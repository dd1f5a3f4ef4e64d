// eb_engine.h -- host side of the batched engine: planning, device orchestration and
// materialisation of EdlibAlignResult.  It restates the reference DRIVER (edlibAlign,
// ref edlib.cpp:146-301) as a batch pipeline; every DP cell is computed by the kernels in
// eb_core.h through a Backend.  The only Backend in the product library is the CUDA one
// (eb_kernels.cu); there is no CPU compute path.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/edlib.h"
#include "../../include/edlib_b200.h"
#include "eb_common.h"

namespace eb {

// Device services + kernel launches.  All pointers handed to launch_* are device pointers.
struct Backend {
    virtual ~Backend() {}
    virtual void* alloc(size_t bytes) = 0;  // >= 256-byte aligned; throws on failure
    virtual void free(void* p) = 0;
    virtual void* alloc_host(size_t bytes) = 0;  // staging memory (pinned on CUDA)
    virtual void free_host(void* p) = 0;
    // Is [p, p + bytes) page-locked host memory the device can read directly (the caller allocated it pinned)?  Then
    // uploads go straight from the caller's buffer, without the staging copy.
    virtual bool host_pinned(const void* /*p*/, size_t /*bytes*/) { return false; }
    virtual void h2d(void* dst, const void* src, size_t bytes) = 0;
    virtual void d2h(void* dst, const void* src, size_t bytes) = 0;  // synchronising
    virtual void zero(void* dst, size_t bytes) = 0;
    virtual void d2d(void* dst, const void* src, size_t bytes) = 0;  // device to device, on the compute stream
    virtual void fill(void* dst, int byteValue, size_t bytes) = 0;
    virtual void sync() = 0;
    // Streamed batches use two more streams beside the compute stream: uploads and result downloads.  A mark is
    // an event recorded on a stream (callable from any host thread); another stream or the host can wait for it.
    // The defaults describe a backend where everything is synchronous.
    enum { STREAM_COMPUTE = 0, STREAM_COPY = 1, STREAM_RESULTS = 2 };
    virtual void h2d_copy(void* dst, const void* src, size_t bytes) { h2d(dst, src, bytes); }  // on the copy stream
    virtual void d2h_async(int /*stream*/, void* dst, const void* src, size_t bytes) { d2h(dst, src, bytes); }
    virtual uint64_t mark(int /*stream*/) { return 1; }
    virtual void wait(int /*stream*/, uint64_t /*mark*/) {}
    virtual void host_wait(uint64_t /*mark*/) {}
    virtual void release_marks() {}
    virtual void sync_all() { sync(); }
    // Makes the calling host thread use this backend's device (CUDA keeps the current device per thread):
    // called on entry of every API call and by pool workers before they issue copies.
    virtual void bind_thread() {}
    // NUMA node the device hangs off (-1: unknown / not applicable)
    virtual int numa_node() { return -1; }
    virtual int sm_count() = 0;
    // Launch shape of the lane-per-alignment kernel for a word class / alphabet size / number of reads
    // (few reads get small CTAs): threads per CTA and how many CTAs are resident on the whole device at
    // once (for wave-aware chunking).  residentCtas == 0: the alphabet is too large for this kernel.
    virtual void k1_shape(int nw32, int ncodes, int numReads, int* blockThreads, int* residentCtas) = 0;
    virtual void launch_mask(const MaskParams& p) = 0;
    virtual void launch_alpha_len(const uint32_t* masks, const int* qset, const int* tset, int numPairs, int* out) = 0;
    virtual void launch_encode(const EncodeParams& p) = 0;
    virtual void launch_k1(const K1Params& p, int nw32) = 0;
    // The same sweep for a HANDFUL of reads: one warp per (read, 32 chunks), lanes = chunks of that read, one profile per warp.
    virtual void launch_k1t(const K1Params& p, int nw32) = 0;
    virtual void launch_k1w(const K1WParams& p, int nw32) = 0;
    // lane-per-alignment sweeps with per-job targets; one launch = one class (mode / reversed / storing)
    virtual void launch_lane(const LParams& p, int nw32, int mode, bool reversed, bool store) = 0;
    virtual void launch_peq(const PeqParams& p) = 0;
    virtual void launch_w(const WParams& p, int R) = 0;
    // k-banded NW sweeps of long queries, one alignment per thread over a sliding window of 4*NB words
    // (eb_core.h: band_job).  band_max_blocks: the largest NB the backend runs for this alphabet size (0: none).
    virtual int band_max_blocks(int ncodes) = 0;
    virtual void launch_band(const WParams& p, int NB, int ncodes) = 0;
    virtual void launch_traceback(const TbParams& p) = 0;
    // one stage of the device-driven start-location / path pipeline of short queries (eb_common.h: ResParams)
    virtual void launch_res(const ResParams& p) = 0;
    virtual void launch_split(const SplitParams& p) = 0;
    // seed stage of the candidate filter: index build (count / scan / fill), per-read planning, window reduction
    virtual void launch_seed_count(const SeedIndexParams& p) = 0;
    virtual void launch_scan(int* data, int count) = 0;  // in place: exclusive prefix sums; data[count] = total
    virtual void launch_seed_fill(const SeedIndexParams& p) = 0;
    virtual void launch_seed_plan(const SeedPlanParams& p) = 0;
    virtual void launch_win_reduce(const WinReduceParams& p) = 0;
    // device-side assembly of distances / end locations of a slice (count -> launch_scan of cnt32 -> fill)
    virtual void launch_fin_count(const FinParams& p) = 0;
    virtual void launch_fin_fill(const FinParams& p) = 0;
    virtual void launch_qalpha(const QAlphaParams& p) = 0;
    // hits (eb_common.h: HitParams): count or fill pass over window jobs / (chunk, read) jobs of a whole-target sweep,
    // and the per-read totals / placement between the two passes.  A backend without these kernels refuses the call.
    virtual void launch_k1w_hits(const K1WParams&, const HitParams&, int /*nw32*/) { no_kernel("k1w_hits"); }
    virtual void launch_k1_hits(const K1Params&, const HitParams&, int /*nw32*/) { no_kernel("k1_hits"); }
    // count or fill pass of the per-pair route (edlibB200FindPairHits): (pair, chunk) jobs over each pair's own target
    virtual void launch_lane_hits(const LaneHitParams&, const HitParams&, int /*nw32*/) { no_kernel("lane_hits"); }
    virtual void launch_hits_total(const HitPlaceParams&) { no_kernel("hits_total"); }
    virtual void launch_hits_place(const HitPlaceParams&) { no_kernel("hits_place"); }
    // start locations / edit scripts of stored hits (eb_common.h: HitResParams)
    virtual void launch_hit_res(const HitResParams&) { no_kernel("hit_res"); }
    // records of a multi-record target (eb_common.h: RecordParams), and the seed index of such a target, whose keys
    // read the separator code as 0 (launch_seed_count / launch_seed_fill otherwise)
    virtual void launch_record(const RecordParams&) { no_kernel("record"); }
    virtual void launch_seed_count_records(const SeedIndexParams&) { no_kernel("seed_count_records"); }
    virtual void launch_seed_fill_records(const SeedIndexParams&) { no_kernel("seed_fill_records"); }
    [[noreturn]] static void no_kernel(const char* name) {
        throw std::runtime_error(std::string(name) + ": no such kernel on this backend");
    }
    // timing of the launches issued since the last reset (device time, ms) and their count
    virtual void reset_timing() = 0;
    virtual double kernel_ms(const char* nameOrNull) = 0;
    virtual int launches() = 0;
    virtual std::string kernel_report() = 0;  // "name:ms:launches;..." of the launches since the last reset
};

struct BatchInput {
    const char* const* queries;
    const int* queryLengths;
    const char* const* targets;
    const int* targetLengths;
    int numPairs;
    EdlibAlignConfig config;
    bool strands = false;  // align every query and its reverse complement, report the better strand (Prepared::strands)
    // A record target (edlibB200FindRecordHits, edlibB200AlignRecords; targets[i] == nullptr, targetLengths[i] == the
    // laid-out length): the records in order, each but the last followed by recordGap separator columns.  numRecords
    // == 0: plain targets.
    const char* const* records = nullptr;
    const int* recordLengths = nullptr;
    int numRecords = 0;
    int recordGap = 0;
    // edlibB200AlignRecords: each pair's result is that of its best record (Pass::pick_records), whose index
    // Engine::records_of reports
    bool bestRecord = false;
};

struct EngineTunables {
    int k1MinGroup = 32;          // pairs sharing one target before the lane-per-alignment kernel is used
    int k1MinChunk = 1024;        // smallest target chunk (columns) when one HW sweep is split
    int ovfCap = 1 << 20;         // overflow entries per launch before the exact-size retry
    size_t sliceBytes = 1ull << 30;  // device memory budget of one slice of W jobs
    size_t pathSliceBytes = 8ull << 30;  // ... of one slice of device-driven paths of short queries (stored matrices)
    size_t packParallelBytes = 32u << 20;  // batches above this are packed and uploaded by several host threads
    // Candidate filter for HW sweeps of reads over a shared target, three stages (0 disables one):
    // exact seeds looked up in a hash index of the target (pigeonhole: t+1 disjoint seeds for threshold
    // t); then, for the reads still undecided, a
    // 32-row prefix sweep finds the target ranges where the prefix matches within filterK1, a 64-row
    // one (for the reads the first stage cannot decide) within filterK0; only windows around those
    // ranges are swept with the whole read; reads no stage decides take the plain full sweep.
    int deviceStage = 1;          // first seed level driven by the device (0: every stage host-driven)
    int devSliceReads = 1 << 20;  // reads per slice of the device-driven level (streamed batches: at least four slices)
    int streamSlices = 8;         // slices of a big streamed batch (the result structs of the last slice are the tail of the call)
    int streamMinPairs = 32768;   // smallest one-target HW batch that edlibAlignBatch streams (upload under compute)
    int longHwMinTarget = 65536;  // HW, query > 256 rows: shortest target worth seeds / chunking (and >= 8 query lengths)
    int longSeedMaxK = 1024;      // ... largest seed threshold tried (thresholds double from 64, capped by the seeds that fit the query)
    int windowCheckAfter = 48;    // banded window sweeps: see K1WParams::checkAfter (-1 disables the early exit)
    int filterSeedK = 20;         // seed stage: largest threshold (needs (t+1) seeds inside the read); 0 disables
    int filterSeedBucket = 128;   // seed stage: longest index range looked at, level 0: twice this; x8 per level (longer: repeat, read passed on)
    int filterSeedLevels = 4;     // seed stage: levels tried (seed length L, L-2, L-4, L-5 for DNA; at most SEED_LEVELS)
    int tinySweepReads = 8;       // plain sweeps of at most this many reads: one warp per (read, 32 chunks) instead of one lane
                                  // per read (k1t_kernel; 0: always the tile kernel)
    int filterMinLevelReads = 64; // seed levels 2 and later: fewest undecided reads worth the level (else: plain sweep)
    int filterSeedSlack = 4;      // seed stage: seed length L is the shortest with sigma^L >= slack * target length
    int filterK1 = 8;
    int filterK0 = 16;
    int filterMinLen = 96;        // shortest query worth the 64-row stage (scaled by P/64 for the other)
    int filterSpread = 1024;      // widest group of candidate ranges verified as one window
    int filterMaxWindows = 32;    // windows per read and stage before the next stage takes the read
    int filterMinTarget = 65536;  // shortest target worth filtering
    size_t directMinBytes = 1u << 20;  // ... grouped batches: from this many query bytes on
    int directUpload = 1;         // queries that are contiguous in PINNED caller memory are uploaded from there (no staging copy)
    int collapseEqualities = 1;   // transitive additional equalities: one code per group of equal bytes, no equality table
    int bandKernel = 1;           // k-banded NW sweeps of long queries on the thread-per-alignment band kernel (0: warp kernel)
    int filterSkipRepeats = 1;    // reads the last seed level found too repetitive skip the prefix stages (plain sweep)
    int hitRunReads = 1 << 18;    // hits: reads per launch group (bounds the per-job arrays of the whole-target and per-pair sweeps)
    EngineTunables();             // reads EDLIB_B200_* environment overrides (used by tests)
};

struct EngineStats {
    double kernelMs = 0;   // device time of all launches of the last compute()
    double k1Ms = 0;       // ... of the K1 launches alone
    int launches = 0;
    long long h2dBytes = 0, d2hBytes = 0;
    long long k1Cells = 0;  // nominal cells (sum m*n) handled by K1
    long long wCells = 0;   // nominal cells of the distance pass handled by W
    long long filterDecided = 0, filterFallback = 0;
    long long filterWindows = 0;  // window sweeps planned by the candidate filter
    std::string kernelReport;  // per-kernel device time of the last compute(): "name:ms:launches;..."
};

// Host vectors of a compute pass, kept between passes so that their pages stay mapped.
struct EngineScratch {
    std::vector<int> best, cnt, posLen, posPool;
    std::vector<long long> posStart;
    int seedWindowsPerRead[SEED_LEVELS] = {0, 0, 0, 0};  // seed stages: windows per read the previous pass produced
    std::vector<int> targetTable;  // prepare(): open-addressing table of the distinct targets
};

class Prepared;  // a batch whose inputs are resident on the device
struct TargetHandle;  // a target kept resident: encoded bytes, presence set, code map, seed index (eb_engine_internal.h)

class Engine {
public:
    explicit Engine(Backend* be);
    ~Engine();
    // One-shot: prepare + compute + materialise (and, for a strand batch, the chosen strand per read into `strands`; for
    // a best-record batch, the record of each result into `records`).  Returns EDLIB_STATUS_OK / EDLIB_STATUS_ERROR.
    int align_batch(const BatchInput& in, EdlibAlignResult* results, unsigned char* strands = nullptr, int* records = nullptr);
    void strands_of(const Prepared* p, unsigned char* strands) const;  // a computed strand batch: 1 where the reverse strand won
    void records_of(const Prepared* p, int* records) const;  // a computed best-record batch: the record of each result

    // Staged form (bench "inputs resident in HBM" measurement, multi-GPU shards):
    Prepared* prepare(const BatchInput& in);                 // upload, alphabet, encode
    void compute(Prepared* p);                               // every kernel; records come back to the host
    // malloc the per-pair arrays, of every result or of the `list`ed ones
    void materialize(Prepared* p, EdlibAlignResult* results, const std::vector<int>* list = nullptr);
    void release(Prepared* p);
    void classify(Prepared* p);                              // pairs -> (target, word class) groups (host only)
    // One-shot streamed path for large HW batches of short reads over one shared target (eb_engine.cpp): returns
    // false when the batch is not of that shape (nothing done), throws on failure.
    bool align_streamed(const BatchInput& in, EdlibAlignResult* results);
    // edlibB200FindHits / edlibB200FindHitAlignments: every end column within config.k of every query over the one
    // shared target (edlibB200FindPairHits: over the pair's own target; in.strands: of its reverse complement too), at
    // most maxHits stored per query; config.task LOC /
    // PATH adds the start location / edit script of every stored hit.  `out` is filled with malloc'd arrays; on
    // failure nothing stays allocated.  Returns EDLIB_STATUS_OK / EDLIB_STATUS_ERROR.  A record target
    // (in.numRecords > 0, edlibB200FindRecordHits): columns and starts count from the start of each hit's record, and
    // *records receives the record of every stored hit (malloc'd).
    int find_hits(const BatchInput& in, long long maxHits, EdlibB200HitAlignments* out, int** records = nullptr);

    void finish_stats();  // fills the device-time fields of `stats` for the last pass (on demand)

    // Targets kept resident for the streamed read-set path (include/edlib_b200.h: edlibB200TargetPrepare).
    TargetHandle* target_prepare(const char* target, int n);
    void target_free(TargetHandle* h);

    EngineTunables tun;
    EngineStats stats;
    EngineScratch scratch;
    std::string lastError;

private:
    Backend* be_;
    Prepared* spare_ = nullptr;  // released batch object whose host vectors the next prepare() reuses
    std::vector<TargetHandle*> targets_;
    TargetHandle* find_target(const char* ptr, int n) const;
    Prepared* take_prepared(const BatchInput& in);  // a batch object reset for `in` (prepare, align_streamed)
    void quiesce();  // error paths: wait for the device, release the marks; never throws
    bool statsPending_ = false;
};

}  // namespace eb
