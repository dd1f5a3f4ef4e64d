// eb_common.h -- types shared by the host engine and the kernels.
//
// Bit layout used by every kernel (differs from the reference on purpose):
//   * bit-vectors are arrays of 32-bit words; query row r lives at global bit  g = r + off,
//     off = 32*nWords - m, i.e. the query is pushed DOWN so that its last row m-1 always sits
//     at bit 31 of the last word.  The reference pads at the bottom with W wildcard rows and
//     reads scores W columns late (ref edlib.cpp:188, 374, 670, 681-693); top padding needs no
//     position shift and lets every kernel read D[m-1][c] from a fixed bit.
//   * padding bits (g < off): vertical deltas 0 (Pv = Mv = 0); Eq = 1 in HW mode (wildcard
//     rows keep D == 0, so the first real row sees the HW boundary D[-1][c] = 0) and Eq = 0 in
//     SHW/NW mode (then Ph is 1 on every padding bit and, with the "| 1" shifted in at bit 0,
//     the first real row sees the NW/SHW boundary delta +1; Pv/Mv stay 0 on the padding bits).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define EB_HD __host__ __device__ __forceinline__
#define EB_D __device__ __forceinline__
#else
#define EB_HD inline
#define EB_D inline
#endif

namespace eb {

struct U2 { uint32_t x, y; };  // {Pv, Ph} of one (column, word) in the stored matrix

constexpr int KPOS = 4;  // end positions kept inline per record; the rest go to the overflow list

// Per-sweep result record (device -> host).  best > bound means "nothing within the bound".
struct Rec {
    int best;       // min over tracked columns of D[m-1][c] (or the sentinel it started from)
    int cnt;        // number of tracked columns attaining `best`
    int last;       // last such column
    int rsv;
    int pos[KPOS];  // first KPOS such columns, ascending
};

// Record of one window sweep (K1W): same header as Rec, more inline positions -- windows are short and the
// reads that tie on many end columns would otherwise need a whole-target sweep.
constexpr int KPOSW = 12;
struct WinRec {
    int best, cnt, last, rsv;
    int pos[KPOSW];
};

// Overflow entry for columns beyond KPOS.  The list is only armed (ovfCap > 0) in the second
// pass over the few sweeps that have more than KPOS end positions; that pass starts from the
// known minimum, so every entry is a final position and the capacity is known exactly.
struct Ovf {
    int rec;    // index of the Rec it belongs to
    int score;
    int pos;
};

// Candidate-filter range list (K1 rangeMode, eb_core.h: k1_range_flush)
#define K1_RANGE_GAP 256    // a candidate this far after the previous one opens a new range
#define K1_RANGE_SPAN 1024  // ... or this far after the first one of the open range
#define K1_RANGE_MAX 16     // ranges per (chunk, read) before the read is marked as saturated

enum Mode : int { MODE_NW = 0, MODE_SHW = 1, MODE_HW = 2 };

// ---------------------------------------------------------------------------------------------
// K1: lane-per-alignment sweep of many short queries over ONE shared target.
// ---------------------------------------------------------------------------------------------
struct K1Params {
    const uint8_t* tcodes;   // encoded target (dense codes), 16-byte aligned, padded to 16
    int n;                   // target length
    const uint8_t* qcodes;   // all encoded queries
    const uint64_t* qoff;    // [pair] offset into qcodes
    const int* qlen;         // [pair]
    const int* readList;     // [numReads] pair indices handled by this launch
    const int* kInit;        // [numReads] initial `best` sentinel (bound + 1)
    int numReads;
    int mode;                // Mode
    int ncodes;              // alphabet size of the batch
    const uint8_t* eqtab;    // ncodes x ncodes match table, or nullptr for identity
    int chunks;              // target chunks (HW only; 1 otherwise)
    int chunkLen;            // multiple of 16
    int halo;                // columns swept before a chunk without tracking (>= 2*max m)
    Rec* recs;               // [chunks][numReads]  (unused in rangeMode)
    Ovf* ovf;
    int* ovfCount;
    int ovfCap;
    int prefixLen;           // > 0: sweep only the first prefixLen rows of every query (candidate filter)
    int rangeMode;           // 1: instead of the running minimum, append the ranges of columns whose prefix score
                             //    is <= kInit to ovf[] as {rec = read slot, score = first, pos = last}
};

// K1W: lane-per-alignment HW sweep of each query over ITS OWN window of the shared target (the
// verification step of the candidate filter).  Columns before trackFrom are halo.
struct K1WParams {
    const uint8_t* tcodes;   // encoded target
    const uint8_t* qcodes;
    const uint64_t* qoff;    // [pair]
    const int* qlen;         // [pair]
    const int* readList;     // [numReads] pair indices
    const int* kInit;        // [numReads] initial best sentinel (threshold + 1)
    const int* winStart;     // [numReads] first target column swept
    const int* winLen;       // [numReads] columns swept
    const int* trackFrom;    // [numReads] first column (relative to winStart) whose score may be recorded
    int numReads;
    const int* countPtr;     // device-planned jobs: the number of jobs is min(*countPtr, numReads); or nullptr
    int checkAfter;          // banded sweeps: columns past the last possible start after which a hopeless window is left (-1: never)
    int ncodes;
    const uint8_t* eqtab;
    WinRec* recs;            // [numReads]; positions are absolute target columns
    // end columns beyond the KPOSW inline ones: appended (window slot, score, column) in sweep order; entries whose
    // score is not the window's final minimum are stale.  ovfCap == 0: not collected.
    Ovf* ovf;
    int* ovfCount;           // zeroed by the host; may run past ovfCap (then the list is incomplete)
    int ovfCap;
};

// L: lane-per-alignment sweep of a short query over its own target (any mode).
struct LJob {
    uint64_t qOff;     // into qcodes (read backwards from qOff+m-1 when the launch is reversed)
    uint64_t tOff;     // into tcodes: first symbol read (reversed launches walk down from it)
    uint64_t matOff;   // into mat (U2 entries, [column][NW]) for storing launches
    int m, n;
    int kInit;         // HW/SHW: initial best sentinel
    int trackFrom;     // HW: first column whose score may be recorded
};
struct LParams {
    const LJob* jobs;
    int numJobs;
    const uint8_t* qcodes;
    const uint8_t* tcodes;
    int ncodes;
    const uint8_t* eqtab;
    Rec* recs;         // [numJobs]
    U2* mat;
    int matStep;       // storing launches: entries between consecutive (column, word) cells of one job; 0 / 1: the job's
                       // matrix is contiguous, 32: the matrices of 32 consecutive jobs are interleaved entry by entry, so
                       // that a warp's stores of one (column, word) form one 256-byte run
};

// ---------------------------------------------------------------------------------------------
// W: warp-per-alignment sweep (any query length, any alphabet, per-job target window).
// ---------------------------------------------------------------------------------------------
enum WFlags : int {
    WF_QREV = 1,      // read the query backwards
    WF_TREV = 2,      // read the target backwards (tBase is then the FIRST symbol read)
    WF_SLIDE = 4,     // NW only: one 1024*R-row window sliding down the k-band
    WF_STORE = 8,     // store Pv/Ph of every column for the traceback kernel
    WF_STOPCOL = 16,  // NW: dump the score column at stopCol and stop (Hirschberg halves)
};

struct WJob {
    uint64_t qOff;     // into qcodes; with WF_QREV the query is q[qOff+m-1 .. qOff] reversed
    uint64_t tOff;     // into tcodes; first symbol read (see WF_TREV)
    uint64_t peqOff;   // into peq (words): ncodes * nWp words, row-major [code][word]
    uint64_t auxOff;   // into mat (U2 entries) when WF_STORE; into colOut (ints) when WF_STOPCOL
    uint64_t hbufOff;  // into hbuf (bytes): 2*n bytes when the job needs more than one strip
    int m, n;
    int nWp;           // padded word count: multiple of R, >= ceil(m/32)
    int mode;          // Mode
    int flags;         // WFlags
    int kInit;         // HW/SHW: initial best sentinel; NW: unused
    int dhi;           // WF_SLIDE: largest diagonal c - r inside the band
    int stopCol;       // WF_STOPCOL: column whose scores are dumped
    int rec;           // index of the output Rec
    int trackFrom;     // HW/SHW: first column whose score may be recorded (earlier ones are halo)
};

struct WParams {
    const WJob* jobs;
    int numJobs;
    const uint8_t* qcodes;
    const uint8_t* tcodes;
    const uint32_t* peq;
    uint8_t* hbuf;
    U2* mat;
    int* colOut;
    Rec* recs;
    Ovf* ovf;
    int* ovfCount;
    int ovfCap;
};

// Query-profile build for W jobs (one Peq per job).
struct PeqParams {
    const WJob* jobs;
    int numJobs;
    const uint8_t* qcodes;
    uint32_t* peq;
    int ncodes;
    const uint8_t* eqtab;  // or nullptr
};

// Traceback over a stored matrix (one thread per job).
struct TbJob {
    uint64_t matOff;   // U2 entries, [column][nWp]
    uint64_t qOff;     // query codes (used when peqOff == ~0)
    uint64_t peqOff;   // Peq of the (forward) query, or ~0: compare symbols directly
    uint64_t tOff;     // target window start in tcodes
    uint64_t outOff;   // into ops: m+n bytes reserved; ops are written back-to-front
    int m, n, nWp;
    int rsv;
};
struct TbParams {
    const TbJob* jobs;
    int numJobs;
    const U2* mat;
    const uint32_t* peq;
    const uint8_t* tcodes;
    const uint8_t* qcodes;
    const uint8_t* eqtab;
    int ncodes;
    uint8_t* ops;
    int* opsStart;     // [job] index of the first op inside the job's reserved area
    int* opsLen;       // [job]
    int matStep;       // as LParams::matStep
};

// Hirschberg split search (ref cpp:1321-1353) over the two stop columns of a node, on the device.
struct SplitNode {
    uint64_t colF;     // into cols: D_fwd[r][leftW-1], r = 0..m-1 (0x3f3f3f3f where outside the band)
    uint64_t colR;     // into cols: D_rev[r'][rightW-1]
    int m, leftW, rightW, best;
};
struct SplitOut {
    int h;             // rows of the query that go with the left half (-1: no split found)
    int left, right;   // scores of the two halves
    int rsv;
};
struct SplitParams {
    const SplitNode* nodes;
    int numNodes;
    const int* cols;
    SplitOut* out;
};

// Seed index of a target (candidate filter, seed stages): ONE radix table serves every seed level.  The key of
// target position i is the base-sigma number of the Lidx codes starting there (codes past the end count as 0),
// so the table is a CSR from key to the positions holding that Lidx-mer, and all positions whose Lidx-mer
// starts with a SHORTER word form one contiguous key range: a seed of length Ls <= Lidx is looked up as the
// range [key(seed) * sigma^(Lidx-Ls), (key(seed)+1) * sigma^(Lidx-Ls)) with no verification at all, a longer
// seed by its first Lidx codes plus a comparison of the remaining ones.  Build: count (seed_count_item),
// exclusive scan of the counts (Backend::launch_scan), fill (seed_fill_item).
struct SeedIndexParams {
    const uint8_t* tcodes;   // encoded target
    int n;
    int Lidx;                // symbols per key
    int sigma;               // radix (>= 2, >= number of target codes)
    int numPos;              // positions indexed: 0 .. numPos-1 (= n - Lmin + 1, Lmin the shortest seed used)
    int numKeys;             // sigma^Lidx
    int* bucketStart;        // [numKeys + 1] counts, then their exclusive prefix sums (last = numPos)
    int* cursor;             // [numKeys] fill cursors, zeroed by the host
    int* positions;          // [numPos]
};
// candidate end columns per read before the read is passed on as saturated, per seed level (shorter seeds
// have more chance occurrences); the planning kernel is instantiated per capacity
#define SEED_LEVELS 4
#define SEED_CAND_0 256
#define SEED_CAND_1 256
#define SEED_CAND_2 4096
enum SeedState : int { SEED_NONE = 0, SEED_WINDOWS = 1, SEED_SATURATED = 2, SEED_LONG_LIST = 3 };
struct SeedPlan {
    int first, count;        // the read's windows in the job arrays
    int state;               // SeedState
    int thr;                 // threshold t the windows were planned for (-1: the read was left out of the stage)
};
// Threshold of a read of m rows at a seed level with seeds of Ls symbols: the largest t with t+1 disjoint
// seeds inside the read, capped by the caller's bound and the stage's cap; -1 if the stage cannot help.
EB_HD int seed_threshold(int m, int kBound, int Ls, int seedK, int excl) {
    const int bound = (kBound < 0 || kBound > m) ? m : kBound;  // distances never exceed m in HW (ref cpp:566-568)
    int t = m / Ls - 1;
    if (t > seedK) t = seedK;
    if (t > bound) t = bound;
    return (m >= 2 * Ls && t > excl) ? t : -1;
}
// Cross-strand rule of one read of a strand batch (DESIGN.md section 3).  Per strand s (0: forward, 1: reverse
// complement): done[s] -- its outcome is final, d[s] then being its distance or 0x7fffffff (none within its bound); or
// pending, with no distance <= excl[s] (-1: nothing known) and bound[s] the largest distance that still counts.  Ties
// go to the forward strand, so the reverse strand only counts below d[0] and the forward strand up to d[1].  Tightens
// the bound of a pending strand and returns the strand that has lost (its outcome becomes "no alignment"), or -1.
EB_HD int strand_rule(const bool (&done)[2], const int (&d)[2], const int (&excl)[2], int (&bound)[2]) {
    if (done[0] && !done[1] && d[0] != 0x7fffffff) {
        if (d[0] - 1 < bound[1]) bound[1] = d[0] - 1;
        if (excl[1] >= bound[1]) return 1;
    }
    if (done[1] && !done[0] && d[1] != 0x7fffffff) {
        if (d[1] < bound[0]) bound[0] = d[1];
        if (excl[0] >= bound[0]) return 0;
    }
    return -1;
}
// Per read: t+1 disjoint seeds are looked up; every exact occurrence yields the expected end column
// of the alignment it belongs to; neighbouring ones share a window (eb_core.h: seed_plan_read).
struct SeedPlanParams {
    const uint8_t* tcodes;
    int n;
    const uint8_t* qcodes;
    const uint64_t* qoff;
    const int* qlen;
    const int* readList;     // [numReads] pair indices, or nullptr: pair = firstPair + slot
    int firstPair;
    const int* thr;          // [numReads] threshold t per read (t < 0: read skipped), or nullptr: seed_threshold(m, kBound, Ls, seedK, -1)
    int kBound, seedK;
    int numReads;
    int maxLen;              // no read of the launch is longer (0: unknown); bounds t and so the lanes a read needs
    int Ls;                  // seed length of this level
    int Lidx, sigma, numKeys;
    const int* bucketStart;
    const int* positions;
    int maxBucket;           // a seed with more index entries than this saturates the read (repeats)
    int level;               // seed level (selects the candidate capacity)
    int spread;              // widest group of candidates verified as one window
    // outputs: K1W jobs (K1WParams arrays) and the per-read plan
    int* winPair;
    int* winK;
    int* winStart;
    int* winLen;
    int* winTf;
    int winCap;
    int* winCount;           // zeroed by the host; may exceed winCap (reads whose windows do not fit are saturated)
    SeedPlan* plan;          // [numReads]
};
// Leftover entry of the device-driven first seed level: a read this level could not decide.
struct Leftover {
    int pair;
    int excl;                // no distance <= excl exists (-1: nothing known); -2: long end-location list (plain sweep)
    int bound;               // largest distance that still counts (strand batches: capped by the other strand's distance)
};
enum RecState : int { REC_DONE = 100, REC_PENDING = 101 };
// Per read: minimum over its windows -> out[slot].
//   host-driven stages (leftover == nullptr): rsv = SeedState (SEED_WINDOWS: decided with best/cnt/pos filled,
//   SEED_NONE: no distance <= t exists); the host works out what happens to the read.
//   device-driven first level (leftover != nullptr): rsv = REC_DONE (best/cnt/pos final; best = 0x7fffffff with
//   cnt = 0 when no alignment within the caller's bound exists) or REC_PENDING, in which case the read is
//   appended to the leftover list for the host-driven stages.  With `strands` set nothing is appended: a pending
//   read keeps its excl (Leftover::excl) in out.last, and fin_count_item applies the cross-strand rule.
struct WinReduceParams {
    const SeedPlan* plan;
    const WinRec* winRecs;
    int numReads;
    Rec* out;                // cnt > KPOS: positions KPOS.. are extra[out.last ...]
    int* extra;
    int* extraCount;         // zeroed by the host
    int extraCap;
    // overflow list of the window sweeps (K1WParams::ovf): windows with more than KPOSW end columns
    const Ovf* ovf;
    const int* ovfCount;
    int ovfCap;
    // device-driven mode
    Leftover* leftover;
    int* leftoverCount;
    const int* readList;     // or nullptr: pair = firstPair + slot
    int firstPair;
    const int* qlen;
    int kBound;
    int strands;
};
// Device-side assembly of editDistance / endLocations of a slice of reads decided on the device (the -1 rule of
// ref cpp:670, 681-693 included): fin_count_item -> exclusive scan of cnt32 -> fin_fill_item.
struct FinParams {
    const Rec* recs;         // [numReads] by slot
    const int* extra;
    const int* readList;     // or nullptr: pair = firstPair + slot
    int firstPair;
    int numReads;
    const int* qlen;
    int kBound;
    int* ed;                 // [pair]: distance, -1 (none within the bound) or -2 (pending: host-driven stages)
    int* endCount;           // [pair]
    long long* endStart;     // [pair] into the batch's end-location pool
    int* cnt32;              // [numReads + 1] counts, then their exclusive prefix sums (last = total)
    int* pool;               // the slice's region of the end-location pool
    long long poolBase;      // offset of that region in the batch pool
    int poolCap;
    int* header;             // [4]: total end locations, reads pending, pool overflow flag, windows planned
    const int* winCount;     // copied into header[3]
    // strand batches: slots 2j / 2j+1 are the two strands of a read; the cross-strand rule (strand_rule) settles the
    // loser as "no alignment", and the strands still pending are appended to the leftover list with their bounds
    int strands;
    Leftover* leftover;
    int* leftoverCount;
};

// ---------------------------------------------------------------------------------------------
// Hits: every end column c of a read whose last-row score D(c) is <= k (edlibB200FindHits).  The jobs are the seed
// windows of a K1W launch (kInit = k + 1, as planned) or the (chunk, read) items of a K1 launch over the whole target
// (kInit = k; a chunk reports the columns it owns).  Each launch runs twice over the same jobs: the count pass writes
// the hits of every job, the fill pass re-sweeps the jobs with room > 0 and stores their first `room` hits in column
// order at at[job].
// ---------------------------------------------------------------------------------------------
struct HitParams {
    int* count;              // count pass (at == nullptr): [job] hits of the job
    const long long* at;     // fill pass: [job] first slot of the job's stored hits in cols / scores
    const int* room;         // fill pass: [job] hits of the job that are stored (0: the job is skipped)
    int* cols;               // fill pass: end columns
    int* scores;             // fill pass: D(column)
    const uint8_t* sepCodes; // record target (edlibB200FindRecordHits): its codes; a column holding code sep is a
    int sep;                 // separator and never a hit (eb_core.h: RecordHitSink).  nullptr: one plain target
};
// Per read of a hits launch: the jobs of read `slot` are plan[slot].first .. + count (windows, in column order), or
// slot + c * numReads for c < chunks (chunks, in column order).
struct HitPlaceParams {
    const SeedPlan* plan;    // windows, or nullptr: chunks
    int chunks;
    int numReads;
    const int* readList;     // [numReads] pair of each slot
    const int* count;        // [job] hits of the job (count pass)
    long long* pairCount;    // hits_total: [pair] hits of the read (reads without windows: 0)
    const long long* pairBase;   // hits_place: [pair] first slot of the read's stored hits
    const long long* pairStored; // hits_place: [pair] hits of the read that are stored
    long long* at;           // hits_place: [job] -> HitParams::at
    int* room;               // hits_place: [job] -> HitParams::room
};
// Hits of the per-pair route (edlibB200FindPairHits): one job per (pair, chunk) of the pair's OWN target, swept as a
// K1 chunk (restart at hs, columns [cs, ce) owned and reported; eb_core.h: lane_hits_job).  The jobs of a pair are
// consecutive and in column order; HitPlaceParams::plan gives each slot its range (state SEED_WINDOWS).
struct LaneHitJob {
    uint64_t qOff;     // into qcodes
    uint64_t tOff;     // into tcodes: the symbol of target column hs
    int m;
    int hs, cs, ce;    // target columns: first swept, first owned, one past the last owned
};
struct LaneHitParams {
    const LaneHitJob* jobs;
    int numJobs;
    int k;                   // fixed threshold
    const uint8_t* qcodes;
    const uint8_t* tcodes;
    int ncodes;
    const uint8_t* eqtab;
};
// Start locations and edit scripts of stored hits (edlibB200FindHitAlignments), one slice of stored hits at a time:
// the lane kernel runs one reversed SHW sweep (start) and one matrix-storing NW sweep + traceback (script) per hit of
// word class nw; `stage` selects the per-item function of hit_res_kernel.  Hit h of the slice is stored hit
// firstHit + h; its pair is the last pair whose first stored slot is <= firstHit + h.
enum HitResStage : int {
    HR_FLAG = 0,        // item = hit h: cnt[h] = 1 if its query is of word class nw                                -> scan
    HR_LOC_JOBS = 1,    // item = hit h of the class: LJob j = cnt[h] of the reversed SHW sweep ending at its column
    HR_LOC_APPLY = 2,   // item = job j: starts[h] = column - last column of the sweep's best (ref cpp:260), best == score
    HR_PATH_JOBS = 3,   // item = hit h of the class: LJob (storing NW) + TbJob j = cnt[h] over [starts[h], column]
    HR_PATH_LEN = 4,    // item = job j: len[h] = ops of its edit script, NW score == score                         -> scan
    HR_PATH_COPY = 5,   // item = job j: edit script into the slice's dense pool at len[h]
};
struct HitResParams {
    int stage;
    int nw;                  // word class handled by this launch
    int numItems;            // hits of the slice (HR_FLAG, HR_*_JOBS) or jobs of the class (the others)
    long long firstHit;      // stored slot of hit 0 of the slice
    int numPairs;
    const long long* pairBase;  // [numPairs] first stored slot of each pair (non-decreasing)
    const int* qlen;         // [pair]
    const uint64_t* qoff;    // [pair]
    uint64_t tOff;           // offset of the shared target in the packed buffer
    const uint64_t* tOffPair;  // [pair] offset of the pair's own target (edlibB200FindPairHits), or nullptr: tOff
    const int* cols;         // [stored hit] end column
    const int* scores;       // [stored hit] D(column)
    int* cnt;                // [hits + 1] flags, then their exclusive prefix sums: job of hit h is cnt[h]
    LJob* jobs;
    int* jobHit;             // [job] hit of the job inside the slice
    const Rec* recs;         // [job] outcome of the lane sweeps
    int* starts;             // [hits] start location of each hit
    TbJob* tb;
    uint64_t matStride;      // HR_PATH_JOBS: U2 entries reserved per job
    uint64_t opsStride;      // bytes reserved per job for its traceback
    const uint8_t* ops;      // traceback output (opsStride per job), opsStart / opsLen per job
    const int* opsStart;
    const int* opsLen;
    int* len;                // [hits + 1] script length of each hit, then their exclusive prefix sums
    uint8_t* pool;           // dense scripts of the slice, in hit order
    int* err;                // set to 1 when a sweep disagrees with the score of its hit
    const int* recOff;       // record target: [numRecords + 1] RecordParams::recOff (a start is clipped at the first
    int numRecords;          // column of its hit's record); nullptr: one plain target
};

// Records of a multi-record target (edlibB200FindRecordHits): the records lie in order in one target, record r at
// columns [recOff[r], recOff[r + 1] - gap), each followed by `gap` columns of the separator code sep (recOff[R] is the
// target length + gap).  `stage` selects the per-item function of record_kernel.
enum RecordStage : int {
    REC_SEPARATORS = 0,  // item = target column c: tcodes[c] = sep when c is a separator column
    REC_STARTS = 1,      // item = hit h of a slice: starts[h] -= first column of the record of stored hit firstHit + h
    REC_HITS = 2,        // item = stored hit firstHit + h: records[.] = its record, cols[.] = its column in the record
};
struct RecordParams {
    int stage;
    int numItems;
    const int* recOff;       // [numRecords + 1]
    int numRecords;
    int gap;
    int sep;
    uint8_t* tcodes;         // REC_SEPARATORS: the encoded target
    long long firstHit;      // REC_STARTS / REC_HITS: stored slot of item 0
    int* cols;               // [stored hit] end column in the target (REC_HITS: in its record, afterwards)
    int* starts;             // REC_STARTS: [item] start of the hit in the target -> in its record
    int* records;            // REC_HITS: [stored hit] record
};

// ---------------------------------------------------------------------------------------------
// Start locations and alignment paths of short queries (<= 256 rows) WITHOUT the host in the loop: the jobs of the
// lane kernel (reversed SHW sweeps of ref cpp:253-257; matrix-storing NW sweeps + traceback of ref cpp:276-289,
// 1161-1213) are derived on the device from the per-pair results, and their outcome is written straight into the
// batch's start-location pool / a dense pool of edit scripts.  `stage` selects the per-item function of res_kernel.
// ---------------------------------------------------------------------------------------------
enum ResStage : int {
    RS_LOC_COUNT = 0,    // cnt[pair] = end locations of the pair if it belongs to word class nw (else 0)        -> scan
    RS_LOC_JOBS = 1,     // item = slot job j: LJob of the reversed sweep from end location j of its pair
    RS_LOC_APPLY = 2,    // item = slot job j: startPool[slot] = end - last best column of the sweep (ref cpp:260)
    RS_PATH_FLAG = 3,    // cnt[pair] = 1 if the pair gets a path from this launch (class nw, found, in [firstPair, lastPair)) -> scan
    RS_PATH_JOBS = 4,    // item = pair: LJob (storing) + TbJob of its first (start, end)
    RS_PATH_LEN = 5,     // item = job: len[j] = ops of its edit script                                          -> scan
    RS_PATH_COPY = 6,    // item = job: edit script into the dense pool; alnStart / alnLen of the pair
};
struct ResParams {
    int stage;
    int nw;                  // word class handled by this launch
    int numPairs;            // N
    int numItems;            // items of this stage (pairs, or jobs)
    int firstPair, lastPair; // RS_PATH_*: the pair range of this slice
    // per-pair inputs
    const int* ed;           // [N] distance or < 0
    const int* endCount;     // [N]
    const long long* endStart;  // [N] into endPool / startPool
    const int* endPool;
    const int* qlen;         // [N]
    const uint64_t* qoff;    // [N]
    const uint64_t* tOffPair;  // [N] offset of the pair's target in the packed buffer, or nullptr: tOff0 for every pair
    uint64_t tOff0;
    // scan arrays / job arrays
    int* cnt;                // [numPairs + 1] or [numJobs + 1]: counts, then exclusive prefix sums
    LJob* jobs;
    int* jobPair;            // [job] pair of the job
    long long* jobSlot;      // [job] RS_LOC_*: slot of the job's end location
    const Rec* recs;         // [job] outcome of the lane sweeps
    int* startPool;          // out (RS_LOC_APPLY); in (RS_PATH_JOBS)
    TbJob* tb;
    int maxPathN;            // RS_PATH_*: longest target slice (columns) a path job of this launch may have
    uint64_t matStride;      // U2 entries reserved per path job
    uint64_t opsStride;      // bytes reserved per path job
    const uint8_t* ops;      // traceback output (opsStride per job), opsStart / opsLen per job
    const int* opsStart;
    const int* opsLen;
    uint8_t* alnPool;        // dense pool of this slice
    long long alnBase;       // offset of that pool in the batch's alignment pool
    long long* alnStart;     // [N]
    int* alnLen;             // [N]
    int* err;                // set to 1 when a sweep disagrees with the distance it was started from
};

// Presence / alphabet kernels.
struct MaskItem {
    uint64_t off;            // into raw
    int len;                 // <= 65536 (long sequences are split by the host)
    int dst;                 // which 256-bit set receives the bytes seen
};
struct MaskParams {
    const uint8_t* raw;      // raw bytes as uploaded
    const MaskItem* items;   // explicit items: targets, and the pieces of queries longer than 65536
    int numItems;
    // implicit items 0..numQueries-1 (work item indices numItems..numItems+numQueries-1): query i at
    // qoff[i], qlen[i] bytes, destination set i; queries longer than 65536 are skipped (explicit pieces)
    const uint64_t* qoff;
    const int* qlen;
    int numQueries;
    uint32_t* masks;         // [numSets][8] 256-bit presence sets, zeroed by the host
    int unionSet;            // set that additionally receives every byte seen (or -1)
    // strand batches (rc != nullptr): the reads are pairs 2i, implicit item q is pair 2q; every byte at offset o < rcBytes
    // (the read block) is also written complemented to rc[rcBytes - 1 - o] (the reverse complement of the block, read
    // i + 1 of it being pair 2i+1), and the presence set of those bytes goes to the set after the item's own
    uint8_t* rc;
    uint64_t rcBytes;
};
struct EncodeParams {
    uint8_t* data;           // encoded in place (any alignment)
    uint64_t numBytes;
    const uint8_t* map;      // [256] byte -> code
};
// alphabetLength of a run of queries that all face ONE target (streamed batches): distinct byte values of the
// query united with the target's presence set (ref transformSequences cpp:1437-1461), straight from the raw bytes.
struct QAlphaParams {
    const uint8_t* raw;      // raw bytes as uploaded
    const uint64_t* qoff;    // [pair]
    const int* qlen;         // [pair]
    int firstPair;
    int numQueries;
    const uint32_t* tmask;   // [8] presence set of the target
    int* alphaLen;           // [pair]
};

}  // namespace eb
