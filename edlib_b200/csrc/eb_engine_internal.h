// eb_engine_internal.h -- shared declarations of the host engine's translation units (eb_engine.cpp: batch
// preparation and the compute driver; eb_wrunner.cpp: warp-per-alignment job runner; eb_pass_lane.cpp: the
// lane-per-alignment distance pass with the candidate filter; eb_pass_results.cpp: end/start locations and
// alignment paths).  Not part of the library's interface.
#pragma once
#include "eb_engine.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <exception>
#include <functional>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <chrono>
#include <map>
#include <memory>
#include <stdexcept>
#include <thread>
#include <unordered_map>

namespace eb {


// EDLIB_B200_TRACE=1: wall-clock of the host phases to stderr (diagnostics only).
struct Trace {
    bool on;
    std::chrono::steady_clock::time_point t0;
    Trace() : on(getenv("EDLIB_B200_TRACE") != nullptr), t0(std::chrono::steady_clock::now()) {}
    void mark(const char* what) {
        if (!on) return;
        const auto t1 = std::chrono::steady_clock::now();
        const char* rank = getenv("RANK");
        fprintf(stderr, "[edlib_b200%s%s] %-28s %8.2f ms\n", rank ? " r" : "", rank ? rank : "", what,
                std::chrono::duration<double, std::milli>(t1 - t0).count());
        t0 = t1;
    }
};

// Persistent host worker threads (spawning threads per loop costs more than most of these loops): run(n, fn)
// executes fn(0) .. fn(n-1), the caller taking part, and returns when all are done.  One client at a time
// (the engine runs under the library's lock).  The workers live until the process ends.
class HostPool {
public:
    // CPUs the workers should run on (the NUMA node of the GPU: packing writes pinned memory that the GPU then
    // reads over PCIe, and a remote node halves that).  Set once, before the pool exists (Engine construction);
    // empty: the workers inherit the creating thread's affinity.
    static std::vector<int>& worker_cpus() {
        static std::vector<int> cpus;
        return cpus;
    }
    static HostPool& get() {
        static HostPool* pool = new HostPool();  // never destroyed: workers may still be parked at exit
        return *pool;
    }
    size_t width() const { return workers_ + 1; }
    void run(size_t n, const std::function<void(size_t)>& fn) {
        if (n == 0) return;
        if (n == 1 || workers_ == 0) {
            for (size_t i = 0; i < n; ++i) fn(i);
            return;
        }
        begin(n, fn);
        end(true);
    }
    // Split form of run(): begin() hands fn(0) .. fn(n-1) to the workers and returns at once (fn must stay alive
    // until end()); end() waits for them, the caller taking part in what is still unclaimed if `participate`.
    // Between the two the caller must not use the pool.  With no workers the tasks run inside end().
    void begin(size_t n, const std::function<void(size_t)>& fn) {
        client_.lock();  // one client at a time (several engines share the pool); released by end()
        {
            std::lock_guard<std::mutex> lock(mu_);
            fn_ = &fn;
            total_ = n;
            next_ = 0;
            pending_ = n;
            activeGen_ = ++generation_;
        }
        cv_.notify_all();
    }
    void end(bool participate) {
        if (participate || workers_ == 0) work(activeGen_);
        std::exception_ptr err;
        {
            std::unique_lock<std::mutex> lock(mu_);
            done_.wait(lock, [this]() { return pending_ == 0; });
            fn_ = nullptr;
            err = error_;
            error_ = nullptr;
        }
        client_.unlock();
        if (err) std::rethrow_exception(err);  // the first exception a task threw, on the caller's thread
    }

private:
    // Pool width: EDLIB_B200_HOST_THREADS if set; else min(16, CPUs this process may use / ranks on this node),
    // where the CPUs are bounded by a cgroup quota when there is one (containers often expose every hardware
    // thread but grant far fewer) and the ranks come from torchrun's LOCAL_WORLD_SIZE.
    static size_t pool_width() {
        if (const char* e = getenv("EDLIB_B200_HOST_THREADS")) {
            const int v = atoi(e);
            if (v > 0) return (size_t)std::min(v, 64);
        }
        double cpus = (double)std::max(1u, std::thread::hardware_concurrency());
        if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {  // cgroup v2: "<quota|max> <period>"
            char quota[32];
            double period = 0;
            if (fscanf(f, "%31s %lf", quota, &period) == 2 && strcmp(quota, "max") != 0 && period > 0)
                cpus = std::min(cpus, std::max(1.0, atof(quota) / period));
            fclose(f);
        } else if (FILE* q = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {  // cgroup v1
            double quotaUs = -1, periodUs = 0;
            if (fscanf(q, "%lf", &quotaUs) != 1) quotaUs = -1;
            fclose(q);
            if (FILE* pf = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
                if (fscanf(pf, "%lf", &periodUs) != 1) periodUs = 0;
                fclose(pf);
            }
            if (quotaUs > 0 && periodUs > 0) cpus = std::min(cpus, std::max(1.0, quotaUs / periodUs));
        }
        int ranks = 1;
        if (const char* e = getenv("LOCAL_WORLD_SIZE")) ranks = std::max(1, atoi(e));
        const size_t w = (size_t)(cpus / ranks + 0.5);
        return std::max<size_t>(2, std::min<size_t>(16, w));
    }
    HostPool() {
        workers_ = pool_width() - 1;
        for (size_t i = 0; i < workers_; ++i) std::thread([this]() { loop(); }).detach();
    }
    // Tasks are few and coarse, so they are claimed under the lock; a worker only ever claims tasks of
    // the generation it woke up for.
    void work(unsigned long long gen) {
        for (;;) {
            const std::function<void(size_t)>* fn;
            size_t i;
            {
                std::lock_guard<std::mutex> lock(mu_);
                if (generation_ != gen || next_ >= total_) return;
                i = next_++;
                fn = fn_;
            }
            std::exception_ptr err;
            try {
                (*fn)(i);
            } catch (...) {
                err = std::current_exception();
            }
            std::lock_guard<std::mutex> lock(mu_);
            if (err && !error_) error_ = err;
            if (--pending_ == 0) done_.notify_all();
        }
    }
    void loop() {
        bind_worker();
        unsigned long long seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lock(mu_);
                cv_.wait(lock, [&]() { return generation_ != seen; });
                seen = generation_;
            }
            work(seen);
        }
    }
    static void bind_worker();  // eb_engine.cpp (sched_setaffinity to worker_cpus(), ignored when not permitted)
    size_t workers_ = 0;
    std::mutex client_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    const std::function<void(size_t)>* fn_ = nullptr;
    std::exception_ptr error_;
    size_t total_ = 0, pending_ = 0, next_ = 0;
    unsigned long long generation_ = 0, activeGen_ = 0;
};

// number of parts a loop over n items is cut into (every part gets >= grain items)
inline size_t host_parts(size_t n, size_t grain) {
    return std::max<size_t>(1, std::min<size_t>(HostPool::get().width(), n / std::max<size_t>(grain, 1)));
}

// fn(begin, end) over [0, n) on the host workers (only when every part gets >= grain items).
template <class F>
void parallel_ranges(size_t n, size_t grain, F fn) {
    if (n == 0) return;  // nothing to do (and callers may hold a null data() for an empty vector)
    const size_t nthr = host_parts(n, grain);
    if (nthr <= 1) {
        fn((size_t)0, n);
        return;
    }
    HostPool::get().run(nthr, [&](size_t t) { fn(n * t / nthr, n * (t + 1) / nthr); });
}

// fn(part, begin, end) over the host_parts(n, grain) parts of [0, n) (one empty part when n == 0), on the host workers.
// Returns the number of parts: at most HostPool::get().width(), and the same for the same n and grain.
template <class F>
size_t parallel_parts(size_t n, size_t grain, F fn) {
    const size_t nparts = host_parts(n, grain);
    HostPool::get().run(nparts, [&](size_t t) { fn(t, n * t / nparts, n * (t + 1) / nparts); });
    return nparts;
}

// Whether pred(i) holds for some i in [0, n), on the host workers.  pred is called on every item (no early exit), so it
// may also write what item i needs.
template <class P>
bool parallel_any(size_t n, size_t grain, P pred) {
    std::atomic<int> any(0);
    parallel_ranges(n, grain, [&](size_t lo, size_t hi) {
        bool a = false;
        for (size_t i = lo; i < hi; ++i) a |= pred(i);
        if (a) any.store(1, std::memory_order_relaxed);
    });
    return any.load() != 0;
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline size_t round_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// Host staging memory from the backend (pinned and cached on CUDA): transfers run at full PCIe rate and
// the host reads / writes it in place.
template <class T>
struct HostBuf {
    Backend* be = nullptr;
    T* p = nullptr;
    size_t n = 0;
    HostBuf(Backend* b, size_t count) : be(b), p(static_cast<T*>(b->alloc_host(std::max<size_t>(count, 1) * sizeof(T)))), n(count) {}
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { be->free_host(p); }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
};

template <class T>
struct DevBuf {
    Backend* be = nullptr;
    T* p = nullptr;
    size_t n = 0;
    DevBuf() {}
    DevBuf(Backend* b, size_t count) { alloc(b, count); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { reset(); }
    void alloc(Backend* b, size_t count) {
        reset();
        be = b;
        n = count;
        p = static_cast<T*>(be->alloc(std::max<size_t>(count, 1) * sizeof(T)));
    }
    void reset() {
        if (p) be->free(p);
        p = nullptr;
        n = 0;
    }
    void upload(const T* src, size_t count) { be->h2d(p, src, count * sizeof(T)); }
    void download(T* dst, size_t count) { be->d2h(dst, p, count * sizeof(T)); }
    void swap(DevBuf& o) {
        std::swap(be, o.be);
        std::swap(p, o.p);
        std::swap(n, o.n);
    }
};

// Growable array in staging memory of the backend (pinned on CUDA): result arrays the device writes with
// asynchronous copies at full PCIe rate and the host then reads in place.  The storage stays with the batch object.
template <class T>
struct PinnedVec {
    Backend* be = nullptr;
    T* p = nullptr;
    size_t n = 0, cap = 0;
    PinnedVec() {}
    PinnedVec(const PinnedVec&) = delete;
    PinnedVec& operator=(const PinnedVec&) = delete;
    ~PinnedVec() { release(); }
    void bind(Backend* b) {
        if (be != b) release();
        be = b;
    }
    void release() {
        if (p) be->free_host(p);
        p = nullptr;
        n = cap = 0;
    }
    void reserve(size_t c) {
        if (c <= cap) return;
        T* q = static_cast<T*>(be->alloc_host(std::max<size_t>(c, 1) * sizeof(T)));
        if (p) {
            if (n) memcpy(q, p, n * sizeof(T));
            be->free_host(p);
        }
        p = q;
        cap = c;
    }
    void resize(size_t c) {  // new elements are NOT initialised
        if (c > cap) reserve(std::max(c, cap + cap / 2));
        n = c;
    }
    void clear() { n = 0; }
    void assign(size_t c, const T& v) {
        resize(c);
        for (size_t i = 0; i < c; ++i) p[i] = v;
    }
    void append(const T* src, size_t c) {
        const size_t at = n;
        resize(n + c);
        if (c) memcpy(p + at, src, c * sizeof(T));
    }
    void append_fill(size_t c, const T& v) {
        const size_t at = n;
        resize(n + c);
        for (size_t i = 0; i < c; ++i) p[at + i] = v;
    }
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    T* data() { return p; }
    const T* data() const { return p; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
};

struct Target {
    const char* ptr;
    int len;
    uint64_t off;  // into the packed sequence buffer
};

// One warp-per-alignment sweep as seen by the host.
struct WTask {
    uint64_t qOff = 0, tOff = 0;
    int m = 0, n = 0, mode = 0, flags = 0, kInit = 0, dhi = 0, stopCol = -1, trackFrom = 0;
    int R = 1, nWp = 0;
    int bandH = 0;               // WF_SLIDE: diagonals of the band the window slides down (plan_w)
    int pair = -1, tag = 0;
    bool wantPositions = false;  // the caller needs every end position, not just best/cnt/last
    int splitSide = -1;          // WF_STOPCOL pairs of a Hirschberg node: 0 forward half, 1 reversed half (adjacent tasks)
    int splitBest = 0;           // ... the node's known score
    SplitOut split{};            // ... the split found on the device (stored on the forward task)
    Rec rec{};
    std::vector<int> extra;  // positions past KPOS that attain rec.best, ascending
    long long opsOff = -1;   // into the ops pool (WF_STORE)
    int opsLen = 0;
};

struct WPlan {
    int R, nWp;
    bool slide;
    int dhi;
    int height;  // slide: diagonals of the band
};

WPlan plan_w(int m, int n, int mode, int kBound);
WPlan plan_w_band(int m, long long height, int dhi);

// ---------------------------------------------------------------------------------------------
// Prepared batch
// ---------------------------------------------------------------------------------------------
class Prepared {
public:
    Backend* be = nullptr;
    int N = 0;
    // Strand batch: read i of the caller is pair 2i (as given) and pair 2i+1 (its reverse complement, written by the
    // presence-set pass into a second query region); N counts both.  `strand` is the chosen strand per read (Pass::pick_strands).
    bool strands = false;
    std::vector<uint8_t> strand;
    EdlibAlignConfig cfg{};
    int mode = MODE_NW;  // normalised: anything that is not SHW/HW runs as NW (ref cpp:205-215)
    std::vector<int> qlen, tlen, tidx;
    std::vector<uint64_t> qoff;
    std::vector<Target> tg;
    DevBuf<uint8_t> dSeq;
    DevBuf<uint64_t> dQoff;
    DevBuf<int> dQlen;
    DevBuf<uint8_t> dEqtab;
    bool hasEq = false;
    int ncodes = 0;
    PinnedVec<int> alphaLen;
    // A record target (BatchInput::numRecords > 0): tg[0] holds the records, recOff the first column of each
    // (eb_common.h: RecordParams; numRecords + 1 entries) on the host and the device.  With more than one record, the
    // separator code sep = ncodes - 1 matches nothing; sep == -1: no separator.
    std::vector<int> recOff;
    DevBuf<int> dRecOff;
    int recGap = 0;
    int sep = -1;
    // A best-record batch (BatchInput::bestRecord): the presence sets of prepare (pair i: set i, record r: set N + r),
    // kept until Pass::pick_records has chosen the record of each pair, `record`, and alphaLen follows from them.
    bool bestRecord = false;
    std::vector<int> record;
    DevBuf<uint32_t> dMasks;

    // classification (Engine::classify): pairs per (target, word class) for the lane kernels, the rest
    struct Part {
        std::map<std::pair<int, int>, std::vector<int>> groups;
        std::vector<int> wPairs, other;
    };
    std::map<std::pair<int, int>, std::vector<int>> groups;
    std::vector<Part> parts;        // per-thread pieces, kept for their storage
    std::vector<int> wPairsBase;    // queries above 256 rows
    std::vector<int> otherPairs;    // pairs without a sweep: an empty sequence, or rejected up front (ref cpp:744)
    bool classified = false;

    // results (the distance pass may fill the first four straight from the device)
    PinnedVec<int> ed;              // distance or -1
    std::vector<uint8_t> special;   // 1: an empty sequence (ref cpp:166-184)
    PinnedVec<long long> endStart;  // end locations of pair i: endPool[endStart[i] .. + endCount[i])
    PinnedVec<int> endCount;
    PinnedVec<int> endPool;         // not compact: regions filled by the device, then the host-assembled tail
    PinnedVec<int> startPool;
    PinnedVec<long long> alnStart;  // -1: none
    PinnedVec<int> alnLen;
    PinnedVec<uint8_t> alnPool;
    bool computed = false;
    void bind(Backend* b) {
        be = b;
        alphaLen.bind(b);
        ed.bind(b);
        endStart.bind(b);
        endCount.bind(b);
        endPool.bind(b);
        startPool.bind(b);
        alnStart.bind(b);
        alnLen.bind(b);
        alnPool.bind(b);
    }
};

// ---------------------------------------------------------------------------------------------
// Runner of warp-per-alignment (and per-job lane) sweeps in memory-bounded slices (eb_wrunner.cpp)
// ---------------------------------------------------------------------------------------------
struct WRunner {
    Engine* eng;
    Backend* be;
    Prepared* p;
    std::vector<uint8_t>* opsPool = nullptr;
    int laneOk[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};

    size_t task_bytes(const WTask& t) const;

    // Can the lane kernels sweep queries of nw 32-bit words (1..8) over this batch's alphabet (Peq rows per thread)?
    bool lane_ok(int nw);

    // Tasks whose query fits 256 rows and whose shape one of the lane-kernel classes covers run one
    // alignment per THREAD (lane_kernel); everything else one alignment per warp (w_kernel).
    static int lane_class(const WTask& t) {  // -1: not a lane task
        if (t.m > 256 || (t.flags & (WF_SLIDE | WF_STOPCOL))) return -1;
        const bool qrev = (t.flags & WF_QREV) != 0, trev = (t.flags & WF_TREV) != 0;
        if (t.flags & WF_STORE) return (t.mode == MODE_NW && !qrev && !trev) ? 4 : -1;
        if (qrev != trev) return -1;
        if (qrev) return t.mode == MODE_SHW ? 3 : -1;
        return t.mode;  // 0 NW, 1 SHW, 2 HW, forward
    }

    void run(std::vector<WTask>& tasks);

    // Window blocks (of four words) the thread-per-alignment band kernel needs for task t, or 0 when the task is not
    // of its kind (plain k-banded NW distance sweep of a query taller than the window).
    int band_blocks(const WTask& t) const;
    // One window size of band tasks, in memory-bounded slices (eb_core.h: band_job).
    void run_band(std::vector<WTask>& tasks, const std::vector<int>& idx, int NB);

    // One class of lane tasks, in memory-bounded slices.  Tasks that need a longer end-location list
    // than a record holds are handed to the warp kernel (`spill`), which owns the list machinery.
    void run_lane(std::vector<WTask>& tasks, const std::vector<int>& idx, int nw, int lc, std::vector<int>& spill);

    // ovfCap == 0: first pass (no position list).  ovfCap > 0: second pass over the tasks whose
    // end-location lists exceed KPOS, started from their known minimum with an exact-size list.
    void run_slice(std::vector<WTask>& tasks, const std::vector<int>& slice, int R, int ovfCap);

    // Traceback of the matrix-storing sweeps just launched over `mat`: tb[i] belongs to tasks[owner[i]], whose edit script
    // is appended to the ops pool.  `peq`: the warp kernel's Peq rows, or nullptr with TbJob::peqOff = ~0 (lane kernel).
    void traceback(std::vector<WTask>& tasks, const std::vector<TbJob>& tb, const std::vector<int>& owner, const U2* mat,
                   const uint32_t* peq);
};

// ---------------------------------------------------------------------------------------------
// One compute() over a prepared batch: shared state + the phases of the reference driver
// ---------------------------------------------------------------------------------------------

// Seed index of one target (eb_common.h: SeedIndexParams) and the seed lengths of the levels it serves.
struct SeedIndex {
    int target = -1;
    bool ok = false;
    int Lidx = 0, sigma = 0, numKeys = 0, n = 0;
    int Ls[SEED_LEVELS] = {0, 0, 0, 0};  // seed length per level (0: level not available)
    DevBuf<int> bucketStart, positions;
};

// Builds the radix seed index of an encoded target (seed lengths per level, bucket table, positions).
// separators: a record target whose separator code (>= ncodes) is left out of the radix (keys read it as 0)
bool build_seed_index(Backend* be, const EngineTunables& tun, SeedIndex& sx, const uint8_t* tcodes, int n, int ncodes,
                      bool separators = false);

// The codes of a target encoded by its own alphabet (encode_target, eb_engine.cpp): dense codes of its bytes in ascending
// order, every byte it lacks one extra code that matches nothing.
struct TargetCodes {
    DevBuf<uint32_t> dMask;    // [8] presence set
    DevBuf<uint8_t> dMap;      // [256] byte -> code
    int ncodes = 0;            // codes the kernels see: the extra one included, 256 when every byte value occurs
};

// A target kept resident on the device (streamed read-set path): its encoded bytes with the padding the kernels rely on,
// its codes and its seed index.
struct TargetHandle {
    const char* ptr = nullptr;
    int n = 0;
    size_t bytes = 0;          // round_up(n, 16) + 32 encoded bytes (zero padding)
    DevBuf<uint8_t> codes;
    TargetCodes tc;
    SeedIndex idx;
};

// Window jobs of the candidate filter on the device (the job arrays of K1WParams): planned by the seed planner, which
// counts them in `count` (zeroed by the caller), or planned on the host and uploaded (count == nullptr).
struct WinJobs {
    DevBuf<int> pair, k, start, len, tf;  // pair, threshold + 1, first column, columns, first tracked column (relative)
    int cap = 0;
    int* count = nullptr;
    void alloc(Backend* be, int n) {
        pair.alloc(be, n);
        k.alloc(be, n);
        start.alloc(be, n);
        len.alloc(be, n);
        tf.alloc(be, n);
        cap = n;
    }
};
// What the sweeps of window jobs record: one WinRec per job, and the end columns beyond its inline ones in ovf (counted
// in *ovfCount, zeroed by the caller; the list is complete while the count stays <= ovfCap).
struct WinRecords {
    WinRec* recs;
    Ovf* ovf;
    int* ovfCount;
    int ovfCap;
};

// One slice of a device-driven group: reads [first, first+count) of the group's list (pair = list[first+slot], or
// firstPair + slot when the group is a run of consecutive pairs), its region of the end-location pool and its
// header {end locations, reads pending, pool overflow, windows}.
// Room of a slice's extra list (end columns beyond the KPOS inline ones of a read) beyond a quarter of its reads.
constexpr int DEV_EXTRA_SLACK = 16384;
// Ints of the end-location pool a slice of `count` reads may fill: <= KPOS inline end columns per read + its extra list.
inline long long dev_slice_pool(long long count) { return 4 * count + count / 4 + DEV_EXTRA_SLACK; }
struct DevSlice {
    int t = 0, nw = 0;
    int firstPair = -1;      // >= 0: consecutive pairs (no read list on the device)
    size_t listOff = 0;      // into the uploaded read lists otherwise
    int count = 0;
    long long poolBase = 0;
    int poolCap = 0;
    int poolFetched = 0;     // ints of the region the first (asynchronous) copy brings to the host
    uint64_t done = 0;       // mark on the results stream: the slice's results are on the host
    bool finished = false;
};

struct Pass {
    Engine& eng;
    Backend* be;
    Prepared* p;
    EngineTunables& tun;
    EngineStats& stats;
    Trace trace;
    const int N, mode, k;
    // per-pair sweep outcome before the "-1" rule (storage reused from pass to pass: EngineScratch).  Only the
    // pairs the host-driven stages handle use these (host_touch): reads decided by the device-driven first seed
    // level never appear here.
    std::vector<int>&best, &cnt;
    std::vector<long long>& posStart;  // end columns of pair i: posPool[posStart[i] .. +posLen[i])
    std::vector<int>&posLen, &posPool;
    std::vector<int> wPairs;          // pairs swept by the warp / lane-job kernels
    std::vector<uint8_t> opsPool;
    WRunner runner;

    // ---- device-driven first seed level (eb_pass_lane.cpp) ----
    bool devMode = false;             // some group of this pass runs it: results are assembled per slice on the device
    std::vector<int> hostPairs;       // devMode: the pairs whose outcome lives in the host vectors above
    std::vector<DevSlice> slices;
    DevBuf<int> dEd, dEndCount, dHeaders, dPool, dLeftCount, dLists;
    DevBuf<long long> dEndStart;
    DevBuf<Leftover> dLeft;
    PinnedVec<int> hHeaders;
    long long poolReserved = 0;       // end-location pool handed out to slices so far
    size_t listsUsed = 0;
    bool wholeArrays = false;
    long long windowsSeen = 0, readsSeen = 0;
    // one more device->host copy to ride with the results of the next slice enqueued (streamed batches: alphabet lengths)
    void* extraCopyDst = nullptr;
    const void* extraCopySrc = nullptr;
    size_t extraCopyBytes = 0;

    Pass(Engine& e, Backend* b, Prepared* pr)
        : eng(e), be(b), p(pr), tun(e.tun), stats(e.stats), N(pr->N), mode(pr->mode), k(pr->cfg.k),
          best(e.scratch.best), cnt(e.scratch.cnt), posStart(e.scratch.posStart), posLen(e.scratch.posLen),
          posPool(e.scratch.posPool), runner{&e, b, pr, &opsPool} {
        hHeaders.bind(b);
        best.resize((size_t)N);
        cnt.resize((size_t)N);
        posStart.resize((size_t)N);
        posLen.resize((size_t)N);
        posPool.clear();
    }
    // Resets the host-side outcome of the pairs list[0..n) (every pair the host-driven stages are about to handle).
    void host_touch(const int* list, size_t n) {
        parallel_ranges(n, 65536, [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) {
                const int pair = list[i];
                best[pair] = -1;
                cnt[pair] = 0;
                posStart[pair] = -1;
                posLen[pair] = 0;
            }
        });
    }
    void host_touch_all() {
        parallel_ranges((size_t)N, 65536, [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) {
                best[i] = -1;
                cnt[i] = 0;
                posStart[i] = -1;
                posLen[i] = 0;
            }
        });
    }

    // The radix seed index of the target the seed stages last worked on (one table for every level); kept in the
    // engine across passes when the caller registered the target (EngineScratch::keptIndex), else rebuilt per pass.
    SeedIndex* seedIdx = nullptr;
    SeedIndex ownIdx;
    bool seed_index(int t);

    // ---- seed windows of the candidate filter: planned (seed_plan), swept (k1w), reduced per read (win_reduce) ----
    // Planner parameters of seed level `level` over target tg; the caller adds its reads (readList / firstPair, thr,
    // numReads, maxLen) and their plans (plan).
    SeedPlanParams seed_plan_params(const Target& tg, int level) const;
    // Plans the windows of sp's reads into `jobs`, with room for `cap` of them (*jobs.count zero).  hostCount: returns their
    // number, planned again with the exact room when they did not fit.  Otherwise the number stays on the device (reads
    // whose windows do not fit are saturated) and -1 is returned.
    int plan_windows(SeedPlanParams sp, WinJobs& jobs, int cap, bool hostCount);
    // Sweeps the first numJobs jobs, or (numJobs < 0) as many as *jobs.count says on the device, into `out`.
    void sweep_windows(const Target& tg, int nw, const WinJobs& jobs, int numJobs, const WinRecords& out);
    // Reduces the window records of the planned reads into out[numReads] (positions past KPOS in extra); rp carries
    // the fields of the device-driven mode, or none.
    void reduce_windows(WinReduceParams rp, const SeedPlan* plan, int numReads, const WinRecords& wr, Rec* out, int* extra,
                        int* extraCount, int extraCap);

    // One group of pairs that share a target and a word class (queries <= 256 rows), on its way through
    // the host-driven stages of the distance pass.  Reads are addressed by their index `s` into `list`.
    struct LaneGroup {
        int t, nw;               // target index, 32-bit words per query
        const std::vector<int>& list;  // the pairs of the group
        const Target& tg;
        int n;                   // target length
        std::vector<int> bound;  // per read: largest distance that still counts as found
        std::vector<int> excl;   // per read: it is known that no distance <= excl[s] exists
        std::vector<int> direct; // reads that take the plain full sweep
        std::vector<uint8_t> repeat;  // per read: the last seed level tried found too many occurrences of its seeds
    };

    // Chunk geometry: a HW sweep may be cut into target chunks (each re-started 2*m columns
    // early, exact because no HW path spans more than 2*m target symbols) so that a small
    // group still fills the machine.
    void lane_geometry(const LaneGroup& c, int g, int nwL, int& chunks, int& chunkLen, bool perChunkRecs);

    // One launch over the reads `sub` (indices into `list`) with sentinels / thresholds subK.
    void lane_sweep(LaneGroup& c, const std::vector<int>& sub, const std::vector<int>& subK, int nwL, int chunks, int chunkLen,
                    int cap, int prefixLen, int rangeMode, std::vector<Rec>& outRecs, std::vector<Ovf>& outOvf);

    // Merge the chunks of every read: the minimum wins; its columns are the inline positions
    // of the chunks attaining it (ascending by construction) plus, in a second pass, the
    // listed ones.  Returns the reads whose lists are incomplete (some chunk holds > KPOS).
    void lane_merge(LaneGroup& c, const std::vector<int>& sub, int chunks, const std::vector<Rec>& rr, const std::vector<Ovf>* oo,
                    std::vector<int>& incomplete, long long& missing);

    // The outcome of `pair` is "no alignment within its bound": no distance, no end columns.
    void no_alignment(int pair) {
        best[pair] = 0x7fffffff;
        cnt[pair] = 0;
        posLen[pair] = 0;
    }
    // It is now known that read s has no alignment within t.  Returns whether that is final (t is the read's bound: its
    // outcome is set); otherwise the read goes on to a later stage.
    bool no_distance_within(LaneGroup& c, int s, int t);

    // Strand batches: the cross-strand rule (eb_core.h: strand_rule) over the reads of `list` whose other strand is in
    // the list as well (at s + 1 for a forward pair s).  The reads of the `pending` lists are undecided (excl / bound
    // per read), the others decided (best[]).  Tightens the bounds; a losing pending read is decided as "no alignment"
    // and leaves its list.
    void strand_prune(const std::vector<int>& list, const std::vector<int>& excl, std::vector<int>& bound,
                      std::initializer_list<std::vector<int>*> pending);
    // After the end locations: per read of a strand batch, the winning strand (Prepared::strand); the loser's result
    // becomes "no alignment", so that start locations and paths are only computed for winners.
    void pick_strands();
    // After the end locations of a best-record batch, before pick_strands: per pair, the first record that holds one of
    // its end columns (Prepared::record), its end columns kept and counted from that record's start; then every pair
    // is rebased onto its record (one Target per record, tidx / tlen) and its alphabet length taken over that record.
    void pick_records();

    // Outcome of the reads `cand` (indices into `list`) of a window stage, with thresholds thr[i] (< 0: the stage left
    // the read out, it goes on), their plans on the device and the records of their swept windows: the reduction
    // (win_reduce), then per read decided (best / cnt / end columns), no distance within thr[i] (no_distance_within),
    // on to `next` (saturated) or to c.direct (long end-location list).  Counts the last two in nSat / nLong.
    void window_outcomes(LaneGroup& c, const std::vector<int>& cand, const int* thr, const SeedPlan* plan, const WinRecords& wr,
                         std::vector<int>& next, int& nSat, int& nLong);

    // Seed stage, host-driven: exact seeds of every read looked up in the index of the target; windows around
    // the expected end columns are planned, swept and reduced on the device (eb_core.h: seed_plan_read).
    void seed_stage(LaneGroup& c, int level, const std::vector<int>& in, std::vector<int>& next);

    // Prefix stage over the reads `in` (indices into `list`): a sweep of the first P rows of every read reports
    // the target ranges where that prefix matches within t = min(K0, bound); the whole read is then swept over
    // one window per range, and the windows are reduced as those of a seed stage (window_outcomes).
    void prefix_stage(LaneGroup& c, int P, int K0, const std::vector<int>& in, std::vector<int>& next);

    // The plain lane-per-alignment sweep of the reads in c.direct over the whole target.
    void plain_sweep(LaneGroup& c);
    bool useK1t = false;  // the next lane_sweep launches the warp-per-read kernel (a handful of reads)

    // Distance pass of one group of pairs that share target `t` and word class `nw` (queries <= 256
    // rows), host-driven: the stages of the candidate filter (HW over a long target; DESIGN.md section 5), each on
    // the reads the previous ones left undecided, then the plain lane-per-alignment sweep of what is left.
    // `excl` (or nullptr) carries what the device-driven first level found out about the reads (-2: plain sweep),
    // `bounds` their bounds, `firstSeedLevel` the first seed level still to try.
    void lane_group(int t, int nw, const std::vector<int>& list, const std::vector<int>* excl = nullptr,
                    const std::vector<int>* bounds = nullptr, int firstSeedLevel = 0);

    // ---- device-driven first seed level ----------------------------------------------------------------
    // May group (t, nw) take it?  (HW over a long target, plain equality, seed stage enabled, index available.)
    bool dev_eligible(int t, int nw);
    // Device arrays of the pass (per-pair results, leftover list, headers, end-location pool, read lists) for at most
    // `maxSlices` slices of `reads` reads in all, `listed` of them in slices of scattered pairs; p->endPool sized to match.
    void dev_begin(long long reads, int maxSlices, long long listed);
    // After the last slice is enqueued: p->endPool trimmed to the regions the slices were handed.
    void dev_enqueued() { p->endPool.resize((size_t)poolReserved); }
    // Enqueues, without any host synchronisation, the whole first level for reads [first, first+count) of a group:
    // seed planning, window sweeps, reduction, assembly of distances and end locations into the slice's pool region.
    // Returns the slice index.
    int dev_enqueue_slice(int t, int nw, int firstPair, const int* listHost, int first, int count);
    // Waits for the results of slice si (their copies were enqueued with the slice).
    void dev_finish_slice(int si);
    // After the last slice: the reads the device could not decide, grouped and run through the host-driven stages.
    void dev_leftovers();

    // ---- hits (edlibB200FindHits; eb_pass_lane.cpp) ----------------------------------------------------------
    // Runs instead of the distance pass: every end column scoring <= k of every pair over its target, into `out`
    // (malloc'd arrays; the two pairs of a read of a strand batch share its cap, forward first).  The pairs of a target
    // group of at least k1MinGroup pairs (or of the batch's only target) take the seed windows of the first level whose
    // threshold reaches k, or the whole-target sweep (no such level, saturated plan, repeats, short target, equality
    // table); every other pair the per-pair route (chunks of its own target, launch_lane_hits).  All routes count,
    // place, then fill.  task LOC / PATH: then the start location / edit script of every stored hit (hit_alignments).
    // A record target: columns (and starts) are mapped into their records on the device, their records into *records.
    void hits(long long maxHits, int task, EdlibB200HitAlignments* out, int** records);
    // Start locations (and, task PATH, edit scripts) of the S stored hits in dCols / dScores, whose pairs start at
    // dBase: lane sweeps per word class over slices of stored hits, jobs built on the device (eb_core.h: hit_res_item).
    void hit_alignments(int task, long long S, const std::vector<long long>& stored, const long long* dBase,
                        const int* dCols, const int* dScores, EdlibB200HitAlignments* out);
    // The K1W launch over the first numJobs jobs (or as many as *jobs.count says, numJobs < 0), records not set.
    K1WParams window_params(const Target& tg, const WinJobs& jobs, int numJobs) const;

    // Distance pass of everything else: one alignment per warp (or per thread with its own target).
    void warp_distance();
    // HW sweeps of long queries (> 256 rows) over a long target: seed levels with doubling thresholds (windows swept
    // by the warp kernel along their diagonals), then the target cut into chunks restarted 2m columns early.
    void long_hw_distance(const std::vector<int>& pairs);

    // editDistance and endLocations from the sweep outcomes (ref cpp:219-225 and the -1 rule), appended to the
    // batch's end-location pool: of every pair (pairs == nullptr) or of the listed ones.
    void collect_ends(const std::vector<int>* pairs);

    void start_locations();

    void paths();

    // ---- start locations / paths of short queries (<= 256 rows) driven from the device (eb_pass_results.cpp) ----
    // Word classes (bit nw) that hold found pairs the lane kernel can sweep, bit 0: some found pair is of no such class.
    unsigned resClasses = 0;
    bool resUploaded = false;
    DevBuf<int> rEd, rEndCount, rEndPool, rStartPool, rErr;
    DevBuf<long long> rEndStart;
    DevBuf<uint64_t> rTOffPair;
    void res_begin();                    // classes + per-pair results on the device
    void res_fill(ResParams& rp, int nw);
    void res_check();
    int resMaxEd = 0;
    // Longest target slice a device-driven path of word class nw may have (longer ones, rare, take the host tree;
    // always inside the reference's 1 MiB rule, ref cpp:1188-1190, for queries of <= 256 rows).
    int res_max_path_n(int nw) const { return std::min(64 * nw, 32 * nw + resMaxEd); }
    bool res_class(int m) const { return m > 0 && m <= 256 && ((resClasses >> ((m + 31) / 32)) & 1u); }
    void start_locations_device();
    void paths_device();
};

}  // namespace eb
