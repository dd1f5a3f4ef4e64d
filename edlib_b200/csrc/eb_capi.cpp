// eb_capi.cpp -- the extern "C" surface declared in include/edlib.h and include/edlib_b200.h.
// Thin: argument checks, one process-wide engine behind a mutex (the reference API is
// re-entrant and is called with the GIL released, ref bindings/python/edlib.pyx:128-129), and
// the two pure-host helpers that carry no DP work (config constructors, CIGAR run-length
// encoding, free).
#include <malloc.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/edlib.h"
#include "../../include/edlib_b200.h"
#include "eb_engine.h"

namespace eb {
void host_parallel_ranges(size_t n, size_t grain, const std::function<void(size_t, size_t)>& fn);  // eb_engine.cpp
void free_result_arrays(EdlibAlignResult* results, size_t lo, size_t hi);  // eb_engine.cpp: frees and clears them
void fail_results(EdlibAlignResult* results, int n);  // eb_engine.cpp: error results (status, distance -1, no arrays)
void free_hits(EdlibB200Hits* h);  // eb_engine.cpp: frees the arrays of a hit list and clears it
void free_hit_alignments(EdlibB200HitAlignments* h);  // eb_engine.cpp: ... and the starts / scripts of its hits
Backend* create_backend(std::string* err);  // provided by the backend object linked into this library
int select_device(int device, std::string* err);  // 0 on success
}

namespace {

std::mutex g_mu;
eb::Backend* g_backend = nullptr;
eb::Engine* g_engine = nullptr;
std::string g_initError;
bool g_initTried = false;

// Small calls (single edlibAlign calls, batches of a few pairs) do not queue behind each other or behind a large batch:
// beside the main engine (large batches, the staged API, target handles; under g_mu) a few more engines, each with
// its own streams, scratch and lock, take them round robin -- concurrent callers (the reference's Python binding
// releases the GIL around edlibAlign, bindings/python/edlib.pyx:128-129) overlap their launches and copies.
struct SideEngine {
    std::mutex mu;
    eb::Backend* be = nullptr;
    eb::Engine* eng = nullptr;
};
constexpr int kMaxSide = 8;
SideEngine g_side[kMaxSide];
int g_numSide = -1;  // -1: not decided yet
std::atomic<unsigned> g_nextSide{0};
constexpr int kSmallBatch = 256;  // pairs; larger batches fill the device on their own and use the main engine
thread_local eb::Engine* t_lastEngine = nullptr;  // engine the calling thread used last (LastStats / LastKernelReport)
thread_local std::string t_lastError;              // text of the last failure of a call made by this thread

eb::Engine* engine_locked() {
    if (!g_initTried) {
        g_initTried = true;
        g_backend = eb::create_backend(&g_initError);
        if (g_backend) g_engine = new eb::Engine(g_backend);
    }
    // the caller may be any host thread: CUDA's current device is per thread
    if (g_backend) {
        try {
            g_backend->bind_thread();
        } catch (const std::exception& e) {
            if (g_engine) g_engine->lastError = e.what();
            return nullptr;
        }
    }
    return g_engine;
}

// A side engine for a small call, locked (nullptr: none configured / the device is unusable: use the main engine).
SideEngine* side_engine_acquire() {
    {
        std::lock_guard<std::mutex> lock(g_mu);
        if (!engine_locked()) return nullptr;
        if (g_numSide < 0) {
            const char* e = getenv("EDLIB_B200_ENGINES");
            g_numSide = std::max(0, std::min(kMaxSide, e && *e ? atoi(e) - 1 : 3));
        }
    }
    if (g_numSide <= 0) return nullptr;
    SideEngine* s = &g_side[g_nextSide.fetch_add(1, std::memory_order_relaxed) % (unsigned)g_numSide];
    s->mu.lock();
    if (!s->eng) {
        std::string err;
        s->be = eb::create_backend(&err);
        if (s->be) s->eng = new eb::Engine(s->be);
        if (!s->eng) {
            s->mu.unlock();
            return nullptr;
        }
    }
    try {
        s->be->bind_thread();
    } catch (...) {
        s->mu.unlock();
        return nullptr;
    }
    return s;
}

// the statistics of the last pass of e (its device times are read now)
void copy_stats(eb::Engine* e, EdlibB200Stats* s) {
    e->finish_stats();
    s->kernelMs = e->stats.kernelMs;
    s->k1Ms = e->stats.k1Ms;
    s->launches = e->stats.launches;
    s->h2dBytes = e->stats.h2dBytes;
    s->d2hBytes = e->stats.d2hBytes;
    s->k1Cells = e->stats.k1Cells;
    s->wCells = e->stats.wCells;
    s->filterDecided = e->stats.filterDecided;
    s->filterFallback = e->stats.filterFallback;
    s->filterWindows = (int)std::min<long long>(e->stats.filterWindows, 0x7fffffff);
}

}  // namespace

extern "C" {

// ref edlib.cpp:1465-1475
EDLIB_API EdlibAlignConfig edlibNewAlignConfig(int k, EdlibAlignMode mode, EdlibAlignTask task,
                                               const EdlibEqualityPair* additionalEqualities,
                                               int additionalEqualitiesLength) {
    EdlibAlignConfig c;
    c.k = k;
    c.mode = mode;
    c.task = task;
    c.additionalEqualities = additionalEqualities;
    c.additionalEqualitiesLength = additionalEqualitiesLength;
    return c;
}

// ref edlib.cpp:1477-1479
EDLIB_API EdlibAlignConfig edlibDefaultAlignConfig(void) {
    return edlibNewAlignConfig(-1, EDLIB_MODE_NW, EDLIB_TASK_DISTANCE, NULL, 0);
}

// ref edlib.cpp:1481-1485
EDLIB_API void edlibFreeAlignResult(EdlibAlignResult result) {
    free(result.endLocations);
    free(result.startLocations);
    free(result.alignment);
}

// edlibAlignBatch and edlibB200AlignBatchStrands (strands != nullptr)
static int align_batch_entry(const char* const* queries, const int* queryLengths, const char* const* targets,
                             const int* targetLengths, int numPairs, const EdlibAlignConfig& config, EdlibAlignResult* results,
                             unsigned char* strands) {
    eb::BatchInput in{queries, queryLengths, targets, targetLengths, numPairs, config};
    in.strands = strands != nullptr;
    if (numPairs <= kSmallBatch) {
        if (SideEngine* s = side_engine_acquire()) {
            t_lastEngine = s->eng;
            const int rc = s->eng->align_batch(in, results, strands);
            if (rc != EDLIB_STATUS_OK) t_lastError = s->eng->lastError;  // (copied while the engine is still ours)
            s->mu.unlock();
            return rc;
        }
    }
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e) {  // no usable device: fail loudly, there is no CPU path
        eb::fail_results(results, numPairs);
        return EDLIB_STATUS_ERROR;
    }
    t_lastEngine = e;
    const int rc = e->align_batch(in, results, strands);
    if (rc != EDLIB_STATUS_OK) t_lastError = e->lastError;
    return rc;
}

EDLIB_API int edlibAlignBatch(const char* const* queries, const int* queryLengths,
                              const char* const* targets, const int* targetLengths,
                              int numPairs, const EdlibAlignConfig config, EdlibAlignResult* results) {
    if (numPairs < 0 || (numPairs > 0 && (!queries || !queryLengths || !targets || !targetLengths || !results)))
        return EDLIB_STATUS_ERROR;
    if (numPairs == 0) return EDLIB_STATUS_OK;
    return align_batch_entry(queries, queryLengths, targets, targetLengths, numPairs, config, results, nullptr);
}

EDLIB_API int edlibB200AlignBatchStrands(const char* const* queries, const int* queryLengths,
                                         const char* const* targets, const int* targetLengths, int numPairs,
                                         const EdlibAlignConfig config, EdlibAlignResult* results, unsigned char* strands) {
    if (numPairs < 0 || (numPairs > 0 && (!queries || !queryLengths || !targets || !targetLengths || !results || !strands)))
        return EDLIB_STATUS_ERROR;
    if (numPairs == 0) return EDLIB_STATUS_OK;
    if (numPairs > 0x3fffffff) return EDLIB_STATUS_ERROR;  // both strands of every read are pairs of one batch
    return align_batch_entry(queries, queryLengths, targets, targetLengths, numPairs, config, results, strands);
}

// ref edlib.cpp:146-301
EDLIB_API EdlibAlignResult edlibAlign(const char* query, int queryLength, const char* target, int targetLength,
                                      const EdlibAlignConfig config) {
    EdlibAlignResult r;
    const char* q = query ? query : "";
    const char* t = target ? target : "";
    edlibAlignBatch(&q, &queryLength, &t, &targetLength, 1, config, &r);
    return r;
}

// ref edlib.cpp:303-350.  Pure formatting of an existing edit script (no DP): kept on the host.
// One pass: runs are found eight operations at a time (EXTENDED: a run is a stretch of equal bytes) and written into a
// scratch buffer of the worst-case size (every run "1X": two characters per operation), then copied into one exact malloc.
static inline int cigar_run_end(const unsigned char* a, int i, int len, unsigned char op) {
    int j = i + 1;
    const uint64_t pat = 0x0101010101010101ull * op;
    while (j + 8 <= len) {
        uint64_t w;
        memcpy(&w, a + j, 8);
        const uint64_t x = w ^ pat;
        if (x) return j + (__builtin_ctzll(x) >> 3);  // first byte that differs (little endian)
        j += 8;
    }
    while (j < len && a[j] == op) ++j;
    return j;
}

// STANDARD format: MATCH (0) and MISMATCH (3) both print 'M' -- the two codes whose low bits agree.  Any other byte
// (I, D, or a bad code) ends the run.
static inline int cigar_m_run_end(const unsigned char* a, int i, int len) {
    int j = i + 1;
    const uint64_t ones = 0x0101010101010101ull;
    while (j + 8 <= len) {
        uint64_t w;
        memcpy(&w, a + j, 8);
        const uint64_t x = ((w ^ (w >> 1)) & ones) | (w & ~(3 * ones));  // per byte: bit0 != bit1, or a bit above them
        if (x) return j + (__builtin_ctzll(x) >> 3);
        j += 8;
    }
    while (j < len && (a[j] == 0 || a[j] == 3)) ++j;
    return j;
}

EDLIB_API char* edlibAlignmentToCigar(const unsigned char* alignment, int alignmentLength, EdlibCigarFormat cigarFormat) {
    if (cigarFormat != EDLIB_CIGAR_EXTENDED && cigarFormat != EDLIB_CIGAR_STANDARD) return NULL;
    const bool ext = cigarFormat == EDLIB_CIGAR_EXTENDED;
    const char* sym = ext ? "=IDX" : "MIDM";
    const int len = alignmentLength < 0 ? 0 : alignmentLength;
    char stackBuf[2048];
    const size_t worst = 2 * (size_t)len + 1;
    char* buf = worst <= sizeof(stackBuf) ? stackBuf : static_cast<char*>(malloc(worst));
    if (!buf) return NULL;
    char* w = buf;
    bool bad = false;
    for (int i = 0; i < len;) {
        const unsigned char op = alignment[i];
        if (op > 3) {
            bad = true;
            break;
        }
        const char c = sym[op];
        // STANDARD: MATCH and MISMATCH share 'M' (ref cpp:311-314); insertions and deletions are plain runs in both formats
        const int j = (ext || c != 'M') ? cigar_run_end(alignment, i, len, op) : cigar_m_run_end(alignment, i, len);
        int run = j - i;
        char digits[12];
        int nd = 0;
        for (; run; run /= 10) digits[nd++] = (char)('0' + run % 10);
        while (nd) *w++ = digits[--nd];
        *w++ = c;
        i = j;
    }
    char* res = NULL;
    if (!bad) {
        const size_t bytes = (size_t)(w - buf) + 1;
        res = static_cast<char*>(malloc(bytes));
        if (res) {
            memcpy(res, buf, bytes - 1);
            res[bytes - 1] = 0;
        }
    }
    if (buf != stackBuf) free(buf);
    return res;
}

// ---- include/edlib_b200.h ------------------------------------------------------------------

EDLIB_API const char* edlibB200LastError(void) {
    // every calling thread reads its own copy: a later call on another thread cannot change it under the reader
    static thread_local std::string copy;
    std::lock_guard<std::mutex> lock(g_mu);
    // failures of edlibAlign / edlibAlignBatch are recorded per calling thread (side engines run concurrently); the
    // staged / handle entry points all use the main engine under this lock
    if (t_lastEngine && t_lastEngine != g_engine) copy = t_lastError;
    else copy = g_engine ? g_engine->lastError : g_initError;
    return copy.c_str();
}

EDLIB_API int edlibB200SetDevice(int device) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (g_initTried) return EDLIB_STATUS_ERROR;
    // remembered by the backend factory: the engine binds to THIS device whichever thread makes the first call
    return eb::select_device(device, &g_initError) == 0 ? EDLIB_STATUS_OK : EDLIB_STATUS_ERROR;
}

EDLIB_API int edlibB200DeviceNumaNode(void) {
    std::lock_guard<std::mutex> lock(g_mu);
    return engine_locked() ? g_backend->numa_node() : -1;
}

EDLIB_API int edlibB200TuneHostAllocator(void) {
#if defined(__GLIBC__)
    const int a = mallopt(M_TRIM_THRESHOLD, 1 << 30);  // freed heap memory stays with the allocator
    const int b = mallopt(M_TOP_PAD, 64 << 20);        // heaps grow in large steps
    return (a && b) ? EDLIB_STATUS_OK : EDLIB_STATUS_ERROR;
#else
    return EDLIB_STATUS_ERROR;
#endif
}

// Large result sets are freed on the host pool, the way they were built: glibc re-serves chunks that ONE thread freed
// (cold in every other core's cache, threaded through its bins one by one) several times slower than chunks the worker
// threads freed themselves.
EDLIB_API void edlibB200FreeResults(EdlibAlignResult* results, int n) {
    if (!results || n <= 0) return;
    if (n < 65536) {
        eb::free_result_arrays(results, 0, (size_t)n);
        return;
    }
    std::lock_guard<std::mutex> lock(g_mu);  // the host pool serves one client at a time
    eb::host_parallel_ranges((size_t)n, 16384, [results](size_t lo, size_t hi) { eb::free_result_arrays(results, lo, hi); });
}

EDLIB_API int edlibB200Available(void) {
    std::lock_guard<std::mutex> lock(g_mu);
    return engine_locked() ? 1 : 0;
}

static EdlibB200Batch* batch_prepare_entry(const char* const* queries, const int* queryLengths, const char* const* targets,
                                           const int* targetLengths, int numPairs, const EdlibAlignConfig& config, bool strands) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e || numPairs <= 0 || (strands && numPairs > 0x3fffffff)) return NULL;
    t_lastEngine = e;
    try {
        eb::BatchInput in{queries, queryLengths, targets, targetLengths, numPairs, config};
        in.strands = strands;
        return reinterpret_cast<EdlibB200Batch*>(e->prepare(in));
    } catch (const std::exception& ex) {
        e->lastError = ex.what();
        return NULL;
    }
}

EDLIB_API EdlibB200Batch* edlibB200BatchPrepare(const char* const* queries, const int* queryLengths,
                                                const char* const* targets, const int* targetLengths,
                                                int numPairs, const EdlibAlignConfig config) {
    return batch_prepare_entry(queries, queryLengths, targets, targetLengths, numPairs, config, false);
}

EDLIB_API EdlibB200Batch* edlibB200BatchPrepareStrands(const char* const* queries, const int* queryLengths,
                                                       const char* const* targets, const int* targetLengths,
                                                       int numPairs, const EdlibAlignConfig config) {
    return batch_prepare_entry(queries, queryLengths, targets, targetLengths, numPairs, config, true);
}

EDLIB_API int edlibB200BatchStrands(EdlibB200Batch* batch, unsigned char* strands) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e || !batch || !strands) return EDLIB_STATUS_ERROR;
    t_lastEngine = e;
    try {
        e->strands_of(reinterpret_cast<eb::Prepared*>(batch), strands);
    } catch (const std::exception& ex) {
        e->lastError = ex.what();
        return EDLIB_STATUS_ERROR;
    }
    return EDLIB_STATUS_OK;
}

EDLIB_API int edlibB200BatchCompute(EdlibB200Batch* batch, EdlibB200Stats* statsOut) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e || !batch) return EDLIB_STATUS_ERROR;
    t_lastEngine = e;
    try {
        e->stats = eb::EngineStats();
        e->compute(reinterpret_cast<eb::Prepared*>(batch));
    } catch (const std::exception& ex) {
        e->lastError = ex.what();
        return EDLIB_STATUS_ERROR;
    }
    if (statsOut) copy_stats(e, statsOut);
    return EDLIB_STATUS_OK;
}

EDLIB_API int edlibB200BatchResults(EdlibB200Batch* batch, EdlibAlignResult* results) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e || !batch || !results) return EDLIB_STATUS_ERROR;
    t_lastEngine = e;
    try {
        e->materialize(reinterpret_cast<eb::Prepared*>(batch), results);
    } catch (const std::exception& ex) {
        e->lastError = ex.what();
        return EDLIB_STATUS_ERROR;
    }
    return EDLIB_STATUS_OK;
}

EDLIB_API void edlibB200BatchFree(EdlibB200Batch* batch) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (batch && engine_locked()) g_engine->release(reinterpret_cast<eb::Prepared*>(batch));
}

EDLIB_API EdlibB200Target* edlibB200TargetPrepare(const char* target, int targetLength) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e) return NULL;
    t_lastEngine = e;
    try {
        return reinterpret_cast<EdlibB200Target*>(e->target_prepare(target, targetLength));
    } catch (const std::exception& ex) {
        e->lastError = ex.what();
        return NULL;
    }
}

EDLIB_API void edlibB200TargetFree(EdlibB200Target* target) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (target && engine_locked()) g_engine->target_free(reinterpret_cast<eb::TargetHandle*>(target));
}

EDLIB_API int edlibB200AlignmentsToCigar(const EdlibAlignResult* results, int n, EdlibCigarFormat cigarFormat, char** cigars) {
    if (n < 0 || (n > 0 && (!results || !cigars))) return EDLIB_STATUS_ERROR;
    if (cigarFormat != EDLIB_CIGAR_EXTENDED && cigarFormat != EDLIB_CIGAR_STANDARD) return EDLIB_STATUS_ERROR;
    std::lock_guard<std::mutex> lock(g_mu);  // the host pool serves one client at a time
    std::atomic<int> bad(0);
    eb::host_parallel_ranges((size_t)n, 4096, [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            cigars[i] = NULL;
            if (!results[i].alignment || results[i].alignmentLength <= 0) continue;
            cigars[i] = edlibAlignmentToCigar(results[i].alignment, results[i].alignmentLength, cigarFormat);
            if (!cigars[i]) bad.store(1, std::memory_order_relaxed);
        }
    });
    if (!bad.load()) return EDLIB_STATUS_OK;
    for (int i = 0; i < n; ++i) {
        free(cigars[i]);
        cigars[i] = NULL;
    }
    return EDLIB_STATUS_ERROR;
}

EDLIB_API void edlibB200FreeCigars(char** cigars, int n) {
    if (!cigars || n <= 0) return;
    auto free_range = [cigars](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            free(cigars[i]);
            cigars[i] = NULL;
        }
    };
    if (n < 65536) {
        free_range(0, (size_t)n);
        return;
    }
    std::lock_guard<std::mutex> lock(g_mu);  // the host pool serves one client at a time
    eb::host_parallel_ranges((size_t)n, 16384, free_range);
}

// The records of edlibB200FindRecordHits / edlibB200AlignRecords.
struct RecordArgs {
    const char* const* records;
    const int* lengths;
    int n;
    int gap;  // separator symbols between two records (set by record_input_error)
};

// What a record call refuses of its records (include/edlib_b200.h), or "", with `at` the message prefix; sets the gap.
// Only lengths are read: a record's bytes are not touched here.
static std::string record_input_error(const std::string& at, RecordArgs* records, int k, int longest) {
    if (records->n < 1) return at + "numRecords must be >= 1";
    if (!records->records || !records->lengths) return at + "no records";
    // an alignment that crosses a separator of gap symbols costs more than k (if k >= 0) and more than any query's length
    records->gap = (k < 0 ? longest : std::min(k, longest)) + 1;
    long long total = (long long)(records->n - 1) * records->gap;
    for (int r = 0; r < records->n; ++r) {
        if (!records->records[r] || records->lengths[r] < 1) return at + "every record must be non-NULL with at least one symbol";
        total += records->lengths[r];
    }
    if (total > EDLIB_B200_MAX_RECORD_TARGET)
        return at + "the records and their separators exceed EDLIB_B200_MAX_RECORD_TARGET symbols";
    return std::string();
}

// The per-pair targets of edlibB200FindPairHits.
struct PairArgs {
    const char* const* targets;
    const int* lengths;
};

// What edlibB200FindHits (alignments == false) / edlibB200FindHitAlignments / edlibB200FindRecordHits (records != NULL)
// / edlibB200FindPairHits (pairs != NULL, one query per pair) refuse (include/edlib_b200.h), or "".
static std::string hits_input_error(const char* entry, bool alignments, const char* const* queries, const int* queryLengths,
                                    int numQueries, const char* target, int targetLength, RecordArgs* records,
                                    const PairArgs* pairs, const EdlibAlignConfig& config, int bothStrands, long long maxHits) {
    const std::string at = std::string(entry) + ": ";
    if (numQueries < 0) return at + (pairs ? "numPairs < 0" : "numQueries < 0");
    if (numQueries > 0 && (!queries || !queryLengths)) return at + "no queries";
    if (bothStrands && numQueries > 0x3fffffff) return at + (pairs ? "too many pairs for both strands" : "too many queries for both strands");
    if (pairs && numQueries > 0 && (!pairs->targets || !pairs->lengths)) return at + "no targets";
    if (!records && !pairs && (!target || targetLength < 1)) return at + "the target must have at least one symbol";
    if (config.mode != EDLIB_MODE_HW) return at + "mode must be EDLIB_MODE_HW";
    if (!alignments && config.task != EDLIB_TASK_DISTANCE) return at + "task must be EDLIB_TASK_DISTANCE";
    if (alignments && config.task != EDLIB_TASK_DISTANCE && config.task != EDLIB_TASK_LOC && config.task != EDLIB_TASK_PATH)
        return at + "task must be EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC or EDLIB_TASK_PATH";
    if (config.k < 0) return at + "k must be >= 0";
    if (maxHits < 0) return at + (pairs ? "maxHitsPerPair must be >= 0" : "maxHitsPerQuery must be >= 0");
    if (config.additionalEqualitiesLength > 0 && !config.additionalEqualities) return at + "no equality pairs";
    int longest = 0;
    for (int i = 0; i < numQueries; ++i) {
        if (!queries[i] || queryLengths[i] < 1 || queryLengths[i] > 256) return at + "query lengths must be 1 .. 256";
        longest = std::max(longest, queryLengths[i]);
        if (pairs && (pairs->lengths[i] < 0 || (pairs->lengths[i] > 0 && !pairs->targets[i])))
            return at + "every target length must be >= 0, with a non-NULL target when it is > 0";
    }
    if (!records) return std::string();
    return record_input_error(at, records, config.k, longest);
}

// The hit entries: `out` (never NULL here) is cleared, then filled on success; on failure nothing stays allocated.
// records: a record call (edlibB200FindRecordHits), whose record of each stored hit goes to *recordsOut.  pairs: a pair
// call (edlibB200FindPairHits), query i searched in pairs->targets[i] only.
static int find_hits_entry(const char* entry, bool alignments, bool outNull, const char* const* queries,
                           const int* queryLengths, int numQueries, const char* target, int targetLength,
                           RecordArgs* records, const PairArgs* pairs, const EdlibAlignConfig& config, int bothStrands,
                           long long maxHitsPerQuery, EdlibB200HitAlignments* out, int** recordsOut) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    memset(out, 0, sizeof(*out));
    if (recordsOut) *recordsOut = nullptr;
    if (!e) return EDLIB_STATUS_ERROR;  // no usable device: there is no CPU path
    t_lastEngine = e;
    const std::string bad = outNull ? std::string(entry) + (alignments ? ": out is NULL" : ": hits is NULL")
                                    : hits_input_error(entry, alignments, queries, queryLengths, numQueries, target,
                                                       targetLength, records, pairs, config, bothStrands, maxHitsPerQuery);
    if (!bad.empty()) {
        e->lastError = bad;
        return EDLIB_STATUS_ERROR;
    }
    if (numQueries == 0) {
        out->hits.offsets = static_cast<long long*>(calloc(1, sizeof(long long)));
        out->hits.counts = static_cast<long long*>(malloc(sizeof(long long)));
        if (config.task == EDLIB_TASK_PATH) out->alignmentOffsets = static_cast<long long*>(calloc(1, sizeof(long long)));
        if (out->hits.offsets && out->hits.counts && (config.task != EDLIB_TASK_PATH || out->alignmentOffsets))
            return EDLIB_STATUS_OK;
        eb::free_hit_alignments(out);
        e->lastError = "out of memory for the hit lists";
        return EDLIB_STATUS_ERROR;
    }
    if (records) {  // one target laid out from the records: its length, no host pointer
        targetLength = (records->n - 1) * records->gap;
        for (int r = 0; r < records->n; ++r) targetLength += records->lengths[r];
        target = nullptr;
    }
    const std::vector<const char*> targets(pairs ? 0 : (size_t)numQueries, target);
    const std::vector<int> targetLengths(pairs ? 0 : (size_t)numQueries, targetLength);
    eb::BatchInput in{queries, queryLengths, pairs ? pairs->targets : targets.data(),
                      pairs ? pairs->lengths : targetLengths.data(), numQueries, config};
    in.strands = bothStrands != 0;
    if (records) {
        in.records = records->records;
        in.recordLengths = records->lengths;
        in.numRecords = records->n;
        in.recordGap = records->gap;
    }
    return e->find_hits(in, maxHitsPerQuery, out, recordsOut);
}

EDLIB_API int edlibB200FindHits(const char* const* queries, const int* queryLengths, int numQueries, const char* target,
                                int targetLength, const EdlibAlignConfig config, int bothStrands, long long maxHitsPerQuery,
                                EdlibB200Hits* hits) {
    EdlibB200HitAlignments out;
    const int st = find_hits_entry("edlibB200FindHits", false, !hits, queries, queryLengths, numQueries, target,
                                   targetLength, nullptr, nullptr, config, bothStrands, maxHitsPerQuery, &out, nullptr);
    if (hits) *hits = out.hits;  // task DISTANCE: nothing else was allocated
    return st;
}

EDLIB_API void edlibB200FreeHits(EdlibB200Hits* hits) {
    if (hits) eb::free_hits(hits);
}

EDLIB_API int edlibB200FindHitAlignments(const char* const* queries, const int* queryLengths, int numQueries,
                                         const char* target, int targetLength, const EdlibAlignConfig config,
                                         int bothStrands, long long maxHitsPerQuery, EdlibB200HitAlignments* out) {
    EdlibB200HitAlignments scratch;
    return find_hits_entry("edlibB200FindHitAlignments", true, !out, queries, queryLengths, numQueries, target,
                           targetLength, nullptr, nullptr, config, bothStrands, maxHitsPerQuery, out ? out : &scratch, nullptr);
}

EDLIB_API void edlibB200FreeHitAlignments(EdlibB200HitAlignments* out) {
    if (out) eb::free_hit_alignments(out);
}

EDLIB_API int edlibB200FindRecordHits(const char* const* queries, const int* queryLengths, int numQueries,
                                      const char* const* records, const int* recordLengths, int numRecords,
                                      const EdlibAlignConfig config, int bothStrands, long long maxHitsPerQuery,
                                      EdlibB200RecordHits* out) {
    EdlibB200RecordHits scratch;
    EdlibB200RecordHits* o = out ? out : &scratch;
    RecordArgs ra{records, recordLengths, numRecords, 0};
    return find_hits_entry("edlibB200FindRecordHits", true, !out, queries, queryLengths, numQueries, nullptr, 0, &ra,
                           nullptr, config, bothStrands, maxHitsPerQuery, &o->aln, &o->records);
}

EDLIB_API int edlibB200FindPairHits(const char* const* queries, const int* queryLengths, const char* const* targets,
                                    const int* targetLengths, int numPairs, const EdlibAlignConfig config, int bothStrands,
                                    long long maxHitsPerPair, EdlibB200HitAlignments* out) {
    EdlibB200HitAlignments scratch;
    const PairArgs pa{targets, targetLengths};
    return find_hits_entry("edlibB200FindPairHits", true, !out, queries, queryLengths, numPairs, nullptr, 0, nullptr, &pa,
                           config, bothStrands, maxHitsPerPair, out ? out : &scratch, nullptr);
}

EDLIB_API void edlibB200FreeRecordHits(EdlibB200RecordHits* out) {
    if (!out) return;
    eb::free_hit_alignments(&out->aln);
    free(out->records);
    out->records = nullptr;
}

// What edlibB200AlignRecords refuses (include/edlib_b200.h), or "".
static std::string align_records_error(const char* const* queries, const int* queryLengths, int numQueries,
                                       RecordArgs* records, const EdlibAlignConfig& config, int bothStrands,
                                       const EdlibAlignResult* results, const int* recordsOut, const unsigned char* strandsOut) {
    const std::string at = "edlibB200AlignRecords: ";
    if (numQueries < 0) return at + "numQueries < 0";
    if (numQueries > 0 && (!queries || !queryLengths)) return at + "no queries";
    if (numQueries > 0 && !results) return at + "results is NULL";
    if (numQueries > 0 && !recordsOut) return at + "recordsOut is NULL";
    if (bothStrands && numQueries > 0 && !strandsOut) return at + "strandsOut is NULL";
    if (bothStrands && numQueries > 0x3fffffff) return at + "too many queries for both strands";
    if (config.mode != EDLIB_MODE_HW) return at + "mode must be EDLIB_MODE_HW";
    if (config.task != EDLIB_TASK_DISTANCE && config.task != EDLIB_TASK_LOC && config.task != EDLIB_TASK_PATH)
        return at + "task must be EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC or EDLIB_TASK_PATH";
    if (config.additionalEqualitiesLength > 0 && !config.additionalEqualities) return at + "no equality pairs";
    int longest = 0;
    for (int i = 0; i < numQueries; ++i) {
        if (queryLengths[i] < 0 || (queryLengths[i] > 0 && !queries[i])) return at + "every query must be non-NULL with a length >= 0";
        longest = std::max(longest, queryLengths[i]);
    }
    return record_input_error(at, records, config.k, longest);
}

EDLIB_API int edlibB200AlignRecords(const char* const* queries, const int* queryLengths, int numQueries,
                                    const char* const* records, const int* recordLengths, int numRecords,
                                    const EdlibAlignConfig config, int bothStrands, EdlibAlignResult* results,
                                    int* recordsOut, unsigned char* strandsOut) {
    std::lock_guard<std::mutex> lock(g_mu);
    eb::Engine* e = engine_locked();
    if (!e) {  // no usable device: there is no CPU path
        if (results && numQueries > 0) eb::fail_results(results, numQueries);
        return EDLIB_STATUS_ERROR;
    }
    t_lastEngine = e;
    RecordArgs ra{records, recordLengths, numRecords, 0};
    const std::string bad = align_records_error(queries, queryLengths, numQueries, &ra, config, bothStrands, results,
                                                recordsOut, strandsOut);
    if (!bad.empty()) {
        e->lastError = bad;
        if (results && numQueries > 0) eb::fail_results(results, numQueries);
        return EDLIB_STATUS_ERROR;
    }
    if (numQueries == 0) return EDLIB_STATUS_OK;
    // one target laid out from the records: its length, no host pointer
    int targetLength = (ra.n - 1) * ra.gap;
    for (int r = 0; r < ra.n; ++r) targetLength += ra.lengths[r];
    const std::vector<const char*> targets((size_t)numQueries, nullptr);
    const std::vector<int> targetLengths((size_t)numQueries, targetLength);
    eb::BatchInput in{queries, queryLengths, targets.data(), targetLengths.data(), numQueries, config};
    in.strands = bothStrands != 0;
    in.records = ra.records;
    in.recordLengths = ra.lengths;
    in.numRecords = ra.n;
    in.recordGap = ra.gap;
    in.bestRecord = true;
    return e->align_batch(in, results, in.strands ? strandsOut : nullptr, recordsOut);
}

EDLIB_API void edlibB200LastStats(EdlibB200Stats* s) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (!s) return;
    memset(s, 0, sizeof(*s));
    if (!g_engine || !engine_locked()) return;
    copy_stats(t_lastEngine ? t_lastEngine : g_engine, s);  // the engine this thread's last call ran on
}

EDLIB_API int edlibB200LastKernelReport(char* buf, int bufLen) {
    std::lock_guard<std::mutex> lock(g_mu);
    if (!buf || bufLen <= 0) return 0;
    eb::Engine* e = t_lastEngine ? t_lastEngine : g_engine;
    if (e && engine_locked()) e->finish_stats();
    const std::string r = e ? e->stats.kernelReport : std::string();
    const int n = (int)std::min<size_t>(r.size(), (size_t)bufLen - 1);
    memcpy(buf, r.data(), (size_t)n);
    buf[n] = 0;
    return (int)r.size();
}

}  // extern "C"
