/*
 * edlib_b200.h -- engine-specific additions to the edlib C ABI (plain C, no CUDA or torch
 * types).  Nothing here exists in the reference; the reference-facing surface is edlib.h.
 *
 * The staged calls split edlibAlignBatch() into its three phases so that a caller (bench.py,
 * a multi-GPU driver running one process per device) can keep a batch resident in HBM and
 * time the device work alone:
 *
 *     b = edlibB200BatchPrepare(...)    pack + upload + alphabet/encoding kernels
 *     edlibB200BatchCompute(b, &st)     every DP kernel; may be repeated on the same batch
 *     edlibB200BatchResults(b, res)     malloc'd EdlibAlignResult per pair (as edlibAlignBatch)
 *     edlibB200BatchFree(b)
 *
 * All calls use the CUDA device that is current for the calling thread at the first call
 * (cudaSetDevice / torch.cuda.set_device before it); one process drives one GPU.
 */
#ifndef EDLIB_B200_H
#define EDLIB_B200_H

#include "edlib.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct EdlibB200Batch EdlibB200Batch; /* opaque */

typedef struct {
    double kernelMs;      /* device time of all kernel launches of the last compute (CUDA events) */
    double k1Ms;          /* ... of the lane-per-alignment sweep kernel alone */
    int launches;         /* kernel launches of the last compute */
    int filterWindows;     /* window sweeps planned by the candidate filter (all stages) */
    long long h2dBytes;   /* host->device bytes since the batch was prepared */
    long long d2hBytes;   /* device->host bytes */
    long long k1Cells;    /* nominal DP cells (sum queryLength*targetLength) swept by that kernel */
    long long wCells;     /* nominal DP cells of the distance pass swept by the warp kernel */
    long long filterDecided;  /* alignments settled by the candidate filter (prefix sweep + window) */
    long long filterFallback; /* alignments the filter could not decide (took the plain full sweep) */
} EdlibB200Stats;

/* Selects the CUDA device this process will use; call before any other entry point (one
 * process drives one GPU).  Returns EDLIB_STATUS_OK, or EDLIB_STATUS_ERROR if the engine was
 * already initialised on another device or the device does not exist. */
EDLIB_API int edlibB200SetDevice(int device);

/* NUMA node the selected device hangs off (-1: unknown).  Host buffers a caller hands to edlibAlignBatch travel fastest
 * when they live on that node (page-locked buffers are read by the device directly, see INTEGRATION.md). */
EDLIB_API int edlibB200DeviceNumaNode(void);

/* Optional, for callers that receive millions of results per call: every result owns malloc'd arrays (the reference's
 * ownership rule), and glibc by default hands freed heap memory back to the kernel, so each batch pays the page faults
 * of tens of megabytes of fresh heap again -- serialised across the threads that build the results.  This call tells the
 * allocator to keep freed memory (mallopt M_TRIM_THRESHOLD / M_TOP_PAD); it changes nothing but the process's resident
 * set.  Returns EDLIB_STATUS_OK when the allocator took the settings. */
EDLIB_API int edlibB200TuneHostAllocator(void);

/* free() the arrays of `n` results at once (same effect as n edlibFreeAlignResult calls). */
EDLIB_API void edlibB200FreeResults(EdlibAlignResult* results, int n);

/* 1 when a CUDA device and the kernels are usable, else 0 (then every align call fails). */
EDLIB_API int edlibB200Available(void);

/* Text of the last engine error on this process (valid until the next call). */
EDLIB_API const char* edlibB200LastError(void);

EDLIB_API EdlibB200Batch* edlibB200BatchPrepare(const char* const* queries, const int* queryLengths,
                                                const char* const* targets, const int* targetLengths,
                                                int numPairs, const EdlibAlignConfig config);
EDLIB_API int edlibB200BatchCompute(EdlibB200Batch* batch, EdlibB200Stats* statsOut);
EDLIB_API int edlibB200BatchResults(EdlibB200Batch* batch, EdlibAlignResult* results);
EDLIB_API void edlibB200BatchFree(EdlibB200Batch* batch);

/* Both strands of DNA reads in one call.  For each pair i, queries[i] and its reverse complement rc(queries[i]) are
 * aligned to targets[i]: rc reverses the query and complements every byte with a fixed table (A<->T, C<->G, R<->Y,
 * K<->M, B<->V, D<->H, upper and lower case; every other byte, N / S / W and non-letters included, is its own
 * complement).  results[i] is the result of edlibAlign(rc(queries[i]), targets[i], config), with strands[i] = 1, when
 * that one has a distance and the forward one has a larger distance or none; otherwise it is the result of
 * edlibAlign(queries[i], targets[i], config), with strands[i] = 0 -- ties and "neither strand within k" report the
 * forward strand.  Every field is that of the chosen strand (the alignment of the reverse strand is that of
 * rc(queries[i])).  Any mode, task, k and additional equalities; for HW read sets over a long target, the distance the
 * seed filter finds on one strand bounds the search on the other.  Returns EDLIB_STATUS_OK / EDLIB_STATUS_ERROR. */
EDLIB_API int edlibB200AlignBatchStrands(const char* const* queries, const int* queryLengths,
                                         const char* const* targets, const int* targetLengths, int numPairs,
                                         const EdlibAlignConfig config, EdlibAlignResult* results, unsigned char* strands);
/* Staged form of edlibB200AlignBatchStrands: the reads are uploaded once, their reverse complements are made on the
 * device.  edlibB200BatchCompute / edlibB200BatchResults then work as for any batch and give numPairs results. */
EDLIB_API EdlibB200Batch* edlibB200BatchPrepareStrands(const char* const* queries, const int* queryLengths,
                                                       const char* const* targets, const int* targetLengths,
                                                       int numPairs, const EdlibAlignConfig config);
/* strands[i] (numPairs bytes) of the last edlibB200BatchCompute of a strand batch; EDLIB_STATUS_ERROR for a batch not
 * prepared with edlibB200BatchPrepareStrands, or one that was not computed. */
EDLIB_API int edlibB200BatchStrands(EdlibB200Batch* batch, unsigned char* strands);

/* Every end location of each query within k edits of one shared target (HW mode).
 *
 * D(c), for a query q of m symbols and the target T of n symbols, is the HW last row at column c: the least edit
 * distance between q and any substring of T that ends at c, the empty substring included.  The hits of q are all pairs
 * (c, D(c)) with 0 <= c < n and D(c) <= k, in ascending c (column -1 is never reported; with k >= m every column is a
 * hit).  So when edlibAlign(q, T, HW, k) gives a distance d >= 0, the least hit score is d and the columns scoring d
 * are its endLocations (without a leading -1); when it gives -1 there are no hits.
 *
 * bothStrands != 0: rc(q) (the complement table of edlibB200AlignBatchStrands) is searched as well, with no pruning
 * between the strands; its hits follow the forward ones and carry strand 1.
 *
 * counts[i] is the exact number of hits of query i over the searched strands; the first min(counts[i],
 * maxHitsPerQuery) of them, in the order above, are stored at [offsets[i], offsets[i+1]) of columns / scores /
 * strands (maxHitsPerQuery = 0: counts only).  Memory for stored hits is bounded by their number.
 *
 * Accepted: 1 <= queryLengths[i] <= 256, targetLength >= 1, config.k >= 0, config.mode == EDLIB_MODE_HW,
 * config.task == EDLIB_TASK_DISTANCE, any additional equalities, maxHitsPerQuery >= 0.  Anything else returns
 * EDLIB_STATUS_ERROR with a message in edlibB200LastError and *hits left empty; on success the arrays are malloc'd
 * and edlibB200FreeHits releases them.  edlibB200LastStats: filterWindows = seed windows planned, filterDecided =
 * query-strands whose hits came from seed windows, filterFallback = query-strands swept over the whole target. */
typedef struct {
    int numQueries;
    long long* counts;      /* numQueries: hits found per query (all searched strands), may exceed what is stored */
    long long* offsets;     /* numQueries + 1: stored hits of query i are [offsets[i], offsets[i+1]) */
    int* columns;           /* end column of each stored hit */
    int* scores;            /* D(column) */
    unsigned char* strands; /* 0 / 1 per stored hit; NULL unless both strands were searched */
} EdlibB200Hits;

EDLIB_API int edlibB200FindHits(const char* const* queries, const int* queryLengths, int numQueries,
                                const char* target, int targetLength, const EdlibAlignConfig config,
                                int bothStrands, long long maxHitsPerQuery, EdlibB200Hits* hits);
/* Frees the arrays of edlibB200FindHits and clears the struct. */
EDLIB_API void edlibB200FreeHits(EdlibB200Hits* hits);

/* The hits of edlibB200FindHits, with the start location and the alignment path of every stored hit.
 *
 * `hits` is exactly what edlibB200FindHits returns for the same arguments.  For a stored hit (c, s) of query q (rc(q)
 * for a strand-1 hit) of m symbols, each hit taken on its own by the rules edlibAlign applies to its best hits:
 *   start  (config.task EDLIB_TASK_LOC or EDLIB_TASK_PATH): the smallest st with ed(q, T[st..c]) = s, i.e. c minus the
 *          last column of score s of the SHW alignment of rev(q) to rev(T[c-m-s+1..c]) (clipped at column 0);
 *   script (EDLIB_TASK_PATH): the EDLIB_EDOP_* codes that edlibAlign(q, T[start..c], NW, k = -1, PATH) returns; its
 *          cost is s.
 * So the starts of the columns of a query's least score are edlibAlign(q, T, HW, k, LOC)'s startLocations, and the
 * script of the first of them is edlibAlign(q, T, HW, k, PATH)'s alignment.  starts / scripts follow the stored hits
 * in their order: starts[h] and alignments[alignmentOffsets[h] .. alignmentOffsets[h+1]) belong to hit h; a script
 * turns into a CIGAR with edlibAlignmentToCigar.
 *
 * Accepted: everything edlibB200FindHits accepts, with config.task EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC or
 * EDLIB_TASK_PATH.  Anything else returns EDLIB_STATUS_ERROR with a message in edlibB200LastError (starting with
 * "edlibB200FindHitAlignments:" for invalid input) and *out left empty; on success the arrays are malloc'd and
 * edlibB200FreeHitAlignments releases them.  edlibB200LastStats reports what edlibB200FindHits reports; its kernel
 * time and launch count include the start-location and path sweeps. */
typedef struct {
    EdlibB200Hits hits;           /* exactly what edlibB200FindHits returns for the same arguments */
    int* starts;                  /* one per stored hit (task LOC / PATH), else NULL */
    long long* alignmentOffsets;  /* task PATH: stored + 1 entries; hit h's script is alignments[off[h] .. off[h+1]) */
    unsigned char* alignments;    /* EDLIB_EDOP_* codes, as EdlibAlignResult.alignment; NULL unless PATH */
} EdlibB200HitAlignments;

EDLIB_API int edlibB200FindHitAlignments(const char* const* queries, const int* queryLengths, int numQueries,
                                         const char* target, int targetLength, const EdlibAlignConfig config,
                                         int bothStrands, long long maxHitsPerQuery, EdlibB200HitAlignments* out);
/* Frees the arrays of edlibB200FindHitAlignments and clears the struct. */
EDLIB_API void edlibB200FreeHitAlignments(EdlibB200HitAlignments* out);

/* The largest multi-record target of edlibB200FindRecordHits, in symbols: the records plus the separators between
 * them (numRecords - 1 runs of min(config.k, longest query) + 1 symbols).  A larger reference is split by the caller
 * over several calls. */
#define EDLIB_B200_MAX_RECORD_TARGET 0x7ffff000

/* Every hit of each query over a reference of several records (chromosomes, plasmids, contigs) in one call.
 *
 * The hits of query q on record r are exactly those of edlibB200FindHitAlignments(q, records[r], ..., bothStrands = 0):
 * column, score, start and script all count from the start of record r, no hit spans two records, and no column outside
 * a record is reported.  With bothStrands != 0 the hits of rc(q) (the complement table of edlibB200AlignBatchStrands)
 * follow, with strand 1.  Within a query, hits are ordered by strand (forward first), then by record index, then by
 * column; counts[i] is exact and the first maxHitsPerQuery hits in that order are stored.  records[h] is the record of
 * stored hit h; the other arrays are those of EdlibB200HitAlignments, for config.task EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC
 * or EDLIB_TASK_PATH.
 *
 * Accepted: the queries and config that edlibB200FindHits accepts (the task may also be LOC or PATH), numRecords >= 1,
 * every records[r] non-NULL with recordLengths[r] >= 1, and records plus separators of at most
 * EDLIB_B200_MAX_RECORD_TARGET symbols (checked before any record byte is read).  The records are laid out in one
 * target, separated by a code that neither the queries nor the records use: when they use all 256 codes (after
 * transitive equalities are merged) and there is more than one record, no code is left and the call is refused.
 * Anything else returns EDLIB_STATUS_ERROR with a message in edlibB200LastError (starting with
 * "edlibB200FindRecordHits:" for invalid input) and *out left empty; on success the arrays are malloc'd and
 * edlibB200FreeRecordHits releases them.  edlibB200LastStats reports what edlibB200FindHits reports. */
typedef struct {
    EdlibB200HitAlignments aln;  /* as edlibB200FindHitAlignments; columns and starts count from the start of the hit's record */
    int* records;                /* record index of each stored hit */
} EdlibB200RecordHits;

EDLIB_API int edlibB200FindRecordHits(const char* const* queries, const int* queryLengths, int numQueries,
                                      const char* const* records, const int* recordLengths, int numRecords,
                                      const EdlibAlignConfig config, int bothStrands, long long maxHitsPerQuery,
                                      EdlibB200RecordHits* out);
/* Frees the arrays of edlibB200FindRecordHits and clears the struct. */
EDLIB_API void edlibB200FreeRecordHits(EdlibB200RecordHits* out);

/* Every hit of each query in its own target: pair i searches queries[i] in targets[i] only (a read's candidate region,
 * its amplicon, the locus a guide is assigned to), all pairs in one call.
 *
 * For a pair with targetLengths[i] >= 1, everything of entry i (counts[i], the stored hits at [offsets[i],
 * offsets[i+1]), their columns, scores, strands, starts and scripts) is exactly what edlibB200FindHitAlignments(
 * &queries[i], &queryLengths[i], 1, targets[i], targetLengths[i], config, bothStrands, maxHitsPerPair, ...) gives for
 * its one query; columns and starts count from the start of targets[i].  A pair with targetLengths[i] == 0 has no
 * hits (columns run over 0 <= c < n), and its targets[i] may be NULL.  The cap and the strand order apply per pair.
 * hits.numQueries = numPairs; edlibB200FreeHitAlignments releases the result.
 *
 * Pairs that share a target (the same pointer and length) are one target group: a group of many pairs is searched as
 * edlibB200FindHitAlignments searches its target, the other pairs by a sweep of each pair over its own target.  A call
 * whose pairs all share one target runs exactly as edlibB200FindHitAlignments over that target.
 *
 * Accepted: numPairs >= 0, and per pair what edlibB200FindHitAlignments accepts: 1 <= queryLengths[i] <= 256,
 * config.k >= 0, config.mode == EDLIB_MODE_HW, config.task EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC or EDLIB_TASK_PATH, any
 * additional equalities, maxHitsPerPair >= 0; targetLengths[i] >= 0 with targets[i] non-NULL when targetLengths[i] > 0.
 * Anything else returns EDLIB_STATUS_ERROR with a message in edlibB200LastError (starting with "edlibB200FindPairHits:"
 * for invalid input) and *out left empty.  edlibB200LastStats: filterWindows = seed windows planned, filterDecided =
 * pair-strands whose hits came from seed windows, filterFallback = pair-strands swept over their whole target (a group's
 * or their own); kernel time and launches include every sweep. */
EDLIB_API int edlibB200FindPairHits(const char* const* queries, const int* queryLengths,
                                    const char* const* targets, const int* targetLengths, int numPairs,
                                    const EdlibAlignConfig config, int bothStrands, long long maxHitsPerPair,
                                    EdlibB200HitAlignments* out);

/* Each query aligned (HW mode) against a reference of several records in one call, with the result of its best record.
 *
 * For query q let A(r) = edlibAlign(q, records[r], config).  The best record r* is the lowest index among the records
 * of least distance, where "none within k" (-1) counts as larger than any distance; so when no record has an alignment
 * within k, and for an empty query, r* = 0.  results[i] is A(r*) in every field: alphabetLength counts the distinct
 * bytes of q and records[r*] only, and endLocations (with the reference's leading -1 where it gives one),
 * startLocations and alignment count from the start of records[r*].  recordsOut[i] = r*.
 *
 * bothStrands != 0: q and rc(q) (the complement table of edlibB200AlignBatchStrands) each get their best record, and
 * the strand is chosen by the rule of edlibB200AlignBatchStrands (the reverse strand only when strictly better);
 * strandsOut[i] receives it, and a reverse result is edlibAlign(rc(q), records[r*], config).
 *
 * Accepted: config.mode EDLIB_MODE_HW with any task, k (-1 included) and additional equalities; queries of any length
 * (0 included); numRecords >= 1, every records[r] non-NULL with recordLengths[r] >= 1; results and recordsOut (and
 * strandsOut with bothStrands) of numQueries entries.  The records are laid out in one target, each but the last
 * followed by g separator symbols, g = min(k, longest query) + 1 (longest query + 1 for k < 0); records plus
 * separators must not exceed EDLIB_B200_MAX_RECORD_TARGET symbols, which is checked before any record byte is read.
 * As for edlibB200FindRecordHits, a call of several records whose queries and records use all 256 codes is refused.
 * One record needs no separator: the results are those of edlibAlignBatch against it.  Errors return
 * EDLIB_STATUS_ERROR with a message in edlibB200LastError (starting with "edlibB200AlignRecords:" for invalid input)
 * and no arrays allocated; results are freed as those of edlibAlignBatch.  edlibB200LastStats reports the distance
 * pass, as for edlibAlignBatch. */
EDLIB_API int edlibB200AlignRecords(const char* const* queries, const int* queryLengths, int numQueries,
                                    const char* const* records, const int* recordLengths, int numRecords,
                                    const EdlibAlignConfig config, int bothStrands,
                                    EdlibAlignResult* results, int* recordsOut, unsigned char* strandsOut);

/* A target kept resident on the device.  edlibAlignBatch calls of read sets (HW, short queries, plain equality) whose
 * targets[i] all equal (target, targetLength) of a live handle skip the target's upload, its encoding and the build of
 * its seed index: a caller that aligns many batches to one genome pays them once.  The bytes at `target` must not
 * change while the handle lives; results are identical with and without a handle.  Returns NULL on failure. */
typedef struct EdlibB200Target EdlibB200Target;
EDLIB_API EdlibB200Target* edlibB200TargetPrepare(const char* target, int targetLength);
EDLIB_API void edlibB200TargetFree(EdlibB200Target* target);

/* edlibAlignmentToCigar (edlib.h) for n results at once, on the engine's host threads: cigars[i] receives a
 * malloc'd C string (caller frees each with free()), or NULL where results[i] holds no alignment.  Returns
 * EDLIB_STATUS_OK, or EDLIB_STATUS_ERROR on a bad format / operation code (then every cigars[i] is NULL). */
EDLIB_API int edlibB200AlignmentsToCigar(const EdlibAlignResult* results, int n, EdlibCigarFormat cigarFormat, char** cigars);

/* free() n strings of edlibB200AlignmentsToCigar at once (on the engine's host threads, like edlibB200FreeResults). */
EDLIB_API void edlibB200FreeCigars(char** cigars, int n);

/* Stats of the most recent edlibAlign / edlibAlignBatch / BatchCompute on this process. */
EDLIB_API void edlibB200LastStats(EdlibB200Stats* statsOut);

/* Device time per kernel of the most recent compute, as text "name:milliseconds:launches;..." written
 * to buf (NUL-terminated, truncated to bufLen); returns the full length. */
EDLIB_API int edlibB200LastKernelReport(char* buf, int bufLen);

#ifdef __cplusplus
}
#endif
#endif /* EDLIB_B200_H */
