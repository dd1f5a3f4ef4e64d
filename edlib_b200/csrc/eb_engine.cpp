// eb_engine.cpp -- batch planner / orchestrator (see eb_engine.h).
//
// Pipeline of one batch (reference driver: edlibAlign, ref edlib.cpp:146-301):
//   prepare : pack + upload raw bytes, byte-presence sets on the device (-> alphabetLength per
//             pair, ref cpp:1417-1462), dense code map, in-place encoding, equality table
//             (ref cpp:63-94)
//   compute : distance + end locations  (K1 lane-per-alignment for groups that share a target,
//             W warp-per-alignment otherwise; ref cpp:199-225)
//             start locations           (reversed SHW sweeps, ref cpp:228-272)
//             alignment path            (stored-matrix NW sweep + traceback kernel inside the
//                                        reference's 1 MiB rule, ref cpp:276-289, 1161-1213)
//   materialize : malloc'd arrays per result (ownership as ref edlib.h:177,186,205)
//
// edlibAlignBatch() on the usual large batch (reads, HW, one shared target) does not run these phases one
// after the other: Engine::align_streamed cuts the reads into slices and overlaps packing + upload of slice
// i+1 with the kernels of slice i and with the result structs of slice i-1 (second half of this file).
#include "eb_engine_internal.h"

#include <sched.h>

namespace eb {

static int env_int(const char* name, int dflt) {
    const char* s = getenv(name);
    return (s && *s) ? atoi(s) : dflt;
}

// "0-3,8,10-11" -> cpu numbers
static std::vector<int> parse_cpulist(const char* path) {
    std::vector<int> cpus;
    FILE* f = fopen(path, "r");
    if (!f) return cpus;
    char buf[4096];
    if (fgets(buf, sizeof(buf), f)) {
        for (char* tok = strtok(buf, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int a = 0, b = 0;
            const int got = sscanf(tok, "%d-%d", &a, &b);
            if (got == 1) b = a;
            if (got >= 1)
                for (int c = a; c <= b && c < 4096; ++c) cpus.push_back(c);
        }
    }
    fclose(f);
    return cpus;
}

void HostPool::bind_worker() {
    const std::vector<int>& cpus = worker_cpus();
    if (cpus.empty()) return;
    cpu_set_t allowed, want;
    CPU_ZERO(&allowed);
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return;
    int n = 0;
    for (int c : cpus)
        if (c < CPU_SETSIZE && CPU_ISSET(c, &allowed)) {
            CPU_SET(c, &want);
            ++n;
        }
    if (n > 0) sched_setaffinity(0, sizeof(want), &want);  // best effort
}

// parallel_ranges for the translation units that do not see the pool (eb_capi.cpp)
void host_parallel_ranges(size_t n, size_t grain, const std::function<void(size_t, size_t)>& fn) {
    parallel_ranges(n, grain, [&](size_t lo, size_t hi) { fn(lo, hi); });
}

// The host workers of the engine run next to the GPU (EDLIB_B200_NUMA=0 leaves them where the caller runs); the
// calling thread itself is never moved.
Engine::Engine(Backend* be) : be_(be) {
    if (env_int("EDLIB_B200_NUMA", 1) == 0) return;
    const int node = be->numa_node();
    if (node < 0) return;
    char path[128];
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    std::vector<int> cpus = parse_cpulist(path);
    if (!cpus.empty() && HostPool::worker_cpus().empty()) HostPool::worker_cpus() = cpus;
}

EngineTunables::EngineTunables() {
    k1MinGroup = env_int("EDLIB_B200_K1_MIN_GROUP", k1MinGroup);
    k1MinChunk = env_int("EDLIB_B200_K1_MIN_CHUNK", k1MinChunk);
    ovfCap = env_int("EDLIB_B200_OVF_CAP", ovfCap);
    filterK0 = env_int("EDLIB_B200_FILTER_K0", filterK0);
    filterK1 = env_int("EDLIB_B200_FILTER_K1", filterK1);
    packParallelBytes = (size_t)env_int("EDLIB_B200_PACK_PARALLEL_KB", (int)(packParallelBytes >> 10)) << 10;
    filterSeedK = env_int("EDLIB_B200_FILTER_SEED_K", filterSeedK);
    filterSeedBucket = env_int("EDLIB_B200_FILTER_SEED_BUCKET", filterSeedBucket);
    filterSeedSlack = env_int("EDLIB_B200_FILTER_SEED_SLACK", filterSeedSlack);
    filterMinLevelReads = env_int("EDLIB_B200_FILTER_MIN_LEVEL_READS", filterMinLevelReads);
    tinySweepReads = env_int("EDLIB_B200_TINY_SWEEP_READS", tinySweepReads);
    filterSeedLevels = std::min(SEED_LEVELS, env_int("EDLIB_B200_FILTER_SEED_LEVELS", filterSeedLevels));
    filterMaxWindows = env_int("EDLIB_B200_FILTER_MAX_WINDOWS", filterMaxWindows);
    filterMinLen = env_int("EDLIB_B200_FILTER_MIN_LEN", filterMinLen);
    filterSpread = env_int("EDLIB_B200_FILTER_SPREAD", filterSpread);
    filterMinTarget = env_int("EDLIB_B200_FILTER_MIN_TARGET", filterMinTarget);
    filterSkipRepeats = env_int("EDLIB_B200_FILTER_SKIP_REPEATS", filterSkipRepeats);
    bandKernel = env_int("EDLIB_B200_BAND_KERNEL", bandKernel);
    collapseEqualities = env_int("EDLIB_B200_COLLAPSE_EQUALITIES", collapseEqualities);
    directUpload = env_int("EDLIB_B200_DIRECT_UPLOAD", directUpload);
    streamSlices = std::max(1, env_int("EDLIB_B200_STREAM_SLICES", streamSlices));
    directMinBytes = (size_t)env_int("EDLIB_B200_DIRECT_MIN_KB", (int)(directMinBytes >> 10)) << 10;
    deviceStage = env_int("EDLIB_B200_DEVICE_STAGE", deviceStage);
    windowCheckAfter = env_int("EDLIB_B200_WINDOW_CHECK", windowCheckAfter);
    longHwMinTarget = env_int("EDLIB_B200_LONG_HW_MIN_TARGET", longHwMinTarget);
    longSeedMaxK = env_int("EDLIB_B200_LONG_SEED_MAX_K", longSeedMaxK);
    devSliceReads = std::max(64, env_int("EDLIB_B200_SLICE_READS", devSliceReads));
    streamMinPairs = env_int("EDLIB_B200_STREAM_MIN_PAIRS", streamMinPairs);
    hitRunReads = std::max(1, env_int("EDLIB_B200_HIT_RUN_READS", hitRunReads));
    const int sliceMb = env_int("EDLIB_B200_SLICE_MB", 0);
    if (sliceMb > 0) sliceBytes = (size_t)sliceMb << 20;
    if (sliceMb > 0) pathSliceBytes = (size_t)sliceMb << 20;
}

// dense codes in ascending byte order for the bytes of `present`; every other byte maps to `other`
static int code_map(const uint32_t (&present)[8], uint8_t (&map)[256], int other) {
    int ncodes = 0;
    for (int b = 0; b < 256; ++b) ncodes += (present[b >> 5] >> (b & 31)) & 1u;
    int next = 0;
    for (int b = 0; b < 256; ++b) {
        if (present[b >> 5] >> (b & 31) & 1u) map[b] = (uint8_t)next++;
        else map[b] = (uint8_t)(other < 0 ? 0 : std::min(other, 255));
    }
    return ncodes;
}

// Encodes a target by its own alphabet, in place: `raw` holds its n bytes on the device, zero-padded to round_up(n, 16).
// Presence set on the device, code map on the host (a byte the target lacks gets the extra code, which matches
// nothing), encoding on the device.  Returns tc.ncodes.
static int encode_target(Backend* be, uint8_t* raw, int n, TargetCodes& tc) {
    std::vector<MaskItem> items;
    for (int s0 = 0; s0 < n; s0 += 65536) items.push_back(MaskItem{(uint64_t)s0, std::min(65536, n - s0), 0});
    DevBuf<MaskItem> dItems(be, items.size());
    dItems.upload(items.data(), items.size());
    tc.dMask.alloc(be, 8);
    be->zero(tc.dMask.p, 8 * sizeof(uint32_t));
    MaskParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.raw = raw;
    mp.items = dItems.p;
    mp.numItems = (int)items.size();
    mp.masks = tc.dMask.p;
    mp.unionSet = -1;
    be->launch_mask(mp);
    uint32_t present[8];
    be->d2h(present, tc.dMask.p, sizeof(present));
    int distinct = 0;
    for (int b = 0; b < 256; ++b) distinct += (present[b >> 5] >> (b & 31)) & 1u;
    uint8_t map[256];
    code_map(present, map, distinct);
    tc.dMap.alloc(be, 256);
    tc.dMap.upload(map, 256);
    EncodeParams ep{raw, (uint64_t)round_up((size_t)n, 16), tc.dMap.p};
    be->launch_encode(ep);
    // no spare code when every byte value occurs in the target: then no read byte is foreign
    tc.ncodes = distinct >= 256 ? 256 : std::max(1, std::min(distinct, 255));
    return tc.ncodes;
}

// The batch object for `in`, with nothing of an earlier batch left in it (staged API: results before compute find
// none) and the per-pair vectors sized for the caller's pairs.  The spare object of the last batch is reused: its host
// vectors keep their pages.  On failure the object stays the spare one.
Prepared* Engine::take_prepared(const BatchInput& in) {
    if (!spare_) spare_ = new Prepared();
    Prepared* p = spare_;
    p->bind(be_);
    p->tg.clear();
    p->hasEq = false;
    p->ncodes = 0;
    p->recOff.clear();
    p->dRecOff.reset();
    p->recGap = 0;
    p->sep = -1;
    p->bestRecord = in.bestRecord;
    p->record.clear();
    p->dMasks.reset();
    p->computed = false;
    p->classified = false;
    p->groups.clear();
    p->wPairsBase.clear();
    p->otherPairs.clear();
    p->ed.clear();
    p->endStart.clear();
    p->endCount.clear();
    p->endPool.clear();
    p->startPool.clear();
    p->alnStart.clear();
    p->alnLen.clear();
    p->alnPool.clear();
    p->N = in.numPairs;
    p->cfg = in.config;
    p->strands = in.strands;
    p->strand.clear();
    p->mode = (in.config.mode == EDLIB_MODE_SHW) ? MODE_SHW : (in.config.mode == EDLIB_MODE_HW) ? MODE_HW : MODE_NW;
    p->qlen.resize(p->N);
    p->tlen.resize(p->N);
    p->tidx.resize(p->N);
    p->qoff.resize(p->N);
    spare_ = nullptr;
    return p;
}

// After a failure: nothing may still run on the device (staging blocks go back to the cache, buffers to the pool) and
// no mark stays live.  Never throws.
void Engine::quiesce() {
    try {
        be_->sync_all();
        be_->release_marks();
    } catch (...) {
    }
}

// ---------------------------------------------------------------------------------------------
// prepare
// ---------------------------------------------------------------------------------------------
Prepared* Engine::prepare(const BatchInput& in) {
    Backend* be = be_;
    Trace trace;
    Prepared* p = take_prepared(in);
    try {
        int N = p->N;  // the caller's pairs; a strand batch doubles it after packing
        if (parallel_any((size_t)N, 65536, [&](size_t i) {
                p->qlen[i] = in.queryLengths[i];
                p->tlen[i] = in.targetLengths[i];
                return p->qlen[i] < 0 || p->tlen[i] < 0;
            }))
            throw std::runtime_error("negative sequence length");

        // identical (pointer, length) targets are uploaded and encoded once: open-addressing table over the pairs
        // (no node allocations: a batch of 100,000 pairs with their own targets spends ~1 ms here)
        struct Key {
            const char* ptr;
            int len;
            bool operator==(const Key& o) const { return ptr == o.ptr && len == o.len; }
        };
        // the usual batch shape (reads over one shared target), checked in parallel
        const bool oneTarget = N >= 131072 && !parallel_any((size_t)N, 65536, [&](size_t i) {
            return in.targets[i] != in.targets[0] || in.targetLengths[i] != in.targetLengths[0];
        });
        if (oneTarget) {
            p->tg.push_back(Target{in.targets[0], in.targetLengths[0], 0});
            parallel_ranges((size_t)N, 65536, [&](size_t lo, size_t hi) {
                for (size_t i = lo; i < hi; ++i) p->tidx[i] = 0;
            });
        } else {
            size_t cap = 64;
            while (cap < 2 * (size_t)N) cap *= 2;
            std::vector<int>& table = scratch.targetTable;  // slot -> index into p->tg, -1: free
            table.assign(cap, -1);
            Key lastKey{nullptr, -1};
            int lastIdx = -1;
            for (int i = 0; i < N; ++i) {
                const Key k{in.targets[i], in.targetLengths[i]};
                if (!(k == lastKey)) {  // neighbours usually share their target
                    uint64_t h = (uint64_t)(uintptr_t)k.ptr * 0x9E3779B97F4A7C15ull + (uint64_t)(uint32_t)k.len * 0xC2B2AE3D27D4EB4Full;
                    h ^= h >> 29;
                    size_t slot = (size_t)h & (cap - 1);
                    for (;;) {
                        const int t = table[slot];
                        if (t < 0) {
                            table[slot] = (int)p->tg.size();
                            lastIdx = (int)p->tg.size();
                            p->tg.push_back(Target{k.ptr, k.len, 0});
                            break;
                        }
                        if (p->tg[(size_t)t].ptr == k.ptr && p->tg[(size_t)t].len == k.len) {
                            lastIdx = t;
                            break;
                        }
                        slot = (slot + 1) & (cap - 1);
                    }
                    lastKey = k;
                }
                p->tidx[i] = lastIdx;
            }
        }
        const int T = (int)p->tg.size();
        trace.mark("prepare: lengths + distinct targets");
        // a record target: record r at columns recOff[r] .., then recGap separator columns (eb_common.h: RecordParams)
        const int numRec = in.numRecords;
        if (numRec > 0) {
            if (T != 1) throw std::runtime_error("internal: a record target is the one target of its batch");
            p->recGap = in.recordGap;
            p->recOff.assign((size_t)numRec + 1, 0);
            for (int r = 0; r < numRec; ++r) p->recOff[(size_t)r + 1] = p->recOff[(size_t)r] + in.recordLengths[r] + in.recordGap;
            if (p->recOff[(size_t)numRec] - in.recordGap != p->tg[0].len) throw std::runtime_error("internal: record target length");
        }

        // pack: queries back to back, then every target 16-aligned with >= 16 bytes of slack
        size_t total = 0;
        for (int i = 0; i < N; ++i) {
            p->qoff[i] = total;
            total += (size_t)p->qlen[i];
        }
        const size_t readBytes = total;
        total = round_up(total, 16);
        for (int t = 0; t < T; ++t) {
            p->tg[t].off = total;
            total += round_up((size_t)p->tg[t].len, 16) + 16;
        }
        total += 16;
        // strand batches: the reverse complements of the reads follow on the device only (written there, never uploaded)
        const size_t rcBase = total;
        const size_t devTotal = in.strands ? rcBase + round_up(readBytes, 16) + 16 : total;
        HostBuf<uint8_t> stageBuf(be, total);  // released on every path out of this function
        uint8_t* stage = stageBuf.p;
        p->dSeq.alloc(be, devTotal);
        // the small per-pair arrays go first: they would otherwise queue behind the sequences
        auto upload_pair_arrays = [&]() {
            p->dQoff.alloc(be, N);
            p->dQoff.upload(p->qoff.data(), N);
            p->dQlen.alloc(be, N);
            p->dQlen.upload(p->qlen.data(), N);
        };
        if (!in.strands) upload_pair_arrays();
        trace.mark("prepare: offsets + buffers");
        {
            // Pure memcpy work, split by bytes over a few host threads when the batch is large: items
            // 0..N-1 are the queries, N..N+T-1 the distinct targets.  Every thread uploads its own byte
            // range as soon as it is packed, so the host->device copy overlaps the packing.
            const size_t qBytes = N ? (size_t)(p->qoff[N - 1] + (uint64_t)p->qlen[N - 1]) : 0;
            // Queries that lie back to back in PINNED caller memory (a read array the caller allocated page-locked) go
            // to the device straight from there: no staging copy, no host memory traffic besides the DMA itself.
            const bool direct = tun.directUpload && N > 0 && qBytes >= tun.directMinBytes &&
                                !parallel_any((size_t)N, 65536, [&](size_t i) {
                                    return i > 0 && in.queries[i] != in.queries[i - 1] + p->qlen[i - 1];
                                }) &&
                                be->host_pinned(in.queries[0], qBytes);
            if (direct) be->h2d(p->dSeq.p, in.queries[0], qBytes);
            const int firstItem = direct ? N : 0;
            size_t allBytes = direct ? 0 : qBytes;
            for (int t = 0; t < T; ++t) allBytes += (size_t)p->tg[t].len;
            const int nthr = allBytes > tun.packParallelBytes ? (int)HostPool::get().width() : 1;
            auto copy_item = [&](int it) {
                if (it < N) {
                    if (p->qlen[it]) memcpy(stage + p->qoff[it], in.queries[it], (size_t)p->qlen[it]);
                } else if (numRec > 0) {  // the records, zeros in the separators until they are written after the encoding
                    uint8_t* dst = stage + p->tg[0].off;
                    for (int r = 0; r < numRec; ++r) {
                        memcpy(dst + p->recOff[(size_t)r], in.records[r], (size_t)in.recordLengths[r]);
                        if (r + 1 < numRec) memset(dst + p->recOff[(size_t)r + 1] - p->recGap, 0, (size_t)p->recGap);
                    }
                } else {
                    const Target& g = p->tg[it - N];
                    if (g.len) memcpy(stage + g.off, g.ptr, (size_t)g.len);
                }
            };
            auto item_off = [&](int it) -> size_t {  // first staging byte of item `it` (N + T: the end)
                if (it >= N + T) return total;
                return it < N ? (size_t)p->qoff[it] : p->tg[it - N].off;
            };
            // padding first: it lies between the items and travels with the neighbouring byte ranges
            {
                size_t pos = qBytes;
                size_t end = p->tg.empty() ? total : p->tg[0].off;
                memset(stage + pos, 0, end - pos);
                for (int t = 0; t < T; ++t) {
                    const Target& g = p->tg[t];
                    const size_t next = (t + 1 < T) ? p->tg[t + 1].off : total;
                    memset(stage + g.off + g.len, 0, next - g.off - (size_t)g.len);
                }
            }
            const size_t firstByte = direct ? qBytes : 0;  // the staging bytes before this travelled directly
            if (nthr > 1) {
                // contiguous item ranges of roughly equal byte counts
                std::vector<int> cut(nthr + 1, N + T);
                cut[0] = firstItem;
                {
                    size_t tAcc = direct ? 0 : qBytes;  // bytes before target `tt`
                    int tt = 0;
                    for (int c = 1; c < nthr; ++c) {
                        const size_t want = allBytes * c / nthr;
                        if (!direct && want < qBytes) {  // qoff is the running byte count of the queries
                            cut[c] = (int)(std::upper_bound(p->qoff.begin(), p->qoff.end(), (uint64_t)want) - p->qoff.begin());
                        } else {
                            while (tt < T && tAcc + (size_t)p->tg[tt].len <= want) tAcc += (size_t)p->tg[tt++].len;
                            cut[c] = N + tt;
                        }
                        if (cut[c] < cut[c - 1]) cut[c] = cut[c - 1];
                    }
                }
                HostPool::get().run((size_t)nthr, [&](size_t t) {  // exceptions of a task are rethrown by run()
                    for (int it = cut[t]; it < cut[t + 1]; ++it) copy_item(it);
                    const size_t a = t == 0 ? firstByte : item_off(cut[t]), b = item_off(cut[t + 1]);
                    be->bind_thread();  // a pool worker: select the backend's device before the copy
                    if (b > a) be->h2d(p->dSeq.p + a, stage + a, b - a);
                });
            } else {
                for (int it = firstItem; it < N + T; ++it) copy_item(it);
                be->h2d(p->dSeq.p + firstByte, stage + firstByte, total - firstByte);
            }
        }
        trace.mark("prepare: pack");
        stats.h2dBytes += (long long)total;
        if (in.strands) {
            // read i becomes pairs 2i (as uploaded) and 2i+1: its reverse complement, which the presence-set pass writes
            // into the region at rcBase on raw bytes, before alphabet lengths and codes are derived
            const int R = N;
            N = p->N = 2 * R;
            p->qlen.resize(N);
            p->tlen.resize(N);
            p->tidx.resize(N);
            p->qoff.resize(N);
            for (int i = R - 1; i >= 0; --i) {
                const int m = p->qlen[i], n = p->tlen[i], t = p->tidx[i];
                const uint64_t off = p->qoff[i];
                p->qlen[2 * i] = p->qlen[2 * i + 1] = m;
                p->tlen[2 * i] = p->tlen[2 * i + 1] = n;
                p->tidx[2 * i] = p->tidx[2 * i + 1] = t;
                p->qoff[2 * i] = off;
                p->qoff[2 * i + 1] = rcBase + (readBytes - off - (uint64_t)m);  // the region is the reversed read block
            }
            upload_pair_arrays();
            be->zero(p->dSeq.p + rcBase + readBytes, devTotal - rcBase - readBytes);
        }
        // the presence-set pass writes the reverse complements (MaskParams::rc): only the reads as given are work items
        const int qstep = in.strands ? 2 : 1;
        std::vector<int> longQueries;  // beyond one presence-set work item
        for (int i = 0; i < N; i += qstep)
            if (p->qlen[i] > 65536) longQueries.push_back(i);

        // byte-presence sets: one per query, one per distinct target (a record target: one per record), one union for
        // the batch.  Queries are implicit work items of the kernel; explicit ones (at most 65536 bytes each) are only
        // needed for the targets and for the pieces of longer queries.
        std::vector<MaskItem> items;
        auto add_items = [&](uint64_t off, int len, int dst) {
            for (int s0 = 0; s0 < len; s0 += 65536) items.push_back(MaskItem{off + (uint64_t)s0, std::min(65536, len - s0), dst});
        };
        for (int i : longQueries) add_items(p->qoff[i], p->qlen[i], i);
        if (numRec > 0) {  // the records only: no separator byte enters a presence set
            for (int r = 0; r < numRec; ++r) add_items(p->tg[0].off + (uint64_t)p->recOff[(size_t)r], in.recordLengths[r], N + r);
        } else {
            for (int t = 0; t < T; ++t) add_items(p->tg[t].off, p->tg[t].len, N + t);
        }
        // (a record target of the hit search: set N, record 0's; its alphabet lengths are not reported)
        HostBuf<int> tset(be, (size_t)N);
        parallel_ranges((size_t)N, 65536, [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) tset[i] = N + p->tidx[i];
        });
        const int numSets = std::max(T, numRec);
        const int unionSet = N + numSets;
        DevBuf<uint32_t> dMasks(be, (size_t)(N + numSets + 1) * 8);
        be->zero(dMasks.p, (size_t)(N + numSets + 1) * 8 * sizeof(uint32_t));
        DevBuf<MaskItem> dItems(be, items.size());
        if (!items.empty()) dItems.upload(items.data(), items.size());
        {
            MaskParams mp;
            memset(&mp, 0, sizeof(mp));
            mp.raw = p->dSeq.p;
            mp.items = dItems.p;
            mp.numItems = (int)items.size();
            mp.qoff = p->dQoff.p;
            mp.qlen = p->dQlen.p;
            mp.numQueries = N / qstep;
            mp.masks = dMasks.p;
            mp.unionSet = unionSet;
            if (in.strands) {
                mp.rc = p->dSeq.p + rcBase;
                mp.rcBytes = (uint64_t)readBytes;
            }
            if (mp.numItems + mp.numQueries > 0) be->launch_mask(mp);
        }
        DevBuf<int> dTset(be, N), dAlpha(be, N);
        trace.mark("prepare: mask items");
        if (!in.bestRecord) {  // a best-record batch: once the record of each pair is known (Pass::pick_records)
            dTset.upload(tset.p, N);
            be->launch_alpha_len(dMasks.p, nullptr, dTset.p, N, dAlpha.p);
        }
        classify(p);  // host work while the upload and the alphabet kernels run
        trace.mark("prepare: classification");
        if (!in.bestRecord) {
            p->alphaLen.resize(N);
            dAlpha.download(p->alphaLen.data(), N);
            stats.d2hBytes += (long long)N * 4;
        }
        uint32_t uni[8];
        be->d2h(uni, dMasks.p + (size_t)unionSet * 8, sizeof(uni));
        stats.d2hBytes += 32;
        if (in.bestRecord) p->dMasks.swap(dMasks);
        trace.mark("prepare: alphabet lengths back");

        // dense codes in ascending byte order; absent bytes (padding) map to code 0
        uint8_t map[256];
        p->ncodes = code_map(uni, map, -1);
        if (p->ncodes == 0) p->ncodes = 1;
        // Additional equalities (ref cpp:63-94) over the codes; a pair naming an absent byte changes nothing.  When the
        // relation they induce on the bytes present is TRANSITIVE (every group of connected bytes is pairwise equal:
        // upper/lower case, synonyms), the bytes of a group get ONE code and the batch runs as a plain-equality batch --
        // the DP only ever asks whether two symbols are equal -- so every fast path (seed filter, lane kernels without
        // the table look-ups) applies.  Otherwise (e.g. a wildcard that equals several mutually different bytes) the
        // kernels test pairs of codes through the table.
        std::vector<uint8_t> eq;
        bool anyEq = false;
        if (in.config.additionalEqualities && in.config.additionalEqualitiesLength > 0) {
            const int s0 = p->ncodes;
            eq.assign((size_t)s0 * s0, 0);
            for (int i = 0; i < s0; ++i) eq[(size_t)i * s0 + i] = 1;
            for (int i = 0; i < in.config.additionalEqualitiesLength; ++i) {
                const int a = (unsigned char)in.config.additionalEqualities[i].first;
                const int b = (unsigned char)in.config.additionalEqualities[i].second;
                const bool ha = uni[a >> 5] >> (a & 31) & 1u, hb = uni[b >> 5] >> (b & 31) & 1u;
                if (ha && hb && a != b) {
                    eq[(size_t)map[a] * s0 + map[b]] = eq[(size_t)map[b] * s0 + map[a]] = 1;
                    anyEq = true;
                }
            }
        }
        if (anyEq && tun.collapseEqualities) {
            const int s0 = p->ncodes;
            std::vector<int> comp(s0, -1);  // connected components of the equality graph, numbered by their smallest code
            int ncomp = 0;
            std::vector<int> stack;
            for (int c = 0; c < s0; ++c) {
                if (comp[c] >= 0) continue;
                comp[c] = ncomp;
                stack.assign(1, c);
                while (!stack.empty()) {
                    const int u = stack.back();
                    stack.pop_back();
                    for (int v = 0; v < s0; ++v)
                        if (eq[(size_t)u * s0 + v] && comp[v] < 0) {
                            comp[v] = ncomp;
                            stack.push_back(v);
                        }
                }
                ++ncomp;
            }
            bool transitive = true;
            for (int u = 0; u < s0 && transitive; ++u)
                for (int v = 0; v < s0; ++v)
                    if ((comp[u] == comp[v]) != (eq[(size_t)u * s0 + v] != 0)) {
                        transitive = false;
                        break;
                    }
            if (transitive) {
                for (int b = 0; b < 256; ++b)
                    if (uni[b >> 5] >> (b & 31) & 1u) map[b] = (uint8_t)comp[map[b]];
                p->ncodes = ncomp;
                anyEq = false;  // nothing left for the table
            }
        }
        // more than one record: the separator takes the code after the batch's codes; it matches nothing, not even a
        // wildcard (its row and column of the equality table stay 0)
        if (numRec > 1) {
            if (p->ncodes >= 256)
                throw std::runtime_error(std::string(in.bestRecord ? "edlibB200AlignRecords" : "edlibB200FindRecordHits") +
                                         ": the queries and records use all 256 codes: none is left for the separator "
                                         "between records");
            p->sep = p->ncodes++;
            if (anyEq) {
                const int s0 = p->sep, s1 = p->ncodes;
                std::vector<uint8_t> grown((size_t)s1 * s1, 0);
                for (int a = 0; a < s0; ++a)
                    for (int b = 0; b < s0; ++b) grown[(size_t)a * s1 + b] = eq[(size_t)a * s0 + b];
                eq.swap(grown);
            }
        }
        DevBuf<uint8_t> dMap(be, 256);
        dMap.upload(map, 256);
        EncodeParams ep{p->dSeq.p, (uint64_t)devTotal, dMap.p};
        be->launch_encode(ep);
        if (numRec > 0) {
            p->dRecOff.alloc(be, (size_t)numRec + 1);
            p->dRecOff.upload(p->recOff.data(), (size_t)numRec + 1);
        }
        if (numRec > 1) {  // separator columns: written over the encoded zeros, before any sweep or index build reads them
            RecordParams rp;
            memset(&rp, 0, sizeof(rp));
            rp.stage = REC_SEPARATORS;
            rp.numItems = p->tg[0].len;
            rp.recOff = p->dRecOff.p;
            rp.numRecords = numRec;
            rp.gap = p->recGap;
            rp.sep = p->sep;
            rp.tcodes = p->dSeq.p + p->tg[0].off;
            be->launch_record(rp);
        }
        if (anyEq) {
            p->dEqtab.alloc(be, eq.size());
            p->dEqtab.upload(eq.data(), eq.size());
            p->hasEq = true;
        }
        be->sync();
        trace.mark("prepare: upload+alphabet");
    } catch (...) {
        quiesce();  // nothing may still be reading the staging block when it goes back to the cache
        delete p;
        throw;
    }
    return p;
}

// Groups the pairs by (target, word class): a pure function of the lengths, the distinct targets and the
// config, so prepare() runs it on the host workers while the sequences travel to the device; the lists stay
// with the batch (and the per-thread pieces, through the spare batch object, keep their storage from call to call).
void Engine::classify(Prepared* p) {
    const int N = p->N;
    const int mode = p->mode;
    const int k = p->cfg.k;
    p->special.resize(N);
    std::map<std::pair<int, int>, std::vector<int>>& groups = p->groups;  // (target, nw32) -> pairs, ascending
    std::vector<int>& wPairs = p->wPairsBase;
    wPairs.clear();
    p->otherPairs.clear();
    for (auto& kv : groups) kv.second.clear();
    {
        // contiguous ranges of pairs are classified on a few host threads and concatenated in order
        std::vector<Prepared::Part>& parts = p->parts;
        parts.resize(HostPool::get().width());
        const size_t nparts = parallel_parts((size_t)N, 65536, [&](size_t t, size_t lo, size_t hi) {
            Prepared::Part& P = parts[t];
            for (auto& kv : P.groups) kv.second.clear();
            P.wPairs.clear();
            P.other.clear();
            std::pair<int, int> lastKey(-1, -1);
            std::vector<int>* lastList = nullptr;
            for (int i = (int)lo; i < (int)hi; ++i) {
                const int m = p->qlen[i], n = p->tlen[i];
                p->special[i] = (m == 0 || n == 0) ? 1 : 0;
                if (p->special[i] || (mode == MODE_NW && k >= 0 && k < abs(n - m))) {  // ref cpp:166-184, 744
                    P.other.push_back(i);
                    continue;
                }
                if (m <= 256) {
                    const std::pair<int, int> key(p->tidx[i], ceil_div(m, 32));
                    if (key != lastKey) {  // neighbours usually share their group
                        lastKey = key;
                        lastList = &P.groups[key];
                        if (lastList->empty()) lastList->reserve(hi - (size_t)i);
                    }
                    lastList->push_back(i);
                } else {
                    P.wPairs.push_back(i);
                }
            }
        });
        for (size_t t = 0; t < nparts; ++t) {
            const Prepared::Part& P = parts[t];
            for (auto& kv : P.groups) {
                if (kv.second.empty()) continue;
                std::vector<int>& dst = groups[kv.first];
                dst.insert(dst.end(), kv.second.begin(), kv.second.end());
            }
            wPairs.insert(wPairs.end(), P.wPairs.begin(), P.wPairs.end());
            p->otherPairs.insert(p->otherPairs.end(), P.other.begin(), P.other.end());
        }
        // drop the keys this batch does not use (bounded memory across differently shaped batches)
        for (auto it = groups.begin(); it != groups.end();) it = it->second.empty() ? groups.erase(it) : std::next(it);
    }
    p->classified = true;
}

static void reset_results(Prepared* p) {
    const int N = p->N;
    // ed / endStart / endCount are written for every pair by the distance pass, special by the classification
    p->ed.resize(N);
    p->endStart.resize(N);
    p->endCount.resize(N);
    p->endPool.clear();
    p->startPool.clear();
    if (p->cfg.task == EDLIB_TASK_PATH) {
        p->alnStart.assign(N, -1);
        p->alnLen.assign(N, 0);
    } else {
        p->alnStart.clear();
        p->alnLen.clear();
    }
    p->alnPool.clear();
}

void Engine::compute(Prepared* p) {
    Backend* be = be_;
    p->computed = false;
    be->reset_timing();
    const int mode = p->mode;
    reset_results(p);
    stats.k1Cells = stats.wCells = 0;
    stats.filterDecided = stats.filterFallback = stats.filterWindows = 0;

    Pass ps(*this, be, p);
    std::vector<int>& wPairs = ps.wPairs;
    Trace& trace = ps.trace;

    // ---- classification (normally done by prepare() while the upload is in flight) --------
    if (!p->classified) classify(p);
    std::map<std::pair<int, int>, std::vector<int>>& groups = p->groups;
    wPairs = p->wPairsBase;

    // ---- routes of the groups of short queries: warp kernel, device-driven first seed level, host-driven --------
    struct Route {
        int t, nw;
        const std::vector<int>* list;
        bool device;
    };
    std::vector<Route> routes;
    long long devReads = 0, devListed = 0;
    int devSlices = 0;
    // a group list of a strand batch holds the two strands of a read next to each other: even slices keep them together
    const int sliceReads = p->strands ? tun.devSliceReads & ~1 : tun.devSliceReads;
    for (auto& kv : groups) {
        const std::vector<int>& list = kv.second;
        // Small groups go to the warp kernel, except HW over a long target: there the lane kernel
        // can cut the target into chunks and spread even one alignment over many CTAs.
        if ((int)list.size() < tun.k1MinGroup && !(mode == MODE_HW && p->tg[kv.first.first].len >= 8 * tun.k1MinChunk)) {
            wPairs.insert(wPairs.end(), list.begin(), list.end());
            continue;
        }
        const int t = kv.first.first, nw = kv.first.second;
        {
            int bt = 0, rc = 0;
            be->k1_shape(nw, p->ncodes, (int)list.size(), &bt, &rc);
            if (rc <= 0) {  // alphabet too large for per-thread Peq rows in shared memory
                wPairs.insert(wPairs.end(), list.begin(), list.end());
                continue;
            }
        }
        const bool dev = ps.dev_eligible(t, nw) && (int)list.size() >= tun.k1MinGroup;
        routes.push_back(Route{t, nw, &list, dev});
        if (dev) {
            devReads += (long long)list.size();
            devSlices += ceil_div((int)list.size(), sliceReads);
            const bool consecutive = (long long)list.back() - list.front() + 1 == (long long)list.size();
            if (!consecutive) devListed += (long long)list.size();
        }
    }
    // ---- device-driven first seed level of every group that may take it: enqueued without waiting --------
    if (devSlices > 0) {
        ps.dev_begin(devReads, devSlices, devListed);
        for (Route& r : routes) {
            if (!r.device) continue;
            const std::vector<int>& list = *r.list;
            if (!ps.seed_index(r.t) || ps.seedIdx->Ls[0] <= 0) {  // target too short for seeds
                r.device = false;
                continue;
            }
            const bool consecutive = (long long)list.back() - list.front() + 1 == (long long)list.size();
            std::atomic<long long> rows(0);
            parallel_ranges(list.size(), 65536, [&](size_t lo, size_t hi) {
                long long s = 0;
                for (size_t i = lo; i < hi; ++i) s += p->qlen[list[i]];
                rows.fetch_add(s, std::memory_order_relaxed);
            });
            stats.k1Cells += rows.load() * (long long)p->tg[r.t].len;
            for (int first = 0; first < (int)list.size(); first += sliceReads)
                ps.dev_enqueue_slice(r.t, r.nw, consecutive ? list.front() : -1, list.data(), first,
                                     std::min(sliceReads, (int)list.size() - first));
        }
        ps.dev_enqueued();
        trace.mark("compute: device stage enqueued");
    } else {
        ps.host_touch_all();
    }
    // ---- host-driven groups ----------------------------------------------------------------
    for (Route& r : routes) {
        if (r.device) continue;
        ps.lane_group(r.t, r.nw, *r.list);
        if (ps.devMode) ps.hostPairs.insert(ps.hostPairs.end(), r.list->begin(), r.list->end());
    }
    trace.mark("compute: K1 groups done");
    if (ps.devMode) {
        ps.host_touch(wPairs.data(), wPairs.size());
        ps.host_touch(p->otherPairs.data(), p->otherPairs.size());
        ps.hostPairs.insert(ps.hostPairs.end(), wPairs.begin(), wPairs.end());
        ps.hostPairs.insert(ps.hostPairs.end(), p->otherPairs.begin(), p->otherPairs.end());
    }
    ps.warp_distance();
    trace.mark("compute: W distance pass");
    if (ps.devMode) {
        ps.dev_leftovers();
        ps.collect_ends(&ps.hostPairs);
    } else {
        ps.collect_ends(nullptr);
    }
    if (p->bestRecord) ps.pick_records();
    if (p->strands) ps.pick_strands();
    trace.mark("compute: end locations");
    ps.start_locations();
    ps.paths();
    trace.mark("compute: starts + paths");
    be->sync_all();
    be->release_marks();
    stats.launches = be->launches();
    statsPending_ = true;  // the per-kernel device times are read from their events when somebody asks (finish_stats)
    p->computed = true;
}

// Device times of the last pass from the CUDA events around its launches: a few hundred event queries, so they are
// only made when the caller asks for statistics, not inside every call.
void Engine::finish_stats() {
    if (!statsPending_) return;
    statsPending_ = false;
    stats.kernelMs = be_->kernel_ms(nullptr);
    stats.k1Ms = be_->kernel_ms("k1") + be_->kernel_ms("k1_prefix");
    stats.kernelReport = be_->kernel_report();
}

// ---------------------------------------------------------------------------------------------
// materialize / release / one-shot
// ---------------------------------------------------------------------------------------------

// The EdlibAlignResult of pair i (arrays malloc'd one by one: each is free()-able on its own, ref edlib.h:177,186,205).
// Returns false when the allocator fails (the arrays of this result are released again).
static bool materialize_one(const Prepared* p, int i, EdlibAlignResult& r) {
    memset(&r, 0, sizeof(r));
    r.status = EDLIB_STATUS_OK;
    r.editDistance = -1;
    r.alphabetLength = p->alphaLen[i];
    const int m = p->qlen[i], n = p->tlen[i];
    if (p->special[i]) {  // ref cpp:166-184
        const int rawMode = (int)p->cfg.mode;
        if (rawMode == EDLIB_MODE_NW || rawMode == EDLIB_MODE_SHW || rawMode == EDLIB_MODE_HW) {
            r.endLocations = static_cast<int*>(malloc(sizeof(int)));
            if (!r.endLocations) return false;
            r.editDistance = rawMode == EDLIB_MODE_NW ? std::max(m, n) : m;
            r.endLocations[0] = rawMode == EDLIB_MODE_NW ? n - 1 : -1;
            r.numLocations = 1;
        } else {
            r.status = EDLIB_STATUS_ERROR;
        }
        return true;
    }
    if (p->ed[i] < 0) return true;
    const int c = p->endCount[i];
    r.endLocations = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(c, 1)));
    if (!r.endLocations) return false;
    memcpy(r.endLocations, p->endPool.data() + p->endStart[i], sizeof(int) * (size_t)c);
    if (!p->startPool.empty() || p->cfg.task == EDLIB_TASK_LOC || p->cfg.task == EDLIB_TASK_PATH) {
        r.startLocations = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(c, 1)));
        if (!r.startLocations) {
            free(r.endLocations);
            r.endLocations = nullptr;
            return false;
        }
        memcpy(r.startLocations, p->startPool.data() + p->endStart[i], sizeof(int) * (size_t)c);
    }
    if (!p->alnStart.empty() && p->alnStart[i] >= 0) {
        r.alignment = static_cast<unsigned char*>(malloc((size_t)std::max(p->alnLen[i], 1)));
        if (!r.alignment) {
            free(r.endLocations);
            free(r.startLocations);
            r.endLocations = r.startLocations = nullptr;
            return false;
        }
        r.alignmentLength = p->alnLen[i];
        memcpy(r.alignment, p->alnPool.data() + p->alnStart[i], (size_t)p->alnLen[i]);
    }
    r.editDistance = p->ed[i];
    r.numLocations = c;
    return true;
}

void free_result_arrays(EdlibAlignResult* results, size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) {
        free(results[i].endLocations);
        free(results[i].startLocations);
        free(results[i].alignment);
        results[i].endLocations = results[i].startLocations = nullptr;
        results[i].alignment = nullptr;
    }
}

void fail_results(EdlibAlignResult* results, int n) {
    for (int i = 0; i < n; ++i) {
        memset(&results[i], 0, sizeof(results[i]));
        results[i].status = EDLIB_STATUS_ERROR;
        results[i].editDistance = -1;
    }
}

void Engine::materialize(Prepared* p, EdlibAlignResult* results, const std::vector<int>* list) {
    if (!p->computed) throw std::runtime_error("results requested from a batch that was not (successfully) computed");
    Trace trace;
    const int N = p->strands ? p->N / 2 : p->N;  // a strand batch: one result per read, from its winning strand
    const size_t n = list ? list->size() : (size_t)N;
    auto result_of = [&](size_t j) { return list ? (*list)[j] : (int)j; };
    const bool failed = parallel_any(n, list ? 4096 : 65536, [&](size_t j) {
        const int i = result_of(j);
        return !materialize_one(p, p->strands ? 2 * i + p->strand[i] : i, results[i]);
    });
    if (failed) {  // every listed result was written: all of them give their arrays back
        for (size_t j = 0; j < n; ++j) free_result_arrays(results, (size_t)result_of(j), (size_t)result_of(j) + 1);
        throw std::runtime_error("out of memory while building the results");
    }
    trace.mark("materialize");
}

void Engine::release(Prepared* p) {
    if (!p) return;
    // device buffers go back to the pool now
    p->dSeq.reset();
    p->dQoff.reset();
    p->dQlen.reset();
    p->dEqtab.reset();
    p->dRecOff.reset();
    p->dMasks.reset();
    p->computed = false;
    if (spare_) {
        delete p;
        return;
    }
    spare_ = p;  // keep the object (host vectors, pinned result arrays) for the next batch
}

Engine::~Engine() {
    delete spare_;
    for (TargetHandle* h : targets_) delete h;
}

TargetHandle* Engine::find_target(const char* ptr, int n) const {
    for (TargetHandle* h : targets_)
        if (h->ptr == ptr && h->n == n) return h;
    return nullptr;
}

// Uploads, encodes and indexes a target once (the steps Engine::align_streamed otherwise repeats per batch).
TargetHandle* Engine::target_prepare(const char* target, int n) {
    Backend* be = be_;
    if (!target || n < 64) throw std::runtime_error("target handle: target too short");
    TargetHandle* h = new TargetHandle();
    try {
        h->ptr = target;
        h->n = n;
        h->bytes = round_up((size_t)n, 16) + 32;
        h->codes.alloc(be, h->bytes);
        {
            HostBuf<uint8_t> stage(be, h->bytes);
            memcpy(stage.p, target, (size_t)n);
            memset(stage.p + n, 0, h->bytes - (size_t)n);
            h->codes.upload(stage.p, h->bytes);
            be->sync();
        }
        build_seed_index(be, tun, h->idx, h->codes.p, n, encode_target(be, h->codes.p, n, h->tc));
        be->sync();
        targets_.push_back(h);
        return h;
    } catch (...) {
        quiesce();
        delete h;
        throw;
    }
}

void Engine::target_free(TargetHandle* h) {
    if (!h) return;
    for (size_t i = 0; i < targets_.size(); ++i)
        if (targets_[i] == h) {
            be_->sync_all();
            targets_.erase(targets_.begin() + (long)i);
            delete h;
            return;
        }
}

void Engine::strands_of(const Prepared* p, unsigned char* strands) const {
    if (!p->strands) throw std::runtime_error("strands requested from a batch not prepared with strands");
    if (!p->computed) throw std::runtime_error("strands requested from a batch that was not (successfully) computed");
    memcpy(strands, p->strand.data(), p->strand.size());
}

void Engine::records_of(const Prepared* p, int* records) const {
    if (!p->bestRecord) throw std::runtime_error("records requested from a batch not prepared as a best-record batch");
    if (!p->computed) throw std::runtime_error("records requested from a batch that was not (successfully) computed");
    const int n = p->strands ? p->N / 2 : p->N;
    for (int i = 0; i < n; ++i) records[i] = p->record[(size_t)(p->strands ? 2 * i + p->strand[(size_t)i] : i)];
}

int Engine::align_batch(const BatchInput& in, EdlibAlignResult* results, unsigned char* strands, int* records) {
    Prepared* p = nullptr;
    stats = EngineStats();
    statsPending_ = false;
    try {
        if (align_streamed(in, results)) return EDLIB_STATUS_OK;
        p = prepare(in);
        compute(p);
        materialize(p, results);  // releases what it built when it fails
        if (strands) strands_of(p, strands);
        if (records) records_of(p, records);
        release(p);
        return EDLIB_STATUS_OK;
    } catch (const std::exception& e) {
        lastError = e.what();
        quiesce();
        if (p) release(p);
        fail_results(results, in.numPairs);
        return EDLIB_STATUS_ERROR;
    }
}

void free_hits(EdlibB200Hits* h) {
    free(h->counts);
    free(h->offsets);
    free(h->columns);
    free(h->scores);
    free(h->strands);
    memset(h, 0, sizeof(*h));
}

void free_hit_alignments(EdlibB200HitAlignments* h) {
    free_hits(&h->hits);
    free(h->starts);
    free(h->alignmentOffsets);
    free(h->alignments);
    memset(h, 0, sizeof(*h));
}

// The grouped batch of every query against the one target (a strand batch for both strands), then the hits pass
// instead of the distance pass.
int Engine::find_hits(const BatchInput& in, long long maxHits, EdlibB200HitAlignments* out, int** records) {
    Prepared* p = nullptr;
    stats = EngineStats();
    statsPending_ = false;
    memset(out, 0, sizeof(*out));
    if (records) *records = nullptr;
    try {
        BatchInput din = in;  // the batch itself is that of edlibB200FindHits: the task only adds a stage
        din.config.task = EDLIB_TASK_DISTANCE;
        p = prepare(din);
        be_->reset_timing();
        {
            Pass ps(*this, be_, p);
            ps.hits(maxHits, in.config.task, out, records);
        }
        be_->sync_all();
        be_->release_marks();
        stats.launches = be_->launches();
        statsPending_ = true;
        release(p);
        return EDLIB_STATUS_OK;
    } catch (const std::exception& e) {
        lastError = e.what();
        quiesce();
        if (p) release(p);
        free_hit_alignments(out);
        if (records) {
            free(*records);
            *records = nullptr;
        }
        return EDLIB_STATUS_ERROR;
    }
}

// =============================================================================================
// Streamed one-shot path of edlibAlignBatch: many short reads, HW, ONE shared target, plain equality.
//
//   caller thread (orchestrator)                      pool workers
//   ---------------------------------------------     --------------------------------------------------
//   target: pack, upload, presence set, code map      pack slice 0 (all workers), upload on the copy stream,
//           encode, seed index                         mark -> slice 1 -> ...
//   per slice: wait for its upload mark; alphabet     then: result structs of the slices whose results the
//           lengths, encode, device-driven seed        orchestrator has seen arrive (DISTANCE task)
//           level, assembly, result copies on the
//           results stream
//   per slice: wait for its results, release it to the workers
//   leftover reads through the host-driven stages; their result structs
//
// Codes: the dense codes of the TARGET's bytes; every other byte of a read becomes one extra code that matches
// nothing (it selects no Peq row and no seed), which is all a byte absent from the target can do under plain
// equality -- so no pass over the reads is needed before the first slice is encoded.
// =============================================================================================
namespace {
struct StreamJob {
    std::mutex mu;
    std::condition_variable cv;
    std::vector<uint64_t> uploadMark;  // per slice: mark on the copy stream (0: not yet)
    std::vector<int> partsLeft;        // per slice: packing parts still running
    std::vector<char> resultsReady;    // per slice: results on the host, result structs may be built
    bool abort = false;
    std::atomic<size_t> nextPack{0}, nextMat{0};
    std::atomic<int> targetIssued{0};  // the target's upload heads the copy stream: the slices queue behind it
    std::atomic<int> failed{0};
    std::vector<char> matDone;         // per result-struct task: its range of results[] was written
};
}  // namespace

bool Engine::align_streamed(const BatchInput& in, EdlibAlignResult* results) {
    Backend* be = be_;
    const int N = in.numPairs;
    if (in.config.mode != EDLIB_MODE_HW || N < tun.streamMinPairs || !tun.deviceStage || in.strands || in.numRecords > 0)
        return false;
    if (in.config.additionalEqualities && in.config.additionalEqualitiesLength > 0) return false;
    if (tun.filterSeedK <= 0 || tun.filterSeedLevels <= 0) return false;
    const char* tptr = in.targets[0];
    const int n = in.targetLengths[0];
    if (n < tun.filterMinTarget || n < 64) return false;
    // one pass over the pairs: same target everywhere, query lengths of at most two neighbouring word classes
    struct Scan {
        int minLen = 0x7fffffff, maxLen = 0;
        long long bytes = 0;
        bool differs = false;
        bool gaps = false;  // some query does not start where its predecessor ends (in the caller's memory)
    };
    // the scan and the offset pass below cut the pairs into the same parts: the offsets start from the scan's byte sums
    auto over_parts = [N](const std::function<void(size_t, size_t, size_t)>& fn) { return parallel_parts((size_t)N, 32768, fn); };
    std::vector<Scan> scans(HostPool::get().width());
    const size_t nparts = over_parts([&](size_t t, size_t lo, size_t hi) {
        Scan s;
        for (size_t i = lo; i < hi; ++i) {
            if (in.targets[i] != tptr || in.targetLengths[i] != n) s.differs = true;
            if (i > 0 && in.queries[i] != in.queries[i - 1] + in.queryLengths[i - 1]) s.gaps = true;
            const int m = in.queryLengths[i];
            s.minLen = std::min(s.minLen, m);
            s.maxLen = std::max(s.maxLen, m);
            s.bytes += m;
        }
        scans[t] = s;
    });
    scans.resize(nparts);
    Scan all;
    for (const Scan& s : scans) {
        all.differs |= s.differs;
        all.gaps |= s.gaps;
        all.minLen = std::min(all.minLen, s.minLen);
        all.maxLen = std::max(all.maxLen, s.maxLen);
        all.bytes += s.bytes;
    }
    if (all.differs || all.minLen < 1 || all.maxLen > 256) return false;
    const int nw = ceil_div(all.maxLen, 32);
    if (ceil_div(all.minLen, 32) * 2 < nw) return false;  // very uneven lengths: the grouped path sorts them by class
    if (all.bytes + n > (1LL << 31) - (1 << 20)) return false;

    Trace trace;
    Prepared* p = take_prepared(in);
    StreamJob job;
    bool poolBusy = false;
    auto stop_workers = [&]() {
        if (!poolBusy) return;
        poolBusy = false;
        {
            std::lock_guard<std::mutex> lock(job.mu);
            job.abort = true;
            job.cv.notify_all();
        }
        HostPool::get().end(true);
    };
    std::function<void()> freeBuilt;
    try {
        p->special.resize(N);
        p->alphaLen.resize(N);
        reset_results(p);
        // offsets of the packed queries: per-part byte sums from the scan, then a running sum inside every part
        // (also into staging memory: the per-pair arrays are uploaded slice by slice with the sequences)
        HostBuf<uint64_t> hQoff(be, (size_t)N);
        HostBuf<int> hQlen(be, (size_t)N);
        std::vector<long long> partOff(nparts + 1, 0);
        for (size_t t = 0; t < nparts; ++t) partOff[t + 1] = partOff[t] + scans[t].bytes;
        over_parts([&](size_t t, size_t lo, size_t hi) {
            uint64_t off = (uint64_t)partOff[t];
            for (size_t i = lo; i < hi; ++i) {
                const int m = in.queryLengths[i];
                p->qlen[i] = m;
                p->tlen[i] = n;
                p->tidx[i] = 0;
                p->special[i] = 0;
                p->qoff[i] = off;
                hQoff[i] = off;
                hQlen[i] = m;
                off += (uint64_t)m;
            }
        });
        const size_t qBytes = (size_t)all.bytes;
        const bool direct = tun.directUpload && !all.gaps && be->host_pinned(in.queries[0], qBytes);
        const size_t tOff = round_up(qBytes, 16);
        const size_t total = tOff + round_up((size_t)n, 16) + 32;
        p->tg.push_back(Target{tptr, n, (uint64_t)tOff});
        HostBuf<uint8_t> stageBuf(be, total);
        uint8_t* stage = stageBuf.p;
        p->dSeq.alloc(be, total);
        p->dQoff.alloc(be, N);
        p->dQlen.alloc(be, N);
        DevBuf<int> dAlpha(be, (size_t)N);
        trace.mark("stream: lengths + offsets + buffers");

        // slices of reads; every slice is packed by all workers together (parts), so that slice 0 is on its way first
        // at least eight slices for big batches: the result structs of the last slice are the tail of the call
        const int sliceReads = std::min(tun.devSliceReads, std::max(4096, ceil_div(N, N >= 262144 ? tun.streamSlices : 4)));
        const int numSlices = ceil_div(N, sliceReads);
        const size_t W = HostPool::get().width();
        const size_t workers = W > 1 ? W - 1 : 0;  // the caller orchestrates
        const int partsPerSlice = (int)std::max<size_t>(1, workers);
        job.uploadMark.assign((size_t)numSlices, 0);
        job.partsLeft.assign((size_t)numSlices, partsPerSlice);
        job.resultsReady.assign((size_t)numSlices, 0);
        const bool matInJob = in.config.task == EDLIB_TASK_DISTANCE;
        const uint64_t allocated = be->mark(Backend::STREAM_COMPUTE);  // the copy stream may use the buffers after this
        be->wait(Backend::STREAM_COPY, allocated);

        // Reads [first, end) of part `part` of slice s, or of the whole slice (part < 0).  Packing, uploads and result
        // structs cut the slices alike; the error path uses it after this scope is gone, so it holds copies.
        const auto part_range = [N, sliceReads, partsPerSlice](int s, int part) {
            const int lo = (int)std::min<long long>((long long)s * sliceReads, N);
            const int hi = (int)std::min<long long>((long long)(s + 1) * sliceReads, N);
            if (part < 0) return std::make_pair(lo, hi);
            return std::make_pair(lo + (int)((long long)(hi - lo) * part / partsPerSlice),
                                  lo + (int)((long long)(hi - lo) * (part + 1) / partsPerSlice));
        };
        auto pack_part = [&](size_t task) {
            const int s = (int)(task / (size_t)partsPerSlice);
            const auto [a, b] = part_range(s, (int)(task % (size_t)partsPerSlice));
            if (b > a) {
                const size_t off = (size_t)p->qoff[a];
                const size_t bytes = (size_t)(p->qoff[b - 1] + (uint64_t)p->qlen[b - 1]) - off;
                const uint8_t* src = stage + off;
                if (direct) {
                    // the reads lie back to back in pinned caller memory: the device reads them from there
                    src = reinterpret_cast<const uint8_t*>(in.queries[0]) + off;
                } else {
                    // runs of queries that are contiguous in the caller's memory are copied in one piece
                    int i = a;
                    while (i < b) {
                        int j = i + 1;
                        while (j < b && in.queries[j] == in.queries[j - 1] + p->qlen[j - 1]) ++j;
                        const size_t run = (size_t)(p->qoff[j - 1] + (uint64_t)p->qlen[j - 1] - p->qoff[i]);
                        memcpy(stage + p->qoff[i], in.queries[i], run);
                        i = j;
                    }
                }
                while (!job.targetIssued.load(std::memory_order_acquire)) {  // (packing went on meanwhile)
                    std::this_thread::yield();
                    std::lock_guard<std::mutex> lock(job.mu);
                    if (job.abort) return;
                }
                be->h2d_copy(p->dSeq.p + off, src, bytes);
                be->h2d_copy(p->dQoff.p + a, hQoff.p + a, (size_t)(b - a) * sizeof(uint64_t));
                be->h2d_copy(p->dQlen.p + a, hQlen.p + a, (size_t)(b - a) * sizeof(int));
            }
            std::lock_guard<std::mutex> lock(job.mu);
            if (--job.partsLeft[(size_t)s] == 0) {  // the last part of the slice: everything of it is on the copy stream
                job.uploadMark[(size_t)s] = be->mark(Backend::STREAM_COPY);
                job.cv.notify_all();
            }
        };
        auto mat_part = [&](size_t task) {
            const int s = (int)(task / (size_t)partsPerSlice);
            {
                std::unique_lock<std::mutex> lock(job.mu);
                job.cv.wait(lock, [&]() { return job.resultsReady[(size_t)s] || job.abort; });
                if (job.abort) return;
            }
            const auto [a, b] = part_range(s, (int)(task % (size_t)partsPerSlice));
            for (int i = a; i < b; ++i) {
                if (p->ed[i] == -2) continue;  // pending: the host-driven stages will settle it
                if (!materialize_one(p, i, results[i])) job.failed.store(1, std::memory_order_relaxed);
            }
            job.matDone[task] = 1;
        };
        // direct uploads need no packing: the orchestrator issues the copies of every slice itself, slice by slice, so
        // that they reach the copy stream in the order the slices are computed in
        const size_t packTasks = direct ? 0 : (size_t)numSlices * partsPerSlice;
        const size_t matTasks = matInJob ? (size_t)numSlices * partsPerSlice : 0;
        job.matDone.assign(matTasks, 0);
        freeBuilt = [&, part_range, partsPerSlice]() {  // error path: the arrays of the result structs built so far
            for (size_t task = 0; task < job.matDone.size(); ++task) {
                if (!job.matDone[task]) continue;
                const auto [a, b] = part_range((int)(task / (size_t)partsPerSlice), (int)(task % (size_t)partsPerSlice));
                for (int i = a; i < b; ++i)
                    if (p->ed[i] != -2) free_result_arrays(results, (size_t)i, (size_t)i + 1);
            }
        };
        const std::function<void(size_t)> workerFn = [&](size_t) {
            try {
                be->bind_thread();
                for (;;) {
                    const size_t t = job.nextPack.fetch_add(1);
                    if (t >= packTasks) break;
                    pack_part(t);
                }
                for (;;) {
                    const size_t t = job.nextMat.fetch_add(1);
                    if (t >= matTasks) break;
                    mat_part(t);
                }
            } catch (...) {
                std::lock_guard<std::mutex> lock(job.mu);
                job.abort = true;
                job.cv.notify_all();
                throw;
            }
        };
        if (workers > 0) {
            HostPool::get().begin(workers, workerFn);
            poolBusy = true;
        }

        // ---- target: upload, presence set, codes, encoding, seed index (while the workers pack slice 0); a target the
        // caller keeps resident (edlibB200TargetPrepare) brings all of that along ----
        // Reads in pinned caller memory: their copies go onto the copy stream right behind the target's, slice by slice (in
        // the order the slices are computed in), and run while the target is prepared below.
        auto issue_direct_uploads = [&]() {
            if (!direct) return;
            for (int s = 0; s < numSlices; ++s) {
                const auto [lo, hi] = part_range(s, -1);
                const size_t off = (size_t)p->qoff[lo];
                const size_t bytes = (size_t)(p->qoff[hi - 1] + (uint64_t)p->qlen[hi - 1]) - off;
                be->h2d_copy(p->dSeq.p + off, reinterpret_cast<const uint8_t*>(in.queries[0]) + off, bytes);
                be->h2d_copy(p->dQoff.p + lo, hQoff.p + lo, (size_t)(hi - lo) * sizeof(uint64_t));
                be->h2d_copy(p->dQlen.p + lo, hQlen.p + lo, (size_t)(hi - lo) * sizeof(int));
                std::lock_guard<std::mutex> lock(job.mu);
                job.uploadMark[(size_t)s] = be->mark(Backend::STREAM_COPY);
            }
        };
        TargetHandle* const kept = find_target(tptr, n);
        TargetCodes ownCodes;
        const TargetCodes& tc = kept ? kept->tc : ownCodes;
        if (kept) {
            if (tOff > qBytes) be->zero(p->dSeq.p + qBytes, tOff - qBytes);
            be->d2d(p->dSeq.p + tOff, kept->codes.p, kept->bytes);  // (bytes == total - tOff)
            job.targetIssued.store(1, std::memory_order_release);
            issue_direct_uploads();
        } else {
            if (tun.directUpload && be->host_pinned(tptr, (size_t)n)) {  // pinned caller memory: no staging copy
                be->h2d_copy(p->dSeq.p + tOff, tptr, (size_t)n);
                if (tOff > qBytes) be->zero(p->dSeq.p + qBytes, tOff - qBytes);  // (compute stream; the encode kernel follows there)
                be->zero(p->dSeq.p + tOff + n, total - tOff - (size_t)n);
            } else {
                memcpy(stage + tOff, tptr, (size_t)n);
                memset(stage + tOff + n, 0, total - tOff - (size_t)n);
                if (tOff > qBytes) memset(stage + qBytes, 0, tOff - qBytes);
                be->h2d_copy(p->dSeq.p + qBytes, stage + qBytes, total - qBytes);
            }
            const uint64_t targetUp = be->mark(Backend::STREAM_COPY);
            job.targetIssued.store(1, std::memory_order_release);
            issue_direct_uploads();
            be->wait(Backend::STREAM_COMPUTE, targetUp);
            encode_target(be, p->dSeq.p + tOff, n, ownCodes);
        }
        p->ncodes = tc.ncodes;
        trace.mark("stream: target uploaded + encoded");
        stats = EngineStats();
        stats.h2dBytes = (long long)(kept ? qBytes : total) + 12LL * N;
        be->reset_timing();
        Pass ps(*this, be, p);
        if (kept) {
            kept->idx.target = 0;
            ps.seedIdx = &kept->idx;
        }
        int bt = 0, rc = 0;
        be->k1_shape(nw, p->ncodes, N, &bt, &rc);
        if (rc <= 0 || !ps.dev_eligible(0, nw) || !ps.seed_index(0) || ps.seedIdx->Ls[0] <= 0) {
            // cannot happen for the batches admitted above except with an exotic alphabet: back to the grouped path
            stop_workers();
            be->sync_all();
            be->release_marks();
            release(p);
            return false;
        }
        stats.k1Cells = all.bytes * (long long)n;
        trace.mark("stream: pass + index");
        ps.dev_begin(N, numSlices, 0);
        trace.mark("stream: target + index");

        // ---- slices: enqueue as their uploads are issued ----
        for (int s = 0; s < numSlices; ++s) {
            if (!direct && workers == 0) {  // no pool: the caller packs the slice itself
                for (int part = 0; part < partsPerSlice; ++part) pack_part((size_t)s * partsPerSlice + part);
            }
            uint64_t up = 0;
            {
                std::unique_lock<std::mutex> lock(job.mu);
                job.cv.wait(lock, [&]() { return job.uploadMark[(size_t)s] != 0 || job.abort; });
                if (job.abort) throw std::runtime_error("a worker failed while packing the batch");
                up = job.uploadMark[(size_t)s];
            }
            be->wait(Backend::STREAM_COMPUTE, up);
            const auto [lo, hi] = part_range(s, -1);
            QAlphaParams qa;
            memset(&qa, 0, sizeof(qa));
            qa.raw = p->dSeq.p;
            qa.qoff = p->dQoff.p;
            qa.qlen = p->dQlen.p;
            qa.firstPair = lo;
            qa.numQueries = hi - lo;
            qa.tmask = tc.dMask.p;
            qa.alphaLen = dAlpha.p;
            be->launch_qalpha(qa);
            const uint64_t b0 = p->qoff[lo], b1 = p->qoff[hi - 1] + (uint64_t)p->qlen[hi - 1];
            EncodeParams ep{p->dSeq.p + b0, b1 - b0, tc.dMap.p};
            be->launch_encode(ep);
            ps.extraCopyDst = p->alphaLen.data() + lo;
            ps.extraCopySrc = dAlpha.p + lo;
            ps.extraCopyBytes = (size_t)(hi - lo) * sizeof(int);
            ps.dev_enqueue_slice(0, nw, 0, nullptr, lo, hi - lo);
            ps.extraCopyBytes = 0;
        }
        ps.dev_enqueued();
        trace.mark("stream: slices enqueued");
        // ---- results of the slices as they arrive: released to the workers ----
        for (int s = 0; s < numSlices; ++s) {
            ps.dev_finish_slice(s);
            std::lock_guard<std::mutex> lock(job.mu);
            job.resultsReady[(size_t)s] = 1;
            job.cv.notify_all();
        }
        if (poolBusy) {
            poolBusy = false;
            HostPool::get().end(true);  // the caller helps with the result structs that are left
        } else if (matInJob) {
            for (size_t t = 0; t < matTasks; ++t) mat_part(t);
        }
        if (job.failed.load()) throw std::runtime_error("out of memory while building the results");
        trace.mark("stream: slices done");
        // ---- the reads the first level could not decide; start locations / paths; their result structs ----
        ps.dev_leftovers();
        ps.collect_ends(&ps.hostPairs);
        ps.start_locations();
        ps.paths();
        be->sync_all();
        be->release_marks();
        stats.launches = be->launches();
        statsPending_ = true;
        p->computed = true;
        materialize(p, results, matInJob ? &ps.hostPairs : nullptr);  // the slices' result structs are built
        trace.mark("stream: leftovers + results");
        release(p);
        return true;
    } catch (...) {
        try {
            stop_workers();
        } catch (...) {
        }
        quiesce();
        // result structs built so far own malloc'd arrays: give them back before the caller's array is reset
        // (entries never written are untouched caller memory: only finished result-struct tasks count)
        if (freeBuilt) freeBuilt();
        release(p);
        throw;
    }
}

}  // namespace eb
