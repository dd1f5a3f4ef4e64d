// eb_pass_lane.cpp -- distance pass of the groups of pairs that share a target and have queries of at most
// 256 rows: the stages of the exact candidate filter (seed index + pigeonhole seeds, prefix sweeps, window
// verification; DESIGN.md section 5) and the plain lane-per-alignment sweep behind them.
#include "eb_engine_internal.h"

namespace eb {

// Seed lengths and the radix index of target t (eb_common.h: SeedIndexParams).  Level 0 uses the shortest seeds
// with sigma^L >= filterSeedSlack * n (a fraction of a chance occurrence per seed: every occurrence costs a window
// sweep); the later levels shorter ones (more seeds fit into a read, so a higher threshold, at the price of more
// chance occurrences) for the reads the previous level could not decide.  One table with keys of Lidx symbols
// (sigma^Lidx <= 2n buckets) serves all of them.
bool build_seed_index(Backend* be, const EngineTunables& tun, SeedIndex& sx, const uint8_t* tcodes, int n, int ncodes,
                      bool separators) {
    sx.n = n;
    sx.ok = false;
    const int sigma = std::max(2, ncodes);
    int L0 = 4;
    double v = std::pow((double)sigma, 4);
    while (v < (double)tun.filterSeedSlack * (double)n && L0 < 32) {
        v *= sigma;
        ++L0;
    }
    if (n < 4 * L0) return false;
    // seed lengths of the levels: small alphabets step by two symbols, then by one (every symbol less multiplies the
    // chance occurrences by sigma: the last level of a DNA target sees ~70 per seed)
    const int step = (sigma * sigma <= 32) ? 2 : 1;
    for (int level = 0; level < SEED_LEVELS; ++level) {
        const int L = level < 3 ? L0 - step * level : L0 - step * 2 - (level - 2);
        // shorter than 4 symbols, or more than ~128 chance occurrences per seed: the level selects nothing
        const bool useful = L >= 4 && (level == 0 || (double)n / std::pow((double)sigma, L) <= 128.0);
        sx.Ls[level] = useful ? L : 0;
    }
    int Lidx = 1;
    long long keys = sigma;
    const long long maxKeys = std::min<long long>(std::max<long long>(2LL * n, 4096), 1LL << 28);
    while (Lidx < 16 && keys * sigma <= maxKeys) {
        keys *= sigma;
        ++Lidx;
    }
    sx.Lidx = Lidx;
    sx.sigma = sigma;
    sx.numKeys = (int)keys;
    sx.bucketStart.alloc(be, (size_t)keys + 1);
    sx.positions.alloc(be, (size_t)n);
    DevBuf<int> cursor(be, (size_t)keys);
    be->zero(sx.bucketStart.p, ((size_t)keys + 1) * sizeof(int));
    be->zero(cursor.p, (size_t)keys * sizeof(int));
    SeedIndexParams ip;
    memset(&ip, 0, sizeof(ip));
    ip.tcodes = tcodes;
    ip.n = n;
    ip.Lidx = Lidx;
    ip.sigma = sigma;
    ip.numPos = n;  // every position: keys near the end are padded with code 0 (hits are checked against n)
    ip.numKeys = (int)keys;
    ip.bucketStart = sx.bucketStart.p;
    ip.cursor = cursor.p;
    ip.positions = sx.positions.p;
    if (separators) be->launch_seed_count_records(ip);
    else be->launch_seed_count(ip);
    be->launch_scan(sx.bucketStart.p, (int)keys);
    if (separators) be->launch_seed_fill_records(ip);
    else be->launch_seed_fill(ip);
    sx.ok = true;
    return true;
}

bool Pass::seed_index(int t) {
    if (!seedIdx) seedIdx = &ownIdx;
    SeedIndex& sx = *seedIdx;
    const Target& tg = p->tg[t];
    const int n = tg.len;
    if (sx.target == t && sx.n == n) return sx.ok;
    sx.target = t;
    // a record target: the radix is that of the records' codes, without the separator
    const bool ok = build_seed_index(be, tun, sx, p->dSeq.p + tg.off, n, p->sep >= 0 ? p->sep : p->ncodes, p->sep >= 0);
    trace.mark("filter: seed index");
    return ok;
}

SeedPlanParams Pass::seed_plan_params(const Target& tg, int level) const {
    const SeedIndex& sx = *seedIdx;
    SeedPlanParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.tcodes = p->dSeq.p + tg.off;
    sp.n = tg.len;
    sp.qcodes = p->dSeq.p;
    sp.qoff = p->dQoff.p;
    sp.qlen = p->dQlen.p;
    sp.kBound = p->cfg.k;
    sp.seedK = tun.filterSeedK;
    sp.Ls = sx.Ls[level];
    sp.Lidx = sx.Lidx;
    sp.sigma = sx.sigma;
    sp.numKeys = sx.numKeys;
    sp.bucketStart = sx.bucketStart.p;
    sp.positions = sx.positions.p;
    sp.maxBucket = std::min(tun.filterSeedBucket << (1 + 3 * level), 8192);  // shorter seeds: longer index ranges are normal
    sp.level = level;
    sp.spread = tun.filterSpread;
    return sp;
}

int Pass::plan_windows(SeedPlanParams sp, WinJobs& jobs, int cap, bool hostCount) {
    for (;;) {
        jobs.alloc(be, cap);
        sp.winPair = jobs.pair.p;
        sp.winK = jobs.k.p;
        sp.winStart = jobs.start.p;
        sp.winLen = jobs.len.p;
        sp.winTf = jobs.tf.p;
        sp.winCap = cap;
        sp.winCount = jobs.count;
        be->launch_seed_plan(sp);
        if (!hostCount) return -1;
        int V = 0;
        be->d2h(&V, jobs.count, sizeof(int));
        stats.d2hBytes += 4;
        if (V <= cap) return V;
        cap = V;  // window list overflow: plan again with the exact size
        be->zero(jobs.count, sizeof(int));
    }
}

K1WParams Pass::window_params(const Target& tg, const WinJobs& jobs, int numJobs) const {
    K1WParams wp;
    memset(&wp, 0, sizeof(wp));
    wp.tcodes = p->dSeq.p + tg.off;
    wp.qcodes = p->dSeq.p;
    wp.qoff = p->dQoff.p;
    wp.qlen = p->dQlen.p;
    wp.readList = jobs.pair.p;
    wp.kInit = jobs.k.p;
    wp.winStart = jobs.start.p;
    wp.winLen = jobs.len.p;
    wp.trackFrom = jobs.tf.p;
    wp.numReads = numJobs < 0 ? jobs.cap : numJobs;
    wp.countPtr = numJobs < 0 ? jobs.count : nullptr;
    wp.checkAfter = tun.windowCheckAfter;
    wp.ncodes = p->ncodes;
    wp.eqtab = p->hasEq ? p->dEqtab.p : nullptr;
    return wp;
}

void Pass::sweep_windows(const Target& tg, int nw, const WinJobs& jobs, int numJobs, const WinRecords& out) {
    K1WParams wp = window_params(tg, jobs, numJobs);
    wp.recs = out.recs;
    wp.ovf = out.ovf;
    wp.ovfCount = out.ovfCount;
    wp.ovfCap = out.ovfCap;
    be->launch_k1w(wp, nw);
}

void Pass::reduce_windows(WinReduceParams rp, const SeedPlan* plan, int numReads, const WinRecords& wr, Rec* out, int* extra,
                          int* extraCount, int extraCap) {
    rp.plan = plan;
    rp.winRecs = wr.recs;
    rp.numReads = numReads;
    rp.out = out;
    rp.extra = extra;
    rp.extraCount = extraCount;
    rp.extraCap = extraCap;
    rp.ovf = wr.ovf;
    rp.ovfCount = wr.ovfCount;
    rp.ovfCap = wr.ovfCap;
    be->launch_win_reduce(rp);
}

// Chunk geometry: a HW sweep may be cut into target chunks (each re-started 2*m columns
// early, exact because no HW path spans more than 2*m target symbols) so that a small
// group still fills the machine.
void Pass::lane_geometry(const LaneGroup& c, int g, int nwL, int& chunks, int& chunkLen, bool perChunkRecs) {
    const int n = c.n;
    int blockThreads = 256, residentCtas = 1;
    be->k1_shape(nwL, p->ncodes, g, &blockThreads, &residentCtas);
    chunks = 1;
    chunkLen = (int)round_up((size_t)n, 16);
    if (mode != MODE_HW) return;
    // the restart lead-in (64 * nwL columns) stays below 1/8 of a chunk; a handful of reads is latency-bound
    // per CTA and may be cut finer (lead-in up to 1/3)
    const int minChunk = std::max(tun.k1MinChunk, (g <= 32 ? 2 : 8) * 64 * nwL);
    long long maxChunks = std::max<long long>(1, n / minChunk);
    // plain sweeps return one record per (chunk, read): keep that below ~64 MB
    if (perChunkRecs) maxChunks = std::min<long long>(maxChunks, std::max<long long>(64, (2LL << 20) / std::max(g, 1)));
    maxChunks = std::min<long long>(maxChunks, 4096);
    const long long tiles = ceil_div(g, blockThreads);
    // CTAs run in waves of `residentCtas`; all CTAs of a launch cost the same, so the launch
    // takes ceil(waves) CTA-times.  Pick the cut with the best (fullness of the last wave) x
    // (1 - halo overhead); more, shorter CTAs fill waves better.
    long long best = 1;
    double bestScore = -1;
    for (long long c = 1; c <= maxChunks; ++c) {
        const double waves = (double)(tiles * c) / residentCtas;
        const double eff = waves / (double)((tiles * c + residentCtas - 1) / residentCtas);
        const double len = (double)n / (double)c;
        const double score = eff * (len / (len + 64.0 * nwL));
        if (score > bestScore + 0.002) {
            bestScore = score;
            best = c;
        }
    }
    chunkLen = (int)round_up((size_t)ceil_div(n, (int)best), 16);
    chunks = ceil_div(n, chunkLen);
}

// One launch over the reads `sub` (indices into `list`) with sentinels / thresholds subK.
void Pass::lane_sweep(LaneGroup& c, const std::vector<int>& sub, const std::vector<int>& subK, int nwL, int chunks, int chunkLen,
                int cap, int prefixLen, int rangeMode, std::vector<Rec>& outRecs, std::vector<Ovf>& outOvf) {
    const std::vector<int>& list = c.list;
    const Target& tg = c.tg;
    const int n = c.n;
    const int g = (int)sub.size();
    std::vector<int> rl(g);
    for (int s = 0; s < g; ++s) rl[s] = list[sub[s]];
    DevBuf<int> dList(be, g), dK(be, g);
    dList.upload(rl.data(), g);
    dK.upload(subK.data(), g);
    const size_t numRecs = rangeMode ? 0 : (size_t)g * chunks;  // range mode reports through the list only
    DevBuf<Rec> dRecs(be, std::max<size_t>(numRecs, 1));
    if (numRecs) be->zero(dRecs.p, numRecs * sizeof(Rec));
    DevBuf<int> dCount(be, 1);
    K1Params kp;
    memset(&kp, 0, sizeof(kp));
    kp.tcodes = p->dSeq.p + tg.off;
    kp.n = n;
    kp.qcodes = p->dSeq.p;
    kp.qoff = p->dQoff.p;
    kp.qlen = p->dQlen.p;
    kp.readList = dList.p;
    kp.kInit = dK.p;
    kp.numReads = g;
    kp.mode = mode;
    kp.ncodes = p->ncodes;
    kp.eqtab = p->hasEq ? p->dEqtab.p : nullptr;
    kp.chunks = chunks;
    kp.chunkLen = chunkLen;
    kp.halo = 64 * nwL;
    kp.recs = dRecs.p;
    kp.ovfCount = dCount.p;
    kp.prefixLen = prefixLen;
    kp.rangeMode = rangeMode;
    for (;;) {
        DevBuf<Ovf> dOvf(be, (size_t)std::max(cap, 1));
        be->zero(dCount.p, sizeof(int));
        kp.ovf = dOvf.p;
        kp.ovfCap = cap;
        if (useK1t && !rangeMode && prefixLen == 0) be->launch_k1t(kp, nwL);
        else be->launch_k1(kp, nwL);
        outOvf.clear();
        if (cap <= 0) break;
        int count = 0;
        dCount.download(&count, 1);
        stats.d2hBytes += 4;
        if (count > cap) {
            if (!rangeMode) throw std::runtime_error("internal: end-location list larger than counted");
            cap = count;  // range list overflow: repeat with the exact size
            continue;
        }
        outOvf.resize(count);
        if (count) dOvf.download(outOvf.data(), count);
        stats.d2hBytes += (long long)count * (long long)sizeof(Ovf);
        break;
    }
    outRecs.resize(numRecs);
    if (numRecs) dRecs.download(outRecs.data(), outRecs.size());
    stats.d2hBytes += (long long)outRecs.size() * (long long)sizeof(Rec);
}

// Merge the chunks of every read: the minimum wins; its columns are the inline positions
// of the chunks attaining it (ascending by construction) plus, in a second pass, the
// listed ones.  Returns the reads whose lists are incomplete (some chunk holds > KPOS).
void Pass::lane_merge(LaneGroup& c, const std::vector<int>& sub, int chunks, const std::vector<Rec>& rr, const std::vector<Ovf>* oo,
                std::vector<int>& incomplete, long long& missing) {
    const std::vector<int>& list = c.list;
    const int g = (int)sub.size();
    std::unordered_map<int, std::vector<int>> extra;  // rec index -> listed positions
    if (oo)
        for (const Ovf& o : *oo)
            if (o.score == rr[o.rec].best) extra[o.rec].push_back(o.pos);
    for (int s = 0; s < g; ++s) {
        const int pair = list[sub[s]];
        int b = 0x7fffffff;
        long long total = 0;
        for (int c = 0; c < chunks; ++c) {
            const Rec& r = rr[(size_t)c * g + s];
            if (r.cnt > 0 && r.best < b) {
                b = r.best;
                total = 0;
            }
            if (r.cnt > 0 && r.best == b) total += r.cnt;
        }
        best[pair] = (total > 0) ? b : 0x7fffffff;
        if (total > 0x7fffffffLL / 4) throw std::runtime_error("end-location list too large");
        cnt[pair] = (int)total;
        std::vector<int>& dst = posPool;
        posStart[pair] = (long long)posPool.size();
        posLen[pair] = 0;
        if (total == 0) continue;
        bool complete = true;
        for (int c = 0; c < chunks; ++c) {
            const Rec& r = rr[(size_t)c * g + s];
            if (r.cnt <= 0 || r.best != b) continue;
            for (int q = 0; q < std::min(r.cnt, KPOS); ++q) dst.push_back(r.pos[q]);
            if (r.cnt > KPOS) {
                if (oo) {
                    const std::vector<int>& ex = extra[(int)((size_t)c * g + s)];
                    dst.insert(dst.end(), ex.begin(), ex.end());
                } else {
                    complete = false;
                }
            }
        }
        posLen[pair] = (int)((long long)posPool.size() - posStart[pair]);
        if (!complete) {
            incomplete.push_back(sub[s]);
            missing += total;
        }
    }
}

// It is now known that read s has no alignment within t: final if t is the read's bound, else the read goes on.
bool Pass::no_distance_within(LaneGroup& c, int s, int t) {
    if (t > c.excl[s]) c.excl[s] = t;
    if (t != c.bound[s]) return false;
    no_alignment(c.list[s]);
    return true;
}

void Pass::strand_prune(const std::vector<int>& list, const std::vector<int>& excl, std::vector<int>& bound,
                        std::initializer_list<std::vector<int>*> pending) {
    const int G = (int)list.size();
    std::vector<uint8_t> state(G, 0);  // 0 decided, 1 pending, 2 lost here
    for (std::vector<int>* v : pending)
        for (int s : *v) state[s] = 1;
    bool lost = false;
    for (int s = 0; s + 1 < G; ++s) {
        if ((list[s] & 1) || list[s + 1] != list[s] + 1) continue;
        bool done[2];
        int d[2], ex[2], bd[2];
        for (int h = 0; h < 2; ++h) {
            done[h] = state[s + h] == 0;
            d[h] = done[h] ? best[list[s + h]] : 0x7fffffff;
            ex[h] = excl[s + h];
            bd[h] = bound[s + h];
        }
        const int loser = strand_rule(done, d, ex, bd);
        bound[s] = bd[0];
        bound[s + 1] = bd[1];
        if (loser < 0) continue;
        no_alignment(list[s + loser]);
        state[s + loser] = 2;
        stats.filterDecided++;
        lost = true;
    }
    if (!lost) return;
    for (std::vector<int>* v : pending) v->erase(std::remove_if(v->begin(), v->end(), [&](int s) { return state[s] == 2; }), v->end());
}

// Outcome of the reads of a window stage (seed or prefix stage): their windows reduced on the device (eb_core.h:
// win_reduce_read), then the switch on each read's reduced record.
void Pass::window_outcomes(LaneGroup& c, const std::vector<int>& cand, const int* thr, const SeedPlan* plan, const WinRecords& wr,
                           std::vector<int>& next, int& nSat, int& nLong) {
    const std::vector<int>& list = c.list;
    const int g = (int)cand.size();
    DevBuf<Rec> dOut(be, g);
    DevBuf<int> dCount(be, 1);
    int extraCap = g / 4 + 16384;
    DevBuf<int> dExtra;
    int nExtra = 0;
    for (;;) {
        dExtra.alloc(be, (size_t)extraCap);
        be->zero(dCount.p, sizeof(int));
        reduce_windows(WinReduceParams{}, plan, g, wr, dOut.p, dExtra.p, dCount.p, extraCap);
        dCount.download(&nExtra, 1);
        if (nExtra <= extraCap) break;
        extraCap = nExtra;  // the extra list ran over (repeat-rich reads): reduce again with the exact size
    }
    HostBuf<Rec> out(be, g);
    dOut.download(out.p, g);
    std::vector<int> extra((size_t)nExtra);
    if (nExtra) dExtra.download(extra.data(), (size_t)nExtra);
    stats.d2hBytes += (long long)g * (long long)sizeof(Rec) + 4 + 4LL * nExtra;
    trace.mark("filter: windows reduced");
    // Outcome per read, on a few host threads: records of decided reads go straight to best / cnt;
    // their positions are appended to posPool in slot order (counts first, then the fill).
    // c.repeat is read between the seed levels and the prefix stages only: what the prefix stages write to it is unused.
    struct Part {
        std::vector<int> next, direct;
        long long decided = 0, positions = 0;
        int nSat = 0, nLong = 0;
    };
    std::vector<Part> parts(HostPool::get().width());
    parts.resize(parallel_parts((size_t)g, 65536, [&](size_t t2, size_t lo, size_t hi) {
        Part& P = parts[t2];
        for (size_t i = lo; i < hi; ++i) {
            const int s = cand[i], pair = list[s];
            const Rec& r = out[i];
            if (thr[i] < 0) {
                P.next.push_back(s);
            } else if (r.rsv == SEED_WINDOWS) {
                P.decided++;
                best[pair] = r.best;
                cnt[pair] = r.cnt;
                posLen[pair] = r.cnt;
                P.positions += r.cnt;
            } else if (r.rsv == SEED_NONE) {
                c.repeat[s] = 0;
                if (no_distance_within(c, s, thr[i])) P.decided++;
                else P.next.push_back(s);
            } else if (r.rsv == SEED_LONG_LIST) {
                P.direct.push_back(s);
                P.nLong++;
            } else {
                P.next.push_back(s);
                P.nSat++;
                c.repeat[s] = 1;  // too many seed occurrences for this level
            }
        }
    }));
    std::vector<long long> partPos(parts.size());
    {
        long long at = (long long)posPool.size();
        for (size_t t2 = 0; t2 < parts.size(); ++t2) {
            partPos[t2] = at;
            at += parts[t2].positions;
            stats.filterDecided += parts[t2].decided;
            nSat += parts[t2].nSat;
            nLong += parts[t2].nLong;
            next.insert(next.end(), parts[t2].next.begin(), parts[t2].next.end());
            c.direct.insert(c.direct.end(), parts[t2].direct.begin(), parts[t2].direct.end());
        }
        posPool.resize((size_t)at);
    }
    parallel_parts((size_t)g, 65536, [&](size_t t2, size_t lo, size_t hi) {
        long long at = partPos[t2];
        for (size_t i = lo; i < hi; ++i) {
            const Rec& r = out[i];
            if (thr[i] < 0 || r.rsv != SEED_WINDOWS) continue;
            const int pair = list[cand[i]];
            posStart[pair] = at;
            for (int q = 0; q < std::min(r.cnt, KPOS); ++q) posPool[(size_t)at++] = r.pos[q];
            for (int q = KPOS; q < r.cnt; ++q) posPool[(size_t)at++] = extra[(size_t)r.last + q - KPOS];
        }
    });
}

// Seed stage, host-driven: exact seeds of every read looked up in the index of the target; windows around
// the expected end columns are planned, swept and reduced on the device (eb_core.h: seed_plan_read).
void Pass::seed_stage(LaneGroup& c, int level, const std::vector<int>& in, std::vector<int>& next) {
    const std::vector<int>& list = c.list;
    const Target& tg = c.tg;
    const int nw = c.nw;
    if (!seed_index(c.t) || seedIdx->Ls[level] <= 0) {
        next = in;
        return;
    }
    const int L = seedIdx->Ls[level];
    // every read of `in` gets a slot; thr < 0 marks the ones this stage cannot help (the kernel skips them)
    const int g = (int)in.size();
    if (g == 0) return;
    HostBuf<int> rl(be, g), thr(be, g);
    parallel_ranges((size_t)g, 65536, [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            const int s = in[i];
            rl[i] = list[s];
            thr[i] = seed_threshold(p->qlen[list[s]], c.bound[s], L, tun.filterSeedK, c.excl[s]);
        }
    });
    DevBuf<int> dList(be, g), dThr(be, g), dCount(be, 1);
    dList.upload(rl.p, g);
    dThr.upload(thr.p, g);
    DevBuf<SeedPlan> dPlan(be, g);
    // room for the window jobs: sized from what the previous pass of this level needed per read
    int& perRead = eng.scratch.seedWindowsPerRead[level];
    const int cap = (int)std::min<long long>((long long)g * std::max(perRead + 2, level == 0 ? 8 : level == 1 ? 96 : level == 2 ? 400 : 1500) + 4096, 1LL << 28);
    SeedPlanParams sp = seed_plan_params(tg, level);
    sp.readList = dList.p;
    sp.thr = dThr.p;
    sp.numReads = g;
    sp.maxLen = 32 * nw;
    sp.plan = dPlan.p;
    WinJobs jobs;
    jobs.count = dCount.p;
    be->zero(dCount.p, sizeof(int));
    const int V = plan_windows(sp, jobs, cap, true);
    perRead = (int)(((long long)V + g - 1) / g);
    stats.filterWindows += V;
    trace.mark("filter: seeds planned");
    DevBuf<WinRec> dWinRecs(be, (size_t)std::max(V, 1));
    // end columns beyond the inline ones of a window (reads that tie on many end columns)
    const int ovfCap = (int)std::min<long long>((long long)V / 8 + 65536, 1 << 24);
    DevBuf<Ovf> dOvf(be, (size_t)ovfCap);
    DevBuf<int> dOvfCount(be, 1);
    be->zero(dOvfCount.p, sizeof(int));
    const WinRecords wr{dWinRecs.p, dOvf.p, dOvfCount.p, ovfCap};
    if (V > 0) sweep_windows(tg, nw, jobs, V, wr);
    int nSat = 0, nLong = 0;
    window_outcomes(c, in, thr.p, dPlan.p, wr, next, nSat, nLong);
    if (trace.on) {
        int nOvf = 0;
        dOvfCount.download(&nOvf, 1);
        fprintf(stderr, "[edlib_b200] filter seed stage %d, L=%d: %d reads, %d windows (%d listed end columns), %d saturated, %d long lists, %zu to the next stage\n",
                level, L, g, V, nOvf, nSat, nLong, next.size());
    }
}

// Prefix stage over the reads `in` (indices into `list`): a sweep of the first P rows of every read reports
// the target ranges where that prefix matches within t = min(K0, bound); the whole read is then swept over
// one window per range.  A read is decided when a window holds a distance <= t (or when t is the caller's
// bound and none does).  Undecided reads go to `next` (a longer prefix or the plain sweep), reads with
// long end-location lists to c.direct.
void Pass::prefix_stage(LaneGroup& c, int P, int K0, const std::vector<int>& in, std::vector<int>& next) {
    const std::vector<int>& list = c.list;
    const Target& tg = c.tg;
    const int n = c.n;
    const int nw = c.nw;
    const std::vector<int>& bound = c.bound;
    const std::vector<int>& excl = c.excl;
    std::vector<int> cand, thr;
    const int minLen = std::max(tun.filterMinLen * P / 64, P + 1);
    for (int s : in) {
        // worth a sweep only if it can decide clearly more than what is already excluded
        if (p->qlen[list[s]] >= minLen && std::min(K0, bound[s]) > excl[s] && (excl[s] < 0 || K0 >= excl[s] + 4)) {
            cand.push_back(s);
            thr.push_back(std::min(K0, bound[s]));
        } else {
            next.push_back(s);
        }
    }
    if (cand.empty()) return;
    const int g = (int)cand.size();
    int chunksA = 1, chunkLenA = 0;
    lane_geometry(c, g, P / 32, chunksA, chunkLenA, false);
    std::vector<Rec> none;
    std::vector<Ovf> ranges;
    lane_sweep(c, cand, thr, P / 32, chunksA, chunkLenA, (int)std::min<long long>(16LL * g + 4096, 1LL << 28), P, 1, none, ranges);
    trace.mark("filter: prefix sweep");
    // ranges of every read, ascending (the list is in completion order)
    std::vector<int> start(g + 1, 0);
    std::vector<char> saturated(g, 0);
    for (const Ovf& o : ranges) {
        if (o.score < 0) saturated[o.rec] = 1;
        else start[o.rec + 1]++;
    }
    for (int i = 0; i < g; ++i) start[i + 1] += start[i];
    std::vector<std::pair<int, int>> rg(start[g]);
    {
        std::vector<int> fill(start.begin(), start.end() - 1);
        for (const Ovf& o : ranges)
            if (o.score >= 0) rg[fill[o.rec]++] = std::make_pair(o.score, o.pos);
    }
    // windows to verify, and the plan of every read: its windows, none (no range or no window: nothing within t),
    // or saturated (its range list ran over, or too many windows: on to the next stage)
    std::vector<int> vPair, vK, vWs, vLen, vTf;
    std::vector<SeedPlan> plan(g);
    for (int i = 0; i < g; ++i) {
        const int s = cand[i];
        const int pair = list[s], m = p->qlen[pair], t = thr[i];
        const int w0 = (int)vPair.size();
        plan[i] = SeedPlan{w0, 0, SEED_NONE, t};
        if (saturated[i]) {
            plan[i].state = SEED_SATURATED;
            continue;
        }
        std::sort(rg.begin() + start[i], rg.begin() + start[i + 1]);
        // An alignment with distance d <= t ending at column e passes, after its first P rows,
        // through a column c' with prefix score <= d and e in [c'+(m-P)-d, c'+(m-P)+d]: the end
        // columns to examine are [first+(m-P)-t, last+(m-P)+t] of every range.  Ranges close to
        // each other share one window; tracked columns of successive windows are kept disjoint.
        long long prevHi = -1;
        for (int a = start[i]; a < start[i + 1];) {
            const int first = rg[a].first;
            int last = rg[a].second;
            int b = a + 1;
            while (b < start[i + 1] && rg[b].first - last <= K1_RANGE_GAP && rg[b].second - first <= tun.filterSpread) {
                last = std::max(last, rg[b].second);
                ++b;
            }
            a = b;
            long long lo = (long long)first + (m - P) - t;
            long long hi = (long long)last + (m - P) + t;
            if (lo <= prevHi) lo = prevHi + 1;
            if (lo < 0) lo = 0;
            if (hi > n - 1) hi = n - 1;
            if (lo > hi) continue;
            prevHi = hi;
            // HW restart: alignments with <= t edits span at most m + t columns (scores <= t stay exact)
            const long long ws = std::max<long long>(0, lo - (long long)(m + t)) & ~15LL;  // windows start at multiples of 16
            vPair.push_back(pair);
            vK.push_back(t + 1);
            vWs.push_back((int)ws);
            vLen.push_back((int)(hi - ws + 1));
            vTf.push_back((int)(lo - ws));
        }
        const int windows = (int)vPair.size() - w0;
        if (windows > tun.filterMaxWindows) {
            vPair.resize(w0);
            vK.resize(w0);
            vWs.resize(w0);
            vLen.resize(w0);
            vTf.resize(w0);
            plan[i].state = SEED_SATURATED;
        } else if (windows > 0) {
            plan[i].count = windows;
            plan[i].state = SEED_WINDOWS;
        }
    }
    trace.mark("filter: windows planned");
    const int V = (int)vPair.size();
    stats.filterWindows += V;
    // Whole reads over their windows, one window per thread (k1w_kernel), reduced per read as in a seed stage.
    DevBuf<SeedPlan> dPlan(be, g);
    dPlan.upload(plan.data(), g);
    DevBuf<WinRec> dRecs(be, V);
    const int ovfCap = (int)std::min<long long>((long long)V / 8 + 65536, 1 << 24);
    DevBuf<Ovf> dOvf(be, (size_t)ovfCap);
    DevBuf<int> dOvfCount(be, 1);
    be->zero(dOvfCount.p, sizeof(int));
    const WinRecords wr{dRecs.p, dOvf.p, dOvfCount.p, ovfCap};
    WinJobs jobs;
    if (V > 0) {
        jobs.alloc(be, V);
        jobs.pair.upload(vPair.data(), V);
        jobs.k.upload(vK.data(), V);
        jobs.start.upload(vWs.data(), V);
        jobs.len.upload(vLen.data(), V);
        jobs.tf.upload(vTf.data(), V);
        sweep_windows(tg, nw, jobs, V, wr);
    }
    int nSat = 0, nLong = 0;
    window_outcomes(c, cand, thr.data(), dPlan.p, wr, next, nSat, nLong);
    if (trace.on) {
        int sat = 0;
        for (char x : saturated) sat += x;
        fprintf(stderr, "[edlib_b200] filter stage P=%d: %d reads, %zu ranges, %d saturated, %d windows, %zu to the next stage\n",
                P, g, rg.size(), sat, V, next.size());
    }
}

// The plain lane-per-alignment sweep of the reads in c.direct over the whole target.
void Pass::plain_sweep(LaneGroup& c) {
    const std::vector<int>& list = c.list;
    const std::vector<int>& direct = c.direct;
    if (direct.empty()) return;
    int chunks = 1, chunkLen = 0;
    lane_geometry(c, (int)direct.size(), c.nw, chunks, chunkLen, true);
    std::vector<int> kInit(direct.size());
    for (size_t s = 0; s < direct.size(); ++s) kInit[s] = c.bound[direct[s]] + 1;
    std::vector<Rec> recs;
    std::vector<Ovf> ovf;
    std::vector<int> incomplete;
    long long missing = 0;
    if (mode == MODE_HW && (int)direct.size() <= tun.tinySweepReads && c.n >= tun.filterMinTarget) {
        // A handful of reads over a long target: the tile kernel would run one wave of CTAs with a few active lanes
        // each, every lane walking thousands of columns (0.5 ms whatever the count).  k1t_kernel gives every read whole
        // warps whose lanes take chunks of a few hundred columns behind their 2m halos.
        const int g = (int)direct.size();
        const long long want = std::max<long long>(1, std::min<long long>(c.n / 256, 32768 / g));
        chunkLen = (int)round_up((size_t)ceil_div(c.n, (int)want), 16);
        chunks = ceil_div(c.n, chunkLen);
        useK1t = true;
    }
    lane_sweep(c, direct, kInit, c.nw, chunks, chunkLen, 0, 0, 0, recs, ovf);
    useK1t = false;
    lane_merge(c, direct, chunks, recs, nullptr, incomplete, missing);
    if (incomplete.empty()) return;
    // Second pass over the few reads with more than KPOS end positions in one chunk: start from the
    // known minimum so that only final positions are recorded, with a list sized from the counts of
    // the first pass, on a finer chunking of the target.
    std::vector<int> subK(incomplete.size());
    for (size_t s = 0; s < incomplete.size(); ++s) subK[s] = best[list[incomplete[s]]];
    int chunks2 = 1, chunkLen2 = 0;
    lane_geometry(c, (int)incomplete.size(), c.nw, chunks2, chunkLen2, true);
    std::vector<Rec> recs2;
    std::vector<Ovf> ovf2;
    std::vector<int> still;
    long long dummy = 0;
    lane_sweep(c, incomplete, subK, c.nw, chunks2, chunkLen2, (int)missing + 16, 0, 0, recs2, ovf2);
    lane_merge(c, incomplete, chunks2, recs2, &ovf2, still, dummy);
}

// Distance pass of one group of pairs that share target `t` and word class `nw` (queries <= 256
// rows), host-driven: the stages of the candidate filter (HW over a long target; DESIGN.md section 5), each on the
// reads the previous ones left undecided, then the plain lane-per-alignment sweep of what is left.
void Pass::lane_group(int t, int nw, const std::vector<int>& list, const std::vector<int>* exclInit, const std::vector<int>* boundInit,
                      int firstSeedLevel) {
    const Target& tg = p->tg[t];
    const int G = (int)list.size();
    LaneGroup c{t, nw, list, tg, tg.len, std::vector<int>(G), std::vector<int>(G, -1), std::vector<int>(), std::vector<uint8_t>(G, 0)};
    host_touch(list.data(), list.size());
    long long rows = 0;
    for (int s = 0; s < G; ++s) {
        const int m = p->qlen[list[s]];
        c.bound[s] = boundInit ? (*boundInit)[s] : (k < 0 || k > m) ? m : k;  // distances never exceed m in HW/SHW (ref cpp:566-568)
        rows += m;
    }
    if (!exclInit) stats.k1Cells += rows * (long long)c.n;  // (device-driven groups were counted when enqueued)
    c.direct.reserve(G);
    std::vector<int> cur;
    cur.reserve(G);
    for (int s = 0; s < G; ++s) {
        if (exclInit && (*exclInit)[s] == -2) {
            c.direct.push_back(s);  // long end-location list: the plain sweep collects it
        } else {
            if (exclInit) c.excl[s] = (*exclInit)[s];
            cur.push_back(s);
        }
    }
    const bool filtered = mode == MODE_HW && c.n >= tun.filterMinTarget;
    if (filtered) {
        trace.mark("lane group: bounds");
        for (int level = firstSeedLevel; level < tun.filterSeedLevels && tun.filterSeedK > 0 && !p->hasEq && !cur.empty(); ++level) {
            // a late level costs about a millisecond whatever it is given (a few reads with thousands of candidates
            // each: one planning group, one reduction thread per read); the plain sweep of a read costs ~15 us
            if (level >= 2 && (int)cur.size() < tun.filterMinLevelReads) break;
            std::vector<int> next;
            seed_stage(c, level, cur, next);
            cur.swap(next);
            if (p->strands) strand_prune(list, c.excl, c.bound, {&cur, &c.direct});
        }
        // Reads that drowned in seed occurrences at the last level tried are repeats: their prefixes match all over
        // the target as well, so the prefix stages would cost two more sweeps and decide few of them.
        if (tun.filterSkipRepeats) {
            std::vector<int> keep;
            for (int s : cur) (c.repeat[s] ? c.direct : keep).push_back(s);
            cur.swap(keep);
        }
        const int stageP[2] = {32, 64};
        const int stageK[2] = {tun.filterK1, tun.filterK0};
        for (int st = 0; st < 2; ++st) {
            if (stageK[st] <= 0 || cur.empty()) continue;
            if (stageP[st] / 32 >= nw) continue;  // the prefix must be shorter than the read's word class
            std::vector<int> next;
            prefix_stage(c, stageP[st], stageK[st], cur, next);
            cur.swap(next);
            if (p->strands) strand_prune(list, c.excl, c.bound, {&cur, &c.direct});
        }
    }
    if (trace.on)
        fprintf(stderr, "[edlib_b200] plain sweep: %zu reads sent directly (long end-location lists, repeats), %zu undecided\n", c.direct.size(), cur.size());
    c.direct.insert(c.direct.end(), cur.begin(), cur.end());
    if (filtered) stats.filterFallback += (long long)c.direct.size();
    trace.mark("filter: collect");
    plain_sweep(c);
}

// =============================================================================================
// Device-driven first seed level.  For the usual batch (a million reads over one genome) the first seed level
// decides 99.8 % of the reads, so it runs without the host in the loop: thresholds are derived in the kernels,
// the window jobs never leave the device (the sweep kernel reads their number from device memory), the
// reduction either finishes a read or appends it to a leftover list, and distances / end locations are
// assembled per slice on the device (-1 rule included) into arrays that travel to the host in four copies.
// Only the leftover reads (a few thousand) see the host-driven stages above.
// =============================================================================================
bool Pass::dev_eligible(int t, int nw) {
    (void)nw;
    if (mode != MODE_HW || p->hasEq || !tun.deviceStage) return false;
    if (tun.filterSeedK <= 0 || tun.filterSeedLevels <= 0) return false;
    if (p->tg[t].len < tun.filterMinTarget) return false;
    return true;
}

void Pass::dev_begin(long long reads, int maxSlices, long long listed) {
    devMode = true;
    dEd.alloc(be, (size_t)N);
    dEndCount.alloc(be, (size_t)N);
    dEndStart.alloc(be, (size_t)N);
    dLeft.alloc(be, (size_t)N);
    dLeftCount.alloc(be, 1);
    be->zero(dLeftCount.p, sizeof(int));
    dHeaders.alloc(be, (size_t)4 * maxSlices);
    be->zero(dHeaders.p, (size_t)4 * maxSlices * sizeof(int));
    hHeaders.resize((size_t)4 * maxSlices);
    slices.clear();
    slices.reserve((size_t)maxSlices);
    poolReserved = 0;
    // the pools of any maxSlices slices of `reads` reads in all: their quarters, rounded down, add up to at most a quarter
    dPool.alloc(be, (size_t)(dev_slice_pool(reads) + (long long)DEV_EXTRA_SLACK * (maxSlices - 1) + 64));
    if (listed > 0) dLists.alloc(be, (size_t)listed);
    p->endPool.resize(dPool.n);
}

int Pass::dev_enqueue_slice(int t, int nw, int firstPair, const int* listHost, int first, int count) {
    const Target& tg = p->tg[t];
    if (!seed_index(t) || seedIdx->Ls[0] <= 0) throw std::runtime_error("internal: device stage without a seed index");
    const int si = (int)slices.size();
    DevSlice sl;
    sl.t = t;
    sl.nw = nw;
    sl.firstPair = firstPair >= 0 ? firstPair + first : -1;
    sl.count = count;
    sl.poolBase = poolReserved;
    sl.poolCap = (int)dev_slice_pool(count);
    poolReserved += sl.poolCap;
    if (poolReserved > (long long)dPool.n) throw std::runtime_error("internal: end-location pool of the device stage too small");
    const int* dList = nullptr;
    if (firstPair < 0) {  // an arbitrary subset of the batch: its pair indices go to the device
        if (listsUsed + (size_t)count > dLists.n) throw std::runtime_error("internal: read lists of the device stage too small");
        be->h2d(dLists.p + listsUsed, listHost + first, (size_t)count * sizeof(int));
        dList = dLists.p + listsUsed;
        listsUsed += (size_t)count;
    }
    int& perRead = eng.scratch.seedWindowsPerRead[0];
    const int cap = (int)std::min<long long>((long long)count * std::max(perRead + 2, 6) + 4096, 1LL << 28);
    const int extraCap = count / 4 + DEV_EXTRA_SLACK;
    const int ovfCap = cap / 8 + 65536;
    DevBuf<Ovf> dOvf(be, (size_t)ovfCap);
    DevBuf<SeedPlan> dPlan(be, count);
    DevBuf<WinRec> dWinRecs(be, cap);
    DevBuf<Rec> dOut(be, count);
    DevBuf<int> dExtra(be, extraCap), dCnt32(be, (size_t)count + 1), dCtr(be, 3);  // counters: windows, extra list, overflow list
    be->zero(dCtr.p, 3 * sizeof(int));
    SeedPlanParams sp = seed_plan_params(tg, 0);
    sp.readList = dList;
    sp.firstPair = sl.firstPair;
    sp.numReads = count;
    sp.maxLen = 32 * nw;
    sp.plan = dPlan.p;
    WinJobs jobs;
    jobs.count = dCtr.p;
    plan_windows(sp, jobs, cap, false);
    const WinRecords wr{dWinRecs.p, dOvf.p, dCtr.p + 2, ovfCap};
    sweep_windows(tg, nw, jobs, -1, wr);
    WinReduceParams rp{};
    rp.leftover = dLeft.p;
    rp.leftoverCount = dLeftCount.p;
    rp.readList = dList;
    rp.firstPair = sl.firstPair;
    rp.qlen = p->dQlen.p;
    rp.kBound = k;
    rp.strands = p->strands;
    reduce_windows(rp, dPlan.p, count, wr, dOut.p, dExtra.p, dCtr.p + 1, extraCap);
    FinParams fp;
    memset(&fp, 0, sizeof(fp));
    fp.recs = dOut.p;
    fp.extra = dExtra.p;
    fp.readList = dList;
    fp.firstPair = sl.firstPair;
    fp.numReads = count;
    fp.qlen = p->dQlen.p;
    fp.kBound = k;
    fp.ed = dEd.p;
    fp.endCount = dEndCount.p;
    fp.endStart = dEndStart.p;
    fp.cnt32 = dCnt32.p;
    fp.pool = dPool.p + sl.poolBase;
    fp.poolBase = sl.poolBase;
    fp.poolCap = sl.poolCap;
    fp.header = dHeaders.p + 4 * si;
    fp.winCount = dCtr.p;
    if (p->strands) {  // the slice holds both strands of its reads (even offsets into a group list of pair couples)
        fp.strands = 1;
        fp.leftover = dLeft.p;
        fp.leftoverCount = dLeftCount.p;
    }
    be->launch_fin_count(fp);
    be->launch_scan(dCnt32.p, count);
    be->launch_fin_fill(fp);
    // the slice's results travel on the results stream while the compute stream goes on with the next slice
    const uint64_t done = be->mark(Backend::STREAM_COMPUTE);
    be->wait(Backend::STREAM_RESULTS, done);
    be->d2h_async(Backend::STREAM_RESULTS, hHeaders.data() + 4 * si, dHeaders.p + 4 * si, 4 * sizeof(int));
    sl.poolFetched = std::min(sl.poolCap, count + count / 4 + 1024);
    be->d2h_async(Backend::STREAM_RESULTS, p->endPool.data() + sl.poolBase, dPool.p + sl.poolBase, (size_t)sl.poolFetched * sizeof(int));
    if (sl.firstPair >= 0) {
        be->d2h_async(Backend::STREAM_RESULTS, p->ed.data() + sl.firstPair, dEd.p + sl.firstPair, (size_t)count * sizeof(int));
        be->d2h_async(Backend::STREAM_RESULTS, p->endCount.data() + sl.firstPair, dEndCount.p + sl.firstPair, (size_t)count * sizeof(int));
        be->d2h_async(Backend::STREAM_RESULTS, p->endStart.data() + sl.firstPair, dEndStart.p + sl.firstPair, (size_t)count * sizeof(long long));
        stats.d2hBytes += 16LL * count;
    } else {
        wholeArrays = true;  // scattered pairs: the per-pair arrays come back in one piece after the last slice
    }
    if (extraCopyBytes) {
        be->d2h_async(Backend::STREAM_RESULTS, extraCopyDst, extraCopySrc, extraCopyBytes);
        stats.d2hBytes += (long long)extraCopyBytes;
    }
    stats.d2hBytes += 16 + 4LL * sl.poolFetched;
    sl.done = be->mark(Backend::STREAM_RESULTS);
    slices.push_back(sl);
    return si;
}

// Waits for the results of slice si; afterwards its reads' ed / endCount / endStart / end locations are valid on
// the host (pending reads carry ed == -2 until the host-driven stages have dealt with them).
void Pass::dev_finish_slice(int si) {
    DevSlice& sl = slices[(size_t)si];
    if (sl.finished) return;
    sl.finished = true;
    be->host_wait(sl.done);
    const int* h = hHeaders.data() + 4 * si;
    if (h[2]) throw std::runtime_error("internal: end-location pool region of a slice overflowed");
    if (h[0] > sl.poolFetched) {  // more end locations than the first copy brought: fetch the rest
        be->d2h(p->endPool.data() + sl.poolBase + sl.poolFetched, dPool.p + sl.poolBase + sl.poolFetched,
                (size_t)(h[0] - sl.poolFetched) * sizeof(int));
        stats.d2hBytes += 4LL * (h[0] - sl.poolFetched);
    }
    stats.filterWindows += h[3];
    stats.filterDecided += sl.count - h[1];
    windowsSeen += h[3];
    readsSeen += sl.count;
}

// After the last slice: per-pair arrays of scattered groups, then the reads the device could not decide, grouped by
// (target, word class) and run through the host-driven stages (their outcome lands in the host vectors; hostPairs).
void Pass::dev_leftovers() {
    for (size_t si = 0; si < slices.size(); ++si) dev_finish_slice((int)si);
    if (readsSeen > 0) eng.scratch.seedWindowsPerRead[0] = (int)((windowsSeen + readsSeen - 1) / readsSeen);
    int L = 0;
    dLeftCount.download(&L, 1);
    if (wholeArrays) {
        be->d2h_async(Backend::STREAM_COMPUTE, p->ed.data(), dEd.p, (size_t)N * sizeof(int));
        be->d2h_async(Backend::STREAM_COMPUTE, p->endCount.data(), dEndCount.p, (size_t)N * sizeof(int));
        be->d2h_async(Backend::STREAM_COMPUTE, p->endStart.data(), dEndStart.p, (size_t)N * sizeof(long long));
        stats.d2hBytes += 16LL * N;
    }
    HostBuf<Leftover> left(be, (size_t)std::max(L, 1));
    if (L) be->d2h(left.p, dLeft.p, (size_t)L * sizeof(Leftover));
    else be->sync();
    stats.d2hBytes += 4 + (long long)sizeof(Leftover) * L;
    trace.mark("device stage: results on the host");
    if (L == 0) return;
    std::sort(left.p, left.p + L, [](const Leftover& a, const Leftover& b) { return a.pair < b.pair; });
    trace.mark("device stage: leftovers sorted");
    struct Group {
        std::vector<int> pairs, excl, bound;
    };
    std::map<std::pair<int, int>, Group> groups;  // (t, nw) -> reads
    for (int i = 0; i < L; ++i) {
        const int pair = left[i].pair;
        Group& g = groups[std::make_pair(p->tidx[pair], ceil_div(p->qlen[pair], 32))];
        g.pairs.push_back(pair);
        g.excl.push_back(left[i].excl);
        g.bound.push_back(left[i].bound);
        hostPairs.push_back(pair);
    }
    trace.mark("device stage: leftovers grouped");
    for (auto& kv : groups) lane_group(kv.first.first, kv.first.second, kv.second.pairs, &kv.second.excl, &kv.second.bound, 1);
}
// =============================================================================================
// Hits (edlibB200FindHits): every end column within k instead of the minimum.  The seed levels are exact pigeonhole
// filters: planned with threshold k, the tracked columns of a read's windows cover every end column of every alignment
// within k, hold every such score exactly and are disjoint and in column order; the whole-target sweep restarts each
// chunk 2m columns early and reports the columns the chunk owns, and so do the (pair, chunk) jobs of the per-pair route
// over each pair's own target.  Either way a read's hits are those of its jobs in job order, so no sort is needed: count
// per job, total per read, the read's place in the output (host), the place of each job, and a fill pass over the jobs
// that store something.
// =============================================================================================
namespace {
// One launch group of the hits pass: reads of one word class on one route, with what the fill pass needs again.
struct HitRun {
    int t = 0, nw = 0, level = -1;  // target (group routes); seed level, -1: whole-target sweep, -2: per-pair route
    std::vector<int> pairs;
    DevBuf<int> dList, dCount, dRoom, dWinCount;
    DevBuf<long long> dAt;
    DevBuf<SeedPlan> dPlan;      // seed route: the windows of each read; per-pair route: the jobs of each read
    WinJobs jobs;                // seed route
    DevBuf<int> dK;              // whole-target sweep: k per read
    DevBuf<LaneHitJob> dJobs;    // per-pair route
    int numJobs = 0, chunks = 0, chunkLen = 0;
};
constexpr int HIT_RUN_JOBS = 1 << 22;  // jobs per launch group of the per-pair route (at most 4096 per read)
}  // namespace

void Pass::hits(long long maxHits, int task, EdlibB200HitAlignments* outAln, int** records) {
    EdlibB200Hits* out = &outAln->hits;
    const int T = (int)p->tg.size();
    // several records (the batch's one target): the sweeps run over all of them at once, and a separator column is
    // never a hit
    const uint8_t* sepCodes = p->sep >= 0 ? p->dSeq.p + p->tg[0].off : nullptr;
    const int Q = p->strands ? N / 2 : N;
    // ---- routes per target group: a group of k1MinGroup pairs (or the batch's only target) takes the seed or
    // whole-target routes over its target, every other pair the per-pair route; a pair with an empty target has no hits
    std::vector<std::vector<int>> byTarget((size_t)T);
    for (int pair = 0; pair < N; ++pair)
        if (p->tlen[pair] > 0) byTarget[(size_t)p->tidx[pair]].push_back(pair);
    std::vector<int> groupTargets, perPair[9];
    for (int t = 0; t < T; ++t) {
        const std::vector<int>& list = byTarget[(size_t)t];
        if (T == 1 || (int)list.size() >= tun.k1MinGroup) {
            if (!list.empty()) groupTargets.push_back(t);
        } else {
            for (int pair : list) perPair[ceil_div(p->qlen[pair], 32)].push_back(pair);
        }
    }
    std::vector<std::unique_ptr<HitRun>> runs;
    DevBuf<long long> dPairCount(be, (size_t)N);
    be->zero(dPairCount.p, (size_t)N * sizeof(long long));
    K1Params kp;
    memset(&kp, 0, sizeof(kp));
    kp.qcodes = p->dSeq.p;
    kp.qoff = p->dQoff.p;
    kp.qlen = p->dQlen.p;
    kp.mode = MODE_HW;
    kp.ncodes = p->ncodes;
    kp.eqtab = p->hasEq ? p->dEqtab.p : nullptr;
    for (int t : groupTargets) {
        const Target& tg = p->tg[(size_t)t];
        const int n = tg.len;
        // ---- routes: the first seed level whose threshold reaches k itself, else the whole-target sweep ----
        const bool seeds = n >= tun.filterMinTarget && !p->hasEq && tun.filterSeedK > 0 && tun.filterSeedLevels > 0 && seed_index(t);
        const size_t firstRun = runs.size();
        std::vector<int> full[9];
        {
            std::map<std::pair<int, int>, std::vector<int>> groups;  // (level, nw) -> pairs
            for (int pair : byTarget[(size_t)t]) {
                const int m = p->qlen[pair], nw = ceil_div(m, 32);
                int level = -1;
                for (int l = 0; seeds && l < tun.filterSeedLevels && level < 0; ++l)
                    if (seedIdx->Ls[l] > 0 && seed_threshold(m, k, seedIdx->Ls[l], tun.filterSeedK, -1) == k) level = l;
                if (level < 0) full[nw].push_back(pair);
                else groups[std::make_pair(level, nw)].push_back(pair);
            }
            for (auto& kv : groups)
                for (size_t a = 0; a < kv.second.size(); a += (size_t)tun.hitRunReads) {
                    runs.emplace_back(new HitRun());
                    HitRun& r = *runs.back();
                    r.t = t;
                    r.level = kv.first.first;
                    r.nw = kv.first.second;
                    r.pairs.assign(kv.second.begin() + a, kv.second.begin() + std::min(kv.second.size(), a + (size_t)tun.hitRunReads));
                }
        }
        // ---- count pass of the seed route: plan at threshold k (one host wait for the window count, one for the plans) ----
        const size_t seedEnd = runs.size();
        for (size_t ri = firstRun; ri < seedEnd; ++ri) {
            HitRun& r = *runs[ri];
            const int g = (int)r.pairs.size();
            r.dList.alloc(be, g);
            r.dList.upload(r.pairs.data(), g);
            const std::vector<int> thr((size_t)g, k);
            DevBuf<int> dThr(be, g);
            dThr.upload(thr.data(), g);
            r.dPlan.alloc(be, g);
            r.dWinCount.alloc(be, 1);
            be->zero(r.dWinCount.p, sizeof(int));
            SeedPlanParams sp = seed_plan_params(tg, r.level);
            sp.readList = r.dList.p;
            sp.thr = dThr.p;
            sp.numReads = g;
            sp.maxLen = 32 * r.nw;
            sp.plan = r.dPlan.p;
            r.jobs.count = r.dWinCount.p;
            const int perRead = r.level == 0 ? 8 : r.level == 1 ? 96 : r.level == 2 ? 400 : 1500;
            r.numJobs = plan_windows(sp, r.jobs, (int)std::min<long long>((long long)g * perRead + 4096, 1LL << 28), true);
            std::vector<SeedPlan> plan((size_t)g);
            be->d2h(plan.data(), r.dPlan.p, (size_t)g * sizeof(SeedPlan));
            stats.d2hBytes += (long long)g * (long long)sizeof(SeedPlan);
            stats.filterWindows += r.numJobs;
            for (int s = 0; s < g; ++s) {
                // saturated: more candidates than the level holds, seeds of repeats, or no room in the job arrays
                if (plan[(size_t)s].state == SEED_SATURATED) full[r.nw].push_back(r.pairs[(size_t)s]);
                else stats.filterDecided++;
            }
            r.dCount.alloc(be, (size_t)std::max(r.numJobs, 1));
            if (r.numJobs > 0) {
                const HitParams h{r.dCount.p, nullptr, nullptr, nullptr, nullptr, sepCodes, p->sep};
                be->launch_k1w_hits(window_params(tg, r.jobs, r.numJobs), h, r.nw);
            }
            HitPlaceParams hp;
            memset(&hp, 0, sizeof(hp));
            hp.plan = r.dPlan.p;
            hp.numReads = g;
            hp.readList = r.dList.p;
            hp.count = r.dCount.p;
            hp.pairCount = dPairCount.p;
            be->launch_hits_total(hp);
        }
        trace.mark("hits: seed windows counted");
        // ---- count pass of the whole-target sweep (launched after the seed route: it overwrites the totals of saturated reads) ----
        kp.tcodes = p->dSeq.p + tg.off;
        kp.n = n;
        for (int nw = 1; nw <= 8; ++nw)
            for (size_t a = 0; a < full[nw].size(); a += (size_t)tun.hitRunReads) {
                runs.emplace_back(new HitRun());
                HitRun& r = *runs.back();
                r.t = t;
                r.nw = nw;
                r.pairs.assign(full[nw].begin() + a, full[nw].begin() + std::min(full[nw].size(), a + (size_t)tun.hitRunReads));
                const int g = (int)r.pairs.size();
                stats.filterFallback += g;
                const LaneGroup c{t, nw, r.pairs, tg, n, {}, {}, {}, {}};
                lane_geometry(c, g, nw, r.chunks, r.chunkLen, true);
                r.numJobs = r.chunks * g;
                r.dList.alloc(be, g);
                r.dList.upload(r.pairs.data(), g);
                const std::vector<int> kk((size_t)g, k);
                r.dK.alloc(be, g);
                r.dK.upload(kk.data(), g);
                r.dCount.alloc(be, (size_t)r.numJobs);
                kp.readList = r.dList.p;
                kp.kInit = r.dK.p;
                kp.numReads = g;
                kp.chunks = r.chunks;
                kp.chunkLen = r.chunkLen;
                kp.halo = 64 * nw;
                const HitParams h{r.dCount.p, nullptr, nullptr, nullptr, nullptr, sepCodes, p->sep};
                be->launch_k1_hits(kp, h, nw);
                stats.k1Cells += (long long)g * 32 * nw * (long long)n;
                HitPlaceParams hp;
                memset(&hp, 0, sizeof(hp));
                hp.chunks = r.chunks;
                hp.numReads = g;
                hp.readList = r.dList.p;
                hp.count = r.dCount.p;
                hp.pairCount = dPairCount.p;
                be->launch_hits_total(hp);
            }
        trace.mark("hits: whole-target sweeps counted");
    }
    // ---- count pass of the per-pair route: (pair, chunk) jobs over each pair's own target, a pair's jobs consecutive
    // and in column order, chunk lengths as lane_geometry cuts a target for the route's pairs of the word class ----
    for (int nw = 1; nw <= 8; ++nw) {
        const std::vector<int>& pl = perPair[nw];
        if (pl.empty()) continue;
        const int G = (int)pl.size();
        stats.filterFallback += G;
        int blockThreads = 0, residentCtas = 0;
        be->k1_shape(nw, p->ncodes, G, &blockThreads, &residentCtas);
        std::vector<int> chunks((size_t)G), chunkLen((size_t)G);
        for (int i = 0; i < G; ++i) {
            const int t = p->tidx[pl[(size_t)i]];
            const Target& tg = p->tg[(size_t)t];
            if (residentCtas > 0) {
                const LaneGroup c{t, nw, pl, tg, tg.len, {}, {}, {}, {}};
                lane_geometry(c, G, nw, chunks[(size_t)i], chunkLen[(size_t)i], true);
            } else {  // no K1 shape for this alphabet (launch_lane_hits decides whether the jobs run): one chunk
                chunks[(size_t)i] = 1;
                chunkLen[(size_t)i] = tg.len;
            }
        }
        for (int a = 0; a < G;) {
            int b = a, numJobs = 0;
            while (b < G && b - a < tun.hitRunReads && numJobs + chunks[(size_t)b] <= HIT_RUN_JOBS) numJobs += chunks[(size_t)b++];
            runs.emplace_back(new HitRun());
            HitRun& r = *runs.back();
            r.nw = nw;
            r.level = -2;
            r.pairs.assign(pl.begin() + a, pl.begin() + b);
            r.numJobs = numJobs;
            const int g = b - a;
            std::vector<SeedPlan> plan((size_t)g);
            std::vector<LaneHitJob> jobs;
            jobs.reserve((size_t)numJobs);
            for (int s = 0; s < g; ++s) {
                const int pair = r.pairs[(size_t)s], m = p->qlen[pair];
                const Target& tg = p->tg[(size_t)p->tidx[pair]];
                const int C = chunks[(size_t)(a + s)], L = chunkLen[(size_t)(a + s)];
                plan[(size_t)s] = SeedPlan{(int)jobs.size(), C, SEED_WINDOWS, k};
                for (int c = 0; c < C; ++c) {
                    const int cs = (int)std::min<long long>((long long)c * L, tg.len);
                    const int ce = (int)std::min<long long>((long long)cs + L, tg.len);
                    const int hs = std::max(0, cs - 64 * nw);  // >= 2m columns of restart: the owned scores are exact
                    jobs.push_back(LaneHitJob{p->qoff[pair], tg.off + (uint64_t)hs, m, hs, cs, ce});
                }
                stats.k1Cells += 32LL * nw * tg.len;
            }
            a = b;
            r.dList.alloc(be, g);
            r.dList.upload(r.pairs.data(), g);
            r.dPlan.alloc(be, g);
            r.dPlan.upload(plan.data(), g);
            r.dJobs.alloc(be, (size_t)numJobs);
            r.dJobs.upload(jobs.data(), (size_t)numJobs);
            r.dCount.alloc(be, (size_t)numJobs);
            const LaneHitParams lp{r.dJobs.p, numJobs, k, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr};
            const HitParams h{r.dCount.p, nullptr, nullptr, nullptr, nullptr, nullptr, -1};
            be->launch_lane_hits(lp, h, nw);
            HitPlaceParams hp;
            memset(&hp, 0, sizeof(hp));
            hp.plan = r.dPlan.p;
            hp.numReads = g;
            hp.readList = r.dList.p;
            hp.count = r.dCount.p;
            hp.pairCount = dPairCount.p;
            be->launch_hits_total(hp);
        }
    }
    trace.mark("hits: per-pair sweeps counted");
    // ---- the place of every read in the output: counts per query, the first maxHits stored, forward strand first ----
    std::vector<long long> cnt((size_t)N), base((size_t)N), stored((size_t)N);
    be->d2h(cnt.data(), dPairCount.p, (size_t)N * sizeof(long long));
    stats.d2hBytes += 8LL * N;
    const int perQuery = p->strands ? 2 : 1;
    out->counts = static_cast<long long*>(malloc(sizeof(long long) * (size_t)std::max(Q, 1)));
    out->offsets = static_cast<long long*>(malloc(sizeof(long long) * ((size_t)Q + 1)));
    if (!out->counts || !out->offsets) throw std::runtime_error("out of memory for the hit lists");
    long long S = 0;
    for (int q = 0; q < Q; ++q) {
        long long total = 0, left = maxHits;
        out->offsets[q] = S;
        for (int s = 0; s < perQuery; ++s) {
            const int pair = q * perQuery + s;
            const long long st = std::min(cnt[(size_t)pair], std::max(left, 0LL));
            base[(size_t)pair] = S;
            stored[(size_t)pair] = st;
            S += st;
            left -= st;
            total += cnt[(size_t)pair];
        }
        out->counts[q] = total;
    }
    out->offsets[Q] = S;
    out->numQueries = Q;
    out->columns = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(S, 1LL)));
    out->scores = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(S, 1LL)));
    if (p->strands) out->strands = static_cast<unsigned char*>(malloc((size_t)std::max(S, 1LL)));
    if (!out->columns || !out->scores || (p->strands && !out->strands)) throw std::runtime_error("out of memory for the hit lists");
    if (p->strands)
        for (int pair = 0; pair < N; ++pair) memset(out->strands + base[(size_t)pair], pair & 1, (size_t)stored[(size_t)pair]);
    if (records) {  // one record: every hit is in record 0, with its column as it is
        *records = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(S, 1LL)));
        if (!*records) throw std::runtime_error("out of memory for the hit lists");
        if (p->sep < 0) memset(*records, 0, sizeof(int) * (size_t)S);
    }
    trace.mark("hits: placed");
    if (S == 0) {
        if (task != EDLIB_TASK_DISTANCE) hit_alignments(task, 0, stored, nullptr, nullptr, nullptr, outAln);
        return;
    }
    // ---- fill pass: only the jobs that store something are swept again ----
    DevBuf<long long> dBase(be, (size_t)N), dStored(be, (size_t)N);
    dBase.upload(base.data(), (size_t)N);
    dStored.upload(stored.data(), (size_t)N);
    DevBuf<int> dCols(be, (size_t)S), dScores(be, (size_t)S);
    for (size_t ri = 0; ri < runs.size(); ++ri) {
        HitRun& r = *runs[ri];
        if (r.numJobs <= 0) continue;
        const int g = (int)r.pairs.size();
        r.dAt.alloc(be, (size_t)r.numJobs);
        r.dRoom.alloc(be, (size_t)r.numJobs);
        HitPlaceParams hp;
        memset(&hp, 0, sizeof(hp));
        hp.plan = r.level != -1 ? r.dPlan.p : nullptr;
        hp.chunks = r.chunks;
        hp.numReads = g;
        hp.readList = r.dList.p;
        hp.count = r.dCount.p;
        hp.pairBase = dBase.p;
        hp.pairStored = dStored.p;
        hp.at = r.dAt.p;
        hp.room = r.dRoom.p;
        be->launch_hits_place(hp);
        const HitParams h{nullptr, r.dAt.p, r.dRoom.p, dCols.p, dScores.p, sepCodes, p->sep};
        const Target& tg = p->tg[(size_t)r.t];
        if (r.level >= 0) {
            be->launch_k1w_hits(window_params(tg, r.jobs, r.numJobs), h, r.nw);
        } else if (r.level == -1) {
            kp.tcodes = p->dSeq.p + tg.off;
            kp.n = tg.len;
            kp.readList = r.dList.p;
            kp.kInit = r.dK.p;
            kp.numReads = g;
            kp.chunks = r.chunks;
            kp.chunkLen = r.chunkLen;
            kp.halo = 64 * r.nw;
            be->launch_k1_hits(kp, h, r.nw);
        } else {
            const LaneHitParams lp{r.dJobs.p, r.numJobs, k, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr};
            be->launch_lane_hits(lp, h, r.nw);
        }
    }
    dScores.download(out->scores, (size_t)S);
    trace.mark("hits: filled");
    if (task != EDLIB_TASK_DISTANCE) hit_alignments(task, S, stored, dBase.p, dCols.p, dScores.p, outAln);
    if (p->sep >= 0) {  // columns into their records (the starts were mapped slice by slice)
        DevBuf<int> dRecords(be, (size_t)S);
        RecordParams rp;
        memset(&rp, 0, sizeof(rp));
        rp.stage = REC_HITS;
        rp.recOff = p->dRecOff.p;
        rp.numRecords = (int)p->recOff.size() - 1;
        rp.cols = dCols.p;
        rp.records = dRecords.p;
        for (long long lo = 0; lo < S; lo += 1LL << 30) {
            rp.firstHit = lo;
            rp.numItems = (int)std::min(S - lo, 1LL << 30);
            be->launch_record(rp);
        }
        dRecords.download(*records, (size_t)S);
        stats.d2hBytes += 4 * S;
    }
    dCols.download(out->columns, (size_t)S);
    stats.d2hBytes += 8 * S;
}

// Start locations and edit scripts of the stored hits.  The stored hits are cut into slices of consecutive slots whose
// jobs (and, task PATH, stored matrices) fit tun.pathSliceBytes and whose scripts stay countable in an int; inside a
// slice, each word class of the lane kernel gets its jobs from a flag scan over the slice's hits, the reversed SHW
// sweeps give the starts, the matrix-storing NW sweeps + traceback the scripts, and the scripts of the slice are
// compacted in hit order into one dense pool that comes back in one copy.
namespace {
struct HitPathClass {  // what the script copy of one word class of a slice needs after its sweeps
    int nw = 0, jobs = 0;
    uint64_t opsStride = 0;
    DevBuf<int> dJobHit, dOpsStart, dOpsLen;
    DevBuf<uint8_t> dOps;
};
}  // namespace

void Pass::hit_alignments(int task, long long S, const std::vector<long long>& stored, const long long* dBase,
                           const int* dCols, const int* dScores, EdlibB200HitAlignments* out) {
    const bool path = task == EDLIB_TASK_PATH;
    out->starts = static_cast<int*>(malloc(sizeof(int) * (size_t)std::max(S, 1LL)));
    if (path) out->alignmentOffsets = static_cast<long long*>(malloc(sizeof(long long) * ((size_t)S + 1)));
    if (!out->starts || (path && !out->alignmentOffsets)) throw std::runtime_error("out of memory for the hit alignments");
    if (path) out->alignmentOffsets[0] = 0;
    if (S == 0) {
        if (path && !(out->alignments = static_cast<unsigned char*>(malloc(1))))
            throw std::runtime_error("out of memory for the hit alignments");
        return;
    }
    unsigned classes = 0;  // word classes of the queries with stored hits
    for (int pair = 0; pair < N; ++pair)
        if (stored[(size_t)pair] > 0) classes |= 1u << ceil_div(p->qlen[pair], 32);
    int maxNw = 0;
    for (int nw = 1; nw <= 8; ++nw) {
        if (!((classes >> nw) & 1u)) continue;
        if (!runner.lane_ok(nw)) throw std::runtime_error("hit alignments: alphabet too large for the lane kernel");
        maxNw = nw;
    }
    // a hit's target slice [start, c] has at most m + s <= min(2m, m + k) columns
    auto maxPathN = [&](int nw) { return (uint64_t)std::min<long long>(64LL * nw, 32LL * nw + k); };
    const uint64_t maxMat = maxPathN(maxNw) * (uint64_t)maxNw, maxOps = 32ull * maxNw + maxPathN(maxNw);
    const size_t perHit = sizeof(LJob) + sizeof(Rec) + 6 * sizeof(int) +
                          (path ? (size_t)maxMat * sizeof(U2) + 2 * (size_t)maxOps + sizeof(TbJob) + 3 * sizeof(int) : 0);
    long long H = std::max<long long>(32, (long long)(tun.pathSliceBytes / perHit));
    H = std::min(H, 1LL << 30);                                      // the flag scans count in an int
    if (path) H = std::min(H, (long long)(0x7fffffff / maxOps) - 1);  // so do the script lengths
    H = std::min(H, S);
    const uint64_t tOff = p->tg[0].off;
    DevBuf<uint64_t> dTOffPair;  // pairs over their own targets: the offset of each pair's target
    if (p->tg.size() > 1) {
        std::vector<uint64_t> off((size_t)N);
        for (int pair = 0; pair < N; ++pair) off[(size_t)pair] = p->tg[(size_t)p->tidx[pair]].off;
        dTOffPair.alloc(be, (size_t)N);
        dTOffPair.upload(off.data(), (size_t)N);
    }
    DevBuf<int> dErr(be, 1);
    be->zero(dErr.p, sizeof(int));
    DevBuf<int> dCnt(be, (size_t)H + 1), dStart(be, (size_t)H), dLen(be, path ? (size_t)H + 1 : 1);
    std::vector<int> lenScan(path ? (size_t)H + 1 : 0);
    long long poolAt = 0;
    for (long long lo = 0; lo < S; lo += H) {
        const int span = (int)std::min(H, S - lo);
        HitResParams hp;
        memset(&hp, 0, sizeof(hp));
        hp.firstHit = lo;
        hp.numPairs = N;
        hp.pairBase = dBase;
        hp.qlen = p->dQlen.p;
        hp.qoff = p->dQoff.p;
        hp.tOff = tOff;
        hp.tOffPair = p->tg.size() > 1 ? dTOffPair.p : nullptr;
        hp.cols = dCols;
        hp.scores = dScores;
        hp.cnt = dCnt.p;
        hp.starts = dStart.p;
        hp.len = dLen.p;
        hp.err = dErr.p;
        if (p->sep >= 0) {  // a start lies in its hit's record
            hp.recOff = p->dRecOff.p;
            hp.numRecords = (int)p->recOff.size() - 1;
        }
        std::vector<std::unique_ptr<HitPathClass>> done;
        for (int nw = 1; nw <= 8; ++nw) {
            if (!((classes >> nw) & 1u)) continue;
            hp.nw = nw;
            hp.stage = HR_FLAG;
            hp.numItems = span;
            be->launch_hit_res(hp);
            be->launch_scan(dCnt.p, span);
            int J = 0;
            be->d2h(&J, dCnt.p + span, sizeof(int));
            if (J <= 0) continue;
            std::unique_ptr<HitPathClass> c(new HitPathClass());
            c->nw = nw;
            c->jobs = J;
            c->dJobHit.alloc(be, (size_t)J);
            DevBuf<LJob> dJobs(be, (size_t)J);
            DevBuf<Rec> dRecs(be, (size_t)J);
            hp.jobs = dJobs.p;
            hp.jobHit = c->dJobHit.p;
            hp.recs = dRecs.p;
            hp.stage = HR_LOC_JOBS;
            be->launch_hit_res(hp);
            const LParams lp{dJobs.p, J, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr, dRecs.p, nullptr, 1};
            be->launch_lane(lp, nw, MODE_SHW, true, false);
            hp.stage = HR_LOC_APPLY;
            hp.numItems = J;
            be->launch_hit_res(hp);
            if (!path) continue;
            const uint64_t maxN = maxPathN(nw);
            hp.matStride = maxN * (uint64_t)nw;
            hp.opsStride = c->opsStride = 32ull * nw + maxN;
            DevBuf<TbJob> dTb(be, (size_t)J);
            DevBuf<U2> dMat(be, (size_t)ceil_div(J, 32) * 32 * hp.matStride);
            c->dOps.alloc(be, (size_t)J * hp.opsStride);
            c->dOpsStart.alloc(be, (size_t)J);
            c->dOpsLen.alloc(be, (size_t)J);
            hp.tb = dTb.p;
            hp.stage = HR_PATH_JOBS;
            hp.numItems = span;
            be->launch_hit_res(hp);
            const LParams sp{dJobs.p, J, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr, dRecs.p, dMat.p, 32};
            be->launch_lane(sp, nw, MODE_NW, false, true);
            const TbParams tp{dTb.p, J, dMat.p, nullptr, p->dSeq.p, p->dSeq.p, p->hasEq ? p->dEqtab.p : nullptr, p->ncodes,
                              c->dOps.p, c->dOpsStart.p, c->dOpsLen.p, 32};
            be->launch_traceback(tp);
            hp.ops = c->dOps.p;
            hp.opsStart = c->dOpsStart.p;
            hp.opsLen = c->dOpsLen.p;
            hp.stage = HR_PATH_LEN;
            hp.numItems = J;
            be->launch_hit_res(hp);
            done.push_back(std::move(c));
        }
        if (p->sep >= 0) {  // starts into their records, while the columns still address the whole target
            RecordParams rp;
            memset(&rp, 0, sizeof(rp));
            rp.stage = REC_STARTS;
            rp.numItems = span;
            rp.recOff = p->dRecOff.p;
            rp.numRecords = (int)p->recOff.size() - 1;
            rp.firstHit = lo;
            rp.cols = const_cast<int*>(dCols);
            rp.starts = dStart.p;
            be->launch_record(rp);
        }
        be->d2h(out->starts + lo, dStart.p, (size_t)span * sizeof(int));
        stats.d2hBytes += 4LL * span;
        if (!path) continue;
        // every hit of the slice has its script length: one scan places them in hit order
        be->launch_scan(dLen.p, span);
        be->d2h(lenScan.data(), dLen.p, ((size_t)span + 1) * sizeof(int));
        const int bytes = lenScan[(size_t)span];
        DevBuf<uint8_t> dPool(be, (size_t)std::max(bytes, 1));
        hp.pool = dPool.p;
        hp.stage = HR_PATH_COPY;
        for (auto& c : done) {
            hp.nw = c->nw;
            hp.numItems = c->jobs;
            hp.jobHit = c->dJobHit.p;
            hp.opsStride = c->opsStride;
            hp.ops = c->dOps.p;
            hp.opsStart = c->dOpsStart.p;
            be->launch_hit_res(hp);
        }
        unsigned char* grown = static_cast<unsigned char*>(realloc(out->alignments, (size_t)std::max(poolAt + bytes, 1LL)));
        if (!grown) throw std::runtime_error("out of memory for the hit alignments");
        out->alignments = grown;
        if (bytes) be->d2h(out->alignments + poolAt, dPool.p, (size_t)bytes);
        for (int h = 0; h < span; ++h) out->alignmentOffsets[lo + h + 1] = poolAt + lenScan[(size_t)h + 1];
        poolAt += bytes;
        stats.d2hBytes += (long long)bytes + 4LL * (span + 1);
    }
    int err = 0;
    dErr.download(&err, 1);
    if (err) throw std::runtime_error("internal: a start-location / path sweep of a hit disagrees with its score");
    trace.mark(path ? "hits: starts and paths" : "hits: starts");
}
}  // namespace eb
