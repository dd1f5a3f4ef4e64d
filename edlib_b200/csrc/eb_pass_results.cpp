// eb_pass_results.cpp -- the remaining phases of a compute pass: warp-per-alignment distance sweeps,
// assembly of distances and end locations (ref cpp:221-225, 658-693), start locations by reversed sweeps
// (ref cpp:228-272), alignment paths (stored-matrix traceback and Hirschberg, ref cpp:276-289, 1161-1396).
#include "eb_engine_internal.h"

namespace eb {

// HW sweeps of long queries over a long target.  The reference keeps these cheap with its band (ref cpp:601-642:
// only the blocks within k of the best diagonal are computed, k doubling from 64, cpp:199-217); here the same
// doubling drives exact seed levels: with threshold t, t+1 disjoint seeds of the query are looked up in the index
// of the target, and the whole query is swept over windows around the end columns their occurrences imply -- by
// the warp kernel, its 1024*R-row window sliding down the <= (4t+1 + spread) diagonals that matter.  A query is
// decided when a window holds a distance <= t.  What no level decides (distances above the largest threshold,
// repeats) is swept over the whole target cut into chunks that restart 2m columns early (no HW path spans more
// than 2m target symbols), so that even one query fills the machine.
void Pass::long_hw_distance(const std::vector<int>& pairs) {
    std::map<int, std::vector<int>> byTarget;
    for (int pair : pairs) byTarget[p->tidx[pair]].push_back(pair);
    for (auto& kv : byTarget) {
        const int t = kv.first;
        const Target& tg = p->tg[t];
        const int n = tg.len;
        const std::vector<int>& list = kv.second;
        const int G = (int)list.size();
        std::vector<int> bound(G), excl(G, -1), cur(G);
        for (int s = 0; s < G; ++s) {
            const int m = p->qlen[list[s]];
            bound[s] = (k < 0 || k > m) ? m : k;
            cur[s] = s;
            stats.wCells += (long long)m * n;
        }
        auto decide = [&](int s, int b, int c, const std::vector<int>& positions) {
            const int pair = list[s];
            best[pair] = c > 0 ? b : 0x7fffffff;
            cnt[pair] = c;
            posStart[pair] = (long long)posPool.size();
            posPool.insert(posPool.end(), positions.begin(), positions.end());
            posLen[pair] = (int)positions.size();
        };
        // ---- seed levels with doubling thresholds ----
        const bool seeds = !p->hasEq && tun.filterSeedK > 0 && tun.longSeedMaxK > 0 && n >= tun.filterMinTarget && seed_index(t) &&
                           seedIdx->Ls[0] > 0;
        std::vector<int> rest;  // reads for the chunked sweep
        if (!seeds) {
            rest.swap(cur);
        }
        for (int thrCap = 64; !cur.empty(); thrCap *= 2) {
            const int L = seedIdx->Ls[0];
            std::vector<int> in, rl, thr, top;
            for (int s : cur) {
                const int m = p->qlen[list[s]];
                const int tp = std::min(std::min(bound[s], m / L - 1), tun.longSeedMaxK);
                const int tt = std::min(tp, thrCap);
                if (m >= 2 * L && tt > excl[s]) {
                    in.push_back(s);
                    rl.push_back(list[s]);
                    thr.push_back(tt);
                    top.push_back(tp);
                } else {
                    rest.push_back(s);  // no (higher) threshold this query can be given
                }
            }
            cur.clear();
            if (in.empty()) break;
            const int g = (int)in.size();
            DevBuf<int> dList(be, g), dThr(be, g), dCount(be, 1);
            dList.upload(rl.data(), g);
            dThr.upload(thr.data(), g);
            DevBuf<SeedPlan> dPlan(be, g);
            SeedPlanParams sp = seed_plan_params(tg, 0);
            sp.readList = dList.p;
            sp.thr = dThr.p;
            sp.seedK = tun.longSeedMaxK;
            sp.numReads = g;
            sp.maxBucket = tun.filterSeedBucket * 8;
            sp.level = SEED_LEVELS - 1;  // the largest candidate capacity
            sp.plan = dPlan.p;
            WinJobs jobs;
            jobs.count = dCount.p;
            be->zero(dCount.p, sizeof(int));
            const int V = plan_windows(sp, jobs, g * 64 + 1024, true);
            std::vector<SeedPlan> plan(g);
            dPlan.download(plan.data(), g);
            std::vector<int> hStart(V), hLen(V), hTf(V);
            if (V) {
                jobs.start.download(hStart.data(), V);
                jobs.len.download(hLen.data(), V);
                jobs.tf.download(hTf.data(), V);
            }
            stats.filterWindows += V;
            stats.d2hBytes += 16LL * g + 12LL * V;
            std::vector<WTask> tasks;
            std::vector<int> taskFirst(g + 1, 0);
            for (int i = 0; i < g; ++i) {
                taskFirst[i] = (int)tasks.size();
                if (plan[i].state != SEED_WINDOWS) continue;
                const int pair = list[in[i]], m = p->qlen[pair], tt = thr[i];
                for (int w = plan[i].first; w < plan[i].first + plan[i].count; ++w) {
                    const int hi = hLen[w] - 1, lo = hTf[w];
                    const int dhi = hi - (m - 1) + tt;
                    const WPlan pl = plan_w_band(m, (long long)(hi - lo) + 2LL * tt + 1, dhi);
                    WTask tk;
                    tk.pair = pair;
                    tk.qOff = p->qoff[pair];
                    tk.tOff = tg.off + (uint64_t)hStart[w];
                    tk.m = m;
                    tk.n = hLen[w];
                    tk.mode = MODE_HW;
                    tk.flags = pl.slide ? WF_SLIDE : 0;
                    tk.dhi = pl.dhi;
                    tk.R = pl.R;
                    tk.nWp = pl.nWp;
                    tk.kInit = tt + 1;
                    tk.trackFrom = lo;
                    tk.tag = hStart[w];  // columns of the task are relative to the window
                    tk.wantPositions = true;
                    tasks.push_back(std::move(tk));
                }
            }
            taskFirst[g] = (int)tasks.size();
            runner.run(tasks);
            if (trace.on)
                fprintf(stderr, "[edlib_b200] long HW queries, seed threshold <= %d: %d queries, %d windows (%zu sliding)\n", thrCap, g, V,
                        (size_t)std::count_if(tasks.begin(), tasks.end(), [](const WTask& x) { return (x.flags & WF_SLIDE) != 0; }));
            for (int i = 0; i < g; ++i) {
                const int s = in[i], tt = thr[i];
                if (plan[i].state == SEED_SATURATED) {  // repeats / too many candidates: the chunked sweep takes it
                    rest.push_back(s);
                    continue;
                }
                int b = 0x7fffffff;
                for (int q = taskFirst[i]; q < taskFirst[i + 1]; ++q)
                    if (tasks[q].rec.cnt > 0 && tasks[q].rec.best < b) b = tasks[q].rec.best;
                if (b <= tt) {
                    std::vector<int> positions;
                    for (int q = taskFirst[i]; q < taskFirst[i + 1]; ++q) {
                        const WTask& tk = tasks[q];
                        if (tk.rec.cnt <= 0 || tk.rec.best != b) continue;
                        for (int x = 0; x < std::min(tk.rec.cnt, KPOS); ++x) positions.push_back(tk.tag + tk.rec.pos[x]);
                        for (int x : tk.extra) positions.push_back(tk.tag + x);
                    }
                    decide(s, b, (int)positions.size(), positions);
                    stats.filterDecided++;
                    continue;
                }
                excl[s] = tt;  // no alignment within tt
                if (tt == bound[s]) {
                    decide(s, 0, 0, std::vector<int>());  // ... which is the caller's bound: final
                    stats.filterDecided++;
                } else if (top[i] > tt) {
                    cur.push_back(s);  // next level: twice the threshold
                } else {
                    rest.push_back(s);
                }
            }
        }
        cur.swap(rest);
        std::sort(cur.begin(), cur.end());
        if (cur.empty()) continue;
        // ---- chunked sweeps of the whole target ----
        stats.filterFallback += (long long)cur.size();
        std::vector<WTask> tasks;
        std::vector<int> taskFirst(cur.size() + 1, 0);
        const long long wantTasks = 4LL * be->sm_count() * 4;  // a few warps per SM sub-partition
        for (size_t i = 0; i < cur.size(); ++i) {
            taskFirst[i] = (int)tasks.size();
            const int s = cur[i], pair = list[s], m = p->qlen[pair];
            // chunks of >= 2m columns (each re-sweeps a 2m halo): a handful of queries is latency-bound per warp, so more,
            // shorter chunks finish sooner even though the halos double the work; many queries get chunks of >= 6m
            const long long minChunk = ((long long)cur.size() * 8 <= wantTasks ? 2LL : 6LL) * m;
            long long chunks = std::max<long long>(1, std::min<long long>(n / minChunk, (wantTasks + (long long)cur.size() - 1) / (long long)cur.size()));
            const int chunkLen = (int)round_up((size_t)((n + chunks - 1) / chunks), 16);
            for (long long cs = 0; cs < n; cs += chunkLen) {
                const long long ce = std::min<long long>(cs + chunkLen, n);
                const long long hs = std::max<long long>(0, cs - 2LL * m);
                const WPlan pl = plan_w(m, (int)(ce - hs), MODE_HW, -1);
                WTask tk;
                tk.pair = pair;
                tk.qOff = p->qoff[pair];
                tk.tOff = tg.off + (uint64_t)hs;
                tk.m = m;
                tk.n = (int)(ce - hs);
                tk.mode = MODE_HW;
                tk.flags = 0;
                tk.R = pl.R;
                tk.nWp = pl.nWp;
                tk.kInit = bound[s] + 1;
                tk.trackFrom = (int)(cs - hs);
                tk.tag = (int)hs;
                tk.wantPositions = true;
                tasks.push_back(std::move(tk));
            }
        }
        taskFirst[cur.size()] = (int)tasks.size();
        runner.run(tasks);
        if (trace.on) fprintf(stderr, "[edlib_b200] long HW queries, chunked sweeps: %zu queries, %zu chunks\n", cur.size(), tasks.size());
        for (size_t i = 0; i < cur.size(); ++i) {
            int b = 0x7fffffff;
            for (int q = taskFirst[i]; q < taskFirst[i + 1]; ++q)
                if (tasks[q].rec.cnt > 0 && tasks[q].rec.best < b) b = tasks[q].rec.best;
            std::vector<int> positions;
            for (int q = taskFirst[i]; q < taskFirst[i + 1]; ++q) {
                const WTask& tk = tasks[q];
                if (tk.rec.cnt <= 0 || tk.rec.best != b) continue;
                for (int x = 0; x < std::min(tk.rec.cnt, KPOS); ++x) positions.push_back(tk.tag + tk.rec.pos[x]);
                for (int x : tk.extra) positions.push_back(tk.tag + x);
            }
            decide(cur[i], b, (int)positions.size(), positions);
        }
    }
}

// Distance pass of everything else: one alignment per warp (or per thread with its own target).
void Pass::warp_distance() {
    // ---- HW, long queries over long targets: seeds + chunks (long_hw_distance) ----
    if (mode == MODE_HW) {
        std::vector<int> longHw, rest;
        for (int pair : wPairs) {
            const int m = p->qlen[pair], n = p->tlen[pair];
            if (m > 256 && n >= tun.longHwMinTarget && (long long)n >= 8LL * m) longHw.push_back(pair);
            else rest.push_back(pair);
        }
        if (!longHw.empty()) {
            long_hw_distance(longHw);
            wPairs.swap(rest);
        }
    }
    // ---- W distance pass ------------------------------------------------------------------
    {
        std::vector<int> pending = wPairs;
        int kRound = 64;  // ref cpp:201: the doubling schedule only matters for speed
        while (!pending.empty()) {
            std::vector<WTask> tasks;
            std::vector<int> later;
            for (int pair : pending) {
                const int m = p->qlen[pair], n = p->tlen[pair];
                int bound = -1;
                if (mode == MODE_NW) {
                    if (k >= 0) {
                        bound = k;
                    } else if (ceil_div(m, 32) > 32) {
                        bound = kRound;
                        if (bound < abs(n - m)) {
                            later.push_back(pair);
                            continue;
                        }
                    }
                }
                // SHW: D[m-1][e] >= e + 1 - m, so columns beyond m + (largest accepted distance) hold no end location
                const int nEff = mode == MODE_SHW ? (int)std::min<long long>(n, (long long)m + ((k < 0 || k > m) ? m : k)) : n;
                WPlan pl = plan_w(m, nEff, mode, bound);
                WTask t;
                t.pair = pair;
                t.qOff = p->qoff[pair];
                t.tOff = p->tg[p->tidx[pair]].off;
                t.m = m;
                t.n = nEff;
                t.mode = mode;
                t.flags = pl.slide ? WF_SLIDE : 0;
                t.dhi = pl.dhi;
                t.bandH = pl.height;
                t.R = pl.R;
                t.nWp = pl.nWp;
                t.kInit = ((k < 0 || k > m) ? m : k) + 1;
                t.tag = pl.slide ? bound : -1;  // a sliding result is only valid when <= bound
                t.wantPositions = (mode != MODE_NW);
                tasks.push_back(std::move(t));
            }
            runner.run(tasks);
            for (WTask& t : tasks) {
                stats.wCells += (long long)t.m * t.n;
                if (t.tag >= 0 && t.rec.best > t.tag) {  // outside the band of this round
                    if (k < 0) later.push_back(t.pair);
                    else best[t.pair] = 0x7fffffff;
                    continue;
                }
                best[t.pair] = t.rec.cnt > 0 ? t.rec.best : 0x7fffffff;
                cnt[t.pair] = t.rec.cnt;
                posStart[t.pair] = (long long)posPool.size();
                for (int q = 0; q < std::min(t.rec.cnt, KPOS); ++q) posPool.push_back(t.rec.pos[q]);
                posPool.insert(posPool.end(), t.extra.begin(), t.extra.end());
                posLen[t.pair] = (int)((long long)posPool.size() - posStart[t.pair]);
            }
            pending.swap(later);
            if (kRound < (1 << 29)) kRound *= 2;
        }
    }
}

// editDistance and endLocations from the sweep outcomes held in the host vectors (ref cpp:219-225 and the -1
// rule), appended to the batch's end-location pool: of every pair (pairs == nullptr) or of the listed ones (the
// rest was assembled on the device).
void Pass::collect_ends(const std::vector<int>* pairs) {
    // ---- counts per pair, offsets, fill (on a few host threads) -------
    // ref cpp:670, 681-693: the padded bottom cell of column W-1 shows up as end location -1
    auto accepted = [&](int i) -> int {  // number of end locations of pair i, or -1 if it has no result
        if (p->special[i]) return -1;
        if (best[i] < 0 || best[i] == 0x7fffffff) return -1;  // rejected up front or nothing tracked
        if (k >= 0 && best[i] > k) return -1;
        if (mode == MODE_NW) return 1;
        const int m = p->qlen[i];
        if (best[i] > m) return -1;
        const int W64 = ceil_div(m, 64) * 64 - m;
        return posLen[i] + ((best[i] == m && W64 > 0) ? 1 : 0);
    };
    const size_t M = pairs ? pairs->size() : (size_t)N;
    auto pair_of = [&](size_t j) -> int { return pairs ? (*pairs)[j] : (int)j; };
    const size_t nparts = host_parts(M, 65536);
    std::vector<long long> partCount(nparts + 1, 0);
    std::vector<int> bad(nparts, 0);
    auto run = [&](const std::function<void(size_t, size_t, size_t)>& fn) {
        HostPool::get().run(nparts, [&](size_t t) { fn(t, M * t / nparts, M * (t + 1) / nparts); });
    };
    run([&](size_t t, size_t lo, size_t hi) {
        long long c = 0;
        for (size_t j = lo; j < hi; ++j) {
            const int i = pair_of(j);
            const int a = accepted(i);
            if (a > 0) c += a;
            if (a >= 0 && mode != MODE_NW && posLen[i] != cnt[i]) bad[t] = 1;
        }
        partCount[t + 1] = c;
    });
    const long long base = (long long)p->endPool.size();  // behind the regions the device filled
    partCount[0] = base;
    for (size_t t = 0; t < nparts; ++t) {
        if (bad[t]) throw std::runtime_error("internal: end-location count mismatch");
        partCount[t + 1] += partCount[t];
    }
    p->endPool.resize((size_t)partCount[nparts]);
    run([&](size_t t, size_t lo, size_t hi) {
        long long at = partCount[t];
        for (size_t j = lo; j < hi; ++j) {
            const int i = pair_of(j);
            p->endStart[i] = at;
            const int a = accepted(i);
            if (a < 0) {
                p->ed[i] = -1;
                p->endCount[i] = 0;
                continue;
            }
            p->ed[i] = best[i];
            p->endCount[i] = a;
            if (mode == MODE_NW) {
                p->endPool[(size_t)at++] = p->tlen[i] - 1;  // ref cpp:221-225
                continue;
            }
            if (a > posLen[i]) p->endPool[(size_t)at++] = -1;
            if (posLen[i]) memcpy(p->endPool.data() + at, posPool.data() + posStart[i], sizeof(int) * (size_t)posLen[i]);
            at += posLen[i];
        }
    });
}

// =============================================================================================
// Start locations and paths of short queries (<= 256 rows) driven from the device.  A read set needs one reversed
// sweep per end location and one matrix-storing sweep + traceback per read: millions of tiny jobs.  Their
// descriptors are derived on the device from the per-pair results (eb_core.h: res_item), the lane / traceback
// kernels run on those lists, and the outcome lands in the batch's start-location pool and in a dense pool of edit
// scripts that comes back in one copy per slice -- the host neither builds nor walks per-job objects.
// =============================================================================================
void Pass::res_begin() {
    if (resUploaded) return;
    resUploaded = true;
    // word classes that hold found pairs; bit 0: found pairs the lane kernel cannot take (long queries, big alphabets)
    const size_t nparts = host_parts((size_t)N, 65536);
    std::vector<unsigned> part(nparts, 0u);
    HostPool::get().run(nparts, [&](size_t t) {
        unsigned bits = 0;
        for (size_t i = (size_t)N * t / nparts, hi = (size_t)N * (t + 1) / nparts; i < hi; ++i) {
            if (p->ed[i] < 0 || p->special[i]) continue;
            const int m = p->qlen[i];
            bits |= (m > 0 && m <= 256) ? (1u << ((m + 31) / 32)) : 1u;
        }
        part[t] = bits;
    });
    resClasses = 0;
    for (unsigned b : part) resClasses |= b;
    for (int nw = 1; nw <= 8; ++nw)
        if (((resClasses >> nw) & 1u) && !lane_ok(32 * nw)) resClasses = (resClasses & ~(1u << nw)) | 1u;
    if (!tun.deviceResults) resClasses = (resClasses & ~0x1feu) | ((resClasses & 0x1feu) ? 1u : 0u);
    if (!(resClasses & 0x1feu)) return;
    rEd.alloc(be, (size_t)N);
    rEndCount.alloc(be, (size_t)N);
    rEndStart.alloc(be, (size_t)N);
    rEndPool.alloc(be, p->endPool.size());
    rEd.upload(p->ed.data(), (size_t)N);
    rEndCount.upload(p->endCount.data(), (size_t)N);
    rEndStart.upload(p->endStart.data(), (size_t)N);
    rEndPool.upload(p->endPool.data(), p->endPool.size());
    stats.h2dBytes += 16LL * N + 4LL * (long long)p->endPool.size();
    if (p->tg.size() > 1) {
        HostBuf<uint64_t> offs(be, (size_t)N);
        parallel_ranges((size_t)N, 65536, [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) offs[i] = p->tg[p->tidx[i]].off;
        });
        rTOffPair.alloc(be, (size_t)N);
        rTOffPair.upload(offs.p, (size_t)N);
        be->sync();  // the staging block goes back to the cache
        stats.h2dBytes += 8LL * N;
    }
    rErr.alloc(be, 1);
    be->zero(rErr.p, sizeof(int));
}

void Pass::res_fill(ResParams& rp, int nw) {
    memset(&rp, 0, sizeof(rp));
    rp.nw = nw;
    rp.numPairs = N;
    rp.ed = rEd.p;
    rp.endCount = rEndCount.p;
    rp.endStart = rEndStart.p;
    rp.endPool = rEndPool.p;
    rp.qlen = p->dQlen.p;
    rp.qoff = p->dQoff.p;
    rp.tOffPair = p->tg.size() > 1 ? rTOffPair.p : nullptr;
    rp.tOff0 = p->tg.empty() ? 0 : p->tg[0].off;
    rp.startPool = rStartPool.p;
    rp.err = rErr.p;
}

void Pass::res_check() {
    int err = 0;
    rErr.download(&err, 1);
    if (err) throw std::runtime_error("internal: a start-location / path sweep disagrees with the distance");
}

// HW start locations (ref cpp:228-272) of every found pair of the lane kernel's word classes.
void Pass::start_locations_device() {
    res_begin();
    if (!(resClasses & 0x1feu)) return;
    rStartPool.alloc(be, p->endPool.size());
    be->zero(rStartPool.p, p->endPool.size() * sizeof(int));
    DevBuf<int> dCnt(be, (size_t)N + 1);
    for (int nw = 1; nw <= 8; ++nw) {
        if (!((resClasses >> nw) & 1u)) continue;
        ResParams rp;
        res_fill(rp, nw);
        rp.cnt = dCnt.p;
        rp.stage = RS_LOC_COUNT;
        rp.numItems = N;
        be->launch_res(rp);
        be->launch_scan(dCnt.p, N);
        int T = 0;
        be->d2h(&T, dCnt.p + N, sizeof(int));
        if (T <= 0) continue;
        DevBuf<LJob> dJobs(be, (size_t)T);
        DevBuf<int> dJobPair(be, (size_t)T);
        DevBuf<long long> dJobSlot(be, (size_t)T);
        DevBuf<Rec> dRecs(be, (size_t)T);
        rp.jobs = dJobs.p;
        rp.jobPair = dJobPair.p;
        rp.jobSlot = dJobSlot.p;
        rp.recs = dRecs.p;
        rp.stage = RS_LOC_JOBS;
        rp.numItems = T;
        be->launch_res(rp);
        LParams lp{dJobs.p, T, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr, dRecs.p, nullptr, 1};
        be->launch_lane(lp, nw, MODE_SHW, true, false);
        rp.stage = RS_LOC_APPLY;
        be->launch_res(rp);
    }
    be->d2h(p->startPool.data(), rStartPool.p, p->endPool.size() * sizeof(int));
    stats.d2hBytes += 4LL * (long long)p->endPool.size();
    res_check();
    trace.mark("starts: device-driven lane sweeps");
}

// Paths (ref cpp:276-289, 1161-1213: inside the 1 MiB rule for every query of <= 256 rows) of the first (start, end)
// of every found pair of the lane kernel's word classes: matrix-storing sweep + traceback per pair, in slices of pairs
// whose stored matrices fit the slice budget; the scripts are compacted on the device and copied into alnPool.
void Pass::paths_device() {
    res_begin();
    if (!(resClasses & 0x1feu)) return;
    if (!rStartPool.p) {  // (start locations were not computed through the device path: cannot happen for PATH)
        rStartPool.alloc(be, p->startPool.size());
        rStartPool.upload(p->startPool.data(), p->startPool.size());
    }
    int maxEd = 0;
    {
        const size_t nparts = host_parts((size_t)N, 65536);
        std::vector<int> part(nparts, 0);
        HostPool::get().run(nparts, [&](size_t t) {
            int mx = 0;
            for (size_t i = (size_t)N * t / nparts, hi = (size_t)N * (t + 1) / nparts; i < hi; ++i) mx = std::max(mx, p->ed[i]);
            part[t] = mx;
        });
        for (int v : part) maxEd = std::max(maxEd, v);
    }
    resMaxEd = maxEd;
    DevBuf<long long> dAlnStart(be, (size_t)N);
    DevBuf<int> dAlnLen(be, (size_t)N);
    be->fill(dAlnStart.p, 0xff, (size_t)N * sizeof(long long));  // -1: no path
    be->zero(dAlnLen.p, (size_t)N * sizeof(int));
    long long poolAt = (long long)p->alnPool.size();
    for (int nw = 1; nw <= 8; ++nw) {
        if (!((resClasses >> nw) & 1u)) continue;
        const uint64_t maxN = (uint64_t)res_max_path_n(nw);  // target slice of a path: at most m + distance symbols
        const uint64_t matStride = maxN * (uint64_t)nw, opsStride = (uint64_t)32 * nw + maxN;
        const size_t perJob = (size_t)matStride * sizeof(U2) + (size_t)opsStride + sizeof(LJob) + sizeof(TbJob) + sizeof(Rec) + 64;
        // pairs per slice: the stored matrices fit the budget, and the scripts of a slice stay countable in an int
        const size_t byScripts = (size_t)0x7fffffff / (size_t)std::max<uint64_t>(opsStride, 1);
        const int S = (int)std::max<size_t>(64, std::min<size_t>(std::min<size_t>((size_t)N, byScripts), tun.pathSliceBytes / perJob));
        DevBuf<int> dCnt(be, (size_t)S + 1), dLen(be, (size_t)S + 1);
        for (int first = 0; first < N; first += S) {
            const int last = std::min(N, first + S), span = last - first;
            ResParams rp;
            res_fill(rp, nw);
            rp.firstPair = first;
            rp.lastPair = last;
            rp.maxPathN = (int)maxN;
            rp.cnt = dCnt.p;
            rp.stage = RS_PATH_FLAG;
            rp.numItems = span;
            be->launch_res(rp);
            be->launch_scan(dCnt.p, span);
            int J = 0;
            be->d2h(&J, dCnt.p + span, sizeof(int));
            if (J <= 0) continue;
            DevBuf<LJob> dJobs(be, (size_t)J);
            DevBuf<TbJob> dTb(be, (size_t)J);
            DevBuf<int> dJobPair(be, (size_t)J), dOpsStart(be, (size_t)J), dOpsLen(be, (size_t)J);
            DevBuf<Rec> dRecs(be, (size_t)J);
            DevBuf<U2> dMat(be, (size_t)ceil_div(J, 32) * 32 * matStride);
            DevBuf<uint8_t> dOps(be, (size_t)J * opsStride);
            rp.jobs = dJobs.p;
            rp.tb = dTb.p;
            rp.jobPair = dJobPair.p;
            rp.recs = dRecs.p;
            rp.matStride = matStride;
            rp.opsStride = opsStride;
            rp.stage = RS_PATH_JOBS;
            be->launch_res(rp);
            LParams lp{dJobs.p, J, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr, dRecs.p, dMat.p, 32};
            be->launch_lane(lp, nw, MODE_NW, false, true);
            TbParams tp{dTb.p, J, dMat.p, nullptr, p->dSeq.p, p->dSeq.p, p->hasEq ? p->dEqtab.p : nullptr, p->ncodes,
                        dOps.p, dOpsStart.p, dOpsLen.p, 32};
            be->launch_traceback(tp);
            rp.cnt = dLen.p;
            rp.ops = dOps.p;
            rp.opsStart = dOpsStart.p;
            rp.opsLen = dOpsLen.p;
            rp.stage = RS_PATH_LEN;
            rp.numItems = J;
            be->launch_res(rp);
            be->launch_scan(dLen.p, J);
            int bytes = 0;
            be->d2h(&bytes, dLen.p + J, sizeof(int));
            DevBuf<uint8_t> dAln(be, (size_t)std::max(bytes, 1));
            rp.alnPool = dAln.p;
            rp.alnBase = poolAt;
            rp.alnStart = dAlnStart.p;
            rp.alnLen = dAlnLen.p;
            rp.stage = RS_PATH_COPY;
            be->launch_res(rp);
            p->alnPool.resize((size_t)(poolAt + bytes));
            if (bytes) be->d2h(p->alnPool.data() + poolAt, dAln.p, (size_t)bytes);
            poolAt += bytes;
            stats.d2hBytes += (long long)bytes + 8;
        }
    }
    // per-pair script positions: the device wrote the pairs it handled, the others stay at -1 / 0
    be->d2h(p->alnStart.data(), dAlnStart.p, (size_t)N * sizeof(long long));
    be->d2h(p->alnLen.data(), dAlnLen.p, (size_t)N * sizeof(int));
    stats.d2hBytes += 12LL * N;
    res_check();
    trace.mark("paths: device-driven leaf sweeps + tracebacks");
}

void Pass::start_locations() {
    // ---- start locations (ref cpp:228-272) ------------------------------------------------
    const bool wantLoc = p->cfg.task == EDLIB_TASK_LOC || p->cfg.task == EDLIB_TASK_PATH;
    if (wantLoc) {
        p->startPool.resize(p->endPool.size());
        if (mode != MODE_HW) {
            parallel_ranges(p->startPool.size(), 1 << 20, [&](size_t lo, size_t hi) { memset(p->startPool.data() + lo, 0, (hi - lo) * sizeof(int)); });
        } else {
            start_locations_device();  // every found pair of the lane kernel's word classes (or nothing)
            if (!(resClasses & 0x1feu))
                parallel_ranges(p->startPool.size(), 1 << 20, [&](size_t lo, size_t hi) { memset(p->startPool.data() + lo, 0, (hi - lo) * sizeof(int)); });
        }
        if (mode == MODE_HW && (resClasses & 1u)) {  // found pairs outside those classes: per-job objects on the host
            std::vector<WTask> tasks;
            std::vector<long long> slotOf;
            std::vector<LJob> lj[9];          // short queries: straight to the lane kernel, per word class
            std::vector<long long> lslot[9];
            std::vector<int> lpair[9];
            for (int i = 0; i < N; ++i) {
                if (p->ed[i] < 0) continue;
                const int m = p->qlen[i];
                if (res_class(m)) continue;  // done on the device
                const bool lane = lane_ok(m);
                for (int q = 0; q < p->endCount[i]; ++q) {
                    p->startPool[(size_t)(p->endStart[i] + q)] = 0;
                    const long long slot = p->endStart[i] + q;
                    const int e = p->endPool[(size_t)slot];
                    if (e < 0) continue;  // ref cpp:237-249: start 0
                    if (lane) {
                        const int nw = ceil_div(m, 32);
                        LJob j;
                        memset(&j, 0, sizeof(j));
                        j.qOff = p->qoff[i];
                        j.tOff = p->tg[p->tidx[i]].off + (uint64_t)e;  // first symbol read, walking backward
                        j.m = m;
                        j.n = (int)std::min<long long>((long long)e + 1, (long long)m + p->ed[i]);
                        j.kInit = p->ed[i] + 1;
                        lj[nw].push_back(j);
                        lslot[nw].push_back(slot);
                        lpair[nw].push_back(i);
                        continue;
                    }
                    WTask t;
                    t.pair = i;
                    t.qOff = p->qoff[i];
                    t.tOff = p->tg[p->tidx[i]].off + (uint64_t)e;  // first symbol read, walking backward
                    t.m = m;
                    t.n = (int)std::min<long long>((long long)e + 1, (long long)m + p->ed[i]);
                    t.mode = MODE_SHW;
                    t.flags = WF_QREV | WF_TREV;
                    t.kInit = p->ed[i] + 1;
                    // the reversed alignment has distance ed: it stays within ed diagonals of the main one, so the
                    // window only has to slide down that band (every last-row score <= ed is exact, larger ones can
                    // only come out larger; ref cpp:253-257 sweeps the same columns with k = ed)
                    WPlan pl = plan_w_band(t.m, 2LL * p->ed[i] + 1, p->ed[i]);
                    t.R = pl.R;
                    t.nWp = pl.nWp;
                    if (pl.slide) {
                        t.flags |= WF_SLIDE;
                        t.dhi = pl.dhi;
                    }
                    tasks.push_back(std::move(t));
                    slotOf.push_back(slot);
                }
            }
            trace.mark("starts: jobs built");
            for (int nw = 1; nw <= 8; ++nw) {
                if (lj[nw].empty()) continue;
                std::vector<Rec> recs;
                lane_launch(lj[nw], nw, MODE_SHW, true, recs);
                for (size_t j = 0; j < recs.size(); ++j) {
                    if (recs[j].cnt <= 0 || recs[j].best != p->ed[lpair[nw][j]])
                        throw std::runtime_error("internal: start-location sweep disagrees");
                    const int e = p->endPool[(size_t)lslot[nw][j]];
                    p->startPool[(size_t)lslot[nw][j]] = e - recs[j].last;  // ref cpp:260
                }
            }
            trace.mark("starts: lane sweeps");
            runner.run(tasks);
            for (size_t j = 0; j < tasks.size(); ++j) {
                const WTask& t = tasks[j];
                if (t.rec.cnt <= 0 || t.rec.best != p->ed[t.pair]) throw std::runtime_error("internal: start-location sweep disagrees");
                const int e = p->endPool[(size_t)slotOf[j]];
                p->startPool[(size_t)slotOf[j]] = e - t.rec.last;  // ref cpp:260
            }
        }
    }
}

void Pass::paths() {
    // ---- alignment path (ref cpp:276-289, 1161-1213, 1231-1396) ---------------------------
    // obtainAlignment as a level-synchronous tree: a node is an NW sub-problem (query slice,
    // target slice, known score).  Inside the reference's 1 MiB rule (cpp:1188-1190) it is a
    // leaf: matrix-storing sweep + traceback kernel.  Otherwise it is split like
    // obtainAlignmentHirschberg: the score column left of the target's middle from a forward
    // sweep and the one right of it from a reversed sweep (both on the device, cpp:1252-1260),
    // the split row chosen by the reference's candidate order (cpp:1321-1353), both halves
    // becoming nodes of the next level (cpp:1372-1380).  All nodes of a level run in one batch.
    if (p->cfg.task == EDLIB_TASK_PATH) {
        struct Node {
            int pair;
            uint64_t qOff, tOff;
            int m, n, best;
            int left = -1, right = -1;
            long long opsOff = -1;  // into opsPool (leaf) ...
            int opsLen = 0;
            int fillOp = -1;        // ... or a run of one op (empty side, cpp:1168-1175)
        };
        std::vector<Node> nodes;
        std::vector<int> rootOf, frontier, leaves;
        paths_device();  // every found pair of the lane kernel's word classes (or nothing)
        {
            std::atomic<int> open(0);  // found pairs the device did not handle (long queries, long target slices)
            parallel_ranges((size_t)N, 65536, [&](size_t lo, size_t hi) {
                bool any = false;
                for (size_t i = lo; i < hi && !any; ++i) any = p->ed[i] >= 0 && p->alnStart[i] < 0;
                if (any) open.store(1, std::memory_order_relaxed);
            });
            if (!open.load()) return;
        }
        rootOf.assign(N, -1);
        for (int i = 0; i < N; ++i) {
            if (p->ed[i] < 0 || p->alnStart[i] >= 0) continue;  // no result / done on the device
            const int s0 = p->startPool[(size_t)p->endStart[i]], e0 = p->endPool[(size_t)p->endStart[i]];
            Node nd;
            nd.pair = i;
            nd.qOff = p->qoff[i];
            nd.tOff = p->tg[p->tidx[i]].off + (uint64_t)s0;
            nd.m = p->qlen[i];
            nd.n = e0 - s0 + 1;
            nd.best = p->ed[i];
            rootOf[i] = (int)nodes.size();
            frontier.push_back((int)nodes.size());
            nodes.push_back(nd);
        }
        while (!frontier.empty()) {
            std::vector<int> split;
            for (int id : frontier) {
                Node& nd = nodes[id];
                if (nd.m == 0 || nd.n <= 0) {
                    nd.fillOp = (nd.m == 0) ? EDLIB_EDOP_DELETE : EDLIB_EDOP_INSERT;
                    nd.opsLen = nd.m + std::max(nd.n, 0);
                    continue;
                }
                const long long matrixBytes = 20LL * ceil_div(nd.m, 64) * nd.n + 8LL * nd.n;  // cpp:1188-1190
                if (matrixBytes < 1024 * 1024) leaves.push_back(id);
                else split.push_back(id);
            }
            frontier.clear();
            if (split.empty()) break;
            std::vector<WTask> tasks;
            tasks.reserve(split.size() * 2);
            for (int id : split) {
                const Node& nd = nodes[id];
                const int leftW = nd.n / 2, rightW = nd.n - leftW;  // cpp:1247-1248
                const WPlan pl = plan_w(nd.m, nd.n, MODE_NW, nd.best);  // band of the WHOLE node
                WTask f;
                f.pair = id;
                f.qOff = nd.qOff;
                f.tOff = nd.tOff;
                f.m = nd.m;
                f.n = leftW;
                f.mode = MODE_NW;
                f.flags = WF_STOPCOL | (pl.slide ? WF_SLIDE : 0);
                f.dhi = pl.dhi;
                f.stopCol = leftW - 1;
                f.R = pl.R;
                f.nWp = pl.nWp;
                f.splitSide = 0;
                f.splitBest = nd.best;
                WTask r = f;
                r.tOff = nd.tOff + (uint64_t)nd.n - 1;  // reversed: first symbol read is the last one
                r.n = rightW;
                r.flags |= WF_QREV | WF_TREV;
                r.stopCol = rightW - 1;
                r.splitSide = 1;
                tasks.push_back(std::move(f));
                tasks.push_back(std::move(r));
            }
            runner.run(tasks);
            for (size_t s = 0; s < split.size(); ++s) {
                const int id = split[s];
                const Node nd = nodes[id];
                const int leftW = nd.n / 2, rightW = nd.n - leftW;
                const SplitOut& so = tasks[2 * s].split;  // found on the device (split_kernel)
                const int h = so.h;
                if (h < 0) throw std::runtime_error("internal: Hirschberg split not found");
                Node a, b;
                a.pair = b.pair = nd.pair;
                a.qOff = nd.qOff;
                a.tOff = nd.tOff;
                a.m = h;
                a.n = leftW;
                a.best = so.left;
                b.qOff = nd.qOff + (uint64_t)h;
                b.tOff = nd.tOff + (uint64_t)leftW;
                b.m = nd.m - h;
                b.n = rightW;
                b.best = so.right;
                nodes[id].left = (int)nodes.size();
                frontier.push_back((int)nodes.size());
                nodes.push_back(a);
                nodes[id].right = (int)nodes.size();
                frontier.push_back((int)nodes.size());
                nodes.push_back(b);
            }
        }
        {
            std::vector<WTask> tasks;
            std::vector<LJob> lj[9];  // leaves with short queries: lane kernel, per word class
            std::vector<int> lnode[9];
            for (int id : leaves) {
                const Node& nd = nodes[id];
                if (lane_ok(nd.m)) {
                    const int nw = ceil_div(nd.m, 32);
                    LJob j;
                    memset(&j, 0, sizeof(j));
                    j.qOff = nd.qOff;
                    j.tOff = nd.tOff;
                    j.m = nd.m;
                    j.n = nd.n;
                    lj[nw].push_back(j);
                    lnode[nw].push_back(id);
                    continue;
                }
                WTask t;
                t.pair = id;
                t.qOff = nd.qOff;
                t.tOff = nd.tOff;
                t.m = nd.m;
                t.n = nd.n;
                t.mode = MODE_NW;
                t.flags = WF_STORE;
                const WPlan pl = plan_w(nd.m, nd.n, MODE_NW, -1);
                t.R = pl.R;
                t.nWp = pl.nWp;
                tasks.push_back(std::move(t));
            }
            trace.mark("paths: tree + leaf jobs built");
            for (int nw = 1; nw <= 8; ++nw) {
                if (lj[nw].empty()) continue;
                lane_paths(lj[nw], nw, [&](size_t j, const uint8_t* ops, int len, int score) {
                    Node& nd = nodes[lnode[nw][j]];
                    if (score != nd.best) throw std::runtime_error("internal: path sweep disagrees with the distance");
                    nd.opsOff = (long long)opsPool.size();
                    nd.opsLen = len;
                    opsPool.insert(opsPool.end(), ops, ops + len);
                });
            }
            runner.run(tasks);
            for (const WTask& t : tasks) {
                Node& nd = nodes[t.pair];
                if (t.rec.best != nd.best) throw std::runtime_error("internal: path sweep disagrees with the distance");
                nd.opsOff = t.opsOff;
                nd.opsLen = t.opsLen;
            }
        }
        trace.mark("paths: leaf sweeps + tracebacks");
        // in-order concatenation (cpp:1388-1391)
        std::vector<int> stack;
        for (int i = 0; i < N; ++i) {
            if (rootOf[i] < 0) continue;
            p->alnStart[i] = (long long)p->alnPool.size();
            stack.assign(1, rootOf[i]);
            while (!stack.empty()) {
                const int id = stack.back();
                stack.pop_back();
                const Node& nd = nodes[id];
                if (nd.left >= 0) {
                    stack.push_back(nd.right);
                    stack.push_back(nd.left);
                } else if (nd.fillOp >= 0) {
                    p->alnPool.append_fill((size_t)nd.opsLen, (uint8_t)nd.fillOp);
                } else {
                    p->alnPool.append(opsPool.data() + nd.opsOff, (size_t)nd.opsLen);
                }
            }
            p->alnLen[i] = (int)(p->alnPool.size() - (size_t)p->alnStart[i]);
        }
    }
}
}  // namespace eb
