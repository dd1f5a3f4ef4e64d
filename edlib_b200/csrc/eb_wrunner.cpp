// eb_wrunner.cpp -- WRunner: runs a list of warp-per-alignment (and per-job lane) sweeps through the backend
// in slices that respect the device-memory budget, handling the Hirschberg stop-column pairs (eb_engine.h).
#include "eb_engine_internal.h"

namespace eb {

// Window shape of a W job.  Short queries (<= 1024 rows) always fit one fixed window, which is
// exact for any k.  Longer NW jobs with a bound use one window sliding down the Ukkonen band
// (cells with |d| + |delta - d| <= k, d = c - r: ref cpp:755, 799-830 keep the same cells) when
// the band is at most half of the query; everything else is swept unbanded in strips.
WPlan plan_w(int m, int n, int mode, int kBound) {
    WPlan pl;
    const int nW = ceil_div(m, 32);
    pl.slide = false;
    pl.dhi = 0;
    pl.height = 0;
    if (nW <= 32) {
        pl.R = 1;
        pl.nWp = nW;
        return pl;
    }
    pl.nWp = (int)round_up((size_t)nW, 8);
    if (mode == MODE_NW && kBound >= 0) {
        const int d = n - m;
        const int ad = d < 0 ? -d : d;
        const long long h = ((long long)kBound - ad) / 2;
        const long long dlo = std::min(0, d) - h, dhi = std::max(0, d) + h;
        const long long height = dhi - dlo + 1;
        for (int R = 1; R <= 8; R *= 2) {
            if (height + 32LL * R <= 1024LL * R && 64 * R <= nW) {
                pl.R = R;
                pl.slide = true;
                pl.dhi = (int)dhi;
                pl.height = (int)height;
                return pl;
            }
        }
    }
    pl.R = 8;
    for (int R = 2; R <= 8; R *= 2)
        if (32 * R >= pl.nWp) {
            pl.R = R;
            break;
        }
    return pl;
}

// Window shape of a W job whose cells of interest lie on `height` diagonals (an HW window sweep of a long query
// around seed hits): one window sliding down those diagonals when it covers them, strips otherwise.
WPlan plan_w_band(int m, long long height, int dhi) {
    WPlan pl = plan_w(m, 0, MODE_HW, -1);
    const int nW = ceil_div(m, 32);
    if (nW <= 32) return pl;  // one fixed window holds every row
    for (int R = 1; R <= 8; R *= 2) {
        if (height + 32LL * R <= 1024LL * R && 64 * R <= nW) {
            pl.R = R;
            pl.slide = true;
            pl.dhi = dhi;
            pl.height = (int)height;
            return pl;
        }
    }
    return pl;
}

bool WRunner::lane_ok(int nw) {
    if (laneOk[nw] < 0) {
        int bt = 0, rc = 0;
        be->k1_shape(nw, p->ncodes, 0x7fffffff, &bt, &rc);
        laneOk[nw] = rc > 0 ? 1 : 0;
    }
    return laneOk[nw] == 1;
}

size_t WRunner::task_bytes(const WTask& t) const {
    size_t b = (size_t)p->ncodes * t.nWp * 4 + sizeof(WJob) + sizeof(Rec);
    if (t.flags & WF_STORE) b += (size_t)t.n * t.nWp * 8 + (size_t)t.m + t.n + 64;
    if (t.flags & WF_STOPCOL) b += (size_t)t.m * 4;
    if (!(t.flags & WF_SLIDE) && t.nWp / t.R > 32) b += 2 * (size_t)t.n;
    return b;
}

// The band kernel's window must hold the band (bandH diagonals), the 31 rows the window lags behind while it waits
// for the next multiple of 32 columns, and the rows by which its top lies above the band's top diagonal (see band_job).
int WRunner::band_blocks(const WTask& t) const {
    if (!eng->tun.bandKernel || t.flags != WF_SLIDE || t.mode != MODE_NW || t.bandH <= 0 || (t.tOff & 15u)) return 0;
    const int nW = ceil_div(t.m, 32);
    const int off = 32 * nW - t.m;
    int A = off - t.dhi;
    A = (A >= 0) ? 0 : -(((-A) + 31) / 32) * 32;
    const long long rows = (long long)t.bandH + 31 + ((off - t.dhi) - A);
    const long long NB = (rows + 127) / 128;
    if (NB > be->band_max_blocks(p->ncodes) || 4 * NB > nW) return 0;
    return (int)NB;
}

void WRunner::run_band(std::vector<WTask>& tasks, const std::vector<int>& idx, int NB) {
    size_t i = 0;
    while (i < idx.size()) {
        size_t bytes = 0, j = i;
        while (j < idx.size()) {
            const WTask& t = tasks[idx[j]];
            const size_t tb = (size_t)p->ncodes * ceil_div(t.m, 32) * 4 + sizeof(WJob) + sizeof(Rec);
            if (j > i && bytes + tb > eng->tun.sliceBytes) break;
            bytes += tb;
            ++j;
        }
        const int J = (int)(j - i);
        HostBuf<WJob> jobs(be, (size_t)J);
        uint64_t peqWords = 0;
        for (int s = 0; s < J; ++s) {
            const WTask& t = tasks[idx[i + s]];
            WJob& wj = jobs[s];
            memset(&wj, 0, sizeof(wj));
            wj.qOff = t.qOff;
            wj.tOff = t.tOff;
            wj.m = t.m;
            wj.n = t.n;
            wj.nWp = ceil_div(t.m, 32);  // no padding words beyond the last one: the window ends on the last row
            wj.mode = t.mode;
            wj.flags = t.flags;
            wj.kInit = t.kInit;
            wj.dhi = t.dhi;
            wj.rec = s;
            wj.peqOff = peqWords;
            peqWords += (uint64_t)p->ncodes * wj.nWp;
        }
        DevBuf<WJob> dJobs(be, (size_t)J);
        dJobs.upload(jobs.p, (size_t)J);
        DevBuf<uint32_t> dPeq(be, peqWords);
        DevBuf<Rec> dRecs(be, (size_t)J);
        PeqParams pp{dJobs.p, J, p->dSeq.p, dPeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr};
        be->launch_peq(pp);
        WParams wp{dJobs.p, J, p->dSeq.p, p->dSeq.p, dPeq.p, nullptr, nullptr, nullptr, dRecs.p, nullptr, nullptr, 0};
        be->launch_band(wp, NB, p->ncodes);
        if (getenv("EDLIB_B200_TRACE")) fprintf(stderr, "[edlib_b200] band kernel: %d sweeps, window of %d words\n", J, 4 * NB);
        HostBuf<Rec> recs(be, (size_t)J);
        dRecs.download(recs.p, (size_t)J);
        eng->stats.d2hBytes += (long long)J * (long long)sizeof(Rec);
        for (int s = 0; s < J; ++s) {
            WTask& t = tasks[idx[i + s]];
            t.rec = recs[s];
            t.extra.clear();
        }
        i = j;
    }
}

void WRunner::run(std::vector<WTask>& tasks) {
    std::vector<int> warp;
    std::map<std::pair<int, int>, std::vector<int>> lanes;  // (word class, lane class) -> tasks
    std::map<int, std::vector<int>> bands;                  // window blocks -> tasks of the band kernel
    for (size_t i = 0; i < tasks.size(); ++i) {
        const int lc = lane_class(tasks[i]);
        if (lc < 0) {
            const int nb = band_blocks(tasks[i]);
            if (nb > 0) bands[nb].push_back((int)i);
            else warp.push_back((int)i);
        } else {
            lanes[std::make_pair(ceil_div(tasks[i].m, 32), lc)].push_back((int)i);
        }
    }
    for (auto& kv : bands) run_band(tasks, kv.second, kv.first);
    for (auto& kv : lanes) {
        if (!lane_ok(kv.first.first) || (int)kv.second.size() < 8) {  // alphabet too large for per-thread Peq rows / too few to bother
            warp.insert(warp.end(), kv.second.begin(), kv.second.end());
            continue;
        }
        run_lane(tasks, kv.second, kv.first.first, kv.first.second, warp);
    }
    std::vector<int>& order = warp;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return tasks[a].R < tasks[b].R; });
    size_t i = 0;
    while (i < order.size()) {
        const int R = tasks[order[i]].R;
        size_t bytes = 0, j = i;
        while (j < order.size() && tasks[order[j]].R == R) {
            const size_t tb = task_bytes(tasks[order[j]]);
            if (j > i && bytes + tb > eng->tun.sliceBytes && tasks[order[j]].splitSide != 1) break;
            bytes += tb;
            ++j;
        }
        std::vector<int> slice(order.begin() + i, order.begin() + j);
        run_slice(tasks, slice, R, 0);
        i = j;
    }
}

// One class of lane tasks, in memory-bounded slices.  Tasks that need a longer end-location list
// than a record holds are handed to the warp kernel (`spill`), which owns the list machinery.
void WRunner::run_lane(std::vector<WTask>& tasks, const std::vector<int>& idx, int nw, int lc, std::vector<int>& spill) {
    const bool store = lc == 4, rev = lc == 3;
    const int mode = store ? MODE_NW : rev ? MODE_SHW : lc;
    size_t i = 0;
    while (i < idx.size()) {
        size_t bytes = 0, j = i;
        while (j < idx.size()) {
            const WTask& t = tasks[idx[j]];
            const size_t tb = sizeof(LJob) + sizeof(Rec) + (store ? (size_t)t.n * nw * 8 + (size_t)t.m + t.n + 64 : 0);
            if (j > i && bytes + tb > eng->tun.sliceBytes) break;
            bytes += tb;
            ++j;
        }
        const int J = (int)(j - i);
        std::vector<LJob> jobs(J);
        std::vector<TbJob> tb;
        std::vector<int> tbTask;
        uint64_t matEntries = 0, opsBytes = 0;
        for (int s = 0; s < J; ++s) {
            const WTask& t = tasks[idx[i + s]];
            LJob& lj = jobs[s];
            memset(&lj, 0, sizeof(lj));
            lj.qOff = t.qOff;
            lj.tOff = t.tOff;
            lj.m = t.m;
            lj.n = t.n;
            lj.kInit = t.kInit;
            lj.trackFrom = t.trackFrom;
            if (store) {
                lj.matOff = matEntries;
                TbJob b;
                memset(&b, 0, sizeof(b));
                b.matOff = matEntries;
                b.qOff = t.qOff;
                b.peqOff = ~0ull;
                b.tOff = t.tOff;
                b.outOff = opsBytes;
                b.m = t.m;
                b.n = t.n;
                b.nWp = nw;
                tb.push_back(b);
                tbTask.push_back(idx[i + s]);
                matEntries += (uint64_t)t.n * nw;
                opsBytes += (uint64_t)t.m + t.n;
            }
        }
        DevBuf<LJob> dJobs(be, J);
        dJobs.upload(jobs.data(), J);
        DevBuf<Rec> dRecs(be, J);
        be->zero(dRecs.p, (size_t)J * sizeof(Rec));
        DevBuf<U2> dMat(be, matEntries);
        LParams lp{dJobs.p, J, p->dSeq.p, p->dSeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr, dRecs.p, dMat.p, 1};
        be->launch_lane(lp, nw, mode, rev, store);
        if (store) traceback(tasks, tb, tbTask, dMat.p, nullptr);
        HostBuf<Rec> recs(be, (size_t)J);
        dRecs.download(recs.p, J);
        eng->stats.d2hBytes += (long long)J * (long long)sizeof(Rec);
        for (int s = 0; s < J; ++s) {
            WTask& t = tasks[idx[i + s]];
            t.rec = recs[s];
            t.extra.clear();
            if (t.wantPositions && t.rec.cnt > KPOS) spill.push_back(idx[i + s]);
        }
        i = j;
    }
}

// ovfCap == 0: first pass (no position list).  ovfCap > 0: second pass over the tasks whose
// end-location lists exceed KPOS, started from their known minimum with an exact-size list.
void WRunner::run_slice(std::vector<WTask>& tasks, const std::vector<int>& slice, int R, int ovfCap) {
    const int J = (int)slice.size();
    std::vector<WJob> jobs(J);
    uint64_t peqWords = 0, matEntries = 0, colInts = 0, hbytes = 0, opsBytes = 0;
    std::vector<TbJob> tb;
    std::vector<int> tbTask;
    for (int s = 0; s < J; ++s) {
        WTask& t = tasks[slice[s]];
        WJob& j = jobs[s];
        memset(&j, 0, sizeof(j));
        j.qOff = t.qOff;
        j.tOff = t.tOff;
        j.m = t.m;
        j.n = t.n;
        j.nWp = t.nWp;
        j.mode = t.mode;
        j.flags = t.flags;
        j.kInit = t.kInit;
        j.dhi = t.dhi;
        j.stopCol = t.stopCol;
        j.trackFrom = t.trackFrom;
        j.rec = s;
        j.peqOff = peqWords;
        peqWords += (uint64_t)p->ncodes * t.nWp;
        if (t.flags & WF_STORE) {
            j.auxOff = matEntries;
            TbJob b;
            memset(&b, 0, sizeof(b));
            b.matOff = matEntries;
            b.qOff = t.qOff;
            b.peqOff = j.peqOff;
            b.tOff = t.tOff;
            b.outOff = opsBytes;
            b.m = t.m;
            b.n = t.n;
            b.nWp = t.nWp;
            tb.push_back(b);
            tbTask.push_back(slice[s]);
            matEntries += (uint64_t)t.n * t.nWp;
            opsBytes += (uint64_t)t.m + t.n;
        } else if (t.flags & WF_STOPCOL) {
            j.auxOff = colInts;
            colInts += (uint64_t)t.m;
        }
        if (!(t.flags & WF_SLIDE) && t.nWp / R > 32) {
            j.hbufOff = hbytes;
            hbytes += 2 * (uint64_t)t.n;
        }
    }
    DevBuf<WJob> dJobs(be, J);
    dJobs.upload(jobs.data(), J);
    DevBuf<uint32_t> dPeq(be, peqWords);
    DevBuf<U2> dMat(be, matEntries);
    DevBuf<int> dCol(be, colInts);
    DevBuf<uint8_t> dH(be, hbytes);
    DevBuf<Rec> dRecs(be, J);
    be->zero(dRecs.p, (size_t)J * sizeof(Rec));
    DevBuf<Ovf> dOvf(be, (size_t)std::max(ovfCap, 1));
    DevBuf<int> dOvfCount(be, 1);
    be->zero(dOvfCount.p, sizeof(int));
    if (colInts) be->fill(dCol.p, 0x3f, (size_t)colInts * sizeof(int));  // rows outside a sliding window: far above any k
    PeqParams pp{dJobs.p, J, p->dSeq.p, dPeq.p, p->ncodes, p->hasEq ? p->dEqtab.p : nullptr};
    be->launch_peq(pp);
    WParams wp{dJobs.p, J, p->dSeq.p, p->dSeq.p, dPeq.p, dH.p, dMat.p, dCol.p, dRecs.p, dOvf.p, dOvfCount.p, ovfCap};
    be->launch_w(wp, R);
    if (!tb.empty()) traceback(tasks, tb, tbTask, dMat.p, dPeq.p);

    std::vector<Rec> recs(J);
    dRecs.download(recs.data(), J);
    int ovfCount = 0;
    dOvfCount.download(&ovfCount, 1);
    eng->stats.d2hBytes += (long long)J * (long long)sizeof(Rec) + 4;
    for (int s = 0; s < J; ++s) tasks[slice[s]].rec = recs[s];
    if (ovfCap > 0) {
        if (ovfCount > ovfCap) throw std::runtime_error("internal: end-location list larger than counted");
        std::vector<Ovf> ov(ovfCount);
        if (ovfCount) dOvf.download(ov.data(), ovfCount);
        eng->stats.d2hBytes += (long long)ovfCount * (long long)sizeof(Ovf);
        for (int s = 0; s < J; ++s) tasks[slice[s]].extra.clear();
        for (const Ovf& o : ov) {
            WTask& t = tasks[slice[o.rec]];
            if (o.score == t.rec.best) t.extra.push_back(o.pos);
        }
    }
    if (colInts) {
        // Hirschberg halves: the split row is searched on the device, only {h, left, right} come back.
        std::vector<SplitNode> nodes;
        std::vector<int> owner;
        for (int s = 0; s + 1 < J; ++s) {
            const WTask& f = tasks[slice[s]];
            const WTask& r = tasks[slice[s + 1]];
            if (f.splitSide != 0 || r.splitSide != 1) continue;
            SplitNode nd;
            nd.colF = jobs[s].auxOff;
            nd.colR = jobs[s + 1].auxOff;
            nd.m = f.m;
            nd.leftW = f.n;
            nd.rightW = r.n;
            nd.best = f.splitBest;
            nodes.push_back(nd);
            owner.push_back(slice[s]);
        }
        if (nodes.empty()) throw std::runtime_error("internal: stop-column tasks without a split pair");
        DevBuf<SplitNode> dNodes(be, nodes.size());
        dNodes.upload(nodes.data(), nodes.size());
        DevBuf<SplitOut> dOut(be, nodes.size());
        SplitParams sp{dNodes.p, (int)nodes.size(), dCol.p, dOut.p};
        be->launch_split(sp);
        std::vector<SplitOut> outs(nodes.size());
        dOut.download(outs.data(), outs.size());
        eng->stats.d2hBytes += (long long)outs.size() * (long long)sizeof(SplitOut);
        for (size_t q = 0; q < outs.size(); ++q) tasks[owner[q]].split = outs[q];
    }
    if (ovfCap == 0) {
        std::vector<int> again;
        long long need = 0;
        for (int s = 0; s < J; ++s) {
            WTask& t = tasks[slice[s]];
            if (t.wantPositions && t.rec.cnt > KPOS) {
                again.push_back(slice[s]);
                need += t.rec.cnt - KPOS;
                t.kInit = t.rec.best;
            }
        }
        if (need > 0x7fffffffLL / 4) throw std::runtime_error("end-location list too large");
        if (!again.empty()) run_slice(tasks, again, R, (int)need + 16);
    }
}

void WRunner::traceback(std::vector<WTask>& tasks, const std::vector<TbJob>& tb, const std::vector<int>& owner, const U2* mat,
                        const uint32_t* peq) {
    const size_t n = tb.size();
    const uint64_t opsBytes = tb.back().outOff + (uint64_t)tb.back().m + tb.back().n;
    DevBuf<TbJob> dTb(be, n);
    dTb.upload(tb.data(), n);
    DevBuf<uint8_t> dOps(be, opsBytes);
    DevBuf<int> dStart(be, n), dLen(be, n);
    TbParams tp{dTb.p, (int)n, mat, peq, p->dSeq.p, p->dSeq.p, p->hasEq ? p->dEqtab.p : nullptr, p->ncodes,
                dOps.p, dStart.p, dLen.p, 1};
    be->launch_traceback(tp);
    // one pinned staging block for everything that comes back (fast D2H, no zero-fill of vectors)
    const size_t offLn = round_up(n * sizeof(int), 64), offOps = offLn + round_up(n * sizeof(int), 64);
    HostBuf<uint8_t> host(be, offOps + opsBytes);
    const int* st = reinterpret_cast<const int*>(host.p);
    const int* ln = reinterpret_cast<const int*>(host.p + offLn);
    const uint8_t* ops = host.p + offOps;
    be->d2h(host.p, dStart.p, n * sizeof(int));
    be->d2h(host.p + offLn, dLen.p, n * sizeof(int));
    be->d2h(host.p + offOps, dOps.p, opsBytes);
    eng->stats.d2hBytes += (long long)opsBytes + 8LL * (long long)n;
    for (size_t q = 0; q < n; ++q) {
        WTask& t = tasks[owner[q]];
        t.opsOff = (long long)opsPool->size();
        t.opsLen = ln[q];
        opsPool->insert(opsPool->end(), ops + tb[q].outOff + st[q], ops + tb[q].outOff + st[q] + ln[q]);
    }
}
}  // namespace eb
