// TEST INFRASTRUCTURE: calls the seed-stage launches of an eb::Backend directly, over a C ABI for ctypes
// (tests/test_seed_stage.py).  Built twice from this one source: linked to the product library (the CUDA backend) and to
// tests/emul/libedlib_emul.so (the CPU emulation).  Every kernel runs through the backend's own launch_*; the probe only
// uploads the inputs and downloads the outputs.
#include <stdint.h>
#include <string.h>

#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "eb_dispatch.h"
#include "eb_engine_internal.h"

namespace eb {
Backend* create_backend(std::string* err);  // the backend of the library the probe is linked to
}

using namespace eb;

namespace {

Backend* g_be = nullptr;
std::string g_err;
SeedIndex g_index;  // the last probe_build_index, until probe_fetch_index

Backend* backend() {
    if (!g_be) {
        std::string err;
        g_be = create_backend(&err);
        if (!g_be) throw std::runtime_error("create_backend: " + err);
    }
    return g_be;
}

// Device copy of host bytes with the zero padding the kernels may read past the end (as a resident target has).
DevBuf<uint8_t>* upload_codes(Backend* be, const uint8_t* src, size_t bytes) {
    const size_t padded = (bytes + 15) / 16 * 16 + 32;
    auto* d = new DevBuf<uint8_t>(be, padded);
    be->zero(d->p, padded);
    if (bytes) d->upload(src, bytes);
    return d;
}

template <class F>
int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_err = e.what();
        return 1;
    }
}

}  // namespace

extern "C" {

const char* probe_error() { return g_err.c_str(); }

// data[0..count) -> exclusive prefix sums in data[0..count], data[count] the total (Backend::launch_scan).
int probe_scan(int* data, int count) {
    return guarded([&] {
        Backend* be = backend();
        DevBuf<int> d(be, (size_t)count + 1);
        be->fill(d.p, 0xA5, ((size_t)count + 1) * sizeof(int));
        if (count) d.upload(data, (size_t)count);
        be->launch_scan(d.p, count);
        d.download(data, (size_t)count + 1);
    });
}

// Index of an encoded target with the given key length and radix: count -> scan -> fill.
// bucketStart: [sigma^Lidx + 1], positions: [numPos].
int probe_index(const uint8_t* tcodes, int n, int Lidx, int sigma, int numPos, int* bucketStart, int* positions) {
    return guarded([&] {
        Backend* be = backend();
        long long keys = 1;
        for (int x = 0; x < Lidx; ++x) keys *= sigma;
        if (keys > (1LL << 28)) throw std::runtime_error("probe_index: too many keys");
        std::unique_ptr<DevBuf<uint8_t>> t(upload_codes(be, tcodes, (size_t)n));
        DevBuf<int> bs(be, (size_t)keys + 1), cursor(be, (size_t)keys), pos(be, (size_t)numPos);
        be->zero(bs.p, ((size_t)keys + 1) * sizeof(int));
        be->zero(cursor.p, (size_t)keys * sizeof(int));
        be->fill(pos.p, 0xff, (size_t)numPos * sizeof(int));
        SeedIndexParams ip;
        memset(&ip, 0, sizeof(ip));
        ip.tcodes = t->p;
        ip.n = n;
        ip.Lidx = Lidx;
        ip.sigma = sigma;
        ip.numPos = numPos;
        ip.numKeys = (int)keys;
        ip.bucketStart = bs.p;
        ip.cursor = cursor.p;
        ip.positions = pos.p;
        be->launch_seed_count(ip);
        be->launch_scan(bs.p, (int)keys);
        be->launch_seed_fill(ip);
        bs.download(bucketStart, (size_t)keys + 1);
        pos.download(positions, (size_t)numPos);
    });
}

// The engine's own index build (build_seed_index, default tunables) of an encoded target with ncodes codes.
// info: ok, Lidx, sigma, numKeys, Ls[SEED_LEVELS].  The index stays until probe_fetch_index.
int probe_build_index(const uint8_t* tcodes, int n, int ncodes, int* info) {
    return guarded([&] {
        Backend* be = backend();
        std::unique_ptr<DevBuf<uint8_t>> t(upload_codes(be, tcodes, (size_t)n));
        EngineTunables tun;
        g_index.bucketStart.reset();
        g_index.positions.reset();
        const bool ok = build_seed_index(be, tun, g_index, t->p, n, ncodes);
        be->sync();
        info[0] = ok ? 1 : 0;
        info[1] = g_index.Lidx;
        info[2] = g_index.sigma;
        info[3] = g_index.numKeys;
        for (int l = 0; l < SEED_LEVELS; ++l) info[4 + l] = g_index.Ls[l];
    });
}
int probe_fetch_index(int* bucketStart, int* positions) {
    return guarded([&] {
        g_index.bucketStart.download(bucketStart, (size_t)g_index.numKeys + 1);
        g_index.positions.download(positions, (size_t)g_index.n);
        g_index.bucketStart.reset();
        g_index.positions.reset();
    });
}

// One launch_seed_plan over host inputs.
//   ip: kBound, seedK, maxLen, Ls, Lidx, sigma, maxBucket, level, spread, winCap, firstPair
//   readList / thr: [numReads] or null.  queries: codes, qoff [numPairs], qlen [numPairs].
//   Outputs: plan [4 * numReads] (first, count, state, thr), win [5 * winCap] (pair, k, start, len, tf; slots never
//   written are -1), winCount, instance [3] (CAP, THREADS, GW of the kernel instance the launch takes).
int probe_plan(const uint8_t* tcodes, int n, const uint8_t* qcodes, size_t qbytes, const uint64_t* qoff, const int* qlen,
               int numPairs, const int* readList, const int* thr, int numReads, const int* ip, const int* bucketStart,
               int numKeys, const int* positions, int numPos, int* plan, int* win, int* winCount, int* instance) {
    return guarded([&] {
        Backend* be = backend();
        std::unique_ptr<DevBuf<uint8_t>> t(upload_codes(be, tcodes, (size_t)n));
        std::unique_ptr<DevBuf<uint8_t>> q(upload_codes(be, qcodes, qbytes));
        DevBuf<uint64_t> dQoff(be, (size_t)numPairs);
        DevBuf<int> dQlen(be, (size_t)numPairs), dList(be, (size_t)numReads), dThr(be, (size_t)numReads);
        DevBuf<int> dBs(be, (size_t)numKeys + 1), dPos(be, (size_t)numPos);
        const int winCap = ip[9];
        DevBuf<int> dWin(be, (size_t)5 * winCap + 1), dCount(be, 1);
        DevBuf<SeedPlan> dPlan(be, (size_t)numReads);
        dQoff.upload(qoff, (size_t)numPairs);
        dQlen.upload(qlen, (size_t)numPairs);
        if (readList) dList.upload(readList, (size_t)numReads);
        if (thr) dThr.upload(thr, (size_t)numReads);
        dBs.upload(bucketStart, (size_t)numKeys + 1);
        if (numPos) dPos.upload(positions, (size_t)numPos);
        be->fill(dWin.p, 0xff, ((size_t)5 * winCap + 1) * sizeof(int));
        be->fill(dPlan.p, 0xA5, (size_t)numReads * sizeof(SeedPlan));
        be->zero(dCount.p, sizeof(int));
        SeedPlanParams sp;
        memset(&sp, 0, sizeof(sp));
        sp.tcodes = t->p;
        sp.n = n;
        sp.qcodes = q->p;
        sp.qoff = dQoff.p;
        sp.qlen = dQlen.p;
        sp.readList = readList ? dList.p : nullptr;
        sp.firstPair = ip[10];
        sp.thr = thr ? dThr.p : nullptr;
        sp.kBound = ip[0];
        sp.seedK = ip[1];
        sp.numReads = numReads;
        sp.maxLen = ip[2];
        sp.Ls = ip[3];
        sp.Lidx = ip[4];
        sp.sigma = ip[5];
        sp.numKeys = numKeys;
        sp.bucketStart = dBs.p;
        sp.positions = dPos.p;
        sp.maxBucket = ip[6];
        sp.level = ip[7];
        sp.spread = ip[8];
        sp.winPair = dWin.p;
        sp.winK = dWin.p + winCap;
        sp.winStart = dWin.p + 2 * (size_t)winCap;
        sp.winLen = dWin.p + 3 * (size_t)winCap;
        sp.winTf = dWin.p + 4 * (size_t)winCap;
        sp.winCap = winCap;
        sp.winCount = dCount.p;
        sp.plan = dPlan.p;
        with_seed_plan_instance(sp, [&](auto cap, auto threads, auto gw) {
            instance[0] = decltype(cap)::value;
            instance[1] = decltype(threads)::value;
            instance[2] = decltype(gw)::value;
        });
        be->launch_seed_plan(sp);
        static_assert(sizeof(SeedPlan) == 4 * sizeof(int), "SeedPlan: four ints");
        dPlan.download(reinterpret_cast<SeedPlan*>(plan), (size_t)numReads);
        dWin.download(win, (size_t)5 * winCap);
        dCount.download(winCount, 1);
    });
}

}  // extern "C"
