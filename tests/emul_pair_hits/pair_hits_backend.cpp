// TEST INFRASTRUCTURE -- the host SIMT emulation of tests/emul/emul_backend.cpp plus every kernel of
// tests/emul_records/records_backend.cpp (the all-hits search, start locations / paths, record targets) and the hit
// sweep of the per-pair route (lane_hits_kernel of eb_kernels.cu), NOT a product path.  The emulated backend is compiled
// from its own source, unchanged; this file only derives from it and runs the bodies of the kernels (eb_core.h) in
// loops.  Linked with the host engine into tests/emul_pair_hits/libedlib_emul_pair_hits.so for the CPU tests of
// tests/test_pair_hits.py.  tests/emul_records stays as it is: a backend without lane_hits, which refuses pair calls that
// need the per-pair route.
#define create_backend emul_backend_without_hits
#include "emul_backend.cpp"
#undef create_backend

namespace {

struct PairHitsEmulBackend : EmulBackend {
    // as k1w_hits_kernel (k1w_hits_records_kernel over a record target): one thread per window job; the profile starts
    // as garbage so that a build that misses a row shows
    void launch_k1w_hits(const K1WParams& p, const HitParams& h, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            constexpr int NW = decltype(w)::value;
            HostWordAcc acc;
            acc.words = NW + 4;
            acc.w.assign((size_t)p.ncodes * (NW + 4), 0xdeadbeefu);
            for (int slot = p.numReads - 1; slot >= 0; --slot) {
                if (h.sepCodes) k1w_hits_thread<NW, HostWordAcc, RecordHitSink>(p, h, slot, acc);
                else k1w_hits_thread<NW>(p, h, slot, acc);
            }
        });
    }
    // as k1_hits_kernel (k1_hits_records_kernel over a record target): one thread per (read, chunk)
    void launch_k1_hits(const K1Params& p, const HitParams& h, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            constexpr int NW = decltype(w)::value;
            HostPeqAcc<NW> acc;
            acc.w.assign((size_t)p.ncodes * NW, 0xdeadbeefu);
            for (int chunk = p.chunks - 1; chunk >= 0; --chunk)
                for (int slot = 0; slot < p.numReads; ++slot) {
                    if (h.sepCodes) k1_hits_thread<NW, HostPeqAcc<NW>, RecordHitSink>(p, h, slot, chunk, acc);
                    else k1_hits_thread<NW>(p, h, slot, chunk, acc);
                }
        });
    }
    // as lane_hits_kernel: one thread per (pair, chunk) job, run in reverse order
    void launch_lane_hits(const LaneHitParams& p, const HitParams& h, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            constexpr int NW = decltype(w)::value;
            HostPeqAcc<NW> acc;
            acc.w.assign((size_t)p.ncodes * NW, 0xdeadbeefu);
            for (int job = p.numJobs - 1; job >= 0; --job) lane_hits_job<NW>(p, h, job, acc);
        });
    }
    void launch_hits_total(const HitPlaceParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numReads; ++i) hits_total_item(p, i);
    }
    void launch_hits_place(const HitPlaceParams& p) override {
        ++launchesCount;
        for (int i = p.numReads - 1; i >= 0; --i) hits_place_item(p, i);
    }
    // as hit_res_kernel / record_kernel: one thread per item, run in reverse order
    void launch_hit_res(const HitResParams& p) override {
        ++launchesCount;
        for (int i = p.numItems - 1; i >= 0; --i) hit_res_item(p, i);
    }
    void launch_record(const RecordParams& p) override {
        ++launchesCount;
        for (int i = p.numItems - 1; i >= 0; --i) record_item(p, i);
    }
    // as seed_count_records_kernel / seed_fill_records_kernel, in the orders of the plain index build
    void launch_seed_count_records(const SeedIndexParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numPos; ++i) seed_count_item<true>(p, i);
    }
    void launch_seed_fill_records(const SeedIndexParams& p) override {
        ++launchesCount;
        for (int i = p.numPos - 1; i >= 0; --i) seed_fill_item<true>(p, i);
    }
};

}  // namespace

namespace eb {
Backend* create_backend(std::string*) { return new PairHitsEmulBackend(); }
}  // namespace eb
