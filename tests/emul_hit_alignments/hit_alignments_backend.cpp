// TEST INFRASTRUCTURE -- the host SIMT emulation of tests/emul/emul_backend.cpp plus every kernel of the all-hits
// search: the hit lists (k1w_hits_kernel, k1_hits_kernel, hits_total_kernel, hits_place_kernel, as in
// tests/emul_hits/hits_backend.cpp) and their start locations / paths (hit_res_kernel of eb_kernels.cu), NOT a product
// path.  The emulated backend is compiled from its own source, unchanged, so every other kernel runs exactly as in
// tests/emul; this file only derives from it and runs the bodies of the hit kernels (eb_core.h) in loops.  Linked with
// the host engine into tests/emul_hit_alignments/libedlib_emul_hit_alignments.so for the CPU tests of
// tests/test_hit_alignments.py.  tests/emul_hits stays as it is: a backend without hit_res_kernel, which refuses LOC /
// PATH hit calls.
#define create_backend emul_backend_without_hits
#include "emul_backend.cpp"
#undef create_backend

namespace {

struct HitAlignmentsEmulBackend : EmulBackend {
    // as k1w_hits_kernel: one thread per window job; the profile starts as garbage so that a build that misses a row shows
    void launch_k1w_hits(const K1WParams& p, const HitParams& h, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            constexpr int NW = decltype(w)::value;
            HostWordAcc acc;
            acc.words = NW + 4;
            acc.w.assign((size_t)p.ncodes * (NW + 4), 0xdeadbeefu);
            for (int slot = p.numReads - 1; slot >= 0; --slot) k1w_hits_thread<NW>(p, h, slot, acc);
        });
    }
    // as k1_hits_kernel: one thread per (read, chunk)
    void launch_k1_hits(const K1Params& p, const HitParams& h, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            constexpr int NW = decltype(w)::value;
            HostPeqAcc<NW> acc;
            acc.w.assign((size_t)p.ncodes * NW, 0xdeadbeefu);
            for (int chunk = p.chunks - 1; chunk >= 0; --chunk)
                for (int slot = 0; slot < p.numReads; ++slot) k1_hits_thread<NW>(p, h, slot, chunk, acc);
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
    // as hit_res_kernel: one thread per hit or job, run in reverse order
    void launch_hit_res(const HitResParams& p) override {
        ++launchesCount;
        for (int i = p.numItems - 1; i >= 0; --i) hit_res_item(p, i);
    }
};

}  // namespace

namespace eb {
Backend* create_backend(std::string*) { return new HitAlignmentsEmulBackend(); }
}  // namespace eb
