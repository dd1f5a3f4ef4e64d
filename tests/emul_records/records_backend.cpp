// TEST INFRASTRUCTURE -- the host SIMT emulation of tests/emul/emul_backend.cpp plus every kernel of the all-hits
// search (as tests/emul_hit_alignments/hit_alignments_backend.cpp) and the kernels of record targets: the hit sweeps
// that skip separator columns (k1w_hits_records_kernel, k1_hits_records_kernel), record_kernel and the separator-aware
// seed index build (seed_count_records_kernel, seed_fill_records_kernel of eb_kernels.cu), NOT
// a product path.  The emulated backend is compiled from its own source, unchanged, so every other kernel runs exactly
// as in tests/emul.  Linked with the host engine into tests/emul_records/libedlib_emul_records.so for the CPU tests of
// tests/test_record_hits.py.  tests/emul_hit_alignments stays as it is: a backend without the record kernels, which
// refuses record calls of more than one record.
#define create_backend emul_backend_without_hits
#include "emul_backend.cpp"
#undef create_backend

namespace {

struct RecordsEmulBackend : EmulBackend {
    // as k1w_hits_kernel (k1w_hits_records_kernel over a record target): one thread per window job; the profile starts as garbage so that a build that misses a row shows
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
Backend* create_backend(std::string*) { return new RecordsEmulBackend(); }
}  // namespace eb
