// TEST INFRASTRUCTURE -- host SIMT emulation of the kernels (NOT a product path).
//
// Implements eb::Backend by running the very same kernel bodies (edlib_b200/csrc/eb_core.h)
// that eb_kernels.cu launches on the GPU: per-thread bodies in plain loops, warp bodies on the
// 32-wide vector backend of host_warp.h.  Linked with eb_engine.cpp + eb_capi.cpp into
// tests/emul/libedlib_emul.so, it lets the CPU test-suite check the kernel logic and the host
// planner against the reference build without a GPU.  The product library never contains it.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

#include "eb_core.h"
#include "eb_dispatch.h"
#include "eb_engine.h"
#include "host_coop.h"
#include "host_warp.h"

namespace ebhost {
template <int R>
void HostWarp::dump_column(int* out, const U (&Pv)[R], const U (&Mv)[R], const U& sb, int topChunk, int, int off, int m) {
    for (int l = 0; l < 32; ++l) {
        uint32_t pv[R], mv[R];
        for (int i = 0; i < R; ++i) {
            pv[i] = Pv[i].x[l];
            mv[i] = Mv[i].x[l];
        }
        eb::dump_chunk_scores<R>(out, pv, mv, sb.x[l], topChunk + l, off, m);
    }
}
}  // namespace ebhost

namespace {

using namespace eb;

// Peq rows of one emulated K1 thread: plain array [code][word].
template <int NW>
struct HostPeqAcc {
    std::vector<uint32_t> w;
    void store(int code, int word, uint32_t bits) { w[(size_t)code * NW + word] = bits; }
    void or_word(int code, int word, uint32_t bits) { w[(size_t)code * NW + word] |= bits; }
    void load(uint32_t code, uint32_t (&Eq)[NW]) const {
        for (int i = 0; i < NW; ++i) Eq[i] = w[(size_t)code * NW + i];
    }
};

template <int NW>
void emul_k1(const K1Params& p) {
    HostPeqAcc<NW> acc;
    acc.w.assign((size_t)p.ncodes * NW, 0);
    for (int chunk = 0; chunk < p.chunks; ++chunk)
        for (int slot = 0; slot < p.numReads; ++slot) k1_thread<NW>(p, slot, chunk, acc);
}

// As k1t_kernel (eb_kernels.cu): the profile of a read is built ONCE (there: by lane 0 of the read's warp), every chunk then
// sweeps with BUILD = false.  The profile starts as garbage so that a build that misses a row shows.
template <int NW>
void emul_k1t(const K1Params& p) {
    HostPeqAcc<NW> acc;
    for (int slot = 0; slot < p.numReads; ++slot) {
        acc.w.assign((size_t)p.ncodes * NW, 0xdeadbeefu);
        const int pair = p.readList[slot];
        k1_build_peq<NW>(acc, p.qcodes + p.qoff[pair], p.qlen[pair], p.mode, p.ncodes, p.eqtab);
        for (int chunk = p.chunks - 1; chunk >= 0; --chunk) k1_thread<NW, HostPeqAcc<NW>, false>(p, slot, chunk, acc);
    }
}

// Word-addressable rows of NW + 4 words (K1W: banded and full sweeps share one profile).
struct HostWordAcc {
    std::vector<uint32_t> w;
    int words;
    void store_word(int code, int word, uint32_t bits) { w[(size_t)code * words + word] = bits; }
    void or_word(int code, int word, uint32_t bits) { w[(size_t)code * words + word] |= bits; }
    uint32_t load_word(uint32_t code, int word) const { return w[(size_t)code * words + word]; }
};

template <int NW>
void emul_k1w(const K1WParams& p) {
    HostWordAcc acc;
    acc.words = NW + 4;
    acc.w.assign((size_t)p.ncodes * (NW + 4), 0xdeadbeefu);
    const int numJobs = p.countPtr ? std::min(p.numReads, *p.countPtr) : p.numReads;
    for (int slot = 0; slot < numJobs; ++slot) k1w_thread<NW>(p, slot, acc);
}

template <int NW, int MODE, bool REV, bool STORE>
void emul_lane(const LParams& p) {
    HostPeqAcc<NW> acc;
    acc.w.assign((size_t)p.ncodes * NW, 0);
    for (int j = 0; j < p.numJobs; ++j) lane_job<NW, MODE, REV, STORE>(p, j, acc);
}

// Window of the profile of one emulated band thread: plain array [code][slot].
struct HostBandAcc {
    std::vector<uint32_t> w;
    int slots = 0, org = 0;
    void set(int code, int slot, uint32_t bits) { w[(size_t)code * slots + slot] = bits; }
    uint32_t get(int code, int slot) const { return w[(size_t)code * slots + slot]; }
    void origin(int slot) { org = slot; }
    uint32_t code_off(uint32_t sym) const { return sym * (uint32_t)slots; }
    uint32_t load(uint32_t codeOff, int word) const { return w[(size_t)codeOff + org + word]; }
};
template <int NB>
void emul_band(const WParams& p, int ncodes) {
    HostBandAcc acc;
    acc.slots = 4 * NB + BAND_SLACK;
    for (int j = 0; j < p.numJobs; ++j) {
        acc.w.assign((size_t)ncodes * acc.slots, 0xdeadbeefu);  // slots never written must never be read
        band_job<NB>(p, j, acc, ncodes);
    }
}

struct EmulBackend : Backend {
    int launchesCount = 0;
    void* alloc(size_t bytes) override {
        void* p = nullptr;
        if (posix_memalign(&p, 256, bytes ? bytes : 1)) throw std::runtime_error("emul alloc failed");
        memset(p, 0xA5, bytes);  // poison: device memory is never implicitly zero
        return p;
    }
    void free(void* p) override { ::free(p); }
    void* alloc_host(size_t bytes) override { return malloc(bytes ? bytes : 1); }
    void free_host(void* p) override { ::free(p); }
    bool host_pinned(const void*, size_t) override { return getenv("EDLIB_EMUL_PINNED") != nullptr; }  // (tests: take the direct-upload path)
    void h2d(void* d, const void* s, size_t n) override { memcpy(d, s, n); }
    void d2h(void* d, const void* s, size_t n) override { memcpy(d, s, n); }
    void zero(void* d, size_t n) override { memset(d, 0, n); }
    void d2d(void* d, const void* s, size_t n) override { memcpy(d, s, n); }
    void fill(void* d, int v, size_t n) override { memset(d, v, n); }
    void sync() override {}
    int sm_count() override {
        const char* s = getenv("EDLIB_EMUL_SMS");
        return s ? atoi(s) : 2;
    }
    void k1_shape(int, int, int, int* blockThreads, int* residentCtas) override {
        *blockThreads = 32;
        *residentCtas = sm_count() * 4;
    }
    void launch_mask(const MaskParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numItems + p.numQueries; ++i) mask_item(p, i, 0, 1);
    }
    void launch_alpha_len(const uint32_t* masks, const int* qset, const int* tset, int n, int* out) override {
        ++launchesCount;
        for (int i = 0; i < n; ++i) out[i] = alpha_len_pair(masks, qset ? qset[i] : i, tset[i]);
    }
    void launch_encode(const EncodeParams& p) override {
        ++launchesCount;
        for (uint64_t i = 0; i < p.numBytes; ++i) p.data[i] = p.map[p.data[i]];
    }
    void launch_seed_count(const SeedIndexParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numPos; ++i) seed_count_item(p, i);
    }
    void launch_seed_fill(const SeedIndexParams& p) override {
        ++launchesCount;
        for (int i = p.numPos - 1; i >= 0; --i) seed_fill_item(p, i);  // any order is valid; not the ascending one
    }
    void launch_scan(int* data, int count) override {
        ++launchesCount;
        int run = 0;
        for (int i = 0; i < count; ++i) {
            const int v = data[i];
            data[i] = run;
            run += v;
        }
        data[count] = run;
    }
    // Serial planning (one member per read) unless EDLIB_EMUL_SEED_GROUP=device: then the instance the CUDA backend
    // launches, its groups as lane threads (host_coop.h).
    void launch_seed_plan(const SeedPlanParams& p) override {
        ++launchesCount;
        const char* mode = getenv("EDLIB_EMUL_SEED_GROUP");
        if (mode && strcmp(mode, "device") == 0) {
            with_seed_plan_instance(p, [&](auto cap, auto threads, auto gw) {
                constexpr int CAP = decltype(cap)::value, THREADS = decltype(threads)::value, GW = decltype(gw)::value;
                constexpr int GROUPS = 32 / GW;  // per warp
                std::vector<int> E((size_t)GROUPS * CAP), ctl((size_t)GROUPS * seed_ctl_words(GW));
                const int ctas = (p.numReads + THREADS / GW - 1) / (THREADS / GW);
                ebhost::run_lane_groups<GW>(ctas, THREADS, [&](int slot, int g) {
                    seed_plan_read<CAP, ebhost::CoopThreads<GW>>(p, slot, E.data() + g * CAP, ctl.data() + g * seed_ctl_words(GW));
                });
            });
            return;
        }
        std::vector<int> E(SEED_CAND_2);
        int ctl[SEED_CTL];
        with_seed_cap(p.level, [&](auto cap) {
            for (int i = p.numReads - 1; i >= 0; --i) seed_plan_read<decltype(cap)::value, CoopSerial>(p, i, E.data(), ctl);
        });
    }
    void launch_fin_count(const FinParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numReads; ++i) fin_count_item(p, i);
    }
    void launch_fin_fill(const FinParams& p) override {
        ++launchesCount;
        for (int i = p.numReads - 1; i >= 0; --i) fin_fill_item(p, i);
    }
    void launch_qalpha(const QAlphaParams& p) override {
        ++launchesCount;
        for (int q = 0; q < p.numQueries; ++q) {
            uint32_t local[8];
            qalpha_scan(p, q, 0, 1, local);
            int total = 0;
            for (int k = 0; k < 8; ++k) total += popcount32(local[k] | p.tmask[k]);
            p.alphaLen[p.firstPair + q] = total;
        }
    }
    void launch_win_reduce(const WinReduceParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numReads; ++i) win_reduce_read(p, i);
    }
    void launch_k1t(const K1Params& p, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) { emul_k1t<decltype(w)::value>(p); });
    }
    void launch_k1(const K1Params& p, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) { emul_k1<decltype(w)::value>(p); });
    }
    void launch_k1w(const K1WParams& p, int nw) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) { emul_k1w<decltype(w)::value>(p); });
    }
    void launch_lane(const LParams& p, int nw, int mode, bool rev, bool store) override {
        ++launchesCount;
        with_nw(nw, [&](auto w) {
            with_lane_class(mode, rev, store, [&](auto c) {
                using C = decltype(c);
                emul_lane<decltype(w)::value, C::MODE, C::REV, C::STORE>(p);
            });
        });
    }
    void launch_peq(const PeqParams& p) override {
        ++launchesCount;
        for (int j = 0; j < p.numJobs; ++j)
            for (int lane = 0; lane < 32; ++lane) peq_build_words(p, j, lane, 32);
    }
    void launch_w(const WParams& p, int R) override {
        ++launchesCount;
        with_r(R, [&](auto r) {
            for (int j = 0; j < p.numJobs; ++j) w_dispatch<ebhost::HostWarp, decltype(r)::value>(p, j);
        });
    }
    void launch_res(const ResParams& p) override {
        ++launchesCount;
        for (int i = 0; i < p.numItems; ++i) res_item(p, i);
    }
    int band_max_blocks(int ncodes) override { return ncodes <= 64 ? 8 : 0; }
    void launch_band(const WParams& p, int NB, int ncodes) override {
        ++launchesCount;
        with_nb(NB, [&](auto nb) { emul_band<decltype(nb)::value>(p, ncodes); });
    }
    void launch_split(const SplitParams& p) override {
        ++launchesCount;
        for (int j = 0; j < p.numNodes; ++j) split_node(p, j);
    }
    void launch_traceback(const TbParams& p) override {
        ++launchesCount;
        for (int j = 0; j < p.numJobs; ++j) traceback_job(p, j);
    }
    void reset_timing() override { launchesCount = 0; }
    double kernel_ms(const char*) override { return 0.0; }
    int launches() override { return launchesCount; }
    std::string kernel_report() override { return std::string(); }
};

}  // namespace

namespace eb {
Backend* create_backend(std::string*) { return new EmulBackend(); }
int select_device(int, std::string*) { return 0; }
}  // namespace eb
