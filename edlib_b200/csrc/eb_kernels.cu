// eb_kernels.cu -- sm_90a kernels and the CUDA Backend of the engine.
//
//   k1_kernel<NW,MODE>  lane-per-alignment Myers sweep over one shared target (the hot path):
//                       query bit-vectors in registers, per-thread Peq rows in shared memory,
//                       the target streamed HBM/L2 -> shared memory by 1-D TMA bulk copies
//                       (cp.async.bulk + mbarrier, double buffered) and consumed by every
//                       thread of the CTA as 32-bit broadcast reads.
//   w_kernel<R>         warp-per-alignment sweep (long queries, per-pair targets, band, strips)
//   peq_kernel, traceback_kernel, mask_kernel, alpha_len_kernel, encode_kernel
//
// The bodies live in eb_core.h (shared with the host emulation used by the CPU tests).
#include <cuda_runtime.h>
#include <ctype.h>
#include <stdio.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "eb_core.h"
#include "eb_dispatch.h"
#include "eb_engine.h"

namespace eb {

// ---------------------------------------------------------------------------------------------
// Device warp backend for w_sweep
// ---------------------------------------------------------------------------------------------
// (Members are __host__ __device__ only because w_sweep is; the host bodies are never run.)
#if defined(__CUDA_ARCH__)
#define EB_DEV(expr, fallback) expr
#else
#define EB_DEV(expr, fallback) fallback
#endif
struct DevWarp {
    using U = uint32_t;
    using P = bool;
    static constexpr unsigned FULL = 0xffffffffu;
    static EB_HD U lane() { return EB_DEV(threadIdx.x & 31u, 0u); }
    template <class F>
    static EB_HD U map(U a, F f) { return f(a); }
    static EB_HD U sel(P p, U a, U b) { return p ? a : b; }
    static EB_HD U toU(P p) { return p ? 1u : 0u; }
    static EB_HD uint32_t ballot(P p) { return EB_DEV(__ballot_sync(FULL, p), (uint32_t)p); }
    static EB_HD bool any(P p) { return EB_DEV(__any_sync(FULL, p) != 0, p); }
    static EB_HD U shfl_up1(U a) { return EB_DEV(__shfl_up_sync(FULL, a, 1), a); }
    static EB_HD U shfl_down1(U a) { return EB_DEV(__shfl_down_sync(FULL, a, 1), a); }
    static EB_HD uint32_t bcast(U a, int src) { return EB_DEV(__shfl_sync(FULL, a, src), a + 0u * (uint32_t)src); }
    static EB_HD U gather8(const uint8_t* base, U idx, P ok) { return ok ? (U)base[idx] : 0u; }
    static EB_HD U gather8_neg(const uint8_t* base, U idx, P ok) { return ok ? (U) * (base - (ptrdiff_t)idx) : 0u; }
    static EB_HD U gather32(const uint32_t* base, U idx, P ok) { return ok ? EB_DEV(__ldg(base + idx), base[idx]) : 0u; }
    static EB_HD void scatterU2(U2* base, U idx, U a, U b, P ok) {
        if (ok) {
            U2 v;
            v.x = a;
            v.y = b;
            *reinterpret_cast<uint2*>(base + idx) = *reinterpret_cast<uint2*>(&v);
        }
    }
    static EB_HD void scatter8(uint8_t* base, U idx, U v, P ok) {
        if (ok) base[idx] = (uint8_t)v;
    }
    static EB_HD void store_uniform(int* p, int v) {
        if (lane() == 0) *p = v;
    }
    static EB_HD int atomic_add_uniform(int* p, int v) {
        int r = 0;
        if (lane() == 0) r = atomic_add_int(p, v);
        return (int)bcast((U)r, 0);
    }
    template <int R>
    static EB_HD void dump_column(int* out, const U (&Pv)[R], const U (&Mv)[R], U sb, int topChunk, int, int off, int m) {
        dump_chunk_scores<R>(out, Pv, Mv, sb, topChunk + (int)lane(), off, m);
    }
};

// ---------------------------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------------------------
constexpr int K1_TILE = 4096;  // target bytes per shared-memory stage (two stages)

// Per-thread Peq rows in shared memory, addressed with explicit 32-bit shared addresses so the
// inner loop is LDS with register+immediate addressing and no generic-address arithmetic.
// Region of one code: [ A: nthreads x 16 B (words 0..3, one LDS.128) | B: nthreads x 4*(NW-4) B
// (words 4.., contiguous per thread) ].  Consecutive threads touch consecutive 16 B slots of A
// and slots of 4/8/12/16 B of B: both patterns are bank-conflict free.
template <int NW>
struct SmemPeqAcc {
    static constexpr int NWB = NW > 4 ? NW - 4 : 0;
    uint32_t a0;          // shared address of this thread's A slot for code 0
    uint32_t b0;          // shared address of this thread's B slot for code 0
    uint32_t codeStride;  // bytes per code region
    EB_D void store(int code, int w, uint32_t bits) {
        const uint32_t addr = (w < 4 ? a0 + 4u * w : b0 + 4u * (w - 4)) + (uint32_t)code * codeStride;
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(bits) : "memory");
    }
    EB_D void or_word(int code, int w, uint32_t bits) {  // the rows are private to the thread: no atomics
        const uint32_t addr = (w < 4 ? a0 + 4u * w : b0 + 4u * (w - 4)) + (uint32_t)code * codeStride;
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v | bits) : "memory");
    }
    EB_D void load(uint32_t code, uint32_t (&Eq)[NW]) const {
        const uint32_t off = code * codeStride;
        uint32_t x, y, z, w;
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a0 + off));
        Eq[0] = x;
        if (NW > 1) Eq[NW > 1 ? 1 : 0] = y;
        if (NW > 2) Eq[NW > 2 ? 2 : 0] = z;
        if (NW > 3) Eq[NW > 3 ? 3 : 0] = w;
        if (NWB == 1) {
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(Eq[NW > 4 ? 4 : 0]) : "r"(b0 + off));
        } else if (NWB == 2) {
            asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(Eq[NW > 4 ? 4 : 0]), "=r"(Eq[NW > 5 ? 5 : 0]) : "r"(b0 + off));
        } else if (NWB == 3) {
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(Eq[NW > 4 ? 4 : 0]) : "r"(b0 + off));
            asm volatile("ld.shared.u32 %0, [%1+4];" : "=r"(Eq[NW > 5 ? 5 : 0]) : "r"(b0 + off));
            asm volatile("ld.shared.u32 %0, [%1+8];" : "=r"(Eq[NW > 6 ? 6 : 0]) : "r"(b0 + off));
        } else if (NWB == 4) {
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                         : "=r"(Eq[NW > 4 ? 4 : 0]), "=r"(Eq[NW > 5 ? 5 : 0]), "=r"(Eq[NW > 6 ? 6 : 0]), "=r"(Eq[NW > 7 ? 7 : 0])
                         : "r"(b0 + off));
        }
    }
};

// Target symbols of the current tile, read as warp-uniform (broadcast) shared loads.
struct SmemSyms {
    uint32_t addr;  // shared address of the first symbol
    EB_D uint32_t read1(int i) const {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr + (uint32_t)i));
        return v;
    }
};

EB_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

EB_D void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
EB_D void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
EB_D void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    uint32_t spins = 0;
    uint64_t t0 = 0;
    do {
        // A copy that never lands must fail the launch, not hang the device -- but only after 20 s of wall
        // time (globaltimer), so that a time-sliced / preempted context is never mistaken for a lost copy.
        if ((++spins & 0xffffu) == 0) {
            uint64_t now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 20000000000ull) __trap();
        }
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier (UBLKCP in SASS).
EB_D void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int NW, int MODE, bool RANGE = false>
__global__ void k1_kernel(const K1Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x;
    const int nthreads = blockDim.x;
    // layout: [tile0 | tile1 | mbar0 mbar1 | PeqA | PeqB]
    uint8_t* tile[2] = {smem, smem + K1_TILE};
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 2 * K1_TILE);
    unsigned char* peqBase = smem + 2 * K1_TILE + 64;

    const int slot = blockIdx.x * nthreads + tid;
    const int chunk = blockIdx.y;
    const bool active = slot < p.numReads;
    const K1Chunk g = k1_chunk(p, chunk);

    if (tid == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int total = g.ce - g.hs;  // columns this CTA sweeps, starting at a 16-byte aligned offset
    const int numTiles = (total + K1_TILE - 1) / K1_TILE;
    auto issue = [&](int i) {
        const int begin = i * K1_TILE;
        int bytes = total - begin;
        if (bytes > K1_TILE) bytes = K1_TILE;
        bytes = (bytes + 15) & ~15;  // the encoded target is padded with >= 16 spare bytes
        mbar_expect_tx(&bar[i & 1], (uint32_t)bytes);
        tma_load_1d(tile[i & 1], p.tcodes + g.hs + begin, (uint32_t)bytes, &bar[i & 1]);
    };
    if (tid == 0 && numTiles > 0) issue(0);

    SmemPeqAcc<NW> acc;
    acc.codeStride = (uint32_t)nthreads * (16u + 4u * SmemPeqAcc<NW>::NWB);
    acc.a0 = smem_u32(peqBase) + 16u * tid;
    acc.b0 = smem_u32(peqBase) + 16u * nthreads + 4u * SmemPeqAcc<NW>::NWB * tid;
    const uint32_t tileAddr[2] = {smem_u32(smem), smem_u32(smem) + (uint32_t)K1_TILE};
    K1State<NW> st;
    Rec* rec = nullptr;
    int recIdx = 0;
    if (active) {
        const int pair = p.readList[slot];
        const int m = p.prefixLen > 0 ? p.prefixLen : p.qlen[pair];
        k1_build_peq<NW>(acc, p.qcodes + p.qoff[pair], m, MODE, p.ncodes, p.eqtab);
        k1_init<NW>(st, m, p.kInit[slot]);
        recIdx = RANGE ? slot : chunk * p.numReads + slot;  // RANGE: events carry the read slot
        rec = RANGE ? nullptr : p.recs + recIdx;
    }

    for (int i = 0; i < numTiles; ++i) {
        if (tid == 0 && i + 1 < numTiles) issue(i + 1);  // its buffer was released by the barrier below
        mbar_wait(&bar[i & 1], (uint32_t)((i >> 1) & 1));
        if (active) {
            const int a = g.hs + i * K1_TILE;                       // absolute column of tile byte 0
            const int b = min(a + K1_TILE, g.ce);
            const uint32_t sa = tileAddr[i & 1];
            if (MODE == MODE_HW) {
                const int mid = min(max(g.cs, a), b);               // columns before cs are halo
                if (mid > a) k1_columns<NW, false, false, RANGE>(st, acc, SmemSyms{sa}, mid - a, a, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
                if (b > mid) k1_columns<NW, false, true, RANGE>(st, acc, SmemSyms{sa + (uint32_t)(mid - a)}, b - mid, mid, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
            } else if (MODE == MODE_SHW) {
                k1_columns<NW, true, true>(st, acc, SmemSyms{sa}, b - a, a, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
            } else {
                k1_columns<NW, true, false>(st, acc, SmemSyms{sa}, b - a, a, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
            }
        }
        __syncthreads();  // everyone is done with tile i before its buffer is refilled
    }
    if (active && RANGE) {
        k1_range_flush<NW>(st, slot, p.ovf, p.ovfCount, p.ovfCap);
    } else if (active) {
        if (MODE == MODE_NW) {
            st.best = st.up - st.down;
            st.cnt = 1;
            rec->last = p.n - 1;
            rec->pos[0] = p.n - 1;
        }
        rec->best = st.best;
        rec->cnt = st.cnt;
    }
}

// Word-addressable per-thread profile rows for K1W: word w of code c of thread t at base + (c * WORDS + w) *
// 4 * THREADS + 4 * t -- consecutive threads in consecutive banks whatever word each of them reads, and (CTA size
// and row length being compile-time constants) every offset an immediate of the shared-memory instruction.
// K1T: the plain sweep for a handful of reads.  The tile kernel gives every read ONE lane per chunk-CTA, so three
// reads occupy three lanes of every warp and walk thousands of columns each; here a warp belongs to one read, its lanes
// take 32 consecutive chunks (each behind its own 2m halo, symbols straight from global memory / L2), and the read's
// profile sits once per warp in shared memory (rows of different codes fall into different banks, equal codes broadcast).
template <int NW>
struct WarpPeqAcc {
    uint32_t* w;  // [ncodes][NW]
    EB_D void store(int code, int word, uint32_t bits) { w[code * NW + word] = bits; }
    EB_D void or_word(int code, int word, uint32_t bits) { w[code * NW + word] |= bits; }
    EB_D void load(uint32_t code, uint32_t (&Eq)[NW]) const {
#pragma unroll
        for (int i = 0; i < NW; ++i) Eq[i] = w[code * NW + i];
    }
};
template <int NW>
__global__ void __launch_bounds__(32) k1t_kernel(const K1Params p) {
    extern __shared__ __align__(16) unsigned char smem[];
    WarpPeqAcc<NW> acc{reinterpret_cast<uint32_t*>(smem)};
    const int slot = blockIdx.y;
    const int chunk = blockIdx.x * 32 + threadIdx.x;
    if (threadIdx.x == 0) {
        const int pair = p.readList[slot];
        k1_build_peq<NW>(acc, p.qcodes + p.qoff[pair], p.qlen[pair], p.mode, p.ncodes, p.eqtab);
    }
    __syncwarp();
    if (chunk < p.chunks) k1_thread<NW, WarpPeqAcc<NW>, false>(p, slot, chunk, acc);
}

template <int THREADS, int WORDS>
struct SmemWordAcc {
    uint32_t base;  // shared address of this thread's word 0 of code 0
    static constexpr uint32_t wordStride = 4u * THREADS, codeStride = wordStride * WORDS;
    EB_D void store_word(int code, int w, uint32_t bits) {
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(base + (uint32_t)code * codeStride + (uint32_t)w * wordStride), "r"(bits) : "memory");
    }
    EB_D void or_word(int code, int w, uint32_t bits) {
        const uint32_t addr = base + (uint32_t)code * codeStride + (uint32_t)w * wordStride;
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v | bits) : "memory");
    }
    EB_D uint32_t load_word(uint32_t code, int w) const {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(base + code * codeStride + (uint32_t)w * wordStride));
        return v;
    }
};

// K1W: every thread over its own target window read through the generic (global) pointer path; no tile
// staging, no barriers.  Banded sweep for windows that span few diagonals, full sweep otherwise (eb_core.h).
template <int NW, int THREADS>
__global__ void __launch_bounds__(THREADS) k1w_kernel(const K1WParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int slot = blockIdx.x * THREADS + threadIdx.x;
    int numJobs = p.numReads;
    if (p.countPtr) numJobs = min(numJobs, *p.countPtr);  // jobs planned on the device (seed_plan_kernel)
    if (slot >= numJobs) return;
    SmemWordAcc<THREADS, NW + 4> acc;
    acc.base = smem_u32(smem) + 4u * threadIdx.x;
    k1w_thread<NW>(p, slot, acc);
}

// L: one alignment per thread over its own target (eb_core.h: lane_job).
template <int NW, int MODE, bool REV, bool STORE>
__global__ void lane_kernel(const LParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int job = blockIdx.x * blockDim.x + threadIdx.x;
    if (job >= p.numJobs) return;
    SmemPeqAcc<NW> acc;
    acc.codeStride = (uint32_t)blockDim.x * (16u + 4u * SmemPeqAcc<NW>::NWB);
    acc.a0 = smem_u32(smem) + 16u * threadIdx.x;
    acc.b0 = smem_u32(smem) + 16u * blockDim.x + 4u * SmemPeqAcc<NW>::NWB * threadIdx.x;
    lane_job<NW, MODE, REV, STORE>(p, job, acc);
}

// ---------------------------------------------------------------------------------------------
// W and the small kernels
// ---------------------------------------------------------------------------------------------
constexpr int W_WARPS = 4;

template <int R>
__global__ void __launch_bounds__(W_WARPS * 32) w_kernel(const WParams p) {
    const int job = blockIdx.x * W_WARPS + (threadIdx.x >> 5);
    if (job >= p.numJobs) return;
    w_dispatch<DevWarp, R>(p, job);
}

// B: k-banded NW sweep of a long query, one alignment per thread (eb_core.h: band_job).  The window's words of
// every code live in shared memory, word-interleaved over the threads of the CTA (slot s of code c of thread t at
// base + ((c * SLOTS + s) * THREADS + t) * 4): conflict-free whatever slot each thread reads, and with the origin
// folded into `cur` every offset of the column loop is an immediate.
template <int THREADS, int SLOTS>
struct SmemBandAcc {
    uint32_t base, cur;
    static constexpr uint32_t wordStride = 4u * THREADS, codeStride = wordStride * SLOTS;
    EB_D void set(int code, int slot, uint32_t bits) {
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(base + (uint32_t)code * codeStride + (uint32_t)slot * wordStride), "r"(bits) : "memory");
    }
    EB_D uint32_t get(int code, int slot) const {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(base + (uint32_t)code * codeStride + (uint32_t)slot * wordStride) : "memory");
        return v;
    }
    EB_D void origin(int slot) { cur = base + (uint32_t)slot * wordStride; }
    EB_D uint32_t code_off(uint32_t sym) const { return sym * codeStride; }
    EB_D uint32_t load(uint32_t codeOff, int w) const {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(cur + codeOff + (uint32_t)w * wordStride) : "memory");
        return v;
    }
};
constexpr int BAND_THREADS = 128;
template <int NB>
__global__ void __launch_bounds__(BAND_THREADS) band_kernel(const WParams p, int ncodes) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int job = blockIdx.x * BAND_THREADS + threadIdx.x;
    if (job >= p.numJobs) return;
    SmemBandAcc<BAND_THREADS, 4 * NB + BAND_SLACK> acc;
    acc.base = smem_u32(smem) + 4u * threadIdx.x;
    acc.cur = acc.base;
    band_job<NB>(p, job, acc, ncodes);
}

__global__ void peq_kernel(const PeqParams p) {
    const int job = blockIdx.x * W_WARPS + (threadIdx.x >> 5);
    if (job >= p.numJobs) return;
    peq_build_words(p, job, threadIdx.x & 31, 32);
}

__global__ void traceback_kernel(const TbParams p) {
    const int job = blockIdx.x * blockDim.x + threadIdx.x;
    if (job < p.numJobs) traceback_job(p, job);
}

__global__ void res_kernel(const ResParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.numItems) res_item(p, i);
}

__global__ void split_kernel(const SplitParams p) {
    const int node = blockIdx.x * blockDim.x + threadIdx.x;
    if (node < p.numNodes) split_node(p, node);
}

__global__ void seed_count_kernel(const SeedIndexParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.numPos) seed_count_item(p, i);
}
__global__ void seed_fill_kernel(const SeedIndexParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.numPos) seed_fill_item(p, i);
}
// One read per group of GW lanes (16: two reads per warp; 32: a warp per read).  The lanes take the seeds of the
// read, so their index lookups (key -> bucket bounds -> positions -> target symbols, a chain of dependent random
// reads) are in flight together; candidates meet in shared memory (eb_core.h: seed_plan_read).
template <int GW>
struct CoopGroup {
    static constexpr int W = GW;
    static EB_D int lane() { return (int)(threadIdx.x & (GW - 1)); }
    static EB_D int width() { return GW; }
    static EB_D unsigned mask() { return GW == 32 ? 0xffffffffu : ((1u << (GW & 31)) - 1u) << (threadIdx.x & 31u & ~(GW - 1u)); }
    static EB_D void sync() { __syncwarp(mask()); }
    static EB_D bool any(bool v) { return __ballot_sync(mask(), v) != 0u; }
    static EB_D int add_shared(int* p, int v) { return atomicAdd(p, v); }
    static EB_D int scan(int v, int& total) {
        int incl = v;
        EB_UNROLL
        for (int d = 1; d < GW; d *= 2) {
            const int y = __shfl_up_sync(mask(), incl, d, GW);
            if (lane() >= d) incl += y;
        }
        total = __shfl_sync(mask(), incl, GW - 1, GW);
        return incl - v;
    }
    // the whole warp: every lane holds its group's n, so a scan in steps of whole groups gives each lane the counts of
    // its own and the earlier groups; one atomic for the warp's total, each group's offset in it
    static EB_D int reserve(int* counter, int n) {
        const int l32 = (int)(threadIdx.x & 31u);
        int incl = n;
        EB_UNROLL
        for (int d = GW; d < 32; d *= 2) {
            const int y = __shfl_up_sync(0xffffffffu, incl, d);
            if (l32 >= d) incl += y;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        int base = 0;
        if (total > 0) {
            if (l32 == 31) base = atomicAdd(counter, total);
            base = __shfl_sync(0xffffffffu, base, 31);
        }
        return base + incl - n;
    }
};
// (registers capped at 40 so that 48 warps fit an SM: the lookups of more reads are in flight together)
template <int CAP, int THREADS, class Group>
__global__ void __launch_bounds__(THREADS, 1536 / THREADS) seed_plan_kernel(const SeedPlanParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    constexpr int GW = Group::W;
    constexpr int GROUPS = THREADS / GW;
    int* E = reinterpret_cast<int*>(smemRaw);              // [groups][CAP]
    int* ctl = E + GROUPS * CAP;                            // [groups][seed_ctl_words(GW)]
    const int g = threadIdx.x / GW;
    // every group runs, also past numReads: the warp reserves its window jobs together
    seed_plan_read<CAP, Group>(p, blockIdx.x * GROUPS + g, E + g * CAP, ctl + g * seed_ctl_words(GW));
}
__global__ void win_reduce_kernel(const WinReduceParams p) {
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot < p.numReads) win_reduce_read(p, slot);
}
__global__ void fin_count_kernel(const FinParams p) {
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot < p.numReads) fin_count_item(p, slot);
}
__global__ void fin_fill_kernel(const FinParams p) {
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot < p.numReads) fin_fill_item(p, slot);
}
// alphabetLength of queries facing one target: one query per warp, lanes stride over its bytes.
__global__ void qalpha_kernel(const QAlphaParams p) {
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (q >= p.numQueries) return;
    uint32_t local[8];
    qalpha_scan(p, q, threadIdx.x & 31, 32, local);
    int total = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) total += __popc(__reduce_or_sync(0xffffffffu, local[k]) | p.tmask[k]);
    if ((threadIdx.x & 31) == 0) p.alphaLen[p.firstPair + q] = total;
}

// Exclusive prefix sums over ints, three launches: per-tile sums, scan of the tile sums (one CTA),
// per-tile scan with the tile offset.  A tile is SCAN_THREADS * SCAN_PER consecutive elements.
constexpr int SCAN_THREADS = 256, SCAN_PER = 16, SCAN_TILE = SCAN_THREADS * SCAN_PER;
template <int THREADS>
__device__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warpSums[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) warpSums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int s = lane < THREADS / 32 ? warpSums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += o;
        }
        warpSums[lane] = s;
    }
    __syncthreads();
    *total = warpSums[THREADS / 32 - 1];
    return incl - v + (wid ? warpSums[wid - 1] : 0);
}
__global__ void scan_tile_sums_kernel(const int* data, int count, int* tileSums) {
    const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER;
    int s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_PER; ++i)
        if (base + i < count) s += data[base + i];
    int total;
    block_exclusive_scan<SCAN_THREADS>(s, &total);
    if (threadIdx.x == 0) tileSums[blockIdx.x] = total;
}
__global__ void scan_top_kernel(int* tileSums, int numTiles, int* totalOut) {
    const int per = (numTiles + 1023) / 1024;
    const int base = threadIdx.x * per;
    int s = 0;
    for (int i = 0; i < per; ++i)
        if (base + i < numTiles) s += tileSums[base + i];
    int total;
    int run = block_exclusive_scan<1024>(s, &total);
    for (int i = 0; i < per; ++i)
        if (base + i < numTiles) {
            const int v = tileSums[base + i];
            tileSums[base + i] = run;
            run += v;
        }
    if (threadIdx.x == 0) *totalOut = total;
}
__global__ void scan_apply_kernel(int* data, int count, const int* tileSums) {
    const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER;
    int v[SCAN_PER];
    int s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_PER; ++i) {
        v[i] = base + i < count ? data[base + i] : 0;
        s += v[i];
    }
    int total;
    int run = block_exclusive_scan<SCAN_THREADS>(s, &total) + tileSums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SCAN_PER; ++i)
        if (base + i < count) {
            data[base + i] = run;
            run += v[i];
        }
}

__global__ void mask_kernel(const MaskParams p) {
    const int item = blockIdx.x * W_WARPS + (threadIdx.x >> 5);
    if (item >= p.numItems + p.numQueries) return;
    // lanes stride over the bytes; the eight words are OR-reduced across the warp and lane k commits word k
    uint32_t local[8], rcLocal[8];
    const MaskItem it = mask_item_scan(p, item, threadIdx.x & 31, 32, local, rcLocal);
    uint32_t mine = 0, rcMine = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t v = __reduce_or_sync(0xffffffffu, local[k]);
        const uint32_t w = __reduce_or_sync(0xffffffffu, rcLocal[k]);
        if ((int)(threadIdx.x & 31) == k) {
            mine = v;
            rcMine = w;
        }
    }
    if ((threadIdx.x & 31) < 8) {
        mask_item_commit(p, it.dst, (int)(threadIdx.x & 31), mine);
        mask_item_commit(p, it.dst + 1, (int)(threadIdx.x & 31), rcMine);  // strand batches: the reverse complement's set
    }
}

__global__ void alpha_len_kernel(const uint32_t* masks, const int* qset, const int* tset, int n, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = alpha_len_pair(masks, qset ? qset[i] : i, tset[i]);
}

__global__ void encode_kernel(const EncodeParams p) {
    __shared__ uint8_t map[256];
    if (threadIdx.x < 256) map[threadIdx.x] = p.map[threadIdx.x];
    __syncthreads();
    // bytes before the first 16-byte boundary and after the last one go one by one (slices of a batch are
    // encoded separately and must not touch their neighbours' bytes)
    uint64_t head = (16 - (reinterpret_cast<uintptr_t>(p.data) & 15)) & 15;
    if (head > p.numBytes) head = p.numBytes;
    const uint64_t nvec = (p.numBytes - head) / 16;
    uint4* v = reinterpret_cast<uint4*>(p.data + head);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (uint64_t)gridDim.x * blockDim.x) {
        uint4 x = v[i];
        uint32_t* w = reinterpret_cast<uint32_t*>(&x);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t a = w[k];
            w[k] = (uint32_t)map[a & 255u] | ((uint32_t)map[(a >> 8) & 255u] << 8) | ((uint32_t)map[(a >> 16) & 255u] << 16) |
                   ((uint32_t)map[a >> 24] << 24);
        }
        v[i] = x;
    }
    if (blockIdx.x == 0) {
        for (uint64_t i = threadIdx.x; i < head; i += blockDim.x) p.data[i] = map[p.data[i]];
        for (uint64_t i = head + nvec * 16 + threadIdx.x; i < p.numBytes; i += blockDim.x) p.data[i] = map[p.data[i]];
    }
}

// ---------------------------------------------------------------------------------------------
// CUDA backend
// ---------------------------------------------------------------------------------------------
#define EB_CUDA(call)                                                                                         \
    do {                                                                                                      \
        cudaError_t e_ = (call);                                                                              \
        if (e_ != cudaSuccess) throw std::runtime_error(std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

struct CudaBackend : Backend {
    cudaStream_t stream = nullptr;      // compute stream: every kernel, the stream-ordered allocations
    cudaStream_t copyStream = nullptr;  // uploads of streamed batches (overlap the kernels of earlier slices)
    cudaStream_t resStream = nullptr;   // result downloads of streamed batches
    std::mutex markMu;                  // marks are recorded by pool workers as well
    std::vector<cudaEvent_t> marks, markPool;
    int sms = 0;
    int maxSmemOptin = 0;
    struct Timed {
        const char* name;
        cudaEvent_t a, b;
    };
    std::vector<Timed> timed;
    std::vector<cudaEvent_t> pool;
    int launchCount = 0;


    int deviceId = 0;
    int numaNode = -1;   // NUMA node of the device's PCIe root (pinned staging memory is placed there)

    int numa_node() override { return numaNode; }

    CudaBackend() {
        int dev = 0;
        EB_CUDA(cudaGetDevice(&dev));
        deviceId = dev;
        {
            char bus[32] = {0};
            if (cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), dev) == cudaSuccess) {
                for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
                const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
                if (FILE* f = fopen(path.c_str(), "r")) {
                    int node = -1;
                    if (fscanf(f, "%d", &node) == 1) numaNode = node;
                    fclose(f);
                }
            }
            const char* e = getenv("EDLIB_B200_NUMA");
            if (e && atoi(e) == 0) numaNode = -1;
        }
        cudaDeviceProp prop;
        EB_CUDA(cudaGetDeviceProperties(&prop, dev));
        sms = prop.multiProcessorCount;
        maxSmemOptin = (int)prop.sharedMemPerBlockOptin;
        EB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        EB_CUDA(cudaStreamCreateWithFlags(&copyStream, cudaStreamNonBlocking));
        EB_CUDA(cudaStreamCreateWithFlags(&resStream, cudaStreamNonBlocking));
        cudaMemPool_t mp;
        EB_CUDA(cudaDeviceGetDefaultMemPool(&mp, dev));
        uint64_t keep = UINT64_MAX;
        EB_CUDA(cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    ~CudaBackend() override {
        for (auto& t : timed) {
            cudaEventDestroy(t.a);
            cudaEventDestroy(t.b);
        }
        for (auto e : pool) cudaEventDestroy(e);
        for (auto& b : hostBlocks) cudaFreeHost(b.p);
        for (auto e : marks) cudaEventDestroy(e);
        for (auto e : markPool) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
        if (copyStream) cudaStreamDestroy(copyStream);
        if (resStream) cudaStreamDestroy(resStream);
    }
    // ---- second and third stream: ordering marks (events) between them, the compute stream and the host ----
    cudaStream_t stream_of(int which) { return which == STREAM_COPY ? copyStream : which == STREAM_RESULTS ? resStream : stream; }
    uint64_t mark(int which) override {
        std::lock_guard<std::mutex> lock(markMu);
        cudaEvent_t e;
        if (!markPool.empty()) {
            e = markPool.back();
            markPool.pop_back();
        } else {
            EB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        }
        EB_CUDA(cudaEventRecord(e, stream_of(which)));
        marks.push_back(e);
        return (uint64_t)marks.size();
    }
    cudaEvent_t mark_event(uint64_t token) {
        std::lock_guard<std::mutex> lock(markMu);
        if (token == 0 || token > marks.size()) throw std::runtime_error("internal: unknown stream mark");
        return marks[(size_t)token - 1];
    }
    void wait(int which, uint64_t token) override { EB_CUDA(cudaStreamWaitEvent(stream_of(which), mark_event(token), 0)); }
    void host_wait(uint64_t token) override { EB_CUDA(cudaEventSynchronize(mark_event(token))); }
    void release_marks() override {
        std::lock_guard<std::mutex> lock(markMu);
        markPool.insert(markPool.end(), marks.begin(), marks.end());
        marks.clear();
    }
    void h2d_copy(void* d, const void* s, size_t n) override {
        if (n) EB_CUDA(cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, copyStream));
    }
    void d2h_async(int which, void* d, const void* s, size_t n) override {
        if (n) EB_CUDA(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToHost, stream_of(which)));
    }
    void sync_all() override {
        EB_CUDA(cudaStreamSynchronize(copyStream));
        EB_CUDA(cudaStreamSynchronize(stream));
        EB_CUDA(cudaStreamSynchronize(resStream));
    }
    // Device memory comes from the stream-ordered pool (cudaMallocAsync) with an unlimited release
    // threshold: after the first batch every alloc/free is a pool hit, ordered on the one stream all
    // work is issued on, so no cudaMalloc/cudaFree (device-wide syncs) remain on the call path.
    void* alloc(size_t bytes) override {
        void* p = nullptr;
        EB_CUDA(cudaMallocAsync(&p, bytes ? bytes : 1, stream));
        return p;
    }
    void free(void* p) override { cudaFreeAsync(p, stream); }
    // Pinned staging blocks are kept and reused (cudaHostAlloc is slow and synchronising).
    struct HostBlock {
        void* p;
        size_t bytes;
        bool used;
    };
    std::vector<HostBlock> hostBlocks;
    std::mutex hostMu;
    void* alloc_host(size_t bytes) override {
        std::lock_guard<std::mutex> lock(hostMu);
        HostBlock* fit = nullptr;  // best fit among the cached blocks
        for (auto& b : hostBlocks)
            if (!b.used && b.bytes >= bytes && (!fit || b.bytes < fit->bytes)) fit = &b;
        if (fit) {
            fit->used = true;
            return fit->p;
        }
        for (size_t i = 0; i < hostBlocks.size() && hostBlocks.size() >= 32; ++i)  // bound the cache: drop an unused block
            if (!hostBlocks[i].used) {
                cudaFreeHost(hostBlocks[i].p);
                hostBlocks.erase(hostBlocks.begin() + i);
                break;
            }
        void* p = nullptr;
        const size_t want = bytes + bytes / 4 + 4096;
        // the pages are faulted in by this thread inside cudaHostAlloc: prefer the GPU's NUMA node for them
        // (set_mempolicy MPOL_PREFERRED for the duration of the call; best effort)
        bool policy = false;
        if (numaNode >= 0 && numaNode < 64) {
            unsigned long mask = 1ul << numaNode;
            policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 65ul) == 0;
        }
        const cudaError_t err = cudaHostAlloc(&p, want, cudaHostAllocDefault);
        if (policy) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
        EB_CUDA(err);
        hostBlocks.push_back(HostBlock{p, want, true});
        return p;
    }
    bool host_pinned(const void* p, size_t bytes) override {
        if (!p || bytes == 0) return false;
        cudaPointerAttributes a0, a1;
        if (cudaPointerGetAttributes(&a0, p) != cudaSuccess || cudaPointerGetAttributes(&a1, static_cast<const char*>(p) + bytes - 1) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        return a0.type == cudaMemoryTypeHost && a1.type == cudaMemoryTypeHost;
    }
    void free_host(void* p) override {
        std::lock_guard<std::mutex> lock(hostMu);
        for (auto& b : hostBlocks)
            if (b.p == p) b.used = false;
    }
    void h2d(void* d, const void* s, size_t n) override {
        if (n) EB_CUDA(cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, stream));
    }
    void d2h(void* d, const void* s, size_t n) override {
        if (n) EB_CUDA(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToHost, stream));
        EB_CUDA(cudaStreamSynchronize(stream));
    }
    void zero(void* d, size_t n) override {
        if (n) EB_CUDA(cudaMemsetAsync(d, 0, n, stream));
    }
    void d2d(void* d, const void* s, size_t n) override {
        if (n) EB_CUDA(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, stream));
    }
    void fill(void* d, int v, size_t n) override {
        if (n) EB_CUDA(cudaMemsetAsync(d, v, n, stream));
    }
    void sync() override { EB_CUDA(cudaStreamSynchronize(stream)); }
    void bind_thread() override { EB_CUDA(cudaSetDevice(deviceId)); }
    int sm_count() override { return sms; }

    cudaEvent_t get_event() {
        if (!pool.empty()) {
            cudaEvent_t e = pool.back();
            pool.pop_back();
            return e;
        }
        cudaEvent_t e;
        EB_CUDA(cudaEventCreate(&e));
        return e;
    }
    static void check_launch(const char* what) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) throw std::runtime_error(std::string(what) + " launch: " + cudaGetErrorString(e));
    }
    // Dynamic shared memory beyond the default 48 KiB needs the kernel's opt-in.  The attribute is the kernel's limit, not
    // a switch: it is only set above 48 KiB, so it never drops below what a later launch within the default needs.
    template <class K>
    static cudaError_t opt_in_smem(K kernel, size_t smem) {
        return smem > 48 * 1024 ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) : cudaSuccess;
    }
    // Every kernel launch: on the compute stream, timed under `name` (kernel_ms, kernel_report).
    template <class... KArgs, class... Args>
    void launch(const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, const Args&... args) {
        EB_CUDA(opt_in_smem(kernel, smem));
        Timed t{name, get_event(), get_event()};
        cudaEventRecord(t.a, stream);
        kernel<<<grid, block, smem, stream>>>(args...);
        cudaEventRecord(t.b, stream);
        timed.push_back(t);
        launchCount++;
        check_launch(name);
    }

    void launch_mask(const MaskParams& p) override {
        launch("mask", mask_kernel, (p.numItems + p.numQueries + W_WARPS - 1) / W_WARPS, W_WARPS * 32, 0, p);
    }
    void launch_alpha_len(const uint32_t* masks, const int* qset, const int* tset, int n, int* out) override {
        launch("alpha", alpha_len_kernel, (n + 255) / 256, 256, 0, masks, qset, tset, n, out);
    }
    void launch_encode(const EncodeParams& p) override {
        const uint64_t nvec = p.numBytes / 16 + 1;
        int blocks = (int)std::min<uint64_t>((nvec + 255) / 256, (uint64_t)sms * 8);
        if (blocks < 1) blocks = 1;
        launch("encode", encode_kernel, blocks, 256, 0, p);
    }

    // CTA size and dynamic shared memory of a K1 launch: four CTAs of 256 threads per SM when the
    // alphabet is small; the CTA shrinks when the per-thread Peq rows would not fit, and when there are
    // only a few reads (more, smaller CTAs are resident: such launches are latency-bound per warp).
    static void k1_block(int nw, int ncodes, int numReads, int* block, size_t* smem) {
        const size_t perThread = (size_t)ncodes * (16 + 4 * (nw > 4 ? nw - 4 : 0));
        const size_t fixed = 2 * K1_TILE + 64;
        int b = 256;
        while (b > 32 && fixed + perThread * b > 44 * 1024) b >>= 1;
        while (b > 32 && b / 2 >= numReads) b >>= 1;
        *block = b;
        *smem = fixed + perThread * b;
    }
    template <int NW>
    int k1_occupancy(int block, size_t smem) {
        int perSm = 0;
        opt_in_smem(k1_kernel<NW, MODE_HW>, smem);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, k1_kernel<NW, MODE_HW>, block, smem) != cudaSuccess) perSm = 1;
        return perSm < 1 ? 1 : perSm;
    }
    std::vector<int> shapeCache;  // [nw*1024 + ncodes] -> block | resident << 12, 0 = unknown
    void k1_shape(int nw, int ncodes, int numReads, int* blockThreads, int* residentCtas) override {
        int block;
        size_t smem;
        k1_block(nw, ncodes, numReads, &block, &smem);
        if (shapeCache.empty()) shapeCache.assign(4 * 9 * 1024, 0);
        const int blockClass = block >= 256 ? 3 : block >= 128 ? 2 : block >= 64 ? 1 : 0;
        const int key = (blockClass * 9 + nw) * 1024 + (ncodes < 1024 ? ncodes : 1023);
        if (ncodes < 1023 && shapeCache[key]) {
            *blockThreads = shapeCache[key] & 0xfff;
            *residentCtas = shapeCache[key] >> 12;
            return;
        }
        // (the window kernel keeps NW + 4 words per row: it must fit too, with 32-thread CTAs at least)
        if (smem > (size_t)maxSmemOptin || (size_t)ncodes * 4 * (nw + 4) * 32 > (size_t)maxSmemOptin) {  // not a K1 case
            *blockThreads = block;
            *residentCtas = 0;
            return;
        }
        int perSm = 1;
        with_nw(nw, [&](auto w) { perSm = k1_occupancy<decltype(w)::value>(block, smem); });
        *blockThreads = block;
        *residentCtas = perSm * sms;
        if (ncodes < 1023) shapeCache[key] = block | ((perSm * sms) << 12);
    }
    void launch_k1t(const K1Params& p, int nw) override {
        if (p.rangeMode || p.prefixLen > 0) throw std::runtime_error("k1t: plain sweeps only");
        const size_t smem = (size_t)p.ncodes * nw * sizeof(uint32_t);
        const dim3 grid((unsigned)((p.chunks + 31) / 32), (unsigned)p.numReads);
        with_nw(nw, [&](auto w) { launch("k1", k1t_kernel<decltype(w)::value>, grid, 32, smem, p); });
    }
    void launch_k1(const K1Params& p, int nw) override {
        int block;
        size_t smem;
        k1_block(nw, p.ncodes, p.numReads, &block, &smem);
        if (smem > (size_t)maxSmemOptin) throw std::runtime_error("K1: alphabet too large for shared memory");
        const dim3 grid((p.numReads + block - 1) / block, p.chunks);
        if (p.rangeMode) {  // candidate-filter sweeps: 32- or 64-row prefixes (one or two words), HW, range recording
            const char* bad = "range mode needs the 1- or 2-word HW kernel";
            if (p.mode != MODE_HW) throw std::runtime_error(bad);
            with_one_of<1, 2>(nw, bad, [&](auto w) { launch("k1_prefix", k1_kernel<decltype(w)::value, MODE_HW, true>, grid, block, smem, p); });
            return;
        }
        with_nw(nw, [&](auto w) {
            with_mode(p.mode, [&](auto m) { launch("k1", k1_kernel<decltype(w)::value, decltype(m)::value>, grid, block, smem, p); });
        });
    }
    void launch_k1w(const K1WParams& p, int nw) override {
        int block = 128;
        const size_t perThread = (size_t)p.ncodes * 4 * (nw + 4);
        while (block > 32 && perThread * block > 96 * 1024) block >>= 1;
        const size_t smem = perThread * block;
        if (smem > (size_t)maxSmemOptin) throw std::runtime_error("K1W: alphabet too large for shared memory");
        with_nw(nw, [&](auto w) {
            with_one_of<128, 64, 32>(block, "bad K1W CTA size", [&](auto threads) {
                constexpr int THREADS = decltype(threads)::value;
                launch("k1w", k1w_kernel<decltype(w)::value, THREADS>, (p.numReads + THREADS - 1) / THREADS, THREADS, smem, p);
            });
        });
    }
    void launch_lane(const LParams& p, int nw, int mode, bool rev, bool store) override {
        int block = 128;
        const size_t perThread = (size_t)p.ncodes * (16 + 4 * (nw > 4 ? nw - 4 : 0));
        while (block > 32 && perThread * block > 96 * 1024) block >>= 1;
        const size_t smem = perThread * block;
        if (smem > (size_t)maxSmemOptin) throw std::runtime_error("lane kernel: alphabet too large for shared memory");
        with_nw(nw, [&](auto w) {
            with_lane_class(mode, rev, store, [&](auto c) {
                using C = decltype(c);
                launch("lane", lane_kernel<decltype(w)::value, C::MODE, C::REV, C::STORE>, (p.numJobs + block - 1) / block, block, smem, p);
            });
        });
    }
    void launch_res(const ResParams& p) override {
        if (p.numItems <= 0) return;
        launch("res", res_kernel, (p.numItems + 255) / 256, 256, 0, p);
    }
    void launch_peq(const PeqParams& p) override {
        launch("peq", peq_kernel, (p.numJobs + W_WARPS - 1) / W_WARPS, W_WARPS * 32, 0, p);
    }
    void launch_w(const WParams& p, int R) override {
        with_r(R, [&](auto r) { launch("w", w_kernel<decltype(r)::value>, (p.numJobs + W_WARPS - 1) / W_WARPS, W_WARPS * 32, 0, p); });
    }
    static size_t band_smem(int NB, int ncodes) { return (size_t)ncodes * (4 * NB + BAND_SLACK) * 4 * BAND_THREADS; }
    int band_max_blocks(int ncodes) override {
        int nb = 0;
        while (nb < 8 && band_smem(nb + 1, ncodes) <= (size_t)110 * 1024) ++nb;  // two CTAs per SM at least
        return nb;
    }
    void launch_band(const WParams& p, int NB, int ncodes) override {
        with_nb(NB, [&](auto nb) {
            launch("band", band_kernel<decltype(nb)::value>, (p.numJobs + BAND_THREADS - 1) / BAND_THREADS, BAND_THREADS, band_smem(NB, ncodes), p,
                   ncodes);
        });
    }
    void launch_seed_count(const SeedIndexParams& p) override { launch("seed_count", seed_count_kernel, (p.numPos + 255) / 256, 256, 0, p); }
    void launch_seed_fill(const SeedIndexParams& p) override { launch("seed_fill", seed_fill_kernel, (p.numPos + 255) / 256, 256, 0, p); }
    void launch_scan(int* data, int count) override {
        if (count <= 0) {  // no tiles (a launch of no CTAs is refused): only the total, 0
            zero(data, sizeof(int));
            return;
        }
        const int numTiles = (count + SCAN_TILE - 1) / SCAN_TILE;
        int* tileSums = static_cast<int*>(alloc((size_t)numTiles * sizeof(int)));
        launch("scan", scan_tile_sums_kernel, numTiles, SCAN_THREADS, 0, data, count, tileSums);
        launch("scan", scan_top_kernel, 1, 1024, 0, tileSums, numTiles, data + count);
        launch("scan", scan_apply_kernel, numTiles, SCAN_THREADS, 0, data, count, tileSums);
        free(tileSums);
    }
    template <int CAP, int THREADS, int GW>
    void launch_seed_plan_t(const SeedPlanParams& p) {
        constexpr int GROUPS = THREADS / GW;
        const size_t smem = (size_t)GROUPS * ((size_t)CAP + seed_ctl_words(GW)) * sizeof(int);
        launch("seed_plan", seed_plan_kernel<CAP, THREADS, CoopGroup<GW>>, (p.numReads + GROUPS - 1) / GROUPS, THREADS, smem, p);
    }
    void launch_seed_plan(const SeedPlanParams& p) override {
        with_seed_plan_instance(p, [&](auto cap, auto threads, auto gw) {
            launch_seed_plan_t<decltype(cap)::value, decltype(threads)::value, decltype(gw)::value>(p);
        });
    }
    void launch_fin_count(const FinParams& p) override { launch("fin_count", fin_count_kernel, (p.numReads + 255) / 256, 256, 0, p); }
    void launch_fin_fill(const FinParams& p) override { launch("fin_fill", fin_fill_kernel, (p.numReads + 255) / 256, 256, 0, p); }
    void launch_qalpha(const QAlphaParams& p) override { launch("qalpha", qalpha_kernel, (p.numQueries + 7) / 8, 256, 0, p); }
    void launch_win_reduce(const WinReduceParams& p) override { launch("win_reduce", win_reduce_kernel, (p.numReads + 127) / 128, 128, 0, p); }
    void launch_split(const SplitParams& p) override { launch("split", split_kernel, (p.numNodes + 63) / 64, 64, 0, p); }
    void launch_traceback(const TbParams& p) override { launch("traceback", traceback_kernel, (p.numJobs + 127) / 128, 128, 0, p); }
    void reset_timing() override {
        for (auto& t : timed) {
            pool.push_back(t.a);
            pool.push_back(t.b);
        }
        timed.clear();
        launchCount = 0;
    }
    double kernel_ms(const char* name) override {
        cudaStreamSynchronize(stream);
        double total = 0;
        for (auto& t : timed) {
            if (name && strcmp(name, t.name) != 0) continue;
            float ms = 0;
            if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) total += ms;
        }
        return total;
    }
    int launches() override { return launchCount; }
    std::string kernel_report() override {
        cudaStreamSynchronize(stream);
        std::vector<std::string> names;
        std::vector<double> ms;
        std::vector<int> count;
        for (auto& t : timed) {
            size_t i = 0;
            while (i < names.size() && names[i] != t.name) ++i;
            if (i == names.size()) {
                names.push_back(t.name);
                ms.push_back(0);
                count.push_back(0);
            }
            float e = 0;
            if (cudaEventElapsedTime(&e, t.a, t.b) == cudaSuccess) ms[i] += e;
            count[i]++;
        }
        std::string out;
        for (size_t i = 0; i < names.size(); ++i) {
            char buf[96];
            snprintf(buf, sizeof(buf), "%s%s:%.4f:%d", i ? ";" : "", names[i].c_str(), ms[i], count[i]);
            out += buf;
        }
        return out;
    }
};

// Device chosen through edlibB200SetDevice (-1: none, the backend takes the creating thread's current device).
static int g_selectedDevice = -1;

int select_device(int device, std::string* err) {
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        if (err) *err = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
        return 1;
    }
    g_selectedDevice = device;  // under the library lock (eb_capi.cpp)
    return 0;
}

Backend* create_backend(std::string* err) {
    try {
        int count = 0;
        cudaError_t e = cudaGetDeviceCount(&count);
        if (e != cudaSuccess || count == 0) {
            if (err) *err = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
            return nullptr;
        }
        // the backend may be created by another host thread than the one that selected the device
        if (g_selectedDevice >= 0 && (e = cudaSetDevice(g_selectedDevice)) != cudaSuccess) {
            if (err) *err = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
            return nullptr;
        }
        return new CudaBackend();
    } catch (const std::exception& ex) {
        if (err) *err = ex.what();
        return nullptr;
    }
}

}  // namespace eb
