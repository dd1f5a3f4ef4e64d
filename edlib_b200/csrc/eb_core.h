// eb_core.h -- the kernel BODIES, written once and compiled twice:
//   * by nvcc for sm_90a (eb_kernels.cu wraps them in __global__ functions), and
//   * by g++ for the host SIMT emulation the CPU test-suite uses to check the kernel logic
//     (tests/emul/): per-thread bodies run in a loop, warp-cooperative bodies are instantiated
//     on a 32-wide vector backend.  The emulation is test infrastructure, never a product path.
//
// Reference functions re-expressed here (all in reference edlib/src/edlib.cpp):
//   calculateBlock 412-447 -> k1_step / w_sweep column step (32-bit words, multi-word carries)
//   buildPeq 358-384       -> K1PeqBuild / peq_build_job
//   myersCalcEditDistanceSemiGlobal 550-704, myersCalcEditDistanceNW 730-928 -> k1_* / w_sweep
//   obtainAlignmentTraceback 942-1141 -> traceback_job
#pragma once
#include <type_traits>

#include "eb_common.h"

#if defined(__CUDA_ARCH__)
#define EB_UNROLL _Pragma("unroll")
#else
#define EB_UNROLL
#endif

namespace eb {

// ---------------------------------------------------------------------------------------------
// Small primitives with a device and a host spelling
// ---------------------------------------------------------------------------------------------

// (hi << 1) | (lo >> 31): one bit moving up across a word boundary.
EB_HD uint32_t funnel_l1(uint32_t lo, uint32_t hi) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, 1);
#else
    return (hi << 1) | (lo >> 31);
#endif
}

EB_HD int popcount32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

EB_HD int atomic_add_int(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    int old = *p;
    *p = old + v;
    return old;
#endif
}

EB_HD void atomic_max_int(int* p, int v) {
#if defined(__CUDA_ARCH__)
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}

EB_HD void atomic_or_u32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}

// S = T + P over NW 32-bit words with the carry rippling from word 0 upward.  On the device the
// whole chain is ONE asm statement so that nothing can be scheduled between the add.cc/addc.cc
// links (IADD3 / IADD3.X in SASS).
template <int NW>
struct AddChain {
    static EB_HD void run(uint32_t (&S)[NW], const uint32_t (&T)[NW], const uint32_t (&P)[NW]) {
        uint32_t carry = 0;
        EB_UNROLL
        for (int w = 0; w < NW; ++w) {
            uint64_t s = (uint64_t)T[w] + P[w] + carry;
            S[w] = (uint32_t)s;
            carry = (uint32_t)(s >> 32);
        }
    }
};
#if defined(__CUDA_ARCH__)
template <>
struct AddChain<1> {
    static EB_HD void run(uint32_t (&S)[1], const uint32_t (&T)[1], const uint32_t (&P)[1]) { S[0] = T[0] + P[0]; }
};
template <>
struct AddChain<2> {
    static EB_HD void run(uint32_t (&S)[2], const uint32_t (&T)[2], const uint32_t (&P)[2]) {
        asm("add.cc.u32 %0, %2, %4;\n\taddc.u32 %1, %3, %5;"
            : "=&r"(S[0]), "=&r"(S[1]) : "r"(T[0]), "r"(T[1]), "r"(P[0]), "r"(P[1]));
    }
};
template <>
struct AddChain<3> {
    static EB_HD void run(uint32_t (&S)[3], const uint32_t (&T)[3], const uint32_t (&P)[3]) {
        asm("add.cc.u32 %0, %3, %6;\n\taddc.cc.u32 %1, %4, %7;\n\taddc.u32 %2, %5, %8;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(P[0]), "r"(P[1]), "r"(P[2]));
    }
};
template <>
struct AddChain<4> {
    static EB_HD void run(uint32_t (&S)[4], const uint32_t (&T)[4], const uint32_t (&P)[4]) {
        asm("add.cc.u32 %0, %4, %8;\n\taddc.cc.u32 %1, %5, %9;\n\taddc.cc.u32 %2, %6, %10;\n\taddc.u32 %3, %7, %11;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(P[0]), "r"(P[1]), "r"(P[2]), "r"(P[3]));
    }
};
template <>
struct AddChain<5> {
    static EB_HD void run(uint32_t (&S)[5], const uint32_t (&T)[5], const uint32_t (&P)[5]) {
        asm("add.cc.u32 %0, %5, %10;\n\taddc.cc.u32 %1, %6, %11;\n\taddc.cc.u32 %2, %7, %12;\n\t"
            "addc.cc.u32 %3, %8, %13;\n\taddc.u32 %4, %9, %14;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(T[4]),
              "r"(P[0]), "r"(P[1]), "r"(P[2]), "r"(P[3]), "r"(P[4]));
    }
};
template <>
struct AddChain<6> {
    static EB_HD void run(uint32_t (&S)[6], const uint32_t (&T)[6], const uint32_t (&P)[6]) {
        asm("add.cc.u32 %0, %6, %12;\n\taddc.cc.u32 %1, %7, %13;\n\taddc.cc.u32 %2, %8, %14;\n\t"
            "addc.cc.u32 %3, %9, %15;\n\taddc.cc.u32 %4, %10, %16;\n\taddc.u32 %5, %11, %17;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(T[4]), "r"(T[5]),
              "r"(P[0]), "r"(P[1]), "r"(P[2]), "r"(P[3]), "r"(P[4]), "r"(P[5]));
    }
};
template <>
struct AddChain<7> {
    static EB_HD void run(uint32_t (&S)[7], const uint32_t (&T)[7], const uint32_t (&P)[7]) {
        asm("add.cc.u32 %0, %7, %14;\n\taddc.cc.u32 %1, %8, %15;\n\taddc.cc.u32 %2, %9, %16;\n\t"
            "addc.cc.u32 %3, %10, %17;\n\taddc.cc.u32 %4, %11, %18;\n\taddc.cc.u32 %5, %12, %19;\n\t"
            "addc.u32 %6, %13, %20;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5]), "=&r"(S[6])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(T[4]), "r"(T[5]), "r"(T[6]),
              "r"(P[0]), "r"(P[1]), "r"(P[2]), "r"(P[3]), "r"(P[4]), "r"(P[5]), "r"(P[6]));
    }
};
template <>
struct AddChain<8> {
    static EB_HD void run(uint32_t (&S)[8], const uint32_t (&T)[8], const uint32_t (&P)[8]) {
        asm("add.cc.u32 %0, %8, %16;\n\taddc.cc.u32 %1, %9, %17;\n\taddc.cc.u32 %2, %10, %18;\n\t"
            "addc.cc.u32 %3, %11, %19;\n\taddc.cc.u32 %4, %12, %20;\n\taddc.cc.u32 %5, %13, %21;\n\t"
            "addc.cc.u32 %6, %14, %22;\n\taddc.u32 %7, %15, %23;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5]), "=&r"(S[6]), "=&r"(S[7])
            : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(T[4]), "r"(T[5]), "r"(T[6]), "r"(T[7]),
              "r"(P[0]), "r"(P[1]), "r"(P[2]), "r"(P[3]), "r"(P[4]), "r"(P[5]), "r"(P[6]), "r"(P[7]));
    }
};
#endif

// S = X << 1 over NW words as the add X + X with the carry rippling upward; the bit shifted out of the
// last word (the last query row, see eb_common.h) is added to `top`.  On the H100 the integer add issues
// at twice the rate of the funnel shift (scripts/microbench/pipes.cu: IADD 0.97 vs SHF 0.49
// warp-instructions/clk/SMSP) and the carry-out replaces the separate extraction of the last-row bit.
template <int NW>
struct ShiftChain {
    static EB_HD void run(uint32_t (&S)[NW], const uint32_t (&X)[NW], int& top) {
        EB_UNROLL
        for (int w = NW - 1; w > 0; --w) S[w] = (X[w] << 1) | (X[w - 1] >> 31);
        S[0] = X[0] << 1;
        top += (int)(X[NW - 1] >> 31);
    }
};
#if defined(__CUDA_ARCH__)
template <>
struct ShiftChain<1> {
    static EB_HD void run(uint32_t (&S)[1], const uint32_t (&X)[1], int& top) {
        asm("add.cc.u32 %0, %2, %2;\n\taddc.u32 %1, %1, 0;"
            : "=&r"(S[0]), "+r"(top) : "r"(X[0]));
    }
};
template <>
struct ShiftChain<2> {
    static EB_HD void run(uint32_t (&S)[2], const uint32_t (&X)[2], int& top) {
        asm("add.cc.u32 %0, %3, %3;\n\taddc.cc.u32 %1, %4, %4;\n\taddc.u32 %2, %2, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "+r"(top) : "r"(X[0]), "r"(X[1]));
    }
};
template <>
struct ShiftChain<3> {
    static EB_HD void run(uint32_t (&S)[3], const uint32_t (&X)[3], int& top) {
        asm("add.cc.u32 %0, %4, %4;\n\taddc.cc.u32 %1, %5, %5;\n\taddc.cc.u32 %2, %6, %6;\n\taddc.u32 %3, %3, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]));
    }
};
template <>
struct ShiftChain<4> {
    static EB_HD void run(uint32_t (&S)[4], const uint32_t (&X)[4], int& top) {
        asm("add.cc.u32 %0, %5, %5;\n\taddc.cc.u32 %1, %6, %6;\n\taddc.cc.u32 %2, %7, %7;\n\taddc.cc.u32 %3, %8, %8;\n\taddc.u32 %4, %4, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]), "r"(X[3]));
    }
};
template <>
struct ShiftChain<5> {
    static EB_HD void run(uint32_t (&S)[5], const uint32_t (&X)[5], int& top) {
        asm("add.cc.u32 %0, %6, %6;\n\taddc.cc.u32 %1, %7, %7;\n\taddc.cc.u32 %2, %8, %8;\n\taddc.cc.u32 %3, %9, %9;\n\taddc.cc.u32 %4, %10, %10;\n\taddc.u32 %5, %5, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]));
    }
};
template <>
struct ShiftChain<6> {
    static EB_HD void run(uint32_t (&S)[6], const uint32_t (&X)[6], int& top) {
        asm("add.cc.u32 %0, %7, %7;\n\taddc.cc.u32 %1, %8, %8;\n\taddc.cc.u32 %2, %9, %9;\n\taddc.cc.u32 %3, %10, %10;\n\taddc.cc.u32 %4, %11, %11;\n\taddc.cc.u32 %5, %12, %12;\n\taddc.u32 %6, %6, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]));
    }
};
template <>
struct ShiftChain<7> {
    static EB_HD void run(uint32_t (&S)[7], const uint32_t (&X)[7], int& top) {
        asm("add.cc.u32 %0, %8, %8;\n\taddc.cc.u32 %1, %9, %9;\n\taddc.cc.u32 %2, %10, %10;\n\taddc.cc.u32 %3, %11, %11;\n\taddc.cc.u32 %4, %12, %12;\n\taddc.cc.u32 %5, %13, %13;\n\taddc.cc.u32 %6, %14, %14;\n\taddc.u32 %7, %7, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5]), "=&r"(S[6]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]));
    }
};
template <>
struct ShiftChain<8> {
    static EB_HD void run(uint32_t (&S)[8], const uint32_t (&X)[8], int& top) {
        asm("add.cc.u32 %0, %9, %9;\n\taddc.cc.u32 %1, %10, %10;\n\taddc.cc.u32 %2, %11, %11;\n\taddc.cc.u32 %3, %12, %12;\n\taddc.cc.u32 %4, %13, %13;\n\taddc.cc.u32 %5, %14, %14;\n\taddc.cc.u32 %6, %15, %15;\n\taddc.cc.u32 %7, %16, %16;\n\taddc.u32 %8, %8, 0;"
            : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(S[4]), "=&r"(S[5]), "=&r"(S[6]), "=&r"(S[7]), "+r"(top) : "r"(X[0]), "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]), "r"(X[7]));
    }
};
#endif

// Pv word for the column before the first one: ones on real rows, zeros on padding bits.
EB_HD uint32_t init_pv_word(int wordIdx, int off) {
    const int lo = wordIdx * 32;
    if (off <= lo) return ~0u;
    if (off >= lo + 32) return 0u;
    return ~0u << (off - lo);
}

// =============================================================================================
// K1 -- one alignment per thread, query words in registers, Peq rows in shared memory
// =============================================================================================

// One DP column for one query held in NW 32-bit words.  Same recurrences as the reference's
// calculateBlock (cpp:421-444) but over ONE NW*32-bit integer: the add carry and the <<1 carry
// cross word boundaries natively, so no per-block hin/hout is needed.  TOP_ONE selects the
// horizontal delta entering above row 0: +1 for NW/SHW (cpp:779, 584), 0 for HW.
// The last-row score is kept as score = up - down: both <<1 shifts are add-with-carry chains whose carry-out
// (the last-row bit of Ph / Mh) accumulates into `up` / `down`.
// (Measured alternative, dropped: doing the <<1 with IMAD/IMAD.HI on the FMA pipe is slower because the
// high-half multiply is quarter-rate on the H100; scripts/microbench/pipes.cu.)
template <int NW, bool TOP_ONE>
EB_HD void k1_step(uint32_t (&Pv)[NW], uint32_t (&Mv)[NW], const uint32_t (&Eq)[NW], int& up, int& down, uint32_t* phOut = nullptr) {
    uint32_t T[NW], S[NW], Ph[NW], Mh[NW];
    EB_UNROLL
    for (int w = 0; w < NW; ++w) T[w] = Eq[w] & Pv[w];
    AddChain<NW>::run(S, T, Pv);
    EB_UNROLL
    for (int w = 0; w < NW; ++w) {
        const uint32_t Xh = (S[w] ^ Pv[w]) | Eq[w];
        Ph[w] = Mv[w] | ~(Xh | Pv[w]);
        Mh[w] = Pv[w] & Xh;
    }
    if (phOut) {  // matrix-storing sweeps keep the unshifted horizontal +1 deltas for the traceback
        EB_UNROLL
        for (int w = 0; w < NW; ++w) phOut[w] = Ph[w];
    }
    uint32_t Phs[NW], Mhs[NW];
    ShiftChain<NW>::run(Phs, Ph, up);
    ShiftChain<NW>::run(Mhs, Mh, down);
    if (TOP_ONE) Phs[0] |= 1u;
    EB_UNROLL
    for (int w = 0; w < NW; ++w) {
        const uint32_t Xv = Eq[w] | Mv[w];
        Pv[w] = Mhs[w] | ~(Xv | Phs[w]);
        Mv[w] = Phs[w] & Xv;
    }
}

// Per-thread K1 state that lives across target tiles.
template <int NW>
struct K1State {
    uint32_t Pv[NW], Mv[NW];
    int up, down;  // D[m-1][c] of the last column swept = up - down
    int best;   // running minimum (starts at the bound sentinel)
    int cnt;    // columns attaining best so far
    int first, last;  // RANGE mode: the open candidate range (cnt columns; 0 = none open)
    int emitted;      // RANGE mode: ranges written to the list so far
};

template <int NW>
EB_HD void k1_init(K1State<NW>& st, int m, int kInit) {
    const int off = 32 * NW - m;
    EB_UNROLL
    for (int w = 0; w < NW; ++w) {
        st.Pv[w] = init_pv_word(w, off);
        st.Mv[w] = 0;
    }
    st.up = m;  // D[m-1][-1] = m  (ref cpp:576, 760)
    st.down = 0;
    st.best = kInit;
    st.cnt = 0;
    st.first = st.last = 0;
    st.emitted = 0;
}

// RANGE mode (candidate filter): the columns whose prefix score is at or below the fixed threshold
// st.best are reported as ranges {read slot, first, last} appended to a list (the Ovf array of the
// launch: rec = slot, score = first, pos = last).  A range is closed when the next candidate lies more
// than K1_RANGE_GAP columns after its last or K1_RANGE_SPAN after its first one.  A thread that has
// written K1_RANGE_MAX ranges appends the marker {slot, -1, -1} and stops recording: the host hands
// such a read to the next stage.
template <int NW>
EB_HD void k1_range_flush(K1State<NW>& st, int slot, Ovf* list, int* listCount, int listCap) {
    if (st.cnt == 0) return;
    int i = atomic_add_int(listCount, 1);
    if (i < listCap) {
        list[i].rec = slot;
        list[i].score = st.first;
        list[i].pos = st.last;
    }
    st.cnt = 0;
    if (++st.emitted >= K1_RANGE_MAX) {
        i = atomic_add_int(listCount, 1);
        if (i < listCap) {
            list[i].rec = slot;
            list[i].score = -1;
            list[i].pos = -1;
        }
        st.best = -1;  // scores are never negative: nothing is recorded any more
    }
}

// Restates the bookkeeping of ref cpp:658-673: a strictly better score restarts the list.
// RecT is Rec (KPOS inline positions) or WinRec (KPOSW).
template <int NW, bool RANGE = false, class RecT>
EB_HD void k1_event(K1State<NW>& st, int score, int column, RecT* rec, int recIdx, Ovf* ovf, int* ovfCount, int ovfCap) {
    constexpr int CAP = (int)(sizeof(rec->pos) / sizeof(rec->pos[0]));
    if (RANGE) {  // candidate filter: recIdx is the read slot, ovf the range list
        if (st.cnt > 0 && (column - st.last > K1_RANGE_GAP || column - st.first > K1_RANGE_SPAN)) {
            k1_range_flush<NW>(st, recIdx, ovf, ovfCount, ovfCap);
            if (st.best < 0) return;
        }
        if (st.cnt == 0) st.first = column;
        st.last = column;
        st.cnt++;
        return;
    }
    if (score < st.best) {
        st.best = score;
        st.cnt = 0;
    }
    if (st.cnt < CAP) {
        rec->pos[st.cnt] = column;
    } else if (ovfCap > 0) {  // second pass only: the list then holds final positions exclusively
        const int slot = atomic_add_int(ovfCount, 1);
        if (slot < ovfCap) {
            ovf[slot].rec = recIdx;
            ovf[slot].score = score;
            ovf[slot].pos = column;
        }
    }
    rec->last = column;
    st.cnt++;
}

// Hits of one job of a hits launch (eb_common.h: HitParams), in the order the sweep meets them (ascending columns):
// all are counted, the first `room` stored.  Sweeps that record into a HitSink compare against a fixed threshold
// (st.best / K1Band::best stays k) instead of a running minimum.
struct HitSink {
    int count, room;
    int* cols;
    int* scores;
    EB_HD void hit(int score, int column) {
        if (count < room) {
            cols[count] = column;
            scores[count] = score;
        }
        ++count;
    }
};
// The sink of job `job`, or false in a fill pass when nothing of the job is stored.
EB_HD bool hit_sink_open(const HitParams& h, int job, HitSink& s) {
    s.count = 0;
    s.room = h.at ? h.room[job] : 0;
    s.cols = h.at ? h.cols + h.at[job] : nullptr;
    s.scores = h.at ? h.scores + h.at[job] : nullptr;
    return !h.at || s.room > 0;
}
// The sink of a record target (HitParams::sepCodes): a separator column is never a hit, so the count pass sees exact
// counts.  Its own kernel instances run it; the plain sink stays free of the test.
struct RecordHitSink : HitSink {
    const uint8_t* sepCodes;
    int sep;
    EB_HD void hit(int score, int column) {
        if (sepCodes[column] != sep) HitSink::hit(score, column);
    }
};
EB_HD bool hit_sink_open(const HitParams& h, int job, RecordHitSink& s) {
    s.sepCodes = h.sepCodes;
    s.sep = h.sep;
    return hit_sink_open(h, job, static_cast<HitSink&>(s));
}
EB_HD void hit_sink_close(const HitParams& h, int job, const HitSink& s) {
    if (!h.at) h.count[job] = s.count;
}
template <int NW, bool RANGE = false>
EB_HD void k1_event(K1State<NW>&, int score, int column, HitSink* sink, int, Ovf*, int*, int) {
    sink->hit(score, column);
}
template <int NW, bool RANGE = false>
EB_HD void k1_event(K1State<NW>&, int score, int column, RecordHitSink* sink, int, Ovf*, int*, int) {
    sink->hit(score, column);
}

// Target symbols addressed through a plain pointer (host emulation; any directly addressable
// target).  The device kernel substitutes a reader over its shared-memory tile.
struct PtrSyms {
    const uint8_t* p;
    EB_HD uint32_t read1(int i) const { return p[i]; }
};
// The same, walking the target backwards from p (reversed sweeps of ref cpp:253-257).
struct RevSyms {
    const uint8_t* p;
    EB_HD uint32_t read1(int i) const { return *(p - i); }
};

// Sweeps `count` consecutive target symbols starting at absolute column cAbs.  `Acc` hands out
// the Eq words of a symbol (shared memory on the device), `Syms` the symbols.  With TRACK the
// running minimum and its columns are recorded; without it only the state advances (halo
// columns of a chunk).  Columns go four at a time: the four last-row scores stay in registers
// and are compared against the running minimum once per group (events are rare).
template <int NW, bool TOP_ONE, bool TRACK, bool RANGE = false, class Acc, class Syms, class RecT>
EB_HD void k1_columns(K1State<NW>& st, const Acc& acc, const Syms& syms, int count, int cAbs,
                      RecT* rec, int recIdx, Ovf* ovf, int* ovfCount, int ovfCap) {
    int i = 0;
    for (; i + 4 <= count; i += 4) {  // body: groups of four columns (byte reads: LSU, not ALU, work)
        int sc[4];
        EB_UNROLL
        for (int j = 0; j < 4; ++j) {
            uint32_t Eq[NW];
            acc.load(syms.read1(i + j), Eq);
            k1_step<NW, TOP_ONE>(st.Pv, st.Mv, Eq, st.up, st.down);
            sc[j] = st.up - st.down;
        }
        if (TRACK) {
            int lo = sc[0] < sc[1] ? sc[0] : sc[1];
            const int lo2 = sc[2] < sc[3] ? sc[2] : sc[3];
            lo = lo < lo2 ? lo : lo2;
            if (lo <= st.best) {
                EB_UNROLL
                for (int j = 0; j < 4; ++j)
                    if (sc[j] <= st.best) k1_event<NW, RANGE>(st, sc[j], cAbs + i + j, rec, recIdx, ovf, ovfCount, ovfCap);
            }
        }
    }
    for (; i < count; ++i) {  // tail
        uint32_t Eq[NW];
        acc.load(syms.read1(i), Eq);
        k1_step<NW, TOP_ONE>(st.Pv, st.Mv, Eq, st.up, st.down);
        if (TRACK && st.up - st.down <= st.best) k1_event<NW, RANGE>(st, st.up - st.down, cAbs + i, rec, recIdx, ovf, ovfCount, ovfCap);
    }
}

// Query profile for one K1 thread (ref buildPeq cpp:358-384 with top padding instead of the
// bottom wildcard rows).  `Acc::store(code, w, bits)` writes one Eq word, `Acc::or_word(code, w, bits)` ORs into it.
// Plain equality: every row starts as its padding bits and ONE pass over the m characters sets the bit of each
// character in the row of its code (m read-modify-writes instead of ncodes * NW * 32 bit tests); a character
// whose code is not a row (the foreign-byte code of streamed batches) matches nothing.  With an equality table
// every (code, bit) is tested as before.
template <int NW, class Acc>
EB_HD void k1_build_peq(Acc& acc, const uint8_t* q, int m, int mode, int ncodes, const uint8_t* eqtab, bool rev = false) {
    const int off = 32 * NW - m;
    const uint32_t padBit = (mode == MODE_HW) ? 1u : 0u;
    if (!eqtab) {
        for (int code = 0; code < ncodes; ++code) {
            EB_UNROLL
            for (int w = 0; w < NW; ++w) acc.store(code, w, padBit ? ~init_pv_word(w, off) : 0u);
        }
        for (int r = 0; r < m; ++r) {
            const int qc = rev ? q[m - 1 - r] : q[r];
            const int g = r + off;
            if (qc < ncodes) acc.or_word(qc, g >> 5, 1u << (g & 31));
        }
        return;
    }
    for (int code = 0; code < ncodes; ++code) {
        for (int w = 0; w < NW; ++w) {
            uint32_t bits = 0;
            for (int b = 0; b < 32; ++b) {
                const int g = w * 32 + b;
                uint32_t bit;
                if (g < off) {
                    bit = padBit;
                } else {
                    const int qc = rev ? q[m - 1 - (g - off)] : q[g - off];
                    bit = eqtab[qc * ncodes + code] ? 1u : 0u;
                }
                bits |= bit << b;
            }
            acc.store(code, w, bits);
        }
    }
}

// Chunk geometry of a K1 launch: chunk j owns columns [cs, ce) and starts sweeping at hs.
struct K1Chunk {
    int hs, cs, ce;
};
EB_HD K1Chunk k1_chunk(const K1Params& p, int chunk) {
    K1Chunk g;
    long long cs = (long long)chunk * p.chunkLen;
    long long ce = cs + p.chunkLen;
    if (cs > p.n) cs = p.n;
    if (ce > p.n) ce = p.n;
    long long hs = cs - p.halo;
    if (hs < 0) hs = 0;
    hs &= ~15LL;  // keep tile copies 16-byte aligned; a longer halo is still exact
    g.hs = (int)hs;
    g.cs = (int)cs;
    g.ce = (int)ce;
    return g;
}

// Whole K1 work item for one thread when the target is directly addressable (host emulation,
// and the reference shape for the device kernel, which adds shared-memory tiling around it).
template <int NW, class Acc, bool BUILD = true>
EB_HD void k1_thread(const K1Params& p, int slot, int chunk, Acc& acc) {
    const int pair = p.readList[slot];
    const int m = p.prefixLen > 0 ? p.prefixLen : p.qlen[pair];
    const uint8_t* q = p.qcodes + p.qoff[pair];
    const int recIdx = chunk * p.numReads + slot;
    Rec* rec = p.rangeMode ? nullptr : p.recs + recIdx;
    if (BUILD) k1_build_peq<NW>(acc, q, m, p.mode, p.ncodes, p.eqtab);  // (else: the caller built the profile, shared by a warp)
    K1State<NW> st;
    k1_init<NW>(st, m, p.kInit[slot]);
    const K1Chunk g = k1_chunk(p, chunk);
    if (p.mode == MODE_HW && p.rangeMode) {
        k1_columns<NW, false, false, true>(st, acc, PtrSyms{p.tcodes + g.hs}, g.cs - g.hs, g.hs, rec, slot, p.ovf, p.ovfCount, p.ovfCap);
        k1_columns<NW, false, true, true>(st, acc, PtrSyms{p.tcodes + g.cs}, g.ce - g.cs, g.cs, rec, slot, p.ovf, p.ovfCount, p.ovfCap);
        k1_range_flush<NW>(st, slot, p.ovf, p.ovfCount, p.ovfCap);
        return;
    } else if (p.mode == MODE_HW) {
        k1_columns<NW, false, false>(st, acc, PtrSyms{p.tcodes + g.hs}, g.cs - g.hs, g.hs, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
        k1_columns<NW, false, true>(st, acc, PtrSyms{p.tcodes + g.cs}, g.ce - g.cs, g.cs, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
    } else if (p.mode == MODE_SHW) {
        k1_columns<NW, true, true>(st, acc, PtrSyms{p.tcodes + g.cs}, g.ce - g.cs, g.cs, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
    } else {
        k1_columns<NW, true, false>(st, acc, PtrSyms{p.tcodes + g.cs}, g.ce - g.cs, g.cs, rec, recIdx, p.ovf, p.ovfCount, p.ovfCap);
        st.best = st.up - st.down;  // NW: the bottom-right cell (ref cpp:916)
        st.cnt = 1;
        rec->last = p.n - 1;
        rec->pos[0] = p.n - 1;
    }
    rec->best = st.best;
    rec->cnt = st.cnt;
}

// (lo:hi) >> sh, low word; sh in 0..31.
EB_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, int sh) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}

// View of a word-addressable profile (rows of NW + 4 words, see k1w_thread) as the NW-word K1 profile.
template <int NW, class WAcc>
struct K1View {
    WAcc& a;
    EB_HD void store(int code, int w, uint32_t bits) { a.store_word(code, w + 2, bits); }
    EB_HD void or_word(int code, int w, uint32_t bits) { a.or_word(code, w + 2, bits); }
    EB_HD void load(uint32_t code, uint32_t (&Eq)[NW]) const {
        EB_UNROLL
        for (int w = 0; w < NW; ++w) Eq[w] = a.load_word(code, w + 2);
    }
};

// Banded window sweep (one K1W work item whose end columns of interest span few diagonals).
//
// Only scores <= t at the tracked columns [lo, hi] matter (t = kInit - 1), and an alignment with <= t edits that
// ends at (m-1, e) stays within t diagonals of its last cell, so every cell that can matter lies on the
// diagonals c - r in [lo-(m-1)-t, hi-(m-1)+t]: H = (hi-lo) + 2t + 1 of them.  With H <= 64 a 64-row window
// that moves down one row per column covers them: bit k of the state of column j is row top(j) + k,
// top(j) = j - dhi.  In that frame the Myers recurrences lose their shifts of the horizontal deltas (they
// cancel against the moving window) and gain one shift of the diagonal vector (Hyyro's banded form):
//     D0 = (((Eq & VP) + VP) ^ VP) | Eq | VN        diagonal zero-delta of the cells of column j
//     HP = VN | ~(D0 | VP),  HN = VP & D0           horizontal deltas
//     X  = D0 >> 1
//     VN' = X & HP,  VP' = HN | ~(X | HP)           vertical deltas of column j, window of column j+1
// Cells outside the window never enter: the top cell gets no contribution from above, the new bottom cell
// none from its left (X brings in a 0), so every value is an upper bound of the true one and exact wherever
// the optimal path stays inside -- which is the case for all scores <= t at tracked columns.  Rows above the
// query (window rows < 0) are the wildcard rows of HW mode: Eq = 1, deltas 0 (two words of ones in front of the
// profile); rows below it carry Eq = 0 and influence nothing above them.  The score of the window's bottom
// cell is carried along (S += 1 - HN[63]); the last-row score at a tracked column is S minus the vertical
// deltas between the last row and the bottom (two popcounts).
// 16 target symbols at once (the device reads them as one 128-bit load; windows start at multiples of 16 symbols
// of a 16-byte aligned target with >= 16 bytes of slack behind it).
struct Sym16 {
    uint32_t w[4];
};
EB_HD Sym16 load_sym16(const uint8_t* p) {
    Sym16 v;
#if defined(__CUDA_ARCH__)
    const uint4 x = __ldg(reinterpret_cast<const uint4*>(p));
    v.w[0] = x.x;
    v.w[1] = x.y;
    v.w[2] = x.z;
    v.w[3] = x.w;
#else
    for (int k = 0; k < 4; ++k)
        v.w[k] = (uint32_t)p[4 * k] | ((uint32_t)p[4 * k + 1] << 8) | ((uint32_t)p[4 * k + 2] << 16) | ((uint32_t)p[4 * k + 3] << 24);
#endif
    return v;
}

// State of one banded sweep (see k1b_sweep) and its column step.
template <class WAcc, class RecT>
struct K1Band {
    const WAcc& acc;
    RecT* rec;
    uint32_t VP0, VP1, VN0, VN1;
    int S;          // score of the window's bottom cell
    int best, cnt;
    int g0;         // profile bit of the window's top row at column 0
    int lo;         // first tracked column
    int kb0;        // window bit of the last query row at column 0 (frame of the following column): kb = kb0 - j
    int ws;         // absolute column of window column 0
    const K1WParams& prm;  // overflow list of end columns beyond the inline ones
    int slot;

    // Smallest value among the cells of the column just swept that lie in the current frame (the window of the
    // next column): D of the bottom cell is S, the vertical deltas lead upwards from there.
    EB_HD int window_min() const {
        int cur = S, mn = S;
        for (int k = 31; k >= 0; --k) {
            cur += (int)((VN1 >> k) & 1u) - (int)((VP1 >> k) & 1u);
            mn = cur < mn ? cur : mn;
        }
        for (int k = 31; k >= 1; --k) {
            cur += (int)((VN0 >> k) & 1u) - (int)((VP0 >> k) & 1u);
            mn = cur < mn ? cur : mn;
        }
        return mn;
    }

    template <bool TRACK>
    EB_HD void column(int j, uint32_t sym) {
        const int gt = j + g0;
        const int wi = gt >> 5, sh = gt & 31;
        const uint32_t w0 = acc.load_word(sym, wi), w1 = acc.load_word(sym, wi + 1), w2 = acc.load_word(sym, wi + 2);
        const uint32_t Eq0 = funnel_r(w0, w1, sh), Eq1 = funnel_r(w1, w2, sh);
        uint32_t T[2] = {Eq0 & VP0, Eq1 & VP1}, P[2] = {VP0, VP1}, Sm[2];
        AddChain<2>::run(Sm, T, P);
        const uint32_t D00 = ((Sm[0] ^ VP0) | Eq0) | VN0, D01 = ((Sm[1] ^ VP1) | Eq1) | VN1;
        const uint32_t HP0 = VN0 | ~(D00 | VP0), HP1 = VN1 | ~(D01 | VP1);
        const uint32_t HN0 = VP0 & D00, HN1 = VP1 & D01;
        const uint32_t X0 = funnel_r(D00, D01, 1), X1 = D01 >> 1;
        VN0 = X0 & HP0;
        VN1 = X1 & HP1;
        VP0 = HN0 | ~(X0 | HP0);
        VP1 = HN1 | ~(X1 | HP1);
        S += 1 - (int)(HN1 >> 31);
        if (TRACK && j >= lo) {
            const int kb = kb0 - j;  // 0..63
            const uint64_t M = kb >= 63 ? 0ull : (~0ull << (kb + 1));
            const int score = S - popcount32(VP0 & (uint32_t)M) - popcount32(VP1 & (uint32_t)(M >> 32)) +
                              popcount32(VN0 & (uint32_t)M) + popcount32(VN1 & (uint32_t)(M >> 32));
            if constexpr (std::is_base_of<HitSink, RecT>::value) {
                if (score <= best) rec->hit(score, ws + j);  // hits: best is the fixed threshold
            } else if (score <= best) {  // same bookkeeping as k1_event (ref cpp:658-673)
                constexpr int CAP = (int)(sizeof(rec->pos) / sizeof(rec->pos[0]));
                if (score < best) {
                    best = score;
                    cnt = 0;
                }
                if (cnt < CAP) {
                    rec->pos[cnt] = ws + j;
                } else if (prm.ovfCap > 0) {
                    const int at = atomic_add_int(prm.ovfCount, 1);
                    if (at < prm.ovfCap) {
                        prm.ovf[at].rec = slot;
                        prm.ovf[at].score = score;
                        prm.ovf[at].pos = ws + j;
                    }
                }
                rec->last = ws + j;
                cnt++;
            }
        }
    }
};

// Hopeless windows (most windows come from chance seed hits) are left early: from column dhi on every alignment
// with <= t edits that ends at a tracked column has begun and crosses each column inside the window, at a cost
// that is at least the banded value of the cell it crosses (the banded values are the cheapest in-band paths); so
// once every cell of a column is above t no tracked column can score <= t.  Checked once, `checkAfter` columns
// past dhi (by then the rows in the window are deep enough for an unrelated read to have left t behind).
template <class WAcc, class RecT>
EB_HD void k1b_sweep(const WAcc& acc, const uint8_t* tsyms, int ws, int m, int off, int c0, int lo, int hi, int t,
                     int checkAfter, int& bestIo, int& cntIo, RecT* rec, const K1WParams& prm, int slot) {
    const int dhi = hi - (m - 1) + t;
    K1Band<WAcc, RecT> b{acc, rec, 0, 0, 0, 0, 0, bestIo, cntIo, off + 64 - dhi, lo, m - 2 + dhi, ws, prm, slot};
    // state before column c0: D[r][c0-1] = r + 1 on the rows of the query, 0 above it
    const int firstReal = off + 64 - (c0 + b.g0);  // window bit of query row 0 (may be <= 0 or >= 64)
    const uint64_t vp64 = firstReal <= 0 ? ~0ull : (firstReal >= 64 ? 0ull : (~0ull << firstReal));
    b.VP0 = (uint32_t)vp64;
    b.VP1 = (uint32_t)(vp64 >> 32);
    const int bottomRow = c0 - dhi + 63;
    b.S = bottomRow >= 0 ? bottomRow + 1 : 0;
    int j = c0;
    for (; j <= hi && (j & 15); ++j) b.template column<true>(j, tsyms[j]);  // up to the next multiple of 16
    if (j + 15 <= hi) {
        Sym16 v = load_sym16(tsyms + j);
        // (t == 0: the one alignment of interest runs along the window's TOP diagonal, whose cell of the column just
        // swept is not part of the frame window_min() looks at -- the cell below it costs 1 > t, so the test would
        // discard an exact occurrence; with t >= 1 that neighbour is within t whenever the path still can be)
        bool checked = checkAfter < 0 || t == 0;
        for (; j + 15 < lo; j += 16) {  // lead-in groups: no column of them is tracked
            if (!checked && j >= dhi + checkAfter) {
                checked = true;
                if (b.window_min() > t) return;  // nothing recorded: the window holds no score <= t
            }
            const Sym16 cur = v;
            if (j + 31 <= hi) v = load_sym16(tsyms + j + 16);  // in flight while the 16 columns below are computed
            EB_UNROLL
            for (int q = 0; q < 16; ++q) b.template column<false>(j + q, (cur.w[q >> 2] >> (8 * (q & 3))) & 255u);
        }
        for (; j + 15 <= hi; j += 16) {
            const Sym16 cur = v;
            if (j + 31 <= hi) v = load_sym16(tsyms + j + 16);
            EB_UNROLL
            for (int q = 0; q < 16; ++q) b.template column<true>(j + q, (cur.w[q >> 2] >> (8 * (q & 3))) & 255u);
        }
    }
    for (; j <= hi; ++j) b.template column<true>(j, tsyms[j]);
    bestIo = b.best;
    cntIo = b.cnt;
}

// One K1W work item: the whole query over its own target window (each lane walks its own window; the target is
// L2-resident).  The profile rows have NW + 4 words: two words of ones (wildcard rows above the query, used by
// the banded sweep), the NW-word K1 profile, two words of zeros.  Windows whose end columns of interest span at
// most 64 diagonals take the banded sweep (k1b_sweep: 2 words per column instead of NW), the others the full one.
// The profile rows of a K1W work item (the layout above), shared by k1w_thread and k1w_hits_thread.
template <int NW, class WAcc>
EB_HD void k1w_profile(const K1WParams& p, int pair, int m, WAcc& acc) {
    for (int code = 0; code < p.ncodes; ++code) {
        acc.store_word(code, 0, ~0u);
        acc.store_word(code, 1, ~0u);
        acc.store_word(code, NW + 2, 0u);
        acc.store_word(code, NW + 3, 0u);
    }
    K1View<NW, WAcc> k1acc{acc};
    k1_build_peq<NW>(k1acc, p.qcodes + p.qoff[pair], m, MODE_HW, p.ncodes, p.eqtab);
}
template <int NW, class WAcc>
EB_HD void k1w_thread(const K1WParams& p, int slot, WAcc& acc) {
    const int pair = p.readList[slot];
    const int m = p.qlen[pair];
    WinRec* rec = p.recs + slot;
    k1w_profile<NW>(p, pair, m, acc);
    K1View<NW, WAcc> k1acc{acc};
    const int ws = p.winStart[slot], tf = p.trackFrom[slot], len = p.winLen[slot];
    const int kInit = p.kInit[slot];
    const int t = kInit - 1;
    const int hi = len - 1;
    if (t >= 0 && (hi - tf) + 2 * t + 1 <= 64) {
        // lead-in: exactly m + t columns before the first tracked one (the window may start a little earlier,
        // at a multiple of 16), or the start of the target
        const int c0 = tf - (m + t) > 0 ? tf - (m + t) : 0;
        int best = kInit, cnt = 0;
        k1b_sweep(acc, p.tcodes + ws, ws, m, 32 * NW - m, c0, tf, hi, t, p.checkAfter, best, cnt, rec, p, slot);
        rec->best = best;
        rec->cnt = cnt;
        return;
    }
    K1State<NW> st;
    k1_init<NW>(st, m, kInit);
    // Lead-in columns in blocks of 32.  The last-row score falls by at most one per column, so once it
    // exceeds the sentinel by more than the columns left in the window no tracked column can reach the
    // threshold any more and the sweep stops (most windows come from chance seed hits and end here).
    bool hopeless = false;
    for (int j = 0; j < tf; j += 32) {
        const int cntj = tf - j < 32 ? tf - j : 32;
        k1_columns<NW, false, false>(st, k1acc, PtrSyms{p.tcodes + ws + j}, cntj, ws + j, rec, slot, nullptr, nullptr, 0);
        if (st.up - st.down - (len - (j + cntj)) >= st.best) {
            hopeless = true;
            break;
        }
    }
    if (!hopeless)
        k1_columns<NW, false, true>(st, k1acc, PtrSyms{p.tcodes + ws + tf}, len - tf, ws + tf, rec, slot, p.ovf, p.ovfCount, p.ovfCap);
    rec->best = st.best;
    rec->cnt = st.cnt;
}

// Hits of one window job (eb_common.h: HitParams): the sweeps of k1w_thread with the window's threshold t = kInit - 1
// held fixed; every tracked column scoring <= t is a hit.  The tracked columns of a read's windows cover every end
// column of every alignment within t, and every such score is exact (seed_windows), so the hits of a read are those of
// its windows in window order.  The early exits stay valid: they only leave windows that hold no score <= t.
template <int NW, class WAcc, class Sink = HitSink>
EB_HD void k1w_hits_thread(const K1WParams& p, const HitParams& h, int slot, WAcc& acc) {
    Sink sink;
    if (!hit_sink_open(h, slot, sink)) return;
    const int pair = p.readList[slot];
    const int m = p.qlen[pair];
    k1w_profile<NW>(p, pair, m, acc);
    K1View<NW, WAcc> k1acc{acc};
    const int ws = p.winStart[slot], tf = p.trackFrom[slot], len = p.winLen[slot];
    const int t = p.kInit[slot] - 1;
    const int hi = len - 1;
    if (t >= 0 && (hi - tf) + 2 * t + 1 <= 64) {
        const int c0 = tf - (m + t) > 0 ? tf - (m + t) : 0;
        int best = t, cnt = 0;
        k1b_sweep(acc, p.tcodes + ws, ws, m, 32 * NW - m, c0, tf, hi, t, p.checkAfter, best, cnt, &sink, p, slot);
    } else {
        K1State<NW> st;
        k1_init<NW>(st, m, t);
        bool hopeless = false;
        for (int j = 0; j < tf; j += 32) {
            const int cntj = tf - j < 32 ? tf - j : 32;
            k1_columns<NW, false, false>(st, k1acc, PtrSyms{p.tcodes + ws + j}, cntj, ws + j, &sink, slot, nullptr, nullptr, 0);
            if (st.up - st.down - (len - (j + cntj)) > t) {
                hopeless = true;
                break;
            }
        }
        if (!hopeless)
            k1_columns<NW, false, true>(st, k1acc, PtrSyms{p.tcodes + ws + tf}, len - tf, ws + tf, &sink, slot, nullptr, nullptr, 0);
    }
    hit_sink_close(h, slot, sink);
}

// Hits of one (chunk, read) job of a whole-target HW sweep (K1Params chunk geometry, kInit = k): the chunk restarts
// halo >= 2m columns early, so every score of the columns it owns is exact, and it reports only those.
template <int NW, class Acc, class Sink = HitSink>
EB_HD void k1_hits_thread(const K1Params& p, const HitParams& h, int slot, int chunk, Acc& acc) {
    const int job = chunk * p.numReads + slot;
    Sink sink;
    if (!hit_sink_open(h, job, sink)) return;
    const int pair = p.readList[slot];
    const int m = p.qlen[pair];
    k1_build_peq<NW>(acc, p.qcodes + p.qoff[pair], m, MODE_HW, p.ncodes, p.eqtab);
    K1State<NW> st;
    k1_init<NW>(st, m, p.kInit[slot]);
    const K1Chunk g = k1_chunk(p, chunk);
    k1_columns<NW, false, false>(st, acc, PtrSyms{p.tcodes + g.hs}, g.cs - g.hs, g.hs, &sink, job, nullptr, nullptr, 0);
    k1_columns<NW, false, true>(st, acc, PtrSyms{p.tcodes + g.cs}, g.ce - g.cs, g.cs, &sink, job, nullptr, nullptr, 0);
    hit_sink_close(h, job, sink);
}

// Hits of one (pair, chunk) job of the per-pair route (eb_common.h: LaneHitParams): the sweep of k1_hits_thread over
// the pair's own target, threshold p.k.  hs lies at least 2m columns before cs (or at column 0), so every score of the
// owned columns is exact.
template <int NW, class Acc>
EB_HD void lane_hits_job(const LaneHitParams& p, const HitParams& h, int job, Acc& acc) {
    HitSink sink;
    if (!hit_sink_open(h, job, sink)) return;
    const LaneHitJob J = p.jobs[job];
    k1_build_peq<NW>(acc, p.qcodes + J.qOff, J.m, MODE_HW, p.ncodes, p.eqtab);
    K1State<NW> st;
    k1_init<NW>(st, J.m, p.k);
    const uint8_t* t = p.tcodes + J.tOff;
    k1_columns<NW, false, false>(st, acc, PtrSyms{t}, J.cs - J.hs, J.hs, &sink, job, nullptr, nullptr, 0);
    k1_columns<NW, false, true>(st, acc, PtrSyms{t + (J.cs - J.hs)}, J.ce - J.cs, J.cs, &sink, job, nullptr, nullptr, 0);
    hit_sink_close(h, job, sink);
}

// Job j of read `slot` of a hits launch (eb_common.h: HitPlaceParams), j = 0 .. hit_jobs(p, slot) - 1, in column order.
EB_HD int hit_jobs(const HitPlaceParams& p, int slot) {
    if (!p.plan) return p.chunks;
    return p.plan[slot].state == SEED_WINDOWS ? p.plan[slot].count : 0;
}
EB_HD int hit_job(const HitPlaceParams& p, int slot, int j) { return p.plan ? p.plan[slot].first + j : slot + j * p.numReads; }
// After the count pass: the hits of the read.
EB_HD void hits_total_item(const HitPlaceParams& p, int slot) {
    long long total = 0;
    for (int j = 0, n = hit_jobs(p, slot); j < n; ++j) total += p.count[hit_job(p, slot, j)];
    p.pairCount[p.readList[slot]] = total;
}
// Before the fill pass: where each job of the read stores its hits, and how many of them (the read's first
// pairStored hits in column order).
EB_HD void hits_place_item(const HitPlaceParams& p, int slot) {
    const int pair = p.readList[slot];
    const long long base = p.pairBase[pair], stored = p.pairStored[pair];
    long long done = 0;
    for (int j = 0, n = hit_jobs(p, slot); j < n; ++j) {
        const int job = hit_job(p, slot, j);
        const int c = p.count[job];
        const long long left = stored - done;
        p.at[job] = base + done;
        p.room[job] = left <= 0 ? 0 : (left < c ? (int)left : c);
        done += c;
    }
}

// =============================================================================================
// Seed stage of the candidate filter (HW, plain symbol equality).  If a read aligns somewhere with
// d <= t edits, then of any t+1 disjoint pieces of the read at least one is untouched by the edits
// and occurs verbatim in the target: piece read[a, a+Ls) == target[p, p+Ls) puts the end column of that
// alignment within d of E = p + (m - a) - 1.  So the columns [E-t, E+t] of all exact piece occurrences
// cover every end column with a distance <= t; the whole read is swept over windows around them
// (k1w_thread) and the minimum is final when it is <= t.
// =============================================================================================

// Radix key of the Lidx codes at s (eb_common.h: SeedIndexParams); only `avail` codes exist, the rest count as 0.
// SEP (a record target): a code >= sigma is a separator and counts as 0 too, so that a seed that ends right before a
// separator is still found by the range lookup of its shorter key.
template <bool SEP = false>
EB_HD uint32_t seed_key(const uint8_t* s, int avail, int Lidx, uint32_t sigma) {
    uint32_t key = 0;
    for (int x = 0; x < Lidx; ++x) {
        const uint32_t c = x < avail ? (uint32_t)s[x] : 0u;
        key = key * sigma + ((SEP && c >= sigma) ? 0u : c);
    }
    return key;
}
template <bool SEP = false>
EB_HD void seed_count_item(const SeedIndexParams& p, int i) {
    atomic_add_int(p.bucketStart + seed_key<SEP>(p.tcodes + i, p.n - i, p.Lidx, (uint32_t)p.sigma), 1);
}
template <bool SEP = false>
EB_HD void seed_fill_item(const SeedIndexParams& p, int i) {
    const uint32_t b = seed_key<SEP>(p.tcodes + i, p.n - i, p.Lidx, (uint32_t)p.sigma);
    p.positions[p.bucketStart[b] + atomic_add_int(p.cursor + b, 1)] = i;
}

// Windows of one read from its sorted candidate end columns E[0..c): f(w, ws, lo, hi) for each window w in order;
// returns their number.  Windows start at multiples of 16 columns (a longer lead-in is still exact).  Candidates are
// verified together as long as the window stays narrow enough for the banded sweep (k1b_sweep: tracked columns +
// 2t + 1 <= 64 diagonals); when t is too large for any banded window, as long as they are neighbours (gap / spread rule).
template <class F>
EB_HD int seed_windows(const SeedPlanParams& p, const int* E, int c, int m, int t, F&& f) {
    const int bandSlack = 63 - 4 * t;  // E[last] - E[first] may be this large in a banded window
    int prevHi = -1;
    int nW = 0;
    for (int i = 0; i < c;) {
        const int first = E[i];
        int last = first;
        ++i;
        if (bandSlack >= 0) {
            while (i < c && E[i] - first <= bandSlack) last = E[i++];
        } else {
            while (i < c && E[i] - last <= K1_RANGE_GAP && E[i] - first <= p.spread) last = E[i++];
        }
        int lo = first - t, hi = last + t;
        if (lo <= prevHi) lo = prevHi + 1;  // tracked columns of successive windows stay disjoint
        if (lo < 0) lo = 0;
        if (hi > p.n - 1) hi = p.n - 1;
        if (lo > hi) continue;
        prevHi = hi;
        // HW restart: an alignment with <= t edits spans at most m + t target columns, so every score <= t
        // of a tracked column is exact (larger ones may come out larger still, which changes nothing)
        int ws = lo - (m + t);
        if (ws < 0) ws = 0;
        ws &= ~15;
        f(nW, ws, lo, hi);
        ++nW;
    }
    return nW;
}
EB_HD void seed_window_store(const SeedPlanParams& p, int w, int pair, int t, int ws, int lo, int hi) {
    p.winPair[w] = pair;
    p.winK[w] = t + 1;
    p.winStart[w] = ws;
    p.winLen[w] = hi - ws + 1;
    p.winTf[w] = lo - ws;
}

// Host spelling of the cooperative group that plans one read (one member); the device kernel passes groups of 16
// or 32 lanes (eb_kernels.cu: CoopGroup).
//   scan(v, total): exclusive prefix sum of v over the members, total = the sum over all of them;
//   reserve(counter, n): every member of the group passes its read's n (all groups of a warp call it together on the
//   device, which adds the warp's total to *counter once); returns the old value plus what the reads before it took.
struct CoopSerial {
    static constexpr int W = 1;
    static EB_HD int lane() { return 0; }
    static EB_HD int width() { return 1; }
    static EB_HD void sync() {}
    static EB_HD bool any(bool v) { return v; }
    static EB_HD int add_shared(int* p, int v) {
        const int old = *p;
        *p = old + v;
        return old;
    }
    static EB_HD int scan(int v, int& total) {
        total = v;
        return 0;
    }
    static EB_HD int reserve(int* counter, int n) { return n > 0 ? atomic_add_int(counter, n) : 0; }
};

// Scratch of one planning group of W members: E[CAP] candidate end columns, then seed_ctl_words(W) ints of control
// words: ctl[0] candidates, ctl[1] saturated, then per member of the current round of seeds the first index entry
// of its seed's range, the range's offset in the round's entries, and the seed's offset a in the read.
EB_HD constexpr int seed_ctl_words(int W) { return 2 + 3 * W; }
// enough control words for a group of any width (at most a warp); the device kernel reserves seed_ctl_words(W)
constexpr int SEED_CTL = seed_ctl_words(32);

// Candidates of one occurrence-list entry per slot k (pos < 0: none): the whole seed read[a, a+Ls) is compared with
// the target (the key covered only its first Lk symbols) and the expected end column of each match recorded.
// The loads of all slots are issued before any is used, so their latencies overlap.
template <int CAP, int K, class C>
EB_HD void seed_try(const SeedPlanParams& p, const uint8_t* q, int m, int Lk, const int (&pos)[K], const int (&a)[K],
                    int* E, int* ctl) {
    bool same[K];
    EB_UNROLL
    for (int k = 0; k < K; ++k) {
        same[k] = pos[k] >= 0 && pos[k] + p.Ls <= p.n;  // keys near the end of the target were padded with code 0
        if (same[k]) {
            uint32_t diff = 0;
            for (int x = Lk; x < p.Ls; ++x) diff |= (uint32_t)(p.tcodes[pos[k] + x] ^ q[a[k] + x]);
            same[k] = diff == 0;
        }
    }
    EB_UNROLL
    for (int k = 0; k < K; ++k) {
        if (!same[k]) continue;
        const int at = C::add_shared(&ctl[0], 1);
        if (at < CAP) E[at] = pos[k] + (m - a[k]) - 1;
    }
}

// One read, planned by a cooperative group C (a single member on the host, 16 or 32 lanes on the device).  Each
// member takes one seed of the read, so that with as many members as seeds the key -> index range lookups of all
// of them are in flight together.  The index entries of the round's ranges are then dealt out over the members as
// one list (a member's entries loaded together: entry -> position -> target symbols), so a read with a long range
// costs little more than one without.  The candidates meet in E and are sorted by a bitonic network over the
// group; every member walks the sorted list to the same windows (seed_windows), keeps the one numbered like it and
// writes it, and the group's reads of a warp take their room in the job arrays with one atomic (C::reserve).
// Every member of every group of a warp must reach C::reserve: slots past numReads pass through with nothing.
template <int CAP, class C>
EB_HD void seed_plan_read(const SeedPlanParams& p, int slot, int* E, int* ctl) {
    const int lane = C::lane();
    constexpr int W = C::W;
    int* rStart = ctl + 2;      // [W]
    int* rPre = rStart + W;     // [W]
    int* rA = rPre + W;         // [W]
    const bool live = slot < p.numReads;
    const int pair = !live ? 0 : (p.readList ? p.readList[slot] : p.firstPair + slot);
    const int m = live ? p.qlen[pair] : 0;
    const int t = !live ? -1 : (p.thr ? p.thr[slot] : seed_threshold(m, p.kBound, p.Ls, p.seedK, -1));
    const uint8_t* q = live ? p.qcodes + p.qoff[pair] : nullptr;
    SeedPlan pl;
    pl.first = pl.count = 0;
    pl.state = SEED_SATURATED;  // left out of the stage (the host, or the threshold rule) unless planned below
    pl.thr = -1;
    int c = 0;
    if (t >= 0) {
        pl.state = SEED_NONE;
        pl.thr = t;
        if (lane == 0) {
            ctl[0] = 0;
            ctl[1] = 0;
        }
        C::sync();
        const int stride = m / (t + 1);  // >= Ls: the t+1 pieces are disjoint
        const int Lk = p.Ls < p.Lidx ? p.Ls : p.Lidx;  // symbols of the seed that go into the key
        uint32_t span = 1;                             // keys sharing that prefix
        for (int x = Lk; x < p.Lidx; ++x) span *= (uint32_t)p.sigma;
        for (int j0 = 0; j0 <= t; j0 += W) {  // one round when the group has t+1 members or more
            const int j = j0 + lane;
            const int a = j * stride;
            int i0 = 0, len = 0;
            if (j <= t) {
                // a code outside the target's alphabet (streamed batches give the reads' foreign bytes one) occurs nowhere
                uint32_t key = 0;
                bool known = true;
                for (int x = 0; x < p.Ls; ++x) {
                    const uint32_t code = q[a + x];
                    known = known && code < (uint32_t)p.sigma;
                    if (x < Lk) key = key * (uint32_t)p.sigma + code;
                }
                if (known) {
                    key *= span;
                    i0 = p.bucketStart[key];
                    len = p.bucketStart[key + span] - i0;
                    if (len > p.maxBucket) {  // repeat: the read is passed on unseen
                        ctl[1] = 1;
                        len = 0;
                    }
                }
            }
            int total;
            const int pre = C::scan(len, total);
            rStart[lane] = i0;
            rPre[lane] = pre;
            rA[lane] = a;
            C::sync();
            constexpr int K = 4;  // entries per member in flight together
            for (int e0 = 0; e0 < total; e0 += K * W) {
                int pos[K], aa[K];
                EB_UNROLL
                for (int k = 0; k < K; ++k) {
                    const int e = e0 + k * W + lane;
                    pos[k] = -1;
                    aa[k] = 0;
                    if (e < total) {
                        int s = 0;  // the seed whose range holds entry e: the last one starting at or before it
                        for (int h = W / 2; h > 0; h /= 2)
                            if (rPre[s + h] <= e) s += h;
                        aa[k] = rA[s];
                        pos[k] = p.positions[rStart[s] + (e - rPre[s])];
                    }
                }
                seed_try<CAP, K, C>(p, q, m, Lk, pos, aa, E, ctl);
            }
            C::sync();  // the round's ranges are walked before the next round overwrites them
        }
        c = ctl[0];
        if (ctl[1] || c > CAP) {
            pl.state = SEED_SATURATED;
            c = 0;
        } else if (c > 1) {
            // bitonic network over the candidates padded to a power of two (<= CAP), compare-exchanges dealt to the members
            int P2 = 2;
            while (P2 < c) P2 *= 2;
            for (int i = c + lane; i < P2; i += W) E[i] = 0x7fffffff;
            C::sync();
            for (int k = 2; k <= P2; k *= 2) {
                for (int jj = k / 2; jj > 0; jj /= 2) {
                    for (int x = lane; x < P2 / 2; x += W) {
                        const int lo = 2 * x - (x & (jj - 1));  // index with bit jj clear
                        const int hi = lo + jj;
                        const bool up = (lo & k) == 0;
                        const int u = E[lo], v = E[hi];
                        if ((u > v) == up) {
                            E[lo] = v;
                            E[hi] = u;
                        }
                    }
                    C::sync();
                }
            }
        }
    }
    // every member walks the sorted candidates to the same windows and keeps the one numbered like it
    int myWs = 0, myLo = 0, myHi = 0;
    const int nW = seed_windows(p, E, c, m, t, [&](int w, int ws, int lo, int hi) {
        if (w == lane) {
            myWs = ws;
            myLo = lo;
            myHi = hi;
        }
    });
    const int base = C::reserve(p.winCount, nW);
    if (nW > 0) {
        if (base + nW <= p.winCap) {
            if (lane < nW) seed_window_store(p, base + lane, pair, t, myWs, myLo, myHi);
            if (nW > W)  // more windows than members (many candidates): the rest in a second walk
                seed_windows(p, E, c, m, t, [&](int w, int ws, int lo, int hi) {
                    if (w >= W && w % W == lane) seed_window_store(p, base + w, pair, t, ws, lo, hi);
                });
            pl.first = base;
            pl.count = nW;
            pl.state = SEED_WINDOWS;
        } else {
            pl.state = SEED_SATURATED;  // the job arrays are full (host-driven stages repeat with the exact size)
        }
    }
    if (live && lane == 0) p.plan[slot] = pl;
}

EB_HD void win_reduce_read(const WinReduceParams& p, int slot) {
    const SeedPlan pl = p.plan[slot];
    Rec out;
    out.best = 0x7fffffff;
    out.cnt = 0;
    out.last = 0;
    out.rsv = pl.state;
    for (int q = 0; q < KPOS; ++q) out.pos[q] = 0;
    if (pl.state == SEED_WINDOWS) {
        const int t = pl.thr;
        int b = 0x7fffffff;
        for (int w = 0; w < pl.count; ++w) {
            const WinRec& r = p.winRecs[pl.first + w];
            if (r.cnt > 0 && r.best < b) b = r.best;
        }
        if (b > t) {
            out.rsv = SEED_NONE;  // every window minimum is above the threshold
        } else {
            int total = 0;
            bool longList = false, listed = false;
            for (int w = 0; w < pl.count; ++w) {
                const WinRec& r = p.winRecs[pl.first + w];
                if (r.cnt <= 0 || r.best != b) continue;
                if (r.cnt > KPOSW) listed = true;  // the columns beyond the inline ones are in the overflow list
                total += r.cnt;
            }
            int listLen = 0;
            if (listed) {
                listLen = p.ovfCap > 0 ? *p.ovfCount : 0x7fffffff;
                if (listLen > p.ovfCap) longList = true;  // no list, or it ran over: the plain sweep collects the columns
            }
            int base = 0;
            if (!longList && total > KPOS) {
                base = atomic_add_int(p.extraCount, total - KPOS);
                if (base + total - KPOS > p.extraCap) longList = true;
            }
            if (longList) {
                out.rsv = SEED_LONG_LIST;
            } else {
                int i = 0;
                for (int w = 0; w < pl.count; ++w) {
                    const WinRec& r = p.winRecs[pl.first + w];
                    if (r.cnt <= 0 || r.best != b) continue;
                    for (int q = 0; q < r.cnt && q < KPOSW; ++q, ++i) {
                        if (i < KPOS) out.pos[i] = r.pos[q];
                        else p.extra[base + i - KPOS] = r.pos[q];
                    }
                    if (r.cnt > KPOSW) {  // rare: the window's entries of the list, which is in sweep order per window
                        int found = 0;
                        for (int e = 0; e < listLen; ++e) {
                            const Ovf o = p.ovf[e];
                            if (o.rec != pl.first + w || o.score != b) continue;
                            if (found < r.cnt - KPOSW) p.extra[base + i++ - KPOS] = o.pos;  // (i >= KPOSW > KPOS here)
                            ++found;
                        }
                        if (found != r.cnt - KPOSW) longList = true;  // cannot happen; the plain sweep would settle it
                    }
                }
                if (longList) {
                    out.rsv = SEED_LONG_LIST;
                } else {
                    out.best = b;
                    out.cnt = total;
                    out.last = base;
                }
            }
        }
    }
    if (p.leftover) {  // device-driven first level: the outcome logic of Pass::window_outcomes, per read
        const int pair = p.readList ? p.readList[slot] : p.firstPair + slot;
        const int m = p.qlen[pair];
        const int bound = (p.kBound < 0 || p.kBound > m) ? m : p.kBound;
        int excl = -3;  // -3: decided
        if (out.rsv == SEED_WINDOWS) {
            out.rsv = REC_DONE;
        } else if (out.rsv == SEED_NONE && pl.thr >= 0 && pl.thr == bound) {
            out.rsv = REC_DONE;  // nothing within the caller's bound: final (best stays at the sentinel)
        } else {
            excl = out.rsv == SEED_LONG_LIST ? -2 : (out.rsv == SEED_NONE ? pl.thr : -1);
            out.rsv = REC_PENDING;
        }
        if (excl != -3 && p.strands) {
            out.last = excl;  // fin_count_item applies the cross-strand rule and appends what goes on
        } else if (excl != -3) {
            const int at = atomic_add_int(p.leftoverCount, 1);
            p.leftover[at].pair = pair;
            p.leftover[at].excl = excl;
            p.leftover[at].bound = bound;
        }
    }
    p.out[slot] = out;
}

// Strand batches, device-driven first level: the cross-strand rule (eb_common.h: strand_rule) on the two records of the
// read that holds `slot` (slots 2j and 2j+1 of a slice are its forward and reverse strand; win_reduce recorded a pending
// strand's excl in its record's `last`).  Both calls of a read see the same two records and reach the same decision;
// each acts on its own slot.  Returns whether the slot's strand has lost; `bound` receives its bound if it goes on.
EB_HD bool strand_lost(const FinParams& p, int slot, int& bound) {
    const int first = slot & ~1;
    bool done[2];
    int d[2], excl[2], bd[2];
    for (int s = 0; s < 2; ++s) {
        const Rec& r = p.recs[first + s];
        const int pair = p.readList ? p.readList[first + s] : p.firstPair + first + s;
        const int m = p.qlen[pair];
        bd[s] = (p.kBound < 0 || p.kBound > m) ? m : p.kBound;
        done[s] = r.rsv != REC_PENDING;
        d[s] = done[s] ? r.best : 0x7fffffff;
        excl[s] = done[s] ? -1 : (r.last < -1 ? -1 : r.last);  // (-2: long end-location list, nothing known)
    }
    int loser = strand_rule(done, d, excl, bd);
    if (done[0] && done[1] && d[1] != 0x7fffffff) loser = d[1] < d[0] ? 0 : 1;  // both final: keep the winner's ends only
    bound = bd[slot & 1];
    return loser == (slot & 1);
}

// Complement of one byte of a read (a fixed involution): A<->T, C<->G and the IUPAC codes R<->Y, K<->M, B<->V, D<->H, in
// upper and lower case; every other byte (N, S, W, non-letters) is its own complement.
EB_HD uint8_t complement_byte(uint8_t b) {
    const uint8_t c = b | 0x20;  // lower case of a letter; b | 0x20 == c only for b == c and b == c - 0x20
    uint8_t o;
    switch (c) {
        case 'a': o = 't'; break;
        case 't': o = 'a'; break;
        case 'c': o = 'g'; break;
        case 'g': o = 'c'; break;
        case 'r': o = 'y'; break;
        case 'y': o = 'r'; break;
        case 'k': o = 'm'; break;
        case 'm': o = 'k'; break;
        case 'b': o = 'v'; break;
        case 'v': o = 'b'; break;
        case 'd': o = 'h'; break;
        case 'h': o = 'd'; break;
        default: return b;
    }
    return (uint8_t)(o ^ (c ^ b));  // the case of b
}

// Number of end locations a finished sweep outcome yields (the -1 rule of ref cpp:670, 681-693: the padded
// bottom cell of column W-1 shows up as end location -1 when editDistance == m), or -1 when there is no result.
EB_HD int hw_accepted_count(int best, int cnt, int m, int kBound, bool* minusOne) {
    *minusOne = false;
    if (best < 0 || best == 0x7fffffff || cnt <= 0) return -1;
    if (kBound >= 0 && best > kBound) return -1;
    if (best > m) return -1;
    const int W64 = (m + 63) / 64 * 64 - m;
    *minusOne = (best == m && W64 > 0);
    return cnt + (*minusOne ? 1 : 0);
}
EB_HD void fin_count_item(const FinParams& p, int slot) {
    Rec r = p.recs[slot];
    const int pair = p.readList ? p.readList[slot] : p.firstPair + slot;
    int count = 0, ed = -1;
    if (p.strands) {
        int bound;
        if (strand_lost(p, slot, bound)) {  // no alignment (fin_fill copies nothing of it)
            r.best = 0x7fffffff;
            r.cnt = 0;
            r.rsv = REC_DONE;
        } else if (r.rsv == REC_PENDING) {
            const int at = atomic_add_int(p.leftoverCount, 1);
            p.leftover[at].pair = pair;
            p.leftover[at].excl = r.last;
            p.leftover[at].bound = bound;
        }
    }
    if (r.rsv == REC_PENDING) {
        ed = -2;
        atomic_add_int(p.header + 1, 1);
    } else {
        bool minusOne;
        const int a = hw_accepted_count(r.best, r.cnt, p.qlen[pair], p.kBound, &minusOne);
        if (a >= 0) {
            ed = r.best;
            count = a;
        }
    }
    p.ed[pair] = ed;
    p.endCount[pair] = count;
    p.cnt32[slot] = count;
}
EB_HD void fin_fill_item(const FinParams& p, int slot) {
    const int pair = p.readList ? p.readList[slot] : p.firstPair + slot;
    const int start = p.cnt32[slot];
    const int count = p.cnt32[slot + 1] - start;
    p.endStart[pair] = p.poolBase + start;
    if (slot == 0) {
        p.header[0] = p.cnt32[p.numReads];
        p.header[3] = p.winCount ? *p.winCount : 0;
    }
    if (count <= 0) return;
    if (start + count > p.poolCap) {
        p.header[2] = 1;
        return;
    }
    const Rec r = p.recs[slot];
    int at = start;
    if (count > r.cnt) p.pool[at++] = -1;
    for (int q = 0; q < r.cnt; ++q) p.pool[at++] = q < KPOS ? r.pos[q] : p.extra[r.last + q - KPOS];
}

// =============================================================================================
// L -- one alignment per thread with its OWN target (per-pair targets, start-location sweeps,
// matrix-storing sweeps of short queries).  Same per-thread sweep as K1; symbols come straight from
// global memory, forward or reversed.  One launch = one (word class, mode, direction, store) class.
// =============================================================================================
template <int NW, int MODE, bool REV, bool STORE, class Acc>
EB_HD void lane_job(const LParams& p, int jobIdx, Acc& acc) {
    const LJob J = p.jobs[jobIdx];
    Rec* rec = p.recs + jobIdx;
    if (J.m <= 0) {  // placeholder job of a device-built list (eb_common.h: ResParams)
        rec->best = 0x7fffffff;
        rec->cnt = 0;
        return;
    }
    k1_build_peq<NW>(acc, p.qcodes + J.qOff, J.m, MODE, p.ncodes, p.eqtab, REV);
    K1State<NW> st;
    k1_init<NW>(st, J.m, J.kInit);
    const uint8_t* t = p.tcodes + J.tOff;
    if (STORE) {
        U2* mat = p.mat + J.matOff;
        const size_t step = p.matStep > 1 ? (size_t)p.matStep : 1;
        for (int c = 0; c < J.n; ++c) {
            uint32_t Eq[NW], Ph[NW];
            acc.load(t[c], Eq);
            k1_step<NW, true>(st.Pv, st.Mv, Eq, st.up, st.down, Ph);
            EB_UNROLL
            for (int w = 0; w < NW; ++w) {
                U2 e;
                e.x = st.Pv[w];
                e.y = Ph[w];
                mat[((size_t)c * NW + w) * step] = e;
            }
        }
    } else if (REV) {
        if (MODE == MODE_HW) {
            k1_columns<NW, false, false>(st, acc, RevSyms{t}, J.trackFrom, 0, rec, jobIdx, nullptr, nullptr, 0);
            k1_columns<NW, false, true>(st, acc, RevSyms{t - J.trackFrom}, J.n - J.trackFrom, J.trackFrom, rec, jobIdx, nullptr, nullptr, 0);
        } else {
            k1_columns<NW, true, MODE == MODE_SHW>(st, acc, RevSyms{t}, J.n, 0, rec, jobIdx, nullptr, nullptr, 0);
        }
    } else {
        if (MODE == MODE_HW) {
            k1_columns<NW, false, false>(st, acc, PtrSyms{t}, J.trackFrom, 0, rec, jobIdx, nullptr, nullptr, 0);
            k1_columns<NW, false, true>(st, acc, PtrSyms{t + J.trackFrom}, J.n - J.trackFrom, J.trackFrom, rec, jobIdx, nullptr, nullptr, 0);
        } else {
            k1_columns<NW, true, MODE == MODE_SHW>(st, acc, PtrSyms{t}, J.n, 0, rec, jobIdx, nullptr, nullptr, 0);
        }
    }
    if (MODE == MODE_NW) {  // the bottom-right cell (ref cpp:916)
        st.best = st.up - st.down;
        st.cnt = 1;
        rec->last = J.n - 1;
        rec->pos[0] = J.n - 1;
    }
    rec->best = st.best;
    rec->cnt = st.cnt;
}

// =============================================================================================
// Start locations / paths of short queries driven from the device (eb_common.h: ResParams): per-item functions of
// the stages around the lane and traceback kernels.
// =============================================================================================
EB_HD bool res_in_class(const ResParams& p, int pair) {
    const int m = p.qlen[pair];
    return p.ed[pair] >= 0 && m > 0 && (m + 31) / 32 == p.nw;
}
EB_HD uint64_t res_target_off(const ResParams& p, int pair) { return p.tOffPair ? p.tOffPair[pair] : p.tOff0; }

// largest i in [0, n) with a[i] <= v (a ascending, a[0] <= v)
EB_HD int res_owner(const int* a, int n, int v) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a[mid] <= v) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

EB_HD void res_item(const ResParams& p, int i) {
    switch (p.stage) {
        case RS_LOC_COUNT: {
            p.cnt[i] = res_in_class(p, i) ? p.endCount[i] : 0;
            break;
        }
        case RS_LOC_JOBS: {  // job i = end location (i - cnt[pair]) of its pair (ref cpp:230-262)
            const int pair = res_owner(p.cnt, p.numPairs, i);
            const long long slot = p.endStart[pair] + (i - p.cnt[pair]);
            const int e = p.endPool[slot], m = p.qlen[pair], d = p.ed[pair];
            LJob J;
            J.qOff = p.qoff[pair];
            J.tOff = res_target_off(p, pair) + (uint64_t)(e < 0 ? 0 : e);  // first symbol read, walking backwards
            J.matOff = 0;
            J.m = e < 0 ? 0 : m;  // end location -1 (ref cpp:237-249): start 0, no sweep (m == 0 jobs are skipped)
            const long long span = (long long)m + d;
            J.n = (int)((long long)e + 1 < span ? (long long)e + 1 : span);
            J.kInit = d + 1;
            J.trackFrom = 0;
            p.jobs[i] = J;
            p.jobPair[i] = pair;
            p.jobSlot[i] = slot;
            break;
        }
        case RS_LOC_APPLY: {
            const int pair = p.jobPair[i];
            const long long slot = p.jobSlot[i];
            const int e = p.endPool[slot];
            if (e < 0) {
                p.startPool[slot] = 0;
            } else {
                const Rec r = p.recs[i];
                if (r.cnt <= 0 || r.best != p.ed[pair]) *p.err = 1;
                p.startPool[slot] = e - r.last;  // ref cpp:260
            }
            break;
        }
        case RS_PATH_FLAG: {  // pairs whose target slice is longer than the launch provides for stay with the host tree
            const int pair = p.firstPair + i;
            int take = 0;
            if (pair < p.lastPair && res_in_class(p, pair)) {
                const long long slot = p.endStart[pair];
                take = (p.endPool[slot] - p.startPool[slot] + 1 <= p.maxPathN) ? 1 : 0;
            }
            p.cnt[i] = take;
            break;
        }
        case RS_PATH_JOBS: {  // item = pair offset inside the slice
            const int pair = p.firstPair + i;
            if (p.cnt[i + 1] == p.cnt[i]) break;
            const int j = p.cnt[i];
            const long long slot = p.endStart[pair];
            const int s0 = p.startPool[slot], e0 = p.endPool[slot];
            LJob J;
            J.qOff = p.qoff[pair];
            J.tOff = res_target_off(p, pair) + (uint64_t)s0;
            J.matOff = (uint64_t)(j / 32) * 32u * p.matStride + (uint64_t)(j % 32);  // interleaved by 32 jobs (LParams::matStep)
            J.m = p.qlen[pair];
            J.n = e0 - s0 + 1;  // <= 0: empty target slice, the script is m inserts (ref cpp:1168-1175)
            if (J.n < 0) J.n = 0;
            J.kInit = 0;
            J.trackFrom = 0;
            if ((uint64_t)J.n * (uint64_t)p.nw > p.matStride) {  // cannot happen: the stride covers m + ed columns
                *p.err = 1;
                J.n = 0;
            }
            p.jobs[j] = J;
            TbJob T;
            T.matOff = J.matOff;
            T.qOff = J.qOff;
            T.peqOff = ~0ull;
            T.tOff = J.tOff;
            T.outOff = (uint64_t)j * p.opsStride;
            T.m = J.m;
            T.n = J.n;
            T.nWp = p.nw;
            T.rsv = 0;
            p.tb[j] = T;
            p.jobPair[j] = pair;
            break;
        }
        case RS_PATH_LEN: {
            const LJob J = p.jobs[i];
            if (J.n > 0 && p.recs[i].best != p.ed[p.jobPair[i]]) *p.err = 1;
            p.cnt[i] = J.n > 0 ? p.opsLen[i] : J.m;
            break;
        }
        case RS_PATH_COPY: {
            const LJob J = p.jobs[i];
            const int pair = p.jobPair[i];
            const int len = p.cnt[i + 1] - p.cnt[i];
            uint8_t* dst = p.alnPool + p.cnt[i];
            if (J.n > 0) {
                const uint8_t* src = p.ops + (uint64_t)i * p.opsStride + (uint64_t)p.opsStart[i];
                for (int x = 0; x < len; ++x) dst[x] = src[x];
            } else {
                for (int x = 0; x < len; ++x) dst[x] = 1;  // EDLIB_EDOP_INSERT
            }
            p.alnStart[pair] = p.alnBase + p.cnt[i];
            p.alnLen[pair] = len;
            break;
        }
        default: break;
    }
}

// Start locations / edit scripts of stored hits (eb_common.h: HitResParams).  The rules are those of a single hit
// of edlibAlign (ref cpp:228-289) applied to each hit (column c, score s) on its own: the start is c minus the last
// column of best score s of the reversed SHW sweep over the last m + s columns, the script that of the NW alignment of
// the query to [start, c].
EB_HD int hit_res_pair(const HitResParams& p, long long slot) {  // last pair whose first slot is <= slot
    int lo = 0, hi = p.numPairs - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (p.pairBase[mid] <= slot) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Record of target column c of a record target (eb_common.h: RecordParams): the last r with recOff[r] <= c.
EB_HD int record_of(const int* recOff, int numRecords, int c) {
    int lo = 0, hi = numRecords - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (recOff[mid] <= c) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

EB_HD void hit_res_item(const HitResParams& p, int i) {
    switch (p.stage) {
        case HR_FLAG: {
            const int m = p.qlen[hit_res_pair(p, p.firstHit + i)];
            p.cnt[i] = (m + 31) / 32 == p.nw ? 1 : 0;
            break;
        }
        case HR_LOC_JOBS: {
            if (p.cnt[i + 1] == p.cnt[i]) break;
            const int j = p.cnt[i];
            const long long slot = p.firstHit + i;
            const int pair = hit_res_pair(p, slot);
            const int c = p.cols[slot], s = p.scores[slot], m = p.qlen[pair];
            LJob J;
            J.qOff = p.qoff[pair];
            J.tOff = (p.tOffPair ? p.tOffPair[pair] : p.tOff) + (uint64_t)c;  // first symbol read, walking backwards
            J.matOff = 0;
            J.m = m;
            const long long span = (long long)m + s;  // a start further back costs more than s
            const int first = p.recOff ? p.recOff[record_of(p.recOff, p.numRecords, c)] : 0;  // nor before the record
            J.n = (int)((long long)c - first + 1 < span ? (long long)c - first + 1 : span);
            J.kInit = s + 1;
            J.trackFrom = 0;
            p.jobs[j] = J;
            p.jobHit[j] = i;
            break;
        }
        case HR_LOC_APPLY: {
            const int h = p.jobHit[i];
            const long long slot = p.firstHit + h;
            const Rec r = p.recs[i];
            if (r.cnt <= 0 || r.best != p.scores[slot]) *p.err = 1;
            p.starts[h] = p.cols[slot] - r.last;  // ref cpp:260
            break;
        }
        case HR_PATH_JOBS: {
            if (p.cnt[i + 1] == p.cnt[i]) break;
            const int j = p.cnt[i];
            const long long slot = p.firstHit + i;
            const int pair = hit_res_pair(p, slot);
            const int st = p.starts[i];
            LJob J;
            J.qOff = p.qoff[pair];
            J.tOff = (p.tOffPair ? p.tOffPair[pair] : p.tOff) + (uint64_t)st;
            J.matOff = (uint64_t)(j / 32) * 32u * p.matStride + (uint64_t)(j % 32);  // interleaved by 32 jobs (LParams::matStep)
            J.m = p.qlen[pair];
            J.n = p.cols[slot] - st + 1;
            J.kInit = 0;
            J.trackFrom = 0;
            if (J.n < 1 || (uint64_t)J.n * (uint64_t)p.nw > p.matStride || (uint64_t)(J.m + J.n) > p.opsStride) {
                *p.err = 1;  // cannot happen: 1 <= c - start + 1 <= m + s, which the strides cover
                J.m = 0;
                J.n = 0;
            }
            p.jobs[j] = J;
            TbJob T;
            T.matOff = J.matOff;
            T.qOff = J.qOff;
            T.peqOff = ~0ull;
            T.tOff = J.tOff;
            T.outOff = (uint64_t)j * p.opsStride;
            T.m = J.m;
            T.n = J.n;
            T.nWp = p.nw;
            T.rsv = 0;
            p.tb[j] = T;
            p.jobHit[j] = i;
            break;
        }
        case HR_PATH_LEN: {
            const int h = p.jobHit[i];
            if (p.jobs[i].n <= 0 || p.recs[i].best != p.scores[p.firstHit + h]) *p.err = 1;
            p.len[h] = p.opsLen[i];
            break;
        }
        case HR_PATH_COPY: {
            const int h = p.jobHit[i];
            const int len = p.len[h + 1] - p.len[h];
            const uint8_t* src = p.ops + (uint64_t)i * p.opsStride + (uint64_t)p.opsStart[i];
            uint8_t* dst = p.pool + p.len[h];
            for (int x = 0; x < len; ++x) dst[x] = src[x];
            break;
        }
        default: break;
    }
}

// One item of record_kernel (eb_common.h: RecordParams).
EB_HD void record_item(const RecordParams& p, int i) {
    switch (p.stage) {
        case REC_SEPARATORS: {
            const int r = record_of(p.recOff, p.numRecords, i);
            if (i >= p.recOff[r + 1] - p.gap) p.tcodes[i] = (uint8_t)p.sep;
            break;
        }
        case REC_STARTS: {
            const int c = p.cols[p.firstHit + i];
            p.starts[i] -= p.recOff[record_of(p.recOff, p.numRecords, c)];
            break;
        }
        case REC_HITS: {
            const long long h = p.firstHit + i;
            const int r = record_of(p.recOff, p.numRecords, p.cols[h]);
            p.records[h] = r;
            p.cols[h] -= p.recOff[r];
            break;
        }
        default: break;
    }
}

// =============================================================================================
// B -- k-banded NW sweep of a LONG query, one alignment per THREAD (ref myersCalcEditDistanceNW cpp:730-928 with
// its Ukkonen band, cpp:755, 799-830).  The thread holds a window of NW = 4*NB words (32*NW rows) of the column in
// registers; the window slides down the band one WORD at a time, at columns that are multiples of 32 for every
// thread of the launch (the window top is 32*floor(c/32) + A, A a multiple of 32 chosen per job so that the top
// stays at or above the band's top diagonal dhi), so control flow stays uniform.  Rows above the window are outside
// the band: the horizontal delta entering its top row is the pessimistic +1 (ref cpp:779; for the true first row
// it is the NW boundary), rows entering at the bottom start from vertical deltas +1.  Every cell whose optimal
// path stays inside the band is exact, everything else an upper bound: the result is valid iff it is <= the bound
// the band was planned for (the host checks that, as for the warp kernel's sliding window).  The profile (peq_kernel:
// [code][nWp] words in global memory) is far too large for per-thread shared memory, so the thread keeps only the
// window's words of every code there (`acc`: NW + BAND_SLACK word slots per code; the origin moves up one slot per
// slide and the slots are moved back every BAND_SLACK slides) and fetches ncodes new words per slide.
// Needs: nWp >= NW, 32*NW >= band height + 31 + ((off - dhi) - A) (WRunner::run_band sizes NB that way).
// =============================================================================================
constexpr int BAND_SLACK = 4;

// S = A + B + cin over four words; returns the carry out.
EB_HD uint32_t chain4(uint32_t (&S)[4], const uint32_t (&A)[4], const uint32_t (&B)[4], uint32_t cin) {
#if defined(__CUDA_ARCH__)
    uint32_t cout;
    asm("{\n\t.reg .u32 t;\n\t"
        "add.cc.u32 t, %13, 0xffffffff;\n\t"
        "addc.cc.u32 %0, %5, %9;\n\t"
        "addc.cc.u32 %1, %6, %10;\n\t"
        "addc.cc.u32 %2, %7, %11;\n\t"
        "addc.cc.u32 %3, %8, %12;\n\t"
        "addc.u32 %4, 0, 0;\n\t}"
        : "=&r"(S[0]), "=&r"(S[1]), "=&r"(S[2]), "=&r"(S[3]), "=&r"(cout)
        : "r"(A[0]), "r"(A[1]), "r"(A[2]), "r"(A[3]), "r"(B[0]), "r"(B[1]), "r"(B[2]), "r"(B[3]), "r"(cin));
    return cout;
#else
    uint32_t carry = cin;
    for (int w = 0; w < 4; ++w) {
        const uint64_t s = (uint64_t)A[w] + B[w] + carry;
        S[w] = (uint32_t)s;
        carry = (uint32_t)(s >> 32);
    }
    return carry;
#endif
}

struct BandCarry {
    uint32_t add, ph, mh;  // carries into the next block of four words: of the add, of Ph << 1, of Mh << 1
};

// Column step of words [4*B, 4*B+4) of the window (k1_step with the carries between blocks spelled out).
template <int NW, int B>
EB_HD void band_block(uint32_t (&Pv)[NW], uint32_t (&Mv)[NW], const uint32_t (&Eq)[4], BandCarry& cy) {
    uint32_t P[4], M[4], T[4], S[4], Ph[4], Mh[4], Phs[4], Mhs[4];
    EB_UNROLL
    for (int i = 0; i < 4; ++i) {
        P[i] = Pv[4 * B + i];
        M[i] = Mv[4 * B + i];
        T[i] = Eq[i] & P[i];
    }
    cy.add = chain4(S, T, P, cy.add);
    EB_UNROLL
    for (int i = 0; i < 4; ++i) {
        const uint32_t Xh = (S[i] ^ P[i]) | Eq[i];
        Ph[i] = M[i] | ~(Xh | P[i]);
        Mh[i] = P[i] & Xh;
    }
    cy.ph = chain4(Phs, Ph, Ph, cy.ph);
    cy.mh = chain4(Mhs, Mh, Mh, cy.mh);
    EB_UNROLL
    for (int i = 0; i < 4; ++i) {
        const uint32_t Xv = Eq[i] | M[i];
        Pv[4 * B + i] = Mhs[i] | ~(Xv | Phs[i]);
        Mv[4 * B + i] = Phs[i] & Xv;
    }
}

template <int NW, int B, int NB, class BAcc>
struct BandBlocks {
    static EB_HD void run(uint32_t (&Pv)[NW], uint32_t (&Mv)[NW], const BAcc& acc, uint32_t codeOff, BandCarry& cy) {
        uint32_t Eq[4];
        EB_UNROLL
        for (int i = 0; i < 4; ++i) Eq[i] = acc.load(codeOff, 4 * B + i);
        band_block<NW, B>(Pv, Mv, Eq, cy);
        BandBlocks<NW, B + 1, NB, BAcc>::run(Pv, Mv, acc, codeOff, cy);
    }
};
template <int NW, int NB, class BAcc>
struct BandBlocks<NW, NB, NB, BAcc> {
    static EB_HD void run(uint32_t (&)[NW], uint32_t (&)[NW], const BAcc&, uint32_t, BandCarry&) {}
};

// BAcc: the thread's window of the profile.  set(code, slot, bits) writes a slot (absolute slot index), get(code, slot)
// reads one; origin(slot) makes `slot` the window's first word for the column loop's load(code_off(sym), w), w a
// compile-time word of the window.
template <int NB, class BAcc>
EB_HD void band_job(const WParams& P, int jobIdx, BAcc& acc, int ncodes) {
    constexpr int NW = 4 * NB;
    const WJob J = P.jobs[jobIdx];
    const int n = J.n, nWp = J.nWp;
    const int off = 32 * nWp - J.m;
    const uint32_t* peq = P.peq + J.peqOff;
    const uint8_t* t = P.tcodes + J.tOff;
    Rec* rec = P.recs + J.rec;
    int A = off - J.dhi;  // window top of column c: 32*floor(c/32) + A rounded down to a multiple of 32, at most 0
    A = (A >= 0) ? 0 : -(((-A) + 31) / 32) * 32;
    const int topMax = nWp - NW;
    int top = 0, org = 0;
    for (int code = 0; code < ncodes; ++code)
        for (int w = 0; w < NW; ++w) acc.set(code, w, peq[(size_t)code * nWp + w]);
    acc.origin(0);
    uint32_t Pv[NW], Mv[NW];
    EB_UNROLL
    for (int w = 0; w < NW; ++w) {
        Pv[w] = init_pv_word(w, off);
        Mv[w] = 0;
    }
    int score = 32 * NW - off;  // D of the window's bottom row in column -1
    Sym16 syms;
    syms.w[0] = syms.w[1] = syms.w[2] = syms.w[3] = 0;
    for (int c = 0; c < n; ++c) {
        if ((c & 15) == 0) {
            syms = load_sym16(t + c);
        } else if ((c & 3) == 0) {  // next four symbols into word 0 (static indices: the words stay in registers)
            syms.w[0] = syms.w[1];
            syms.w[1] = syms.w[2];
            syms.w[2] = syms.w[3];
        }
        if ((c & 31) == 0 && ((c + A) >> 5) > top && top < topMax) {
            // slide: drop the top word, open a fresh one at the bottom (vertical deltas +1: ref cpp:799-809 grows the
            // band the same way), fetch its profile words
            EB_UNROLL
            for (int w = 0; w + 1 < NW; ++w) {
                Pv[w] = Pv[w + 1];
                Mv[w] = Mv[w + 1];
            }
            Pv[NW - 1] = ~0u;
            Mv[NW - 1] = 0u;
            score += 32;
            ++top;
            ++org;
            if (org == BAND_SLACK) {  // move the slots back to the front
                for (int code = 0; code < ncodes; ++code)
                    for (int w = 0; w + 1 < NW; ++w) acc.set(code, w, acc.get(code, w + BAND_SLACK));
                org = 0;
            }
            for (int code = 0; code < ncodes; ++code) acc.set(code, org + NW - 1, peq[(size_t)code * nWp + top + NW - 1]);
            acc.origin(org);
        }
        const uint32_t sym = (syms.w[0] >> (8 * (c & 3))) & 255u;
        BandCarry cy;
        cy.add = 0;
        cy.ph = 1;  // +1 enters above the window's top row
        cy.mh = 0;
        BandBlocks<NW, 0, NB, BAcc>::run(Pv, Mv, acc, acc.code_off(sym), cy);
        score += (int)cy.ph - (int)cy.mh;  // horizontal delta of the window's bottom row
    }
    // the window ends on the query's last row (top == topMax by the band's geometry); a window that did not get
    // there cannot hold the bottom-right cell: report a score above every bound
    rec->best = (top == topMax) ? score : 0x3fffffff;  // ref cpp:916
    rec->cnt = 1;
    rec->last = n - 1;
    rec->pos[0] = n - 1;
}

// =============================================================================================
// W -- one alignment per warp.  Lane l holds R consecutive words (a "chunk"); the 32 chunks of
// a warp form a window of 1024*R rows.  A query taller than the window is swept in strips
// (fixed windows stacked vertically, the horizontal deltas of a strip's bottom row feeding the
// next strip), or -- NW with a k-band narrower than the window -- by ONE window sliding down
// the band.  The backend B supplies the warp primitives (device: shuffles/votes; host
// emulation: 32-wide vectors).  All control flow is warp-uniform.
// =============================================================================================

struct InitPvFn {
    int off;
    EB_HD uint32_t operator()(uint32_t wordIdx) const { return init_pv_word((int)wordIdx, off); }
};
struct InitSbFn {  // D at the bottom row of a chunk in column -1: rows above it that are real
    int off, rowsPerChunk;
    EB_HD uint32_t operator()(uint32_t chunkIdx) const {
        const long long v = (long long)(chunkIdx + 1) * rowsPerChunk - off;
        return v > 0 ? (uint32_t)v : 0u;
    }
};

// FEAT is a compile-time superset of what the job may need (WM_* bits): a feature whose bit is clear is
// compiled out, so the per-column loop of the common job shapes carries no test for sliding, matrix
// stores, stop columns, tracking or strip hand-over (w_dispatch picks the instantiation).
enum WMask : int { WM_SLIDE = 1, WM_STORE = 2, WM_STOPCOL = 4, WM_TRACK = 8, WM_STRIPS = 16, WM_ALL = 31 };

template <class B, int R, int FEAT = WM_ALL>
EB_HD void w_sweep(const WParams& P, int jobIdx) {
    using U = typename B::U;
    using Pr = typename B::P;
    const WJob J = P.jobs[jobIdx];
    const int m = J.m, n = J.n, nWp = J.nWp;
    const int off = 32 * nWp - m;
    const int chunksTotal = nWp / R;
    const bool slide = (FEAT & WM_SLIDE) && (J.flags & WF_SLIDE) != 0;
    const bool store = (FEAT & WM_STORE) && (J.flags & WF_STORE) != 0;
    const bool stopcol = (FEAT & WM_STOPCOL) && (J.flags & WF_STOPCOL) != 0;
    const bool trev = (J.flags & WF_TREV) != 0;
    const int strips = (slide || !(FEAT & WM_STRIPS)) ? 1 : (chunksTotal + 31) / 32;
    const uint8_t* tptr = P.tcodes + J.tOff;
    const uint32_t* peq = P.peq + J.peqOff;
    const U lane = B::lane();
    const Pr isTop = (lane == 0u);
    const Pr isBot = (lane == 31u);
    const int topOne = (J.mode != MODE_HW) ? 1 : 0;
    Rec* rec = P.recs + J.rec;
    int bestU = J.kInit, cntU = 0;
    const int rowsPerChunk = 32 * R;

    for (int strip = 0; strip < strips; ++strip) {
        int topChunk = strip * 32;
        const bool lastStrip = (strip == strips - 1);
        const bool track = (FEAT & WM_TRACK) && lastStrip && J.mode != MODE_NW && !stopcol;
        const uint8_t* hin = nullptr;
        uint8_t* hout = nullptr;
        if (strips > 1) {
            uint8_t* h0 = P.hbuf + J.hbufOff;
            uint8_t* h1 = h0 + n;
            if (strip > 0) hin = (strip & 1) ? h0 : h1;
            if (!lastStrip) hout = (strip & 1) ? h1 : h0;
        }
        U Pv[R], Mv[R];
        EB_UNROLL
        for (int i = 0; i < R; ++i) {
            Pv[i] = B::map((U(topChunk) + lane) * U(R) + U(i), InitPvFn{off});
            Mv[i] = U(0u);
        }
        U sb = B::map(U(topChunk) + lane, InitSbFn{off, rowsPerChunk});
        U symsV = U(0u), hinV = U(0u);

        for (int c = 0; c < n; ++c) {
            if ((c & 31) == 0) {  // 32 target symbols (and strip inputs) per refill, one per lane
                const U idx = U(c) + lane;
                const Pr ok = idx < U(n);
                symsV = trev ? B::gather8_neg(tptr, idx, ok) : B::gather8(tptr, idx, ok);
                if (hin) hinV = B::gather8(hin, idx, ok);
            }
            const int sym = (int)B::bcast(symsV, c & 31);
            if (slide) {
                const int want = c - J.dhi + off;
                const int wantChunk = want > 0 ? want / rowsPerChunk : 0;
                while (topChunk < wantChunk) {  // drop the top chunk, open a fresh one at the bottom
                    const uint32_t old31 = B::bcast(sb, 31);
                    EB_UNROLL
                    for (int i = 0; i < R; ++i) {
                        Pv[i] = B::sel(isBot, U(~0u), B::shfl_down1(Pv[i]));
                        Mv[i] = B::sel(isBot, U(0u), B::shfl_down1(Mv[i]));
                    }
                    sb = B::sel(isBot, U(old31 + (uint32_t)rowsPerChunk), B::shfl_down1(sb));
                    ++topChunk;
                }
            }
            const int ownerLane = chunksTotal - 1 - topChunk;  // lane whose chunk ends at row m-1

            // Eq words of this lane's chunk for the column's symbol
            U Eq[R], EqX[R];
            const uint32_t* peqRow = peq + (size_t)sym * nWp;
            EB_UNROLL
            for (int i = 0; i < R; ++i) {
                const U widx = (U(topChunk) + lane) * U(R) + U(i);
                Eq[i] = B::gather32(peqRow, widx, widx < U(nWp));
            }
            // horizontal delta entering the window's top row
            int hinP, hinM;
            if (hin) {
                const int hv = (int)B::bcast(hinV, c & 31);
                hinP = hv & 1;
                hinM = (hv >> 1) & 1;
            } else if (slide && topChunk > 0) {
                hinP = 1;  // rows above a sliding window are outside the band: pessimistic +1 (ref cpp:779)
                hinM = 0;
            } else {
                hinP = topOne;
                hinM = 0;
            }
            // (Eq & Pv) + Pv over the whole window: ripple inside the lane, ballot across lanes
            U S[R];
            U carry = U(0u);
            Pr allOnes = (lane == lane);
            EB_UNROLL
            for (int i = 0; i < R; ++i) {
                U e = Eq[i];
                if (i == 0) e = e | B::sel(isTop, U((uint32_t)hinM), U(0u));  // ref cpp:423
                EqX[i] = e;
                const U t = e & Pv[i];
                U s = t + Pv[i];
                const U c1 = B::toU(s < t);
                s = s + carry;
                const U c2 = B::toU(s < carry);
                carry = c1 | c2;
                S[i] = s;
                allOnes = allOnes & (s == U(~0u));
            }
            const uint32_t G = B::ballot(carry != U(0u));
            const uint32_t Pg = B::ballot(allOnes);
            const uint32_t cinMask = ((G | Pg) + G) ^ Pg;  // bit l = carry entering lane l
            U cin = (U(cinMask) >> lane) & U(1u);
            EB_UNROLL
            for (int i = 0; i < R; ++i) {
                S[i] = S[i] + cin;
                cin = cin & B::toU(S[i] == U(0u));
            }
            U Ph[R], Mh[R];
            EB_UNROLL
            for (int i = 0; i < R; ++i) {
                const U Xh = (S[i] ^ Pv[i]) | EqX[i];
                Ph[i] = Mv[i] | ~(Xh | Pv[i]);
                Mh[i] = Pv[i] & Xh;
            }
            const U hp = Ph[R - 1] >> 31, hm = Mh[R - 1] >> 31;  // delta leaving this chunk's bottom row
            const U inP = B::sel(isTop, U((uint32_t)hinP), B::shfl_up1(hp));
            const U inM = B::sel(isTop, U((uint32_t)hinM), B::shfl_up1(hm));
            EB_UNROLL
            for (int i = R - 1; i >= 0; --i) {
                const U Phs = (Ph[i] << 1) | (i ? (Ph[i ? i - 1 : 0] >> 31) : inP);
                const U Mhs = (Mh[i] << 1) | (i ? (Mh[i ? i - 1 : 0] >> 31) : inM);
                const U Xv = Eq[i] | Mv[i];
                Pv[i] = Mhs | ~(Xv | Phs);
                Mv[i] = Phs & Xv;
            }
            sb = sb + hp - hm;

            if (store) {
                EB_UNROLL
                for (int i = 0; i < R; ++i) {
                    const U widx = (U(topChunk) + lane) * U(R) + U(i);
                    B::scatterU2(P.mat + J.auxOff, U((uint32_t)c * (uint32_t)nWp) + widx, Pv[i], Ph[i], widx < U(nWp));
                }
            }
            if (hout) B::scatter8(hout, U((uint32_t)c), hp | (hm << 1), isBot);
            if (track && c >= J.trackFrom) {
                const Pr ev = (lane == U((uint32_t)ownerLane)) & (sb <= U((uint32_t)bestU));
                if (B::any(ev)) {  // ref cpp:658-673
                    const int s = (int)B::bcast(sb, ownerLane);
                    if (s < bestU) {
                        bestU = s;
                        cntU = 0;
                    }
                    if (cntU < KPOS) {
                        B::store_uniform(&rec->pos[cntU], c);
                    } else if (P.ovfCap > 0) {  // second pass only (see k1_event)
                        const int slot = B::atomic_add_uniform(P.ovfCount, 1);
                        if (slot < P.ovfCap) {
                            B::store_uniform(&P.ovf[slot].rec, J.rec);
                            B::store_uniform(&P.ovf[slot].score, s);
                            B::store_uniform(&P.ovf[slot].pos, c);
                        }
                    }
                    B::store_uniform(&rec->last, c);
                    ++cntU;
                }
            }
            if (stopcol && c == J.stopCol) {
                // Dump D[r][c] for the rows inside the window (ref cpp:896-908 keeps the stop
                // column); later strips still need their rows, so only this strip's sweep ends.
                B::dump_column(P.colOut + J.auxOff, Pv, Mv, sb, topChunk, R, off, m);
                break;
            }
        }
        if (lastStrip) {
            if (stopcol) {
                B::store_uniform(&rec->best, -1);
                B::store_uniform(&rec->cnt, 0);
            } else if (J.mode == MODE_NW) {
                const int ownerLane = chunksTotal - 1 - topChunk;
                const int s = (int)B::bcast(sb, ownerLane);
                B::store_uniform(&rec->best, s);  // ref cpp:916: bottom-right cell
                B::store_uniform(&rec->cnt, 1);
                B::store_uniform(&rec->last, n - 1);
                B::store_uniform(&rec->pos[0], n - 1);
            } else {
                B::store_uniform(&rec->best, bestU);
                B::store_uniform(&rec->cnt, cntU);
            }
        }
    }
}

// Picks the leanest instantiation that covers the job (all branches warp-uniform).
template <class B, int R>
EB_HD void w_dispatch(const WParams& P, int jobIdx) {
    const int flags = P.jobs[jobIdx].flags, mode = P.jobs[jobIdx].mode;
    const int nWp = P.jobs[jobIdx].nWp;
    const bool slide = (flags & WF_SLIDE) != 0;
    const bool strips = !slide && (nWp / R) > 32;
    int need = (slide ? WM_SLIDE : 0) | ((flags & WF_STORE) ? WM_STORE : 0) | ((flags & WF_STOPCOL) ? WM_STOPCOL : 0) |
               ((mode != MODE_NW && !(flags & WF_STOPCOL)) ? WM_TRACK : 0) | (strips ? WM_STRIPS : 0);
    if (need == 0) w_sweep<B, R, 0>(P, jobIdx);                                         // NW, one fixed window
    else if (need == WM_SLIDE) w_sweep<B, R, WM_SLIDE>(P, jobIdx);                      // banded NW
    else if (need == WM_TRACK) w_sweep<B, R, WM_TRACK>(P, jobIdx);                      // HW / SHW, one window
    else if (need == WM_STORE) w_sweep<B, R, WM_STORE>(P, jobIdx);                      // matrix-storing NW
    else if (need == WM_STOPCOL) w_sweep<B, R, WM_STOPCOL>(P, jobIdx);                  // Hirschberg half, fixed
    else if (need == (WM_STOPCOL | WM_SLIDE)) w_sweep<B, R, WM_STOPCOL | WM_SLIDE>(P, jobIdx);  // ... banded
    else w_sweep<B, R, WM_ALL>(P, jobIdx);                                              // strips and mixtures
}

// Scalar helper used by both backends' dump_column: writes the scores of one lane's chunk.
// Bits are walked from the chunk's bottom row upward (ref getBlockCellValues cpp:470-482).
template <int R>
EB_HD void dump_chunk_scores(int* out, const uint32_t* Pv, const uint32_t* Mv, uint32_t sb,
                             int chunkIdx, int off, int m) {
    int score = (int)sb;
    for (int i = R - 1; i >= 0; --i) {
        for (int b = 31; b >= 0; --b) {
            const long long g = ((long long)chunkIdx * R + i) * 32 + b;
            const long long r = g - off;
            if (r >= 0 && r < m) out[r] = score;
            score -= (int)((Pv[i] >> b) & 1u);
            score += (int)((Mv[i] >> b) & 1u);
        }
    }
}

// Query profile of one W job: lanes stride over the words (ref buildPeq cpp:358-384, top
// padding instead of bottom wildcards, optional reversed query for cpp:232-234).
EB_HD void peq_build_words(const PeqParams& p, int jobIdx, int firstWord, int wordStride) {
    const WJob J = p.jobs[jobIdx];
    const int off = 32 * J.nWp - J.m;
    const uint32_t padBit = (J.mode == MODE_HW) ? 1u : 0u;
    const uint8_t* q = p.qcodes + J.qOff;
    const bool rev = (J.flags & WF_QREV) != 0;
    uint32_t* dst = p.peq + J.peqOff;
    for (int w = firstWord; w < J.nWp; w += wordStride) {
        for (int code = 0; code < p.ncodes; ++code) {
            uint32_t bits = 0;
            for (int b = 0; b < 32; ++b) {
                const int g = w * 32 + b;
                uint32_t bit;
                if (g < off) {
                    bit = padBit;
                } else {
                    const int r = g - off;
                    const int qc = rev ? q[J.m - 1 - r] : q[r];
                    bit = p.eqtab ? (p.eqtab[qc * p.ncodes + code] ? 1u : 0u) : (qc == code ? 1u : 0u);
                }
                bits |= bit << b;
            }
            dst[(size_t)code * J.nWp + w] = bits;
        }
    }
}

// Traceback over the stored {Pv, Ph} matrix of an NW sweep (restates obtainAlignmentTraceback,
// ref cpp:942-1141): from the bottom-right cell prefer UP (vertical delta +1 -> INSERT,
// cpp:1020), then LEFT (horizontal delta +1 -> DELETE, cpp:1054), else the diagonal, which is a
// MATCH exactly when the symbols are equal (cpp:1086 decides by score; equal symbols <=> equal
// scores on a diagonal step that is neither UP- nor LEFT-explained).  Edges run out as in
// cpp:1025-1029, 1059-1065, 1090-1103.  Ops are written back-to-front, so no final reverse.
EB_HD void traceback_job(const TbParams& p, int jobIdx) {
    const TbJob J = p.jobs[jobIdx];
    if (J.n <= 0 || J.m <= 0) {  // empty side: the caller fills the script (ref cpp:1168-1175)
        p.opsStart[jobIdx] = 0;
        p.opsLen[jobIdx] = 0;
        return;
    }
    const U2* mat = p.mat + J.matOff;
    const size_t step = p.matStep > 1 ? (size_t)p.matStep : 1;
    const uint32_t* peq = p.peq + (J.peqOff != ~0ull ? J.peqOff : 0);
    const uint8_t* t = p.tcodes + J.tOff;
    uint8_t* ops = p.ops + J.outOff;
    const int off = 32 * J.nWp - J.m;
    int w = J.m + J.n;  // next write position + 1
    int r = J.m - 1, c = J.n - 1;
    for (;;) {
        const int g = r + off;
        const U2 e = mat[((size_t)c * J.nWp + (g >> 5)) * step];
        const uint32_t bit = 1u << (g & 31);
        if (e.x & bit) {  // up
            ops[--w] = 1;
            if (--r < 0) {
                for (int i = 0; i <= c; ++i) ops[--w] = 2;
                break;
            }
        } else if (e.y & bit) {  // left
            ops[--w] = 2;
            if (--c < 0) {
                for (int i = 0; i <= r; ++i) ops[--w] = 1;
                break;
            }
        } else {
            uint32_t eq;
            if (J.peqOff != ~0ull) {
                eq = peq[(size_t)t[c] * J.nWp + (g >> 5)] & bit;
            } else {  // lane sweeps keep no Peq in global memory: compare the symbols directly
                const int qc = p.qcodes[J.qOff + (uint64_t)r];
                eq = p.eqtab ? p.eqtab[qc * p.ncodes + t[c]] : (uint32_t)(qc == t[c]);
            }
            ops[--w] = eq ? 0 : 3;
            --r;
            --c;
            if (c < 0) {
                for (int i = 0; i <= r; ++i) ops[--w] = 1;
                break;
            }
            if (r < 0) {
                for (int i = 0; i <= c; ++i) ops[--w] = 2;
                break;
            }
        }
    }
    p.opsStart[jobIdx] = w;
    p.opsLen[jobIdx] = J.m + J.n - w;
}

// Split row of one Hirschberg node.  With L[h] = distance(q[0..h), left half) and R[s] = distance(last s
// query rows, right half): the first h in 1..m-1 with L[h] + R[m-h] == best (cpp:1327-1335), else the
// top boundary h = 0 (cpp:1337-1344), else the bottom boundary h = m (cpp:1345-1353).
EB_HD void split_node(const SplitParams& p, int nodeIdx) {
    const SplitNode nd = p.nodes[nodeIdx];
    const int* colF = p.cols + nd.colF;
    const int* colR = p.cols + nd.colR;
    int h = -1;
    for (int cand = 1; cand <= nd.m - 1; ++cand) {
        if (colF[cand - 1] + colR[nd.m - cand - 1] == nd.best) {
            h = cand;
            break;
        }
    }
    if (h < 0 && nd.leftW + colR[nd.m - 1] == nd.best) h = 0;
    if (h < 0 && colF[nd.m - 1] + nd.rightW == nd.best) h = nd.m;
    SplitOut o;
    o.h = h;
    o.left = h < 0 ? 0 : (h == 0 ? nd.leftW : colF[h - 1]);
    o.right = h < 0 ? 0 : (h == nd.m ? nd.rightW : colR[nd.m - h - 1]);
    o.rsv = 0;
    p.out[nodeIdx] = o;
}

// Presence set of one item (<= 64 KiB of raw bytes): the bytes at first, first+stride, ... into local[8].  Strand batches
// (p.rc): bytes of the read block are also written complemented to their place in the reverse-complement block, whose
// presence set goes to rcLocal[8] (zero for targets).
EB_HD MaskItem mask_item_scan(const MaskParams& p, int itemIdx, int first, int stride, uint32_t (&local)[8], uint32_t (&rcLocal)[8]) {
    MaskItem it;
    if (itemIdx < p.numItems) {
        it = p.items[itemIdx];
    } else {
        const int q = itemIdx - p.numItems;
        const int pair = p.rc ? 2 * q : q;
        it.off = p.qoff[pair];
        it.len = p.qlen[pair] <= 65536 ? p.qlen[pair] : 0;
        it.dst = pair;
    }
    for (int k = 0; k < 8; ++k) local[k] = rcLocal[k] = 0;
    const uint8_t* s = p.raw + it.off;
    const bool rc = p.rc && it.off < p.rcBytes;
    for (int i = first; i < it.len; i += stride) {
        const uint32_t b = s[i];
        local[b >> 5] |= 1u << (b & 31);
        if (rc) {
            const uint32_t c = complement_byte((uint8_t)b);
            p.rc[p.rcBytes - 1 - (it.off + (uint64_t)i)] = (uint8_t)c;
            rcLocal[c >> 5] |= 1u << (c & 31);
        }
    }
    return it;
}
// OR word k of an item's presence set into its destination set and into the union set.  The union is
// read first: after the first few items it already holds every byte value, and the atomics disappear.
EB_HD void mask_item_commit(const MaskParams& p, int dst, int k, uint32_t bits) {
    if (!bits) return;
    atomic_or_u32(&p.masks[(size_t)dst * 8 + k], bits);
    if (p.unionSet >= 0) {
        uint32_t* u = &p.masks[(size_t)p.unionSet * 8 + k];
        if (bits & ~*u) atomic_or_u32(u, bits);
    }
}
// Whole item by one caller (host emulation).
EB_HD void mask_item(const MaskParams& p, int itemIdx, int first, int stride) {
    uint32_t local[8], rcLocal[8];
    const MaskItem it = mask_item_scan(p, itemIdx, first, stride, local, rcLocal);
    for (int k = 0; k < 8; ++k) mask_item_commit(p, it.dst, k, local[k]);
    for (int k = 0; k < 8; ++k) mask_item_commit(p, it.dst + 1, k, rcLocal[k]);  // (nothing for targets and plain batches)
}

// Presence set of query `q` of a QAlphaParams run: the bytes at first, first+stride, ... into local[8].
EB_HD void qalpha_scan(const QAlphaParams& p, int q, int first, int stride, uint32_t (&local)[8]) {
    const int pair = p.firstPair + q;
    const uint8_t* s = p.raw + p.qoff[pair];
    const int len = p.qlen[pair];
    for (int k = 0; k < 8; ++k) local[k] = 0;
    for (int i = first; i < len; i += stride) {
        const uint32_t b = s[i];
        local[b >> 5] |= 1u << (b & 31);
    }
}
// alphabetLength of one pair: distinct byte values in query and target together
// (ref transformSequences cpp:1437-1461 counts them while recoding).
EB_HD int alpha_len_pair(const uint32_t* masks, int qset, int tset) {
    int c = 0;
    for (int k = 0; k < 8; ++k) {
        const uint32_t v = masks[(size_t)qset * 8 + k] | masks[(size_t)tset * 8 + k];
#if defined(__CUDA_ARCH__)
        c += __popc(v);
#else
        c += __builtin_popcount(v);
#endif
    }
    return c;
}

}  // namespace eb
