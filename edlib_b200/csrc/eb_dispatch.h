// eb_dispatch.h -- run-time launch values to the template arguments of the kernel instances.  The CUDA backend
// (eb_kernels.cu) and the CPU emulation (tests/emul/emul_backend.cpp) both select through these, so they accept the
// same values and instantiate the same classes.  Plain C++17, no CUDA.
#pragma once
#include <algorithm>
#include <stdexcept>
#include <type_traits>

#include "eb_common.h"

namespace eb {

// f(std::integral_constant<int, V>{}) for the V of Vs equal to v; throws std::runtime_error(what) when there is none.
template <int... Vs, class F>
void with_one_of(int v, const char* what, F&& f) {
    const bool found = ((v == Vs ? (f(std::integral_constant<int, Vs>{}), true) : false) || ...);
    if (!found) throw std::runtime_error(what);
}

// Word class: 32-row words per query (queries of up to 256 rows).
template <class F>
void with_nw(int nw, F&& f) {
    with_one_of<1, 2, 3, 4, 5, 6, 7, 8>(nw, "bad word class", f);
}
// Window blocks (of four words) of the band kernel.
template <class F>
void with_nb(int nb, F&& f) {
    with_one_of<1, 2, 3, 4, 5, 6, 7, 8>(nb, "bad band window size", f);
}
// Words per lane of the warp kernel.
template <class F>
void with_r(int R, F&& f) {
    with_one_of<1, 2, 4, 8>(R, "bad W chunk size", f);
}
template <class F>
void with_mode(int mode, F&& f) {
    with_one_of<MODE_NW, MODE_SHW, MODE_HW>(mode, "bad alignment mode", f);
}

// The lane-kernel classes that exist: matrix-storing NW, reversed SHW, forward NW / SHW / HW.
template <int M, bool R, bool S>
struct LaneClass {
    static constexpr int MODE = M;
    static constexpr bool REV = R, STORE = S;
};
template <class F>
void with_lane_class(int mode, bool rev, bool store, F&& f) {
    if (store) f(LaneClass<MODE_NW, false, true>{});
    else if (rev && mode == MODE_SHW) f(LaneClass<MODE_SHW, true, false>{});
    else if (!rev && mode == MODE_HW) f(LaneClass<MODE_HW, false, false>{});
    else if (!rev && mode == MODE_SHW) f(LaneClass<MODE_SHW, false, false>{});
    else if (!rev && mode == MODE_NW) f(LaneClass<MODE_NW, false, false>{});
    else throw std::runtime_error("unsupported lane class");
}

// Candidate capacity of the seed planner (per read) at a seed level.
template <class F>
void with_seed_cap(int level, F&& f) {
    if (level <= 0) f(std::integral_constant<int, SEED_CAND_0>{});
    else if (level == 1) f(std::integral_constant<int, SEED_CAND_1>{});
    else f(std::integral_constant<int, SEED_CAND_2>{});
}

// Instance of the seed planning kernel for a launch (eb_kernels.cu: seed_plan_kernel<CAP, THREADS, CoopGroup<GW>>):
// f(cap, threads, gw), each an integral constant.  A read has t + 1 <= min(maxLen / Ls, seedK + 1) seeds: groups of
// 16 lanes look them all up in one round when that is at most 16, whole warps otherwise (or when the read lengths
// are not known); the last level is planned by a warp per read, two reads per CTA.
template <class F>
void with_seed_plan_instance(const SeedPlanParams& p, F&& f) {
    const bool narrow = p.maxLen > 0 && p.Ls > 0 && std::min(p.maxLen / p.Ls, p.seedK + 1) <= 16;
    with_seed_cap(p.level, [&](auto cap) {
        using I64 = std::integral_constant<int, 64>;
        using I128 = std::integral_constant<int, 128>;
        using I16 = std::integral_constant<int, 16>;
        using I32 = std::integral_constant<int, 32>;
        if constexpr (decltype(cap)::value == SEED_CAND_2) f(cap, I64{}, I32{});
        else if (narrow) f(cap, I128{}, I16{});
        else f(cap, I128{}, I32{});
    });
}

}  // namespace eb
