// TEST INFRASTRUCTURE: host spelling of the planning group CoopGroup<W> of eb_kernels.cu, so that the emulation runs
// seed_plan_read (eb_core.h) at the width the device uses.  One std::thread per lane of a warp; a barrier per group for
// sync(), a warp barrier for reserve(); scans go through an exchange array.  Used only by tests/emul/emul_backend.cpp
// (EDLIB_EMUL_SEED_GROUP=device).
#pragma once
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace ebhost {

struct LaneBarrier {
    explicit LaneBarrier(int members) : n(members) {}
    void wait() {
        std::unique_lock<std::mutex> lock(m);
        const long g = gen;
        if (++arrived == n) {
            arrived = 0;
            ++gen;
            cv.notify_all();
        } else {
            cv.wait(lock, [&] { return gen != g; });
        }
    }
    std::mutex m;
    std::condition_variable cv;
    const int n;
    int arrived = 0;
    long gen = 0;
};

// The shared state of one emulated warp: its groups' barriers, the warp barrier and the exchange words.
struct LaneWarp {
    explicit LaneWarp(int groupWidth) : warp(32) {
        for (int g = 0; g < 32 / groupWidth; ++g) group.emplace_back(new LaneBarrier(groupWidth));
    }
    LaneBarrier warp;
    std::vector<std::unique_ptr<LaneBarrier>> group;
    int xchg[32] = {};
    int base = 0;
};

inline thread_local LaneWarp* tlWarp = nullptr;
inline thread_local int tlLane = 0;  // lane of the calling thread in its warp (0..31)

template <int GW>
struct CoopThreads {
    static_assert(GW >= 1 && GW <= 32 && (GW & (GW - 1)) == 0, "group width: a power of two up to a warp");
    static constexpr int W = GW;
    static int lane() { return tlLane & (GW - 1); }
    static int width() { return GW; }
    static int first() { return tlLane & ~(GW - 1); }
    static void sync() { tlWarp->group[tlLane / GW]->wait(); }
    static bool any(bool v) {
        tlWarp->xchg[tlLane] = v ? 1 : 0;
        sync();
        bool r = false;
        for (int l = first(); l < first() + GW; ++l) r = r || tlWarp->xchg[l] != 0;
        sync();  // every member has read the exchange before it is written again
        return r;
    }
    static int add_shared(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
    static int scan(int v, int& total) {
        tlWarp->xchg[tlLane] = v;
        sync();
        int pre = 0;
        total = 0;
        for (int l = first(); l < first() + GW; ++l) {
            if (l < tlLane) pre += tlWarp->xchg[l];
            total += tlWarp->xchg[l];
        }
        sync();
        return pre;
    }
    // the whole warp, as on the device: one atomic for the warp's total, each group's offset in it (groups in lane order)
    static int reserve(int* counter, int n) {
        LaneWarp& w = *tlWarp;
        w.xchg[tlLane] = n;
        w.warp.wait();
        int before = 0, total = 0;
        for (int l = 0; l < 32; l += GW) {
            if (l < first()) before += w.xchg[l];
            total += w.xchg[l];
        }
        if (tlLane == 31 && total > 0) w.base = __atomic_fetch_add(counter, total, __ATOMIC_SEQ_CST);
        w.warp.wait();
        const int base = total > 0 ? w.base : 0;
        w.warp.wait();  // base and the exchange are read before the next reserve writes them
        return base + before;
    }
};

// Runs body(slot) on 32 lane threads per warp, warp after warp, for the slots of `ctas` CTAs of `threads` threads in
// groups of GW lanes (slot = CTA * (threads / GW) + group, as seed_plan_kernel numbers them).  body gets the group's
// index within the warp; every lane of every warp runs, also past the last read.
template <int GW, class F>
void run_lane_groups(int ctas, int threads, F&& body) {
    const int warps = ctas * (threads / 32);
    LaneWarp w(GW);
    std::vector<std::thread> lanes;
    for (int l = 0; l < 32; ++l)
        lanes.emplace_back([&, l] {
            tlWarp = &w;
            tlLane = l;
            for (int wi = 0; wi < warps; ++wi) {
                body(wi * (32 / GW) + l / GW, l / GW);
                w.warp.wait();  // the warp's scratch is reused by the next warp
            }
        });
    for (auto& t : lanes) t.join();
}

}  // namespace ebhost
