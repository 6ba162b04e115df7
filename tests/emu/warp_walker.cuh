// TEST INFRASTRUCTURE ONLY — lock-step warp emulation of a generated walker, for the host emulation (emu.cpp).
//
// The generated walkers emit the items of top-level lists/maps item-parallel across the warp (jit.cpp items_par): warp
// shuffles, votes and scans, and an item-position table filled by the count walk.  emu.cpp walks one lane at a time, so
// this header wraps the generated walker (EMU_LANE_WALKER) into the `rv::gen::Walker` that emu.cpp drives
// (EMU_GEN_WALKER = this file): the count walks and the precise emit pass straight through, and the FAST emit of a warp
// is deferred until its 32nd lane has been handed in, then runs the 32 lanes as coroutines that meet at every warp
// collective (dev_core.cuh HostWarpEmu).  A collective reached by only part of the warp aborts.
#pragma once
#include <ucontext.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "dev_core.cuh"

#define gen gen_lanes
#include EMU_LANE_WALKER
#undef gen

namespace rv {
namespace warp_emu {
namespace {  // one emulation state per library: each is built for one schema

constexpr size_t kLaneStack = 256 * 1024;

struct State {
    HostWarpEmu hook;
    std::vector<uint8_t> items;
    std::vector<char> stacks;
    ucontext_t sched;
    ucontext_t lane_ctx[32];
    uint32_t vals[32], snap[32];
    bool done[32];
    int pending = 0;                 // lanes of the current warp handed in so far
    WalkCtx<true> ctx[32];
    gen_lanes::Cur q[32];
    int n_nodes = 0;
    long long collectives = 0;       // warp collectives met by whole warps
};

inline State& state();

inline const uint32_t* exchange(uint32_t lane, uint32_t v) {
    State& s = state();
    s.vals[lane] = v;
    swapcontext(&s.lane_ctx[lane], &s.sched);
    return s.snap;
}

inline State& state() {
    static State* s = [] {
        State* n = new State;
        n->items.assign(gen_lanes::Walker::kItemBytes + 1, uint8_t(0xA5));  // (the device table is not cleared either)
        n->stacks.resize(32 * kLaneStack);
        n->hook.items = n->items.data();
        n->hook.exchange = exchange;
        host_warp_emu() = &n->hook;  // from the first walk on: the count walks fill the item-position table
        return n;
    }();
    return *s;
}

inline void lane_entry(int lane) {
    State& s = state();
    gen_lanes::Walker::walk<WM_EMIT>(s.ctx[lane], s.n_nodes, s.q[lane]);
    s.done[lane] = true;
}

inline void run_warp() {
    State& s = state();
    for (int l = 0; l < 32; ++l) {
        s.done[l] = false;
        getcontext(&s.lane_ctx[l]);
        s.lane_ctx[l].uc_stack.ss_sp = s.stacks.data() + size_t(l) * kLaneStack;
        s.lane_ctx[l].uc_stack.ss_size = kLaneStack;
        s.lane_ctx[l].uc_link = &s.sched;
        makecontext(&s.lane_ctx[l], reinterpret_cast<void (*)()>(lane_entry), 1, l);
    }
    for (;;) {
        for (int l = 0; l < 32; ++l)
            if (!s.done[l]) swapcontext(&s.sched, &s.lane_ctx[l]);  // lane l runs to its next collective or its end
        int n_done = 0;
        for (int l = 0; l < 32; ++l) n_done += s.done[l];
        if (n_done == 32) break;
        if (n_done) { std::fprintf(stderr, "emu: warp collective reached by %d of 32 lanes\n", 32 - n_done); std::abort(); }
        std::memcpy(s.snap, s.vals, sizeof s.snap);
        ++s.collectives;
    }
}

}  // namespace
}  // namespace warp_emu

namespace gen {
using Cur = gen_lanes::Cur;
struct Walker {
    static constexpr bool kRegCursors = gen_lanes::Walker::kRegCursors;
    static constexpr int kStreams = gen_lanes::Walker::kStreams;
    static constexpr uint32_t kItemBytes = gen_lanes::Walker::kItemBytes;
    using Cur = gen_lanes::Cur;
    template <int MODE, class C>
    static void walk(C& c, int n_nodes, Cur& q) {
        warp_emu::State& s = warp_emu::state();
        if constexpr (MODE == WM_EMIT && C::kShared) {
            const int lane = int(c.row0 % 32u);
            if (lane != s.pending) { std::fprintf(stderr, "emu: lane %d of a warp handed in out of order\n", lane); std::abort(); }
            s.ctx[lane] = c;
            s.q[lane] = q;
            s.n_nodes = n_nodes;
            if (++s.pending == 32) {
                s.pending = 0;
                warp_emu::run_warp();
            }
        } else {
            gen_lanes::Walker::walk<MODE>(c, n_nodes, q);
        }
    }
    template <class C>
    static void zero_offsets(C& c, int tid) { gen_lanes::Walker::zero_offsets(c, tid); }
};
}  // namespace gen

}  // namespace rv

// Warp collectives run so far by this library (a test's proof that the item-parallel emit was taken).
extern "C" long long emu_warp_collectives() { return rv::warp_emu::state().collectives; }
