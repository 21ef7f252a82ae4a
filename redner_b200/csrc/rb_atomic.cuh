// Gradient scatter: warp-aggregated atomics.
// The reference issues one global atomic per scalar per thread (src/atomic.h:41-57; call sites e.g.
// src/primary_intersection.cpp:41-65, src/path_contribution.cpp:287-292).  Neighbouring paths of a warp mostly hit
// the same triangle / material / light, so we first combine the lanes that target the same address
// (__match_any_sync on the address) with a log-depth shuffle tree and let one lane per group issue the
// red.global.add.f32.  For a warp whose 32 lanes share the target this is 32x fewer atomics.
#pragma once
#include "rb_exact.cuh"
#include "rb_math.cuh"

#ifdef RB_CPU_EMU
// host-compiled debug emulator (tools/cpu_emu): single "lane", plain adds.  In deterministic mode its rb_render points this at the
// exact accumulators of the virtual gradient addresses (rb_exact.cuh), and every scatter goes there.  One pointer for the process:
// deterministic renders of the emulator must not run concurrently (the emulator is a single-threaded debug aid).
static long long* rb_emu_exact_acc = nullptr;
RB_D void rb_red_add(float* addr, float v) {
    if (rb_emu_exact_acc == nullptr) *addr += v;
    else if (v != 0.f) exact_add_serial(exact_slot(rb_emu_exact_acc, addr), v);
}
RB_D void warp_agg_add3(float* addr, float x, float y, float z) { rb_red_add(addr, x); rb_red_add(addr + 1, y); rb_red_add(addr + 2, z); }
#elif defined(RB_DETERMINISTIC)
// Deterministic scatter (rb_kernels_det.cu): every contribution goes into the exact accumulator of its element.  rb_render sets
// this to the accumulator array before the backward kernels run; the gradient buffers the kernels see are virtual addresses into it.
__device__ long long* rb_exact_acc;
// Add one float to the exact accumulator `acc` (global or shared memory).  The lanes of the convergence group that target the same
// (accumulator, limb) first add their integer chunks with the pointer-doubling scheme of the default scatter below, and the group
// leader issues one 64-bit integer reduction per limb.  Integer sums are exact, so the grouping cannot change the result.  A zero
// contributes nothing and is not written.  Must stay inline, like warp_agg_add3 below.
RB_D void exact_agg_add(long long* acc, float v) {
    const ExactTerm t = exact_term(v);
    if (t.flag) atomicOr((unsigned long long*)(acc + RB_EXACT_LIMBS), (unsigned long long)t.flag);
    long long lo = t.lo, hi = t.hi;
    const unsigned long long key = (lo | hi) != 0 ? (unsigned long long)(acc + t.limb) : 0ull;
    unsigned active = __activemask();
    unsigned peers = __match_any_sync(active, key);
    int lane = threadIdx.x & 31;
    unsigned above = peers & (0xfffffffeu << lane);
    int nxt = above ? __ffs(above) - 1 : -1;
    int n = __popc(peers);
#pragma unroll 1
    for (int span = 1; span < n; span <<= 1) {
        int src = nxt >= 0 ? nxt : lane;
        long long olo = __shfl_sync(peers, lo, src), ohi = __shfl_sync(peers, hi, src);
        int nn = __shfl_sync(peers, nxt, src);
        if (nxt >= 0) {
            lo += olo;
            hi += ohi;
            nxt = nn;
        }
    }
    if (key != 0ull && lane == __ffs(peers) - 1) {
        unsigned long long* limb = (unsigned long long*)(acc + t.limb);
        if (lo != 0) atomicAdd(limb, (unsigned long long)lo); // two's complement: the unsigned add is the signed one
        if (hi != 0) atomicAdd(limb + 1, (unsigned long long)hi);
    }
}
RB_D void rb_red_add(float* addr, float v) { exact_agg_add(exact_slot(rb_exact_acc, addr), v); }
// (a zero component is skipped inside exact_agg_add, so the accumulator of an unused component is never touched)
RB_D void warp_agg_add3(float* addr, float x, float y, float z) {
    long long* acc = exact_slot(rb_exact_acc, addr);
    exact_agg_add(acc, x);
    exact_agg_add(acc + RB_EXACT_WORDS, y);
    exact_agg_add(acc + 2 * RB_EXACT_WORDS, z);
}
#else
RB_D void rb_red_add(float* addr, float v) { atomicAdd(addr, v); } // result unused -> RED.E.ADD.F32 (fire and forget)
// (A per-block shared-memory cache in front of the REDs was tried and measured 1.4x - 4.6x SLOWER on the backward kernel:
//  the 64-bit CAS + shared atomic per scalar costs more than a fire-and-forget L2 reduction; see DESIGN.md.)

// Combine up to three consecutive floats across the lanes of the current convergence group that target the same `addr`;
// the group leader issues the reductions.  Must stay INLINE: inside a real function the callers' lanes are not
// reconverged, __activemask() degenerates to single lanes and every lane issues its own atomics.
// The peers of one address form a linked list in lane order; pointer doubling turns every lane's value into the
// suffix sum of its list in ceil(log2 n) rounds, so the lowest lane ends with the group total.  One code path for
// every group shape and no __fns(): a rank-based tree made this helper a large share of the backward kernel's SASS, and the kernel
// instruction-fetch bound.
RB_D void warp_agg_add3(float* addr, float x, float y, float z) {
    unsigned active = __activemask();
    unsigned peers = __match_any_sync(active, (unsigned long long)addr);
    int lane = threadIdx.x & 31;
    unsigned above = peers & (0xfffffffeu << lane);
    int nxt = above ? __ffs(above) - 1 : -1;
    int n = __popc(peers);
#pragma unroll 1
    for (int span = 1; span < n; span <<= 1) {
        int src = nxt >= 0 ? nxt : lane;
        float ox = __shfl_sync(peers, x, src), oy = __shfl_sync(peers, y, src), oz = __shfl_sync(peers, z, src);
        int nn = __shfl_sync(peers, nxt, src);
        if (nxt >= 0) {
            x += ox;
            y += oy;
            z += oz;
            nxt = nn;
        }
    }
    if (lane == __ffs(peers) - 1) {
        if (x != 0.f) rb_red_add(addr, x);
        if (y != 0.f) rb_red_add(addr + 1, y);
        if (z != 0.f) rb_red_add(addr + 2, z);
    }
}
#endif // RB_CPU_EMU
// NOTE: a zero component is never written, so the 1- and 2-component variants may pass 0 for the unused lanes of the
// triple without touching memory beyond their target.
RB_D void agg_add3(float* addr, V3 v) { warp_agg_add3(addr, (float)v.x, (float)v.y, (float)v.z); }
RB_D void agg_add2(float* addr, V2 v) { warp_agg_add3(addr, (float)v.x, (float)v.y, 0.f); }
RB_D void agg_add1(float* addr, Real v) { warp_agg_add3(addr, (float)v, 0.f, 0.f); }
