// Triangle BVH traversal (own structure; replaces Embree rtcIntersect1/rtcOccluded1 and OptiX Prime queries,
// reference call sites src/scene.cpp:503-597 (closest hit) and :629-690 (any hit)).
//
// Layout: binary LBVH, 64-byte nodes holding BOTH children's boxes (one 4x16 B fetch per step, served by L1/L2 --
// every BASELINE scene's BVH is < 2 MB and L2-resident).  Leaves reference one pre-gathered triangle (48 B,
// three float4 loads) stored in Morton order, so neighbouring rays touch neighbouring memory.
// Each thread walks its own ray with a short stack in local memory; rays of a warp are coherent by construction
// (lanes of a warp are samples of the same / adjacent pixels, see rb_render.cuh).
//
// The triangle test is a Pluecker edge-function test evaluated in fp32 with the same operation nesting as
// Embree 3.6's robust-mode intersector (edge tests U, V, W with fused multiply-adds, inclusive zero), because
// parity with the reference means agreeing with Embree's hit/miss decisions on silhouette pixels
// (including its one-ulp edge tolerance).
#pragma once
#include "rb_types.cuh"


RB_D float rb_msub(float a, float b, float c) { return fmaf(a, b, -c); }
struct F3 {
    float x, y, z;
};
RB_D F3 f3(float x, float y, float z) { F3 r; r.x = x; r.y = y; r.z = z; return r; }
RB_D F3 f3_sub(F3 a, F3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
RB_D F3 f3_add(F3 a, F3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
RB_D F3 f3_cross(F3 a, F3 b) { return f3(rb_msub(a.y, b.z, a.z * b.y), rb_msub(a.z, b.x, a.x * b.z), rb_msub(a.x, b.y, a.y * b.x)); }
RB_D float f3_dot(F3 a, F3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }

// Returns true and the hit distance if the ray hits the triangle within (tnear, tfar].
RB_D bool tri_test(F3 O, F3 D, float tnear, float tfar, const BVHTri& tri, float& t_out) {
    F3 v0 = f3_sub(f3(tri.v0.x, tri.v0.y, tri.v0.z), O);
    F3 v1 = f3_sub(f3(tri.v1.x, tri.v1.y, tri.v1.z), O);
    F3 v2 = f3_sub(f3(tri.v2.x, tri.v2.y, tri.v2.z), O);
    F3 e0 = f3_sub(v2, v0), e1 = f3_sub(v0, v1), e2 = f3_sub(v1, v2);
    float U = f3_dot(f3_cross(f3_add(v2, v0), e0), D);
    float V = f3_dot(f3_cross(f3_add(v0, v1), e1), D);
    float W = f3_dot(f3_cross(f3_add(v1, v2), e2), D);
    float mn = fminf(U, fminf(V, W)), mx = fmaxf(U, fmaxf(V, W));
    // edge tolerance of one ulp of the summed edge functions, as in Embree's robust intersector (without it, 5 of
    // 16.8 M primary samples of the C2 image miss the floor edge that the reference hits)
    float eps = 1.1920929e-7f * fabsf(U + V + W);
    if (!(mn >= -eps || mx <= eps)) return false;
    F3 Ng = f3_cross(e2, e1);
    float den = 2.0f * f3_dot(Ng, D);
    if (den == 0.0f) return false;
    float T = 2.0f * f3_dot(v0, Ng);
    float absDen = fabsf(den);
    float Ts = den < 0.0f ? -T : T;
    if (!(absDen * tnear < Ts && Ts <= absDen * tfar)) return false;
    t_out = Ts / absDen;
    return true;
}

struct BoxRay {
    float nx, ny, nz;    // -org / dir
    float ix, iy, iz;    // 1 / dir
};
RB_D float safe_rcp(float d) { return 1.0f / (fabsf(d) > 1e-30f ? d : copysignf(1e-30f, d)); }

// slab test for one child box; returns entry distance or +inf when missed.  One FMA per plane: (b - o) / d == b * (1/d) - o * (1/d).
RB_D float box_test(const BoxRay& r, float lox, float hix, float loy, float hiy, float loz, float hiz, float tnear, float tfar) {
    float tx0 = fmaf(lox, r.ix, r.nx), tx1 = fmaf(hix, r.ix, r.nx);
    float ty0 = fmaf(loy, r.iy, r.ny), ty1 = fmaf(hiy, r.iy, r.ny);
    float tz0 = fmaf(loz, r.iz, r.nz), tz1 = fmaf(hiz, r.iz, r.nz);
    float t0 = fmaxf(fmaxf(fminf(tx0, tx1), fminf(ty0, ty1)), fmaxf(fminf(tz0, tz1), tnear));
    float t1 = fminf(fminf(fmaxf(tx0, tx1), fmaxf(ty0, ty1)), fminf(fmaxf(tz0, tz1), tfar));
    // boxes are padded at build time; the extra relative slack covers the rounding of the slab products
    return (t0 <= t1 * 1.0000004f) ? t0 : INFINITY;
}

struct BvhHit { // returned in registers
    int shape_id, tri_id;
    float t;
    int hit;
};
// Out of line on purpose: the traversal is instantiated at ~8 call sites of the backward kernel; as a real function with a
// register-only interface (no references into the caller's frame) it is shared by all of them, which keeps the kernel
// closer to the instruction caches (L0 6 KB / L1.5 32 KB per SM).
// One loop with "inner node or leaf" per iteration.  With ONE triangle per leaf a leaf test costs about as much as an inner step,
// so "while-while" (Aila & Laine 2009: descend to a leaf, then test) was no faster and has been removed.
template <bool ANY_HIT>
RB_DFN BvhHit bvh_trace_impl(const float4* __restrict__ nodes4, const float4* __restrict__ tris4, int root, int num_tris, float ox, float oy,
                             float oz, float dx, float dy, float dz, float tnear, float tfar) {
    BvhHit res;
    res.shape_id = -1;
    res.tri_id = -1;
    res.t = tfar;
    res.hit = 0;
    F3 O = f3(ox, oy, oz);
    F3 D = f3(dx, dy, dz);
    if (num_tris <= 0) return res;
    // zero / degenerate directions never hit (src/scene.cpp:577-578)
    if (D.x * D.x + D.y * D.y + D.z * D.z <= 1e-3f) return res;
    if (!(tfar >= tnear)) return res;
    BoxRay br;
    br.ix = safe_rcp(D.x); br.iy = safe_rcp(D.y); br.iz = safe_rcp(D.z);
    br.nx = -O.x * br.ix; br.ny = -O.y * br.iy; br.nz = -O.z * br.iz;
    int stack[RB_BVH_STACK];
    int sp = 0;
    int node = root;
    while (true) {
        if (node >= 0) {
            float4 bx = __ldg(nodes4 + 4 * (size_t)node + 0);
            float4 by = __ldg(nodes4 + 4 * (size_t)node + 1);
            float4 bz = __ldg(nodes4 + 4 * (size_t)node + 2);
            float4 ch = __ldg(nodes4 + 4 * (size_t)node + 3);
            int left = __float_as_int(ch.x), right = __float_as_int(ch.y);
            float tl = box_test(br, bx.x, bx.y, by.x, by.y, bz.x, bz.y, tnear, tfar);
            float tr = box_test(br, bx.z, bx.w, by.z, by.w, bz.z, bz.w, tnear, tfar);
            bool hl = tl < INFINITY, hr = tr < INFINITY;
            if (hl && hr) {
                int first = left, second = right;
                if (tr < tl) { first = right; second = left; }
                if (sp < RB_BVH_STACK) stack[sp++] = second;
                node = first;
                continue;
            } else if (hl) {
                node = left;
                continue;
            } else if (hr) {
                node = right;
                continue;
            }
        } else {
            int slot = ~node;
            BVHTri tri;
            tri.v0 = __ldg(tris4 + 3 * (size_t)slot + 0);
            tri.v1 = __ldg(tris4 + 3 * (size_t)slot + 1);
            tri.v2 = __ldg(tris4 + 3 * (size_t)slot + 2);
            float t;
            if (tri_test(O, D, tnear, tfar, tri, t)) {
                res.hit = 1;
                tfar = t;
                res.shape_id = __float_as_int(tri.v0.w);
                res.tri_id = __float_as_int(tri.v1.w);
                if (ANY_HIT) break;
            }
        }
        if (sp == 0) break;
        node = stack[--sp];
    }
    res.t = tfar;
    return res;
}
// The exact answer the traversal must give (test hook rb_scene_trace_rays): tri_test on every triangle in leaf order, with the
// early-outs of bvh_trace_impl.  Closest hit: a triangle replaces the best hit only with a strictly smaller t, so of exactly tied
// triangles the first in leaf order wins.  Any hit: the first triangle hit in leaf order.
template <bool ANY_HIT>
RB_D BvhHit bvh_brute_force(const float4* __restrict__ tris4, int num_tris, float ox, float oy, float oz, float dx, float dy, float dz,
                            float tnear, float tfar) {
    BvhHit res;
    res.shape_id = -1;
    res.tri_id = -1;
    res.t = tfar;
    res.hit = 0;
    F3 O = f3(ox, oy, oz);
    F3 D = f3(dx, dy, dz);
    if (num_tris <= 0) return res;
    if (D.x * D.x + D.y * D.y + D.z * D.z <= 1e-3f) return res;
    if (!(tfar >= tnear)) return res;
    for (int slot = 0; slot < num_tris; slot++) {
        BVHTri tri;
        tri.v0 = __ldg(tris4 + 3 * (size_t)slot + 0);
        tri.v1 = __ldg(tris4 + 3 * (size_t)slot + 1);
        tri.v2 = __ldg(tris4 + 3 * (size_t)slot + 2);
        float t;
        if (tri_test(O, D, tnear, tfar, tri, t) && (!res.hit || t < res.t)) {
            res.hit = 1;
            res.t = t;
            res.shape_id = __float_as_int(tri.v0.w);
            res.tri_id = __float_as_int(tri.v1.w);
            if (ANY_HIT) break;
        }
    }
    return res;
}

template <bool ANY_HIT>
RB_D bool bvh_trace(const DevScene& sc, const Ray& ray, int& shape_id, int& tri_id, float& t_hit) {
    BvhHit h = bvh_trace_impl<ANY_HIT>(reinterpret_cast<const float4*>(sc.bvh_nodes), reinterpret_cast<const float4*>(sc.bvh_tris), sc.bvh_root,
                                       sc.num_tris, (float)ray.org.x, (float)ray.org.y, (float)ray.org.z, (float)ray.dir.x, (float)ray.dir.y,
                                       (float)ray.dir.z, (float)ray.tmin, (float)ray.tmax);
    shape_id = h.shape_id;
    tri_id = h.tri_id;
    t_hit = h.t;
    return h.hit != 0;
}
