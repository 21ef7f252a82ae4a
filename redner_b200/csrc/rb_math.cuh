// Small vector / matrix / frame algebra for the sm_90a path tracer, with the reverse-mode
// ("adjoint") counterpart of every primitive the hot path differentiates through.
// Semantics mirror the reference helpers so that results agree with the oracle:
//   normalize / d_normalize        src/vector.h:443-467
//   cross / d_cross                src/vector.h:486-503
//   coordinate_system (+adjoint)   src/vector.h:532-577   (Frisvad-style basis)
//   look_at_matrix (+adjoint)      src/transform.h:9-71
//   xfm_point / xfm_vector (+adj)  src/transform.h:73-179
// The working precision is `Real` (fp32 by default; compile with -DRB_REAL_DOUBLE for an
// fp64 validation build).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#ifdef RB_REAL_DOUBLE
typedef double Real;
#else
typedef float Real;
#endif

#define RB_HD __host__ __device__ __forceinline__
#define RB_D __device__ __forceinline__
// Out-of-line functions: the differentiable path tracer is far larger than the SM instruction caches (L0 6 KB / L1.5 32 KB),
// so the big building blocks are real calls that every kernel and every call site shares instead of being inlined N times.
#ifndef __CUDACC__
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
#endif
#define RB_FN inline __host__ __device__ __noinline__
#define RB_DFN inline __device__ __noinline__

// Feature tests.  rb_kernels_lean.cu compiles the same kernels a second time with RB_LEAN defined: no environment map, pinhole
// camera without lens model, channels == [radiance], 1-pixel box filter -- the configuration of nearly every optimisation loop.
// There the tests are compile-time constants and the rarely used code disappears from the instruction stream (DESIGN.md section 2).
#ifdef RB_LEAN
#define RB_ENVMAP(sc) false
#define RB_CAM_GENERAL(cam) false
#define RB_CAM_DISTORT(cam) false
#define RB_ONLY_RADIANCE(rp) true
#define RB_PIXEL_BOX(cam) true
#define RB_GGX(m) false
#define RB_CAM_LENS(cam) false
#define RB_LIGHT_TEX(t) false
#define RB_LIGHT_TEX_KERNELS 0
#else
#define RB_ENVMAP(sc) ((sc).has_envmap != 0)
#define RB_CAM_GENERAL(cam) ((cam).type != RB_CAMERA_PERSPECTIVE || (cam).has_distortion != 0)
#define RB_CAM_DISTORT(cam) ((cam).has_distortion != 0)
#define RB_ONLY_RADIANCE(rp) ((rp).only_radiance != 0)
#define RB_PIXEL_BOX(cam) ((cam).filter_type == RB_FILTER_BOX && (cam).filter_width == 1.0f)
// The GGX specular lobe (rb_material::specular_model) lives in the general and deterministic kernels only; rb_render keeps scenes that
// use it off the lean and diffuse-only sets.
#define RB_GGX(m) ((m).specular_model == RB_SPECULAR_GGX)
// The thin lens (rb_camera::lens_radius) likewise: rb_render keeps lens cameras off the lean and diffuse-only sets.
#define RB_CAM_LENS(cam) ((cam).lens_radius > 0)
// The emission texture of an area light (rb_area_light::emission, `t`) likewise: rb_render keeps scenes with one off those sets.
#define RB_LIGHT_TEX(t) ((t).num_levels > 0)
// (for the adjoint's bookkeeping, which is compiled only where RB_LIGHT_TEX can be true, so that the lean kernels stay as they were)
#define RB_LIGHT_TEX_KERNELS 1
#endif
// Material features.  rb_kernels_diffuse.cu compiles the lean kernels once more with RB_DIFFUSE defined as well: no material
// computes specular lighting, uses vertex colours or has a normal map -- the diffuse-only scenes of shape and pose optimisation.
// Only the host-known flags are folded; texel values (the specular reflectance that weights lobe selection included) are read
// and used as in every other build.
#ifdef RB_DIFFUSE
#ifndef RB_LEAN
#error "RB_DIFFUSE is a refinement of RB_LEAN"
#endif
#define RB_SPECULAR(m) false
#define RB_VERTEX_COLOR(m) false
#define RB_NORMAL_MAP(m) false
#else
#define RB_SPECULAR(m) ((m).compute_specular_lighting != 0)
#define RB_VERTEX_COLOR(m) ((m).use_vertex_color != 0)
#define RB_NORMAL_MAP(m) ((m).normal_map.num_levels > 0)
#endif

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#define RB_PI Real(3.14159265358979323846)
#define RB_INV_PI Real(0.31830988618379067154)

RB_HD Real rb_sq(Real x) { return x * x; }
// a * b + c with TWO roundings, never contracted into an FMA.  Used where the reference's un-fused double arithmetic produces
// exact values that decisions hang on: a hit point `org + t * dir` on an axis-aligned plane comes out EXACTLY on the plane for
// ~85 % of the rays when product and sum are rounded separately (t is the rounded root of that very equation), and a few ulps
// above or BELOW it with an FMA -- and `inside(box, p)` of the edge hierarchy (src/edge.cpp:1181, src/aabb.h:131-135) flips with it.
// With the contracted form the boundary terms of C2's lamp drift many standard errors off the reference; without it they agree
// within the noise (c2_all_vertices_secondary_stat in the GPU suite).
RB_HD Real rb_mul_add_unfused(Real a, Real b, Real c) {
#ifdef __CUDA_ARCH__
#ifdef RB_REAL_DOUBLE
    return __dadd_rn(__dmul_rn(a, b), c);
#else
    return __fadd_rn(__fmul_rn(a, b), c);
#endif
#else
    volatile Real p = a * b; // (host build: keep the compiler from contracting under -mfma / -ffp-contract=fast)
    return p + c;
#endif
}
RB_HD Real rb_max(Real a, Real b) { return a > b ? a : b; }
RB_HD Real rb_min(Real a, Real b) { return a < b ? a : b; }
RB_HD int rb_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
RB_HD Real rb_clamp(Real v, Real lo, Real hi) { return v < lo ? lo : (v > hi ? hi : v); }
RB_HD int rb_modulo(int a, int b) {
    int r = a % b;
    return (r < 0) ? r + b : r;
}

struct V2 {
    Real x, y;
    RB_HD Real& operator[](int i) { return (&x)[i]; }
    RB_HD const Real& operator[](int i) const { return (&x)[i]; }
};
struct V3 {
    Real x, y, z;
    RB_HD Real& operator[](int i) { return (&x)[i]; }
    RB_HD const Real& operator[](int i) const { return (&x)[i]; }
};

RB_HD V2 mk2(Real x, Real y) { V2 v; v.x = x; v.y = y; return v; }
RB_HD V3 mk3(Real x, Real y, Real z) { V3 v; v.x = x; v.y = y; v.z = z; return v; }
RB_HD V3 zero3() { return mk3(0, 0, 0); }
RB_HD V2 zero2() { return mk2(0, 0); }

RB_HD V2 operator+(V2 a, V2 b) { return mk2(a.x + b.x, a.y + b.y); }
RB_HD V2 operator-(V2 a, V2 b) { return mk2(a.x - b.x, a.y - b.y); }
RB_HD V2 operator-(V2 a) { return mk2(-a.x, -a.y); }
RB_HD V2 operator*(V2 a, Real s) { return mk2(a.x * s, a.y * s); }
RB_HD V2 operator*(Real s, V2 a) { return mk2(a.x * s, a.y * s); }
RB_HD V2 operator*(V2 a, V2 b) { return mk2(a.x * b.x, a.y * b.y); }
RB_HD V2 operator/(V2 a, Real s) { return mk2(a.x / s, a.y / s); }
RB_HD V2& operator+=(V2& a, V2 b) { a.x += b.x; a.y += b.y; return a; }
RB_HD V2& operator-=(V2& a, V2 b) { a.x -= b.x; a.y -= b.y; return a; }
RB_HD V2& operator*=(V2& a, Real s) { a.x *= s; a.y *= s; return a; }
RB_HD Real sum(V2 a) { return a.x + a.y; }
RB_HD Real dot(V2 a, V2 b) { return a.x * b.x + a.y * b.y; }
RB_HD Real length(V2 a) { return sqrt(dot(a, a)); }

RB_HD V3 operator+(V3 a, V3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
RB_HD V3 operator-(V3 a, V3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
RB_HD V3 operator-(V3 a) { return mk3(-a.x, -a.y, -a.z); }
RB_HD V3 operator*(V3 a, Real s) { return mk3(a.x * s, a.y * s, a.z * s); }
RB_HD V3 operator*(Real s, V3 a) { return mk3(a.x * s, a.y * s, a.z * s); }
RB_HD V3 operator*(V3 a, V3 b) { return mk3(a.x * b.x, a.y * b.y, a.z * b.z); }
RB_HD V3 operator/(V3 a, Real s) { return mk3(a.x / s, a.y / s, a.z / s); }
RB_HD V3 operator/(V3 a, V3 b) { return mk3(a.x / b.x, a.y / b.y, a.z / b.z); }
RB_HD V3& operator+=(V3& a, V3 b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
RB_HD V3& operator-=(V3& a, V3 b) { a.x -= b.x; a.y -= b.y; a.z -= b.z; return a; }
RB_HD V3& operator*=(V3& a, Real s) { a.x *= s; a.y *= s; a.z *= s; return a; }
RB_HD V3& operator*=(V3& a, V3 b) { a.x *= b.x; a.y *= b.y; a.z *= b.z; return a; }
RB_HD V3& operator/=(V3& a, Real s) { a.x /= s; a.y /= s; a.z /= s; return a; }
RB_HD Real sum(V3 a) { return a.x + a.y + a.z; }
RB_HD Real dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
RB_HD V3 cross(V3 a, V3 b) { return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
RB_HD Real length_sq(V3 a) { return dot(a, a); }
RB_HD Real length(V3 a) { return sqrt(dot(a, a)); }
RB_HD V3 max3(V3 a, Real s) { return mk3(rb_max(a.x, s), rb_max(a.y, s), rb_max(a.z, s)); }
RB_HD bool is_zero(V3 a) { return a.x == 0 && a.y == 0 && a.z == 0; }
RB_HD bool finite3(V3 a) { return isfinite(a.x) && isfinite(a.y) && isfinite(a.z); }
// src/vector.h:506-510
RB_HD Real luminance(V3 v) { return Real(0.212671) * v.x + Real(0.715160) * v.y + Real(0.072169) * v.z; }

// ---- adjoints of the basic primitives -------------------------------------------------
// l_sq = |v|^2
RB_HD V3 d_length_sq(V3 v, Real d_lsq) { return (2 * d_lsq) * v; }
// l = |v|
RB_HD V3 d_length(V3 v, Real d_l) {
    Real l = length(v);
    return d_length_sq(v, Real(0.5) * d_l / l);
}
RB_HD V2 d_length2(V2 v, Real d_l) {
    Real l = length(v);
    Real s = 2 * (Real(0.5) * d_l / l);
    return mk2(s * v.x, s * v.y);
}
RB_HD V3 normalize(V3 v) {
    Real l = length(v);
    if (l <= 0) return zero3();
    return v / l;
}
RB_HD V2 normalize2(V2 v) { return v / length(v); }
RB_HD V3 d_normalize(V3 v, V3 d_n) {
    Real l = length(v);
    if (l <= 0) return zero3();
    V3 n = v / l;
    V3 d_v = d_n / l;
    Real d_l = -dot(d_n, n) / l;
    d_v += d_length(v, d_l);
    return d_v;
}
// out = cross(a, b)
RB_HD void d_cross(V3 a, V3 b, V3 d_out, V3& d_a, V3& d_b) {
    d_a += cross(b, d_out);
    d_b += cross(d_out, a);
}

// Orthonormal basis from a unit normal.
RB_HD void coordinate_system(V3 n, V3& x, V3& y) {
    if (n.z < Real(-1) + Real(1e-6)) {
        x = mk3(0, -1, 0);
        y = mk3(-1, 0, 0);
    } else {
        Real a = 1 / (1 + n.z);
        Real b = -n.x * n.y * a;
        x = mk3(1 - rb_sq(n.x) * a, b, -n.x);
        y = mk3(b, 1 - rb_sq(n.y) * a, -n.y);
    }
}
RB_HD void d_coordinate_system(V3 n, V3 d_x, V3 d_y, V3& d_n) {
    if (n.z < Real(-1) + Real(1e-6)) return;
    Real a = 1 / (1 + n.z);
    // x = (1 - n.x^2 a, b, -n.x),  y = (b, 1 - n.y^2 a, -n.y),  b = -n.x n.y a
    d_n.x -= 2 * n.x * d_x.x * a;
    Real d_a = -rb_sq(n.x) * d_x.x;
    Real d_b = d_x.y;
    d_n.x -= d_x.z;
    d_b += d_y.x;
    d_n.y -= 2 * d_y.y * n.y * a;
    d_a -= d_y.y * rb_sq(n.y);
    d_n.y -= d_y.z;
    d_n.x -= d_b * n.y * a;
    d_n.y -= d_b * n.x * a;
    d_a -= d_b * n.x * n.y;
    d_n.z -= d_a * a / (1 + n.z);
}

struct Frame {
    V3 x, y, n;
    RB_HD V3& operator[](int i) { return (&x)[i]; }
    RB_HD const V3& operator[](int i) const { return (&x)[i]; }
};
RB_HD Frame mk_frame(V3 x, V3 y, V3 n) { Frame f; f.x = x; f.y = y; f.n = n; return f; }
RB_HD Frame frame_from_normal(V3 n) {
    Frame f;
    f.n = n;
    coordinate_system(n, f.x, f.y);
    return f;
}
RB_HD Frame zero_frame() { return mk_frame(zero3(), zero3(), zero3()); }
RB_HD V3 to_local(const Frame& f, V3 v) { return mk3(dot(v, f.x), dot(v, f.y), dot(v, f.n)); }
RB_HD V3 to_world(const Frame& f, V3 v) { return f.x * v.x + f.y * v.y + f.n * v.z; }
RB_HD void d_to_world(const Frame& f, V3 v, V3 d_dir, Frame& d_f, V3& d_v) {
    d_f.x += d_dir * v.x;
    d_f.y += d_dir * v.y;
    d_f.n += d_dir * v.z;
    d_v.x += dot(d_dir, f.x);
    d_v.y += dot(d_dir, f.y);
    d_v.z += dot(d_dir, f.n);
}

// Row-major matrices.
struct M3 {
    Real m[3][3];
};
struct M4 {
    Real m[4][4];
};
RB_HD M3 zero_m3() {
    M3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[i][j] = 0;
    return r;
}
RB_HD M4 zero_m4() {
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) r.m[i][j] = 0;
    return r;
}
RB_HD V3 mul(const M3& a, V3 v) {
    return mk3(a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z, a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
               a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z);
}
// v^T A
RB_HD V3 mul_t(V3 v, const M3& a) {
    return mk3(a.m[0][0] * v.x + a.m[1][0] * v.y + a.m[2][0] * v.z, a.m[0][1] * v.x + a.m[1][1] * v.y + a.m[2][1] * v.z,
               a.m[0][2] * v.x + a.m[1][2] * v.y + a.m[2][2] * v.z);
}
RB_HD void d_outer_acc(M3& d_a, V3 d_out, V3 v) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) d_a.m[i][j] += d_out[i] * v[j];
}
RB_HD M4 mul(const M4& a, const M4& b) {
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            Real s = 0;
            for (int k = 0; k < 4; k++) s += a.m[i][k] * b.m[k][j];
            r.m[i][j] = s;
        }
    return r;
}
RB_HD M4 transpose(const M4& a) {
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) r.m[i][j] = a.m[j][i];
    return r;
}
RB_HD V3 xfm_point(const M4& a, V3 p) {
    Real x = a.m[0][0] * p.x + a.m[0][1] * p.y + a.m[0][2] * p.z + a.m[0][3];
    Real y = a.m[1][0] * p.x + a.m[1][1] * p.y + a.m[1][2] * p.z + a.m[1][3];
    Real z = a.m[2][0] * p.x + a.m[2][1] * p.y + a.m[2][2] * p.z + a.m[2][3];
    Real w = a.m[3][0] * p.x + a.m[3][1] * p.y + a.m[3][2] * p.z + a.m[3][3];
    Real iw = 1 / w;
    return mk3(x * iw, y * iw, z * iw);
}
RB_HD V3 xfm_vector(const M4& a, V3 v) {
    return mk3(a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z, a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
               a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z);
}
RB_HD void d_xfm_point(const M4& a, V3 p, V3 d_out, M4& d_a, V3& d_p) {
    Real t[4];
    for (int i = 0; i < 4; i++) t[i] = a.m[i][0] * p.x + a.m[i][1] * p.y + a.m[i][2] * p.z + a.m[i][3];
    Real iw = 1 / t[3];
    Real d_t[4];
    d_t[0] = d_out.x * iw;
    d_t[1] = d_out.y * iw;
    d_t[2] = d_out.z * iw;
    Real d_iw = d_out.x * t[0] + d_out.y * t[1] + d_out.z * t[2];
    d_t[3] = -d_iw * iw * iw;
    for (int i = 0; i < 4; i++) {
        d_a.m[i][0] += d_t[i] * p.x;
        d_a.m[i][1] += d_t[i] * p.y;
        d_a.m[i][2] += d_t[i] * p.z;
        d_a.m[i][3] += d_t[i];
    }
    for (int j = 0; j < 3; j++) d_p[j] += d_t[0] * a.m[0][j] + d_t[1] * a.m[1][j] + d_t[2] * a.m[2][j] + d_t[3] * a.m[3][j];
}
RB_HD void d_xfm_vector(const M4& a, V3 v, V3 d_out, M4& d_a, V3& d_v) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) d_a.m[i][j] += d_out[i] * v[j];
    for (int j = 0; j < 3; j++) d_v[j] += d_out.x * a.m[0][j] + d_out.y * a.m[1][j] + d_out.z * a.m[2][j];
}
// Camera frame from position / look-at / up: columns (right, up', dir, pos).
RB_HD M4 look_at_matrix(V3 pos, V3 look, V3 up) {
    V3 d = normalize(look - pos);
    V3 right = normalize(cross(d, normalize(up)));
    V3 new_up = normalize(cross(right, d));
    M4 r;
    r.m[0][0] = right.x; r.m[0][1] = new_up.x; r.m[0][2] = d.x; r.m[0][3] = pos.x;
    r.m[1][0] = right.y; r.m[1][1] = new_up.y; r.m[1][2] = d.y; r.m[1][3] = pos.y;
    r.m[2][0] = right.z; r.m[2][1] = new_up.z; r.m[2][2] = d.z; r.m[2][3] = pos.z;
    r.m[3][0] = 0; r.m[3][1] = 0; r.m[3][2] = 0; r.m[3][3] = 1;
    return r;
}
RB_HD void d_look_at_matrix(V3 pos, V3 look, V3 up, const M4& d_m, V3& d_pos, V3& d_look, V3& d_up) {
    V3 look_pos = look - pos;
    V3 d = normalize(look_pos);
    V3 nup = normalize(up);
    V3 c_d_up = cross(d, nup);
    V3 right = normalize(c_d_up);
    V3 c_right_d = cross(right, d);
    V3 d_right = mk3(d_m.m[0][0], d_m.m[1][0], d_m.m[2][0]);
    V3 d_new_up = mk3(d_m.m[0][1], d_m.m[1][1], d_m.m[2][1]);
    V3 d_d = mk3(d_m.m[0][2], d_m.m[1][2], d_m.m[2][2]);
    d_pos += mk3(d_m.m[0][3], d_m.m[1][3], d_m.m[2][3]);
    V3 d_c_right_d = d_normalize(c_right_d, d_new_up);
    d_cross(right, d, d_c_right_d, d_right, d_d);
    V3 d_c_d_up = d_normalize(c_d_up, d_right);
    V3 d_nup = zero3();
    d_cross(d, nup, d_c_d_up, d_d, d_nup);
    d_up += d_normalize(up, d_nup);
    V3 d_look_pos = d_normalize(look_pos, d_d);
    d_look += d_look_pos;
    d_pos -= d_look_pos;
}
// General 4x4 inverse (host side; used once per scene for the look-at camera, src/camera.h:53).
inline __host__ M4 inverse_m4(const M4& a) {
    double inv[16], m[16];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) m[4 * i + j] = a.m[i][j];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) r.m[i][j] = (Real)(inv[4 * i + j] / det);
    return r;
}
