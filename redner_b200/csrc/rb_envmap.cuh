// Environment map: radiance lookup with ray-differential filtering, its adjoint, importance sampling and pdf.
//   envmap_eval / d_envmap_eval   src/envmap.h:63-197
//   envmap_sample                 src/envmap.h:199-250 (luminance x sin(theta) tables built by the caller, pyredner/envmap.py:36-61)
//   envmap_pdf                    src/envmap.h:252-306
// Latitude-longitude parametrisation, y up: uv = (atan2(x, -z) / 2pi, acos(y) / pi) in the map's local frame.
#pragma once
#include "rb_material.cuh"

RB_HD V3 env_xfm_vector(const float* m, V3 v) { // upper 3x3 of a row-major 4x4
    return mk3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z);
}
RB_HD Real env_safe_acos(Real x) { return x >= 1 ? Real(0) : (x <= -1 ? Real(RB_PI) : acos(x)); }
RB_HD int env_modulo(int a, int b) {
    int r = a % b;
    return r < 0 ? r + b : r;
}
struct EnvUV {
    V2 uv, du_dxy, dv_dxy;
};
// shared by eval and its adjoint: uv and the screen-space derivatives of uv
RB_HD EnvUV envmap_uv(const DevEnvmap& e, V3 local_dir, const RayDiff& rd, bool with_diff) {
    EnvUV r;
    r.uv = mk2(atan2(local_dir.x, -local_dir.z) / Real(2 * RB_PI), env_safe_acos(local_dir.y) / Real(RB_PI));
    r.du_dxy = r.dv_dxy = zero2();
    if (with_diff) {
        // (no handling of scaling in world_to_env, like the reference)
        V3 ldx = env_xfm_vector(e.w2e, rd.dir_dx), ldy = env_xfm_vector(e.w2e, rd.dir_dy);
        Real xz = rb_sq(local_dir.x) + rb_sq(local_dir.z);
        Real du_dx = local_dir.x / (Real(2 * RB_PI) * xz), du_dz = local_dir.z / (Real(2 * RB_PI) * xz);
        r.du_dxy = mk2(du_dx * ldx.x + du_dz * ldx.z, du_dx * ldy.x + du_dz * ldy.z);
        Real dv_dy = -1 / (Real(RB_PI) * sqrt(1 - rb_sq(local_dir.y)));
        r.dv_dxy = mk2(dv_dy * ldx.y, dv_dy * ldy.y);
    }
    return r;
}
// The pole rule (DESIGN.md section 4), one for both poles: the lookup is filtered only where |l.y| < 1 and l.x^2 + l.z^2 > 0.  The
// footprint's d(v) / d(l.y) = -1 / (pi sqrt(1 - l.y^2)) and d(u) / d(l.x, l.z) = (l.x, l.z) / (2 pi (l.x^2 + l.z^2)) are singular at the
// poles, and every direction within ~2.4e-4 rad of a pole rounds onto it in float32.  There the lookup is unfiltered, and the adjoint
// has neither footprint nor acos terms; the atan2 terms need xz > 0 (the reference is undefined at exactly |y| = 1).
RB_HD bool env_filtered(V3 l, Real xz) { return fabs(l.y) < 1 && xz > 0; }
RB_HD V3 envmap_eval(const DevEnvmap& e, V3 dir, const RayDiff& rd) {
    V3 local_dir = normalize(env_xfm_vector(e.w2e, dir));
    EnvUV q = envmap_uv(e, local_dir, rd, env_filtered(local_dir, rb_sq(local_dir.x) + rb_sq(local_dir.z)));
    return tex_eval(e.values, 3, q.uv, q.du_dxy, q.dv_dxy);
}
// d_values: gradient texture; d_w2e: 16 floats (row-major 4x4) accumulated with aggregated atomics
RB_D void d_envmap_eval(const DevEnvmap& e, V3 dir, const RayDiff& rd, V3 d_out, const rb_texture& d_values, float* d_w2e, V3& d_dir, RayDiff& d_rd) {
    V3 n_local = env_xfm_vector(e.w2e, dir);
    V3 l = normalize(n_local);
    Real xz = rb_sq(l.x) + rb_sq(l.z);
    const bool filtered = env_filtered(l, xz); // (the branch envmap_eval took; the reference always differentiates the filtered one, src/envmap.h:118-130)
    EnvUV q = envmap_uv(e, l, rd, filtered);
    V2 d_uv = zero2(), d_du = zero2(), d_dv = zero2();
    Real d_o[3] = {d_out.x, d_out.y, d_out.z};
    d_tex_eval(e.values, d_values, 3, q.uv, q.du_dxy, q.dv_dxy, d_o, d_uv, d_du, d_dv);
    V3 d_l = zero3();
    // adjoint of the three xfm_vector calls: d_m[i][j] += d_out[i] * v[j], d_v[j] += m[i][j] * d_out[i]
    Real dm[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    auto d_xfm = [&](V3 v, V3 d_o3, V3& d_v) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                dm[i][j] += d_o3[i] * v[j];
                d_v[j] += e.w2e[4 * i + j] * d_o3[i];
            }
    };
    if (filtered) { // the footprint terms
        V3 ldx = env_xfm_vector(e.w2e, rd.dir_dx), ldy = env_xfm_vector(e.w2e, rd.dir_dy);
        Real du_dx = l.x / (Real(2 * RB_PI) * xz), du_dz = l.z / (Real(2 * RB_PI) * xz);
        Real dv_dy = -1 / (Real(RB_PI) * sqrt(1 - rb_sq(l.y)));
        Real d_dv_dy = d_dv.x * ldx.y + d_dv.y * ldy.y;
        V3 d_ldx = mk3(0, d_dv.x * dv_dy, 0), d_ldy = mk3(0, d_dv.y * dv_dy, 0);
        d_l.y = -d_dv_dy * l.y / (Real(RB_PI) * sqrt(1 - rb_sq(l.y)) * (1 - rb_sq(l.y)));
        Real d_du_dx = d_du.x * ldx.x + d_du.y * ldy.x, d_du_dz = d_du.x * ldx.z + d_du.y * ldy.z;
        d_ldx.x += d_du.x * du_dx;
        d_ldx.z += d_du.x * du_dz;
        d_ldy.x += d_du.y * du_dx;
        d_ldy.z += d_du.y * du_dz;
        Real den = Real(2 * RB_PI) * rb_sq(xz);
        d_l.z += d_du_dz * (rb_sq(l.x) - rb_sq(l.z)) / den;
        d_l.x -= d_du_dz * l.x * l.z / den;
        d_l.x += d_du_dx * (rb_sq(l.z) - rb_sq(l.x)) / den;
        d_l.z -= d_du_dx * l.x * l.z / den;
        d_xfm(rd.dir_dx, d_ldx, d_rd.dir_dx);
        d_xfm(rd.dir_dy, d_ldy, d_rd.dir_dy);
    }
    if (xz > 0) { // the reference differentiates atan2(x, -z) with these signs (src/envmap.h:184-188)
        d_l.x += -d_uv.x * l.z / (xz * Real(2 * RB_PI));
        d_l.z += -d_uv.x * l.x / (xz * Real(2 * RB_PI));
    }
    if (fabs(l.y) < 1) d_l.y += -d_uv.y / (sqrt(1 - rb_sq(l.y)) * Real(2 * RB_PI)); // (2 pi, not pi: as in the reference, :190)
    V3 d_n_local = d_normalize(n_local, d_l);
    d_xfm(dir, d_n_local, d_dir);
    if (d_w2e != nullptr)
        for (int i = 0; i < 3; i++) agg_add3(d_w2e + 4 * i, mk3(dm[i][0], dm[i][1], dm[i][2]));
}
RB_HD double env_tent_inv_cdf(double x) { return x < 0.5 ? 1 - sqrt(2 * x) : sqrt(2 * x - 0.5f) - 1; }
// upper_bound on an ascending float table against a double sample (thrust::upper_bound, src/envmap.h:210-231)
RB_HD int env_cdf_pick(const float* cdf, int n, double x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if ((double)cdf[mid] <= x) lo = mid + 1; else hi = mid;
    }
    return rb_clampi(lo - 1, 0, n - 1);
}
RB_HD V3 envmap_sample(const DevEnvmap& e, double sx, double sy) {
    int w = e.values.width[0], h = e.values.height[0];
    int yp = env_cdf_pick(e.cdf_ys, h, sy);
    sy = yp < h - 1 ? (sy - e.cdf_ys[yp]) / ((double)e.cdf_ys[yp + 1] - e.cdf_ys[yp]) : (sy - e.cdf_ys[yp]) / (1 - (double)e.cdf_ys[yp]);
    const float* cx = e.cdf_xs + (size_t)yp * w;
    int xp = env_cdf_pick(cx, w, sx);
    sx = xp < w - 1 ? (sx - cx[xp]) / ((double)cx[xp + 1] - cx[xp]) : (sx - cx[xp]) / (1 - (double)cx[xp]);
    // importance sampling of the bilinear (tent) reconstruction
    double u = xp + env_tent_inv_cdf(sx), v = yp + env_tent_inv_cdf(sy);
    const double pi = 3.14159265358979323846;
    double phi = (2 * pi / w) * (u + 0.5f), theta = (pi / h) * (v + 0.5f);
    double sp = sin(phi), cp = cos(phi), st = sin(theta), ct = cos(theta);
    V3 local = mk3((Real)(sp * st), (Real)ct, (Real)(-cp * st));
    return env_xfm_vector(e.e2w, local);
}
RB_HD Real envmap_pdf(const DevEnvmap& e, V3 dir) {
    V3 l = env_xfm_vector(e.w2e, dir);
    V2 uv = mk2(atan2(l.x, -l.z) / Real(2 * RB_PI), env_safe_acos(l.y) / Real(RB_PI));
    int w = e.values.width[0], h = e.values.height[0];
    Real x = uv.x * w - Real(0.5), y = uv.y * h - Real(0.5);
    int xfi = env_modulo((int)floor(x), w), yfi = env_modulo((int)floor(y), h);
    int xci = env_modulo(xfi + 1, w), yci = env_modulo(yfi + 1, h);
    Real dx = x - xfi, dy = y - yfi;
    if (dx < 0) dx += w;
    if (dy < 0) dy += h;
    const float* t = e.values.texels[0];
    auto lum = [&](int yy, int xx) {
        const float* p = t + 3 * ((size_t)yy * w + xx);
        return Real(0.212671) * p[0] + Real(0.715160) * p[1] + Real(0.072169) * p[2];
    };
    Real lum_fy = lum(yfi, xfi) * (1 - dx) * (1 - dy) + lum(yfi, xci) * dx * (1 - dy);
    Real lum_cy = lum(yci, xfi) * (1 - dx) * dy + lum(yci, xci) * dx * dy;
    Real sin_theta = sqrt(rb_max(1 - rb_sq(l.y), Real(0)));
    if (sin_theta == 0) return 0;
    Real s_fy = fabs(sin(Real(RB_PI) * (yfi + Real(0.5)) / h)), s_cy = fabs(sin(Real(RB_PI) * (yci + Real(0.5)) / h));
    return e.pdf_norm * fabs(lum_fy * s_fy + lum_cy * s_cy) / sin_theta;
}
