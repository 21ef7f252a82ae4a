// Light tables of a scene as element steps (reference: Scene::Scene src/scene.cpp:156-253, compute_area_cdf :38-61):
//
//   lt_triangle_area     area of one emissive triangle, in double
//   lt_sum_and_scan      the in-order sum of one light's triangle areas and the exclusive scan of them divided by that sum (the
//                        light's area CDF); serial in triangle order, like thrust::reduce / exclusive_scan on the CPP backend
//   lt_light_weight      luminance-weighted selection weight of an area light
//   lt_env_weight        selection weight of the environment map, the LAST entry of the light PMF
//   lt_normalize         the PMF divided by its in-order total, and the CDF
//   lt_bsphere_radius    radius of the scene's bounding sphere from the X and Y extent of all vertices (the reference folds each
//                        shape's Y extent into the Z bounds, src/scene.cpp:156-195, so Z never enters)
//
// The functions are RB_HD: host_build_lights (rb_scene_host.hpp) runs them in serial loops; rb_light_build.cu runs the areas in parallel,
// a warp per light for the sum and scan (the additions of lt_sum_and_scan in the same order, loads and divisions spread over the lanes),
// and one thread for the PMF / CDF.  Both must give the same doubles, so rb_light_build.cu is compiled without FMA contraction and with
// IEEE division / square root (build.py); tests/test_scene_update_cpu.py compares the decomposition below with host_build_lights byte for
// byte, tests/test_scene_update_gpu.py the device tables with a NumPy float64 restatement.
#pragma once
#include "rb_types.cuh"

RB_HD double lt_triangle_area(const float* V, const int* id) {
    double v[3][3];
    for (int k = 0; k < 3; k++)
        for (int c = 0; c < 3; c++) v[k][c] = V[3 * (size_t)id[k] + c];
    double e1[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]};
    double e2[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
    double cx = e1[1] * e2[2] - e1[2] * e2[1], cy = e1[2] * e2[0] - e1[0] * e2[2], cz = e1[0] * e2[1] - e1[1] * e2[0];
    return 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
}
// Returns the light's area; cdf[t] = (sum of a[0 .. t)) / area.
RB_HD double lt_sum_and_scan(const double* a, int T, double* cdf) {
    double sum = 0;
    for (int t = 0; t < T; t++) sum += a[t];
    double run = 0;
    for (int t = 0; t < T; t++) {
        cdf[t] = run / sum;
        run += a[t];
    }
    return sum;
}
RB_HD double lt_light_weight(const DevLight& light, double area) {
    double lum = 0.212671f * (double)light.intensity[0] + 0.715160f * (double)light.intensity[1] + 0.072169f * (double)light.intensity[2];
    return area * lum * double(M_PI);
}
RB_HD double lt_env_weight(double bsphere_radius, double pdf_norm) {
    double area = 4 * double(M_PI) * bsphere_radius * bsphere_radius;
    return area > 0 ? area / pdf_norm : 1.0;
}
// false: the total importance is not positive (src/scene.cpp:243)
RB_HD bool lt_normalize(double* pmf, double* cdf, int n) {
    double total = 0;
    for (int l = 0; l < n; l++) total += pmf[l];
    if (!(total > 0)) return false;
    for (int l = 0; l < n; l++) pmf[l] /= total;
    cdf[0] = 0;
    for (int l = 1; l < n; l++) cdf[l] = cdf[l - 1] + pmf[l - 1];
    return true;
}
// lo / hi: minimum and maximum X and Y over every vertex of every shape
RB_HD double lt_bsphere_radius(const float lo[2], const float hi[2]) {
    float dx = hi[0] - lo[0], dy = hi[1] - lo[1];
    return 0.5f * sqrtf(dx * dx + dy * dy + dy * dy);
}

// ---- the decomposition rb_light_build.cu launches
struct LTScene {
    const rb_shape* shapes;  // pointers valid in the calling address space
    const DevLight* lights;
    const int* offsets;      // [L + 1]: first entry of every light in the area-CDF pool, then the pool size
    int L;
};
// one thread per pool entry: the area of that emissive triangle
RB_HD double lt_pool_area(const LTScene& S, int i) {
    int lo = 0, hi = S.L; // the last light l with offsets[l] <= i (lights without triangles are skipped)
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (S.offsets[mid] <= i) lo = mid;
        else hi = mid;
    }
    const rb_shape& sh = S.shapes[S.lights[lo].shape_id];
    return lt_triangle_area(sh.vertices, sh.indices + 3 * (size_t)(i - S.offsets[lo]));
}
// per light: area and area CDF from the triangle areas `a` (pool layout).  k_lt_scan performs the same additions and divisions in the
// same order with a warp per light.
RB_HD double lt_light_scan(const LTScene& S, int l, const double* a, double* pool) {
    const int o = S.offsets[l];
    return lt_sum_and_scan(a + o, S.offsets[l + 1] - o, pool + o);
}

// ---- emission sampling (rb_area_light::emission_sampling, DESIGN.md "Emission sampling")
//
//   ls_cell_weight       weight of one bilinear cell of the emission texture's level 0: the mean of |luminance| of its four taps
//   ls_sat_row / _col    the periodic summed-area table of the cell weights: prefix sums along each row (left to right), then down each column
//   ls_prefix            mass of the cells [0, X) x [0, Y) of the periodic continuation, for any integers X, Y (negative ones included)
//   ls_tri_corners       a triangle's uv corners in continuous cell coordinates X = u sx w - 0.5, Y = v sy h - 0.5
//   ls_tri_record        per triangle: its cell rectangle R_t, mass M_t, weight a_t and (until ls_scan) |T_t| / (M_t area_t)
//   ls_scan              per light: S = sum of a_t in triangle order, the exclusive CDF of a_t / S and the pdf factor
//                        P_t |T_t| / (M_t area_t)
// Like the area tables, host_build_light_sampling (rb_scene_host.hpp) runs them in serial loops and rb_light_build.cu as kernels, with
// the same additions in the same order, so that both give the same doubles.
#define RB_LS_DELTA 0.125     // share of the area branch in the mixture
#define RB_LS_MAX_CELLS 16777216.0 // 2^24: bound on |X|, |Y| of every scaled triangle corner (rb_scene_create refuses more): cell indices and
                                   // cell counts stay exact integers in double
#define RB_LS_TRI 8           // doubles per triangle record: x0, y0, x1, y1, M_t, a_t, CDF_t, pdf factor
RB_HD double ls_luminance(const float* texels, int channels, size_t i) {
    const float* p = texels + (size_t)channels * i;
    if (channels == 1) return (double)p[0];
    return 0.212671f * (double)p[0] + 0.715160f * (double)p[1] + 0.072169f * (double)p[2];
}
RB_HD double ls_cell_weight(const float* texels, int channels, int w, int h, int i, int j) {
    const int i1 = i + 1 < w ? i + 1 : 0, j1 = j + 1 < h ? j + 1 : 0;
    double s = fabs(ls_luminance(texels, channels, (size_t)j * w + i));
    s += fabs(ls_luminance(texels, channels, (size_t)j * w + i1));
    s += fabs(ls_luminance(texels, channels, (size_t)j1 * w + i));
    s += fabs(ls_luminance(texels, channels, (size_t)j1 * w + i1));
    return 0.25 * s;
}
RB_HD void ls_sat_row(const double* cells, double* sat, int w, int j) {
    double run = 0;
    for (int i = 0; i < w; i++) {
        run += cells[(size_t)j * w + i];
        sat[(size_t)j * w + i] = run;
    }
}
RB_HD void ls_sat_col(double* sat, int w, int h, int i) {
    for (int j = 1; j < h; j++) sat[(size_t)j * w + i] += sat[(size_t)(j - 1) * w + i];
}
RB_HD long long ls_floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
// sum of the cells [0, a) x [0, b) of one period, 0 <= a <= w, 0 <= b <= h
RB_HD double ls_sat_at(const double* sat, int w, long long a, long long b) { return a > 0 && b > 0 ? sat[(size_t)(b - 1) * w + (a - 1)] : 0.0; }
RB_HD double ls_prefix(const double* sat, int w, int h, long long X, long long Y) {
    const long long qx = ls_floor_div(X, w), qy = ls_floor_div(Y, h), rx = X - qx * w, ry = Y - qy * h;
    const double tot = ls_sat_at(sat, w, w, h);
    return (double)qx * (double)qy * tot + (double)qx * ls_sat_at(sat, w, w, ry) + (double)qy * ls_sat_at(sat, w, rx, h) + ls_sat_at(sat, w, rx, ry);
}
// Mass of [x0, x1) x [y0, y1), the rectangle first moved by whole periods so that (x0, y0) lies in [0, w) x [0, h): the prefixes then hold a
// few periods' mass at most, whatever the rectangle's distance from the origin.
RB_HD double ls_rect_mass(const double* sat, int w, int h, long long x0, long long y0, long long x1, long long y1) {
    const long long bx = ls_floor_div(x0, w) * w, by = ls_floor_div(y0, h) * h;
    x0 -= bx;
    x1 -= bx;
    y0 -= by;
    y1 -= by;
    return (ls_prefix(sat, w, h, x1, y1) - ls_prefix(sat, w, h, x0, y1)) - (ls_prefix(sat, w, h, x1, y0) - ls_prefix(sat, w, h, x0, y0));
}
// The corners of triangle t in cell coordinates (uvs as tri_attribs supplies them: the shape's, or (0, 0), (1, 0), (1, 1) without).
RB_HD void ls_tri_corners(const rb_shape& s, int t, double sx, double sy, int w, int h, double X[3], double Y[3]) {
    for (int k = 0; k < 3; k++) {
        const int vi = s.indices[3 * (size_t)t + k];
        const int ui = s.uv_indices ? s.uv_indices[3 * (size_t)t + k] : vi;
        double u, v;
        if (s.uvs) {
            u = s.uvs[2 * (size_t)ui];
            v = s.uvs[2 * (size_t)ui + 1];
        } else {
            u = k == 0 ? 0.0 : 1.0;
            v = k == 2 ? 1.0 : 0.0;
        }
        X[k] = u * sx * w - 0.5;
        Y[k] = v * sy * h - 0.5;
    }
}
// rec[0..7] of triangle t; returns false when a corner is not finite or reaches RB_LS_MAX_CELLS.
RB_HD bool ls_tri_record(const rb_shape& s, int t, double sx, double sy, int w, int h, const double* sat, double* rec) {
    double X[3], Y[3];
    ls_tri_corners(s, t, sx, sy, w, h, X, Y);
    for (int k = 0; k < 8; k++) rec[k] = 0;
    for (int k = 0; k < 3; k++)
        if (!(fabs(X[k]) < RB_LS_MAX_CELLS && fabs(Y[k]) < RB_LS_MAX_CELLS)) return false;
    const double lx = fmin(X[0], fmin(X[1], X[2])), hx = fmax(X[0], fmax(X[1], X[2]));
    const double ly = fmin(Y[0], fmin(Y[1], Y[2])), hy = fmax(Y[0], fmax(Y[1], Y[2]));
    const long long x0 = (long long)floor(lx), y0 = (long long)floor(ly), x1 = (long long)floor(hx) + 1, y1 = (long long)floor(hy) + 1;
    rec[0] = (double)x0;
    rec[1] = (double)y0;
    rec[2] = (double)x1;
    rec[3] = (double)y1;
    double M = ls_rect_mass(sat, w, h, x0, y0, x1, y1);
    if (!(M > 0)) M = 0;
    const double T = 0.5 * fabs((X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0]));
    const double area = lt_triangle_area(s.vertices, s.indices + 3 * (size_t)t);
    rec[4] = M;
    if (T > 0 && M > 0 && area > 0) {
        rec[5] = area * (M / ((double)(x1 - x0) * (double)(y1 - y0)));
        rec[7] = T / (M * area);
    }
    return true;
}
// Per light, over its T triangle records: returns S; CDF_t = (a_0 + ... + a_{t-1}) / S and the pdf factor (a_t / S) |T_t| / (M_t area_t)
// (all 0 when S is 0).  k_ls_scan performs the same additions and divisions in the same order with a warp.
RB_HD double ls_scan(double* recs, int T) {
    double sum = 0;
    for (int t = 0; t < T; t++) sum += recs[RB_LS_TRI * (size_t)t + 5];
    double run = 0;
    for (int t = 0; t < T; t++) {
        double* r = recs + RB_LS_TRI * (size_t)t;
        r[6] = sum > 0 ? run / sum : 0.0;
        r[7] = sum > 0 ? (r[5] / sum) * r[7] : 0.0;
        run += r[5];
    }
    return sum;
}
// The light's selection area: S of its texture branch, or its area when that branch is off.
RB_HD double ls_selection_area(double area, double S) { return S > 0 ? S : area; }
// Offsets of a light's data (in doubles): { S, 0 }, cells, SAT, triangle records.
RB_HD size_t ls_cells(int w, int h) { (void)w; (void)h; return 2; }
RB_HD size_t ls_sat(int w, int h) { return 2 + (size_t)w * h; }
RB_HD size_t ls_tris(int w, int h) { return 2 + 2 * (size_t)w * h; }
RB_HD size_t ls_size(int w, int h, int T) { return ls_tris(w, h) + RB_LS_TRI * (size_t)T; }
