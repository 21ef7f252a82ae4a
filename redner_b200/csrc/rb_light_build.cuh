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
