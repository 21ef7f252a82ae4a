// Per-path device code: light sampling, per-vertex radiance estimate (NEE + BSDF sampling with power-2 MIS),
// the bounce loop, and the hand-derived adjoint of one path vertex.
//   light_point_sampler             src/scene.cpp:692-741
//   primary_contribs_accumulator    src/primary_contribution.cpp:6-35  (radiance channel)
//   path_contribs_accumulator       src/path_contribution.cpp:5-154
//   d_path_contribs_accumulator     src/path_contribution.cpp:156-592
//   bounce loop                     src/pathtracer.cpp:292-390
// One thread carries one path from the camera (or from an edge ray) to its end; nothing but the final pixel /
// gradient contributions leaves the SM.
#pragma once
#include "rb_bvh.cuh"
#include "rb_camera.cuh"
#include "rb_envmap.cuh"
#include "rb_material.cuh"
#include "rb_sampler.cuh"
#include "rb_shape.cuh"

// upper_bound on an ascending double table: number of entries <= x (thrust::upper_bound, src/scene.cpp:698)
RB_D int cdf_pick(const double* cdf, int n, double x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (cdf[mid] <= x) lo = mid + 1; else hi = mid;
    }
    return rb_clampi(lo - 1, 0, n - 1);
}

struct LightSampleRec {
    Isect isect;      // (light shape, triangle); environment map: shape_id = -1 and tri_id = bits of dir.z
    V2 uv;            // the 2-D sample used on the triangle; environment map: (dir.x, dir.y) of the sampled direction
    bool unoccluded;  // shadow ray reached the light (nee_ray.tmax >= 0)
#if RB_LIGHT_TEX_KERNELS
    bool rejected;    // emission sampling placed the point outside the triangle: no light sample at all (unoccluded is false too)
#endif
};
// The environment-map sample keeps its world direction in the record (the adjoint pass needs exactly the direction the
// primal pass used; re-sampling from rounded random numbers would not give it).
RB_HD void light_rec_set_env_dir(LightSampleRec& r, V3 dir) {
    r.isect.shape_id = -1;
    float z = (float)dir.z;
    memcpy(&r.isect.tri_id, &z, sizeof(int));
    r.uv = mk2(dir.x, dir.y);
}
RB_HD V3 light_rec_env_dir(const LightSampleRec& r) {
    float z;
    memcpy(&z, &r.isect.tri_id, sizeof(float));
    return mk3(r.uv.x, r.uv.y, (Real)z);
}

RB_D bool closest_hit(const DevScene& sc, const Ray& ray, Isect& is) {
    float t;
    return bvh_trace<false>(sc, ray, is.shape_id, is.tri_id, t);
}
RB_D bool any_hit(const DevScene& sc, const Ray& ray) {
    int s, tr;
    float t;
    return bvh_trace<true>(sc, ray, s, tr, t);
}

// Hit point in double precision.  The reference keeps rays and hit points in double and only rounds the rays it hands to
// Embree (src/scene.cpp:556-567); a shadow ray that starts at an fp32 hit point differs from the reference's in the last
// bit and resolves differently when it grazes a blocker edge (measured: 4 of 16.8 M samples at 512x512x64 == 1.6e-4
// relative L2).  Carrying the hit point (only) in double makes the rounded shadow / bounce rays identical again.
RB_D D3 hit_point_d(const rb_shape& s, int tri, D3 o, D3 d) {
    int idx[3];
    shape_tri(s, tri, idx);
    const float *p0 = s.vertices + 3 * (size_t)idx[0], *p1 = s.vertices + 3 * (size_t)idx[1], *p2 = s.vertices + 3 * (size_t)idx[2];
    double e1x = (double)p1[0] - p0[0], e1y = (double)p1[1] - p0[1], e1z = (double)p1[2] - p0[2];
    double e2x = (double)p2[0] - p0[0], e2y = (double)p2[1] - p0[1], e2z = (double)p2[2] - p0[2];
    double pvx = d.y * e2z - d.z * e2y, pvy = d.z * e2x - d.x * e2z, pvz = d.x * e2y - d.y * e2x;
    double div = pvx * e1x + pvy * e1y + pvz * e1z;
    if (fabs(div) < 1e-8) div = div > 0 ? 1e-8 : -1e-8;
    double sx = o.x - p0[0], sy = o.y - p0[1], sz = o.z - p0[2];
    double qx = sy * e1z - sz * e1y, qy = sz * e1x - sx * e1z, qz = sx * e1y - sy * e1x;
    double t = (e2x * qx + e2y * qy + e2z * qz) / div;
    return d3(o.x + d.x * t, o.y + d.y * t, o.z + d.z * t);
}

// ---- emission sampling (rb_area_light::emission_sampling, DESIGN.md "Emission sampling")
#if RB_LIGHT_TEX_KERNELS
#include "rb_light_build.cuh"
#endif
// The tables of light l's texture branch, or null when the light samples by area (always null where RB_LIGHT_TEX cannot hold).
RB_HD const LightSampling* light_sampling(const DevScene& sc, int l) {
#if RB_LIGHT_TEX_KERNELS
    const LightSampling* t = light_sampling_table(sc);
    if (t == nullptr || t[l].data == nullptr || !(t[l].data[0] > 0)) return nullptr;
    return t + l;
#else
    (void)sc;
    (void)l;
    return nullptr;
#endif
}
#if RB_LIGHT_TEX_KERNELS // (the kernel sets without emission textures compile none of it: their code stays what it was)
// THE density of light l's point sampler (per unit area, without the light's selection probability) at the point of triangle `tri`
// whose texture coordinate, before uv_scale, is `uv`: delta / A_l + (1 - delta) P_t (w_c / M_t) |T_t| / area_t, with c the cell at uv
// clamped into the triangle's rectangle R_t.  Every estimator that weighs a point of such a light calls it, from the point alone.
RB_HD double light_point_density(const DevScene& sc, const LightSampling& s, int l, int tri, V2 uv) {
    const rb_texture& et = light_emission(sc, l);
    const double* r = s.data + ls_tris(s.w, s.h) + RB_LS_TRI * (size_t)tri;
    const double X = (double)uv.x * (double)et.uv_scale[0] * s.w - 0.5, Y = (double)uv.y * (double)et.uv_scale[1] * s.h - 0.5;
    const long long ix = (long long)fmin(fmax(floor(X), r[0]), r[2] - 1), iy = (long long)fmin(fmax(floor(Y), r[1]), r[3] - 1);
    const long long cx = ix - ls_floor_div(ix, s.w) * s.w, cy = iy - ls_floor_div(iy, s.h) * s.h;
    const double wc = s.data[ls_cells(s.w, s.h) + (size_t)cy * s.w + (size_t)cx];
    return RB_LS_DELTA / sc.light_areas[l] + (1 - RB_LS_DELTA) * r[7] * wc;
}
// The texture branch: triangle by the CDF of a_t at u1, then a row of R_t by sv and a column within it by su from the summed-area table,
// each continuous inside its cell, and the barycentrics (b1, b2) of that point in the triangle's cell-space corners.  False: rejected (the
// point lies outside the triangle, or a degenerate table row).
RB_HD bool ls_sample_tex(const LightSampling& s, const rb_texture& et, const rb_shape& shape, double u1, double su, double sv, int& tri, double& b1,
                         double& b2) {
    const int T = shape.num_triangles, w = s.w, h = s.h;
    const double *recs = s.data + ls_tris(w, h), *sat = s.data + ls_sat(w, h);
    int lo = 0, hi = T; // (upper_bound, as cdf_pick)
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (recs[RB_LS_TRI * (size_t)mid + 6] <= u1) lo = mid + 1;
        else hi = mid;
    }
    tri = rb_clampi(lo - 1, 0, T - 1);
    const double* r = recs + RB_LS_TRI * (size_t)tri;
    if (!(r[5] > 0)) return false;
    // (in R_t moved by whole periods so that its corner lies in the first period, as ls_rect_mass does: small prefixes)
    const long long bx = ls_floor_div((long long)r[0], w) * w, by = ls_floor_div((long long)r[1], h) * h;
    const long long x0 = (long long)r[0] - bx, y0 = (long long)r[1] - by, x1 = (long long)r[2] - bx, y1 = (long long)r[3] - by;
    // rows: the mass of [x0, x1) x [y0, y) is strip(y) - strip(y0)
    auto strip = [&](long long y) { return ls_prefix(sat, w, h, x1, y) - ls_prefix(sat, w, h, x0, y); };
    const double rbase = strip(y0), ty = sv * (strip(y1) - rbase);
    long long a = y0, b = y1;
    while (b - a > 1) {
        const long long mid = a + (b - a) / 2;
        if (strip(mid) - rbase <= ty) a = mid;
        else b = mid;
    }
    const long long j = a;
    const double r0 = strip(j) - rbase, r1 = strip(j + 1) - rbase;
    if (!(r1 > r0)) return false;
    // columns of row j: the mass of [x0, x) x [j, j + 1) is col(x) - col(x0)
    auto col = [&](long long x) { return ls_prefix(sat, w, h, x, j + 1) - ls_prefix(sat, w, h, x, j); };
    const double cbase = col(x0), tx = su * (col(x1) - cbase);
    a = x0;
    b = x1;
    while (b - a > 1) {
        const long long mid = a + (b - a) / 2;
        if (col(mid) - cbase <= tx) a = mid;
        else b = mid;
    }
    const long long i = a;
    const double c0 = col(i) - cbase, c1 = col(i + 1) - cbase;
    if (!(c1 > c0)) return false;
    const double X = (double)(i + bx) + fmin(fmax((tx - c0) / (c1 - c0), 0.0), 1.0), Y = (double)(j + by) + fmin(fmax((ty - r0) / (r1 - r0), 0.0), 1.0);
    double CX[3], CY[3];
    ls_tri_corners(shape, tri, et.uv_scale[0], et.uv_scale[1], w, h, CX, CY);
    const double e1x = CX[1] - CX[0], e1y = CY[1] - CY[0], e2x = CX[2] - CX[0], e2y = CY[2] - CY[0], dx = X - CX[0], dy = Y - CY[0];
    const double det = e1x * e2y - e1y * e2x;
    b1 = (dx * e2y - dy * e2x) / det;
    b2 = (e1x * dy - e1y * dx) / det;
    return b1 >= 0 && b2 >= 0 && b1 + b2 <= 1;
}
// A point on area light l: the triangle and the barycentrics (b1, b2) the shadow ray is built from, the equivalent uniform sample
// (su', sv') = ((1 - b1)^2, b2 / (1 - b1)) that the record keeps (sample_light_triangle and light_sample_uv reproduce the point from it),
// the branch (0: by area, 1: by texture) and whether the texture branch rejected the point.  A light without emission sampling takes
// today's uniform map of (su, sv).
struct LightPoint {
    int tri, branch;
    bool rejected;
    double b1, b2, su, sv;
};
RB_D LightPoint sample_light_point(const DevScene& sc, int l, double tri_sel, double su, double sv) {
    const rb_shape& shape = sc.shapes[sc.lights[l].shape_id];
    const double* acdf = sc.area_cdf_pool + sc.area_cdf_offset[l];
    const LightSampling* s = light_sampling(sc, l);
    LightPoint p;
    p.branch = 0;
    p.rejected = false;
    if (s == nullptr || tri_sel < RB_LS_DELTA) {
        p.tri = cdf_pick(acdf, shape.num_triangles, s ? tri_sel / RB_LS_DELTA : tri_sel);
        double a = sqrt(su);
        p.b1 = 1.0 - a;
        p.b2 = a * sv;
        p.su = su;
        p.sv = sv;
        return p;
    }
    p.branch = 1;
    p.rejected = !ls_sample_tex(*s, light_emission(sc, l), shape, (tri_sel - RB_LS_DELTA) / (1 - RB_LS_DELTA), su, sv, p.tri, p.b1, p.b2);
    if (p.rejected) {
        p.b1 = p.b2 = p.su = p.sv = 0;
        return p;
    }
    const double a = 1 - p.b1;
    p.su = a * a;
    p.sv = a > 0 ? p.b2 / a : 0.0;
    return p;
}
// light_point_density for any area light: 1 / A_l for a light that samples by area.
RB_HD double light_point_pdf(const DevScene& sc, int l, int tri, V2 uv) {
    const LightSampling* s = light_sampling(sc, l);
    return s ? light_point_density(sc, *s, l, tri, uv) : 1.0 / sc.light_areas[l];
}
// Test hook rb_light_sample_test, sample i: { branch, triangle, rejected } and { b1, b2, density } of the record sample_light would keep
// (b1, b2 as sample_light_triangle reproduces them from it); query k: the density at { triangle, u, v } (NaN for a triangle out of range).
RB_D void light_sample_test_one(const DevScene& sc, int l, const double* samples, int n, int* ints, double* doubles, const float* queries, int m,
                                 double* query_pdfs, long long i) {
    const rb_shape& shape = sc.shapes[sc.lights[l].shape_id];
    if (i < n) {
        const double* q = samples + 3 * i;
        const LightPoint p = sample_light_point(sc, l, q[0], q[1], q[2]);
        ints[3 * i] = p.branch;
        ints[3 * i + 1] = p.tri;
        ints[3 * i + 2] = p.rejected ? 1 : 0;
        double* o = doubles + 3 * i;
        o[0] = o[1] = o[2] = 0;
        if (!p.rejected) {
            const V2 rec = mk2((Real)p.su, (Real)p.sv);
            const Real a = sqrt(rec.x);
            o[0] = 1 - a;
            o[1] = a * rec.y;
            o[2] = light_point_pdf(sc, l, p.tri, light_sample_uv(shape, p.tri, rec));
        }
    }
    if (i < m) {
        const float* q = queries + 3 * i;
        const int tri = (int)q[0];
        query_pdfs[i] = tri >= 0 && tri < shape.num_triangles ? light_point_pdf(sc, l, tri, mk2(q[1], q[2])) : NAN;
    }
}
// Whether the shadow ray from the double hit point `p_d` to the point (b1, b2) of triangle `tri` reaches it (built in double, then
// rounded once -- src/scene.cpp:692-741; sample_light's uniform path spells the same steps out, so that the kernels without emission
// textures compile to the code they had).
RB_D bool light_point_unoccluded(const DevScene& sc, const rb_shape& shape, int tri, double b1, double b2, D3 p_d) {
    int idx[3];
    shape_tri(shape, tri, idx);
    const float *p0 = shape.vertices + 3 * (size_t)idx[0], *p1 = shape.vertices + 3 * (size_t)idx[1], *p2 = shape.vertices + 3 * (size_t)idx[2];
    double lx = p0[0] + ((double)p1[0] - p0[0]) * b1 + ((double)p2[0] - p0[0]) * b2;
    double ly = p0[1] + ((double)p1[1] - p0[1]) * b1 + ((double)p2[1] - p0[1]) * b2;
    double lz = p0[2] + ((double)p1[2] - p0[2]) * b1 + ((double)p2[2] - p0[2]) * b2;
    double dx = lx - p_d.x, dy = ly - p_d.y, dz = lz - p_d.z;
    double len = sqrt(dx * dx + dy * dy + dz * dz);
    Ray sh;
    sh.org = mk3((Real)p_d.x, (Real)p_d.y, (Real)p_d.z);
    sh.dir = len > 0 ? mk3((Real)(dx / len), (Real)(dy / len), (Real)(dz / len)) : zero3();
    sh.tmin = Real(1e-3);
    sh.tmax = (Real)((1 - 1e-3f) * len);
    return !any_hit(sc, sh);
}
#endif

// Pick a light, a triangle on it and a point on the triangle; trace the shadow ray (built in double from the double hit
// point `p_d`, then rounded once -- src/scene.cpp:692-741).
RB_D void sample_light(const DevScene& sc, D3 p_d, double light_sel, double tri_sel, double su, double sv, LightSampleRec& rec, SurfacePoint& lp) {
    int light_id = cdf_pick(sc.light_cdf, sc.num_lights, light_sel);
#if RB_LIGHT_TEX_KERNELS
    rec.rejected = false;
#endif
    if (RB_ENVMAP(sc) && light_id == sc.num_lights - 1) {
        // environment map: direction by importance sampling, shadow ray to infinity (src/scene.cpp:703-711)
        V3 dir = envmap_sample(sc.env, su, sv);
        light_rec_set_env_dir(rec, dir);
        lp = zero_point();
        Ray sh;
        sh.org = mk3((Real)p_d.x, (Real)p_d.y, (Real)p_d.z);
        sh.dir = dir;
        sh.tmin = Real(1e-3);
        sh.tmax = INFINITY;
        rec.unoccluded = !any_hit(sc, sh);
        return;
    }
    const DevLight& light = sc.lights[light_id];
    const rb_shape& shape = sc.shapes[light.shape_id];
#if RB_LIGHT_TEX_KERNELS
    if (light_sampling(sc, light_id) != nullptr) { // emission sampling: the point from sample_light_point, the record from its equivalent sample
        const LightPoint q = sample_light_point(sc, light_id, tri_sel, su, sv);
        rec.isect.shape_id = light.shape_id;
        rec.isect.tri_id = q.tri;
        rec.uv = mk2((Real)q.su, (Real)q.sv);
        if (q.rejected) {
            rec.rejected = true;
            rec.unoccluded = false;
            lp = zero_point();
            return;
        }
        lp = sample_light_triangle(shape, q.tri, rec.uv);
        rec.unoccluded = light_point_unoccluded(sc, shape, q.tri, q.b1, q.b2, p_d);
        return;
    }
#endif
    const double* acdf = sc.area_cdf_pool + sc.area_cdf_offset[light_id];
    int tri = cdf_pick(acdf, shape.num_triangles, tri_sel);
    rec.isect.shape_id = light.shape_id;
    rec.isect.tri_id = tri;
    rec.uv = mk2((Real)su, (Real)sv);
    lp = sample_light_triangle(shape, tri, rec.uv);
    int idx[3];
    shape_tri(shape, tri, idx);
    const float *p0 = shape.vertices + 3 * (size_t)idx[0], *p1 = shape.vertices + 3 * (size_t)idx[1], *p2 = shape.vertices + 3 * (size_t)idx[2];
    double a = sqrt(su), b1 = 1.0 - a, b2 = a * sv;
    double lx = p0[0] + ((double)p1[0] - p0[0]) * b1 + ((double)p2[0] - p0[0]) * b2;
    double ly = p0[1] + ((double)p1[1] - p0[1]) * b1 + ((double)p2[1] - p0[1]) * b2;
    double lz = p0[2] + ((double)p1[2] - p0[2]) * b1 + ((double)p2[2] - p0[2]) * b2;
    double dx = lx - p_d.x, dy = ly - p_d.y, dz = lz - p_d.z;
    double len = sqrt(dx * dx + dy * dy + dz * dz);
    Ray sh;
    sh.org = mk3((Real)p_d.x, (Real)p_d.y, (Real)p_d.z);
    sh.dir = len > 0 ? mk3((Real)(dx / len), (Real)(dy / len), (Real)(dz / len)) : zero3();
    sh.tmin = Real(1e-3);
    sh.tmax = (Real)((1 - 1e-3f) * len);
    rec.unoccluded = !any_hit(sc, sh);
}

// Adjoint of light_sample_uv (rb_shape.cuh): d(uv) into the light's uv gradient buffer `d_uvs` (for a shape with uvs).
RB_D void d_light_sample_uv(const rb_shape& s, int tri, V2 sample, V2 d_uv, float* d_uvs) {
    TriAttribs a;
    tri_attribs(s, tri, a);
    Real r = sqrt(sample.x);
    Real b1 = 1 - r, b2 = r * sample.y;
    agg_add2(d_uvs + 2 * (size_t)a.uv_ind[0], d_uv * (1 - (b1 + b2)));
    agg_add2(d_uvs + 2 * (size_t)a.uv_ind[1], d_uv * b1);
    agg_add2(d_uvs + 2 * (size_t)a.uv_ind[2], d_uv * b2);
}
// Emission texture of area light `l` (RB_LIGHT_TEX) at texture coordinate uv with footprint (du_dxy, dv_dxy), broadcast to RGB from one
// channel: the factor E(uv) of Le = intensity * E(uv).
RB_D V3 light_tex_eval(const rb_texture& t, V2 uv, V2 du_dxy, V2 dv_dxy) { return tex_eval(t, t.channels, uv, du_dxy, dv_dxy); }
// Adjoint of that lookup for d(loss)/d(E) `d_E`: scatters into the light's gradient texture, and returns d(uv) (d(du_dxy) and d(dv_dxy)
// are added to the two references).  Nothing when the backward pass has no gradient texture for the light.
RB_D V2 d_light_tex_eval(const DevScene& sc, const DevDScene& ds, int l, V2 uv, V2 du_dxy, V2 dv_dxy, V3 d_E, V2& d_du_dxy, V2& d_dv_dxy) {
    const rb_texture& t = light_emission(sc, l);
    const rb_texture& dt = light_d_emission(sc, ds, l);
    if (dt.num_levels <= 0) return zero2();
    const Real d0 = t.channels == 1 ? sum(d_E) : d_E.x; // (one channel is read three times)
    if (tex_is_constant(t)) {
        if (t.channels == 3) agg_add3(dt.texels[0], d_E);
        else agg_add1(dt.texels[0], d0);
        return zero2();
    }
    TexAdjoint r = d_tex_eval_mip(t, dt, t.channels, uv, du_dxy, dv_dxy, d0, d_E.y, d_E.z);
    d_du_dxy += r.d_du_dxy;
    d_dv_dxy += r.d_dv_dxy;
    return r.d_uv;
}

// Emission seen along a primary / edge ray (radiance channel of accumulate_primary_contribs).  An emission texture is looked up with the
// footprint the material textures use at the hit.
RB_D V3 hit_emission(const DevScene& sc, const Isect& is, const SurfacePoint& sp, V3 wi) {
    if (!is.valid()) return zero3();
    const rb_shape& shape = sc.shapes[is.shape_id];
    if (shape.light_id >= 0) {
        const DevLight& light = sc.lights[shape.light_id];
        if (light.directly_visible && (light.two_sided || dot(wi, sp.shading_frame.n) > 0)) {
            const rb_texture& et = light_emission(sc, shape.light_id);
            if (RB_LIGHT_TEX(et)) return mk3(light.intensity[0], light.intensity[1], light.intensity[2]) * light_tex_eval(et, sp.uv, sp.du_dxy, sp.dv_dxy);
            return mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
        }
    }
    return zero3();
}

// Radiance of the environment map seen along a ray that left the scene (src/primary_contribution.cpp:25-29).
RB_D V3 miss_emission(const DevScene& sc, V3 dir, const RayDiff& rd) {
    if (!RB_ENVMAP(sc) || !sc.env.directly_visible) return zero3();
    return envmap_eval(sc.env, dir, rd);
}

RB_D Real mis_power2(Real p_other, Real p_this) {
    double r = (double)p_other / (double)p_this;
    return (Real)(1.0 / (1.0 + r * r));
}

// Radiance estimate at one vertex: returns nee + scatter (not yet multiplied by the throughput) and the
// throughput factor for the next vertex.
RB_D V3 vertex_estimate(const DevScene& sc, const rb_material& mat, const SurfacePoint& sp, const MatTex& tx, V3 wi, Real min_rough, const LightSampleRec& ls,
                        const SurfacePoint& lp, const Isect& bis, const SurfacePoint& bp, V3 bdir, V3& scatter_factor, bool& scatter_ok) {
    // Both estimators exist for two kinds of light (area light / environment map).  Each first settles the direction and
    // what the light contributes along it, then ONE bsdf_eval / bsdf_pdf pair serves either kind (the BSDF with its texture
    // lookups is the bulk of this function's code).
    V3 nee = zero3();
    if (ls.unoccluded) {
        V3 wo = zero3(), Le = zero3();
        Real pdf_nee = 0, G = 1;
        bool on = false;
        if (ls.isect.valid()) { // area light, src/path_contribution.cpp:28-49
            const rb_shape& lshape = sc.shapes[ls.isect.shape_id];
            V3 dir = lp.position - sp.position;
            Real dist_sq = length_sq(dir);
            wo = dir / sqrt(dist_sq);
            if (dist_sq > Real(1e-20) && lshape.light_id >= 0) {
                const DevLight& light = sc.lights[lshape.light_id];
                if (light.two_sided || dot(-wo, lp.shading_frame.n) > 0) {
                    G = fabs(dot(wo, lp.geom_normal)) / dist_sq;
#if !RB_LIGHT_TEX_KERNELS
                    pdf_nee = (Real)(sc.light_pmf[lshape.light_id] / sc.light_areas[lshape.light_id]);
#endif
                    Le = mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
                    // (an emission texture: at the sample's uv, unfiltered like the environment map's lookups)
                    const rb_texture& et = light_emission(sc, lshape.light_id);
#if RB_LIGHT_TEX_KERNELS
                    const LightSampling* lsm = light_sampling(sc, lshape.light_id);
                    if (RB_LIGHT_TEX(et)) {
                        const V2 luv = light_sample_uv(lshape, ls.isect.tri_id, ls.uv);
                        Le = Le * light_tex_eval(et, luv, zero2(), zero2());
                        if (lsm) pdf_nee = (Real)(sc.light_pmf[lshape.light_id] * light_point_density(sc, *lsm, lshape.light_id, ls.isect.tri_id, luv));
                    }
                    if (!lsm) pdf_nee = (Real)(sc.light_pmf[lshape.light_id] / sc.light_areas[lshape.light_id]);
#else
                    if (RB_LIGHT_TEX(et)) Le = Le * light_tex_eval(et, light_sample_uv(lshape, ls.isect.tri_id, ls.uv), zero2(), zero2());
#endif
                    on = true;
                }
            }
        } else if (RB_ENVMAP(sc)) { // environment light (:51-67); the lookup is unfiltered (zero ray differential)
            wo = light_rec_env_dir(ls);
            pdf_nee = envmap_pdf(sc.env, wo) * (Real)sc.light_pmf[sc.num_lights - 1];
            if (pdf_nee > 0) {
                Le = envmap_eval(sc.env, wo, zero_raydiff());
                on = true;
            }
        }
        if (on) {
            V3 f = bsdf_eval(mat, sp, tx, wi, wo, min_rough);
            Real pdf_b = bsdf_pdf(mat, sp, tx, wi, wo, min_rough) * G;
            nee = (mis_power2(pdf_b, pdf_nee) * G / pdf_nee) * f * Le;
        }
    }
    V3 scatter = zero3();
    scatter_factor = zero3();
    scatter_ok = false;
    const bool hit = bis.valid();
    if (hit || RB_ENVMAP(sc)) {
        V3 wo = bdir;
        Real dist_sq = 1;
        if (hit) {
            V3 dir = bp.position - sp.position;
            dist_sq = length_sq(dir);
            wo = dir / sqrt(dist_sq);
        }
        Real pdf_b = bsdf_pdf(mat, sp, tx, wi, wo, min_rough);
        // (hit: src/path_contribution.cpp:71-98; miss: :99-118 -- bdir is zero when the BSDF sample failed)
        if ((hit ? dist_sq > Real(1e-20) : length_sq(wo) > 0) && pdf_b > Real(1e-20)) {
            V3 f = bsdf_eval(mat, sp, tx, wi, wo, min_rough);
            if (hit) {
                const rb_shape& bshape = sc.shapes[bis.shape_id];
                if (bshape.light_id >= 0) {
                    const DevLight& light = sc.lights[bshape.light_id];
                    if (light.two_sided || dot(-wo, bp.shading_frame.n) > 0) {
                        Real G = fabs(dot(wo, bp.geom_normal)) / dist_sq;
#if RB_LIGHT_TEX_KERNELS
                        const LightSampling* lsm = light_sampling(sc, bshape.light_id);
                        Real pdf_nee = (Real)(lsm ? sc.light_pmf[bshape.light_id] * light_point_density(sc, *lsm, bshape.light_id, bis.tri_id, bp.uv)
                                                  : sc.light_pmf[bshape.light_id] * (1.0 / sc.light_areas[bshape.light_id])) / G;
#else
                        Real pdf_nee = (Real)(sc.light_pmf[bshape.light_id] * (1.0 / sc.light_areas[bshape.light_id])) / G;
#endif
                        V3 Le = mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
                        const rb_texture& et = light_emission(sc, bshape.light_id);
                        if (RB_LIGHT_TEX(et)) Le = Le * light_tex_eval(et, bp.uv, zero2(), zero2());
                        scatter = (mis_power2(pdf_nee, pdf_b) / pdf_b) * f * Le;
                    }
                }
                scatter_factor = f / pdf_b;
                scatter_ok = true;
            } else {
                V3 Le = envmap_eval(sc.env, wo, zero_raydiff());
                Real pdf_nee = envmap_pdf(sc.env, wo) * (Real)sc.light_pmf[sc.num_lights - 1];
                scatter = (mis_power2(pdf_nee, pdf_b) / pdf_b) * f * Le;
            }
        }
    }
    return nee + scatter;
}

// What the adjoint pass needs to know about path vertex d (everything else is recomputed).  16-byte aligned so that
// the records move through HBM / L2 as 128-bit loads and stores (a quarter of the memory instructions).
struct alignas(16) VertexRec {
    Ray ray;       // ray that reached the vertex
    RayDiff rd_in; // its differential before the hit
    Isect isect;
    V3 thr;
    Real min_rough;
    LightSampleRec light;
};

// Follows a path from an already intersected vertex through at most (max_bounces - depth_begin) bounces and
// returns the sum of throughput-weighted vertex estimates.  `smp` must be positioned at the light-sample
// dimension of depth `depth_begin`.  If REC, vertices are written to rec[depth - depth_begin] and *num_rec is
// the number of vertices at which an estimate was formed.
template <bool REC>
RB_D V3 trace_bounces(const DevScene& sc, Sampler& smp, Ray ray, RayDiff rd_in, Isect is, V3 thr, Real min_rough, int depth_begin,
                      int max_bounces, VertexRec* rec, int rec_stride, int* num_rec, const D3* ray_org_d = nullptr, const D3* ray_dir_d = nullptr) {
    V3 L = zero3();
    int count = 0;
    // double-precision copy of the current ray (exact for camera rays, promoted fp32 otherwise)
    D3 od = ray_org_d ? *ray_org_d : d3(ray.org.x, ray.org.y, ray.org.z);
    D3 dd = ray_dir_d ? *ray_dir_d : d3(ray.dir.x, ray.dir.y, ray.dir.z);
    if (sc.num_lights > 0) {
        for (int depth = depth_begin; depth < max_bounces && is.valid(); depth++) {
            RayDiff rd;
            SurfacePoint sp = make_surface_point(sc.shapes[is.shape_id], is.tri_id, ray, rd_in, rd);
            const rb_material& mat = sc.materials[sc.shapes[is.shape_id].material_id];
            V3 wi = -ray.dir;
            double l_sel = smp.next(), t_sel = smp.next(), lu = smp.next(), lv = smp.next();
            LightSampleRec ls;
            SurfacePoint lp;
            D3 p_d = hit_point_d(sc.shapes[is.shape_id], is.tri_id, od, dd);
            sample_light(sc, p_d, l_sel, t_sel, lu, lv, ls, lp);
            double bu = smp.next(), bv = smp.next(), bw = smp.next();
            if (REC) {
                VertexRec& r = rec[(size_t)count * rec_stride];
                r.ray = ray;
                r.rd_in = rd_in;
                r.isect = is;
                r.thr = thr;
                r.min_rough = min_rough;
                r.light = ls;
            }
            RayDiff rd_b;
            Real next_rough;
            const MatTex tx = mat_textures(mat, sp);
            V3 dir = bsdf_sample_dir(mat, sp, tx, wi, mk2((Real)bu, (Real)bv), bw, min_rough, rd, rd_b, next_rough);
            Ray nray;
            nray.org = mk3((Real)p_d.x, (Real)p_d.y, (Real)p_d.z);
            nray.dir = dir;
            od = p_d;
            dd = d3(dir.x, dir.y, dir.z);
            nray.tmin = Real(1e-3);
            nray.tmax = INFINITY;
            Isect bis = no_isect();
            SurfacePoint bp = zero_point();
            RayDiff rd_after;
            if (closest_hit(sc, nray, bis)) bp = make_surface_point(sc.shapes[bis.shape_id], bis.tri_id, nray, rd_b, rd_after);
            V3 factor;
            bool ok;
            V3 est = vertex_estimate(sc, mat, sp, tx, wi, min_rough, ls, lp, bis, bp, dir, factor, ok);
            L += thr * est;
            count++;
            thr = ok ? thr * factor : zero3();
            ray = nray;
            rd_in = rd_b;
            is = bis;
            min_rough = next_rough;
        }
    }
    if (REC) {
        // terminal vertex: no estimate is formed there, but the adjoint of the previous vertex needs its hit
        VertexRec& r = rec[(size_t)count * rec_stride];
        r.ray = ray;
        r.rd_in = rd_in;
        r.isect = is;
        r.thr = thr;
        r.min_rough = min_rough;
        *num_rec = count;
    }
    return L;
}

// Gradient sinks for geometry: per-corner scatter with warp aggregation.
RB_D void scatter_vertex_grads(const DevScene& sc, const DevDScene& ds, const Isect& is, const V3 d_vp[3], const V3 d_vn[3], const V2 d_vuv[3],
                               const V3 d_vc[3]) {
    const rb_shape& s = sc.shapes[is.shape_id];
    const rb_dshape& d = ds.shapes[is.shape_id];
    TriAttribs a;
    tri_attribs(s, is.tri_id, a);
    for (int k = 0; k < 3; k++) {
        if (d.vertices) agg_add3(d.vertices + 3 * (size_t)a.ind[k], d_vp[k]);
        if (s.uvs && d.uvs) agg_add2(d.uvs + 2 * (size_t)a.uv_ind[k], d_vuv[k]);
        if (s.normals && d.normals) agg_add3(d.normals + 3 * (size_t)a.n_ind[k], d_vn[k]);
        if (s.colors && d.colors) agg_add3(d.colors + 3 * (size_t)a.ind[k], d_vc[k]);
    }
}

// Adjoint state flowing from vertex d+1 to vertex d.
struct VertexAdjoint {
    V3 d_thr;
    DRay d_ray;
    SurfacePoint d_point;
};
RB_D VertexAdjoint zero_vertex_adjoint() {
    VertexAdjoint a;
    a.d_thr = zero3();
    a.d_ray = zero_dray();
    a.d_point = zero_point();
    return a;
}

// Adjoint of vertex_estimate + throughput update at vertex `cur`, given the adjoint arriving from vertex `nxt`.
// d_contrib = weight * d_image[pixel] (radiance channels).
RB_D VertexAdjoint d_vertex(const DevScene& sc, const DevDScene& ds, const VertexRec& cur, const VertexRec* nxt, V3 d_contrib,
                            const VertexAdjoint& next) {
    VertexAdjoint out = zero_vertex_adjoint();
    const rb_shape& shape = sc.shapes[cur.isect.shape_id];
    const rb_material& mat = sc.materials[shape.material_id];
    const rb_material& d_mat = ds.materials[shape.material_id];
    RayDiff rd;
    SurfacePoint sp = make_surface_point(shape, cur.isect.tri_id, cur.ray, cur.rd_in, rd);
    V3 wi = -cur.ray.dir;
    V3 p = sp.position;
    V3 thr = cur.thr;
    Real min_rough = cur.min_rough;
    // The two estimators of this vertex (light sample, BSDF sample) share ONE rolled call of d_bsdf_eval: each prepares
    // (wo, d_f, d_wo) in a "pre" block and consumes the returned d_wo in a "post" block.  Besides halving the code of
    // the largest adjoint this reconverges the lanes of a warp that took only one of the two branches.
    bool on_l = false, on_b = false, env_l = false, env_b = false;
    V3 wo_l = zero3(), d_f_l = zero3(), d_wo_l = zero3(), dir_l = zero3();
    V3 wo_b = zero3(), d_f_b = zero3(), d_wo_b = zero3(), dir_b = zero3();
    Real dist_sq_l = 1, d_dist_sq_l = 0, dist_sq_b = 1, d_cos_l = 0;
    V3 d_lv[3] = {zero3(), zero3(), zero3()};
    // ---- next event estimation (pre): area light (src/path_contribution.cpp:212-293) or environment map (:295-337).
    // Direction and light-side quantities first, then ONE bsdf_eval / bsdf_pdf pair for either kind.
    if (cur.light.unoccluded) {
        const bool area = cur.light.isect.valid();
        const Isect& lis = cur.light.isect;
        SurfacePoint lp = zero_point();
        V3 wo = zero3(), dir = zero3(), Le = zero3();
        Real dist_sq = 1, pdf_nee = 0;
        bool ok = false;
#if RB_LIGHT_TEX_KERNELS
        bool tex_l = false; // an emission texture (RB_LIGHT_TEX): its value E_l at the sample's uv `luv`
        V3 E_l = zero3();
        V2 luv = zero2();
#endif
        if (area) {
            const rb_shape& lshape = sc.shapes[lis.shape_id];
            lp = sample_light_triangle(lshape, lis.tri_id, cur.light.uv);
            dir = lp.position - p;
            dist_sq = length_sq(dir);
            wo = dir / sqrt(dist_sq);
            if (lshape.light_id >= 0) {
                const DevLight& light = sc.lights[lshape.light_id];
                if (light.two_sided || dot(-wo, lp.shading_frame.n) > 0) {
                    Le = mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
#if RB_LIGHT_TEX_KERNELS
                    const rb_texture& et = light_emission(sc, lshape.light_id);
                    if (RB_LIGHT_TEX(et)) {
                        tex_l = true;
                        luv = light_sample_uv(lshape, lis.tri_id, cur.light.uv);
                        E_l = light_tex_eval(et, luv, zero2(), zero2());
                        Le = Le * E_l;
                    }
                    const LightSampling* lsm = light_sampling(sc, lshape.light_id);
                    pdf_nee = (Real)(lsm ? sc.light_pmf[lshape.light_id] * light_point_density(sc, *lsm, lshape.light_id, lis.tri_id, luv)
                                         : sc.light_pmf[lshape.light_id] * (1.0 / sc.light_areas[lshape.light_id]));
#else
                    pdf_nee = (Real)(sc.light_pmf[lshape.light_id] * (1.0 / sc.light_areas[lshape.light_id]));
#endif
                    ok = true;
                }
            }
        } else if (RB_ENVMAP(sc)) {
            wo = light_rec_env_dir(cur.light);
            pdf_nee = envmap_pdf(sc.env, wo) * (Real)sc.light_pmf[sc.num_lights - 1];
            if (pdf_nee > 0) {
                Le = envmap_eval(sc.env, wo, zero_raydiff());
                ok = true;
            }
        }
        if (ok) {
            V3 f = bsdf_eval(mat, sp, wi, wo, min_rough);
            Real pdf_b0 = bsdf_pdf(mat, sp, wi, wo, min_rough);
            V3 d_nee = d_contrib * thr;
            if (area) {
                const rb_shape& lshape = sc.shapes[lis.shape_id];
                Real cos_l = dot(wo, lp.geom_normal);
                Real G = fabs(cos_l) / dist_sq;
                Real mis = mis_power2(pdf_b0 * G, pdf_nee);
                out.d_thr += d_contrib * ((mis * G / pdf_nee) * f * Le);
                Real wgt = mis / pdf_nee;
                // derivatives of the MIS weight and of the light-selection pmf are ignored (src/path_contribution.cpp:239)
                Real d_wgt = G * sum(d_nee * f * Le);
                Real d_pdf_nee = -d_wgt * wgt / pdf_nee;
                Real d_G = wgt * sum(d_nee * f * Le);
                Real d_area = -d_pdf_nee * pdf_nee / shape_tri_area(lshape, lis.tri_id);
                d_shape_tri_area(lshape, lis.tri_id, d_area, d_lv);
#if RB_LIGHT_TEX_KERNELS
                if (tex_l) { // Le = intensity * E(uv): into the intensity, the texture and the light's uvs
                    const int lid = lshape.light_id;
                    const DevLight& light = sc.lights[lid];
                    const V3 d_Le = wgt * G * (d_nee * f);
                    agg_add3(ds.light_intensity[lid], d_Le * E_l);
                    V2 d_du = zero2(), d_dv = zero2();
                    V2 d_uv = d_light_tex_eval(sc, ds, lid, luv, zero2(), zero2(), d_Le * mk3(light.intensity[0], light.intensity[1], light.intensity[2]), d_du, d_dv);
                    const rb_dshape& dls = ds.shapes[lis.shape_id];
                    if (lshape.uvs && dls.uvs) d_light_sample_uv(lshape, lis.tri_id, cur.light.uv, d_uv, dls.uvs);
                } else {
                    agg_add3(ds.light_intensity[lshape.light_id], wgt * G * (d_nee * f));
                }
#else
                agg_add3(ds.light_intensity[lshape.light_id], wgt * G * (d_nee * f));
#endif
                d_cos_l = cos_l > 0 ? d_G / dist_sq : -d_G / dist_sq;
                dir_l = dir;
                dist_sq_l = dist_sq;
                d_dist_sq_l = -d_G * G / dist_sq;
                d_f_l = wgt * G * (d_nee * Le);
                d_wo_l = d_cos_l * lp.geom_normal;
            } else { // no dependence of the direction on the vertex position
                Real wgt = mis_power2(pdf_b0, pdf_nee) / pdf_nee;
                out.d_thr += d_contrib * (wgt * f * Le);
                RayDiff d_rd0 = zero_raydiff();
                d_envmap_eval(sc.env, wo, zero_raydiff(), wgt * (d_nee * f), ds.env_values, ds.env_w2e, d_wo_l, d_rd0);
                env_l = true;
                d_f_l = wgt * (d_nee * Le);
            }
            on_l = true;
            wo_l = wo;
        }
    }
    // ---- BSDF-sampled continuation (pre): the ray hit something (:339-518) or left the scene into the map (:520-590)
    SurfacePoint bp;
#if RB_LIGHT_TEX_KERNELS
    bool tex_b = false; // the hit is on a light with an emission texture (RB_LIGHT_TEX); d(uv) of the hit
    V2 d_buv = zero2();
#endif
    if (nxt != nullptr && (nxt->isect.valid() || RB_ENVMAP(sc))) {
        const bool hit = nxt->isect.valid();
        const Isect& bis = nxt->isect;
        V3 wo = nxt->ray.dir, dir = zero3();
        Real dist_sq = 1;
        if (hit) {
            RayDiff rd_after;
            bp = make_surface_point(sc.shapes[bis.shape_id], bis.tri_id, nxt->ray, nxt->rd_in, rd_after);
            dir = bp.position - p;
            dist_sq = length_sq(dir);
            wo = dir / sqrt(dist_sq);
        }
        Real pdf_b = bsdf_pdf(mat, sp, wi, wo, min_rough);
        if (pdf_b > 0 && (hit || length_sq(wo) > 0)) {
            V3 f = bsdf_eval(mat, sp, wi, wo, min_rough);
            V3 d_scatter = d_contrib * thr;
            if (hit) {
                const rb_shape& bshape = sc.shapes[bis.shape_id];
                out.d_thr += next.d_thr * (f / pdf_b);
                // the derivative w.r.t. pdf_bsdf is dropped on purpose (src/path_contribution.cpp:369-376)
                V3 d_f = (next.d_thr * thr) / pdf_b;
                if (bshape.light_id >= 0) {
                    const DevLight& light = sc.lights[bshape.light_id];
                    if (light.two_sided || dot(-wo, bp.shading_frame.n) > 0) {
                        Real G = fabs(dot(wo, bp.geom_normal)) / dist_sq;
                        V3 Le = mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
#if RB_LIGHT_TEX_KERNELS
                        const rb_texture& et = light_emission(sc, bshape.light_id);
                        V3 E_b = zero3();
                        if (RB_LIGHT_TEX(et)) {
                            tex_b = true;
                            E_b = light_tex_eval(et, bp.uv, zero2(), zero2());
                            Le = Le * E_b;
                        }
#endif
#if RB_LIGHT_TEX_KERNELS
                        const LightSampling* lsm = light_sampling(sc, bshape.light_id);
                        Real pdf_nee = (Real)(lsm ? sc.light_pmf[bshape.light_id] * light_point_density(sc, *lsm, bshape.light_id, bis.tri_id, bp.uv)
                                                  : sc.light_pmf[bshape.light_id] * (1.0 / sc.light_areas[bshape.light_id])) / G;
#else
                        Real pdf_nee = (Real)(sc.light_pmf[bshape.light_id] * (1.0 / sc.light_areas[bshape.light_id])) / G;
#endif
                        Real wgt = mis_power2(pdf_nee, pdf_b) / pdf_b;
                        out.d_thr += d_contrib * (wgt * f * Le);
                        d_f += wgt * (d_scatter * Le);
#if RB_LIGHT_TEX_KERNELS
                        if (tex_b) { // into the intensity and the texture; d(uv) reaches the hit's uvs and vertices through d_make_surface_point
                            const V3 d_Le = wgt * (d_scatter * f);
                            agg_add3(ds.light_intensity[bshape.light_id], d_Le * E_b);
                            V2 d_du = zero2(), d_dv = zero2();
                            d_buv = d_light_tex_eval(sc, ds, bshape.light_id, bp.uv, zero2(), zero2(),
                                                     d_Le * mk3(light.intensity[0], light.intensity[1], light.intensity[2]), d_du, d_dv);
                        } else {
                            agg_add3(ds.light_intensity[bshape.light_id], wgt * (d_scatter * f));
                        }
#else
                        agg_add3(ds.light_intensity[bshape.light_id], wgt * (d_scatter * f));
#endif
                    }
                }
                dir_b = dir;
                dist_sq_b = dist_sq;
                d_f_b = d_f;
                d_wo_b = next.d_ray.dir;
            } else { // nothing flows back into the sampling procedure
                V3 Le = envmap_eval(sc.env, wo, zero_raydiff());
                Real pdf_nee = envmap_pdf(sc.env, wo) * (Real)sc.light_pmf[sc.num_lights - 1];
                Real wgt = mis_power2(pdf_nee, pdf_b) / pdf_b;
                out.d_thr += d_contrib * (wgt * f * Le);
                RayDiff d_rd0 = zero_raydiff();
                d_envmap_eval(sc.env, wo, zero_raydiff(), wgt * (d_scatter * f), ds.env_values, ds.env_w2e, d_wo_b, d_rd0);
                env_b = true;
                d_f_b = wgt * (d_scatter * Le);
            }
            on_b = true;
            wo_b = wo;
        }
    }
    // ---- shared BSDF adjoint
#pragma unroll 1
    for (int k = 0; k < 2; k++) {
        if (!(k ? on_b : on_l)) continue;
        V3 d_wi = zero3();
        V3 d_wo = k ? d_wo_b : d_wo_l;
        d_bsdf_eval(mat, d_mat, sp, wi, k ? wo_b : wo_l, min_rough, k ? d_f_b : d_f_l, out.d_point, d_wi, d_wo);
        out.d_ray.dir -= d_wi;
        if (k) d_wo_b = d_wo; else d_wo_l = d_wo;
    }
    // ---- next event estimation (post)
    if (on_l && !env_l) {
        const Isect& lis = cur.light.isect;
        const rb_shape& lshape = sc.shapes[lis.shape_id];
        V3 d_dir = d_wo_l / sqrt(dist_sq_l);
        Real d_sqrt = -sum(d_wo_l * dir_l) / dist_sq_l;
        Real d_dist_sq = d_dist_sq_l + Real(0.5) * d_sqrt / sqrt(dist_sq_l);
        d_dir += d_length_sq(dir_l, d_dist_sq);
        SurfacePoint d_lp = zero_point();
        d_lp.geom_normal = d_cos_l * wo_l;
        d_lp.position += d_dir;
        out.d_point.position -= d_dir;
        d_sample_light_triangle(lshape, lis.tri_id, cur.light.uv, d_lp, d_lv);
        int idx[3];
        shape_tri(lshape, lis.tri_id, idx);
        float* dv = ds.shapes[lis.shape_id].vertices;
        if (dv) {
            agg_add3(dv + 3 * (size_t)idx[0], d_lv[0]);
            agg_add3(dv + 3 * (size_t)idx[1], d_lv[1]);
            agg_add3(dv + 3 * (size_t)idx[2], d_lv[2]);
        }
    }
    // ---- BSDF-sampled continuation (post)
    if (on_b && !env_b) {
        const Isect& bis = nxt->isect;
        const rb_shape& bshape = sc.shapes[bis.shape_id];
        V3 d_bvp[3] = {zero3(), zero3(), zero3()}, d_bvn[3] = {zero3(), zero3(), zero3()}, d_bvc[3] = {zero3(), zero3(), zero3()};
        V2 d_bvuv[3] = {zero2(), zero2(), zero2()};
        V3 d_dir = d_wo_b / sqrt(dist_sq_b);
        Real d_sqrt = -sum(d_wo_b * dir_b) / dist_sq_b;
        Real d_dist_sq = Real(0.5) * d_sqrt / sqrt(dist_sq_b);
        d_dir += d_length_sq(dir_b, d_dist_sq);
        SurfacePoint d_bp = next.d_point;
        d_bp.position += d_dir;
#if RB_LIGHT_TEX_KERNELS
        if (tex_b) d_bp.uv += d_buv;
#endif
        DRay d_ray = zero_dray();
        RayDiff d_rd_b = zero_raydiff();
        Ray bray;
        bray.org = sp.position;
        bray.dir = wo_b;
        bray.tmin = Real(1e-3);
        bray.tmax = INFINITY;
        d_make_surface_point(bshape, bis.tri_id, bray, nxt->rd_in, d_bp, zero_raydiff(), d_ray, d_rd_b, d_bvp, d_bvn, d_bvuv, d_bvc);
        // position gradient through the sampled direction only below glossy vertices (src/path_contribution.cpp:447-455)
        if (min_rough > Real(0.01)) {
            out.d_point.position -= d_dir;
            out.d_point.position += d_ray.org;
        }
        scatter_vertex_grads(sc, ds, bis, d_bvp, d_bvn, d_bvuv, d_bvc);
    }
    return out;
}
