// One query of the test hook rb_surface_test (rb_surface_test.cu, and the host emulator's export): the geometry functions of rb_shape.cuh
// that the render kernels call -- tri_solve, make_surface_point and its adjoint, the light-point sampler, its uv and the triangle area with
// their adjoints -- and the gradient scatters of rb_path.cuh, on the scene's shapes.  Query i reads row i of `in` ([n, RB_SURFTEST_IN]
// doubles) and writes row i of `out` ([n, RB_SURFTEST_OUT] doubles).  The layouts are listed in include/redner_b200.h.
#pragma once
#include "rb_path.cuh"

#define RB_SURFTEST_IN 96
#define RB_SURFTEST_OUT 96

RB_HD V3 surftest_v3(const double* p) { return mk3((Real)p[0], (Real)p[1], (Real)p[2]); }
RB_HD void surftest_put(double* out, V3 v) {
    out[0] = v.x;
    out[1] = v.y;
    out[2] = v.z;
}
// SurfacePoint <-> 35 doubles: position, geom_normal, shading_frame x / y / n, dpdu, uv, du_dxy, dv_dxy, dn_dx, dn_dy, color, bary
RB_HD SurfacePoint surftest_point(const double* p) {
    SurfacePoint s;
    s.position = surftest_v3(p);
    s.geom_normal = surftest_v3(p + 3);
    s.shading_frame = mk_frame(surftest_v3(p + 6), surftest_v3(p + 9), surftest_v3(p + 12));
    s.dpdu = surftest_v3(p + 15);
    s.uv = mk2((Real)p[18], (Real)p[19]);
    s.du_dxy = mk2((Real)p[20], (Real)p[21]);
    s.dv_dxy = mk2((Real)p[22], (Real)p[23]);
    s.dn_dx = surftest_v3(p + 24);
    s.dn_dy = surftest_v3(p + 27);
    s.color = surftest_v3(p + 30);
    s.bary = mk2((Real)p[33], (Real)p[34]);
    return s;
}
RB_HD void surftest_put_point(double* o, const SurfacePoint& s) {
    const V3 v[6] = {s.position, s.geom_normal, s.shading_frame.x, s.shading_frame.y, s.shading_frame.n, s.dpdu};
    for (int k = 0; k < 6; k++) surftest_put(o + 3 * k, v[k]);
    const V2 w[3] = {s.uv, s.du_dxy, s.dv_dxy};
    for (int k = 0; k < 3; k++) {
        o[18 + 2 * k] = w[k].x;
        o[19 + 2 * k] = w[k].y;
    }
    surftest_put(o + 24, s.dn_dx);
    surftest_put(o + 27, s.dn_dy);
    surftest_put(o + 30, s.color);
    o[33] = s.bary.x;
    o[34] = s.bary.y;
}
RB_HD RayDiff surftest_rd(const double* p) {
    RayDiff r;
    r.org_dx = surftest_v3(p);
    r.org_dy = surftest_v3(p + 3);
    r.dir_dx = surftest_v3(p + 6);
    r.dir_dy = surftest_v3(p + 9);
    return r;
}
RB_HD void surftest_put_rd(double* o, const RayDiff& r) {
    surftest_put(o, r.org_dx);
    surftest_put(o + 3, r.org_dy);
    surftest_put(o + 6, r.dir_dx);
    surftest_put(o + 9, r.dir_dy);
}

// `ds`: the gradient buffers the adjoint ops scatter into, or null (DevDScene::shapes is the only member read).
RB_D void surface_test_one(const DevScene& sc, const DevDScene* ds, int op, const double* in_, int n, double* out_, long long i) {
    if (i >= n) return;
    const double* in = in_ + RB_SURFTEST_IN * i;
    double* out = out_ + RB_SURFTEST_OUT * i;
    Isect is;
    is.shape_id = (int)in[0];
    is.tri_id = (int)in[1];
    const rb_shape& s = sc.shapes[is.shape_id];
    if (op == RB_SURFTEST_POINT || op == RB_SURFTEST_D_POINT) {
        Ray ray;
        ray.org = surftest_v3(in + 2);
        ray.dir = surftest_v3(in + 5);
        ray.tmin = 0;
        ray.tmax = INFINITY;
        const RayDiff rd = surftest_rd(in + 8);
        if (op == RB_SURFTEST_POINT) {
            V3 v0, v1, v2;
            shape_tri_vertices(s, is.tri_id, v0, v1, v2);
            const TriSolve h = tri_solve(v0, v1, v2, ray, rd);
            const double hv[9] = {h.u, h.v, h.t, h.u_dxy.x, h.u_dxy.y, h.v_dxy.x, h.v_dxy.y, h.t_dxy.x, h.t_dxy.y};
            for (int k = 0; k < 9; k++) out[k] = hv[k];
            RayDiff rd_out;
            const SurfacePoint p = make_surface_point(s, is.tri_id, ray, rd, rd_out);
            surftest_put_point(out + 9, p);
            surftest_put_rd(out + 44, rd_out);
            // The decisions, read back from the outputs so that make_surface_point stays as the kernels compile it: the geometric normal
            // is +-normalize(cross(e1, e2)) exactly; fy = cross(sn, normalize(dpdu)) is recomputed from the exact sn and dpdu by the same
            // functions; the determinant is formed without FMA contraction, so recomputing it gives the kernel's value.
            TriAttribs a;
            tri_attribs(s, is.tri_id, a);
            const double det = tri_uv_det(a);
            const bool flipped = dot(p.geom_normal, normalize(cross(v1 - v0, v2 - v0))) < 0;
            const Frame& f = p.shading_frame;
            const bool fy_degenerate = !(length_sq(cross(f.n, normalize(p.dpdu))) > 0);
            const V3 gn0 = flipped ? -p.geom_normal : p.geom_normal;
            out[56] = det == 0;
            out[57] = flipped;
            out[58] = fy_degenerate;
            out[59] = gn0.z < Real(-1) + Real(1e-6);
            out[60] = f.n.z < Real(-1) + Real(1e-6);
            out[61] = det;
        } else {
            const SurfacePoint d_p = surftest_point(in + 20);
            const RayDiff d_rd_out = surftest_rd(in + 55);
            DRay d_ray = zero_dray();
            RayDiff d_rd = zero_raydiff();
            V3 d_vp[3], d_vn[3], d_vc[3];
            V2 d_vuv[3];
            for (int k = 0; k < 3; k++) {
                d_vp[k] = d_vn[k] = d_vc[k] = zero3();
                d_vuv[k] = zero2();
            }
            d_make_surface_point(s, is.tri_id, ray, rd, d_p, d_rd_out, d_ray, d_rd, d_vp, d_vn, d_vuv, d_vc);
            surftest_put(out, d_ray.org);
            surftest_put(out + 3, d_ray.dir);
            surftest_put_rd(out + 6, d_rd);
            for (int k = 0; k < 3; k++) {
                surftest_put(out + 18 + 3 * k, d_vp[k]);
                surftest_put(out + 27 + 3 * k, d_vn[k]);
                out[36 + 2 * k] = d_vuv[k].x;
                out[37 + 2 * k] = d_vuv[k].y;
                surftest_put(out + 42 + 3 * k, d_vc[k]);
            }
            if (ds != nullptr) scatter_vertex_grads(sc, *ds, is, d_vp, d_vn, d_vuv, d_vc);
        }
    } else {
        const V2 sample = mk2((Real)in[2], (Real)in[3]);
        if (op == RB_SURFTEST_LIGHT) {
            const SurfacePoint p = sample_light_triangle(s, is.tri_id, sample);
            const V3 v[5] = {p.position, p.geom_normal, p.shading_frame.x, p.shading_frame.y, p.shading_frame.n};
            for (int k = 0; k < 5; k++) surftest_put(out + 3 * k, v[k]);
            out[15] = p.bary.x;
            out[16] = p.bary.y;
            out[17] = p.uv.x;
            out[18] = p.uv.y;
            const V2 uv = light_sample_uv(s, is.tri_id, sample);
            out[19] = uv.x;
            out[20] = uv.y;
            out[21] = shape_tri_area(s, is.tri_id);
        } else {
            SurfacePoint d_p = zero_point();
            d_p.position = surftest_v3(in + 4);
            d_p.geom_normal = surftest_v3(in + 7);
            d_p.shading_frame = mk_frame(surftest_v3(in + 10), surftest_v3(in + 13), surftest_v3(in + 16));
            V3 d_v[3] = {zero3(), zero3(), zero3()}, d_va[3] = {zero3(), zero3(), zero3()};
            d_sample_light_triangle(s, is.tri_id, sample, d_p, d_v);
            d_shape_tri_area(s, is.tri_id, (Real)in[19], d_va);
            for (int k = 0; k < 3; k++) {
                surftest_put(out + 3 * k, d_v[k]);
                surftest_put(out + 9 + 3 * k, d_va[k]);
            }
            const rb_dshape* dsh = ds != nullptr ? &ds->shapes[is.shape_id] : nullptr;
            if (dsh != nullptr && s.uvs && dsh->uvs) d_light_sample_uv(s, is.tri_id, sample, mk2((Real)in[20], (Real)in[21]), dsh->uvs);
        }
    }
}

// The checks the library and the emulator share: the op, the count, and every query's shape and triangle (`rows`: the inputs on the host).
template <typename Scene>
inline const char* surface_test_check(const Scene* sc, int op, int n, const double* in, const double* rows) {
    if (sc == nullptr) return "null scene";
    if (sc->incomplete) return "the scene's last update failed";
    if (op < RB_SURFTEST_POINT || op > RB_SURFTEST_D_LIGHT) return "unknown op";
    if (n < 0) return "negative number of queries";
    if (n > 0 && in == nullptr) return "null buffer";
    for (long long i = 0; i < n; i++) {
        const double sh = rows[RB_SURFTEST_IN * i], tr = rows[RB_SURFTEST_IN * i + 1];
        if (!(sh >= 0 && sh < (double)sc->shapes.size()) || sh != (double)(int)sh) return "shape out of range";
        if (!(tr >= 0 && tr < (double)sc->shapes[(int)sh].num_triangles) || tr != (double)(int)tr) return "triangle out of range";
    }
    return nullptr;
}
