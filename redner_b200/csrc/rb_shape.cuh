// Triangle meshes: ray/triangle solve with ray-differential propagation, surface-point reconstruction,
// light-point sampling -- and the reverse-mode adjoint of each.
//   intersect / d_intersect               src/intersection.h:55-109 / :111-289
//   intersect_shape / d_intersect_shape   src/shape.h:258-382 / :384-747
//   sample_shape / d_sample_shape         src/shape.h:184-210 / :212-256
//   get_area / d_get_area                 src/shape.h:156-182
// Geometry is fetched straight from the caller's buffers (float [V,3] / int [T,3]); the BVH only decides WHICH
// triangle, the reported (u, v, t) are re-derived here, like the reference does after Embree (src/scene.cpp:583-592).
#pragma once
#include "rb_types.cuh"

RB_HD V3 shape_vertex(const rb_shape& s, int i) {
    const float* p = s.vertices + 3 * (size_t)i;
    return mk3(p[0], p[1], p[2]);
}
RB_HD void shape_tri(const rb_shape& s, int t, int idx[3]) {
    const int* p = s.indices + 3 * (size_t)t;
    idx[0] = p[0];
    idx[1] = p[1];
    idx[2] = p[2];
}
RB_HD void shape_tri_vertices(const rb_shape& s, int t, V3& v0, V3& v1, V3& v2) {
    int idx[3];
    shape_tri(s, t, idx);
    v0 = shape_vertex(s, idx[0]);
    v1 = shape_vertex(s, idx[1]);
    v2 = shape_vertex(s, idx[2]);
}
RB_HD Real shape_tri_area(const rb_shape& s, int t) {
    V3 v0, v1, v2;
    shape_tri_vertices(s, t, v0, v1, v2);
    return Real(0.5) * length(cross(v1 - v0, v2 - v0));
}
RB_HD void d_shape_tri_area(const rb_shape& s, int t, Real d_area, V3 d_v[3]) {
    V3 v0, v1, v2;
    shape_tri_vertices(s, t, v0, v1, v2);
    V3 dir = cross(v1 - v0, v2 - v0);
    V3 d_dir = d_length(dir, d_area * Real(0.5));
    V3 d_e1 = zero3(), d_e2 = zero3();
    d_cross(v1 - v0, v2 - v0, d_dir, d_e1, d_e2);
    d_v[0] -= (d_e1 + d_e2);
    d_v[1] += d_e1;
    d_v[2] += d_e2;
}

// ---- ray / triangle solve with screen-space differentials of (u, v, t) ----
struct TriSolve {
    Real u, v, t;
    V2 u_dxy, v_dxy, t_dxy;
};
struct TriTerms { // intermediate quantities shared by the primal and the adjoint
    V3 e1, e2, pvec, pvec_dx, pvec_dy, s, qvec, qvec_dx, qvec_dy;
    Real div, div_dx, div_dy;
    Real nu, nu_dx, nu_dy, nv, nv_dx, nv_dy, nt, nt_dx, nt_dy;
};
RB_HD void tri_terms(V3 v0, V3 v1, V3 v2, const Ray& ray, const RayDiff& rd, TriTerms& k) {
    k.e1 = v1 - v0;
    k.e2 = v2 - v0;
    k.pvec = cross(ray.dir, k.e2);
    k.pvec_dx = cross(rd.dir_dx, k.e2);
    k.pvec_dy = cross(rd.dir_dy, k.e2);
    k.div = dot(k.pvec, k.e1);
    k.div_dx = dot(k.pvec_dx, k.e1);
    k.div_dy = dot(k.pvec_dy, k.e1);
    // near-parallel rays: the reference clamps the divisor instead of rejecting (src/intersection.h:73-80)
    if (fabs(k.div) < Real(1e-8)) k.div = (k.div > 0) ? Real(1e-8) : Real(-1e-8);
    k.s = ray.org - v0;
    k.nu = dot(k.s, k.pvec);
    k.nu_dx = dot(rd.org_dx, k.pvec) + dot(k.s, k.pvec_dx);
    k.nu_dy = dot(rd.org_dy, k.pvec) + dot(k.s, k.pvec_dy);
    k.qvec = cross(k.s, k.e1);
    k.qvec_dx = cross(rd.org_dx, k.e1);
    k.qvec_dy = cross(rd.org_dy, k.e1);
    k.nv = dot(ray.dir, k.qvec);
    k.nv_dx = dot(rd.dir_dx, k.qvec) + dot(ray.dir, k.qvec_dx);
    k.nv_dy = dot(rd.dir_dy, k.qvec) + dot(ray.dir, k.qvec_dy);
    k.nt = dot(k.e2, k.qvec);
    k.nt_dx = dot(k.e2, k.qvec_dx);
    k.nt_dy = dot(k.e2, k.qvec_dy);
}
RB_HD Real quot_d(Real n, Real n_d, Real dv, Real dv_d) { return (n_d * dv - n * dv_d) / rb_sq(dv); }
RB_HD TriSolve tri_solve(V3 v0, V3 v1, V3 v2, const Ray& ray, const RayDiff& rd) {
    TriTerms k;
    tri_terms(v0, v1, v2, ray, rd, k);
    TriSolve r;
    r.u = k.nu / k.div;
    r.v = k.nv / k.div;
    r.t = k.nt / k.div;
    r.u_dxy = mk2(quot_d(k.nu, k.nu_dx, k.div, k.div_dx), quot_d(k.nu, k.nu_dy, k.div, k.div_dy));
    r.v_dxy = mk2(quot_d(k.nv, k.nv_dx, k.div, k.div_dx), quot_d(k.nv, k.nv_dy, k.div, k.div_dy));
    r.t_dxy = mk2(quot_d(k.nt, k.nt_dx, k.div, k.div_dx), quot_d(k.nt, k.nt_dy, k.div, k.div_dy));
    return r;
}
// Adjoint of q = n / dv, q_dx = (n_dx dv - n dv_dx) / dv^2, q_dy likewise.
RB_HD void quot_adjoint(Real n, Real n_dx, Real n_dy, Real dv, Real dv_dx, Real dv_dy, Real d_q, V2 d_q_dxy, Real& d_n, Real& d_n_dx,
                        Real& d_n_dy, Real& d_dv, Real& d_dv_dx, Real& d_dv_dy) {
    Real dv2 = dv * dv, dv3 = dv2 * dv;
    d_n_dx = d_q_dxy.x / dv;
    d_n_dy = d_q_dxy.y / dv;
    d_n = d_q / dv - d_q_dxy.x * dv_dx / dv2 - d_q_dxy.y * dv_dy / dv2;
    d_dv += -d_q * (n / dv) / dv - d_q_dxy.x * (n_dx / dv2 - 2 * n * dv_dx / dv3) - d_q_dxy.y * (n_dy / dv2 - 2 * n * dv_dy / dv3);
    d_dv_dx += -d_q_dxy.x * n / dv2;
    d_dv_dy += -d_q_dxy.y * n / dv2;
}
RB_HD void d_tri_solve(V3 v0, V3 v1, V3 v2, const Ray& ray, const RayDiff& rd, Real d_u, Real d_v, Real d_t, V2 d_u_dxy, V2 d_v_dxy,
                       V2 d_t_dxy, V3& d_v0, V3& d_v1, V3& d_v2, DRay& d_ray, RayDiff& d_rd) {
    TriTerms k;
    tri_terms(v0, v1, v2, ray, rd, k);
    Real d_div = 0, d_div_dx = 0, d_div_dy = 0;
    Real d_nt, d_nt_dx, d_nt_dy, d_nv, d_nv_dx, d_nv_dy, d_nu, d_nu_dx, d_nu_dy;
    quot_adjoint(k.nt, k.nt_dx, k.nt_dy, k.div, k.div_dx, k.div_dy, d_t, d_t_dxy, d_nt, d_nt_dx, d_nt_dy, d_div, d_div_dx, d_div_dy);
    quot_adjoint(k.nv, k.nv_dx, k.nv_dy, k.div, k.div_dx, k.div_dy, d_v, d_v_dxy, d_nv, d_nv_dx, d_nv_dy, d_div, d_div_dx, d_div_dy);
    quot_adjoint(k.nu, k.nu_dx, k.nu_dy, k.div, k.div_dx, k.div_dy, d_u, d_u_dxy, d_nu, d_nu_dx, d_nu_dy, d_div, d_div_dx, d_div_dy);
    // nt* = dot(e2, qvec*)
    V3 d_e2 = d_nt * k.qvec + d_nt_dx * k.qvec_dx + d_nt_dy * k.qvec_dy;
    V3 d_qvec = d_nt * k.e2, d_qvec_dx = d_nt_dx * k.e2, d_qvec_dy = d_nt_dy * k.e2;
    // nv* = dot(dir*, qvec) + dot(dir, qvec*)
    d_ray.dir += d_nv * k.qvec + d_nv_dx * k.qvec_dx + d_nv_dy * k.qvec_dy;
    d_qvec += d_nv * ray.dir + d_nv_dx * rd.dir_dx + d_nv_dy * rd.dir_dy;
    d_rd.dir_dx += d_nv_dx * k.qvec;
    d_rd.dir_dy += d_nv_dy * k.qvec;
    d_qvec_dx += d_nv_dx * ray.dir;
    d_qvec_dy += d_nv_dy * ray.dir;
    // qvec* = cross(s*, e1)
    V3 d_s = zero3(), d_s_dx = zero3(), d_s_dy = zero3(), d_e1 = zero3();
    d_cross(rd.org_dx, k.e1, d_qvec_dx, d_s_dx, d_e1);
    d_cross(rd.org_dy, k.e1, d_qvec_dy, d_s_dy, d_e1);
    d_cross(k.s, k.e1, d_qvec, d_s, d_e1);
    // nu* = dot(s*, pvec) + dot(s, pvec*)
    d_s += d_nu * k.pvec + d_nu_dx * k.pvec_dx + d_nu_dy * k.pvec_dy;
    V3 d_pvec = d_nu * k.s + d_nu_dx * rd.org_dx + d_nu_dy * rd.org_dy;
    d_s_dx += d_nu_dx * k.pvec;
    d_s_dy += d_nu_dy * k.pvec;
    V3 d_pvec_dx = d_nu_dx * k.s, d_pvec_dy = d_nu_dy * k.s;
    d_rd.org_dx += d_s_dx;
    d_rd.org_dy += d_s_dy;
    d_ray.org += d_s;
    d_v0 -= d_s;
    // div* = dot(pvec*, e1)
    d_pvec_dx += d_div_dx * k.e1;
    d_pvec_dy += d_div_dy * k.e1;
    d_pvec += d_div * k.e1;
    d_e1 += d_div_dx * k.pvec_dx + d_div_dy * k.pvec_dy + d_div * k.pvec;
    // pvec* = cross(dir*, e2)
    d_cross(rd.dir_dx, k.e2, d_pvec_dx, d_rd.dir_dx, d_e2);
    d_cross(rd.dir_dy, k.e2, d_pvec_dy, d_rd.dir_dy, d_e2);
    d_cross(ray.dir, k.e2, d_pvec, d_ray.dir, d_e2);
    d_v2 += d_e2;
    d_v0 -= d_e2;
    d_v1 += d_e1;
    d_v0 -= d_e1;
}

// ---- surface point at a known (shape, triangle) ----
struct TriAttribs { // per-corner attribute indices and uv values
    int ind[3], uv_ind[3], n_ind[3];
    V2 uv0, uv1, uv2;
};
RB_HD void tri_attribs(const rb_shape& s, int t, TriAttribs& a) {
    shape_tri(s, t, a.ind);
    for (int i = 0; i < 3; i++) {
        a.uv_ind[i] = s.uv_indices ? s.uv_indices[3 * (size_t)t + i] : a.ind[i];
        a.n_ind[i] = s.normal_indices ? s.normal_indices[3 * (size_t)t + i] : a.ind[i];
    }
    if (s.uvs) {
        a.uv0 = mk2(s.uvs[2 * a.uv_ind[0]], s.uvs[2 * a.uv_ind[0] + 1]);
        a.uv1 = mk2(s.uvs[2 * a.uv_ind[1]], s.uvs[2 * a.uv_ind[1] + 1]);
        a.uv2 = mk2(s.uvs[2 * a.uv_ind[2]], s.uvs[2 * a.uv_ind[2] + 1]);
    } else {
        a.uv0 = mk2(0, 0);
        a.uv1 = mk2(1, 0);
        a.uv2 = mk2(1, 1);
    }
}
// Texture coordinate at barycentrics (u, v) of a triangle (weights 1 - u - v, u, v of its corners): the uv of a ray hit
// (make_surface_point) and of a light sample (light_sample_uv) alike.
RB_HD V2 tri_uv(const TriAttribs& a, Real u, Real v) {
    Real w = 1 - (u + v);
    return w * a.uv0 + u * a.uv1 + v * a.uv2;
}
// Determinant of the uv triangle's edge matrix as the reference computes it (src/shape.h:299-301): the float uv corners are subtracted in
// double and the two products are rounded separately before their difference, never contracted into an FMA.  Two equal uv corners then
// give two identical products and exactly 0, whatever the third corner is; a fused form leaves the rounding residual of one product
// (about 1e-17 for uv0 = uv1 = (0.3, 0.7), uv2 = (0.01, 0.02)), and the dpdu branch flips.  make_surface_point and its adjoint both call
// this, so they take the same branch.
RB_HD double tri_uv_det(const TriAttribs& a) {
    const double x02 = (double)a.uv0.x - a.uv2.x, y02 = (double)a.uv0.y - a.uv2.y, x12 = (double)a.uv1.x - a.uv2.x, y12 = (double)a.uv1.y - a.uv2.y;
#ifdef __CUDA_ARCH__
    return __dsub_rn(__dmul_rn(x02, y12), __dmul_rn(y02, x12));
#else
    volatile double p = x02 * y12, q = y02 * x12; // (host build: keep the compiler from contracting under -mfma / -ffp-contract=fast)
    return p - q;
#endif
}
RB_HD V3 shape_normal(const rb_shape& s, int i) {
    const float* p = s.normals + 3 * (size_t)i;
    return mk3(p[0], p[1], p[2]);
}
RB_HD V3 shape_color(const rb_shape& s, int i) {
    const float* p = s.colors + 3 * (size_t)i;
    return mk3(p[0], p[1], p[2]);
}

RB_HD SurfacePoint make_surface_point(const rb_shape& s, int tri, const Ray& ray, const RayDiff& rd, RayDiff& rd_out) {
    TriAttribs a;
    tri_attribs(s, tri, a);
    V3 v0 = shape_vertex(s, a.ind[0]), v1 = shape_vertex(s, a.ind[1]), v2 = shape_vertex(s, a.ind[2]);
    TriSolve h = tri_solve(v0, v1, v2, ray, rd);
    Real u = h.u, v = h.v, w = 1 - (u + v), t = h.t;
    SurfacePoint p;
    p.uv = tri_uv(a, u, v);
    // hit point: product and sum rounded separately like the reference's (src/shape.h:295), see rb_mul_add_unfused
    p.position = mk3(rb_mul_add_unfused(ray.dir.x, t, ray.org.x), rb_mul_add_unfused(ray.dir.y, t, ray.org.y), rb_mul_add_unfused(ray.dir.z, t, ray.org.z));
    V3 gn = normalize(cross(v1 - v0, v2 - v0));
    V2 uv02 = a.uv0 - a.uv2, uv12 = a.uv1 - a.uv2;
    const double det = tri_uv_det(a);
    V3 dpdu = zero3(), dpdv = zero3();
    if (det == 0) {
        coordinate_system(gn, dpdu, dpdv);
    } else {
        Real inv = 1 / (Real)det;
        V3 v02 = v0 - v2, v12 = v1 - v2;
        dpdu = (uv12.y * v02 - uv02.y * v12) * inv;
    }
    V2 neg = -h.u_dxy - h.v_dxy;
    p.du_dxy = neg * a.uv0.x + h.u_dxy * a.uv1.x + h.v_dxy * a.uv2.x;
    p.dv_dxy = neg * a.uv0.y + h.u_dxy * a.uv1.y + h.v_dxy * a.uv2.y;
    V3 dpdx = rd.org_dx + ray.dir * h.t_dxy.x + rd.dir_dx * t;
    V3 dpdy = rd.org_dy + ray.dir * h.t_dxy.y + rd.dir_dy * t;
    V3 sn = gn;
    p.dn_dx = p.dn_dy = zero3();
    if (s.normals) {
        V3 n0 = shape_normal(s, a.n_ind[0]), n1 = shape_normal(s, a.n_ind[1]), n2 = shape_normal(s, a.n_ind[2]);
        V3 nn = w * n0 + u * n1 + v * n2;
        V3 dnn_dx = neg.x * n0 + h.u_dxy.x * n1 + h.v_dxy.x * n2;
        V3 dnn_dy = neg.y * n0 + h.u_dxy.y * n1 + h.v_dxy.y * n2;
        Real l2 = dot(nn, nn), l = sqrt(l2);
        // (an interpolated normal of length 0 has no derivative: zero there instead of 0 / 0, as the adjoint skips it)
        if (l2 * l > 0) {
            p.dn_dx = (l2 * dnn_dx - dot(nn, dnn_dx) * nn) / (l2 * l);
            p.dn_dy = (l2 * dnn_dy - dot(nn, dnn_dy) * nn) / (l2 * l);
        }
        sn = normalize(nn);
        if (dot(gn, sn) < 0) gn = -gn;
    }
    V3 fx = normalize(dpdu);
    V3 fy = cross(sn, fx);
    if (length_sq(fy) > 0) {
        fy = normalize(fy);
        fx = cross(fy, sn);
    } else {
        coordinate_system(sn, fx, fy);
    }
    p.geom_normal = gn;
    p.shading_frame = mk_frame(fx, fy, sn);
    p.dpdu = dpdu;
    rd_out.org_dx = dpdx;
    rd_out.org_dy = dpdy;
    rd_out.dir_dx = rd.dir_dx;
    rd_out.dir_dy = rd.dir_dy;
    p.color = zero3();
    if (s.colors) p.color = w * shape_color(s, a.ind[0]) + u * shape_color(s, a.ind[1]) + v * shape_color(s, a.ind[2]);
    p.bary = mk2(u, v);
    return p;
}

// Adjoint of make_surface_point.  d_vp / d_vn / d_vuv / d_vc receive the per-corner gradients.
// The treatment of the shading frame follows the reference statement by statement (including the places where
// it double-counts or drops a term, src/shape.h:533-549, :565-574, :634-638) because gradient parity with the
// oracle is the acceptance test.
RB_HD void d_make_surface_point(const rb_shape& s, int tri, const Ray& ray, const RayDiff& rd, const SurfacePoint& d_p,
                                const RayDiff& d_rd_out, DRay& d_ray, RayDiff& d_rd, V3 d_vp[3], V3 d_vn[3], V2 d_vuv[3], V3 d_vc[3]) {
    TriAttribs a;
    tri_attribs(s, tri, a);
    V3 v0 = shape_vertex(s, a.ind[0]), v1 = shape_vertex(s, a.ind[1]), v2 = shape_vertex(s, a.ind[2]);
    TriSolve h = tri_solve(v0, v1, v2, ray, rd);
    Real u = h.u, v = h.v, w = 1 - (u + v), t = h.t;
    V3 ugn = cross(v1 - v0, v2 - v0);
    V3 gn = normalize(ugn);
    V2 uv02 = a.uv0 - a.uv2, uv12 = a.uv1 - a.uv2;
    const double det = tri_uv_det(a);
    V3 dpdu = zero3(), dpdv = zero3();
    if (det == 0) {
        coordinate_system(gn, dpdu, dpdv);
    } else {
        Real inv = 1 / (Real)det;
        dpdu = (uv12.y * (v0 - v2) - uv02.y * (v1 - v2)) * inv;
    }
    V2 neg = -h.u_dxy - h.v_dxy;
    V3 sn = gn;
    bool flipped = false;
    V3 n0 = zero3(), n1 = zero3(), n2 = zero3(), nn = zero3(), dnn_dx = zero3(), dnn_dy = zero3(), dn_dx = zero3(), dn_dy = zero3();
    Real l2 = 0, l = 0;
    if (s.normals) {
        n0 = shape_normal(s, a.n_ind[0]);
        n1 = shape_normal(s, a.n_ind[1]);
        n2 = shape_normal(s, a.n_ind[2]);
        nn = w * n0 + u * n1 + v * n2;
        dnn_dx = neg.x * n0 + h.u_dxy.x * n1 + h.v_dxy.x * n2;
        dnn_dy = neg.y * n0 + h.u_dxy.y * n1 + h.v_dxy.y * n2;
        l2 = dot(nn, nn);
        l = sqrt(l2);
        dn_dx = (l2 * dnn_dx - dot(nn, dnn_dx) * nn) / (l2 * l);
        dn_dy = (l2 * dnn_dy - dot(nn, dnn_dy) * nn) / (l2 * l);
        sn = normalize(nn);
        if (dot(gn, sn) < 0) {
            gn = -gn;
            flipped = true;
        }
    }
    V3 fx_org = normalize(dpdu);
    V3 fy_org = cross(sn, fx_org);
    bool fy_ok = length_sq(fy_org) > 0;
    V3 fx = zero3(), fy = zero3();
    if (fy_ok) {
        fy = normalize(fy_org);
        fx = cross(fy, sn);
    } else {
        coordinate_system(sn, fx, fy);
    }

    // ---- reverse sweep ----
    Real d_u = d_p.bary.x, d_v = d_p.bary.y, d_w = 0;
    if (s.colors) {
        V3 c0 = shape_color(s, a.ind[0]), c1 = shape_color(s, a.ind[1]), c2 = shape_color(s, a.ind[2]);
        d_vc[0] += d_p.color * w;
        d_vc[1] += d_p.color * u;
        d_vc[2] += d_p.color * v;
        d_w += sum(d_p.color * c0);
        d_u += sum(d_p.color * c1);
        d_v += sum(d_p.color * c2);
    }
    V3 d_fx = d_p.shading_frame.x, d_fy = d_p.shading_frame.y, d_sn = d_p.shading_frame.n;
    V3 d_dpdu = d_p.dpdu;
    if (fy_ok) {
        d_cross(fy, sn, d_fx, d_fy, d_sn);
        V3 d_fy_org = d_normalize(fy_org, d_fy);
        V3 d_fx_org = zero3();
        d_cross(sn, fx_org, d_fy_org, d_sn, d_fx_org);
        d_dpdu = d_normalize(dpdu, d_fx_org);
    } else {
        d_coordinate_system(sn, d_fx, d_fy, d_sn);
    }
    V3 d_gn = d_p.geom_normal;
    V3 d_dpdx = d_rd_out.org_dx, d_dpdy = d_rd_out.org_dy;
    d_rd.dir_dx += d_rd_out.dir_dx;
    d_rd.dir_dy += d_rd_out.dir_dy;
    V2 d_u_dxy = zero2(), d_v_dxy = zero2();
    V3 d_v0 = zero3(), d_v1 = zero3(), d_v2 = zero3();
    if (s.normals) {
        if (flipped) d_gn = -d_gn;
        d_coordinate_system(sn, d_p.shading_frame.x, d_p.shading_frame.y, d_sn);
        if (l2 > 0) {
            V3 d_nn = d_normalize(nn, d_sn);
            Real denom = l2 * l;
            V3 d_dn_dx = d_p.dn_dx, d_dn_dy = d_p.dn_dy;
            // NOTE: the reference keeps d_nn_len_sq / d_nn_denom as *vectors* (elementwise products that are never
            // summed, src/shape.h:595-610); reproduced.  These terms only carry d_point.dn_dx/dn_dy, which no
            // stage of the path produces (d_bsdf_sample is disabled, src/path_contribution.cpp:458-474).
            V3 d_l2 = (d_dn_dx * dnn_dx + d_dn_dy * dnn_dy) / denom;
            V3 d_dnn_dx = d_dn_dx * l2 / denom;
            V3 d_dnn_dy = d_dn_dy * l2 / denom;
            Real d_dot_x = sum(d_dn_dx * nn) / denom;
            Real d_dot_y = sum(d_dn_dy * nn) / denom;
            d_nn += (d_dn_dx * dot(nn, dnn_dx) + d_dn_dy * dot(nn, dnn_dy)) / denom;
            V3 d_denom = (d_dn_dx * (-dn_dx) + d_dn_dy * (-dn_dy)) / denom;
            d_nn += d_dot_x * dnn_dx + d_dot_y * dnn_dy;
            d_dnn_dx += d_dot_x * nn;
            d_dnn_dy += d_dot_y * nn;
            d_l2 += d_denom * (l * Real(1.5));
            d_nn += 2 * (d_l2 * nn);
            d_u_dxy.x += sum(d_dnn_dx * (n1 - n0));
            d_u_dxy.y += sum(d_dnn_dy * (n1 - n0));
            d_v_dxy.x += sum(d_dnn_dx * (n2 - n0));
            d_v_dxy.y += sum(d_dnn_dy * (n2 - n0));
            V3 d_n0 = d_dnn_dx * neg.x + d_dnn_dy * neg.y;
            V3 d_n1 = d_dnn_dx * h.u_dxy.x + d_dnn_dy * h.u_dxy.y;
            V3 d_n2 = d_dnn_dx * h.v_dxy.x + d_dnn_dy * h.v_dxy.y;
            d_w += sum(d_nn * n0);
            d_u += sum(d_nn * n1);
            d_v += sum(d_nn * n2);
            d_n0 += d_nn * w;
            d_n1 += d_nn * u;
            d_n2 += d_nn * v;
            d_vn[0] += d_n0;
            d_vn[1] += d_n1;
            d_vn[2] += d_n2;
        }
    } else {
        d_gn += d_p.shading_frame.n;
        d_coordinate_system(sn, d_p.shading_frame.x, d_p.shading_frame.y, d_gn);
    }
    // dpdx = org_dx + dir * t_dx + dir_dx * t
    V2 d_t_dxy = zero2();
    d_rd.org_dx += d_dpdx;
    d_ray.dir += d_dpdx * h.t_dxy.x;
    d_t_dxy.x += sum(d_dpdx * ray.dir);
    d_rd.dir_dx += d_dpdx * t;
    Real d_t = sum(d_dpdx * rd.dir_dx);
    d_rd.org_dy += d_dpdy;
    d_ray.dir += d_dpdy * h.t_dxy.y;
    d_t_dxy.y += sum(d_dpdy * ray.dir);
    d_rd.dir_dy += d_dpdy * t;
    d_t += sum(d_dpdy * rd.dir_dy);
    // dpdu
    V2 d_uv0 = zero2(), d_uv1 = zero2(), d_uv2 = zero2();
    if (det == 0) {
        d_coordinate_system(gn, d_dpdu, zero3(), d_gn);
    } else {
        Real inv = 1 / (Real)det;
        V3 v02 = v0 - v2, v12 = v1 - v2;
        V2 d_uv02 = zero2(), d_uv12 = zero2();
        d_uv12.y += sum(d_dpdu * v02) * inv;
        V3 d_v02 = d_dpdu * uv12.y * inv;
        d_uv02.y += sum(d_dpdu * v12) * inv;
        V3 d_v12 = d_dpdu * uv02.y * inv;
        Real d_inv = sum(d_dpdu * (uv12.y * v02 - uv02.y * v12));
        Real d_det = -d_inv * inv * inv;
        d_uv02.x += d_det * uv12.y;
        d_uv12.y += d_det * uv02.x;
        d_uv02.y -= d_det * uv12.x;
        d_uv12.x -= d_det * uv02.y;
        d_uv0 += d_uv02;
        d_uv1 += d_uv12;
        d_uv2 -= (d_uv02 + d_uv12);
        d_v0 += d_v02;
        d_v1 += d_v12;
        d_v2 -= (d_v02 + d_v12);
    }
    V2 d_du = d_p.du_dxy, d_dv = d_p.dv_dxy;
    d_u_dxy += d_du * (a.uv1.x - a.uv0.x) + d_dv * (a.uv1.y - a.uv0.y);
    d_v_dxy += d_du * (a.uv2.x - a.uv0.x) + d_dv * (a.uv2.y - a.uv0.y);
    d_uv0.x += sum(d_du * neg);
    d_uv0.y += sum(d_dv * neg);
    d_uv1.x += sum(d_du * h.u_dxy);
    d_uv1.y += sum(d_dv * h.u_dxy);
    d_uv2.x += sum(d_du * h.v_dxy);
    d_uv2.y += sum(d_dv * h.v_dxy);
    // geometric normal
    V3 d_ugn = d_normalize(ugn, d_gn);
    V3 d_e1 = zero3(), d_e2 = zero3();
    d_cross(v1 - v0, v2 - v0, d_ugn, d_e1, d_e2);
    d_v0 += (-d_e1 - d_e2);
    d_v1 += d_e1;
    d_v2 += d_e2;
    // hit position
    d_ray.org += d_p.position;
    d_ray.dir += d_p.position * t;
    d_t += sum(d_p.position * ray.dir);
    // uv
    d_w += sum(d_p.uv * a.uv0);
    d_u += sum(d_p.uv * a.uv1);
    d_v += sum(d_p.uv * a.uv2);
    d_uv0 += d_p.uv * w;
    d_uv1 += d_p.uv * u;
    d_uv2 += d_p.uv * v;
    d_u -= d_w;
    d_v -= d_w;
    d_tri_solve(v0, v1, v2, ray, rd, d_u, d_v, d_t, d_u_dxy, d_v_dxy, d_t_dxy, d_v0, d_v1, d_v2, d_ray, d_rd);
    if (s.uvs) {
        d_vuv[0] += d_uv0;
        d_vuv[1] += d_uv1;
        d_vuv[2] += d_uv2;
    }
    d_vp[0] += d_v0;
    d_vp[1] += d_v1;
    d_vp[2] += d_v2;
}

// ---- uniform point on a triangle of an area light ----
RB_HD SurfacePoint sample_light_triangle(const rb_shape& s, int tri, V2 sample) {
    V3 v0, v1, v2;
    shape_tri_vertices(s, tri, v0, v1, v2);
    Real a = sqrt(sample.x);
    Real b1 = 1 - a, b2 = a * sample.y;
    V3 e1 = v1 - v0, e2 = v2 - v0;
    V3 n = normalize(cross(e1, e2));
    SurfacePoint p = zero_point();
    p.position = v0 + e1 * b1 + e2 * b2;
    p.geom_normal = n;
    p.shading_frame = frame_from_normal(n);
    p.uv = sample;
    p.bary = mk2(b1, b2);
    return p;
}
RB_HD void d_sample_light_triangle(const rb_shape& s, int tri, V2 sample, const SurfacePoint& d_p, V3 d_v[3]) {
    V3 v0, v1, v2;
    shape_tri_vertices(s, tri, v0, v1, v2);
    Real a = sqrt(sample.x);
    Real b1 = 1 - a, b2 = a * sample.y;
    V3 e1 = v1 - v0, e2 = v2 - v0;
    V3 n = cross(e1, e2);
    V3 nn = normalize(n);
    V3 d_v0 = d_p.position;
    V3 d_e1 = d_p.position * b1, d_e2 = d_p.position * b2;
    V3 d_nn = d_p.geom_normal + d_p.shading_frame.n;
    d_coordinate_system(nn, d_p.shading_frame.x, d_p.shading_frame.y, d_nn);
    V3 d_n = d_normalize(n, d_nn);
    d_cross(e1, e2, d_n, d_e1, d_e2);
    d_v0 -= d_e1;
    d_v0 -= d_e2;
    d_v[0] += d_v0;
    d_v[1] += d_e1;
    d_v[2] += d_e2;
}
// Texture coordinate of the light sample `sample` on triangle `tri` (sample_light_triangle keeps the sample itself in
// SurfacePoint::uv): the hit's interpolation at the sample's barycentrics.  It depends on the uv vertices only, not on the positions.
RB_HD V2 light_sample_uv(const rb_shape& s, int tri, V2 sample) {
    TriAttribs a;
    tri_attribs(s, tri, a);
    Real r = sqrt(sample.x);
    return tri_uv(a, 1 - r, r * sample.y);
}
