// Secondary (shadow / interreflection) edge sampling at one path vertex.
//   secondary_edge_sampler                    src/edge.cpp:826-1773  (ltc_bound :838-875, importance :885-917,
//                                             leaf_importance :943-1067, sample_edge_h :1115-1237, sample_edge_l :1239-1364,
//                                             operator() :1366-1744)
//   get_ltc_matrix                            src/edge.cpp:803-814
//   secondary_edge_weights_updater            src/edge.cpp:1856-1972 (intersect_jacobian :1829-1853)
//   secondary_edge_derivatives_accumulator    src/edge.cpp:2001-2043
// The estimator is the reference's and so is the hierarchy it walks (a restatement of src/edge_tree.cpp incl. the treelet
// pass, flattened into EdgeNode records); what differs from the reference is only which Sobol point a vertex gets (the
// reference indexes that stream by the rank of the pixel in its compacted wavefront), hence statistical parity on the GPU
// and sample-exact parity in the host build with -DRB_EMU_REF_STREAMS.
// Every path keeps its traversal state in a <= 24-entry stack: each stack item carries at least one of the 16
// stochastic descents, so the hierarchical sampler never holds more than 16 items; the gather variant holds at
// most two per level of the balanced tree.
#pragma once
#include "rb_edge.cuh"
#include "rb_path.cuh"

#define RB_EDGE_H_SAMPLES 16
#define RB_EDGE_STACK_H 24
#define RB_EDGE_STACK_L 64
#define RB_GATHER_BATCH 8

RB_HD M3 m3_rows(V3 a, V3 b, V3 c) {
    M3 r;
    r.m[0][0] = a.x; r.m[0][1] = a.y; r.m[0][2] = a.z;
    r.m[1][0] = b.x; r.m[1][1] = b.y; r.m[1][2] = b.z;
    r.m[2][0] = c.x; r.m[2][1] = c.y; r.m[2][2] = c.z;
    return r;
}
RB_HD M3 m3_mul(const M3& a, const M3& b) {
    M3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}
RB_HD M3 m3_inverse(const M3& m) {
    Real det = m.m[0][0] * (m.m[1][1] * m.m[2][2] - m.m[2][1] * m.m[1][2]) - m.m[0][1] * (m.m[1][0] * m.m[2][2] - m.m[1][2] * m.m[2][0]) +
               m.m[0][2] * (m.m[1][0] * m.m[2][1] - m.m[1][1] * m.m[2][0]);
    Real id = 1 / det;
    M3 r;
    r.m[0][0] = (m.m[1][1] * m.m[2][2] - m.m[2][1] * m.m[1][2]) * id;
    r.m[0][1] = (m.m[0][2] * m.m[2][1] - m.m[0][1] * m.m[2][2]) * id;
    r.m[0][2] = (m.m[0][1] * m.m[1][2] - m.m[0][2] * m.m[1][1]) * id;
    r.m[1][0] = (m.m[1][2] * m.m[2][0] - m.m[1][0] * m.m[2][2]) * id;
    r.m[1][1] = (m.m[0][0] * m.m[2][2] - m.m[0][2] * m.m[2][0]) * id;
    r.m[1][2] = (m.m[1][0] * m.m[0][2] - m.m[0][0] * m.m[1][2]) * id;
    r.m[2][0] = (m.m[1][0] * m.m[2][1] - m.m[2][0] * m.m[1][1]) * id;
    r.m[2][1] = (m.m[2][0] * m.m[0][1] - m.m[0][0] * m.m[2][1]) * id;
    r.m[2][2] = (m.m[0][0] * m.m[1][1] - m.m[1][0] * m.m[0][1]) * id;
    return r;
}

struct EdgeCtx { // per-vertex constants of the sampler
    const DevScene* sc;
    V3 pos; // shading point
    M3 m, m_inv;
    M3 abs_m_inv; // |M^-1| element-wise (box transform)
    V3 cam_org;
    // Olson & Zhang sphere of the shading point: centre 0.5 (p - cam_org), radius^2
    V3 hough_center;
    Real hough_r2;
};
RB_HD void edge_ctx_finish(EdgeCtx& c) { // call after m_inv / cam_org / p are set
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) c.abs_m_inv.m[i][j] = fabs(c.m_inv.m[i][j]);
    c.hough_center = Real(0.5) * (c.pos - c.cam_org);
    c.hough_r2 = rb_sq(Real(0.5) * length(c.pos - c.cam_org));
}

RB_HD Real min_abs_bound(Real lo, Real hi) {
    if (lo <= 0 && hi >= 0) return 0;
    if (lo <= 0 && hi <= 0) return hi;
    return lo;
}
// p inside the PARENT's box == inside the union of its children's boxes (the builder takes exact min / max)
RB_HD bool parent_contains(const EdgeNode& n, V3 p) {
    for (int k = 0; k < 3; k++) {
        Real lo = n.c[0].pmin[k] < n.c[1].pmin[k] ? n.c[0].pmin[k] : n.c[1].pmin[k], hi = n.c[0].pmax[k] > n.c[1].pmax[k] ? n.c[0].pmax[k] : n.c[1].pmax[k];
        if (!(p[k] >= lo && p[k] <= hi)) return false;
    }
    return true;
}
RB_HD bool node_contains(const EdgeChild& n, V3 p) {
    return p.x >= n.pmin[0] && p.x <= n.pmax[0] && p.y >= n.pmin[1] && p.y <= n.pmax[1] && p.z >= n.pmin[2] && p.z <= n.pmax[2];
}
// Upper bound of the (linearly transformed) cosine lobe over a position box, src/edge.cpp:838-875.
//  * The reference transforms the 8 corners and takes min / max: the map is affine, so that box is the transformed centre
//    +- |M^-1| * half-extent -- a fifth of the arithmetic.
//  * Its tail  max_dir = normalize(M dir); local = M^-1 max_dir; return local.z / |local|^4  is  dir.z * |M dir|^3  for a unit `dir`
//    (local == dir / |M dir|): one matrix product and one normalisation less.
//  * Written without divergent branches: lanes of a warp walk different nodes, and "shading point inside the box" is a per-lane fact.
RB_D Real ltc_bound(const EdgeChild& n, const EdgeCtx& c) {
    const bool inside = node_contains(n, c.pos);
    V3 ctr = Real(0.5) * (mk3(n.pmin[0], n.pmin[1], n.pmin[2]) + mk3(n.pmax[0], n.pmax[1], n.pmax[2])) - c.pos;
    V3 ext = Real(0.5) * (mk3(n.pmax[0], n.pmax[1], n.pmax[2]) - mk3(n.pmin[0], n.pmin[1], n.pmin[2]));
    V3 q = mul(c.m_inv, ctr), r = mul(c.abs_m_inv, ext);
    V3 lo = q - r, hi = q + r;
    V3 dir = mk3(min_abs_bound(lo.x, hi.x), min_abs_bound(lo.y, hi.y), hi.z);
    Real l = length(dir);
    dir = (inside || l <= 0) ? mk3(0, 0, 1) : dir / l;
    if (!inside && hi.z < 0) return 0;
    if (dir.z <= 0) return 0;
    Real len2 = length_sq(mul(c.m, dir));
    return dir.z * len2 * sqrt(len2);
}
// Olson & Zhang: an edge of the non-camera-silhouette set can only be a silhouette from p if the sphere with diameter
// (cam_org, p) touches its Hough-space box.  The reference's box / sphere test (Arvo's, src/aabb.h:155-171) returns from INSIDE
// its loop over the axes as soon as the accumulated distance is within the radius; the accumulated distance only grows, so its
// verdict is the verdict of the FIRST axis alone -- which is what this evaluates (same result, a third of the work).
RB_HD bool hough_may_be_silhouette_at(const EdgeChild& n, V3 center, Real r2) {
    Real d = center.x < n.dmin[0] ? rb_sq(center.x - n.dmin[0]) : (center.x > n.dmax[0] ? rb_sq(center.x - n.dmax[0]) : Real(0));
    return d <= r2;
}
RB_HD bool hough_may_be_silhouette(const EdgeChild& n, V3 p, V3 cam_org) {
    return hough_may_be_silhouette_at(n, Real(0.5) * (p - cam_org), rb_sq(Real(0.5) * length(p - cam_org)));
}
RB_D Real node_importance(const EdgeChild& n, bool is6d, const EdgeCtx& c) {
    if (is6d && !hough_may_be_silhouette_at(n, c.hough_center, c.hough_r2)) return 0;
    Real brdf = ltc_bound(n, c);
    V3 center = Real(0.5) * (mk3(n.pmin[0], n.pmin[1], n.pmin[2]) + mk3(n.pmax[0], n.pmax[1], n.pmax[2]));
    return brdf * n.wlen / rb_max(length(center - c.pos), Real(1e-3));
}
// Integral of the transformed cosine along the (clipped) edge, src/edge.cpp:951-983
RB_D Real edge_ltc_integral(V3 v0, V3 v1, const EdgeCtx& c) {
    if (!(length_sq(v1 - v0) > Real(1e-10))) return 0;
    V3 a = mul(c.m_inv, v0 - c.pos), b = mul(c.m_inv, v1 - c.pos);
    if (!(a.z > 0 || b.z > 0)) return 0;
    if (a.z < 0) a = (a * b.z - b * a.z) / (b.z - a.z);
    if (b.z < 0) b = (a * b.z - b * a.z) / (b.z - a.z);
    V3 wt = normalize(b - a);
    Real l0 = dot(a, wt), l1 = dot(b, wt);
    V3 vo = a - l0 * wt;
    Real d = length(vo);
    auto I = [&](Real l) { return (l / (d * (d * d + l * l)) + atan(l / d) / (d * d)) * vo.z + (l * l / (d * (d * d + l * l))) * wt.z; };
    return rb_max(I(l1) - I(l0), Real(0));
}
RB_D Real leaf_importance_h(const Edge& e, const EdgeCtx& c) {
    if (!edge_is_silhouette(c.sc->shapes, c.pos, e)) return 0;
    return edge_ltc_integral(edge_v0(c.sc->shapes, e), edge_v1(c.sc->shapes, e), c);
}
// gather variant: the edge must also be a silhouette seen from the light point and its "billboard" must be hit
// by the shadow ray, src/edge.cpp:998-1067
RB_D Real leaf_importance_l(const Edge& e, const EdgeCtx& c, const Ray& nee, Real billboard) {
    if (!edge_is_silhouette(c.sc->shapes, c.pos, e)) return 0;
    V3 nee_pt = nee.org + nee.tmax * nee.dir;
    if (!edge_is_silhouette(c.sc->shapes, nee_pt, e)) return 0;
    V3 v0 = edge_v0(c.sc->shapes, e), v1 = edge_v1(c.sc->shapes, e);
    Real t = -(dot(nee.org, nee.dir) - dot(v0, nee.dir)) / dot(nee.dir, nee.dir);
    V3 ip = nee.org + nee.dir * t;
    V3 v0_p = v0 - ip;
    V3 ed = normalize(v1 - v0);
    V3 ept = ip + v0_p - dot(v0_p, ed) * ed;
    if (length_sq(ept - ip) > rb_sq(billboard)) return 0;
    return edge_ltc_integral(v0, v1, c);
}
// pbrt-style slab test with the box grown by `expand`, src/aabb.h:172-195
RB_HD bool node_hit_by_ray(const EdgeChild& n, const Ray& r, Real expand) {
    Real t0 = r.tmin, t1 = r.tmax;
    for (int i = 0; i < 3; i++) {
        Real inv = 1 / r.dir[i];
        Real tn = (n.pmin[i] - expand - r.org[i]) * inv, tf = (n.pmax[i] + expand - r.org[i]) * inv;
        if (tn > tf) {
            Real tmp = tn;
            tn = tf;
            tf = tmp;
        }
        tf *= (1 + Real(1e-6));
        t0 = tn > t0 ? tn : t0;
        t1 = tf < t1 ? tf : t1;
        if (t0 > t1) return false;
    }
    return true;
}

struct StackH {
    int node;
    short num;
    short is6d;
    Real pmf;
};
// Split `num` stochastic descents between two children proportionally to their importance.
RB_D void split_samples(int num, Real prob0, Real& u, int& n0, int& n1) {
    Real e0 = num * prob0, e1 = num * (1 - prob0);
    n0 = (int)floor(e0);
    n1 = (int)floor(e1);
    if (n0 + n1 < num) {
        Real prob = e0 - n0;
        if (u < prob) {
            n0++;
            u /= prob;
        } else {
            n1++;
            u = (u - prob) / (1 - prob);
        }
    }
}
// 16 correlated stochastic descents through both trees followed by reservoir resampling among the reached leaves, in three
// pieces: hier_begin, hier_step (ONE stack item per call) and hier_end.  sample_edge_hier runs them back to back.
struct HierWalk {
    StackH stack[RB_EDGE_STACK_H];
    StackH leaves[RB_EDGE_H_SAMPLES];
    int sp, nl;
    Real u;
};
RB_D bool hier_begin(const EdgeCtx& c, Real u, HierWalk& w) {
    const DevScene& sc = *c.sc;
    w.sp = 0;
    w.nl = 0;
    Real imp_cs = sc.edge_root_cs != RB_EDGE_EMPTY ? Real(1) : Real(0), imp_ncs = sc.edge_root_ncs != RB_EDGE_EMPTY ? Real(1) : Real(0);
    if (imp_cs <= 0 && imp_ncs <= 0) return false;
    Real prob_cs = imp_cs / (imp_cs + imp_ncs);
    int n_cs, n_ncs;
    split_samples(RB_EDGE_H_SAMPLES, prob_cs, u, n_cs, n_ncs);
    if (n_cs > 0) { w.stack[w.sp].node = sc.edge_root_cs; w.stack[w.sp].num = (short)n_cs; w.stack[w.sp].is6d = 0; w.stack[w.sp].pmf = prob_cs; w.sp++; }
    if (n_ncs > 0) { w.stack[w.sp].node = sc.edge_root_ncs; w.stack[w.sp].num = (short)n_ncs; w.stack[w.sp].is6d = 1; w.stack[w.sp].pmf = 1 - prob_cs; w.sp++; }
    w.u = u;
    return true;
}
// Interior nodes first, leaves afterwards (in the order the descent reached them, so the reservoir of hier_end consumes
// `resample_u` exactly as a combined loop would): lanes of a warp would otherwise sit in the leaf branch (silhouette
// test + LTC line integral) and the interior branch (two box bounds) of the same loop at the same time.
RB_D void hier_step(const EdgeCtx& c, HierWalk& w) { // requires w.sp > 0
    const DevScene& sc = *c.sc;
    StackH it = w.stack[--w.sp];
    if (it.node < 0) { // leaf: ~edge id
        if (w.nl < RB_EDGE_H_SAMPLES) {
            w.leaves[w.nl] = it;
            w.leaves[w.nl].node = ~it.node;
            w.nl++;
        }
        return;
    }
    const EdgeNode n = sc.edge_nodes[it.node]; // one 128-byte fetch: both children's bounds and references
    Real i0, i1;
    if (parent_contains(n, c.pos)) {
        i0 = i1 = 1;
    } else {
        i0 = node_importance(n.c[0], it.is6d != 0, c);
        i1 = node_importance(n.c[1], it.is6d != 0, c);
    }
    if (i0 > 0 || i1 > 0) {
        Real p0 = i0 / (i0 + i1);
        int n0, n1;
        split_samples(it.num, p0, w.u, n0, n1);
        if (n0 > 0 && w.sp < RB_EDGE_STACK_H) { w.stack[w.sp].node = n.c[0].ref; w.stack[w.sp].num = (short)n0; w.stack[w.sp].is6d = it.is6d; w.stack[w.sp].pmf = it.pmf * p0; w.sp++; }
        if (n1 > 0 && w.sp < RB_EDGE_STACK_H) { w.stack[w.sp].node = n.c[1].ref; w.stack[w.sp].num = (short)n1; w.stack[w.sp].is6d = it.is6d; w.stack[w.sp].pmf = it.pmf * (1 - p0); w.sp++; }
    }
}
RB_D int hier_end(const EdgeCtx& c, const HierWalk& w, Real resample_u, Real& sample_weight) {
    const DevScene& sc = *c.sc;
    int selected = -1;
    Real edge_weight = 0, wsum = 0;
    for (int k = 0; k < w.nl; k++) {
        const StackH it = w.leaves[k];
        Real wt = it.num * leaf_importance_h(sc.edges[it.node], c) / it.pmf;
        if (wt > 0) {
            Real prev = wsum;
            wsum += wt;
            Real nw = wt / wsum;
            if (resample_u <= nw || prev == 0) {
                selected = it.node;
                edge_weight = wt * it.pmf;
                resample_u /= nw;
            } else {
                resample_u = (resample_u - nw) / (1 - nw);
            }
        }
    }
    if (edge_weight <= 0 || wsum <= 0) return -1;
    sample_weight = 1 / (edge_weight * RB_EDGE_H_SAMPLES / wsum);
    return selected;
}
RB_D int sample_edge_hier(const EdgeCtx& c, Real u, Real resample_u, Real& sample_weight) {
    HierWalk w;
    if (!hier_begin(c, u, w)) return -1;
    while (w.sp > 0) hier_step(c, w);
    return hier_end(c, w, resample_u, sample_weight);
}
// Gather all silhouette edges whose billboard the shadow ray crosses and pick one by reservoir resampling.
RB_D int sample_edge_gather(const EdgeCtx& c, const Ray& nee, const Isect& lis, const SurfacePoint& lp, Real resample_u, Real& sample_weight,
                            V3& edge_pt, V3& mwt) {
    const DevScene& sc = *c.sc;
    int stack[RB_EDGE_STACK_L];
    int sp = 0;
    int selected = -1;
    Real edge_weight = 0, wsum = 0;
    Real expand = sc.edge_bounds_expand;
    // stack items: child references.  Inner nodes (index >= 0) carry the tree kind in bit 30; leaves (~edge id < 0) need none.
    if (sc.edge_root_cs != RB_EDGE_EMPTY) stack[sp++] = sc.edge_root_cs;
    if (sc.edge_root_ncs != RB_EDGE_EMPTY) stack[sp++] = sc.edge_root_ncs < 0 ? sc.edge_root_ncs : (sc.edge_root_ncs | (1 << 30));
    // Same two-phase structure as the hierarchical sampler: box tests run until RB_GATHER_BATCH leaves are pending (or the
    // stack is empty), then the pending leaves are weighed in arrival order.
    int pending[RB_GATHER_BATCH];
    int np = 0;
    while (sp > 0 || np > 0) {
        while (sp > 0 && np < RB_GATHER_BATCH) {
            int item = stack[--sp];
            if (item < 0) {
                pending[np++] = ~item;
                continue;
            }
            bool is6d = (item & (1 << 30)) != 0;
            const EdgeNode n = sc.edge_nodes[item & ~(1 << 30)];
            for (int k = 0; k < 2; k++) {
                const EdgeChild& ch = n.c[k];
                bool ok = true;
                if (is6d) ok = hough_may_be_silhouette_at(ch, c.hough_center, c.hough_r2) && hough_may_be_silhouette(ch, lp.position, c.cam_org);
                if (ok && node_hit_by_ray(ch, nee, expand) && sp < RB_EDGE_STACK_L) stack[sp++] = ch.ref < 0 ? ch.ref : (ch.ref | (is6d ? (1 << 30) : 0));
            }
        }
        for (int k = 0; k < np; k++) {
            Real w = leaf_importance_l(sc.edges[pending[k]], c, nee, expand);
            if (w > 0) {
                Real prev = wsum;
                wsum += w;
                Real nw = w / wsum;
                if (resample_u <= nw || prev == 0) {
                    selected = pending[k];
                    edge_weight = w;
                    resample_u /= nw;
                } else {
                    resample_u = (resample_u - nw) / (1 - nw);
                }
            }
        }
        np = 0;
    }
    if (selected == -1) return -1;
    Real pmf = edge_weight / wsum;
    const Edge& e = sc.edges[selected];
    V3 v0 = edge_v0(sc.shapes, e), v1 = edge_v1(sc.shapes, e);
    Real t = -(dot(nee.org, nee.dir) - dot(v0, nee.dir)) / dot(nee.dir, nee.dir);
    if (t < nee.tmin || t > nee.tmax) return -1;
    V3 ip = nee.org + nee.dir * t;
    V3 nn = lp.geom_normal;
    V3 omega = ip - nee.org;
    Real tau = dot(lp.position - nee.org, nn) / dot(omega, nn);
    Real jac = length(tau * ((v1 - v0) - omega * (dot(v1 - v0, nn) / dot(omega, nn))));
    const rb_shape& lshape = sc.shapes[lis.shape_id];
#if RB_LIGHT_TEX_KERNELS
    // (emission sampling: the density at the light point, whose record sample lp.uv gives its texture coordinate)
    const LightSampling* lsm = light_sampling(sc, lshape.light_id);
    Real pdf_nee = (Real)(lsm ? sc.light_pmf[lshape.light_id] * light_point_density(sc, *lsm, lshape.light_id, lis.tri_id, light_sample_uv(lshape, lis.tri_id, lp.uv))
                              : sc.light_pmf[lshape.light_id] / sc.light_areas[lshape.light_id]);
#else
    Real pdf_nee = (Real)(sc.light_pmf[lshape.light_id] / sc.light_areas[lshape.light_id]);
#endif
    if (pmf <= 0 || jac <= 0 || pdf_nee <= 0) return -1;
    sample_weight = 1 / (2 * expand * pmf * jac * pdf_nee);
    V3 v0_p = v0 - ip;
    V3 ed = normalize(v1 - v0);
    edge_pt = ip + v0_p - dot(v0_p, ed) * ed - nee.org;
    mwt = v1 - v0;
    return selected;
}

// d(intersection point)/d(line parameter), src/edge.cpp:1829-1853
RB_HD V3 intersect_jacobian(V3 org, V3 dir, V3 p, V3 n, V3 l) {
    Real dn = dot(dir, n);
    if (fabs(dn) < Real(1e-10)) return zero3();
    Real t = -(dot(org, n) - dot(p, n)) / dn;
    if (t <= 0) return zero3();
    return t * (l - dir * (dot(l, n) / dn));
}

// Boundary term of one path vertex in two steps (src/edge.cpp:826-2053):
//   secondary_edge_pick   chooses a silhouette edge and a point on it as seen from the vertex (hierarchy or gather)
//   secondary_edge_shade  traces the two rays on either side of it with their sub-paths and accumulates the gradient
//                         of the shading-point position (returned) and of the two edge vertices (scattered)
// k_bwd_secondary_pick / _shade run them as two kernels with a sort by edge in between: after the pick only about half
// of the lanes are still alive and each continues towards a different edge.
struct alignas(16) EdgePick {
    int edge_id;
    int flags; // bit 0: diffuse lobe, bit 1: gather strategy, bit 2: diffuse or glossy
    float w;   // edge_weight / strategy pmf
    V3 sample_p, mwt;
};
// The pick in three pieces -- pick_setup (frame, lobe, LTC matrices, strategy), the edge choice (hierarchy walk or gather), and
// pick_finish_hier (point on the chosen edge by inverting the LTC line CDF); secondary_edge_pick runs them back to back.
struct PickSetup {
    EdgeCtx c;
    Real m_pmf, nee_pmf, edge_sel, resample, t_sel;
    int flags; // bit 0: diffuse lobe, bit 1: gather strategy, bit 2: diffuse or glossy
};
// `smp` is the edge sampler positioned at this depth's first dimension (4 dimensions are consumed here).  `nee` / `lp` (may be null)
// receive the vertex's shadow ray and light point, which only the gather strategy needs.
RB_D bool pick_setup(const DevScene& sc, const VertexRec& cur, Sampler& smp, PickSetup& ps, Ray* nee_out, SurfacePoint* lp_out) {
    double s_edge_sel = smp.next(), s_resample = smp.next(), s_component = smp.next(), s_t = smp.next();
    Real min_rough = cur.min_rough;
    // secondary edges are only sampled until the first rough bounce (src/edge.cpp:1396-1401)
    if (min_rough > Real(1e-2)) return false;
    const rb_shape& shape = sc.shapes[cur.isect.shape_id];
    const rb_material& mat = sc.materials[shape.material_id];
    RayDiff rd;
    SurfacePoint sp = make_surface_point(shape, cur.isect.tri_id, cur.ray, cur.rd_in, rd);
    V3 wi = -cur.ray.dir;
    if (nee_out != nullptr) {
        // shadow ray of this vertex with its true length (src/edge.cpp:1377-1385)
        const rb_shape& lshape = sc.shapes[cur.light.isect.shape_id];
        SurfacePoint lp = sample_light_triangle(lshape, cur.light.isect.tri_id, cur.light.uv);
        nee_out->org = sp.position;
        nee_out->dir = normalize(lp.position - sp.position);
        nee_out->tmin = Real(1e-3);
        nee_out->tmax = length(lp.position - sp.position);
        *lp_out = lp;
    }
    V3 kd = mat_diffuse(mat, sp), ks = mat_specular(mat, sp);
    Real wd = luminance(kd), ws = luminance(ks), wsum = wd + ws;
    if (wsum <= 0) return false;
    Real pd = wd / wsum, pspec = ws / wsum;
    V3 n = sp.shading_frame.n;
    if (mat.two_sided && dot(wi, n) < 0) n = -n;
    V3 fx = normalize(wi - n * dot(wi, n));
    V3 fy = cross(n, fx);
    if (dot(wi, n) > 1 - Real(1e-6)) coordinate_system(n, fx, fy);
    EdgeCtx& c = ps.c;
    c.sc = &sc;
    c.pos = sp.position;
    {
        double iw = 1.0 / sc.cam.c2w[15];
        c.cam_org = mk3((Real)(sc.cam.c2w[3] * iw), (Real)(sc.cam.c2w[7] * iw), (Real)(sc.cam.c2w[11] * iw));
    }
    Real roughness = rb_max(mat_roughness(mat, sp), min_rough);
    bool diffuse_lobe = s_component <= (double)pd;
    if (diffuse_lobe) {
        c.m_inv = m3_rows(fx, fy, n);
        c.m = m3_inverse(c.m_inv);
        ps.m_pmf = pd;
    } else {
        // LTC fitted to the Blinn-Phong lobe, src/edge.cpp:803-814
        Real theta = acos(dot(wi, sp.shading_frame.n));
        int rid = rb_clampi(int(roughness * 127), 0, 127);
        int tid = rb_clampi(int((theta / (RB_PI / 2)) * 127), 0, 127);
        const float* t = sc.ltc_table + 9 * (rid + tid * 128);
        M3 ltc;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) ltc.m[i][j] = t[3 * i + j];
        c.m_inv = m3_mul(m3_inverse(ltc), m3_rows(fx, fy, n));
        c.m = m3_inverse(c.m_inv);
        ps.m_pmf = pspec;
    }
    edge_ctx_finish(c);
    ps.edge_sel = (Real)s_edge_sel;
    ps.resample = (Real)s_resample;
    ps.t_sel = (Real)s_t;
    bool use_nee = false;
    ps.nee_pmf = 1;
    bool diffuse_or_glossy = diffuse_lobe || roughness > Real(0.1);
    if (diffuse_or_glossy) {
        // The strategy coin is the reference's: the upper half of `edge_sel` goes to the hierarchy (rescaled), the lower half
        // to the gather (src/edge.cpp:1461-1472).  A cheaper-to-run block-wide coin (every warp in one strategy) was tried and
        // is NOT equivalent: the reference scrambles all Sobol dimensions of a pixel with one value, so edge_sel, resample_sel,
        // bsdf_component and t of a sample are strongly related (identical for sample 0) and the mean over seeds at a fixed
        // sample count depends on exactly how the dimensions are consumed (measured on C2 at 8 spp: boundary term of the lamp
        // off by 22 % with an independent coin, 0.6 standard errors with this one).  It also makes the pick a pure function of
        // (pixel, sample, depth), independent of bands, stripes and block size.
        use_nee = s_edge_sel < 0.5;
        if (!use_nee) ps.edge_sel = (Real)((s_edge_sel - 0.5) * 2);
        if (roughness > Real(0.1)) ps.nee_pmf = Real(0.5);
        else ps.nee_pmf = use_nee ? pd * Real(0.5) : 1 - pd * Real(0.5);
    }
    ps.flags = (diffuse_lobe ? 1 : 0) | (use_nee ? 2 : 0) | (diffuse_or_glossy ? 4 : 0);
    return true;
}
// Point on the edge the hierarchy chose: invert the CDF of the transformed cosine along the (clipped) edge.
RB_D bool pick_finish_hier(const DevScene& sc, const PickSetup& ps, int edge_id, Real edge_weight, EdgePick& pk) {
    const EdgeCtx& c = ps.c;
    if (edge_id == -1 || edge_weight <= 0) return false;
    const Edge& e = sc.edges[edge_id];
    if (!edge_is_silhouette(sc.shapes, c.pos, e)) return false;
    V3 a = mul(c.m_inv, edge_v0(sc.shapes, e) - c.pos), b = mul(c.m_inv, edge_v1(sc.shapes, e) - c.pos);
    if (a.z <= 0 && b.z <= 0) return false;
    if (a.z < 0) a = (a * b.z - b * a.z) / (b.z - a.z);
    if (b.z < 0) b = (a * b.z - b * a.z) / (b.z - a.z);
    V3 wt = normalize(b - a);
    Real l0 = dot(a, wt), l1 = dot(b, wt);
    V3 vo = a - l0 * wt;
    Real d = length(vo);
    auto I = [&](Real l) { return (l / (d * (d * d + l * l)) + atan(l / d) / (d * d)) * vo.z + (l * l / (d * (d * d + l * l))) * wt.z; };
    Real Il0 = I(l0), Il1 = I(l1);
    Real norm = Il1 - Il0;
    auto line_pdf = [&](Real l) {
        Real ds2 = d * d + l * l;
        return 2 * d * (vo + l * wt).z / (norm * ds2 * ds2);
    };
    // invert the line CDF by bisection-safeguarded Newton, src/edge.cpp:1618-1643
    Real lb = l0, ub = l1;
    if (lb > ub) {
        Real tmp = lb;
        lb = ub;
        ub = tmp;
    }
    Real l = Real(0.5) * (lb + ub);
    for (int it = 0; it < 20; it++) {
        if (!(l >= lb && l <= ub)) l = Real(0.5) * (lb + ub);
        Real value = (I(l) - Il0) / norm - ps.t_sel;
        if (fabs(value) < Real(1e-5) || it == 19) break;
        if (value > 0) ub = l; else lb = l;
        l -= value / line_pdf(l);
    }
    Real lpdf = line_pdf(l);
    if (!(lpdf > 0)) return false;
    pk.edge_id = edge_id;
    pk.flags = ps.flags;
    pk.w = (float)(edge_weight / (ps.m_pmf * lpdf) / ps.nee_pmf);
    pk.sample_p = mul(c.m, vo + l * wt);
    pk.mwt = mul(c.m, wt);
    return true;
}
RB_D bool secondary_edge_pick(const DevScene& sc, const VertexRec& cur, Sampler& smp, EdgePick& pk) {
    PickSetup ps;
    Ray nee;
    SurfacePoint lp;
    if (!pick_setup(sc, cur, smp, ps, &nee, &lp)) return false;
    if (!(ps.flags & 2)) {
        Real edge_weight = 0;
        int edge_id = sample_edge_hier(ps.c, ps.edge_sel, ps.resample, edge_weight);
        return pick_finish_hier(sc, ps, edge_id, edge_weight, pk);
    }
#if RB_LIGHT_TEX_KERNELS
    if (cur.light.rejected) return false; // (emission sampling rejected the light point: no shadow ray to gather along)
#endif
    Real edge_weight = 0;
    V3 sample_p = zero3(), mwt = zero3();
    int edge_id = sample_edge_gather(ps.c, nee, cur.light.isect, lp, ps.resample, edge_weight, sample_p, mwt);
    if (edge_id == -1 || edge_weight <= 0) return false;
    pk.edge_id = edge_id;
    pk.flags = ps.flags;
    pk.w = (float)(edge_weight / ps.nee_pmf);
    pk.sample_p = sample_p;
    pk.mwt = mwt;
    return true;
}
// `smp` must be positioned 4 dimensions after the start of this depth (both edge rays share the following light / bsdf
// samples); `d_color` is the raw d_image pixel.
RB_D void secondary_edge_shade(const DevScene& sc, const DevDScene& ds, const RenderParams& rp, const VertexRec& cur, int depth, Sampler smp, V3 d_color,
                               const EdgePick& pk, V3& d_position) {
    const Real weight = Real(1) / Real(rp.spp);
    const Real min_rough = cur.min_rough;
    const rb_shape& shape = sc.shapes[cur.isect.shape_id];
    const rb_material& mat = sc.materials[shape.material_id];
    RayDiff rd;
    SurfacePoint sp = make_surface_point(shape, cur.isect.tri_id, cur.ray, cur.rd_in, rd);
    V3 wi = -cur.ray.dir;
    const int edge_id = pk.edge_id;
    const bool diffuse_lobe = (pk.flags & 1) != 0, use_nee = (pk.flags & 2) != 0, diffuse_or_glossy = (pk.flags & 4) != 0;
    const V3 sample_p = pk.sample_p, mwt = pk.mwt;
    const Edge edge = sc.edges[edge_id];
    V3 v0 = edge_v0(sc.shapes, edge), v1 = edge_v1(sc.shapes, edge);
    // The two edge rays differ by 1e-5 / |sample_p| in direction -- ten to thirty fp32 ulps.  The reference builds them in double and
    // rounds to float once for Embree (src/edge.cpp:1670-1678, src/scene.cpp:559-566); so do we (in fp32, with 2-ulp division and
    // square root, the perturbation drowns in the rounding of the normalisations and the +nt / -nt sides stop being symmetric).
    D3 hp_d, sd_d;
    double plen_d;
    {
        D3 a = d3((double)v0.x - (double)sp.position.x, (double)v0.y - (double)sp.position.y, (double)v0.z - (double)sp.position.z);
        D3 b = d3((double)v1.x - (double)sp.position.x, (double)v1.y - (double)sp.position.y, (double)v1.z - (double)sp.position.z);
        hp_d = d3_normalize(d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x));
        plen_d = sqrt((double)sample_p.x * (double)sample_p.x + (double)sample_p.y * (double)sample_p.y + (double)sample_p.z * (double)sample_p.z);
        sd_d = d3((double)sample_p.x / plen_d, (double)sample_p.y / plen_d, (double)sample_p.z / plen_d);
    }
    const double offset_d = (double)1e-5f / plen_d;
    V3 hpn = mk3((Real)hp_d.x, (Real)hp_d.y, (Real)hp_d.z);
    Real plen = (Real)plen_d;
    V3 sdir = mk3((Real)sd_d.x, (Real)sd_d.y, (Real)sd_d.z);
    V3 f = bsdf_eval(mat, sp, wi, sdir, min_rough);
    if (sum(f) < Real(1e-6)) return;
    // ray differential of the two edge rays (src/edge.cpp:1703-1733)
    RayDiff rd_e;
    rd_e.org_dx = rd.org_dx;
    rd_e.org_dy = rd.org_dy;
    if (diffuse_lobe) {
        rd_e.dir_dx = rd_e.dir_dy = mk3(Real(0.03), Real(0.03), Real(0.03));
    } else {
        V3 h = normalize(wi + sdir);
        Real hz = dot(h, sp.shading_frame.n);
        V3 dmdx = sp.dn_dx * hz, dmdy = sp.dn_dy * hz;
        // (elementwise products, as in the reference: src/edge.cpp:1724-1730)
        V3 ddn_dx = rd.dir_dx * h - wi * dmdx, ddn_dy = rd.dir_dy * h - wi * dmdy;
        rd_e.dir_dx = rd.dir_dx - 2 * (-dot(wi, h) * sp.dn_dx + ddn_dx * h);
        rd_e.dir_dy = rd.dir_dy - 2 * (-dot(wi, h) * sp.dn_dy + ddn_dy * h);
    }
    V3 nt = cur.thr * f * d_color * (Real)pk.w;
    // advance the sampler past this depth's 4 dimensions: both edge rays share the following light/bsdf samples
    Isect eis[2];
    SurfacePoint esp[2];
    Ray eray[2];
    bool hit[2];
    int light_id[2] = {-1, -1};
    for (int k = 0; k < 2; k++) {
        eray[k].org = sp.position;
        {
            double sg = k == 0 ? offset_d : -offset_d;
            D3 dk = d3_normalize(d3(sd_d.x + sg * hp_d.x, sd_d.y + sg * hp_d.y, sd_d.z + sg * hp_d.z));
            eray[k].dir = mk3((Real)dk.x, (Real)dk.y, (Real)dk.z);
        }
        eray[k].tmin = Real(1e-3) * plen;
        eray[k].tmax = INFINITY;
        eis[k] = no_isect();
        hit[k] = closest_hit(sc, eray[k], eis[k]);
        if (hit[k]) {
            RayDiff tmp;
            esp[k] = make_surface_point(sc.shapes[eis[k].shape_id], eis[k].tri_id, eray[k], rd_e, tmp);
            light_id[k] = sc.shapes[eis[k].shape_id].light_id;
        }
    }
    bool hit_light = light_id[0] != -1 || light_id[1] != -1;
    Real scale = 1;
    if (use_nee) {
        scale = hit_light ? Real(0.5) : Real(0);
    } else if (hit_light && diffuse_or_glossy) {
        scale = Real(0.5);
    }
    if (scale == 0) return;
    V3 dp = zero3(), dv0 = zero3(), dv1 = zero3();
    for (int k = 0; k < 2; k++) {
        if (!hit[k]) continue;
        V3 thr = (k == 0 ? nt : -nt) * scale;
        // geometry term and Jacobians (Eq. 15-18), src/edge.cpp:1857-1898
        V3 dir = esp[k].position - sp.position;
        Real dist_sq = length_sq(dir);
        if (dist_sq < Real(1e-8)) continue;
        V3 ndir = dir / sqrt(dist_sq);
        Real G = fabs(dot(esp[k].geom_normal, ndir)) / dist_sq;
        V3 ij = intersect_jacobian(sp.position, sample_p, esp[k].position, esp[k].geom_normal, mwt);
        Real line_jac = length(ij) / length(cross(esp[k].geom_normal, hpn));
        Real dirac_jac = length(cross(v0 - sp.position, v1 - sp.position));
        thr *= G * (line_jac / dirac_jac);
        if (!finite3(thr)) continue;
        // radiance carried by this side: emission at the hit + the remaining bounces
        Real contrib = sum(weight * thr * hit_emission(sc, eis[k], esp[k], -eray[k].dir));
        Sampler sub = smp;
        V3 Lb = trace_bounces<false>(sc, sub, eray[k], rd_e, eis[k], thr, min_rough, depth + 1, rp.max_bounces, nullptr, 0, nullptr);
        contrib += sum(weight * Lb);
        if (contrib == 0) continue;
        // Eq. 16 (with the errata), src/edge.cpp:2020-2033
        V3 x = esp[k].position, p = sp.position;
        V3 d0 = v0 - p, d1 = v1 - p;
        dp += (cross(d1, d0) + cross(x - p, d1) + cross(d0, x - p)) * contrib;
        dv0 += cross(d1, x - p) * contrib;
        dv1 += cross(x - p, d0) * contrib;
    }
    d_position += dp;
    float* dv = ds.shapes[edge.shape_id].vertices;
    if (dv) {
        agg_add3(dv + 3 * (size_t)edge.v0, dv0);
        agg_add3(dv + 3 * (size_t)edge.v1, dv1);
    }
}

// pick + shade for one vertex (host-compiled emulator; the kernels run the two steps separately)
RB_D void secondary_edge_sample(const DevScene& sc, const DevDScene& ds, const RenderParams& rp, const VertexRec& cur, int depth, Sampler smp,
                                V3 d_color, V3& d_position) {
    EdgePick pk;
    if (!secondary_edge_pick(sc, cur, smp, pk)) return;
    secondary_edge_shade(sc, ds, rp, cur, depth, smp, d_color, pk, d_position);
}
