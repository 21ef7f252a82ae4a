// Mesh-edge helpers shared by the scene build (host) and the edge-sampling kernels (device).
//   Edge, get_v0/v1, get_non_shared_v0/v1, is_silhouette     src/edge.h:13-204
//   clip_line (Cohen-Sutherland against the unit square)      src/line_clip.h:37-102
// All functions take an array of rb_shape whose pointers are valid in the calling address space
// (device pointers inside kernels, host mirrors during rb_scene_create).
#pragma once
#include "rb_camera.cuh"
#include "rb_shape.cuh"

RB_HD V3 edge_v0(const rb_shape* shapes, const Edge& e) { return shape_vertex(shapes[e.shape_id], e.v0); }
RB_HD V3 edge_v1(const rb_shape* shapes, const Edge& e) { return shape_vertex(shapes[e.shape_id], e.v1); }
RB_HD bool same_pos(V3 a, V3 b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
// third vertex of face f0 (by index), src/edge.h:84-94
RB_HD V3 edge_opposite0(const rb_shape* shapes, const Edge& e) {
    int idx[3];
    shape_tri(shapes[e.shape_id], e.f0, idx);
    for (int i = 0; i < 3; i++)
        if (idx[i] != e.v0 && idx[i] != e.v1) return shape_vertex(shapes[e.shape_id], idx[i]);
    return edge_v0(shapes, e);
}
// third vertex of face f1 (by POSITION, because f1 may come from a duplicated seam edge), src/edge.h:96-121
RB_HD V3 edge_opposite1(const rb_shape* shapes, const Edge& e) {
    int idx[3];
    shape_tri(shapes[e.shape_id], e.f1, idx);
    V3 a = edge_v0(shapes, e), b = edge_v1(shapes, e);
    for (int i = 0; i < 3; i++) {
        V3 v = shape_vertex(shapes[e.shape_id], idx[i]);
        if (!same_pos(v, a) && !same_pos(v, b)) return v;
    }
    return b;
}
RB_HD bool edge_is_silhouette(const rb_shape* shapes, V3 p, const Edge& e) {
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    if (e.f0 == -1 || e.f1 == -1) {
        if (e.f0 != -1) {
            V3 o = edge_opposite0(shapes, e);
            if (length_sq(cross(v0 - o, v1 - o)) < Real(1e-20)) return false;
        }
        if (e.f1 != -1) {
            V3 o = edge_opposite1(shapes, e);
            if (length_sq(cross(v1 - o, v0 - o)) < Real(1e-20)) return false;
        }
        return true;
    }
    V3 o0 = edge_opposite0(shapes, e), o1 = edge_opposite1(shapes, e);
    V3 n0 = cross(v0 - o0, v1 - o0), n1 = cross(v1 - o1, v0 - o1);
    Real l0 = length_sq(n0), l1 = length_sq(n1);
    if (l0 < Real(1e-20) || l1 < Real(1e-20)) return false;
    n0 = n0 / sqrt(l0);
    n1 = n1 / sqrt(l1);
    if (shapes[e.shape_id].normals == nullptr) {
        // without interpolated normals every non-flat edge can be a silhouette
        return !(dot(n0, n1) >= 1 - Real(1e-6));
    }
    bool f0 = dot(p - o0, n0) > 0, f1 = dot(p - o1, n1) > 0;
    return (f0 && !f1) || (!f0 && f1);
}
// dihedral filter used when the edge list is built, src/edge.cpp:168-184
RB_HD bool edge_is_flat(const rb_shape* shapes, const Edge& e) {
    if (e.f0 == -1 || e.f1 == -1) return false;
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    V3 o0 = edge_opposite0(shapes, e), o1 = edge_opposite1(shapes, e);
    V3 n0 = normalize(cross(v0 - o0, v1 - o0)), n1 = normalize(cross(v1 - o1, v0 - o1));
    return dot(n0, n1) >= (1 - Real(1e-6));
}

RB_HD int clip_code(V2 v) {
    int c = 0;
    if (v.x < 0) c |= 1; else if (v.x > 1) c |= 2;
    if (v.y < 0) c |= 4; else if (v.y > 1) c |= 8;
    return c;
}
RB_HD bool clip_line_unit(V2 v0, V2 v1, V2& a, V2& b) {
    int c0 = clip_code(v0), c1 = clip_code(v1);
    a = v0;
    b = v1;
    for (int it = 0; it < 16; it++) {
        if (!(c0 | c1)) return true;
        if (c0 & c1) return false;
        int co = c0 ? c0 : c1;
        V2 v = zero2();
        if (co & 8) {
            v.x = a.x + (b.x - a.x) * (1 - a.y) / (b.y - a.y);
            v.y = 1;
        } else if (co & 4) {
            v.x = a.x + (b.x - a.x) * (0 - a.y) / (b.y - a.y);
            v.y = 0;
        } else if (co & 2) {
            v.y = a.y + (b.y - a.y) * (1 - a.x) / (b.x - a.x);
            v.x = 1;
        } else if (co & 1) {
            v.y = a.y + (b.y - a.y) * (0 - a.x) / (b.x - a.x);
            v.x = 0;
        }
        if (co == c0) {
            a = v;
            c0 = clip_code(a);
        } else {
            b = v;
            c1 = clip_code(b);
        }
    }
    return false;
}

// Clip against the image grown by filter_grow(cam) pixels on each side: the unit-square clip in the coordinates where that rectangle
// is the unit square.  Without growth (every filter up to 1 pixel wide) it is clip_line_unit itself.
RB_HD bool clip_line_filter(const DevCamera& cam, V2 v0, V2 v1, V2& a, V2& b) {
    const double g = filter_grow(cam);
    if (g == 0) return clip_line_unit(v0, v1, a, b);
    const Real gx = (Real)(g / cam.width), gy = (Real)(g / cam.height), sx = 1 + 2 * gx, sy = 1 + 2 * gy;
    if (!clip_line_unit(mk2((v0.x + gx) / sx, (v0.y + gy) / sy), mk2((v1.x + gx) / sx, (v1.y + gy) / sy), a, b)) return false;
    a = mk2(a.x * sx - gx, a.y * sy - gy);
    b = mk2(b.x * sx - gx, b.y * sy - gy);
    return true;
}
// Weight of an edge in the primary-edge distribution (src/edge.cpp:186-214): its screen-space length after clipping to the image (grown
// by the pixel filter's reach) if it is a silhouette seen from the camera, else 0.
// With a thin lens: positive for every edge that is a silhouette from some lens point and whose projection from that point meets the
// image (only that makes the lens estimator unbiased).  On the film, the projection of camera-space P from lens point L is its projection
// from the centre moved by the intrinsic scaling of L (1 / f - 1 / P.z), at most m(P.z) = r |1 / f - 1 / P.z| times that scaling in
// screen units; 1 / z is monotone along a segment, so the near-clipped ends bound it.  The weight is the centre projection clipped to
// the image grown by the larger bound, plus the two bounds.  The silhouette test keeps the edge unless the signed distance of the lens
// point to each face plane, s(o) +- r |(n.ex, n.ey)| over the disc, stays strictly on one side and on the same side for both faces.
RB_HD bool edge_is_lens_silhouette(const DevCamera& cam, const rb_shape* shapes, V3 org, const Edge& e) {
    if (e.f0 == -1 || e.f1 == -1 || shapes[e.shape_id].normals == nullptr) return edge_is_silhouette(shapes, org, e);
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    V3 o0 = edge_opposite0(shapes, e), o1 = edge_opposite1(shapes, e);
    V3 n0 = cross(v0 - o0, v1 - o0), n1 = cross(v1 - o1, v0 - o1);
    Real l0 = length_sq(n0), l1 = length_sq(n1);
    if (l0 < Real(1e-20) || l1 < Real(1e-20)) return false;
    n0 = n0 / sqrt(l0);
    n1 = n1 / sqrt(l1);
    const V3 ex = mk3((Real)cam.c2w[0], (Real)cam.c2w[4], (Real)cam.c2w[8]), ey = mk3((Real)cam.c2w[1], (Real)cam.c2w[5], (Real)cam.c2w[9]);
    const Real r = (Real)cam.lens_radius;
    const Real s0 = dot(org - o0, n0), s1 = dot(org - o1, n1);
    const Real h0 = r * sqrt(rb_sq(dot(n0, ex)) + rb_sq(dot(n0, ey))), h1 = r * sqrt(rb_sq(dot(n1, ex)) + rb_sq(dot(n1, ey)));
    const bool front = s0 - h0 > 0 && s1 - h1 > 0, back = s0 + h0 < 0 && s1 + h1 < 0;
    return !(front || back);
}
// Screen-space radius of the circle of confusion at camera depth z (the larger of its x and y extents).
RB_HD Real lens_confusion_radius(const DevCamera& cam, Real z) {
    const Real aspect = Real(cam.width) / Real(cam.height), k = (Real)fabs(cam.intr[8]);
    const Real sx = Real(0.5) * ((Real)fabs(cam.intr[0]) + (Real)fabs(cam.intr[1])) / k, sy = Real(0.5) * aspect * ((Real)fabs(cam.intr[3]) + (Real)fabs(cam.intr[4])) / k;
    return (Real)cam.lens_radius * (Real)fabs(Real(1) / (Real)cam.focus_distance - Real(1) / z) * (sx > sy ? sx : sy);
}
RB_HD double primary_edge_weight_lens(const DevCamera& cam, const rb_shape* shapes, const Edge& e, V3 org) {
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    M4 W = cam_m4(cam.w2c);
    V3 a = xfm_point(W, v0), b = xfm_point(W, v1);
    const Real cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return 0;
    const Real za = a.z < cn ? cn : a.z, zb = b.z < cn ? cn : b.z;
    const Real m0 = lens_confusion_radius(cam, za), m1 = lens_confusion_radius(cam, zb), g = m0 > m1 ? m0 : m1;
    V2 p0, p1, c0, c1;
    if (!cam_project(cam, v0, v1, p0, p1)) return 0;
    if (!clip_line_unit(mk2((p0.x + g) / (1 + 2 * g), (p0.y + g) / (1 + 2 * g)), mk2((p1.x + g) / (1 + 2 * g), (p1.y + g) / (1 + 2 * g)), c0, c1)) return 0;
    if (!edge_is_lens_silhouette(cam, shapes, org, e)) return 0;
    return (double)(length(c1 - c0) * (1 + 2 * g) + m0 + m1);
}
RB_HD double primary_edge_weight(const DevCamera& cam, const rb_shape* shapes, const Edge& e) {
    double iw = 1.0 / cam.c2w[15];
    if (RB_CAM_LENS(cam)) return primary_edge_weight_lens(cam, shapes, e, mk3((Real)(cam.c2w[3] * iw), (Real)(cam.c2w[7] * iw), (Real)(cam.c2w[11] * iw)));
    V3 org = mk3((Real)(cam.c2w[3] * iw), (Real)(cam.c2w[7] * iw), (Real)(cam.c2w[11] * iw));
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    V2 p0, p1, c0, c1;
    if (cam_project(cam, v0, v1, p0, p1) && clip_line_filter(cam, p0, p1, c0, c1) && edge_is_silhouette(shapes, org, e)) return length(c1 - c0);
    return 0;
}
