// Camera: primary ray generation (with finite-difference ray differentials), screen projection of
// edges, and their adjoints.
//   sample_primary            src/camera.h:121-197       primary_ray_sampler   src/camera.cpp:8-43
//   d_sample_primary_ray      src/camera.h:199-500       camera_to_screen      src/camera.h:508-559
//   project / d_project       src/camera.h:561-591, :731-830   in_screen       src/camera.h:1049-1067
// The forward ray is evaluated in double from the float camera parameters exactly like the reference
// (Real == double there) and rounded to fp32 once, so the rays entering the fp32 BVH traversal are the
// same fp32 rays the reference hands to Embree (src/scene.cpp:556-567).
// Supported: perspective, orthographic, fisheye (equi-angular) and panorama cameras without distortion parameters
// (Brown-Conrady distortion is rejected by rb_scene_create).  A fisheye sample outside the unit disc gives a NULL ray
// (zero origin and direction, src/camera.h:160-162): it is traced by nobody and contributes nothing.
#pragma once
#include "rb_atomic.cuh"
#include "rb_types.cuh"

struct D3 {
    double x, y, z;
};
RB_HD D3 d3(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
RB_HD D3 d3_normalize(D3 v) {
    double l = sqrt(v.x * v.x + v.y * v.y + v.z * v.z);
    if (l <= 0) return d3(0, 0, 0);
    return d3(v.x / l, v.y / l, v.z / l);
}

struct D2 {
    double x, y;
};
RB_HD D2 d2(double x, double y) { D2 r; r.x = x; r.y = y; return r; }

// ---- Brown-Conrady lens distortion on normalised screen coordinates (src/camera_distortion.h) ----
// distort: undistorted -> distorted position; optional forward-mode rows d(out.x)/d(pos), d(out.y)/d(pos).
RB_HD D2 cam_distort_impl(const DevCamera& cam, D2 pos, D2* dx_dpos, D2* dy_dpos) {
    const double* k = cam.distortion;
    const double p0 = k[6], p1 = k[7];
    double x = 2.0 * (pos.x - 0.5), y = 2.0 * (pos.y - 0.5);
    double r = sqrt(x * x + y * y), r2 = r * r, r4 = r2 * r2, r6 = r4 * r2;
    double num = 1 + k[0] * r2 + k[1] * r4 + k[2] * r6, den = 1 + k[3] * r2 + k[4] * r4 + k[5] * r6, rr = num / den;
    double xx = x * rr + 2 * p0 * x * y + p1 * (r2 + 2 * x * x), yy = y * rr + p0 * (r2 + 2 * y * y) + 2 * p1 * x * y;
    if (dx_dpos != nullptr && dy_dpos != nullptr) {
        D2 dx = d2(2, 0), dy = d2(0, 2); // d(x)/d(pos), d(y)/d(pos)
        // d(r2) = 2 (x dx + y dy), formed without dividing by r: finite at the centre, where r = 0 (the reference's d(r) / r is NaN there)
        D2 dr2 = d2(2 * (dx.x * x + dy.x * y), 2 * (dx.y * x + dy.y * y)), dr4 = d2(2 * r2 * dr2.x, 2 * r2 * dr2.y);
        D2 dr6 = d2(r4 * dr2.x + dr4.x * r2, r4 * dr2.y + dr4.y * r2);
        D2 dnum = d2(k[0] * dr2.x + k[1] * dr4.x + k[2] * dr6.x, k[0] * dr2.y + k[1] * dr4.y + k[2] * dr6.y);
        D2 dden = d2(k[3] * dr2.x + k[4] * dr4.x + k[5] * dr6.x, k[3] * dr2.y + k[4] * dr4.y + k[5] * dr6.y);
        D2 drr = d2((dnum.x * den - num * dden.x) / (den * den), (dnum.y * den - num * dden.y) / (den * den));
        D2 dxx = d2(dx.x * rr + x * drr.x + 2 * p0 * (dx.x * y + x * dy.x) + p1 * (dr2.x + 4 * dx.x * x),
                    dx.y * rr + x * drr.y + 2 * p0 * (dx.y * y + x * dy.y) + p1 * (dr2.y + 4 * dx.y * x));
        D2 dyy = d2(dy.x * rr + y * drr.x + p0 * (dr2.x + 4 * dy.x * y) + 2 * p1 * (dx.x * y + x * dy.x),
                    dy.y * rr + y * drr.y + p0 * (dr2.y + 4 * dy.y * y) + 2 * p1 * (dx.y * y + x * dy.y));
        *dx_dpos = d2(dxx.x / 2, dxx.y / 2);
        *dy_dpos = d2(dyy.x / 2, dyy.y / 2);
    }
    return d2((xx + 1) / 2, (yy + 1) / 2);
}
RB_HD D2 cam_distort(const DevCamera& cam, D2 pos, D2* dx_dpos = nullptr, D2* dy_dpos = nullptr) {
    if (!RB_CAM_DISTORT(cam)) return pos;
    return cam_distort_impl(cam, pos, dx_dpos, dy_dpos);
}
// Adjoint of cam_distort; d_params (8 doubles, may be null) receives the parameter gradient.
RB_HD void d_cam_distort_impl(const DevCamera& cam, D2 pos, D2 d_out, double* d_params, D2& d_pos) {
    const double* k = cam.distortion;
    const double p0 = k[6], p1 = k[7];
    double x = 2.0 * (pos.x - 0.5), y = 2.0 * (pos.y - 0.5);
    double r = sqrt(x * x + y * y), r2 = r * r, r4 = r2 * r2, r6 = r4 * r2;
    double num = 1 + k[0] * r2 + k[1] * r4 + k[2] * r6, den = 1 + k[3] * r2 + k[4] * r4 + k[5] * r6, rr = num / den;
    double d_k[6] = {0, 0, 0, 0, 0, 0}, d_p[2] = {0, 0};
    double d_xx = d_out.x / 2, d_yy = d_out.y / 2;
    double d_x = d_xx * (rr + 2 * p0 * y + 4 * p1 * x), d_rr = d_xx * x, d_y = d_xx * 2 * p0 * x;
    d_p[0] += d_xx * 2 * x * y;
    d_p[1] += d_xx * (r2 + 2 * x * x);
    double d_r2 = d_xx * p1;
    d_y += d_yy * (rr + 4 * p0 * y + 2 * p1 * x);
    d_rr += d_yy * y;
    d_p[0] += d_yy * (r2 + 2 * y * y);
    d_r2 += d_yy * p0;
    d_p[1] += d_yy * 2 * x * y;
    d_x += d_yy * 2 * p1 * y;
    double d_num = d_rr / den, d_den = -d_rr * rr / den;
    d_k[0] += d_num * r2; d_r2 += d_num * k[0];
    d_k[1] += d_num * r4; double d_r4 = d_num * k[1];
    d_k[2] += d_num * r6; double d_r6 = d_num * k[2];
    d_k[3] += d_den * r2; d_r2 += d_den * k[3];
    d_k[4] += d_den * r4; d_r4 += d_den * k[4];
    d_k[5] += d_den * r6; d_r6 += d_den * k[5];
    d_r4 += d_r6 * r2;
    d_r2 += d_r6 * r2; // (r2 where r4 belongs: as in the reference :160)
    d_r2 += 2 * d_r4 * r2;
    d_x += 2 * d_r2 * x; // (d(r2)/dx = 2 x, without the reference's division by r, which is NaN at the centre)
    d_y += 2 * d_r2 * y;
    d_pos.x += d_x * 2;
    d_pos.y += d_y * 2;
    if (d_params != nullptr) {
        for (int i = 0; i < 6; i++) d_params[i] += d_k[i];
        d_params[6] += d_p[0];
        d_params[7] += d_p[1];
    }
}
RB_HD void d_cam_distort(const DevCamera& cam, D2 pos, D2 d_out, double* d_params, D2& d_pos) {
    if (!RB_CAM_DISTORT(cam)) {
        d_pos = d_out; // (assignment, as in the reference :96-99)
        return;
    }
    d_cam_distort_impl(cam, pos, d_out, d_params, d_pos);
}
// distorted -> undistorted position by Gauss-Newton (src/camera_distortion.h:171-198)
RB_HD D2 cam_inverse_distort_impl(const DevCamera& cam, D2 pos) {
    D2 result = pos;
    double err = 0;
    int iter = 0;
    do {
        D2 jx, jy;
        D2 next = cam_distort(cam, result, &jx, &jy);
        D2 res = d2(next.x - pos.x, next.y - pos.y);
        err = fabs(res.x) + fabs(res.y);
        double inv_det = 1 / (jx.x * jy.y - jx.y * jy.x);
        result = d2(result.x - inv_det * (jy.y * res.x - jx.y * res.y), result.y - inv_det * (-jy.x * res.x + jx.x * res.y));
    } while (err > 1e-3 && iter++ < 1000);
    return result;
}
RB_HD D2 cam_inverse_distort(const DevCamera& cam, D2 pos) {
    if (!RB_CAM_DISTORT(cam)) return pos;
    return cam_inverse_distort_impl(cam, pos);
}
// Adjoint through the implicit function theorem (src/camera_distortion.h:200-258)
RB_HD void d_cam_inverse_distort_impl(const DevCamera& cam, D2 pos, D2 d_out, double* d_params, D2& d_pos) {
    D2 result = cam_inverse_distort(cam, pos);
    D2 fx, fy;
    cam_distort(cam, result, &fx, &fy);
    double inv_det = 1 / (fx.x * fy.y - fx.y * fy.x);
    D2 d_result = d2(-inv_det * (fy.y * d_out.x - fy.x * d_out.y), -inv_det * (-fx.y * d_out.x + fx.x * d_out.y));
    D2 unused = d2(0, 0);
    if (d_params != nullptr) d_cam_distort(cam, result, d_result, d_params, unused);
    d_pos.x -= d_result.x;
    d_pos.y -= d_result.y;
}
RB_HD void d_cam_inverse_distort(const DevCamera& cam, D2 pos, D2 d_out, double* d_params, D2& d_pos) {
    if (!RB_CAM_DISTORT(cam)) {
        d_pos = d_out;
        return;
    }
    d_cam_inverse_distort_impl(cam, pos, d_out, d_params, d_pos);
}

RB_HD void cam_sample_primary_any(const DevCamera& cam, double sx_, double sy_, D3& org, D3& dir) {
    D2 undist = cam_inverse_distort(cam, d2(sx_, sy_)); // (identity without a lens model)
    const double sx = undist.x, sy = undist.y;
    const double* C = cam.c2w;
    const double* I = cam.intr_inv;
    double aspect = double(cam.width) / double(cam.height);
    if (cam.type == RB_CAMERA_PERSPECTIVE) {
        // org = xfm_point(c2w, 0)
        double iw = 1.0 / C[15];
        org = d3(C[3] * iw, C[7] * iw, C[11] * iw);
        double px = (sx - 0.5) * 2.0, py = (sy - 0.5) * (-2.0) / aspect, pz = 1.0;
        D3 d = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
        D3 n = d3_normalize(d);
        D3 w = d3(C[0] * n.x + C[1] * n.y + C[2] * n.z, C[4] * n.x + C[5] * n.y + C[6] * n.z, C[8] * n.x + C[9] * n.y + C[10] * n.z);
        dir = d3_normalize(w);
    } else if (cam.type == RB_CAMERA_FISHEYE || cam.type == RB_CAMERA_PANORAMA) {
        const double pi = 3.14159265358979323846;
        double lx, ly, lz;
        if (cam.type == RB_CAMERA_FISHEYE) { // equi-angular: radius on the unit disc -> polar angle
            double x = 2.0 * (sx - 0.5), y = 2.0 * (sy - 0.5);
            if (x * x + y * y > 1.0) {
                org = d3(0, 0, 0);
                dir = d3(0, 0, 0);
                return;
            }
            double r = sqrt(x * x + y * y), phi = atan2(y, x), theta = r * (pi / 2);
            lx = -cos(phi) * sin(theta);
            ly = -sin(phi) * sin(theta);
            lz = cos(theta);
        } else { // latitude-longitude
            double theta = pi * sy, phi = 2 * pi * sx;
            lx = cos(phi) * sin(theta);
            ly = cos(theta);
            lz = sin(phi) * sin(theta);
        }
        double iw = 1.0 / C[15];
        org = d3(C[3] * iw, C[7] * iw, C[11] * iw);
        dir = d3_normalize(d3(C[0] * lx + C[1] * ly + C[2] * lz, C[4] * lx + C[5] * ly + C[6] * lz, C[8] * lx + C[9] * ly + C[10] * lz));
    } else { // orthographic
        double px = (sx - 0.5) * 2.0, py = (sy - 0.5) * (-2.0) / aspect, pz = 0.0;
        D3 l = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
        double tx = C[0] * l.x + C[1] * l.y + C[2] * l.z + C[3];
        double ty = C[4] * l.x + C[5] * l.y + C[6] * l.z + C[7];
        double tz = C[8] * l.x + C[9] * l.y + C[10] * l.z + C[11];
        double tw = C[12] * l.x + C[13] * l.y + C[14] * l.z + C[15];
        double iw = 1.0 / tw;
        org = d3(tx * iw, ty * iw, tz * iw);
        dir = d3_normalize(d3(C[2], C[6], C[10]));
    }
}

// ---- thin lens (rb_camera::lens_radius > 0, perspective cameras without distortion only; DESIGN.md "thin-lens camera") ----
// A lens sample is the point `lu` of the unit disc; the lens point is L = lens_radius * (lu.x, lu.y, 0) in camera space.
// Shirley-Chiu concentric map of [0, 1)^2 onto the unit disc: uniform, and continuous inside each of its four wedges.
RB_HD D2 concentric_disc(double u1, double u2) {
    const double a = 2.0 * u1 - 1.0, b = 2.0 * u2 - 1.0;
    if (a == 0.0 && b == 0.0) return d2(0, 0);
    const double quarter_pi = 0.78539816339744830962;
    double r, phi;
    if (a * a > b * b) {
        r = a;
        phi = quarter_pi * (b / a);
    } else {
        r = b;
        phi = 2.0 * quarter_pi - quarter_pi * (a / b);
    }
    return d2(r * cos(phi), r * sin(phi));
}
// Ray of film position (sx, sy) through lens point lu: from L towards F = d f / d.z, the point of the focal plane z = f on the pinhole
// ray d = intr_inv (px, py, 1).
RB_HD void cam_sample_lens(const DevCamera& cam, double sx, double sy, D2 lu, D3& org, D3& dir) {
    const double* C = cam.c2w;
    const double* I = cam.intr_inv;
    double aspect = double(cam.width) / double(cam.height);
    double px = (sx - 0.5) * 2.0, py = (sy - 0.5) * (-2.0) / aspect, pz = 1.0;
    D3 d = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
    const double t = cam.focus_distance / d.z, lx = cam.lens_radius * lu.x, ly = cam.lens_radius * lu.y;
    D3 n = d3_normalize(d3(d.x * t - lx, d.y * t - ly, d.z * t));
    double iw = 1.0 / (C[12] * lx + C[13] * ly + C[15]);
    org = d3((C[0] * lx + C[1] * ly + C[3]) * iw, (C[4] * lx + C[5] * ly + C[7]) * iw, (C[8] * lx + C[9] * ly + C[11]) * iw);
    D3 w = d3(C[0] * n.x + C[1] * n.y + C[2] * n.z, C[4] * n.x + C[5] * n.y + C[6] * n.z, C[8] * n.x + C[9] * n.y + C[10] * n.z);
    dir = d3_normalize(w);
}

// The common camera (pinhole, no lens model) has its own short path; everything else goes through the general one.  `lu` is the lens
// sample of a camera with a lens, and unused otherwise.
RB_HD void cam_sample_primary(const DevCamera& cam, double sx, double sy, D3& org, D3& dir, D2 lu = D2{0, 0}) {
    if (RB_CAM_GENERAL(cam)) {
        cam_sample_primary_any(cam, sx, sy, org, dir);
        return;
    }
    if (RB_CAM_LENS(cam)) {
        cam_sample_lens(cam, sx, sy, lu, org, dir);
        return;
    }
    const double* C = cam.c2w;
    const double* I = cam.intr_inv;
    double aspect = double(cam.width) / double(cam.height);
    double iw = 1.0 / C[15];
    org = d3(C[3] * iw, C[7] * iw, C[11] * iw);
    double px = (sx - 0.5) * 2.0, py = (sy - 0.5) * (-2.0) / aspect, pz = 1.0;
    D3 d = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
    D3 n = d3_normalize(d);
    D3 w = d3(C[0] * n.x + C[1] * n.y + C[2] * n.z, C[4] * n.x + C[5] * n.y + C[6] * n.z, C[8] * n.x + C[9] * n.y + C[10] * n.z);
    dir = d3_normalize(w);
}

RB_HD Ray make_ray(D3 o, D3 d) {
    Ray r;
    r.org = mk3((Real)o.x, (Real)o.y, (Real)o.z);
    r.dir = mk3((Real)d.x, (Real)d.y, (Real)d.z);
    r.tmin = Real(1e-3);
    r.tmax = INFINITY;
    return r;
}

// Primary ray + ray differential at normalised screen position (sx, sy).
// With a lens all three rays leave the same lens point.
RB_HD void cam_primary_ray(const DevCamera& cam, double sx, double sy, Ray& ray, RayDiff& rd, D2 lu = D2{0, 0}) {
    D3 o, d, ox, dx, oy, dy;
    cam_sample_primary(cam, sx, sy, o, d, lu);
    const double delta = 1e-3;
    cam_sample_primary(cam, sx + delta, sy, ox, dx, lu);
    cam_sample_primary(cam, sx, sy + delta, oy, dy, lu);
    double psx = 0.5 / cam.width, psy = 0.5 / cam.height;
    ray = make_ray(o, d);
    rd.org_dx = mk3((Real)(psx * (ox.x - o.x) / delta), (Real)(psx * (ox.y - o.y) / delta), (Real)(psx * (ox.z - o.z) / delta));
    rd.org_dy = mk3((Real)(psy * (oy.x - o.x) / delta), (Real)(psy * (oy.y - o.y) / delta), (Real)(psy * (oy.z - o.z) / delta));
    rd.dir_dx = mk3((Real)(psx * (dx.x - d.x) / delta), (Real)(psx * (dx.y - d.y) / delta), (Real)(psx * (dx.z - d.z) / delta));
    rd.dir_dy = mk3((Real)(psy * (dy.x - d.x) / delta), (Real)(psy * (dy.y - d.y) / delta), (Real)(psy * (dy.z - d.z) / delta));
}

RB_HD M4 cam_m4(const double* a) {
    M4 r;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) r.m[i][j] = (Real)a[4 * i + j];
    return r;
}
RB_HD M3 cam_m3(const double* a) {
    M3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[i][j] = (Real)a[3 * i + j];
    return r;
}

// Per-thread camera-gradient accumulator.  The reference does one atomic per scalar per pixel into the same
// <= 30 addresses (src/camera.h:244-259) -- its worst contention point.  Here every thread owns a strided
// column in shared memory; the block reduces once at kernel end and issues one double atomic per scalar.
// Layout (RB_CAM_ACC floats): [0..15] d_cam_to_world, [16..31] d_world_to_cam, [32..40] d_intr_inv, [41..49] d_intr,
// [50..57] d_distortion, and with a lens [58] d_lens_radius, [59] d_focus_distance: cam_acc_count(cam) floats in all.
// Deterministic mode (rb_kernels_det.cu) keeps one exact accumulator (rb_exact.cuh) per scalar for the whole block instead: each
// (float) contribution goes there, the block flushes them into the global exact accumulators at kernel end.
#define RB_CAM_ACC 58
#define RB_CAM_ACC_LENS 60
RB_HD int cam_acc_count(const DevCamera& cam) { return RB_CAM_LENS(cam) ? RB_CAM_ACC_LENS : RB_CAM_ACC; }
struct CamAcc {
#if defined(RB_DETERMINISTIC) && !defined(RB_CPU_EMU)
    long long* exact; // shared memory, [RB_CAM_ACC][RB_EXACT_WORDS]
    RB_D void add(int k, Real v) { exact_agg_add(exact + k * RB_EXACT_WORDS, (float)v); }
#else
    float* base; // shared memory, element k of this thread at base[k * stride]
    int stride;
#ifdef RB_CPU_EMU
    long long* exact = nullptr; // the emulator's deterministic mode: host exact accumulators, [RB_CAM_ACC][RB_EXACT_WORDS]
    RB_D void add(int k, Real v) {
        if (exact) exact_add_serial(exact + k * RB_EXACT_WORDS, (float)v);
        else base[k * stride] += (float)v;
    }
#else
    RB_D void add(int k, Real v) { base[k * stride] += (float)v; }
#endif
#endif
    RB_D void add_c2w(const M4& d) {
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++)
                if (d.m[i][j] != 0) add(4 * i + j, d.m[i][j]);
    }
    RB_D void add_w2c(const M4& d) {
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++)
                if (d.m[i][j] != 0) add(16 + 4 * i + j, d.m[i][j]);
    }
    RB_D void add_intr_inv(const M3& d) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) add(32 + 3 * i + j, d.m[i][j]);
    }
    RB_D void add_intr(const M3& d) {
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) add(41 + 3 * i + j, d.m[i][j]);
    }
    RB_D void add_distortion(const double* d) {
        for (int i = 0; i < 8; i++)
            if (d[i] != 0) add(50 + i, (Real)d[i]);
    }
    RB_D void add_lens(Real d_radius, Real d_focus) {
        if (d_radius != 0) add(58, d_radius);
        if (d_focus != 0) add(59, d_focus);
    }
};

// Adjoint of cam_sample_lens w.r.t. cam_to_world (the origin c2w (L, 1) included), intr_inv, lens_radius and focus_distance.
RB_D void d_cam_sample_lens(const DevCamera& cam, Real sx, Real sy, D2 lu, const DRay& d_ray, CamAcc& acc) {
    M4 C = cam_m4(cam.c2w);
    M3 I = cam_m3(cam.intr_inv);
    Real aspect = Real(cam.width) / Real(cam.height);
    const Real r = (Real)cam.lens_radius, f = (Real)cam.focus_distance, ux = (Real)lu.x, uy = (Real)lu.y;
    M4 d_C = zero_m4();
    M3 d_I = zero_m3();
    V3 L = mk3(r * ux, r * uy, 0);
    V3 pt = mk3((sx - Real(0.5)) * 2, (sy - Real(0.5)) * (-2) / aspect, 1);
    V3 d = mul(I, pt);
    Real t = f / d.z;
    V3 v = d * t - L;
    V3 n_dir = normalize(v);
    V3 world_dir = xfm_vector(C, n_dir);
    V3 d_world_dir = d_normalize(world_dir, d_ray.dir);
    V3 d_n_dir = zero3();
    d_xfm_vector(C, n_dir, d_world_dir, d_C, d_n_dir);
    V3 d_v = d_normalize(v, d_n_dir);
    V3 d_d = d_v * t;
    Real d_t = dot(d_v, d);
    V3 d_L = -d_v;
    Real d_f = d_t / d.z;
    d_d.z -= d_t * t / d.z;
    d_outer_acc(d_I, d_d, pt);
    d_xfm_point(C, L, d_ray.org, d_C, d_L);
    acc.add_intr_inv(d_I);
    acc.add_c2w(d_C);
    acc.add_lens(d_L.x * ux + d_L.y * uy, d_f);
}

// Adjoint of cam_sample_primary w.r.t. camera parameters (screen-position gradients are only needed for
// distortion / screen_gradient_image; the latter is accumulated by the caller through d_screen).
RB_D void d_cam_sample_primary_any(const DevCamera& cam, Real sx_, Real sy_, const DRay& d_ray, CamAcc& acc, V2* d_screen_out) {
    // With a lens model the ray is generated at the UNDISTORTED position and the adjoint w.r.t. that position flows back
    // through inverse_distort (parameters + original position), src/camera.h:205-206,262-277.
    const D2 spos = d2(sx_, sy_);
    const D2 undist = cam_inverse_distort(cam, spos);
    const Real sx = (Real)undist.x, sy = (Real)undist.y;
    V2 d_und = zero2();
    V2* d_screen = (RB_CAM_DISTORT(cam) || d_screen_out != nullptr) ? &d_und : nullptr;
    M4 C = cam_m4(cam.c2w);
    M3 I = cam_m3(cam.intr_inv);
    Real aspect = Real(cam.width) / Real(cam.height);
    M4 d_C = zero_m4();
    M3 d_I = zero_m3();
    if (cam.type == RB_CAMERA_PERSPECTIVE) {
        V3 pt = mk3((sx - Real(0.5)) * 2, (sy - Real(0.5)) * (-2) / aspect, 1);
        V3 dir = mul(I, pt);
        V3 n_dir = normalize(dir);
        V3 world_dir = xfm_vector(C, n_dir);
        V3 d_world_dir = d_normalize(world_dir, d_ray.dir);
        V3 d_n_dir = zero3();
        d_xfm_vector(C, n_dir, d_world_dir, d_C, d_n_dir);
        V3 d_dir = d_normalize(dir, d_n_dir);
        d_outer_acc(d_I, d_dir, pt);
        V3 d_cam_org = zero3();
        d_xfm_point(C, zero3(), d_ray.org, d_C, d_cam_org);
        if (d_screen != nullptr) {
            V3 d_pt = mul_t(d_dir, I);
            d_screen->x += d_pt.x * 2;
            d_screen->y += d_pt.y * (-2 / aspect);
        }
    } else if (cam.type == RB_CAMERA_FISHEYE || cam.type == RB_CAMERA_PANORAMA) {
        // src/camera.h:343-498: camera matrix always, the screen position only when somebody asks for it
        bool fish = cam.type == RB_CAMERA_FISHEYE;
        Real x = fish ? 2 * (sx - Real(0.5)) : sx, y = fish ? 2 * (sy - Real(0.5)) : sy;
        if (fish && x * x + y * y > 1) return;
        Real r = sqrt(x * x + y * y);
        Real phi = fish ? atan2(y, x) : Real(2 * RB_PI) * x, theta = fish ? r * Real(RB_PI) / 2 : Real(RB_PI) * y;
        Real sp = sin(phi), cp = cos(phi), st = sin(theta), ct = cos(theta);
        V3 dir = fish ? mk3(-cp * st, -sp * st, ct) : mk3(cp * st, ct, sp * st);
        V3 world_dir = xfm_vector(C, dir);
        V3 d_world_dir = d_normalize(world_dir, d_ray.dir);
        V3 d_dir = zero3();
        d_xfm_vector(C, dir, d_world_dir, d_C, d_dir);
        V3 d_cam_org = zero3();
        d_xfm_point(C, zero3(), d_ray.org, d_C, d_cam_org);
        if (d_screen != nullptr) {
            if (fish) {
                Real d_cp = d_dir.x * (-st), d_sp = d_dir.y * (-st), d_st = d_dir.x * (-cp) + d_dir.y * (-sp), d_ct = d_dir.z;
                Real d_phi = d_cp * (-sp) + d_sp * cp, d_theta = d_ct * (-st) + d_st * ct;
                Real d_r = d_theta * (Real(RB_PI) / 2);
                // at the centre phi is atan2(0, 0) = 0 and d_phi / r tends to -(pi / 2) d_dir.y: the limit of the two quotients below
                Real d_x = r > 0 ? d_phi * (-y / (x * x + y * y)) + d_r * (x / r) : d_r;
                Real d_y = r > 0 ? d_phi * (x / (x * x + y * y)) + d_r * (y / r) : -(Real(RB_PI) / 2) * d_dir.y;
                d_screen->x += 2 * d_x;
                d_screen->y += 2 * d_y;
            } else {
                Real d_cp = d_dir.x * st, d_sp = d_dir.z * st, d_st = d_dir.x * cp + d_dir.z * sp, d_ct = d_dir.y;
                Real d_phi = d_cp * (-sp) + d_sp * cp, d_theta = d_ct * (-st) + d_st * ct;
                d_screen->x += d_phi * Real(2 * RB_PI);
                d_screen->y += d_theta * Real(RB_PI);
            }
        }
    } else {
        // NOTE: the reference's adjoint uses pt.z = 1 here although the forward uses 0 (src/camera.h:283-285 vs :146-148);
        // reproduced for parity.
        V3 pt = mk3((sx - Real(0.5)) * 2, (sy - Real(0.5)) * (-2) / aspect, 1);
        V3 local_org = mul(I, pt);
        V3 dir = xfm_vector(C, mk3(0, 0, 1));
        V3 d_dir = d_normalize(dir, d_ray.dir);
        V3 d_local_dir = zero3();
        d_xfm_vector(C, mk3(0, 0, 1), d_dir, d_C, d_local_dir);
        V3 d_local_org = zero3();
        d_xfm_point(C, local_org, d_ray.org, d_C, d_local_org);
        d_outer_acc(d_I, d_local_org, pt);
        if (d_screen != nullptr) {
            V3 d_pt = mul_t(d_local_org, I);
            d_screen->x += d_pt.x * 2;
            d_screen->y += d_pt.y * (-2 / aspect);
        }
    }
    acc.add_intr_inv(d_I);
    acc.add_c2w(d_C);
    if (d_screen != nullptr) {
        double d_par[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        D2 d_pos = d2(0, 0);
        d_cam_inverse_distort(cam, spos, d2(d_und.x, d_und.y), RB_CAM_DISTORT(cam) ? d_par : nullptr, d_pos);
        if (RB_CAM_DISTORT(cam)) acc.add_distortion(d_par);
        if (d_screen_out != nullptr) {
            d_screen_out->x += (Real)d_pos.x;
            d_screen_out->y += (Real)d_pos.y;
        }
    }
}

// (rb_render refuses a screen_gradient_image with a lens: d_screen is null there)
RB_D void d_cam_sample_primary(const DevCamera& cam, Real sx, Real sy, const DRay& d_ray, CamAcc& acc, V2* d_screen, D2 lu = D2{0, 0}) {
    if (RB_CAM_GENERAL(cam)) {
        d_cam_sample_primary_any(cam, sx, sy, d_ray, acc, d_screen);
        return;
    }
    if (RB_CAM_LENS(cam)) {
        d_cam_sample_lens(cam, sx, sy, lu, d_ray, acc);
        return;
    }
    M4 C = cam_m4(cam.c2w);
    M3 I = cam_m3(cam.intr_inv);
    Real aspect = Real(cam.width) / Real(cam.height);
    M4 d_C = zero_m4();
    M3 d_I = zero_m3();
    V3 pt = mk3((sx - Real(0.5)) * 2, (sy - Real(0.5)) * (-2) / aspect, 1);
    V3 dir = mul(I, pt);
    V3 n_dir = normalize(dir);
    V3 world_dir = xfm_vector(C, n_dir);
    V3 d_world_dir = d_normalize(world_dir, d_ray.dir);
    V3 d_n_dir = zero3();
    d_xfm_vector(C, n_dir, d_world_dir, d_C, d_n_dir);
    V3 d_dir = d_normalize(dir, d_n_dir);
    d_outer_acc(d_I, d_dir, pt);
    V3 d_cam_org = zero3();
    d_xfm_point(C, zero3(), d_ray.org, d_C, d_cam_org);
    if (d_screen != nullptr) {
        V3 d_pt = mul_t(d_dir, I);
        d_screen->x += d_pt.x * 2;
        d_screen->y += d_pt.y * (-2 / aspect);
    }
    acc.add_intr_inv(d_I);
    acc.add_c2w(d_C);
}

// Adjoint of cam_primary_ray's ray differential, which is psx (ray(sx + delta, sy) - ray(sx, sy)) / delta and likewise in y, psx = 0.5 / width,
// psy = 0.5 / height: d_prd becomes the adjoints of the two offset rays (d_ray_dx at (sx + delta, sy), d_ray_dy at (sx, sy + delta)) and a
// term added to the centre ray's d_ray.  Each of the three then goes through d_cam_sample_primary.
RB_D void d_cam_primary_ray_diff(const DevCamera& cam, const RayDiff& d_prd, DRay& d_ray, DRay& d_ray_dx, DRay& d_ray_dy) {
    const Real delta = Real(1e-3);
    Real psx = Real(0.5) / cam.width, psy = Real(0.5) / cam.height;
    d_ray_dx.org = d_prd.org_dx * (psx / delta);
    d_ray_dx.dir = d_prd.dir_dx * (psx / delta);
    d_ray_dy.org = d_prd.org_dy * (psy / delta);
    d_ray_dy.dir = d_prd.dir_dy * (psy / delta);
    d_ray.org += (d_prd.org_dx * (-psx) + d_prd.org_dy * (-psy)) / delta;
    d_ray.dir += (d_prd.dir_dx * (-psx) + d_prd.dir_dy * (-psy)) / delta;
}

// ---- screen projection of a world-space segment (primary edge sampling) ----
RB_HD V2 cam_to_screen_undistorted(const DevCamera& cam, V3 pt);
RB_HD V2 cam_to_screen(const DevCamera& cam, V3 pt) {
    V2 q = cam_to_screen_undistorted(cam, pt);
    if (!RB_CAM_DISTORT(cam)) return q;
    D2 r = cam_distort(cam, d2(q.x, q.y));
    return mk2((Real)r.x, (Real)r.y);
}
RB_HD V2 cam_to_screen_undistorted(const DevCamera& cam, V3 pt) {
    if (RB_CAM_GENERAL(cam) && cam.type == RB_CAMERA_FISHEYE) { // src/camera.h:533-543
        V3 d = normalize(pt);
        Real phi = atan2(d.y, d.x), r = acos(d.z) * 2 / Real(RB_PI);
        return mk2(Real(0.5) * (-r * cos(phi) + 1), Real(0.5) * (-r * sin(phi) + 1));
    }
    if (RB_CAM_GENERAL(cam) && cam.type == RB_CAMERA_PANORAMA) { // src/camera.h:544-553
        V3 d = normalize(pt);
        return mk2(atan2(d.z, d.x) / Real(2 * RB_PI), acos(d.y) / Real(RB_PI));
    }
    M3 K = cam_m3(cam.intr);
    Real aspect = Real(cam.width) / Real(cam.height);
    V3 ip = mul(K, pt);
    if (!RB_CAM_GENERAL(cam) || cam.type == RB_CAMERA_PERSPECTIVE) {
        Real x = (ip.x / ip.z + 1) * Real(0.5);
        Real y = (-(ip.y / ip.z) * aspect + 1) * Real(0.5);
        return mk2(x, y);
    } else {
        Real x = (ip.x + 1) * Real(0.5);
        Real y = (-ip.y * aspect + 1) * Real(0.5);
        return mk2(x, y);
    }
}
RB_HD bool cam_project(const DevCamera& cam, V3 p0, V3 p1, V2& pp0, V2& pp1) {
    M4 W = cam_m4(cam.w2c);
    V3 a = xfm_point(W, p0), b = xfm_point(W, p1);
    Real cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return false;
    if (a.z < cn) {
        V3 dir = a - b;
        Real t = -(b.z - cn) / dir.z;
        a = b + t * dir;
    } else if (b.z < cn) {
        V3 dir = b - a;
        Real t = -(a.z - cn) / dir.z;
        b = a + t * dir;
    }
    pp0 = cam_to_screen(cam, a);
    pp1 = cam_to_screen(cam, b);
    return true;
}
RB_D void d_cam_to_screen_any(const DevCamera& cam, V3 pt, Real dx, Real dy, CamAcc& acc, V3& d_pt) {
    if (RB_CAM_DISTORT(cam)) { // adjoint of the final distort(): parameters, and the undistorted position for the rest
        V2 q = cam_to_screen_undistorted(cam, pt);
        double d_par[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        D2 d_q = d2(0, 0);
        d_cam_distort(cam, d2(q.x, q.y), d2(dx, dy), d_par, d_q);
        acc.add_distortion(d_par);
        dx = (Real)d_q.x;
        dy = (Real)d_q.y;
    }
    if (cam.type == RB_CAMERA_FISHEYE) { // src/camera.h:669-697
        // On the unit sphere the map is s = 1/2 - G(theta) (d.x, d.y) / pi with G = theta / sin(theta), theta = atan2(rho, d.z) and
        // rho = sqrt(d.x^2 + d.y^2) = sin(theta): smooth at the axis.  Any extension off the sphere gives the same d_pt once
        // d_normalize drops the radial part, so G is differentiated as a function of d.z alone: G'(z) = -F(theta), with
        // F = (sin(theta) - theta cos(theta)) / sin(theta)^3, taken from its Taylor series near the axis, where the quotient cancels.
        // (The reference's acos(d.z) and 1 / sqrt(1 - d.z^2) lose all accuracy there and divide by zero where d.z rounds to 1.)
        V3 d = normalize(pt);
        Real rho = sqrt(d.x * d.x + d.y * d.y), theta = atan2(rho, d.z), t2 = theta * theta;
        Real G = rho > 0 ? theta / rho : Real(1);
        Real F = theta < Real(0.5) ? Real(1.0 / 3) + t2 * (Real(2.0 / 15) + t2 * (Real(2.0 / 63) + t2 * (Real(4.0 / 675) + t2 * (Real(2.0 / 2079) +
                                                                                                                             t2 * Real(2764.0 / 19348875)))))
                                   : (rho - theta * d.z) / (rho * rho * rho);
        Real w = dx * d.x + dy * d.y;
        d_pt += d_normalize(pt, mk3(-G * dx, -G * dy, w * F) * Real(1 / RB_PI));
        return;
    }
    if (cam.type == RB_CAMERA_PANORAMA) { // src/camera.h:698-724
        // theta = atan2(rho, d.y), rho = sqrt(d.x^2 + d.z^2): its gradient (d.y d.x / rho, -rho, d.y d.z / rho) differs from the
        // reference's (0, -1 / sqrt(1 - d.y^2), 0) by a radial part only, and stays accurate up to the poles.  At an exact pole the
        // azimuth is undefined: both terms are dropped there, as the environment map's pole rule does.
        V3 d = normalize(pt);
        Real d_phi = dx / Real(2 * RB_PI), d_theta = dy / Real(RB_PI);
        Real q = d.x * d.x + d.z * d.z, rho = sqrt(q);
        if (q > 0) d_pt += d_normalize(pt, mk3(-d_phi * d.z / q + d_theta * d.y * d.x / rho, -d_theta * rho, d_phi * d.x / q + d_theta * d.y * d.z / rho));
        return;
    }
    M3 K = cam_m3(cam.intr);
    Real aspect = Real(cam.width) / Real(cam.height);
    V3 ip = mul(K, pt);
    M3 d_K = zero_m3();
    V3 d_ip;
    if (cam.type == RB_CAMERA_PERSPECTIVE) {
        V2 q = mk2(ip.x / ip.z, ip.y / ip.z);
        V2 d_q = mk2(dx * Real(0.5), dy * Real(-0.5) * aspect);
        d_ip = mk3(d_q.x / ip.z, d_q.y / ip.z, -(d_q.x * q.x / ip.z + d_q.y * q.y / ip.z));
    } else {
        d_ip = mk3(dx * Real(0.5), dy * Real(-0.5) * aspect, 0);
    }
    d_outer_acc(d_K, d_ip, pt);
    acc.add_intr(d_K);
    d_pt += mul_t(d_ip, K);
}
RB_D void d_cam_to_screen(const DevCamera& cam, V3 pt, Real dx, Real dy, CamAcc& acc, V3& d_pt) {
    if (RB_CAM_GENERAL(cam)) {
        d_cam_to_screen_any(cam, pt, dx, dy, acc, d_pt);
        return;
    }
    M3 K = cam_m3(cam.intr);
    Real aspect = Real(cam.width) / Real(cam.height);
    V3 ip = mul(K, pt);
    M3 d_K = zero_m3();
    V2 q = mk2(ip.x / ip.z, ip.y / ip.z);
    V2 d_q = mk2(dx * Real(0.5), dy * Real(-0.5) * aspect);
    V3 d_ip = mk3(d_q.x / ip.z, d_q.y / ip.z, -(d_q.x * q.x / ip.z + d_q.y * q.y / ip.z));
    d_outer_acc(d_K, d_ip, pt);
    acc.add_intr(d_K);
    d_pt += mul_t(d_ip, K);
}
RB_D void d_cam_project(const DevCamera& cam, V3 p0, V3 p1, Real dp0x, Real dp0y, Real dp1x, Real dp1y, CamAcc& acc, V3& d_p0,
                        V3& d_p1) {
    M4 W = cam_m4(cam.w2c);
    V3 a = xfm_point(W, p0), b = xfm_point(W, p1);
    Real cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return;
    V3 ca = a, cb = b;
    if (a.z < cn) {
        V3 dir = a - b;
        Real t = -(b.z - cn) / dir.z;
        ca = b + t * dir;
    } else if (b.z < cn) {
        V3 dir = b - a;
        Real t = -(a.z - cn) / dir.z;
        cb = a + t * dir;
    }
    V3 d_ca = zero3(), d_cb = zero3();
    d_cam_to_screen(cam, ca, dp0x, dp0y, acc, d_ca);
    d_cam_to_screen(cam, cb, dp1x, dp1y, acc, d_cb);
    V3 d_a = zero3(), d_b = zero3();
    // The "+ clip_near" below reproduces the reference's sign (src/camera.h:776,:791 vs :578,:584).
    if (a.z < cn) {
        V3 dir = a - b;
        Real t = -(b.z + cn) / dir.z;
        d_b += d_ca;
        Real dt = dot(dir, d_ca);
        V3 ddir = t * d_ca;
        d_b.z += (-dt / dir.z);
        ddir.z -= dt * t / dir.z;
        d_a += ddir;
        d_b -= ddir;
        d_b += d_cb;
    } else if (b.z < cn) {
        V3 dir = b - a;
        Real t = -(a.z + cn) / dir.z;
        d_a += d_cb;
        Real dt = dot(dir, d_cb);
        V3 ddir = t * d_cb;
        d_a.z += (-dt / dir.z);
        ddir.z -= dt * t / dir.z;
        d_b += ddir;
        d_a -= ddir;
        d_a += d_ca;
    } else {
        d_a += d_ca;
        d_b += d_cb;
    }
    M4 d_W = zero_m4();
    d_xfm_point(W, p0, d_a, d_W, d_p0);
    d_xfm_point(W, p1, d_b, d_W, d_p1);
    // d_cam_to_world = -W^T d_W W^T is applied once, at the end, on the reduced accumulator (it is linear in d_W).
    acc.add_w2c(d_W);
}
// Projection from the lens point L = (lx, ly, 0) with focal plane z = f: camera-space P lands where the pinhole screen map puts
// Q = (lx / f + (P.x - lx) / P.z, ly / f + (P.y - ly) / P.z, 1), the point where the ray from L through P meets the focal plane, seen from
// the origin.  For a fixed L it is a pinhole at L with a sheared frustum: lines stay lines on the film.
RB_HD V3 lens_film_point(V3 P, Real lx, Real ly, Real f) { return mk3(lx / f + (P.x - lx) / P.z, ly / f + (P.y - ly) / P.z, 1); }
RB_D void d_lens_film_point(const DevCamera& cam, V3 P, Real lx, Real ly, Real f, Real dx, Real dy, CamAcc& acc, V3& d_P, Real& d_lx, Real& d_ly, Real& d_f) {
    V3 d_Q = zero3();
    d_cam_to_screen(cam, lens_film_point(P, lx, ly, f), dx, dy, acc, d_Q);
    d_P.x += d_Q.x / P.z;
    d_P.y += d_Q.y / P.z;
    d_P.z -= (d_Q.x * (P.x - lx) + d_Q.y * (P.y - ly)) / (P.z * P.z);
    d_lx += d_Q.x * (1 / f - 1 / P.z);
    d_ly += d_Q.y * (1 / f - 1 / P.z);
    d_f -= (d_Q.x * lx + d_Q.y * ly) / (f * f);
}
// Adjoint of the projection of segment (p0, p1) from lens sample lu (cam_project_lens_d) w.r.t. the vertices, world_to_cam, intrinsic_mat,
// lens_radius and focus_distance.  The near clip is the camera-space clip of cam_project, differentiated as written.
RB_D void d_cam_project_lens(const DevCamera& cam, V3 p0, V3 p1, D2 lu, Real dp0x, Real dp0y, Real dp1x, Real dp1y, CamAcc& acc, V3& d_p0,
                             V3& d_p1) {
    M4 W = cam_m4(cam.w2c);
    V3 a = xfm_point(W, p0), b = xfm_point(W, p1);
    Real cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return;
    V3 ca = a, cb = b;
    if (a.z < cn) ca = b + ((cn - b.z) / (a.z - b.z)) * (a - b);
    else if (b.z < cn) cb = a + ((cn - a.z) / (b.z - a.z)) * (b - a);
    const Real r = (Real)cam.lens_radius, f = (Real)cam.focus_distance, ux = (Real)lu.x, uy = (Real)lu.y;
    Real d_lx = 0, d_ly = 0, d_f = 0;
    V3 d_ca = zero3(), d_cb = zero3();
    d_lens_film_point(cam, ca, r * ux, r * uy, f, dp0x, dp0y, acc, d_ca, d_lx, d_ly, d_f);
    d_lens_film_point(cam, cb, r * ux, r * uy, f, dp1x, dp1y, acc, d_cb, d_lx, d_ly, d_f);
    V3 d_a = zero3(), d_b = zero3();
    // clipped end c = q + t (p - q), t = (cn - q.z) / (p.z - q.z), p the end behind the plane
    if (a.z < cn) {
        V3 dir = a - b;
        Real t = (cn - b.z) / dir.z, dt = dot(dir, d_ca);
        V3 ddir = t * d_ca;
        ddir.z -= dt * t / dir.z;
        d_b += d_ca + ddir * Real(-1);
        d_b.z -= dt / dir.z;
        d_a += ddir;
        d_b += d_cb;
    } else if (b.z < cn) {
        V3 dir = b - a;
        Real t = (cn - a.z) / dir.z, dt = dot(dir, d_cb);
        V3 ddir = t * d_cb;
        ddir.z -= dt * t / dir.z;
        d_a += d_cb + ddir * Real(-1);
        d_a.z -= dt / dir.z;
        d_b += ddir;
        d_a += d_ca;
    } else {
        d_a += d_ca;
        d_b += d_cb;
    }
    M4 d_W = zero_m4();
    d_xfm_point(W, p0, d_a, d_W, d_p0);
    d_xfm_point(W, p1, d_b, d_W, d_p1);
    acc.add_w2c(d_W);
    acc.add_lens(d_lx * ux + d_ly * uy, d_f);
}
RB_HD bool cam_in_screen(const DevCamera& cam, V2 pt) {
    int xi = int(pt.x * cam.width), yi = int(pt.y * cam.height);
    if (xi < cam.vp_beg[0] || xi >= cam.vp_end[0] || yi < cam.vp_beg[1] || yi >= cam.vp_end[1]) return false;
    if (RB_CAM_GENERAL(cam) && cam.type == RB_CAMERA_FISHEYE) return rb_sq(pt.x - Real(0.5)) + rb_sq(pt.y - Real(0.5)) < Real(0.25); // src/camera.h:1059-1066
    return pt.x >= 0 && pt.x < 1 && pt.y >= 0 && pt.y < 1;
}

// ---- pixel reconstruction filter (rb_pixel_filter; DESIGN.md "pixel filters").  Separable: f(dx, dy) = f1(dx) f1(dy), offsets in pixels
// from the pixel centre.  Cameras with a filter other than the 1-pixel box (RB_PIXEL_BOX) are linear: rb_scene_create refuses the rest.
RB_HD double filter_radius(const DevCamera& cam) { return 0.5 * (double)cam.filter_width; }
// Pixels by which the support of the viewport's pixels reaches past the viewport: the primary-edge distribution covers the image
// grown by this much on each side.
RB_HD double filter_grow(const DevCamera& cam) { return filter_radius(cam) > 0.5 ? filter_radius(cam) - 0.5 : 0.0; }
// The Gaussian's sigma = width / 6, truncated at +-3 sigma: erf(r / (sigma sqrt 2)) = erf(3 / sqrt 2).
#define RB_FILTER_GAUSS_ERF_R 0.99730020393673979
// f1, normalised over its support (the 1-pixel box: 1).
RB_HD double filter_density(const DevCamera& cam, double t) {
    const double r = filter_radius(cam);
    t = fabs(t);
    if (!(t < r)) return 0.0;
    if (cam.filter_type == RB_FILTER_TENT) return (r - t) / (r * r);
    if (cam.filter_type == RB_FILTER_GAUSSIAN) {
        const double sigma = (double)cam.filter_width / 6.0;
        return exp(-t * t / (2.0 * sigma * sigma)) / (sigma * 2.50662827463100050 * RB_FILTER_GAUSS_ERF_R);
    }
    return 1.0 / (double)cam.filter_width;
}
// Inverse CDF of f1: u in [0, 1) -> offset from the pixel centre.
RB_D double filter_offset(const DevCamera& cam, double u) {
    const double r = filter_radius(cam);
    if (cam.filter_type == RB_FILTER_TENT) return u < 0.5 ? r * (sqrt(2.0 * u) - 1.0) : r * (1.0 - sqrt(2.0 * (1.0 - u)));
    if (cam.filter_type == RB_FILTER_GAUSSIAN) {
        const double sigma = (double)cam.filter_width / 6.0;
        return sigma * 1.41421356237309515 * erfinv((2.0 * u - 1.0) * RB_FILTER_GAUSS_ERF_R);
    }
    return (u - 0.5) * (double)cam.filter_width;
}
// A primary-edge point can reach a viewport pixel through the filter: the viewport grown by filter_grow (inside the grown image
// the distribution covers).
RB_HD bool cam_in_filter_reach(const DevCamera& cam, D2 pt) {
    const double g = filter_grow(cam), x = pt.x * cam.width, y = pt.y * cam.height;
    return x >= cam.vp_beg[0] - g && x < cam.vp_end[0] + g && y >= cam.vp_beg[1] - g && y < cam.vp_end[1] + g;
}
RB_HD bool ray_is_null(const Ray& r) { return r.dir.x == 0 && r.dir.y == 0 && r.dir.z == 0; }
