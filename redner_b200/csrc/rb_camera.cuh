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
        D2 dr = d2((dx.x * x + dy.x * y) / r, (dx.y * x + dy.y * y) / r);
        D2 dr2 = d2(2 * r * dr.x, 2 * r * dr.y), dr4 = d2(2 * r2 * dr2.x, 2 * r2 * dr2.y);
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
    double d_r = 2 * d_r2 * r;
    d_x += d_r * x / r;
    d_y += d_r * y / r;
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

// The common camera (pinhole, no lens model) has its own short path; everything else goes through the general one.
RB_HD void cam_sample_primary(const DevCamera& cam, double sx, double sy, D3& org, D3& dir) {
    if (RB_CAM_GENERAL(cam)) {
        cam_sample_primary_any(cam, sx, sy, org, dir);
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
RB_HD void cam_primary_ray(const DevCamera& cam, double sx, double sy, Ray& ray, RayDiff& rd) {
    D3 o, d, ox, dx, oy, dy;
    cam_sample_primary(cam, sx, sy, o, d);
    const double delta = 1e-3;
    cam_sample_primary(cam, sx + delta, sy, ox, dx);
    cam_sample_primary(cam, sx, sy + delta, oy, dy);
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
// [50..57] d_distortion.
// Deterministic mode (rb_kernels_det.cu) keeps one exact accumulator (rb_exact.cuh) per scalar for the whole block instead: each
// (float) contribution goes there, the block flushes them into the global exact accumulators at kernel end.
#define RB_CAM_ACC 58
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
};

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
                Real d_x = d_phi * (-y / (x * x + y * y)) + d_r * (x / r), d_y = d_phi * (x / (x * x + y * y)) + d_r * (y / r);
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

RB_D void d_cam_sample_primary(const DevCamera& cam, Real sx, Real sy, const DRay& d_ray, CamAcc& acc, V2* d_screen) {
    if (RB_CAM_GENERAL(cam)) {
        d_cam_sample_primary_any(cam, sx, sy, d_ray, acc, d_screen);
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
        V3 d = normalize(pt);
        Real phi = atan2(d.y, d.x), r = acos(d.z) * 2 / Real(RB_PI);
        Real dr = Real(-0.5) * (cos(phi) * dx + sin(phi) * dy), dphi = Real(0.5) * r * sin(phi) * dx - Real(0.5) * r * cos(phi) * dy;
        Real dtheta = dr * (2 / Real(RB_PI));
        Real q = d.x * d.x + d.y * d.y;
        d_pt += d_normalize(pt, mk3(-dphi * d.y / q, dphi * d.x / q, -dtheta / sqrt(1 - d.z * d.z)));
        return;
    }
    if (cam.type == RB_CAMERA_PANORAMA) { // src/camera.h:698-724
        V3 d = normalize(pt);
        Real d_phi = dx / Real(2 * RB_PI), d_theta = dy / Real(RB_PI);
        Real q = d.x * d.x + d.z * d.z;
        d_pt += d_normalize(pt, mk3(-d_phi * d.z / q, -d_theta / sqrt(1 - d.y * d.y), d_phi * d.x / q));
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
RB_HD bool cam_in_screen(const DevCamera& cam, V2 pt) {
    int xi = int(pt.x * cam.width), yi = int(pt.y * cam.height);
    if (xi < cam.vp_beg[0] || xi >= cam.vp_end[0] || yi < cam.vp_beg[1] || yi >= cam.vp_end[1]) return false;
    if (RB_CAM_GENERAL(cam) && cam.type == RB_CAMERA_FISHEYE) return rb_sq(pt.x - Real(0.5)) + rb_sq(pt.y - Real(0.5)) < Real(0.25); // src/camera.h:1059-1066
    return pt.x >= 0 && pt.x < 1 && pt.y >= 0 && pt.y < 1;
}
RB_HD bool ray_is_null(const Ray& r) { return r.dir.x == 0 && r.dir.y == 0 && r.dir.z == 0; }
