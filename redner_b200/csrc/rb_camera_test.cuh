// One query of the test hook rb_camera_test (rb_camera_test.cu, and the host emulator's export): the camera functions of rb_camera.cuh
// and rb_render.cuh that the render kernels call, on the scene's DevCamera.  Query i reads row i of `in` ([n, RB_CAMTEST_IN] doubles) and
// writes row i of `out` ([n, RB_CAMTEST_OUT] doubles); the adjoints accumulate into column i of `acc` ([cam_acc_count, n] floats) through a
// CamAcc with base = acc + i and stride = n, exactly as the kernels' per-thread columns.  The layouts are listed in include/redner_b200.h.
#pragma once
#include "rb_render.cuh"

#define RB_CAMTEST_IN 64
#define RB_CAMTEST_OUT 64

RB_D void camera_test_one(const DevCamera& cam, int op, const double* in_, int n, double* out_, float* acc, long long i) {
    if (i >= n) return;
    const double* in = in_ + RB_CAMTEST_IN * i;
    double* out = out_ + RB_CAMTEST_OUT * i;
    CamAcc ca;
    ca.base = acc != nullptr ? acc + i : nullptr;
    ca.stride = n;
    if (op == RB_CAMTEST_CAMERA) {
        for (int k = 0; k < 16; k++) out[k] = cam.c2w[k];
        for (int k = 0; k < 16; k++) out[16 + k] = cam.w2c[k];
        for (int k = 0; k < 9; k++) out[32 + k] = cam.intr_inv[k];
        for (int k = 0; k < 9; k++) out[41 + k] = cam.intr[k];
        for (int k = 0; k < 8; k++) out[50 + k] = cam.distortion[k];
        out[58] = cam.lens_radius;
        out[59] = cam.focus_distance;
        out[60] = cam.clip_near;
        out[61] = cam_acc_count(cam);
    } else if (op == RB_CAMTEST_RAY) {
        const D2 lu = concentric_disc(in[2], in[3]);
        D3 o, d;
        cam_sample_primary(cam, in[0], in[1], o, d, lu);
        Ray ray;
        RayDiff rd;
        cam_primary_ray(cam, in[0], in[1], ray, rd, lu);
        const double v[26] = {o.x, o.y, o.z, d.x, d.y, d.z, ray.org.x, ray.org.y, ray.org.z, ray.dir.x, ray.dir.y, ray.dir.z,
                              rd.org_dx.x, rd.org_dx.y, rd.org_dx.z, rd.org_dy.x, rd.org_dy.y, rd.org_dy.z,
                              rd.dir_dx.x, rd.dir_dx.y, rd.dir_dx.z, rd.dir_dy.x, rd.dir_dy.y, rd.dir_dy.z, lu.x, lu.y};
        for (int k = 0; k < 26; k++) out[k] = v[k];
    } else if (op == RB_CAMTEST_D_RAY) {
        const D2 lu = concentric_disc(in[2], in[3]);
        DRay d_ray;
        d_ray.org = mk3((Real)in[4], (Real)in[5], (Real)in[6]);
        d_ray.dir = mk3((Real)in[7], (Real)in[8], (Real)in[9]);
        V2 d_screen = zero2();
        V2* ds = in[10] != 0 ? &d_screen : nullptr;
        if (in[23] != 0) { // with the ray differential's adjoint, as bwd_sweep does it
            RayDiff d_prd;
            d_prd.org_dx = mk3((Real)in[11], (Real)in[12], (Real)in[13]);
            d_prd.org_dy = mk3((Real)in[14], (Real)in[15], (Real)in[16]);
            d_prd.dir_dx = mk3((Real)in[17], (Real)in[18], (Real)in[19]);
            d_prd.dir_dy = mk3((Real)in[20], (Real)in[21], (Real)in[22]);
            DRay d_ray_dx, d_ray_dy;
            d_cam_primary_ray_diff(cam, d_prd, d_ray, d_ray_dx, d_ray_dy);
            const Real delta = Real(1e-3);
            for (int k = 0; k < 3; k++) {
                DRay dr = k == 0 ? d_ray : k == 1 ? d_ray_dx : d_ray_dy;
                d_cam_sample_primary(cam, (Real)in[0] + (k == 1 ? delta : Real(0)), (Real)in[1] + (k == 2 ? delta : Real(0)), dr, ca, ds, lu);
            }
        } else {
            d_cam_sample_primary(cam, (Real)in[0], (Real)in[1], d_ray, ca, ds, lu);
        }
        out[0] = d_screen.x;
        out[1] = d_screen.y;
    } else if (op == RB_CAMTEST_PROJECT) {
        const D3 p0 = d3(in[0], in[1], in[2]), p1 = d3(in[3], in[4], in[5]);
        const D2 lu = concentric_disc(in[6], in[7]);
        D2 q0 = d2(0, 0), q1 = d2(0, 0);
        out[0] = RB_CAM_LENS(cam) ? cam_project_lens_d(cam, p0, p1, lu, q0, q1) : cam_project_d(cam, p0, p1, q0, q1);
        out[1] = q0.x; out[2] = q0.y; out[3] = q1.x; out[4] = q1.y;
        V2 f0 = zero2(), f1 = zero2();
        out[5] = cam_project(cam, mk3((Real)in[0], (Real)in[1], (Real)in[2]), mk3((Real)in[3], (Real)in[4], (Real)in[5]), f0, f1);
        out[6] = f0.x; out[7] = f0.y; out[8] = f1.x; out[9] = f1.y;
    } else if (op == RB_CAMTEST_D_PROJECT) {
        const V3 p0 = mk3((Real)in[0], (Real)in[1], (Real)in[2]), p1 = mk3((Real)in[3], (Real)in[4], (Real)in[5]);
        const D2 lu = concentric_disc(in[6], in[7]);
        V3 d_p0 = zero3(), d_p1 = zero3();
        if (RB_CAM_LENS(cam)) d_cam_project_lens(cam, p0, p1, lu, (Real)in[8], (Real)in[9], (Real)in[10], (Real)in[11], ca, d_p0, d_p1);
        else d_cam_project(cam, p0, p1, (Real)in[8], (Real)in[9], (Real)in[10], (Real)in[11], ca, d_p0, d_p1);
        const double v[6] = {d_p0.x, d_p0.y, d_p0.z, d_p1.x, d_p1.y, d_p1.z};
        for (int k = 0; k < 6; k++) out[k] = v[k];
    } else if (op == RB_CAMTEST_DISTORT) {
        const D2 pos = d2(in[0], in[1]), d_out = d2(in[2], in[3]);
        D2 jx = d2(0, 0), jy = d2(0, 0);
        const D2 q = cam_distort(cam, pos, &jx, &jy), u = cam_inverse_distort(cam, pos);
        double par[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ipar[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        D2 d_pos = d2(0, 0), d_ipos = d2(0, 0);
        d_cam_distort(cam, pos, d_out, par, d_pos);
        d_cam_inverse_distort(cam, pos, d_out, ipar, d_ipos);
        const double v[12] = {q.x, q.y, jx.x, jx.y, jy.x, jy.y, u.x, u.y, d_pos.x, d_pos.y, d_ipos.x, d_ipos.y};
        for (int k = 0; k < 12; k++) out[k] = v[k];
        for (int k = 0; k < 8; k++) out[12 + k] = par[k];
        for (int k = 0; k < 8; k++) out[20 + k] = ipar[k];
    } else if (op == RB_CAMTEST_FINISH) {
        float g[55];
        for (int k = 0; k < 55; k++) g[k] = 0.f;
        rb_dcamera dc;
        dc.position = g;
        dc.look = g + 3;
        dc.up = g + 6;
        dc.cam_to_world = g + 9;
        dc.world_to_cam = nullptr;
        dc.intrinsic_mat_inv = g + 25;
        dc.intrinsic_mat = g + 34;
        dc.distortion = g + 43;
        dc.lens = g + 51;
        finish_camera(cam, in, dc);
        for (int k = 0; k < 53; k++) out[k] = g[k];
    }
}
