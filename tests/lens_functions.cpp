// TEST INFRASTRUCTURE.  The thin-lens camera functions of rb_camera.cuh / rb_render.cuh / rb_edge.cuh on the host build of the device
// headers with Real = double (g++ -DRB_REAL_DOUBLE -include tools/cpu_emu/emu_shim.h).  Built and run by tests/test_lens_functions_cpu.py,
// which holds the float64 restatement (tests/lens_ref.py).  One mode per run:
//   disc   concentric_disc at given (u1, u2): one line "u1 u2 x y" per point of a grid that includes the wedge boundaries
//   ray    per case: the camera, (sx, sy), the lens sample and what cam_sample_lens returns
//   proj   per case: the camera, the two world-space ends, the lens sample and what cam_project_lens_d returns
//   fd     d_cam_sample_lens and d_cam_project_lens against central differences of the forward functions, w.r.t. every input they
//          differentiate: cam_to_world and intr_inv (ray); the two vertices, world_to_cam and intrinsic_mat (projection); lens_radius and
//          focus_distance (both).  Exits non-zero on the first failure.
//   dist   the distribution invariant: on random edges (among them edges on a ray through the lens centre and edges outside the centre view
//          but within reach of the circle of confusion), every edge that is a silhouette from one of 10^4 lens points and whose projection
//          from it meets the image has primary_edge_weight > 0.  Exits non-zero on the first violation.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../redner_b200/csrc/rb_render.cuh"
#include "../redner_b200/csrc/rb_scene_host.hpp"

static std::mt19937_64 rng(12345);
static double uni(double a, double b) { return std::uniform_real_distribution<double>(a, b)(rng); }

// A perspective camera with a lens, look-at form; a non-square image and a skewed intrinsic matrix exercise every term.
static DevCamera make_camera(double r, double f) {
    rb_camera c;
    memset(&c, 0, sizeof(c));
    c.width = 40;
    c.height = 30;
    c.use_look_at = 1;
    const float pos[3] = {(float)uni(-1, 1), (float)uni(-1, 1), (float)uni(-6, -4)}, look[3] = {(float)uni(-.3, .3), (float)uni(-.3, .3), 0.f},
                up[3] = {(float)uni(-.2, .2), 1.f, (float)uni(-.2, .2)};
    memcpy(c.position, pos, sizeof(pos));
    memcpy(c.look, look, sizeof(look));
    memcpy(c.up, up, sizeof(up));
    const float fx = (float)uni(1.5, 2.5), fy = (float)uni(1.5, 2.5), sk = (float)uni(-.1, .1), cx = (float)uni(-.1, .1), cy = (float)uni(-.1, .1);
    const float K[9] = {fx, sk, cx, 0, fy, cy, 0, 0, 1};
    memcpy(c.intrinsic_mat, K, sizeof(K));
    // intr_inv of the upper-triangular K
    const float Ki[9] = {1 / fx, -sk / (fx * fy), (sk * cy - cx * fy) / (fx * fy), 0, 1 / fy, -cy / fy, 0, 0, 1};
    memcpy(c.intrinsic_mat_inv, Ki, sizeof(Ki));
    c.clip_near = 1e-2f;
    c.camera_type = RB_CAMERA_PERSPECTIVE;
    c.viewport_end[0] = c.width;
    c.viewport_end[1] = c.height;
    c.lens_radius = (float)r;
    c.focus_distance = (float)f;
    DevCamera dc;
    memset(&dc, 0, sizeof(dc));
    host_setup_camera(c, dc);
    dc.filter_type = RB_FILTER_BOX;
    dc.filter_width = 1.f;
    return dc;
}
static void print_camera(const DevCamera& c) {
    printf("%d %d %.17g %.17g", c.width, c.height, (double)c.lens_radius, (double)c.focus_distance);
    for (int i = 0; i < 16; i++) printf(" %.17g", c.c2w[i]);
    for (int i = 0; i < 16; i++) printf(" %.17g", c.w2c[i]);
    for (int i = 0; i < 9; i++) printf(" %.17g", c.intr_inv[i]);
    for (int i = 0; i < 9; i++) printf(" %.17g", c.intr[i]);
    printf(" %.17g", (double)c.clip_near);
}

static int fails = 0;
static void check(const char* what, int k, double ana, double num, double scale) {
    const double tol = 2e-5 * scale + 1e-7;
    if (!(std::fabs(ana - num) <= tol)) {
        printf("FAIL %s[%d]: adjoint %.10g, central difference %.10g\n", what, k, ana, num);
        fails++;
    }
}

// scalar of the ray: d_org . org + d_dir . dir
static double ray_dot(const DevCamera& c, double sx, double sy, D2 lu, const DRay& w) {
    D3 o, d;
    cam_sample_lens(c, sx, sy, lu, o, d);
    return w.org.x * o.x + w.org.y * o.y + w.org.z * o.z + w.dir.x * d.x + w.dir.y * d.y + w.dir.z * d.z;
}
static double proj_dot(const DevCamera& c, V3 p0, V3 p1, D2 lu, const double* w) {
    D2 q0, q1;
    if (!cam_project_lens_d(c, d3(p0.x, p0.y, p0.z), d3(p1.x, p1.y, p1.z), lu, q0, q1)) return 0;
    return w[0] * q0.x + w[1] * q0.y + w[2] * q1.x + w[3] * q1.y;
}
// central difference of g() in the float parameter *p (the camera keeps lens_radius / focus_distance in float)
template <typename G>
static double fd_float(float* p, double rel, G g) {
    const float p0 = *p;
    const float hi = p0 * (float)(1 + rel), lo = p0 * (float)(1 - rel);
    *p = hi;
    double a = g();
    *p = lo;
    double b = g();
    *p = p0;
    return (a - b) / ((double)hi - (double)lo);
}
template <typename G>
static double fd_double(double* p, double h, G g) {
    const double p0 = *p;
    *p = p0 + h;
    double a = g();
    *p = p0 - h;
    double b = g();
    *p = p0;
    return (a - b) / (2 * h);
}

static void mode_fd() {
    std::vector<float> acc(RB_CAM_ACC_LENS * 1);
    for (int cs = 0; cs < 200; cs++) {
        DevCamera c = make_camera(uni(0.05, 0.6), uni(2, 9));
        const D2 lu = concentric_disc(uni(0, 1), uni(0, 1));
        // ray
        {
            const double sx = uni(0.05, 0.95), sy = uni(0.05, 0.95);
            DRay w;
            w.org = mk3(uni(-1, 1), uni(-1, 1), uni(-1, 1));
            w.dir = mk3(uni(-1, 1), uni(-1, 1), uni(-1, 1));
            std::fill(acc.begin(), acc.end(), 0.f);
            CamAcc a;
            a.base = acc.data();
            a.stride = 1;
            d_cam_sample_lens(c, sx, sy, lu, w, a);
            auto g = [&]() { return ray_dot(c, sx, sy, lu, w); };
            double scale = 0;
            for (int k = 0; k < RB_CAM_ACC_LENS; k++) scale = std::max(scale, (double)std::fabs(acc[k]));
            for (int k = 0; k < 12; k++) check("ray d_cam_to_world", k, acc[k], fd_double(&c.c2w[k], 1e-6, g), scale);
            for (int k = 0; k < 9; k++) check("ray d_intr_inv", k, acc[32 + k], fd_double(&c.intr_inv[k], 1e-6, g), scale);
            check("ray d_lens_radius", 0, acc[58], fd_float(&c.lens_radius, 1e-3, g), scale);
            check("ray d_focus_distance", 0, acc[59], fd_float(&c.focus_distance, 1e-3, g), scale);
        }
        // projection; every fourth case has an end behind the near plane
        {
            V3 p0 = mk3(uni(-2, 2), uni(-2, 2), uni(-1.5, 2)), p1 = mk3(uni(-2, 2), uni(-2, 2), uni(-1.5, 2));
            if (cs % 4 == 0) {
                const double* C = c.c2w; // a point just behind the camera, in world space
                p1 = mk3(C[3] - 0.3 * C[2] + 0.2 * C[0], C[7] - 0.3 * C[6] + 0.2 * C[4], C[11] - 0.3 * C[10] + 0.2 * C[8]);
            }
            const double w[4] = {uni(-1, 1), uni(-1, 1), uni(-1, 1), uni(-1, 1)};
            std::fill(acc.begin(), acc.end(), 0.f);
            CamAcc a;
            a.base = acc.data();
            a.stride = 1;
            V3 d0 = zero3(), d1 = zero3();
            d_cam_project_lens(c, p0, p1, lu, w[0], w[1], w[2], w[3], a, d0, d1);
            auto g = [&]() { return proj_dot(c, p0, p1, lu, w); };
            double scale = 0;
            for (int k = 0; k < RB_CAM_ACC_LENS; k++) scale = std::max(scale, (double)std::fabs(acc[k]));
            for (int j = 0; j < 3; j++) scale = std::max(scale, std::max(std::fabs(d0[j]), std::fabs(d1[j])));
            for (int j = 0; j < 3; j++) {
                check("proj d_v0", j, d0[j], fd_double(&p0[j], 1e-6, g), scale);
                check("proj d_v1", j, d1[j], fd_double(&p1[j], 1e-6, g), scale);
            }
            for (int k = 0; k < 12; k++) check("proj d_world_to_cam", k, acc[16 + k], fd_double(&c.w2c[k], 1e-6, g), scale);
            for (int k = 0; k < 9; k++) check("proj d_intrinsic_mat", k, acc[41 + k], fd_double(&c.intr[k], 1e-6, g), scale);
            check("proj d_lens_radius", 0, acc[58], fd_float(&c.lens_radius, 1e-3, g), scale);
            check("proj d_focus_distance", 0, acc[59], fd_float(&c.focus_distance, 1e-3, g), scale);
        }
        if (fails) break;
    }
    printf(fails ? "fd failed\n" : "fd ok\n");
}

static void mode_ray() {
    for (int cs = 0; cs < 64; cs++) {
        DevCamera c = make_camera(uni(0.05, 0.6), uni(2, 9));
        const double sx = uni(-0.1, 1.1), sy = uni(-0.1, 1.1), u1 = uni(0, 1), u2 = uni(0, 1);
        const D2 lu = concentric_disc(u1, u2);
        D3 o, d;
        cam_sample_lens(c, sx, sy, lu, o, d);
        print_camera(c);
        printf(" %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", sx, sy, u1, u2, o.x, o.y, o.z, d.x, d.y, d.z);
    }
}

static void mode_proj() {
    for (int cs = 0; cs < 64; cs++) {
        DevCamera c = make_camera(uni(0.05, 0.6), uni(2, 9));
        const double u1 = uni(0, 1), u2 = uni(0, 1);
        const D2 lu = concentric_disc(u1, u2);
        D3 p0 = d3(uni(-2, 2), uni(-2, 2), uni(-1.5, 2)), p1 = d3(uni(-2, 2), uni(-2, 2), uni(-1.5, 2));
        if (cs % 4 == 0) p1 = d3(c.c2w[3] - 0.3 * c.c2w[2], c.c2w[7] - 0.3 * c.c2w[6], c.c2w[11] - 0.3 * c.c2w[10]);
        D2 q0 = d2(0, 0), q1 = d2(0, 0);
        const int ok = cam_project_lens_d(c, p0, p1, lu, q0, q1);
        print_camera(c);
        printf(" %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d %.17g %.17g %.17g %.17g\n", p0.x, p0.y, p0.z, p1.x, p1.y, p1.z, u1, u2, ok, q0.x,
               q0.y, q1.x, q1.y);
    }
}

static void mode_disc() {
    const double us[] = {0.0, 0.125, 0.25, 0.375, 0.5, 0.625, 0.75, 0.875, 0.999};
    for (double a : us)
        for (double b : us) {
            D2 p = concentric_disc(a, b);
            printf("%.17g %.17g %.17g %.17g\n", a, b, p.x, p.y);
        }
}

// Two faces sharing edge (v0, v1) with per-vertex normals (so that silhouettes depend on the viewpoint).
struct Hinge {
    float v[12], n[12];
    int idx[6];
    rb_shape s;
};
static void make_hinge(Hinge& h, V3 a, V3 b, V3 o0, V3 o1) {
    const V3 p[4] = {a, b, o0, o1};
    for (int i = 0; i < 4; i++) {
        h.v[3 * i] = (float)p[i].x;
        h.v[3 * i + 1] = (float)p[i].y;
        h.v[3 * i + 2] = (float)p[i].z;
        h.n[3 * i] = 0.f;
        h.n[3 * i + 1] = 0.f;
        h.n[3 * i + 2] = 1.f;
    }
    const int idx[6] = {0, 1, 2, 1, 0, 3};
    memcpy(h.idx, idx, sizeof(idx));
    memset(&h.s, 0, sizeof(h.s));
    h.s.vertices = h.v;
    h.s.indices = h.idx;
    h.s.normals = h.n;
    h.s.num_vertices = 4;
    h.s.num_normal_vertices = 4;
    h.s.num_triangles = 2;
}

static void mode_dist() {
    long long edges = 0, seen = 0, kept_only_by_lens = 0;
    for (int cs = 0; cs < 600; cs++) {
        DevCamera c = make_camera(uni(0.05, 0.8), uni(1, 10));
        const double* C = c.c2w;
        auto world = [&](double x, double y, double z) {
            return mk3(C[0] * x + C[1] * y + C[2] * z + C[3], C[4] * x + C[5] * y + C[6] * z + C[7], C[8] * x + C[9] * y + C[10] * z + C[11]);
        };
        V3 a, b;
        const int kind = cs % 3;
        if (kind == 0) { // anywhere in front of the camera
            a = world(uni(-3, 3), uni(-3, 3), uni(0.3, 8));
            b = world(uni(-3, 3), uni(-3, 3), uni(0.3, 8));
        } else if (kind == 1) { // on a ray through the lens centre: a point from the centre, a segment from any other lens point
            const double x = uni(-0.3, 0.3), y = uni(-0.3, 0.3), z0 = uni(0.3, 3), z1 = z0 + uni(0.5, 5);
            a = world(x * z0, y * z0, z0);
            b = world(x * z1, y * z1, z1);
        } else { // just outside the centre view, close to the camera where the circle of confusion is large
            const double z = uni(0.2, 1.0), side = (rng() & 1) ? 1 : -1;
            const double x = side * (1.0 / c.intr[0] + uni(0.0, 0.3)) * z;
            a = world(x, uni(-0.4, 0.4) * z, z);
            b = world(x + side * uni(0, 0.2) * z, uni(-0.4, 0.4) * z, z * uni(1, 1.3));
        }
        const V3 m = (a + b) * Real(0.5), e = b - a;
        V3 t = cross(e, mk3(uni(-1, 1), uni(-1, 1), uni(-1, 1)));
        V3 t2 = cross(e, mk3(uni(-1, 1), uni(-1, 1), uni(-1, 1)));
        Hinge h;
        make_hinge(h, a, b, m + t * Real(uni(0.1, 1) / length(t)), m + t2 * Real(uni(0.1, 1) / length(t2)));
        Edge edge;
        edge.shape_id = 0;
        edge.v0 = 0;
        edge.v1 = 1;
        edge.f0 = 0;
        edge.f1 = 1;
        if (edge_is_flat(&h.s, edge)) continue;
        edges++;
        const double w = primary_edge_weight(c, &h.s, edge);
        bool reachable = false;
        for (int k = 0; k < 10000 && !reachable; k++) {
            const D2 lu = concentric_disc(uni(0, 1), uni(0, 1));
            const double lx = c.lens_radius * lu.x, ly = c.lens_radius * lu.y;
            const V3 lw = world(lx, ly, 0);
            if (!edge_is_silhouette(&h.s, lw, edge)) continue;
            D2 q0, q1;
            if (!cam_project_lens_d(c, d3(a.x, a.y, a.z), d3(b.x, b.y, b.z), lu, q0, q1)) continue;
            V2 c0, c1;
            if (clip_line_unit(mk2(q0.x, q0.y), mk2(q1.x, q1.y), c0, c1) && length(c1 - c0) > 0) reachable = true;
        }
        if (!reachable) continue;
        seen++;
        DevCamera pin = c;
        pin.lens_radius = 0.f;
        pin.focus_distance = 0.f;
        if (primary_edge_weight(pin, &h.s, edge) == 0) kept_only_by_lens++;
        if (!(w > 0)) {
            printf("FAIL case %d (kind %d): the edge is a silhouette from a lens point and its projection from it meets the image, weight %g\n", cs, kind, w);
            fails++;
            break;
        }
    }
    printf("edges %lld reachable %lld zero-weight-for-the-pinhole %lld\n", edges, seen, kept_only_by_lens);
    printf(fails ? "dist failed\n" : "dist ok\n");
}

int main(int argc, char** argv) {
    const std::string m = argc > 1 ? argv[1] : "";
    if (m == "disc") mode_disc();
    else if (m == "ray") mode_ray();
    else if (m == "proj") mode_proj();
    else if (m == "fd") mode_fd();
    else if (m == "dist") mode_dist();
    else {
        fprintf(stderr, "usage: lens_functions disc|ray|proj|fd|dist\n");
        return 2;
    }
    return fails ? 1 : 0;
}
