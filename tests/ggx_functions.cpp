// TEST INFRASTRUCTURE.  The GGX specular lobe of rb_material.cuh (bsdf_eval, bsdf_pdf, bsdf_sample_dir, d_bsdf_eval) on the host build
// of the device headers with Real = double (g++ -DRB_REAL_DOUBLE -include tools/cpu_emu/emu_shim.h).  Built and run by
// tests/test_ggx_cpu.py, which holds the float64 restatement of the lobe and the statistics.  One mode per run:
//   grid   one line per case: the inputs of the lobe as bsdf_ctx sees them and what eval, pdf and sample return
//   quad   per (alpha, angle) case: the spec pdf (ggx_pdf) integrated over the sphere of reflected directions, and over the directions a
//          sample keeps
//   hist   per case: observed and expected counts of 10^6 samples over bins of the sphere, plus the failed samples
//   fd     d_bsdf_eval's GGX branch against central differences of bsdf_eval; exits non-zero on the first failure
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../redner_b200/csrc/rb_render.cuh"

static rb_texture const_tex(float* data, int channels, float* uv_scale) {
    rb_texture t;
    memset(&t, 0, sizeof(t));
    t.texels[0] = data;
    t.channels = channels;
    t.num_levels = 1;
    t.uv_scale = uv_scale;
    return t;
}

// One shading point and material: constant textures, a shading normal tilted away from the geometric one, optionally a normal map.
struct Setup {
    float kd[3], ks[3], ro[1], nm[3], uvs[2] = {1.f, 1.f};
    float d_kd[3] = {0, 0, 0}, d_ks[3] = {0, 0, 0}, d_ro[1] = {0}, d_nm[3] = {0, 0, 0}, d_uvs[2] = {0, 0};
    rb_material m, d_m;
    SurfacePoint p;
    Setup(Real kd_, Real ks_, Real rough, bool two_sided, bool normal_map, Real tilt) {
        for (int i = 0; i < 3; i++) {
            kd[i] = (float)(kd_ * (1 - Real(0.1) * i));
            ks[i] = (float)(ks_ * (1 - Real(0.15) * i));
        }
        ro[0] = (float)rough;
        nm[0] = 0.62f;
        nm[1] = 0.44f;
        nm[2] = 0.93f;
        memset(&m, 0, sizeof(m));
        memset(&d_m, 0, sizeof(d_m));
        m.diffuse_reflectance = const_tex(kd, 3, uvs);
        m.specular_reflectance = const_tex(ks, 3, uvs);
        m.roughness = const_tex(ro, 1, uvs);
        d_m.diffuse_reflectance = const_tex(d_kd, 3, d_uvs);
        d_m.specular_reflectance = const_tex(d_ks, 3, d_uvs);
        d_m.roughness = const_tex(d_ro, 1, d_uvs);
        if (normal_map) {
            m.normal_map = const_tex(nm, 3, uvs);
            d_m.normal_map = const_tex(d_nm, 3, d_uvs);
        }
        m.compute_specular_lighting = 1;
        m.two_sided = two_sided ? 1 : 0;
        m.specular_model = RB_SPECULAR_GGX;
        p = zero_point();
        p.geom_normal = mk3(0, 0, 1);
        p.shading_frame = frame_from_normal(normalize(mk3(tilt, Real(0.5) * tilt, 1)));
        p.dpdu = mk3(1, 0, 0);
        p.uv = mk2(Real(0.5), Real(0.5));
    }
};

static V3 dir_at(Real theta, Real phi) { return mk3(sin(theta) * cos(phi), sin(theta) * sin(phi), cos(theta)); }
static void put(V3 v) { printf(" %.17g %.17g %.17g", (double)v.x, (double)v.y, (double)v.z); }

static const Real ALPHAS[] = {1e-3, 0.05, 0.3, 0.7, 1.0};
static const Real THETAS[] = {0.0, 0.5, 1.1, 1.48};

static void mode_grid() {
    std::mt19937_64 rng(7);
    std::uniform_real_distribution<double> U(0, 1);
    for (Real alpha : ALPHAS)
        for (Real theta : THETAS)
            for (int variant = 0; variant < 4; variant++) { // 0 plain, 1 normal map, 2 two-sided seen from below, 3 two-sided + normal map from below
                const bool nmap = variant & 1, below = variant & 2;
                Setup s(Real(0.4), Real(0.7), alpha * alpha, below, nmap, Real(0.15));
                BsdfCtx c = bsdf_ctx(s.m, s.p);
                MatTex tx = mat_textures(s.m, s.p);
                V3 wi = dir_at(theta, Real(0.3) + theta);
                if (below) wi = -wi;
                for (int k = 0; k < 6; k++) {
                    V2 suv = mk2((Real)U(rng), (Real)U(rng));
                    double w_sel = 0.5 + 0.5 * U(rng); // above pd = lum(kd) / (lum(kd) + lum(ks)) ~ 0.38: the specular lobe
                    RayDiff rd_in, rd_out;
                    memset(&rd_in, 0, sizeof(rd_in));
                    Real nmr;
                    V3 ws = bsdf_sample_dir(s.m, s.p, tx, wi, suv, w_sel, Real(0), rd_in, rd_out, nmr);
                    // wo: the sample itself (k even) or a direction of either hemisphere (k odd)
                    V3 wo = (k % 2 == 0 && length_sq(ws) > 0) ? ws : dir_at((Real)(U(rng) * 3.1), (Real)(U(rng) * 6.28));
                    V3 f = bsdf_eval(s.m, s.p, tx, wi, wo, Real(0));
                    Real pdf = bsdf_pdf(s.m, s.p, tx, wi, wo, Real(0));
                    printf("case %.17g %d %.17g %.17g %.17g %.17g %.17g %.17g", (double)tx.rough, s.m.two_sided, (double)tx.kd.x, (double)tx.kd.y, (double)tx.kd.z,
                           (double)tx.ks.x, (double)tx.ks.y, (double)tx.ks.z);
                    put(c.frame.x), put(c.frame.y), put(c.frame.n), put(c.geom_n), put(wi), put(wo);
                    put(f);
                    printf(" %.17g %.17g %.17g %.17g", (double)pdf, (double)suv.x, (double)suv.y, w_sel);
                    put(ws);
                    printf("\n");
                }
            }
}

// Directions around the mirror direction mdir: gamma = pi t^3 concentrates the grid where the lobe is.
struct Sphere {
    V3 m, t1, t2;
    explicit Sphere(V3 mdir) : m(mdir) { coordinate_system(m, t1, t2); }
    V3 at(Real t, Real phi) const {
        Real g = RB_PI * t * t * t;
        return m * cos(g) + (t1 * cos(phi) + t2 * sin(phi)) * sin(g);
    }
    // d(omega) / (dt dphi)
    Real jac(Real t) const { return sin(RB_PI * t * t * t) * 3 * RB_PI * t * t; }
    void coords(V3 d, Real& t, Real& phi) const {
        Real g = acos(rb_max(Real(-1), rb_min(Real(1), dot(d, m))));
        t = cbrt(g / RB_PI);
        phi = atan2(dot(d, t2), dot(d, t1));
        if (phi < 0) phi += 2 * RB_PI;
    }
};
struct LobeCase {
    Real alpha, theta;
    int variant;
};
static std::vector<LobeCase> lobe_cases() {
    std::vector<LobeCase> v;
    for (Real alpha : {0.02, 0.1, 0.3, 0.6, 1.0})
        for (Real theta : {0.0, 0.7, 1.3, 1.55}) v.push_back({alpha, theta, 0});
    v.push_back({0.2, 0.9, 1});
    v.push_back({0.2, 0.9, 2});
    v.push_back({0.5, 1.2, 3});
    return v;
}
struct Lobe {
    Setup s;
    MatTex tx;
    V3 wi, n;
    Real geom_wi;
    Lobe(const LobeCase& lc) : s(0, 1, lc.alpha * lc.alpha, lc.variant & 2, lc.variant & 1, Real(0.15)) {
        tx = mat_textures(s.m, s.p);
        BsdfCtx c = bsdf_ctx(s.m, s.p);
        n = c.frame.n;
        wi = to_world(c.frame, dir_at(lc.theta, Real(0.4)));
        if (lc.variant & 2) wi = -wi;
        geom_wi = dot(c.geom_n, wi);
        if (dot(wi, n) < 0) n = -n;
    }
    // the spec pdf itself (bsdf_pdf is zero on the far side of the geometric surface, whatever the lobe)
    Real pdf(V3 wo) const { return ggx_pdf(s.m, bsdf_ctx(s.m, s.p), tx.rough, wi, wo); }
    // what bsdf_sample_dir keeps: nothing seen from below a one-sided surface, else the directions on wi's side of it
    bool kept(V3 wo) const { return (s.m.two_sided || geom_wi >= 0) && dot(s.p.geom_normal, wo) * geom_wi >= 0; }
    V3 mirror() const { return 2 * dot(wi, n) * n - wi; }
};

static void mode_quad() {
    const int NT = 4000, NP = 512;
    for (const LobeCase& lc : lobe_cases()) {
        Lobe l(lc);
        Sphere sp(l.mirror());
        double all = 0, kept = 0;
        for (int i = 0; i < NT; i++) {
            Real t = (i + Real(0.5)) / NT;
            for (int j = 0; j < NP; j++) {
                Real phi = 2 * RB_PI * (j + Real(0.5)) / NP;
                V3 wo = sp.at(t, phi);
                double w = (double)(l.pdf(wo) * sp.jac(t)) * (1.0 / NT) * (2 * M_PI / NP);
                all += w;
                if (l.kept(wo)) kept += w;
            }
        }
        printf("quad %.17g %.17g %d %.17g %.17g\n", (double)lc.alpha, (double)lc.theta, lc.variant, all, kept);
    }
}

static void mode_hist() {
    const int NT = 24, NP = 12, SUB_T = 64, SUB_P = 32;
    const long N = 1000000;
    for (const LobeCase& lc : lobe_cases()) {
        if (lc.theta == Real(0.0)) continue; // (the normal-incidence cases are covered by quad)
        Lobe l(lc);
        Sphere sp(l.mirror());
        std::vector<long> obs(NT * NP + 1, 0);
        std::mt19937_64 rng(1234);
        std::uniform_real_distribution<double> U(0, 1);
        for (long k = 0; k < N; k++) {
            RayDiff rd_in, rd_out;
            memset(&rd_in, 0, sizeof(rd_in));
            Real nmr;
            V2 suv = mk2((Real)U(rng), (Real)U(rng));
            V3 wo = bsdf_sample_dir(l.s.m, l.s.p, l.tx, l.wi, suv, 1.0 - U(rng), Real(0), rd_in, rd_out, nmr);
            if (length_sq(wo) == 0) {
                obs[NT * NP]++;
                continue;
            }
            Real t, phi;
            sp.coords(wo, t, phi);
            int a = rb_clampi((int)(t * NT), 0, NT - 1), b = rb_clampi((int)(phi / (2 * RB_PI) * NP), 0, NP - 1);
            obs[a * NP + b]++;
        }
        double kept_total = 0;
        printf("hist %.17g %.17g %d", (double)lc.alpha, (double)lc.theta, lc.variant);
        for (int a = 0; a < NT; a++)
            for (int b = 0; b < NP; b++) {
                double e = 0;
                for (int i = 0; i < SUB_T; i++)
                    for (int j = 0; j < SUB_P; j++) {
                        Real t = (a + (i + Real(0.5)) / SUB_T) / NT, phi = 2 * RB_PI * (b + (j + Real(0.5)) / SUB_P) / NP;
                        V3 wo = sp.at(t, phi);
                        if (l.kept(wo)) e += (double)(l.pdf(wo) * sp.jac(t));
                    }
                e *= (1.0 / (NT * SUB_T)) * (2 * M_PI / (NP * SUB_P));
                kept_total += e;
                printf(" %ld %.17g", obs[a * NP + b], e * N);
            }
        printf(" %ld %.17g\n", obs[NT * NP], (1 - kept_total) * N);
    }
}

static int g_checks = 0;
static void check(const char* what, int i, double fd, double analytic) {
    g_checks++;
    double tol = 1e-3 * (fabs(analytic) > 1 ? fabs(analytic) : 1.0); // the reference's 1e-3, relative where the value exceeds 1
    if (!(fabs(fd - analytic) <= tol)) {
        fprintf(stderr, "FD check failed: %s[%d]: finite difference %.9g, adjoint %.9g\n", what, i, fd, analytic);
        exit(1);
    }
}

static void fd_case(Real alpha, Real theta_i, Real theta_o, bool below, bool nmap) {
    Setup s(Real(0.4), Real(0.7), alpha * alpha, below, nmap, Real(0.15));
    V3 wi = dir_at(theta_i, Real(0.3)), wo = dir_at(theta_o, Real(0.3) + Real(2.9));
    if (below) {
        wi = -wi;
        wo = -wo;
    }
    V3 w = mk3(Real(0.9), Real(-0.6), Real(1.3)); // loss weights of the three channels
    SurfacePoint d_p = zero_point();
    V3 d_wi = zero3(), d_wo = zero3();
    d_bsdf_eval(s.m, s.d_m, s.p, wi, wo, Real(0), w, d_p, d_wi, d_wo);
    auto eval = [&](const SurfacePoint& q, V3 a, V3 b) { return (double)dot(w, bsdf_eval(s.m, q, a, b, Real(0))); };
    auto tex_fd = [&](const char* name, float* texel, int n, const float* grad, float h) {
        for (int i = 0; i < n; i++) {
            float keep = texel[i];
            texel[i] = keep + h;
            double fp = eval(s.p, wi, wo);
            texel[i] = keep - h;
            double fn = eval(s.p, wi, wo);
            texel[i] = keep;
            check(name, i, (fp - fn) / ((double)(keep + h) - (double)(keep - h)), grad[i]);
        }
    };
    tex_fd("d_diffuse", s.kd, 3, s.d_kd, 1e-3f);
    tex_fd("d_specular", s.ks, 3, s.d_ks, 1e-3f);
    tex_fd("d_roughness", s.ro, 1, s.d_ro, s.ro[0] * 1e-3f);
    if (nmap) tex_fd("d_normal_map", s.nm, 3, s.d_nm, 1e-4f);
    const Real h = Real(1e-6);
    for (int i = 0; i < 3; i++) {
        V3 a = wi, b = wi;
        a[i] += h;
        b[i] -= h;
        check("d_wi", i, (eval(s.p, a, wo) - eval(s.p, b, wo)) / (2 * h), d_wi[i]);
        a = wo;
        b = wo;
        a[i] += h;
        b[i] -= h;
        check("d_wo", i, (eval(s.p, wi, a) - eval(s.p, wi, b)) / (2 * h), d_wo[i]);
        if (!nmap) {
            SurfacePoint qa = s.p, qb = s.p;
            qa.shading_frame.n[i] += h;
            qb.shading_frame.n[i] -= h;
            check("d_shading_normal", i, (eval(qa, wi, wo) - eval(qb, wi, wo)) / (2 * h), d_p.shading_frame.n[i]);
        }
    }
}

static void mode_fd() {
    for (Real alpha : {0.05, 0.1, 0.3, 0.6, 1.0})
        for (int variant = 0; variant < 4; variant++)
            for (Real ti : {0.2, 0.8, 1.3})
                for (Real to : {0.3, 0.9, 1.4}) fd_case(alpha, ti, to, variant & 2, variant & 1);
    printf("fd checks %d\n", g_checks);
}

int main(int argc, char** argv) {
    std::string mode = argc > 1 ? argv[1] : "";
    if (mode == "grid") mode_grid();
    else if (mode == "quad") mode_quad();
    else if (mode == "hist") mode_hist();
    else if (mode == "fd") mode_fd();
    else {
        fprintf(stderr, "usage: ggx_functions grid | quad | hist | fd\n");
        return 2;
    }
    return 0;
}
