// CPU check of the decomposition rb_light_build.cu launches (TEST infrastructure).  Its element steps -- one area per emissive triangle
// found through the pool offsets (lt_pool_area), one serial sum and scan per light (lt_light_scan), a min / max over every vertex in
// another order, one PMF / CDF pass -- are run here in serial loops, and the light tables are compared byte for byte with
// host_build_lights / host_bsphere_radius (rb_scene_host.hpp).  Both sides call the same arithmetic of rb_light_build.cuh, so this checks
// the decomposition (offsets, binary search, pool layout, bounds order, environment-map entry), not the arithmetic: that is compared with
// an independent NumPy float64 restatement in tests/test_scene_update_gpu.py.
//
//   light_tables_check <file.bin>...   meshes (int S, then per shape int nv, nt, float[3 nv], int[3 nt]); every shape is a light
//   light_tables_check --random N      N random scenes: random shapes, some of them lights, some empty, with and without an environment map
#include <cstdio>
#include <cstdlib>
#include <limits>
#include <random>
#include <string>
#include <vector>

#include "../redner_b200/csrc/rb_render.cuh"
#include "../redner_b200/csrc/rb_scene_host.hpp"

struct Scene {
    std::vector<HostMesh> meshes;
    std::vector<rb_shape> shapes;
    std::vector<DevLight> lights;
    bool env = false;
    float pdf_norm = 0.f;
    void finish() {
        shapes.assign(meshes.size(), rb_shape());
        for (size_t s = 0; s < meshes.size(); s++) {
            memset(&shapes[s], 0, sizeof(rb_shape));
            shapes[s].num_vertices = (int)meshes[s].vertices.size() / 3;
            shapes[s].num_triangles = (int)meshes[s].indices.size() / 3;
            shapes[s].vertices = meshes[s].vertices.data();
            shapes[s].indices = meshes[s].indices.data();
        }
    }
};

// the decomposition of rb_light_build.cu, in serial loops
static bool tables_by_steps(const Scene& sc, HostLightTables& t) {
    const int L = (int)sc.lights.size();
    std::vector<int> off(L + 1, 0);
    for (int l = 0; l < L; l++) off[l + 1] = off[l] + sc.shapes[sc.lights[l].shape_id].num_triangles;
    const LTScene S{sc.shapes.data(), sc.lights.data(), off.data(), L};
    std::vector<double> a(off[L]);
    t.pool.assign(off[L], 0.0);
    t.areas.assign(L, 0.0);
    for (int i = 0; i < off[L]; i++) a[i] = lt_pool_area(S, i);          // k_lt_areas
    for (int l = 0; l < L; l++) t.areas[l] = lt_light_scan(S, l, a.data(), t.pool.data()); // k_lt_scan
    t.offsets.assign(off.begin(), off.end() - 1);
    double radius = 0;
    if (sc.env && !sc.shapes.empty()) { // k_lt_bounds
        float lo[2] = {INFINITY, INFINITY}, hi[2] = {-INFINITY, -INFINITY};
        for (const rb_shape& sh : sc.shapes)
            for (int v = sh.num_vertices - 1; v >= 0; v--) // (any order)
                for (int k = 0; k < 2; k++) {
                    lo[k] = fminf(lo[k], sh.vertices[3 * v + k]);
                    hi[k] = fmaxf(hi[k], sh.vertices[3 * v + k]);
                }
        radius = lt_bsphere_radius(lo, hi);
    }
    const int n = L + (sc.env ? 1 : 0); // k_lt_pmf
    t.pmf.assign(n, 0.0);
    t.cdf.assign(n, 0.0);
    for (int l = 0; l < L; l++) t.pmf[l] = lt_light_weight(sc.lights[l], t.areas[l]);
    if (sc.env) t.pmf[L] = lt_env_weight(radius, sc.pdf_norm);
    return lt_normalize(t.pmf.data(), t.cdf.data(), n);
}

template <typename T>
static bool same_bytes(const std::vector<T>& a, const std::vector<T>& b) {
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), sizeof(T) * a.size()) == 0);
}

static int compare(const Scene& sc, const char* label, bool verbose) {
    HostLightTables h, d;
    std::string err;
    const bool ok_h = host_build_lights(sc.lights, sc.meshes, h, err, sc.env, sc.env ? sc.pdf_norm : 0.0, sc.env ? host_bsphere_radius(sc.meshes) : 0.0);
    const bool ok_d = tables_by_steps(sc, d);
    if (ok_h != ok_d) {
        printf("MISMATCH %s: host %s, steps %s\n", label, ok_h ? "ok" : "refused", ok_d ? "ok" : "refused");
        return 1;
    }
    if (!ok_h) return 0;
    const char* bad = !same_bytes(h.pmf, d.pmf) ? "pmf" : !same_bytes(h.cdf, d.cdf) ? "cdf" : !same_bytes(h.areas, d.areas) ? "areas" :
                      !same_bytes(h.pool, d.pool) ? "pool" : !same_bytes(h.offsets, d.offsets) ? "offsets" : nullptr;
    if (bad) {
        printf("MISMATCH %s: %s\n", label, bad);
        return 1;
    }
    if (verbose) printf("ok %s lights %zu pool %zu env %d\n", label, sc.lights.size(), h.pool.size(), sc.env ? 1 : 0);
    return 0;
}

static bool load(const char* path, Scene& sc) {
    FILE* f = fopen(path, "rb");
    if (!f) return false;
    int S = 0;
    if (fread(&S, 4, 1, f) != 1) return false;
    sc.meshes.assign(S, HostMesh());
    for (int s = 0; s < S; s++) {
        int nv[2];
        if (fread(nv, 4, 2, f) != 2) return false;
        sc.meshes[s].vertices.resize(3 * (size_t)nv[0]);
        sc.meshes[s].indices.resize(3 * (size_t)nv[1]);
        if (fread(sc.meshes[s].vertices.data(), 4, 3 * (size_t)nv[0], f) != 3 * (size_t)nv[0]) return false;
        if (fread(sc.meshes[s].indices.data(), 4, 3 * (size_t)nv[1], f) != 3 * (size_t)nv[1]) return false;
    }
    fclose(f);
    sc.finish();
    return true;
}

static DevLight light(int shape, float r, float g, float b) {
    DevLight l;
    memset(&l, 0, sizeof(l));
    l.shape_id = shape;
    l.intensity[0] = r;
    l.intensity[1] = g;
    l.intensity[2] = b;
    return l;
}

static void random_scene(std::mt19937& rng, Scene& sc) {
    auto U = [&](int lo, int hi) { return std::uniform_int_distribution<int>(lo, hi)(rng); };
    auto F = [&](float lo, float hi) { return std::uniform_real_distribution<float>(lo, hi)(rng); };
    const int S = U(0, 6);
    sc.meshes.assign(S, HostMesh());
    for (HostMesh& m : sc.meshes) {
        const int nv = U(0, 1) ? U(3, 300) : U(0, 2), nt = nv >= 3 ? U(0, 2000) : 0;
        const float scale = std::pow(10.f, F(-3.f, 3.f));
        for (int v = 0; v < 3 * nv; v++) m.vertices.push_back(scale * F(-1.f, 1.f));
        for (int t = 0; t < 3 * nt; t++) m.indices.push_back(U(0, nv - 1));
    }
    sc.finish();
    if (S > 0)
        for (int l = U(0, 4); l > 0; l--) sc.lights.push_back(light(U(0, S - 1), F(0.f, 30.f), F(0.f, 30.f), U(0, 5) == 0 ? 0.f : F(0.f, 30.f)));
    sc.env = U(0, 1) == 1;
    sc.pdf_norm = F(0.01f, 2.f);
}

int main(int argc, char** argv) {
    int bad = 0;
    if (argc >= 3 && std::string(argv[1]) == "--random") {
        const int N = atoi(argv[2]);
        std::mt19937 rng(20261015u);
        for (int i = 0; i < N; i++) {
            Scene sc;
            random_scene(rng, sc);
            bad += compare(sc, ("random" + std::to_string(i)).c_str(), false);
        }
        printf("random scenes %d mismatching %d\n", N, bad);
        return bad != 0;
    }
    for (int a = 1; a < argc; a++) {
        Scene sc;
        if (!load(argv[a], sc)) {
            printf("cannot read %s\n", argv[a]);
            return 2;
        }
        for (int s = 0; s < (int)sc.shapes.size(); s++) sc.lights.push_back(light(s, 1.f + s, 2.f, 0.5f * s));
        for (int env = 0; env < 2; env++) {
            sc.env = env == 1;
            sc.pdf_norm = 0.37f;
            bad += compare(sc, (std::string(argv[a]) + (env ? " env" : "")).c_str(), true);
        }
    }
    return bad != 0;
}
