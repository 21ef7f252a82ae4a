// DEVELOPMENT AID ONLY (see emu_shim.h).  Exports the same C ABI as libredner_b200.so, but every buffer is a HOST
// pointer and the "kernels" are plain loops over the per-sample functions of rb_render.cuh.  The triangle BVH is a
// simple median-split tree in the same node format (the GPU LBVH builder itself is exercised on the GPU only, by
// tests/test_bvh_gpu.py; rb_scene_trace_rays queries this tree with the same traversal).
#include "emu_shim.h"

#include <algorithm>
#include <numeric>
#include <string>
#include <vector>

#include "../../redner_b200/csrc/rb_render.cuh"
#include "../../redner_b200/csrc/rb_exact_layout.hpp"
#include "../../redner_b200/csrc/rb_scene_host.hpp"

static thread_local std::string g_err;
extern "C" const char* rb_last_error(void) { return g_err.c_str(); }
extern "C" const char* rb_version(void) { return "redner_b200 CPU emulator (debug only)"; }

struct rb_scene {
    DevScene dev;
    rb_camera cam;
    std::vector<rb_shape> shapes;
    std::vector<rb_material> materials;
    std::vector<DevLight> lights;
    HostLightTables lt;
    HostEdgeTables et;
    HostEdgeTree tree;
    std::vector<float> ltc;
    std::vector<BVHNode> nodes;
    std::vector<BVHTri> tris;
    std::vector<unsigned long long> sobol;
    int max_generic = 0;
    int gpu_index = -1;
    bool incomplete = false; // the last update failed part-way (as in the library: rb_render refuses the scene)
    int part = 0, num_parts = 1, rps = 16;
};

static int build_node(rb_scene* sc, std::vector<int>& order, std::vector<float>& boxes, int lo, int hi, float out_box[6]) {
    // returns child reference (>=0 inner, <0 leaf) for the range [lo, hi) of `order`
    if (hi - lo == 1) {
        for (int k = 0; k < 6; k++) out_box[k] = boxes[6 * (size_t)order[lo] + k];
        return ~order[lo];
    }
    float cb[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int i = lo; i < hi; i++)
        for (int a = 0; a < 3; a++) {
            float c = 0.5f * (boxes[6 * (size_t)order[i] + a] + boxes[6 * (size_t)order[i] + 3 + a]);
            cb[a] = std::min(cb[a], c);
            cb[3 + a] = std::max(cb[3 + a], c);
        }
    int axis = 0;
    for (int a = 1; a < 3; a++)
        if (cb[3 + a] - cb[a] > cb[3 + axis] - cb[axis]) axis = a;
    int mid = (lo + hi) / 2;
    std::nth_element(order.begin() + lo, order.begin() + mid, order.begin() + hi, [&](int x, int y) {
        return boxes[6 * (size_t)x + axis] + boxes[6 * (size_t)x + 3 + axis] < boxes[6 * (size_t)y + axis] + boxes[6 * (size_t)y + 3 + axis];
    });
    int me = (int)sc->nodes.size();
    sc->nodes.push_back(BVHNode());
    float l[6], r[6];
    int left = build_node(sc, order, boxes, lo, mid, l);
    int right = build_node(sc, order, boxes, mid, hi, r);
    BVHNode& n = sc->nodes[me];
    n.left = left;
    n.right = right;
    n.pad0 = n.pad1 = 0;
    n.lo_x_hi_x = make_float4(l[0], l[3], r[0], r[3]);
    n.lo_y_hi_y = make_float4(l[1], l[4], r[1], r[4]);
    n.lo_z_hi_z = make_float4(l[2], l[5], r[2], r[5]);
    for (int k = 0; k < 3; k++) {
        out_box[k] = std::min(l[k], r[k]);
        out_box[3 + k] = std::max(l[3 + k], r[3 + k]);
    }
    return me;
}

static bool load_table(const char* path, size_t bytes_per, std::vector<unsigned char>& out, size_t count) {
    FILE* f = fopen(path, "rb");
    if (!f) return false;
    out.resize(bytes_per * count);
    bool ok = fread(out.data(), bytes_per, count, f) == count;
    fclose(f);
    return ok;
}

// Every table from the descriptor with the host builders (rb_scene_create and rb_scene_update).
static int emu_build(rb_scene* sc, const rb_scene_desc* desc) {
    DevScene& d = sc->dev;
    const unsigned long long* sobol = d.sobol_matrices;
    const float* ltc = d.ltc_table;
    memset(&d, 0, sizeof(DevScene));
    d.sobol_matrices = sobol;
    d.sobol_dims = 1024;
    sc->cam = desc->camera;
    host_setup_camera(desc->camera, d.cam);
    sc->shapes.assign(desc->shapes, desc->shapes + desc->num_shapes);
    sc->materials.assign(desc->materials, desc->materials + desc->num_materials);
    sc->lights = host_area_lights(*desc);
    sc->max_generic = host_max_generic_texture_dimension(*desc);
    d.edge_root_cs = d.edge_root_ncs = RB_EDGE_EMPTY;
    d.shapes = sc->shapes.data();
    d.num_shapes = (int)sc->shapes.size();
    d.materials = sc->materials.data();
    d.num_materials = (int)sc->materials.size();
    d.use_primary_edge = desc->use_primary_edge_sampling;
    d.use_secondary_edge = desc->use_secondary_edge_sampling;
    // BVH
    sc->nodes.clear();
    sc->tris.clear();
    std::vector<float> boxes;
    for (int s = 0; s < d.num_shapes; s++)
        for (int t = 0; t < sc->shapes[s].num_triangles; t++) {
            V3 v0, v1, v2;
            shape_tri_vertices(sc->shapes[s], t, v0, v1, v2);
            BVHTri tr;
            tr.v0 = make_float4((float)v0.x, (float)v0.y, (float)v0.z, __int_as_float(s));
            tr.v1 = make_float4((float)v1.x, (float)v1.y, (float)v1.z, __int_as_float(t));
            tr.v2 = make_float4((float)v2.x, (float)v2.y, (float)v2.z, 0.f);
            sc->tris.push_back(tr);
            for (int a = 0; a < 3; a++) {
                float lo = std::min((float)v0[a], std::min((float)v1[a], (float)v2[a])), hi = std::max((float)v0[a], std::max((float)v1[a], (float)v2[a]));
                float pad = std::max(std::fabs(lo), std::fabs(hi)) * 4e-7f + 1e-6f;
                boxes.push_back(lo - pad);
            }
            for (int a = 0; a < 3; a++) {
                float hi = std::max((float)v0[a], std::max((float)v1[a], (float)v2[a]));
                float lo = std::min((float)v0[a], std::min((float)v1[a], (float)v2[a]));
                float pad = std::max(std::fabs(lo), std::fabs(hi)) * 4e-7f + 1e-6f;
                boxes.push_back(hi + pad);
            }
        }
    int T = (int)sc->tris.size();
    d.num_tris = T;
    if (T > 0) {
        std::vector<int> order(T);
        std::iota(order.begin(), order.end(), 0);
        float box[6];
        d.bvh_root = build_node(sc, order, boxes, 0, T, box);
        if (sc->nodes.empty()) sc->nodes.push_back(BVHNode());
        d.bvh_nodes = sc->nodes.data();
        d.bvh_tris = sc->tris.data();
    }
    // lights + edges
    std::vector<HostMesh> meshes(d.num_shapes);
    for (int s = 0; s < d.num_shapes; s++) {
        meshes[s].vertices.assign(sc->shapes[s].vertices, sc->shapes[s].vertices + 3 * (size_t)sc->shapes[s].num_vertices);
        meshes[s].indices.assign(sc->shapes[s].indices, sc->shapes[s].indices + 3 * (size_t)sc->shapes[s].num_triangles);
    }
    host_setup_envmap(desc->envmap, d);
    d.num_lights = (int)sc->lights.size() + (d.has_envmap ? 1 : 0);
    if (d.num_lights > 0) {
        if (!host_build_lights(sc->lights, meshes, sc->lt, g_err, d.has_envmap != 0, d.has_envmap ? desc->envmap->pdf_norm : 0.0, host_bsphere_radius(meshes))) return 1;
        d.lights = sc->lights.data();
        d.light_pmf = sc->lt.pmf.data();
        d.light_cdf = sc->lt.cdf.data();
        d.light_areas = sc->lt.areas.data();
        d.area_cdf_pool = sc->lt.pool.data();
        d.area_cdf_offset = sc->lt.offsets.data();
    }
    if (d.use_primary_edge || d.use_secondary_edge) {
        host_build_edges(sc->shapes, meshes, d.cam, d.use_primary_edge != 0, sc->et);
        d.edges = sc->et.edges.data();
        d.num_edges = (int)sc->et.edges.size();
        d.prim_edge_pmf = sc->et.prim_pmf.data();
        d.prim_edge_cdf = sc->et.prim_cdf.data();
        d.edge_root_cs = d.edge_root_ncs = RB_EDGE_EMPTY;
        if (d.use_secondary_edge) {
            host_build_edge_tree(sc->shapes, meshes, sc->et.edges, d.cam, sc->tree);
            d.edge_nodes = sc->tree.nodes.data();
            d.edge_root_cs = sc->tree.root_cs;
            d.edge_root_ncs = sc->tree.root_ncs;
            d.edge_bounds_expand = sc->tree.expand;
            d.ltc_table = ltc;
        }
    }
    return 0;
}

extern "C" int rb_scene_create(const rb_scene_desc* desc, rb_scene** out) {
    if (const char* err = host_check_scene_desc(*desc)) {
        g_err = err;
        return 1;
    }
    rb_scene* sc = new rb_scene();
    memset(&sc->dev, 0, sizeof(DevScene));
    sc->gpu_index = desc->gpu_index;
    std::vector<unsigned char> bytes;
    if (!load_table(RB_DATA_DIR "/sobol_joe_kuo_1024x52_u64.bin", 8, bytes, 1024 * 52)) { g_err = "emu: sobol table not found"; delete sc; return 1; }
    sc->sobol.resize(1024 * 52);
    memcpy(sc->sobol.data(), bytes.data(), bytes.size());
    if (!load_table(RB_DATA_DIR "/ltc_blinn_phong_128x128x9_f32.bin", 4, bytes, 128 * 128 * 9)) { g_err = "emu: ltc table not found"; delete sc; return 1; }
    sc->ltc.resize(128 * 128 * 9);
    memcpy(sc->ltc.data(), bytes.data(), bytes.size());
    sc->dev.sobol_matrices = sc->sobol.data();
    sc->dev.ltc_table = sc->ltc.data();
    if (emu_build(sc, desc)) {
        delete sc;
        return 1;
    }
    *out = sc;
    return 0;
}
// Re-target at a descriptor of the same structure: the same checks as the library, then every table is rebuilt from the descriptor with
// the host builders (the library rebuilds only what changed, on the GPU; the tables are the same either way).
extern "C" int rb_scene_update(rb_scene* sc, const rb_scene_desc* desc, int, void*) {
    const char* err = host_check_scene_desc(*desc);
    if (!err) err = host_check_same_structure(*desc, sc->shapes, (int)sc->materials.size(), sc->lights, sc->dev, sc->gpu_index, sc->max_generic);
    if (err) {
        g_err = err;
        if (g_err.compare(0, 16, "rb_scene_create:") == 0) g_err = "rb_scene_update:" + g_err.substr(16);
        return 1;
    }
    sc->incomplete = emu_build(sc, desc) != 0;
    if (sc->incomplete && g_err.compare(0, 16, "rb_scene_create:") == 0) g_err = "rb_scene_update:" + g_err.substr(16);
    return sc->incomplete ? 1 : 0;
}
extern "C" int rb_scene_table(const rb_scene* sc, int which, void* out, size_t bytes, size_t* size) {
    const DevScene& d = sc->dev;
    const bool prim = d.use_primary_edge && d.num_edges > 0, lights = d.num_lights > 0;
    const void* src = nullptr;
    size_t n = 0;
    switch (which) {
        case RB_TABLE_BVH_NODES: src = sc->nodes.data(); n = sizeof(BVHNode) * (size_t)std::max(d.num_tris - 1, 0); break;
        case RB_TABLE_BVH_TRIANGLES: src = sc->tris.data(); n = sizeof(BVHTri) * sc->tris.size(); break;
        case RB_TABLE_LIGHT_PMF: src = sc->lt.pmf.data(); n = lights ? sizeof(double) * sc->lt.pmf.size() : 0; break;
        case RB_TABLE_LIGHT_CDF: src = sc->lt.cdf.data(); n = lights ? sizeof(double) * sc->lt.cdf.size() : 0; break;
        case RB_TABLE_LIGHT_AREAS: src = sc->lt.areas.data(); n = lights ? sizeof(double) * sc->lt.areas.size() : 0; break;
        case RB_TABLE_AREA_CDF_POOL: src = sc->lt.pool.data(); n = lights ? sizeof(double) * sc->lt.pool.size() : 0; break;
        case RB_TABLE_AREA_CDF_OFFSETS: src = sc->lt.offsets.data(); n = lights ? sizeof(int) * sc->lt.offsets.size() : 0; break;
        case RB_TABLE_PRIMARY_EDGE_PMF: src = sc->et.prim_pmf.data(); n = prim ? sizeof(double) * (size_t)d.num_edges : 0; break;
        case RB_TABLE_PRIMARY_EDGE_CDF: src = sc->et.prim_cdf.data(); n = prim ? sizeof(double) * (size_t)d.num_edges : 0; break;
        default: g_err = "rb_scene_table: unknown table"; return 1;
    }
    if (size) *size = n;
    if (out && bytes > 0 && n > 0) memcpy(out, src, std::min(bytes, n));
    return 0;
}
// Ray queries against this build's median-split tree, through the same traversal and brute force as the library (host pointers).
extern "C" int rb_scene_trace_rays(const rb_scene* sc, const float* rays, int num_rays, int flags, int* ids, float* t) {
    if (!sc || num_rays < 0) {
        g_err = !sc ? "rb_scene_trace_rays: null scene" : "rb_scene_trace_rays: negative number of rays";
        return 1;
    }
    const DevScene& d = sc->dev;
    const float4* nodes4 = reinterpret_cast<const float4*>(d.bvh_nodes);
    const float4* tris4 = reinterpret_cast<const float4*>(d.bvh_tris);
    for (int i = 0; i < num_rays; i++) {
        const float* r = rays + 8 * (size_t)i;
        BvhHit h;
        switch (flags & (RB_TRACE_ANY_HIT | RB_TRACE_BRUTE_FORCE)) {
            case 0: h = bvh_trace_impl<false>(nodes4, tris4, d.bvh_root, d.num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7]); break;
            case RB_TRACE_ANY_HIT: h = bvh_trace_impl<true>(nodes4, tris4, d.bvh_root, d.num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7]); break;
            case RB_TRACE_BRUTE_FORCE: h = bvh_brute_force<false>(tris4, d.num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7]); break;
            default: h = bvh_brute_force<true>(tris4, d.num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7]); break;
        }
        ids[2 * (size_t)i] = h.shape_id;
        ids[2 * (size_t)i + 1] = h.tri_id;
        t[i] = h.t;
    }
    return 0;
}
// Texture lookups and adjoints through the same functions as the library's hook, one query after another (host pointers; the scatter
// is the emulator's single-lane plain add).  The argument checks that do not involve device memory are the library's.
extern "C" int rb_texture_test(const rb_texture* tex, const rb_texture* d_tex, const float* queries, int n, const float* d_values, float* values,
                               float* d_queries, void*) {
    const char* err = nullptr;
    if (n < 0) err = "negative number of queries";
    else if (tex == nullptr) err = "null texture";
    else if (d_values != nullptr && d_tex == nullptr) err = "d_values needs a gradient texture";
    else if (tex->channels < 1) err = "channels must be at least 1";
    else if (tex->num_levels < 1 || tex->num_levels > RB_MAX_MIP_LEVELS) err = "num_levels must be in [1, RB_MAX_MIP_LEVELS]";
    else if (d_values != nullptr && (d_tex->num_levels != tex->num_levels || d_tex->channels != tex->channels))
        err = "the gradient texture must have the texture's levels and channels";
    if (err == nullptr && !tex_is_constant(*tex))
        for (int l = 0; l < tex->num_levels; l++)
            if (tex->width[l] < 1 || tex->height[l] < 1) err = "every level of a texture that is not constant needs a positive width and height";
    if (err != nullptr) {
        g_err = std::string("rb_texture_test: ") + err;
        return 1;
    }
    const int nch = tex->channels;
    for (int i = 0; i < n; i++) {
        const float* q = queries + 6 * (size_t)i;
        const V2 uv = mk2(q[0], q[1]), du_dxy = mk2(q[2], q[3]), dv_dxy = mk2(q[4], q[5]);
        float* out = values + (size_t)nch * i;
        if (nch == 1 || nch == 3) {
            const V3 v = tex_eval(*tex, nch, uv, du_dxy, dv_dxy);
            out[0] = v.x;
            if (nch == 3) {
                out[1] = v.y;
                out[2] = v.z;
            }
        } else {
            tex_eval_channels(*tex, nch, uv, du_dxy, dv_dxy, out);
        }
        if (d_values == nullptr) continue;
        V2 d_uv = zero2(), d_du = zero2(), d_dv = zero2();
        d_tex_eval(*tex, *d_tex, nch, uv, du_dxy, dv_dxy, d_values + (size_t)nch * i, d_uv, d_du, d_dv);
        if (d_queries != nullptr) {
            float* dq = d_queries + 6 * (size_t)i;
            dq[0] = d_uv.x;
            dq[1] = d_uv.y;
            dq[2] = d_du.x;
            dq[3] = d_du.y;
            dq[4] = d_dv.x;
            dq[5] = d_dv.y;
        }
    }
    return 0;
}
extern "C" int rb_scene_edge_list(const rb_scene* sc, int* num_edges, int* edges_out, size_t edges_bytes) {
    if (num_edges) *num_edges = sc->dev.num_edges;
    if (edges_out && edges_bytes > 0) memcpy(edges_out, sc->et.edges.data(), std::min(edges_bytes, sizeof(Edge) * (size_t)sc->dev.num_edges));
    return 0;
}
// Re-target at another camera: the camera-dependent tables (primary-edge distribution, both edge trees) are rebuilt with the host
// builders; geometry, BVH, lights and the edge list are kept (mirrors rb_scene_set_camera of the product, which rebuilds them on the GPU).
extern "C" int rb_scene_set_camera(rb_scene* sc, const rb_camera* cam) {
    DevScene& d = sc->dev;
    sc->cam = *cam;
    host_setup_camera(*cam, d.cam);
    if (d.num_edges > 0) {
        std::vector<HostMesh> meshes(d.num_shapes);
        for (int s = 0; s < d.num_shapes; s++) {
            meshes[s].vertices.assign(sc->shapes[s].vertices, sc->shapes[s].vertices + 3 * (size_t)sc->shapes[s].num_vertices);
            meshes[s].indices.assign(sc->shapes[s].indices, sc->shapes[s].indices + 3 * (size_t)sc->shapes[s].num_triangles);
        }
        if (d.use_primary_edge) {
            host_primary_edge_distribution(sc->shapes, meshes, d.cam, sc->et);
            d.prim_edge_pmf = sc->et.prim_pmf.data();
            d.prim_edge_cdf = sc->et.prim_cdf.data();
        }
        if (d.use_secondary_edge) {
            host_build_edge_tree(sc->shapes, meshes, sc->et.edges, d.cam, sc->tree);
            d.edge_nodes = sc->tree.nodes.data();
            d.edge_root_cs = sc->tree.root_cs;
            d.edge_root_ncs = sc->tree.root_ncs;
            d.edge_bounds_expand = sc->tree.expand;
        }
    }
    return 0;
}
extern "C" void rb_scene_destroy(rb_scene* sc) { delete sc; }
extern "C" int rb_scene_max_generic_texture_dimension(const rb_scene* sc) { return sc->max_generic; }
extern "C" int rb_compute_num_channels(const int* ch, int n, int mg) { return host_compute_num_channels(ch, n, mg); }
extern "C" int rb_scene_set_partition(rb_scene* sc, int part, int num_parts, int rps) {
    sc->part = part; sc->num_parts = num_parts; sc->rps = rps;
    return 0;
}
extern "C" int rb_scene_last_stage_stats(const rb_scene*, float* ms, double* v, double* h) {
    if (ms) for (int i = 0; i < 4; i++) ms[i] = 0;
    if (v) *v = 0;
    if (h) *h = 0;
    return 0;
}
extern "C" int rb_scene_build_ms(const rb_scene*, float* ms) { ms[0] = ms[1] = ms[2] = 0; return 0; }
extern "C" int rb_scene_last_stats(const rb_scene*, int* n, float* ms) {
    if (n) *n = 0;
    if (ms) *ms = 0;
    return 0;
}

// rb_render (records == nullptr) and rb_render_exact (the accumulators are added into `records` instead of rounded), as in the library.
static int emu_render(const rb_scene* scene, const rb_options* opt, float* image, const float* d_image, const rb_dscene_desc* d_scene, float* screen_grad,
                      long long* records, size_t count) {
    if (!scene || !opt) {
        g_err = "rb_render: null scene / options";
        return 1;
    }
    if (scene->incomplete) {
        g_err = "rb_render: the scene's last update failed; update it again or build a new scene";
        return 1;
    }
    KernelArgs ka;
    if (const char* err = setup_kernel_args(*opt, scene->cam, scene->max_generic, scene->part, scene->num_parts, scene->rps, image, d_image, d_scene,
                                            screen_grad, ka)) {
        g_err = err;
        return 1;
    }
    const RenderParams& rp = ka.rp;
    if (rp.vp_w <= 0 || rp.vp_h <= 0 || rp.spp == 0) return 0;
    const DevScene& sc = scene->dev;
    if (image && !rp.only_radiance) {
        for (int j = 0; j < ka.owned_rows; j++)
            for (int x = 0; x < rp.vp_w; x++) {
                const int y = owned_row_to_row(rp, j), pixel = y * rp.vp_w + x;
                float acc[RB_MAX_ND] = {0};
                int ids[3] = {-1, -1, -1}, last = -1;
                for (int s = 0; s < rp.spp; s++) {
                    int cur[3] = {-1, -1, -1};
                    if (forward_sample_channels(sc, rp, pixel, x, y, s, acc, cur)) { last = s; ids[0] = cur[0]; ids[1] = cur[1]; ids[2] = cur[2]; }
                }
                write_gbuffer_pixel(rp, acc, ids, last >= 0, image + (size_t)rp.nd * pixel);
            }
    } else if (image) {
        for (int j = 0; j < ka.owned_rows; j++)
            for (int x = 0; x < rp.vp_w; x++) {
                const int y = owned_row_to_row(rp, j), pixel = y * rp.vp_w + x;
                V3 acc = zero3();
                for (int s = 0; s < rp.spp; s++) acc += forward_sample(sc, rp, pixel, x, y, s);
                float* px = image + (size_t)rp.nd * pixel + rp.rad_dim;
                px[0] += (float)acc.x; px[1] += (float)acc.y; px[2] += (float)acc.z;
            }
    }
    if (d_image) {
        if (const char* err = setup_backward(*d_scene, sc, ka)) {
            g_err = err;
            return 1;
        }
        std::vector<double> cam_accum(RB_CAM_ACC, 0.0);
        std::vector<float> cam_f(RB_CAM_ACC, 0.f);
        ka.ds.shapes = d_scene->shapes;
        ka.ds.materials = d_scene->materials;
        ka.ds.light_intensity = d_scene->light_intensity;
        ka.ds.cam_accum = cam_accum.data();
        CamAcc acc;
        acc.base = cam_f.data();
        acc.stride = 1;
        // deterministic mode: every scatter and camera contribution into the exact accumulators of the library's layout
        const bool det = opt->deterministic != 0 || records != nullptr;
        ExactLayout xl;
        std::vector<long long> xacc;
        struct ExactReset {
            ~ExactReset() { rb_emu_exact_acc = nullptr; }
        } exact_reset;
        long long exact_samples = 0;
        const long long exact_max_samples = std::max(1LL, exact_band_samples(rp.max_bounces));
        auto exact_sample_done = [&]() { // the library's bound: normalise after as many samples as one of its bands holds at most
            if (det && ++exact_samples % exact_max_samples == 0)
                for (long long i = 0; i <= xl.num_acc; i++) exact_normalise(&xacc[(size_t)i * RB_EXACT_WORDS]);
        };
        if (det) {
            exact_layout(*d_scene, scene->shapes.data(), scene->materials.data(), sc, ka, xl);
            if (records && xl.overlaps) {
                g_err = "rb_render_exact: gradient buffers of d_scene overlap; records need disjoint buffers";
                return 1;
            }
            if (records && (size_t)xl.num_records != count) {
                g_err = "rb_render_exact: count is " + std::to_string(count) + " but the descriptor has " + std::to_string(xl.num_records) +
                        " records (rb_exact_record_count)";
                return 1;
            }
            xacc.assign((size_t)(xl.num_acc + 1) * RB_EXACT_WORDS, 0);
            ka.ds.shapes = xl.shapes.data();
            ka.ds.materials = xl.materials.data();
            ka.ds.light_intensity = xl.lights.data();
            ka.ds.env_values = xl.env_values;
            ka.ds.env_w2e = xl.env_w2e;
            ka.screen_grad = xl.screen_grad;
            rb_emu_exact_acc = xacc.data();
            acc.exact = xacc.data();
        }
        std::vector<VertexRec> recs(rp.max_bounces + 2);
#ifdef RB_EMU_REF_STREAMS
        // rank of every (sample, pixel) in the reference's compacted active list of each depth (pixels in ascending order)
        const int mbr = std::max(rp.max_bounces, 1);
        const size_t npx = (size_t)rp.vp_w * rp.vp_h;
        std::vector<int> ranks((size_t)rp.spp * npx * mbr, 0);
        for (int s = 0; s < rp.spp; s++) {
            std::vector<int> counter(mbr, 0);
            for (size_t pixel = 0; pixel < npx; pixel++) {
                int nrec = bwd_trace(sc, rp, (int)pixel, (int)(pixel % rp.vp_w), (int)(pixel / rp.vp_w), s, recs.data(), 1);
                for (int d = 0; d < nrec && d < mbr; d++) ranks[((size_t)s * npx + pixel) * mbr + d] = counter[d]++;
            }
        }
#endif
        for (int j = 0; j < ka.owned_rows; j++)
            for (int x = 0; x < rp.vp_w; x++)
                for (int s = 0; s < rp.spp; s++) {
                    const int y = owned_row_to_row(rp, j);
#ifdef RB_EMU_REF_STREAMS
                    rb_emu_rank = &ranks[((size_t)s * npx + (size_t)y * rp.vp_w + x) * mbr];
#endif
                    backward_sample(sc, ka, y * rp.vp_w + x, x, y, s, recs.data(), acc);
                    for (int k = 0; k < RB_CAM_ACC; k++) { cam_accum[k] += cam_f[k]; cam_f[k] = 0.f; }
                    exact_sample_done();
                }
        if (primary_edge_pass_runs(sc)) {
            long long n_px = (long long)rp.vp_w * rp.vp_h;
            for (long long i = 0; i < n_px; i++)
                for (int s = 0; s < rp.spp; s++) {
                    if (i % rp.num_parts != rp.part) continue; // primary-edge samples are sharded by sample index
                    primary_edge_sample(sc, ka, i, s, primary_edge_dim_base(sc, rp), acc);
                    for (int k = 0; k < RB_CAM_ACC; k++) { cam_accum[k] += cam_f[k]; cam_f[k] = 0.f; }
                    exact_sample_done();
                }
        }
        if (records) {
            for (long long i = 0; i < xl.num_acc; i++)
                exact_export(&xacc[(size_t)i * RB_EXACT_WORDS],
                             records + exact_record_of(i, xl.ranges.data(), xl.rec_first.data(), (int)xl.ranges.size(), RB_CAM_ACC) * RB_EXACT_RECORD_WORDS);
            return 0;
        }
        if (det)
            for (long long i = 0; i < xl.num_acc; i++) exact_finalise(xacc.data(), i, xl.ranges.data(), (int)xl.ranges.size(), cam_accum.data(), RB_CAM_ACC);
        finish_camera(sc.cam, cam_accum.data(), d_scene->camera);
    }
    return 0;
}
extern "C" int rb_render(const rb_scene* scene, const rb_options* opt, float* image, const float* d_image, const rb_dscene_desc* d_scene,
                         float* screen_grad, void*) {
    return emu_render(scene, opt, image, d_image, d_scene, screen_grad, nullptr, 0);
}
extern "C" int rb_exact_record_count(const rb_scene* scene, const rb_options* opt, const rb_dscene_desc* d_scene, float* screen_grad, size_t* count,
                                     uint64_t* fingerprint) {
    if (!scene || !opt || !count) {
        g_err = "rb_exact_record_count: null scene / options / count";
        return 1;
    }
    KernelArgs ka;
    ExactLayout xl;
    std::string err;
    if (const char* e = exact_record_layout("rb_exact_record_count", *opt, scene->cam, scene->max_generic, d_scene, screen_grad, scene->shapes.data(),
                                            scene->materials.data(), scene->dev, ka, xl, err)) {
        g_err = e;
        return 1;
    }
    *count = (size_t)xl.num_records;
    if (fingerprint) *fingerprint = xl.fingerprint;
    return 0;
}
extern "C" int rb_render_exact(const rb_scene* scene, const rb_options* opt, const float* d_image, const rb_dscene_desc* d_scene, float* screen_grad,
                               long long* records, size_t count, void*) {
    if (!d_image || !d_scene || !records) {
        g_err = "rb_render_exact: null d_rendered_image / d_scene / records";
        return 1;
    }
    return emu_render(scene, opt, nullptr, d_image, d_scene, screen_grad, records, count);
}
extern "C" int rb_exact_round(const rb_scene* scene, const rb_options* opt, const rb_dscene_desc* d_scene, float* screen_grad, const long long* records,
                              size_t count, void*) {
    if (!scene || !opt || !records) {
        g_err = "rb_exact_round: null scene / options / records";
        return 1;
    }
    if (scene->incomplete) {
        g_err = "rb_exact_round: the scene's last update failed; update it again or build a new scene";
        return 1;
    }
    KernelArgs ka;
    ExactLayout xl;
    std::string err;
    if (const char* e = exact_record_layout("rb_exact_round", *opt, scene->cam, scene->max_generic, d_scene, screen_grad, scene->shapes.data(),
                                            scene->materials.data(), scene->dev, ka, xl, err)) {
        g_err = e;
        return 1;
    }
    if ((size_t)xl.num_records != count) {
        g_err = "rb_exact_round: count is " + std::to_string(count) + " but the descriptor has " + std::to_string(xl.num_records) +
                " records (rb_exact_record_count)";
        return 1;
    }
    std::vector<long long> acc((size_t)(xl.num_acc + 1) * RB_EXACT_WORDS, 0);
    std::vector<double> cam_accum(RB_CAM_ACC, 0.0);
    for (long long i = 0; i < xl.num_acc; i++)
        exact_import(records + exact_record_of(i, xl.ranges.data(), xl.rec_first.data(), (int)xl.ranges.size(), RB_CAM_ACC) * RB_EXACT_RECORD_WORDS,
                     &acc[(size_t)i * RB_EXACT_WORDS]);
    for (long long i = 0; i < xl.num_acc; i++) exact_finalise(acc.data(), i, xl.ranges.data(), (int)xl.ranges.size(), cam_accum.data(), RB_CAM_ACC);
    finish_camera(scene->dev.cam, cam_accum.data(), d_scene->camera);
    return 0;
}
