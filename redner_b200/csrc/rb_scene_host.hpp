// Host-side scene preprocessing shared by rb_scene.cu and the debug emulator (tools/cpu_emu):
//   light PMF/CDF + per-light triangle-area CDFs   src/scene.cpp:197-253, compute_area_cdf :38-61 (serial, double; steps shared with
//                                                  rb_light_build.cu: rb_light_build.cuh)
//   edge list + primary-edge distribution          src/edge.cpp:43-214, :233-331
//   secondary-edge trees                           src/edge_tree.cpp:724-882 (steps shared with rb_edge_tree.cu: rb_edge_tree.cuh)
//   camera matrices in double                      src/camera.h:44-55, src/transform.h:9-27
#pragma once
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <thread>
#include <vector>

#include "rb_edge_tree.cuh"
#include "rb_light_build.cuh"

struct HostMesh {
    std::vector<float> vertices;
    std::vector<int> indices;
};
struct HostLightTables {
    std::vector<double> pmf, cdf, areas, pool;
    std::vector<int> offsets;
};
struct HostEdgeTables {
    std::vector<Edge> edges;
    std::vector<double> prim_pmf, prim_cdf;
};

// ---- scene descriptor -> scene, shared by both rb_scene_create (rb_scene.cu and the emulator's)
// The pixel filter as the kernels see it: { 0, 0 } is the 1-pixel box.
inline rb_pixel_filter host_pixel_filter(const rb_pixel_filter& f) {
    if (f.type == 0 && f.width == 0.f) return rb_pixel_filter{RB_FILTER_BOX, 1.f};
    return f;
}
inline bool host_pixel_box(const rb_pixel_filter& f) { return f.type == RB_FILTER_BOX && f.width == 1.f; }
// The camera against the scene's pixel filter: a filter other than the 1-pixel box needs a linear projection without a lens model, and a
// thin lens (rb_camera::lens_radius > 0) a perspective camera without distortion, with the 1-pixel box and an intrinsic matrix whose
// last row is (0, 0, k) (the primary-edge distribution bounds the circle of confusion through it).
inline const char* host_check_camera(const rb_pixel_filter& f, const rb_camera& cam) {
    if (!host_pixel_box(host_pixel_filter(f)) && (cam.camera_type == RB_CAMERA_FISHEYE || cam.camera_type == RB_CAMERA_PANORAMA || cam.has_distortion))
        return "rb_scene_create: pixel filters other than the 1-pixel box need a perspective or orthographic camera without lens distortion";
    if (!(std::isfinite(cam.lens_radius) && cam.lens_radius >= 0.f)) return "rb_scene_create: the lens_radius of a thin lens must be finite and >= 0";
    if (cam.lens_radius == 0.f) return nullptr;
    if (!(std::isfinite(cam.focus_distance) && cam.focus_distance > 0.f)) return "rb_scene_create: the focus_distance of a thin lens must be finite and > 0";
    if (cam.camera_type != RB_CAMERA_PERSPECTIVE) return "rb_scene_create: a thin lens (lens_radius > 0) needs a perspective camera";
    if (cam.has_distortion) return "rb_scene_create: a thin lens (lens_radius > 0) cannot be combined with a distortion model";
    if (!host_pixel_box(host_pixel_filter(f))) return "rb_scene_create: a thin lens (lens_radius > 0) needs the 1-pixel box pixel filter";
    if (cam.intrinsic_mat[6] != 0.f || cam.intrinsic_mat[7] != 0.f || cam.intrinsic_mat[8] == 0.f)
        return "rb_scene_create: a thin lens (lens_radius > 0) needs an intrinsic_mat whose last row is (0, 0, k) with k != 0";
    return nullptr;
}
inline const char* host_check_pixel_filter(const rb_scene_desc& desc) {
    const rb_pixel_filter f = host_pixel_filter(desc.pixel_filter);
    if (f.type != RB_FILTER_BOX && f.type != RB_FILTER_TENT && f.type != RB_FILTER_GAUSSIAN) return "rb_scene_create: unknown pixel filter type";
    if (!(f.width > 0.f && f.width <= 4.f)) return "rb_scene_create: pixel filter width must lie in (0, 4] pixels";
    return host_check_camera(f, desc.camera);
}
inline void host_setup_pixel_filter(const rb_pixel_filter& f, DevCamera& dc) {
    const rb_pixel_filter g = host_pixel_filter(f);
    dc.filter_type = g.type;
    dc.filter_width = g.width;
}
// An area light's emission texture (rb_area_light::emission); returns the error message, or null.
inline const char* host_check_emission(const rb_texture& t) {
    if (t.num_levels == 0) return nullptr;
    if (t.num_levels < 0 || t.num_levels > RB_MAX_MIP_LEVELS) return "rb_scene_create: a light's emission texture needs num_levels in [0, RB_MAX_MIP_LEVELS]";
    if (t.channels != 1 && t.channels != 3) return "rb_scene_create: a light's emission texture needs 1 or 3 channels";
    if (t.uv_scale == nullptr) return "rb_scene_create: a light's emission texture needs a uv_scale";
    const bool constant = t.width[0] == 0 && t.height[0] == 0;
    for (int k = 0; k < t.num_levels; k++) {
        if (t.texels[k] == nullptr) return "rb_scene_create: a level of a light's emission texture has no texels";
        if (!constant && (t.width[k] <= 0 || t.height[k] <= 0)) return "rb_scene_create: a level of a light's emission texture needs a positive size";
    }
    return nullptr;
}
// Index, pixel-filter, specular-model and emission-texture checks of the descriptor; returns the error message, or null.
inline const char* host_check_scene_desc(const rb_scene_desc& desc) {
    if (const char* err = host_check_pixel_filter(desc)) return err;
    for (int m = 0; m < desc.num_materials; m++)
        if (desc.materials[m].specular_model != RB_SPECULAR_BLINN_PHONG && desc.materials[m].specular_model != RB_SPECULAR_GGX)
            return "rb_scene_create: material specular_model must be RB_SPECULAR_BLINN_PHONG (0) or RB_SPECULAR_GGX (1)";
    for (int l = 0; l < desc.num_lights; l++) {
        if (desc.lights[l].shape_id < 0 || desc.lights[l].shape_id >= desc.num_shapes) return "rb_scene_create: area light refers to an invalid shape";
        if (const char* err = host_check_emission(desc.lights[l].emission)) return err;
        if (desc.lights[l].emission_sampling != RB_EMISSION_SAMPLE_AREA && desc.lights[l].emission_sampling != RB_EMISSION_SAMPLE_TEXTURE)
            return "rb_scene_create: a light's emission_sampling must be RB_EMISSION_SAMPLE_AREA (0) or RB_EMISSION_SAMPLE_TEXTURE (1)";
    }
    for (int s = 0; s < desc.num_shapes; s++) {
        const rb_shape& sh = desc.shapes[s];
        if (sh.material_id < 0 || sh.material_id >= desc.num_materials) return "rb_scene_create: shape refers to an invalid material";
        if (sh.vertices == nullptr || sh.indices == nullptr) return "rb_scene_create: shape without vertices / indices";
    }
    return nullptr;
}
inline std::vector<DevLight> host_area_lights(const rb_scene_desc& desc) {
    std::vector<DevLight> out;
    for (int l = 0; l < desc.num_lights; l++) {
        DevLight dl;
        dl.shape_id = desc.lights[l].shape_id;
        for (int k = 0; k < 3; k++) dl.intensity[k] = desc.lights[l].intensity[k];
        dl.two_sided = desc.lights[l].two_sided;
        dl.directly_visible = desc.lights[l].directly_visible;
        out.push_back(dl);
    }
    return out;
}
// The lights' emission textures (one per area light, num_levels == 0: none).
inline std::vector<rb_texture> host_light_emission(const rb_scene_desc& desc) {
    std::vector<rb_texture> out;
    for (int l = 0; l < desc.num_lights; l++) out.push_back(desc.lights[l].emission);
    return out;
}
// Per area light: 1 when it samples by its emission texture (RB_EMISSION_SAMPLE_TEXTURE and a texture that is not constant), else 0.
inline std::vector<int> host_light_sampling(const rb_scene_desc& desc) {
    std::vector<int> out;
    for (int l = 0; l < desc.num_lights; l++) {
        const rb_texture& t = desc.lights[l].emission;
        out.push_back(desc.lights[l].emission_sampling == RB_EMISSION_SAMPLE_TEXTURE && t.num_levels > 0 && !(t.width[0] == 0 && t.height[0] == 0) ? 1 : 0);
    }
    return out;
}
inline bool host_any(const std::vector<int>& v) {
    for (int x : v)
        if (x) return true;
    return false;
}
// Layout of the emission-sampling data: per light its offset into the pool (doubles) and its level-0 size; returns the pool size.
inline size_t host_light_sampling_layout(const std::vector<int>& on, const std::vector<rb_texture>& emission, const std::vector<DevLight>& lights,
                                         const std::vector<rb_shape>& shapes, std::vector<size_t>& offsets) {
    size_t n = 0;
    offsets.assign(on.size(), 0);
    for (size_t l = 0; l < on.size(); l++) {
        offsets[l] = n;
        if (on[l]) n += ls_size(emission[l].width[0], emission[l].height[0], shapes[lights[l].shape_id].num_triangles);
    }
    return n;
}
const char* const RB_LS_UV_ERROR =
    "rb_scene_create: emission sampling needs the scaled texture coordinates of a light (uv * uv_scale * level-0 size) to be finite and below 2^24 cells in magnitude";
// The emission-sampling tables with the steps of rb_light_build.cuh in serial loops (`shapes` and the textures hold host pointers): fills
// `pool` and, per light, S[l] (0 for a light that samples by area).  Returns false with `err` set when a light's texture coordinates are out
// of range.
inline bool host_build_light_sampling(const std::vector<int>& on, const std::vector<rb_texture>& emission, const std::vector<DevLight>& lights,
                                      const std::vector<rb_shape>& shapes, const std::vector<size_t>& offsets, std::vector<double>& pool,
                                      std::vector<double>& S, std::string& err) {
    S.assign(on.size(), 0.0);
    for (size_t l = 0; l < on.size(); l++) {
        if (!on[l]) continue;
        const rb_texture& t = emission[l];
        const int w = t.width[0], h = t.height[0];
        const rb_shape& sh = shapes[lights[l].shape_id];
        double* d = pool.data() + offsets[l];
        double *cells = d + ls_cells(w, h), *sat = d + ls_sat(w, h), *recs = d + ls_tris(w, h);
        for (int j = 0; j < h; j++)
            for (int i = 0; i < w; i++) cells[(size_t)j * w + i] = ls_cell_weight(t.texels[0], t.channels, w, h, i, j);
        for (int j = 0; j < h; j++) ls_sat_row(cells, sat, w, j);
        for (int i = 0; i < w; i++) ls_sat_col(sat, w, h, i);
        for (int k = 0; k < sh.num_triangles; k++)
            if (!ls_tri_record(sh, k, t.uv_scale[0], t.uv_scale[1], w, h, sat, recs + RB_LS_TRI * (size_t)k)) {
                err = RB_LS_UV_ERROR;
                return false;
            }
        d[0] = S[l] = ls_scan(recs, sh.num_triangles);
        d[1] = 0;
    }
    return true;
}
inline int host_max_generic_texture_dimension(const rb_scene_desc& desc) {
    int n = 0;
    for (int m = 0; m < desc.num_materials; m++)
        if (desc.materials[m].generic_texture.num_levels > 0) n = std::max(n, desc.materials[m].generic_texture.channels);
    return n;
}
// The environment map of the descriptor (may be null) -> has_envmap and env of the scene.
inline void host_setup_envmap(const rb_envmap* e, DevScene& d) {
    d.has_envmap = e != nullptr;
    if (!e) return;
    d.env.values = e->values;
    memcpy(d.env.w2e, e->world_to_env, sizeof(d.env.w2e));
    memcpy(d.env.e2w, e->env_to_world, sizeof(d.env.e2w));
    d.env.cdf_ys = e->sample_cdf_ys;
    d.env.cdf_xs = e->sample_cdf_xs;
    d.env.pdf_norm = e->pdf_norm;
    d.env.directly_visible = e->directly_visible;
}
// rb_scene_update re-targets a scene only at a descriptor with the structure of its build: the scene's shapes, light list and
// DevScene flags against the new descriptor.  Returns the error message, or null.
inline const char* host_check_same_structure(const rb_scene_desc& d, const std::vector<rb_shape>& shapes, int num_materials, const std::vector<DevLight>& lights,
                                             const DevScene& dev, int gpu_index, int max_generic_texture_dimension) {
    if (d.num_shapes != (int)shapes.size() || d.num_materials != num_materials || d.num_lights != (int)lights.size())
        return "rb_scene_update: the numbers of shapes, materials and lights must not change";
    for (int s = 0; s < d.num_shapes; s++) {
        const rb_shape &a = d.shapes[s], &b = shapes[s];
        if (a.num_vertices != b.num_vertices || a.num_triangles != b.num_triangles || a.num_uv_vertices != b.num_uv_vertices ||
            a.num_normal_vertices != b.num_normal_vertices)
            return "rb_scene_update: a shape's vertex, triangle, uv or normal count changed";
        if (a.material_id != b.material_id || a.light_id != b.light_id) return "rb_scene_update: a shape's material or light id changed";
        if ((a.uvs == nullptr) != (b.uvs == nullptr) || (a.normals == nullptr) != (b.normals == nullptr) || (a.uv_indices == nullptr) != (b.uv_indices == nullptr) ||
            (a.normal_indices == nullptr) != (b.normal_indices == nullptr) || (a.colors == nullptr) != (b.colors == nullptr))
            return "rb_scene_update: a shape gained or lost an optional buffer";
    }
    for (int l = 0; l < d.num_lights; l++)
        if (d.lights[l].shape_id != lights[l].shape_id) return "rb_scene_update: an area light's shape changed";
    if ((d.envmap != nullptr) != (dev.has_envmap != 0)) return "rb_scene_update: the environment map was added or removed";
    if (d.use_primary_edge_sampling != dev.use_primary_edge || d.use_secondary_edge_sampling != dev.use_secondary_edge)
        return "rb_scene_update: the edge-sampling flags changed";
    if (d.gpu_index != gpu_index) return "rb_scene_update: gpu_index changed";
    if (host_max_generic_texture_dimension(d) != max_generic_texture_dimension) return "rb_scene_update: the generic texture dimension changed";
    return nullptr;
}

// Radius of the scene's bounding sphere as the reference computes it (src/scene.cpp:156-195) -- including its slip of
// folding each shape's Y extent into the Z bounds; the radius only scales the environment map's selection weight.
inline double host_bsphere_radius(const std::vector<HostMesh>& meshes) {
    if (meshes.empty()) return 0;
    float inf = std::numeric_limits<float>::infinity();
    float lo[2] = {inf, inf}, hi[2] = {-inf, -inf};
    for (const HostMesh& m : meshes)
        for (size_t v = 0; v + 2 < m.vertices.size(); v += 3)
            for (int a = 0; a < 2; a++) {
                lo[a] = std::min(lo[a], m.vertices[v + a]);
                hi[a] = std::max(hi[a], m.vertices[v + a]);
            }
    return lt_bsphere_radius(lo, hi);
}
// `has_env` appends the environment map as the last light (src/scene.cpp:197-253).  The steps are those of rb_light_build.cuh, which
// rb_light_build.cu runs on the device.
// `sel`: per light, S of its emission sampling (ls_selection_area), or null.
inline bool host_build_lights(const std::vector<DevLight>& lights, const std::vector<HostMesh>& meshes, HostLightTables& out, std::string& err,
                              bool has_env = false, double env_pdf_norm = 0, double bsphere_radius = 0, const std::vector<double>* sel = nullptr) {
    int L = (int)lights.size();
    out.pmf.assign(L, 0);
    out.cdf.assign(L, 0);
    out.areas.assign(L, 0);
    out.offsets.assign(L, 0);
    out.pool.clear();
    for (int l = 0; l < L; l++) {
        const HostMesh& m = meshes[lights[l].shape_id];
        int T = (int)m.indices.size() / 3;
        out.offsets[l] = (int)out.pool.size();
        std::vector<double> a(T);
        for (int t = 0; t < T; t++) a[t] = lt_triangle_area(m.vertices.data(), &m.indices[3 * (size_t)t]);
        out.pool.resize(out.pool.size() + T);
        out.areas[l] = lt_sum_and_scan(a.data(), T, out.pool.data() + out.offsets[l]);
        out.pmf[l] = lt_light_weight(lights[l], sel ? ls_selection_area(out.areas[l], (*sel)[l]) : out.areas[l]);
    }
    if (has_env) {
        out.pmf.push_back(lt_env_weight(bsphere_radius, env_pdf_norm));
        out.cdf.push_back(0);
        L++;
    }
    if (L == 0 || !lt_normalize(out.pmf.data(), out.cdf.data(), L)) {
        err = "rb_scene_create: total light importance is not positive (src/scene.cpp:243)";
        return false;
    }
    return true;
}

inline bool host_pos_less(const float* a, const float* b) { // strict lexicographic order on positions
    if (a[0] != b[0]) return a[0] < b[0];
    if (a[1] != b[1]) return a[1] < b[1];
    return a[2] < b[2];
}
inline bool host_pos_eq(const float* a, const float* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; }

// Host sort of the reference's Thrust (sequential backend, thrust/system/detail/sequential/stable_merge_sort.inl,
// insertion_sort.h, merge.inl): insertion sort for <= 32 elements, otherwise sort both halves recursively and merge,
// taking from the right run whenever comp(right, left).  Identical to std::stable_sort for a strict weak ordering;
// restated because one of the reference's comparators is not strict.
template <typename T, typename Comp>
inline void host_merge_sort_range(std::vector<T>& v, size_t first, size_t last, Comp comp) {
    if (last - first <= 32) {
        for (size_t i = first + 1; i < last; i++) {
            T tmp = v[i];
            if (comp(tmp, v[first])) {
                for (size_t j = i; j > first; j--) v[j] = v[j - 1];
                v[first] = tmp;
            } else {
                size_t j = i, k = i - 1;
                while (comp(tmp, v[k])) {
                    v[j] = v[k];
                    j = k;
                    --k;
                }
                v[j] = tmp;
            }
        }
        return;
    }
    size_t middle = first + (last - first) / 2;
    host_merge_sort_range(v, first, middle, comp);
    host_merge_sort_range(v, middle, last, comp);
    std::vector<T> a(v.begin() + first, v.begin() + middle), b(v.begin() + middle, v.begin() + last);
    size_t i = 0, j = 0, o = first;
    while (i < a.size() && j < b.size()) v[o++] = comp(b[j], a[i]) ? b[j++] : a[i++];
    while (i < a.size()) v[o++] = a[i++];
    while (j < b.size()) v[o++] = b[j++];
}
template <typename T, typename Comp>
inline void host_merge_sort_like_reference(std::vector<T>& v, Comp comp) {
    host_merge_sort_range(v, 0, v.size(), comp);
}

// `shapes` carries device (or emulator-host) pointers; the builders below read only material / light ids and the null-ness of
// `normals` from it, geometry comes from `meshes`.  This is the copy of `shapes` whose geometry pointers are the host mirrors.
inline std::vector<rb_shape> host_shapes(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes) {
    std::vector<rb_shape> hs(shapes);
    for (size_t s = 0; s < hs.size(); s++) {
        hs[s].vertices = meshes[s].vertices.data();
        hs[s].indices = meshes[s].indices.data();
    }
    return hs;
}

// screen-space length of camera silhouettes -> PMF / CDF (src/edge.cpp:186-214, :298-331)
inline void host_primary_edge_distribution(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const DevCamera& cam, HostEdgeTables& out) {
    const std::vector<rb_shape> hs = host_shapes(shapes, meshes);
    int E = (int)out.edges.size();
    out.prim_pmf.assign(E, 0);
    out.prim_cdf.assign(E, 0);
    double total = 0;
    for (int i = 0; i < E; i++) {
        out.prim_pmf[i] = primary_edge_weight(cam, hs.data(), out.edges[i]);
        total += out.prim_pmf[i];
    }
    double run = 0;
    for (int i = 0; i < E; i++) {
        out.prim_pmf[i] = total > 0 ? out.prim_pmf[i] / total : 0.0;
        out.prim_cdf[i] = run;
        run += out.prim_pmf[i];
    }
}
inline void host_build_edges(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const DevCamera& cam, bool want_primary,
                             HostEdgeTables& out) {
    int S = (int)shapes.size();
    const std::vector<rb_shape> hs = host_shapes(shapes, meshes);
    std::vector<Edge> edges;
    for (int s = 0; s < S; s++) {
        const HostMesh& m = meshes[s];
        int T = (int)m.indices.size() / 3;
        std::vector<Edge> he(3 * (size_t)T);
        for (int t = 0; t < T; t++) {
            const int* id = &m.indices[3 * (size_t)t];
            for (int k = 0; k < 3; k++) {
                int a = id[k], b = id[(k + 1) % 3];
                Edge e;
                e.shape_id = s;
                e.v0 = std::min(a, b);
                e.v1 = std::max(a, b);
                e.f0 = t;
                e.f1 = -1;
                he[3 * (size_t)t + k] = e;
            }
        }
        std::stable_sort(he.begin(), he.end(), [](const Edge& x, const Edge& y) { return x.v0 != y.v0 ? x.v0 < y.v0 : x.v1 < y.v1; });
        // merge runs of equal (v0, v1): f0 of the first, f1 = f0 of the last (src/edge.cpp:86-90, :266-273)
        std::vector<Edge> merged;
        for (size_t i = 0; i < he.size();) {
            size_t j = i + 1;
            while (j < he.size() && he[j].v0 == he[i].v0 && he[j].v1 == he[i].v1) j++;
            Edge e = he[i];
            if (j - i >= 2) e.f1 = he[j - 1].f0;
            merged.push_back(e);
            i = j;
        }
        // seam repair: sort by end-point POSITIONS and pair up unmatched duplicates (src/edge.cpp:103-166, :280-288)
        const float* V = m.vertices.data();
        auto key = [&](const Edge& e, const float*& lo, const float*& hi) {
            lo = V + 3 * (size_t)e.v0;
            hi = V + 3 * (size_t)e.v1;
            if (host_pos_less(hi, lo)) std::swap(lo, hi);
        };
        // The reference's comparator answers TRUE for equal keys (src/edge.cpp:93-131), so the order of seam twins -- and
        // with it which copy of a duplicated vertex a sample's gradient lands on -- is whatever its sort algorithm makes
        // of that: restated step by step above (host_merge_sort_like_reference).
        host_merge_sort_like_reference(merged, [&](const Edge& x, const Edge& y) {
            const float *xl, *xh, *yl, *yh;
            key(x, xl, xh);
            key(y, yl, yh);
            if (!host_pos_eq(xl, yl)) return host_pos_less(xl, yl);
            if (!host_pos_eq(xh, yh)) return host_pos_less(xh, yh);
            return true;
        });
        std::vector<int> new_f1(merged.size());
        for (size_t i = 0; i < merged.size(); i++) {
            new_f1[i] = merged[i].f1;
            if (merged[i].f1 != -1) continue;
            const float *l, *h, *cl, *ch;
            key(merged[i], l, h);
            if (i > 0) {
                key(merged[i - 1], cl, ch);
                if (host_pos_eq(l, cl) && host_pos_eq(h, ch)) new_f1[i] = merged[i - 1].f0;
            }
            if (i + 1 < merged.size()) {
                key(merged[i + 1], cl, ch);
                if (host_pos_eq(l, cl) && host_pos_eq(h, ch)) new_f1[i] = merged[i + 1].f0;
            }
        }
        for (size_t i = 0; i < merged.size(); i++) {
            merged[i].f1 = new_f1[i];
            edges.push_back(merged[i]);
        }
    }
    // drop edges between coplanar faces (src/edge.cpp:293-296)
    out.edges.clear();
    for (const Edge& e : edges)
        if (!edge_is_flat(hs.data(), e)) out.edges.push_back(e);
    int E = (int)out.edges.size();
    out.prim_pmf.assign(E, 0);
    out.prim_cdf.assign(E, 0);
    if (want_primary && E > 0) host_primary_edge_distribution(shapes, meshes, cam, out);
}
// ---- secondary-edge hierarchy (host build) ----
// The hierarchical edge sampler's expectation depends on the tree when a scene has few edges (an edge that receives
// more than one of the 16 stochastic descents is still only counted once, src/edge.cpp:1173-1190), so gradient parity
// with the oracle on small scenes needs the SAME tree as EdgeTree::EdgeTree (src/edge_tree.cpp:724-882).  The steps that
// decide it -- leaf records, Morton codes, the Karras split, the node algebra and the treelet pieces, record emission -- are
// those of rb_edge_tree.cuh, which the CUDA builder (rb_edge_tree.cu) runs too.  What is this builder's own is the serial
// orchestration: partition into camera silhouettes / rest (:749-756), billboard size from the mean absolute deviation
// (:763-773), stable sort (:795, :846), the Karras loop, bottom-up bounds in post-order, the treelet pass (post-order, or
// threaded from 8 192 leaves) and the depth-first flattening into the EdgeNode array the kernels traverse.
struct HostEdgeTree {
    std::vector<EdgeNode> nodes;
    int root_cs = RB_EDGE_EMPTY, root_ncs = RB_EDGE_EMPTY;
    float expand = 0.f;
};
struct HostPrefix { // et_prefix of sorted leaves i and j: ids in sorted order, codes by edge id
    const unsigned long long* codes;
    const int* ids;
    RB_HD int operator()(int i, int j) const { return et_prefix(codes[ids[i]], codes[ids[j]], ids[i], ids[j]); }
};
struct HostTreeBuilder {
    std::vector<ETNode> n; // [0, L-1) internal, [L-1, 2L-1) leaves (leaf j at L-1+j)
    ETOps ops{nullptr, 0}; // over n
    int L = 0;
    void treelet_optimize(int root) { // src/edge_tree.cpp:627-684
        if (n[root].edge_id != -1) return;
        int lv[7], inner[5];
        const int cnt = ops.treelet_form(root, lv, inner);
        unsigned char optimal[128];
        double a[128], c_opt[128];
        unsigned num_subsets = (1u << cnt) - 1;
        {
            // a[s] = area(union(leaf 0, leaves of s)): built incrementally, box[s] = box[s without its lowest leaf] + that leaf
            // (min / max are exact and associative, so this equals the reference's from-scratch union, which the CUDA builder keeps)
            ETNode box[128];
            box[0] = n[lv[0]];
            for (unsigned s = 1; s <= num_subsets; s++) {
                int low = __builtin_ctz(s);
                box[s] = box[s & (s - 1u)];
                if (low != 0) ETOps::merge_into(box[s], box[s], n[lv[low]]);
                a[s] = ops.area(box[s]);
            }
        }
        for (int i = 0; i < cnt; i++) c_opt[1u << i] = n[lv[i]].cost;
        for (int k = 2; k <= cnt; k++)
            for (unsigned s = 1; s <= num_subsets; s++)
                if (__builtin_popcount(s) == k) et_best_partition(s, a, c_opt, optimal);
        ops.treelet_rewire(root, lv, inner, optimal, cnt);
    }
    // The reference runs the treelet pass bottom-up in parallel: every thread starts at a leaf and climbs, the SECOND thread to
    // arrive at a node optimises it (src/edge_tree.cpp:685-707).  A node's treelet lies in its own subtree, concurrently
    // processed nodes sit in disjoint subtrees, and a node's result depends on its (finished) subtree only -- so the tree
    // is the same as with the serial post-order, which small scenes keep using.
    void optimize_parallel(int num_threads) {
        const int LB = std::max(L - 1, 1);
        std::vector<std::atomic<int>> arrived(LB);
        for (auto& x : arrived) x.store(0, std::memory_order_relaxed);
        auto worker = [&](int j0, int j1) {
            for (int j = j0; j < j1; j++) {
                int cur = n[LB + j].parent;
                while (cur != -1) {
                    if (arrived[cur].fetch_add(1, std::memory_order_acq_rel) == 0) break; // first arrival: the sibling subtree is not done
                    treelet_optimize(cur);
                    cur = n[cur].parent;
                }
            }
        };
        std::vector<std::thread> pool;
        int per = (L + num_threads - 1) / num_threads;
        for (int t = 0; t < num_threads; t++) {
            int j0 = t * per, j1 = std::min(L, j0 + per);
            if (j0 < j1) pool.emplace_back(worker, j0, j1);
        }
        for (auto& th : pool) th.join();
    }
    template <typename F>
    void postorder(F visit) { // every inner node after both of its child subtrees
        std::vector<std::pair<int, int>> st;
        st.push_back({0, 0});
        while (!st.empty()) {
            auto& top = st.back();
            int i = top.first;
            if (n[i].edge_id != -1) {
                st.pop_back();
                continue;
            }
            if (top.second == 0) {
                top.second = 1;
                st.push_back({n[i].child[0], 0});
            } else if (top.second == 1) {
                top.second = 2;
                st.push_back({n[i].child[1], 0});
            } else {
                st.pop_back();
                visit(i);
            }
        }
    }
    // returns the root index in `n` (or -1)
    int build(const std::vector<ETNode>& leaf_nodes, const std::vector<unsigned long long>& codes, const std::vector<int>& ids, bool six) {
        L = (int)ids.size();
        if (L == 0) return -1;
        int LB = std::max(L - 1, 1); // leaf base
        n.assign(LB + L, et_blank_node());
        ops = ETOps{n.data(), six};
        for (int j = 0; j < L; j++) {
            n[LB + j] = leaf_nodes[ids[j]];
            n[LB + j].cost = ops.area(n[LB + j]);
        }
        if (L == 1) {
            n[0] = n[LB]; // src/edge_tree.cpp:303-308
            return 0;
        }
        for (int i = 0; i < L - 1; i++) {
            int c0, c1;
            et_karras_split(i, L, HostPrefix{codes.data(), ids.data()}, c0, c1);
            n[i].child[0] = c0;
            n[i].child[1] = c1;
            n[c0].parent = i;
            n[c1].parent = i;
        }
        // bottom-up bounds / weighted lengths (costs of internal nodes are set by the optimiser)
        postorder([&](int i) {
            ETOps::merge_into(n[i], n[n[i].child[0]], n[n[i].child[1]]);
            n[i].wlen = n[n[i].child[0]].wlen + n[n[i].child[1]].wlen;
        });
        int threads = 1;
        if (L >= 8192) threads = (int)std::min<unsigned>(16u, std::max(1u, std::thread::hardware_concurrency()));
        if (threads > 1) optimize_parallel(threads);
        else postorder([&](int i) { treelet_optimize(i); }); // the order the reference's atomic-counter walk guarantees (:685-707)
        return 0;
    }
};
inline void host_build_edge_tree(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const std::vector<Edge>& edges,
                                 const DevCamera& cam, HostEdgeTree& out) {
    out.nodes.clear();
    out.root_cs = out.root_ncs = RB_EDGE_EMPTY;
    out.expand = 0.f;
    int E = (int)edges.size();
    if (E == 0) return;
    const std::vector<rb_shape> hs = host_shapes(shapes, meshes);
    double iw = 1.0 / cam.c2w[15];
    const double co[3] = {cam.c2w[3] * iw, cam.c2w[7] * iw, cam.c2w[11] * iw};
    std::vector<ETNode> leaves(E);
    std::vector<int> ids_cs, ids_ncs;
    double mean[3] = {0, 0, 0};
    for (int i = 0; i < E; i++) {
        V3 v0 = edge_v0(hs.data(), edges[i]), v1 = edge_v1(hs.data(), edges[i]);
        for (int k = 0; k < 3; k++) mean[k] += (double)v0[k] + (double)v1[k];
        (et_leaf(hs.data(), edges[i], i, co, leaves[i]) ? ids_cs : ids_ncs).push_back(i);
    }
    for (int k = 0; k < 3; k++) mean[k] /= 2.0 * E;
    double mad[3] = {0, 0, 0};
    for (int i = 0; i < E; i++) {
        V3 v0 = edge_v0(hs.data(), edges[i]), v1 = edge_v1(hs.data(), edges[i]);
        for (int k = 0; k < 3; k++) mad[k] += std::fabs((double)v0[k] - mean[k]) + std::fabs((double)v1[k] - mean[k]);
    }
    for (int k = 0; k < 3; k++) mad[k] /= E;
    out.expand = (float)(0.01 * std::sqrt(mad[0] * mad[0] + mad[1] * mad[1] + mad[2] * mad[2]));
    auto build = [&](std::vector<int>& ids, bool six) -> int {
        if (ids.empty()) return RB_EDGE_EMPTY;
        double lo[6], hi[6];
        for (int k = 0; k < 6; k++) { lo[k] = INFINITY; hi[k] = -INFINITY; }
        for (int id : ids)
            for (int k = 0; k < 3; k++) {
                lo[k] = std::min(lo[k], leaves[id].pmin[k]);
                hi[k] = std::max(hi[k], leaves[id].pmax[k]);
                lo[3 + k] = std::min(lo[3 + k], leaves[id].dmin[k]);
                hi[3 + k] = std::max(hi[3 + k], leaves[id].dmax[k]);
            }
        std::vector<unsigned long long> codes(E, 0);
        for (int id : ids) codes[id] = et_morton(leaves[id], lo, hi, six);
        std::stable_sort(ids.begin(), ids.end(), [&](int a, int b) { return codes[a] < codes[b]; });
        HostTreeBuilder tb;
        int root = tb.build(leaves, codes, ids, six);
        if (tb.n[root].edge_id != -1) return ~tb.n[root].edge_id;
        // flatten the inner nodes (depth-first) into EdgeNode records that carry both children's bounds
        int base = (int)out.nodes.size();
        std::vector<int> number(tb.n.size(), -1);
        std::vector<int> st;
        std::vector<int> order;
        st.push_back(root);
        while (!st.empty()) {
            int i = st.back();
            st.pop_back();
            number[i] = base + (int)order.size();
            order.push_back(i);
            for (int k = 1; k >= 0; k--)
                if (tb.n[tb.n[i].child[k]].edge_id == -1) st.push_back(tb.n[i].child[k]);
        }
        for (int i : order) out.nodes.push_back(et_record(tb.n.data(), i, number.data()));
        return base; // the root is numbered first
    };
    out.root_cs = build(ids_cs, false);
    out.root_ncs = build(ids_ncs, true);
}

inline void host_look_at(const float* pos, const float* look, const float* up, double* m) {
    auto norm = [](double* v) {
        double l = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        if (l > 0) { v[0] /= l; v[1] /= l; v[2] /= l; } else { v[0] = v[1] = v[2] = 0; }
    };
    auto crs = [](const double* a, const double* b, double* c) {
        c[0] = a[1] * b[2] - a[2] * b[1];
        c[1] = a[2] * b[0] - a[0] * b[2];
        c[2] = a[0] * b[1] - a[1] * b[0];
    };
    double d[3] = {(double)look[0] - pos[0], (double)look[1] - pos[1], (double)look[2] - pos[2]};
    norm(d);
    double u[3] = {up[0], up[1], up[2]};
    norm(u);
    double r[3];
    crs(d, u, r);
    norm(r);
    double nu[3];
    crs(r, d, nu);
    norm(nu);
    double o[16] = {r[0], nu[0], d[0], pos[0], r[1], nu[1], d[1], pos[1], r[2], nu[2], d[2], pos[2], 0, 0, 0, 1};
    std::memcpy(m, o, sizeof(o));
}
inline void host_inverse4(const double* m, double* o) {
    double A[4][8];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            A[i][j] = m[4 * i + j];
            A[i][4 + j] = (i == j) ? 1.0 : 0.0;
        }
    for (int c = 0; c < 4; c++) {
        int piv = c;
        for (int r = c + 1; r < 4; r++)
            if (std::fabs(A[r][c]) > std::fabs(A[piv][c])) piv = r;
        for (int k = 0; k < 8; k++) std::swap(A[c][k], A[piv][k]);
        double d = A[c][c];
        for (int k = 0; k < 8; k++) A[c][k] /= d;
        for (int r = 0; r < 4; r++)
            if (r != c) {
                double f = A[r][c];
                for (int k = 0; k < 8; k++) A[r][k] -= f * A[c][k];
            }
    }
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) o[4 * i + j] = A[i][4 + j];
}
// rb_camera (C ABI) -> DevCamera (double copies of the host-read parameters)
inline void host_setup_camera(const rb_camera& c, DevCamera& dc) {
    dc.width = c.width;
    dc.height = c.height;
    dc.use_look_at = c.use_look_at;
    for (int i = 0; i < 3; i++) {
        dc.position[i] = c.position[i];
        dc.look[i] = c.look[i];
        dc.up[i] = c.up[i];
    }
    if (c.use_look_at) {
        host_look_at(c.position, c.look, c.up, dc.c2w);
        host_inverse4(dc.c2w, dc.w2c);
    } else {
        for (int i = 0; i < 16; i++) {
            dc.c2w[i] = c.cam_to_world[i];
            dc.w2c[i] = c.world_to_cam[i];
        }
    }
    for (int i = 0; i < 9; i++) {
        dc.intr_inv[i] = c.intrinsic_mat_inv[i];
        dc.intr[i] = c.intrinsic_mat[i];
    }
    dc.clip_near = c.clip_near;
    dc.type = c.camera_type;
    dc.has_distortion = c.has_distortion;
    for (int i = 0; i < 8; i++) dc.distortion[i] = c.has_distortion ? c.distortion[i] : 0.0;
    dc.vp_beg[0] = c.viewport_beg[0];
    dc.vp_beg[1] = c.viewport_beg[1];
    dc.vp_end[0] = c.viewport_end[0];
    dc.vp_end[1] = c.viewport_end[1];
    dc.lens_radius = c.lens_radius > 0.f ? c.lens_radius : 0.f;
    dc.focus_distance = c.lens_radius > 0.f ? c.focus_distance : 0.f;
}
// compute_num_channels, src/channels.cpp:42-113
inline int host_compute_num_channels(const int* channels, int n, int max_generic) {
    int total = 0;
    for (int i = 0; i < n; i++) {
        switch (channels[i]) {
            case RB_CH_RADIANCE: case RB_CH_POSITION: case RB_CH_GEOMETRY_NORMAL: case RB_CH_SHADING_NORMAL:
            case RB_CH_DIFFUSE_REFLECTANCE: case RB_CH_SPECULAR_REFLECTANCE: case RB_CH_VERTEX_COLOR:
                total += 3;
                break;
            case RB_CH_ALPHA: case RB_CH_DEPTH: case RB_CH_ROUGHNESS: case RB_CH_SHAPE_ID: case RB_CH_TRIANGLE_ID: case RB_CH_MATERIAL_ID:
                total += 1;
                break;
            case RB_CH_UV: case RB_CH_BARYCENTRIC:
                total += 2;
                break;
            case RB_CH_GENERIC_TEXTURE:
                total += max_generic;
                break;
            default:
                return -1;
        }
    }
    return total;
}
