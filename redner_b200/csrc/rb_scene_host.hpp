// Host-side scene preprocessing shared by rb_scene.cu and the debug emulator (tools/cpu_emu):
//   light PMF/CDF + per-light triangle-area CDFs   src/scene.cpp:197-253, compute_area_cdf :38-61 (serial, double)
//   edge list + primary-edge distribution          src/edge.cpp:43-214, :233-331
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

#include "rb_edge.cuh"

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
// Index checks of the descriptor; returns the error message, or null.
inline const char* host_check_scene_desc(const rb_scene_desc& desc) {
    for (int l = 0; l < desc.num_lights; l++)
        if (desc.lights[l].shape_id < 0 || desc.lights[l].shape_id >= desc.num_shapes) return "rb_scene_create: area light refers to an invalid shape";
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

// Radius of the scene's bounding sphere as the reference computes it (src/scene.cpp:156-195) -- including its slip of
// folding each shape's Y extent into the Z bounds; the radius only scales the environment map's selection weight.
inline double host_bsphere_radius(const std::vector<HostMesh>& meshes) {
    if (meshes.empty()) return 0;
    float inf = std::numeric_limits<float>::infinity();
    float lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
    for (const HostMesh& m : meshes) {
        float mn[3] = {inf, inf, inf}, mx[3] = {-inf, -inf, -inf};
        for (size_t v = 0; v + 2 < m.vertices.size(); v += 3)
            for (int a = 0; a < 3; a++) {
                mn[a] = std::min(mn[a], m.vertices[v + a]);
                mx[a] = std::max(mx[a], m.vertices[v + a]);
            }
        lo[0] = std::min(mn[0], lo[0]);
        lo[1] = std::min(mn[1], lo[1]);
        lo[2] = std::min(mn[1], lo[2]);
        hi[0] = std::max(mx[0], hi[0]);
        hi[1] = std::max(mx[1], hi[1]);
        hi[2] = std::max(mx[1], hi[2]);
    }
    float d[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
    return 0.5f * std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
}
// `env_pdf_norm` > 0 appends the environment map as the last light (src/scene.cpp:197-253).
inline bool host_build_lights(const std::vector<DevLight>& lights, const std::vector<HostMesh>& meshes, HostLightTables& out, std::string& err,
                              bool has_env = false, double env_pdf_norm = 0, double bsphere_radius = 0) {
    int L = (int)lights.size();
    out.pmf.assign(L, 0);
    out.cdf.assign(L, 0);
    out.areas.assign(L, 0);
    out.offsets.assign(L, 0);
    out.pool.clear();
    double total = 0;
    for (int l = 0; l < L; l++) {
        const DevLight& light = lights[l];
        const HostMesh& m = meshes[light.shape_id];
        int T = (int)m.indices.size() / 3;
        out.offsets[l] = (int)out.pool.size();
        std::vector<double> a(T);
        double sum_area = 0; // serial sum in triangle order == thrust::reduce on the CPP backend (src/scene.cpp:43-45)
        for (int t = 0; t < T; t++) {
            const int* id = &m.indices[3 * (size_t)t];
            double v[3][3];
            for (int k = 0; k < 3; k++)
                for (int c = 0; c < 3; c++) v[k][c] = m.vertices[3 * (size_t)id[k] + c];
            double e1[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]};
            double e2[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
            double cx = e1[1] * e2[2] - e1[2] * e2[1], cy = e1[2] * e2[0] - e1[0] * e2[2], cz = e1[0] * e2[1] - e1[1] * e2[0];
            a[t] = 0.5 * std::sqrt(cx * cx + cy * cy + cz * cz);
            sum_area += a[t];
        }
        double run = 0;
        for (int t = 0; t < T; t++) { // exclusive scan, then normalise
            out.pool.push_back(run / sum_area);
            run += a[t];
        }
        out.areas[l] = sum_area;
        double lum = 0.212671f * (double)light.intensity[0] + 0.715160f * (double)light.intensity[1] + 0.072169f * (double)light.intensity[2];
        out.pmf[l] = sum_area * lum * double(M_PI);
        total += out.pmf[l];
    }
    if (has_env) {
        double area = 4 * double(M_PI) * bsphere_radius * bsphere_radius;
        out.pmf.push_back(area > 0 ? area / env_pdf_norm : 1.0);
        out.cdf.push_back(0);
        total += out.pmf.back();
        L++;
    }
    if (!(total > 0)) {
        err = "rb_scene_create: total light importance is not positive (src/scene.cpp:243)";
        return false;
    }
    for (int l = 0; l < L; l++) out.pmf[l] /= total;
    out.cdf[0] = 0;
    for (int l = 1; l < L; l++) out.cdf[l] = out.cdf[l - 1] + out.pmf[l - 1];
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


inline void host_primary_edge_distribution(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const DevCamera& cam, HostEdgeTables& out);
// `shapes` carries device (or emulator-host) pointers; only material / light ids and the null-ness of `normals` are
// read from it here, geometry comes from `meshes`.
inline void host_build_edges(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const DevCamera& cam, bool want_primary,
                             HostEdgeTables& out) {
    int S = (int)shapes.size();
    std::vector<rb_shape> hs(shapes);
    for (int s = 0; s < S; s++) {
        hs[s].vertices = meshes[s].vertices.data();
        hs[s].indices = meshes[s].indices.data();
    }
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
// screen-space length of camera silhouettes -> PMF / CDF (src/edge.cpp:186-214, :298-331)
inline void host_primary_edge_distribution(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const DevCamera& cam, HostEdgeTables& out) {
    int S = (int)shapes.size(), E = (int)out.edges.size();
    std::vector<rb_shape> hs(shapes);
    for (int s = 0; s < S; s++) {
        hs[s].vertices = meshes[s].vertices.data();
        hs[s].indices = meshes[s].indices.data();
    }
    out.prim_pmf.assign(E, 0);
    out.prim_cdf.assign(E, 0);
    double iw = 1.0 / cam.c2w[15];
    V3 org = mk3((Real)(cam.c2w[3] * iw), (Real)(cam.c2w[7] * iw), (Real)(cam.c2w[11] * iw));
    double total = 0;
    for (int i = 0; i < E; i++) {
        const Edge& e = out.edges[i];
        V3 v0 = edge_v0(hs.data(), e), v1 = edge_v1(hs.data(), e);
        V2 p0, p1, c0, c1;
        double w = 0;
        if (cam_project(cam, v0, v1, p0, p1) && clip_line_unit(p0, p1, c0, c1) && edge_is_silhouette(hs.data(), org, e)) w = length(c1 - c0);
        out.prim_pmf[i] = w;
        total += w;
    }
    double run = 0;
    for (int i = 0; i < E; i++) {
        out.prim_pmf[i] = total > 0 ? out.prim_pmf[i] / total : 0.0;
        out.prim_cdf[i] = run;
        run += out.prim_pmf[i];
    }
}

// ---- secondary-edge hierarchy (host build) ----
// The hierarchical edge sampler's expectation depends on the tree when a scene has few edges (an edge that receives
// more than one of the 16 stochastic descents is still only counted once, src/edge.cpp:1173-1190), so gradient parity
// with the oracle on small scenes needs the SAME tree.  This is therefore a step-by-step restatement of
// EdgeTree::EdgeTree (src/edge_tree.cpp:724-882) in index form:
//   partition into camera silhouettes / rest (:749-756), 6-D edge bounds with the Hough transform (:23-66),
//   billboard size from the mean absolute deviation (:763-773), Morton codes (:166-266), stable sort (:795, :846),
//   Karras radix tree with the reference's tie break (:282-376), bottom-up bounds and weighted lengths (:391-445)
//   and the treelet (<= 7 leaves) SAH re-optimisation (:464-711) including its quirks.
// The result is flattened into the EdgeNode array the kernels traverse (one record per inner node, both children's bounds).
struct HostEdgeTree {
    std::vector<EdgeNode> nodes;
    int root_cs = RB_EDGE_EMPTY, root_ncs = RB_EDGE_EMPTY;
    float expand = 0.f;
};
struct HNode { // node of the reference-shaped tree (double precision like the reference's Real)
    double pmin[3], pmax[3], dmin[3], dmax[3];
    double wlen;
    int parent;
    int child[2];
    int edge_id;
    double cost;
};
inline int host_clz64(unsigned long long x) { return x == 0 ? 64 : __builtin_clzll(x); }
inline unsigned long long host_expand21(unsigned long long x) {
    x &= 0x1fffffULL;
    x = (x | x << 32) & 0x1f00000000ffffULL;
    x = (x | x << 16) & 0x1f0000ff0000ffULL;
    x = (x | x << 8) & 0x100f00f00f00f00fULL;
    x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
    x = (x | x << 2) & 0x1249249249249249ULL;
    return x;
}
inline unsigned long long host_expand10(unsigned long long x) { // 5 zeros before each bit of a 10-bit integer
    unsigned long long r = 0;
    for (int b = 0; b < 10; b++) r |= ((x >> b) & 1ULL) << (5 * b);
    return r;
}
struct HostTreeBuilder {
    bool six;
    std::vector<HNode> n; // [0, L-1) internal, [L-1, 2L-1) leaves (leaf j at L-1+j)
    int L = 0;
    static void merge_into(HNode& o, const HNode& a, const HNode& b) {
        for (int k = 0; k < 3; k++) {
            o.pmin[k] = std::min(a.pmin[k], b.pmin[k]);
            o.pmax[k] = std::max(a.pmax[k], b.pmax[k]);
            o.dmin[k] = std::min(a.dmin[k], b.dmin[k]);
            o.dmax[k] = std::max(a.dmax[k], b.dmax[k]);
        }
    }
    double area(const HNode& a) const {
        double dx = a.pmax[0] - a.pmin[0], dy = a.pmax[1] - a.pmin[1], dz = a.pmax[2] - a.pmin[2];
        double s = dx * dy + dx * dz + dy * dz;
        if (six) {
            double ex = a.dmax[0] - a.dmin[0], ey = a.dmax[1] - a.dmin[1], ez = a.dmax[2] - a.dmin[2];
            s += ex * ey + ex * ez + ey * ez;
        }
        return 2 * s;
    }
    void refresh(int i) { // bounds, weighted length and SAH cost of an internal node from its children
        HNode &o = n[i];
        const HNode &a = n[o.child[0]], &b = n[o.child[1]];
        merge_into(o, a, b);
        o.wlen = a.wlen + b.wlen;
        o.cost = area(o) + a.cost + b.cost;
    }
    // src/edge_tree.cpp:491-500: NOTE the union always starts from leaf 0, also for subsets that do not contain it
    double subset_area(int cnt, const int* lv, unsigned s) const {
        HNode t = n[lv[0]];
        for (int i = 1; i < cnt; i++)
            if ((s >> i) & 1u) merge_into(t, t, n[lv[i]]);
        return area(t);
    }
    void propagate_cost(int root, const int* lv, int cnt) { // src/edge_tree.cpp:546-579
        for (int i = 0; i < cnt; i++) {
            int cur = lv[i];
            while (cur != root) {
                if (n[cur].cost < 0) {
                    if (n[n[cur].child[0]].cost >= 0 && n[n[cur].child[1]].cost >= 0) refresh(cur); else break;
                }
                cur = n[cur].parent;
            }
        }
        refresh(root);
    }
    void restruct(int parent, int child_index, const int* lv, const int* inner, unsigned char partition, const unsigned char* optimal, int& index,
                  int cnt) { // src/edge_tree.cpp:586-626
        struct Entry { unsigned char partition, child; int parent; } stack[8];
        int sp = 0;
        stack[sp++] = Entry{partition, (unsigned char)child_index, parent};
        while (sp > 0) {
            Entry e = stack[--sp];
            if (__builtin_popcount(e.partition) == 1) {
                int leaf = lv[__builtin_ffs(e.partition) - 1];
                n[e.parent].child[e.child] = leaf;
                n[leaf].parent = e.parent;
            } else {
                int node = inner[index++];
                n[node].cost = -1;
                n[e.parent].child[e.child] = node;
                n[node].parent = e.parent;
                unsigned char lp = optimal[e.partition];
                unsigned char rp = (unsigned char)((~lp) & e.partition);
                stack[sp++] = Entry{lp, 0, node};
                stack[sp++] = Entry{rp, 1, node};
            }
        }
        propagate_cost(parent, lv, cnt);
    }
    void treelet_optimize(int root) { // src/edge_tree.cpp:627-684
        if (n[root].edge_id != -1) return;
        int lv[7], inner[5];
        int cnt = 0, icnt = 0;
        lv[cnt++] = n[root].child[0];
        lv[cnt++] = n[root].child[1];
        int max_idx = 0;
        while (cnt < 7 && max_idx != -1) {
            max_idx = -1;
            double max_area = -1;
            for (int i = 0; i < cnt; i++)
                if (n[lv[i]].edge_id == -1) {
                    double a = area(n[lv[i]]);
                    if (a > max_area) {
                        max_area = a;
                        max_idx = i;
                    }
                }
            if (max_idx != -1) {
                int tmp = lv[max_idx];
                inner[icnt++] = tmp;
                lv[max_idx] = lv[cnt - 1];
                lv[cnt - 1] = n[tmp].child[0];
                lv[cnt] = n[tmp].child[1];
                cnt++;
            }
        }
        // Algorithm 2 of Karras & Aila 2013 (src/edge_tree.cpp:502-544)
        unsigned char optimal[128];
        double a[128], c_opt[128];
        unsigned num_subsets = (1u << cnt) - 1;
        {
            // a[s] = area(union(leaf 0, leaves of s)): built incrementally, box[s] = box[s without its lowest leaf] + that leaf
            // (min / max are exact and associative, so this equals the reference's from-scratch union, subset_area above)
            HNode box[128];
            box[0] = n[lv[0]];
            for (unsigned s = 1; s <= num_subsets; s++) {
                int low = __builtin_ctz(s);
                box[s] = box[s & (s - 1u)];
                if (low != 0) merge_into(box[s], box[s], n[lv[low]]);
                a[s] = area(box[s]);
            }
        }
        for (int i = 0; i < cnt; i++) c_opt[1u << i] = n[lv[i]].cost;
        for (int k = 2; k <= cnt; k++)
            for (unsigned s = 1; s <= num_subsets; s++)
                if (__builtin_popcount(s) == k) {
                    double c_s = INFINITY;
                    unsigned p_s = 0;
                    unsigned d = (s - 1u) & s;
                    unsigned p = (0u - d) & s;
                    do {
                        double c = c_opt[p] + c_opt[s ^ p];
                        if (c < c_s) {
                            c_s = c;
                            p_s = p;
                        }
                        p = (p - d) & s;
                    } while (p != 0);
                    c_opt[s] = a[s] + c_s;
                    optimal[s] = (unsigned char)p_s;
                }
        unsigned char mask = (unsigned char)((1u << cnt) - 1);
        int index = 0;
        unsigned char left = optimal[mask];
        restruct(root, 0, lv, inner, left, optimal, index, cnt);
        unsigned char right = (unsigned char)((~left) & mask);
        restruct(root, 1, lv, inner, right, optimal, index, cnt);
        refresh(root);
    }
    // The reference runs the treelet pass bottom-up in parallel: every thread starts at a leaf and climbs, the SECOND thread to
    // arrive at a node optimises it (src/edge_tree.cpp:685-707).  A node's treelet lies in its own subtree, concurrently
    // processed nodes sit in disjoint subtrees, and a node's result depends on its (finished) subtree only -- so the tree
    // is the same as with the serial post-order below, which small scenes keep using.
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
    void optimize_postorder(int root) {
        // every internal node is optimised after both of its (already optimised) child subtrees, which is the order the
        // reference's atomic-counter walk guarantees (src/edge_tree.cpp:685-707)
        std::vector<std::pair<int, int>> st;
        st.push_back({root, 0});
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
                treelet_optimize(i);
            }
        }
    }
    // returns the root index in `n` (or -1)
    int build(const std::vector<HNode>& leaf_nodes, const std::vector<unsigned long long>& codes, const std::vector<int>& ids) {
        L = (int)ids.size();
        if (L == 0) return -1;
        n.assign(std::max(L - 1, 1) + L, HNode());
        for (auto& x : n) {
            x.parent = -1;
            x.child[0] = x.child[1] = -1;
            x.edge_id = -1;
            x.cost = 0;
            x.wlen = 0;
            for (int k = 0; k < 3; k++) {
                x.pmin[k] = x.dmin[k] = INFINITY;
                x.pmax[k] = x.dmax[k] = -INFINITY;
            }
        }
        int LB = std::max(L - 1, 1); // leaf base
        for (int j = 0; j < L; j++) {
            n[LB + j] = leaf_nodes[ids[j]];
            n[LB + j].parent = -1;
            n[LB + j].cost = area(n[LB + j]);
        }
        if (L == 1) {
            n[0] = n[LB]; // src/edge_tree.cpp:303-308
            return 0;
        }
        auto lcp = [&](int i, int j) -> int {
            if (i < 0 || i >= L || j < 0 || j >= L) return -1;
            unsigned long long a = codes[ids[i]], b = codes[ids[j]];
            if (a == b) return host_clz64(a ^ b) + host_clz64((unsigned long long)ids[i] ^ (unsigned long long)ids[j]);
            return host_clz64(a ^ b);
        };
        for (int i = 0; i < L - 1; i++) {
            int d = (lcp(i, i + 1) - lcp(i, i - 1)) >= 0 ? 1 : -1;
            int dmin = lcp(i, i - d);
            int lmax = 2;
            while (lcp(i, i + lmax * d) > dmin) lmax *= 2;
            int l = 0;
            for (int t = lmax / 2; t >= 1; t /= 2)
                if (lcp(i, i + (l + t) * d) > dmin) l += t;
            int j = i + l * d;
            int dnode = lcp(i, j);
            int s = 0, div = 2;
            for (int t = (l + (div - 1)) / div; t >= 1;) {
                if (lcp(i, i + (s + t) * d) > dnode) s += t;
                if (t == 1) break;
                div *= 2;
                t = (l + (div - 1)) / div;
            }
            int gamma = i + s * d + std::min(d, 0);
            int c0 = (std::min(i, j) == gamma) ? LB + gamma : gamma;
            int c1 = (std::max(i, j) == gamma + 1) ? LB + gamma + 1 : gamma + 1;
            n[i].child[0] = c0;
            n[i].child[1] = c1;
            n[c0].parent = i;
            n[c1].parent = i;
        }
        // bottom-up bounds / weighted lengths (costs of internal nodes are set by the optimiser)
        {
            std::vector<int> order; // post-order over internal nodes
            std::vector<std::pair<int, int>> st;
            st.push_back({0, 0});
            while (!st.empty()) {
                auto& top = st.back();
                int i = top.first;
                if (n[i].edge_id != -1 || i >= LB) { st.pop_back(); continue; }
                if (top.second == 0) { top.second = 1; st.push_back({n[i].child[0], 0}); }
                else if (top.second == 1) { top.second = 2; st.push_back({n[i].child[1], 0}); }
                else { st.pop_back(); order.push_back(i); }
            }
            for (int i : order) {
                merge_into(n[i], n[n[i].child[0]], n[n[i].child[1]]);
                n[i].wlen = n[n[i].child[0]].wlen + n[n[i].child[1]].wlen;
            }
        }
        int threads = 1;
        if (L >= 8192) threads = (int)std::min<unsigned>(16u, std::max(1u, std::thread::hardware_concurrency()));
        if (const char* env = getenv("RB_TREE_THREADS")) threads = std::max(1, atoi(env)); // (test hook)
        if (threads > 1) optimize_parallel(threads);
        else optimize_postorder(0);
        return 0;
    }
};
inline V3 host_edge_normal(const rb_shape* hs, const Edge& e, int which) {
    V3 v0 = edge_v0(hs, e), v1 = edge_v1(hs, e);
    V3 n;
    if (which == 0) {
        V3 o = edge_opposite0(hs, e);
        n = cross(v0 - o, v1 - o);
    } else {
        V3 o = edge_opposite1(hs, e);
        n = cross(v1 - o, v0 - o);
    }
    Real l2 = length_sq(n);
    if (l2 < Real(1e-20)) return zero3();
    return n / std::sqrt(l2);
}
inline void host_build_edge_tree(const std::vector<rb_shape>& shapes, const std::vector<HostMesh>& meshes, const std::vector<Edge>& edges,
                                 const DevCamera& cam, HostEdgeTree& out) {
    out.nodes.clear();
    out.root_cs = out.root_ncs = RB_EDGE_EMPTY;
    out.expand = 0.f;
    int E = (int)edges.size();
    if (E == 0) return;
    std::vector<rb_shape> hs(shapes);
    for (size_t s = 0; s < shapes.size(); s++) {
        hs[s].vertices = meshes[s].vertices.data();
        hs[s].indices = meshes[s].indices.data();
    }
    double iw = 1.0 / cam.c2w[15];
    double co[3] = {cam.c2w[3] * iw, cam.c2w[7] * iw, cam.c2w[11] * iw};
    V3 cam_org = mk3((Real)co[0], (Real)co[1], (Real)co[2]);
    std::vector<HNode> leaves(E);
    std::vector<int> ids_cs, ids_ncs;
    double mean[3] = {0, 0, 0};
    for (int i = 0; i < E; i++) {
        const Edge& e = edges[i];
        V3 v0 = edge_v0(hs.data(), e), v1 = edge_v1(hs.data(), e);
        for (int k = 0; k < 3; k++) mean[k] += (double)v0[k] + (double)v1[k];
        HNode n;
        V3 n0 = host_edge_normal(hs.data(), e, 0);
        V3 n1 = e.f1 == -1 ? -n0 : host_edge_normal(hs.data(), e, 1);
        double p[3], p0d = 0, p1d = 0;
        for (int k = 0; k < 3; k++) p[k] = 0.5 * ((double)v0[k] + (double)v1[k]) - co[k];
        for (int k = 0; k < 3; k++) {
            p0d += p[k] * (double)n0[k];
            p1d += p[k] * (double)n1[k];
        }
        for (int k = 0; k < 3; k++) {
            double h0 = (double)n0[k] * p0d, h1 = (double)n1[k] * p1d;
            n.pmin[k] = std::min((double)v0[k], (double)v1[k]);
            n.pmax[k] = std::max((double)v0[k], (double)v1[k]);
            n.dmin[k] = std::min(h0, h1);
            n.dmax[k] = std::max(h0, h1);
        }
        double ext = M_PI;
        if (e.f1 != -1) ext = std::acos(std::min(1.0, std::max(-1.0, (double)dot(n0, n1))));
        n.wlen = (double)length(v1 - v0) * ext;
        n.parent = -1;
        n.child[0] = n.child[1] = -1;
        n.edge_id = i;
        n.cost = 0;
        leaves[i] = n;
        (edge_is_silhouette(hs.data(), cam_org, e) ? ids_cs : ids_ncs).push_back(i);
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
        for (int id : ids) {
            double q[6];
            for (int k = 0; k < 3; k++) {
                double cp = 0.5 * (leaves[id].pmin[k] + leaves[id].pmax[k]), cd = 0.5 * (leaves[id].dmin[k] + leaves[id].dmax[k]);
                q[k] = hi[k] - lo[k] <= 0 ? 0.5 : (cp - lo[k]) / (hi[k] - lo[k]);
                q[3 + k] = hi[3 + k] - lo[3 + k] <= 0 ? 0.5 : (cd - lo[3 + k]) / (hi[3 + k] - lo[3 + k]);
            }
            if (!six) {
                double sc = (1 << 21) - 1;
                codes[id] = (host_expand21((unsigned long long)(q[0] * sc)) << 2) | (host_expand21((unsigned long long)(q[1] * sc)) << 1) |
                            host_expand21((unsigned long long)(q[2] * sc));
            } else {
                unsigned long long c = 0;
                for (int k = 0; k < 6; k++) c |= host_expand10((unsigned long long)(q[k] * 1023)) << (5 - k);
                codes[id] = c;
            }
        }
        std::stable_sort(ids.begin(), ids.end(), [&](int a, int b) { return codes[a] < codes[b]; });
        HostTreeBuilder tb;
        tb.six = six;
        int root = tb.build(leaves, codes, ids);
        // flatten the inner nodes (depth-first) into EdgeNode records that carry both children's bounds
        auto ref_of = [&](int i, const std::vector<int>& map) { return tb.n[i].edge_id != -1 ? ~tb.n[i].edge_id : map[i]; };
        int base = (int)out.nodes.size();
        std::vector<int> map(tb.n.size(), -1);
        std::vector<int> st;
        std::vector<int> order;
        if (tb.n[root].edge_id == -1) st.push_back(root);
        while (!st.empty()) {
            int i = st.back();
            st.pop_back();
            map[i] = base + (int)order.size();
            order.push_back(i);
            for (int k = 1; k >= 0; k--)
                if (tb.n[tb.n[i].child[k]].edge_id == -1) st.push_back(tb.n[i].child[k]);
        }
        for (int i : order) {
            EdgeNode en;
            memset(&en, 0, sizeof(en));
            for (int c = 0; c < 2; c++) {
                const HNode& h = tb.n[tb.n[i].child[c]];
                for (int k = 0; k < 3; k++) {
                    en.c[c].pmin[k] = (float)h.pmin[k];
                    en.c[c].pmax[k] = (float)h.pmax[k];
                    en.c[c].dmin[k] = (float)h.dmin[k];
                    en.c[c].dmax[k] = (float)h.dmax[k];
                }
                en.c[c].wlen = (float)h.wlen;
                en.c[c].ref = ref_of(tb.n[i].child[c], map);
            }
            out.nodes.push_back(en);
        }
        return ref_of(root, map);
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
