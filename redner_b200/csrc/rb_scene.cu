// Scene construction: GPU LBVH over all triangles of all shapes, light distributions, edge list.
// Reference counterpart: Scene::Scene src/scene.cpp:63-307 (Embree/OptiX build :78-155, light CDFs :197-253,
// compute_area_cdf :38-61) and EdgeSampler::EdgeSampler src/edge.cpp:233-383.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "rb_bvh.cuh"
#include "rb_scene.cuh"
#include "rb_scene_host.hpp"

static thread_local std::string g_last_error;
void rb_set_error(const std::string& msg) { g_last_error = msg; }
// The builders name rb_scene_create in their messages; a failure inside another entry point is reported under that entry point's name.
static void retitle_error(const char* fn) {
    static const std::string create = "rb_scene_create:";
    if (g_last_error.compare(0, create.size(), create) == 0) g_last_error = std::string(fn) + ":" + g_last_error.substr(create.size());
}
extern "C" const char* rb_last_error(void) { return g_last_error.c_str(); }
extern "C" const char* rb_version(void) { return "redner_b200 0.1 (sm_90a)"; }

// Scene buffers come from the device's default stream-ordered pool.  Its default release threshold (0) hands the memory
// back to the driver at every synchronisation, so a scene rebuilt each optimiser step would pay a real allocation each
// time: keep up to 256 MiB cached in the pool.
static void keep_pool_warm(int device) {
    static std::mutex m;
    static bool done[64] = {};
    std::lock_guard<std::mutex> lock(m);
    if (done[device & 63]) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        unsigned long long keep = 256ULL << 20;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    done[device & 63] = true;
}
int scene_buffer(rb_scene* sc, SceneSlot slot, size_t bytes, cudaStream_t stream, void** out) {
    SceneBuffer& b = sc->bufs[slot];
    if (b.p == nullptr || b.bytes != bytes) {
        if (b.p) RB_CUDA_OK(cudaFreeAsync(b.p, stream));
        b.p = nullptr;
        b.bytes = 0;
        keep_pool_warm(sc->device);
        RB_CUDA_OK(cudaMallocAsync(&b.p, bytes, stream));
        b.bytes = bytes;
    }
    *out = b.p;
    return 0;
}
template <typename T>
static int dev_upload(rb_scene* sc, SceneSlot slot, T** out, const T* host, size_t count, cudaStream_t stream) {
    if (scene_table(sc, slot, count, stream, out)) return 1;
    if (count > 0) RB_CUDA_OK(cudaMemcpyAsync(*out, host, count * sizeof(T), cudaMemcpyHostToDevice, stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------ BVH build
__device__ __forceinline__ unsigned int f2ord(float f) {
    unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int o) {
    unsigned int b = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    return __uint_as_float(b);
}
__device__ __forceinline__ void global_to_shape(const int* tri_offset, int num_shapes, int g, int& shape, int& tri) {
    int lo = 0, hi = num_shapes; // offsets has num_shapes + 1 entries
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (tri_offset[mid] <= g) lo = mid; else hi = mid;
    }
    shape = lo;
    tri = g - tri_offset[lo];
}

__global__ void k_scene_bounds(const rb_shape* shapes, const int* tri_offset, int num_shapes, int T, unsigned int* bounds) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < T; g += gridDim.x * blockDim.x) {
        int s, t;
        global_to_shape(tri_offset, num_shapes, g, s, t);
        const rb_shape& sh = shapes[s];
        for (int k = 0; k < 3; k++) {
            int vi = sh.indices[3 * (size_t)t + k];
            for (int a = 0; a < 3; a++) {
                float c = sh.vertices[3 * (size_t)vi + a];
                lo[a] = fminf(lo[a], c);
                hi[a] = fmaxf(hi[a], c);
            }
        }
    }
    for (int a = 0; a < 3; a++) {
        for (int off = 16; off > 0; off >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], off));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], off));
        }
    }
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; a++) {
            atomicMin(&bounds[a], f2ord(lo[a]));
            atomicMax(&bounds[3 + a], f2ord(hi[a]));
        }
    }
}
__global__ void k_morton(const rb_shape* shapes, const int* tri_offset, int num_shapes, int T, const unsigned int* bounds,
                         unsigned long long* keys, int* vals) {
    int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T) return;
    int s, t;
    global_to_shape(tri_offset, num_shapes, g, s, t);
    const rb_shape& sh = shapes[s];
    float c[3] = {0, 0, 0};
    for (int k = 0; k < 3; k++) {
        int vi = sh.indices[3 * (size_t)t + k];
        for (int a = 0; a < 3; a++) c[a] += sh.vertices[3 * (size_t)vi + a];
    }
    unsigned int q[3];
    for (int a = 0; a < 3; a++) {
        float lo = ord2f(bounds[a]), hi = ord2f(bounds[3 + a]);
        float ext = fmaxf(hi - lo, 1e-30f);
        float u = (c[a] * (1.0f / 3.0f) - lo) / ext;
        u = fminf(fmaxf(u, 0.f), 1.f);
        q[a] = (unsigned int)fminf(u * 2097152.0f, 2097151.0f);
    }
    keys[g] = (expand21(q[0]) << 2) | (expand21(q[1]) << 1) | expand21(q[2]);
    vals[g] = g;
}
__global__ void k_leaves(const rb_shape* shapes, const int* tri_offset, int num_shapes, int T, const int* sorted_vals,
                         const unsigned int* bounds, BVHTri* tris, float* leaf_box) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    int g = sorted_vals[i];
    int s, t;
    global_to_shape(tri_offset, num_shapes, g, s, t);
    const rb_shape& sh = shapes[s];
    float v[3][3];
    for (int k = 0; k < 3; k++) {
        int vi = sh.indices[3 * (size_t)t + k];
        for (int a = 0; a < 3; a++) v[k][a] = sh.vertices[3 * (size_t)vi + a];
    }
    BVHTri tr;
    tr.v0 = make_float4(v[0][0], v[0][1], v[0][2], __int_as_float(s));
    tr.v1 = make_float4(v[1][0], v[1][1], v[1][2], __int_as_float(t));
    tr.v2 = make_float4(v[2][0], v[2][1], v[2][2], 0.f);
    tris[i] = tr;
    float ext = 0.f;
    for (int a = 0; a < 3; a++) ext = fmaxf(ext, ord2f(bounds[3 + a]) - ord2f(bounds[a]));
    for (int a = 0; a < 3; a++) {
        float lo = fminf(v[0][a], fminf(v[1][a], v[2][a])), hi = fmaxf(v[0][a], fmaxf(v[1][a], v[2][a]));
        float pad = fmaxf(fabsf(lo), fabsf(hi)) * 4e-7f + ext * 1e-7f;
        leaf_box[6 * (size_t)i + a] = lo - pad;
        leaf_box[6 * (size_t)i + 3 + a] = hi + pad;
    }
}
__device__ __forceinline__ int lbvh_delta(const unsigned long long* keys, int T, int i, int j) {
    if (j < 0 || j >= T) return -1;
    unsigned long long a = keys[i], b = keys[j];
    if (a == b) return 64 + __clz(i ^ j);
    return __clzll(a ^ b);
}
// Karras 2012: one thread per internal node.
__global__ void k_karras(const unsigned long long* keys, int T, BVHNode* nodes, int* parent_inner, int* parent_leaf) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T - 1) return;
    int d = (lbvh_delta(keys, T, i, i + 1) - lbvh_delta(keys, T, i, i - 1)) >= 0 ? 1 : -1;
    int dmin = lbvh_delta(keys, T, i, i - d);
    int lmax = 2;
    while (lbvh_delta(keys, T, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (lbvh_delta(keys, T, i, i + (l + t) * d) > dmin) l += t;
    int j = i + l * d;
    int dnode = lbvh_delta(keys, T, i, j);
    int s = 0;
    int t = l;
    do {
        t = (t + 1) >> 1;
        if (lbvh_delta(keys, T, i, i + (s + t) * d) > dnode) s += t;
    } while (t > 1);
    int gamma = i + s * d + min(d, 0);
    int lo = min(i, j), hi = max(i, j);
    int left = (lo == gamma) ? ~gamma : gamma;
    int right = (hi == gamma + 1) ? ~(gamma + 1) : (gamma + 1);
    nodes[i].left = left;
    nodes[i].right = right;
    nodes[i].pad0 = nodes[i].pad1 = 0;
    if (left >= 0) parent_inner[left] = i; else parent_leaf[~left] = i;
    if (right >= 0) parent_inner[right] = i; else parent_leaf[~right] = i;
    if (i == 0) parent_inner[0] = -1;
}
__device__ __forceinline__ void load_box(const float* leaf_box, const float* inner_box, int child, float b[6]) {
    const float* p = child >= 0 ? inner_box + 6 * (size_t)child : leaf_box + 6 * (size_t)(~child);
    for (int k = 0; k < 6; k++) b[k] = p[k];
}
// (`height`: levels below each inner node; the root's bounds the traversal stack, checked by rb_build_bvh)
__global__ void k_refit(int T, BVHNode* nodes, const int* parent_inner, const int* parent_leaf, const float* leaf_box, float* inner_box,
                        int* flags, int* height) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    int node = parent_leaf[i];
    while (node >= 0) {
        __threadfence();
        if (atomicAdd(&flags[node], 1) == 0) return; // first arrival: sibling subtree not finished yet
        __threadfence();
        float l[6], r[6];
        load_box(leaf_box, inner_box, nodes[node].left, l);
        load_box(leaf_box, inner_box, nodes[node].right, r);
        nodes[node].lo_x_hi_x = make_float4(l[0], l[3], r[0], r[3]);
        nodes[node].lo_y_hi_y = make_float4(l[1], l[4], r[1], r[4]);
        nodes[node].lo_z_hi_z = make_float4(l[2], l[5], r[2], r[5]);
        for (int k = 0; k < 3; k++) {
            inner_box[6 * (size_t)node + k] = fminf(l[k], r[k]);
            inner_box[6 * (size_t)node + 3 + k] = fmaxf(l[3 + k], r[3 + k]);
        }
        int hl = nodes[node].left >= 0 ? height[nodes[node].left] : 0, hr = nodes[node].right >= 0 ? height[nodes[node].right] : 0;
        height[node] = (hl > hr ? hl : hr) + 1;
        node = parent_inner[node];
    }
}

int rb_build_bvh(rb_scene* sc, cudaStream_t stream) {
    int num_shapes = (int)sc->shapes.size();
    std::vector<int> offs(num_shapes + 1, 0);
    for (int i = 0; i < num_shapes; i++) offs[i + 1] = offs[i] + sc->shapes[i].num_triangles;
    int T = offs[num_shapes];
    sc->dev.num_tris = T;
    sc->dev.bvh_nodes = nullptr;
    sc->dev.bvh_tris = nullptr;
    sc->dev.bvh_root = 0;
    if (T == 0) return 0;
    std::vector<void*> temps; // builder temporaries (~100 B / triangle) go back to the pool in stream order
    auto talloc = [&](auto** p, size_t count) {
        void* q = nullptr;
        if (cudaMallocAsync(&q, std::max<size_t>(count, 1) * sizeof(**p), stream) != cudaSuccess) return true;
        temps.push_back(q);
        *p = (std::remove_reference_t<decltype(**p)>*)q;
        return false;
    };
    auto release = [&]() {
        for (void* p : temps) cudaFreeAsync(p, stream);
        temps.clear();
    };
    int* d_offs;
    unsigned int* d_bounds;
    unsigned long long *keys, *keys_sorted;
    int *vals, *vals_sorted, *parent_inner, *parent_leaf, *flags, *height;
    float *leaf_box, *inner_box;
    BVHTri* tris;
    BVHNode* nodes;
    if (talloc(&d_offs, offs.size()) || talloc(&d_bounds, 6) || talloc(&keys, T) || talloc(&keys_sorted, T) || talloc(&vals, T) || talloc(&vals_sorted, T) ||
        talloc(&parent_inner, T) || talloc(&parent_leaf, T) || talloc(&flags, T) || talloc(&height, T) || talloc(&leaf_box, 6 * (size_t)T) ||
        talloc(&inner_box, 6 * (size_t)T) || scene_table(sc, SS_BVH_TRIS, T, stream, &tris) || scene_table(sc, SS_BVH_NODES, T, stream, &nodes)) {
        release();
        rb_set_error("rb_scene_create: out of device memory for the triangle BVH");
        return 1;
    }
    RB_CUDA_OK(cudaMemcpyAsync(d_offs, offs.data(), sizeof(int) * offs.size(), cudaMemcpyHostToDevice, stream));
    unsigned int init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
    RB_CUDA_OK(cudaMemcpyAsync(d_bounds, init, sizeof(init), cudaMemcpyHostToDevice, stream));
    int B = 256, G = (T + B - 1) / B;
    k_scene_bounds<<<std::min(G, 1184), B, 0, stream>>>(sc->dev.shapes, d_offs, num_shapes, T, d_bounds);
    k_morton<<<G, B, 0, stream>>>(sc->dev.shapes, d_offs, num_shapes, T, d_bounds, keys, vals);
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys_sorted, vals, vals_sorted, T, 0, 63, stream);
    unsigned char* tmp;
    if (talloc(&tmp, tmp_bytes)) {
        release();
        rb_set_error("rb_scene_create: out of device memory for the triangle BVH");
        return 1;
    }
    RB_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys_sorted, vals, vals_sorted, T, 0, 63, stream));
    k_leaves<<<G, B, 0, stream>>>(sc->dev.shapes, d_offs, num_shapes, T, vals_sorted, d_bounds, tris, leaf_box);
    if (T > 1) {
        RB_CUDA_OK(cudaMemsetAsync(flags, 0, sizeof(int) * T, stream));
        k_karras<<<G, B, 0, stream>>>(keys_sorted, T, nodes, parent_inner, parent_leaf);
        k_refit<<<G, B, 0, stream>>>(T, nodes, parent_inner, parent_leaf, leaf_box, inner_box, flags, height);
        sc->dev.bvh_root = 0;
        // The traversal keeps at most one deferred sibling per level on a RB_BVH_STACK-entry stack.  Morton keys with an index
        // tie-break can make a radix tree deeper than that on heavily clustered / duplicated geometry: refuse instead of
        // silently dropping subtrees.
        int root_height = 0;
        RB_CUDA_OK(cudaMemcpyAsync(&root_height, height, sizeof(int), cudaMemcpyDeviceToHost, stream));
        RB_CUDA_OK(cudaStreamSynchronize(stream));
        if (root_height >= RB_BVH_STACK) {
            release();
            rb_set_error("rb_scene_create: triangle BVH is " + std::to_string(root_height) + " levels deep (limit " + std::to_string(RB_BVH_STACK - 1) +
                         "): degenerate / heavily duplicated geometry");
            return 1;
        }
    } else {
        sc->dev.bvh_root = ~0;
    }
    RB_CUDA_OK(cudaGetLastError());
    sc->dev.bvh_nodes = nodes;
    sc->dev.bvh_tris = tris;
    release();
    return 0;
}

// ------------------------------------------------------------------------------------------------ edges
// The light tables are built on the device (rb_light_build.cu).  The host edge builders of small scenes (rb_scene_host.hpp, shared
// with the debug emulator) work on host mirrors of the meshes; here we only move data.
static int fetch_mesh(const rb_shape& s, HostMesh& m, cudaStream_t stream) {
    m.vertices.resize(3 * (size_t)s.num_vertices);
    m.indices.resize(3 * (size_t)s.num_triangles);
    if (s.num_vertices > 0)
        RB_CUDA_OK(cudaMemcpyAsync(m.vertices.data(), s.vertices, m.vertices.size() * sizeof(float), cudaMemcpyDeviceToHost, stream));
    if (s.num_triangles > 0)
        RB_CUDA_OK(cudaMemcpyAsync(m.indices.data(), s.indices, m.indices.size() * sizeof(int), cudaMemcpyDeviceToHost, stream));
    return 0;
}

static std::vector<HostMesh>& host_meshes() {
    static thread_local std::vector<HostMesh> meshes;
    return meshes;
}

#ifndef RB_GPU_TABLES_MIN_EDGES
#define RB_GPU_TABLES_MIN_EDGES 1024
#endif
#ifndef RB_GPU_EDGE_LIST_MIN_TRIANGLES
#define RB_GPU_EDGE_LIST_MIN_TRIANGLES 1024
#endif
// Host mirror of every mesh of the scene (topology + positions) for the host edge builders; released when it goes out of scope.
struct MeshMirror {
    std::vector<HostMesh>& meshes = host_meshes();
    int fetch(const rb_scene* sc, cudaStream_t stream) {
        meshes.assign(sc->shapes.size(), HostMesh());
        for (size_t s = 0; s < sc->shapes.size(); s++)
            if (fetch_mesh(sc->shapes[s], meshes[s], stream)) return 1;
        if (cudaStreamSynchronize(stream) != cudaSuccess) {
            rb_set_error("rb_scene_create: device-to-host geometry copy failed (are the shape buffers device pointers?)");
            return 1;
        }
        return 0;
    }
    ~MeshMirror() { meshes.clear(); }
};
// The camera-dependent tables of a scene whose edge list was built on the host, built on the host too: the primary-edge distribution
// and the two secondary-edge trees, from the mirrors and the host copy of the list.
static int host_camera_tables(rb_scene* sc, const std::vector<HostMesh>& meshes, cudaStream_t stream) {
    const int E = (int)sc->host_edges.size();
    HostEdgeTables t;
    t.edges = sc->host_edges;
    HostEdgeTree tree;
    if (sc->dev.use_primary_edge) {
        host_primary_edge_distribution(sc->shapes, meshes, sc->dev.cam, t);
        double *d_pmf, *d_cdf;
        if (dev_upload(sc, SS_PRIM_PMF, &d_pmf, t.prim_pmf.data(), E, stream) || dev_upload(sc, SS_PRIM_CDF, &d_cdf, t.prim_cdf.data(), E, stream)) return 1;
        sc->dev.prim_edge_pmf = d_pmf;
        sc->dev.prim_edge_cdf = d_cdf;
    }
    if (sc->dev.use_secondary_edge) {
        host_build_edge_tree(sc->shapes, meshes, t.edges, sc->dev.cam, tree);
        EdgeNode* d_nodes;
        sc->num_edge_nodes = (int)tree.nodes.size();
        if (tree.nodes.empty()) tree.nodes.push_back(EdgeNode()); // (single-edge trees have no inner node)
        if (dev_upload(sc, SS_EDGE_NODES, &d_nodes, tree.nodes.data(), tree.nodes.size(), stream)) return 1;
        sc->dev.edge_nodes = d_nodes;
        sc->dev.edge_root_cs = tree.root_cs;
        sc->dev.edge_root_ncs = tree.root_ncs;
        sc->dev.edge_bounds_expand = tree.expand;
    }
    RB_CUDA_OK(cudaStreamSynchronize(stream)); // (the host vectors go out of scope)
    return 0;
}

int rb_build_edges(rb_scene* sc, cudaStream_t stream) {
    sc->camera_tables_as_built = true;
    sc->host_tables = false;
    sc->host_edges.clear();
    sc->dev.edges = nullptr;
    sc->dev.num_edges = 0;
    sc->dev.prim_edge_pmf = sc->dev.prim_edge_cdf = nullptr;
    sc->dev.edge_nodes = nullptr;
    sc->num_edge_nodes = 0;
    sc->dev.edge_root_cs = sc->dev.edge_root_ncs = RB_EDGE_EMPTY;
    sc->dev.edge_bounds_expand = 0.f;
    if (!sc->dev.use_primary_edge && !sc->dev.use_secondary_edge) return 0;
    long long num_triangles = 0;
    for (const rb_shape& s : sc->shapes) num_triangles += s.num_triangles;
    sc->edge_list_on_device = getenv("RB_HOST_TREES") == nullptr && getenv("RB_HOST_EDGE_LIST") == nullptr &&
                              (num_triangles >= RB_GPU_EDGE_LIST_MIN_TRIANGLES || getenv("RB_GPU_TREES") != nullptr || getenv("RB_GPU_EDGE_LIST") != nullptr);
    // Small scenes (a few hundred edges: C1, C2) build the edge list and the tables that depend on the camera -- the primary-edge
    // distribution and the two secondary-edge trees -- on the host: faster than ~35 kernel launches and four synchronisations.  From
    // RB_GPU_EDGE_LIST_MIN_TRIANGLES triangles on everything is built on the device (rb_edge_list.cu, rb_edge_tree.cu); in between
    // (host list of >= RB_GPU_TABLES_MIN_EDGES edges, or RB_HOST_EDGE_LIST=1) the list comes from the host and the tables from the
    // device.  A camera update of rb_scene_update rebuilds the tables on the side chosen here; rb_scene_set_camera / rb_render_batch
    // always rebuild them on the device.  The builders produce the same list and
    // the same tables (tests/test_scene_build_gpu.py); RB_GPU_TREES=1 / RB_HOST_TREES=1 force everything onto one side.
    if (sc->edge_list_on_device) {
        // Larger scenes: the list too is built on the device (rb_edge_list.cu), and no mesh leaves the GPU for it.
        if (rb_build_edge_list_gpu(sc, stream)) return 1;
        if (sc->dev.num_edges == 0) return 0;
        if (sc->dev.use_primary_edge && rb_build_primary_edge_cdf_gpu(sc, stream)) return 1;
        if (sc->dev.use_secondary_edge && rb_build_edge_trees_gpu(sc, stream)) return 1;
        RB_CUDA_OK(cudaStreamSynchronize(stream));
        return 0;
    }
    MeshMirror mirror;
    if (mirror.fetch(sc, stream)) return 1;
    const std::vector<HostMesh>& meshes = mirror.meshes;
    HostEdgeTables t;
    host_build_edges(sc->shapes, meshes, sc->dev.cam, false, t);
    int E = (int)t.edges.size();
    sc->host_tables = getenv("RB_HOST_TREES") != nullptr || (E < RB_GPU_TABLES_MIN_EDGES && getenv("RB_GPU_TREES") == nullptr);
    sc->dev.num_edges = E;
    if (E == 0) return 0;
    Edge* d_edges;
    if (dev_upload(sc, SS_EDGES, &d_edges, t.edges.data(), E, stream)) return 1;
    sc->dev.edges = d_edges;
    if (sc->host_tables) {
        sc->host_edges = t.edges;
        if (host_camera_tables(sc, meshes, stream)) return 1;
    } else {
        if (sc->dev.use_primary_edge && rb_build_primary_edge_cdf_gpu(sc, stream)) return 1;
        if (sc->dev.use_secondary_edge && rb_build_edge_trees_gpu(sc, stream)) return 1;
    }
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------ tables (per device, uploaded once)
struct DeviceTables {
    unsigned long long* sobol = nullptr;
    float* ltc = nullptr;
    int sobol_dims = 0;
};
static std::mutex g_tab_mutex;
static DeviceTables g_tables[64];
static int get_tables(int device, DeviceTables& out) {
    std::lock_guard<std::mutex> lock(g_tab_mutex);
    DeviceTables& t = g_tables[device & 63];
    if (t.sobol == nullptr) {
        size_t sb = rb_sobol_table_end - rb_sobol_table_begin;
        size_t lb = rb_ltc_table_end - rb_ltc_table_begin;
        RB_CUDA_OK(cudaMalloc(&t.sobol, sb));
        RB_CUDA_OK(cudaMemcpy(t.sobol, rb_sobol_table_begin, sb, cudaMemcpyHostToDevice));
        RB_CUDA_OK(cudaMalloc(&t.ltc, lb));
        RB_CUDA_OK(cudaMemcpy(t.ltc, rb_ltc_table_begin, lb, cudaMemcpyHostToDevice));
        t.sobol_dims = (int)(sb / (52 * sizeof(unsigned long long)));
    }
    out = t;
    return 0;
}

// ------------------------------------------------------------------------------------------------ build / update steps
// Checks of a descriptor that do not depend on a previous build; returns the error message, or null.
static const char* check_desc(const rb_scene_desc& desc) {
    if (!desc.use_gpu) return "rb_scene_create: use_gpu == 0 requested, but redner_b200 has no CPU path (CUDA sm_90a only)";
    if (desc.envmap != nullptr && desc.use_secondary_edge_sampling)
        return "rb_scene_create: secondary edge sampling with an environment map is not implemented yet (interior terms and primary edges are)";
    if (desc.envmap != nullptr && (desc.envmap->values.num_levels <= 0 || desc.envmap->values.width[0] <= 0 || desc.envmap->sample_cdf_ys == nullptr ||
                                   desc.envmap->sample_cdf_xs == nullptr))
        return "rb_scene_create: the environment map needs an image texture ([h, w, 3] mip pyramid) and its two sampling tables";
    if (desc.camera.camera_type < RB_CAMERA_PERSPECTIVE || desc.camera.camera_type > RB_CAMERA_PANORAMA) return "rb_scene_create: unknown camera type";
    return host_check_scene_desc(desc);
}

// The tables that depend on the camera: primary-edge distribution and secondary-edge trees.  `like_build`: on the side rb_build_edges
// chose for them (so that they are the tables a new scene would have); else on the device.
static int camera_step(rb_scene* sc, const rb_camera& cam, bool like_build, cudaStream_t stream) {
    sc->cam = cam;
    host_setup_camera(cam, sc->dev.cam);
    sc->camera_tables_as_built = like_build || !sc->host_tables;
    if (sc->dev.num_edges > 0 && like_build && sc->host_tables) {
        MeshMirror mirror;
        return mirror.fetch(sc, stream) || host_camera_tables(sc, mirror.meshes, stream);
    }
    if (sc->dev.num_edges > 0) {
        if (sc->dev.use_primary_edge && rb_build_primary_edge_cdf_gpu(sc, stream)) return 1;
        if (sc->dev.use_secondary_edge && rb_build_edge_trees_gpu(sc, stream)) return 1;
    }
    return 0;
}

// The steps of rb_scene_update; rb_scene_create_on_stream runs them with everything marked changed.  `geometry`: vertices may have moved
// (BVH, light areas and bounds, edge list and camera tables are rebuilt); else `camera`: the camera differs (camera tables only).  The
// descriptors, the DevLights and the light PMF / CDF are always refreshed.  Runs on `stream`, which becomes the scene's stream.
// A failure part-way leaves tables of the old and the new descriptor side by side: the scene is marked incomplete, rb_render refuses it
// and the next rb_scene_update rebuilds everything.
static int scene_apply(rb_scene* sc, const rb_scene_desc& desc, bool geometry, bool camera, cudaStream_t stream) {
    sc->incomplete = true;
    sc->stream = stream;
    sc->shapes.assign(desc.shapes, desc.shapes + desc.num_shapes);
    sc->materials.assign(desc.materials, desc.materials + desc.num_materials);
    sc->lights = host_area_lights(desc);
    host_setup_envmap(desc.envmap, sc->dev);
    rb_shape* d_shapes;
    rb_material* d_materials;
    if (dev_upload(sc, SS_SHAPES, &d_shapes, sc->shapes.data(), sc->shapes.size(), stream) ||
        dev_upload(sc, SS_MATERIALS, &d_materials, sc->materials.data(), sc->materials.size(), stream))
        return 1;
    sc->dev.shapes = d_shapes;
    sc->dev.num_shapes = (int)sc->shapes.size();
    sc->dev.materials = d_materials;
    sc->dev.num_materials = (int)sc->materials.size();
    auto t0 = std::chrono::high_resolution_clock::now();
    if (geometry && rb_build_bvh(sc, stream)) return 1;
    auto t1 = std::chrono::high_resolution_clock::now();
    if (rb_build_lights(sc, geometry, stream)) return 1;
    int light_status = 0;
    if (rb_light_status(sc, stream, &light_status)) return 1; // (synchronises: the light kernels are timed here)
    if (light_status != 0) {
        rb_set_error("rb_scene_create: total light importance is not positive (src/scene.cpp:243)");
        return 1;
    }
    auto t2 = std::chrono::high_resolution_clock::now();
    if (geometry) {
        sc->cam = desc.camera;
        host_setup_camera(desc.camera, sc->dev.cam);
        if (rb_build_edges(sc, stream)) return 1;
    } else if (camera && camera_step(sc, desc.camera, true, stream)) {
        return 1;
    }
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    auto t3 = std::chrono::high_resolution_clock::now();
    sc->build_ms_bvh = std::chrono::duration<float, std::milli>(t1 - t0).count();
    sc->build_ms_lights = std::chrono::duration<float, std::milli>(t2 - t1).count();
    sc->build_ms_edges = std::chrono::duration<float, std::milli>(t3 - t2).count();
    if (cudaStreamSynchronize(stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
        rb_set_error("rb_scene_create: scene build kernels failed");
        return 1;
    }
    sc->incomplete = false;
    return 0;
}

// ------------------------------------------------------------------------------------------------ C ABI
extern "C" int rb_scene_create(const rb_scene_desc* desc, rb_scene** out) { return rb_scene_create_on_stream(desc, out, nullptr); }
// Uploads, the device->host mesh mirror and the build kernels run on `stream_` (the stream the caller's geometry tensors were produced
// on: work queued there is ordered before the build; with the legacy default stream a non-blocking side stream would not be).
extern "C" int rb_scene_create_on_stream(const rb_scene_desc* desc, rb_scene** out, void* stream_) {
    if (!desc || !out) {
        rb_set_error("rb_scene_create: null argument");
        return 1;
    }
    *out = nullptr;
    if (const char* err = check_desc(*desc)) {
        rb_set_error(err);
        return 1;
    }
    int count = 0;
    RB_CUDA_OK(cudaGetDeviceCount(&count));
    if (count <= 0) {
        rb_set_error("rb_scene_create: no CUDA device visible; redner_b200 has no CPU fallback");
        return 1;
    }
    int prev = 0;
    RB_CUDA_OK(cudaGetDevice(&prev));
    int device = desc->gpu_index >= 0 ? desc->gpu_index : prev;
    RB_CUDA_OK(cudaSetDevice(device));
    rb_scene* sc = new rb_scene();
    sc->device = device;
    sc->gpu_index = desc->gpu_index;
    memset(&sc->dev, 0, sizeof(DevScene));
    sc->max_generic_texture_dimension = host_max_generic_texture_dimension(*desc);
    sc->dev.use_primary_edge = desc->use_primary_edge_sampling;
    sc->dev.use_secondary_edge = desc->use_secondary_edge_sampling;
    sc->dev.edge_root_cs = sc->dev.edge_root_ncs = RB_EDGE_EMPTY;
    DeviceTables tabs;
    if (get_tables(device, tabs) || scene_apply(sc, *desc, true, true, (cudaStream_t)stream_)) {
        rb_scene_destroy(sc);
        cudaSetDevice(prev);
        return 1;
    }
    sc->dev.sobol_matrices = tabs.sobol;
    sc->dev.sobol_dims = tabs.sobol_dims;
    sc->dev.ltc_table = tabs.ltc;
    cudaSetDevice(prev);
    *out = sc;
    return 0;
}

// Re-target the scene at a descriptor of the same structure (see the header).  Nothing changes before the structure checks pass.
extern "C" int rb_scene_update(rb_scene* sc, const rb_scene_desc* desc, int geometry_changed, void* stream_) {
    if (!sc || !desc) {
        rb_set_error("rb_scene_update: null argument");
        return 1;
    }
    const char* err = check_desc(*desc);
    if (!err) err = host_check_same_structure(*desc, sc->shapes, (int)sc->materials.size(), sc->lights, sc->dev, sc->gpu_index, sc->max_generic_texture_dimension);
    if (err) {
        rb_set_error(err);
        retitle_error("rb_scene_update");
        return 1;
    }
    // (after a failed build or update every table is rebuilt; after rb_scene_set_camera on a scene whose camera tables the build made on
    // the host, they are made on the host again)
    bool geometry = geometry_changed != 0 || sc->incomplete;
    for (int s = 0; s < desc->num_shapes; s++) geometry = geometry || desc->shapes[s].vertices != sc->shapes[s].vertices;
    const bool camera = memcmp(&desc->camera, &sc->cam, sizeof(rb_camera)) != 0 || !sc->camera_tables_as_built;
    int prev = 0;
    cudaGetDevice(&prev);
    if (cudaSetDevice(sc->device) != cudaSuccess) {
        rb_set_error("rb_scene_update: cudaSetDevice failed");
        return 1;
    }
    int rc = scene_apply(sc, *desc, geometry, camera, (cudaStream_t)stream_);
    cudaSetDevice(prev);
    if (rc != 0) retitle_error("rb_scene_update");
    return rc;
}

extern "C" void rb_scene_destroy(rb_scene* sc) {
    if (!sc) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(sc->device);
    for (SceneBuffer& b : sc->bufs)
        if (b.p) cudaFreeAsync(b.p, sc->stream);
    sc->events.destroy();
    cudaSetDevice(prev);
    delete sc;
}

// Test hook: the secondary-edge trees as the kernels see them ({records, root of the camera-silhouette tree, root of the other tree},
// the billboard size, and optionally the records themselves).
extern "C" int rb_scene_edge_trees(const rb_scene* sc, int* info3, float* expand, void* records_out, size_t records_bytes) {
    if (!sc) return 1;
    if (info3) {
        info3[0] = sc->num_edge_nodes;
        info3[1] = sc->dev.edge_root_cs;
        info3[2] = sc->dev.edge_root_ncs;
    }
    if (expand) *expand = sc->dev.edge_bounds_expand;
    if (records_out && sc->dev.edge_nodes && records_bytes > 0) {
        size_t n = std::min(records_bytes, sizeof(EdgeNode) * (size_t)sc->num_edge_nodes);
        if (cudaMemcpy(records_out, sc->dev.edge_nodes, n, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    }
    return 0;
}

// Test hook: the edge list as the kernels see it (5 ints per edge: shape, v0, v1, f0, f1).
extern "C" int rb_scene_edge_list(const rb_scene* sc, int* num_edges, int* edges_out, size_t edges_bytes) {
    if (!sc) return 1;
    if (num_edges) *num_edges = sc->dev.num_edges;
    if (edges_out && sc->dev.edges && edges_bytes > 0) {
        size_t n = std::min(edges_bytes, sizeof(Edge) * (size_t)sc->dev.num_edges);
        if (cudaMemcpy(edges_out, sc->dev.edges, n, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    }
    return 0;
}

// Test hook: one table of the scene as the kernels see it.
extern "C" int rb_scene_table(const rb_scene* sc, int which, void* out, size_t bytes, size_t* size) {
    if (!sc) return 1;
    const DevScene& d = sc->dev;
    const int L = (int)sc->lights.size();
    const bool prim = d.use_primary_edge && d.num_edges > 0;
    const void* src = nullptr;
    size_t n = 0;
    switch (which) {
        case RB_TABLE_BVH_NODES: src = d.bvh_nodes; n = sizeof(BVHNode) * (size_t)std::max(d.num_tris - 1, 0); break;
        case RB_TABLE_BVH_TRIANGLES: src = d.bvh_tris; n = sizeof(BVHTri) * (size_t)d.num_tris; break;
        case RB_TABLE_LIGHT_PMF: src = d.light_pmf; n = sizeof(double) * (size_t)d.num_lights; break;
        case RB_TABLE_LIGHT_CDF: src = d.light_cdf; n = sizeof(double) * (size_t)d.num_lights; break;
        case RB_TABLE_LIGHT_AREAS: src = d.light_areas; n = sizeof(double) * (size_t)L; break;
        case RB_TABLE_AREA_CDF_POOL: src = d.area_cdf_pool; n = sizeof(double) * (size_t)(sc->light_offsets.empty() ? 0 : sc->light_offsets.back()); break;
        case RB_TABLE_AREA_CDF_OFFSETS: src = d.area_cdf_offset; n = sizeof(int) * (size_t)L; break;
        case RB_TABLE_PRIMARY_EDGE_PMF: src = d.prim_edge_pmf; n = prim ? sizeof(double) * (size_t)d.num_edges : 0; break;
        case RB_TABLE_PRIMARY_EDGE_CDF: src = d.prim_edge_cdf; n = prim ? sizeof(double) * (size_t)d.num_edges : 0; break;
        default: rb_set_error("rb_scene_table: unknown table"); return 1;
    }
    if (src == nullptr || (d.num_lights == 0 && which >= RB_TABLE_LIGHT_PMF && which <= RB_TABLE_AREA_CDF_OFFSETS)) n = 0;
    if (size) *size = n;
    if (out && bytes > 0 && n > 0) {
        int prev = 0;
        cudaGetDevice(&prev);
        cudaSetDevice(sc->device);
        cudaError_t e = cudaMemcpy(out, src, std::min(bytes, n), cudaMemcpyDeviceToHost);
        cudaSetDevice(prev);
        if (e != cudaSuccess) {
            rb_set_error(std::string("rb_scene_table: ") + cudaGetErrorString(e));
            return 1;
        }
    }
    return 0;
}

// Test hook: one ray query per thread, through the traversal the render kernels call or by brute force over every triangle.
template <bool ANY_HIT, bool BRUTE>
__global__ void k_trace_rays(const float4* nodes4, const float4* tris4, int root, int num_tris, const float* rays, int num_rays, int* ids, float* t) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_rays) return;
    const float* r = rays + 8 * (size_t)i;
    BvhHit h = BRUTE ? bvh_brute_force<ANY_HIT>(tris4, num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7])
                     : bvh_trace_impl<ANY_HIT>(nodes4, tris4, root, num_tris, r[0], r[1], r[2], r[4], r[5], r[6], r[3], r[7]);
    ids[2 * (size_t)i] = h.shape_id;
    ids[2 * (size_t)i + 1] = h.tri_id;
    t[i] = h.t;
}
// (memory of the scene's own device: the kernel runs there, and another GPU's memory would be read without peer access)
static bool on_device(const void* p, int device) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}
extern "C" int rb_scene_trace_rays(const rb_scene* sc, const float* rays, int num_rays, int flags, int* ids, float* t) {
    if (!sc) {
        rb_set_error("rb_scene_trace_rays: null scene");
        return 1;
    }
    if (num_rays < 0) {
        rb_set_error("rb_scene_trace_rays: negative number of rays");
        return 1;
    }
    if (sc->incomplete) {
        rb_set_error("rb_scene_trace_rays: the scene's last update failed; update it again or build a new scene");
        return 1;
    }
    if (num_rays == 0) return 0;
    int prev = 0;
    cudaGetDevice(&prev);
    if (cudaSetDevice(sc->device) != cudaSuccess) {
        rb_set_error("rb_scene_trace_rays: cudaSetDevice failed");
        return 1;
    }
    if (!on_device(rays, sc->device) || !on_device(ids, sc->device) || !on_device(t, sc->device)) {
        cudaSetDevice(prev);
        rb_set_error("rb_scene_trace_rays: rays, ids and t must be memory of the scene's device");
        return 1;
    }
    // (synchronises the device before and after: the rays may come from any stream)
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) {
        const float4* nodes4 = reinterpret_cast<const float4*>(sc->dev.bvh_nodes);
        const float4* tris4 = reinterpret_cast<const float4*>(sc->dev.bvh_tris);
        const int B = 128, G = (num_rays + B - 1) / B, root = sc->dev.bvh_root, T = sc->dev.num_tris;
        switch (flags & (RB_TRACE_ANY_HIT | RB_TRACE_BRUTE_FORCE)) {
            case 0: k_trace_rays<false, false><<<G, B>>>(nodes4, tris4, root, T, rays, num_rays, ids, t); break;
            case RB_TRACE_ANY_HIT: k_trace_rays<true, false><<<G, B>>>(nodes4, tris4, root, T, rays, num_rays, ids, t); break;
            case RB_TRACE_BRUTE_FORCE: k_trace_rays<false, true><<<G, B>>>(nodes4, tris4, root, T, rays, num_rays, ids, t); break;
            default: k_trace_rays<true, true><<<G, B>>>(nodes4, tris4, root, T, rays, num_rays, ids, t); break;
        }
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_scene_trace_rays: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}

// Re-target the scene at another camera: only the camera-dependent tables are rebuilt (on the device).
extern "C" int rb_scene_set_camera(rb_scene* sc, const rb_camera* cam) {
    if (!sc || !cam) {
        rb_set_error("rb_scene_set_camera: null argument");
        return 1;
    }
    if (cam->width <= 0 || cam->height <= 0 || cam->viewport_end[0] <= cam->viewport_beg[0] || cam->viewport_end[1] <= cam->viewport_beg[1]) {
        rb_set_error("rb_scene_set_camera: empty image / viewport");
        return 1;
    }
    if (sc->incomplete) {
        rb_set_error("rb_scene_set_camera: the scene's last update failed; update it again or build a new scene");
        return 1;
    }
    int prev = 0;
    cudaGetDevice(&prev);
    if (cudaSetDevice(sc->device) != cudaSuccess) {
        rb_set_error("rb_scene_set_camera: cudaSetDevice failed");
        return 1;
    }
    cudaStream_t stream = sc->stream;
    int rc = camera_step(sc, *cam, false, stream);
    if (rc == 0 && cudaStreamSynchronize(stream) != cudaSuccess) {
        rb_set_error("rb_scene_set_camera: device failure");
        rc = 1;
    }
    if (rc != 0) {
        sc->incomplete = true;
        retitle_error("rb_scene_set_camera");
    }
    cudaSetDevice(prev);
    return rc;
}

extern "C" int rb_scene_max_generic_texture_dimension(const rb_scene* sc) { return sc ? sc->max_generic_texture_dimension : 0; }

extern "C" int rb_scene_set_partition(rb_scene* sc, int part, int num_parts, int rows_per_stripe) {
    if (!sc || num_parts < 1 || part < 0 || part >= num_parts || rows_per_stripe < 1) {
        rb_set_error("rb_scene_set_partition: invalid arguments");
        return 1;
    }
    sc->part = part;
    sc->num_parts = num_parts;
    sc->rows_per_stripe = rows_per_stripe;
    return 0;
}

extern "C" int rb_scene_last_stats(const rb_scene* sc, int* launches, float* ms) {
    if (!sc) return 1;
    if (launches) *launches = sc->last_launches;
    if (ms) *ms = sc->last_kernel_ms;
    return 0;
}

extern "C" int rb_scene_last_stage_stats(const rb_scene* sc, float* stage_ms4, double* path_vertices, double* primary_hits) {
    if (!sc) return 1;
    if (stage_ms4)
        for (int i = 0; i < 4; i++) stage_ms4[i] = sc->last_stage_ms[i];
    if (path_vertices) *path_vertices = sc->last_path_vertices;
    if (primary_hits) *primary_hits = sc->last_primary_hits;
    return 0;
}
extern "C" int rb_scene_last_backward_stats(const rb_scene* sc, float* bwd_ms3) {
    if (!sc || !bwd_ms3) return 1;
    for (int i = 0; i < 3; i++) bwd_ms3[i] = sc->last_bwd_ms[i];
    return 0;
}
extern "C" int rb_scene_last_exact_bytes(const rb_scene* sc, size_t* bytes) {
    if (!sc || !bytes) return 1;
    *bytes = sc->last_exact_bytes;
    return 0;
}
extern "C" int rb_scene_build_ms(const rb_scene* sc, float* bvh_lights_edges3) {
    if (!sc || !bvh_lights_edges3) return 1;
    bvh_lights_edges3[0] = sc->build_ms_bvh;
    bvh_lights_edges3[1] = sc->build_ms_lights;
    bvh_lights_edges3[2] = sc->build_ms_edges;
    return 0;
}

// compute_num_channels, src/channels.cpp:42-113
extern "C" int rb_compute_num_channels(const int* channels, int n, int max_generic) { return host_compute_num_channels(channels, n, max_generic); }
