// Secondary-edge hierarchy on the GPU (reference: EdgeTree::EdgeTree, src/edge_tree.cpp:724-882, Thrust-parallel there too).
//
// Builds, per rb_scene_create, the two trees the boundary sampler walks -- a 3-D tree over the camera-silhouette edges and a
// 6-D (position x Hough) tree over the rest.  The steps that decide the trees (leaf records, Morton codes, the Karras split, the
// node algebra, treelet formation / subset search / re-wiring, record emission) are those of rb_edge_tree.cuh, which the host
// builder of rb_scene_host.hpp runs too; tests/test_scene_build_gpu.py compares the two builders' records.  The orchestration is
// this file's own:
//   k_et_leaves     leaf records and camera-silhouette flags, sums for the mean end point (block sums + atomics)
//   k_et_mad        mean absolute deviation of the end points -> billboard size; per-tree bounds of the leaf boxes (ordered-integer
//                   atomic min / max)
//   k_et_codes      Morton codes with the tree bit on top
//   radix sort      stable, by (tree, code); ties keep edge order, which the Karras split resolves by index like the reference
//   k_et_karras     radix tree, one thread per inner node
//   k_et_climb<0>   bottom-up boxes / weighted lengths, atomic arrival counters
//   k_et_optimize   treelet pass, bottom-up, one warp per treelet
//   k_et_climb<2> / k_et_rank / k_et_emit   depth-first numbering of the inner nodes and their records
// The subset areas of a treelet are filled lane-parallel from scratch here and incrementally on the host; the mean absolute deviation
// is summed in a different order (`expand` agrees to ~1e-15 relative).
// This translation unit is compiled with -fmad=false -prec-div=true -prec-sqrt=true (redner_b200/build.py): the float parts (face
// normals) must round like the host builder's, and -Xptxas -dlcm=cg keeps the bottom-up passes' loads out of the (incoherent) L1.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "rb_edge_tree.cuh"
#include "rb_scene.cuh"

struct ETGlobals {
    double sum[3];            // sum of all end points
    double mad[3];            // sum of |end point - mean|
    unsigned long long lo[2][6], hi[2][6]; // per tree: ordered-integer bounds of the leaf boxes (position, Hough)
    int n_cs;                 // camera-silhouette edges
};

__device__ __forceinline__ unsigned long long d2ord(double d) {
    unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b & 0x8000000000000000ULL) ? ~b : (b | 0x8000000000000000ULL);
}
__device__ __forceinline__ double ord2d(unsigned long long o) {
    unsigned long long b = (o & 0x8000000000000000ULL) ? (o & 0x7fffffffffffffffULL) : ~o;
    return __longlong_as_double((long long)b);
}
__global__ void k_et_leaves(const rb_shape* shapes, const Edge* edges, int E, double cx, double cy, double cz, ETNode* leaves, unsigned char* is_cs,
                            ETGlobals* g) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double s[3] = {0, 0, 0};
    int cs = 0;
    if (i < E) {
        const Edge e = edges[i];
        const double co[3] = {cx, cy, cz};
        V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
        for (int k = 0; k < 3; k++) s[k] = (double)v0[k] + (double)v1[k];
        ETNode n;
        cs = et_leaf(shapes, e, i, co, n) ? 1 : 0;
        leaves[i] = n;
        is_cs[i] = (unsigned char)cs;
    }
    // block sums (order of the additions differs from the host's sequential loop: `expand` agrees to ~1e-15 relative)
    __shared__ double sh[3][256];
    __shared__ int shc[256];
    for (int k = 0; k < 3; k++) sh[k][threadIdx.x] = s[k];
    shc[threadIdx.x] = cs;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off) {
            for (int k = 0; k < 3; k++) sh[k][threadIdx.x] += sh[k][threadIdx.x + off];
            shc[threadIdx.x] += shc[threadIdx.x + off];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        for (int k = 0; k < 3; k++) atomicAdd(&g->sum[k], sh[k][0]);
        atomicAdd(&g->n_cs, shc[0]);
    }
}
__global__ void k_et_mad(const rb_shape* shapes, const Edge* edges, int E, const ETNode* leaves, const unsigned char* is_cs, ETGlobals* g) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    double s[3] = {0, 0, 0};
    if (i < E) {
        const Edge e = edges[i];
        V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
        for (int k = 0; k < 3; k++) {
            double mean = g->sum[k] / (2.0 * E);
            s[k] = fabs((double)v0[k] - mean) + fabs((double)v1[k] - mean);
        }
        // bounds of the leaf boxes of this edge's tree
        const ETNode& n = leaves[i];
        int t = is_cs[i] ? 0 : 1;
        for (int k = 0; k < 3; k++) {
            atomicMin(&g->lo[t][k], d2ord(n.pmin[k]));
            atomicMax(&g->hi[t][k], d2ord(n.pmax[k]));
            atomicMin(&g->lo[t][3 + k], d2ord(n.dmin[k]));
            atomicMax(&g->hi[t][3 + k], d2ord(n.dmax[k]));
        }
    }
    __shared__ double sh[3][256];
    for (int k = 0; k < 3; k++) sh[k][threadIdx.x] = s[k];
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if ((int)threadIdx.x < off)
            for (int k = 0; k < 3; k++) sh[k][threadIdx.x] += sh[k][threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0)
        for (int k = 0; k < 3; k++) atomicAdd(&g->mad[k], sh[k][0]);
}
// key = tree bit (0: camera silhouettes, 1: the rest) on top of the Morton code of the leaf centre inside its tree's bounds
__global__ void k_et_codes(int E, const ETNode* leaves, const unsigned char* is_cs, const ETGlobals* g, unsigned long long* keys, int* vals) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E) return;
    int t = is_cs[i] ? 0 : 1;
    double lo[6], hi[6];
    for (int k = 0; k < 6; k++) {
        lo[k] = ord2d(g->lo[t][k]);
        hi[k] = ord2d(g->hi[t][k]);
    }
    unsigned long long c = et_morton(leaves[i], lo, hi, t == 1);
    if (t == 1) c |= 1ULL << 63;
    keys[i] = c;
    vals[i] = i;
}

// Tree t lives in nodes[base .. base + LB + L): inner nodes first (LB = max(L - 1, 1)), then the leaves in sorted order.
struct ETTree {
    int first; // first sorted position of this tree's edges
    int L;     // leaves
    int base;  // first node
    int six;
};
__device__ __forceinline__ int et_lb(const ETTree& t) { return t.L - 1 > 1 ? t.L - 1 : 1; }

__global__ void k_et_init(ETTree t, const ETNode* leaves, const int* ids_sorted, ETNode* nodes) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int LB = et_lb(t);
    if (j < LB) nodes[t.base + j] = et_blank_node();
    if (j < t.L) {
        ETNode x = leaves[ids_sorted[t.first + j]];
        x.cost = ETOps{nodes, t.six}.area(x);
        nodes[t.base + LB + j] = x;
        if (t.L == 1) nodes[t.base] = x; // src/edge_tree.cpp:303-308
    }
}
__global__ void k_et_karras(ETTree t, const unsigned long long* keys, const int* ids, ETNode* nodes) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.L - 1) return;
    keys += t.first;
    ids += t.first;
    const unsigned long long M = 0x7fffffffffffffffULL; // without the tree bit
    int c0, c1;
    et_karras_split(i, t.L, [&](int a, int b) { return et_prefix(keys[a] & M, keys[b] & M, ids[a], ids[b]); }, c0, c1);
    nodes[t.base + i].child[0] = t.base + c0;
    nodes[t.base + i].child[1] = t.base + c1;
    nodes[t.base + c0].parent = t.base + i;
    nodes[t.base + c1].parent = t.base + i;
}

// One WARP optimises one treelet: lane 0 forms it and rewires the tree afterwards; the 127 subset areas and, round by round, the
// optimal partition of every subset of k leaves are spread over the lanes.  Each subset is still evaluated by ONE lane in the
// reference's order, so ties resolve identically.  (A single thread per treelet -- the host builder's shape -- costs ~0.2 ms per
// node here and the pass climbs ~30 levels.)
struct ETScratch { // shared memory, per warp
    double a[128], c_opt[128], bx[7][12];
    unsigned char optimal[128];
    int lv[7], inner[5], cnt;
};
__device__ void treelet_optimize_warp(ETOps ops, int root, ETScratch& w) {
    const int lane = threadIdx.x & 31;
    if (ops.n[root].edge_id != -1) return; // (warp-uniform)
    if (lane == 0) {
        const int cnt = ops.treelet_form(root, w.lv, w.inner);
        w.cnt = cnt;
        for (int i = 0; i < cnt; i++) {
            const ETNode& l = ops.n[w.lv[i]];
            for (int k = 0; k < 3; k++) {
                w.bx[i][k] = l.pmin[k];
                w.bx[i][3 + k] = l.pmax[k];
                w.bx[i][6 + k] = l.dmin[k];
                w.bx[i][9 + k] = l.dmax[k];
            }
            w.c_opt[1u << i] = l.cost;
        }
    }
    __syncwarp();
    const int cnt = w.cnt;
    const unsigned num_subsets = (1u << cnt) - 1;
    // a[s] = area(union(leaf 0, leaves of s)) -- the reference's union always starts from leaf 0 (src/edge_tree.cpp:491-500)
    for (unsigned s = 1 + lane; s <= num_subsets; s += 32) {
        ETNode t;
        for (int k = 0; k < 3; k++) {
            t.pmin[k] = w.bx[0][k];
            t.pmax[k] = w.bx[0][3 + k];
            t.dmin[k] = w.bx[0][6 + k];
            t.dmax[k] = w.bx[0][9 + k];
        }
        for (int i = 1; i < cnt; i++)
            if ((s >> i) & 1u)
                for (int k = 0; k < 3; k++) {
                    t.pmin[k] = et_min(t.pmin[k], w.bx[i][k]);
                    t.pmax[k] = et_max(t.pmax[k], w.bx[i][3 + k]);
                    t.dmin[k] = et_min(t.dmin[k], w.bx[i][6 + k]);
                    t.dmax[k] = et_max(t.dmax[k], w.bx[i][9 + k]);
                }
        w.a[s] = ops.area(t);
    }
    __syncwarp();
    for (int k = 2; k <= cnt; k++) {
        for (unsigned s = 1 + lane; s <= num_subsets; s += 32)
            if (__popc(s) == k) et_best_partition(s, w.a, w.c_opt, w.optimal);
        __syncwarp();
    }
    if (lane == 0) ops.treelet_rewire(root, w.lv, w.inner, w.optimal, cnt);
    __syncwarp();
}
// Bottom-up pass: every thread starts at a leaf and climbs; the SECOND thread to arrive at a node processes it (its two subtrees are
// finished then) -- boxes / weighted lengths (PASS 0) or inner-node counts of the subtrees (PASS 2); pass 1 is k_et_optimize below.
// Concurrently processed nodes sit in disjoint subtrees.
template <int PASS>
__global__ void k_et_climb(ETTree t, ETNode* nodes, int* arrived, int* inner_count) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= t.L || t.L < 2) return;
    int cur = nodes[t.base + et_lb(t) + j].parent;
    while (cur != -1) {
        __threadfence();
        if (atomicAdd(&arrived[cur], 1) == 0) break; // first arrival: the sibling subtree is not done
        __threadfence();
        if (PASS == 0) {
            ETNode o = nodes[cur];
            const ETNode a = nodes[o.child[0]], b = nodes[o.child[1]];
            ETOps::merge_into(o, a, b);
            o.wlen = a.wlen + b.wlen;
            nodes[cur] = o;
        } else {
            int c0 = nodes[cur].child[0], c1 = nodes[cur].child[1];
            inner_count[cur] = 1 + (nodes[c0].edge_id == -1 ? inner_count[c0] : 0) + (nodes[c1].edge_id == -1 ? inner_count[c1] : 0);
        }
        cur = nodes[cur].parent;
    }
}
// The treelet pass (src/edge_tree.cpp:685-707): one warp per leaf climbs; lane 0 owns the arrival counters.
#define RB_ET_WARPS 4
__global__ void __launch_bounds__(32 * RB_ET_WARPS) k_et_optimize(ETTree t, ETNode* nodes, int* arrived) {
    __shared__ ETScratch scratch[RB_ET_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int j = blockIdx.x * RB_ET_WARPS + warp;
    if (j >= t.L || t.L < 2) return;
    ETOps ops{nodes, t.six};
    int cur = nodes[t.base + et_lb(t) + j].parent;
    while (cur != -1) {
        int go = 0;
        if (lane == 0) {
            __threadfence();
            go = atomicAdd(&arrived[cur], 1) != 0;
            __threadfence();
        }
        go = __shfl_sync(0xffffffffu, go, 0);
        if (!go) break; // first arrival: the sibling subtree is not done
        treelet_optimize_warp(ops, cur, scratch[warp]);
        __threadfence();
        cur = nodes[cur].parent;
    }
}
// depth-first (left first) number of every inner node: the number of inner nodes visited before it
__global__ void k_et_rank(ETTree t, const ETNode* nodes, const int* inner_count, int rank_base, int* rank) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.L - 1) return;
    int node = t.base + i, r = 0;
    int cur = node;
    while (nodes[cur].parent != -1) {
        int par = nodes[cur].parent;
        r += 1; // the parent itself
        if (nodes[par].child[1] == cur) {
            int sib = nodes[par].child[0];
            if (nodes[sib].edge_id == -1) r += inner_count[sib];
        }
        cur = par;
    }
    rank[node] = rank_base + r;
}
__global__ void k_et_emit(ETTree t, const ETNode* nodes, const int* rank, EdgeNode* out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.L - 1) return;
    int node = t.base + i;
    out[rank[node]] = et_record(nodes, node, rank);
}

// Builds both trees for the scene's current edge list and camera.  Device temporaries are released in stream order.
int rb_build_edge_trees_gpu(rb_scene* sc, cudaStream_t stream) {
    const int E = sc->dev.num_edges;
    sc->dev.edge_nodes = nullptr;
    sc->num_edge_nodes = 0;
    sc->dev.edge_root_cs = sc->dev.edge_root_ncs = RB_EDGE_EMPTY;
    sc->dev.edge_bounds_expand = 0.f;
    if (E == 0) return 0;
    const double iw = 1.0 / sc->dev.cam.c2w[15];
    const double co[3] = {sc->dev.cam.c2w[3] * iw, sc->dev.cam.c2w[7] * iw, sc->dev.cam.c2w[11] * iw};
    std::vector<void*> temps;
    auto talloc = [&](size_t bytes) -> void* {
        void* p = nullptr;
        if (cudaMallocAsync(&p, std::max<size_t>(bytes, 16), stream) != cudaSuccess) return nullptr;
        temps.push_back(p);
        return p;
    };
    auto release = [&]() {
        for (void* p : temps) cudaFreeAsync(p, stream);
    };
    EdgeNode* out = nullptr; // (kept across rebuilds while the number of edges stays the same)
    if (scene_table(sc, SS_EDGE_NODES, E, stream, &out)) return 1;
    ETNode* leaves = (ETNode*)talloc(sizeof(ETNode) * (size_t)E);
    ETNode* nodes = (ETNode*)talloc(sizeof(ETNode) * (2 * (size_t)E + 2));
    unsigned char* is_cs = (unsigned char*)talloc(E);
    ETGlobals* g = (ETGlobals*)talloc(sizeof(ETGlobals));
    unsigned long long *keys = (unsigned long long*)talloc(8 * (size_t)E), *keys_sorted = (unsigned long long*)talloc(8 * (size_t)E);
    int *vals = (int*)talloc(4 * (size_t)E), *ids = (int*)talloc(4 * (size_t)E);
    int* counters = (int*)talloc(4 * 3 * (2 * (size_t)E + 2)); // arrival flags of the passes, inner counts / ranks
    size_t sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, keys_sorted, vals, ids, E, 0, 64, stream);
    void* sort_tmp = talloc(sort_bytes);
    if (!leaves || !nodes || !is_cs || !g || !keys || !keys_sorted || !vals || !ids || !counters || !sort_tmp) {
        release();
        rb_set_error("rb_scene_create: out of device memory for the edge trees");
        return 1;
    }
    ETGlobals g0;
    memset(&g0, 0, sizeof(g0));
    for (int t = 0; t < 2; t++)
        for (int k = 0; k < 6; k++) {
            g0.lo[t][k] = ~0ULL;
            g0.hi[t][k] = 0ULL;
        }
    RB_CUDA_OK(cudaMemcpyAsync(g, &g0, sizeof(g0), cudaMemcpyHostToDevice, stream));
    const int B = 256, G = (E + B - 1) / B;
    k_et_leaves<<<G, B, 0, stream>>>(sc->dev.shapes, sc->dev.edges, E, co[0], co[1], co[2], leaves, is_cs, g);
    k_et_mad<<<G, B, 0, stream>>>(sc->dev.shapes, sc->dev.edges, E, leaves, is_cs, g);
    k_et_codes<<<G, B, 0, stream>>>(E, leaves, is_cs, g, keys, vals);
    RB_CUDA_OK(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, keys, keys_sorted, vals, ids, E, 0, 64, stream));
    ETGlobals gh;
    RB_CUDA_OK(cudaMemcpyAsync(&gh, g, sizeof(gh), cudaMemcpyDeviceToHost, stream));
    RB_CUDA_OK(cudaStreamSynchronize(stream)); // the tree sizes decide the launches below
    double mad[3];
    for (int k = 0; k < 3; k++) mad[k] = gh.mad[k] / E;
    sc->dev.edge_bounds_expand = (float)(0.01 * std::sqrt(mad[0] * mad[0] + mad[1] * mad[1] + mad[2] * mad[2]));
    ETTree trees[2];
    trees[0] = ETTree{0, gh.n_cs, 0, 0};
    trees[1] = ETTree{gh.n_cs, E - gh.n_cs, gh.n_cs > 0 ? std::max(gh.n_cs - 1, 1) + gh.n_cs : 0, 1};
    const size_t NN = 2 * (size_t)E + 2;
    int *arrived = counters, *inner_count = counters + NN, *rank = counters + 2 * NN;
    int roots[2] = {RB_EDGE_EMPTY, RB_EDGE_EMPTY};
    int rank_base = 0;
    std::vector<int> first_ids(2, -1);
    for (int t = 0; t < 2; t++) {
        const ETTree& tr = trees[t];
        if (tr.L == 0) continue;
        const int GL = (tr.L + B - 1) / B;
        k_et_init<<<GL, B, 0, stream>>>(tr, leaves, ids, nodes);
        if (tr.L >= 2) {
            k_et_karras<<<GL, B, 0, stream>>>(tr, keys_sorted, ids, nodes);
            for (int pass = 0; pass < 3; pass++) {
                RB_CUDA_OK(cudaMemsetAsync(arrived, 0, sizeof(int) * NN, stream));
                if (pass == 0) k_et_climb<0><<<GL, B, 0, stream>>>(tr, nodes, arrived, inner_count);
                else if (pass == 1) k_et_optimize<<<(tr.L + RB_ET_WARPS - 1) / RB_ET_WARPS, 32 * RB_ET_WARPS, 0, stream>>>(tr, nodes, arrived);
                else k_et_climb<2><<<GL, B, 0, stream>>>(tr, nodes, arrived, inner_count);
            }
            k_et_rank<<<GL, B, 0, stream>>>(tr, nodes, inner_count, rank_base, rank);
            k_et_emit<<<GL, B, 0, stream>>>(tr, nodes, rank, out);
            roots[t] = rank_base; // the root is visited first
            rank_base += tr.L - 1;
        } else {
            RB_CUDA_OK(cudaMemcpyAsync(&first_ids[t], ids + tr.first, sizeof(int), cudaMemcpyDeviceToHost, stream));
        }
    }
    RB_CUDA_OK(cudaGetLastError());
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    for (int t = 0; t < 2; t++)
        if (trees[t].L == 1) roots[t] = ~first_ids[t];
    sc->dev.edge_nodes = out;
    sc->dev.edge_root_cs = roots[0];
    sc->dev.edge_root_ncs = roots[1];
    sc->num_edge_nodes = rank_base;
    release();
    return 0;
}

// ------------------------------------------------------------------------------------------------ primary-edge distribution
// Screen-space length of every camera-silhouette edge -> PMF / CDF of the primary-edge sampler (src/edge.cpp:186-214, :298-331),
// on the device: the other camera-dependent table of a scene (rb_scene_set_camera rebuilds it together with the trees).
__global__ void k_prim_weights(DevCamera cam, const rb_shape* shapes, const Edge* edges, int E, double* w) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E) return;
    w[i] = primary_edge_weight(cam, shapes, edges[i]);
}
__global__ void k_prim_normalize(int E, const double* total, double* pmf) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E) return;
    double t = *total;
    pmf[i] = t > 0 ? pmf[i] / t : 0.0;
}
int rb_build_primary_edge_cdf_gpu(rb_scene* sc, cudaStream_t stream) {
    const int E = sc->dev.num_edges;
    if (E == 0 || !sc->dev.use_primary_edge) return 0;
    double *pmf = nullptr, *cdf = nullptr; // (kept across rebuilds while the number of edges stays the same)
    if (scene_table(sc, SS_PRIM_PMF, E, stream, &pmf) || scene_table(sc, SS_PRIM_CDF, E, stream, &cdf)) return 1;
    sc->dev.prim_edge_pmf = pmf;
    sc->dev.prim_edge_cdf = cdf;
    size_t b1 = 0, b2 = 0;
    cub::DeviceReduce::Sum(nullptr, b1, pmf, (double*)nullptr, E, stream);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, pmf, cdf, E, stream);
    void* tmp = nullptr;
    if (cudaMallocAsync(&tmp, std::max(b1, b2) + 256, stream) != cudaSuccess) {
        rb_set_error("rb_scene_create: out of device memory for the primary-edge distribution");
        return 1;
    }
    double* total = (double*)tmp;
    char* work = (char*)tmp + 256;
    const int B = 256, G = (E + B - 1) / B;
    k_prim_weights<<<G, B, 0, stream>>>(sc->dev.cam, sc->dev.shapes, sc->dev.edges, E, pmf);
    RB_CUDA_OK(cub::DeviceReduce::Sum(work, b1, pmf, total, E, stream));
    k_prim_normalize<<<G, B, 0, stream>>>(E, total, pmf);
    RB_CUDA_OK(cub::DeviceScan::ExclusiveSum(work, b2, pmf, cdf, E, stream));
    RB_CUDA_OK(cudaGetLastError());
    RB_CUDA_OK(cudaFreeAsync(tmp, stream));
    return 0;
}
