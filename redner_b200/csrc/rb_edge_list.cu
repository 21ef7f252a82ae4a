// Edge list of a scene on the device: the steps of rb_edge_list.cuh as kernels between CUB sorts and scans.  Replaces the host pass
// (device->host mirror of every mesh, std::stable_sort, a serial merge sort and three serial loops: 5.6 ms for the 15.7 k-triangle
// teapot scene) for scenes above RB_GPU_EDGE_LIST_MIN_TRIANGLES; the two produce the same list, element for element
// (tests/test_edge_list_cpu.py for the steps, tests/test_scene_build_gpu.py on the device).
// Reference: Thrust sort / reduce / remove_if per shape in src/edge.cpp:233-296.
//
// Compiled like rb_edge_tree.cu (no FMA contraction, IEEE division / square root): edge_is_flat compares a dot product of two unit
// normals with 1 - 1e-6 and must round like the host build of the same function.
#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

#include "rb_edge_list.cuh"
#include "rb_scene.cuh"

__global__ void k_el_keys(ELScene L, int n, unsigned long long* keys, int* half_edges) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = el_half_edge_key(L, i);
    half_edges[i] = i;
}
__global__ void k_el_heads(int n, const unsigned long long* keys, int* is_head) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    is_head[i] = el_is_run_head(keys, i) ? 1 : 0;
}
__global__ void k_el_merge(ELScene L, int n, const unsigned long long* keys, const int* half_edges, const int* head_rank, Edge* merged) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !el_is_run_head(keys, i)) return;
    merged[head_rank[i] - 1] = el_merge_run(L, keys, half_edges, n, i);
}
__global__ void k_el_reverse(int M, int* order) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < M) order[p] = M - 1 - p;
}
__global__ void k_el_pair(const rb_shape* shapes, const Edge* merged, const int* order, int M, Edge* paired, int* keep) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= M) return;
    Edge e = el_pair_seam(shapes, merged, order, M, p);
    paired[p] = e;
    keep[p] = edge_is_flat(shapes, e) ? 0 : 1;
}
__global__ void k_el_compact(int M, const Edge* paired, const int* keep, const int* keep_rank, Edge* edges) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < M && keep[p]) edges[keep_rank[p] - 1] = paired[p];
}

// Fills sc->dev.edges / num_edges from the device meshes.  Two small device->host reads (the number of distinct edges, the number that
// survive the filter) size the buffers; temporaries are released in stream order.
int rb_build_edge_list_gpu(rb_scene* sc, cudaStream_t stream) {
    const int S = (int)sc->shapes.size();
    sc->dev.edges = nullptr;
    sc->dev.num_edges = 0;
    std::vector<int> offsets(2 * ((size_t)S + 1), 0); // [0, S]: triangles, [S + 1, 2 S + 1]: vertices
    long long T = 0, V = 0;
    for (int s = 0; s < S; s++) {
        T += sc->shapes[s].num_triangles;
        V += sc->shapes[s].num_vertices;
        if (3 * T > 0x7fffffffLL || V > 0x7fffffffLL) {
            rb_set_error("rb_scene_create: too many triangles for the edge list (3 * triangles must fit a 32-bit integer)");
            return 1;
        }
        offsets[s + 1] = (int)T;
        offsets[(size_t)S + 1 + s + 1] = (int)V;
    }
    if (T == 0) return 0;
    const int n = (int)(3 * T);
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
    auto fail = [&](const char* what) {
        release();
        rb_set_error(std::string("rb_scene_create: ") + what);
        return 1;
    };
    ELScene L;
    L.shapes = sc->dev.shapes;
    L.S = S;
    L.key_bits = el_bits_for(V);
    int* d_offsets = (int*)talloc(sizeof(int) * offsets.size());
    unsigned long long *keys = (unsigned long long*)talloc(8 * (size_t)n), *keys_sorted = (unsigned long long*)talloc(8 * (size_t)n);
    int *half_edges = (int*)talloc(4 * (size_t)n), *half_sorted = (int*)talloc(4 * (size_t)n);
    int *flags = (int*)talloc(4 * (size_t)n), *ranks = (int*)talloc(4 * (size_t)n);
    size_t b_sort = 0, b_scan = 0, b_merge = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b_sort, keys, keys_sorted, half_edges, half_sorted, n, 0, 2 * L.key_bits, stream);
    cub::DeviceScan::InclusiveSum(nullptr, b_scan, flags, ranks, n, stream);
    cub::DeviceMergeSort::StableSortKeys(nullptr, b_merge, half_edges, n, ELPositionLess{nullptr, nullptr}, stream); // (n bounds the merged count)
    const size_t work_bytes = std::max(b_sort, std::max(b_scan, b_merge));
    void* work = talloc(work_bytes);
    if (!d_offsets || !keys || !keys_sorted || !half_edges || !half_sorted || !flags || !ranks || !work) return fail("out of device memory for the edge list");
    L.tri_off = d_offsets;
    L.vert_off = d_offsets + S + 1;
    RB_CUDA_OK(cudaMemcpyAsync(d_offsets, offsets.data(), sizeof(int) * offsets.size(), cudaMemcpyHostToDevice, stream));
    const int B = 256, G = (n + B - 1) / B;
    size_t bytes = work_bytes;
    // A: keys of the half-edges, grouped by a stable sort
    k_el_keys<<<G, B, 0, stream>>>(L, n, keys, half_edges);
    RB_CUDA_OK(cub::DeviceRadixSort::SortPairs(work, bytes, keys, keys_sorted, half_edges, half_sorted, n, 0, 2 * L.key_bits, stream));
    // B: one edge per run of equal keys
    k_el_heads<<<G, B, 0, stream>>>(n, keys_sorted, flags);
    bytes = work_bytes;
    RB_CUDA_OK(cub::DeviceScan::InclusiveSum(work, bytes, flags, ranks, n, stream));
    int M = 0;
    RB_CUDA_OK(cudaMemcpyAsync(&M, ranks + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, stream));
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    if (M <= 0 || M > n) return fail("edge list: inconsistent run count");
    Edge *merged = (Edge*)talloc(sizeof(Edge) * (size_t)M), *paired = (Edge*)talloc(sizeof(Edge) * (size_t)M);
    int* order = half_edges; // (the unsorted half-edge ids are no longer needed; M <= n)
    if (!merged || !paired) return fail("out of device memory for the edge list");
    k_el_merge<<<G, B, 0, stream>>>(L, n, keys_sorted, half_sorted, ranks, merged);
    // C: position order with ties in reverse input order
    const int GM = (M + B - 1) / B;
    k_el_reverse<<<GM, B, 0, stream>>>(M, order);
    bytes = work_bytes;
    RB_CUDA_OK(cub::DeviceMergeSort::StableSortKeys(work, bytes, order, M, ELPositionLess{sc->dev.shapes, merged}, stream));
    // D + E: seam twins, then drop the flat edges
    k_el_pair<<<GM, B, 0, stream>>>(sc->dev.shapes, merged, order, M, paired, flags);
    bytes = work_bytes;
    RB_CUDA_OK(cub::DeviceScan::InclusiveSum(work, bytes, flags, ranks, M, stream));
    int E = 0;
    RB_CUDA_OK(cudaMemcpyAsync(&E, ranks + (M - 1), sizeof(int), cudaMemcpyDeviceToHost, stream));
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    if (E < 0 || E > M) return fail("edge list: inconsistent edge count");
    if (E > 0) {
        Edge* edges = nullptr;
        if (scene_table(sc, SS_EDGES, E, stream, &edges)) {
            release();
            return 1;
        }
        k_el_compact<<<GM, B, 0, stream>>>(M, paired, flags, ranks, edges);
        sc->dev.edges = edges;
    }
    sc->dev.num_edges = E;
    RB_CUDA_OK(cudaGetLastError());
    release();
    return 0;
}
