// Light tables of a scene on the device: the steps of rb_light_build.cuh as kernels.  Replaces the host pass (device->host mirror of
// every light mesh, and of every mesh when there is an environment map, then serial loops), so that neither rb_scene_create nor a
// geometry update of rb_scene_update copies meshes to the host for the lights.  The two give the same doubles
// (tests/test_scene_update_cpu.py for the steps, tests/test_scene_update_gpu.py on the device).
//
//   k_lt_areas    one thread per emissive triangle: its area
//   k_lt_scan     one warp per light: the serial in-order sum and exclusive scan of its triangle areas (one dependent double add
//                 per triangle, as the reference's CPP-backend Thrust does it), with loads, divisions and stores spread over the lanes
//   k_lt_bounds   min / max of X and Y over all vertices of all shapes (environment map only); min and max do not depend on the order
//   k_lt_pmf      one thread: selection weights, environment map last, normalisation and CDF
//
// Compiled like rb_edge_list.cu (no FMA contraction, IEEE division / square root) so that the doubles round like the host build.
#include <algorithm>
#include <vector>

#include "rb_light_build.cuh"
#include "rb_scene.cuh"
#include "rb_scene_host.hpp"

// persistent per scene (slot SS_LIGHT_AUX): the vertex bounds survive updates that do not move vertices
struct LightAux {
    unsigned int bounds[4]; // lo x, lo y, hi x, hi y as order-preserving integers
    int status;             // 1: the total light importance is not positive
    int uv_status;          // 1: a light's scaled texture coordinates are out of the range of emission sampling (RB_LS_MAX_CELLS)
};

__device__ __forceinline__ unsigned int lt_f2ord(float f) {
    unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float lt_ord2f(unsigned int o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

__global__ void k_lt_areas(LTScene S, int n, double* a) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = lt_pool_area(S, i);
}
// One warp per light, the arithmetic of lt_light_scan: the lanes load 32 areas at a time and every lane performs the same in-order
// additions on the shuffled values, so the sum and the prefix sums are lt_sum_and_scan's bit for bit; the loads, the divisions and the
// stores are spread over the lanes (one thread per light, doing all of it, took 16 ms for a 129 k-triangle emissive mesh).
__global__ void k_lt_scan(LTScene S, const double* a, double* pool, double* areas) {
    const int l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (l >= S.L) return; // (uniform per warp)
    const int o = S.offsets[l], T = S.offsets[l + 1] - o;
    double sum = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const double v = t0 + lane < T ? a[o + t0 + lane] : 0.0;
        const int n = min(32, T - t0);
        for (int j = 0; j < n; j++) sum += __shfl_sync(0xffffffffu, v, j);
    }
    double run = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const double v = t0 + lane < T ? a[o + t0 + lane] : 0.0;
        const int n = min(32, T - t0);
        double mine = 0;
        for (int j = 0; j < n; j++) {
            if (lane == j) mine = run;
            run += __shfl_sync(0xffffffffu, v, j);
        }
        if (t0 + lane < T) pool[o + t0 + lane] = mine / sum;
    }
    if (lane == 0) areas[l] = sum;
}
__global__ void k_lt_bounds(const rb_shape* shapes, int num_shapes, LightAux* aux) {
    float lo[2] = {INFINITY, INFINITY}, hi[2] = {-INFINITY, -INFINITY};
    for (int s = blockIdx.y; s < num_shapes; s += gridDim.y) {
        const rb_shape& sh = shapes[s];
        for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < sh.num_vertices; v += gridDim.x * blockDim.x)
            for (int a = 0; a < 2; a++) {
                float c = sh.vertices[3 * (size_t)v + a];
                lo[a] = fminf(lo[a], c);
                hi[a] = fmaxf(hi[a], c);
            }
    }
    for (int a = 0; a < 2; a++)
        for (int off = 16; off > 0; off >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], off));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], off));
        }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 2; a++) {
            atomicMin(&aux->bounds[a], lt_f2ord(lo[a]));
            atomicMax(&aux->bounds[2 + a], lt_f2ord(hi[a]));
        }
}
// ---- emission sampling (the ls_* steps of rb_light_build.cuh), per light that samples by its texture
//   k_ls_cells    one thread per cell: its weight
//   k_ls_rows     one thread per row: prefix sums along it; then k_ls_cols, one thread per column: prefix sums down it
//   k_ls_tris     one thread per triangle: its record (R_t, M_t, a_t, |T_t| / (M_t area_t)); flags coordinates out of range
//   k_ls_scan     one warp: S, the CDF of a_t and the pdf factors, with ls_scan's additions in its order (as k_lt_scan does it)
__global__ void k_ls_cells(rb_texture t, double* d) {
    const int w = t.width[0], h = t.height[0];
    const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (c < (long long)w * h) d[ls_cells(w, h) + c] = ls_cell_weight(t.texels[0], t.channels, w, h, (int)(c % w), (int)(c / w));
}
__global__ void k_ls_rows(int w, int h, double* d) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < h) ls_sat_row(d + ls_cells(w, h), d + ls_sat(w, h), w, j);
}
__global__ void k_ls_cols(int w, int h, double* d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < w) ls_sat_col(d + ls_sat(w, h), w, h, i);
}
__global__ void k_ls_tris(const rb_shape* shapes, int shape_id, rb_texture t, double* d, LightAux* aux) {
    const rb_shape& sh = shapes[shape_id];
    const int k = blockIdx.x * blockDim.x + threadIdx.x, w = t.width[0], h = t.height[0];
    if (k < sh.num_triangles && !ls_tri_record(sh, k, t.uv_scale[0], t.uv_scale[1], w, h, d + ls_sat(w, h), d + ls_tris(w, h) + RB_LS_TRI * (size_t)k))
        aux->uv_status = 1;
}
__global__ void k_ls_scan(int T, int w, int h, double* d) {
    const int lane = threadIdx.x & 31;
    double* recs = d + ls_tris(w, h);
    double sum = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const double v = t0 + lane < T ? recs[RB_LS_TRI * (size_t)(t0 + lane) + 5] : 0.0;
        const int n = min(32, T - t0);
        for (int j = 0; j < n; j++) sum += __shfl_sync(0xffffffffu, v, j);
    }
    double run = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const double v = t0 + lane < T ? recs[RB_LS_TRI * (size_t)(t0 + lane) + 5] : 0.0;
        const int n = min(32, T - t0);
        double mine = 0;
        for (int j = 0; j < n; j++) {
            if (lane == j) mine = run;
            run += __shfl_sync(0xffffffffu, v, j);
        }
        if (t0 + lane < T) {
            double* r = recs + RB_LS_TRI * (size_t)(t0 + lane);
            r[6] = sum > 0 ? mine / sum : 0.0;
            r[7] = sum > 0 ? (v / sum) * r[7] : 0.0;
        }
    }
    if (lane == 0) {
        d[0] = sum;
        d[1] = 0;
    }
}

// sel: the descriptors of the lights' emission sampling (null when no light uses it); a light with S > 0 is selected by S instead of its area
__global__ void k_lt_pmf(const DevLight* lights, int L, const double* areas, const LightSampling* sel, int has_env, int num_shapes, double pdf_norm, LightAux* aux,
                         double* pmf, double* cdf) {
    for (int l = 0; l < L; l++) pmf[l] = lt_light_weight(lights[l], sel && sel[l].data ? ls_selection_area(areas[l], sel[l].data[0]) : areas[l]);
    if (has_env) {
        double radius = 0;
        if (num_shapes > 0) {
            const float lo[2] = {lt_ord2f(aux->bounds[0]), lt_ord2f(aux->bounds[1])}, hi[2] = {lt_ord2f(aux->bounds[2]), lt_ord2f(aux->bounds[3])};
            radius = lt_bsphere_radius(lo, hi);
        }
        pmf[L] = lt_env_weight(radius, pdf_norm);
    }
    aux->status = lt_normalize(pmf, cdf, L + (has_env ? 1 : 0)) ? 0 : 1;
}

// Fills the light tables of sc->dev.  `geometry`: vertices may have moved, so the areas, area CDFs and bounds are rebuilt; otherwise
// only the DevLights and the PMF / CDF (intensities and the environment map's pdf_norm are values of the descriptor).  The status of the
// normalisation is in the LightAux slot; rb_scene.cu reads it after the build.
int rb_build_lights(rb_scene* sc, bool geometry, cudaStream_t stream) {
    const int L = (int)sc->lights.size();
    const bool env = sc->dev.has_envmap != 0;
    sc->dev.num_lights = L + (env ? 1 : 0);
    sc->dev.lights = nullptr;
    if (sc->dev.num_lights == 0) return 0;
    DevLight* d_lights;
    double *d_pmf, *d_cdf, *d_areas, *d_pool;
    int* d_off;
    LightAux* aux;
    unsigned long long* d_table; // the DevLights, then the lights' emission textures (sc->light_table, rb_types.cuh)
    if (scene_table(sc, SS_LIGHTS, sc->light_table.size(), stream, &d_table) || scene_table(sc, SS_LIGHT_PMF, sc->dev.num_lights, stream, &d_pmf) ||
        scene_table(sc, SS_LIGHT_CDF, sc->dev.num_lights, stream, &d_cdf) || scene_table(sc, SS_LIGHT_AUX, 1, stream, &aux))
        return 1;
    d_lights = (DevLight*)d_table;
    RB_CUDA_OK(cudaMemcpyAsync(d_table, sc->light_table.data(), sizeof(unsigned long long) * sc->light_table.size(), cudaMemcpyHostToDevice, stream));
    if (geometry) {
        std::vector<int>& off = sc->light_offsets;
        off.assign(L + 1, 0);
        for (int l = 0; l < L; l++) off[l + 1] = off[l] + sc->shapes[sc->lights[l].shape_id].num_triangles;
        const int P = off[L];
        if (scene_table(sc, SS_LIGHT_AREAS, L, stream, &d_areas) || scene_table(sc, SS_AREA_POOL, P, stream, &d_pool) ||
            scene_table(sc, SS_AREA_OFFSETS, L + 1, stream, &d_off))
            return 1;
        RB_CUDA_OK(cudaMemcpyAsync(d_off, off.data(), sizeof(int) * (L + 1), cudaMemcpyHostToDevice, stream));
        const LTScene S{sc->dev.shapes, d_lights, d_off, L};
        const int B = 256;
        if (L > 0) {
            double* a = nullptr;
            if (P > 0) {
                if (cudaMallocAsync((void**)&a, sizeof(double) * (size_t)P, stream) != cudaSuccess) {
                    rb_set_error("rb_scene_create: out of device memory for the light tables");
                    return 1;
                }
                k_lt_areas<<<(P + B - 1) / B, B, 0, stream>>>(S, P, a);
            }
            k_lt_scan<<<(L + 3) / 4, 128, 0, stream>>>(S, a, d_pool, d_areas);
            if (a) RB_CUDA_OK(cudaFreeAsync(a, stream));
        }
        if (env) {
            LightAux init;
            init.bounds[0] = init.bounds[1] = 0xff800000u; // +inf
            init.bounds[2] = init.bounds[3] = 0x007fffffu; // -inf
            init.status = init.uv_status = 0;
            RB_CUDA_OK(cudaMemcpyAsync(aux, &init, sizeof(init), cudaMemcpyHostToDevice, stream));
            long long V = 0;
            for (const rb_shape& s : sc->shapes) V = std::max<long long>(V, s.num_vertices);
            const int S_ = (int)sc->shapes.size();
            if (S_ > 0 && V > 0) {
                dim3 grid((unsigned)std::min<long long>((V + B - 1) / B, 64), (unsigned)std::min(S_, 1024));
                k_lt_bounds<<<grid, B, 0, stream>>>(sc->dev.shapes, S_, aux);
            }
        }
    } else {
        d_areas = (double*)sc->bufs[SS_LIGHT_AREAS].p;
        d_pool = (double*)sc->bufs[SS_AREA_POOL].p;
        d_off = (int*)sc->bufs[SS_AREA_OFFSETS].p;
    }
    // emission sampling: every table of every light that samples by its texture, on every call (texels change in place between updates)
    LightSampling* d_sel = nullptr;
    std::vector<size_t> off_unused;
    RB_CUDA_OK(cudaMemsetAsync(&aux->uv_status, 0, sizeof(int), stream));
    if (host_any(sc->light_sampling)) {
        std::vector<size_t> off;
        const size_t n = host_light_sampling_layout(sc->light_sampling, sc->light_emission, sc->lights, sc->shapes, off);
        const size_t head = (sizeof(LightSampling) * (size_t)L + sizeof(double) - 1) / sizeof(double); // (descriptors, then the data)
        double* pool;
        if (scene_table(sc, SS_LIGHT_SAMPLING, head + n, stream, &pool)) return 1;
        d_sel = (LightSampling*)pool;
        std::vector<LightSampling> desc(L);
        const int B = 256;
        for (int l = 0; l < L; l++) {
            if (!sc->light_sampling[l]) {
                desc[l] = LightSampling{nullptr, 0, 0};
                continue;
            }
            const rb_texture& t = sc->light_emission[l];
            const int w = t.width[0], h = t.height[0], T = sc->shapes[sc->lights[l].shape_id].num_triangles;
            double* d = pool + head + off[l];
            desc[l] = LightSampling{d, w, h};
            const long long C = (long long)w * h;
            k_ls_cells<<<(unsigned)((C + B - 1) / B), B, 0, stream>>>(t, d);
            k_ls_rows<<<(h + B - 1) / B, B, 0, stream>>>(w, h, d);
            k_ls_cols<<<(w + B - 1) / B, B, 0, stream>>>(w, h, d);
            if (T > 0) k_ls_tris<<<(T + B - 1) / B, B, 0, stream>>>(sc->dev.shapes, sc->lights[l].shape_id, t, d, aux);
            k_ls_scan<<<1, 32, 0, stream>>>(T, w, h, d);
        }
        RB_CUDA_OK(cudaMemcpyAsync(d_sel, desc.data(), sizeof(LightSampling) * (size_t)L, cudaMemcpyHostToDevice, stream));
    }
    sc->light_sampling_bytes = 0;
    if (d_sel) {
        sc->light_sampling_head = ((sizeof(LightSampling) * (size_t)L + sizeof(double) - 1) / sizeof(double)) * sizeof(double);
        sc->light_sampling_bytes = sizeof(double) * host_light_sampling_layout(sc->light_sampling, sc->light_emission, sc->lights, sc->shapes, off_unused);
    }
    // the light table's last word: the descriptors' address (rb_types.cuh)
    const unsigned long long word = (unsigned long long)(uintptr_t)d_sel;
    RB_CUDA_OK(cudaMemcpyAsync(d_table + sc->light_table.size() - 1, &word, sizeof(word), cudaMemcpyHostToDevice, stream));
    k_lt_pmf<<<1, 1, 0, stream>>>(d_lights, L, d_areas, d_sel, env ? 1 : 0, (int)sc->shapes.size(), env ? (double)sc->dev.env.pdf_norm : 0.0, aux, d_pmf, d_cdf);
    RB_CUDA_OK(cudaGetLastError());
    sc->dev.lights = d_lights;
    sc->dev.light_pmf = d_pmf;
    sc->dev.light_cdf = d_cdf;
    sc->dev.light_areas = d_areas;
    sc->dev.area_cdf_pool = d_pool;
    sc->dev.area_cdf_offset = d_off;
    return 0;
}

// 0: the light tables of the last rb_build_lights are valid; 1: their total importance was not positive; 2: a light's texture coordinates
// are out of the range of emission sampling.  Synchronises the stream.
int rb_light_status(const rb_scene* sc, cudaStream_t stream, int* status) {
    *status = 0;
    if (sc->dev.num_lights == 0) return 0;
    int st[2] = {0, 0};
    RB_CUDA_OK(cudaMemcpyAsync(st, (const char*)sc->bufs[SS_LIGHT_AUX].p + offsetof(LightAux, status), 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    *status = st[1] ? 2 : st[0];
    return 0;
}
