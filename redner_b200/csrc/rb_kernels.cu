// Render kernels and the rb_render driver (reference: render(), src/pathtracer.cpp:177-958).
//
// Execution model (DESIGN.md section 2).  The reference runs a host-driven wavefront: ~20 launches and 2 host syncs per
// bounce per sample, with every per-path field (5.5 - 9.4 KB/pixel in double) streamed through managed memory between
// stage functors.  Here a path lives in registers inside a kernel and only a 128-byte record per path vertex crosses kernels:
//   forward    k_forward / k_forward_channels   camera sample -> primary hit -> emission -> bounce loop -> pixel
//   backward   per band of samples:  k_bwd_trace (primal replay, records, work lists by warp ballot) -> k_bwd_sec_pick ->
//              counting sort by edge (k_sec_offsets, k_sec_scatter) -> k_bwd_sec_shade (boundary terms) -> k_bwd_sweep (reverse
//              sweep, first-hit and camera adjoints);  then k_prim_keys -> radix sort -> k_primary_edge;  k_finish_camera
// Every kernel is small enough for the GPC instruction cache and walks the stages of a sample block-synchronously
// (RB_PHASE_SYNC): a fused megakernel of the same code ran instruction-fetch bound at 6 % issue utilisation.
// Forward: a warp owns 32/L pixels with L lanes per pixel (L = min(32, 2^floor(log2 spp))); lanes of a pixel are its
// samples, so rays of a warp are coherent in the BVH, the pixel is reduced with shuffles and written by one lane
// without atomics (deterministic image).  Gradient atomics are aggregated per warp before they reach L2.
// The per-sample logic itself lives in rb_render.cuh.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "rb_kernel_set.h"
#include "rb_render.cuh"
#include "rb_scene.cuh"

#include "rb_kernels_body.cuh"

// ------------------------------------------------------------------------------------------------ driver
// Backward scratch (gradient descriptors, band records and work lists): ONE grow-only allocation per device, kept for
// the life of the process so that a training loop pays no cudaMalloc / pool growth per step (measured: ~20 ms per step
// with per-call cudaMallocAsync of the 1 GiB band).  rb_render holds the lock for the whole backward pass, which also
// serialises concurrent backward passes on one device; rb_release_scratch() frees everything.
#include <mutex>
struct DeviceScratch {
    std::mutex mutex; // one backward pass per DEVICE at a time; passes on different devices of one process run concurrently
    char* ptr = nullptr;
    size_t bytes = 0;
};
static DeviceScratch g_scratch[64];
static char* scratch_ensure(DeviceScratch& sc, size_t bytes) { // (caller holds sc.mutex and has made the device current)
    if (sc.bytes >= bytes) return sc.ptr;
    if (sc.ptr) {
        cudaDeviceSynchronize();
        cudaFree(sc.ptr);
        sc.ptr = nullptr;
        sc.bytes = 0;
    }
    if (cudaMalloc((void**)&sc.ptr, bytes) != cudaSuccess) {
        sc.ptr = nullptr;
        return nullptr;
    }
    sc.bytes = bytes;
    return sc.ptr;
}
extern "C" void rb_release_scratch(void) {
    int prev = 0;
    cudaGetDevice(&prev);
    for (int d = 0; d < 64; d++) {
        std::lock_guard<std::mutex> lock(g_scratch[d].mutex);
        if (g_scratch[d].ptr) {
            cudaSetDevice(d);
            cudaDeviceSynchronize();
            cudaFree(g_scratch[d].ptr);
            g_scratch[d].ptr = nullptr;
            g_scratch[d].bytes = 0;
        }
    }
    cudaSetDevice(prev);
}
// Restores the caller's current device on EVERY exit path of rb_render (RB_CUDA_OK returns).
struct RenderGuard {
    int prev_device = -1;
    ~RenderGuard() {
        if (prev_device >= 0) cudaSetDevice(prev_device);
    }
};
// Persistent grid of a kernel: SMs x resident blocks per SM for its block size and dynamic shared memory.
static int pick_grid(const void* kernel, int device, int block = RB_BLOCK, size_t smem = 0) {
    int sms = 132, per_sm = 1;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem);
    if (per_sm < 1) per_sm = 1;
    return sms * per_sm;
}

// CUDA events of one rb_render on the render stream, for the stage timings of rb_scene_last_stage_stats and
// rb_scene_last_backward_stats: the fixed ones first, then BAND_EVENTS per backward band.  The events belong to the scene and are
// reused by every call (creating ~40 events per call cost more than the kernels of a small render).
enum { EV_BEGIN, EV_AFTER_FORWARD, EV_AFTER_BANDS, EV_AFTER_PRIMARY_EDGE, EV_END, NUM_FIXED_EVENTS };
enum { BAND_BEGIN, BAND_AFTER_TRACE, BAND_BEFORE_SWEEP, BAND_END, BAND_EVENTS };

extern "C" int rb_render(const rb_scene* scene_, const rb_options* opt, float* image, const float* d_image, const rb_dscene_desc* d_scene,
                         float* screen_grad, void* stream_) {
    rb_scene* scene = const_cast<rb_scene*>(scene_);
    if (!scene || !opt) {
        rb_set_error("rb_render: null scene / options");
        return 1;
    }
    if (scene->incomplete) {
        rb_set_error("rb_render: the scene's last update failed; update it again or build a new scene");
        return 1;
    }
    KernelArgs ka;
    if (const char* err = setup_kernel_args(*opt, scene->cam, scene->max_generic_texture_dimension, scene->part, scene->num_parts, scene->rows_per_stripe,
                                            image, d_image, d_scene, screen_grad, ka)) {
        rb_set_error(err);
        return 1;
    }
    const RenderParams& rp = ka.rp;
    if (rp.vp_w <= 0 || rp.vp_h <= 0 || rp.spp == 0) return 0;
    // The feature-free instantiation of the kernels (rb_kernels_lean.cu) serves the common configuration; `kern` holds the kernels of
    // the chosen instantiation, and every launch of one of them below goes through it.
    const bool lean_allowed = getenv("RB_NO_LEAN") == nullptr; // (test hook: force the general kernels)
    const bool lean = lean_allowed && rp.only_radiance && !scene->dev.has_envmap && scene->dev.cam.type == RB_CAMERA_PERSPECTIVE && !scene->dev.cam.has_distortion;
    const RenderKernels kern = lean ? rb_lean::render_kernels() : render_kernels();

    RenderGuard guard;
    int prev = 0;
    RB_CUDA_OK(cudaGetDevice(&prev));
    RB_CUDA_OK(cudaSetDevice(scene->device));
    guard.prev_device = prev;
    cudaStream_t stream = (cudaStream_t)stream_;
    EventPool& events = scene->events;
    if (!events.ensure(NUM_FIXED_EVENTS)) {
        rb_set_error("rb_render: cudaEventCreate failed");
        return 1;
    }
    std::vector<cudaEvent_t>& ev = events.ev;
    int launches = 0;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, scene->device);
    std::vector<BandCounters> host_counters;
    long long num_bands_done = 0;
    std::unique_lock<std::mutex> scratch_lock; // per-device scratch, held for the backward pass (released before the guard runs)
    void* args[] = {&scene->dev, &ka}; // parameters of every kernel in `kern` but the primary-edge pair (read at each launch)
    RB_CUDA_OK(cudaEventRecord(ev[EV_BEGIN], stream));
    if (image != nullptr) {
        if (rp.only_radiance) {
            int grid = pick_grid(kern.forward, scene->device, RB_BLOCK_FWD);
            RB_CUDA_OK(cudaLaunchKernel(kern.forward, grid, RB_BLOCK_FWD, args, 0, stream));
        } else {
            int grid = pick_grid((const void*)k_forward_channels, scene->device);
            k_forward_channels<<<grid, RB_BLOCK, 0, stream>>>(scene->dev, ka);
        }
        launches++;
    }
    RB_CUDA_OK(cudaEventRecord(ev[EV_AFTER_FORWARD], stream));
    if (d_image == nullptr) {
        for (int i = EV_AFTER_BANDS; i <= EV_END; i++) RB_CUDA_OK(cudaEventRecord(ev[i], stream));
    }
    if (d_image != nullptr) {
        if (const char* err = setup_backward(*d_scene, scene->dev, ka)) {
            rb_set_error(err);
            return 1;
        }
        const bool secondary = boundary_stage_runs(scene->dev, rp);
        const long long total_samples = (long long)ka.owned_rows * rp.vp_w * rp.spp;
        ka.rec_per_sample = rp.max_bounces + 1;
        const size_t per_sample = (size_t)ka.rec_per_sample * (sizeof(VertexRec) + (secondary ? sizeof(V3) + sizeof(EdgePick) + 16 : 0)) + 2 * sizeof(int) +
                                  sizeof(ListCount) + (secondary ? sizeof(ulonglong2) : 0);
        size_t band_bytes = RB_BAND_BYTES;
        if (const char* env = getenv("RB_BAND_BYTES")) { // test hook: force many small bands
            long long v = atoll(env);
            if (v > 0) band_bytes = (size_t)v;
        }
        long long band = (long long)std::max<size_t>(band_bytes / per_sample, 1024);
        band = std::min<long long>(band, (1LL << 30) / ka.rec_per_sample);
        band = std::min<long long>(band, std::max<long long>(total_samples, 1));
        const long long num_bands = (total_samples + band - 1) / band;
        if (!events.ensure((size_t)(NUM_FIXED_EVENTS + BAND_EVENTS * num_bands))) {
            rb_set_error("rb_render: cudaEventCreate failed");
            return 1;
        }
        auto count_it = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), ListCountOf{nullptr, nullptr});
        size_t scan_bytes = 0;
        cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, count_it, (ListCount*)nullptr, ListCountSum(), ListCount{0, 0, 0, 0}, (int)band, stream);
        // boundary terms: vertex list, edge picks, (edge, vertex) per slot, slots in edge order
        const size_t vert_cap = (size_t)band * ka.rec_per_sample, slots = vert_cap + 32;
        ka.vert_cap = (int)vert_cap;
        const bool primary = primary_edge_pass_runs(scene->dev);
        const long long n_px_all = (long long)rp.vp_w * rp.vp_h;
        const long long total_e = primary ? ((n_px_all - rp.part + rp.num_parts - 1) / rp.num_parts) * rp.spp : 0; // i % num_parts == part
        const long long band_e = std::min<long long>(std::max<long long>(total_e, 1), 1LL << 26);
        size_t sort_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned*)nullptr, (unsigned*)nullptr, (int)band_e, 0, 32, stream);

        // ---- scratch layout, in carving order, every buffer 256-byte aligned: gradient descriptors | camera accumulators | band counters |
        //      edge histogram, offsets and cursors | band (records, boundary terms, work lists).  The primary-edge pass runs after the
        //      bands and reuses the band area for its keys / values (double buffers) and radix-sort temporaries.  The buffers of the
        //      boundary stage are empty when it does not run.  carve(nullptr) only measures; both calls return the size.
        rb_dshape* d_shapes;
        rb_material* d_mats;
        float** d_lights;
        double* cam_accum;
        BandCounters* counters;
        ListCount* list_offs;
        void *scan_tmp, *sort_tmp;
        unsigned *k0, *k1, *v0, *v1;
        size_t zeroed_bytes = 0;
        auto carve = [&](char* base) {
            size_t off = 0;
            auto take = [&](size_t bytes) -> void* {
                void* p = base ? base + off : nullptr;
                off += (bytes + 255) & ~(size_t)255;
                return p;
            };
            const size_t n_edges = (size_t)std::max(scene->dev.num_edges, 1), n_rec = (size_t)band * ka.rec_per_sample;
            d_shapes = (rb_dshape*)take(std::max(1, d_scene->num_shapes) * sizeof(rb_dshape));
            d_mats = (rb_material*)take(std::max(1, d_scene->num_materials) * sizeof(rb_material));
            d_lights = (float**)take(std::max(1, d_scene->num_lights) * sizeof(float*));
            // Every pass starts with these three at zero.  They stay adjacent, carved one after the other, so that one memset clears them.
            const size_t zeroed_begin = off;
            cam_accum = (double*)take(RB_CAM_ACC * sizeof(double));
            counters = (BandCounters*)take((size_t)num_bands * sizeof(BandCounters));
            ka.edge_hist = (unsigned*)take(secondary ? n_edges * 4 : 0);
            zeroed_bytes = off - zeroed_begin;
            ka.edge_offs = (unsigned*)take(secondary ? n_edges * 4 : 0);
            ka.edge_cursor = (unsigned*)take(secondary ? n_edges * 4 : 0);
            const size_t band_begin = off;
            ka.records = (VertexRec*)take(n_rec * sizeof(VertexRec));
            V3* dpos = (V3*)take(secondary ? n_rec * sizeof(V3) : 0);
            ka.dpos = secondary ? dpos : nullptr;
            ka.nrec = (int*)take((size_t)band * sizeof(int));
            ka.vmask = (ulonglong2*)take(secondary ? (size_t)band * sizeof(ulonglong2) : 0);
            list_offs = (ListCount*)take((size_t)band * sizeof(ListCount));
            scan_tmp = take(scan_bytes);
            ka.path_list = (int*)take((size_t)band * sizeof(int));
            ka.vert_list = (int*)take(secondary ? vert_cap * sizeof(int) : 0);
            ka.picks = (EdgePick*)take(secondary ? slots * sizeof(EdgePick) : 0);
            ka.sec_keys = (unsigned*)take(secondary ? slots * 4 : 0);
            ka.sec_vals = (unsigned*)take(secondary ? slots * 4 : 0);
            ka.sec_order = (unsigned*)take(secondary ? slots * 4 : 0);
            const size_t band_end = off;
            off = band_begin;
            k0 = (unsigned*)take((size_t)band_e * 4);
            k1 = (unsigned*)take((size_t)band_e * 4);
            v0 = (unsigned*)take((size_t)band_e * 4);
            v1 = (unsigned*)take((size_t)band_e * 4);
            sort_tmp = take(sort_bytes);
            return primary ? std::max(band_end, off) : band_end;
        };
        const size_t scratch_bytes = carve(nullptr);
        DeviceScratch& dscratch = g_scratch[scene->device & 63];
        scratch_lock = std::unique_lock<std::mutex>(dscratch.mutex);
        char* scratch = scratch_ensure(dscratch, scratch_bytes);
        if (!scratch) {
            rb_set_error("rb_render: out of device memory for the backward scratch");
            return 1;
        }
        carve(scratch);
        if (d_scene->num_shapes) RB_CUDA_OK(cudaMemcpyAsync(d_shapes, d_scene->shapes, d_scene->num_shapes * sizeof(rb_dshape), cudaMemcpyHostToDevice, stream));
        if (d_scene->num_materials)
            RB_CUDA_OK(cudaMemcpyAsync(d_mats, d_scene->materials, d_scene->num_materials * sizeof(rb_material), cudaMemcpyHostToDevice, stream));
        if (d_scene->num_lights)
            RB_CUDA_OK(cudaMemcpyAsync(d_lights, d_scene->light_intensity, d_scene->num_lights * sizeof(float*), cudaMemcpyHostToDevice, stream));
        RB_CUDA_OK(cudaMemsetAsync(cam_accum, 0, zeroed_bytes, stream)); // camera accumulators, band counters, edge histogram
        ka.ds.shapes = d_shapes;
        ka.ds.materials = d_mats;
        ka.ds.light_intensity = d_lights;
        ka.ds.cam_accum = cam_accum;

        // ---- interior + first-hit adjoints, band by band: trace (+ work lists) -> boundary terms (pick, counting sort by edge, shade)
        //      -> sweep.  Every list size stays on the device: fixed persistent grids, no host synchronisation inside the pass.
        const int grid_t = pick_grid(kern.bwd_trace, scene->device, RB_BLOCK_TRACE);
        const int grid_p = pick_grid(kern.bwd_sec_pick, scene->device, RB_BLOCK_SEC);
        const int grid_s = pick_grid(kern.bwd_sec_shade, scene->device, RB_BLOCK_SEC);
        const int grid_w = pick_grid(kern.bwd_sweep, scene->device, RB_BLOCK_SWEEP, RB_SMEM_CAM(RB_BLOCK_SWEEP));
        long long band_idx = 0;
        for (long long i0 = 0; i0 < total_samples; i0 += band, band_idx++) {
            ka.band_i0 = i0;
            ka.band_n = (int)std::min<long long>(band, total_samples - i0);
            ka.counters = counters + band_idx;
            cudaEvent_t* bev = &ev[(size_t)(NUM_FIXED_EVENTS + BAND_EVENTS * band_idx)];
            RB_CUDA_OK(cudaEventRecord(bev[BAND_BEGIN], stream));
            RB_CUDA_OK(cudaLaunchKernel(kern.bwd_trace, grid_t, RB_BLOCK_TRACE, args, 0, stream));
            RB_CUDA_OK(cudaEventRecord(bev[BAND_AFTER_TRACE], stream));
            {
                auto counts = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), ListCountOf{ka.nrec, secondary ? ka.vmask : nullptr});
                RB_CUDA_OK(cub::DeviceScan::ExclusiveScan(scan_tmp, scan_bytes, counts, list_offs, ListCountSum(), ListCount{0, 0, 0, 0}, ka.band_n, stream));
                k_bwd_compact<<<std::min((ka.band_n + 255) / 256, sms * 8), 256, 0, stream>>>(ka, list_offs);
            }
            launches += 4;
            if (secondary) {
                RB_CUDA_OK(cudaLaunchKernel(kern.bwd_sec_pick, grid_p, RB_BLOCK_SEC, args, 0, stream));
                k_sec_offsets<<<1, 1024, 0, stream>>>(ka, scene->dev.num_edges);
                k_sec_scatter<<<sms * 8, 256, 0, stream>>>(ka);
                RB_CUDA_OK(cudaLaunchKernel(kern.bwd_sec_shade, grid_s, RB_BLOCK_SEC, args, 0, stream));
                launches += 4;
            }
            RB_CUDA_OK(cudaEventRecord(bev[BAND_BEFORE_SWEEP], stream));
            RB_CUDA_OK(cudaLaunchKernel(kern.bwd_sweep, grid_w, RB_BLOCK_SWEEP, args, RB_SMEM_CAM(RB_BLOCK_SWEEP), stream));
            launches++;
            RB_CUDA_OK(cudaEventRecord(bev[BAND_END], stream));
        }
        num_bands_done = band_idx;
        if (num_bands_done > 0) {
            host_counters.resize((size_t)num_bands_done);
            RB_CUDA_OK(cudaMemcpyAsync(host_counters.data(), counters, (size_t)num_bands_done * sizeof(BandCounters), cudaMemcpyDeviceToHost, stream));
        }
        RB_CUDA_OK(cudaEventRecord(ev[EV_AFTER_BANDS], stream));
        if (primary) {
            int grid_e = pick_grid(kern.primary_edge, scene->device, RB_BLOCK_PRIM, RB_SMEM_CAM(RB_BLOCK_PRIM));
            int dim_base = primary_edge_dim_base(scene->dev, rp);
            int ebits = 1;
            while ((1 << ebits) < scene->dev.num_edges && ebits < 31) ebits++;
            for (long long t0 = 0; t0 < total_e; t0 += band_e) {
                int n = (int)std::min<long long>(band_e, total_e - t0);
                int grid_k = std::min((n + 255) / 256, sms * 16);
                void* key_args[] = {&scene->dev, &ka, &dim_base, &t0, &n, &k0, &v0};
                RB_CUDA_OK(cudaLaunchKernel(kern.prim_keys, grid_k, 256, key_args, 0, stream));
                // sort on the edge bits and the top 8 bits of the position only (coarser order is enough for coherence)
                int lo = std::max(0, 31 - ebits - 8);
                cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, k0, k1, v0, v1, n, lo, 32, stream);
                void* edge_args[] = {&scene->dev, &ka, &dim_base, &t0, &n, &k1, &v1};
                RB_CUDA_OK(cudaLaunchKernel(kern.primary_edge, grid_e, RB_BLOCK_PRIM, edge_args, RB_SMEM_CAM(RB_BLOCK_PRIM), stream));
                launches += 2 + 4;
            }
        }
        RB_CUDA_OK(cudaEventRecord(ev[EV_AFTER_PRIMARY_EDGE], stream));
        k_finish_camera<<<1, 32, 0, stream>>>(scene->dev.cam, cam_accum, d_scene->camera);
        launches++;
        RB_CUDA_OK(cudaEventRecord(ev[EV_END], stream));
    }
    cudaError_t err = cudaStreamSynchronize(stream);
    if (err == cudaSuccess) err = cudaGetLastError();
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[EV_BEGIN], ev[EV_END]);
    scene->last_launches = launches;
    scene->last_kernel_ms = ms;
    for (int i = EV_BEGIN; i < EV_END; i++) { // k_forward, backward bands, primary edges, k_finish_camera
        scene->last_stage_ms[i] = 0.f;
        if (err == cudaSuccess) cudaEventElapsedTime(&scene->last_stage_ms[i], ev[i], ev[i + 1]);
    }
    for (int i = 0; i < 3; i++) scene->last_bwd_ms[i] = 0.f;
    double host_stats[2] = {0, 0};
    if (err == cudaSuccess)
        for (long long b = 0; b < num_bands_done; b++) {
            const cudaEvent_t* bev = &ev[(size_t)(NUM_FIXED_EVENTS + BAND_EVENTS * b)];
            for (int i = BAND_BEGIN; i < BAND_END; i++) { // trace, work lists + boundary stage, sweep
                float t = 0.f;
                cudaEventElapsedTime(&t, bev[i], bev[i + 1]);
                scene->last_bwd_ms[i] += t;
            }
            host_stats[0] += (double)host_counters[(size_t)b].total_vertices;
            host_stats[1] += (double)host_counters[(size_t)b].total_hits;
        }
    scene->last_path_vertices = host_stats[0];
    scene->last_primary_hits = host_stats[1];
    if (err != cudaSuccess) {
        rb_set_error(std::string("rb_render: kernel failure: ") + cudaGetErrorString(err));
        return 1;
    }
    return 0;
}

// Batch of views of ONE scene (the multi-view loops of pyredner/render_utils.py:407-430 and of BASELINE config 5 rebuild the whole
// Scene per view): geometry, BVH, light tables and the edge list are shared; per view only the camera-dependent tables are rebuilt,
// on the device (rb_scene_set_camera), followed by the usual kernel set.  Gradients of all views ACCUMULATE into the buffers of
// d_scenes[k] (pass the same descriptor for every view to sum them: one gradient buffer for the batch).
extern "C" int rb_render_batch(rb_scene* scene, int num_views, const rb_camera* cameras, const rb_options* options, float* const* images,
                               const float* const* d_images, const rb_dscene_desc* const* d_scenes, void* stream) {
    if (!scene || num_views < 0 || (num_views > 0 && (!cameras || !options))) {
        rb_set_error("rb_render_batch: null argument");
        return 1;
    }
    for (int k = 0; k < num_views; k++) {
        if (rb_scene_set_camera(scene, &cameras[k])) return 1;
        if (rb_render(scene, &options[k], images ? images[k] : nullptr, d_images ? d_images[k] : nullptr, d_scenes ? d_scenes[k] : nullptr, nullptr, stream)) return 1;
    }
    return 0;
}
