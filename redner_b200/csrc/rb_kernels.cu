// Render kernels and the rb_render driver (reference: render(), src/pathtracer.cpp:177-958).
//
// Execution model (DESIGN.md section 2).  The reference runs a host-driven wavefront: ~20 launches and 2 host syncs per
// bounce per sample, with every per-path field (5.5 - 9.4 KB/pixel in double) streamed through managed memory between
// stage functors.  Here a path lives in registers inside a kernel and only a 128-byte record per path vertex crosses kernels:
//   forward    k_forward / k_forward_channels   camera sample -> primary hit -> emission -> bounce loop -> pixel
//   backward   per band of samples:  k_bwd_trace (primal replay, records, work lists by warp ballot) -> k_bwd_sec_pick ->
//              counting sort by edge (k_sec_offsets, k_sec_scatter) -> k_bwd_sec_shade (boundary terms) -> k_bwd_sweep (reverse
//              sweep, first-hit and camera adjoints);  then k_prim_keys -> radix sort -> k_primary_edge per band of edge samples,
//              k_prim_edge_project;  k_finish_camera
// Every kernel is small enough for the GPC instruction cache and walks the stages of a sample block-synchronously
// (RB_PHASE_SYNC): a fused megakernel of the same code ran instruction-fetch bound at 6 % issue utilisation.
// Forward: a warp owns 32/L pixels with L lanes per pixel (L = min(32, 2^floor(log2 spp))); lanes of a pixel are its
// samples, so rays of a warp are coherent in the BVH, the pixel is reduced with shuffles and written by one lane
// without atomics (deterministic image).  Gradient atomics are aggregated per warp before they reach L2.
// The per-sample logic itself lives in rb_render.cuh.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
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
#include "rb_exact_layout.hpp"

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

// Live-pixel list of a backward pass (KernelArgs::live_pixels): owned pixel k, row-major over the owned rows, -> its viewport pixel, kept
// by cub::DeviceSelect::If when its adjoint is not zero.  The selection keeps the input order, so the list is ascending.
struct OwnedPixelOf {
    RenderParams rp;
    __host__ __device__ int operator()(int k) const {
        int j = k / rp.vp_w;
        return owned_row_to_row(rp, j) * rp.vp_w + (k - j * rp.vp_w);
    }
};
struct PixelIsLive {
    KernelArgs ka;
    __host__ __device__ bool operator()(int pixel) const { return !ka.zero_cull || !pixel_adjoint_is_zero(ka, pixel); }
};

// The caller's records of rb_render_exact: the backward pass ends by adding its accumulators into them instead of rounding.
struct ExactExport {
    long long* records;
    size_t count;
};

// rb_render and rb_render_exact: the same passes, which differ only in the last step of the backward pass (xo == nullptr: round into
// the caller's buffers and finish the camera; otherwise: add the accumulators into xo->records).
static int render_pass(const rb_scene* scene_, const rb_options* opt, float* image, const float* d_image, const rb_dscene_desc* d_scene,
                       float* screen_grad, void* stream_, const ExactExport* xo) {
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
    if (const char* err = check_pixel_filter_options(scene->dev.cam, *opt, screen_grad)) {
        rb_set_error(err);
        return 1;
    }
    const RenderParams& rp = ka.rp;
    if (rp.vp_w <= 0 || rp.vp_h <= 0 || rp.spp == 0) return 0;
    // The feature-free instantiation of the kernels (rb_kernels_lean.cu) serves the common configuration, and its diffuse-only refinement
    // (rb_kernels_diffuse.cu) the scenes of that configuration whose materials are all diffuse; `kern` holds the kernels of the chosen
    // instantiation, and every launch of one of them below goes through it.  The materials are read from the scene's host copies on every
    // call: rb_scene_update may have changed their flags.  Neither set has the GGX lobe (RB_GGX is false there), nor emission textures
    // (RB_LIGHT_TEX), which the lights' host copies tell likewise.
    const bool lean_allowed = getenv("RB_NO_LEAN") == nullptr;       // (test hook: force the general kernels)
    const bool diffuse_allowed = getenv("RB_NO_DIFFUSE") == nullptr; // (test hook: force the lean kernels where the diffuse ones would run)
    const DevCamera& cam = scene->dev.cam;
    const bool lean = lean_allowed && !materials_use_ggx(scene->materials.data(), (int)scene->materials.size()) && !lights_use_emission(scene->light_emission) &&
                      rp.only_radiance && !scene->dev.has_envmap && cam.type == RB_CAMERA_PERSPECTIVE && !cam.has_distortion &&
                      cam.filter_type == RB_FILTER_BOX && cam.filter_width == 1.0f && cam.lens_radius == 0;
    const bool diffuse = lean && diffuse_allowed && materials_diffuse_only(scene->materials.data(), (int)scene->materials.size());
    const RenderKernels kern = diffuse ? rb_diffuse::render_kernels() : lean ? rb_lean::render_kernels() : render_kernels();
    // Deterministic mode: the backward kernels of rb_kernels_det.cu (the forward kernels are deterministic as they are).  Records
    // come from the exact accumulators, so rb_render_exact runs them whatever the options say.
    const bool det = opt->deterministic != 0 || xo != nullptr;
    const RenderKernels bkern = det ? rb_det::render_kernels() : kern;
    const rb_det::ExactKernels xk = rb_det::exact_kernels();

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
    long long live_samples = 0; // samples of the pixels whose adjoint is not zero (backward)
    size_t exact_bytes = 0; // exact accumulators of a deterministic backward pass
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
        if (const char* err = setup_backward(*d_scene, scene->dev, scene->light_emission.data(), ka)) {
            rb_set_error(err);
            return 1;
        }
        ExactLayout xl;
        if (det) {
            exact_layout(*d_scene, scene->shapes.data(), scene->materials.data(), scene->light_emission.data(), scene->dev, ka, xl);
            if (xo && xl.overlaps) {
                rb_set_error("rb_render_exact: gradient buffers of d_scene overlap; records need disjoint buffers");
                return 1;
            }
            if (xo && (size_t)xl.num_records != xo->count) {
                rb_set_error("rb_render_exact: count is " + std::to_string(xo->count) + " but the descriptor has " + std::to_string(xl.num_records) +
                             " records (rb_exact_record_count)");
                return 1;
            }
            ka.ds.env_values = xl.env_values;
            ka.ds.env_w2e = xl.env_w2e;
            ka.screen_grad = xl.screen_grad;
        }
        int n_cam = cam_acc_count(cam);
        // Without a lens the default sets sum each edge's screen-space adjoints and project them once per edge (k_prim_edge_project):
        // k_primary_edge then needs no camera columns in shared memory.
        const bool primary = primary_edge_pass_runs(scene->dev);
        const bool per_edge = primary && !det && !RB_CAM_LENS(cam);
        const size_t cam_smem_sweep = det ? RB_SMEM_CAM_EXACT(n_cam) : RB_SMEM_CAM(n_cam, RB_BLOCK_SWEEP),
                     cam_smem_prim = det ? RB_SMEM_CAM_EXACT(n_cam) : per_edge ? 0 : RB_SMEM_CAM(n_cam, RB_BLOCK_PRIM);
        const long long exact_max_samples = exact_band_samples(rp.max_bounces);
        if (det && exact_max_samples < 1) {
            rb_set_error("rb_render: deterministic mode supports at most 2097150 bounces");
            return 1;
        }
        const bool secondary = boundary_stage_runs(scene->dev, rp);
        const int owned_px = ka.owned_rows * rp.vp_w;
        const long long total_samples = (long long)owned_px * rp.spp; // (the bands run over the live ones only; this bounds their number)
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
        if (det) band = std::min(band, exact_max_samples);
        band = std::min<long long>(band, std::max<long long>(total_samples, 1));
        const long long max_bands = (total_samples + band - 1) / band;
        auto owned_it = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), OwnedPixelOf{rp});
        size_t select_bytes = 0;
        cub::DeviceSelect::If(nullptr, select_bytes, owned_it, (int*)nullptr, (int*)nullptr, owned_px, PixelIsLive{ka}, stream);
        auto count_it = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), ListCountOf{nullptr, nullptr});
        size_t scan_bytes = 0;
        cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, count_it, (ListCount*)nullptr, ListCountSum(), ListCount{0, 0, 0, 0}, (int)band, stream);
        // boundary terms: vertex list, edge picks, (edge, vertex) per slot, slots in edge order
        const size_t vert_cap = (size_t)band * ka.rec_per_sample, slots = vert_cap + 32;
        ka.vert_cap = (int)vert_cap;
        const long long n_px_all = (long long)rp.vp_w * rp.vp_h;
        const long long total_e = primary ? ((n_px_all - rp.part + rp.num_parts - 1) / rp.num_parts) * rp.spp : 0; // i % num_parts == part
        const long long band_e = std::min<long long>(std::max<long long>(total_e, 1), det ? std::min(1LL << 26, exact_max_samples) : 1LL << 26);
        size_t sort_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned*)nullptr, (unsigned*)nullptr, (int)band_e, 0, 32, stream);

        // ---- scratch layout, in carving order, every buffer 256-byte aligned: gradient descriptors | camera accumulators | band counters |
        //      edge histogram | per-edge primary-edge adjoint sums | edge offsets and cursors | live-pixel list, its count and its selection
        //      temporaries | band (records, boundary terms, work lists).  The primary-edge pass runs after the
        //      bands and reuses the band area for its keys / values (double buffers) and radix-sort temporaries.  The buffers of the
        //      boundary stage are empty when it does not run.  carve(nullptr) only measures; both calls return the size.
        rb_dshape* d_shapes;
        rb_material* d_mats;
        float** d_lights;
        double* cam_accum;
        BandCounters* counters;
        ListCount* list_offs;
        long long* exact_acc; // deterministic mode: xl.num_acc accumulators and the spare
        ExactRange* exact_ranges;
        long long* exact_rec_first; // (rb_render_exact)
        int *live_pixels, *live_count;
        void *select_tmp, *scan_tmp, *sort_tmp;
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
            // (the intensity-gradient pointers, then the gradients of the emission textures: light_d_emission, rb_types.cuh)
            d_lights = (float**)take(std::max<size_t>(light_table_offset(d_scene->num_lights * sizeof(float*)) + d_scene->num_lights * sizeof(rb_texture), 8));
            exact_acc = (long long*)take(det ? (size_t)(xl.num_acc + 1) * RB_EXACT_WORDS * sizeof(long long) : 0);
            exact_ranges = (ExactRange*)take(det ? std::max<size_t>(xl.ranges.size(), 1) * sizeof(ExactRange) : 0);
            exact_rec_first = (long long*)take(xo ? std::max<size_t>(xl.rec_first.size(), 1) * sizeof(long long) : 0);
            // Every pass starts with these four at zero.  They stay adjacent, carved one after the other, so that one memset clears them.
            // The per-edge sums span every primary-edge band, outside the band area that the keys and values reuse.
            const size_t zeroed_begin = off;
            cam_accum = (double*)take(RB_CAM_ACC_LENS * sizeof(double));
            counters = (BandCounters*)take((size_t)max_bands * sizeof(BandCounters));
            ka.edge_hist = (unsigned*)take(secondary ? n_edges * 4 : 0);
            double* edge_adj = (double*)take(per_edge ? n_edges * 4 * sizeof(double) : 0);
            ka.edge_adj = per_edge ? edge_adj : nullptr;
            zeroed_bytes = off - zeroed_begin;
            ka.edge_offs = (unsigned*)take(secondary ? n_edges * 4 : 0);
            ka.edge_cursor = (unsigned*)take(secondary ? n_edges * 4 : 0);
            live_pixels = (int*)take((size_t)owned_px * sizeof(int));
            live_count = (int*)take(sizeof(int));
            select_tmp = take(select_bytes);
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
            rb_set_error(det ? "rb_render: out of device memory for the backward scratch and the exact gradient accumulators of deterministic mode"
                             : "rb_render: out of device memory for the backward scratch");
            return 1;
        }
        carve(scratch);
        // (deterministic mode: the descriptors with the virtual addresses of the accumulators; no kernel reads a gradient buffer)
        const rb_dshape* h_shapes = det ? xl.shapes.data() : d_scene->shapes;
        const rb_material* h_mats = det ? xl.materials.data() : d_scene->materials;
        const std::vector<unsigned long long> h_lights = light_table_words(det ? xl.lights.data() : d_scene->light_intensity,
                                                                           det ? (xl.light_emission.empty() ? nullptr : xl.light_emission.data()) : d_scene->light_emission,
                                                                           d_scene->num_lights);
        if (d_scene->num_shapes) RB_CUDA_OK(cudaMemcpyAsync(d_shapes, h_shapes, d_scene->num_shapes * sizeof(rb_dshape), cudaMemcpyHostToDevice, stream));
        if (d_scene->num_materials)
            RB_CUDA_OK(cudaMemcpyAsync(d_mats, h_mats, d_scene->num_materials * sizeof(rb_material), cudaMemcpyHostToDevice, stream));
        if (d_scene->num_lights)
            RB_CUDA_OK(cudaMemcpyAsync(d_lights, h_lights.data(), h_lights.size() * 8, cudaMemcpyHostToDevice, stream));
        if (det) {
            if (!xl.ranges.empty())
                RB_CUDA_OK(cudaMemcpyAsync(exact_ranges, xl.ranges.data(), xl.ranges.size() * sizeof(ExactRange), cudaMemcpyHostToDevice, stream));
            if (xo && !xl.rec_first.empty())
                RB_CUDA_OK(cudaMemcpyAsync(exact_rec_first, xl.rec_first.data(), xl.rec_first.size() * sizeof(long long), cudaMemcpyHostToDevice, stream));
            exact_bytes = (size_t)(xl.num_acc + 1) * RB_EXACT_WORDS * sizeof(long long);
            RB_CUDA_OK(cudaMemsetAsync(exact_acc, 0, exact_bytes, stream));
            RB_CUDA_OK((cudaError_t)rb_det::bind_exact_accumulators(exact_acc, stream));
        }
        long long n_acc = xl.num_acc;
        void* normalise_args[] = {&exact_acc, &n_acc};
        const int grid_x = sms * 4;
        RB_CUDA_OK(cudaMemsetAsync(cam_accum, 0, zeroed_bytes, stream)); // camera accumulators, band counters, edge histogram, edge sums
        ka.ds.shapes = d_shapes;
        ka.ds.materials = d_mats;
        ka.ds.light_intensity = d_lights;
        ka.ds.cam_accum = cam_accum;

        // ---- the live pixels: those of the owned rows whose adjoint is not zero, in ascending order.  Their count is the one value
        //      read back inside the pass: the bands then cover the live samples only, so a mostly-zero adjoint runs few bands.
        ka.live_pixels = live_pixels;
        RB_CUDA_OK(cub::DeviceSelect::If(select_tmp, select_bytes, owned_it, live_pixels, live_count, owned_px, PixelIsLive{ka}, stream));
        launches += 2;
        int n_live_px = 0;
        RB_CUDA_OK(cudaMemcpyAsync(&n_live_px, live_count, sizeof(int), cudaMemcpyDeviceToHost, stream));
        RB_CUDA_OK(cudaStreamSynchronize(stream));
        live_samples = (long long)n_live_px * rp.spp;
        if (!events.ensure((size_t)(NUM_FIXED_EVENTS + BAND_EVENTS * ((live_samples + band - 1) / band)))) {
            rb_set_error("rb_render: cudaEventCreate failed");
            return 1;
        }

        // ---- interior + first-hit adjoints, band by band: trace (+ work lists) -> boundary terms (pick, counting sort by edge, shade)
        //      -> sweep.  Every list size stays on the device: fixed persistent grids, no host synchronisation inside the bands.
        const int grid_t = pick_grid(bkern.bwd_trace, scene->device, RB_BLOCK_TRACE);
        const int grid_p = pick_grid(bkern.bwd_sec_pick, scene->device, RB_BLOCK_SEC);
        const int grid_s = pick_grid(bkern.bwd_sec_shade, scene->device, RB_BLOCK_SEC);
        const int grid_w = pick_grid(bkern.bwd_sweep, scene->device, RB_BLOCK_SWEEP, cam_smem_sweep);
        long long band_idx = 0;
        for (long long i0 = 0; i0 < live_samples; i0 += band, band_idx++) {
            ka.band_i0 = i0;
            ka.band_n = (int)std::min<long long>(band, live_samples - i0);
            ka.counters = counters + band_idx;
            cudaEvent_t* bev = &ev[(size_t)(NUM_FIXED_EVENTS + BAND_EVENTS * band_idx)];
            RB_CUDA_OK(cudaEventRecord(bev[BAND_BEGIN], stream));
            RB_CUDA_OK(cudaLaunchKernel(bkern.bwd_trace, grid_t, RB_BLOCK_TRACE, args, 0, stream));
            RB_CUDA_OK(cudaEventRecord(bev[BAND_AFTER_TRACE], stream));
            {
                auto counts = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), ListCountOf{ka.nrec, secondary ? ka.vmask : nullptr});
                RB_CUDA_OK(cub::DeviceScan::ExclusiveScan(scan_tmp, scan_bytes, counts, list_offs, ListCountSum(), ListCount{0, 0, 0, 0}, ka.band_n, stream));
                k_bwd_compact<<<std::min((ka.band_n + 255) / 256, sms * 8), 256, 0, stream>>>(ka, list_offs);
            }
            launches += 4;
            if (secondary) {
                RB_CUDA_OK(cudaLaunchKernel(bkern.bwd_sec_pick, grid_p, RB_BLOCK_SEC, args, 0, stream));
                k_sec_offsets<<<1, 1024, 0, stream>>>(ka, scene->dev.num_edges);
                k_sec_scatter<<<sms * 8, 256, 0, stream>>>(ka);
                RB_CUDA_OK(cudaLaunchKernel(bkern.bwd_sec_shade, grid_s, RB_BLOCK_SEC, args, 0, stream));
                launches += 4;
            }
            RB_CUDA_OK(cudaEventRecord(bev[BAND_BEFORE_SWEEP], stream));
            RB_CUDA_OK(cudaLaunchKernel(bkern.bwd_sweep, grid_w, RB_BLOCK_SWEEP, args, cam_smem_sweep, stream));
            launches++;
            if (det) {
                RB_CUDA_OK(cudaLaunchKernel(xk.normalise, grid_x, 256, normalise_args, 0, stream));
                launches++;
            }
            RB_CUDA_OK(cudaEventRecord(bev[BAND_END], stream));
        }
        num_bands_done = band_idx;
        if (num_bands_done > 0) {
            host_counters.resize((size_t)num_bands_done);
            RB_CUDA_OK(cudaMemcpyAsync(host_counters.data(), counters, (size_t)num_bands_done * sizeof(BandCounters), cudaMemcpyDeviceToHost, stream));
        }
        RB_CUDA_OK(cudaEventRecord(ev[EV_AFTER_BANDS], stream));
        if (primary) {
            int grid_e = pick_grid(bkern.primary_edge, scene->device, RB_BLOCK_PRIM, cam_smem_prim);
            int dim_base = primary_edge_dim_base(scene->dev, rp);
            int ebits = 1;
            while ((1 << ebits) < scene->dev.num_edges && ebits < 31) ebits++;
            for (long long t0 = 0; t0 < total_e; t0 += band_e) {
                int n = (int)std::min<long long>(band_e, total_e - t0);
                int grid_k = std::min((n + 255) / 256, sms * 16);
                void* key_args[] = {&scene->dev, &ka, &dim_base, &t0, &n, &k0, &v0};
                RB_CUDA_OK(cudaLaunchKernel(bkern.prim_keys, grid_k, 256, key_args, 0, stream));
                // sort on the edge bits and the top 8 bits of the position only (coarser order is enough for coherence)
                int lo = std::max(0, 31 - ebits - 8);
                cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, k0, k1, v0, v1, n, lo, 32, stream);
                void* edge_args[] = {&scene->dev, &ka, &dim_base, &t0, &n, &k1, &v1};
                RB_CUDA_OK(cudaLaunchKernel(bkern.primary_edge, grid_e, RB_BLOCK_PRIM, edge_args, cam_smem_prim, stream));
                launches += 2 + 4;
                if (det) {
                    RB_CUDA_OK(cudaLaunchKernel(xk.normalise, grid_x, 256, normalise_args, 0, stream));
                    launches++;
                }
            }
            if (per_edge) {
                RB_CUDA_OK(cudaLaunchKernel(bkern.prim_edge_project, (scene->dev.num_edges + RB_BLOCK_PRIM - 1) / RB_BLOCK_PRIM, RB_BLOCK_PRIM, args, 0, stream));
                launches++;
            }
        }
        RB_CUDA_OK(cudaEventRecord(ev[EV_AFTER_PRIMARY_EDGE], stream));
        int num_ranges = (int)xl.ranges.size();
        if (xo) { // rb_render_exact: every accumulator, the camera's included, into the caller's records; no buffer of d_scene is written
            long long* records = xo->records;
            void* exp_args[] = {&exact_acc, &n_acc, &exact_ranges, &exact_rec_first, &num_ranges, &records, &n_cam};
            RB_CUDA_OK(cudaLaunchKernel(xk.export_records, grid_x, 256, exp_args, 0, stream));
            launches++;
        } else {
            if (det) { // round every accumulator once: into the caller's buffers, and the camera's into cam_accum
                void* fin_args[] = {&exact_acc, &n_acc, &exact_ranges, &num_ranges, &cam_accum, &n_cam};
                RB_CUDA_OK(cudaLaunchKernel(xk.finalise, grid_x, 256, fin_args, 0, stream));
                launches++;
            }
            k_finish_camera<<<1, 32, 0, stream>>>(scene->dev.cam, cam_accum, d_scene->camera);
            launches++;
        }
        RB_CUDA_OK(cudaEventRecord(ev[EV_END], stream));
    }
    cudaError_t err = cudaStreamSynchronize(stream);
    if (err == cudaSuccess) err = cudaGetLastError();
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[EV_BEGIN], ev[EV_END]);
    scene->last_launches = launches;
    scene->last_live_samples = live_samples;
    scene->last_bands = num_bands_done;
    scene->last_exact_bytes = exact_bytes;
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

extern "C" int rb_render(const rb_scene* scene, const rb_options* opt, float* image, const float* d_image, const rb_dscene_desc* d_scene,
                         float* screen_grad, void* stream) {
    return render_pass(scene, opt, image, d_image, d_scene, screen_grad, stream, nullptr);
}

// ------------------------------------------------------------------------------------------------ records (rb_exact.cuh)
extern "C" int rb_exact_record_count(const rb_scene* scene, const rb_options* opt, const rb_dscene_desc* d_scene, float* screen_grad, size_t* count,
                                     uint64_t* fingerprint) {
    if (!scene || !opt || !count) {
        rb_set_error("rb_exact_record_count: null scene / options / count");
        return 1;
    }
    KernelArgs ka;
    ExactLayout xl;
    std::string err;
    if (const char* e = exact_record_layout("rb_exact_record_count", *opt, scene->cam, scene->max_generic_texture_dimension, d_scene, screen_grad,
                                            scene->shapes.data(), scene->materials.data(), scene->light_emission.data(), scene->dev, ka, xl, err)) {
        rb_set_error(e);
        return 1;
    }
    *count = (size_t)xl.num_records;
    if (fingerprint) *fingerprint = xl.fingerprint;
    return 0;
}

extern "C" int rb_render_exact(const rb_scene* scene, const rb_options* opt, const float* d_image, const rb_dscene_desc* d_scene, float* screen_grad,
                               long long* records, size_t count, void* stream) {
    if (!d_image || !d_scene || !records) {
        rb_set_error("rb_render_exact: null d_rendered_image / d_scene / records");
        return 1;
    }
    const ExactExport xo{records, count};
    return render_pass(scene, opt, nullptr, d_image, d_scene, screen_grad, stream, &xo);
}

extern "C" int rb_exact_round(const rb_scene* scene, const rb_options* opt, const rb_dscene_desc* d_scene, float* screen_grad, const long long* records,
                              size_t count, void* stream_) {
    if (!scene || !opt || !records) {
        rb_set_error("rb_exact_round: null scene / options / records");
        return 1;
    }
    if (scene->incomplete) {
        rb_set_error("rb_exact_round: the scene's last update failed; update it again or build a new scene");
        return 1;
    }
    KernelArgs ka;
    ExactLayout xl;
    std::string err;
    if (const char* e = exact_record_layout("rb_exact_round", *opt, scene->cam, scene->max_generic_texture_dimension, d_scene, screen_grad, scene->shapes.data(),
                                            scene->materials.data(), scene->light_emission.data(), scene->dev, ka, xl, err)) {
        rb_set_error(e);
        return 1;
    }
    if ((size_t)xl.num_records != count) {
        rb_set_error("rb_exact_round: count is " + std::to_string(count) + " but the descriptor has " + std::to_string(xl.num_records) +
                     " records (rb_exact_record_count)");
        return 1;
    }
    RenderGuard guard;
    int prev = 0;
    RB_CUDA_OK(cudaGetDevice(&prev));
    RB_CUDA_OK(cudaSetDevice(scene->device));
    guard.prev_device = prev;
    cudaStream_t stream = (cudaStream_t)stream_;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, scene->device);
    // scratch: accumulators | ranges | record of each range | camera doubles, every buffer 256-byte aligned
    auto align = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t acc_bytes = align((size_t)(xl.num_acc + 1) * RB_EXACT_WORDS * sizeof(long long));
    const size_t range_bytes = align(std::max<size_t>(xl.ranges.size(), 1) * sizeof(ExactRange));
    const size_t rec_bytes = align(std::max<size_t>(xl.rec_first.size(), 1) * sizeof(long long));
    DeviceScratch& dscratch = g_scratch[scene->device & 63];
    std::lock_guard<std::mutex> lock(dscratch.mutex);
    char* scratch = scratch_ensure(dscratch, acc_bytes + range_bytes + rec_bytes + RB_CAM_ACC_LENS * sizeof(double));
    if (!scratch) {
        rb_set_error("rb_exact_round: out of device memory for the exact accumulators");
        return 1;
    }
    long long* acc = (long long*)scratch;
    ExactRange* ranges = (ExactRange*)(scratch + acc_bytes);
    long long* rec_first = (long long*)(scratch + acc_bytes + range_bytes);
    double* cam_accum = (double*)(scratch + acc_bytes + range_bytes + rec_bytes);
    if (!xl.ranges.empty()) {
        RB_CUDA_OK(cudaMemcpyAsync(ranges, xl.ranges.data(), xl.ranges.size() * sizeof(ExactRange), cudaMemcpyHostToDevice, stream));
        RB_CUDA_OK(cudaMemcpyAsync(rec_first, xl.rec_first.data(), xl.rec_first.size() * sizeof(long long), cudaMemcpyHostToDevice, stream));
    }
    RB_CUDA_OK(cudaMemsetAsync(cam_accum, 0, RB_CAM_ACC_LENS * sizeof(double), stream));
    const rb_det::ExactKernels xk = rb_det::exact_kernels();
    long long n_acc = xl.num_acc;
    int num_ranges = (int)xl.ranges.size();
    int n_cam = cam_acc_count(scene->dev.cam);
    void* imp_args[] = {&acc, &n_acc, &ranges, &rec_first, &num_ranges, (void*)&records, &n_cam};
    RB_CUDA_OK(cudaLaunchKernel(xk.import_records, sms * 4, 256, imp_args, 0, stream));
    // from here on the end of a deterministic rb_render: round every accumulator once, then the camera
    void* fin_args[] = {&acc, &n_acc, &ranges, &num_ranges, &cam_accum, &n_cam};
    RB_CUDA_OK(cudaLaunchKernel(xk.finalise, sms * 4, 256, fin_args, 0, stream));
    k_finish_camera<<<1, 32, 0, stream>>>(scene->dev.cam, cam_accum, d_scene->camera);
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    RB_CUDA_OK(cudaGetLastError());
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

// Test hook: exact sums through the deterministic scatter (see the header).  Contribution j of [0, n * repeat) adds values[j % n] to
// slot slots[j % n]; the slots are accumulators of the device scratch, normalised after every RB_EXACT_MAX_ADDS contributions.
extern "C" int rb_exact_sum_test(const float* values, const int* slots, int n, int num_slots, long long repeat, float* out_f32, double* out_f64, void* stream_) {
    if (n < 0 || num_slots < 0 || repeat < 0 || (n > 0 && (!values || !slots)) || (num_slots > 0 && (!out_f32 || !out_f64))) {
        rb_set_error("rb_exact_sum_test: bad arguments");
        return 1;
    }
    if (num_slots == 0) return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    std::vector<int> h_slots((size_t)n);
    if (n > 0) { // (read on the caller's stream, which wrote them)
        RB_CUDA_OK(cudaMemcpyAsync(h_slots.data(), slots, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, stream));
        RB_CUDA_OK(cudaStreamSynchronize(stream));
    }
    for (int s : h_slots)
        if (s < 0 || s >= num_slots) {
            rb_set_error("rb_exact_sum_test: slot out of range");
            return 1;
        }
    int device = 0, sms = 132;
    RB_CUDA_OK(cudaGetDevice(&device));
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    DeviceScratch& dscratch = g_scratch[device & 63];
    std::lock_guard<std::mutex> lock(dscratch.mutex); // the accumulator binding is per device, like a backward pass
    long long* acc = (long long*)scratch_ensure(dscratch, (size_t)num_slots * RB_EXACT_WORDS * sizeof(long long));
    if (!acc) {
        rb_set_error("rb_exact_sum_test: out of device memory");
        return 1;
    }
    const rb_det::ExactKernels xk = rb_det::exact_kernels();
    RB_CUDA_OK(cudaMemsetAsync(acc, 0, (size_t)num_slots * RB_EXACT_WORDS * sizeof(long long), stream));
    RB_CUDA_OK((cudaError_t)rb_det::bind_exact_accumulators(acc, stream));
    long long n_acc = num_slots;
    void* normalise_args[] = {&acc, &n_acc};
    const long long total = (long long)n * repeat;
    for (long long j0 = 0; j0 < total; j0 += RB_EXACT_MAX_ADDS) {
        long long count = std::min<long long>(RB_EXACT_MAX_ADDS, total - j0);
        void* args[] = {(void*)&values, (void*)&slots, &n, &j0, &count};
        RB_CUDA_OK(cudaLaunchKernel(xk.sum_test, sms * 8, 256, args, 0, stream));
        RB_CUDA_OK(cudaLaunchKernel(xk.normalise, sms * 4, 256, normalise_args, 0, stream));
    }
    void* out_args[] = {&acc, &num_slots, &out_f32, &out_f64};
    RB_CUDA_OK(cudaLaunchKernel(xk.readout, std::min((num_slots + 255) / 256, sms * 8), 256, out_args, 0, stream));
    RB_CUDA_OK(cudaStreamSynchronize(stream));
    RB_CUDA_OK(cudaGetLastError());
    return 0;
}
