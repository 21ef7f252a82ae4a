// Kernels of rb_render, included by rb_kernels.cu (general instantiation, global namespace) and by rb_kernels_lean.cu
// (feature-free instantiation, namespace rb_lean, RB_LEAN defined).  No include guard on purpose.  Both translation units
// include rb_kernel_set.h at global scope first.
// Threads per block and minimum resident blocks per SM (the __launch_bounds__ below) of each kernel family.  The per-sample stages
// are walked block-synchronously (RB_PHASE_SYNC), so the block size is also the number of threads that share one pass over the
// instruction stream; see DESIGN.md sections 2 and 6.  k_bwd_sweep is bound by the instruction cache (its SASS is far larger than
// the cache), so wide blocks that share one pass over the instruction stream win; k_bwd_trace and k_bwd_sec_* stay at <= 80
// registers so that more warps hide the dependent BVH and edge-tree fetches.
constexpr int RB_BLOCK = 128;                                // k_forward_channels (2 blocks / SM)
constexpr int RB_BLOCK_FWD = 256, RB_MIN_BLOCKS_FWD = 3;     // k_forward
constexpr int RB_BLOCK_TRACE = 256, RB_MIN_BLOCKS_TRACE = 3; // k_bwd_trace
constexpr int RB_BLOCK_SEC = 128, RB_MIN_BLOCKS_SEC = 6;     // k_bwd_sec_pick, k_bwd_sec_shade: 24 warps / SM at <= 80 registers
constexpr int RB_BLOCK_SWEEP = 512, RB_MIN_BLOCKS_SWEEP = 1; // k_bwd_sweep
constexpr int RB_BLOCK_PRIM = 128, RB_MIN_BLOCKS_PRIM = 5;   // k_primary_edge
// dynamic shared memory: per-thread columns of the n_cam = cam_acc_count(cam) camera accumulators (k_bwd_sweep, k_primary_edge)
#define RB_SMEM_CAM(n_cam, block) ((size_t)(n_cam) * (block) * sizeof(float))
// ... in the deterministic instantiation: the block's exact camera accumulators, [n_cam][RB_EXACT_WORDS]
#define RB_SMEM_CAM_EXACT(n_cam) ((size_t)(n_cam) * RB_EXACT_WORDS * sizeof(long long))
#ifndef RB_BAND_BYTES
#define RB_BAND_BYTES (1ULL << 30) // scratch budget of one backward band (records + lists)
#endif

struct WorkItem {
    bool valid;
    int pixel;    // viewport-relative pixel id (y * vp_w + x)
    int px, py;   // viewport-relative pixel coordinates
    int sample_lane;
};
RB_D WorkItem warp_work(const RenderParams& rp, int L, int owned_rows, long long group) {
    int lane = threadIdx.x & 31;
    int P = 32 / L;
    long long k = group * P + lane / L;
    WorkItem w;
    w.sample_lane = lane % L;
    long long n = (long long)owned_rows * rp.vp_w;
    w.valid = k < n;
    if (!w.valid) k = 0;
    int j = (int)(k / rp.vp_w), x = (int)(k % rp.vp_w);
    int y = owned_row_to_row(rp, j);
    w.pixel = y * rp.vp_w + x;
    w.px = x;
    w.py = y;
    return w;
}

// ------------------------------------------------------------------------------------------------ forward
// ---- optional: stage the Sobol rows of the main sampler in shared memory with ONE bulk asynchronous copy (TMA engine,
// cp.async.bulk + mbarrier) issued by one thread at kernel start -- north_star's "Sobol state staged through TMA into shared memory".
// Measured (DESIGN.md section 6): no gain -- the <= 4 KB of rows a configuration touches sit in L1 anyway -- so it is off by default.
#ifdef RB_TMA_SOBOL
#define RB_TMA_SOBOL_DIMS 32
RB_D unsigned rb_smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
RB_D const unsigned long long* stage_sobol_rows(const DevScene& sc, const RenderParams& rp, unsigned long long* smem_rows, unsigned long long* mbar) {
    const int dims = (int)main_draws_per_sample(sc, rp);
    if (rp.sampler_type != RB_SAMPLER_SOBOL || dims > RB_TMA_SOBOL_DIMS || dims == 0) return sc.sobol_matrices;
    const unsigned bytes = (unsigned)(dims * RB_SOBOL_BITS * sizeof(unsigned long long)); // 416 B per dimension: a multiple of 16
    const unsigned bar = rb_smem_addr(mbar), dst = rb_smem_addr(smem_rows);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(sc.sobol_matrices), "r"(bytes),
                     "r"(bar)
                     : "memory");
    }
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "RB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
        "@p bra RB_DONE;\n"
        "bra RB_WAIT;\n"
        "RB_DONE:\n"
        "}\n" ::"r"(bar)
        : "memory");
    return smem_rows;
}
#endif
#define RB_FWD_SYNC() RB_PHASE_SYNC() // measured: k_forward 5.2 -> 3.7 ms on C2 (one I-cache miss serves the block)
__global__ void __launch_bounds__(RB_BLOCK_FWD, RB_MIN_BLOCKS_FWD) k_forward(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const RenderParams& rp = ka.rp;
    const int L = ka.lanes_per_pixel;
    const int P = 32 / L;
    long long n_px = (long long)ka.owned_rows * rp.vp_w;
    long long groups = (n_px + P - 1) / P;
    long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int nb = (rp.spp + L - 1) / L;
#ifdef RB_TMA_SOBOL
    __shared__ alignas(16) unsigned long long sobol_rows[RB_TMA_SOBOL_DIMS * RB_SOBOL_BITS];
    __shared__ alignas(8) unsigned long long sobol_bar;
    const unsigned long long* sobol = stage_sobol_rows(sc, rp, sobol_rows, &sobol_bar);
#else
    const unsigned long long* sobol = nullptr;
#endif
    for (long long g0 = 0; g0 < groups; g0 += nwarps) { // block-uniform trip count (phase barrier inside)
        long long g = g0 + warp;
        WorkItem w = warp_work(rp, L, ka.owned_rows, g < groups ? g : 0);
        if (g >= groups) w.valid = false;
        V3 acc = zero3();
        for (int b = 0; b < nb; b++) {
            int s = b * L + w.sample_lane;
            RB_FWD_SYNC();
            if (w.valid && s < rp.spp) acc += forward_sample(sc, rp, w.pixel, w.px, w.py, s, sobol);
        }
        for (int off = L >> 1; off > 0; off >>= 1) {
            acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
            acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
            acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
        }
        if (w.valid && w.sample_lane == 0) {
            float* px = ka.image + (size_t)rp.nd * w.pixel + rp.rad_dim;
            px[0] += (float)acc.x;
            px[1] += (float)acc.y;
            px[2] += (float)acc.z;
        }
    }
}

#ifndef RB_LEAN // only the general instantiation renders G-buffer channels
// G-buffer forward (any channel list): one warp per pixel group like k_forward, channels reduced with shuffles; id
// channels take the value of the highest-numbered sample that hit (the reference overwrites them sample after sample).
__global__ void __launch_bounds__(RB_BLOCK, 2) k_forward_channels(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const RenderParams& rp = ka.rp;
    const int L = ka.lanes_per_pixel;
    const int P = 32 / L;
    long long n_px = (long long)ka.owned_rows * rp.vp_w;
    long long groups = (n_px + P - 1) / P;
    long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int nb = (rp.spp + L - 1) / L;
    const int nd = rp.nd < RB_MAX_ND ? rp.nd : RB_MAX_ND;
    for (long long g = warp; g < groups; g += nwarps) {
        WorkItem w = warp_work(rp, L, ka.owned_rows, g);
        float acc[RB_MAX_ND];
        for (int i = 0; i < nd; i++) acc[i] = 0.f;
        int ids[3] = {-1, -1, -1};
        int last = -1;
        for (int b = 0; b < nb; b++) {
            int s = b * L + w.sample_lane;
            if (w.valid && s < rp.spp) {
                int cur[3] = {-1, -1, -1};
                if (forward_sample_channels(sc, rp, w.pixel, w.px, w.py, s, acc, cur)) {
                    last = s;
                    ids[0] = cur[0]; ids[1] = cur[1]; ids[2] = cur[2];
                }
            }
        }
        for (int off = L >> 1; off > 0; off >>= 1) {
            for (int i = 0; i < nd; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
            int ol = __shfl_xor_sync(0xffffffffu, last, off);
            int o0 = __shfl_xor_sync(0xffffffffu, ids[0], off), o1 = __shfl_xor_sync(0xffffffffu, ids[1], off), o2 = __shfl_xor_sync(0xffffffffu, ids[2], off);
            if (ol > last) { last = ol; ids[0] = o0; ids[1] = o1; ids[2] = o2; }
        }
        if (w.valid && w.sample_lane == 0) write_gbuffer_pixel(rp, acc, ids, last >= 0, ka.image + (size_t)rp.nd * w.pixel);
    }
}

#endif
// ------------------------------------------------------------------------------------------------ backward (interior + first hit)
RB_D void block_reduce_camera(float* cam_smem, double* cam_accum, int n_cam) {
    // cam_smem: [n_cam][blockDim.x]; reduce each row and add to the global double accumulators
    __syncthreads();
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int k = warp; k < n_cam; k += nw) {
        float s = 0.f;
        for (int i = lane; i < (int)blockDim.x; i += 32) s += cam_smem[k * blockDim.x + i];
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0 && s != 0.f) atomicAdd(&cam_accum[k], (double)s);
    }
}
#ifdef RB_DETERMINISTIC
// Deterministic mode: the block's exact camera accumulators (shared memory, [n_cam][RB_EXACT_WORDS]) start at zero and end in
// the global exact accumulators 0 .. n_cam - 1, normalised first so that a block adds less than 2^32 to each limb.
RB_D void exact_camera_begin(long long* cam_exact, int n_cam) {
    for (int i = threadIdx.x; i < n_cam * RB_EXACT_WORDS; i += blockDim.x) cam_exact[i] = 0;
    __syncthreads();
}
RB_D void exact_camera_flush(long long* cam_exact, int n_cam) {
    __syncthreads();
    for (int k = threadIdx.x; k < n_cam; k += blockDim.x) {
        long long a[RB_EXACT_WORDS];
        for (int i = 0; i < RB_EXACT_WORDS; i++) a[i] = cam_exact[k * RB_EXACT_WORDS + i];
        exact_normalise(a);
        unsigned long long* g = (unsigned long long*)(rb_exact_acc + k * RB_EXACT_WORDS);
        for (int i = 0; i < RB_EXACT_LIMBS; i++)
            if (a[i] != 0) atomicAdd(g + i, (unsigned long long)a[i]);
        if (a[RB_EXACT_LIMBS] != 0) atomicOr(g + RB_EXACT_LIMBS, (unsigned long long)a[RB_EXACT_LIMBS]);
    }
}
#endif

// Dense live sample index -> (pixel, px, py, s): sample s of live pixel I / spp.  Consecutive lanes are consecutive samples of a pixel.
struct SampleId {
    int pixel, px, py, s;
};
RB_D SampleId band_sample(const KernelArgs& ka, long long I) {
    const RenderParams& rp = ka.rp;
    long long k = I / rp.spp;
    SampleId id;
    id.s = (int)(I - k * rp.spp);
    id.pixel = ka.live_pixels[k];
    id.py = id.pixel / rp.vp_w;
    id.px = id.pixel - id.py * rp.vp_w;
    return id;
}
// The work loops below are BLOCK-uniform (every thread of a block runs the same number of iterations, idle ones with
// act == false) because the per-sample stages contain phase barriers (RB_PHASE_SYNC, rb_render.cuh).
#define RB_BLOCK_LOOP(t, n) \
    for (long long t##_base = (long long)blockIdx.x * blockDim.x, t = t##_base + threadIdx.x; t##_base < (n); \
         t##_base += (long long)gridDim.x * blockDim.x, t = t##_base + threadIdx.x)
// Stage 1: replay the primal path of every sample of the band, one VertexRec per vertex.  Also decides, per vertex, whether the
// boundary stage will look at it at all (secondary edges are only sampled until the first rough bounce, src/edge.cpp:1396-1401)
// and which strategy its boundary sample takes: the first number of its edge-sampler point < 0.5 -> GATHER, else HIERARCHY
// (the reference's own per-sample coin, src/edge.cpp:1461-1472); one bit per depth in `vmask`.
// The bands hold the samples of live pixels only (KernelArgs::live_pixels): a sample whose pixel's adjoint is exactly zero adds
// nothing and never reaches this kernel.
__global__ void __launch_bounds__(RB_BLOCK_TRACE, RB_MIN_BLOCKS_TRACE) k_bwd_trace(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const RenderParams& rp = ka.rp;
    RB_BLOCK_LOOP(t, ka.band_n) {
        bool act = t < ka.band_n;
        SampleId id = band_sample(ka, ka.band_i0 + (act ? t : 0));
        VertexRec* recs = ka.records + (size_t)(act ? t : 0) * ka.rec_per_sample;
        int n = bwd_trace(sc, rp, id.pixel, id.px, id.py, id.s, recs, 1, act); // (-1 when not traced)
        if (!act) continue;
        ka.nrec[t] = n;
        if (ka.dpos != nullptr) {
            unsigned long long has = 0, gather = 0;
            for (int d = 0; d < n && d < 64; d++) {
                ka.dpos[(size_t)t * ka.rec_per_sample + d] = zero3();
                if (recs[d].min_rough <= Real(1e-2)) {
                    has |= 1ULL << d;
                    if (bwd_edge_sampler(sc, rp, id.pixel, id.s, d, 0).next() < 0.5) gather |= 1ULL << d;
                }
            }
            ka.vmask[t] = make_ulonglong2(has, gather);
        }
    }
}
#ifndef RB_LEAN // the work lists do not depend on scene features
// Stage 2: the work lists of the later stages, in SAMPLE ORDER (an exclusive scan over the band + this kernel; the reference
// compacts its wavefront with thrust::copy_if and a host read-back per bounce, src/active_pixels.cpp:17-49 -- here every
// list size stays on the device, `counters`, and the later kernels run fixed persistent grids):
//   path_list            samples whose primary ray hit something (work items of k_bwd_sweep)
//   vert_list, front     path vertices whose boundary sample takes the GATHER strategy
//   vert_list, back      ... the HIERARCHY strategy, filled downwards from the end of the same array: every warp of
//                        k_bwd_sec_pick then runs one strategy, while the coin itself stays the reference's per-sample one
struct ListCount {
    unsigned paths, gather, hier, vertices;
};
struct ListCountSum {
    __host__ __device__ ListCount operator()(const ListCount& a, const ListCount& b) const {
        ListCount r;
        r.paths = a.paths + b.paths;
        r.gather = a.gather + b.gather;
        r.hier = a.hier + b.hier;
        r.vertices = a.vertices + b.vertices;
        return r;
    }
};
struct ListCountOf {
    const int* nrec;
    const ulonglong2* vmask; // null without secondary edge sampling
    __host__ __device__ ListCount operator()(int t) const {
        ListCount r;
        int n = nrec[t];
        r.paths = n >= 0 ? 1u : 0u;
        r.vertices = n > 0 ? (unsigned)n : 0u;
        r.gather = r.hier = 0;
#ifdef __CUDA_ARCH__
        if (vmask != nullptr && n > 0) {
            ulonglong2 m = vmask[t];
            r.gather = (unsigned)__popcll(m.x & m.y);
            r.hier = (unsigned)__popcll(m.x & ~m.y);
        }
#endif
        return r;
    }
};
__global__ void k_bwd_compact(const __grid_constant__ KernelArgs ka, const ListCount* offs) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < ka.band_n; t += (long long)gridDim.x * blockDim.x) {
        ListCount o = offs[t];
        ListCount c = ListCountOf{ka.nrec, ka.dpos != nullptr ? ka.vmask : nullptr}((int)t);
        if (c.paths) ka.path_list[o.paths] = (int)t;
        if (c.gather + c.hier > 0) {
            ulonglong2 m = ka.vmask[t];
            unsigned g = o.gather, h = o.hier;
            for (unsigned long long bits = m.x; bits != 0; bits &= bits - 1) {
                int d = __ffsll((long long)bits) - 1;
                int e = (int)t * ka.rec_per_sample + d;
                if ((m.y >> d) & 1ULL) ka.vert_list[g++] = e;
                else ka.vert_list[(unsigned)ka.vert_cap - 1u - (h++)] = e;
            }
        }
        if (t == ka.band_n - 1) {
            BandCounters* cnt = ka.counters;
            cnt->n_paths = o.paths + c.paths;
            cnt->n_gather = o.gather + c.gather;
            cnt->n_hier = o.hier + c.hier;
            cnt->total_vertices = o.vertices + c.vertices; // statistics for the roofline accounting (mean path length, hit fraction)
            cnt->total_hits = o.paths + c.paths;
        }
    }
}
#endif
// Slot t of the boundary stage -> entry of vert_list: [0, n_gather) from the front, then (after padding to a warp boundary) the
// hierarchy entries from the back.
struct SecRange {
    unsigned n_g, pad, total;
};
RB_D SecRange sec_range(const KernelArgs& ka) {
    SecRange r;
    r.n_g = ka.counters->n_gather;
    r.pad = (r.n_g + 31u) & ~31u;
    r.total = r.pad + ka.counters->n_hier;
    return r;
}
RB_D int sec_entry(const KernelArgs& ka, const SecRange& r, long long t) {
    if (t < (long long)r.n_g) return ka.vert_list[t];
    if (t >= (long long)r.pad && t < (long long)r.total) return ka.vert_list[(unsigned)ka.vert_cap - 1u - (unsigned)(t - r.pad)];
    return -1;
}
// Stage 2a: edge pick of every listed path vertex (secondary edge sampling).  Writes the pick, its vertex and its edge per
// slot and counts the picks per edge (aggregated per warp) for the counting sort below.
__global__ void __launch_bounds__(RB_BLOCK_SEC, RB_MIN_BLOCKS_SEC) k_bwd_sec_pick(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const SecRange r = sec_range(ka);
    const long long n = r.total;
    RB_BLOCK_LOOP(t, n) {
        RB_PHASE_SYNC();
        if (t < n) {
            int e = sec_entry(ka, r, t);
            unsigned key = 0xffffffffu;
            if (e >= 0) {
                int ts = e / ka.rec_per_sample, d = e - ts * ka.rec_per_sample;
                SampleId id = band_sample(ka, ka.band_i0 + ts);
                VertexRec cur = ka.records[e];
                EdgePick pk;
                if (bwd_secondary_pick(sc, ka, id.pixel, id.s, d, cur, pk)) {
                    ka.picks[t] = pk;
                    key = (unsigned)pk.edge_id;
                }
            }
            ka.sec_keys[t] = key;
            ka.sec_vals[t] = (unsigned)e;
            if (key != 0xffffffffu) {
                unsigned peers = __match_any_sync(__activemask(), key);
                if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&ka.edge_hist[key], (unsigned)__popc(peers));
            }
        }
    }
}
#ifndef RB_LEAN // the counting sort does not depend on scene features
// Stage 2b: exclusive scan of the per-edge pick counts (one block; the histogram is zeroed again for the next band).
__global__ void __launch_bounds__(1024) k_sec_offsets(const __grid_constant__ KernelArgs ka, int num_edges) {
    __shared__ unsigned warp_sums[32];
    __shared__ unsigned carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < num_edges; base += 1024) {
        int i = base + tid;
        unsigned v = i < num_edges ? ka.edge_hist[i] : 0u, x = v;
        for (int off = 1; off < 32; off <<= 1) {
            unsigned y = __shfl_up_sync(0xffffffffu, x, off);
            if (lane >= off) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned w = warp_sums[lane], ws = w;
            for (int off = 1; off < 32; off <<= 1) {
                unsigned y = __shfl_up_sync(0xffffffffu, ws, off);
                if (lane >= off) ws += y;
            }
            warp_sums[lane] = ws - w; // exclusive prefix of the warp totals
        }
        __syncthreads();
        unsigned carry = carry_s;
        if (i < num_edges) {
            ka.edge_offs[i] = carry + warp_sums[warp] + x - v;
            ka.edge_hist[i] = 0;
            ka.edge_cursor[i] = 0;
        }
        __syncthreads();
        if (tid == 1023) carry_s = carry + warp_sums[31] + x;
        __syncthreads();
    }
    if (tid == 0) ka.counters->n_picked = carry_s;
}
// Stage 2c: scatter the slots into edge order (rank inside an edge: warp-aggregated cursor).
__global__ void __launch_bounds__(256) k_sec_scatter(const __grid_constant__ KernelArgs ka) {
    const SecRange r = sec_range(ka);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < (long long)r.total; t += (long long)gridDim.x * blockDim.x) {
        unsigned key = ka.sec_keys[t];
        if (key == 0xffffffffu) continue;
        unsigned peers = __match_any_sync(__activemask(), key);
        int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
        unsigned base = 0;
        if (lane == leader) base = atomicAdd(&ka.edge_cursor[key], (unsigned)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        ka.sec_order[ka.edge_offs[key] + base + __popc(peers & ((1u << lane) - 1u))] = (unsigned)t;
    }
}
#endif
// Stage 2d: the two edge rays and their sub-paths, in edge order (neighbouring lanes aim at the same edge).
__global__ void __launch_bounds__(RB_BLOCK_SEC, RB_MIN_BLOCKS_SEC) k_bwd_sec_shade(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const long long n = ka.counters->n_picked;
    RB_BLOCK_LOOP(j, n) {
        RB_PHASE_SYNC();
        if (j < n) {
            unsigned t = ka.sec_order[j];
            int e = (int)ka.sec_vals[t];
            int ts = e / ka.rec_per_sample, d = e - ts * ka.rec_per_sample;
            SampleId id = band_sample(ka, ka.band_i0 + ts);
            VertexRec cur = ka.records[e];
            EdgePick pk = ka.picks[t];
            ka.dpos[e] = bwd_secondary_shade(sc, ka, id.pixel, id.s, d, cur, pk);
        }
    }
}
// Stage 3: reverse sweep of every path, first-hit and camera adjoints.
__global__ void __launch_bounds__(RB_BLOCK_SWEEP, RB_MIN_BLOCKS_SWEEP) k_bwd_sweep(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    const int n_cam = cam_acc_count(sc.cam);
#ifdef RB_DETERMINISTIC
    extern __shared__ long long cam_exact[]; // [n_cam][RB_EXACT_WORDS]
    exact_camera_begin(cam_exact, n_cam);
    CamAcc cam_acc;
    cam_acc.exact = cam_exact;
#else
    extern __shared__ float cam_smem[]; // [n_cam][blockDim.x]
    for (int k = 0; k < n_cam; k++) cam_smem[k * blockDim.x + threadIdx.x] = 0.f;
    CamAcc cam_acc;
    cam_acc.base = cam_smem + threadIdx.x;
    cam_acc.stride = blockDim.x;
#endif
    const long long n = ka.counters->n_paths;
    RB_BLOCK_LOOP(t, n) {
        bool act = t < n;
        int ts = act ? ka.path_list[t] : 0;
        SampleId id = band_sample(ka, ka.band_i0 + ts);
        size_t base = (size_t)ts * ka.rec_per_sample;
        bwd_sweep(sc, ka, id.pixel, id.px, id.py, id.s, ka.records + base, 1, act ? ka.nrec[ts] : 0, ka.dpos ? ka.dpos + base : nullptr, cam_acc, act);
    }
#ifdef RB_DETERMINISTIC
    exact_camera_flush(cam_exact, n_cam);
#else
    block_reduce_camera(cam_smem, ka.ds.cam_accum, n_cam);
#endif
}

// ------------------------------------------------------------------------------------------------ primary edges
// One thread per (edge sample i, spp sample s), in two steps: k_prim_keys computes each sample's (edge, position on
// the edge) key, a radix sort orders the band by it, and k_primary_edge shades in that order -- neighbouring lanes then
// shoot nearly identical camera rays and scatter into the same two vertices.  (In sample order every lane picks an
// unrelated edge: 13 of 32 lanes active per instruction on C2.)  Sums are order-independent, so parity is unaffected.
#define RB_PRIM_SYNC() RB_PHASE_SYNC() // measured: k_primary_edge 19.2 -> 14.3 ms on C2
// dense index t of this device's primary-edge samples -> (i, s): i with i % num_parts == part
RB_D void prim_sample_id(const RenderParams& rp, long long t, long long& i, int& s) {
    long long k = t / rp.spp;
    i = k * rp.num_parts + rp.part;
    s = (int)(t - k * rp.spp);
}
__global__ void __launch_bounds__(256) k_prim_keys(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka, int dim_base, long long t0, int n,
                                                   unsigned* keys, unsigned* vals) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        long long i;
        int s;
        prim_sample_id(ka.rp, t0 + t, i, s);
        keys[t] = primary_edge_key(sc, ka, i, s, dim_base);
        vals[t] = (unsigned)t;
    }
}
#ifndef RB_DETERMINISTIC
// Adds a thread's run of primary-edge adjoints (the sums s[0..3] of edge e's samples) to the edge's sums in edge_adj.  The lanes of the
// current convergence group that flush the same edge are added together first (pointer doubling, as in warp_agg_add3) and the group
// leader issues the reductions.  Must stay inline for the same reason as warp_agg_add3.
RB_D void flush_edge_adjoint(double* edge_adj, int e, double s0, double s1, double s2, double s3) {
    unsigned peers = __match_any_sync(__activemask(), e);
    int lane = threadIdx.x & 31;
    unsigned above = peers & (0xfffffffeu << lane);
    int nxt = above ? __ffs(above) - 1 : -1;
    int n = __popc(peers);
#pragma unroll 1
    for (int span = 1; span < n; span <<= 1) {
        int src = nxt >= 0 ? nxt : lane;
        double o0 = __shfl_sync(peers, s0, src), o1 = __shfl_sync(peers, s1, src), o2 = __shfl_sync(peers, s2, src), o3 = __shfl_sync(peers, s3, src);
        int nn = __shfl_sync(peers, nxt, src);
        if (nxt >= 0) {
            s0 += o0; s1 += o1; s2 += o2; s3 += o3;
            nxt = nn;
        }
    }
    if (lane == __ffs(peers) - 1) {
        double* a = edge_adj + 4 * (size_t)e;
        if (s0 != 0) atomicAdd(a + 0, s0);
        if (s1 != 0) atomicAdd(a + 1, s1);
        if (s2 != 0) atomicAdd(a + 2, s2);
        if (s3 != 0) atomicAdd(a + 3, s3);
    }
}
#endif
// Shades the band's primary-edge samples in key order.  The deterministic instantiation and a camera with a lens project every sample
// (primary_edge_sample), the camera's gradients in per-thread shared-memory columns.  Otherwise the projection is linear in the
// screen-space adjoints and fixed per edge: each thread sums the adjoints of its run of samples of one edge in double, adds the run to
// ka.edge_adj when the edge changes, and k_prim_edge_project projects each edge's sum once.  The sort puts the samples of one edge next to
// each other, so a thread meets few edges (at most three on C2) and every lane of a warp mostly flushes the same one.  That path launches
// with no dynamic shared memory.
__global__ void __launch_bounds__(RB_BLOCK_PRIM, RB_MIN_BLOCKS_PRIM) k_primary_edge(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka, int dim_base,
                                                                               long long t0, int n, const unsigned* keys, const unsigned* vals) {
    const int n_cam = cam_acc_count(sc.cam);
#ifdef RB_DETERMINISTIC
    extern __shared__ long long cam_exact[]; // [n_cam][RB_EXACT_WORDS]
    exact_camera_begin(cam_exact, n_cam);
    CamAcc cam_acc;
    cam_acc.exact = cam_exact;
    RB_BLOCK_LOOP(t, n) {
        RB_PRIM_SYNC();
        if (t < n && keys[t] != 0xffffffffu) {
            long long i;
            int s;
            prim_sample_id(ka.rp, t0 + vals[t], i, s);
            primary_edge_sample(sc, ka, i, s, dim_base, cam_acc);
        }
    }
    exact_camera_flush(cam_exact, n_cam);
#else
    const bool lens = RB_CAM_LENS(sc.cam); // (block-uniform; always false in the sets without lenses)
    extern __shared__ float cam_smem[];   // [n_cam][blockDim.x], with a lens only
    CamAcc cam_acc;
    cam_acc.base = cam_smem + threadIdx.x;
    cam_acc.stride = blockDim.x;
    if (lens)
        for (int k = 0; k < n_cam; k++) cam_smem[k * blockDim.x + threadIdx.x] = 0.f;
    int run_e = -1; // the edge of this thread's run, and its sums
    double r0 = 0, r1 = 0, r2 = 0, r3 = 0;
    RB_BLOCK_LOOP(t, n) {
        RB_PRIM_SYNC();
        PrimEdgeAdjoint a;
        bool hit = false;
        if (t < n && keys[t] != 0xffffffffu) {
            long long i;
            int s;
            prim_sample_id(ka.rp, t0 + vals[t], i, s);
            hit = primary_edge_screen_adjoint(sc, ka, i, s, dim_base, a);
        }
        if (hit && lens) primary_edge_project(sc, ka, a.edge_id, a.lu, a.d0x, a.d0y, a.d1x, a.d1y, cam_acc);
        else if (hit) {
            if (a.edge_id != run_e) {
                if (run_e >= 0) flush_edge_adjoint(ka.edge_adj, run_e, r0, r1, r2, r3);
                run_e = a.edge_id;
                r0 = r1 = r2 = r3 = 0;
            }
            r0 += a.d0x; r1 += a.d0y;
            r2 += a.d1x; r3 += a.d1y;
        }
    }
    if (run_e >= 0) flush_edge_adjoint(ka.edge_adj, run_e, r0, r1, r2, r3);
    if (lens) block_reduce_camera(cam_smem, ka.ds.cam_accum, n_cam);
#endif
}
#ifndef RB_DETERMINISTIC
// After the last primary-edge band: one thread per edge projects the edge's summed screen-space adjoints (edge_adj) into its vertices'
// gradients and the camera accumulators, exactly as primary_edge_project does for one sample.  Edges no sample contributed to are skipped.
__global__ void __launch_bounds__(RB_BLOCK_PRIM) k_prim_edge_project(const __grid_constant__ DevScene sc, const __grid_constant__ KernelArgs ka) {
    __shared__ float cam_smem[RB_CAM_ACC * RB_BLOCK_PRIM]; // [RB_CAM_ACC][blockDim.x]
    for (int k = 0; k < RB_CAM_ACC; k++) cam_smem[k * blockDim.x + threadIdx.x] = 0.f;
    CamAcc cam_acc;
    cam_acc.base = cam_smem + threadIdx.x;
    cam_acc.stride = blockDim.x;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < sc.num_edges) {
        const double* a = ka.edge_adj + 4 * (size_t)e;
        const double s0 = a[0], s1 = a[1], s2 = a[2], s3 = a[3];
        if (s0 != 0 || s1 != 0 || s2 != 0 || s3 != 0) primary_edge_project(sc, ka, e, d2(0, 0), (Real)s0, (Real)s1, (Real)s2, (Real)s3, cam_acc);
    }
    block_reduce_camera(cam_smem, ka.ds.cam_accum, RB_CAM_ACC);
}
#endif

// The kernels of this instantiation that rb_render launches through a RenderKernels table (rb_kernel_set.h).
RenderKernels render_kernels() {
    RenderKernels k;
    k.forward = (const void*)k_forward;
    k.bwd_trace = (const void*)k_bwd_trace;
    k.bwd_sec_pick = (const void*)k_bwd_sec_pick;
    k.bwd_sec_shade = (const void*)k_bwd_sec_shade;
    k.bwd_sweep = (const void*)k_bwd_sweep;
    k.prim_keys = (const void*)k_prim_keys;
    k.primary_edge = (const void*)k_primary_edge;
#ifdef RB_DETERMINISTIC
    k.prim_edge_project = nullptr;
#else
    k.prim_edge_project = (const void*)k_prim_edge_project;
#endif
    return k;
}

#ifndef RB_LEAN
__global__ void k_finish_camera(DevCamera cam, const double* acc, rb_dcamera out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    finish_camera(cam, acc, out);
}
#endif

