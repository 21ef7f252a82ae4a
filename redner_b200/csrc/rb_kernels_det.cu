// Deterministic instantiation of the render kernels: the very same source (rb_kernels_body.cuh and every per-sample header) with
// the general features, compiled with RB_DETERMINISTIC inside namespace rb_det.  Every gradient scatter then adds into exact
// fixed-point accumulators (rb_exact.cuh, rb_atomic.cuh) instead of issuing float atomics, and the camera goes through exact
// per-block accumulators, so the gradients do not depend on the order in which threads, warps and blocks add.  rb_render launches
// these backward kernels when rb_options::deterministic is set, rb_render_exact always, and the kernels below normalise, round and hand
// out the sums, or move them to and from records.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "../../include/redner_b200.h"
#include "rb_kernel_set.h"

#define RB_DETERMINISTIC 1
namespace rb_det {
#include "rb_render.cuh"
#include "rb_kernels_body.cuh"

// Carries of accumulators [0, n), between bands (the overflow bound of rb_exact.cuh).
__global__ void k_exact_normalise(long long* acc, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long a[RB_EXACT_WORDS];
        long long* p = acc + i * RB_EXACT_WORDS;
        for (int k = 0; k < RB_EXACT_LIMBS; k++) a[k] = p[k];
        exact_normalise(a);
        for (int k = 0; k < RB_EXACT_LIMBS; k++) p[k] = a[k];
    }
}
// End of a deterministic backward pass: every accumulator that received something is rounded once (exact_finalise); the camera's
// become the doubles k_finish_camera reads.
__global__ void k_exact_finalise(const long long* acc, long long n, const ExactRange* ranges, int num_ranges, double* cam_accum) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        exact_finalise(acc, i, ranges, num_ranges, cam_accum, RB_CAM_ACC);
}
// rb_render_exact: every accumulator [0, n) is added into its record and the record left normalised (exact_export).  Accumulators
// and records are disjoint one-to-one (the layout refuses overlapping buffers), so no two threads touch one record.
__global__ void k_exact_export(const long long* acc, long long n, const ExactRange* ranges, const long long* rec_first, int num_ranges, long long* records) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        exact_export(acc + i * RB_EXACT_WORDS, records + exact_record_of(i, ranges, rec_first, num_ranges, RB_CAM_ACC) * RB_EXACT_RECORD_WORDS);
}
// rb_exact_round: accumulators [0, n) from their records (exact_import), ready for k_exact_finalise.
__global__ void k_exact_import(long long* acc, long long n, const ExactRange* ranges, const long long* rec_first, int num_ranges, const long long* records) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        exact_import(records + exact_record_of(i, ranges, rec_first, num_ranges, RB_CAM_ACC) * RB_EXACT_RECORD_WORDS, acc + i * RB_EXACT_WORDS);
}
// Test hook rb_exact_sum_test: contribution j of [j0, j0 + count) adds values[j % n] to slot slots[j % n] through the scatter of the
// render kernels (rb_red_add: the same warp aggregation and integer reductions), slot s being accumulator s.
__global__ void k_exact_sum_test(const float* values, const int* slots, int n, long long j0, long long count) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (long long)gridDim.x * blockDim.x) {
        const int k = (int)((j0 + t) % n);
        rb_red_add(exact_virtual(slots[k]), values[k]);
    }
}
__global__ void k_exact_readout(const long long* acc, int n, float* out_f32, double* out_f64) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        out_f32[i] = exact_to_float(acc + (size_t)i * RB_EXACT_WORDS);
        out_f64[i] = exact_to_double(acc + (size_t)i * RB_EXACT_WORDS);
    }
}
ExactKernels exact_kernels() {
    ExactKernels k;
    k.normalise = (const void*)k_exact_normalise;
    k.finalise = (const void*)k_exact_finalise;
    k.sum_test = (const void*)k_exact_sum_test;
    k.readout = (const void*)k_exact_readout;
    k.export_records = (const void*)k_exact_export;
    k.import_records = (const void*)k_exact_import;
    return k;
}
int bind_exact_accumulators(long long* acc, void* stream) {
    return (int)cudaMemcpyToSymbolAsync(rb_exact_acc, &acc, sizeof(acc), 0, cudaMemcpyHostToDevice, (cudaStream_t)stream);
}
} // namespace rb_det
