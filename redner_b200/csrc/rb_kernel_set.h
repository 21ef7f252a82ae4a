// The render kernels that exist in every instantiation of rb_kernels_body.cuh, as host-side kernel pointers for
// cudaLaunchKernel: ::render_kernels() returns the general set (rb_kernels.cu), rb_lean::render_kernels() the feature-free
// set (rb_kernels_lean.cu), rb_diffuse::render_kernels() the feature-free set for diffuse-only materials (rb_kernels_diffuse.cu),
// rb_det::render_kernels() the general set with the deterministic gradient scatter (rb_kernels_det.cu).
// All sets take the same arguments: the other translation units declare the same DevScene / KernelArgs layouts inside their
// namespaces, so the driver's structs are passed to any of them as they are.
#pragma once
// prim_edge_project is null in the deterministic set, which projects every primary-edge sample itself.
struct RenderKernels {
    const void *forward, *bwd_trace, *bwd_sec_pick, *bwd_sec_shade, *bwd_sweep, *prim_keys, *primary_edge, *prim_edge_project;
};
RenderKernels render_kernels();
namespace rb_lean {
RenderKernels render_kernels();
}
namespace rb_diffuse {
RenderKernels render_kernels();
}
namespace rb_det {
RenderKernels render_kernels();
// Kernels of the exact accumulators (rb_exact.cuh), arguments as in rb_kernels_det.cu:
//   normalise  (long long* acc, long long n)                                           carries of accumulators [0, n)
//   finalise   (const long long* acc, long long n, const ExactRange* ranges, int num_ranges, double* cam_accum, int n_cam)
//   sum_test   (const float* values, const int* slots, int n, long long j0, long long count)
//   readout    (const long long* acc, int n, float* out_f32, double* out_f64)
//   export_records  (const long long* acc, long long n, const ExactRange* ranges, const long long* rec_first, int num_ranges, long long* records, int n_cam)
//   import_records  (long long* acc, long long n, const ExactRange* ranges, const long long* rec_first, int num_ranges, const long long* records, int n_cam)
struct ExactKernels {
    const void *normalise, *finalise, *sum_test, *readout, *export_records, *import_records;
};
ExactKernels exact_kernels();
// Points the deterministic scatter at the accumulator array `acc` (stream-ordered); returns a cudaError_t.
int bind_exact_accumulators(long long* acc, void* stream);
} // namespace rb_det
