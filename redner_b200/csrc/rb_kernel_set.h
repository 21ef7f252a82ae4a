// The render kernels that exist in both instantiations of rb_kernels_body.cuh, as host-side kernel pointers for
// cudaLaunchKernel: ::render_kernels() returns the general set (rb_kernels.cu), rb_lean::render_kernels() the feature-free
// set (rb_kernels_lean.cu).  Both sets take the same arguments: the lean translation unit declares the same DevScene /
// KernelArgs layouts inside namespace rb_lean, so the driver's structs are passed to either as they are.
#pragma once
struct RenderKernels {
    const void *forward, *bwd_trace, *bwd_sec_pick, *bwd_sec_shade, *bwd_sweep, *prim_keys, *primary_edge;
};
RenderKernels render_kernels();
namespace rb_lean {
RenderKernels render_kernels();
}
