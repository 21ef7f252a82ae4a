// Test hook rb_surface_test: ray/triangle solves, surface points, light-sample points and their adjoints, one query per thread, through the
// functions of rb_shape.cuh and the gradient scatters of rb_path.cuh that the render kernels call (rb_surface_test.cuh).  Compiled with the
// default flags of build.py, so the hook rounds as the render kernels do.
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "rb_scene.cuh"
#include "rb_surface_test.cuh"

__global__ void k_surface_test(DevScene sc, const rb_dshape* d_shapes, int op, const double* in, int n, double* out) {
    DevDScene ds;
    ds.shapes = d_shapes;
    surface_test_one(sc, d_shapes != nullptr ? &ds : nullptr, op, in, n, out, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

extern "C" int rb_surface_test(const rb_scene* sc, int op, const double* in, int n, double* out, const rb_dshape* d_shapes, void* stream_) {
#ifdef RB_REAL_DOUBLE
    rb_set_error("rb_surface_test: not available in the double-precision build");
    return 1;
#endif
    cudaStream_t stream = (cudaStream_t)stream_;
    std::vector<double> rows;
    const char* err = nullptr;
    if (sc != nullptr && n > 0 && in != nullptr && out != nullptr) {
        rows.resize((size_t)RB_SURFTEST_IN * n);
        if (cudaMemcpyAsync(rows.data(), in, rows.size() * sizeof(double), cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
            cudaStreamSynchronize(stream) != cudaSuccess) {
            rb_set_error(std::string("rb_surface_test: ") + cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
    } else if (n > 0 && out == nullptr) {
        err = "null buffer";
    }
    if (err == nullptr) err = surface_test_check(sc, op, n, in, rows.data());
    if (err != nullptr) {
        rb_set_error(std::string("rb_surface_test: ") + err);
        return 1;
    }
    if (n == 0) return 0;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(sc->device);
    rb_dshape* dsh = nullptr;
    cudaError_t e = cudaSuccess;
    if (d_shapes != nullptr) {
        const size_t bytes = sizeof(rb_dshape) * sc->shapes.size();
        e = cudaMallocAsync((void**)&dsh, bytes, stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dsh, d_shapes, bytes, cudaMemcpyHostToDevice, stream);
    }
    if (e == cudaSuccess) {
        const int B = 128;
        k_surface_test<<<(n + B - 1) / B, B, 0, stream>>>(sc->dev, dsh, op, in, n, out);
        e = cudaGetLastError();
    }
    if (dsh != nullptr) cudaFreeAsync(dsh, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_surface_test: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}
