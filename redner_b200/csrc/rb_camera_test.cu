// Test hook rb_camera_test: the camera's rays, projections, lens model, pixel filter and their adjoints, one query per thread, through the
// functions the render kernels call (rb_camera_test.cuh).  Compiled with the default flags of build.py, so the hook rounds as the render
// kernels do.
#include <cuda_runtime.h>

#include <string>

#include "rb_camera_test.cuh"
#include "rb_scene.cuh"

__global__ void k_camera_test(DevCamera cam, int op, const double* in, int n, double* out, float* acc) {
    camera_test_one(cam, op, in, n, out, acc, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

extern "C" int rb_camera_test(const rb_scene* sc, int op, const double* in, int n, double* out, float* acc, void* stream_) {
#ifdef RB_REAL_DOUBLE
    rb_set_error("rb_camera_test: not available in the double-precision build");
    return 1;
#endif
    const char* err = nullptr;
    if (sc == nullptr) err = "null scene";
    else if (sc->incomplete) err = "the scene's last update failed";
    else if (op < RB_CAMTEST_CAMERA || op > RB_CAMTEST_FINISH) err = "unknown op";
    else if (n < 0) err = "negative number of queries";
    else if (n > 0 && (in == nullptr || out == nullptr)) err = "null buffer";
    else if (n > 0 && acc == nullptr && (op == RB_CAMTEST_D_RAY || op == RB_CAMTEST_D_PROJECT))
        err = "the adjoint ops need an accumulator";
    if (err != nullptr) {
        rb_set_error(std::string("rb_camera_test: ") + err);
        return 1;
    }
    if (n == 0) return 0;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(sc->device);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = 128;
    k_camera_test<<<(n + B - 1) / B, B, 0, stream>>>(sc->dev.cam, op, in, n, out, acc);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_camera_test: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}
