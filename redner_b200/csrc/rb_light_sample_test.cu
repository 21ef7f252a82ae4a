// Test hook rb_light_sample_test: the point-on-light sampler of emission sampling and its density, one sample or query per thread,
// through the functions of rb_path.cuh that the render kernels call (sample_light_point, light_point_pdf).  Compiled with the default
// flags of build.py, so the hook rounds as the render kernels do.
#include <cuda_runtime.h>

#include <string>

#include "rb_path.cuh"
#include "rb_scene.cuh"

__global__ void k_light_sample_test(DevScene sc, int l, const double* samples, int n, int* ints, double* doubles, const float* queries, int m,
                                    double* query_pdfs) {
    light_sample_test_one(sc, l, samples, n, ints, doubles, queries, m, query_pdfs, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

extern "C" int rb_light_sample_test(const rb_scene* sc, int light, const double* samples, int n, int* ints, double* doubles, const float* queries, int m,
                                    double* query_pdfs, void* stream_) {
    const char* err = nullptr;
    if (sc == nullptr) err = "null scene";
    else if (sc->incomplete) err = "the scene's last update failed";
    else if (light < 0 || light >= (int)sc->lights.size()) err = "light out of range";
    else if (n < 0 || m < 0) err = "negative number of samples or queries";
    else if ((n > 0 && (samples == nullptr || ints == nullptr || doubles == nullptr)) || (m > 0 && (queries == nullptr || query_pdfs == nullptr)))
        err = "null buffer";
    if (err != nullptr) {
        rb_set_error(std::string("rb_light_sample_test: ") + err);
        return 1;
    }
    if (n == 0 && m == 0) return 0;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(sc->device);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = 256, total = n > m ? n : m;
    k_light_sample_test<<<(total + B - 1) / B, B, 0, stream>>>(sc->dev, light, samples, n, ints, doubles, queries, m, query_pdfs);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_light_sample_test: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}
