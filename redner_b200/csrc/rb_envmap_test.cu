// Test hook rb_envmap_test: environment-map lookups, their adjoints, samples and pdfs, one query per thread, through the functions of
// rb_envmap.cuh that the render kernels call (envmap_eval, d_envmap_eval with its aggregated scatters, envmap_sample, envmap_pdf).
// Compiled with the default flags of build.py, so the hook rounds as the render kernels do.
#include <cuda_runtime.h>

#include <string>

#include "rb_envmap.cuh"
#include "rb_scene.cuh"
#include "rb_scene_host.hpp"

// queries: [n, 9] = dir, dir_dx, dir_dy.  values: [n, 3].  pdfs: [n] or NULL.  d_out: [n, 3] or NULL.  d_queries: [n, 9] or NULL.
// samples: [m, 2] doubles (sx, sy).  sample_dirs: [m, 3].
__global__ void k_envmap_test(DevEnvmap e, rb_texture d_values, float* d_w2e, const float* queries, int n, const float* d_out, float* values,
                              float* pdfs, float* d_queries, const double* samples, int m, float* sample_dirs) {
#ifndef RB_REAL_DOUBLE // (directions and adjoints are read and written in place as Real)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float* q = queries + 9 * (size_t)i;
        const V3 dir = mk3(q[0], q[1], q[2]);
        RayDiff rd = zero_raydiff();
        rd.dir_dx = mk3(q[3], q[4], q[5]);
        rd.dir_dy = mk3(q[6], q[7], q[8]);
        const V3 v = envmap_eval(e, dir, rd);
        values[3 * (size_t)i] = v.x;
        values[3 * (size_t)i + 1] = v.y;
        values[3 * (size_t)i + 2] = v.z;
        if (pdfs != nullptr) pdfs[i] = envmap_pdf(e, dir);
        if (d_out != nullptr) {
            const float* g = d_out + 3 * (size_t)i;
            V3 d_dir = zero3();
            RayDiff d_rd = zero_raydiff();
            d_envmap_eval(e, dir, rd, mk3(g[0], g[1], g[2]), d_values, d_w2e, d_dir, d_rd);
            if (d_queries != nullptr) {
                float* dq = d_queries + 9 * (size_t)i;
                const V3 o[3] = {d_dir, d_rd.dir_dx, d_rd.dir_dy};
                for (int k = 0; k < 3; k++) {
                    dq[3 * k] = o[k].x;
                    dq[3 * k + 1] = o[k].y;
                    dq[3 * k + 2] = o[k].z;
                }
            }
        }
    }
    if (i < m) {
        const V3 d = envmap_sample(e, samples[2 * (size_t)i], samples[2 * (size_t)i + 1]);
        sample_dirs[3 * (size_t)i] = d.x;
        sample_dirs[3 * (size_t)i + 1] = d.y;
        sample_dirs[3 * (size_t)i + 2] = d.z;
    }
#endif
}

static bool on_current_device(const void* p, int device) {
    cudaPointerAttributes a;
    if (p == nullptr || cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device;
}

// The map's layout (the emulator's hook checks the same): a 3-channel pyramid with positive level sizes, and a gradient pyramid of the same shape.
static const char* check_envmap_shape(const rb_envmap& env, const rb_texture* d_values) {
    const rb_texture& t = env.values;
    if (t.channels != 3) return "the map must have 3 channels";
    if (t.num_levels < 1 || t.num_levels > RB_MAX_MIP_LEVELS) return "num_levels must be in [1, RB_MAX_MIP_LEVELS]";
    for (int l = 0; l < t.num_levels; l++)
        if (t.width[l] < 1 || t.height[l] < 1) return "every level of the map needs a positive width and height";
    if (d_values != nullptr) {
        if (d_values->channels != t.channels || d_values->num_levels != t.num_levels) return "the gradient pyramid must have the map's levels and channels";
        for (int l = 0; l < t.num_levels; l++)
            if (d_values->width[l] != t.width[l] || d_values->height[l] != t.height[l]) return "the gradient pyramid must have the map's level sizes";
    }
    return nullptr;
}

extern "C" int rb_envmap_test(const rb_envmap* env, const rb_texture* d_values, float* d_w2e, const float* queries, int n, const float* d_out, float* values,
                              float* pdfs, float* d_queries, const double* samples, int m, float* sample_dirs, void* stream_) {
#ifdef RB_REAL_DOUBLE
    rb_set_error("rb_envmap_test: not available in the double-precision build");
    return 1;
#endif
    const char* err = nullptr;
    int device = 0;
    if (n < 0 || m < 0) err = "negative number of queries or samples";
    else if (env == nullptr) err = "null environment map";
    else if (d_out != nullptr && d_values == nullptr) err = "d_out needs a gradient pyramid";
    else if (cudaGetDevice(&device) != cudaSuccess) err = "no current device";
    if (err == nullptr) err = check_envmap_shape(*env, d_out != nullptr ? d_values : nullptr);
    if (err == nullptr) {
        const rb_texture& t = env->values;
        for (int l = 0; l < t.num_levels && err == nullptr; l++) {
            if (!on_current_device(t.texels[l], device)) err = "the map's texels must be memory of the current device";
            else if (d_out != nullptr && !on_current_device(d_values->texels[l], device)) err = "the gradient pyramid must be memory of the current device";
        }
        if (err == nullptr && !on_current_device(t.uv_scale, device)) err = "the map's uv_scale must be memory of the current device";
        if (err == nullptr && (!on_current_device(env->sample_cdf_ys, device) || !on_current_device(env->sample_cdf_xs, device)))
            err = "the sampling tables must be memory of the current device";
        if (err == nullptr && d_out != nullptr && d_values->uv_scale != nullptr && !on_current_device(d_values->uv_scale, device))
            err = "the gradient's uv_scale must be NULL or memory of the current device";
        if (err == nullptr && d_out != nullptr && d_w2e != nullptr && !on_current_device(d_w2e, device))
            err = "d_w2e must be NULL or memory of the current device";
    }
    if (err == nullptr && n > 0) {
        if (!on_current_device(queries, device) || !on_current_device(values, device) || (pdfs != nullptr && !on_current_device(pdfs, device)) ||
            (d_out != nullptr && !on_current_device(d_out, device)) || (d_queries != nullptr && !on_current_device(d_queries, device)))
            err = "queries, values, pdfs, d_out and d_queries must be memory of the current device";
    }
    if (err == nullptr && m > 0 && (!on_current_device(samples, device) || !on_current_device(sample_dirs, device)))
        err = "samples and sample_dirs must be memory of the current device";
    if (err != nullptr) {
        rb_set_error(std::string("rb_envmap_test: ") + err);
        return 1;
    }
    if (n == 0 && m == 0) return 0;
    DevScene ds{};
    host_setup_envmap(env, ds); // (the descriptor -> DevEnvmap step of rb_scene_create)
    cudaStream_t stream = (cudaStream_t)stream_;
    const rb_texture dv = d_out != nullptr ? *d_values : rb_texture{};
    const int B = 256, total = n > m ? n : m;
    k_envmap_test<<<(total + B - 1) / B, B, 0, stream>>>(ds.env, dv, d_out != nullptr ? d_w2e : nullptr, queries, n, d_out, values, pdfs,
                                                         d_out != nullptr ? d_queries : nullptr, samples, m, sample_dirs);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_envmap_test: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}
