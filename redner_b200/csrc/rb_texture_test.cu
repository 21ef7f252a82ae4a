// Test hook rb_texture_test: texture lookups and their adjoints, one query per thread, through the functions of rb_material.cuh
// that the render kernels call (tex_eval / tex_eval_channels forward, d_tex_eval with its warp-aggregated scatter backward).
// Compiled with the default flags of build.py, so the hook rounds as the render kernels do.
#include <cuda_runtime.h>

#include <string>

#include "rb_material.cuh"
#include "rb_scene.cuh"

// queries: [n, 6] = u, v, du/dx, du/dy, dv/dx, dv/dy.  values: [n, nch].  d_values: [n, nch] or NULL.  d_queries: [n, 6] or NULL.
__global__ void k_texture_test(rb_texture t, rb_texture dt, const float* queries, int n, const float* d_values, float* values, float* d_queries) {
#ifndef RB_REAL_DOUBLE // (values and adjoints are read and written in place as Real)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int nch = t.channels;
    const float* q = queries + 6 * (size_t)i;
    const V2 uv = mk2(q[0], q[1]), du_dxy = mk2(q[2], q[3]), dv_dxy = mk2(q[4], q[5]);
    float* out = values + (size_t)nch * i;
    if (nch == 1 || nch == 3) { // the BSDF's textures (mat_roughness, mat_diffuse, ...)
        const V3 v = tex_eval(t, nch, uv, du_dxy, dv_dxy);
        out[0] = v.x;
        if (nch == 3) {
            out[1] = v.y;
            out[2] = v.z;
        }
    } else { // generic textures
        tex_eval_channels(t, nch, uv, du_dxy, dv_dxy, out);
    }
    if (d_values == nullptr) return;
    V2 d_uv = zero2(), d_du = zero2(), d_dv = zero2();
    d_tex_eval(t, dt, nch, uv, du_dxy, dv_dxy, d_values + (size_t)nch * i, d_uv, d_du, d_dv);
    if (d_queries != nullptr) {
        float* dq = d_queries + 6 * (size_t)i;
        dq[0] = d_uv.x;
        dq[1] = d_uv.y;
        dq[2] = d_du.x;
        dq[3] = d_du.y;
        dq[4] = d_dv.x;
        dq[5] = d_dv.y;
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

// The layout checks of one texture: levels in range, every level's texels on the device, positive level sizes unless constant.
static const char* check_texture(const rb_texture& t, int device, bool need_uv_scale) {
    if (t.channels < 1) return "channels must be at least 1";
    if (t.num_levels < 1 || t.num_levels > RB_MAX_MIP_LEVELS) return "num_levels must be in [1, RB_MAX_MIP_LEVELS]";
    const bool constant = t.width[0] <= 0 && t.height[0] <= 0;
    for (int l = 0; l < t.num_levels; l++) {
        if (!on_current_device(t.texels[l], device)) return "texels must be memory of the current device";
        if (!constant && (t.width[l] < 1 || t.height[l] < 1)) return "every level of a texture that is not constant needs a positive width and height";
        if (constant) break; // (a constant texture reads texels[0] only)
    }
    if (need_uv_scale && !constant && !on_current_device(t.uv_scale, device)) return "uv_scale must be memory of the current device";
    return nullptr;
}

extern "C" int rb_texture_test(const rb_texture* tex, const rb_texture* d_tex, const float* queries, int n, const float* d_values, float* values,
                               float* d_queries, void* stream_) {
#ifdef RB_REAL_DOUBLE
    rb_set_error("rb_texture_test: not available in the double-precision build");
    return 1;
#endif
    const char* err = nullptr;
    int device = 0;
    if (n < 0) err = "negative number of queries";
    else if (tex == nullptr) err = "null texture";
    else if (d_values != nullptr && d_tex == nullptr) err = "d_values needs a gradient texture";
    else if (cudaGetDevice(&device) != cudaSuccess) err = "no current device";
    if (err == nullptr) err = check_texture(*tex, device, true);
    if (err == nullptr && d_values != nullptr) {
        err = check_texture(*d_tex, device, false);
        if (err == nullptr && (d_tex->num_levels != tex->num_levels || d_tex->channels != tex->channels))
            err = "the gradient texture must have the texture's levels and channels";
        if (err == nullptr && d_tex->uv_scale != nullptr && !on_current_device(d_tex->uv_scale, device))
            err = "the gradient's uv_scale must be NULL or memory of the current device";
    }
    if (err == nullptr && n > 0) {
        if (!on_current_device(queries, device) || !on_current_device(values, device) ||
            (d_values != nullptr && !on_current_device(d_values, device)) || (d_queries != nullptr && !on_current_device(d_queries, device)))
            err = "queries, values, d_values and d_queries must be memory of the current device";
    }
    if (err != nullptr) {
        rb_set_error(std::string("rb_texture_test: ") + err);
        return 1;
    }
    if (n == 0) return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    const rb_texture dt = d_values != nullptr ? *d_tex : rb_texture{};
    const int B = 256;
    k_texture_test<<<(n + B - 1) / B, B, 0, stream>>>(*tex, dt, queries, n, d_values, values, d_values != nullptr ? d_queries : nullptr);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        rb_set_error(std::string("rb_texture_test: ") + cudaGetErrorString(e));
        return 1;
    }
    return 0;
}
