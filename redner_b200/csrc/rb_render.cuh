// Per-sample render logic and the render set-up, shared by the CUDA kernels and their driver (rb_kernels.cu) and by the
// host-compiled debug emulator (tools/cpu_emu, development aid only).  One call == one (pixel, sample) or one primary-edge sample.
//   forward_sample         src/pathtracer.cpp:240-390 for one pixel-sample
//   backward_sample        src/pathtracer.cpp:392-762 (reverse sweep, first-hit adjoint)
//   primary_edge_sample    src/edge.cpp:385-625 + src/pathtracer.cpp:766-942 + src/edge.cpp:700-783
//   finish_camera          d_look_at_matrix / d_project tail, src/transform.h:29-71, src/camera.h:811-829
#pragma once
#include <cstdlib>

#include "rb_edge.cuh"
#include "rb_path.cuh"
#include "rb_secondary.cuh"

#define RB_MAX_ND 64                // floats per pixel of an image, at most
#define RB_MAX_BOUNDARY_BOUNCES 64  // bounces the boundary stage supports: one bit per depth in KernelArgs::vmask
// Phase barrier: the warps of a block enter each stage of a sample together, so one instruction-cache miss serves the
// whole block (measured 2.1x - 7.4x on the backward pass, DESIGN.md "instruction supply").  Every call site is reached
// by all threads of the block: the kernels iterate block-uniformly and pass an `act` flag instead of branching around.
#ifdef RB_CPU_EMU
#define RB_PHASE_SYNC()
#else
#define RB_PHASE_SYNC() __syncthreads()
#endif
struct BandCounters {
    unsigned n_paths, n_gather, n_hier, n_picked;
    unsigned long long total_vertices, total_hits; // statistics (mean path length, primary-hit fraction)
};
struct KernelArgs {
    RenderParams rp;
    int lanes_per_pixel; // L
    int owned_rows;      // rows of the viewport this device renders
    int zero_cull;       // backward: skip the samples of pixels whose adjoint is exactly zero (pixel_adjoint_is_zero)
    float* image;        // forward
    const float* d_image;
    float* screen_grad;
    DevDScene ds;
    // ---- backward band state (rb_kernels.cu): the adjoint pass walks the samples of the live pixels in bands of `band_n`
    const int* live_pixels;      // viewport pixels of the owned rows whose adjoint is not zero (all of them without zero_cull), ascending
    long long band_i0;           // first dense live sample index (index into live_pixels * spp + s) of the band
    int band_n;                  // samples in the band
    int rec_per_sample;          // max_bounces + 1 records per sample
    VertexRec* records;          // [band_n][rec_per_sample]
    V3* dpos;                    // [band_n][rec_per_sample] boundary terms (null without secondary edge sampling)
    int* nrec;                   // [band_n] vertices with an estimate, -1: primary ray missed
    ulonglong2* vmask;           // [band_n] per depth: (vertex takes part in the boundary stage, its sample uses the gather strategy)
    BandCounters* counters;      // list sizes of THIS band, written by k_bwd_trace / k_sec_offsets, read by the later kernels
    int* path_list;              // samples that hit something
    int* vert_list;              // (sample * rec_per_sample + depth): gather-strategy vertices from the front, hierarchy from the back
    int vert_cap;                // capacity of vert_list
    EdgePick* picks;             // [slot] edge chosen for each listed vertex
    unsigned *sec_keys, *sec_vals; // [slot] picked edge (or 0xffffffff) / vert_list entry
    unsigned *edge_hist, *edge_offs, *edge_cursor; // [num_edges] counting sort of the picks by edge
    unsigned* sec_order;         // [picks] slots in edge order
    double* edge_adj;            // [num_edges][4] primary-edge screen-space adjoints summed per edge (k_primary_edge without a lens), or null
};

RB_HD int rb_channel_width(int ch, int max_generic) { // floats of one channel, src/channels.cpp:42-113
    switch (ch) {
        case RB_CH_RADIANCE: case RB_CH_POSITION: case RB_CH_GEOMETRY_NORMAL: case RB_CH_SHADING_NORMAL: case RB_CH_DIFFUSE_REFLECTANCE:
        case RB_CH_SPECULAR_REFLECTANCE: case RB_CH_VERTEX_COLOR: return 3;
        case RB_CH_UV: case RB_CH_BARYCENTRIC: return 2;
        case RB_CH_GENERIC_TEXTURE: return max_generic;
        default: return 1;
    }
}

// Row partition over devices: round-robin stripes of `rows_per_stripe` viewport rows, stripe k rendered by part k % num_parts.
// j-th owned row -> viewport row
RB_HD int owned_row_to_row(const RenderParams& rp, int j) {
    int s = j / rp.rows_per_stripe, w = j % rp.rows_per_stripe;
    return (s * rp.num_parts + rp.part) * rp.rows_per_stripe + w;
}
inline int count_owned_rows(int H, int part, int num_parts, int rps) {
    int n = 0;
    for (int r = 0; r < H; r++)
        if ((r / rps) % num_parts == part) n++;
    return n;
}

// ---- render set-up shared by both rb_render drivers: the kernels' (rb_kernels.cu) and the host emulator's (tools/cpu_emu)
// Fills `ka` from the options, the scene's camera, generic-texture width and partition, and the image pointers.  Returns the
// error message, or null.  An empty viewport or zero samples passes: there is nothing to render then.
inline const char* setup_kernel_args(const rb_options& opt, const rb_camera& cam, int max_generic, int part, int num_parts, int rows_per_stripe,
                                     float* image, const float* d_image, const rb_dscene_desc* d_scene, float* screen_grad, KernelArgs& ka) {
    if (image == nullptr && d_image == nullptr) return "rb_render: neither rendered_image nor d_rendered_image given";
    if (d_image != nullptr && d_scene == nullptr) return "rb_render: d_rendered_image given without d_scene";
    if (opt.max_bounces < 0 || opt.num_samples < 0) return "rb_render: negative max_bounces / num_samples";
    memset(&ka, 0, sizeof(ka));
    RenderParams& rp = ka.rp;
    rp.seed = opt.seed;
    rp.spp = opt.num_samples;
    rp.max_bounces = opt.max_bounces;
    rp.sampler_type = opt.sampler_type;
    rp.sample_pixel_center = opt.sample_pixel_center;
    rp.num_channels = opt.num_channels;
    rp.max_generic = max_generic;
    rp.rad_dim = -1;
    if (opt.num_channels > RB_CH_COUNT) return "rb_render: too many channels";
    for (int i = 0; i < opt.num_channels; i++) {
        rp.channels[i] = opt.channels[i];
        if (opt.channels[i] < 0 || opt.channels[i] >= RB_CH_COUNT) return "rb_render: unknown channel";
        if (opt.channels[i] == RB_CH_RADIANCE) {
            if (rp.rad_dim != -1) return "Duplicated radiance channel"; // src/channels.cpp:24-26
            // the reference stores the CHANNEL INDEX and uses it as a float offset (src/channels.cpp:27,
            // src/path_contribution.cpp:125-129); identical whenever radiance is the first channel
            rp.rad_dim = i;
        }
    }
    rp.only_radiance = opt.num_channels == 1 && opt.channels[0] == RB_CH_RADIANCE ? 1 : 0;
    rp.nd = 0;
    rp.rad_off = -1;
    for (int i = 0; i < opt.num_channels; i++) {
        if (opt.channels[i] == RB_CH_RADIANCE) rp.rad_off = rp.nd;
        rp.nd += rb_channel_width(opt.channels[i], max_generic);
    }
    if (rp.nd > RB_MAX_ND) return "rb_render: more than 64 image dimensions requested";
    rp.part = part;
    rp.num_parts = num_parts;
    rp.rows_per_stripe = rows_per_stripe;
    rp.vp_w = cam.viewport_end[0] - cam.viewport_beg[0];
    rp.vp_h = cam.viewport_end[1] - cam.viewport_beg[1];
    int L = 1;
    while (L * 2 <= 32 && L * 2 <= rp.spp) L *= 2;
    ka.lanes_per_pixel = L;
    ka.owned_rows = count_owned_rows(rp.vp_h, part, num_parts, rows_per_stripe);
    ka.zero_cull = getenv("RB_NO_ZERO_CULL") == nullptr; // (test hook: trace every sample whatever its pixel's adjoint)
    ka.image = image;
    ka.d_image = d_image;
    ka.screen_grad = screen_grad;
    return nullptr;
}
// True iff all rp.nd floats of d_image at viewport pixel `pixel` compare equal to zero (-0 included; NaN and inf are not zero).
// Every term the backward pass computes for a sample of such a pixel is a product with one of these floats, and the samplers are
// pure functions of (pixel, sample, depth): its samples add exact zeros, and leaving them out changes no other sample.  All nd
// floats are tested, not only radiance's, so that G-buffer channels and the rad_dim offset (reads inside [0, nd)) are covered.
RB_HD bool pixel_adjoint_is_zero(const KernelArgs& ka, int pixel) {
    const float* p = ka.d_image + (size_t)ka.rp.nd * pixel;
    for (int k = 0; k < ka.rp.nd; k++)
        if (p[k] != 0.0f) return false;
    return true;
}
// rb_render's refusals under a pixel filter other than the 1-pixel box; returns the error message, or null.
inline const char* check_pixel_filter_options(const DevCamera& cam, const rb_options& opt, const float* screen_grad) {
    if (cam.lens_radius > 0 && screen_grad != nullptr) return "rb_render: a screen_gradient_image needs a camera without a lens (lens_radius 0)";
    if (cam.filter_type == RB_FILTER_BOX && cam.filter_width == 1.0f) return nullptr;
    if (opt.sample_pixel_center) return "rb_render: sample_pixel_center needs the 1-pixel box pixel filter (the scene's filter places samples around the centre)";
    if (screen_grad != nullptr) return "rb_render: a screen_gradient_image needs the 1-pixel box pixel filter";
    return nullptr;
}
// The boundary (secondary-edge) stage of the backward pass runs: it needs edges, a light and a radiance channel.
RB_HD bool boundary_stage_runs(const DevScene& sc, const RenderParams& rp) {
    return sc.use_secondary_edge && sc.num_edges > 0 && sc.num_lights > 0 && rp.rad_dim >= 0;
}
// The primary-edge pass of the backward pass runs.
RB_HD bool primary_edge_pass_runs(const DevScene& sc) { return sc.use_primary_edge && sc.num_edges > 0 && sc.prim_edge_cdf != nullptr; }
// The gradients of the lights' emission textures (rb_dscene_desc::light_emission) against the scene's textures (`emission`, host copies,
// one per area light).  Returns the error message, or null.
inline const char* check_light_emission_grads(const rb_dscene_desc& d_scene, const rb_texture* emission) {
    if (d_scene.light_emission == nullptr) return nullptr;
    for (int l = 0; l < d_scene.num_lights; l++) {
        const rb_texture &dt = d_scene.light_emission[l], &t = emission[l];
        if (dt.num_levels == 0) continue;
        bool same = dt.num_levels == t.num_levels && dt.channels == t.channels;
        for (int k = 0; same && k < t.num_levels; k++) same = dt.width[k] == t.width[k] && dt.height[k] == t.height[k] && dt.texels[k] != nullptr;
        if (!same) return "rb_render: a light's emission texture gradient (d_scene light_emission) needs the levels, sizes and channels of the light's emission texture";
    }
    return nullptr;
}
// Checks the gradient descriptor against the scene (`emission`: its lights' emission textures, host copies) and the options, and points
// the environment-map gradients of `ka.ds` at d_scene's.  Returns the error message, or null.  Each driver fills the shape, material,
// light and camera gradients itself.
inline const char* setup_backward(const rb_dscene_desc& d_scene, const DevScene& sc, const rb_texture* emission, KernelArgs& ka) {
    if (d_scene.num_shapes != sc.num_shapes || d_scene.num_materials != sc.num_materials || d_scene.num_lights != sc.num_lights - (sc.has_envmap ? 1 : 0))
        return "rb_render: d_scene does not match the scene (shape / material / light counts)";
    if (const char* err = check_light_emission_grads(d_scene, emission)) return err;
    if (boundary_stage_runs(sc, ka.rp) && ka.rp.max_bounces > RB_MAX_BOUNDARY_BOUNCES) return "rb_render: secondary edge sampling supports at most 64 bounces";
    memset(&ka.ds.env_values, 0, sizeof(rb_texture));
    ka.ds.env_w2e = nullptr;
    if (d_scene.envmap != nullptr) {
        ka.ds.env_values = d_scene.envmap->values;
        ka.ds.env_w2e = d_scene.envmap->world_to_env;
    } else if (sc.has_envmap) {
        return "rb_render: the scene has an environment map but d_scene has no envmap gradient buffers";
    }
    return nullptr;
}
// Writes one G-buffer pixel from the sums over its samples (`acc`) and the ids of the last sample that hit (`hit`: some sample
// did): channel sums are added to the pixel, id channels are overwritten.
RB_HD void write_gbuffer_pixel(const RenderParams& rp, const float* acc, const int* ids, bool hit, float* px) {
    const int nd = rp.nd < RB_MAX_ND ? rp.nd : RB_MAX_ND;
    int d = 0;
    for (int c = 0; c < rp.num_channels; c++) {
        int ch = rp.channels[c];
        int width = rb_channel_width(ch, rp.max_generic);
        if (ch == RB_CH_SHAPE_ID || ch == RB_CH_TRIANGLE_ID || ch == RB_CH_MATERIAL_ID) {
            if (hit && d < nd) px[d] = (float)ids[ch - RB_CH_SHAPE_ID];
        } else {
            for (int i = 0; i < width && d + i < nd; i++) px[d + i] += acc[d + i];
        }
        d += width;
    }
}

// Main-sampler dimensions per sample: camera (2, or 0 with sample_pixel_center) | lens (2, with a lens only) | 7 per bounce.
RB_HD unsigned long long main_draws_per_sample(const DevScene& sc, const RenderParams& rp) {
    return (unsigned long long)((rp.sample_pixel_center ? 0 : 2) + (RB_CAM_LENS(sc.cam) ? 2 : 0) + 7 * rp.max_bounces);
}
// Edge-sampler dimension layout per sample, in the order of the reference's next_* calls on `edge_sampler`
// (src/pathtracer.cpp:505, :630-641 inside the reverse depth loop, then :788, :871-882):
//   for depth = mb-1 .. 0:  secondary edge (4) + 7 per remaining bounce of its two sub-paths
//   primary edge (2) + lens (2, with a lens only) + 7 per bounce of its two sub-paths
RB_HD int secondary_edge_dim_base(const RenderParams& rp, int depth) {
    int off = 0;
    for (int d = rp.max_bounces - 1; d > depth; d--) off += 4 + 7 * (rp.max_bounces - 1 - d);
    return off;
}
// (not boundary_stage_runs: the reference reserves these dimensions whenever secondary edge sampling is on and a light exists)
RB_HD int primary_edge_dim_base(const DevScene& sc, const RenderParams& rp) {
    return (sc.use_secondary_edge && sc.num_lights > 0) ? secondary_edge_dim_base(rp, -1) : 0;
}
RB_HD unsigned long long edge_draws_per_sample(const DevScene& sc, const RenderParams& rp) {
    return (unsigned long long)(primary_edge_dim_base(sc, rp) + 2 + (RB_CAM_LENS(sc.cam) ? 2 : 0) + 7 * rp.max_bounces);
}

// Screen position of a pixel sample: consumes the first two sampler dimensions unless sample_pixel_center.  Under a pixel filter
// other than the 1-pixel box each of the two numbers becomes an offset from the pixel centre through the filter's inverse CDF
// (rb_render refuses sample_pixel_center there); the 1-pixel box keeps its own expression, which rounds differently.
RB_D void primary_sample_pos(const DevScene& sc, const RenderParams& rp, int px, int py, Sampler& smp, double& sx, double& sy) {
    double jx = 0.5, jy = 0.5;
    if (!rp.sample_pixel_center) {
        jx = smp.next();
        jy = smp.next();
    }
    if (!RB_PIXEL_BOX(sc.cam)) {
        jx = 0.5 + filter_offset(sc.cam, jx);
        jy = 0.5 + filter_offset(sc.cam, jy);
    }
    sx = (double(px + sc.cam.vp_beg[0]) + jx) / double(sc.cam.width);
    sy = (double(py + sc.cam.vp_beg[1]) + jy) / double(sc.cam.height);
}
// Lens sample of a camera with a lens (the two sampler dimensions after the camera's), a point of the unit disc; (0, 0) without a lens.
RB_D D2 primary_lens_sample(const DevScene& sc, Sampler& smp) {
    if (!RB_CAM_LENS(sc.cam)) return d2(0, 0);
    const double u1 = smp.next();
    const double u2 = smp.next();
    return concentric_disc(u1, u2);
}
// Camera sample -> primary ray (px, py are viewport-relative pixel coordinates), src/camera.cpp:8-43.
RB_D void primary_ray_for(const DevScene& sc, const RenderParams& rp, int px, int py, Sampler& smp, double& sx, double& sy, Ray& ray, RayDiff& rd,
                          D3* org_d = nullptr, D3* dir_d = nullptr) {
    primary_sample_pos(sc, rp, px, py, smp, sx, sy);
    const D2 lu = primary_lens_sample(sc, smp);
    cam_primary_ray(sc.cam, sx, sy, ray, rd, lu);
    if (org_d) cam_sample_primary(sc.cam, sx, sy, *org_d, *dir_d, lu);
}

// Radiance of one pixel sample, already multiplied by 1/spp.
// `sobol`: the Sobol rows of the main sampler (global memory, or the block's shared-memory copy when k_forward stages them)
RB_D V3 forward_sample(const DevScene& sc, const RenderParams& rp, int pixel, int px, int py, int s, const unsigned long long* sobol = nullptr) {
    const Real weight = Real(1) / Real(rp.spp);
    Sampler smp;
    smp.init(rp.sampler_type, rp.seed, pixel, (unsigned)s, sobol ? sobol : sc.sobol_matrices, RB_SOBOL_BITS, (unsigned long long)s * main_draws_per_sample(sc, rp));
    double sx, sy;
    Ray ray;
    RayDiff rd;
    D3 od, dd;
    primary_ray_for(sc, rp, px, py, smp, sx, sy, ray, rd, &od, &dd);
    Isect is = no_isect();
    V3 acc = zero3();
    if (ray_is_null(ray)) return acc; // fisheye sample outside the image disc
    if (closest_hit(sc, ray, is)) {
        RayDiff rd_after;
        SurfacePoint sp = make_surface_point(sc.shapes[is.shape_id], is.tri_id, ray, rd, rd_after);
        acc += weight * hit_emission(sc, is, sp, -ray.dir);
        acc += weight * trace_bounces<false>(sc, smp, ray, rd, is, mk3(1, 1, 1), Real(0), 0, rp.max_bounces, nullptr, 0, nullptr, &od, &dd);
    } else {
        acc += weight * miss_emission(sc, ray.dir, rd);
    }
    return acc;
}

// Values of every non-radiance, non-id channel at a first hit, at their float offsets in vals[0..nd) (unweighted;
// src/primary_contribution.cpp:36-253).  Radiance and id slots are left untouched.
RB_D void channel_values_at_hit(const DevScene& sc, const RenderParams& rp, const Isect& is, const SurfacePoint& sp, const Ray& ray, Real* vals) {
    const rb_shape& shape = sc.shapes[is.shape_id];
    const rb_material& mat = sc.materials[shape.material_id];
    int d = 0;
    for (int c = 0; c < rp.num_channels; c++) {
        switch (rp.channels[c]) {
            case RB_CH_RADIANCE: d += 3; break;
            case RB_CH_ALPHA: vals[d] = 1; d += 1; break;
            case RB_CH_DEPTH: vals[d] = length(sp.position - ray.org); d += 1; break;
            case RB_CH_POSITION: vals[d] = sp.position.x; vals[d + 1] = sp.position.y; vals[d + 2] = sp.position.z; d += 3; break;
            case RB_CH_GEOMETRY_NORMAL: vals[d] = sp.geom_normal.x; vals[d + 1] = sp.geom_normal.y; vals[d + 2] = sp.geom_normal.z; d += 3; break;
            case RB_CH_SHADING_NORMAL: {
                V3 n = sp.shading_frame.n;
                if (mat_has_normal_map(mat)) n = perturb_shading_frame(mat, sp).n;
                vals[d] = n.x; vals[d + 1] = n.y; vals[d + 2] = n.z;
                d += 3;
            } break;
            case RB_CH_UV: vals[d] = sp.uv.x; vals[d + 1] = sp.uv.y; d += 2; break;
            case RB_CH_BARYCENTRIC: vals[d] = sp.bary.x; vals[d + 1] = sp.bary.y; d += 2; break;
            case RB_CH_DIFFUSE_REFLECTANCE: {
                V3 r = RB_VERTEX_COLOR(mat) ? sp.color : mat_diffuse(mat, sp);
                vals[d] = r.x; vals[d + 1] = r.y; vals[d + 2] = r.z;
                d += 3;
            } break;
            case RB_CH_SPECULAR_REFLECTANCE: {
                V3 r = mat_specular(mat, sp);
                vals[d] = r.x; vals[d + 1] = r.y; vals[d + 2] = r.z;
                d += 3;
            } break;
            case RB_CH_ROUGHNESS: vals[d] = mat_roughness(mat, sp); d += 1; break;
            case RB_CH_GENERIC_TEXTURE: {
                if (mat.generic_texture.num_levels > 0) {
                    int n = mat.generic_texture.channels < RB_MAX_ND ? mat.generic_texture.channels : RB_MAX_ND;
                    tex_eval_channels(mat.generic_texture, n, sp.uv, sp.du_dxy, sp.dv_dxy, vals + d);
                }
                d += rp.max_generic;
            } break;
            case RB_CH_VERTEX_COLOR: vals[d] = sp.color.x; vals[d + 1] = sp.color.y; vals[d + 2] = sp.color.z; d += 3; break;
            default: d += 1; break; // ids
        }
    }
}
// Adjoint of channel_values_at_hit (src/primary_contribution.cpp:486-692): d_vals[0..nd) are the (already weighted)
// adjoints of the channel values; results go to the surface-point adjoint, the ray origin (depth) and the textures.
RB_D void d_channel_values_at_hit(const DevScene& sc, const DevDScene& ds, const RenderParams& rp, const Isect& is, const SurfacePoint& sp, const Ray& ray,
                                  const Real* d_vals, SurfacePoint& d_sp, V3& d_ray_org) {
    const rb_shape& shape = sc.shapes[is.shape_id];
    const rb_material& mat = sc.materials[shape.material_id];
    const rb_material& d_mat = ds.materials[shape.material_id];
    int d = 0;
    for (int c = 0; c < rp.num_channels; c++) {
        switch (rp.channels[c]) {
            case RB_CH_RADIANCE: d += 3; break;
            case RB_CH_DEPTH: {
                V3 diff = sp.position - ray.org;
                Real l = length(diff);
                if (l > 0) {
                    V3 g = diff * (d_vals[d] / l);
                    d_sp.position += g;
                    d_ray_org -= g;
                }
                d += 1;
            } break;
            case RB_CH_POSITION: d_sp.position += mk3(d_vals[d], d_vals[d + 1], d_vals[d + 2]); d += 3; break;
            case RB_CH_GEOMETRY_NORMAL: d_sp.geom_normal += mk3(d_vals[d], d_vals[d + 1], d_vals[d + 2]); d += 3; break;
            // (the reference sends this adjoint to the unperturbed shading normal even under a normal map, :551-566)
            case RB_CH_SHADING_NORMAL: d_sp.shading_frame.n += mk3(d_vals[d], d_vals[d + 1], d_vals[d + 2]); d += 3; break;
            case RB_CH_UV: d_sp.uv += mk2(d_vals[d], d_vals[d + 1]); d += 2; break;
            case RB_CH_BARYCENTRIC: d_sp.bary += mk2(d_vals[d], d_vals[d + 1]); d += 2; break;
            case RB_CH_DIFFUSE_REFLECTANCE:
                if (RB_VERTEX_COLOR(mat)) d_sp.color += mk3(d_vals[d], d_vals[d + 1], d_vals[d + 2]);
                else d_tex_eval(mat.diffuse_reflectance, d_mat.diffuse_reflectance, 3, sp.uv, sp.du_dxy, sp.dv_dxy, d_vals + d, d_sp.uv, d_sp.du_dxy, d_sp.dv_dxy);
                d += 3;
                break;
            case RB_CH_SPECULAR_REFLECTANCE:
                d_tex_eval(mat.specular_reflectance, d_mat.specular_reflectance, 3, sp.uv, sp.du_dxy, sp.dv_dxy, d_vals + d, d_sp.uv, d_sp.du_dxy, d_sp.dv_dxy);
                d += 3;
                break;
            case RB_CH_ROUGHNESS:
                d_tex_eval(mat.roughness, d_mat.roughness, 1, sp.uv, sp.du_dxy, sp.dv_dxy, d_vals + d, d_sp.uv, d_sp.du_dxy, d_sp.dv_dxy);
                d += 1;
                break;
            case RB_CH_GENERIC_TEXTURE:
                if (mat.generic_texture.num_levels > 0 && d_mat.generic_texture.num_levels > 0) {
                    int n = mat.generic_texture.channels < RB_MAX_ND ? mat.generic_texture.channels : RB_MAX_ND;
                    d_tex_eval(mat.generic_texture, d_mat.generic_texture, n, sp.uv, sp.du_dxy, sp.dv_dxy, d_vals + d, d_sp.uv, d_sp.du_dxy, d_sp.dv_dxy);
                }
                d += rp.max_generic;
                break;
            case RB_CH_VERTEX_COLOR: d_sp.color += mk3(d_vals[d], d_vals[d + 1], d_vals[d + 2]); d += 3; break;
            default: d += 1; break; // alpha and ids: nothing to propagate
        }
    }
}
// G-buffer variant of forward_sample: accumulates every requested channel of the first hit into out[0..nd)
// plus the path-traced radiance.  Id channels (shape / triangle / material) are assigned, not averaged ("the last
// sample wins" in the reference); they are returned in ids[] and resolved by the kernel.
RB_D bool forward_sample_channels(const DevScene& sc, const RenderParams& rp, int pixel, int px, int py, int s, float* out, int* ids) {
    const Real weight = Real(1) / Real(rp.spp);
    Sampler smp;
    smp.init(rp.sampler_type, rp.seed, pixel, (unsigned)s, sc.sobol_matrices, RB_SOBOL_BITS, (unsigned long long)s * main_draws_per_sample(sc, rp));
    double sx, sy;
    Ray ray;
    RayDiff rd;
    D3 od, dd;
    primary_ray_for(sc, rp, px, py, smp, sx, sy, ray, rd, &od, &dd);
    Isect is = no_isect();
    if (ray_is_null(ray)) return false;
    if (!closest_hit(sc, ray, is)) {
        if (rp.rad_off >= 0) {
            V3 L = weight * miss_emission(sc, ray.dir, rd);
            out[rp.rad_off] += (float)L.x; out[rp.rad_off + 1] += (float)L.y; out[rp.rad_off + 2] += (float)L.z;
        }
        return false;
    }
    RayDiff rd_after;
    const rb_shape& shape = sc.shapes[is.shape_id];
    SurfacePoint sp = make_surface_point(shape, is.tri_id, ray, rd, rd_after);
    Real vals[RB_MAX_ND];
    for (int i = 0; i < rp.nd; i++) vals[i] = 0;
    channel_values_at_hit(sc, rp, is, sp, ray, vals);
    int d = 0;
    for (int c = 0; c < rp.num_channels; c++) {
        int w = rb_channel_width(rp.channels[c], rp.max_generic);
        if (rp.channels[c] == RB_CH_RADIANCE) {
            V3 L = hit_emission(sc, is, sp, -ray.dir);
            out[d] += (float)(weight * L.x); out[d + 1] += (float)(weight * L.y); out[d + 2] += (float)(weight * L.z);
        } else if (rp.channels[c] == RB_CH_SHAPE_ID) {
            ids[0] = is.shape_id;
        } else if (rp.channels[c] == RB_CH_TRIANGLE_ID) {
            ids[1] = is.tri_id;
        } else if (rp.channels[c] == RB_CH_MATERIAL_ID) {
            ids[2] = shape.material_id;
        } else {
            for (int i = 0; i < w; i++) out[d + i] += (float)(vals[d + i] * weight);
        }
        d += w;
    }
    if (rp.rad_dim >= 0) {
        V3 Lb = weight * trace_bounces<false>(sc, smp, ray, rd, is, mk3(1, 1, 1), Real(0), 0, rp.max_bounces, nullptr, 0, nullptr, &od, &dd);
        // path contributions land at float offset `rad_dim` == the channel INDEX of radiance, like the reference
        // (src/channels.cpp:27, src/path_contribution.cpp:125-129)
        out[rp.rad_dim] += (float)Lb.x; out[rp.rad_dim + 1] += (float)Lb.y; out[rp.rad_dim + 2] += (float)Lb.z;
    }
    return true;
}

// ---- adjoint of one pixel sample, in three stages (src/pathtracer.cpp:392-762) ----
// The stages run as three kernels over compacted work lists (rb_kernels.cu); records travel through HBM:
//   bwd_trace      replays the primal path and writes one VertexRec per vertex             (k_bwd_trace)
//   bwd_secondary  boundary term of one path vertex -> d(position) of that vertex          (k_bwd_secondary)
//   bwd_sweep      reverse sweep over the vertices, first-hit and camera adjoints          (k_bwd_sweep)
// A fused megakernel of the three is instruction-fetch bound: 0.6 - 1.6 MB of SASS walked once per sample.
// Returns the number of vertices at which a radiance estimate was formed (-1: the primary ray missed).  Writes
// recs[0 .. nrec] (the last one is the terminal vertex), `stride` records apart.
RB_D int bwd_trace(const DevScene& sc, const RenderParams& rp, int pixel, int px, int py, int s, VertexRec* recs, int stride, bool act = true) {
    Sampler smp;
    double sx, sy;
    Ray ray;
    RayDiff rd;
    D3 od, dd;
    Isect is = no_isect();
    RB_PHASE_SYNC();
    if (act) {
        smp.init(rp.sampler_type, rp.seed, pixel, (unsigned)s, sc.sobol_matrices, RB_SOBOL_BITS, (unsigned long long)s * main_draws_per_sample(sc, rp));
        primary_ray_for(sc, rp, px, py, smp, sx, sy, ray, rd, &od, &dd);
        bool null_ray = ray_is_null(ray);
        act = !null_ray && closest_hit(sc, ray, is);
        if (!act && !null_ray) is.shape_id = -2; // "traced and missed" (as opposed to an idle lane or a null ray)
    }
    RB_PHASE_SYNC();
    if (!act) {
        // a primary ray that leaves the scene still has an adjoint when it sees the environment map
        if (is.shape_id == -2 && RB_ENVMAP(sc) && sc.env.directly_visible && rp.rad_off >= 0) {
            VertexRec& r = recs[0];
            r.ray = ray;
            r.rd_in = rd;
            r.isect = no_isect();
            r.thr = mk3(1, 1, 1);
            r.min_rough = 0;
            return 0;
        }
        return -1;
    }
    int nrec = 0;
    // (without a radiance channel only the first hit matters: the terminal record alone)
    trace_bounces<true>(sc, smp, ray, rd, is, mk3(1, 1, 1), Real(0), 0, rp.rad_dim >= 0 ? rp.max_bounces : 0, recs, stride, &nrec, &od, &dd);
    return nrec;
}
// Boundary (visibility) term at vertex `depth` of the path of (pixel, s), src/pathtracer.cpp:500-707, in two steps (see
// rb_secondary.cuh).
#ifdef RB_EMU_REF_STREAMS
// Host emulator only: the reference indexes the boundary-sample stream of a vertex by the RANK of its pixel in the compacted
// active list of that depth (src/pathtracer.cpp:504-505).  A sequential emulator can know that rank (tools/cpu_emu fills
// this table per sample), which makes the boundary terms comparable sample by sample; kernels cannot.
static const int* rb_emu_rank = nullptr; // rank of the current (pixel, sample) at each depth
#endif
RB_D Sampler bwd_edge_sampler(const DevScene& sc, const RenderParams& rp, int pixel, int s, int depth, int consumed) {
    Sampler es;
#ifdef RB_EMU_REF_STREAMS
    if (rb_emu_rank != nullptr) pixel = rb_emu_rank[depth];
#endif
    es.init(rp.sampler_type, rp.seed + 131071ULL, pixel, (unsigned)s, sc.sobol_matrices, RB_SOBOL_BITS, (unsigned long long)s * edge_draws_per_sample(sc, rp));
    es.skip(secondary_edge_dim_base(rp, depth) + consumed);
    return es;
}
RB_D bool bwd_secondary_pick(const DevScene& sc, const KernelArgs& ka, int pixel, int s, int depth, const VertexRec& cur, EdgePick& pk) {
    Sampler es = bwd_edge_sampler(sc, ka.rp, pixel, s, depth, 0);
    return secondary_edge_pick(sc, cur, es, pk);
}
// Returns d(position of the vertex).
RB_D V3 bwd_secondary_shade(const DevScene& sc, const KernelArgs& ka, int pixel, int s, int depth, const VertexRec& cur, const EdgePick& pk) {
    const RenderParams& rp = ka.rp;
    V3 d_position = zero3();
    const float* dpx = ka.d_image + (size_t)rp.nd * pixel + (rp.rad_dim >= 0 ? rp.rad_dim : 0);
    secondary_edge_shade(sc, ka.ds, rp, cur, depth, bwd_edge_sampler(sc, rp, pixel, s, depth, 4), mk3(dpx[0], dpx[1], dpx[2]), pk, d_position);
    return d_position;
}
RB_D V3 bwd_secondary(const DevScene& sc, const KernelArgs& ka, int pixel, int s, int depth, const VertexRec& cur) {
    EdgePick pk;
    if (!bwd_secondary_pick(sc, ka, pixel, s, depth, cur, pk)) return zero3();
    return bwd_secondary_shade(sc, ka, pixel, s, depth, cur, pk);
}
// Reverse sweep (src/pathtracer.cpp:431-714) + first-hit and camera adjoints.  `dpos` (may be null) holds the
// boundary terms of the vertices, laid out like `recs`.
RB_D void bwd_sweep(const DevScene& sc, const KernelArgs& ka, int pixel, int px, int py, int s, const VertexRec* recs, int stride, int nrec,
                    const V3* dpos, CamAcc& cam_acc, bool act = true) {
    const RenderParams& rp = ka.rp;
    const DevDScene& ds = ka.ds;
    const Real weight = Real(1) / Real(rp.spp);
    const float* dpx_all = ka.d_image + (size_t)rp.nd * pixel;
    const float* dpx = dpx_all + (rp.rad_dim >= 0 ? rp.rad_dim : 0);
    V3 d_contrib = (act && rp.rad_dim >= 0) ? weight * mk3(dpx[0], dpx[1], dpx[2]) : zero3();
    // first-hit emission sits at the channel's true offset (differs from rad_dim only when radiance is not the first channel)
    const float* dpe = dpx_all + (rp.rad_off >= 0 ? rp.rad_off : 0);
    V3 d_emission = (act && rp.rad_off >= 0) ? weight * mk3(dpe[0], dpe[1], dpe[2]) : zero3();
    VertexAdjoint adj = zero_vertex_adjoint();
    for (int d = rp.max_bounces - 1; d >= 0; d--) { // block-uniform trip count (phase barrier inside)
        RB_PHASE_SYNC();
        if (act && d < nrec) {
            VertexRec cur = recs[(size_t)d * stride];
            VertexRec nxt = recs[(size_t)(d + 1) * stride];
            adj = d_vertex(sc, ds, cur, &nxt, d_contrib, adj);
            if (dpos) adj.d_point.position += dpos[(size_t)d * stride];
        }
    }
    RB_PHASE_SYNC();
    if (!act) return;
    const Ray ray = recs[0].ray;
    const RayDiff rd = recs[0].rd_in;
    const Isect is = recs[0].isect;
    DRay d_ray = adj.d_ray;
    RayDiff d_prd = zero_raydiff();
    if (is.valid()) {
        // first vertex: emission adjoint (src/primary_contribution.cpp:449-466) ...
        RayDiff rd_after;
        SurfacePoint sp = make_surface_point(sc.shapes[is.shape_id], is.tri_id, ray, rd, rd_after);
        {
            const rb_shape& shape = sc.shapes[is.shape_id];
            V3 wi = -ray.dir;
            if (shape.light_id >= 0 && RB_LIGHT_TEX(light_emission(sc, shape.light_id))) {
                // An emission texture: under the forward's condition (the untextured branch below keeps the reference's gate), into the
                // intensity, the texture, and through d(uv) and the footprint into the hit (DESIGN.md "Emission textures").
                const DevLight& light = sc.lights[shape.light_id];
                if (light.directly_visible && (light.two_sided || dot(wi, sp.shading_frame.n) > 0)) {
                    const V3 I = mk3(light.intensity[0], light.intensity[1], light.intensity[2]);
                    agg_add3(ds.light_intensity[shape.light_id], d_emission * light_tex_eval(light_emission(sc, shape.light_id), sp.uv, sp.du_dxy, sp.dv_dxy));
                    V2 d_du = zero2(), d_dv = zero2();
                    adj.d_point.uv += d_light_tex_eval(sc, ds, shape.light_id, sp.uv, sp.du_dxy, sp.dv_dxy, d_emission * I, d_du, d_dv);
                    adj.d_point.du_dxy += d_du;
                    adj.d_point.dv_dxy += d_dv;
                }
            } else if (shape.light_id >= 0 && dot(wi, sp.shading_frame.n) > 0) {
                const DevLight& light = sc.lights[shape.light_id];
                if (light.directly_visible) agg_add3(ds.light_intensity[shape.light_id], d_emission);
            }
        }
        // G-buffer channels of the first hit (src/primary_contribution.cpp:486-692)
        if (!RB_ONLY_RADIANCE(rp)) {
            Real d_vals[RB_MAX_ND];
            for (int i = 0; i < rp.nd; i++) d_vals[i] = weight * dpx_all[i];
            d_channel_values_at_hit(sc, ds, rp, is, sp, ray, d_vals, adj.d_point, d_ray.org);
        }
        // ... and the hit itself back to the mesh and the camera (src/primary_intersection.cpp:5-130)
        V3 d_vp[3] = {zero3(), zero3(), zero3()}, d_vn[3] = {zero3(), zero3(), zero3()}, d_vc[3] = {zero3(), zero3(), zero3()};
        V2 d_vuv[3] = {zero2(), zero2(), zero2()};
        d_make_surface_point(sc.shapes[is.shape_id], is.tri_id, ray, rd, adj.d_point, zero_raydiff(), d_ray, d_prd, d_vp, d_vn, d_vuv, d_vc);
        scatter_vertex_grads(sc, ds, is, d_vp, d_vn, d_vuv, d_vc);
    } else {
        // the primary ray left the scene: environment map seen directly (src/primary_contribution.cpp:469-483)
        // Only the direction adjoint reaches the camera: the reference feeds the footprint adjoint of a primary ray to the
        // camera through d_intersect_shape, i.e. for hits only (src/primary_intersection.cpp:9-16,:30-41).
        RayDiff d_footprint = zero_raydiff();
        d_envmap_eval(sc.env, ray.dir, rd, d_emission, ds.env_values, ds.env_w2e, d_ray.dir, d_footprint);
    }
    const Real delta = Real(1e-3);
    DRay d_ray_dx, d_ray_dy;
    d_cam_primary_ray_diff(sc.cam, d_prd, d_ray, d_ray_dx, d_ray_dy);
    Sampler smp;
    smp.init(rp.sampler_type, rp.seed, pixel, (unsigned)s, sc.sobol_matrices, RB_SOBOL_BITS, (unsigned long long)s * main_draws_per_sample(sc, rp));
    double sx, sy;
    primary_sample_pos(sc, rp, px, py, smp, sx, sy);
    const D2 lu = primary_lens_sample(sc, smp);
    V2 d_screen = zero2();
    V2* d_screen_ptr = ka.screen_grad ? &d_screen : nullptr;
#pragma unroll 1
    for (int k = 0; k < 3; k++) { // centre ray and its two offset rays; rolled to keep one copy of the camera adjoint
        DRay dr = k == 0 ? d_ray : k == 1 ? d_ray_dx : d_ray_dy;
        d_cam_sample_primary(sc.cam, (Real)sx + (k == 1 ? delta : Real(0)), (Real)sy + (k == 2 ? delta : Real(0)), dr, cam_acc, d_screen_ptr, lu);
    }
    if (ka.screen_grad) {
        rb_red_add(&ka.screen_grad[2 * (size_t)pixel + 0], (float)d_screen.x);
        rb_red_add(&ka.screen_grad[2 * (size_t)pixel + 1], (float)d_screen.y);
    }
}
// The three stages back to back for ONE sample: used by the host-compiled debug emulator (tools/cpu_emu) only.
RB_D int backward_sample(const DevScene& sc, const KernelArgs& ka, int pixel, int px, int py, int s, VertexRec* recs, CamAcc& cam_acc) {
    const RenderParams& rp = ka.rp;
    if (ka.zero_cull && pixel_adjoint_is_zero(ka, pixel)) return -1; // (like the bands, which hold the samples of live pixels only)
    int nrec = bwd_trace(sc, rp, pixel, px, py, s, recs, 1);
    if (nrec < 0) return -1;
    V3 dpos[RB_MAX_BOUNDARY_BOUNCES]; // (setup_backward rejects deeper paths when the stage runs)
    const bool sec = boundary_stage_runs(sc, rp);
    for (int d = 0; sec && d < nrec; d++) dpos[d] = bwd_secondary(sc, ka, pixel, s, d, recs[d]);
    bwd_sweep(sc, ka, pixel, px, py, s, recs, 1, nrec, sec ? dpos : nullptr, cam_acc);
    return nrec;
}

// ---- primary edges ----
// Projection of an edge in double (the +-1e-6 offsets across the edge need more than fp32 screen coordinates).
RB_HD D3 w2c_point(const DevCamera& cam, D3 p) {
    const double* W = cam.w2c;
    double x = W[0] * p.x + W[1] * p.y + W[2] * p.z + W[3];
    double y = W[4] * p.x + W[5] * p.y + W[6] * p.z + W[7];
    double z = W[8] * p.x + W[9] * p.y + W[10] * p.z + W[11];
    double w = W[12] * p.x + W[13] * p.y + W[14] * p.z + W[15];
    double iw = 1.0 / w;
    return d3(x * iw, y * iw, z * iw);
}
RB_HD D2 cam_to_screen_sphere_d(const DevCamera& cam, D3 p) { // fisheye / panorama, src/camera.h:533-553
    const double pi = 3.14159265358979323846;
    D3 d = d3_normalize(p);
    D2 r;
    if (cam.type == RB_CAMERA_FISHEYE) {
        double phi = atan2(d.y, d.x), rr = acos(d.z) * 2.0 / pi;
        r.x = 0.5 * (-rr * cos(phi) + 1.0);
        r.y = 0.5 * (-rr * sin(phi) + 1.0);
    } else {
        r.x = atan2(d.z, d.x) / (2 * pi);
        r.y = acos(d.y) / pi;
    }
    return r;
}
RB_HD D2 cam_to_screen_undistorted_d(const DevCamera& cam, D3 p);
RB_HD D2 cam_to_screen_d(const DevCamera& cam, D3 p) { return cam_distort(cam, cam_to_screen_undistorted_d(cam, p)); } // (cam_distort: identity without a lens model)
RB_HD D2 cam_to_screen_undistorted_d(const DevCamera& cam, D3 p) {
    const double* K = cam.intr;
    double aspect = double(cam.width) / double(cam.height);
    double ix = K[0] * p.x + K[1] * p.y + K[2] * p.z, iy = K[3] * p.x + K[4] * p.y + K[5] * p.z, iz = K[6] * p.x + K[7] * p.y + K[8] * p.z;
    D2 r;
    if (RB_CAM_GENERAL(cam) && (cam.type == RB_CAMERA_FISHEYE || cam.type == RB_CAMERA_PANORAMA)) return cam_to_screen_sphere_d(cam, p);
    if (!RB_CAM_GENERAL(cam) || cam.type == RB_CAMERA_PERSPECTIVE) {
        r.x = (ix / iz + 1.0) * 0.5;
        r.y = (-(iy / iz) * aspect + 1.0) * 0.5;
    } else {
        r.x = (ix + 1.0) * 0.5;
        r.y = (-iy * aspect + 1.0) * 0.5;
    }
    return r;
}
RB_HD bool cam_project_d(const DevCamera& cam, D3 p0, D3 p1, D2& q0, D2& q1) {
    D3 a = w2c_point(cam, p0), b = w2c_point(cam, p1);
    double cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return false;
    if (a.z < cn) {
        D3 dir = d3(a.x - b.x, a.y - b.y, a.z - b.z);
        double t = -(b.z - cn) / dir.z;
        a = d3(b.x + t * dir.x, b.y + t * dir.y, b.z + t * dir.z);
    } else if (b.z < cn) {
        D3 dir = d3(b.x - a.x, b.y - a.y, b.z - a.z);
        double t = -(a.z - cn) / dir.z;
        b = d3(a.x + t * dir.x, a.y + t * dir.y, a.z + t * dir.z);
    }
    q0 = cam_to_screen_d(cam, a);
    q1 = cam_to_screen_d(cam, b);
    return true;
}

// Screen position -> direction in camera space and its adjoint, fisheye / panorama only (src/camera.h:858-890, :962-1037;
// the panorama adjoint carries the reference's slips: sin(phi) where sin(theta) belongs, and the fisheye's factor 2).
RB_HD D3 cam_screen_to_camera_d(const DevCamera& cam, D2 p_) {
    const double pi = 3.14159265358979323846;
    const D2 p = cam_inverse_distort(cam, p_);
    if (cam.type == RB_CAMERA_PERSPECTIVE || cam.type == RB_CAMERA_ORTHOGRAPHIC) { // src/camera.h:839-862
        const double* I = cam.intr_inv;
        double aspect = double(cam.width) / double(cam.height);
        double px = (p.x - 0.5) * 2.0, py = (p.y - 0.5) * (-2.0) / aspect, pz = 1.0;
        D3 d = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
        return cam.type == RB_CAMERA_PERSPECTIVE ? d3(d.x / d.z, d.y / d.z, 1.0) : d3(d.x, d.y, 1.0);
    }
    if (cam.type == RB_CAMERA_FISHEYE) {
        double x = 2.0 * (p.x - 0.5), y = 2.0 * (p.y - 0.5);
        double phi = atan2(y, x), theta = sqrt(x * x + y * y) * pi / 2.0;
        return d3(-cos(phi) * sin(theta), -sin(phi) * sin(theta), cos(theta));
    }
    double theta = pi * p.y, phi = 2 * pi * p.x;
    return d3(cos(phi) * sin(theta), cos(theta), sin(phi) * sin(theta));
}
RB_HD D2 d_cam_screen_to_camera_undistorted_d(const DevCamera& cam, D2 p, D3 d_dir);
RB_HD D2 d_cam_screen_to_camera_d(const DevCamera& cam, D2 p_, D3 d_dir) {
    D2 g = d_cam_screen_to_camera_undistorted_d(cam, cam_inverse_distort(cam, p_), d_dir);
    D2 d_pos = d2(0, 0);
    d_cam_inverse_distort(cam, p_, g, nullptr, d_pos); // (no parameter gradient on this path, src/camera.h:951-960)
    return d_pos;
}
RB_HD D2 d_cam_screen_to_camera_undistorted_d(const DevCamera& cam, D2 p, D3 d_dir) {
    const double pi = 3.14159265358979323846;
    D2 r;
    if (cam.type == RB_CAMERA_PERSPECTIVE || cam.type == RB_CAMERA_ORTHOGRAPHIC) { // src/camera.h:908-960
        const double* I = cam.intr_inv;
        double aspect = double(cam.width) / double(cam.height);
        double px = (p.x - 0.5) * 2.0, py = (p.y - 0.5) * (-2.0) / aspect, pz = 1.0;
        D3 d = d3(I[0] * px + I[1] * py + I[2] * pz, I[3] * px + I[4] * py + I[5] * pz, I[6] * px + I[7] * py + I[8] * pz);
        D3 dd = cam.type == RB_CAMERA_PERSPECTIVE ? d3(d_dir.x / d.z, d_dir.y / d.z, -(d_dir.x * (d.x / d.z) / d.z + d_dir.y * (d.y / d.z) / d.z))
                                                  : d3(d_dir.x, d_dir.y, 0.0);
        double d_px = I[0] * dd.x + I[3] * dd.y + I[6] * dd.z, d_py = I[1] * dd.x + I[4] * dd.y + I[7] * dd.z;
        r.x = d_px * 2;
        r.y = d_py * (-2) / aspect;
        return r;
    }
    if (cam.type == RB_CAMERA_FISHEYE) {
        double x = 2.0 * (p.x - 0.5), y = 2.0 * (p.y - 0.5);
        double rr = sqrt(x * x + y * y), phi = atan2(y, x), theta = rr * pi / 2.0;
        double sp = sin(phi), cp = cos(phi), st = sin(theta), ct = cos(theta);
        double d_cp = -d_dir.x * st, d_sp = -d_dir.y * st, d_st = -(d_dir.x * cp + d_dir.y * sp), d_ct = d_dir.z;
        double d_phi = d_sp * cp - d_cp * sp, d_theta = d_st * ct - d_ct * st;
        double d_r = d_theta * (pi / 2.0);
        // at the centre phi is atan2(0, 0) = 0 and d_phi / rr tends to -(pi / 2) d_dir.y: the limit of the two quotients below
        double d_x = rr > 0 ? d_phi * (-y / (x * x + y * y)) + d_r * (x / rr) : d_r;
        double d_y = rr > 0 ? d_phi * (x / (x * x + y * y)) + d_r * (y / rr) : -(pi / 2.0) * d_dir.y;
        r.x = d_x * 2;
        r.y = d_y * 2;
        return r;
    }
    double theta = pi * p.y, phi = 2 * pi * p.x;
    double sp = sin(phi), cp = cos(phi), st = sin(theta), ct = cos(theta);
    double d_cp = d_dir.x * st, d_sp = d_dir.z * sp, d_st = d_dir.x * cp + d_dir.z * sp, d_ct = d_dir.y;
    double d_phi = d_sp * cp - d_cp * sp, d_theta = d_st * ct - d_ct * st;
    r.x = d_phi * (2 * pi) * 2;
    r.y = d_theta * pi * 2;
    return r;
}
RB_HD D3 d3_cross(D3 a, D3 b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
RB_HD bool cam_is_linear(const DevCamera& cam) { return !RB_CAM_GENERAL(cam) || ((cam.type == RB_CAMERA_PERSPECTIVE || cam.type == RB_CAMERA_ORTHOGRAPHIC) && !cam.has_distortion); }

// One primary-edge sample: edge sample index i (seeds the stream like a pixel index), spp sample s.
// Edge and point on it chosen by primary-edge sample (i, s); false if the sample contributes nothing (edge behind the
// camera, zero probability, point off screen).  `smp` is left positioned at the first light/bsdf dimension.
struct PrimEdgePick {
    int edge_id;
    double pmf, e_t;
    D2 q0, q1, ept;
    D2 upper, lower; // screen positions of the two rays on either side of the edge
    double jacobian; // 1 for linear projections (there the edge length and the gradient of the edge equation cancel)
#ifndef RB_LEAN
    D2 lu; // lens sample (unit disc) of a camera with a lens: the edge is projected from it, and both rays leave it
#endif
};
// The lens sample of a pick; the lean kernels have no lens (RB_CAM_LENS is false there) and keep PrimEdgePick as it was without one.
RB_D D2 pick_lens(const PrimEdgePick& pk) {
#ifdef RB_LEAN
    return d2(0, 0);
#else
    return pk.lu;
#endif
}
// Gradients of the edge equation alpha(p) = dot(p, cross(v0_dir, v1_dir)) on the camera-space film w.r.t. the two projected
// end points and the edge point (src/edge.cpp:737-757).
RB_HD void primary_edge_grad_nonlinear(const DevCamera& cam, D2 q0, D2 q1, D2 ept, double* g) {
    D3 a = cam_screen_to_camera_d(cam, q0), b = cam_screen_to_camera_d(cam, q1), e = cam_screen_to_camera_d(cam, ept);
    D2 g0 = d_cam_screen_to_camera_d(cam, q0, d3_cross(b, e)), g1 = d_cam_screen_to_camera_d(cam, q1, d3_cross(e, a));
    D2 ge = d_cam_screen_to_camera_d(cam, q1, d3_cross(a, b)); // (evaluated at v1_ss like the reference, :757)
    g[0] = g0.x; g[1] = g0.y; g[2] = g1.x; g[3] = g1.y; g[4] = ge.x; g[5] = ge.y;
}
// Fisheye / panorama / distorted cameras (cold for the usual pinhole camera).
RB_HD bool primary_edge_pick_nonlinear(const DevScene& sc, V3 v0, V3 v1, PrimEdgePick& pk) {
    // src/edge.cpp:486-592: the edge is a straight segment on the film in CAMERA space, so the
    // point is sampled there and projected back; the two rays leave the edge plane by an offset shrinking with distance.
    D3 a = cam_screen_to_camera_d(sc.cam, pk.q0), b = cam_screen_to_camera_d(sc.cam, pk.q1);
    D3 ab = d3(b.x - a.x, b.y - a.y, b.z - a.z);
    D3 p3 = d3(a.x + pk.e_t * ab.x, a.y + pk.e_t * ab.y, a.z + pk.e_t * ab.z);
    pk.ept = cam_to_screen_d(sc.cam, p3);
    if (!cam_in_screen(sc.cam, mk2((Real)pk.ept.x, (Real)pk.ept.y))) return false;
    D3 axb = d3_cross(a, b);
    D3 hn = d3_normalize(axb);
    D3 l0 = w2c_point(sc.cam, d3(v0.x, v0.y, v0.z)), l1 = w2c_point(sc.cam, d3(v1.x, v1.y, v1.z));
    D3 el = d3(l0.x + pk.e_t * l1.x, l0.y + pk.e_t * l1.y, l0.z + pk.e_t * l1.z); // (v0 + t v1, as in the reference :527)
    double offset = 1e-5f / sqrt(el.x * el.x + el.y * el.y + el.z * el.z);
    pk.upper = cam_to_screen_d(sc.cam, d3_normalize(d3(p3.x + offset * hn.x, p3.y + offset * hn.y, p3.z + offset * hn.z)));
    pk.lower = cam_to_screen_d(sc.cam, d3_normalize(d3(p3.x - offset * hn.x, p3.y - offset * hn.y, p3.z - offset * hn.z)));
    D2 d_ept = d_cam_screen_to_camera_d(sc.cam, pk.ept, axb);
    double dirac_jacobian = 1.0 / sqrt(d_ept.x * d_ept.x + d_ept.y * d_ept.y);
    const double jac_offset = 1e-6;
    D2 pd = cam_to_screen_d(sc.cam, d3(a.x + (pk.e_t + jac_offset) * ab.x, a.y + (pk.e_t + jac_offset) * ab.y, a.z + (pk.e_t + jac_offset) * ab.z));
    // (finite difference divided by the RAY offset, not by jac_offset: src/edge.cpp:577)
    double line_jacobian = sqrt(rb_sq((pd.x - pk.ept.x) / offset) + rb_sq((pd.y - pk.ept.y) / offset));
    pk.jacobian = line_jacobian * dirac_jacobian;
    return true;
}
// Ends of edge (v0, v1) projected from lens sample lu (lens_film_point in double), after the camera-space near clip of cam_project_d.
RB_HD bool cam_project_lens_d(const DevCamera& cam, D3 p0, D3 p1, D2 lu, D2& q0, D2& q1) {
    D3 a = w2c_point(cam, p0), b = w2c_point(cam, p1);
    double cn = cam.clip_near;
    if (a.z < cn && b.z < cn) return false;
    if (a.z < cn) {
        D3 dir = d3(a.x - b.x, a.y - b.y, a.z - b.z);
        double t = -(b.z - cn) / dir.z;
        a = d3(b.x + t * dir.x, b.y + t * dir.y, b.z + t * dir.z);
    } else if (b.z < cn) {
        D3 dir = d3(b.x - a.x, b.y - a.y, b.z - a.z);
        double t = -(a.z - cn) / dir.z;
        b = d3(a.x + t * dir.x, a.y + t * dir.y, a.z + t * dir.z);
    }
    const double f = cam.focus_distance, lx = cam.lens_radius * lu.x, ly = cam.lens_radius * lu.y;
    q0 = cam_to_screen_d(cam, d3(lx / f + (a.x - lx) / a.z, ly / f + (a.y - ly) / a.z, 1.0));
    q1 = cam_to_screen_d(cam, d3(lx / f + (b.x - lx) / b.z, ly / f + (b.y - ly) / b.z, 1.0));
    return true;
}
// The lens camera's pick: the edge projected from the lens point, a uniform point on the projected segment, dropped when it is off
// screen or when the edge is no silhouette seen from the lens point.  The projection is linear, so the pinhole's offsets and jacobian
// carry over.
RB_D bool primary_edge_pick_lens(const DevScene& sc, const Edge& edge, V3 v0, V3 v1, D2 lu, PrimEdgePick& pk) {
    if (pk.pmf <= 0) return false;
    if (!cam_project_lens_d(sc.cam, d3(v0.x, v0.y, v0.z), d3(v1.x, v1.y, v1.z), lu, pk.q0, pk.q1)) return false;
    pk.ept.x = pk.q0.x + pk.e_t * (pk.q1.x - pk.q0.x);
    pk.ept.y = pk.q0.y + pk.e_t * (pk.q1.y - pk.q0.y);
    if (!cam_in_screen(sc.cam, mk2((Real)pk.ept.x, (Real)pk.ept.y))) return false;
    const double* C = sc.cam.c2w;
    const double lx = sc.cam.lens_radius * lu.x, ly = sc.cam.lens_radius * lu.y, iw = 1.0 / (C[12] * lx + C[13] * ly + C[15]);
    const V3 lens_world = mk3((Real)((C[0] * lx + C[1] * ly + C[3]) * iw), (Real)((C[4] * lx + C[5] * ly + C[7]) * iw), (Real)((C[8] * lx + C[9] * ly + C[11]) * iw));
    if (!edge_is_silhouette(sc.shapes, lens_world, edge)) return false;
    double ddx = pk.q0.x - pk.q1.x, ddy = pk.q0.y - pk.q1.y;
    double dl = sqrt(ddx * ddx + ddy * ddy);
    double nx = ddy / dl, ny = -ddx / dl;
    const double offset = 1e-6;
    pk.upper.x = pk.ept.x + nx * offset;
    pk.upper.y = pk.ept.y + ny * offset;
    pk.lower.x = pk.ept.x - nx * offset;
    pk.lower.y = pk.ept.y - ny * offset;
    pk.jacobian = 1;
    return true;
}
RB_D bool primary_edge_pick(const DevScene& sc, const RenderParams& rp, long long i, int s, int dim_base, Sampler& smp, PrimEdgePick& pk) {
    smp.init(rp.sampler_type, rp.seed + 131071ULL, (int)i, (unsigned)s, sc.sobol_matrices, RB_SOBOL_BITS,
             (unsigned long long)s * edge_draws_per_sample(sc, rp));
    smp.skip(dim_base);
    double e_sel = smp.next();
    pk.e_t = smp.next();
#ifndef RB_LEAN
    pk.lu = primary_lens_sample(sc, smp);
#endif
    pk.edge_id = cdf_pick(sc.prim_edge_cdf, sc.num_edges, e_sel);
    pk.pmf = sc.prim_edge_pmf[pk.edge_id];
    const Edge edge = sc.edges[pk.edge_id];
    V3 v0 = edge_v0(sc.shapes, edge), v1 = edge_v1(sc.shapes, edge);
    if (RB_CAM_LENS(sc.cam)) return primary_edge_pick_lens(sc, edge, v0, v1, pick_lens(pk), pk);
    if (!cam_project_d(sc.cam, d3(v0.x, v0.y, v0.z), d3(v1.x, v1.y, v1.z), pk.q0, pk.q1)) return false;
    if (pk.pmf <= 0) return false;
    if (cam_is_linear(sc.cam)) {
        pk.ept.x = pk.q0.x + pk.e_t * (pk.q1.x - pk.q0.x);
        pk.ept.y = pk.q0.y + pk.e_t * (pk.q1.y - pk.q0.y);
        if (RB_PIXEL_BOX(sc.cam) ? !cam_in_screen(sc.cam, mk2((Real)pk.ept.x, (Real)pk.ept.y)) : !cam_in_filter_reach(sc.cam, pk.ept)) return false;
        // unit normal of the projected edge: get_normal(normalize(v0_ss - v1_ss)) = (d.y, -d.x); rays at +-1e-6 across it
        double ddx = pk.q0.x - pk.q1.x, ddy = pk.q0.y - pk.q1.y;
        double dl = sqrt(ddx * ddx + ddy * ddy);
        double nx = ddy / dl, ny = -ddx / dl;
        const double offset = 1e-6;
        pk.upper.x = pk.ept.x + nx * offset;
        pk.upper.y = pk.ept.y + ny * offset;
        pk.lower.x = pk.ept.x - nx * offset;
        pk.lower.y = pk.ept.y - ny * offset;
        pk.jacobian = 1;
        return true;
    }
    return primary_edge_pick_nonlinear(sc, v0, v1, pk);
}
// Viewport pixel whose d_image a primary-edge point reads under the 1-pixel box (clamped to [0, vp_w] x [0, vp_h], like the reference).
RB_HD void edge_point_pixel(const DevCamera& cam, D2 ept, int& xi, int& yi) {
    xi = rb_clampi(int(ept.x * cam.width - cam.vp_beg[0]), 0, cam.vp_end[0] - cam.vp_beg[0]);
    yi = rb_clampi(int(ept.y * cam.height - cam.vp_beg[1]), 0, cam.vp_end[1] - cam.vp_beg[1]);
}
// Viewport pixels [cx0, cx1] x [cy0, cy1] whose filter support holds the screen point p (empty when cx1 < cx0 or cy1 < cy0), and
// p's offsets (x, y) from the centre of viewport pixel (0, 0): pixel c is reached when |offset - c| < the filter's radius.
struct FilterReach {
    double x, y;
    int cx0, cx1, cy0, cy1;
};
RB_HD FilterReach filter_reach(const DevCamera& cam, const RenderParams& rp, D2 p) {
    FilterReach f;
    const double r = filter_radius(cam);
    f.x = p.x * cam.width - cam.vp_beg[0] - 0.5;
    f.y = p.y * cam.height - cam.vp_beg[1] - 0.5;
    f.cx0 = rb_clampi((int)floor(f.x - r) + 1, 0, rp.vp_w);
    f.cx1 = rb_clampi((int)ceil(f.x + r) - 1, -1, rp.vp_w - 1);
    f.cy0 = rb_clampi((int)floor(f.y - r) + 1, 0, rp.vp_h);
    f.cy1 = rb_clampi((int)ceil(f.y + r) - 1, -1, rp.vp_h - 1);
    return f;
}
// True iff every d_image float that primary_edge_sample reads for the edge point `ept` is zero: the sample then adds nothing.  The
// 1-pixel box reads edge_point_pixel's pixel, every other filter the pixels of its reach (filter_splat).
RB_D bool edge_point_adjoint_is_zero(const DevScene& sc, const KernelArgs& ka, D2 ept) {
    if (RB_PIXEL_BOX(sc.cam)) {
        int xi, yi;
        edge_point_pixel(sc.cam, ept, xi, yi);
        return pixel_adjoint_is_zero(ka, yi * ka.rp.vp_w + xi);
    }
    const FilterReach f = filter_reach(sc.cam, ka.rp, ept);
    for (int cy = f.cy0; cy <= f.cy1; cy++)
        for (int cx = f.cx0; cx <= f.cx1; cx++)
            if (!pixel_adjoint_is_zero(ka, cy * ka.rp.vp_w + cx)) return false;
    return true;
}
// Sort key of a primary-edge sample: (edge, position along the edge).  Samples that are neighbours under this key
// shoot nearly the same camera rays and scatter into the same two vertices; ~0u = contributes nothing (no edge point, or one
// whose pixels' adjoint is zero).
RB_D unsigned primary_edge_key(const DevScene& sc, const KernelArgs& ka, long long i, int s, int dim_base) {
    Sampler smp;
    PrimEdgePick pk;
    if (!primary_edge_pick(sc, ka.rp, i, s, dim_base, smp, pk)) return 0xffffffffu;
    if (ka.zero_cull && edge_point_adjoint_is_zero(sc, ka, pk.ept)) return 0xffffffffu;
    int ebits = 1;
    while ((1 << ebits) < sc.num_edges && ebits < 31) ebits++;
    int tbits = 31 - ebits; // (the top bit stays clear so that no key equals ~0u)
    unsigned tq = tbits > 0 ? (unsigned)rb_clampi((int)(pk.e_t * (double)(1u << tbits)), 0, (1 << tbits) - 1) : 0u;
    return ((unsigned)pk.edge_id << tbits) | tq;
}
// out[0, nd) = sum of f(p - c) d_image[c] over the viewport pixels c whose filter support holds the screen point p (at most 4 x 4 of
// them for widths up to 4 pixels), in a fixed order.
RB_D void filter_splat(const DevCamera& cam, const RenderParams& rp, const float* d_image, D2 p, float* out) {
    const int nd = rp.nd < RB_MAX_ND ? rp.nd : RB_MAX_ND;
    for (int k = 0; k < nd; k++) out[k] = 0.f;
    const FilterReach f = filter_reach(cam, rp, p);
    for (int cy = f.cy0; cy <= f.cy1; cy++) {
        const double wy = filter_density(cam, f.y - cy);
        for (int cx = f.cx0; cx <= f.cx1; cx++) {
            const float w = (float)(wy * filter_density(cam, f.x - cx));
            const float* px = d_image + (size_t)rp.nd * ((size_t)cy * rp.vp_w + cx);
            for (int k = 0; k < nd; k++) out[k] += w * px[k];
        }
    }
}
// What one primary-edge sample hands to the projection: its edge, its lens point and the screen-space adjoints of the edge's two
// projected end points.
struct PrimEdgeAdjoint {
    int edge_id;
    D2 lu;
    Real d0x, d0y, d1x, d1y;
};
// The per-sample part of a primary-edge sample: the pick, the two edge rays, the contribution, and the screen_grad scatter.  False when the
// sample adds nothing; otherwise `a` holds the adjoints that primary_edge_project turns into vertex and camera gradients.
RB_D bool primary_edge_screen_adjoint(const DevScene& sc, const KernelArgs& ka, long long i, int s, int dim_base, PrimEdgeAdjoint& a) {
    const RenderParams& rp = ka.rp;
    const Real weight = Real(1) / Real(rp.spp);
    Sampler smp;
    PrimEdgePick pk;
    if (!primary_edge_pick(sc, rp, i, s, dim_base, smp, pk)) return false;
    const D2 lu = pick_lens(pk);
    if (ka.zero_cull && edge_point_adjoint_is_zero(sc, ka, pk.ept)) return false; // (before any ray: k_prim_keys drops these samples too)
    const double pmf = pk.pmf;
    const D2 q0 = pk.q0, q1 = pk.q1, ept = pk.ept;
    const Edge edge = sc.edges[pk.edge_id];
    int vp_w = rp.vp_w;
    int xi, yi;
    edge_point_pixel(sc.cam, ept, xi, yi);
    const float* dpx_all = ka.d_image + (size_t)rp.nd * ((size_t)yi * vp_w + xi);
    // Under a pixel filter the edge point weighs into every viewport pixel whose support holds it.  The integrand is linear in the
    // d_image multipliers, so the rays and the scatter below run once, on their filter-weighted sum.
    float d_splat[RB_MAX_ND];
    if (!RB_PIXEL_BOX(sc.cam)) {
        filter_splat(sc.cam, rp, ka.d_image, ept, d_splat);
        dpx_all = d_splat;
    }
    const float* dpx = dpx_all + (rp.rad_dim >= 0 ? rp.rad_dim : 0);
    V3 d_color = rp.rad_dim >= 0 ? mk3(dpx[0], dpx[1], dpx[2]) : zero3();
    V3 wgt = d_color * (Real)(pk.jacobian / pmf);
    // ray differential of the un-offset ray, shared by both sides (src/edge.cpp:594-608)
    Ray cray;
    RayDiff rd;
    cam_primary_ray(sc.cam, ept.x, ept.y, cray, rd, lu);
    Real contrib = 0;
    Ray rays[2];
    Isect hits[2];
    bool connected = false;
    for (int side = 0; side < 2; side++) {
        D3 o, d;
        cam_sample_primary(sc.cam, side == 0 ? pk.upper.x : pk.lower.x, side == 0 ? pk.upper.y : pk.lower.y, o, d, lu);
        rays[side] = make_ray(o, d);
        hits[side] = no_isect();
        if (!ray_is_null(rays[side])) closest_hit(sc, rays[side], hits[side]);
        // at least one side must see a face of the edge, otherwise the edge is hidden here and the sample is dropped
        // (primary_edge_weights_updater, src/edge.cpp:653-676)
        connected = connected || (hits[side].shape_id == edge.shape_id && (hits[side].tri_id == edge.f0 || hits[side].tri_id == edge.f1));
    }
    if (!connected) return false;
    for (int side = 0; side < 2; side++) {
        const Ray ray = rays[side];
        const Isect is = hits[side];
        V3 thr = side == 0 ? wgt : -wgt;
        if (!is.valid()) { // this side looks past the edge into the environment (src/primary_contribution.cpp:25-29)
            if (rp.rad_dim >= 0 && !ray_is_null(ray)) contrib += sum(weight * thr * miss_emission(sc, ray.dir, rd));
            continue;
        }
        RayDiff rd_after;
        SurfacePoint sp = make_surface_point(sc.shapes[is.shape_id], is.tri_id, ray, rd, rd_after);
        if (rp.rad_dim >= 0) {
            contrib += sum(weight * thr * hit_emission(sc, is, sp, -ray.dir));
            Sampler sub = smp; // both sides consume the same light / bsdf samples (src/pathtracer.cpp:871-886)
            V3 Lb = trace_bounces<false>(sc, sub, ray, rd, is, thr, Real(0), 0, rp.max_bounces, nullptr, 0, nullptr);
            contrib += sum(weight * Lb);
        }
        if (!RB_ONLY_RADIANCE(rp)) {
            // every other channel enters the edge integrand with its own d_image component as the multiplier
            // (channel_multipliers, src/edge.cpp:476-481; src/primary_contribution.cpp:256-435)
            Real vals[RB_MAX_ND];
            for (int k = 0; k < rp.nd; k++) vals[k] = 0;
            channel_values_at_hit(sc, rp, is, sp, ray, vals);
            Real acc = 0;
            int d = 0;
            for (int c = 0; c < rp.num_channels; c++) {
                int w = rb_channel_width(rp.channels[c], rp.max_generic);
                int ch = rp.channels[c];
                if (ch != RB_CH_RADIANCE && ch != RB_CH_SHAPE_ID && ch != RB_CH_TRIANGLE_ID && ch != RB_CH_MATERIAL_ID)
                    for (int k = 0; k < w; k++) acc += vals[d + k] * (Real)dpx_all[d + k];
                d += w;
            }
            contrib += (side == 0 ? weight : -weight) * acc * (Real)(pk.jacobian / pmf);
        }
    }
    if (contrib == 0) return false;
    // gradients of the edge equation w.r.t. the projected end points and the edge point
    Real d0x, d0y, d1x, d1y, dex, dey;
    if (cam_is_linear(sc.cam)) { // Eq. 8
        d0x = (Real)(q1.y - ept.y) * contrib; d0y = (Real)(ept.x - q1.x) * contrib;
        d1x = (Real)(ept.y - q0.y) * contrib; d1y = (Real)(q0.x - ept.x) * contrib;
        dex = (Real)(q0.y - q1.y) * contrib; dey = (Real)(q1.x - q0.x) * contrib;
    } else {
        double g[6];
        primary_edge_grad_nonlinear(sc.cam, q0, q1, ept, g);
        d0x = (Real)g[0] * contrib; d0y = (Real)g[1] * contrib;
        d1x = (Real)g[2] * contrib; d1y = (Real)g[3] * contrib;
        dex = (Real)g[4] * contrib; dey = (Real)g[5] * contrib;
    }
    if (ka.screen_grad) {
        size_t pix = (size_t)yi * vp_w + xi;
        rb_red_add(&ka.screen_grad[2 * pix + 0], (float)dex);
        rb_red_add(&ka.screen_grad[2 * pix + 1], (float)dey);
    }
    a.edge_id = pk.edge_id;
    a.lu = lu;
    a.d0x = d0x; a.d0y = d0y;
    a.d1x = d1x; a.d1y = d1y;
    return true;
}
// The projection of a primary-edge sample: the adjoints (d0x, d0y, d1x, d1y) of edge `edge_id`'s projected end points, through the camera
// projection, into its two vertices' gradients and the camera accumulators.  Linear in the adjoints, and apart from the lens point it
// depends on the edge alone, so without a lens k_primary_edge runs it once per edge on the sum of the edge's samples (k_prim_edge_project).
RB_D void primary_edge_project(const DevScene& sc, const KernelArgs& ka, int edge_id, D2 lu, Real d0x, Real d0y, Real d1x, Real d1y, CamAcc& cam_acc) {
    const Edge edge = sc.edges[edge_id];
    V3 v0 = edge_v0(sc.shapes, edge), v1 = edge_v1(sc.shapes, edge);
    V3 d_v0 = zero3(), d_v1 = zero3();
    if (RB_CAM_LENS(sc.cam)) d_cam_project_lens(sc.cam, v0, v1, lu, d0x, d0y, d1x, d1y, cam_acc, d_v0, d_v1);
    else d_cam_project(sc.cam, v0, v1, d0x, d0y, d1x, d1y, cam_acc, d_v0, d_v1);
    float* dv = ka.ds.shapes[edge.shape_id].vertices;
    if (dv) {
        agg_add3(dv + 3 * (size_t)edge.v0, d_v0);
        agg_add3(dv + 3 * (size_t)edge.v1, d_v1);
    }
}
RB_D void primary_edge_sample(const DevScene& sc, const KernelArgs& ka, long long i, int s, int dim_base, CamAcc& cam_acc) {
    PrimEdgeAdjoint a;
    if (primary_edge_screen_adjoint(sc, ka, i, s, dim_base, a)) primary_edge_project(sc, ka, a.edge_id, a.lu, a.d0x, a.d0y, a.d1x, a.d1y, cam_acc);
}

// Turns the reduced matrix gradients into the user-facing camera gradients (everything is linear in the accumulated
// matrices): d_project's world_to_cam term (src/camera.h:811-829) and d_look_at_matrix (src/transform.h:29-71).
RB_HD void finish_camera(const DevCamera& cam, const double* acc, const rb_dcamera& out) {
    double C[4][4], W[4][4], Dw[4][4];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            C[i][j] = acc[4 * i + j];
            Dw[i][j] = acc[16 + 4 * i + j];
            W[i][j] = cam.w2c[4 * i + j];
        }
    // d_cam_to_world += -W^T * d_W * W^T
    double tmp[4][4];
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double s = 0;
            for (int k = 0; k < 4; k++) s += W[k][i] * Dw[k][j];
            tmp[i][j] = s;
        }
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            double s = 0;
            for (int k = 0; k < 4; k++) s += tmp[i][k] * W[j][k];
            C[i][j] -= s;
        }
    if (cam.use_look_at) {
        M4 d_m;
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++) d_m.m[i][j] = (Real)C[i][j];
        V3 pos = mk3((Real)cam.position[0], (Real)cam.position[1], (Real)cam.position[2]);
        V3 look = mk3((Real)cam.look[0], (Real)cam.look[1], (Real)cam.look[2]);
        V3 up = mk3((Real)cam.up[0], (Real)cam.up[1], (Real)cam.up[2]);
        V3 d_p = zero3(), d_l = zero3(), d_u = zero3();
        d_look_at_matrix(pos, look, up, d_m, d_p, d_l, d_u);
        if (out.position) { out.position[0] += (float)d_p.x; out.position[1] += (float)d_p.y; out.position[2] += (float)d_p.z; }
        if (out.look) { out.look[0] += (float)d_l.x; out.look[1] += (float)d_l.y; out.look[2] += (float)d_l.z; }
        if (out.up) { out.up[0] += (float)d_u.x; out.up[1] += (float)d_u.y; out.up[2] += (float)d_u.z; }
    } else if (out.cam_to_world) {
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++) out.cam_to_world[4 * i + j] += (float)C[i][j];
    }
    if (out.intrinsic_mat_inv)
        for (int k = 0; k < 9; k++) out.intrinsic_mat_inv[k] += (float)acc[32 + k];
    if (out.intrinsic_mat)
        for (int k = 0; k < 9; k++) out.intrinsic_mat[k] += (float)acc[41 + k];
    if (out.distortion)
        for (int k = 0; k < 8; k++) out.distortion[k] += (float)acc[50 + k];
    if (out.lens && cam.lens_radius > 0)
        for (int k = 0; k < 2; k++) out.lens[k] += (float)acc[RB_CAM_ACC + k];
}
