/*
 * redner_b200 -- C ABI of the H100-native differentiable path tracer.
 *
 * This is the drop-in boundary for the one hot path of BachiLi/redner:
 *   pyredner.RenderFunction.forward/backward  ->  redner.render(...)
 * Every entry point below replaces one piece of the reference's pybind11 surface
 * (reference file:line given per item; paths relative to the reference checkout).
 * Signatures use plain pointers and sizes only (no torch / pybind types).
 *
 * Memory convention (same as the reference, pyredner/render_pytorch.py:314-617):
 *   - the CALLER owns every buffer; the library stores raw pointers only;
 *   - mesh, texture, image and gradient buffers are DEVICE pointers (cuda:<gpu_index>);
 *   - camera parameters, light intensities and other small "host-read" parameters are
 *     passed BY VALUE inside the descriptors (the reference copies them at construction
 *     time: src/camera.h:44-65, src/area_light.h:18-20);
 *   - image and gradient buffers are pre-zeroed by the caller and are ACCUMULATED into.
 *
 * Error convention: every call returns 0 on success, non-zero on failure;
 * rb_last_error() returns a thread-local message (the reference assert()/exit(1)s instead:
 * src/cuda_utils.h:9-13, src/redner.h:173).
 */
#ifndef REDNER_B200_H
#define REDNER_B200_H

#include <stdint.h>

#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define RB_MAX_MIP_LEVELS 8 /* src/texture.h:11 max_num_texels */

/* src/camera.h:12-17 */
enum rb_camera_type { RB_CAMERA_PERSPECTIVE = 0, RB_CAMERA_ORTHOGRAPHIC = 1, RB_CAMERA_FISHEYE = 2, RB_CAMERA_PANORAMA = 3 };
/* src/pathtracer.h:11-14 */
enum rb_sampler_type { RB_SAMPLER_INDEPENDENT = 0, RB_SAMPLER_SOBOL = 1 };
/* src/channels.h:6-23 */
enum rb_channel {
    RB_CH_RADIANCE = 0, RB_CH_ALPHA, RB_CH_DEPTH, RB_CH_POSITION, RB_CH_GEOMETRY_NORMAL, RB_CH_SHADING_NORMAL,
    RB_CH_UV, RB_CH_BARYCENTRIC, RB_CH_DIFFUSE_REFLECTANCE, RB_CH_SPECULAR_REFLECTANCE, RB_CH_ROUGHNESS,
    RB_CH_GENERIC_TEXTURE, RB_CH_VERTEX_COLOR, RB_CH_SHAPE_ID, RB_CH_TRIANGLE_ID, RB_CH_MATERIAL_ID, RB_CH_COUNT
};

/* Camera -- src/camera.h:19-83 (constructor semantics: cam_to_world given <=> use_look_at == 0). */
typedef struct rb_camera {
    int width, height;
    int use_look_at;
    float position[3], look[3], up[3]; /* valid if use_look_at */
    float cam_to_world[16];            /* row-major; valid if !use_look_at */
    float world_to_cam[16];            /* row-major; valid if !use_look_at */
    float intrinsic_mat_inv[9];        /* row-major 3x3 */
    float intrinsic_mat[9];
    int has_distortion;
    float distortion[8]; /* k1..k6, p1, p2 -- src/camera.h:56-62 */
    float clip_near;
    int camera_type; /* rb_camera_type */
    int viewport_beg[2], viewport_end[2]; /* (x, y) -- src/camera.h:82 */
    /* Thin lens (no reference counterpart; DESIGN.md "thin-lens camera"), in world units.  lens_radius == 0 (the zero-initialised
     * struct) is the pinhole, and focus_distance is then ignored.  With lens_radius > 0 each camera sample also picks a point L on the
     * disc of that radius around the camera origin, in the plane z = 0 of camera space, uniformly, and the ray leaves L towards the
     * point of the plane z = focus_distance that the pinhole ray of the same film position meets.  rb_scene_create, rb_scene_update and
     * rb_scene_set_camera refuse, with a message naming the lens, a lens_radius that is negative or not finite, a focus_distance that is
     * not finite or not > 0, and a lens on anything but a perspective camera without distortion and with the 1-pixel box pixel filter;
     * rb_render refuses a lens together with a screen_gradient_image. */
    float lens_radius, focus_distance;
} rb_camera;

/* Shape -- src/shape.h:9-63.  All pointers are device pointers; optional ones may be NULL. */
typedef struct rb_shape {
    const float* vertices;     /* [num_vertices, 3] */
    const int* indices;        /* [num_triangles, 3] */
    const float* uvs;          /* [num_uv_vertices, 2] or NULL */
    const float* normals;      /* [num_normal_vertices, 3] or NULL */
    const int* uv_indices;     /* [num_triangles, 3] or NULL */
    const int* normal_indices; /* [num_triangles, 3] or NULL */
    const float* colors;       /* [num_vertices, 3] or NULL */
    int num_vertices, num_uv_vertices, num_normal_vertices, num_triangles;
    int material_id, light_id;
} rb_shape;

/* Texture<N> -- src/texture.h:14-46.  Constant texture <=> width[0] == 0 && height[0] == 0 (src/texture.h:342). */
typedef struct rb_texture {
    float* texels[RB_MAX_MIP_LEVELS]; /* device pointers, [h, w, channels] per level, or [channels] if constant */
    int width[RB_MAX_MIP_LEVELS];
    int height[RB_MAX_MIP_LEVELS];
    int channels;
    int num_levels;  /* 0 == texture absent */
    float* uv_scale; /* device pointer to 2 floats (may be NULL when num_levels == 0) */
} rb_texture;

/* Specular lobe of a material (rb_material::specular_model).  Blinn-Phong is the reference's lobe (a Phong exponent 2 / r - 2 with a
 * rational fit of the Smith term).  GGX (no reference counterpart) is the Trowbridge-Reitz distribution with alpha = sqrt(r),
 * height-correlated Smith masking-shadowing and sampling of the visible normals; DESIGN.md section "GGX" defines it. */
enum rb_specular_model { RB_SPECULAR_BLINN_PHONG = 0, RB_SPECULAR_GGX = 1 };

/* Material -- src/material.h:12-91; DMaterial (src/material.h:93-99) uses the same layout with gradient buffers. */
typedef struct rb_material {
    rb_texture diffuse_reflectance;  /* 3 channels */
    rb_texture specular_reflectance; /* 3 channels */
    rb_texture roughness;            /* 1 channel */
    rb_texture generic_texture;      /* N channels, optional */
    rb_texture normal_map;           /* 3 channels, optional */
    int compute_specular_lighting, two_sided, use_vertex_color;
    /* rb_specular_model; zero-initialised == Blinn-Phong.  Matters only with compute_specular_lighting and without use_vertex_color.
     * rb_scene_create and rb_scene_update refuse any other value; rb_dscene_desc::materials ignores the field. */
    int specular_model;
} rb_material;

/* AreaLight -- src/area_light.h:8-36 */
typedef struct rb_area_light {
    int shape_id;
    float intensity[3];
    int two_sided, directly_visible;
    /* Emission texture (no reference counterpart; DESIGN.md "Emission textures").  num_levels == 0 (the zero-initialised field) is no
     * texture: the light emits `intensity` everywhere, as in the reference.  Otherwise the light emits intensity * E(uv) at a point of its
     * shape, where E is this 1- or 3-channel mip-mapped texture (1 channel is broadcast to RGB) and uv the shape's texture coordinate there
     * (its uvs, or the default per-triangle uvs, times uv_scale).  Rays from the camera and edge rays look it up with the footprint of the
     * material textures at that hit; light samples and BSDF-sampled hits with a zero footprint.  Light selection and the point on the
     * light are sampled as without a texture unless emission_sampling asks otherwise.  rb_scene_create and rb_scene_update refuse, with a message naming the emission texture, a
     * channel count other than 1 or 3, num_levels outside [0, RB_MAX_MIP_LEVELS], a level without texels, a non-constant level without a
     * positive size and a missing uv_scale.  rb_scene_update may add, change or remove the texture: it is a value of the light, like
     * intensity. */
    rb_texture emission;
    /* One of rb_emission_sampling, below (no reference counterpart; DESIGN.md "Emission sampling").  RB_EMISSION_SAMPLE_AREA (the zero-initialised field)
     * places light samples uniformly by area, as the reference does.  RB_EMISSION_SAMPLE_TEXTURE, on a light whose emission texture is not
     * constant, places them by a defensive mixture: with probability 1/8 uniformly by area, otherwise by the luminance of the texture's
     * level 0 (a triangle by its area times the mean cell weight over its uv bounding box, then a texel cell, then a point uniformly in
     * the cell; a point outside the triangle is rejected and contributes nothing).  The light's selection weight then uses the sum of
     * those triangle weights in place of its area.  Without a texture, or with a constant one, the option changes nothing.  The tables
     * are rebuilt from the texels by every rb_scene_create and rb_scene_update; texels written in place without an update leave them
     * stale, which costs variance but no bias.  rb_scene_create and rb_scene_update refuse, with a message naming the emission sampling,
     * any other value and a light whose scaled texture coordinates (uv * uv_scale * level-0 size) reach 2^24 cells in magnitude or are
     * not finite. */
    int emission_sampling;
} rb_area_light;
/* rb_area_light::emission_sampling */
enum rb_emission_sampling { RB_EMISSION_SAMPLE_AREA = 0, RB_EMISSION_SAMPLE_TEXTURE = 1 };

/* EnvironmentMap -- src/envmap.h:19-51, constructor src/redner.cpp:169-178.  `values` is the [h, w, 3] mip pyramid, the two
 * tables are the caller's importance-sampling CDFs (pyredner/envmap.py:36-61); all device memory, matrices row-major. */
typedef struct rb_envmap {
    rb_texture values;
    float env_to_world[16], world_to_env[16];
    const float* sample_cdf_ys;
    const float* sample_cdf_xs;
    float pdf_norm;
    int directly_visible;
} rb_envmap;

/* Pixel reconstruction filter (no reference counterpart; the reference integrates radiance over the 1 x 1 pixel box).  Widths are in
 * pixels: the box's side length; the tent's base width (radius width / 2); the Gaussian's truncation interval [-width / 2, width / 2],
 * with sigma = width / 6.  The filter is separable and importance-sampled: a camera sample is placed at the pixel centre plus an offset
 * drawn from the filter, and keeps weight 1 / num_samples, so a pixel is the filter-weighted integral of the radiance around its
 * centre.  Samples may land outside their pixel and outside the image. */
enum rb_filter_type { RB_FILTER_BOX = 0, RB_FILTER_TENT = 1, RB_FILTER_GAUSSIAN = 2 };
typedef struct rb_pixel_filter {
    int type;    /* rb_filter_type */
    float width; /* in (0, 4] pixels; { 0, 0 } == { RB_FILTER_BOX, 1 } */
} rb_pixel_filter;

/* Scene -- constructor arguments of src/scene.cpp:63-75 / src/redner.cpp:62-73 */
typedef struct rb_scene_desc {
    rb_camera camera;
    int num_shapes;
    const rb_shape* shapes; /* host array */
    int num_materials;
    const rb_material* materials; /* host array */
    int num_lights;
    const rb_area_light* lights; /* host array */
    const rb_envmap* envmap;     /* host pointer or NULL */
    int use_gpu;                 /* must be 1: there is no CPU fallback */
    int gpu_index;               /* -1 == current device (src/pathtracer.cpp:186-191) */
    int use_primary_edge_sampling;
    int use_secondary_edge_sampling;
    /* A zero-initialised field is the 1-pixel box: the reference's image formation, bit for bit.  The filter belongs to the scene because
     * the primary-edge distribution depends on its radius: it covers the image grown by max(0, width / 2 - 0.5) pixels on each side.
     * rb_scene_create and rb_scene_update refuse, with a message naming the pixel filter, an unknown type, a width outside (0, 4], and any
     * filter but the 1-pixel box with a fisheye or panorama camera or a lens-distortion model; rb_scene_set_camera refuses those
     * cameras on a scene with such a filter.  rb_render refuses such a filter together with sample_pixel_center or a
     * screen_gradient_image. */
    rb_pixel_filter pixel_filter;
} rb_scene_desc;

/* RenderOptions -- src/pathtracer.h:16-23 */
typedef struct rb_options {
    uint64_t seed;
    int num_samples;
    int max_bounces;
    int num_channels;
    const int* channels; /* host array of rb_channel */
    int sampler_type;    /* rb_sampler_type */
    int sample_pixel_center;
    /* 0: gradients are summed with float atomics, in whatever order the GPU schedules them (the last bits vary between runs).
     * Non-zero: every gradient the backward pass writes -- every buffer of d_scene, the camera and screen_gradient_image -- is the
     * correctly rounded exact sum of the per-sample float contributions, the same run after run whatever the band size, grid or
     * device scheduling (fixed-point accumulators, DESIGN.md section 2).  It is added once into the caller's buffer; elements that
     * received nothing are left as they are.  The accumulators take 88 bytes per gradient float from the backward scratch (see
     * rb_release_scratch).  The forward pass is deterministic either way.  A zero-initialised struct keeps the default. */
    int deterministic;
} rb_options;

/* DShape -- src/shape.h:65-80 (device pointers, any may be NULL) */
typedef struct rb_dshape {
    float *vertices, *uvs, *normals, *colors;
} rb_dshape;

/* DCamera -- src/camera.h:85-112 (device pointers) */
typedef struct rb_dcamera {
    float *position, *look, *up;      /* 3 floats each, used when the camera uses look-at */
    float *cam_to_world, *world_to_cam; /* 16 floats each */
    float *intrinsic_mat_inv, *intrinsic_mat; /* 9 floats each */
    float* distortion;                /* 8 floats or NULL */
    float* lens;                      /* 2 floats { d(lens_radius), d(focus_distance) }, or NULL; written only when the camera has a lens */
} rb_dcamera;

/* DEnvironmentMap -- src/envmap.h:53-61: gradient mip pyramid and the 16 floats of d(world_to_env) (device memory) */
typedef struct rb_denvmap {
    rb_texture values;
    float* world_to_env;
} rb_denvmap;

/* DScene -- src/scene.h DScene / src/redner.cpp:75-82 */
typedef struct rb_dscene_desc {
    rb_dcamera camera;
    int num_shapes;
    const rb_dshape* shapes; /* host array */
    int num_materials;
    const rb_material* materials; /* host array; texel pointers are gradient buffers */
    int num_lights;
    float* const* light_intensity; /* host array of device pointers (3 floats each) -- src/area_light.h:38-43 */
    const rb_denvmap* envmap;      /* host pointer or NULL */
    /* Gradients of the lights' emission textures (rb_area_light::emission): a host array of num_lights gradient pyramids (device memory),
     * or NULL for none.  An entry with num_levels == 0 wants no gradient; then neither the texels and uv_scale nor the uvs and vertex
     * positions receive what flows through that light's texture.  Otherwise the entry has the levels, sizes and channels of the scene's
     * texture (rb_render refuses anything else, naming the emission texture), and uv_scale (2 floats) may be NULL.  The intensity gradient
     * of a textured light is sum(d_Le * E(uv)). */
    const rb_texture* light_emission;
} rb_dscene_desc;

typedef struct rb_scene rb_scene;

/* Scene::Scene (src/scene.cpp:63-307): flattens the scene, builds the triangle BVH (replaces Embree / OptiX Prime,
 * src/scene.cpp:78-155), the light PMF/CDF and per-light area CDFs (src/scene.cpp:197-253), the edge list and
 * primary-edge distribution (src/edge.cpp:233-383). */
int rb_scene_create(const rb_scene_desc* desc, rb_scene** out);
/* The same on a caller-chosen CUDA stream (a cudaStream_t; NULL == legacy default stream, which is what rb_scene_create uses): uploads,
 * mesh read-back and build kernels are ordered after the work already queued on that stream -- pass the stream the geometry tensors
 * were produced on.  rb_scene_set_camera and rb_scene_destroy keep using it. */
int rb_scene_create_on_stream(const rb_scene_desc* desc, rb_scene** out, void* stream);
/* Re-target an existing scene at a descriptor of the SAME structure, without building a new scene (an optimisation step that moves
 * vertices or changes materials, lights or the camera).  The structure is:
 *   - the numbers of shapes, materials and lights;
 *   - per shape: num_vertices, num_triangles, num_uv_vertices, num_normal_vertices, material_id, light_id, and which optional
 *     buffers (uvs, normals, uv_indices, normal_indices, colors) are present;
 *   - per light: shape_id;
 *   - the presence of the environment map, both edge-sampling flags, gpu_index and the largest generic texture dimension.
 * All of it is checked before any work; on a mismatch the call fails with a message and the scene is left unchanged and usable.
 * The CONTENTS of every index buffer must be those of the build as well: the caller promises this, the library does not check it.
 * Any pointer may change, and so may every value passed by value (camera, light intensities, the environment map's matrices and
 * pdf_norm).
 * The build reads vertex positions in place, so an in-place write to them is invisible to the library: pass geometry_changed != 0
 * after one.  Texels are read in place too: the emission-sampling tables (rb_area_light::emission_sampling) are rebuilt from them by every
 * update, and an in-place texel write without one leaves them stale, which keeps the image unbiased but noisier.  Then -- or when any `vertices` pointer changed -- the BVH, the light areas and area CDFs, the environment map's
 * bounding sphere, the edge list and the camera-dependent tables are rebuilt.  Otherwise, when the camera or the pixel filter differs by
 * value, only the camera-dependent tables are, as rb_scene_set_camera does (but on the host for the small scenes whose build made them there, so
 * that they stay the build's tables byte for byte).  The shape / material descriptors, the lights and the light PMF / CDF are
 * refreshed on every call.
 * After a successful update every table of the scene is the one rb_scene_create would build from the same descriptor, byte for
 * byte.  `stream` becomes the scene's stream (as with rb_scene_create_on_stream), rb_scene_build_ms reports this update and the
 * partition of rb_scene_set_partition is kept.  After rb_scene_set_camera on a scene whose build made the camera-dependent tables on
 * the host, the next update makes them on the host again.  A failure after the checks (a BVH too deep for the traversal stack, a
 * total light importance that is not positive, a device error) leaves the scene incomplete: rb_render and rb_scene_set_camera refuse
 * it, and the next rb_scene_update rebuilds every table whatever geometry_changed says. */
int rb_scene_update(rb_scene* scene, const rb_scene_desc* desc, int geometry_changed, void* stream);
void rb_scene_destroy(rb_scene* scene);
/* Scene::max_generic_texture_dimension (src/scene.cpp:293-300, bound at src/redner.cpp:72) */
int rb_scene_max_generic_texture_dimension(const rb_scene* scene);

/* compute_num_channels (src/channels.cpp:42-113, bound at src/redner.cpp:201) */
int rb_compute_num_channels(const int* channels, int num_channels, int max_generic_texture_dimension);

/* render (src/pathtracer.cpp:177-958, declared src/pathtracer.h:25-31, bound at src/redner.cpp:257).
 * Forward pass <=> rendered_image != NULL; backward pass <=> d_rendered_image != NULL (then d_scene is required).
 * screen_gradient_image may be NULL.  `stream` is a cudaStream_t (NULL == legacy default stream); the call
 * synchronises the stream before returning, like the reference (src/pathtracer.cpp:947-949). */
int rb_render(const rb_scene* scene, const rb_options* options, float* rendered_image, const float* d_rendered_image,
              const rb_dscene_desc* d_scene, float* screen_gradient_image, void* stream);

/* Re-target a scene at another camera.  Only what depends on the camera is rebuilt, on the device: the primary-edge distribution
 * (src/edge.cpp:298-331) and the two secondary-edge trees (src/edge_tree.cpp:724-882); geometry, BVH, light tables and the edge
 * list are kept, and so is the scene's pixel filter.  (The reference rebuilds the whole Scene per view, pyredner/render_pytorch.py:608-617.) */
int rb_scene_set_camera(rb_scene* scene, const rb_camera* camera);

/* A batch of views of one scene -- the native form of the per-view Python loops of pyredner/render_utils.py:407-430 and of
 * BASELINE config 5: for k in [0, num_views): rb_scene_set_camera(cameras[k]) then rb_render(options[k], images[k], d_images[k],
 * d_scenes[k]).  images / d_images / d_scenes may be NULL (or hold NULL entries) like the arguments of rb_render; gradients
 * ACCUMULATE, so one descriptor passed for every view sums the batch's gradients into one set of buffers. */
int rb_render_batch(rb_scene* scene, int num_views, const rb_camera* cameras, const rb_options* options, float* const* images,
                    const float* const* d_images, const rb_dscene_desc* const* d_scenes, void* stream);

/* Multi-GPU tile sharding (no reference counterpart; SURVEY.md section 8e).  Restricts subsequent rb_render calls on
 * this scene to the rows r with (r / rows_per_stripe) % num_parts == part of the viewport, while samplers stay
 * seeded by the full-viewport pixel index, so the union over parts equals the single-GPU result.  Primary-edge
 * samples are sharded by sample index.  num_parts == 1 restores the full image. */
int rb_scene_set_partition(rb_scene* scene, int part, int num_parts, int rows_per_stripe);

/* Statistics of the last rb_render on this scene: number of kernels launched and device milliseconds (CUDA events on
 * the render stream) spent inside the traced kernels. */
int rb_scene_last_stats(const rb_scene* scene, int* num_kernel_launches, float* kernel_ms);

/* Per-kernel device times of the last rb_render (CUDA events on the render stream), in launch order
 * { k_forward, backward bands (trace + boundary terms + sweep), k_primary_edge, k_finish_camera } (0 for kernels that
 * did not run), the number of path
 * vertices at which the last backward pass formed a radiance estimate and its number of primary hits (mean executed
 * bounces per sample = path_vertices / (W*H*spp), SURVEY.md section 8d).  Both count the samples the backward pass traced:
 * it skips the samples of pixels whose d_rendered_image is exactly zero in every float. */
int rb_scene_last_stage_stats(const rb_scene* scene, float* stage_ms4, double* path_vertices, double* primary_hits);
/* Split of the backward bands of the last rb_render, summed over the bands:
 * { k_bwd_trace, scan + compaction + k_bwd_secondary, k_bwd_sweep } in milliseconds. */
int rb_scene_last_backward_stats(const rb_scene* scene, float* bwd_ms3);
/* Work of the backward bands of the last rb_render: the samples of the owned pixels whose d_rendered_image is not exactly zero in
 * every float (every owned sample with RB_NO_ZERO_CULL=1), which are the only ones the bands run over, and the number of bands they
 * took.  Both are 0 after a call without d_rendered_image. */
int rb_scene_last_live_samples(const rb_scene* scene, long long* live_samples, long long* num_bands);
/* Bytes of exact gradient accumulators (rb_options::deterministic) the last rb_render on this scene took from the backward scratch:
 * 88 per accumulator, one per camera scalar and per float of the gradient buffers (overlapping buffers share them), plus a spare;
 * 0 when the last call was not a deterministic backward pass. */
int rb_scene_last_exact_bytes(const rb_scene* scene, size_t* bytes);
/* Deterministic gradients summed over several calls, devices or processes (for example the stripes of rb_scene_set_partition on one
 * GPU per rank).  Each call hands out its exact accumulators as RECORDS instead of rounding them; the caller sums the records, word by
 * word in signed 64-bit integers (an all-reduce SUM), and rounds the sum once.  The gradients are then those of ONE deterministic
 * rb_render over all the samples, bit for bit, however the samples were split.
 * A record is 13 signed 64-bit words: 10 limbs of a fixed-point number (limb k weighs 2^(32 k - 149)) and three counts of non-finite
 * contributions (+inf, -inf, NaN).  There are `count` records: one per camera gradient scalar, then one per float of every gradient
 * buffer of d_scene and screen_gradient_image, in the order: shapes (vertices, uvs, normals, colors), materials (the five textures:
 * levels, then uv_scale), light intensities, the lights' emission textures (for every light with one, when d_scene->light_emission is
 * not NULL: levels, then uv_scale), the environment map (levels, uv_scale, world_to_env), the screen-gradient image.  The
 * position of a record depends on the structure of the descriptor only, never on where its buffers are; descriptors whose gradient
 * buffers overlap are refused.  `fingerprint` hashes that structure: compare it across ranks before summing.  Records live in memory
 * of the scene's device; `stream` as for rb_render, and both calls synchronise it. */
int rb_exact_record_count(const rb_scene* scene, const rb_options* options, const rb_dscene_desc* d_scene, float* screen_gradient_image, size_t* count,
                          uint64_t* fingerprint);
/* The backward pass of rb_render in deterministic mode (whatever options->deterministic says), except its end: instead of rounding,
 * every accumulator is ADDED into records[0, count) (zeroed by the caller, or holding the records of earlier calls), which are left
 * normalised.  No buffer of d_scene or screen_gradient_image is written: their pointers only give the layout. */
int rb_render_exact(const rb_scene* scene, const rb_options* options, const float* d_rendered_image, const rb_dscene_desc* d_scene,
                    float* screen_gradient_image, long long* records, size_t count, void* stream);
/* The end of a deterministic rb_render on records (any sum of records of this layout): every record that holds a non-zero value or a
 * non-finite count is rounded once and added into the caller's gradient buffer, and the camera gradients are finished with the scene's
 * camera.  Records that sum to zero leave their element untouched, as in rb_render. */
int rb_exact_round(const rb_scene* scene, const rb_options* options, const rb_dscene_desc* d_scene, float* screen_gradient_image, const long long* records,
                   size_t count, void* stream);
/* rb_render keeps one grow-only scratch allocation per device for the backward pass (gradient descriptors, path
 * records, work lists; at most ~1 GiB + small).  This frees them all; the next backward pass allocates again. */
void rb_release_scratch(void);
/* Host wall-clock milliseconds the last rb_scene_create or rb_scene_update spent in { BVH build, light tables, edge list + edge tree }. */
int rb_scene_build_ms(const rb_scene* scene, float* bvh_lights_edges3);

/* Test hook: the secondary-edge trees as the kernels see them.  info3 = { number of 128-byte records, root reference of the
 * camera-silhouette tree, root reference of the other tree } (reference >= 0: record index, < 0: ~edge id, INT_MIN: empty tree);
 * *expand = billboard size (src/edge_tree.cpp:773); records_out (may be NULL) receives up to records_bytes of the records. */
int rb_scene_edge_trees(const rb_scene* scene, int* info3, float* expand, void* records_out, size_t records_bytes);
/* Test hook: the scene's edge list (what collect_edges builds, src/edge.cpp:233-296): *num_edges, and up to edges_bytes of
 * { shape, v0, v1, f0, f1 } int records into edges_out (may be NULL). */
int rb_scene_edge_list(const rb_scene* scene, int* num_edges, int* edges_out, size_t edges_bytes);

/* Test hook: one table of the scene as the kernels see it.  *size (may be NULL) receives its size in bytes; out (may be NULL) receives
 * up to `bytes` of it. */
enum rb_scene_table_id {
    RB_TABLE_BVH_NODES = 0,      /* triangle BVH inner nodes (scene triangles - 1 of them) */
    RB_TABLE_BVH_TRIANGLES,      /* triangles in BVH leaf order */
    RB_TABLE_LIGHT_PMF,          /* double per light, the environment map last (src/scene.cpp:197-253) */
    RB_TABLE_LIGHT_CDF,
    RB_TABLE_LIGHT_AREAS,        /* double per area light */
    RB_TABLE_AREA_CDF_POOL,      /* double per emissive triangle: every light's triangle-area CDF */
    RB_TABLE_AREA_CDF_OFFSETS,   /* int per area light: first entry in the pool */
    RB_TABLE_PRIMARY_EDGE_PMF,   /* double per edge (src/edge.cpp:298-331); empty without primary-edge sampling */
    RB_TABLE_PRIMARY_EDGE_CDF,
    RB_TABLE_LIGHTS,             /* the area lights as the kernels read them: { shape_id, intensity, two_sided, directly_visible } per light
                                    (24 bytes), then from the next 16-byte boundary the lights' emission textures (rb_texture each) */
    RB_TABLE_LIGHT_SAMPLING      /* doubles, for every light that samples by its emission texture (RB_EMISSION_SAMPLE_TEXTURE with a texture
                                    that is not constant), in light order: { S, 0 } (S: the sum of the triangle weights a_t), the w x h cell
                                    weights of level 0 (row-major), their w x h summed-area table, then per triangle { x0, y0, x1, y1, M_t,
                                    a_t, CDF_t, pdf factor } (DESIGN.md "Emission sampling"); empty when no light does */
};
int rb_scene_table(const rb_scene* scene, int which, void* out, size_t bytes, size_t* size);

/* Test hook: ray queries against the scene's triangle BVH.  All three buffers are memory of the scene's device.  rays: 8 floats per ray, { origin xyz,
 * tnear, direction xyz, tfar }; ids receives { shape id, triangle id } per ray, { -1, -1 } for a miss; t the hit distance, tfar for a
 * miss.  Without flags the query is the closest-hit traversal the render kernels call (rb_bvh.cuh, bvh_trace_impl), on the scene's own
 * nodes, leaf triangles and root; RB_TRACE_ANY_HIT asks for its any-hit form.  RB_TRACE_BRUTE_FORCE skips the tree: the same triangle
 * test on every leaf triangle in leaf order, with the traversal's early-outs (no triangles, |dir|^2 <= 1e-3, tfar < tnear); a closer hit
 * replaces the best one only with a strictly smaller t, and an any-hit query stops at the first hit.  The exact answer the traversal
 * must give.  Synchronises the device before and after. */
enum rb_trace_flags { RB_TRACE_ANY_HIT = 1, RB_TRACE_BRUTE_FORCE = 2 };
int rb_scene_trace_rays(const rb_scene* scene, const float* rays, int num_rays, int flags, int* ids, float* t);

/* Test hook: exact sums through the scatter of the deterministic backward pass (warp aggregation and integer reductions included).
 * values (float) and slots (int) are n device entries; contribution j of [0, n * repeat) adds values[j % n] to slot slots[j % n], so
 * `repeat` drives slots past the per-accumulator bound between normalisations.  out_f32 / out_f64 (device, num_slots entries) receive
 * each slot's sum rounded to float and to double (+0 for a slot without contributions).  Synchronises `stream`. */
int rb_exact_sum_test(const float* values, const int* slots, int n, int num_slots, long long repeat, float* out_f32, double* out_f64, void* stream);

/* Test hook: n texture lookups, one per thread, through the lookup and its adjoint that the render kernels call (rb_material.cuh).
 * queries: [n, 6] floats per lookup { u, v, du/dx, du/dy, dv/dx, dv/dy }; values receives [n, channels].  1 and 3 channels take the
 * BSDF's path (tex_eval from channel 0), other counts the generic texture's (tex_eval_channels).  With d_values ([n, channels]) the
 * adjoint (d_tex_eval) scatters into d_tex -- same levels, sizes and channels as tex, zeroed by the caller, uv_scale may be NULL --
 * and d_queries (may be NULL) receives { d_u, d_v, d(du/dx), d(du/dy), d(dv/dx), d(dv/dy) } per lookup.  Every buffer is memory of the
 * current device; a negative n, channels < 1, num_levels outside [1, RB_MAX_MIP_LEVELS] or a level without a size (unless the
 * texture is constant) are refused.  Runs on `stream` (a cudaStream_t, NULL == legacy default stream) and synchronises it. */
int rb_texture_test(const rb_texture* tex, const rb_texture* d_tex, const float* queries, int n, const float* d_values, float* values,
                    float* d_queries, void* stream);

/* Test hook: n environment-map lookups and m samples, one per thread, through the functions the render kernels call (rb_envmap.cuh).
 * `env` is turned into the scene's map exactly as rb_scene_create does.  queries: [n, 9] floats { dir, dir_dx, dir_dy } per lookup;
 * values receives [n, 3] (envmap_eval) and pdfs, unless NULL, [n] (envmap_pdf of dir).  With d_out ([n, 3]) the adjoint
 * (d_envmap_eval) scatters into d_values -- the map's levels, sizes and channels, zeroed by the caller, uv_scale may be NULL -- and, unless
 * NULL, into d_w2e (16 floats, row-major 4x4); d_queries (may be NULL) receives { d_dir, d_dir_dx, d_dir_dy } per lookup.  samples: [m, 2]
 * doubles (sx, sy) for envmap_sample; sample_dirs receives [m, 3].  Every buffer is memory of the current device; negative counts, a map
 * without 3 channels or positive level sizes, and a gradient pyramid of another shape are refused, as is the double-precision build.
 * Runs on `stream` (a cudaStream_t, NULL == legacy default stream) and synchronises it. */
int rb_envmap_test(const rb_envmap* env, const rb_texture* d_values, float* d_w2e, const float* queries, int n, const float* d_out, float* values,
                   float* pdfs, float* d_queries, const double* samples, int m, float* sample_dirs, void* stream);

/* Test hook: the point-on-light sampler and its density for area light `light` of a built scene, through the functions the render
 * kernels call (rb_path.cuh).  samples: [n, 3] doubles (tri_sel, su, sv); ints receives [n, 3] { branch (0: by area, 1: by texture),
 * triangle, rejected }; doubles receives [n, 3] { b1, b2, density }, where (b1, b2) are the barycentrics of the point as the light-sample
 * record reproduces it and density the area density of that point evaluated from the record (0 for a rejected sample).  queries: [m, 3]
 * floats { triangle, u, v } (u, v: the light's texture coordinate before uv_scale); query_pdfs receives the area density at each.  The
 * densities do not include the light-selection probability; a query whose triangle is out of range gets NaN.  Every buffer is memory of
 * the scene's device; a light out of range and a negative count are refused.  Runs on `stream` and synchronises it. */
int rb_light_sample_test(const rb_scene* scene, int light, const double* samples, int n, int* ints, double* doubles, const float* queries, int m,
                         double* query_pdfs, void* stream);

/* Test hook: n camera queries of one kind (`op`), one per thread, through the camera functions the render kernels call (rb_camera.cuh,
 * rb_render.cuh), on the camera of a built scene (rb_scene_set_camera re-targets it).  in: [n, 64] doubles, out: [n, 64] doubles, one row per
 * query; acc: NULL, or [cam_acc_count, n] floats (cam_acc_count: 58, 60 with a lens), the camera-gradient accumulator with query i's column
 * at acc + i (stride n), which the adjoint ops add to.  lu below is concentric_disc(u1, u2).  Rows (indices):
 *   RB_CAMTEST_CAMERA      out: c2w 0-15, w2c 16-31, intr_inv 32-40, intr 41-49, distortion 50-57, lens_radius 58, focus_distance 59,
 *                          clip_near 60, cam_acc_count 61 (the DevCamera the kernels see)
 *   RB_CAMTEST_RAY         in: sx, sy, u1, u2.  out: cam_sample_primary org 0-2, dir 3-5 (double); cam_primary_ray org 6-8, dir 9-11,
 *                          org_dx 12-14, org_dy 15-17, dir_dx 18-20, dir_dy 21-23 (float); lu 24-25
 *   RB_CAMTEST_D_RAY       in: sx, sy, u1, u2, d_org 4-6, d_dir 7-9, want d_screen 10, d(org_dx, org_dy, dir_dx, dir_dy) 11-22, with the
 *                          differential 23.  d_cam_sample_primary at ((float)sx, (float)sy) or, with the differential, the adjoint of
 *                          cam_primary_ray as bwd_sweep forms it (d_cam_primary_ray_diff, then d_cam_sample_primary of the three rays); out:
 *                          d_screen 0-1
 *   RB_CAMTEST_PROJECT     in: p0 0-2, p1 3-5, u1 6, u2 7.  out: cam_project_d (cam_project_lens_d with a lens) visible 0, q0 1-2, q1 3-4;
 *                          cam_project of the float ends visible 5, q0 6-7, q1 8-9
 *   RB_CAMTEST_D_PROJECT   in: p0 0-2, p1 3-5 (rounded to float), u1 6, u2 7, d_q0 8-9, d_q1 10-11.  d_cam_project (d_cam_project_lens with a
 *                          lens); out: d_p0 0-2, d_p1 3-5
 *   RB_CAMTEST_DISTORT     in: pos 0-1, d_out 2-3.  out: cam_distort 0-1 with Jacobian rows d(x)/d(pos) 2-3, d(y)/d(pos) 4-5;
 *                          cam_inverse_distort 6-7; d_pos of d_cam_distort 8-9 and of d_cam_inverse_distort 10-11; their parameter
 *                          gradients 12-19 and 20-27
 *   RB_CAMTEST_FINISH      in: the 60 reduced accumulator doubles.  out: finish_camera's d(position) 0-2, d(look) 3-5, d(up) 6-8 (look-at
 *                          cameras), d(cam_to_world) 9-24 (the others), d(intrinsic_mat_inv) 25-33, d(intrinsic_mat) 34-42, d(distortion)
 *                          43-50, d(lens) 51-52
 * Every buffer is memory of the scene's device; an unknown op, a negative count and an adjoint op without `acc` are refused, as is the
 * double-precision build.  Runs on `stream` and synchronises it. */
enum {
    RB_CAMTEST_CAMERA = 0, RB_CAMTEST_RAY = 1, RB_CAMTEST_D_RAY = 2, RB_CAMTEST_PROJECT = 3, RB_CAMTEST_D_PROJECT = 4, RB_CAMTEST_DISTORT = 5,
    RB_CAMTEST_FINISH = 6
};
int rb_camera_test(const rb_scene* scene, int op, const double* in, int n, double* out, float* acc, void* stream);

/* Test hook: n geometry queries of one kind (`op`), one per thread, through the functions of rb_shape.cuh and the gradient scatters of
 * rb_path.cuh that the render kernels call, on the shapes of a built scene.  in: [n, 96] doubles, out: [n, 96] doubles, one row per query;
 * every row starts with the shape and triangle index (0, 1).  Inputs are rounded to float, as the kernels hold them.  A SurfacePoint is
 * 35 numbers: position 0-2, geom_normal 3-5, shading frame x 6-8, y 9-11, n 12-14, dpdu 15-17, uv 18-19, du_dxy 20-21, dv_dxy 22-23,
 * dn_dx 24-26, dn_dy 27-29, color 30-32, bary 33-34; a ray differential 12: org_dx, org_dy, dir_dx, dir_dy.  Rows (indices):
 *   RB_SURFTEST_POINT    in: ray org 2-4, dir 5-7, differential 8-19.  out: tri_solve's u, v, t 0-2, u_dxy 3-4, v_dxy 5-6, t_dxy 7-8;
 *                        make_surface_point's SurfacePoint 9-43 and rd_out 44-55; its decisions (0 / 1): the uv determinant is 0 56,
 *                        the geometric normal flipped 57, the frame's y degenerate 58, coordinate_system's n.z < -1 + 1e-6 branch at
 *                        the unflipped geometric normal 59 and at the shading normal 60; the uv determinant 61
 *   RB_SURFTEST_D_POINT  in: the POINT inputs 2-19, d(SurfacePoint) 20-54, d(rd_out) 55-66.  out: d_make_surface_point's d_ray org 0-2,
 *                        dir 3-5, d(ray differential) 6-17, d_vp 18-26, d_vn 27-35, d_vuv 36-41, d_vc 42-50 (per corner, zero-seeded);
 *                        with d_shapes, scatter_vertex_grads adds them to the shape's gradient buffers
 *   RB_SURFTEST_LIGHT    in: su 2, sv 3.  out: sample_light_triangle's position 0-2, geom_normal 3-5, frame x 6-8, y 9-11, n 12-14,
 *                        bary 15-16, uv (the sample) 17-18; light_sample_uv 19-20; shape_tri_area 21
 *   RB_SURFTEST_D_LIGHT  in: su 2, sv 3, d(position) 4-6, d(geom_normal) 7-9, d(frame x, y, n) 10-18, d(area) 19, d(uv) 20-21.
 *                        out: d_sample_light_triangle's d_v 0-8, d_shape_tri_area's d_v 9-17; with d_shapes, d_light_sample_uv adds
 *                        d(uv) to the shape's uv gradient
 * d_shapes: NULL, or a host array of one rb_dshape per shape of the scene (device buffers, any may be NULL), scattered into with the
 * kernels' warp-aggregated atomics.  `in` and `out` are memory of the scene's device.  An unknown op, a negative count, a shape or
 * triangle index out of range, and the double-precision build are refused.  Runs on `stream` and synchronises it. */
enum { RB_SURFTEST_POINT = 0, RB_SURFTEST_D_POINT = 1, RB_SURFTEST_LIGHT = 2, RB_SURFTEST_D_LIGHT = 3 };
int rb_surface_test(const rb_scene* scene, int op, const double* in, int n, double* out, const rb_dshape* d_shapes, void* stream);

const char* rb_last_error(void);
const char* rb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* REDNER_B200_H */
