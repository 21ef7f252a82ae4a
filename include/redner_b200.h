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

/* Material -- src/material.h:12-91; DMaterial (src/material.h:93-99) uses the same layout with gradient buffers. */
typedef struct rb_material {
    rb_texture diffuse_reflectance;  /* 3 channels */
    rb_texture specular_reflectance; /* 3 channels */
    rb_texture roughness;            /* 1 channel */
    rb_texture generic_texture;      /* N channels, optional */
    rb_texture normal_map;           /* 3 channels, optional */
    int compute_specular_lighting, two_sided, use_vertex_color;
} rb_material;

/* AreaLight -- src/area_light.h:8-36 */
typedef struct rb_area_light {
    int shape_id;
    float intensity[3];
    int two_sided, directly_visible;
} rb_area_light;

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
 * after one.  Then -- or when any `vertices` pointer changed -- the BVH, the light areas and area CDFs, the environment map's
 * bounding sphere, the edge list and the camera-dependent tables are rebuilt.  Otherwise, when the camera differs by value, only the
 * camera-dependent tables are, as rb_scene_set_camera does (but on the host for the small scenes whose build made them there, so
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
 * list are kept.  (The reference rebuilds the whole Scene per view, pyredner/render_pytorch.py:608-617.) */
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
 * bounces per sample = path_vertices / (W*H*spp), SURVEY.md section 8d). */
int rb_scene_last_stage_stats(const rb_scene* scene, float* stage_ms4, double* path_vertices, double* primary_hits);
/* Split of the backward bands of the last rb_render, summed over the bands:
 * { k_bwd_trace, scan + compaction + k_bwd_secondary, k_bwd_sweep } in milliseconds. */
int rb_scene_last_backward_stats(const rb_scene* scene, float* bwd_ms3);
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
 * levels, then uv_scale), light intensities, the environment map (levels, uv_scale, world_to_env), the screen-gradient image.  The
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
    RB_TABLE_PRIMARY_EDGE_CDF
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

const char* rb_last_error(void);
const char* rb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* REDNER_B200_H */
