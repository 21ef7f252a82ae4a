// Device-side scene description shared by all kernels.
#pragma once
#include <cstring>
#include <vector>

#include "../../include/redner_b200.h"
#include "rb_math.cuh"

// ---- rays and path vertices (reference: src/ray.h:9-41, src/intersection.h:8-51) ----
struct Ray {
    V3 org, dir;
    Real tmin, tmax;
};
struct RayDiff {
    V3 org_dx, org_dy, dir_dx, dir_dy;
};
struct DRay {
    V3 org, dir;
};
RB_HD RayDiff zero_raydiff() {
    RayDiff r;
    r.org_dx = r.org_dy = r.dir_dx = r.dir_dy = zero3();
    return r;
}
RB_HD DRay zero_dray() {
    DRay r;
    r.org = r.dir = zero3();
    return r;
}
struct Isect {
    int shape_id, tri_id;
    RB_HD bool valid() const { return shape_id >= 0 && tri_id >= 0; }
};
RB_HD Isect no_isect() {
    Isect i;
    i.shape_id = -1;
    i.tri_id = -1;
    return i;
}
struct SurfacePoint {
    V3 position;
    V3 geom_normal;
    Frame shading_frame;
    V3 dpdu;
    V2 uv;
    V2 du_dxy, dv_dxy;
    V3 dn_dx, dn_dy;
    V3 color;
    V2 bary;
};
RB_HD SurfacePoint zero_point() {
    SurfacePoint p;
    p.position = p.geom_normal = zero3();
    p.shading_frame = zero_frame();
    p.dpdu = zero3();
    p.uv = p.du_dxy = p.dv_dxy = zero2();
    p.dn_dx = p.dn_dy = p.color = zero3();
    p.bary = zero2();
    return p;
}

// ---- camera (double precision copies of the host-read parameters; src/camera.h:72-82) ----
struct DevCamera {
    int width, height;
    int use_look_at;
    // thin lens (rb_camera::lens_radius / focus_distance); lens_radius == 0: the pinhole, focus_distance is then 0 as well.  The two floats
    // sit in what was alignment padding, so that DevCamera, and the kernels' parameter layout behind it, keep their size and offsets.
    float lens_radius;
    double position[3], look[3], up[3];
    double c2w[16], w2c[16];
    double intr_inv[9], intr[9];
    float clip_near;
    int type;
    int vp_beg[2], vp_end[2];
    int has_distortion;   // Brown-Conrady lens model, src/camera_distortion.h
    float focus_distance; // (thin lens, see lens_radius)
    double distortion[8]; // k1..k6 (radial, rational), p1, p2 (tangential)
    // the scene's pixel filter (rb_scene_desc::pixel_filter, { 0, 0 } made { RB_FILTER_BOX, 1 }); rb_scene_set_camera keeps it
    int filter_type;
    float filter_width;
};

// ---- BVH (own LBVH; replaces Embree/OptiX Prime) ----
#define RB_BVH_STACK 64 // traversal stack entries per ray; rb_build_bvh refuses trees that could overflow it
// Node i stores the AABBs of BOTH children so that one 64-byte fetch decides the descent.
// child index >= 0: inner node; < 0: leaf, triangle slot = ~child.
struct __align__(16) BVHNode {
    float4 lo_x_hi_x; // (l.min.x, l.max.x, r.min.x, r.max.x)
    float4 lo_y_hi_y;
    float4 lo_z_hi_z;
    int left, right;
    int pad0, pad1;
};
// Triangle in BVH (sorted) order: three vertices (w of v0/v1 carry shape_id / tri_id bits).
struct __align__(16) BVHTri {
    float4 v0; // .w = __int_as_float(shape_id)
    float4 v1; // .w = __int_as_float(tri_id)
    float4 v2;
};

// ---- edges (src/edge.h:13-31) ----
struct Edge {
    int shape_id, v0, v1, f0, f1;
};

struct DevLight {
    int shape_id;
    float intensity[3];
    int two_sided, directly_visible;
};

// Secondary-edge trees (own flat layout; replaces the pointer-linked BVHNode3 / BVHNode6 of src/edge_tree.h:14-30).  One 128-byte
// record per INNER node holding BOTH children's bounds: every step of the two edge-tree walks is one fetch followed by
// arithmetic, instead of "load node, then load its two children" (the walks are bound by those dependent loads).  The camera-silhouette tree only uses the position
// box, the other tree also the box in Hough space (src/edge_tree.cpp:23-66).
// A child reference is >= 0: index of an inner node, < 0: leaf, edge id = ~ref; RB_EDGE_EMPTY: no tree.
#define RB_EDGE_EMPTY ((int)0x80000000)
struct EdgeChild {
    float pmin[3], pmax[3];
    float dmin[3], dmax[3];
    float wlen; // sum of length * exterior dihedral angle below this child
    int ref;
};
struct __align__(16) EdgeNode {
    EdgeChild c[2];
    int pad[4];
};

// EnvironmentMap, src/envmap.h:19-51 (the texture and the two sampling tables are caller-owned device memory)
struct DevEnvmap {
    rb_texture values;
    float w2e[16], e2w[16];
    const float* cdf_ys; // [height]
    const float* cdf_xs; // [height][width]
    float pdf_norm;
    int directly_visible;
};

struct DevScene {
    DevCamera cam;
    const rb_shape* shapes;
    int num_shapes;
    const rb_material* materials;
    int num_materials;
    const DevLight* lights;
    int num_lights; // area lights + 1 if there is an environment map (it is the LAST entry of light_pmf / light_cdf)
    int has_envmap;
    DevEnvmap env;
    const double* light_pmf;
    const double* light_cdf;
    const double* light_areas;
    const double* area_cdf_pool;
    const int* area_cdf_offset; // per light, offset into the pool
    // triangle BVH
    const BVHNode* bvh_nodes;
    const BVHTri* bvh_tris;
    int bvh_root; // >=0 inner, <0 single leaf, or INT_MIN when the scene is empty
    int num_tris;
    // edges
    const Edge* edges;
    int num_edges;
    const double* prim_edge_pmf;
    const double* prim_edge_cdf;
    // secondary edge trees
    const EdgeNode* edge_nodes;
    int edge_root_cs, edge_root_ncs; // camera-silhouette tree / rest: child reference of the root (RB_EDGE_EMPTY if empty)
    float edge_bounds_expand;
    const float* ltc_table;
    // samplers
    const unsigned long long* sobol_matrices; // [dims][52]
    int sobol_dims;
    int use_primary_edge, use_secondary_edge;
};

// Gradient targets (device pointers supplied by the caller) + internal accumulators.
struct DevDScene {
    const rb_dshape* shapes;
    const rb_material* materials; // texel pointers are gradient buffers
    float* const* light_intensity;
    rb_texture env_values; // gradient mip pyramid of the environment map (num_levels == 0: none)
    float* env_w2e;        // 16 floats, gradient of world_to_env
    // internal double accumulators for the camera (reduced per block, finished by one tiny kernel):
    // [0..15] d_cam_to_world, [16..31] d_world_to_cam, [32..40] d_intrinsic_mat_inv, [41..49] d_intrinsic_mat, ... (CamAcc, rb_camera.cuh)
    double* cam_accum;
};

// Emission textures of the area lights (rb_area_light::emission) and their gradients sit in tables of their own, so that DevLight,
// DevScene and DevDScene keep the layout the lean and diffuse-only kernels are compiled against.  The scene's table follows its DevLight
// array in the same allocation; the gradient table of a backward pass follows the array of intensity-gradient pointers that
// DevDScene::light_intensity points at.  Each starts at the first 16-byte boundary after its array and holds one rb_texture per area
// light (num_levels == 0: no texture, or no gradient).  Only kernels with RB_LIGHT_TEX read them.
RB_HD size_t light_table_offset(size_t array_bytes) { return (array_bytes + 15) & ~(size_t)15; }
RB_HD int num_area_lights(const DevScene& sc) { return sc.num_lights - (sc.has_envmap ? 1 : 0); }
RB_HD const rb_texture& light_emission(const DevScene& sc, int l) {
    return ((const rb_texture*)((const char*)sc.lights + light_table_offset((size_t)num_area_lights(sc) * sizeof(DevLight))))[l];
}
RB_HD const rb_texture& light_d_emission(const DevScene& sc, const DevDScene& ds, int l) {
    return ((const rb_texture*)((const char*)ds.light_intensity + light_table_offset((size_t)num_area_lights(sc) * sizeof(float*))))[l];
}
// Host image of such a table: the n entries of `head`, then the n textures of `tex` (zeroed when `tex` is null), in 8-byte words.
template <typename T>
inline std::vector<unsigned long long> light_table_words(const T* head, const rb_texture* tex, int n) {
    const size_t off = light_table_offset((size_t)n * sizeof(T));
    std::vector<unsigned long long> w((off + (size_t)n * sizeof(rb_texture) + 7) / 8, 0ull);
    if (n > 0) {
        memcpy(w.data(), head, (size_t)n * sizeof(T));
        if (tex) memcpy((char*)w.data() + off, tex, (size_t)n * sizeof(rb_texture));
    }
    return w;
}
// Emission sampling (rb_area_light::emission_sampling, DESIGN.md "Emission sampling").  The scene's light table ends with one more 8-byte
// word after the emission textures: 0, or the address of L LightSampling descriptors, when some light samples by its texture.  A light
// whose descriptor has data == nullptr, or whose S = data[0] is 0, samples by area.  data points at { S, 0 }, the w x h cell weights, their
// w x h summed-area table and 8 doubles per triangle (ls_cells / ls_sat / ls_tris, rb_light_build.cuh).  The word is not part of
// RB_TABLE_LIGHTS, so that table is what it was for every scene.
struct LightSampling {
    const double* data;
    int w, h;
};
RB_HD size_t light_sampling_word(int num_area_lights) { return light_table_offset((size_t)num_area_lights * sizeof(DevLight)) + (size_t)num_area_lights * sizeof(rb_texture); }
RB_HD const LightSampling* light_sampling_table(const DevScene& sc) {
    return *(const LightSampling* const*)((const char*)sc.lights + light_sampling_word(num_area_lights(sc)));
}

// True when some light has an emission texture (RB_LIGHT_TEX), i.e. when only the general and deterministic kernels compute what the
// scene asks for.
inline bool lights_use_emission(const std::vector<rb_texture>& emission) {
    for (const rb_texture& t : emission)
        if (t.num_levels > 0) return true;
    return false;
}

struct RenderParams {
    unsigned long long seed;
    int spp;
    int max_bounces;
    int sampler_type;
    int sample_pixel_center;
    int nd;        // total image dimensions per pixel
    int rad_dim;   // float offset of the radiance channel (reference stores the channel index here, see DESIGN.md)
    int rad_off;   // TRUE float offset of the radiance channel: where first-hit emission goes (src/primary_contribution.cpp:36-45)
    int num_channels;
    int channels[RB_CH_COUNT];
    int max_generic;
    int only_radiance; // channels == [radiance]: the common case, skips every G-buffer branch
    // multi-GPU partition over viewport rows
    int part, num_parts, rows_per_stripe;
    int vp_w, vp_h;
};
