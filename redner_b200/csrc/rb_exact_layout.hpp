// The exact accumulators of one deterministic backward pass (rb_options::deterministic), shared by the CUDA driver (rb_kernels.cu)
// and the host emulator (tools/cpu_emu): one accumulator per camera scalar (accumulators 0 .. RB_CAM_ACC - 1), then one per float of
// every gradient buffer the pass can write, and the gradient descriptors the kernels see in place of the caller's, whose buffer
// pointers are virtual addresses of those accumulators (rb_exact.cuh).  A NULL pointer stays NULL.  Caller buffers that overlap share
// accumulators: the memory ranges are merged before they are numbered, so every caller float has exactly one accumulator and the
// finalisation adds into it once.
//
// Accumulators are numbered in address order, which differs between processes and between descriptors of separately allocated
// buffers.  Records (rb_exact.cuh), the form in which accumulators are summed across calls and devices, are numbered by the structure
// of the descriptor alone: the camera scalars, then one record per float of every gradient buffer in the order exact_layout visits
// them -- shapes (vertices, uvs, normals, colours), materials (the five textures: their levels, then uv_scale), light intensities, the
// environment map (levels, uv_scale), world_to_env, the screen-gradient image.  Overlapping buffers have no such position: the entry
// points that take or give records (rb_exact_record_count, rb_render_exact, rb_exact_round) refuse descriptors whose gradient buffers
// overlap.  ExactLayout::fingerprint hashes that structure, so that callers can check that their records line up before they sum them.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "rb_exact.cuh"

// The exact accumulators take at most RB_EXACT_MAX_ADDS contributions between two normalisations, and the drivers normalise after
// every band of samples.  A path vertex adds fewer than RB_EXACT_ADDS_PER_VERTEX values to any one accumulator.  One texture lookup
// (d_tex_eval_mip) adds at most 8 values to one texel accumulator (2 mip levels x 4 bilinear taps, which can all land on one texel of a
// small or clamped level) and ceil(channels / 3) <= 22 to its uv_scale (one per channel triple of a 64-channel generic texture); a
// vertex evaluates the adjoint of each of its material's five textures a few times and scatters into its shape's vertex, uv, normal and
// colour buffers and the light intensities a handful of times more.  That is a few hundred adds in the worst case, where every gradient
// buffer of a material is one caller buffer, so a band of at most exact_band_samples(max_bounces) samples stays within the bound.  A
// primary-edge sample adds fewer still.  The bound is argued here, not counted at run time.
#define RB_EXACT_ADDS_PER_VERTEX 1024
inline long long exact_band_samples(int max_bounces) { return RB_EXACT_MAX_ADDS / (RB_EXACT_ADDS_PER_VERTEX * ((long long)max_bounces + 1)); }

struct ExactLayout {
    long long num_acc = 0;              // accumulators with a meaning; the array has one more, a spare (see virt below)
    std::vector<ExactRange> ranges;     // caller memory per accumulator range, sorted by `first`
    std::vector<long long> rec_first;   // record of the first float of each range (meaningful when !overlaps)
    long long num_records = 0;          // records: the camera scalars and every float of every span, in visiting order
    bool overlaps = false;              // two gradient buffers overlap (and share accumulators)
    uint64_t fingerprint = 0;           // FNV-1a of the structure: every buffer slot visited and its size (0 if absent)
    std::vector<rb_dshape> shapes;      // the descriptors with virtual addresses
    std::vector<rb_material> materials;
    std::vector<float*> lights;
    rb_texture env_values;
    float* env_w2e = nullptr;
    float* screen_grad = nullptr;
};

// Floats of every gradient buffer the backward pass of `sc` can write through `ka.ds` / `ka.screen_grad` (as set up by
// setup_backward), with shape and texture sizes from the scene's descriptors (`shapes`, `materials`): the kernels index gradient
// buffers like the scene's own buffers.
inline void exact_layout(const rb_dscene_desc& d, const rb_shape* shapes, const rb_material* materials, const DevScene& sc, const KernelArgs& ka,
                         ExactLayout& out) {
    struct Span {
        uintptr_t begin, end;
        long long rec; // record of its first float
    };
    std::vector<Span> spans;
    uint64_t h = 14695981039346656037ull;
    auto hash = [&](uint64_t v) {
        for (int b = 0; b < 8; b++) h = (h ^ ((v >> (8 * b)) & 0xffu)) * 1099511628211ull;
    };
    hash(RB_CAM_ACC);
    out.num_records = RB_CAM_ACC;
    auto add = [&](const float* p, long long n) {
        const bool present = p != nullptr && n > 0;
        hash(present ? (uint64_t)n : 0);
        if (!present) return;
        spans.push_back(Span{(uintptr_t)p, (uintptr_t)(p + n), out.num_records});
        out.num_records += n;
    };
    // a texture's gradient: `nch` floats per texel (the channel count its d_tex_eval call uses), or per level of a constant texture
    auto add_texture = [&](const rb_texture& t, const rb_texture& dt, int nch) {
        const bool constant = t.width[0] == 0 && t.height[0] == 0;
        for (int l = 0; l < t.num_levels && l < RB_MAX_MIP_LEVELS; l++)
            add(dt.texels[l], constant ? nch : (long long)std::max(t.width[l], 1) * std::max(t.height[l], 1) * nch);
        add(dt.uv_scale, 2);
    };
    for (int s = 0; s < d.num_shapes; s++) {
        const rb_shape& sh = shapes[s];
        const rb_dshape& ds = d.shapes[s];
        add(ds.vertices, 3LL * sh.num_vertices);
        add(ds.uvs, 2LL * std::max(sh.num_uv_vertices, sh.num_vertices));
        add(ds.normals, 3LL * std::max(sh.num_normal_vertices, sh.num_vertices));
        add(ds.colors, 3LL * sh.num_vertices);
    }
    for (int m = 0; m < d.num_materials; m++) {
        const rb_material &mt = materials[m], &dm = d.materials[m];
        add_texture(mt.diffuse_reflectance, dm.diffuse_reflectance, 3);
        add_texture(mt.specular_reflectance, dm.specular_reflectance, 3);
        add_texture(mt.roughness, dm.roughness, 1);
        add_texture(mt.generic_texture, dm.generic_texture, std::min(std::max(mt.generic_texture.channels, 1), RB_MAX_ND));
        add_texture(mt.normal_map, dm.normal_map, 3);
    }
    for (int l = 0; l < d.num_lights; l++) add(d.light_intensity[l], 3);
    if (sc.has_envmap) add_texture(sc.env.values, ka.ds.env_values, 3);
    add(ka.ds.env_w2e, 16);
    add(ka.screen_grad, 2LL * ka.rp.vp_w * ka.rp.vp_h);
    hash((uint64_t)spans.size());
    out.fingerprint = h;

    std::sort(spans.begin(), spans.end(), [](const Span& a, const Span& b) { return a.begin < b.begin; });
    out.ranges.clear();
    out.rec_first.clear();
    out.overlaps = false;
    out.num_acc = RB_CAM_ACC;
    for (const Span& sp : spans) {
        if (!out.ranges.empty()) {
            ExactRange& r = out.ranges.back();
            const uintptr_t end = (uintptr_t)(r.dst + r.count);
            if (sp.begin < end) { // overlaps the previous range: extend it
                out.overlaps = true;
                if (sp.end > end) {
                    const long long more = (long long)((sp.end - end) / sizeof(float));
                    r.count += more;
                    out.num_acc += more;
                }
                continue;
            }
        }
        const long long n = (long long)((sp.end - sp.begin) / sizeof(float));
        out.ranges.push_back(ExactRange{out.num_acc, n, (float*)sp.begin});
        out.rec_first.push_back(sp.rec);
        out.num_acc += n;
    }
    // caller pointer -> virtual address of its accumulator (NULL stays NULL).  A pointer of no range (a buffer of zero size) gets the
    // spare accumulator `num_acc`, which nothing reads.
    auto virt = [&](const float* p) -> float* {
        if (p == nullptr) return nullptr;
        size_t lo = 0, hi = out.ranges.size(); // ranges [0, lo) start at or before p
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if ((uintptr_t)out.ranges[mid].dst <= (uintptr_t)p) lo = mid + 1;
            else hi = mid;
        }
        if (lo == 0 || p >= out.ranges[lo - 1].dst + out.ranges[lo - 1].count) return exact_virtual(out.num_acc);
        return exact_virtual(out.ranges[lo - 1].first + (long long)(p - out.ranges[lo - 1].dst));
    };
    auto virt_texture = [&](const rb_texture& t) {
        rb_texture v = t;
        for (int l = 0; l < RB_MAX_MIP_LEVELS; l++) v.texels[l] = virt(t.texels[l]);
        v.uv_scale = virt(t.uv_scale);
        return v;
    };
    out.shapes.assign(d.shapes, d.shapes + d.num_shapes);
    for (rb_dshape& s : out.shapes) {
        s.vertices = virt(s.vertices);
        s.uvs = virt(s.uvs);
        s.normals = virt(s.normals);
        s.colors = virt(s.colors);
    }
    out.materials.assign(d.materials, d.materials + d.num_materials);
    for (rb_material& m : out.materials) {
        m.diffuse_reflectance = virt_texture(m.diffuse_reflectance);
        m.specular_reflectance = virt_texture(m.specular_reflectance);
        m.roughness = virt_texture(m.roughness);
        m.generic_texture = virt_texture(m.generic_texture);
        m.normal_map = virt_texture(m.normal_map);
    }
    out.lights.assign(d.light_intensity, d.light_intensity + d.num_lights);
    for (float*& l : out.lights) l = virt(l);
    out.env_values = virt_texture(ka.ds.env_values);
    out.env_w2e = virt(ka.ds.env_w2e);
    out.screen_grad = virt(ka.screen_grad);
}

// The records of a backward pass of `opt` over d_scene / screen_grad on a scene (camera `cam`, generic-texture width `max_generic`,
// descriptors `shapes` / `materials`, device-side scene `sc`): the checks and the layout of rb_render's backward pass, and the refusal of
// overlapping gradient buffers.  `who` prefixes the messages of this function's own checks.  Returns the error message, or null.
inline const char* exact_record_layout(const char* who, const rb_options& opt, const rb_camera& cam, int max_generic, const rb_dscene_desc* d_scene,
                                       float* screen_grad, const rb_shape* shapes, const rb_material* materials, const DevScene& sc, KernelArgs& ka,
                                       ExactLayout& xl, std::string& err) {
    if (d_scene == nullptr) return (err = std::string(who) + ": null d_scene").c_str();
    static const float no_image = 0.f; // (the layout does not depend on the image: any non-null d_image passes the checks)
    const char* e = setup_kernel_args(opt, cam, max_generic, 0, 1, 1, nullptr, &no_image, d_scene, screen_grad, ka);
    if (e == nullptr) e = setup_backward(*d_scene, sc, ka);
    if (e != nullptr) return e;
    exact_layout(*d_scene, shapes, materials, sc, ka, xl);
    if (xl.overlaps) return (err = std::string(who) + ": gradient buffers of d_scene overlap; records need disjoint buffers").c_str();
    return nullptr;
}
