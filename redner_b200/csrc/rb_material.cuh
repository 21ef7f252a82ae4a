// Textures and the BSDF (Lambert + Blinn-Phong or GGX microfacet lobe), sampling, pdf and the adjoint of the BSDF value.
//   get_texture_value / d_get_texture_value   src/texture.h:335-355 / :357-419 (trilinear mip: :53-140, :142-333)
//   bsdf / d_bsdf                             src/material.h:353-449 / :451-692
//   bsdf_sample                               src/material.h:702-811
//   bsdf_pdf                                  src/material.h:1023-1093
//   perturb_shading_frame (+adjoints)         src/material.h:273-351
// d_bsdf_sample / d_bsdf_pdf are not on the path (commented out at src/path_contribution.cpp:410-412,:463-474).
// The GGX lobe (rb_material::specular_model) has no reference counterpart; DESIGN.md section "GGX" defines it.
#pragma once
#include "rb_atomic.cuh"
#include "rb_types.cuh"

// ---------------------------------------------------------------- textures
struct BilerpTap {
    int i_ff, i_cf, i_fc, i_cc; // texel indices (before the channel multiply)
    Real u, v;
};
RB_HD BilerpTap bilerp_tap(const rb_texture& t, int li, V2 uv) {
    int w = t.width[li], h = t.height[li];
    Real x = uv.x * w - Real(0.5), y = uv.y * h - Real(0.5);
    int xf = (int)floor(x), yf = (int)floor(y);
    BilerpTap b;
    b.u = x - xf;
    b.v = y - yf;
    int xfi = rb_modulo(xf, w), yfi = rb_modulo(yf, h), xci = rb_modulo(xf + 1, w), yci = rb_modulo(yf + 1, h);
    b.i_ff = yfi * w + xfi;
    b.i_cf = yfi * w + xci;
    b.i_fc = yci * w + xfi;
    b.i_cc = yci * w + xci;
    return b;
}
RB_HD Real bilerp_eval(const float* tex, int nch, int c, const BilerpTap& b) {
    Real ff = tex[nch * b.i_ff + c], cf = tex[nch * b.i_cf + c], fc = tex[nch * b.i_fc + c], cc = tex[nch * b.i_cc + c];
    return ff * (1 - b.u) * (1 - b.v) + fc * (1 - b.u) * b.v + cf * b.u * (1 - b.v) + cc * b.u * b.v;
}
RB_HD bool tex_is_constant(const rb_texture& t) { return t.width[0] <= 0 && t.height[0] <= 0; }
RB_HD Real tex_level(const rb_texture& t, V2 du, V2 dv, Real& fu, Real& fv) {
    fu = length(du) * t.width[0];
    fv = length(dv) * t.height[0];
    return log2(rb_max(rb_max(fu, fv), Real(1e-8)));
}
// Mip-mapped (trilinear) fetch of channels c0, c0 + 1, c0 + 2 of an `nch`-channel texture; channels past nch - 1 repeat the last
// one.  Out of line (~15 inlined copies per kernel otherwise) and returned by value, so that neither side keeps an addressable
// array in local memory.
RB_FN V3 tex_eval_mip(const rb_texture& t, int nch, int c0, V2 uv_, V2 du_dxy_, V2 dv_dxy_) {
    const int c1 = c0 + 1 < nch ? c0 + 1 : nch - 1, c2 = c0 + 2 < nch ? c0 + 2 : nch - 1;
    Real sx = t.uv_scale[0], sy = t.uv_scale[1];
    V2 uv = mk2(uv_.x * sx, uv_.y * sy);
    V2 du = du_dxy_ * sx, dv = dv_dxy_ * sy;
    Real fu, fv;
    Real level = tex_level(t, du, dv, fu, fv);
    if (level <= 0 || level >= t.num_levels - 1) {
        int li = level <= 0 ? 0 : t.num_levels - 1;
        BilerpTap b = bilerp_tap(t, li, uv);
        const float* tex = t.texels[li];
        return mk3(bilerp_eval(tex, nch, c0, b), bilerp_eval(tex, nch, c1, b), bilerp_eval(tex, nch, c2, b));
    }
    int li = (int)floor(level);
    Real ld = level - li;
    BilerpTap b0 = bilerp_tap(t, li, uv), b1 = bilerp_tap(t, li + 1, uv);
    const float *tex0 = t.texels[li], *tex1 = t.texels[li + 1];
    V3 a0 = mk3(bilerp_eval(tex0, nch, c0, b0), bilerp_eval(tex0, nch, c1, b0), bilerp_eval(tex0, nch, c2, b0));
    V3 a1 = mk3(bilerp_eval(tex1, nch, c0, b1), bilerp_eval(tex1, nch, c1, b1), bilerp_eval(tex1, nch, c2, b1));
    return mk3(a0.x * (1 - ld) + a1.x * ld, a0.y * (1 - ld) + a1.y * ld, a0.z * (1 - ld) + a1.z * ld);
}
// Channels c0 .. c0 + 2 of a texture lookup (see tex_eval_mip); a constant texture is read directly, without the call.
RB_HD V3 tex_eval(const rb_texture& t, int nch, V2 uv_, V2 du_dxy_, V2 dv_dxy_, int c0 = 0) {
    if (tex_is_constant(t)) {
        const float* v = t.texels[0];
        return mk3(v[c0], v[c0 + 1 < nch ? c0 + 1 : nch - 1], v[c0 + 2 < nch ? c0 + 2 : nch - 1]);
    }
    return tex_eval_mip(t, nch, c0, uv_, du_dxy_, dv_dxy_);
}
// All `nch` channels into out[0 .. nch) (textures of any width: the G-buffer's generic texture).
RB_HD void tex_eval_channels(const rb_texture& t, int nch, V2 uv_, V2 du_dxy_, V2 dv_dxy_, Real* out) {
    for (int c0 = 0; c0 < nch; c0 += 3) {
        V3 v = tex_eval(t, nch, uv_, du_dxy_, dv_dxy_, c0);
        out[c0] = v.x;
        if (c0 + 1 < nch) out[c0 + 1] = v.y;
        if (c0 + 2 < nch) out[c0 + 2] = v.z;
    }
}
struct TexAdjoint { // returned by value so that the caller's SurfacePoint adjoint can stay in registers
    V2 d_uv, d_du_dxy, d_dv_dxy;
};
// Adjoint of the trilinear lookup (src/texture.h:146-276): scatters into the gradient mip pyramid and returns d(uv),
// d(du_dxy), d(dv_dxy).  Levels and taps are walked by ROLLED loops and each texel takes one aggregated 3-float
// reduction (nch <= 3 on this path: reflectances, roughness, normal map), so the whole adjoint is ~0.5k SASS
// instructions instead of the 36 unrolled aggregated atomics it used to be.
// `nch` is the texel stride; the call covers channels [c0, c0 + ncomp), ncomp <= 3 (wider textures: one call per triple).
RB_D TexAdjoint d_tex_eval_mip(const rb_texture& t, const rb_texture& d_t, int nch, V2 uv_, V2 du_dxy_, V2 dv_dxy_, Real d0, Real d1, Real d2, int c0 = 0,
                               int ncomp = 3) {
    V2 d_uv_ = zero2(), d_du_dxy_ = zero2(), d_dv_dxy_ = zero2();
    Real sx = t.uv_scale[0], sy = t.uv_scale[1];
    V2 uv = mk2(uv_.x * sx, uv_.y * sy);
    V2 du = du_dxy_ * sx, dv = dv_dxy_ * sy;
    Real fu, fv;
    Real level = tex_level(t, du, dv, fu, fv);
    bool u_is_max = !(fv > fu);
    Real max_fp = u_is_max ? fu : fv;
    V2 d_uv = zero2();
    Real d_level = 0;
    int l0, nl;
    Real ld = 0;
    if (level <= 0) {
        l0 = 0;
        nl = 1;
    } else if (level >= t.num_levels - 1) {
        l0 = t.num_levels - 1;
        nl = 1;
    } else {
        l0 = (int)floor(level);
        nl = 2;
        ld = level - l0;
    }
    if (ncomp > nch - c0) ncomp = nch - c0;
    if (ncomp < 2) d1 = 0;
    if (ncomp < 3) d2 = 0;
#pragma unroll 1
    for (int j = 0; j < nl; j++) {
        int li = l0 + j;
        Real wl = j ? ld : 1 - ld;
        BilerpTap b = bilerp_tap(t, li, uv);
        const float* tex = t.texels[li];
        float* d_tex = d_t.texels[li];
        Real d_u = 0, d_v = 0, val = 0;
#pragma unroll 1
        for (int k = 0; k < 4; k++) { // bit 0: ceil in x, bit 1: ceil in y
            int idx = nch * (k == 0 ? b.i_ff : k == 1 ? b.i_cf : k == 2 ? b.i_fc : b.i_cc) + c0;
            Real wu = (k & 1) ? b.u : 1 - b.u, wv = (k & 2) ? b.v : 1 - b.v;
            Real tv = d0 * tex[idx];
            if (ncomp > 1) tv += d1 * tex[idx + 1];
            if (ncomp > 2) tv += d2 * tex[idx + 2];
            val += tv * wu * wv;
            d_u += (k & 1) ? tv * wv : -tv * wv;
            d_v += (k & 2) ? tv * wu : -tv * wu;
            Real w = wl * wu * wv;
            warp_agg_add3(d_tex + idx, (float)(d0 * w), (float)(d1 * w), (float)(d2 * w));
        }
        if (nl == 2) d_level += j ? val : -val;
        d_uv.x += wl * d_u * t.width[li];
        d_uv.y += wl * d_v * t.height[li];
    }
    V2 d_du = zero2(), d_dv = zero2();
    if (max_fp > Real(1e-8)) {
        Real d_max_fp = d_level / (max_fp * log(Real(2)));
        if (u_is_max) {
            d_du += d_length2(du, d_max_fp) * Real(t.width[0]);
        } else {
            d_dv += d_length2(dv, d_max_fp) * Real(t.height[0]);
        }
    }
    d_uv_ += mk2(d_uv.x * sx, d_uv.y * sy);
    d_du_dxy_ += d_du * sx;
    d_dv_dxy_ += d_dv * sy;
    if (d_t.uv_scale != nullptr)
        agg_add2(d_t.uv_scale, mk2(d_uv.x * uv_.x + sum(d_du * du_dxy_), d_uv.y * uv_.y + sum(d_dv * dv_dxy_)));
    TexAdjoint r;
    r.d_uv = d_uv_;
    r.d_du_dxy = d_du_dxy_;
    r.d_dv_dxy = d_dv_dxy_;
    return r;
}
RB_D void d_tex_eval(const rb_texture& t, const rb_texture& d_t, int nch, V2 uv_, V2 du_dxy_, V2 dv_dxy_, const Real* d_out, V2& d_uv_,
                     V2& d_du_dxy_, V2& d_dv_dxy_) {
    if (tex_is_constant(t)) {
        if (nch == 3) {
            agg_add3(d_t.texels[0], mk3(d_out[0], d_out[1], d_out[2]));
        } else {
            for (int c = 0; c < nch; c++) agg_add1(&d_t.texels[0][c], d_out[c]);
        }
        return;
    }
#pragma unroll 1
    for (int c0 = 0; c0 < nch; c0 += 3) { // one pass for every texture of the BSDF (nch <= 3); generic textures take more
        TexAdjoint r = d_tex_eval_mip(t, d_t, nch, uv_, du_dxy_, dv_dxy_, d_out[c0], c0 + 1 < nch ? d_out[c0 + 1] : Real(0),
                                      c0 + 2 < nch ? d_out[c0 + 2] : Real(0), c0, 3);
        d_uv_ += r.d_uv;
        d_du_dxy_ += r.d_du_dxy;
        d_dv_dxy_ += r.d_dv_dxy;
    }
}

// ---------------------------------------------------------------- material helpers
RB_HD V3 mat_diffuse(const rb_material& m, const SurfacePoint& p) { return tex_eval(m.diffuse_reflectance, 3, p.uv, p.du_dxy, p.dv_dxy); }
RB_HD V3 mat_specular(const rb_material& m, const SurfacePoint& p) { return tex_eval(m.specular_reflectance, 3, p.uv, p.du_dxy, p.dv_dxy); }
RB_HD Real mat_roughness(const rb_material& m, const SurfacePoint& p) { return tex_eval(m.roughness, 1, p.uv, p.du_dxy, p.dv_dxy).x; }
RB_HD V3 mat_normal_tex(const rb_material& m, const SurfacePoint& p) { return tex_eval(m.normal_map, 3, p.uv, p.du_dxy, p.dv_dxy); }
RB_HD bool mat_has_normal_map(const rb_material& m) { return RB_NORMAL_MAP(m); }
// True when no material sets a flag that RB_SPECULAR, RB_VERTEX_COLOR or RB_NORMAL_MAP tests, i.e. when the diffuse-only kernels
// (RB_DIFFUSE, rb_kernels_diffuse.cu) compute what the others do.  Tests the fields themselves, so that it answers the same in every build.
inline bool materials_diffuse_only(const rb_material* m, int n) {
    for (int i = 0; i < n; i++)
        if (m[i].compute_specular_lighting != 0 || m[i].use_vertex_color != 0 || m[i].normal_map.num_levels > 0) return false;
    return true;
}
// True when some material's specular lobe is GGX (RB_SPECULAR && !RB_VERTEX_COLOR && RB_GGX), i.e. when only the general and deterministic
// kernels compute what the scene asks for.  Tests the fields themselves, so that it answers the same in every build.
inline bool materials_use_ggx(const rb_material* m, int n) {
    for (int i = 0; i < n; i++)
        if (m[i].compute_specular_lighting != 0 && m[i].use_vertex_color == 0 && m[i].specular_model == RB_SPECULAR_GGX) return true;
    return false;
}
RB_HD Real roughness_to_phong(Real r) { return rb_max(2 / r - 2, Real(0)); }
RB_HD Real d_roughness_to_phong(Real r, Real d_e) { return (r > 0 && r <= 1) ? -2 * d_e / rb_sq(r) : Real(0); }

RB_HD Frame perturb_shading_frame(const rb_material& m, const SurfacePoint& p) {
    V3 n_local = 2 * mat_normal_tex(m, p) - mk3(1, 1, 1);
    V3 pn = normalize(to_world(p.shading_frame, n_local));
    V3 px = normalize(p.dpdu - pn * dot(pn, p.dpdu));
    V3 py = cross(pn, px);
    return mk_frame(px, py, pn);
}
// normal-only adjoint (the BSDF value only depends on the perturbed normal; src/material.h:331-351)
// Returns the adjoint of the normal-map texel; the caller scatters it into the texture gradient.
RB_D V3 d_perturb_shading_normal(const rb_material& m, const SurfacePoint& p, V3 d_n, SurfacePoint& d_p) {
    V3 n_local = 2 * mat_normal_tex(m, p) - mk3(1, 1, 1);
    V3 n_world = to_world(p.shading_frame, n_local);
    V3 d_n_world = d_normalize(n_world, d_n);
    V3 d_local = zero3();
    d_to_world(p.shading_frame, n_local, d_n_world, d_p.shading_frame, d_local);
    return 2 * d_local;
}

struct BsdfCtx { // quantities shared by eval / pdf / sample
    Frame frame;
    V3 geom_n;
};
RB_HD BsdfCtx bsdf_ctx(const rb_material& m, const SurfacePoint& p) {
    BsdfCtx c;
    c.frame = p.shading_frame;
    if (mat_has_normal_map(m)) c.frame = perturb_shading_frame(m, p);
    c.geom_n = p.geom_normal;
    if (dot(c.geom_n, c.frame.n) < 0) c.geom_n = -c.geom_n;
    return c;
}
// The texture values the BSDF reads at one shading point.  trace_bounces fetches them once per vertex for its sample, eval and
// pdf calls.  d_vertex goes through the overloads that fetch per call: holding the values across its body costs more spills there.
struct MatTex {
    V3 kd, ks;  // reflectances, clamped at zero
    Real rough; // roughness as stored (each user clamps it its own way)
};
RB_HD MatTex mat_textures(const rb_material& m, const SurfacePoint& p) {
    MatTex t;
    t.kd = max3(RB_VERTEX_COLOR(m) ? p.color : mat_diffuse(m, p), 0);
    t.ks = max3(RB_VERTEX_COLOR(m) ? zero3() : mat_specular(m, p), 0);
    t.rough = mat_roughness(m, p);
    return t;
}
RB_HD Real smith_g1(V3 v, V3 n, Real roughness) {
    Real cos_t = dot(v, n);
    Real tan_t = sqrt(rb_max(1 / (cos_t * cos_t) - 1, Real(0)));
    if (tan_t == 0) return 1;
    Real alpha = sqrt(roughness);
    Real a = 1 / (alpha * tan_t);
    if (a >= Real(1.6)) return 1;
    Real a2 = a * a;
    return (Real(3.535) * a + Real(2.181) * a2) / (1 + Real(2.276) * a + Real(2.577) * a2);
}

// ---------------------------------------------------------------- GGX lobe
// RB_SPECULAR && !RB_VERTEX_COLOR && RB_GGX: the material's specular lobe is GGX (false in the lean and diffuse-only kernels).
#define RB_GGX_LOBE(m) (RB_SPECULAR(m) && !RB_VERTEX_COLOR(m) && RB_GGX(m))
// r is redner's roughness after its clamps; alpha^2 == r.  Every quantity is a function of the lobe's normal, wi and wo only, so that
// the adjoint reaches the shading normal (and through it the normal map) and nothing else of the frame.
// The lobe's normal: the (perturbed) shading normal, mirrored when a two-sided material is seen from below.
RB_HD V3 ggx_normal(const rb_material& m, const BsdfCtx& c, V3 wi) { return m.two_sided && dot(wi, c.frame.n) < 0 ? -c.frame.n : c.frame.n; }
// Smith Lambda (-1 + sqrt(1 + x)) / 2 with x = alpha^2 tan^2(theta_v), written x / (2 (1 + sqrt(1 + x))) and with sin^2 = |n x v|^2,
// so that it keeps its digits at small alpha and near the normal.
RB_HD Real ggx_lambda(V3 v, V3 n, Real r) {
    Real c = dot(v, n);
    Real x = r * length_sq(cross(n, v)) / (c * c);
    return x / (2 * (1 + sqrt(1 + x)));
}
// NDF alpha^2 / (pi ((n.h)^2 (alpha^2 - 1) + 1)^2) for a unit h, written alpha^2 / (pi (alpha^2 (n.h)^2 + |n x h|^2)^2) (no cancellation).
RB_HD Real ggx_ndf(V3 h, V3 n, Real r) {
    Real hz = dot(h, n);
    Real q = r * hz * hz + length_sq(cross(n, h));
    return r / (RB_PI * q * q);
}
// The specular term of bsdf_eval: F(h.wo) D(h) G2(wi, wo) / (4 |n.wi|), height-correlated G2 = 1 / (1 + Lambda(wi) + Lambda(wo)).
RB_HD V3 ggx_eval(const rb_material& m, const BsdfCtx& c, V3 ks, Real r, V3 wi, V3 wo) {
    V3 n = ggx_normal(m, c, wi);
    V3 h = normalize(wi + wo);
    Real cwi = dot(n, wi);
    if (!(cwi > 0 && dot(n, h) > 0)) return zero3();
    Real G = 1 / (1 + ggx_lambda(wi, n, r) + ggx_lambda(wo, n, r));
    V3 F = ks + (mk3(1, 1, 1) - ks) * pow(rb_max(1 - fabs(dot(h, wo)), Real(0)), Real(5));
    return F * (ggx_ndf(h, n, r) * G / (4 * cwi));
}
// Density of ggx_sample over wo: the visible-normal density G1(wi) D(h) max(0, wi.h) / (n.wi) times the reflection Jacobian 1 / (4 wo.h).
RB_HD Real ggx_pdf(const rb_material& m, const BsdfCtx& c, Real r, V3 wi, V3 wo) {
    V3 n = ggx_normal(m, c, wi);
    V3 h = normalize(wi + wo);
    Real cwi = dot(n, wi);
    if (!(cwi > 0 && dot(n, h) > 0)) return 0;
    return ggx_ndf(h, n, r) / ((1 + ggx_lambda(wi, n, r)) * 4 * cwi);
}
// A half vector drawn from the visible normals seen from wi (spherical caps, Dupuy & Benyoub 2023, in the configuration stretched to
// alpha = 1), in the local coordinates of c.frame; zero when wi lies below the lobe's normal.
RB_HD V3 ggx_sample_half(const rb_material& m, const BsdfCtx& c, Real r, V3 wi, V2 suv) {
    V3 wl = to_local(c.frame, wi);
    const Real s = m.two_sided && wl.z < 0 ? Real(-1) : Real(1);
    wl.z *= s;
    if (!(wl.z > 0)) return zero3();
    Real alpha = sqrt(r);
    V3 ws = normalize(mk3(alpha * wl.x, alpha * wl.y, wl.z));
    Real phi = 2 * RB_PI * suv.x;
    Real z = (1 - suv.y) * (1 + ws.z) - ws.z;
    Real sin_t = sqrt(rb_max(1 - z * z, Real(0)));
    V3 hs = mk3(sin_t * cos(phi) + ws.x, sin_t * sin(phi) + ws.y, z + ws.z);
    if (!(hs.z > 0)) return zero3();
    V3 hl = normalize(mk3(alpha * hs.x, alpha * hs.y, hs.z));
    hl.z *= s;
    return hl;
}

RB_HD V3 bsdf_eval(const rb_material& m, const SurfacePoint& p, const MatTex& tx, V3 wi, V3 wo, Real min_rough) {
    BsdfCtx c = bsdf_ctx(m, p);
    Real geom_wi = dot(c.geom_n, wi), geom_wo = dot(c.geom_n, wo);
    Real sh_wi = fabs(dot(c.frame.n, wi)), sh_wo = fabs(dot(c.frame.n, wo));
    if (geom_wi * geom_wo < 0) return zero3();
    if (!m.two_sided && geom_wi < 0 && geom_wo < 0) return zero3();
    if (sh_wi == 0 || sh_wo <= Real(1e-3) || fabs(geom_wo) <= Real(1e-3)) return zero3();
    const V3 kd = tx.kd, ks = tx.ks;
    Real roughness = rb_max(tx.rough, min_rough);
    V3 diffuse = kd * (sh_wo / RB_PI);
    V3 spec = zero3();
    if (RB_GGX_LOBE(m)) {
        spec = ggx_eval(m, c, ks, rb_max(roughness, Real(1e-6)), wi, wo);
    } else if (RB_SPECULAR(m) && !RB_VERTEX_COLOR(m)) {
        V3 h = normalize(wi + wo);
        V3 hl = to_local(c.frame, h);
        if (m.two_sided && hl.z < 0) hl = -hl;
        if (hl.z > 0) {
            Real e = roughness_to_phong(roughness);
            Real D = pow(rb_max(hl.z, Real(0)), e) * (e + 2) / (2 * RB_PI);
            Real G = smith_g1(wi, c.frame.n, roughness) * smith_g1(wo, c.frame.n, roughness);
            Real cos_d = fabs(dot(h, wo));
            V3 F = ks + (mk3(1, 1, 1) - ks) * pow(rb_max(1 - cos_d, Real(0)), Real(5));
            spec = F * (D * G / (4 * sh_wi));
        }
    }
    return diffuse + spec;
}
RB_HD V3 bsdf_eval(const rb_material& m, const SurfacePoint& p, V3 wi, V3 wo, Real min_rough) { return bsdf_eval(m, p, mat_textures(m, p), wi, wo, min_rough); }

RB_HD Real bsdf_pdf(const rb_material& m, const SurfacePoint& p, const MatTex& tx, V3 wi, V3 wo, Real min_rough) {
    BsdfCtx c = bsdf_ctx(m, p);
    Real geom_wi = dot(c.geom_n, wi), geom_wo = dot(c.geom_n, wo);
    Real sh_wo = fabs(dot(c.frame.n, wo));
    if (geom_wi * geom_wo < 0) return 0;
    if (!m.two_sided && geom_wi < 0 && geom_wo < 0) return 0;
    Real wd = luminance(tx.kd), ws = luminance(tx.ks), wsum = wd + ws;
    Real pd = Real(0.5), ps = Real(0.5);
    if (wsum > 0) {
        pd = wd / wsum;
        ps = ws / wsum;
    }
    Real diffuse_pdf = 0;
    if (pd > 0) diffuse_pdf = pd * sh_wo / RB_PI;
    Real spec_pdf = 0;
    if (ps > 0 && RB_GGX_LOBE(m)) {
        spec_pdf = ps * ggx_pdf(m, c, rb_max(rb_max(tx.rough, min_rough), Real(1e-6)), wi, wo);
    } else if (ps > 0) {
        V3 h = normalize(wi + wo);
        // the reference projects on the UNPERTURBED frame here (src/material.h:1078); reproduced
        V3 hl = to_local(p.shading_frame, h);
        if (m.two_sided && hl.z < 0) hl = -hl;
        Real hdwo = fabs(dot(h, wo));
        if (hl.z > 0 && hdwo > 0) {
            Real roughness = rb_max(rb_max(tx.rough, min_rough), Real(1e-6));
            Real e = roughness_to_phong(roughness);
            Real D = pow(hl.z, e) * (e + 2) / (2 * RB_PI);
            spec_pdf = ps * D * hl.z / (4 * hdwo);
        }
    }
    return diffuse_pdf + spec_pdf;
}
RB_HD Real bsdf_pdf(const rb_material& m, const SurfacePoint& p, V3 wi, V3 wo, Real min_rough) { return bsdf_pdf(m, p, mat_textures(m, p), wi, wo, min_rough); }

// Returns the sampled direction (zero vector when sampling fails).  `w_sel` is the lobe-selection sample kept in
// double so that the decision agrees with the reference's double comparison.
RB_HD V3 bsdf_sample_dir(const rb_material& m, const SurfacePoint& p, const MatTex& tx, V3 wi, V2 suv, double w_sel, Real min_rough, const RayDiff& wi_diff,
                         RayDiff& wo_diff, Real& next_min_rough) {
    next_min_rough = min_rough;
    BsdfCtx c = bsdf_ctx(m, p);
    Real geom_wi = dot(c.geom_n, wi);
    if (!m.two_sided && geom_wi < 0) return zero3();
    Real wd = luminance(tx.kd), ws = luminance(tx.ks), wsum = wd + ws;
    Real pd = Real(0.5);
    if (wsum > 0) pd = wd / wsum;
    if (w_sel <= (double)pd) {
        next_min_rough = 1;
        Real phi = 2 * RB_PI * suv.x;
        Real tmp = sqrt(rb_max(1 - suv.y, Real(0)));
        V3 local = mk3(cos(phi) * tmp, sin(phi) * tmp, sqrt(suv.y));
        wo_diff.org_dx = wi_diff.org_dx;
        wo_diff.org_dy = wi_diff.org_dy;
        wo_diff.dir_dx = mk3(Real(0.03), Real(0.03), Real(0.03));
        wo_diff.dir_dy = mk3(Real(0.03), Real(0.03), Real(0.03));
        V3 dir = to_world(c.frame, local);
        if (dot(c.geom_n, dir) * geom_wi < 0) dir = to_world(c.frame, -local);
        return dir;
    } else if (RB_GGX_LOBE(m)) {
        Real roughness = rb_max(rb_max(tx.rough, min_rough), Real(1e-6));
        next_min_rough = rb_max(roughness, min_rough);
        V3 hl = ggx_sample_half(m, c, roughness, wi, suv);
        if (hl.z == 0) return zero3();
        V3 h = to_world(c.frame, hl);
        V3 dir = 2 * dot(wi, h) * h - wi;
        // below the geometric surface eval is zero; a flipped direction would not have the density ggx_pdf gives it
        if (dot(c.geom_n, dir) * geom_wi < 0) return zero3();
        // the ray differential of the Blinn-Phong branch (it only selects mip levels)
        V3 dmdx = p.dn_dx * hl.z, dmdy = p.dn_dy * hl.z;
        V3 wi_dx = -wi_diff.dir_dx, wi_dy = -wi_diff.dir_dy;
        Real wdm_dx = dot(wi_dx, h) + dot(wi, dmdx);
        Real wdm_dy = dot(wi_dy, h) + dot(wi, dmdy);
        wo_diff.org_dx = wi_diff.org_dx;
        wo_diff.org_dy = wi_diff.org_dy;
        wo_diff.dir_dx = 2 * (dot(wi, h) * dmdx + wdm_dx * h) - wi_dx;
        wo_diff.dir_dy = 2 * (dot(wi, h) * dmdy + wdm_dy * h) - wi_dy;
        return dir;
    } else {
        Real roughness = rb_max(rb_max(tx.rough, min_rough), Real(1e-6));
        next_min_rough = rb_max(roughness, min_rough);
        Real e = roughness_to_phong(roughness);
        Real phi = 2 * RB_PI * suv.y;
        Real sin_phi = sin(phi), cos_phi = cos(phi);
        Real cos_t = pow(suv.x, 1 / (e + 2));
        Real sin_t = sqrt(rb_max(1 - cos_t * cos_t, Real(0)));
        V3 hl = mk3(sin_t * cos_phi, sin_t * sin_phi, cos_t);
        V3 h = to_world(c.frame, hl);
        V3 dir = 2 * dot(wi, h) * h - wi;
        if (dot(c.geom_n, dir) * geom_wi < 0) {
            hl = -hl;
            h = to_world(c.frame, hl);
            dir = 2 * dot(wi, h) * h - wi;
        }
        V3 dmdx = p.dn_dx * hl.z, dmdy = p.dn_dy * hl.z;
        V3 wi_dx = -wi_diff.dir_dx, wi_dy = -wi_diff.dir_dy;
        Real wdm_dx = dot(wi_dx, h) + dot(wi, dmdx);
        Real wdm_dy = dot(wi_dy, h) + dot(wi, dmdy);
        wo_diff.org_dx = wi_diff.org_dx;
        wo_diff.org_dy = wi_diff.org_dy;
        wo_diff.dir_dx = 2 * (dot(wi, h) * dmdx + wdm_dx * h) - wi_dx;
        wo_diff.dir_dy = 2 * (dot(wi, h) * dmdy + wdm_dy * h) - wi_dy;
        return dir;
    }
}

// Adjoint of bsdf_eval with respect to material textures, the shading point, wi and wo.
RB_D void d_bsdf_eval(const rb_material& m, const rb_material& d_m, const SurfacePoint& p, const MatTex& tx, V3 wi, V3 wo, Real min_rough,
                      V3 d_out, SurfacePoint& d_p, V3& d_wi, V3& d_wo) {
    BsdfCtx c = bsdf_ctx(m, p);
    const V3 n = c.frame.n;
    V3 d_n = zero3();
    Real geom_wi = dot(c.geom_n, wi), geom_wo = dot(c.geom_n, wo);
    Real sh_wi = fabs(dot(n, wi)), sh_wo = fabs(dot(n, wo));
    if (geom_wi * geom_wo < 0) return;
    if (!m.two_sided && geom_wi < 0 && geom_wo < 0) return;
    if (sh_wi == 0 || sh_wo <= Real(1e-3) || fabs(geom_wo) <= Real(1e-3)) return;
    const V3 kd = tx.kd, ks = tx.ks;
    // diffuse = kd * sh_wo / pi   (gradient passes through the clamp unchanged, src/material.h:505-518)
    V3 d_kd = d_out * (sh_wo / RB_PI);
    if (RB_VERTEX_COLOR(m)) d_p.color += d_kd;
    // texture adjoints are collected here and scattered by ONE rolled loop at the end (one copy of the mip adjoint)
    V3 d_slot[4] = {d_kd, zero3(), zero3(), zero3()};
    unsigned slot_on = RB_VERTEX_COLOR(m) ? 0u : 1u;
    Real d_sh_wo = sum(d_out * kd) / RB_PI;
    if (dot(n, wo) < 0) d_sh_wo = -d_sh_wo;
    d_wo += n * d_sh_wo;
    d_n += wo * d_sh_wo;

    Real roughness = rb_max(rb_max(tx.rough, min_rough), Real(1e-6));
    if (RB_GGX_LOBE(m)) {
        // ggx_eval with x_v = r |n x v|^2 / (n.v)^2, Lambda_v = (sqrt(1 + x_v) - 1) / 2, D = r / (pi q^2), q = r (n'.h)^2 + |n x h|^2,
        // n' = sg n the lobe's normal
        const Real sg = m.two_sided && dot(wi, n) < 0 ? Real(-1) : Real(1);
        const V3 ns = n * sg;
        V3 h = normalize(wi + wo);
        Real cwi = dot(ns, wi), hz = dot(ns, h);
        if (cwi > 0 && hz > 0) {
            const Real r = roughness;
            V3 nxh = cross(n, h), nxi = cross(n, wi), nxo = cross(n, wo);
            Real q = r * hz * hz + length_sq(nxh);
            Real D = r / (RB_PI * q * q);
            Real ci = dot(n, wi), co = dot(n, wo);
            Real xi = r * length_sq(nxi) / (ci * ci), xo = r * length_sq(nxo) / (co * co);
            Real sqi = sqrt(1 + xi), sqo = sqrt(1 + xo);
            Real G = 1 / (1 + xi / (2 * (1 + sqi)) + xo / (2 * (1 + sqo)));
            Real cos_d = dot(h, wo);
            Real cos5 = pow(rb_max(1 - cos_d, Real(0)), Real(5));
            V3 one = mk3(1, 1, 1);
            V3 F = ks + (one - ks) * cos5;
            Real k = D * G / (4 * cwi);
            V3 d_F = d_out * k;
            Real d_k = sum(d_out * F);
            Real d_D = d_k * G / (4 * cwi), d_G = d_k * D / (4 * cwi);
            Real d_cwi = -d_k * k / cwi;
            d_wi += d_cwi * ns;
            d_n += (d_cwi * sg) * wi;
            V3 d_ks = d_F * (1 - cos5);
            Real d_cos5 = sum(d_F * (one - ks));
            Real d_cos_d = -5 * d_cos5 * pow(rb_max(1 - cos_d, Real(0)), Real(4));
            V3 d_h = d_cos_d * wo;
            d_wo += d_cos_d * h;
            Real d_r = 0;
            Real d_lambda = -d_G * G * G; // dLambda / dx = 1 / (4 sqrt(1 + x))
            auto d_x = [&](V3 v, V3 nxv, Real cv, Real x, Real d_xv) -> V3 {
                d_r += d_xv * length_sq(nxv) / (cv * cv);
                Real d_cv = -2 * d_xv * x / cv;
                V3 d_v = d_cv * n;
                d_n += d_cv * v;
                d_cross(n, v, nxv * (2 * d_xv * r / (cv * cv)), d_n, d_v);
                return d_v;
            };
            d_wi += d_x(wi, nxi, ci, xi, d_lambda / (4 * sqi));
            d_wo += d_x(wo, nxo, co, xo, d_lambda / (4 * sqo));
            Real d_q = -2 * d_D * D / q;
            d_r += d_D / (RB_PI * q * q) + d_q * hz * hz;
            Real d_hz = d_q * 2 * r * hz;
            d_h += d_hz * ns;
            d_n += (d_hz * sg) * h;
            d_cross(n, h, nxh * (2 * d_q), d_n, d_h);
            V3 d_wiwo = d_normalize(wi + wo, d_h);
            d_wi += d_wiwo;
            d_wo += d_wiwo;
            d_slot[1] = d_ks;
            slot_on |= 2u;
            if (roughness > min_rough) {
                d_slot[2] = mk3(d_r, 0, 0);
                slot_on |= 4u;
            }
        }
    } else if (RB_SPECULAR(m) && !RB_VERTEX_COLOR(m)) {
        V3 h = normalize(wi + wo);
        V3 hl = to_local(c.frame, h);
        bool flipped = false;
        if (m.two_sided && hl.z < 0) {
            hl = -hl;
            flipped = true;
        }
        if (hl.z > 0) {
            Real e = roughness_to_phong(roughness);
            Real D = pow(hl.z, e) * (e + 2) / (2 * RB_PI);
            Real d_roughness = 0;
            Real Gwi = smith_g1(wi, n, roughness), Gwo = smith_g1(wo, n, roughness);
            Real G = Gwi * Gwo;
            Real cos_d = dot(h, wo);
            Real cos5 = pow(rb_max(1 - cos_d, Real(0)), Real(5));
            V3 one = mk3(1, 1, 1);
            V3 F = ks + (one - ks) * cos5;
            V3 spec = F * (D * G / (4 * sh_wi));
            V3 d_F = d_out * (D * G / (4 * sh_wi));
            Real d_D = sum(d_out * F) * (G / (4 * sh_wi));
            Real d_G = sum(d_out * F) * (D / (4 * sh_wi));
            Real d_sh_wi = -sum(d_out * spec) / sh_wi;
            // (the reference flips sh_wi instead of d_sh_wi here -- no effect on the result, src/material.h:615-620)
            d_wi += d_sh_wi * n;
            d_n += d_sh_wi * wi;
            V3 d_ks = d_F * (1 - cos5);
            Real d_cos5 = sum(d_F * (one - ks));
            Real d_cos_d = -5 * d_cos5 * pow(rb_max(1 - cos_d, Real(0)), Real(4));
            V3 d_h = d_cos_d * wo;
            d_wo += d_cos_d * h;
            Real d_Gwi = d_G * Gwo, d_Gwo = d_G * Gwi;
            // adjoint of the Smith G1 fit; uses 2.557 where the primal uses 2.577 (src/material.h:581,586) -- reproduced
            auto d_smith = [&](V3 v, Real d_G1) -> V3 {
                Real cos_t = dot(v, n);
                if (dot(v, h) * cos_t <= 0) return zero3();
                Real tan_t = sqrt(rb_max(1 / rb_sq(cos_t) - 1, Real(0)));
                if (tan_t <= Real(1e-10)) return zero3();
                Real alpha = sqrt(roughness);
                Real a = 1 / (alpha * tan_t);
                if (a >= Real(1.6)) return zero3();
                Real num = Real(3.535) * a + Real(2.181) * rb_sq(a);
                Real den = 1 + Real(2.276) * a + Real(2.557) * rb_sq(a);
                Real d_num = d_G1 / den;
                Real d_den = -d_G1 * num / rb_sq(den);
                Real d_a = d_num * (Real(3.535) + Real(2.181) * 2 * a) + d_den * (Real(2.276) + Real(2.557) * 2 * a);
                Real d_alpha = -d_a * a / alpha;
                Real d_tan = -d_a * a / tan_t;
                d_roughness += Real(0.5) * d_alpha / alpha;
                Real d_tan_sq = d_tan * Real(0.5) / tan_t;
                Real d_cos_t = -2 * d_tan_sq / (cos_t * cos_t * cos_t);
                d_n += d_cos_t * v;
                return d_cos_t * n;
            };
            d_wi += d_smith(wi, d_Gwi);
            d_wo += d_smith(wo, d_Gwo);
            Real d_D_pow = d_D * (e + 2) / (2 * RB_PI);
            Real d_D_factor = d_D * pow(hl.z, e);
            Real d_hlz = d_D_pow * pow(rb_max(hl.z, Real(0)), e - 1) * e;
            Real d_e = d_D_pow * pow(rb_max(hl.z, Real(0)), e) * log(hl.z);
            d_e += d_D_factor / (2 * RB_PI);
            d_roughness += d_roughness_to_phong(roughness, d_e);
            if (flipped) d_hlz = -d_hlz;
            d_h += d_hlz * n;
            d_n += d_hlz * h;
            V3 d_wiwo = d_normalize(wi + wo, d_h);
            d_wi += d_wiwo;
            d_wo += d_wiwo;
            d_slot[1] = d_ks;
            slot_on |= 2u;
            if (roughness > min_rough) {
                d_slot[2] = mk3(d_roughness, 0, 0);
                slot_on |= 4u;
            }
        }
    }
    if (mat_has_normal_map(m)) {
        d_slot[3] = d_perturb_shading_normal(m, p, d_n, d_p);
        slot_on |= 8u;
    } else {
        d_p.shading_frame.n += d_n;
    }
#pragma unroll 1
    for (int k = 0; k < 4; k++) {
        if (!((slot_on >> k) & 1u)) continue;
        const rb_texture* t = k == 0 ? &m.diffuse_reflectance : k == 1 ? &m.specular_reflectance : k == 2 ? &m.roughness : &m.normal_map;
        const rb_texture* dt = k == 0 ? &d_m.diffuse_reflectance : k == 1 ? &d_m.specular_reflectance : k == 2 ? &d_m.roughness : &d_m.normal_map;
        V3 d = k == 0 ? d_slot[0] : k == 1 ? d_slot[1] : k == 2 ? d_slot[2] : d_slot[3];
        Real d_o[3] = {d.x, d.y, d.z};
        d_tex_eval(*t, *dt, k == 2 ? 1 : 3, p.uv, p.du_dxy, p.dv_dxy, d_o, d_p.uv, d_p.du_dxy, d_p.dv_dxy);
    }
}
RB_D void d_bsdf_eval(const rb_material& m, const rb_material& d_m, const SurfacePoint& p, V3 wi, V3 wo, Real min_rough, V3 d_out, SurfacePoint& d_p,
                      V3& d_wi, V3& d_wo) {
    d_bsdf_eval(m, d_m, p, mat_textures(m, p), wi, wo, min_rough, d_out, d_p, d_wi, d_wo);
}
