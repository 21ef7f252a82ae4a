"""GPU suite: texture lookups and their adjoints (rb_material.cuh: tex_eval, tex_eval_channels, d_tex_eval with the warp-aggregated
scatter) through the test hook rb_texture_test, lookup by lookup, against the float64 restatement in tests/texture_ref.py.

Textures are api.Texture pyramids of sizes 1x1, 1x7, 7x1, 2x2, 5x3, 13x7, 64x64 and 1024x1024 (cut at 8 levels), with 1 and 3
channels (the BSDF's path) and 2, 4, 5, 6, 7 (generic: tail triples of 1 and 2 channels), constant textures of 1, 3 and 5 channels,
uv_scale (1, 1), (2, 3) and (-1.5, 0.5), with and without a uv_scale gradient.  Query families: uv random in [0, 1), wrapping
(negative, above 1, the environment map's [-0.5, 0.5]), exactly 0 and 1, texel centres and edges of every level (and 1e-3 texel off
them), large |x| from 2^8 up to just below 2^22; footprints zero, below a texel, inside each level interval, at integer levels and
1e-4 off them, above the top level up to 1e18 texels, anisotropic both ways, exact ties fu == fv.  |x| stays below 2^22 because there
the float32 spacing of x is at most 0.25, so rounding moves floor(x) by at most one and the one-sided answers are two; from 2^23 on
every float32 is an integer, the bilinear weights are always 0 and the lookup degenerates to the nearest texel, and beyond 2^31
floor(x) does not fit the int the texel index is computed in.

Comparison rules (tolerances from texture_ref: the float32 error bounds of x, y and level times each output's sensitivity to them,
plus ARITH = 32 ulps of the few rounded products and sums):
- values of every query (the value is continuous across floor and level flips);
- d(uv), d(du_dxy), d(dv_dxy) per query: strictly for queries whose answer does not depend on rounding, and for the others equal to
  one of their one-sided float64 answers; both counted per family, and every family compares some queries strictly;
- texel and uv_scale gradients of a batch of queries that do not depend on rounding: each element within
  gamma_k * sum(|c| + err) + sum(err) of the float64 sum, where k is its number of contributions, gamma_k = k u / (1 - k u) with
  u = 2^-24 is the bound for summing k floats in any order, and err is each contribution's own float32 error (4 ulps of it plus its
  sensitivity to the rounding of x, y and level) -- the widening; an element without contributions must be exactly zero;
- queries that depend on rounding are scattered one per call and must match one of their one-sided scatters;
- exact sums: power-of-two sizes, uv at texel centres or midpoints, clamped levels and small integer d(value) make every contribution
  and partial sum exact, so the gradient must equal the float64 sum bit for bit at every lane pattern, including 10^6 lookups of
  a 1x1 texture (a lane lost or counted twice by warp_agg_add3 shows);
- guard zones: each gradient pyramid is a set of views into one allocation with 64 guard floats before, between and after the
  levels and after the uv_scale gradient; guards and untouched elements must stay exactly zero.

The checks are shared with tests/test_texture_cpu.py, which runs them on the host build of the device headers (tools/cpu_emu)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import texture_ref as R

pytestmark = pytest.mark.gpu

GUARD = 64
SCALES = [(1.0, 1.0), (2.0, 3.0), (-1.5, 0.5)]
# (height, width, channels): every size, every channel count, 1024^2 with the BSDF's channel counts
TEXTURES = [(1, 1, 1), (1, 7, 3), (7, 1, 2), (2, 2, 4), (5, 3, 5), (13, 7, 6), (64, 64, 7), (64, 64, 3), (13, 7, 1), (1024, 1024, 3),
            (1024, 1024, 1), (5, 3, 3), (1, 7, 7)]
CONSTANTS = [1, 3, 5]


# ---------------------------------------------------------------------------------------------------- textures and buffers
class Setup:
    """A texture on `dev` through the library's wrappers, its float64 restatement and a guarded gradient pyramid."""

    def __init__(self, rb, dev, texels, uv_scale, d_uv_scale=True):
        from redner_b200 import api
        self.rb, self.dev = rb, dev
        if texels.dim() == 1:
            mips = [texels.contiguous()]
        else:
            mips = api.Texture(texels).mipmap
        self.mips = [m.to(dev).contiguous() for m in mips]
        self.uv_scale = torch.tensor(uv_scale, dtype=torch.float32, device=dev)
        self.ref = R.Tex([m.cpu().numpy() for m in self.mips], self.uv_scale.cpu().numpy())
        nch, self.constant = self.ref.nch, self.ref.constant
        cls = rb.TextureN if nch not in (1, 3) else (rb.Texture1 if nch == 1 else rb.Texture3)
        self.cls = cls
        fp = lambda t: rb.float_ptr(t.data_ptr())  # noqa: E731
        wh = ([0], [0]) if self.constant else ([int(m.shape[1]) for m in self.mips], [int(m.shape[0]) for m in self.mips])
        self.tex = cls([fp(m) for m in self.mips], wh[0], wh[1], nch, fp(self.uv_scale))
        # one allocation: guard, level 0, guard, level 1, ..., guard, uv_scale gradient (2), guard
        sizes = [m.numel() for m in self.mips]
        total = GUARD + sum(s + GUARD for s in sizes) + 2 + GUARD
        self.buf = torch.zeros(total, dtype=torch.float32, device=dev)
        self.views, off = [], GUARD
        for s in sizes:
            self.views.append((off, s))
            off += s + GUARD
        self.uvs_off = off
        self.with_uvs = d_uv_scale
        self.d_tex = cls([rb.float_ptr(self.buf.data_ptr() + 4 * o) for o, _ in self.views], wh[0], wh[1], nch,
                         rb.float_ptr(self.buf.data_ptr() + 4 * off) if d_uv_scale else None)

    def run(self, q, d=None):
        """(values, d_queries, gradient levels [size, nch], uv_scale gradient) of one call, after zeroing the gradient pyramid; the
        guard zones (and the uv_scale gradient when the call has none) must stay zero."""
        self.buf.zero_()
        qt = torch.as_tensor(q, dtype=torch.float32).to(self.dev)
        dt = None if d is None else torch.as_tensor(d, dtype=torch.float32).to(self.dev)
        values, dq = self.rb.texture_test(self.tex, qt, dt, self.d_tex if d is not None else None)
        buf = self.buf.cpu().numpy()
        guard = np.ones(buf.size, bool)
        levels = []
        for o, s in self.views:
            guard[o:o + s] = False
            levels.append(buf[o:o + s].reshape(-1, self.ref.nch).astype(np.float64))
        if self.with_uvs:
            guard[self.uvs_off:self.uvs_off + 2] = False
        bad = np.nonzero(guard & (buf != 0))[0]
        assert bad.size == 0, "a write outside the gradient pyramid: %d guard floats touched, first at offset %d" % (bad.size, bad[0])
        return (values.cpu().numpy().astype(np.float64), None if dq is None else dq.cpu().numpy().astype(np.float64), levels,
                buf[self.uvs_off:self.uvs_off + 2].astype(np.float64))


def random_texels(h, w, nch, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(h, w, nch, generator=g) * 2 - 1).float()


# ---------------------------------------------------------------------------------------------------- query families
def _dirs(rng, n):
    a = rng.uniform(0, 2 * math.pi, n)
    return np.stack([np.cos(a), np.sin(a)], 1)


def _footprint(rng, n, length_u, length_v):
    return np.concatenate([_dirs(rng, n) * length_u[:, None], _dirs(rng, n) * length_v[:, None]], 1)


def families(ref, n, seed):
    """{family: [n', 6] float32 queries} for texture `ref` (a texture_ref.Tex)."""
    rng = np.random.default_rng(seed)
    L, w0, h0 = ref.L, max(ref.w[0], 1), max(ref.h[0], 1)
    top = L - 1

    def fp_at_level(level, aniso=0.25):
        # footprints whose larger side (u or v) is 2^level texels of level 0 after uv_scale, the other a fraction of that
        fu = np.exp2(level) / (w0 * abs(ref.sx))
        fv = np.exp2(level) / (h0 * abs(ref.sy))
        frac = rng.uniform(0, aniso, level.size)
        swap = rng.random(level.size) < 0.5
        return _footprint(rng, level.size, np.where(swap, fu * frac, fu), np.where(swap, fv, fv * frac))

    def mixed_fp(k):
        return fp_at_level(rng.uniform(-3, top + 2, k))

    def rand_uv(k):
        return rng.uniform(-0.5, 1.5, (k, 2))
    fam = {}
    fam["uv_random"] = np.concatenate([rng.random((n, 2)), mixed_fp(n)], 1)
    wrap = np.concatenate([rng.uniform(-7, 8, (n // 2, 2)), rng.uniform(-0.5, 0.5, (n - n // 2, 2))])
    fam["uv_wrap"] = np.concatenate([wrap, mixed_fp(n)], 1)
    zo = rng.choice(np.array([0.0, 1.0, -0.0]), (n, 2))
    fam["uv_zero_one"] = np.concatenate([zo, mixed_fp(n)], 1)
    # texel centres (x integer) and edges (x + 0.5 integer) of a random level, exactly and 1e-3 texel off
    lv = rng.integers(0, L, n)
    W = np.array([max(w, 1) for w in ref.w])[lv] * abs(ref.sx)
    H = np.array([max(h, 1) for h in ref.h])[lv] * abs(ref.sy)
    k = rng.integers(-3, 12, (n, 2)).astype(np.float64) + rng.choice([0.5, 0.0], (n, 2))
    off = np.where(rng.random((n, 1)) < 0.5, 0.0, rng.choice([-1e-3, 1e-3], (n, 2)))
    sgn = np.sign(np.array([ref.sx, ref.sy]))
    uv = (k + off) / np.stack([W, H], 1) * sgn
    fam["uv_centres_edges"] = np.concatenate([uv, fp_at_level(lv + rng.uniform(-0.3, 0.3, n))], 1)
    mag = np.exp2(rng.uniform(8, 21.99, (n, 2))) / (np.array([w0, h0]) * np.abs([ref.sx, ref.sy]))
    fam["uv_large"] = np.concatenate([mag * rng.choice([-1.0, 1.0], (n, 2)), mixed_fp(n)], 1)
    fam["fp_zero"] = np.concatenate([rand_uv(n), np.zeros((n, 4))], 1)
    fam["fp_sub_texel"] = np.concatenate([rand_uv(n), fp_at_level(rng.uniform(-12, 0, n))], 1)
    fam["fp_interior"] = np.concatenate([rand_uv(n), fp_at_level(rng.uniform(0, max(top, 1e-9), n))], 1)
    # integer levels 0 .. L - 1, axis-aligned (exact where the size is a power of two), and 1e-4 off them
    lk = rng.integers(0, L, n).astype(np.float64) + np.where(rng.random(n) < 0.5, 0.0, rng.choice([-1e-4, 1e-4], n))
    ax = np.zeros((n, 4))
    ax[:, 0] = np.exp2(lk) / (w0 * abs(ref.sx))
    ax[:, 3] = np.exp2(lk) / (h0 * abs(ref.sy)) * rng.choice([0.0, 0.5, 0.25], n)
    fam["fp_integer_levels"] = np.concatenate([rand_uv(n), ax], 1)
    lev_top = rng.uniform(top, top + 6, n)
    lev_top[: n // 4] = math.log2(1e18)  # (a very large finite footprint: 1e18 texels, its square still a finite float32)
    fam["fp_above_top"] = np.concatenate([rand_uv(n), fp_at_level(lev_top)], 1)
    ratio = np.exp2(rng.uniform(3, 12, n))
    base = np.exp2(rng.uniform(-2, top + 1, n)) / (w0 * abs(ref.sx))
    sw = rng.random(n) < 0.5
    fam["fp_anisotropic"] = np.concatenate([rand_uv(n), _footprint(rng, n, np.where(sw, base, base / ratio), np.where(sw, base / ratio, base))], 1)
    a = np.exp2(rng.uniform(-2, top + 1, n)) / max(w0, h0)
    tie = np.zeros((n, 4))
    kind = rng.integers(0, 3, n)
    sg = rng.choice([-1.0, 1.0], (n, 4))
    tie[kind == 0] = np.stack([a, 0 * a, 0 * a, a], 1)[kind == 0]
    tie[kind == 1] = np.stack([0 * a, a, a, 0 * a], 1)[kind == 1]
    tie[kind == 2] = np.stack([a, 0.5 * a, a, 0.5 * a], 1)[kind == 2]
    fam["fp_ties"] = np.concatenate([rand_uv(n), tie * sg], 1)
    return {k: np.asarray(v, dtype=np.float32) for k, v in fam.items()}


# ---------------------------------------------------------------------------------------------------- comparisons
def _close(got, want, tol):
    return np.abs(got - want) <= tol + 1e-30


def check_values(name, got, ans, rows):
    """values of `rows` (every query) within the tolerance of the nominal answer"""
    ok = _close(got[rows], ans.value, ans.value_tol)
    bad = np.nonzero(~ok.all(1))[0]
    assert bad.size == 0, "%s: %d values differ from float64, e.g. query row %d: got %s want %s tol %s" % (
        name, bad.size, rows[bad[0]], got[rows[bad[0]]].tolist(), ans.value[bad[0]].tolist(), ans.value_tol[bad[0]].tolist())


def check_dq_strict(name, got, ans):
    ok = _close(got, ans.d_q, ans.dq_tol).all(1)
    bad = np.nonzero(~ok)[0]
    assert bad.size == 0, "%s: %d adjoints differ from float64, e.g. row %d: got %s want %s tol %s" % (
        name, bad.size, bad[0], got[bad[0]].tolist(), ans.d_q[bad[0]].tolist(), ans.dq_tol[bad[0]].tolist())


def check_dq_one_sided(name, got, answers, rows):
    """every query of `rows` matches one of its one-sided answers (got indexed by query)"""
    matched = np.zeros(got.shape[0], bool)
    for a in answers:
        ok = _close(got[a.qid], a.d_q, a.dq_tol).all(1)
        matched[a.qid[ok]] = True
    bad = [int(r) for r in rows if not matched[r]]
    assert not bad, "%s: %d rounding-dependent queries match none of their one-sided answers, e.g. query %d: got %s, answers %s" % (
        name, len(bad), bad[0], got[bad[0]].tolist(), [a.d_q[a.qid == bad[0]].tolist() for a in answers if (a.qid == bad[0]).any()])


def scatter_ok(ref, levels, uvs, sc, with_uvs, exact=False):
    """(ok, message): the gradient pyramid of one call against the float64 scatter `sc` of texture_ref.scatter"""
    lv, (us, uab, uer, uct) = sc
    for l, (got, (s, ab, er, ct)) in enumerate(zip(levels, lv)):
        if exact:
            assert np.all(s.astype(np.float32).astype(np.float64) == s), "exact family whose float64 sum is not a float32"
            bad = got != s
        else:
            tol = R.gamma(ct) * (ab + er) + er
            bad = np.abs(got - s) > tol
        bad |= (ct == 0) & (got != 0)
        if bad.any():
            i = np.argwhere(bad)[0]
            return False, "level %d texel %d channel %d: got %r, float64 %r (sum |c| %r, err %r, %d contributions)" % (
                l, i[0], i[1], float(got[i[0], i[1]]), float(s[i[0], i[1]]), float(ab[i[0], i[1]]), float(er[i[0], i[1]]), int(ct[i[0], i[1]]))
    if with_uvs and not ref.constant:
        tol = R.gamma(uct) * (uab + uer) + uer
        if (np.abs(uvs - us) > tol).any():
            return False, "uv_scale gradient %s, float64 %s, tol %s" % (uvs.tolist(), us.tolist(), tol.tolist())
    if ref.constant or not with_uvs:
        if (uvs != 0).any():
            return False, "uv_scale gradient written: %s" % uvs.tolist()
    return True, ""


def d_values_for(rng, n, nch):
    return rng.uniform(-1, 1, (n, nch)).astype(np.float32)


def check_texture(rb, dev, size_ch, scale_i, n=256, n_dep_scatter=4, seed=0):
    """Every family on one texture and uv_scale; returns {family: {check: count}}."""
    h, w, nch = size_ch
    texels = random_texels(h, w, nch, seed=1000 * h + 10 * w + nch) if h else (torch.rand(nch, generator=torch.Generator().manual_seed(nch)) * 2 - 1)
    S = Setup(rb, dev, texels, SCALES[scale_i], d_uv_scale=scale_i != 1)
    ref = S.ref
    fam = families(ref, n, seed + 17 * scale_i) if not ref.constant else {"constant": np.random.default_rng(seed).uniform(-2, 2, (n, 6)).astype(np.float32)}
    rng = np.random.default_rng(seed + 1)
    report = {}
    all_strict_q, all_strict_d = [], []
    for fname, q in fam.items():
        d = d_values_for(rng, q.shape[0], nch)
        p = R.plan(ref, q)
        tag = "%dx%dx%d scale %s %s" % (h, w, nch, SCALES[scale_i], fname)
        values, dq, _, _ = S.run(q, d)
        nom = R.nominal(ref, q, d, p)
        check_values(tag, values, nom, np.arange(q.shape[0]))
        strict = np.nonzero(~p.depends)[0]
        dep = np.nonzero(p.depends)[0]
        check_dq_strict(tag, dq[strict], R.nominal(ref, q, d, p, strict))
        if dep.size:
            check_dq_one_sided(tag, dq, R.answers(ref, q, d, p, dep), dep)
        report[fname] = {"strict": int(strict.size), "one_sided": int(dep.size)}
        assert strict.size > 0, tag + ": no query compared strictly"
        all_strict_q.append(q[strict])
        all_strict_d.append(d[strict])
        # rounding-dependent queries: one per call, against their one-sided scatters
        for r in dep[:n_dep_scatter]:
            q1, d1 = q[r:r + 1], d[r:r + 1]
            p1 = R.plan(ref, q1)
            _, _, levels, uvs = S.run(q1, d1)
            msgs = []
            for a in R.answers(ref, q1, d1, p1, np.array([0])):
                ok, msg = scatter_ok(ref, levels, uvs, R.scatter(ref, a), S.with_uvs)
                if ok:
                    break
                msgs.append(msg)
            else:
                raise AssertionError("%s: query %s matches none of its one-sided scatters: %s" % (tag, q1.tolist(), msgs))
    # the scatter of every strictly compared query in one batch
    q = np.concatenate(all_strict_q)
    d = np.concatenate(all_strict_d)
    p = R.plan(ref, q)
    assert not p.depends.any()
    _, _, levels, uvs = S.run(q, d)
    ok, msg = scatter_ok(ref, levels, uvs, R.scatter(ref, R.nominal(ref, q, d, p)), S.with_uvs)
    assert ok, "%dx%dx%d scale %s, batch of %d queries: %s" % (h, w, nch, SCALES[scale_i], q.shape[0], msg)
    print(h, w, nch, SCALES[scale_i], report)
    return report


# ---------------------------------------------------------------------------------------------------- lane patterns
def lane_batch(ref, pattern, n, rng):
    """[n, 6] queries of a lane pattern for the scatter (the first 32 lanes of a warp are consecutive queries)."""
    L, w0 = ref.L, max(ref.w[0], 1)
    if pattern == "one_query":
        q = np.tile(np.array([[0.3172, 0.6211, 3.1 / w0, 0.4 / w0, -0.2 / w0, 1.7 / w0]]), (n, 1))
    elif pattern == "one_texel":  # every lane inside the same cell of level 0 with its own weights (clamped level)
        cell = np.array([2.0, 1.0])
        q = np.zeros((n, 6))
        q[:, :2] = (cell + 0.5 + rng.uniform(0.02, 0.98, (n, 2))) / np.array([w0, max(ref.h[0], 1)])
        q[:, 2:] = rng.uniform(-0.1, 0.1, (n, 4)) / w0
    elif pattern == "alternate_clamped":  # even lanes clamped at level 0 (one level), odd lanes between two levels
        q = np.zeros((n, 6))
        q[:, :2] = rng.random((n, 2))
        lev = np.where(np.arange(n) % 2 == 0, -2.0, rng.uniform(0.1, max(L - 1.1, 0.2), n))
        q[:, 2] = np.exp2(lev) / w0
        q[:, 5] = q[:, 2] * 0.3
    else:
        raise ValueError(pattern)
    return q.astype(np.float32)


# (texture, pattern, n); the 1x7 texture and the top levels of 13x7 wrap several taps of one lane onto one texel
LANE_CASES = [((13, 7, 3), "one_query", 32), ((13, 7, 3), "one_texel", 32), ((13, 7, 3), "alternate_clamped", 1000), ((1, 7, 5), "one_texel", 33),
              ((1, 7, 5), "alternate_clamped", 31), ((64, 64, 1), "alternate_clamped", 1), ((64, 64, 1), "one_query", 1 << 20),
              ((2, 2, 3), "one_texel", 1 << 20)]


def check_lanes(rb, dev, tex, pattern, n, seed=0):
    h, w, nch = tex
    S = Setup(rb, dev, random_texels(h, w, nch, seed=7 * h + w), (1.0, 1.0))
    rng = np.random.default_rng(seed)
    q = lane_batch(S.ref, pattern, n, rng)
    d = d_values_for(rng, n, nch)
    p = R.plan(S.ref, q)
    keep = ~p.depends
    q, d = q[keep], d[keep]
    assert q.shape[0] > 0
    p = R.plan(S.ref, q)
    sc = R.scatter(S.ref, R.nominal(S.ref, q, d, p))
    for perm in (None, rng.permutation(q.shape[0])):
        qq, dd = (q, d) if perm is None else (q[perm], d[perm])
        _, _, levels, uvs = S.run(qq, dd)
        ok, msg = scatter_ok(S.ref, levels, uvs, sc, True)
        assert ok, "%s %s n=%d%s: %s" % (tex, pattern, q.shape[0], "" if perm is None else " permuted", msg)
    return q.shape[0]


# exact sums: power-of-two sizes, texel centres / midpoints, clamped levels (zero or huge footprint), small integer d(value)
EXACT_CASES = [((1, 1, 1), 1 << 20), ((1, 1, 3), 1000), ((2, 2, 3), 33), ((64, 64, 1), 1 << 20), ((64, 64, 5), 31), ((1024, 1024, 3), 1 << 18),
               ((1024, 1024, 1), 1)]


def exact_batch(ref, n, rng):
    L = ref.L
    q = np.zeros((n, 6))
    top = rng.random(n) < 0.5
    lvl = np.where(top, L - 1, 0)
    W = np.array(ref.w, dtype=np.float64)[lvl]
    H = np.array(ref.h, dtype=np.float64)[lvl]
    kx = rng.integers(-2 * W.astype(np.int64) - 1, 3 * W.astype(np.int64) + 2) + rng.choice([0.5, 1.0], n)
    ky = rng.integers(-2 * H.astype(np.int64) - 1, 3 * H.astype(np.int64) + 2) + rng.choice([0.5, 1.0], n)
    q[:, 0], q[:, 1] = kx / W, ky / H
    big = np.exp2(rng.integers(L + 1, L + 20, n).astype(np.float64)) / ref.w[0]
    q[:, 2] = np.where(top, big, 0.0)
    q[:, 5] = np.where(top, big * 0.5, 0.0)
    # runs of equal queries (1 to 40 lanes long), so that warps aggregate groups of every size
    q = q[np.minimum(np.cumsum(rng.integers(1, 40, n)) // 20, n - 1)]
    return q.astype(np.float32)


def check_exact(rb, dev, tex, n, seed=0):
    h, w, nch = tex
    S = Setup(rb, dev, random_texels(h, w, nch, seed=3 * h + w), (1.0, 1.0))
    rng = np.random.default_rng(seed)
    q = exact_batch(S.ref, n, rng)
    d = rng.integers(-2, 3, (n, nch)).astype(np.float32)
    p = R.plan(S.ref, q)
    assert not p.depends.any()
    ans = R.nominal(S.ref, q, d, p)
    # every contribution a multiple of 1/4 and every element's sum of |c| below 2^22: all partial sums are exact float32
    assert np.all(np.mod(ans.tap_c * 4, 1) == 0), "a contribution that is not a multiple of 1/4"
    sc = R.scatter(S.ref, ans)
    for s, ab, _, _ in sc[0]:
        assert (ab * 4 < 2 ** 24).all(), "partial sums could round"
    for perm in (None, rng.permutation(n)):
        qq, dd = (q, d) if perm is None else (q[perm], d[perm])
        _, _, levels, uvs = S.run(qq, dd)
        ok, msg = scatter_ok(S.ref, levels, uvs, sc, True, exact=True)
        assert ok, "%s n=%d%s: %s" % (tex, n, "" if perm is None else " permuted", msg)


def check_arguments(rb, dev, lib, last_error, device_checks):
    """The hook refuses bad arguments with a message."""
    S = Setup(rb, dev, random_texels(2, 2, 3, 0), (1.0, 1.0))
    q = torch.zeros(4, 6, device=dev)
    v = torch.zeros(4, 3, device=dev)
    vp = ctypes.c_void_p
    assert lib.rb_texture_test(ctypes.byref(S.tex._c), None, vp(q.data_ptr()), -1, None, vp(v.data_ptr()), None, None) == 1
    assert "negative number of queries" in last_error(lib)
    for field, value, msg in (("channels", 0, "channels"), ("num_levels", 0, "num_levels"), ("num_levels", 9, "num_levels")):
        t = type(S.tex._c).from_buffer_copy(S.tex._c)
        setattr(t, field, value)
        assert lib.rb_texture_test(ctypes.byref(t), None, vp(q.data_ptr()), 4, None, vp(v.data_ptr()), None, None) == 1
        assert msg in last_error(lib), last_error(lib)
    if device_checks:
        host = torch.zeros(4, 6)
        assert lib.rb_texture_test(ctypes.byref(S.tex._c), None, vp(host.data_ptr()), 4, None, vp(v.data_ptr()), None, None) == 1
        assert "memory of the current device" in last_error(lib), last_error(lib)
        t = type(S.tex._c).from_buffer_copy(S.tex._c)
        t.texels[0] = host.data_ptr()
        assert lib.rb_texture_test(ctypes.byref(t), None, vp(q.data_ptr()), 4, None, vp(v.data_ptr()), None, None) == 1
        assert "memory of the current device" in last_error(lib), last_error(lib)
    with pytest.raises(ValueError):
        rb.texture_test(S.tex, torch.zeros(4, 5, device=dev))
    values, dq = rb.texture_test(S.tex, torch.zeros(0, 6, device=dev))
    assert values.shape == (0, 3) and dq is None


# ---------------------------------------------------------------------------------------------------- tests
DEV = torch.device("cuda:0")


def _rb():
    from redner_b200 import redner as rb
    return rb


@pytest.mark.parametrize("scale", range(len(SCALES)))
@pytest.mark.parametrize("tex", TEXTURES + [(0, 0, c) for c in CONSTANTS], ids=lambda t: "%dx%dx%d" % t if isinstance(t, tuple) else str(t))
def test_lookup_and_adjoint_against_float64(tex, scale):
    check_texture(_rb(), DEV, tex, scale, n=512)


@pytest.mark.parametrize("case", range(len(LANE_CASES)))
def test_scatter_lane_patterns(case):
    tex, pattern, n = LANE_CASES[case]
    check_lanes(_rb(), DEV, tex, pattern, n)


@pytest.mark.parametrize("case", range(len(EXACT_CASES)))
def test_exact_sums_bit_for_bit(case):
    tex, n = EXACT_CASES[case]
    check_exact(_rb(), DEV, tex, n)


def test_hook_rejects_bad_arguments():
    from redner_b200 import _lib
    check_arguments(_rb(), DEV, _lib.load(), _lib.last_error, device_checks=True)
