"""GPU suite: the environment map (rb_envmap.cuh: envmap_eval, d_envmap_eval with its aggregated scatters, envmap_sample, envmap_pdf)
through the test hook rb_envmap_test, query by query, against the float64 restatement in tests/envmap_ref.py; and the backward pass of
environment-lit scenes that look at or bounce towards the map's poles.

Maps (api.EnvironmentMap, so the pyramid and the sampling tables are the real ones): 1x1, 1x2, 2x1, 5x13, 16x32 and 1024x2048 with its
full pyramid, a 16x32 map with zero-luminance rows and columns, one with one hot texel and one black except its last row; each with an
identity env_to_world, a general rotation and a rotation with non-uniform scale.  Direction families: uniform on the sphere, exact seam
directions with both signs of zero, both poles exactly and rings at 1e-6 ... 1e-2 rad around each, unnormalised directions of length
1e-3 ... 1e3, and ray differentials that are zero, below a texel, inside each level, above the top level and anisotropic.  Sample
families: a uniform grid, every CDF entry as a double and one double ulp either side, 0 and 1 - 2^-53, and values in zero-width CDF
segments; an entry of a column table is paired with an sy that picks its own row (every pickable row of the smaller maps, eight of the
wide one).

Comparison rules (tolerances from envmap_ref: the float32 error bound of every rounded step before the lookup, turned into each
output's tolerance by evaluating the restatement at +- that bound; texture_ref's bounds for the lookup itself; 64 ulps of the adjoint's
own arithmetic relative to the sum of the magnitudes of its terms):
- every output of every finite query is finite: values, pdfs, d(dir), d(dir_dx), d(dir_dy), texel and world_to_env gradients, samples;
- values and d(dir, dir_dx, dir_dy) strictly where no decision depends on rounding, and otherwise equal to one of the one-sided answers
  (each perturbed point's, and texture_ref's one-sided answers there); both counted per family.  Where the float32 error of the local
  direction moves u or v by more than half a texel of level 0 (close to a pole, more so on a wide map) the answer is not linear in that
  error any more, and where it reaches the size of the local (x, z) the azimuth is not determined by the inputs at all: there the value
  must lie between the smallest and largest texel of the rows at that pole, and every output must be finite; these are counted too.  Where float32 may or may not round the direction onto a pole, the
  adjoint of the filtered side goes like (1 - l.y^2)^(-3/2) with 1 - l.y^2 a few float32 ulps: there the value is compared with the
  one-sided answers and the adjoint must be finite (counted as pole_ambiguous);
- pdfs within their bound; where the pole decision (sin theta == 0) flips within the bound, 0 or a finite non-negative value;
- samples: with an identity env_to_world the float32 rounding of the restated double direction, bit for bit (either neighbour where the
  double lies within 16 double ulps of a rounding midpoint); otherwise within gamma_3 of the float32 transform of that direction;
- texel and world_to_env gradients of a batch of strict queries within gamma_k * sum(|c| + err) + sum(err) of the float64 sum, k the
  element's number of contributions (every query adds into the same 12 floats of world_to_env); elements without contributions, the
  fourth column and the last row of world_to_env exactly zero; a few rounding-dependent queries alone, each matching one of its
  one-sided world_to_env contributions;
- exact sums: directions that float32 rounds onto the north pole with u = 0 put weight 1/4 on the same four texels, so with integer
  d_out every contribution and partial sum is exact, and the texel gradient must equal the float64 sum bit for bit at several lane
  patterns (a lane lost or counted twice shows); there the pole branch is deterministic, so d(dir, dir_dx, dir_dy) and the
  world_to_env sum are compared with the restated pole branch (atan2 term only) within its bounds;
- guard zones: the gradient pyramid and world_to_env gradient are views into one allocation with 64 guard floats around each; guards
  must stay exactly zero.

The lookup checks are shared with tests/test_envmap_cpu.py, which runs them on the host build of the device headers (tools/cpu_emu)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import envmap_ref as R
import texture_ref as T

pytestmark = pytest.mark.gpu

GUARD = 64
MAPS = ["1x1", "1x2", "2x1", "5x13", "16x32", "zero_rows_cols", "hot_texel", "last_row", "1024x2048"]
XFORMS = ["identity", "rotation", "rotation_scale"]


# ---------------------------------------------------------------------------------------------------- maps and buffers
def map_texels(name, seed=0):
    g = torch.Generator().manual_seed(seed + 31 * MAPS.index(name))
    if "x" in name and name[0].isdigit():
        h, w = (int(s) for s in name.split("x"))
        return (torch.rand(h, w, 3, generator=g) * 2).float()
    t = (torch.rand(16, 32, 3, generator=g) * 2).float()
    if name == "zero_rows_cols":
        t[[0, 5, 15]] = 0
        t[:, [3, 7, 8, 31]] = 0
    elif name == "hot_texel":
        t[:] = 1e-3
        t[9, 21] = 100.0
    elif name == "last_row":
        t[:-1] = 0
    return t


def _rot(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def env_to_world(name):
    m = np.eye(4)
    if name == "rotation":
        m[:3, :3] = _rot([0.3, -0.8, 0.52], 1.1)
    elif name == "rotation_scale":
        m[:3, :3] = _rot([-0.6, 0.2, 0.77], 2.3) @ np.diag([1.7, 0.45, 1.2])
    return torch.tensor(m, dtype=torch.float32)


class Setup:
    """An environment map on `dev` through api.EnvironmentMap and the library's wrappers, its float64 restatement and a guarded gradient
    buffer (pyramid and world_to_env gradient)."""

    def __init__(self, rb, dev, texels, e2w):
        from redner_b200 import api
        self.rb, self.dev = rb, dev
        env = api.EnvironmentMap(texels.to(dev), env_to_world=e2w.contiguous())
        self.env = env
        self.mips = [m.contiguous() for m in env.values.mipmap]
        fp = lambda t: rb.float_ptr(t.data_ptr())  # noqa: E731
        ws, hs = [int(m.shape[1]) for m in self.mips], [int(m.shape[0]) for m in self.mips]
        self.tex = rb.Texture3([fp(m) for m in self.mips], ws, hs, 3, fp(env.values.uv_scale))
        self.renv = rb.EnvironmentMap(self.tex, fp(env.env_to_world), fp(env.world_to_env), fp(env.sample_cdf_ys), fp(env.sample_cdf_xs),
                                      env.pdf_norm, True)
        self.ref = R.Env([m.cpu().numpy() for m in self.mips], env.world_to_env.numpy(), env.env_to_world.numpy(), env.sample_cdf_ys.cpu().numpy(),
                         env.sample_cdf_xs.cpu().numpy(), self.renv._c.pdf_norm)
        sizes = [m.numel() for m in self.mips]
        self.buf = torch.zeros(GUARD + sum(s + GUARD for s in sizes) + 16 + GUARD, dtype=torch.float32, device=dev)
        self.views, off = [], GUARD
        for s in sizes:
            self.views.append((off, s))
            off += s + GUARD
        self.w2e_off = off
        self.d_tex = rb.Texture3([rb.float_ptr(self.buf.data_ptr() + 4 * o) for o, _ in self.views], ws, hs, 3, None)
        self.ws, self.hs = ws, hs

    def run(self, q, d_out=None, samples=None):
        """(values, pdfs, d_queries, sample_dirs, gradient levels [size, 3], d_w2e [4, 4]) of one call, after zeroing the gradients;
        guard zones must stay zero."""
        self.buf.zero_()
        qt = torch.as_tensor(np.asarray(q, np.float32)).to(self.dev)
        dt = None if d_out is None else torch.as_tensor(np.asarray(d_out, np.float32)).to(self.dev)
        st = None if samples is None else torch.as_tensor(np.asarray(samples, np.float64)).to(self.dev)
        w2e = self.buf[self.w2e_off:self.w2e_off + 16]
        values, pdfs, dq, sd = self.rb.envmap_test(self.renv, qt, dt, self.d_tex if dt is not None else None, w2e if dt is not None else None, st)
        buf = self.buf.cpu().numpy()
        guard = np.ones(buf.size, bool)
        levels = []
        for o, s in self.views:
            guard[o:o + s] = False
            levels.append(buf[o:o + s].reshape(-1, 3).astype(np.float64))
        guard[self.w2e_off:self.w2e_off + 16] = False
        bad = np.nonzero(guard & (buf != 0))[0]
        assert bad.size == 0, "a write outside the gradient buffers: %d guard floats touched, first at offset %d" % (bad.size, bad[0])
        f = lambda t: None if t is None else t.cpu().numpy().astype(np.float64)  # noqa: E731
        return f(values), f(pdfs), f(dq), None if sd is None else sd.cpu().numpy(), levels, buf[self.w2e_off:self.w2e_off + 16].astype(np.float64).reshape(4, 4)


# ---------------------------------------------------------------------------------------------------- query families
def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _tangents(d, rng):
    a = np.where(np.abs(d[:, 1:2]) < 0.9, np.array([[0.0, 1.0, 0.0]]), np.array([[1.0, 0.0, 0.0]]))
    t1 = np.cross(d, a)
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(d, t1)
    ang = rng.uniform(0, 2 * math.pi, (len(d), 1))
    return np.cos(ang) * t1 + np.sin(ang) * t2, -np.sin(ang) * t1 + np.cos(ang) * t2


def ray_diffs(ref, d, rng, kind):
    """dir_dx, dir_dy [n, 3] of a kind: zero, sub_texel, levels, above_top, anisotropic or mixed (angles in units of a texel of level 0)"""
    n = len(d)
    texel = 2 * math.pi / ref.w
    L = ref.tex.L
    if kind == "mixed":
        kinds = rng.choice(["zero", "sub_texel", "levels", "above_top", "anisotropic"], n)
        out = np.zeros((n, 6))
        for k in set(kinds):
            s = kinds == k
            out[s] = ray_diffs(ref, d[s], rng, k)
        return out
    if kind == "zero":
        return np.zeros((n, 6))
    t1, t2 = _tangents(d, rng)
    lo, hi = {"sub_texel": (-12, -1), "levels": (0, max(L - 1, 0.5)), "above_top": (L, L + 6), "anisotropic": (-2, L + 1)}[kind]
    m1 = np.exp2(rng.uniform(lo, hi, (n, 1))) * texel
    m2 = m1 * (np.exp2(-rng.uniform(3, 10, (n, 1))) if kind == "anisotropic" else rng.uniform(0.3, 1, (n, 1)))
    sw = rng.random((n, 1)) < 0.5
    return np.concatenate([np.where(sw, m1, m2) * t1, np.where(sw, m2, m1) * t2], 1)


def families(ref, n, seed):
    """{family: [n', 9] float32 queries}; local directions are mapped to the world by env_to_world, so that poles and seam are the map's"""
    rng = np.random.default_rng(seed)
    E = ref.E

    def world(local):
        w = local @ E.T
        return w / np.linalg.norm(w, axis=1, keepdims=True)

    def q(d, kind="mixed"):
        return np.concatenate([d, ray_diffs(ref, d / np.linalg.norm(d, axis=1, keepdims=True), rng, kind)], 1).astype(np.float32)
    fam = {}
    fam["uniform"] = q(_unit(rng, n))
    # the seam: local x = +-0, local z > 0 (atan2(+-0, -z) = +-pi); with an identity transform the zero's sign reaches atan2
    k = n // 2
    th = rng.uniform(0.05, math.pi - 0.05, k)
    loc = np.stack([np.where(rng.random(k) < 0.5, 0.0, -0.0), np.cos(th), np.sin(th)], 1)
    seam = world(loc) if not np.array_equal(E, np.eye(3)) else loc
    fam["seam"] = q(seam)
    # the poles exactly and rings around them
    rings = []
    for pole in (1.0, -1.0):
        for theta in (0.0, 1e-6, 1e-5, 1e-4, 2.4e-4, 3e-4, 1e-3, 1e-2):
            m = max(n // 16, 2)
            ph = rng.uniform(0, 2 * math.pi, m)
            loc = np.stack([math.sin(theta) * np.sin(ph), pole * math.cos(theta) * np.ones(m), -math.sin(theta) * np.cos(ph)], 1)
            rings.append(loc)
    loc = np.concatenate(rings)
    fam["poles"] = q(world(loc) if not np.array_equal(E, np.eye(3)) else loc)
    fam["unnormalised"] = q(_unit(rng, n) * np.exp(rng.uniform(math.log(1e-3), math.log(1e3), (n, 1))))
    for kind in ("zero", "sub_texel", "levels", "above_top", "anisotropic"):
        fam["rd_" + kind] = q(_unit(rng, n), kind)
    return fam


def d_out_for(rng, n):
    return rng.uniform(-1, 1, (n, 3)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- comparisons
def _within(got, want, tol):
    return np.abs(got - want) <= tol + 1e-30


def _match(name, what, got, r, strict_want, strict_tol, cand_index, fam, skip=None):
    """strict rows of the family mask `fam` against the nominal answer, its rounding-dependent rows (but `skip`) against any candidate;
    returns (strict, one_sided)"""
    st, dep = r.strict_rows[fam[r.strict_rows]], r.dependent[fam[r.dependent]]
    if skip is not None:
        dep = dep[~skip[dep]]
    ok = _within(got[st], strict_want[st], strict_tol[st]).all(1)
    bad = st[~ok]
    assert bad.size == 0, "%s: %d %s differ from float64, e.g. query %d: got %s want %s tol %s" % (
        name, bad.size, what, bad[0], got[bad[0]].tolist(), strict_want[bad[0]].tolist(), strict_tol[bad[0]].tolist())
    matched = np.zeros(got.shape[0], bool)
    for c in r.candidates:
        g, want, tol = c[0], c[cand_index[0]], c[cand_index[1]]
        matched[g[_within(got[g], want, tol).all(1)]] = True
    miss = [int(i) for i in dep if not matched[i]]
    assert not miss, "%s: %d rounding-dependent queries' %s match none of their one-sided answers, e.g. query %d: got %s, answers %s" % (
        name, len(miss), what, miss[0], got[miss[0]].tolist(), [c[cand_index[0]][c[0] == miss[0]].tolist() for c in r.candidates if (c[0] == miss[0]).any()][:6])
    return int(st.size), int(dep.size)


def _finite(name, **arrays):
    for k, a in arrays.items():
        if a is None:
            continue
        bad = ~np.isfinite(a)
        assert not bad.any(), "%s: %d non-finite %s, e.g. at %s" % (name, int(bad.sum()), k, np.argwhere(bad)[0].tolist())


def sums_ok(ref, levels, d_w2e, taps, dm, dm_tol):
    """(ok, message): texel and world_to_env gradients of a batch of strict queries against the float64 sums"""
    if taps is not None:
        lv, _ = T.scatter(ref.tex, taps)
        for l, (got, (s, ab, er, ct)) in enumerate(zip(levels, lv)):
            tol = T.gamma(ct) * (ab + er) + er
            bad = (np.abs(got - s) > tol) | ((ct == 0) & (got != 0))
            if bad.any():
                i = np.argwhere(bad)[0]
                return False, "level %d texel %d channel %d: got %r, float64 %r, tol %r, %d contributions" % (
                    l, i[0], i[1], float(got[i[0], i[1]]), float(s[i[0], i[1]]), float(tol[i[0], i[1]]), int(ct[i[0], i[1]]))
    k = dm.shape[0]
    s, ab, er = dm.sum(0), np.abs(dm).sum(0), dm_tol.sum(0)
    tol = T.gamma(k) * (ab + er) + er
    got = d_w2e[:3, :3]
    if (np.abs(got - s) > tol).any():
        return False, "d_w2e %s, float64 %s, tol %s" % (got.tolist(), s.tolist(), tol.tolist())
    if (d_w2e[:, 3] != 0).any() or (d_w2e[3] != 0).any():
        return False, "d_w2e outside its upper 3x3: %s" % d_w2e.tolist()
    return True, ""


def check_lookups(rb, dev, map_name, xform, n=128, n_dep_scatter=3, seed=0):
    """Every direction family on one map and transform, restated in one batch; returns {family: counts}."""
    S = Setup(rb, dev, map_texels(map_name), env_to_world(xform))
    ref = S.ref
    rng = np.random.default_rng(seed + 1)
    fams = families(ref, n, seed + 7 * XFORMS.index(xform))
    q = np.concatenate(list(fams.values()))
    fam_of = np.concatenate([np.full(len(v), i) for i, v in enumerate(fams.values())])
    d = d_out_for(rng, q.shape[0])
    values, pdfs, dq, _, levels, d_w2e = S.run(q, d)
    _finite("%s %s" % (map_name, xform), values=values, pdfs=pdfs, d_queries=dq, d_w2e=d_w2e, texel_gradients=np.concatenate(levels))
    r = R.lookup(ref, q, d)
    p0, ptol, one_sided, _ = R.pdf(ref, q)
    report = {}
    for i, fname in enumerate(fams):
        tag = "%s %s %s" % (map_name, xform, fname)
        fam = fam_of == i
        und = np.nonzero(r.undetermined & fam)[0]
        inside = ((values[und] >= r.pole_lo[und] * (1 - 1e-6)) & (values[und] <= r.pole_hi[und] * (1 + 1e-6))).all(1)
        assert inside.all(), "%s: query %d, azimuth undetermined at the pole: value %s outside the pole rows' [%s, %s]" % (
            tag, und[~inside][0], values[und[~inside][0]].tolist(), r.pole_lo[und[~inside][0]].tolist(), r.pole_hi[und[~inside][0]].tolist())
        ns, nd = _match(tag, "values", values, r, r.value, r.value_tol, (1, 4), fam)
        _match(tag, "d(dir, dir_dx, dir_dy)", dq, r, r.dq, r.dq_tol, (2, 5), fam, skip=r.pole_ambiguous)
        ok = _within(pdfs, p0, ptol) | (one_sided & (pdfs >= 0))
        bad = np.nonzero(~ok & fam)[0]
        assert bad.size == 0, "%s: %d pdfs differ, e.g. query %d: got %r want %r tol %r" % (tag, bad.size, bad[0], pdfs[bad[0]], p0[bad[0]], ptol[bad[0]])
        report[fname] = {"strict": ns, "one_sided": nd, "pole_unresolved": int(und.size), "pole_ambiguous": int((r.pole_ambiguous & fam).sum()),
                         "pdf_one_sided": int((one_sided & fam).sum())}
        if fname not in ("poles",):
            assert ns > 0, tag + ": no query compared strictly"
        # rounding-dependent queries alone: their world_to_env contribution against the one-sided ones
        for k in r.dependent[fam[r.dependent]][:n_dep_scatter]:
            _, _, _, _, _, w1 = S.run(q[k:k + 1], d[k:k + 1])
            got = w1[:3, :3]
            if not any(np.all(np.abs(got - c[3][c[0] == k][0]) <= T.gamma(1) * np.abs(c[3][c[0] == k][0]) + c[6][c[0] == k][0] + 1e-30)
                       for c in r.candidates if (c[0] == k).any()):
                raise AssertionError("%s: query %d's d_w2e %s matches none of its one-sided contributions" % (tag, k, got.tolist()))
    # every strict query in one batch: texel and world_to_env sums
    st = r.strict_rows
    _, _, _, _, levels, d_w2e = S.run(q[st], d[st])
    ok, msg = sums_ok(ref, levels, d_w2e, r.taps, r.dm_strict, r.dm_tol_strict)
    assert ok, "%s %s, batch of %d strict queries: %s" % (map_name, xform, st.size, msg)
    print(map_name, xform, report)
    return report


# ---------------------------------------------------------------------------------------------------- samples
MAX_ENTRY_ROWS = 8  # (rows of a wide map whose column entries are all sampled; smaller maps: every pickable row)


def sample_families(ref, seed):
    """{family: [m, 2] double samples (sx, sy)}.  Column-table samples are paired with an sy that picks the row they belong to."""
    rng = np.random.default_rng(seed)
    one = 1 - 2.0 ** -53
    fam = {}
    g = (np.arange(16) + 0.5) / 16
    fam["grid"] = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    ys, xs = ref.cdf_ys, ref.cdf_xs
    # the rows env_cdf_pick can return, and an sy inside each one's interval [ys[r], next entry or 1)
    nxt = np.append(ys[1:], 1.0)
    rows = np.nonzero(nxt > ys)[0]
    sy_row = ys[rows] + 0.5 * (nxt[rows] - ys[rows])
    assert (R._pick(ys, sy_row) == rows).all()
    near = lambda c: np.concatenate([c, np.nextafter(c, -1), np.nextafter(c, 2)])  # noqa: E731
    # every entry of the row table, and one double ulp either side, with a random sx
    sy = near(ys)
    ent = [np.stack([rng.random(sy.size), sy], 1)]
    # every entry of the column tables of the pickable rows (a few rows of a wide map), and one double ulp either side, in their row
    pick = rows if rows.size <= MAX_ENTRY_ROWS or ref.w * rows.size <= 4096 else rng.choice(rows, MAX_ENTRY_ROWS, replace=False)
    for r in pick:
        sx = near(xs[r])
        ent.append(np.stack([sx, np.full(sx.size, sy_row[rows == r][0])], 1))
    fam["cdf_entries"] = np.clip(np.concatenate(ent), 0, one)
    fam["ends"] = np.array([[0, 0], [0, one], [one, 0], [one, one], [0.5, 0], [0, 0.5], [one, 0.5], [0.5, one]])
    # zero-width segments: a repeated entry of the row table with a random sx, and a repeated entry of a pickable row's column table in
    # that row
    zs = [np.stack([rng.random(int((np.diff(ys) == 0).sum())), ys[1:][np.diff(ys) == 0]], 1)]
    for r, sy_r in zip(rows, sy_row):
        zx = xs[r, 1:][np.diff(xs[r]) == 0]
        zs.append(np.stack([zx, np.full(zx.size, sy_r)], 1))
    fam["zero_width"] = np.concatenate(zs)
    # (a sampler draws from [0, 1): a table entry of exactly 1, the end of a zero-width last segment, is not a sample)
    return {k: np.asarray(v, np.float64)[(np.asarray(v) < 1).all(1)] for k, v in fam.items() if len(v)}


def check_samples(rb, dev, map_name, xform, seed=0):
    S = Setup(rb, dev, map_texels(map_name), env_to_world(xform))
    ref = S.ref
    identity = np.array_equal(ref.E, np.eye(3))
    report = {}
    for fname, s in sample_families(ref, seed).items():
        tag = "%s %s samples %s" % (map_name, xform, fname)
        _, _, _, got, _, _ = S.run(np.zeros((0, 9), np.float32), None, s)
        _finite(tag, samples=got.astype(np.float64))
        cand, amb = R.sample(ref, s)
        if identity:
            ok = ((got == cand[:, 0]) | (got == cand[:, 1])).all(1)
        else:
            ok = np.zeros(len(s), bool)
            for c in range(2):
                want, tol = R.transform_tol(ref, cand[:, c])
                ok |= _within(got.astype(np.float64), want, tol).all(1)
        bad = np.nonzero(~ok)[0]
        assert bad.size == 0, "%s: %d samples differ, e.g. sample %r: got %s want %s" % (tag, bad.size, s[bad[0]].tolist(), got[bad[0]].tolist(), cand[bad[0]].tolist())
        report[fname] = {"n": int(len(s)), "rounding_ambiguous": int(amb.any(1).sum())}
    print(map_name, xform, report)
    return report


# ---------------------------------------------------------------------------------------------------- exact sums, lane patterns
EXACT_CASES = [1, 31, 32, 33, 1000, 1 << 18]


def check_exact(rb, dev, n, seed=0):
    """Directions that float32 normalises onto the north pole with u = +-0: the lookup is unfiltered at level 0, x = y = -0.5, and every
    query puts weight 1/4 on the same four texels.  Integer d_out makes every contribution and partial sum exact."""
    S = Setup(rb, dev, map_texels("16x32"), env_to_world("identity"))
    rng = np.random.default_rng(seed)
    c = rng.choice([1.0, 2.0, 0.5, 4.0], n)
    delta = rng.uniform(1e-6, 1e-4, n)
    q = np.zeros((n, 9), np.float32)
    q[:, 0] = rng.choice([0.0, -0.0], n)
    q[:, 1] = c
    q[:, 2] = -c * delta
    q[:, 3:] = rng.uniform(-1e-2, 1e-2, (n, 6))  # (ignored at the pole)
    q32 = q[:, :3]
    nn = np.sqrt((q32 * q32).sum(1, dtype=np.float32))
    assert (q32[:, 1] / nn == 1).all(), "a direction float32 does not normalise onto the pole"
    d = rng.integers(-2, 3, (n, 3)).astype(np.float32)
    d = d[np.minimum(np.cumsum(rng.integers(1, 40, n)) // 20, n - 1)]  # runs of equal d_out, so that warps aggregate groups of every size
    tq = np.zeros((n, 6), np.float32)
    p = T.plan(S.ref.tex, tq)
    assert not p.depends.any()
    ans = T.nominal(S.ref.tex, tq, d.astype(np.float64), p)
    assert np.all(np.mod(ans.tap_c * 4, 1) == 0)
    lv, _ = T.scatter(S.ref.tex, ans)
    # the pole branch's adjoint there: no footprint and no acos term, the atan2 term d_l.x = -d_uv.x l.z / (2 pi (l.x^2 + l.z^2))
    l32 = np.stack([q32[:, 0], np.ones(n, np.float32), q32[:, 2] / nn], 1)
    want_v, want_dq, want_dm, tol_v, tol_dq, tol_dm = R.at_local(S.ref, q, d, l32, nn)
    assert (np.abs(want_dq[:, 0]) > 0).any(), "no query with a non-zero atan2 term"
    for perm in (None, rng.permutation(n)):
        qq, dd = (q, d) if perm is None else (q[perm], d[perm])
        values, _, dq, _, levels, d_w2e = S.run(qq, dd)
        tag = "exact n=%d%s" % (n, "" if perm is None else " permuted")
        _finite(tag, values=values, d_queries=dq, d_w2e=d_w2e)
        order = np.arange(n) if perm is None else perm
        for what, got, want, tol in (("values", values, want_v[order], tol_v[order]), ("d(dir, dir_dx, dir_dy)", dq, want_dq[order], tol_dq[order])):
            bad = np.nonzero(~_within(got, want, tol).all(1))[0]
            assert bad.size == 0, "%s: %d %s differ from the pole branch's, e.g. query %d: got %s want %s tol %s" % (
                tag, bad.size, what, bad[0], got[bad[0]].tolist(), want[bad[0]].tolist(), tol[bad[0]].tolist())
        ok, msg = sums_ok(S.ref, [np.zeros_like(g) for g in levels], d_w2e, None, want_dm, tol_dm)
        assert ok, tag + ": " + msg
        for l, (got, (s, ab, _, ct)) in enumerate(zip(levels, lv)):
            assert (ab * 4 < 2 ** 24).all()
            bad = got != s
            assert not bad.any(), "exact n=%d%s level %d: got %s, float64 %s" % (n, "" if perm is None else " permuted", l, got[bad][:4].tolist(), s[bad][:4].tolist())


def check_arguments(rb, dev, lib, last_error, device_checks):
    """The hook refuses bad arguments with a message."""
    from redner_b200 import _lib
    S = Setup(rb, dev, map_texels("2x1"), env_to_world("identity"))
    q = torch.zeros(4, 9, device=dev)
    v = torch.zeros(4, 3, device=dev)
    vp = ctypes.c_void_p

    def call(env=S.renv._c, d_values=None, d_out=None, n=4, m=0, queries=q):
        return lib.rb_envmap_test(ctypes.byref(env) if env is not None else None, ctypes.byref(d_values) if d_values is not None else None, None,
                                  vp(queries.data_ptr()), n, vp(d_out.data_ptr()) if d_out is not None else None, vp(v.data_ptr()), None, None, None, m,
                                  None, None)
    assert call(n=-1) == 1 and "negative number" in last_error(lib)
    assert call(m=-1) == 1 and "negative number" in last_error(lib)
    assert call(env=None) == 1 and "null environment map" in last_error(lib)
    assert call(d_out=v) == 1 and "needs a gradient pyramid" in last_error(lib)
    bad = _lib.rb_envmap.from_buffer_copy(S.renv._c)
    bad.values.channels = 1
    assert call(env=bad) == 1 and "3 channels" in last_error(lib), last_error(lib)
    wrong = _lib.rb_texture.from_buffer_copy(S.d_tex._c)
    wrong.width[0] += 1
    assert call(d_values=wrong, d_out=v) == 1 and "level sizes" in last_error(lib), last_error(lib)
    wrong = _lib.rb_texture.from_buffer_copy(S.d_tex._c)
    wrong.num_levels -= 1
    assert call(d_values=wrong, d_out=v) == 1 and "levels and channels" in last_error(lib), last_error(lib)
    if device_checks:
        assert call(queries=torch.zeros(4, 9)) == 1 and "memory of the current device" in last_error(lib), last_error(lib)
        host = _lib.rb_envmap.from_buffer_copy(S.renv._c)
        host_table = torch.zeros(4)
        host.sample_cdf_ys = host_table.data_ptr()
        assert call(env=host) == 1 and "sampling tables" in last_error(lib), last_error(lib)
    with pytest.raises(ValueError):
        rb.envmap_test(S.renv, torch.zeros(4, 6, device=dev))
    values, pdfs, dq, sd = rb.envmap_test(S.renv, torch.zeros(0, 9, device=dev))
    assert values.shape == (0, 3) and dq is None and sd is None


# ---------------------------------------------------------------------------------------------------- tests
DEV = torch.device("cuda:0")


def _rb():
    from redner_b200 import redner as rb
    return rb


@pytest.mark.parametrize("xform", XFORMS)
@pytest.mark.parametrize("map_name", MAPS)
def test_lookup_and_adjoint_against_float64(map_name, xform):
    check_lookups(_rb(), DEV, map_name, xform, n=48 if map_name == "1024x2048" else 128)  # (the wide map's restatement is the slow part)


@pytest.mark.parametrize("xform", XFORMS)
@pytest.mark.parametrize("map_name", MAPS)
def test_samples_against_float64(map_name, xform):
    check_samples(_rb(), DEV, map_name, xform)


@pytest.mark.parametrize("n", EXACT_CASES)
def test_exact_sums_bit_for_bit(n):
    check_exact(_rb(), DEV, n)


def test_hook_rejects_bad_arguments():
    from redner_b200 import _lib
    check_arguments(_rb(), DEV, _lib.load(), _lib.last_error, device_checks=True)


# ---------------------------------------------------------------------------------------------------- end to end
def _pole_scene(kind, device):
    """Environment-lit scenes whose rays reach the map's poles: a glossy upward floor seen straight from above (its reflections of the
    centre pixels leave towards the zenith), a pinhole camera and a fisheye camera looking straight up, and a pinhole camera looking at
    the pole of a map rotated so that the pole is not a world axis.  Every input that has a gradient requires one.  Pixels are sampled at
    their centres and the resolution is odd, so the centre pixel's ray is the optical axis, on the pole (a random position in one of these
    65 x 65 pixels at 45 degrees would reach the 2.4e-4 rad cap around it with probability ~1e-3)."""
    from redner_b200 import api
    g = torch.Generator().manual_seed(5)
    tilt = 0.7 if kind == "pinhole_tilted_pole" else 0.0
    e2w = torch.tensor([[1.0, 0.0, 0.0, 0.0], [0.0, math.cos(tilt), -math.sin(tilt), 0.0], [0.0, math.sin(tilt), math.cos(tilt), 0.0],
                        [0.0, 0.0, 0.0, 1.0]], requires_grad=True)
    pole = [0.0, math.cos(tilt), math.sin(tilt)]
    sky = (0.2 + 1.5 * torch.rand(16, 32, 3, generator=g)).to(device).requires_grad_(True)
    env = api.EnvironmentMap(sky, e2w)
    if kind == "mirror_floor":
        pos, look, up, ctype = [0.0, 2.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 1.0], 0
    else:
        pos = [0.0, 0.5, 0.0]
        look, up, ctype = [pos[i] + pole[i] for i in range(3)], [0.0, -pole[2], pole[1]] if tilt else [0.0, 0.0, 1.0], 2 if kind == "fisheye_up" else 0
    cam = api.Camera(position=torch.tensor(pos, requires_grad=True), look_at=torch.tensor(look, requires_grad=True), up=torch.tensor(up),
                     fov=torch.tensor([45.0]), clip_near=1e-2, resolution=(65, 65), camera_type=ctype)
    tex = (0.2 + 0.6 * torch.rand(8, 8, 3, generator=g)).to(device).requires_grad_(True)
    spec = torch.tensor([0.8, 0.8, 0.8], device=device, requires_grad=True)
    rough = torch.tensor([0.002], device=device, requires_grad=True)
    m_floor = api.Material(diffuse_reflectance=api.Texture(tex), specular_reflectance=spec, roughness=rough)
    v = torch.tensor([[-3.0, 0.0, -3.0], [-3.0, 0.0, 3.0], [3.0, 0.0, -3.0], [3.0, 0.0, 3.0]], device=device, requires_grad=True)
    floor = api.Shape(v, torch.tensor([[0, 1, 2], [1, 3, 2]], dtype=torch.int32, device=device), 0,
                      uvs=torch.tensor([[0.0, 0.0], [0.0, 1.0], [1.0, 0.0], [1.0, 1.0]], device=device))
    scene = api.Scene(cam, [floor], [m_floor], [], envmap=env)
    return scene, {"sky texels": sky, "env_to_world": e2w, "camera position": cam.position, "camera look_at": cam.look_at, "floor vertices": v,
                   "floor texture": tex, "specular": spec, "roughness": rough}


def render_pole_scene(kind, deterministic, device=DEV, spp=64):
    """{input: number of non-finite gradient elements} of one backward pass of a pole scene"""
    from redner_b200 import api
    rb = _rb()
    scene, inputs = _pole_scene(kind, device)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic, warn_only=True)
    try:
        # (secondary edges are not available with an environment map; primary edges carry the camera's boundary gradient)
        args = api.RenderFunction.serialize_scene(scene, spp, 2, device=device, backend=rb, sample_pixel_center=True,
                                                  use_secondary_edge_sampling=False)
        img = api.RenderFunction.apply(3, *args)
        assert torch.isfinite(img).all(), "%s: non-finite image" % kind
        img.sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    counts = {}
    for name, t in inputs.items():
        assert t.grad is not None, "%s: no gradient for %s" % (kind, name)
        counts[name] = int((~torch.isfinite(t.grad)).sum())
    return counts


POLE_SCENES = ["mirror_floor", "pinhole_zenith", "fisheye_up", "pinhole_tilted_pole"]


@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("kind", POLE_SCENES)
def test_gradients_finite_at_the_poles(kind, deterministic):
    counts = render_pole_scene(kind, deterministic)
    print(kind, deterministic, counts)
    assert not any(counts.values()), "%s: non-finite gradient elements: %s" % (kind, counts)
