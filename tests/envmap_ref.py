"""A float64 restatement of the environment map (rb_envmap.cuh), for tests/test_envmap_gpu.py and tests/test_envmap_cpu.py.

Written from the reference's semantics (src/envmap.h:63-306), NumPy only, on top of tests/texture_ref.py for the texture lookup and its
adjoint.  It takes the float32 inputs exactly as the kernels see them: the direction and its ray differential, `world_to_env` /
`env_to_world`, the mip pyramid and the sampling tables that api.EnvironmentMap built, and restates
- envmap_eval: uv = (atan2(x, -z) / 2pi, acos(y) / pi) of the normalised local direction l, and the footprint
  du/d(l.x, l.z) = (l.x, l.z) / (2pi (l.x^2 + l.z^2)), dv/d(l.y) = -1 / (pi sqrt(1 - l.y^2)) applied to the transformed ray
  differential (no correction for a scaled `world_to_env`, as in the reference);
- d_envmap_eval: d(dir), d(dir_dx), d(dir_dy) and the 3x3 contribution to d(world_to_env), with the reference's 2pi (not pi) in the
  acos term;
- the pole rule (DESIGN.md section 4): the lookup is filtered only where |l.y| < 1 and l.x^2 + l.z^2 > 0; the acos term needs |l.y| < 1
  and the atan2 terms l.x^2 + l.z^2 > 0;
- envmap_sample in double, as the kernel computes it: the CDFs shifted by their first entry (api.py), upper_bound picks, the tent
  inverse CDF with its `0.5f`, then one rounding to float32 and the float32 transform by `env_to_world`;
- envmap_pdf of the direction as given (not normalised), bilinear in luminance with the reference's wrap of the row below the last.

Rounding.  The kernels compute the lookup in float32 with approximate division and square root; the restatement computes it in float64
and bounds the difference by linearisation.  Every place where float32 rounds on the way is an axis: the three components of l (the
transform, gamma_3, and the normalisation), the two transformed ray differentials, u and v (atan2 / acos and the division), 1 - l.y^2,
l.x^2 + l.z^2 and the two footprint lengths.  The answer is evaluated at the nominal point and at +- the error bound along each axis;
an output's tolerance is the sum over axes of the largest change, plus texture_ref's own bound for the lookup, plus CHAIN of the sum of
the magnitudes of the terms of the adjoint's own arithmetic.  Near a pole the change along l.y grows like 1 / theta and more: the bound
follows it because it is evaluated, not assumed.

Decisions.  A query depends on rounding when a decision differs at some perturbation from the nominal one: the filtered / pole branch,
l.x^2 + l.z^2 > 0, the mip levels, the floors of every level used (wrapped, so the atan2 seam itself is not a decision) and the u / v
branch of the footprint maximum; or when texture_ref says the lookup depends on rounding.  For those every perturbed point's answers
(and texture_ref's one-sided answers at each) are candidates."""
import math

import numpy as np

import texture_ref as T

U = T.EPS  # 2^-24
G3 = 4 * U  # a float32 3-term dot product (gamma_3, with room for a fused multiply-add)
CHAIN = 64 * U  # relative error of the adjoint's own float32 chain (a dozen rounded operations, several approximate divisions)
TWO_PI = 2 * math.pi
AXES = ("lx", "ly", "lz", "dxx", "dxy", "dxz", "dyx", "dyy", "dyz", "u", "v", "s", "xz", "fu", "fv")


def ulp32(x):
    return T._ulp32(x)


class Env:
    """An environment map as the kernels see it: the mip pyramid (list of [h, w, 3] float32), `w2e` / `e2w` [4, 4] float32, the sampling
    tables cdf_ys [h] and cdf_xs [h, w] float32, and pdf_norm as the float32 of rb_envmap."""

    def __init__(self, mips, w2e, e2w, cdf_ys, cdf_xs, pdf_norm):
        self.tex = T.Tex(mips, np.ones(2, np.float32))
        self.M = np.asarray(w2e, np.float32).astype(np.float64)[:3, :3]
        self.E = np.asarray(e2w, np.float32).astype(np.float64)[:3, :3]
        self.cdf_ys = np.asarray(cdf_ys, np.float32).astype(np.float64)
        self.cdf_xs = np.asarray(cdf_xs, np.float32).astype(np.float64)
        self.pdf_norm = float(np.float32(pdf_norm))
        self.h, self.w = self.tex.h[0], self.tex.w[0]
        lum_w = np.array([0.212671, 0.715160, 0.072169], np.float32).astype(np.float64)
        self.lum = (self.tex.f64[0] * lum_w).sum(1).reshape(self.h, self.w)
        self.lum_max = float(np.abs(self.lum).max())


# ---------------------------------------------------------------------------------------------------- lookup and adjoint
class Inputs:
    pass


def _xfm(M, v):
    """env_xfm_vector in the kernel's order, term by term (a matrix product in BLAS may lose the sign of a zero, which decides atan2 at
    the seam and u at the poles)"""
    return np.stack([(M[i, 0] * v[:, 0] + M[i, 1] * v[:, 1]) + M[i, 2] * v[:, 2] for i in range(3)], 1)


def inputs(env, q):
    """Float64 values of the float32 steps before the lookup, and their error bounds: n = w2e dir, l = n / |n|, ldx, ldy."""
    q = np.asarray(q, np.float32).astype(np.float64)
    x = Inputs()
    x.dir, x.ddx, x.ddy = q[:, 0:3], q[:, 3:6], q[:, 6:9]
    M, aM = env.M, np.abs(env.M)
    x.n = _xfm(M, x.dir)
    e_n = G3 * (np.abs(x.dir) @ aM.T)
    x.nn = np.sqrt((x.n ** 2).sum(1))
    pos = x.nn > 0
    x.l = np.zeros_like(x.n)
    x.l[pos] = x.n[pos] / x.nn[pos, None]
    r = np.zeros(len(q))
    r[pos] = np.sqrt((e_n[pos] ** 2).sum(1)) / x.nn[pos]
    x.e_l = np.zeros_like(x.n)
    x.e_l[pos] = e_n[pos] / x.nn[pos, None] + np.abs(x.l[pos]) * (r[pos, None] + 8 * U)
    x.ldx, x.ldy = _xfm(M, x.ddx), _xfm(M, x.ddy)
    x.e_ldx, x.e_ldy = G3 * (np.abs(x.ddx) @ aM.T), G3 * (np.abs(x.ddy) @ aM.T)
    return x


def _forward(l, ldx, ldy, sh):
    """uv, footprint and branches of local directions l (float64) with the perturbations sh (dict of axis -> [n] shift)."""
    X, Y, Z = l[:, 0], l[:, 1], l[:, 2]
    f = {}
    f["xz"] = (X ** 2 + Z ** 2) * (1 + sh.get("xz", 0.0))
    f["s"] = np.maximum(1 - Y ** 2 + sh.get("s", 0.0), 2.0 ** -24)  # (where |l.y| < 1 the float32 1 - l.y^2 is at least 2^-23)
    f["ylt1"] = np.abs(Y) < 1
    f["xzpos"] = f["xz"] > 0
    f["filtered"] = f["ylt1"] & f["xzpos"]
    u = np.arctan2(X, -Z) / TWO_PI + sh.get("u", 0.0)
    v = np.where(Y >= 1, 0.0, np.where(Y <= -1, math.pi, np.arccos(np.clip(Y, -1, 1)))) / math.pi + sh.get("v", 0.0)
    fl = f["filtered"]
    xz = np.where(fl, f["xz"], 1.0)
    sq = np.sqrt(np.where(fl, f["s"], 1.0))
    f["du_dx"] = np.where(fl, X / (TWO_PI * xz), 0.0)
    f["du_dz"] = np.where(fl, Z / (TWO_PI * xz), 0.0)
    f["dv_dy"] = np.where(fl, -1 / (math.pi * sq), 0.0)
    du = np.stack([f["du_dx"] * ldx[:, 0] + f["du_dz"] * ldx[:, 2], f["du_dx"] * ldy[:, 0] + f["du_dz"] * ldy[:, 2]], 1) * (1 + np.asarray(sh.get("fu", 0.0)))[..., None]
    dv = np.stack([f["dv_dy"] * ldx[:, 1], f["dv_dy"] * ldy[:, 1]], 1) * (1 + np.asarray(sh.get("fv", 0.0)))[..., None]
    f["q"] = np.concatenate([u[:, None], v[:, None], du, dv], 1)
    return f


def _adjoint(M, l, nn, ldx, ldy, dirs, f, dq, absmode=False):
    """d(dir), d(dir_dx), d(dir_dy) [n, 9] and the d(world_to_env) contribution [n, 3, 3] for the texture adjoint dq [n, 6].  With
    absmode every factor is taken by magnitude and every difference becomes a sum: the sum of the magnitudes of the terms."""
    A = (lambda a: np.abs(a)) if absmode else (lambda a: a)
    sub = (lambda a, b: a + b) if absmode else (lambda a, b: a - b)
    neg = (lambda a: np.abs(a)) if absmode else (lambda a: -a)
    M = A(M)
    X, Y, Z = A(l[:, 0]), A(l[:, 1]), A(l[:, 2])
    ldx, ldy, dirs = A(ldx), A(ldy), [A(d) for d in dirs]
    d_uv, d_du, d_dv = A(dq[:, 0:2]), A(dq[:, 2:4]), A(dq[:, 4:6])
    n = len(l)
    fl, xzp, ylt = f["filtered"], f["xzpos"], f["ylt1"]
    xz = np.where(xzp, f["xz"], 1.0)
    s = np.where(ylt, f["s"], 1.0)
    sq = np.sqrt(np.abs(s))
    du_dx, du_dz, dv_dy = A(f["du_dx"]), A(f["du_dz"]), A(f["dv_dy"])
    d_l = np.zeros((n, 3))
    d_ldx = np.zeros((n, 3))
    d_ldy = np.zeros((n, 3))
    # the footprint terms (filtered only)
    d_dv_dy = d_dv[:, 0] * ldx[:, 1] + d_dv[:, 1] * ldy[:, 1]
    d_ldx[:, 1] = d_dv[:, 0] * dv_dy
    d_ldy[:, 1] = d_dv[:, 1] * dv_dy
    d_l[:, 1] = neg(d_dv_dy) * Y / (math.pi * sq * s)
    d_du_dx = d_du[:, 0] * ldx[:, 0] + d_du[:, 1] * ldy[:, 0]
    d_du_dz = d_du[:, 0] * ldx[:, 2] + d_du[:, 1] * ldy[:, 2]
    d_ldx[:, 0] = d_du[:, 0] * du_dx
    d_ldx[:, 2] = d_du[:, 0] * du_dz
    d_ldy[:, 0] = d_du[:, 1] * du_dx
    d_ldy[:, 2] = d_du[:, 1] * du_dz
    den = TWO_PI * xz ** 2
    d_l[:, 2] += d_du_dz * sub(X ** 2, Z ** 2) / den
    d_l[:, 0] = sub(d_l[:, 0], d_du_dz * X * Z / den)
    d_l[:, 0] += d_du_dx * sub(Z ** 2, X ** 2) / den
    d_l[:, 2] = sub(d_l[:, 2], d_du_dx * X * Z / den)
    for a in (d_l, d_ldx, d_ldy):
        a[~fl] = 0
    # atan2 and acos terms
    d_l[:, 0] += np.where(xzp, neg(d_uv[:, 0]) * Z / (xz * TWO_PI), 0.0)
    d_l[:, 2] += np.where(xzp, neg(d_uv[:, 0]) * X / (xz * TWO_PI), 0.0)
    d_l[:, 1] += np.where(ylt, neg(d_uv[:, 1]) / (sq * TWO_PI), 0.0)
    # d_normalize: (d_l - l (d_l . l)) / |n|
    pos = nn > 0
    L3 = np.stack([X, Y, Z], 1)
    dot = (d_l * L3).sum(1)
    d_n = np.zeros((n, 3))
    d_n[pos] = (sub(d_l[pos], L3[pos] * dot[pos, None])) / nn[pos, None]
    dm = np.zeros((n, 3, 3))
    out = np.zeros((n, 9))
    for k, (dv3, v) in enumerate(((d_n, dirs[0]), (d_ldx, dirs[1]), (d_ldy, dirs[2]))):
        dm += dv3[:, :, None] * v[:, None, :]
        out[:, 3 * k:3 * k + 3] = dv3 @ M
    return out, dm


def _decisions(t, f, p):
    """One int64 row of decisions per query: the branches and texture_ref's decisions at the float64 point (floors wrapped)."""
    cols = [f["filtered"], f["xzpos"], f["ylt1"], p.l0[:, 0], p.nl[:, 0], p.u_is_max]
    for l in range(t.L):
        cols.append(np.where(p.used[:, l], np.mod(p.xf[:, l, 0], t.w[l]), -1))
        cols.append(np.where(p.used[:, l], np.mod(p.yf[:, l, 0], t.h[l]), -1))
    return np.stack([np.asarray(c, np.int64) for c in cols], 1)


class Eval:
    pass


def _evaluate(env, x, d_out, sh, rows=None):
    """The answer at one perturbed point: forward branches, texture plan and nominal texture answer, adjoint."""
    t = env.tex
    rows = np.arange(len(x.l)) if rows is None else rows
    sh = {k: np.broadcast_to(np.asarray(v, np.float64), (len(x.l),)) for k, v in sh.items()}
    g = lambda *names: np.stack([sh[a] if a in sh else np.zeros(len(x.l)) for a in names], 1)[rows]  # noqa: E731
    l = x.l[rows] + g("lx", "ly", "lz")
    ldx = x.ldx[rows] + g("dxx", "dxy", "dxz")
    ldy = x.ldy[rows] + g("dyx", "dyy", "dyz")
    shr = {k: v[rows] for k, v in sh.items()}
    f = _forward(l, ldx, ldy, shr)
    q32 = f["q"].astype(np.float32)
    p = T.plan(t, q32)
    d = np.asarray(d_out, np.float32).astype(np.float64)[rows]
    a = T.nominal(t, q32, d, p)
    e = Eval()
    e.f, e.p, e.a, e.q32, e.l, e.ldx, e.ldy, e.d = f, p, a, q32, l, ldx, ldy, d
    e.key = _decisions(t, f, p)
    dirs = (x.dir[rows], x.ddx[rows], x.ddy[rows])
    e.dq, e.dm = _adjoint(env.M, l, x.nn[rows], ldx, ldy, dirs, f, a.d_q)
    e.value = a.value
    return e


def _axis_shift(x, axis, sign):
    n = len(x.l)
    e = {"lx": x.e_l[:, 0], "ly": x.e_l[:, 1], "lz": x.e_l[:, 2], "dxx": x.e_ldx[:, 0], "dxy": x.e_ldx[:, 1], "dxz": x.e_ldx[:, 2],
         "dyx": x.e_ldy[:, 0], "dyy": x.e_ldy[:, 1], "dyz": x.e_ldy[:, 2]}
    if axis in e:
        return {axis: sign * e[axis]}
    X, Y, Z = x.l[:, 0], x.l[:, 1], x.l[:, 2]
    if axis == "u":  # atan2 (a few ulps), the float32 2pi and the approximate division
        u = np.arctan2(X, -Z) / TWO_PI
        return {"u": sign * (8 * ulp32(u) + 1e-45)}
    if axis == "v":
        v = np.arccos(np.clip(Y, -1, 1)) / math.pi
        return {"v": sign * 8 * ulp32(v)}
    if axis == "s":  # 1 - y * y: the rounding of the product (the difference is then exact or within an ulp of the result)
        return {"s": sign * (U * Y ** 2 + U * np.abs(1 - Y ** 2))}
    if axis == "xz":
        return {"xz": sign * 3 * U * np.ones(n)}
    return {axis: sign * 8 * U * np.ones(n)}  # fu, fv: the footprint's products, sums and approximate square root


class Result:
    """Per query: value [n, 3], value_tol, dq [n, 9] (d_dir, d_dir_dx, d_dir_dy), dq_tol, dm [n, 3, 3], dm_tol; `strict` [n];
    `undetermined` [n]: queries so close to a pole that the float32 error of l moves u or v by more than half a texel of level 0 (or
    reaches the size of (l.x, l.z)), whose value can only be bounded by the texels of the rows at that pole (pole_lo, pole_hi: the rows next to it, and the wrapped row, of every level); for the
    rounding-dependent queries `candidates`: list of (rows, value, dq, dm, value_tol, dq_tol, dm_tol); `taps`: texture_ref Answer of the
    strict rows with widened tap_err (for texture_ref.scatter)."""
    pass


def _merge(a, b):
    out = dict(a)
    for k, v in b.items():
        out[k] = out[k] + v if k in out else v
    return out


def _spread(env, x, d_out, base, rows):
    """Around the point shifted by `base`, for queries `rows`: that point's evaluation, the sum over axes of the largest change of value
    (among the perturbations that keep its pole branch), d(queries) and d(world_to_env) (among those that keep all its decisions), and whether every perturbation kept them.  Also
    the perturbed evaluations whose decisions differ (shift, rows where they differ).  The evaluation keeps every perturbed point's
    texture answer (axis_evals)."""
    b = _evaluate(env, x, d_out, base, rows)
    m = len(rows)
    sv, sq, sm = np.zeros((m, 3)), np.zeros((m, 9)), np.zeros((m, 3, 3))
    same = ~b.p.depends
    flips = []
    b.axis_evals = []
    for axis in AXES:
        bv, bq, bm = np.zeros((m, 3)), np.zeros((m, 9)), np.zeros((m, 3, 3))
        for sign in (1.0, -1.0):
            sh = _merge(base, _axis_shift(x, axis, sign))
            ev = _evaluate(env, x, d_out, sh, rows)
            b.axis_evals.append((axis, ev.a))
            ok = (ev.key == b.key).all(1) & ~ev.p.depends
            same &= ok
            if (~ok).any():
                flips.append((sh, ~ok))
            # (the value is continuous across the floors, levels and the branch of the footprint maximum: only the pole branch cuts it)
            same_branch = ev.f["filtered"] == b.f["filtered"]
            bv = np.maximum(bv, np.where(same_branch[:, None], np.abs(ev.value - b.value), 0))
            bq = np.maximum(bq, np.where(ok[:, None], np.abs(ev.dq - b.dq), 0))
            bm = np.maximum(bm, np.where(ok[:, None, None], np.abs(ev.dm - b.dm), 0))
        sv, sq, sm = sv + bv, sq + bq, sm + bm
    return b, (sv, sq, sm), same, flips


def lookup(env, q, d_out):
    """The restated lookup, adjoint and their bounds for queries q [n, 9] float32 and d_out [n, 3] float32."""
    x = inputs(env, q)
    n = len(x.l)
    allrows = np.arange(n)
    nom, (spread_v, spread_q, spread_m), same, flips = _spread(env, x, d_out, {}, allrows)
    r = Result()
    r.value, r.dq, r.dm = nom.value, nom.dq, nom.dm
    # near a pole the float32 error of l moves u (and v) by more than half a texel of level 0, where the value is not linear in it any
    # more, and where the error of (l.x, l.z) reaches their size the azimuth is not determined by the inputs at all
    e_xz = np.hypot(x.e_l[:, 0], x.e_l[:, 2])
    r_xz = np.hypot(x.l[:, 0], x.l[:, 2])
    Y, e_y = x.l[:, 1], x.e_l[:, 1]
    dv_err = (np.arccos(np.clip(Y - e_y, -1, 1)) - np.arccos(np.clip(Y + e_y, -1, 1))) / math.pi
    with np.errstate(divide="ignore", invalid="ignore"):
        du_err = np.where(r_xz > 0, e_xz / (TWO_PI * r_xz), np.where(e_xz > 0, np.inf, 0.0))
    r.undetermined = (r_xz < 4 * e_xz) | (du_err * env.w > 0.5) | (dv_err * env.h > 0.5)
    north = x.l[:, 1] > 0
    r.pole_lo, r.pole_hi = np.zeros((n, 3)), np.zeros((n, 3))
    for side, rows_of in ((True, lambda h: [0, 1] if h > 1 else [0]), (False, lambda h: [h - 2, h - 1] if h > 1 else [0])):
        vals = np.concatenate([m.reshape(m.shape[0], m.shape[1], 3)[rows_of(m.shape[0]) + [0, m.shape[0] - 1]].reshape(-1, 3) for m in env.tex.mips])
        sel = north == side
        r.pole_lo[sel], r.pole_hi[sel] = vals.min(0), vals.max(0)
    r.strict = same & ~r.undetermined
    # where float32 may or may not round l onto a pole, the filtered side's footprint terms go like (1 - l.y^2)^(-3/2) with 1 - l.y^2 a
    # few float32 ulps, and no perturbation bounds them: there only the value is compared, and the adjoint must be finite
    r.pole_ambiguous = np.zeros(n, bool)
    for axis in ("lx", "ly", "lz", "s", "xz"):
        for sign in (1.0, -1.0):
            sh = _axis_shift(x, axis, sign)
            l = x.l + np.stack([sh.get(a, np.zeros(n)) for a in ("lx", "ly", "lz")], 1)
            f = _forward(l, x.ldx, x.ldy, {k: v for k, v in sh.items() if k in ("s", "xz")})
            r.pole_ambiguous |= f["filtered"] != nom.f["filtered"]
    r.pole_ambiguous &= ~r.strict & ~r.undetermined

    def tols(ev, rows):
        # texture_ref's bounds through the adjoint, and the adjoint's own arithmetic
        tq, tm = _adjoint(env.M, ev.l, x.nn[rows], ev.ldx, ev.ldy, (x.dir[rows], x.ddx[rows], x.ddy[rows]), ev.f, ev.a.dq_tol, absmode=True)
        aq, am = _adjoint(env.M, ev.l, x.nn[rows], ev.ldx, ev.ldy, (x.dir[rows], x.ddx[rows], x.ddy[rows]), ev.f, ev.a.d_q, absmode=True)
        return ev.a.value_tol, tq + CHAIN * aq, tm + CHAIN * am
    vt, qt, mt = tols(nom, allrows)
    r.value_tol = vt + spread_v
    r.dq_tol = qt + spread_q
    r.dm_tol = mt + spread_m
    # one-sided candidates of the rounding-dependent queries: the nominal point and every perturbed point whose decisions differ, each
    # with its own spread and texture_ref's one-sided answers there
    dep = np.nonzero(~r.strict & ~r.undetermined)[0]
    r.dependent = dep
    r.candidates = []
    if dep.size:
        is_dep = np.zeros(n, bool)
        is_dep[dep] = True
        # every flip point lies inside the +- bound box of every other one (they differ by one step along at most two axes), so one
        # point per query and new set of decisions is enough: the linear bound of its box covers the others with the same decisions
        covered = {int(i): {nom.key[i].tobytes()} for i in dep}
        points = [({}, dep)]
        for sh, mask in flips:
            rows = np.nonzero(mask & is_dep)[0]
            if rows.size == 0:
                continue
            ev = _evaluate(env, x, d_out, sh, rows)
            new = np.array([ev.p.depends[i] or ev.key[i].tobytes() not in covered[int(r)] for i, r in enumerate(rows)], bool)
            for i in np.nonzero(new)[0]:
                covered[int(rows[i])].add(ev.key[i].tobytes())
            points.append((sh, rows[new]))
        for sh, rows in points:
            if rows.size == 0:
                continue
            if sh:
                b, (sv, sq, sm), _, _ = _spread(env, x, d_out, sh, rows)
            else:  # (the nominal point: its spread is already known)
                b, sv, sq, sm = _evaluate(env, x, d_out, {}, rows), spread_v[rows], spread_q[rows], spread_m[rows]
            for a in T.answers(env.tex, b.q32, b.d, b.p, np.arange(rows.size)):
                k = a.qid
                evr = Eval()
                evr.f = {key: (v[k] if np.ndim(v) else v) for key, v in b.f.items()}
                evr.l, evr.ldx, evr.ldy, evr.a = b.l[k], b.ldx[k], b.ldy[k], a
                g = rows[k]
                dq, dm = _adjoint(env.M, evr.l, x.nn[g], evr.ldx, evr.ldy, (x.dir[g], x.ddx[g], x.ddy[g]), evr.f, a.d_q)
                vt, qt, mt = tols(evr, g)
                r.candidates.append((g, a.value, dq, dm, vt + sv[k], qt + sq[k], mt + sm[k]))
    # texel contributions of the strict rows: texture_ref's taps at the nominal point, widened by their change along every axis
    st = np.nonzero(r.strict)[0]
    r.strict_rows = st
    # (the perturbed points of the nominal spread: a strict query keeps its decisions at every one, so its taps line up with the nominal's)
    r.taps = None
    if st.size:
        sel = np.isin(nom.a.tap_qrow, st)
        c0 = nom.a.tap_c[sel]
        widen = np.zeros(c0.size)
        for axis in AXES:
            best = np.zeros_like(widen)
            for name, a in nom.axis_evals:
                if name != axis:
                    continue
                k = np.isin(a.tap_qrow, st)
                assert k.sum() == c0.size and (a.tap_index[k] == nom.a.tap_index[sel]).all()
                best = np.maximum(best, np.abs(a.tap_c[k] - c0))
            widen += best
        r.taps = Taps(nom.a.tap_level[sel], nom.a.tap_index[sel], nom.a.tap_channel[sel], c0, nom.a.tap_err[sel] + widen)
    r.dm_strict, r.dm_tol_strict = r.dm[st], r.dm_tol[st]
    return r


class Taps:
    """Texel contributions (texture_ref.Answer's tap arrays) for texture_ref.scatter."""

    def __init__(self, level, index, channel, c, err):
        self.tap_level, self.tap_index, self.tap_channel, self.tap_c, self.tap_err = level, index, channel, c, err
        self.tap_qrow = np.zeros(c.size, np.int64)
        self.uvs = self.uvs_err = np.zeros((0, 1, 2))


def at_local(env, q, d_out, l, nn):
    """The answer where the kernel's float32 local direction l [n, 3] and |w2e dir| nn [n] are known exactly (a direction that float32
    normalises onto a pole): (value, d(queries) [n, 9], d(world_to_env) [n, 3, 3]) and their bounds, texture_ref's own and the adjoint's
    arithmetic.  No decision may depend on rounding there."""
    x = inputs(env, q)
    l = np.asarray(l, np.float64)
    nn = np.asarray(nn, np.float64)
    f = _forward(l, x.ldx, x.ldy, {})
    q32 = f["q"].astype(np.float32)
    p = T.plan(env.tex, q32)
    assert not p.depends.any()
    d = np.asarray(d_out, np.float32).astype(np.float64)
    a = T.nominal(env.tex, q32, d, p)
    dirs = (x.dir, x.ddx, x.ddy)
    dq, dm = _adjoint(env.M, l, nn, x.ldx, x.ldy, dirs, f, a.d_q)
    tq, tm = _adjoint(env.M, l, nn, x.ldx, x.ldy, dirs, f, a.dq_tol, absmode=True)
    aq, am = _adjoint(env.M, l, nn, x.ldx, x.ldy, dirs, f, a.d_q, absmode=True)
    return a.value, dq, dm, a.value_tol, tq + CHAIN * aq, tm + CHAIN * am


# ---------------------------------------------------------------------------------------------------- pdf
def _pdf64(env, l, sh):
    X, Y, Z = l[:, 0], l[:, 1], l[:, 2]
    u = np.arctan2(X, -Z) / TWO_PI + sh.get("u", 0.0)
    v = np.where(Y >= 1, 0.0, np.where(Y <= -1, math.pi, np.arccos(np.clip(Y, -1, 1)))) / math.pi + sh.get("v", 0.0)
    w, h = env.w, env.h
    x, y = u * w - 0.5, v * h - 0.5
    xfi, yfi = np.mod(np.floor(x), w).astype(np.int64), np.mod(np.floor(y), h).astype(np.int64)
    xci, yci = np.mod(xfi + 1, w), np.mod(yfi + 1, h)
    dx, dy = x - xfi, y - yfi
    dx = np.where(dx < 0, dx + w, dx)
    dy = np.where(dy < 0, dy + h, dy)
    L = env.lum
    lum_fy = L[yfi, xfi] * (1 - dx) * (1 - dy) + L[yfi, xci] * dx * (1 - dy)
    lum_cy = L[yci, xfi] * (1 - dx) * dy + L[yci, xci] * dx * dy
    s2 = np.maximum(1 - Y ** 2 + sh.get("s", 0.0), 0)
    st = np.sqrt(s2)
    s_fy = np.abs(np.sin(math.pi * (yfi + 0.5) / h))
    s_cy = np.abs(np.sin(math.pi * (yci + 0.5) / h))
    zero = st == 0
    pdf = np.where(zero, 0.0, env.pdf_norm * np.abs(lum_fy * s_fy + lum_cy * s_cy) / np.where(zero, 1.0, st))
    mag = env.pdf_norm * (np.abs(lum_fy) * s_fy + np.abs(lum_cy) * s_cy) / np.where(zero, 1.0, st)
    # the float32 bilinear weights: x = u w - 0.5, x - floor(x) and its wrap by + w each round to the spacing of their result, which
    # for the wrap is that of w (and likewise in y); the pdf moves by at most the weight error times the taps' luminance
    e_dx = 2 * ulp32(np.abs(x) + w) + ulp32(x)
    e_dy = 2 * ulp32(np.abs(y) + h) + ulp32(y)
    taps = (np.abs(L[yfi, xfi]) + np.abs(L[yfi, xci])) * s_fy + (np.abs(L[yci, xfi]) + np.abs(L[yci, xci])) * s_cy
    werr = env.pdf_norm * (e_dx + e_dy) * taps / np.where(zero, 1.0, st)
    return pdf, zero, mag, werr


def pdf(env, q):
    """(pdf [n], tol [n], one_sided [n]): envmap_pdf of the directions q[:, 0:3] as given.  Where the pole decision (sin_theta == 0)
    flips within the bounds, both 0 and the other side are answers: `one_sided` marks them and `alt` holds the non-zero side."""
    x = inputs(env, q)
    aM = np.abs(env.M)
    n_ = x.n
    e_n = G3 * (np.abs(x.dir) @ aM.T)
    p0, z0, mag, werr = _pdf64(env, n_, {})
    X, Y, Z = n_[:, 0], n_[:, 1], n_[:, 2]
    spread = np.zeros(len(p0))
    one_sided = np.zeros(len(p0), bool)
    alt = np.where(z0, 0.0, p0)
    alt_tol = np.zeros(len(p0))
    axes = [{"l": k} for k in range(3)] + [{"u": 8 * ulp32(np.arctan2(X, -Z) / TWO_PI) + 1e-45},
                                           {"v": 8 * ulp32(np.arccos(np.clip(Y, -1, 1)) / math.pi)}, {"s": U * Y ** 2 + U * np.abs(1 - Y ** 2)}]
    for ax in axes:
        best = np.zeros(len(p0))
        for sign in (1.0, -1.0):
            if "l" in ax:
                nl = n_.copy()
                nl[:, ax["l"]] += sign * e_n[:, ax["l"]]
                p1, z1, _, _ = _pdf64(env, nl, {})
            else:
                k, v = next(iter(ax.items()))
                p1, z1, _, _ = _pdf64(env, n_, {k: sign * v})
            flip = z1 != z0
            one_sided |= flip
            alt = np.where(flip & z0, np.maximum(alt, p1), alt)
            best = np.maximum(best, np.where(flip, 0.0, np.abs(p1 - p0)))
        spread += best
    tol = spread + 32 * U * mag + werr + 1e-45
    return p0, tol, one_sided, alt


# ---------------------------------------------------------------------------------------------------- sampling
def _pick(cdf, x):
    """env_cdf_pick: upper_bound of x in the ascending float table, minus one, clamped"""
    return np.clip(np.searchsorted(cdf, x, side="right") - 1, 0, len(cdf) - 1)


def _tent(x):
    return np.where(x < 0.5, 1 - np.sqrt(2 * x), np.sqrt(np.maximum(2 * x - 0.5, 0)) - 1)


def sample_local(env, s):
    """The double local direction of envmap_sample for samples s [m, 2] (sx, sy), before the rounding to float32."""
    s = np.asarray(s, np.float64)
    sx, sy = s[:, 0].copy(), s[:, 1].copy()
    w, h = env.w, env.h
    cy = env.cdf_ys
    yp = _pick(cy, sy)
    last = yp >= h - 1
    nxt = cy[np.minimum(yp + 1, h - 1)]
    with np.errstate(divide="ignore", invalid="ignore"):
        sy = np.where(last, (sy - cy[yp]) / (1 - cy[yp]), (sy - cy[yp]) / (nxt - cy[yp]))
    # the column pick in the picked row's table, one row at a time (a [samples, width] gather of a wide map would not fit)
    xp = np.zeros(len(sx), np.int64)
    c0, c1 = np.zeros(len(sx)), np.ones(len(sx))
    for r in np.unique(yp):
        k = yp == r
        row = env.cdf_xs[r]
        xp[k] = _pick(row, sx[k])
        c0[k] = row[xp[k]]
        c1[k] = np.where(xp[k] < w - 1, row[np.minimum(xp[k] + 1, w - 1)], 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        sx = (sx - c0) / (c1 - c0)
    u = xp + _tent(sx)
    v = yp + _tent(sy)
    phi = (2 * math.pi / w) * (u + 0.5)
    theta = (math.pi / h) * (v + 0.5)
    sp, cp, st, ct = np.sin(phi), np.cos(phi), np.sin(theta), np.cos(theta)
    return np.stack([sp * st, ct, -cp * st], 1)


def sample(env, s):
    """(candidates [m, 2, 3] float32 local directions, ambiguous [m, 3]): the float32 rounding of the double local direction, and the
    other neighbour where the double lies within 16 double ulps of a float32 rounding midpoint (double sin / cos and the products on the
    device may differ from NumPy's by a few double ulps)."""
    loc = sample_local(env, s)
    r = loc.astype(np.float32)
    r64 = r.astype(np.float64)
    other = np.where(loc > r64, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf)))
    mid = 0.5 * (r64 + other.astype(np.float64))
    amb = np.abs(loc - mid) <= 16 * np.spacing(np.abs(loc)) + 1e-300
    return np.stack([r, np.where(amb, other, r)], 1), amb


def transform_tol(env, local32):
    """the float32 transform of local32 by env_to_world: float64 value and gamma_3 bound"""
    l = np.asarray(local32, np.float32).astype(np.float64)
    return l @ env.E.T, G3 * (np.abs(l) @ np.abs(env.E).T) + 1e-45
