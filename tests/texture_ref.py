"""A float64 restatement of the texture lookup and its adjoint, for tests/test_texture_gpu.py and tests/test_texture_cpu.py.

Written from the reference's semantics (src/texture.h:53-140 trilinear_interp, :142-323 d_trilinear_interp, :335-419
get_texture_value / d_get_texture_value), NumPy only.  It takes the mip pyramid that api.Texture builds (so the box filter is not
re-derived here) and evaluates, per query:
- the value of every channel;
- d(uv), d(du_dxy), d(dv_dxy) for the given d(value);
- every texel contribution of the adjoint, per level, and the uv_scale contribution;
- constant textures (value = texels[0], adjoint = d(value) into texels[0]).

The kernels compute in float32, so some decisions of a lookup can go either way by rounding.  For each query `plan` reports whether
its answer depends on rounding: one of these lies within the float32 error bound of its computation (a few float32 ulps; zero when
every float32 operation on the way is exact):
- x = u * sx * w - 0.5 or y at a level the query uses is near an integer, so `floor` can flip;
- level is near 0, near an integer, or near num_levels - 1, so the level pair can change;
- fu is near fv, so the branch of the maximum can flip (an exact tie that float32 computes with the same operations on the same
  values, e.g. du = (a, 0), dv = (0, a) on a square texture with sx == sy, is not rounding-dependent: it takes the u branch).
For such queries `answers` gives every one-sided answer: each combination of the sides of its ambiguous decisions.

Error bounds (`Bounds`), also from the float32 rounding of each step: dx, dy and dlevel bound |x32 - x|, |y32 - y| and
|level32 - level|; the tests turn them into tolerances through the sensitivity of each output to x, y and level."""
import itertools
import math

import numpy as np

EPS = 2.0 ** -24  # unit roundoff of float32
F32_1E8 = float(np.float32(1e-8))  # the footprint clamp, a float32 literal in both codes
LN2 = math.log(2.0)
ARITH = 32 * EPS  # relative error of the few rounded products and sums of one bilinear tap set, with room to spare


def _ulp32(x):
    """the spacing of float32 at |x| (its normal range; float32's smallest normal spacing below it)"""
    a = np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** -126)
    return np.ldexp(1.0, np.frexp(a)[1] - 24)


def _is_f32(x):
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore"):
        return x.astype(np.float32).astype(np.float64) == x


class Tex:
    """A texture as the kernels see it: `mips` is the list of [h, w, channels] float32 arrays of api.Texture (cut at 8 levels), or one
    [channels] array for a constant texture; `uv_scale` two float32."""

    def __init__(self, mips, uv_scale):
        self.mips = [np.asarray(m, dtype=np.float32) for m in mips]
        self.constant = self.mips[0].ndim == 1
        self.nch = int(self.mips[0].shape[-1])
        self.L = len(self.mips)
        self.w = [int(m.shape[1]) if not self.constant else 0 for m in self.mips]
        self.h = [int(m.shape[0]) if not self.constant else 0 for m in self.mips]
        self.sx, self.sy = (float(s) for s in np.asarray(uv_scale, dtype=np.float32))
        self.f64 = [m.astype(np.float64).reshape(-1, self.nch) for m in self.mips]
        self.M = max(float(np.abs(m).max()) for m in self.f64)  # (bounds use the largest texel magnitude)


class Plan:
    """The float64 decisions of every query, their float32 error bounds and which of them may flip."""
    pass


def plan(t, q):
    """Decisions and rounding dependence of queries q [n, 6] (float32 values) on texture t."""
    q32 = np.asarray(q, dtype=np.float32)
    q = q32.astype(np.float64)
    n = q.shape[0]
    p = Plan()
    p.n = n
    if t.constant:
        p.depends = np.zeros(n, bool)
        return p
    sx, sy = t.sx, t.sy
    f32 = np.float32
    # uv * uv_scale: one float32 product each, reproduced exactly (float32 multiplication is correctly rounded)
    pu32 = (q32[:, 0] * f32(sx)).astype(np.float64)
    pv32 = (q32[:, 1] * f32(sy)).astype(np.float64)
    pu, pv = q[:, 0] * sx, q[:, 1] * sy
    L = t.L
    p.x = np.stack([pu * t.w[l] - 0.5 for l in range(L)], 1)  # [n, L] in float64 from the float32 inputs
    p.y = np.stack([pv * t.h[l] - 0.5 for l in range(L)], 1)

    def coord_bound(p32, pe, size):
        # |x32 - x|: the error of the product, scaled by the level size, plus the final rounding of p * size - 0.5 (fused: half an
        # ulp; two roundings: at most one ulp of the larger operand); zero where both steps are exact
        out = []
        for s in size:
            xe = p32 * s - 0.5  # (exact in float64)
            exact = (p32 == pe) & _is_f32(p32 * s) & _is_f32(xe)
            out.append(np.where(exact, 0.0, np.abs(p32 - pe) * s + _ulp32(np.abs(p32 * s) + 0.5)))
        return np.stack(out, 1)
    p.dx = coord_bound(pu32, pu, t.w)
    p.dy = coord_bound(pv32, pv, t.h)
    # footprint and level
    du, dv = q[:, 2:4] * sx, q[:, 4:6] * sy
    p.fu = np.sqrt((du ** 2).sum(1)) * t.w[0]
    p.fv = np.sqrt((dv ** 2).sum(1)) * t.h[0]
    p.max_fp = np.maximum(p.fu, p.fv)
    p.level = np.log2(np.maximum(p.max_fp, F32_1E8))

    def fp_exact(d_in, s, size):
        # every float32 step exact and the footprint a power of two with one zero component (sqrt of a power of four): then the
        # approximate square root and log2 are exact as well
        d32 = (d_in.astype(np.float32) * f32(s)).astype(np.float64)
        one_zero = (d32 == 0).any(1)
        sq = (d32 ** 2).sum(1)
        fp = np.sqrt(sq) * size
        m, e = np.frexp(fp)
        return (d32 == d_in * s).all(1) & _is_f32(d32 ** 2).all(1) & one_zero & (m == 0.5) & _is_f32(fp)
    exact_u = fp_exact(q[:, 2:4], sx, t.w[0])
    exact_v = fp_exact(q[:, 4:6], sy, t.h[0])
    level_exact = np.where(p.fu >= p.fv, exact_u, exact_v) | (p.max_fp < F32_1E8 / 2)
    # |level32 - level|: the footprint's relative error (ARITH: products, squares, sum, approximate sqrt) through log2, plus the
    # rounding of log2 itself (4 ulps of the level)
    p.dlevel = np.where(level_exact, 0.0, ARITH / LN2 + 4 * _ulp32(p.level))
    # the u / v branch of the maximum: fu and fv within their error of each other, unless float32 computes them identically
    a_du, a_dv = np.abs(q[:, 2:4]), np.abs(q[:, 4:6])
    same = (f32(sx) == f32(sy)) & (t.w[0] == t.h[0]) & (
        (a_du == a_dv).all(1) | ((a_du[:, ::-1] == a_dv).all(1) & (a_du.min(1) == 0)))
    p.u_is_max = ~(p.fv > p.fu)
    p.tie_amb = ~same & (np.abs(p.fu - p.fv) <= ARITH * p.max_fp) & (p.max_fp > 0)  # (two zero footprints are zero in float32 too)
    # level sides: (l0, nl) per side; ld follows from the float64 level
    lev = p.level
    nominal = np.where(lev <= 0, 0, np.where(lev >= L - 1, L - 1, np.floor(np.clip(lev, 0, L - 1)))).astype(np.int64)
    p.l0 = np.stack([nominal, nominal], 1)
    p.nl = np.stack([np.where((lev <= 0) | (lev >= L - 1), 1, 2)] * 2, 1)
    p.level_amb = np.zeros(n, bool)
    if L > 1:
        near0 = np.abs(lev) < p.dlevel
        near_top = np.abs(lev - (L - 1)) < p.dlevel
        k = np.round(lev)
        near_k = (np.abs(lev - k) < p.dlevel) & (k > 0) & (k < L - 1)
        # (side 0 is the float64 decision, side 1 the other one)
        below = (lev <= 0)[near0]
        p.l0[near0] = 0
        p.nl[near0] = np.stack([np.where(below, 1, 2), np.where(below, 2, 1)], 1)
        above = (lev >= L - 1)[near_top]
        p.l0[near_top] = np.stack([np.where(above, L - 1, L - 2), np.where(above, L - 2, L - 1)], 1)
        p.nl[near_top] = np.stack([np.where(above, 1, 2), np.where(above, 2, 1)], 1)
        kk = k[near_k].astype(np.int64)
        lo = (lev < k)[near_k]
        p.l0[near_k] = np.stack([np.where(lo, kk - 1, kk), np.where(lo, kk, kk - 1)], 1)
        p.nl[near_k] = [2, 2]
        p.level_amb = near0 | near_top | near_k
    # floor sides per level: [n, L, 2]
    def floor_sides(c, dc):
        # float32 may floor c anywhere in [c - dc, c + dc]: two candidates while dc < 0.5 (|x| < 2^22)
        assert (dc < 0.5).all(), "a coordinate beyond what float32 resolves to half a texel"
        lo, hi, fl = np.floor(c - dc), np.floor(c + dc), np.floor(c)
        return np.stack([fl, np.where(fl == lo, hi, lo)], 2).astype(np.int64), lo != hi  # (side 0: the float64 floor)
    p.xf, p.x_amb = floor_sides(p.x, p.dx)
    p.yf, p.y_amb = floor_sides(p.y, p.dy)
    # which levels a query may use
    used = np.zeros((n, L), bool)
    for s in range(2):
        for j in range(2):
            li = np.clip(p.l0[:, s] + j, 0, L - 1)
            ok = j < p.nl[:, s]
            used[np.arange(n)[ok], li[ok]] = True
    p.used = used
    p.depends = p.level_amb | p.tie_amb | ((p.x_amb | p.y_amb) & used).any(1)
    return p


class Answer:
    """One answer per row: `qid` the query, value [m, nch], d_q [m, 6] (d_u, d_v, d(du/dxy), d(dv/dxy)), their error bounds
    value_tol [m, nch], dq_tol [m, 6]; the uv_scale contributions uvs [m, triples, 2] and uvs_err; and the texel contributions
    (tap_qrow, tap_level, tap_index, tap_channel, tap_c, tap_err) where tap_qrow indexes the rows."""
    pass


def evaluate(t, q, d, p, rows, side):
    """The answer of queries `rows` of plan p with the decisions chosen by side [m, 6] bits: level side, x / y side at the first used
    level, x / y side at the second, branch of the maximum (flipped when 1 and the tie is ambiguous)."""
    q = np.asarray(q, dtype=np.float32).astype(np.float64)[rows]
    d = None if d is None else np.asarray(d, dtype=np.float32).astype(np.float64)[rows]
    m, nch = q.shape[0], t.nch
    a = Answer()
    a.qid = rows
    if t.constant:
        a.value = np.repeat(t.f64[0][None, 0, :nch], m, 0) if m else np.zeros((0, nch))
        a.value_tol = np.zeros((m, nch))
        a.d_q = np.zeros((m, 6))
        a.dq_tol = np.zeros((m, 6))
        ntr = (nch + 2) // 3
        a.uvs, a.uvs_err = np.zeros((m, ntr, 2)), np.zeros((m, ntr, 2))
        if d is None:
            d = np.zeros((m, nch))
        a.tap_qrow = np.repeat(np.arange(m), nch)
        a.tap_level = np.zeros(m * nch, np.int64)
        a.tap_index = np.zeros(m * nch, np.int64)
        a.tap_channel = np.tile(np.arange(nch), m)
        a.tap_c = d.reshape(-1)
        a.tap_err = np.zeros(m * nch)
        return a
    if d is None:
        d = np.zeros((m, nch))
    ar = np.arange(m)
    L, sx, sy, M = t.L, t.sx, t.sy, t.M
    ls = side[:, 0]
    l0, nl = p.l0[rows, ls], p.nl[rows, ls]
    lev = p.level[rows]
    ld = np.where(nl == 2, lev - l0, 0.0)
    u_is_max = p.u_is_max[rows] ^ (p.tie_amb[rows] & (side[:, 5] == 1))
    dlev = p.dlevel[rows]
    ntr = (nch + 2) // 3
    value = np.zeros((m, nch))
    value_tol = np.full((m, nch), ARITH * M)
    d_uv = np.zeros((m, ntr, 2))
    d_uv_err = np.zeros((m, ntr, 2))
    d_level = np.zeros((m, ntr))
    d_level_err = np.zeros((m, ntr))
    taps = []
    for j in range(2):
        act = j < nl
        li = np.clip(l0 + j, 0, L - 1)
        wl = np.where(nl == 2, np.where(j == 1, ld, 1 - ld), 1.0)
        xs, ys = side[:, 1 + 2 * j], side[:, 2 + 2 * j]
        xf = p.xf[rows, li, xs]
        yf = p.yf[rows, li, ys]
        x, y = p.x[rows, li], p.y[rows, li]
        # the error of the bilinear weights: that of x (y) plus the rounding of u = x - floor(x) itself (inexact for a small negative
        # x: then 1 - u loses digits by cancellation)
        dx, dy = p.dx[rows, li] + EPS, p.dy[rows, li] + EPS
        W = np.array(t.w)[li]
        H = np.array(t.h)[li]
        uu, vv = x - xf, y - yf
        val = np.zeros((m, ntr))
        d_u = np.zeros((m, ntr))
        d_v = np.zeros((m, ntr))
        for k in range(4):
            cx, cy = k & 1, (k >> 1) & 1
            xi = np.mod(xf + cx, W)
            yi = np.mod(yf + cy, H)
            idx = yi * W + xi
            wu = uu if cx else 1 - uu
            wv = vv if cy else 1 - vv
            texv = np.zeros((m, nch))
            for l in range(L):
                s = act & (li == l)
                if s.any():
                    texv[s] = t.f64[l][idx[s]]
            w = np.where(act, wl * wu * wv, 0.0)
            value += w[:, None] * texv
            for tr in range(ntr):
                cs = slice(3 * tr, min(3 * tr + 3, nch))
                tv = (d[:, cs] * texv[:, cs]).sum(1)
                val[:, tr] += tv * wu * wv
                d_u[:, tr] += (tv if cx else -tv) * wv
                d_v[:, tr] += (tv if cy else -tv) * wu
            # texel contributions d * wl * wu * wv: their own rounding (a few ulps) and their sensitivity to x, y and level
            err_w = wl * (np.abs(wv) * dx + np.abs(wu) * dy) + np.where(nl == 2, dlev, 0.0) * np.abs(wu * wv)
            for c in range(nch):
                c_val = d[:, c] * w
                c_err = np.abs(d[:, c]) * err_w + 4 * EPS * np.abs(c_val)
                taps.append((ar[act], li[act], idx[act], np.full(int(act.sum()), c), c_val[act], c_err[act]))
        for tr in range(ntr):
            cs = slice(3 * tr, min(3 * tr + 3, nch))
            D = np.abs(d[:, cs]).sum(1)
            aw = np.where(act, wl, 0.0)
            d_level[:, tr] += np.where(act & (nl == 2), np.where(j == 1, val[:, tr], -val[:, tr]), 0.0)
            # d_level: continuous in x and y (slope <= 2 D M each), arithmetic ARITH D M per level
            d_level_err[:, tr] += np.where(act & (nl == 2), 2 * D * M * (dx + dy) + ARITH * D * M, 0.0)
            d_uv[:, tr, 0] += aw * d_u[:, tr] * W
            d_uv[:, tr, 1] += aw * d_v[:, tr] * H
            # d_u is piecewise constant in x and linear in y (slope <= 4 D M); ld moves it by <= 2 D M per unit
            lev_term = np.where(act & (nl == 2), dlev * 2 * D * M, 0.0)
            d_uv_err[:, tr, 0] += np.where(act, W * (aw * (4 * D * M * dy + ARITH * D * M) + lev_term), 0.0)
            d_uv_err[:, tr, 1] += np.where(act, H * (aw * (4 * D * M * dx + ARITH * D * M) + lev_term), 0.0)
        vt = 2 * M * (dx + dy)
        value_tol += np.where(act, aw, 0.0)[:, None] * vt[:, None]
    value_tol += 2 * M * np.where(nl == 2, dlev, 0.0)[:, None]
    # d(level) -> d(footprint) -> d(du_dxy) or d(dv_dxy) (src/texture.h:394-408)
    du, dv = q[:, 2:4] * sx, q[:, 4:6] * sy
    max_fp = np.where(u_is_max, p.fu[rows], p.fv[rows])
    on = max_fp > F32_1E8
    g = np.zeros(m)
    g[on] = 1.0 / (max_fp[on] * LN2)
    vec = np.where(u_is_max[:, None], du, dv)
    nrm = np.sqrt((vec ** 2).sum(1))
    unit = np.zeros_like(vec)
    unit[on] = vec[on] / nrm[on, None]
    size0 = np.where(u_is_max, t.w[0], t.h[0])
    d_fp = d_level * (g * size0)[:, None]  # [m, ntr] d(footprint vector length) per unit
    d_fp_err = d_level_err * (g * size0)[:, None] + ARITH * np.abs(d_fp)
    d_du = np.where(u_is_max[:, None, None], d_fp[:, :, None] * unit[:, None, :], 0.0)
    d_dv = np.where(u_is_max[:, None, None], 0.0, d_fp[:, :, None] * unit[:, None, :])
    e_du = np.where(u_is_max[:, None, None], d_fp_err[:, :, None], 0.0) * np.ones((1, 1, 2))
    e_dv = np.where(u_is_max[:, None, None], 0.0, d_fp_err[:, :, None]) * np.ones((1, 1, 2))
    # to the caller's uv and footprint (uv = uv_ * uv_scale, du = du_ * sx, dv = dv_ * sy) and the uv_scale contribution
    s2 = np.array([sx, sy])
    a.d_q = np.concatenate([(d_uv * s2).sum(1), (d_du * sx).sum(1), (d_dv * sy).sum(1)], 1)
    a.dq_tol = np.concatenate([(d_uv_err * np.abs(s2)).sum(1), (e_du * abs(sx)).sum(1), (e_dv * abs(sy)).sum(1)], 1)
    a.dq_tol += ARITH * np.abs(a.d_q)
    uv_ = q[:, 0:2]
    a.uvs = np.stack([d_uv[:, :, 0] * uv_[:, None, 0] + (d_du * q[:, None, 2:4]).sum(2),
                      d_uv[:, :, 1] * uv_[:, None, 1] + (d_dv * q[:, None, 4:6]).sum(2)], 2)
    a.uvs_err = np.stack([d_uv_err[:, :, 0] * np.abs(uv_[:, None, 0]) + (e_du * np.abs(q[:, None, 2:4])).sum(2),
                          d_uv_err[:, :, 1] * np.abs(uv_[:, None, 1]) + (e_dv * np.abs(q[:, None, 4:6])).sum(2)], 2) + ARITH * np.abs(a.uvs)
    a.value = value
    a.value_tol = value_tol
    cat = lambda i: np.concatenate([tp[i] for tp in taps]) if taps else np.zeros(0)  # noqa: E731
    a.tap_qrow, a.tap_level, a.tap_index, a.tap_channel = (cat(i).astype(np.int64) for i in range(4))
    a.tap_c, a.tap_err = cat(4), cat(5)
    return a


def nominal(t, q, d, p, rows=None):
    """The answer with the float64 decisions (every side bit 0)."""
    rows = np.arange(p.n) if rows is None else np.asarray(rows)
    return evaluate(t, q, d, p, rows, np.zeros((len(rows), 6), np.int64))


def answers(t, q, d, p, rows):
    """Every one-sided answer of the queries `rows`: a list of Answers whose qid say which query each row is (a query appears once per
    combination of the sides of its ambiguous decisions)."""
    rows = np.asarray(rows)
    if t.constant or rows.size == 0:
        return [nominal(t, q, d, p, rows)]
    out = []
    for bits in itertools.product((0, 1), repeat=6):
        b = np.array(bits)
        ok = np.ones(rows.size, bool)
        if b[0]:
            ok &= p.level_amb[rows]
        if b[5]:
            ok &= p.tie_amb[rows]
        for j in range(2):
            li = np.clip(p.l0[rows, b[0]] + j, 0, t.L - 1)
            used = j < p.nl[rows, b[0]]
            if b[1 + 2 * j]:
                ok &= used & p.x_amb[rows, li]
            if b[2 + 2 * j]:
                ok &= used & p.y_amb[rows, li]
        if ok.any():
            r = rows[ok]
            out.append(evaluate(t, q, d, p, r, np.repeat(b[None], r.size, 0)))
    return out


def scatter(t, a, rows_of=None):
    """The gradient pyramid of the answer rows `rows_of` (all by default): per level the float64 sum, the sum of |contribution|, the sum
    of the contributions' error bounds and the number of contributions, [h * w (or 1), nch] each; and the uv_scale gradient (sum, sum
    of |c|, error, count) [2]."""
    sel = np.ones(a.tap_qrow.size, bool) if rows_of is None else np.isin(a.tap_qrow, rows_of)
    out = []
    for l in range(t.L):
        size = t.f64[l].shape[0]
        k = sel & (a.tap_level == l)
        flat = a.tap_index[k] * t.nch + a.tap_channel[k]  # (np.add.at over (texel, channel), by bincount)
        acc = lambda w: np.bincount(flat, weights=w, minlength=size * t.nch).reshape(size, t.nch)  # noqa: E731
        out.append((acc(a.tap_c[k]), acc(np.abs(a.tap_c[k])), acc(a.tap_err[k]), acc(np.ones(flat.size))))
    r = slice(None) if rows_of is None else rows_of
    u = a.uvs[r].reshape(-1, 2)
    ue = a.uvs_err[r].reshape(-1, 2)
    uvs = (u.sum(0), np.abs(u).sum(0), ue.sum(0), np.full(2, float(u.shape[0])))
    return out, uvs


def gamma(k):
    """The bound on the relative error of a float32 sum of k terms in any order, as a fraction of the sum of their magnitudes."""
    k = np.asarray(k, dtype=np.float64)
    return k * EPS / (1 - k * EPS)
