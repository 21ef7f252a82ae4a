"""Float64 restatement of emission sampling (DESIGN.md "Emission sampling"): the tables a light that samples by its emission texture
builds, and the probabilities and density its point sampler has.  The tables are restated with the library's additions in the library's
order, so they equal its doubles bit for bit; the probabilities of the sampler use exact polygon clipping.

Everything takes plain NumPy arrays: `tex` [h, w, c] float32 (level 0), `uv_scale` (sx, sy) float32, per triangle the uv corners `uv`
[T, 3, 2] float32 (the shape's uvs, or (0, 0), (1, 0), (1, 1) without) and the world corners `pos` [T, 3, 3] float32."""
import numpy as np

DELTA = 0.125
REC = 8  # doubles per triangle record


def luminance(tex):
    t = tex.astype(np.float64)
    if tex.shape[-1] == 1:
        return t[..., 0]
    c = np.float32([0.212671, 0.715160, 0.072169]).astype(np.float64)
    return (c[0] * t[..., 0] + c[1] * t[..., 1]) + c[2] * t[..., 2]


def cell_weights(tex):
    """w[j, i]: the mean |luminance| of the four wrapped taps (i, j), (i + 1, j), (i, j + 1), (i + 1, j + 1), summed in that order."""
    a = np.abs(luminance(tex))
    cf = np.roll(a, -1, axis=1)
    fc = np.roll(a, -1, axis=0)
    cc = np.roll(cf, -1, axis=0)
    return 0.25 * (((a + cf) + fc) + cc)


def sat(cells):
    """Row prefix sums left to right, then column sums top to bottom."""
    return np.cumsum(np.cumsum(cells, axis=1), axis=0)


def prefix(S, X, Y):
    """Mass of the cells [0, X) x [0, Y) of the periodic continuation (integers, negative ones included)."""
    h, w = S.shape
    qx, rx = X // w, X % w
    qy, ry = Y // h, Y % h

    def at(a, b):
        return S[b - 1, a - 1] if a > 0 and b > 0 else 0.0
    return float(qx) * float(qy) * at(w, h) + float(qx) * at(w, ry) + float(qy) * at(rx, h) + at(rx, ry)


def rect_mass(S, x0, y0, x1, y1):
    """Mass of [x0, x1) x [y0, y1), moved by whole periods so that (x0, y0) lies in the first period."""
    h, w = S.shape
    bx, by = (x0 // w) * w, (y0 // h) * h
    x0, x1, y0, y1 = x0 - bx, x1 - bx, y0 - by, y1 - by
    return (prefix(S, x1, y1) - prefix(S, x0, y1)) - (prefix(S, x1, y0) - prefix(S, x0, y0))


def corners(uv, uv_scale, w, h):
    """Cell coordinates X = u sx w - 0.5, Y = v sy h - 0.5 of [..., 2] uvs."""
    u, v = uv[..., 0].astype(np.float64), uv[..., 1].astype(np.float64)
    return u * float(uv_scale[0]) * w - 0.5, v * float(uv_scale[1]) * h - 0.5


def triangle_area(p):
    p = p.astype(np.float64)
    e1, e2 = p[1] - p[0], p[2] - p[0]
    cx, cy, cz = e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]
    return 0.5 * np.sqrt(cx * cx + cy * cy + cz * cz)


def tables(tex, uv_scale, uv, pos):
    """{S, cells, sat, recs [T, 8], area_t [T], T_cells [T]} of one light, as RB_TABLE_LIGHT_SAMPLING lays them out."""
    h, w = tex.shape[:2]
    cells = cell_weights(tex)
    S = sat(cells)
    recs = np.zeros((len(uv), REC))
    areas, tcell = np.zeros(len(uv)), np.zeros(len(uv))
    for t in range(len(uv)):
        X, Y = corners(uv[t], uv_scale, w, h)
        x0, y0 = int(np.floor(min(X[0], min(X[1], X[2])))), int(np.floor(min(Y[0], min(Y[1], Y[2]))))
        x1, y1 = int(np.floor(max(X[0], max(X[1], X[2])))) + 1, int(np.floor(max(Y[0], max(Y[1], Y[2])))) + 1
        M = rect_mass(S, x0, y0, x1, y1)
        M = M if M > 0 else 0.0
        T = 0.5 * abs((X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0]))
        a = triangle_area(pos[t])
        areas[t], tcell[t] = a, T
        recs[t, :5] = [x0, y0, x1, y1, M]
        if T > 0 and M > 0 and a > 0:
            recs[t, 5] = a * (M / (float(x1 - x0) * float(y1 - y0)))
            recs[t, 7] = T / (M * a)
    tot, run = 0.0, 0.0
    for t in range(len(uv)):
        tot += recs[t, 5]
    for t in range(len(uv)):
        recs[t, 6] = run / tot if tot > 0 else 0.0
        recs[t, 7] = (recs[t, 5] / tot) * recs[t, 7] if tot > 0 else 0.0
        run += recs[t, 5]
    return dict(S=tot, cells=cells, sat=S, recs=recs, areas=areas, tcell=tcell)


def light_weight(intensity, area):
    """lt_light_weight: the selection weight of a light of this intensity (float32) and (selection) area."""
    c = np.float32([0.212671, 0.715160, 0.072169]).astype(np.float64)
    i = np.asarray(intensity, np.float32).astype(np.float64)
    lum = (c[0] * i[0] + c[1] * i[1]) + c[2] * i[2]
    return area * lum * np.pi


def flat(tab):
    """The light's doubles in RB_TABLE_LIGHT_SAMPLING order."""
    return np.concatenate([[tab["S"], 0.0], tab["cells"].ravel(), tab["sat"].ravel(), tab["recs"].ravel()])


def density(tab, tex_shape, uv_scale, t, uv, light_area):
    """The mixture's area density at the point of triangle t with texture coordinate uv (before uv_scale)."""
    h, w = tex_shape[:2]
    r = tab["recs"][t]
    X, Y = corners(np.asarray(uv), uv_scale, w, h)
    ix = int(min(max(np.floor(X), r[0]), r[2] - 1))
    iy = int(min(max(np.floor(Y), r[1]), r[3] - 1))
    return DELTA / light_area + (1 - DELTA) * r[7] * tab["cells"][iy % h, ix % w]


def _clip(poly, axis, value, keep_below):
    out = []
    n = len(poly)
    for k in range(n):
        a, b = poly[k], poly[(k + 1) % n]
        ina = a[axis] <= value if keep_below else a[axis] >= value
        inb = b[axis] <= value if keep_below else b[axis] >= value
        if ina:
            out.append(a)
        if ina != inb:
            s = (value - a[axis]) / (b[axis] - a[axis])
            out.append((a[0] + s * (b[0] - a[0]), a[1] + s * (b[1] - a[1])))
    return out


def _area(poly):
    if len(poly) < 3:
        return 0.0
    x = np.array([p[0] for p in poly])
    y = np.array([p[1] for p in poly])
    return 0.5 * abs(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


def cell_overlaps(X, Y, rect):
    """{(i, j): area of cell [i, i+1) x [j, j+1) inside the triangle (X, Y)} over the integer rectangle `rect` (cell units)."""
    x0, y0, x1, y1 = (int(v) for v in rect)
    tri = list(zip(X, Y))
    out = {}
    for j in range(y0, y1):
        row = _clip(_clip(tri, 1, j, False), 1, j + 1, True)
        if len(row) < 3:
            continue
        for i in range(x0, x1):
            a = _area(_clip(_clip(row, 0, i, False), 0, i + 1, True))
            if a > 0:
                out[(i, j)] = a
    return out


def bin_probabilities(tab, tex_shape, uv_scale, uv, light_area):
    """({(t, i, j): probability that a sample lands in cell (i, j) of triangle t}, probability of a rejection)."""
    h, w = tex_shape[:2]
    recs, areas = tab["recs"], tab["areas"]
    S = tab["S"]
    probs, rejected = {}, 0.0
    for t in range(len(uv)):
        X, Y = corners(uv[t], uv_scale, w, h)
        ov = cell_overlaps(X, Y, recs[t, :4])
        T = tab["tcell"][t]
        P = recs[t, 5] / S if S > 0 else 0.0
        inside = 0.0
        for (i, j), a in ov.items():
            p = DELTA * areas[t] / light_area * (a / T) if T > 0 else 0.0
            if P > 0:
                q = P * tab["cells"][j % h, i % w] / recs[t, 4] * a
                inside += q
                p += (1 - DELTA) * q
            probs[(t, i, j)] = probs.get((t, i, j), 0.0) + p
        rejected += (1 - DELTA) * (P - inside)
    return probs, rejected


# ---------------------------------------------------------------------------------------------------- the MIS scene's quadrature
KD = 0.7
INTENSITY = np.array([3.0, 2.0, 1.5])
LIGHT = dict(x0=1.4, x1=2.4, y0=-0.5, y1=0.5, z=1.0)


def bilinear(tex, uv):
    """E(uv) at level 0 (uv already scaled, wrapping), as the renderer's zero-footprint lookup."""
    h, w, _ = tex.shape
    x, y = uv[..., 0] * w - 0.5, uv[..., 1] * h - 0.5
    xf, yf = np.floor(x).astype(int), np.floor(y).astype(int)
    fx, fy = (x - xf)[..., None], (y - yf)[..., None]
    ff, cf, fc, cc = tex[yf % h, xf % w], tex[yf % h, (xf + 1) % w], tex[(yf + 1) % h, xf % w], tex[(yf + 1) % h, (xf + 1) % w]
    return ff * (1 - fx) * (1 - fy) + cf * fx * (1 - fy) + fc * (1 - fx) * fy + cc * fx * fy


def light_grid(tex, n=256):
    """(E [n, n, 3], light points x [n, n], y [n, n], dA) of the midpoint rule over the unit-square uvs of the light LIGHT."""
    L = LIGHT
    s = (np.arange(n) + 0.5) / n
    u, v = np.meshgrid(s, s, indexing="xy")
    E = bilinear(tex, np.stack([u, v], -1))
    if E.shape[-1] == 1:
        E = np.repeat(E, 3, -1)
    xs = L["x0"] + u * (L["x1"] - L["x0"])
    ys = L["y0"] + v * (L["y1"] - L["y0"])
    return E, xs, ys, (L["x1"] - L["x0"]) * (L["y1"] - L["y0"]) / (n * n)


def quadrature(points, tex, n=256):
    """kd / pi * integral of I E(uv) cos cos' / r^2 dA' over the light, per floor point (float64, midpoint rule)."""
    E, xs, ys, dA = light_grid(tex, n)
    out = np.zeros(points.shape[:-1] + (3,))
    for idx in np.ndindex(points.shape[:-1]):
        p = points[idx]
        d = np.stack([xs - p[0], ys - p[1], np.full_like(xs, LIGHT["z"] - p[2])], -1)
        r2 = (d * d).sum(-1)
        cos_f = d[..., 2] / np.sqrt(r2)  # at the floor (normal +z) and at the light (normal -z): the same
        out[idx] = KD / np.pi * INTENSITY * (E * (cos_f * cos_f / r2)[..., None]).sum((0, 1)) * dA
    return out


def mis_variance(points, tex, density, n=128):
    """Sum over the floor points and channels of the variance of ONE sample of the renderer's estimate of the quadrature's integral with
    max_bounces 1: a light sample of area density `density` [n, n] over the light's uv grid (0 where it never lands) and a cosine BSDF
    sample, weighed by the power heuristic; a rejected light sample contributes 0.  Both estimators are integrated over the light in
    float64: Var = sum over k of (integral (w_k f / p_k)^2 p_k dA - (integral w_k f dA)^2)."""
    E, xs, ys, dA = light_grid(tex, n)
    tot = 0.0
    for idx in np.ndindex(points.shape[:-1]):
        p = points[idx]
        d = np.stack([xs - p[0], ys - p[1], np.full_like(xs, LIGHT["z"] - p[2])], -1)
        r2 = (d * d).sum(-1)
        cos_f = d[..., 2] / np.sqrt(r2)
        f = KD / np.pi * INTENSITY * E * (cos_f * cos_f / r2)[..., None]
        p_b = cos_f * cos_f / (np.pi * r2)  # (cosine sampling at the floor, as an area density on the light)
        p_l = density
        for pk in (p_l, p_b):
            w = pk * pk / (p_l * p_l + p_b * p_b)
            on = pk > 0
            second = ((w[on, None] * f[on]) ** 2 / pk[on, None] * dA).sum(0)
            first = (w[..., None] * f * dA).sum((0, 1))
            tot += float((second - first ** 2).sum())
    return tot
