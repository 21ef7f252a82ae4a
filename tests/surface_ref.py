"""Float64 restatement of the geometry functions of rb_shape.cuh: tri_solve, make_surface_point, sample_light_triangle, light_sample_uv
and shape_tri_area, the adjoint d_make_surface_point as written, and central differences for the true derivatives.

d_make_surface_point follows the reference statement by statement (src/shape.h:384-747) and so reproduces its slips.  Each is a named,
separate term that `point_adjoint(..., slips=...)` can leave out; without them the restatement is the true adjoint:
- S1  with vertex normals, d_coordinate_system(sn, d_frame.x, d_frame.y) is added to d_sn on top of the frame adjoint (src/shape.h:573);
- S2  without vertex normals, the frame adjoint's d_sn is dropped: d_frame.n goes to d_gn, and the frame seeds go through
      d_coordinate_system(sn) whichever way the frame was built (src/shape.h:635-637);
- S3  on the non-degenerate fy branch, d_point.dpdu is overwritten by d_normalize(dpdu, d_fx_org) instead of added to (src/shape.h:546);
- S4  d_l2 and d_denom of the dn_dx / dn_dy adjoint are vectors, never summed (src/shape.h:595-610);
- S5  on the det == 0 branch, coordinate_system is differentiated at the flipped geometric normal (src/shape.h:660);
- S6  the uv02.y * v12 term of dpdu is differentiated with a + sign, into d_uv02.y and into d_v12 (src/shape.h:670-671);
- S7  the - dot(nn, dnn) nn term of dn_dx / dn_dy is differentiated with a + sign, into d_nn and through d(dot) (src/shape.h:598-600).

Queries are vectorised: every argument is an [n, k] array.  A triangle block `T` is a dict with the float32 corner values the kernel reads
(v0, v1, v2; uv0, uv1, uv2, the default (0,0), (1,0), (1,1) without uvs; n0, n1, n2 or None; c0, c1, c2 or None)."""
import numpy as np

CS_EPS = -1.0 + 1e-6
SLIPS = ("S1", "S2", "S3", "S4", "S5", "S6", "S7")


def dot(a, b):
    return (a * b).sum(-1)


def cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def length(a):
    return np.sqrt(dot(a, a))


def normalize(v):
    l = length(v)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(l > 0, v / np.where(l > 0, l, 1), 0.0)


def d_normalize(v, d_n):
    l = length(v)[:, None]
    ls = np.where(l > 0, l, 1)
    n = v / ls
    return np.where(l > 0, d_n / ls - dot(d_n, n)[:, None] * n / ls, 0.0)


def d_cross(a, b, d_out):
    return cross(b, d_out), cross(d_out, a)


def coordinate_system(n):
    low = n[:, 2] < CS_EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        a = 1 / (1 + n[:, 2])
    a = np.where(low, 0.0, a)
    b = -n[:, 0] * n[:, 1] * a
    x = np.stack([1 - n[:, 0] ** 2 * a, b, -n[:, 0]], 1)
    y = np.stack([b, 1 - n[:, 1] ** 2 * a, -n[:, 1]], 1)
    x[low] = [0.0, -1.0, 0.0]
    y[low] = [-1.0, 0.0, 0.0]
    return x, y


def d_coordinate_system(n, d_x, d_y):
    """The gradient d_coordinate_system adds to d_n (zero on the n.z < -1 + 1e-6 branch)."""
    low = n[:, 2] < CS_EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(low, 0.0, 1 / (1 + n[:, 2]))
    nx, ny = n[:, 0], n[:, 1]
    d_a = -nx ** 2 * d_x[:, 0] - d_y[:, 1] * ny ** 2
    d_b = d_x[:, 1] + d_y[:, 0]
    d_a = d_a - d_b * nx * ny
    gx = -2 * nx * d_x[:, 0] * a - d_x[:, 2] - d_b * ny * a
    gy = -2 * d_y[:, 1] * ny * a - d_y[:, 2] - d_b * nx * a
    with np.errstate(divide="ignore", invalid="ignore"):
        gz = np.where(low, 0.0, -d_a * a / np.where(low, 1.0, 1 + n[:, 2]))
    return np.where(low[:, None], 0.0, np.stack([gx, gy, gz], 1))


# ---------------------------------------------------------------------------------------------------- inputs as one flat vector
# A query's differentiable inputs, in this order: v0, v1, v2 (9), uv0, uv1, uv2 (6), n0, n1, n2 (9), c0, c1, c2 (9), org, dir (6),
# org_dx, org_dy, dir_dx, dir_dy (12): 51 numbers.
NX = 51


def pack(T, org, dir_, rd):
    n = len(org)
    z3 = np.zeros((n, 3))
    parts = [T["v0"], T["v1"], T["v2"], T["uv0"], T["uv1"], T["uv2"]]
    parts += [T[k] if T.get("n0") is not None else z3 for k in ("n0", "n1", "n2")]
    parts += [T[k] if T.get("c0") is not None else z3 for k in ("c0", "c1", "c2")]
    return np.concatenate(parts + [org, dir_, rd], 1).astype(np.float64)


def unpack(X, has_n, has_c):
    sl = lambda a, b: X[:, a:b]  # noqa: E731
    T = dict(v0=sl(0, 3), v1=sl(3, 6), v2=sl(6, 9), uv0=sl(9, 11), uv1=sl(11, 13), uv2=sl(13, 15),
             n0=sl(15, 18) if has_n else None, n1=sl(18, 21) if has_n else None, n2=sl(21, 24) if has_n else None,
             c0=sl(24, 27) if has_c else None, c1=sl(27, 30) if has_c else None, c2=sl(30, 33) if has_c else None)
    return T, sl(33, 36), sl(36, 39), sl(39, 51)


# ---------------------------------------------------------------------------------------------------- forward
def tri_terms(v0, v1, v2, org, dir_, rd):
    odx, ody, ddx, ddy = rd[:, 0:3], rd[:, 3:6], rd[:, 6:9], rd[:, 9:12]
    k = {}
    e1, e2 = v1 - v0, v2 - v0
    pvec, pdx, pdy = cross(dir_, e2), cross(ddx, e2), cross(ddy, e2)
    div = dot(pvec, e1)
    k["clamped"] = np.abs(div) < 1e-8
    div = np.where(k["clamped"], np.where(div > 0, 1e-8, -1e-8), div)
    s = org - v0
    qvec, qdx, qdy = cross(s, e1), cross(odx, e1), cross(ody, e1)
    k.update(e1=e1, e2=e2, pvec=pvec, pdx=pdx, pdy=pdy, s=s, qvec=qvec, qdx=qdx, qdy=qdy, div=div, div_dx=dot(pdx, e1), div_dy=dot(pdy, e1))
    k["nu"], k["nu_dx"], k["nu_dy"] = dot(s, pvec), dot(odx, pvec) + dot(s, pdx), dot(ody, pvec) + dot(s, pdy)
    k["nv"], k["nv_dx"], k["nv_dy"] = dot(dir_, qvec), dot(ddx, qvec) + dot(dir_, qdx), dot(ddy, qvec) + dot(dir_, qdy)
    k["nt"], k["nt_dx"], k["nt_dy"] = dot(e2, qvec), dot(e2, qdx), dot(e2, qdy)
    return k


def tri_solve(v0, v1, v2, org, dir_, rd):
    """[n, 9]: u, v, t, u_dxy, v_dxy, t_dxy."""
    k = tri_terms(v0, v1, v2, org, dir_, rd)
    dv = k["div"]
    q = lambda n, n_d, dv_d: (n_d * dv - n * dv_d) / dv ** 2  # noqa: E731
    cols = [k["nu"] / dv, k["nv"] / dv, k["nt"] / dv]
    for nm in ("nu", "nv", "nt"):
        cols += [q(k[nm], k[nm + "_dx"], k["div_dx"]), q(k[nm], k[nm + "_dy"], k["div_dy"])]
    return np.stack(cols, 1)


def uv_det(T):
    uv02, uv12 = T["uv0"] - T["uv2"], T["uv1"] - T["uv2"]
    return uv02[:, 0] * uv12[:, 1] - uv02[:, 1] * uv12[:, 0]


def point(X, has_n, has_c):
    """make_surface_point at the flat inputs X.  Returns (out [n, 56] in the hook's layout: tri_solve 0-8, SurfacePoint 9-43, rd_out
    44-55; dict: det, the decision operands flip (dot(gn, sn)), fy (|cross(sn, fx)|), cs_gn (gn.z - (-1 + 1e-6)), cs_sn, whether tri_solve
    clamped its divisor, and dn_scale, |dnn_dx| / |nn| and |dnn_dy| / |nn|, the size of the terms dn_dx and dn_dy cancel)."""
    T, org, dir_, rd = unpack(X, has_n, has_c)
    v0, v1, v2 = T["v0"], T["v1"], T["v2"]
    h = tri_solve(v0, v1, v2, org, dir_, rd)
    u, v, t = h[:, 0:1], h[:, 1:2], h[:, 2:3]
    w = 1 - (u + v)
    u_dxy, v_dxy, t_dxy = h[:, 3:5], h[:, 5:7], h[:, 7:9]
    uv = w * T["uv0"] + u * T["uv1"] + v * T["uv2"]
    pos = org + dir_ * t
    gn = normalize(cross(v1 - v0, v2 - v0))
    gn0 = gn
    uv02, uv12 = T["uv0"] - T["uv2"], T["uv1"] - T["uv2"]
    det = uv_det(T)
    zero = det == 0
    inv = 1 / np.where(zero, 1.0, det)
    dpdu = (uv12[:, 1:2] * (v0 - v2) - uv02[:, 1:2] * (v1 - v2)) * inv[:, None]
    dpdu = np.where(zero[:, None], coordinate_system(gn)[0], dpdu)
    neg = -u_dxy - v_dxy
    du_dxy = neg * T["uv0"][:, 0:1] + u_dxy * T["uv1"][:, 0:1] + v_dxy * T["uv2"][:, 0:1]
    dv_dxy = neg * T["uv0"][:, 1:2] + u_dxy * T["uv1"][:, 1:2] + v_dxy * T["uv2"][:, 1:2]
    odx, ody, ddx, ddy = rd[:, 0:3], rd[:, 3:6], rd[:, 6:9], rd[:, 9:12]
    dpdx = odx + dir_ * t_dxy[:, 0:1] + ddx * t
    dpdy = ody + dir_ * t_dxy[:, 1:2] + ddy * t
    sn = gn
    n = len(X)
    dn_dx = dn_dy = np.zeros((n, 3))
    flip = np.ones(n)
    if has_n:
        n0, n1, n2 = T["n0"], T["n1"], T["n2"]
        nn = w * n0 + u * n1 + v * n2
        dnn_dx = neg[:, 0:1] * n0 + u_dxy[:, 0:1] * n1 + v_dxy[:, 0:1] * n2
        dnn_dy = neg[:, 1:2] * n0 + u_dxy[:, 1:2] * n1 + v_dxy[:, 1:2] * n2
        l2 = dot(nn, nn)[:, None]
        den = l2 * np.sqrt(l2)
        ok = den > 0
        with np.errstate(invalid="ignore", divide="ignore"):
            dn_dx = np.where(ok, (l2 * dnn_dx - dot(nn, dnn_dx)[:, None] * nn) / np.where(ok, den, 1), 0.0)
            dn_dy = np.where(ok, (l2 * dnn_dy - dot(nn, dnn_dy)[:, None] * nn) / np.where(ok, den, 1), 0.0)
        sn = normalize(nn)
        flip = dot(gn, sn)
        gn = np.where((flip < 0)[:, None], -gn, gn)
    fx = normalize(dpdu)
    fy = cross(sn, fx)
    fy_len = length(fy)
    good = (fy_len ** 2 > 0)[:, None]
    fyn = normalize(fy)
    csx, csy = coordinate_system(sn)
    fx = np.where(good, cross(fyn, sn), csx)
    fy = np.where(good, fyn, csy)
    col = np.zeros((n, 3))
    if has_c:
        col = w * T["c0"] + u * T["c1"] + v * T["c2"]
    sp = np.concatenate([pos, gn, fx, fy, sn, dpdu, uv, du_dxy, dv_dxy, dn_dx, dn_dy, col, np.concatenate([u, v], 1)], 1)
    out = np.concatenate([h, sp, dpdx, dpdy, ddx, ddy], 1)
    dn_scale = np.zeros((n, 2))
    if has_n:
        with np.errstate(invalid="ignore", divide="ignore"):
            dn_scale = np.stack([length(dnn_dx), length(dnn_dy)], 1) / np.where(ok, np.sqrt(l2), np.inf)
    kk = tri_terms(v0, v1, v2, org, dir_, rd)
    dec = dict(div_cond=length(kk["pvec"]) * length(kk["e1"]) / np.abs(kk["div"]), dn_scale=dn_scale, det=det, flip=flip, fy=fy_len, cs_gn=gn0[:, 2] - CS_EPS, cs_sn=sn[:, 2] - CS_EPS, clamped=tri_terms(v0, v1, v2, org, dir_, rd)["clamped"])
    return out, dec


def decisions(dec, has_n):
    """The branches the restatement takes, in the hook's order: det == 0, flipped, fy degenerate, cs branch at gn, cs branch at sn."""
    return np.stack([dec["det"] == 0, (dec["flip"] < 0) & has_n, ~(dec["fy"] ** 2 > 0), dec["cs_gn"] < 0, dec["cs_sn"] < 0], 1).astype(float)


# ---------------------------------------------------------------------------------------------------- d_make_surface_point as written
def d_tri_solve(k, dir_, rd, d_h):
    """The adjoint of tri_solve for the seeds d_h [n, 9] (u, v, t, u_dxy, v_dxy, t_dxy), the divisor clamp ignored as in the kernel:
    returns d_v0, d_v1, d_v2, d_org, d_dir, d_rd."""
    odx, ody, ddx, ddy = rd[:, 0:3], rd[:, 3:6], rd[:, 6:9], rd[:, 9:12]
    dv, dvx, dvy = k["div"], k["div_dx"], k["div_dy"]
    d_div, d_div_dx, d_div_dy = np.zeros(len(dv)), np.zeros(len(dv)), np.zeros(len(dv))
    res = {}
    for j, nm in enumerate(("nu", "nv", "nt")):
        n_, nx, ny = k[nm], k[nm + "_dx"], k[nm + "_dy"]
        dq, dqx, dqy = d_h[:, j], d_h[:, 3 + 2 * j], d_h[:, 4 + 2 * j]
        res[nm] = (dq / dv - dqx * dvx / dv ** 2 - dqy * dvy / dv ** 2, dqx / dv, dqy / dv)
        d_div += -dq * n_ / dv ** 2 - dqx * (nx / dv ** 2 - 2 * n_ * dvx / dv ** 3) - dqy * (ny / dv ** 2 - 2 * n_ * dvy / dv ** 3)
        d_div_dx += -dqx * n_ / dv ** 2
        d_div_dy += -dqy * n_ / dv ** 2
    c = lambda a: a[:, None]  # noqa: E731
    (d_nu, d_nux, d_nuy), (d_nv, d_nvx, d_nvy), (d_nt, d_ntx, d_nty) = res["nu"], res["nv"], res["nt"]
    e1, e2 = k["e1"], k["e2"]
    d_e2 = c(d_nt) * k["qvec"] + c(d_ntx) * k["qdx"] + c(d_nty) * k["qdy"]
    d_q, d_qx, d_qy = c(d_nt) * e2, c(d_ntx) * e2, c(d_nty) * e2
    d_dir = c(d_nv) * k["qvec"] + c(d_nvx) * k["qdx"] + c(d_nvy) * k["qdy"]
    d_q = d_q + c(d_nv) * dir_ + c(d_nvx) * ddx + c(d_nvy) * ddy
    d_ddx, d_ddy = c(d_nvx) * k["qvec"], c(d_nvy) * k["qvec"]
    d_qx, d_qy = d_qx + c(d_nvx) * dir_, d_qy + c(d_nvy) * dir_
    d_odx, d_e1 = d_cross(odx, e1, d_qx)
    a, b = d_cross(ody, e1, d_qy)
    d_ody, d_e1 = a, d_e1 + b
    d_s, b = d_cross(k["s"], e1, d_q)
    d_e1 = d_e1 + b
    d_s = d_s + c(d_nu) * k["pvec"] + c(d_nux) * k["pdx"] + c(d_nuy) * k["pdy"]
    d_p = c(d_nu) * k["s"] + c(d_nux) * odx + c(d_nuy) * ody
    d_odx, d_ody = d_odx + c(d_nux) * k["pvec"], d_ody + c(d_nuy) * k["pvec"]
    d_px, d_py = c(d_nux) * k["s"] + c(d_div_dx) * e1, c(d_nuy) * k["s"] + c(d_div_dy) * e1
    d_p = d_p + c(d_div) * e1
    d_e1 = d_e1 + c(d_div_dx) * k["pdx"] + c(d_div_dy) * k["pdy"] + c(d_div) * k["pvec"]
    a, b = d_cross(ddx, e2, d_px)
    d_ddx, d_e2 = d_ddx + a, d_e2 + b
    a, b = d_cross(ddy, e2, d_py)
    d_ddy, d_e2 = d_ddy + a, d_e2 + b
    a, b = d_cross(dir_, e2, d_p)
    d_dir, d_e2 = d_dir + a, d_e2 + b
    return -d_s - d_e1 - d_e2, d_e1, d_e2, d_s, d_dir, np.concatenate([d_odx, d_ody, d_ddx, d_ddy], 1)


def point_adjoint(X, has_n, has_c, seed, slips=SLIPS):
    """d_make_surface_point at the flat inputs X for seeds [n, 47] (d SurfacePoint 35, d rd_out 12), as written with the named `slips`
    (all of them by default, none for the true adjoint).  Returns the gradient of the 51 flat inputs."""
    T, org, dir_, rd = unpack(X, has_n, has_c)
    n = len(X)
    c = lambda a: a[:, None]  # noqa: E731
    v0, v1, v2 = T["v0"], T["v1"], T["v2"]
    k = tri_terms(v0, v1, v2, org, dir_, rd)
    h = tri_solve(v0, v1, v2, org, dir_, rd)
    u, v, t = h[:, 0], h[:, 1], h[:, 2]
    w = 1 - (u + v)
    u_dxy, v_dxy, t_dxy = h[:, 3:5], h[:, 5:7], h[:, 7:9]
    ugn = cross(v1 - v0, v2 - v0)
    gn = normalize(ugn)
    gn0 = gn
    uv02, uv12 = T["uv0"] - T["uv2"], T["uv1"] - T["uv2"]
    det = uv_det(T)
    zero = det == 0
    inv = 1 / np.where(zero, 1.0, det)
    dpdu = np.where(c(zero), coordinate_system(gn)[0], (uv12[:, 1:2] * (v0 - v2) - uv02[:, 1:2] * (v1 - v2)) * c(inv))
    neg = -u_dxy - v_dxy
    sn = gn
    flipped = np.zeros(n, bool)
    if has_n:
        n0, n1, n2 = T["n0"], T["n1"], T["n2"]
        nn = c(w) * n0 + c(u) * n1 + c(v) * n2
        dnn_dx = neg[:, 0:1] * n0 + u_dxy[:, 0:1] * n1 + v_dxy[:, 0:1] * n2
        dnn_dy = neg[:, 1:2] * n0 + u_dxy[:, 1:2] * n1 + v_dxy[:, 1:2] * n2
        l2 = dot(nn, nn)
        sn = normalize(nn)
        flipped = dot(gn, sn) < 0
        gn = np.where(c(flipped), -gn, gn)
    fx_org = normalize(dpdu)
    fy_org = cross(sn, fx_org)
    fy_ok = dot(fy_org, fy_org) > 0
    fy = normalize(fy_org)
    S = seed
    d_pos, d_gn_s, d_fx, d_fy, d_fn, d_dpdu_s = (S[:, 3 * j:3 * j + 3] for j in range(6))
    d_uv, d_du, d_dv = S[:, 18:20], S[:, 20:22], S[:, 22:24]
    d_dndx, d_dndy, d_col, d_bary = S[:, 24:27], S[:, 27:30], S[:, 30:33], S[:, 33:35]
    d_rdo = S[:, 35:47]
    d_u, d_v, d_w = d_bary[:, 0].copy(), d_bary[:, 1].copy(), np.zeros(n)
    G = np.zeros((n, NX))
    if has_c:
        G[:, 24:27], G[:, 27:30], G[:, 30:33] = d_col * c(w), d_col * c(u), d_col * c(v)
        d_w += dot(d_col, T["c0"])
        d_u += dot(d_col, T["c1"])
        d_v += dot(d_col, T["c2"])
    # the shading frame
    a, b = d_cross(fy, sn, d_fx)
    d_fy_t, d_sn_t = d_fy + a, d_fn + b
    d_fy_org = d_normalize(fy_org, d_fy_t)
    a, d_fx_org = d_cross(sn, fx_org, d_fy_org)
    d_sn_t = d_sn_t + a
    d_dpdu = np.where(c(fy_ok), d_normalize(dpdu, d_fx_org) + (0 if "S3" in slips else d_dpdu_s), d_dpdu_s)
    d_sn = np.where(c(fy_ok), d_sn_t, d_fn + d_coordinate_system(sn, d_fx, d_fy))
    d_gn = d_gn_s.copy()
    d_rd = np.zeros((n, 12))
    d_rd[:, 6:12] += d_rdo[:, 6:12]
    d_u_dxy, d_v_dxy = np.zeros((n, 2)), np.zeros((n, 2))
    d_v0, d_v1, d_v2 = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3))
    if has_n:
        d_gn = np.where(c(flipped), -d_gn, d_gn)
        if "S1" in slips:
            d_sn = d_sn + d_coordinate_system(sn, d_fx, d_fy)
        live = l2 > 0
        ls = np.where(live, np.sqrt(l2), 1.0)
        den = ls ** 3
        d_nn = d_normalize(nn, d_sn)
        dn_dx = (c(ls ** 2) * dnn_dx - c(dot(nn, dnn_dx)) * nn) / c(den)
        dn_dy = (c(ls ** 2) * dnn_dy - c(dot(nn, dnn_dy)) * nn) / c(den)
        d_l2 = (d_dndx * dnn_dx + d_dndy * dnn_dy) / c(den)
        d_dnn_dx = d_dndx * c(ls ** 2 / den)
        d_dnn_dy = d_dndy * c(ls ** 2 / den)
        s7 = 1.0 if "S7" in slips else -1.0
        d_dot_x = s7 * dot(d_dndx, nn) / den
        d_dot_y = s7 * dot(d_dndy, nn) / den
        d_nn = d_nn + s7 * (d_dndx * c(dot(nn, dnn_dx)) + d_dndy * c(dot(nn, dnn_dy))) / c(den)
        d_den = (d_dndx * -dn_dx + d_dndy * -dn_dy) / c(den)
        d_nn = d_nn + c(d_dot_x) * dnn_dx + c(d_dot_y) * dnn_dy
        d_dnn_dx = d_dnn_dx + c(d_dot_x) * nn
        d_dnn_dy = d_dnn_dy + c(d_dot_y) * nn
        if "S4" in slips:
            d_l2 = d_l2 + d_den * c(ls * 1.5)
            d_nn = d_nn + 2 * (d_l2 * nn)
        else:
            d_nn = d_nn + 2 * c(d_l2.sum(1) + d_den.sum(1) * ls * 1.5) * nn
        d_u_dxy = d_u_dxy + np.stack([dot(d_dnn_dx, n1 - n0), dot(d_dnn_dy, n1 - n0)], 1)
        d_v_dxy = d_v_dxy + np.stack([dot(d_dnn_dx, n2 - n0), dot(d_dnn_dy, n2 - n0)], 1)
        d_n0 = d_dnn_dx * neg[:, 0:1] + d_dnn_dy * neg[:, 1:2] + d_nn * c(w)
        d_n1 = d_dnn_dx * u_dxy[:, 0:1] + d_dnn_dy * u_dxy[:, 1:2] + d_nn * c(u)
        d_n2 = d_dnn_dx * v_dxy[:, 0:1] + d_dnn_dy * v_dxy[:, 1:2] + d_nn * c(v)
        lv = c(live)
        G[:, 15:18], G[:, 18:21], G[:, 21:24] = np.where(lv, d_n0, 0), np.where(lv, d_n1, 0), np.where(lv, d_n2, 0)
        d_w += np.where(live, dot(d_nn, n0), 0)
        d_u += np.where(live, dot(d_nn, n1), 0)
        d_v += np.where(live, dot(d_nn, n2), 0)
        d_u_dxy, d_v_dxy = np.where(lv, d_u_dxy, 0), np.where(lv, d_v_dxy, 0)
    elif "S2" in slips:
        d_gn = d_gn + d_fn + d_coordinate_system(sn, d_fx, d_fy)
    else:
        d_gn = d_gn + d_sn
    # dpdx, dpdy
    ddx, ddy = rd[:, 6:9], rd[:, 9:12]
    d_dpdx, d_dpdy = d_rdo[:, 0:3], d_rdo[:, 3:6]
    d_rd[:, 0:3] += d_dpdx
    d_rd[:, 3:6] += d_dpdy
    d_dir = d_dpdx * t_dxy[:, 0:1] + d_dpdy * t_dxy[:, 1:2]
    d_t_dxy = np.stack([dot(d_dpdx, dir_), dot(d_dpdy, dir_)], 1)
    d_rd[:, 6:9] += d_dpdx * c(t)
    d_rd[:, 9:12] += d_dpdy * c(t)
    d_t = dot(d_dpdx, ddx) + dot(d_dpdy, ddy)
    # dpdu
    d_uv0, d_uv1, d_uv2 = np.zeros((n, 2)), np.zeros((n, 2)), np.zeros((n, 2))
    d_gn = d_gn + np.where(c(zero), d_coordinate_system(gn if "S5" in slips else gn0, d_dpdu, np.zeros((n, 3))), 0)
    nz = c(~zero)
    v02, v12 = v0 - v2, v1 - v2
    sg = 1.0 if "S6" in slips else -1.0
    d_uv12y = dot(d_dpdu, v02) * inv
    d_v02 = d_dpdu * uv12[:, 1:2] * c(inv)
    d_uv02y = sg * dot(d_dpdu, v12) * inv
    d_v12 = sg * d_dpdu * uv02[:, 1:2] * c(inv)
    d_det = -dot(d_dpdu, uv12[:, 1:2] * v02 - uv02[:, 1:2] * v12) * inv * inv
    d_uv02 = np.stack([d_det * uv12[:, 1], d_uv02y - d_det * uv12[:, 0]], 1)
    d_uv12 = np.stack([-d_det * uv02[:, 1], d_uv12y + d_det * uv02[:, 0]], 1)
    d_uv0 += np.where(nz, d_uv02, 0)
    d_uv1 += np.where(nz, d_uv12, 0)
    d_uv2 -= np.where(nz, d_uv02 + d_uv12, 0)
    d_v0 += np.where(nz, d_v02, 0)
    d_v1 += np.where(nz, d_v12, 0)
    d_v2 -= np.where(nz, d_v02 + d_v12, 0)
    d_u_dxy = d_u_dxy + d_du * c(T["uv1"][:, 0] - T["uv0"][:, 0]) + d_dv * c(T["uv1"][:, 1] - T["uv0"][:, 1])
    d_v_dxy = d_v_dxy + d_du * c(T["uv2"][:, 0] - T["uv0"][:, 0]) + d_dv * c(T["uv2"][:, 1] - T["uv0"][:, 1])
    d_uv0 += np.stack([dot(d_du, neg), dot(d_dv, neg)], 1)
    d_uv1 += np.stack([dot(d_du, u_dxy), dot(d_dv, u_dxy)], 1)
    d_uv2 += np.stack([dot(d_du, v_dxy), dot(d_dv, v_dxy)], 1)
    # geometric normal
    d_e1, d_e2 = d_cross(v1 - v0, v2 - v0, d_normalize(ugn, d_gn))
    d_v0 += -d_e1 - d_e2
    d_v1 += d_e1
    d_v2 += d_e2
    # hit position, uv
    d_org = d_pos.copy()
    d_dir = d_dir + d_pos * c(t)
    d_t = d_t + dot(d_pos, dir_)
    d_w += dot(d_uv, T["uv0"])
    d_u += dot(d_uv, T["uv1"])
    d_v += dot(d_uv, T["uv2"])
    d_uv0 += d_uv * c(w)
    d_uv1 += d_uv * c(u)
    d_uv2 += d_uv * c(v)
    d_u, d_v = d_u - d_w, d_v - d_w
    d_h = np.concatenate([c(d_u), c(d_v), c(d_t), d_u_dxy, d_v_dxy, d_t_dxy], 1)
    a0, a1, a2, a_org, a_dir, a_rd = d_tri_solve(k, dir_, rd, d_h)
    G[:, 0:3], G[:, 3:6], G[:, 6:9] = d_v0 + a0, d_v1 + a1, d_v2 + a2
    G[:, 9:11], G[:, 11:13], G[:, 13:15] = d_uv0, d_uv1, d_uv2
    G[:, 33:36] = d_org + a_org
    G[:, 36:39] = d_dir + a_dir
    G[:, 39:51] = d_rd + a_rd
    return G


# ---------------------------------------------------------------------------------------------------- light samples
def light(V, UV, s):
    """sample_light_triangle, light_sample_uv and shape_tri_area at flat inputs V [n, 9] (v0, v1, v2), UV [n, 6] and samples s [n, 2]:
    [n, 22] in the hook's layout."""
    v0, v1, v2 = V[:, 0:3], V[:, 3:6], V[:, 6:9]
    a = np.sqrt(s[:, 0:1])
    b1, b2 = 1 - a, a * s[:, 1:2]
    e1, e2 = v1 - v0, v2 - v0
    nrm = normalize(cross(e1, e2))
    fx, fy = coordinate_system(nrm)
    pos = v0 + e1 * b1 + e2 * b2
    r = a
    bu, bv = 1 - r, r * s[:, 1:2]
    uv = (1 - (bu + bv)) * UV[:, 0:2] + bu * UV[:, 2:4] + bv * UV[:, 4:6]
    area = 0.5 * length(cross(e1, e2))[:, None]
    return np.concatenate([pos, nrm, fx, fy, nrm, b1, b2, s, uv, area], 1)


def light_adjoint(V, s, seed):
    """The true adjoint of sample_light_triangle's position, geometric normal and frame (seed [n, 15]) and of shape_tri_area (seed
    [n, 1]) with respect to the vertices V [n, 9]: ([n, 9], [n, 9])."""
    v0, v1, v2 = V[:, 0:3], V[:, 3:6], V[:, 6:9]
    a = np.sqrt(s[:, 0:1])
    b1, b2 = 1 - a, a * s[:, 1:2]
    e1, e2 = v1 - v0, v2 - v0
    cr = cross(e1, e2)
    nrm = normalize(cr)
    d_pos, d_gn, d_fx, d_fy, d_fn = (seed[:, 3 * j:3 * j + 3] for j in range(5))
    d_n = d_normalize(cr, d_gn + d_fn + d_coordinate_system(nrm, d_fx, d_fy))
    out = []
    for d_cr, dp in ((d_n, d_pos), (0.5 * seed[:, 15:16] * nrm, 0 * d_pos)):
        d_e1, d_e2 = d_cross(e1, e2, d_cr)
        d_e1, d_e2 = d_e1 + dp * b1, d_e2 + dp * b2
        out.append(np.concatenate([dp - d_e1 - d_e2, d_e1, d_e2], 1))
    return out[0], out[1]


def central_jacobian(f, X, rel=1e-6, floor=None, nonneg=(), absolute=False):
    """Central differences of f: [n, m] -> [n, p] at X, one input column at a time: [n, m, p].  Step rel * max(|x|, floor), or rel * floor
    with `absolute`; floor [m] or per query [n, m].  The columns
    `nonneg` take a one-sided difference where the lower point would be negative (square roots of light samples at 0)."""
    floor = np.ones(X.shape[1]) if floor is None else floor
    cols = []
    for j in range(X.shape[1]):
        hj = rel * (floor[..., j] * np.ones(len(X)) if absolute else np.maximum(np.abs(X[:, j]), floor[..., j]))
        Xp, Xm = X.copy(), X.copy()
        Xp[:, j] += hj
        Xm[:, j] -= hj
        if j in nonneg:
            Xm[:, j] = np.maximum(Xm[:, j], 0.0)
            Xp[:, j] = Xm[:, j] + 2 * hj
        cols.append((f(Xp) - f(Xm)) / (2 * hj[:, None]))
    return np.stack(cols, 1)
