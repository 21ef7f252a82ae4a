"""Float64 restatement of the camera (rb_camera.cuh, the projection half of rb_render.cuh), written from the formulas, for
tests/test_camera_gpu.py.  Every function takes the camera dict `c` built by `camera(row, ...)` from the DevCamera doubles the hook reports
(RB_CAMTEST_CAMERA), and works on batches: numpy arrays of shape [N, ...].

Adjoints are not restated by hand: `jacobian` takes float64 central differences of the restated forward, whose error (about 1e-9 of the
derivative) is far below the float32 rounding the kernels' adjoints are judged by.  So an adjoint of the restatement cannot share a slip
with the kernel.  The places where the kernels reproduce the reference's slips on purpose are restated as written, by name:
- `near_clip_slip`: d_cam_project's near-clip adjoint uses t = -(q.z + clip_near) / dir.z where the forward has -(q.z - clip_near);
- `ortho_pt_z`: the orthographic d_cam_sample_primary is the adjoint of the forward with pt.z = 1, where the forward has pt.z = 0;
- `distort_r6_slip`: d_cam_distort adds d_r6 * r2 to d_r2 where r6 = r4 * r2 asks for d_r6 * r4."""
import math

import numpy as np

import lens_ref

PI = math.pi


def camera(row, width, height, ctype, use_look_at=True):
    """The DevCamera as RB_CAMTEST_CAMERA reports it (row: 64 doubles)."""
    r = np.asarray(row, np.float64)
    return dict(c2w=r[0:16].reshape(4, 4), w2c=r[16:32].reshape(4, 4), intr_inv=r[32:41].reshape(3, 3), intr=r[41:50].reshape(3, 3),
                k=r[50:58].copy(), r=r[58], f=r[59], clip_near=r[60], width=width, height=height, type=ctype,
                distort=bool(np.any(r[50:58] != 0)), use_look_at=use_look_at)


def rounded(c):
    """The camera with the matrices cam_m4 / cam_m3 round to float32, as the float32 adjoints see them."""
    d = dict(c)
    for key in ("c2w", "w2c", "intr_inv", "intr"):
        d[key] = c[key].astype(np.float32).astype(np.float64)
    return d


# ---------------------------------------------------------------------------------------------------- lens model
def distort(c, q):
    """Brown-Conrady distortion of normalised screen positions q [N, 2] (identity without parameters)."""
    if not c["distort"]:
        return q.copy()
    k = c["k"]
    x, y = 2 * (q[:, 0] - 0.5), 2 * (q[:, 1] - 0.5)
    r2 = x * x + y * y
    rr = (1 + k[0] * r2 + k[1] * r2 ** 2 + k[2] * r2 ** 3) / (1 + k[3] * r2 + k[4] * r2 ** 2 + k[5] * r2 ** 3)
    xx = x * rr + 2 * k[6] * x * y + k[7] * (r2 + 2 * x * x)
    yy = y * rr + k[6] * (r2 + 2 * y * y) + 2 * k[7] * x * y
    return np.stack([(xx + 1) / 2, (yy + 1) / 2], 1)


def inverse_distort(c, p):
    """cam_inverse_distort as written: Gauss-Newton from p, stopping once |residual|_1 <= 1e-3 (at most 1001 steps)."""
    if not c["distort"]:
        return p.copy()
    out = np.empty_like(p)
    for i in range(len(p)):
        u = p[i:i + 1].copy()
        for _ in range(1001):
            J = jacobian(lambda v: distort(c, v), u)[0]
            res = distort(c, u)[0] - p[i]
            u = u - np.linalg.solve(J, res)[None]
            if np.abs(res).sum() <= 1e-3:
                break
        out[i] = u[0]
    return out


def distort_r6_slip(c, q, d_out):
    """What d_cam_distort adds to d_pos on top of the true adjoint: 4 d_r6 (r2 - r4) (x, y)."""
    k = c["k"]
    x, y = 2 * (q[:, 0] - 0.5), 2 * (q[:, 1] - 0.5)
    r2 = x * x + y * y
    num, den = 1 + k[0] * r2 + k[1] * r2 ** 2 + k[2] * r2 ** 3, 1 + k[3] * r2 + k[4] * r2 ** 2 + k[5] * r2 ** 3
    d_rr = d_out[:, 0] / 2 * x + d_out[:, 1] / 2 * y
    d_r6 = d_rr / den * k[2] - d_rr * (num / den) / den * k[5]
    return 4 * (d_r6 * (r2 - r2 * r2))[:, None] * np.stack([x, y], 1)


# ---------------------------------------------------------------------------------------------------- rays
def ray(c, s, u=None, ortho_pt_z=0.0, disc_test=True):
    """(org, dir) [N, 3] of screen positions s [N, 2] (after inverse distortion) as cam_sample_primary defines them; u [N, 2] the lens
    samples in [0, 1)^2 of a camera with a lens.  Fisheye samples outside the unit disc give zero vectors, unless disc_test is False."""
    s = inverse_distort(c, s)
    C, I, aspect = c["c2w"], c["intr_inv"], c["width"] / c["height"]
    n = len(s)
    px, py = (s[:, 0] - 0.5) * 2, (s[:, 1] - 0.5) * -2 / aspect
    org = np.broadcast_to(C[:3, 3] / C[3, 3], (n, 3)).copy()
    t = c["type"]
    if t == 0 and c["r"] > 0:  # the thin lens: tests/lens_ref.py
        o, w = zip(*[lens_ref.lens_ray(c, si[0], si[1], ui[0], ui[1]) for si, ui in zip(s, u)])
        return np.array(o), np.array(w)
    elif t == 0:
        d = (I @ np.stack([px, py, np.ones(n)])).T
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        w = (C[:3, :3] @ d.T).T
    elif t == 1:
        lo = (I @ np.stack([px, py, np.full(n, ortho_pt_z)])).T
        oh = (C @ np.concatenate([lo, np.ones((n, 1))], 1).T).T
        org = oh[:, :3] / oh[:, 3:4]
        w = np.broadcast_to(C[:3, 2], (n, 3)).copy()
    else:
        if t == 2:
            x, y = 2 * (s[:, 0] - 0.5), 2 * (s[:, 1] - 0.5)
            r = np.hypot(x, y)
            th = r * PI / 2
            # (-cos(phi) sin(theta), -sin(phi) sin(theta)) with the limit sin(theta) / r -> pi / 2 at the centre
            sr = np.where(r > 0, np.sin(th) / np.where(r > 0, r, 1), PI / 2)
            l = np.stack([-x * sr, -y * sr, np.cos(th)], 1)
            out = (x * x + y * y > 1) & disc_test
        else:
            th, ph = PI * s[:, 1], 2 * PI * s[:, 0]
            l = np.stack([np.cos(ph) * np.sin(th), np.cos(th), np.sin(ph) * np.sin(th)], 1)
            out = np.zeros(n, bool)
        w = (C[:3, :3] @ l.T).T
        org[out] = 0
        w[out] = 0
    nw = np.linalg.norm(w, axis=1, keepdims=True)
    return org, w / np.where(nw > 0, nw, 1)


# ---------------------------------------------------------------------------------------------------- projection
def to_screen(c, P):
    """Camera-space points P [N, 3] to normalised screen positions (cam_to_screen: the map, then the distortion)."""
    t, aspect = c["type"], c["width"] / c["height"]
    if t in (2, 3):
        d = P / np.linalg.norm(P, axis=1, keepdims=True)
        if t == 2:  # s = 1/2 - (theta / (pi sin(theta))) (d.x, d.y), smooth at the axis
            rho = np.hypot(d[:, 0], d[:, 1])
            th = np.arctan2(rho, d[:, 2])
            G = np.where(rho > 0, th / np.where(rho > 0, rho, 1), 1.0)
            q = 0.5 - G[:, None] * d[:, :2] / PI
        else:
            q = np.stack([np.arctan2(d[:, 2], d[:, 0]) / (2 * PI), np.arctan2(np.hypot(d[:, 0], d[:, 2]), d[:, 1]) / PI], 1)
    else:
        ip = (c["intr"] @ P.T).T
        if t == 0:
            q = np.stack([(ip[:, 0] / ip[:, 2] + 1) * 0.5, (-(ip[:, 1] / ip[:, 2]) * aspect + 1) * 0.5], 1)
        else:
            q = np.stack([(ip[:, 0] + 1) * 0.5, (-ip[:, 1] * aspect + 1) * 0.5], 1)
    return distort(c, q)


def to_camera(c, p):
    ph = (c["w2c"] @ np.concatenate([p, np.ones((len(p), 1))], 1).T).T
    return ph[:, :3] / ph[:, 3:4]


def clip(c, a, b):
    """cam_project's near clip in camera space: (clipped a, clipped b, a was clipped, b was clipped, visible)."""
    cn = c["clip_near"]
    ca, cb = a < cn, b < cn
    a, b = a.copy(), b.copy()
    ia, ib = ca[:, 2] & ~cb[:, 2], cb[:, 2] & ~ca[:, 2]
    ta = -(b[:, 2] - cn) / (a[:, 2] - b[:, 2])
    a[ia] = (b + ta[:, None] * (a - b))[ia]
    tb = -(a[:, 2] - cn) / (b[:, 2] - a[:, 2])
    b[ib] = (a + tb[:, None] * (b - a))[ib]
    return a, b, ia, ib, ~(ca[:, 2] & cb[:, 2])


def project(c, p0, p1, lu=None):
    """(visible [N], q0 [N, 2], q1 [N, 2]) of world-space segments: cam_project_d, or cam_project_lens_d for a camera with a lens."""
    a, b, _, _, vis = clip(c, to_camera(c, p0), to_camera(c, p1))
    if c["r"] > 0:
        L = c["r"] * lu
        f = c["f"]
        film = lambda P: np.stack([L[:, 0] / f + (P[:, 0] - L[:, 0]) / P[:, 2], L[:, 1] / f + (P[:, 1] - L[:, 1]) / P[:, 2], np.ones(len(P))], 1)
        a, b = film(a), film(b)
    return vis, to_screen(c, a), to_screen(c, b)


def near_clip_slip(c, a, b, d_ca, d_cb):
    """What d_cam_project adds to the camera-space (d_a, d_b) on top of the true adjoint, from the '+ clip_near' in its clip adjoint:
    with q the end in front and dir = p - q (p the clipped end), (t' - t) (d_c - e_z dot(dir, d_c) / dir.z) goes to d_p and its negative
    to d_q, t' - t = -2 clip_near / dir.z."""
    cn = c["clip_near"]
    da, db = np.zeros_like(a), np.zeros_like(b)
    for p, q, d_c, dp, dq, m in ((a, b, d_ca, da, db, (a[:, 2] < cn) & (b[:, 2] >= cn)), (b, a, d_cb, db, da, (b[:, 2] < cn) & (a[:, 2] >= cn))):
        dirv = p - q
        dt = (dirv * d_c).sum(1)
        delta = (-2 * cn / dirv[:, 2])[:, None] * (d_c - np.outer(dt / dirv[:, 2], [0, 0, 1]))
        dp[m] += delta[m]
        dq[m] -= delta[m]
    return da, db


# ---------------------------------------------------------------------------------------------------- differentiation
def jacobian(f, x, rel=1e-6, floor=1e-3):
    """Float64 central differences of f: [N, m] -> [N, k] at x: [N, k, m], steps rel * max(|x|, floor) per coordinate."""
    x = np.asarray(x, np.float64)
    cols = []
    for j in range(x.shape[1]):
        h = rel * np.maximum(np.abs(x[:, j]), floor)
        xp, xm = x.copy(), x.copy()
        xp[:, j] += h
        xm[:, j] -= h
        cols.append((f(xp) - f(xm)) / (2 * h)[:, None])
    return np.stack(cols, 2)
