"""GPU suite: the camera (rb_camera.cuh and the projection half of rb_render.cuh) through the test hook rb_camera_test, query by query,
against the float64 restatement in tests/camera_ref.py; and the backward pass of scenes whose cameras look straight at a vertex along the
fisheye axis, at a panorama pole, and through the centre of a distorted lens.

Cameras: a square look-at pinhole, a 40x30 pinhole with a skewed intrinsic matrix, a cam_to_world pinhole 10^3 from the origin, clip_near
1, an orthographic camera, fisheye and panorama cameras, distortion on a perspective and on a fisheye camera, and a thin lens.

Query families:
- rays: uniform screen positions, the exact centre, pixel centres of odd resolutions, 0 and 1 - 2^-53, the fisheye disc boundary +- 1 ulp,
  the panorama seam and poles;
- segments: uniform in front, one end behind the near plane, both behind, one end exactly on it, near the z = 0 plane, at 10^4 distance,
  degenerate (both ends equal), and for the fisheye / panorama ends exactly on the axis / pole and at 1e-7 ... 1e-1 rad from it;
- seeds: random, unit, and all zero.

Comparison rules:
- double outputs (cam_sample_primary, cam_distort and its Jacobian rows, the distortion adjoints): within 1e-12 (rays), 1e-13 (distort)
  of the restatement, relative to the output's scale, and within 1e-7 where the restatement differentiates or inverts numerically
  (Jacobian rows, Gauss-Newton steps); the float32 ray equals the double ray rounded to float32, bit for bit;
- float32 adjoints (d_cam_project's d_p0, d_p1; d_cam_sample_primary's d_screen and camera columns): the restatement is evaluated at the
  float32 inputs and float32-rounded matrices the kernel sees, and the error must be within K u (sum_i |dy/dx_i| |x_i| + |J|^T |s| + |y|),
  u = 2^-24, K = 64.  The first term is the conditioning of the adjoint itself, measured by perturbing the restatement's inputs; the second
  the conditioning of the linear map applied to the seed.  K covers the longest rounding chain, about 30 float operations between an
  input and an output (transform, clip, normalize, the screen map, d_normalize, the transform back) with the 2-ulp division and square root
  of the fast build;
- a clipped end lies on z = clip_near, computed as q.z + t (p.z - q.z) in float32: its rounding relative to clip_near, and so the bound,
  grows by (|a.z| + |b.z|) / clip_near;
- where float32 rounding can flip the near-clip decision (an end within 1e-5 of the plane), either answer is accepted: only finiteness is
  checked, and such queries are counted per family; every family but "both behind" and "on the plane" (a rounding decision by
  construction) compares some queries strictly.  With distortion, clipped segments are checked for finiteness only: the restatement
  carries d_cam_distort's slip through the screen map of ends in front of the plane only;
- zero seeds give exactly zero and leave the accumulator column untouched;
- every output is finite, on the fisheye axis, at the panorama poles and at the distortion centre included."""
import math

import numpy as np
import pytest
import torch

import camera_ref as R
from redner_b200 import api
from redner_b200 import _lib as L

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K = 64
CAMERAS = ["pinhole", "skewed", "c2w_far", "clip1", "ortho", "fisheye", "panorama", "panorama_clip0", "distort_persp", "distort_fish", "lens"]


# ---------------------------------------------------------------------------------------------------- cameras and scenes
def make_camera(name, res=None):
    t = lambda v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    pos, look, up = t([0.3, 1.4, -4.5]), t([0.0, 0.6, 0.0]), t([0.0, 1.0, 0.0])
    kw = dict(position=pos, look_at=look, up=up, fov=t([45.0]), clip_near=1e-2, resolution=res or (32, 32))
    if name == "skewed":
        kw.update(resolution=res or (30, 40), intrinsic_mat=t([[1.4, 0.2, 0.05], [0.0, 1.3, -0.03], [0.0, 0.0, 1.0]]))
    elif name == "c2w_far":
        c2w = torch.eye(4)
        c2w[:3, :3] = torch.tensor([[0.8, 0.0, 0.6], [0.0, 1.0, 0.0], [-0.6, 0.0, 0.8]])
        c2w[:3, 3] = t([600.0, 300.0, -742.0])
        kw = dict(cam_to_world=c2w, fov=t([45.0]), clip_near=1e-2, resolution=res or (32, 32))
    elif name == "clip1":
        kw.update(clip_near=1.0)
    elif name == "ortho":
        kw.update(intrinsic_mat=t([[0.4, 0.0, 0.0], [0.0, 0.4, 0.0], [0.0, 0.0, 1.0]]), camera_type=1)
    elif name == "panorama_clip0":  # clip_near 0 and an axis-aligned pose: points on the poles reach the map exactly
        c2w = torch.eye(4)
        c2w[:3, 3] = t([0.5, 1.0, -2.0])
        kw = dict(cam_to_world=c2w, clip_near=0.0, resolution=res or (32, 32), camera_type=3)
    elif name in ("fisheye", "panorama", "distort_fish"):
        kw.update(position=t([0.4, 1.2, -1.6]), look_at=t([0.1, 0.7, 0.2]), fov=None, camera_type=2 if name != "panorama" else 3)
    if name.startswith("distort"):
        kw.update(distortion_params=t([0.1, -0.05, 0.02, 0.03, 0.01, -0.01, 0.004, -0.003]))
    if name == "lens":
        kw.update(lens_radius=t([0.08]), focus_distance=t([4.0]))
    return api.Camera(**kw)


def native_scene(rb, dev, cam):
    v = torch.tensor([[-1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], device=dev)
    i = torch.tensor([[0, 1, 2]], dtype=torch.int32, device=dev)
    sc = api.Scene(cam, [api.Shape(v, i, 0)], [api.Material(diffuse_reflectance=torch.tensor([0.5, 0.5, 0.5], device=dev))], [])
    args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev, backend=rb)
    c = api.RenderFunction._unpack([0], args)
    c.args = args  # (keeps the tensors the native scene points into alive)
    return c


class Hook:
    def __init__(self, rb, dev, name):
        self.cam = make_camera(name)
        self.ctx = native_scene(rb, dev, self.cam)
        self.dev = dev
        row = self.run(L.RB_CAMTEST_CAMERA, np.zeros((1, 1)))[0][0]
        h, w = self.cam.resolution
        self.c = R.camera(row, w, h, self.cam.camera_type)
        self.n_acc = int(row[61])

    def run(self, op, x, acc=None):
        out, acc = self.ctx.scene.camera_test(op, torch.from_numpy(np.asarray(x, np.float64)).to(self.dev), acc)
        return out.cpu().numpy(), (acc.cpu().numpy() if acc is not None else None)


# ---------------------------------------------------------------------------------------------------- query families
def screen_families(c, rng, n):
    w, h = c["width"], c["height"]
    fam = {"uniform": rng.random((n, 2)), "centre": np.array([[0.5, 0.5]]),
           "odd_pixel_centres": np.stack([(np.arange(7) + 0.5) / 7, (np.arange(7) + 0.5) / 7], 1),
           "edges": np.array([[0.0, 0.0], [1 - 2.0 ** -53, 1 - 2.0 ** -53], [0.0, 1 - 2.0 ** -53]])}
    if c["type"] == 2:
        a = rng.random(n) * 2 * math.pi
        r = np.concatenate([np.nextafter(np.ones(n // 2), 2), np.nextafter(np.ones(n - n // 2), 0)])
        fam["disc_boundary"] = np.stack([0.5 + 0.5 * r * np.cos(a), 0.5 + 0.5 * r * np.sin(a)], 1)
    if c["type"] == 3:
        fam["seam_poles"] = np.array([[0.0, 0.3], [1 - 2.0 ** -53, 0.3], [0.3, 0.0], [0.7, 1 - 2.0 ** -53], [0.25, 0.5]])
    return fam


def axis_points(c, n, rng):
    """Camera-space directions exactly on the fisheye axis / panorama poles and at 1e-7 ... 1e-1 rad from them, placed in world space.
    Every point lies in front of the near plane, which would otherwise move it off the pole: the panorama's are tilted towards +z and
    placed far enough out that z >= 2 clip_near, at most 10^3 away (further out, the float32 transform to camera space rounds the offset
    from the pole by more than the bound's linear model covers), so a camera with clip_near > 0 gets the angles from 1e-4 rad; the
    axis-aligned clip_near 0 camera, whose transform is exact, gets the exact poles (z = 0) and every angle."""
    axis = np.array([0.0, 0.0, 1.0]) if c["type"] == 2 else np.array([0.0, 1.0, 0.0])
    pts = [axis * 2.0]
    if c["type"] == 3:
        pts = [axis * 2.0, -axis * 2.0] if c["clip_near"] == 0 else []
    for e in 10.0 ** np.arange(-7, 0):
        for sign in ((1.0,) if c["type"] == 2 else (1.0, -1.0)):
            a = rng.uniform(math.pi / 6, 5 * math.pi / 6)
            perp = np.array([math.cos(a), math.sin(a), 0.0]) if c["type"] == 2 else np.array([math.cos(a), 0.0, math.sin(a)])
            L = 2.0 if c["type"] == 2 else max(2.0, 4 * c["clip_near"] / math.sin(e))
            if L <= 1e3:
                pts.append(L * (math.cos(e) * sign * axis + math.sin(e) * perp))
    P = np.array(pts)
    Ph = (c["c2w"] @ np.concatenate([P, np.ones((len(P), 1))], 1).T).T
    return Ph[:, :3] / Ph[:, 3:4]


def world(c, P):
    Ph = (c["c2w"] @ np.concatenate([P, np.ones((len(P), 1))], 1).T).T
    return Ph[:, :3] / Ph[:, 3:4]


def segment_families(c, rng, n):
    cn = c["clip_near"]
    front = lambda m: np.stack([rng.uniform(-1, 1, m), rng.uniform(-1, 1, m), rng.uniform(cn + 0.5, 6, m)], 1)  # noqa: E731
    behind = lambda m: np.stack([rng.uniform(-1, 1, m), rng.uniform(-1, 1, m), rng.uniform(-3, cn - 0.2, m)], 1)  # noqa: E731
    fam = {"front": (front(n), front(n)), "one_behind": (behind(n), front(n)), "other_behind": (front(n), behind(n)),
           "both_behind": (behind(n), behind(n))}
    on = front(n)
    on[:, 2] = cn
    fam["plane_rounding"] = (on, front(n))  # (on the plane in double; the float32 ends lie within rounding of it)
    near = front(n)
    near[:, 2] = cn * (1 + rng.random(n))
    fam["just_in_front"] = (near, front(n))
    fam["far"] = (front(n) * 1e4 / 6, front(n) * 1e4 / 6)
    d = front(n)
    fam["degenerate"] = (d, d.copy())
    if c["type"] in (2, 3):
        A = axis_points(c, n, rng)
        fam["axis"] = (A, world(c, front(len(A))))
        return {k: (v[0], v[1]) if k == "axis" else (world(c, v[0]), world(c, v[1])) for k, v in fam.items()}
    return {k: (world(c, a), world(c, b)) for k, (a, b) in fam.items()}


def seeds(rng, n, k):
    s = rng.normal(size=(n, k))
    s[1::5] = 0
    s[2::5] = 0
    s[1::5, 0] = 1.0
    s[3::7] = 0.0
    return s


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def assert_within(name, got, want, tol, mask=None):
    err = np.abs(got - want)
    tol = np.broadcast_to(tol, err.shape)
    bad = ~(err <= tol)
    if mask is not None:
        bad &= mask[:, None] if bad.ndim == 2 else mask
    assert not bad.any(), "%s: %d bad, worst %s got %s want %s tol %s" % (name, bad.sum(), np.argwhere(bad)[:3].tolist(), got[bad][:4], want[bad][:4], tol[bad][:4])


# ---------------------------------------------------------------------------------------------------- checks
def check_rays(rb, dev, name, n=64, seed=1):
    h = Hook(rb, dev, name)
    c, rng = h.c, np.random.default_rng(seed)
    for fam, s in screen_families(c, rng, n).items():
        u = rng.random((len(s), 2))
        out, _ = h.run(L.RB_CAMTEST_RAY, np.concatenate([s, u], 1))
        assert np.isfinite(out[:, :26]).all(), (name, fam)
        org, d = R.ray(c, s, u)
        tol = 1e-7 if c["distort"] else 1e-12
        scale = 1 + np.abs(org).max(1, keepdims=True)
        # the disc test x^2 + y^2 > 1 of a position 1 ulp from the fisheye boundary is a rounding decision (the device contracts it into
        # an FMA): there either the null ray or the restated ray without the disc test is accepted
        null = (out[:, 3:6] == 0).all(1) & (out[:, 0:3] == 0).all(1)
        keep = np.ones(len(s), bool)
        if fam == "disc_boundary":
            keep = ~null
            org, d = R.ray(c, s, u, disc_test=False)
        assert_within("%s/%s org" % (name, fam), out[:, 0:3], org, tol * scale, keep)
        assert_within("%s/%s dir" % (name, fam), out[:, 3:6], d, np.full_like(d, tol), keep)
        assert np.array_equal(out[:, 6:12], f32(out[:, 0:6])), (name, fam, "float ray is not the rounded double ray")
        lu = np.array([R.lens_ref.concentric(*ui) for ui in u])
        assert_within("%s/%s concentric_disc" % (name, fam), out[:, 24:26], lu, np.full_like(lu, 1e-15))
        # the ray differential: psx (ray(sx + delta, sy) - ray(sx, sy)) / delta and likewise in y, rounded to float32 once
        if fam != "disc_boundary":
            o1, d1 = R.ray(c, s + [1e-3, 0], u)
            o2, d2 = R.ray(c, s + [0, 1e-3], u)
            psx, psy = 0.5 / c["width"], 0.5 / c["height"]
            diff = np.concatenate([psx * (o1 - org), psy * (o2 - org), psx * (d1 - d), psy * (d2 - d)], 1) / 1e-3
            # one float32 ulp, and the restatement's own error over delta
            one = np.ones_like(scale)
            err = (tol / 1e-3) * np.concatenate([psx * scale, psy * scale, psx * one, psy * one], 1).repeat(3, 1)
            assert_within("%s/%s differential" % (name, fam), out[:, 12:24], diff, np.abs(diff) * 2.0 ** -23 + 2 * err)


def pole_ends(c, p0, p1):
    """[N, 2]: which end lies exactly on a panorama pole in camera space (x = z = 0), where the adjoint's pole rule drops both terms."""
    cr = R.rounded(c)
    if c["type"] != 3:
        return np.zeros((len(p0), 2), bool)
    return np.stack([(P[:, 0] == 0) & (P[:, 2] == 0) for P in (R.to_camera(cr, p0), R.to_camera(cr, p1))], 1)


def dproject_reference(c, p0, p1, lu, s):
    """(d_p0 d_p1 [N, 6], |J|^T |s|, J [N, 4, 6]) of the restated projection at float32 inputs, with d_cam_project's near-clip slip; an
    end exactly on a panorama pole contributes nothing (the pole rule)."""
    cr = R.rounded(c)
    x = np.concatenate([p0, p1], 1)
    J = R.jacobian(lambda v: np.concatenate(R.project(cr, v[:, :3], v[:, 3:], lu)[1:], 1), x)  # [N, 4, 6]
    pole = pole_ends(c, p0, p1)
    J[pole[:, 0], :, 0:3] = 0
    J[pole[:, 1], :, 3:6] = 0
    y = np.einsum("nk,nkm->nm", s, J)
    mag = np.einsum("nk,nkm->nm", np.abs(s), np.abs(J))
    if cr["r"] == 0:
        a, b = R.to_camera(cr, p0), R.to_camera(cr, p1)
        ca, cb, _, _, _ = R.clip(cr, a, b)
        Ja, Jb = R.jacobian(lambda v: R.to_screen(cr, v), ca), R.jacobian(lambda v: R.to_screen(cr, v), cb)
        da, db = R.near_clip_slip(cr, a, b, np.einsum("nk,nkm->nm", s[:, :2], Ja), np.einsum("nk,nkm->nm", s[:, 2:], Jb))
        W3 = cr["w2c"][:3, :3]
        y = y + np.concatenate([da @ W3, db @ W3], 1)
        if cr["distort"]:  # d_cam_distort's r6 slip, through the undistorted screen map, for ends in front of the plane
            und = dict(cr, distort=False)
            for k, (P, e) in enumerate(((a, ca), (b, cb))):
                Ju = R.jacobian(lambda v: R.to_screen(und, v), e)
                dq = R.distort_r6_slip(cr, R.to_screen(und, e), s[:, 2 * k:2 * k + 2])
                y[:, 3 * k:3 * k + 3] += np.einsum("nk,nkm->nm", dq, Ju) @ W3
    return y, mag, J


def check_project(rb, dev, name, n=48, seed=2):
    h = Hook(rb, dev, name)
    c, rng = h.c, np.random.default_rng(seed)
    counts = {}
    for fam, (p0, p1) in segment_families(c, rng, n).items():
        p0, p1 = f32(p0), f32(p1)
        m = len(p0)
        u = rng.random((m, 2))
        lu = np.array([R.lens_ref.concentric(*ui) for ui in u])
        s = f32(seeds(rng, m, 4))
        x = np.concatenate([p0, p1, u, s], 1)
        acc0 = torch.full((60, m), 0.25, dtype=torch.float32, device=dev)
        out, acc = h.run(L.RB_CAMTEST_D_PROJECT, x, acc0)
        got = out[:, :6]
        assert np.isfinite(got).all() and np.isfinite(acc).all(), (name, fam)
        zero = (s == 0).all(1)
        assert (got[zero] == 0).all() and (acc[:, zero] == 0.25).all(), (name, fam, "zero seed")
        # the double projection the primary-edge pick uses
        pout, _ = h.run(L.RB_CAMTEST_PROJECT, np.concatenate([p0, p1, u], 1))
        vis, q0, q1 = R.project(c, p0, p1, lu)
        assert np.array_equal(pout[:, 0] != 0, vis), (name, fam)
        sc = 1 + np.abs(np.concatenate([q0, q1], 1))
        if c["type"] == 3:  # the seam: atan2 of a direction on it gives s.x = -1/2 or 1/2 by the sign of a zero, the same direction
            pout = pout.copy()
            for k, want in ((1, q0[:, 0]), (3, q1[:, 0]), (6, q0[:, 0]), (8, q1[:, 0])):
                pout[:, k] -= np.round(pout[:, k] - want)
        # (the fisheye and panorama maps of cam_project_d take acos of d.z / d.y in double: about 1e-16 / theta near the axis and poles)
        qtol = 1e-7 if c["distort"] or c["type"] in (2, 3) else 1e-11
        assert_within("%s/%s project_d" % (name, fam), pout[:, 1:5], np.concatenate([q0, q1], 1), qtol * sc, vis)
        # the float32 adjoint
        cr = R.rounded(c)
        a, b = R.to_camera(cr, p0), R.to_camera(cr, p1)
        cn = cr["clip_near"]
        near = lambda z: (np.abs(z - cn) <= 1e-5 * (1 + np.abs(z))) & (z != cn)  # noqa: E731  (an end exactly on the plane is exact)
        # (clip_near 0: the axis-aligned camera, whose float32 camera-space z is exact, so its near-clip decision is too)
        ambiguous = near(a[:, 2]) | near(b[:, 2]) if cn > 0 else np.zeros(m, bool)
        clipped = vis & ((a[:, 2] < cn) | (b[:, 2] < cn))
        if c["distort"] or cn == 0:
            ambiguous |= clipped  # (the distortion slip is restated for ends in front of the plane only; clip_near 0 clips onto z = 0)
        strict = ~ambiguous & vis & ~zero
        y, mag, J = dproject_reference(c, p0, p1, lu, s)
        pole = pole_ends(c, p0, p1)
        assert (got[pole[:, 0] & vis, 0:3] == 0).all() and (got[pole[:, 1] & vis, 3:6] == 0).all(), (name, fam, "pole rule")
        # the float projection primary_edge_weight uses: within the same bound, of the map (the fisheye / panorama maps of cam_project
        # take acos in float32, about u / theta near the axis and poles: not compared on that family)
        xin = np.abs(np.concatenate([p0, p1], 1)) + np.abs(c["w2c"][:3, 3]).max() + 1
        qmag = np.einsum("nkm,nm->nk", np.abs(J), xin) + np.abs(np.concatenate([q0, q1], 1)) + 1
        fstrict = strict if fam != "axis" else np.zeros(m, bool)
        if c["r"] > 0:  # (cam_project is the pinhole's projection; the lens camera's pick uses cam_project_lens_d)
            _, q0, q1 = R.project(dict(c, r=0.0), p0, p1)
            qmag = np.abs(np.concatenate([q0, q1], 1)) * 64 + 1
        assert np.array_equal(pout[strict, 5] != 0, vis[strict]), (name, fam)
        amp_q = np.where(clipped, 1 + (np.abs(a[:, 2]) + np.abs(b[:, 2])) / max(cn, 1e-30), 1.0)[:, None]
        assert_within("%s/%s cam_project" % (name, fam), pout[:, 6:10], np.concatenate([q0, q1], 1), K * U * qmag * amp_q, fstrict)
        # conditioning of the adjoint itself: the restatement at ends moved by 2^-20 of their scale (the float32 transform to camera
        # space rounds every coordinate to about u times |W| |(p, 1)|), scaled back to u
        sens = np.zeros_like(y)
        e = 2.0 ** -20
        scale = np.abs(np.concatenate([p0, p1], 1)).max(1) + np.abs(c["w2c"][:3, 3]).max() + 1
        for j in range(6):
            xp, xm = np.concatenate([p0, p1], 1), np.concatenate([p0, p1], 1)
            xp[:, j] += e * scale
            xm[:, j] -= e * scale
            yp, ym = dproject_reference(c, xp[:, :3], xp[:, 3:], lu, s)[0], dproject_reference(c, xm[:, :3], xm[:, 3:], lu, s)[0]
            sens += np.abs(yp - ym) / 2
        # a clipped end lies on z = clip_near, computed as q.z + t (p.z - q.z): rounded by about u (|a.z| + |b.z|), relative to clip_near
        amp = amp_q
        tol = K * U * (sens / e + mag + np.abs(y).max(1, keepdims=True)) * amp
        assert_within("%s/%s d_project" % (name, fam), got, y, tol, strict)
        counts[fam] = (int(strict.sum()), int((ambiguous & vis & ~zero).sum()))
    for fam, (ns, na) in counts.items():
        # (both behind: nothing to compare; on the plane: every end is a rounding decision by construction)
        assert ns > 0 or fam in ("both_behind", "plane_rounding") or ((c["distort"] or cn == 0) and "behind" in fam), (name, fam, counts)
    return counts


def check_distort(rb, dev, name, n=64, seed=3):
    h = Hook(rb, dev, name)
    c, rng = h.c, np.random.default_rng(seed)
    pos = np.concatenate([np.array([[0.5, 0.5]]), rng.uniform(0.05, 0.95, (n, 2)), np.array([[0.5, 0.5 + 1e-9], [0.5 + 2.0 ** -30, 0.5]])])
    d_out = rng.normal(size=(len(pos), 2))
    d_out[1] = 0
    out, _ = h.run(L.RB_CAMTEST_DISTORT, np.concatenate([pos, d_out], 1))
    assert np.isfinite(out[:, :28]).all(), name
    assert np.array_equal(out[0, 0:2], [0.5, 0.5]) and np.array_equal(out[0, 6:8], [0.5, 0.5]), (name, "the centre maps to itself")
    q = R.distort(c, pos)
    assert_within(name + " distort", out[:, 0:2], q, np.full_like(q, 1e-13))
    J = R.jacobian(lambda v: R.distort(c, v), pos)  # [N, 2 (out), 2 (pos)]
    assert_within(name + " jacobian", out[:, 2:6], J.reshape(-1, 4), 1e-7 * (1 + np.abs(J.reshape(-1, 4))))
    want = np.einsum("nk,nkm->nm", d_out, J) + R.distort_r6_slip(c, pos, d_out)
    assert_within(name + " d_distort", out[:, 8:10], want, 1e-7 * (1 + np.abs(want)))
    inv = out[:, 6:8]
    assert np.abs(R.distort(c, inv) - pos).sum(1).max() <= 2e-3, name
    Ji = R.jacobian(lambda v: R.distort(c, v), inv)
    want = np.linalg.solve(np.transpose(Ji, (0, 2, 1)), d_out[:, :, None])[:, :, 0]
    assert_within(name + " d_inverse_distort", out[:, 10:12], want, 1e-6 * (1 + np.abs(want)))
    assert (out[1, 8:28] == 0).all(), (name, "zero seed")
    # parameter gradients: d_out . d(distort)/dk, and through the implicit function -(J^-T d_out) . d(distort)/dk at the inverse
    k0 = c["k"].copy()

    def by_k(pos_):
        return lambda v: np.concatenate([R.distort(dict(c, k=v[i]), pos_[i:i + 1]) for i in range(len(v))])
    # (distort is linear in k1..k3, p1, p2 and rational in k4..k6: wide steps keep the differences above the rounding of tiny r^n terms)
    Jk = R.jacobian(by_k(pos), np.tile(k0, (len(pos), 1)), rel=1e-4, floor=0.1)  # [N, 2, 8]
    want = np.einsum("nk,nkm->nm", d_out, Jk)
    assert_within(name + " d_distort params", out[:, 12:20], want, 1e-6 * np.einsum("nk,nkm->nm", np.abs(d_out), np.abs(Jk)) + 1e-9 * np.abs(want).max())
    Jki = R.jacobian(by_k(inv), np.tile(k0, (len(pos), 1)), rel=1e-4, floor=0.1)
    lam = np.linalg.solve(np.transpose(Ji, (0, 2, 1)), d_out[:, :, None])[:, :, 0]
    want = -np.einsum("nk,nkm->nm", lam, Jki)
    assert_within(name + " d_inverse_distort params", out[:, 20:28], want, 1e-6 * np.einsum("nk,nkm->nm", np.abs(lam), np.abs(Jki)) + 1e-9 * np.abs(want).max())


def check_ray_adjoint(rb, dev, name, n=48, seed=4):
    h = Hook(rb, dev, name)
    c, rng = h.c, np.random.default_rng(seed)
    cr = R.rounded(c)
    pt_z = 1.0 if c["type"] == 1 else 0.0  # (the orthographic adjoint's pt.z = 1, camera_ref.ortho_pt_z)
    for fam, s in screen_families(c, rng, n).items():
        m = len(s)
        u = rng.random((m, 2))
        dr = f32(seeds(rng, m, 6))
        want_screen = 0.0 if c["r"] > 0 else 1.0
        acc0 = torch.full((60, m), 0.25, dtype=torch.float32, device=dev)
        out, acc = h.run(L.RB_CAMTEST_D_RAY, np.concatenate([s, u, dr, np.full((m, 1), want_screen)], 1), acc0)
        assert np.isfinite(out[:, :2]).all() and np.isfinite(acc).all(), (name, fam)
        zero = (dr == 0).all(1)
        assert (out[zero, :2] == 0).all() and (acc[:, zero] == 0.25).all(), (name, fam, "zero seed")
        sf = f32(s)
        inside = np.ones(m, bool) if c["type"] != 2 else ((2 * (sf - 0.5)) ** 2).sum(1) <= 1 - 1e-6
        # d_screen against differences of the restated ray at the float32 screen position
        if want_screen and not c["distort"]:
            def f(v):
                o, d = R.ray(cr, v, u, ortho_pt_z=pt_z)
                return np.concatenate([o, d], 1)
            J = R.jacobian(f, sf)
            y = np.einsum("nk,nkm->nm", dr, J)
            mag = np.einsum("nk,nkm->nm", np.abs(dr), np.abs(J))
            ok = inside & (np.abs(sf - 0.5) < 0.5 - 1e-6).all(1) if c["type"] == 3 else inside
            assert_within("%s/%s d_screen" % (name, fam), out[:, :2], y, 4 * K * U * (mag + np.abs(y).max(1, keepdims=True) + 1e-3 * mag.max()), ok & ~zero)
        # the accumulator columns: c2w (0-15), intr_inv (32-40) and, with a lens, lens_radius (58) and focus_distance (59); alone, and
        # with the ray differential's adjoint (three rays, at s, s + (delta, 0) and s + (0, delta) as the kernel forms them in float32)
        if not c["distort"]:
            check_ray_columns(h, cr, name, fam, sf, u, dr, inside & ~zero, pt_z, acc, rng)


def ray_columns_reference(cr, pos, u, w, pt_z):
    """(y, |w|^T |J|) of the 25 (27 with a lens) accumulator entries for one ray at screen position pos [2] with adjoint w [6]."""
    lens = cr["r"] > 0
    base = np.concatenate([cr["c2w"].ravel(), cr["intr_inv"].ravel()] + ([[cr["r"], cr["f"]]] if lens else []))

    def g(v):
        d = dict(cr)
        d["c2w"], d["intr_inv"] = v[0, :16].reshape(4, 4), v[0, 16:25].reshape(3, 3)
        if lens:
            d["r"], d["f"] = v[0, 25], v[0, 26]
        o, dd = R.ray(d, pos[None], u[None], ortho_pt_z=pt_z)
        return np.concatenate([o, dd], 1)
    Jc = R.jacobian(g, base[None])[0]
    return w @ Jc, np.abs(w) @ np.abs(Jc)


def check_ray_columns(h, cr, name, fam, sf, u, dr, ok, pt_z, acc, rng):
    rows = np.r_[0:16, 32:41] if cr["r"] == 0 else np.r_[0:16, 32:41, 58:60]
    for j in np.flatnonzero(ok)[:8]:
        y, mag = ray_columns_reference(cr, sf[j], u[j], dr[j], pt_z)
        got = acc[rows, j] - 0.25
        tol = 4 * K * U * (mag + np.abs(y).max() + 1) + 1e-7
        assert (np.abs(got - y) <= tol).all(), (name, fam, j, got, y, tol)
    # the differential: d(org_dx, org_dy, dir_dx, dir_dy) -> the two offset rays and the centre ray (bwd_sweep's d_cam_primary_ray_diff)
    j = np.flatnonzero(ok)[:4]
    if len(j) == 0 or (cr["type"] == 2 and fam == "disc_boundary"):
        return
    m = len(j)
    dprd = f32(rng.normal(size=(m, 12)))
    x = np.zeros((m, 24))
    x[:, 0:2], x[:, 2:4], x[:, 4:10], x[:, 11:23], x[:, 23] = sf[j], u[j], dr[j], dprd, 1
    acc0 = torch.full((60, m), 0.25, dtype=torch.float32, device=h.dev)
    _, acc2 = h.run(L.RB_CAMTEST_D_RAY, x, acc0)
    f = np.float32
    delta = f(1e-3)
    psx, psy = float(f(0.5) / f(cr["width"])), float(f(0.5) / f(cr["height"]))
    for i in range(m):
        sx, sy = f(sf[j[i], 0]), f(sf[j[i], 1])
        pos = [np.array([sx, sy], np.float64), np.array([f(sx + delta), sy], np.float64), np.array([sx, f(sy + delta)], np.float64)]
        odx, ody, ddx, ddy = dprd[i, 0:3], dprd[i, 3:6], dprd[i, 6:9], dprd[i, 9:12]
        w0 = dr[j[i]] + np.concatenate([-psx * odx - psy * ody, -psx * ddx - psy * ddy]) / float(delta)
        w = [w0, np.concatenate([odx, ddx]) * psx / float(delta), np.concatenate([ody, ddy]) * psy / float(delta)]
        y, mag = 0, 0
        for k in range(3):
            yk, mk = ray_columns_reference(cr, pos[k], u[j[i]], w[k], pt_z)
            y, mag = y + yk, mag + mk
        got = acc2[rows, i] - 0.25
        tol = 4 * K * U * (mag + np.abs(y).max() + 1) + 1e-7
        assert (np.abs(got - y) <= tol).all(), (name, fam, "differential", i, got, y, tol)


def look_at(pos, look, up):
    """The look-at cam_to_world of the host set-up, in float64 (rows: right, up, forward, position)."""
    n = lambda v: v / np.linalg.norm(v)  # noqa: E731
    d = n(look - pos)
    r = n(np.cross(d, n(up)))
    nu = n(np.cross(r, d))
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = r, nu, d, pos
    return m


def check_finish(rb, dev, name, n=16, seed=5):
    """finish_camera on given reduced accumulators: d_cam_to_world = C - W^T Dw W^T, then d_look_at_matrix for a look-at camera."""
    h = Hook(rb, dev, name)
    c, rng = h.c, np.random.default_rng(seed)
    A = rng.normal(size=(n, 60)) * np.exp(rng.uniform(-3, 3, (n, 1)))
    A[1] = 0
    out, _ = h.run(L.RB_CAMTEST_FINISH, A)
    assert np.isfinite(out[:, :53]).all(), name
    W = c["w2c"]
    C = A[:, 0:16].reshape(-1, 4, 4) - np.einsum("ki,nkl,jl->nij", W, A[:, 16:32].reshape(-1, 4, 4), W)
    assert np.array_equal(out[:, 25:51], f32(A[:, 32:58])), name
    assert np.array_equal(out[:, 51:53], f32(A[:, 58:60]) if c["r"] > 0 else np.zeros((n, 2))), name
    if h.cam.cam_to_world is not None:
        Cf = C.reshape(-1, 16)
        assert_within(name + " d_cam_to_world", out[:, 9:25], Cf, np.abs(Cf) * 2.0 ** -23 + 1e-12 * np.abs(Cf).max(1, keepdims=True))
        assert (out[:, 0:9] == 0).all(), name
        return
    x = np.concatenate([h.cam.position.numpy(), h.cam.look_at.numpy(), h.cam.up.numpy()]).astype(np.float64)
    JM = R.jacobian(lambda v: look_at(v[0, 0:3], v[0, 3:6], v[0, 6:9]).reshape(1, 16), x[None])[0]  # [16, 9]
    Cr = f32(C.reshape(-1, 16))
    want = Cr @ JM
    mag = np.abs(Cr) @ np.abs(JM)
    assert_within(name + " d_look_at", out[:, 0:9], want, 4 * K * U * (mag + np.abs(want).max(1, keepdims=True)) + 1e-30)
    assert (out[:, 9:25] == 0).all() and (out[1, :] == 0).all(), name


# ---------------------------------------------------------------------------------------------------- the tests
@pytest.fixture(scope="module")
def rb():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from redner_b200 import redner
    return redner


DEV = torch.device("cuda:0")


@pytest.mark.parametrize("name", CAMERAS)
def test_rays_against_float64(rb, name):
    check_rays(rb, DEV, name)


@pytest.mark.parametrize("name", CAMERAS)
def test_projection_adjoint_against_float64(rb, name):
    check_project(rb, DEV, name)


@pytest.mark.parametrize("name", ["distort_persp", "distort_fish"])
def test_distortion_against_float64(rb, name):
    check_distort(rb, DEV, name)


@pytest.mark.parametrize("name", CAMERAS)
def test_ray_adjoint_against_float64(rb, name):
    check_ray_adjoint(rb, DEV, name)


@pytest.mark.parametrize("name", CAMERAS)
def test_finish_camera_against_float64(rb, name):
    check_finish(rb, DEV, name)


# ---------------------------------------------------------------------------------------------------- whole scenes
def singular_scene(dev, kind, res):
    """The glossy room seen by a fisheye camera aimed at a sphere vertex, a panorama camera with a sphere vertex straight below it (on its
    pole), or the distorted camera (kind 'distort', or 'plain' for the same camera without distortion)."""
    import scenes
    if kind in ("distort", "plain"):
        sc = scenes.glossy_room(dev, resolution=res, distortion=kind == "distort")
        return sc, [sc.camera.position, sc.camera.look_at, sc.camera.up] + ([sc.camera.distortion_params] if kind == "distort" else [])
    sc = scenes.glossy_room(dev, resolution=res, camera_type=2 if kind == "fisheye" else 3)
    v = sc.shapes[3].vertices.detach().cpu()[0]
    t = lambda x: torch.tensor(x, dtype=torch.float32, requires_grad=True)  # noqa: E731
    if kind == "fisheye":
        cam = api.Camera(position=t([0.4, 1.2, -1.6]), look_at=v.clone().requires_grad_(True), up=t([0.0, 1.0, 0.0]), clip_near=1e-2, resolution=res,
                         camera_type=2)
    else:
        p = v + torch.tensor([0.0, 1.0, 0.0])
        # (clip_near 0: the vertex lies at camera-space z = 0, which a positive clip_near would move off the pole)
        cam = api.Camera(position=p.clone().requires_grad_(True), look_at=(p + torch.tensor([0.0, 0.0, 1.0])).requires_grad_(True), up=t([0.0, 1.0, 0.0]),
                         clip_near=0.0, resolution=res, camera_type=3)
    sc.camera = cam
    return sc, [cam.position, cam.look_at, cam.up]


def render_grads(rb, dev, kind, res, deterministic):
    sc, cam_params = singular_scene(dev, kind, res)
    verts = sc.shapes[3].vertices
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic, warn_only=True)
    try:
        args = api.RenderFunction.serialize_scene(sc, 4, 1, device=dev, backend=rb, sample_pixel_center=kind in ("distort", "plain"),
                                                  use_primary_edge_sampling=True, use_secondary_edge_sampling=False)
        img = api.RenderFunction.apply(0, *args)
        (img * img).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    grads = [p.grad for p in cam_params + [verts]]
    return img.detach().cpu(), grads


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("kind", ["fisheye", "panorama", "distort"])
def test_singular_cameras_give_finite_gradients(rb, kind, deterministic):
    img, grads = render_grads(rb, DEV, kind, (25, 25), deterministic)
    assert torch.isfinite(img).all()
    for g in grads:
        assert g is not None and torch.isfinite(g).all(), (kind, g)
    if kind == "distort":
        # the distortion maps the centre to itself, so the centre pixel is the undistorted camera's centre pixel
        plain, _ = render_grads(rb, DEV, "plain", (25, 25), deterministic)
        assert torch.equal(img[12, 12], plain[12, 12]), (img[12, 12], plain[12, 12])
