"""GPU suite: ray/triangle solves, surface points, light-sample points and their adjoints (rb_shape.cuh) and the vertex-gradient scatters
(rb_path.cuh) through the test hook rb_surface_test, query by query, against the float64 restatement in tests/surface_ref.py; and the
backward pass of scenes with uv-degenerate triangles under a normal map and with flipped and zero-sum vertex normals.

Meshes (one native scene, built through api.Scene / api.Shape): a bare triangle (default uvs); a quad in z = 0 with uvs, vertex normals and
colours; a seamed mesh whose uv_indices and normal_indices differ from its indices; uv-degenerate triangles (all three uvs equal, two
equal corners at values whose products are not exact in float32, collinear uvs on a diagonal), without and with vertex normals opposite to
the winding; vertex normals opposite to the winding, nearly perpendicular to it, summing to exactly zero at an edge midpoint and to near
zero, and within 1e-7 ... 1e-2 rad of -z on both sides of coordinate_system's threshold; edges of 1e-4 and 1e3, and a mesh 10^3 from the
origin.

Query families: uniform hits, hits on the edges (u = 0, v = 0, u + v = 1) and on the vertices, grazing rays (|div| below the 1e-8 clamp
among them), axis-aligned planes; ray differentials zero, camera-like and random; light samples su, sv in {0, 1 - 2^-24, uniform}.

Comparison rules:
- forward outputs: within K u (sum_i |dy/dx_i| |x_i| + |y|), u = 2^-24, K = 64 as in the camera module (the longest chain, tri_solve's
  quotient derivatives through the normal's derivative, is about 30 float operations); the conditioning is measured by central
  differences of the restatement's inputs;
- the hit position equals fl(fl(dir t) + org) for the kernel's own float t, bit for bit;
- the uv determinant equals the restatement's bit for bit, so the det == 0 decision always matches; the other decisions (flip, degenerate
  fy, coordinate_system's branch) match wherever the margin says float32 rounding cannot flip them, and elsewhere either branch is accepted
  and counted;
- the hit position and dpdx / dpdy are sums whose terms cancel, and dn_dx / dn_dy a difference of two terms of size |dnn| / |nn|: their
  bound adds K u times the size of those terms;
- d_make_surface_point: within K u (sum_i |dg/dx_i| |x_i| + |A|^T |s| + |g|) + K_J E of the restatement as written (slips S1-S7), E the
  restatement's own rounding scale (rounding_scale), K_J = 16; the restatement without its slips equals the central-difference
  derivative wherever that is reliable, and so does the as-written one for every query no slip touches; every slip has a non-zero term;
- the light sample and area adjoints: within the same kind of bound of their true adjoint, a float64 restatement that itself matches
  central differences; the uv-of-sample adjoint's scatter matches the central-difference derivative;
- scatters: buffer sums within gamma_k of the per-query outputs mapped through uv_indices / normal_indices, bit-exact for exactly
  representable values at several lane patterns, untouched elements zero;
- zero seeds give exactly zero; every output is finite."""
import math

import numpy as np
import pytest
import torch

import surface_ref as R
from redner_b200 import api
from redner_b200 import _lib as L

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K = 64
K_J = 16
MESHES = ["bare", "attrs", "seamed", "uvdeg", "uvdeg_flip", "normals", "near_minus_z", "scale"]


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------------- meshes
def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def mesh_arrays():
    """name -> dict of numpy arrays (vertices, indices, and the optional uvs, normals, uv_indices, normal_indices, colors)."""
    rng = np.random.default_rng(7)
    M = {}
    M["bare"] = dict(vertices=[[-1.0, -0.5, 0.2], [1.2, -0.3, -0.1], [0.1, 1.1, 0.3]], indices=[[0, 1, 2]])
    quad = [[-1.0, -1.0, 0.0], [1.0, -1.0, 0.0], [-1.0, 1.0, 0.0], [1.0, 1.0, 0.0]]
    M["attrs"] = dict(vertices=quad, indices=[[0, 1, 2], [1, 3, 2]], uvs=[[0.0, 0.0], [1.0, 0.0], [0.0, 1.0], [1.0, 1.0]],
                      normals=_unit([[0.1, 0.2, -1.0], [-0.2, 0.1, -1.0], [0.0, -0.3, -1.0], [0.2, 0.2, -1.0]]),
                      colors=[[0.25, 0.5, 0.75], [1.0, 0.5, 0.25], [0.5, 0.5, 0.5], [0.75, 0.25, 1.0]])
    # a strip whose uv seam and normal seam split corners that share a position
    M["seamed"] = dict(vertices=[[0, 0, 0], [1, 0, 0.1], [0, 1, 0.2], [1, 1, 0.1], [2, 0.5, -0.1]], indices=[[0, 1, 2], [1, 3, 2], [1, 4, 3]],
                       uvs=[[0.1, 0.1], [0.9, 0.2], [0.2, 0.8], [0.7, 0.9], [0.0, 0.5], [0.4, 0.4]],
                       uv_indices=[[0, 1, 2], [4, 3, 2], [5, 4, 3]],
                       normals=_unit([[0.1, 0, 1], [0, 0.1, 1], [0.1, 0.1, 1], [-0.1, 0, 1], [0, -0.1, 1], [0.2, 0, 1], [0, 0.2, 1]]),
                       normal_indices=[[0, 1, 2], [3, 4, 5], [6, 3, 4]], colors=rng.random((5, 3)))
    # uv-degenerate triangles: all three equal, two equal corners (products not exact in float32), collinear on a diagonal
    two_eq = [(0.3, 0.7), (0.1, 0.9), (1 / 3, 0.2), (0.7, 0.3), (0.45, 0.55), (2 / 3, 1 / 7)]
    # ... and with the third corner non-zero and of another magnitude, so that the differences carry more than 26 bits and a fused
    # determinant leaves the residual of one product
    two_eq_off = [((0.3, 0.7), (0.01, 0.02)), ((0.45, 0.55), (0.001, 0.9)), ((0.7, 0.3), (3e-3, 1e-4)), ((1 / 3, 2 / 3), (0.9, 7e-3))]
    tris, uvs, verts = [], [], []
    def add(tv, tuv):  # noqa: E306
        b = len(verts)
        verts.extend(tv)
        uvs.extend(tuv)
        tris.append([b, b + 1, b + 2])
    for k in range(len(two_eq) + 2 + len(two_eq_off)):
        o = np.array([0.3 * k, 0.1 * k, 0.05 * k])
        tv = (o + np.array([[0.0, 0.0, 0.0], [1.0, 0.1, 0.2], [0.2, 1.0, -0.1]])).tolist()
        if k == 0:
            tuv = [[0.5, 0.5]] * 3
        elif k == 1:
            tuv = [[0.1, 0.1], [0.3, 0.3], [0.7, 0.7]]
        elif k < len(two_eq) + 2:
            a = list(two_eq[k - 2])
            tuv = [a, a, [0.0, 0.0]] if k % 2 == 0 else [[0.0, 0.0], a, a]
        else:
            a, c = (list(x) for x in two_eq_off[k - 2 - len(two_eq)])
            tuv = [a, a, c] if k % 2 == 0 else [c, a, a]
        add(tv, tuv)
    M["uvdeg"] = dict(vertices=verts, indices=tris, uvs=uvs)
    # the same, with vertex normals opposite to the winding (flip branch, and S5 on the det == 0 branch)
    V = np.array(verts)
    fn = np.array([-_unit(np.cross(V[t[1]] - V[t[0]], V[t[2]] - V[t[0]])) for t in tris])
    M["uvdeg_flip"] = dict(vertices=verts, indices=tris, uvs=uvs, normals=np.repeat(fn, 3, 0) + rng.normal(0, 0.05, (len(verts), 3)))
    # vertex normals: opposite, nearly perpendicular, summing to exactly zero at the edge midpoint, near zero
    base = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    nv, nn = [], []
    n0 = _unit([0.2, 0.3, 1.0])
    for k, ns in enumerate([[[0, 0, -1], [0.1, 0, -1], [0, 0.1, -1]],
                            [[1, 0, 1e-3], [0, 1, 1e-3], [-1, 0, 2e-3]],
                            [n0, -n0, [0.0, 0.0, 1.0]],
                            [[0, 0, 1], [0, 1e-3, -1], [0.5, 0.5, 0.2]]]):
        nv.extend((base + [2.0 * k, 0, 0]).tolist())
        nn.extend(ns)
    M["normals"] = dict(vertices=nv, indices=[[3 * k, 3 * k + 1, 3 * k + 2] for k in range(4)], normals=nn)
    # shading normals within 1e-7 ... 1e-2 rad of -z, each side of coordinate_system's n.z < -1 + 1e-6 (1.41e-3 rad)
    nv, nn = [], []
    for k, a in enumerate([1e-7, 1e-5, 1e-3, 1.5e-3, 1e-2]):
        nv.extend((base + [2.0 * k, 0, 0]).tolist())
        nrm = [math.sin(a), 0.0, -math.cos(a)]
        nn.extend([nrm, nrm, nrm])
    M["near_minus_z"] = dict(vertices=nv, indices=[[3 * k, 3 * k + 1, 3 * k + 2] for k in range(5)], normals=nn, uvs=[[0, 0], [1, 0], [0, 1]] * 5)
    M["scale"] = dict(vertices=(base * 1e-4).tolist() + (base * 1e3 + [0, 0, 5]).tolist() + (base + [1e3, -1e3, 1e3]).tolist(),
                      indices=[[0, 1, 2], [3, 4, 5], [6, 7, 8]])
    return M


class Hook:
    """One native scene holding every mesh of MESHES, its restatement blocks, and the hook."""

    def __init__(self, rb, dev):
        self.dev = dev
        self.M = mesh_arrays()
        shapes = []
        for name in MESHES:
            m = self.M[name]
            t = lambda k, dt=torch.float32: torch.tensor(np.asarray(m[k]), dtype=dt, device=dev).contiguous() if k in m else None  # noqa: E731
            shapes.append(api.Shape(t("vertices"), t("indices", torch.int32), 0, uvs=t("uvs"), normals=t("normals"), uv_indices=t("uv_indices", torch.int32),
                                    normal_indices=t("normal_indices", torch.int32), colors=t("colors")))
        cam = api.Camera(position=torch.tensor([0.0, 0.0, -5.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                         fov=torch.tensor([45.0]), clip_near=1e-2, resolution=(8, 8))
        self.shapes = shapes
        sc = api.Scene(cam, shapes, [api.Material(diffuse_reflectance=torch.tensor([0.5, 0.5, 0.5], device=dev))], [])
        args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev, backend=rb)
        self.ctx = api.RenderFunction._unpack([0], args)
        self.ctx.args = args

    def sid(self, name):
        return MESHES.index(name)

    def flags(self, name):
        m = self.M[name]
        return "normals" in m, "colors" in m, "uvs" in m

    def corners(self, name, tris):
        """The float32 corner values the kernel reads for triangles `tris`: the restatement's block T."""
        m = self.M[name]
        ind = np.asarray(m["indices"])[tris]
        g = lambda k, idx: f32(np.asarray(m[k], np.float64)[idx])  # noqa: E731
        T = {"v%d" % j: g("vertices", ind[:, j]) for j in range(3)}
        uvi = np.asarray(m["uv_indices"])[tris] if "uv_indices" in m else ind
        ni = np.asarray(m["normal_indices"])[tris] if "normal_indices" in m else ind
        dflt = [[0.0, 0.0], [1.0, 0.0], [1.0, 1.0]]
        for j in range(3):
            T["uv%d" % j] = g("uvs", uvi[:, j]) if "uvs" in m else np.tile(dflt[j], (len(tris), 1))
            T["n%d" % j] = g("normals", ni[:, j]) if "normals" in m else None
            T["c%d" % j] = g("colors", ind[:, j]) if "colors" in m else None
        return T

    def run(self, op, x, d_shapes=None):
        out = self.ctx.scene.surface_test(op, torch.from_numpy(np.asarray(x, np.float64)).to(self.dev), d_shapes)
        return out.cpu().numpy()


# ---------------------------------------------------------------------------------------------------- query families
def ray_queries(h, name, rng, n):
    """family -> (tris, X flat inputs [m, 51]) for mesh `name`: the rays and differentials are float32 values."""
    m = h.M[name]
    nt = len(m["indices"])
    fams = {}
    def make(tris, bary, dirs, rdk):  # noqa: E306
        T = h.corners(name, tris)
        b = np.asarray(bary)
        P = (1 - b[:, 0:1] - b[:, 1:2]) * T["v0"] + b[:, 0:1] * T["v1"] + b[:, 1:2] * T["v2"]
        scale = np.maximum(np.linalg.norm(T["v1"] - T["v0"], axis=1), np.linalg.norm(T["v2"] - T["v0"], axis=1))[:, None]
        d = f32(_unit(dirs))
        org = f32(P - d * 3 * scale)
        rd = np.zeros((len(tris), 12))
        if rdk == "camera":
            rd[:, 6:9] = f32(np.cross(d, [0.0, 1.0, 0.0]) * 1e-3)
            rd[:, 9:12] = f32(np.cross(d, [1.0, 0.0, 0.0]) * 1e-3)
        elif rdk == "random":
            rd = f32(rng.normal(0, 1e-2, (len(tris), 12)))
        return tris, R.pack(T, org, d, rd)
    def normal_dirs(tris, spread):  # noqa: E306
        T = h.corners(name, tris)
        g = _unit(np.cross(T["v1"] - T["v0"], T["v2"] - T["v0"]))
        sg = np.where(rng.random((len(tris), 1)) < 0.5, 1.0, -1.0)
        return -sg * g + rng.normal(0, spread, g.shape)
    tris = rng.integers(0, nt, n)
    b = rng.random((n, 2))
    b = np.where(b.sum(1, keepdims=True) > 1, 1 - b, b)
    for rdk in ("zero", "camera", "random"):
        fams["uniform_" + rdk] = make(tris, b, normal_dirs(tris, 0.4), rdk)
    te = np.repeat(np.arange(nt), 6)
    r = rng.random(len(te))
    eb = np.stack([np.select([np.arange(len(te)) % 6 == k for k in range(6)], [np.zeros_like(r), r, 1 - r, np.zeros_like(r), np.ones_like(r), np.zeros_like(r)]),
                   np.select([np.arange(len(te)) % 6 == k for k in range(6)], [r, np.zeros_like(r), r, np.zeros_like(r), np.zeros_like(r), np.ones_like(r)])], 1)
    fams["edges_vertices"] = make(te, eb, normal_dirs(te, 0.3), "camera")
    # grazing: the direction in the triangle's plane, tilted by 1e-2 ... 1e-9 (|div| below the 1e-8 clamp at the end)
    tg = np.repeat(np.arange(nt), 8)
    T = h.corners(name, tg)
    g = _unit(np.cross(T["v1"] - T["v0"], T["v2"] - T["v0"]))
    e = _unit(T["v1"] - T["v0"] + 0.3 * (T["v2"] - T["v0"]))
    tilt = 10.0 ** -np.tile(np.arange(2, 10), nt)[:, None]
    fams["grazing"] = make(tg, np.tile([[0.3, 0.3]], (len(tg), 1)), e - tilt * g, "camera")
    return fams


def seeds(rng, n, kind):
    if kind == "zero":
        return np.zeros((n, 47))
    if kind == "ones":
        return np.ones((n, 47))
    if kind == "random":
        return f32(rng.normal(size=(n, 47)))
    s = np.zeros((n, 47))
    fields = [(0, 3), (3, 6), (6, 9), (9, 12), (12, 15), (15, 18), (18, 20), (20, 22), (22, 24), (24, 27), (27, 30), (30, 33), (33, 35), (35, 47)]
    for i in range(n):
        a, b = fields[i % len(fields)]
        s[i, a:b] = f32(rng.normal(size=b - a))
    return s


# hook layout <-> flat inputs of surface_ref
def hook_rows(h, name, tris, X, seed=None):
    rows = np.zeros((len(X), 96))
    rows[:, 0] = h.sid(name)
    rows[:, 1] = tris
    rows[:, 2:20] = X[:, 33:51]
    if seed is not None:
        rows[:, 20:67] = seed
    return rows


def assert_within(what, got, want, tol, mask=None):
    err = np.abs(got - want)
    tol = np.broadcast_to(tol, err.shape)
    bad = ~(err <= tol)
    if mask is not None:
        bad &= mask[:, None]
    assert not bad.any(), "%s: %d bad, worst at %s: got %s want %s tol %s" % (what, bad.sum(), np.argwhere(bad)[:3].tolist(), got[bad][:4], want[bad][:4], tol[bad][:4])


def forward_all(X, has_n, has_c):
    out, dec = R.point(X, has_n, has_c)
    return np.concatenate([out, np.stack([dec["flip"], dec["fy"], dec["cs_gn"], dec["cs_sn"]], 1)], 1)


def conditioning(f, X, floor):
    J = R.central_jacobian(f, X, floor=floor, absolute=True)
    return np.abs(J * X[:, :, None]).sum(1), J


def input_floor(X):
    """The scale of each input of each query, the central-difference step being 1e-6 of it: positions (vertices, ray origin) at the size
    of the query's triangle, not at their distance from the origin (a unit triangle 10^3 away would otherwise be stepped by 1e-3 of its
    size); directions, uvs, normals and colours at 1; the ray differential at its largest component, at least 1e-3."""
    size = np.maximum(np.linalg.norm(X[:, 3:6] - X[:, 0:3], axis=1), np.linalg.norm(X[:, 6:9] - X[:, 0:3], axis=1))[:, None]
    floor = np.ones(X.shape)
    floor[:, 0:9] = size
    floor[:, 33:36] = size
    floor[:, 39:51] = np.maximum(np.abs(X[:, 39:51]).max(1, keepdims=True), 1e-3)
    return floor


# ---------------------------------------------------------------------------------------------------- checks
def check_point(rb, dev, name, n=48, seed=1, counts=None):
    h = Hook(rb, dev)
    has_n, has_c, _ = h.flags(name)
    rng = np.random.default_rng(seed)
    for fam, (tris, X) in ray_queries(h, name, rng, n).items():
        o = h.run(L.RB_SURFTEST_POINT, hook_rows(h, name, tris, X))
        assert np.isfinite(o[:, :62]).all(), (name, fam, np.argwhere(~np.isfinite(o[:, :62]))[:4])
        ref, dec = R.point(X, has_n, has_c)
        # the uv determinant: exact in double from the float uv corners, so bit for bit and the det == 0 branch always agrees
        assert (o[:, 61] == dec["det"]).all(), (name, fam, o[:, 61][o[:, 61] != dec["det"]][:4], dec["det"][o[:, 61] != dec["det"]][:4])
        assert (o[:, 56] == (dec["det"] == 0)).all(), (name, fam)
        # the hit position: fl(fl(dir t) + org) with the kernel's float t
        t = o[:, 2].astype(np.float32)
        org, d = X[:, 33:36].astype(np.float32), X[:, 36:39].astype(np.float32)
        assert (o[:, 9:12] == (d * t[:, None] + org).astype(np.float64)).all(), (name, fam)
        Y = forward_all(X, has_n, has_c)
        floor = input_floor(X)
        cond, _ = conditioning(lambda Z: forward_all(Z, has_n, has_c), X, floor)
        tol = K * U * (cond + np.abs(Y))
        # the hit position and dpdx / dpdy are sums whose terms cancel (org + dir t lies on the plane whatever org is): their rounding is
        # relative to the terms, not to the result
        org, d, rd, hs = X[:, 33:36], X[:, 36:39], X[:, 39:51], Y[:, 0:9]
        tol[:, 9:12] += K * U * (np.abs(org) + np.abs(d * hs[:, 2:3]))
        tol[:, 44:47] += K * U * (np.abs(rd[:, 0:3]) + np.abs(d * hs[:, 7:8]) + np.abs(rd[:, 6:9] * hs[:, 2:3]))
        tol[:, 47:50] += K * U * (np.abs(rd[:, 3:6]) + np.abs(d * hs[:, 8:9]) + np.abs(rd[:, 9:12] * hs[:, 2:3]))
        # the ray-differential outputs divide by div^2, and div = dot(pvec, e1) cancels on grazing rays: its relative rounding,
        # |pvec| |e1| / |div| u, enters them twice
        dxy = np.r_[3:9, 29:33, 33:39, 44:50]
        tol[:, dxy] += K * U * 2 * dec["div_cond"][:, None] * np.abs(Y[:, dxy])
        tol[:, 33:36] += K * U * 2 * dec["dn_scale"][:, 0:1]
        tol[:, 36:39] += K * U * 2 * dec["dn_scale"][:, 1:2]
        # decisions: must agree where the margin says float32 rounding cannot flip them
        want = R.decisions(dec, has_n)[:, 1:]
        got = o[:, 57:61]
        margin = np.stack([np.abs(Y[:, 56]) > tol[:, 56], np.abs(Y[:, 57]) > tol[:, 57], np.abs(Y[:, 58]) > tol[:, 58], np.abs(Y[:, 59]) > tol[:, 59]], 1)
        margin[:, 0] |= not has_n
        amb = ~margin
        assert ((got == want) | amb).all(), (name, fam, np.argwhere((got != want) & ~amb)[:4].tolist(), Y[:, 56:60][(got != want).any(1)][:3])
        if counts is not None:
            counts[(name, fam)] = int(amb.any(1).sum())
        same = (got == want).all(1) & ~dec["clamped"]
        # outputs 0-55: tri_solve, SurfacePoint, rd_out, on the queries whose decisions agree (elsewhere finiteness only)
        assert_within("%s/%s forward" % (name, fam), o[:, :56], Y[:, :56], tol[:, :56], same)


def hook_grad_to_flat(o):
    """d_make_surface_point's outputs in the hook's layout -> the gradient of surface_ref's 51 flat inputs."""
    G = np.zeros((len(o), R.NX))
    G[:, 0:9], G[:, 9:15], G[:, 15:24], G[:, 24:33] = o[:, 18:27], o[:, 36:42], o[:, 27:36], o[:, 42:51]
    G[:, 33:36], G[:, 36:39], G[:, 39:51] = o[:, 0:3], o[:, 3:6], o[:, 6:18]
    return G


JITTERED = ("dot", "cross", "normalize", "d_normalize", "d_cross", "coordinate_system", "d_coordinate_system")


def rounding_scale(f, rng, runs=8):
    """How far rounding inside `f` can move its result: the largest deviation of f over `runs` evaluations in which every vector
    primitive of surface_ref (dot, cross, normalize, their adjoints, coordinate_system) returns its value times (1 + 4u r), r uniform in
    [-1, 1].  It covers cancellation among intermediates (an adjoint term of size 1 / (1 + n.z)^2 near -z, removed again by a projection)
    that the conditioning in the inputs and seeds does not see."""
    clean = f()
    saved = {k: getattr(R, k) for k in JITTERED}
    jit = lambda v: tuple(jit(x) for x in v) if isinstance(v, tuple) else v * (1 + 4 * U * rng.uniform(-1, 1, np.shape(v)))  # noqa: E731
    dev = np.zeros_like(clean)
    try:
        for k in JITTERED:
            setattr(R, k, (lambda g: lambda *a: jit(g(*a)))(saved[k]))
        for _ in range(runs):
            dev = np.maximum(dev, np.abs(f() - clean))
    finally:
        for k, g in saved.items():
            setattr(R, k, g)
    return dev


def central_reliable(f, X, floor, rel=1e-6, skip=None):
    """Central differences of f at two step sizes; where they disagree by more than 1e-6 of the row's scale the difference quotient is not
    trusted (a branch within the step, the divisor clamp, a near-zero normal), and the row is reported unreliable.  `skip` [m, inputs]
    masks inputs that have no derivative (their rows of the Jacobian are zeroed)."""
    J1 = R.central_jacobian(f, X, rel=rel, floor=floor, absolute=True)
    J2 = R.central_jacobian(f, X, rel=rel * 10, floor=floor, absolute=True)
    if skip is not None:
        J1[skip], J2[skip] = 0, 0
    scale = np.abs(J1).reshape(len(X), -1).max(1)
    ok = (np.abs(J1 - J2).reshape(len(X), -1).max(1) <= 1e-6 * scale + 1e-12) & np.isfinite(J1).reshape(len(X), -1).all(1)
    return J1, ok


def check_adjoint(rb, dev, name, n=24, seed=2, slip_terms=None, counts=None):
    """d_make_surface_point against the restatement as written (slips S1-S6 included), within
    K u (sum_i |dg/dx_i| |x_i| + |A|^T |s| + |g|) + K_J E, E the rounding scale of the restatement (rounding_scale); the restatement
    without its slips against central differences of the forward wherever those are reliable, and the restatement as written there too
    wherever no slip term is non-zero; finite outputs; zero seeds exactly zero."""
    h = Hook(rb, dev)
    has_n, has_c, has_uv = h.flags(name)
    rng = np.random.default_rng(seed)
    for fam, (tris, X) in ray_queries(h, name, rng, n).items():
        _, dec = R.point(X, has_n, has_c)
        floor = input_floor(X)
        # (the uv inputs of a degenerate uv triangle have no derivative: any perturbation changes the dpdu branch)
        skip = np.zeros(X.shape, bool)
        skip[dec["det"] == 0, 9:15] = True
        J, reliable = central_reliable(lambda Z: R.point(Z, has_n, has_c)[0][:, 9:56], X, floor, skip=skip)
        reliable &= ~dec["clamped"]
        if fam == "grazing":  # (|div| down to the clamp: difference quotients of 1 / div^2 terms are not trustworthy at any step)
            reliable[:] = False
        units = [R.point_adjoint(X, has_n, has_c, np.eye(47)[[j] * len(X)]) for j in range(47)]
        for kind in ("onehot", "ones", "random", "zero"):
            S = seeds(rng, len(X), kind)
            o = h.run(L.RB_SURFTEST_D_POINT, hook_rows(h, name, tris, X, S))
            assert np.isfinite(o[:, :51]).all(), (name, fam, kind, np.argwhere(~np.isfinite(o[:, :51]))[:4].tolist())
            if kind == "zero":
                assert (o[:, :51] == 0).all(), (name, fam)
                continue
            got = hook_grad_to_flat(o)
            want = R.point_adjoint(X, has_n, has_c, S)
            AS = sum(np.abs(units[j]) * np.abs(S[:, j:j + 1]) for j in range(47))
            condg = np.abs(R.central_jacobian(lambda Z: R.point_adjoint(Z, has_n, has_c, S), X, floor=floor, absolute=True) * X[:, :, None]).sum(1)
            E = rounding_scale(lambda: R.point_adjoint(X, has_n, has_c, S), rng)
            if not has_uv:  # (the kernel adds no uv gradient to a shape without uvs)
                want[:, 9:15] = AS[:, 9:15] = condg[:, 9:15] = E[:, 9:15] = 0
            tol = K * U * (condg + AS + np.abs(want)) + K_J * E
            fin = np.isfinite(tol).all(1)
            assert_within("%s/%s/%s adjoint vs as-written" % (name, fam, kind), got, want, np.where(np.isfinite(tol), tol, np.inf), fin)
            # the true derivative; the uv columns of a degenerate uv triangle have none (the dpdu branch changes under any perturbation)
            true = np.einsum("mij,mj->mi", J, S)
            off = R.point_adjoint(X, has_n, has_c, S, slips=())
            if not has_uv:
                true[:, 9:15] = off[:, 9:15] = 0
            true[dec["det"] == 0, 9:15] = off[dec["det"] == 0, 9:15]
            scale = np.einsum("mij,mj->mi", np.abs(J), np.abs(S)).max(1, keepdims=True)
            assert_within("%s/%s/%s restatement without slips vs central differences" % (name, fam, kind), off, true, 1e-5 * scale + 1e-12, reliable)
            untouched = (np.abs(want - off).max(1) == 0) & reliable
            assert_within("%s/%s/%s as written, no slip touched, vs central differences" % (name, fam, kind), want, true, 1e-5 * scale + 1e-12, untouched)
            if counts is not None:
                counts[(name, fam, kind)] = (int(reliable.sum()), int(untouched.sum()), len(X))
            if slip_terms is not None:
                for sl in R.SLIPS:
                    term = want - R.point_adjoint(X, has_n, has_c, S, slips=tuple(x for x in R.SLIPS if x != sl))
                    slip_terms[sl] = max(slip_terms.get(sl, 0.0), float(np.abs(term).max()))


def light_queries(h, name, rng, n):
    nt = len(h.M[name]["indices"])
    e = 1 - 2.0 ** -24
    grid = np.array([[a, b] for a in (0.0, e) for b in (0.0, e)])
    tris = np.concatenate([rng.integers(0, nt, n), np.repeat(np.arange(nt), 4)])
    s = np.concatenate([f32(rng.random((n, 2))), np.tile(grid, (nt, 1))])
    T = h.corners(name, tris)
    V = np.concatenate([T["v0"], T["v1"], T["v2"]], 1)
    UV = np.concatenate([T["uv0"], T["uv1"], T["uv2"]], 1)
    return tris, V, UV, s


def check_light(rb, dev, name, n=32, seed=3):
    h = Hook(rb, dev)
    rng = np.random.default_rng(seed)
    tris, V, UV, s = light_queries(h, name, rng, n)
    rows = np.zeros((len(tris), 96))
    rows[:, 0], rows[:, 1], rows[:, 2:4] = h.sid(name), tris, s
    o = h.run(L.RB_SURFTEST_LIGHT, rows)
    assert np.isfinite(o[:, :22]).all()
    X = np.concatenate([V, UV, s], 1)
    f = lambda Z: R.light(Z[:, 0:9], Z[:, 9:15], Z[:, 15:17])  # noqa: E731
    Y = f(X)
    size = np.maximum(np.linalg.norm(V[:, 3:6] - V[:, 0:3], axis=1), np.linalg.norm(V[:, 6:9] - V[:, 0:3], axis=1))[:, None]
    floor = np.concatenate([np.repeat(size, 9, 1), np.ones((len(V), 8))], 1)
    J = R.central_jacobian(f, X, floor=floor, nonneg=np.arange(15, 17), absolute=True)
    tol = K * U * (np.abs(J * X[:, :, None]).sum(1) + np.abs(Y))
    assert_within("%s light forward" % name, o[:, :22], Y, tol)
    # adjoints: against the true adjoint (light_adjoint, itself checked against central differences), within
    # K u (|A|^T |s| + sum_i |dg/dx_i| |x_i| + |g|) + K_J E
    for kind in ("random", "ones", "zero"):
        S = np.zeros((len(tris), 18)) if kind == "zero" else (np.ones((len(tris), 18)) if kind == "ones" else f32(rng.normal(size=(len(tris), 18))))
        rows2 = rows.copy()
        rows2[:, 4:22] = S
        o2 = h.run(L.RB_SURFTEST_D_LIGHT, rows2)
        assert np.isfinite(o2[:, :18]).all(), (name, kind)
        if kind == "zero":
            assert (o2[:, :18] == 0).all(), name
            continue
        g = lambda VV: np.concatenate(R.light_adjoint(VV, s, S[:, :16]), 1)  # noqa: E731
        want = g(V)
        seed_out = np.zeros((len(tris), 22))
        seed_out[:, 0:15], seed_out[:, 21] = S[:, 0:15], S[:, 15]
        true = np.concatenate([np.einsum("mij,mj->mi", J[:, 0:9, :], seed_out * (np.arange(22) < 15)),
                               np.einsum("mij,mj->mi", J[:, 0:9, :], seed_out * (np.arange(22) == 21))], 1)
        Jr, reliable = central_reliable(f, X, floor)  # (rows with a sample at 0 step outside the square root's domain: unreliable)
        sc = np.abs(want).max(1, keepdims=True)
        assert_within("%s light adjoint restatement vs central differences" % name, want, true, 1e-5 * sc + 1e-12, reliable)
        units = [np.concatenate(R.light_adjoint(V, s, np.eye(16)[[j] * len(V)]), 1) for j in range(16)]
        AS = sum(np.abs(units[j]) * np.abs(S[:, j:j + 1]) for j in range(16))
        # (the samples are inputs too: b1 = 1 - sqrt(su) near su = 1 carries the rounding of the float square root ~1e7-fold)
        gs = lambda Z: np.concatenate(R.light_adjoint(Z[:, :9], Z[:, 9:11], S[:, :16]), 1)  # noqa: E731
        Vs = np.concatenate([V, s], 1)
        condg = np.abs(R.central_jacobian(gs, Vs, floor=np.concatenate([floor[..., :9], np.ones(floor.shape[:-1] + (2,))], -1), nonneg=(9, 10), absolute=True) * Vs[:, :, None]).sum(1)
        E = rounding_scale(lambda: g(V), rng)
        assert_within("%s d_sample_light_triangle / d_shape_tri_area" % name, o2[:, :18], want, K * U * (AS + condg + np.abs(want)) + K_J * E)


def _dshapes(h, dev):
    out = []
    for name in MESHES:
        m = h.M[name]
        d = {}
        for k in ("vertices", "uvs", "normals", "colors"):
            if k in m:
                d[k] = torch.zeros(np.asarray(m[k]).shape, dtype=torch.float32, device=dev)
        out.append(d)
    return out


def check_scatter(rb, dev, seed=4):
    """scatter_vertex_grads and d_light_sample_uv into real gradient buffers."""
    h = Hook(rb, dev)
    rng = np.random.default_rng(seed)
    # 1. exactly representable values: dyadic hits on the axis-aligned quad with colours and uvs, seeded on colour and uv only, so that
    #    every per-query output is a short dyadic and any summation order gives the same float; several lane patterns
    name = "attrs"
    pats = {"one_triangle": np.zeros(64, int), "alternating": np.arange(64) % 2, "halves": (np.arange(64) >= 32).astype(int),
            "random": rng.integers(0, 2, 64)}
    for pat, tris in pats.items():
        T = h.corners(name, tris)
        b = np.stack([rng.integers(1, 4, 64) / 8.0, rng.integers(1, 4, 64) / 8.0], 1)
        P = (1 - b[:, 0:1] - b[:, 1:2]) * T["v0"] + b[:, 0:1] * T["v1"] + b[:, 1:2] * T["v2"]
        d = np.tile([0.0, 0.0, 1.0], (64, 1))
        X = R.pack(T, P - d, d, np.zeros((64, 12)))
        S = np.zeros((64, 47))
        S[:, 30:33] = rng.integers(-8, 9, (64, 3)) / 4.0
        S[:, 18:20] = rng.integers(-8, 9, (64, 2)) / 4.0
        ds = _dshapes(h, dev)
        o = h.run(L.RB_SURFTEST_D_POINT, hook_rows(h, name, tris, X, S), ds)
        ind = np.asarray(h.M[name]["indices"])[tris]
        want_c = np.zeros((4, 3))
        want_uv = np.zeros((4, 2))
        for j in range(3):
            np.add.at(want_c, ind[:, j], o[:, 42 + 3 * j:45 + 3 * j])
            np.add.at(want_uv, ind[:, j], o[:, 36 + 2 * j:38 + 2 * j])
        assert (ds[h.sid(name)]["colors"].cpu().numpy() == want_c).all(), pat
        assert (ds[h.sid(name)]["uvs"].cpu().numpy() == want_uv).all(), pat
        for k, sname in enumerate(MESHES):
            if sname != name:
                assert all((v == 0).all() for v in ds[k].values()), (pat, sname)
    # 2. random seeds on the seamed mesh: buffer sums within gamma_k of the per-query outputs mapped through uv_indices / normal_indices
    name = "seamed"
    tris, X = ray_queries(h, name, rng, 96)["uniform_random"]
    S = seeds(rng, len(X), "random")
    ds = _dshapes(h, dev)
    o = h.run(L.RB_SURFTEST_D_POINT, hook_rows(h, name, tris, X, S), ds)
    m = h.M[name]
    maps = {"vertices": (np.asarray(m["indices"]), 18, 3), "normals": (np.asarray(m["normal_indices"]), 27, 3), "uvs": (np.asarray(m["uv_indices"]), 36, 2),
            "colors": (np.asarray(m["indices"]), 42, 3)}
    for k, (idx, col, w) in maps.items():
        ref = np.zeros(np.asarray(m[k]).shape)
        mag = np.zeros_like(ref)
        cnt = np.zeros(len(ref))
        for j in range(3):
            np.add.at(ref, idx[tris, j], o[:, col + w * j:col + w * (j + 1)])
            np.add.at(mag, idx[tris, j], np.abs(o[:, col + w * j:col + w * (j + 1)]))
            np.add.at(cnt, idx[tris, j], 1)
        got = ds[h.sid(name)][k].cpu().numpy()
        gam = (cnt * U / (1 - cnt * U))[:, None]
        assert (np.abs(got - ref) <= gam * mag).all(), (k, got, ref)
        assert (got[cnt == 0] == 0).all(), k
    # 3. d_light_sample_uv into the uv gradient of the seamed mesh
    tl, V, UV, s = light_queries(h, name, rng, 64)
    rows = np.zeros((len(tl), 96))
    rows[:, 0], rows[:, 1], rows[:, 2:4] = h.sid(name), tl, s
    duv = f32(rng.normal(size=(len(tl), 2)))
    rows[:, 20:22] = duv
    ds = _dshapes(h, dev)
    h.run(L.RB_SURFTEST_D_LIGHT, rows, ds)
    f = lambda Z: R.light(V, Z, s)[:, 19:21]  # noqa: E731
    J = R.central_jacobian(f, UV, floor=np.ones(6))  # [m, 6, 2], linear in UV
    per = np.einsum("mij,mj->mi", J, duv)
    ui = np.asarray(m["uv_indices"])
    ref = np.zeros((len(m["uvs"]), 2))
    mag = np.zeros_like(ref)
    cnt = np.zeros(len(ref))
    for j in range(3):
        np.add.at(ref, ui[tl, j], per[:, 2 * j:2 * j + 2])
        np.add.at(mag, ui[tl, j], np.abs(per[:, 2 * j:2 * j + 2]))
        np.add.at(cnt, ui[tl, j], 1)
    got = ds[h.sid(name)]["uvs"].cpu().numpy()
    assert (np.abs(got - ref) <= (cnt[:, None] * 8 * U) * mag + 1e-12).all(), (got, ref)
    assert (got[cnt == 0] == 0).all()


def check_errors(rb, dev):
    h = Hook(rb, dev)
    row = np.zeros((1, 96))
    for bad, msg in (((L.RB_SURFTEST_D_LIGHT + 1, row), "unknown op"), ((L.RB_SURFTEST_POINT, np.array([[len(MESHES)] + [0] * 95])), "shape out of range"),
                     ((L.RB_SURFTEST_POINT, np.array([[0, 1] + [0] * 94])), "triangle out of range"), ((L.RB_SURFTEST_POINT, np.array([[-1] + [0] * 95])), "shape out of range")):
        with pytest.raises(RuntimeError, match=msg):
            h.run(*bad)
    from redner_b200 import _lib
    assert h.ctx.scene._lib.rb_surface_test(h.ctx.scene._handle, 0, None, -1, None, None, None) != 0
    assert "negative" in _lib.last_error(h.ctx.scene._lib)


# ---------------------------------------------------------------------------------------------------- GPU tests
@pytest.fixture(scope="module")
def rb():
    from redner_b200 import redner
    return redner


DEV = torch.device("cuda:0")


@pytest.mark.parametrize("name", MESHES)
def test_point_against_float64(rb, name):
    check_point(rb, DEV, name)


@pytest.mark.parametrize("name", MESHES)
def test_adjoint_against_float64(rb, name):
    check_adjoint(rb, DEV, name)


def test_every_slip_is_exercised_and_the_suite_compares_enough(rb):
    terms, counts = {}, {}
    for name in MESHES:
        check_adjoint(rb, DEV, name, n=8, slip_terms=terms, counts=counts)
    assert all(terms.get(sl, 0) > 0 for sl in R.SLIPS), terms
    # central differences were reliable, and compared, on at least half of every mesh's queries outside the grazing family (which never
    # uses them)
    for name in MESHES:
        rel = sum(v[0] for k, v in counts.items() if k[0] == name and k[1] != "grazing")
        tot = sum(v[2] for k, v in counts.items() if k[0] == name and k[1] != "grazing")
        assert rel >= tot // 2, (name, rel, tot)


@pytest.mark.parametrize("name", MESHES)
def test_light_sample_against_float64(rb, name):
    check_light(rb, DEV, name)


def test_scatters(rb):
    check_scatter(rb, DEV)


def test_refusals(rb):
    check_errors(rb, DEV)


def singular_scene(dev, deterministic_grad=True):
    """uv-degenerate triangles (two equal corners) under a normal map, and a mesh with flipped and zero-sum vertex normals."""
    M = mesh_arrays()
    t = lambda x, dt=torch.float32: torch.tensor(np.asarray(x), dtype=dt, device=dev).contiguous()  # noqa: E731
    a = M["uvdeg"]
    V = np.asarray(a["vertices"]) * 0.6 + [-1.2, -0.8, 0.0]
    s0 = api.Shape(t(V).requires_grad_(), t(a["indices"], torch.int32), 0, uvs=t(a["uvs"]).requires_grad_())
    b = M["normals"]
    s1 = api.Shape(t(np.asarray(b["vertices"]) * 0.4 + [-1.0, 0.2, -0.3]).requires_grad_(), t(b["indices"], torch.int32), 0,
                   normals=t(b["normals"]).requires_grad_())
    light = api.Shape(t([[-1.0, -1.0, -7.0], [1.0, -1.0, -7.0], [-1.0, 1.0, -7.0], [1.0, 1.0, -7.0]]), t([[0, 1, 2], [1, 3, 2]], torch.int32), 0)
    nm = torch.rand(8, 8, 3, device=dev) * 0.4 + torch.tensor([0.3, 0.3, 0.6], device=dev)
    mat = api.Material(diffuse_reflectance=torch.tensor([0.6, 0.5, 0.4], device=dev, requires_grad=True),
                       normal_map=api.Texture(nm.requires_grad_(), torch.tensor([1.0, 1.0], device=dev)))
    cam = api.Camera(position=torch.tensor([0.0, 0.0, -5.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([45.0]), clip_near=1e-2, resolution=(48, 48))
    return api.Scene(cam, [s0, s1, light], [mat], [api.AreaLight(2, torch.tensor([20.0, 20.0, 20.0]))])


@pytest.mark.parametrize("deterministic", [False, True])
def test_singular_geometry_backward_is_finite(rb, deterministic):
    import parity_utils as pu
    torch.manual_seed(0)
    sc = singular_scene(DEV)
    args = api.RenderFunction.serialize_scene(sc, 4, 2, device=DEV, backend=rb)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic, warn_only=True)
    try:
        img = api.RenderFunction.apply(1, *args)
        img.pow(2).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.isfinite(img).all()
    grads = pu.collect_grads(sc)
    assert {"shape0.vertices", "shape0.uvs", "shape1.vertices", "shape1.normals"} <= set(grads), sorted(grads)
    for k, g in grads.items():
        assert torch.isfinite(g).all(), k
