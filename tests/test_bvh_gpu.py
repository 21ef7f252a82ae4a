"""GPU suite: the triangle LBVH (rb_build_bvh in rb_scene.cu) and its traversal (bvh_trace_impl in rb_bvh.cuh).

The BVH is an acceleration structure, so its answers have an exact oracle: the same triangle test on every triangle.  For every scene
below, built through api.Scene / redner.Scene:
- structure: T - 1 inner nodes and T leaf triangles; the walk from the root reaches every node and every leaf slot exactly once, at most
  63 levels deep; the leaves are a permutation of all (shape, triangle) pairs with the scene's coordinates bit for bit; an inner child's
  box is the min / max of that child's two boxes bit for bit; a leaf's box strictly contains its triangle with a bounded pad; two builds
  give the same bytes.
- queries (Scene.trace_rays, closest hit and any hit) from ten ray families: the traversal equals brute force over the leaf triangles
  (hit flag, triangle and t bit for bit); any-hit triangles really intersect the ray within (tnear, tfar] in float64; and on rays whose
  answer does not depend on rounding, a float64 closest hit computed with torch gives the same triangle and t to 1e-5.

Traversal and brute force may differ only in three ways, each counted per family, and all else fails:
- an exact tie: two triangles whose float64 distances agree to 1e-6 relative, with t at most 2 ulps apart (rays through a shared vertex
  or edge; the triangle test bounds Ts <= |den| * tfar as Embree does, so after a hit at t it still accepts a triangle whose rounded t
  is an ulp larger);
- the traversal returns the exact answer and brute force does not: the traversal's triangle is hit by the exact float64 test, and brute
  force's is missed by it or hit no closer (at grazing angles the triangle test's t can fall short of the exact t by more than the leaf
  box's pad);
- a hit only brute force finds on a triangle the exact float64 test misses and float32 cannot resolve: a zero-area triangle, or a ray
  whose origin float32 places no better than 1e-3 of the triangle's smallest height (at most 1 % of a family).
With tfar at a hit's own t (steep hits on triangles that are neither needles nor zero-area) the two modes must agree exactly.  Such a
ray can miss in both, because the triangle test compares Ts with |den| * tfar rather than its rounded t: the test counts those, and
with tfar 4 ulps larger both modes must hit.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: the module runs in about 18 s.  With tfar at the hit, 15 442 of
112 974 steep rays (14 %) miss in both modes and all hit 4 ulps above; no other lost hit occurs outside the zero-area slivers and the
63-level tree, whose unit triangles are seen from 4e6 away.  Each planted bug makes it fail: k_refit storing the left child's box for
both sides (30 of 33 tests), the traversal dropping the deferred sibling (13 query tests), leaf boxes without pad (24: every structure
test and 9 query tests).

The query checks are shared with tests/test_bvh_cpu.py, which runs them on the host build of the device headers (tools/cpu_emu) and
its median-split tree."""
import math

import numpy as np
import pytest
import torch

import scenes
from redner_b200 import api

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
STACK = 64  # RB_BVH_STACK


# ---------------------------------------------------------------------------------------------------- scenes
# Each generator returns a list of (vertices [V, 3] float32, indices [F, 3] int32) CPU tensors, one per shape.
def _shapes_of(sc):
    return [(s.vertices.detach().cpu().float().contiguous(), s.indices.cpu().int().contiguous()) for s in sc.shapes]


def _flat(shapes):
    """one shape of independent triangles [T, 3, 3] -> (vertices, indices)"""
    P = shapes.reshape(-1, 3).float().contiguous()
    return [(P, torch.arange(P.shape[0], dtype=torch.int32).reshape(-1, 3).contiguous())]


def _soup(n, seed=3):
    return _shapes_of(scenes.random_soup(torch.device("cpu"), num_tris=n, seed=seed))


def _transformed(shapes, scale=1.0, offset=(0.0, 0.0, 0.0)):
    return [((v * scale + torch.tensor(offset)).float().contiguous(), i) for v, i in shapes]


def _negative(shapes):
    """every coordinate <= 0: the soup moved so that its maximum is 0, those zeros and some others made -0.0"""
    hi = torch.stack([v.max(0).values for v, _ in shapes]).max(0).values
    g = torch.Generator().manual_seed(11)
    out = []
    for v, i in shapes:
        v = v - hi
        v = torch.where(v == 0, torch.full_like(v, -0.0), v)
        snap = torch.rand(v.shape, generator=g) < 0.05
        out.append((torch.where(snap, torch.full_like(v, -0.0), v).contiguous(), i))
    return out


def _ties():
    """5 000 copies of one triangle plus three others: every Morton key of the copies is equal"""
    one = torch.tensor([[0.1, 0.2, 0.3], [1.1, 0.25, 0.35], [0.4, 1.3, 0.2]])
    others = torch.tensor([[[-1.0, -1.0, 0.0], [1.0, -1.0, 0.1], [0.0, -0.5, 0.2]], [[2.0, 2.0, 2.0], [3.0, 2.0, 2.0], [2.0, 3.0, 2.5]],
                           [[0.3, 0.4, -1.0], [0.8, 0.4, -1.0], [0.5, 0.9, -1.2]]])
    return _flat(torch.cat([one.expand(5000, 3, 3), others]))


def _floor(n=256):
    """n x n quads at z = 0: zero extent on one axis"""
    s = torch.linspace(-2.0, 2.0, n + 1)
    y, x = torch.meshgrid(s, s, indexing="ij")
    v = torch.stack([x, y, torch.zeros_like(x)], -1).reshape(-1, 3).contiguous()
    a = (torch.arange(n)[:, None] * (n + 1) + torch.arange(n)[None, :]).reshape(-1)
    i = torch.cat([torch.stack([a, a + 1, a + n + 1], -1), torch.stack([a + 1, a + n + 2, a + n + 1], -1)]).int().contiguous()
    return [(v, i)]


def _slivers(n=1500, n_zero=250, seed=5):
    """slivers of aspect ratio 1e4 mixed with zero-area triangles (a repeated vertex; exactly collinear vertices)"""
    g = torch.Generator().manual_seed(seed)
    p = (torch.rand(n, 3, generator=g) - 0.5) * 4.0
    u = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1)
    w = torch.nn.functional.normalize(torch.cross(u, torch.randn(n, 3, generator=g), dim=1), dim=1)
    L = 0.2 + 0.6 * torch.rand(n, 1, generator=g)
    sl = torch.stack([p, p + L * u, p + 0.5 * L * u + (L / 1e4) * w], 1)
    a = torch.randint(-16, 16, (n_zero, 3), generator=g).float() / 8
    b = torch.randint(-16, 16, (n_zero, 3), generator=g).float() / 8
    rep = torch.stack([a, a, b], 1)
    s = torch.randint(1, 4, (n_zero, 3), generator=g).float() / 8
    col = torch.stack([a, a + s, a + 2 * s], 1)
    return _flat(torch.cat([sl, rep, col])[torch.randperm(n + 2 * n_zero, generator=g)])


def _multi_shape():
    """shapes of 1, 2 and many triangles, so that global_to_shape has to search"""
    P = _soup(1200, seed=9)[0]
    tris = P[0][P[1].long()]
    cuts = [1, 2, 500, 1, 2, 300, 1, 390]
    out, k = [], 0
    for c in cuts:
        out += _flat(tris[k:k + c])
        k += c
    return out


def _few(T):
    v, i = _soup(3, seed=4)[0]
    return [(v, i[:T].contiguous())]


def _depth_keys(duplicate=False):
    """Triangles whose Morton codes are 0, 1, 2, 4, ..., 2^62, under scene bounds of exactly [0, 2^21] per axis: a caterpillar radix tree of
    height 63 (RB_BVH_STACK - 1).  Bit 3j + 2 of a code is bit j of the x cell, 3j + 1 of y, 3j of z.  A cell q is reached with the vertex
    coordinates (q, q + 0.5, q + 1) (sum 3q + 1.5, centroid q + 0.5, all exact), rotated per axis so the triangle is not degenerate; the
    three triangles with a cell 2^20 use (0, 2^20 + 1.5, 2^21) on that axis, which also sets the bounds.  `duplicate`: one more triangle
    with code 0 (height 64)."""
    tris = []
    for b in [None] + list(range(63)) + ([None] if duplicate else []):
        q = [0, 0, 0]
        if b is not None:
            q[2 - b % 3] = 1 << (b // 3)
        tri = [[0.0] * 3 for _ in range(3)]
        for a in range(3):
            c = [0.0, q[a] + 1.5, 2.0 ** 21] if q[a] == 1 << 20 else [q[a], q[a] + 0.5, q[a] + 1.0]
            for k in range(3):
                tri[k][a] = float(c[(k + a) % 3])
        tris.append(tri)
    return _flat(torch.tensor(tris, dtype=torch.float32))


SCENES = {
    "teapot": lambda: _shapes_of(scenes.teapot_geometry(torch.device("cpu"), resolution=(8, 8), grad=False)),
    "bunny_box": lambda: _shapes_of(scenes.bunny_box_shifted(torch.device("cpu"), resolution=(8, 8), grad=False)),
    "hires_room": lambda: _shapes_of(scenes.hires_room(torch.device("cpu"), resolution=(8, 8), grad=False)),
    "soup_2000": lambda: _soup(2000),
    "soup_400000": lambda: _soup(400000),
    "morton_ties": _ties,
    "flat_floor": _floor,
    "soup_far": lambda: _transformed(_soup(2000), offset=(1e4, -1e4, 1e4)),
    "soup_small": lambda: _transformed(_soup(2000), scale=1e-3),
    "soup_negative": lambda: _negative(_soup(2000)),
    "slivers": _slivers,
    "one_triangle": lambda: _few(1),
    "two_triangles": lambda: _few(2),
    "three_triangles": lambda: _few(3),
    "multi_shape": _multi_shape,
    "depth_63": _depth_keys,
}


def make_scene(shapes, dev, rb):
    """The native scene of `shapes` (one material, no light, no edge sampling) -> (redner.Scene, shapes on `dev`)"""
    shapes = [(v.to(dev), i.to(dev)) for v, i in shapes]
    cam = api.Camera(position=torch.tensor([0.0, 0.0, -10.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([45.0]), clip_near=1e-2, resolution=(8, 8))
    sc = api.Scene(cam, [api.Shape(v, i, 0) for v, i in shapes], [api.Material(diffuse_reflectance=torch.tensor([0.5, 0.5, 0.5], device=dev))], [])
    args = api.RenderFunction.serialize_scene(sc, 1, 1, use_primary_edge_sampling=False, use_secondary_edge_sampling=False, device=dev, backend=rb)
    c = api.RenderFunction._unpack((1, 2), args)
    c.scene._keep = args  # (the native scene holds raw pointers into these)
    return c.scene, shapes


# ---------------------------------------------------------------------------------------------------- rays
def _unit(x):
    return x / x.norm(dim=-1, keepdim=True).clamp_min(1e-30)


def _rays(o, d, tnear=0.0, tfar=math.inf):
    n = o.shape[0]
    tn = torch.as_tensor(tnear, dtype=torch.float32, device=o.device).expand(n)
    tf = torch.as_tensor(tfar, dtype=torch.float32, device=o.device).expand(n)
    return torch.cat([o.float(), tn[:, None], d.float(), tf[:, None]], 1).contiguous()


class Geometry:
    """The scene's triangles in shape order, float32 [T, 3, 3], with their (shape, triangle) ids and bounds."""

    def __init__(self, shapes):
        self.P = torch.cat([v[i.long()] for v, i in shapes])
        self.offsets = [0]
        for _, i in shapes:
            self.offsets.append(self.offsets[-1] + i.shape[0])
        self.T = self.P.shape[0]
        flat = self.P.reshape(-1, 3)
        self.lo, self.hi = flat.min(0).values, flat.max(0).values
        self.center = 0.5 * (self.lo + self.hi)
        self.radius = float((self.hi - self.lo).norm().clamp_min(1e-6))
        self.magnitude = float(flat.abs().max())
        _, self.hmin, self.vmax = _triangle_tolerance(self.P.double())
        P = self.P.double()
        self.area2 = torch.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0], dim=1).norm(dim=1)
        # whether float32 resolves the typical triangle from rays starting outside the bounds (not so for unit triangles 1e6 away)
        self.resolvable = 3e-6 * (self.magnitude + 1.5 * self.radius) < 1e-2 * float(self.hmin.median())

    def index(self, ids):
        """(shape, triangle) -> index into P"""
        off = torch.tensor(self.offsets[:-1], device=ids.device, dtype=torch.int64)
        return off[ids[:, 0].long().clamp_min(0)] + ids[:, 1].long()


def primary_families(geo, n, n_aim, gen):
    """the ray families that do not depend on a query: {name: [N, 8] rays}"""
    dev, lo, hi = geo.P.device, geo.lo, geo.hi

    def uniform(k):
        return lo + (hi - lo) * torch.rand(k, 3, generator=gen, device=dev)

    def outside(k):
        return geo.center + 1.5 * geo.radius * _unit(torch.randn(k, 3, generator=gen, device=dev))
    fam = {}
    o = outside(n)
    fam["outside"] = _rays(o, _unit(uniform(n) - o))
    grow = 0.05 * geo.radius  # (so that the origins of a flat scene are not all in its plane)
    fam["inside"] = _rays(lo - grow + (hi - lo + 2 * grow) * torch.rand(n, 3, generator=gen, device=dev), _unit(torch.randn(n, 3, generator=gen, device=dev)))
    # every triangle (from several origins when there are few), or a sample of n_aim / 7 of them
    if 7 * geo.T <= n_aim:
        sel = torch.arange(geo.T, device=dev).repeat(min(16, n_aim // (7 * geo.T)))
    else:
        sel = torch.randperm(geo.T, generator=gen, device=dev)[:n_aim // 7]
    P = geo.P[sel]
    tg = torch.cat([P.mean(1), P[:, 0], P[:, 1], P[:, 2], 0.5 * (P[:, 0] + P[:, 1]), 0.5 * (P[:, 1] + P[:, 2]), 0.5 * (P[:, 2] + P[:, 0])])
    o = outside(tg.shape[0])
    fam["aimed"] = _rays(o, _unit(tg - o))
    # axis-parallel, with exact +-0.0 in the other components; half of them through triangle centroids
    axis = torch.randint(0, 3, (n,), generator=gen, device=dev)
    sign = torch.where(torch.rand(n, generator=gen, device=dev) < 0.5, -1.0, 1.0)
    d = torch.zeros(n, 3, device=dev)
    d[torch.arange(n, device=dev), axis] = sign
    d = torch.where((d == 0) & (torch.rand(n, 3, generator=gen, device=dev) < 0.5), torch.full_like(d, -0.0), d)
    o = uniform(n)
    half = n // 2
    o[:half] = geo.P[torch.randint(0, geo.T, (half,), generator=gen, device=dev)].mean(1)
    start = torch.where(sign > 0, lo[axis] - 0.25 * geo.radius, hi[axis] + 0.25 * geo.radius)
    o[torch.arange(n, device=dev), axis] = start
    fam["axis_parallel"] = _rays(o, d)
    # zero and tiny directions: |d| = 0 (+0.0 or -0.0), 1e-20, 1e-2 (|d|^2 below the 1e-3 cut-off: no hit), and 0.1 (above it)
    k = n // 5
    u = _unit(torch.randn(5 * k, 3, generator=gen, device=dev))
    scale = torch.tensor([0.0, -0.0, 1e-20, 1e-2, 0.1], device=dev).repeat_interleave(k)[:, None]
    o = outside(5 * k)
    aim = _unit(uniform(5 * k) - o)
    d = torch.where(scale == 0, scale * u, scale * aim)
    fam["tiny_direction"] = _rays(o, d)
    o = outside(n)
    tnear = geo.radius * (0.5 + 2.0 * torch.rand(n, generator=gen, device=dev))
    fam["tnear_above_tfar"] = _rays(o, _unit(uniform(n) - o), tnear, tnear * 0.999)
    return fam


def derived_families(geo, fam, first, gen):
    """families built from brute-force closest hits `first` of fam["outside"] + fam["aimed"]: {name: rays}"""
    dev = geo.P.device
    rays = torch.cat([fam["outside"], fam["aimed"]])
    ids, t = first
    hit = ids[:, 0] >= 0
    rays, t, ids = rays[hit], t[hit], ids[hit]
    out = {}
    o, d = rays[:, :3], rays[:, 4:7]
    # tfar equal to the hit distance (inclusive), and one float below it.  Only for hits at least 30 degrees off the plane of a triangle
    # that is not a needle (aspect ratio up to 100) and has an area: at a grazing angle, and on a needle whose float32 plane is tilted by
    # rounding, the triangle test's t is less accurate than the leaf box's pad, so with tfar at that t the box may end short of it.
    hit_idx = geo.index(ids)
    Q = geo.P[hit_idx].double()
    nrm = torch.cross(Q[:, 1] - Q[:, 0], Q[:, 2] - Q[:, 0], dim=1)
    steep = (nrm * d.double()).sum(1).abs() >= 0.5 * nrm.norm(dim=1) * d.double().norm(dim=1)
    tol_tri, _, _ = _triangle_tolerance(geo.P.double())
    steep &= (nrm.norm(dim=1) > 0) & (tol_tri[hit_idx] <= 1e-3)
    if bool(steep.any()):  # (none on a scene of needles and zero-area triangles only)
        out["tfar_at_hit"] = torch.cat([o, rays[:, 3:4], d, t[:, None]], 1)[steep]
        out["tfar_below_hit"] = torch.cat([o, rays[:, 3:4], d, torch.nextafter(t, torch.zeros_like(t))[:, None]], 1)[steep]
    # secondary rays from the hit points with the renderer's tnear: random directions, and towards a point of another triangle with
    # tfar just short of it (shadow rays)
    p = o + t[:, None] * d
    n = p.shape[0]
    out["secondary"] = _rays(p, _unit(torch.randn(n, 3, generator=gen, device=dev)), 1e-4)
    other = torch.randint(0, geo.T, (n,), generator=gen, device=dev)
    same = other == geo.index(ids)
    other = torch.where(same, (other + 1) % geo.T, other)
    w = torch.rand(n, 3, generator=gen, device=dev)
    w = w / w.sum(1, keepdim=True)
    q = (w[:, :, None] * geo.P[other]).sum(1)
    dist = (q - p).norm(dim=1)
    ok = dist > 0
    out["shadow"] = _rays(p[ok], _unit(q - p)[ok], 1e-4, (dist * (1 - 1e-4))[ok])
    return out


# ---------------------------------------------------------------------------------------------------- float64
def _f64_pairs(o, d, P):
    """Moeller-Trumbore in float64 for every (ray, triangle) pair: t, barycentric margin, |cos| [R, C]"""
    v0, v1, v2 = P[:, 0][None], P[:, 1][None], P[:, 2][None]
    e1, e2 = v1 - v0, v2 - v0
    o, d = o[:, None], d[:, None]
    pv = torch.cross(d.expand(-1, P.shape[0], -1), e2.expand(o.shape[0], -1, -1), dim=2)
    det = (e1 * pv).sum(2)
    s = o - v0
    qv = torch.cross(s, e1.expand(o.shape[0], -1, -1), dim=2)
    inv = 1.0 / torch.where(det == 0, torch.ones_like(det), det)
    u = (s * pv).sum(2) * inv
    v = (d * qv).sum(2) * inv
    t = (e2 * qv).sum(2) * inv
    margin = torch.minimum(torch.minimum(u, v), 1 - u - v)
    nrm = torch.cross(e1, e2, dim=2)
    cos = det.abs() / (nrm.norm(dim=2) * d.norm(dim=2)).clamp_min(1e-300)
    degenerate = nrm.norm(dim=2) == 0
    margin = torch.where((det == 0) | degenerate, torch.full_like(margin, -math.inf), margin)
    return t, margin, cos


def _triangle_tolerance(P):
    """per triangle: the barycentric margin within which float32 may decide either way by its own shape (1e-4, more for needles), its
    smallest height, and its largest coordinate"""
    e = torch.stack([P[:, 1] - P[:, 0], P[:, 2] - P[:, 1], P[:, 0] - P[:, 2]], 1)
    area2 = torch.cross(e[:, 0], e[:, 1], dim=1).norm(dim=1)
    longest = e.norm(dim=2).max(1).values
    aspect = longest ** 2 / area2.clamp_min(1e-300)
    return 1e-4 * torch.clamp(aspect / 10.0, min=1.0), area2 / longest.clamp_min(1e-300), P.abs().amax((1, 2))


def _line_distance(o, d, c):
    """distance of the points c [C, 3] from the lines o + s d [R, 3] -> [R, C]"""
    u = _unit(d)[:, None]
    w = c[None] - o[:, None]
    return torch.cross(w, u.expand_as(w), dim=2).norm(dim=2)


def f64_closest(geo, rays, chunk=2048):
    """Closest hit in float64 over all triangles, and whether the answer depends on rounding.  Returns (index of the closest hit or -1,
    its t, robust [R] bool, the uncertainty of that t).

    float32 places the ray and the triangle to within about 1e-7 of their coordinates' magnitude; `pos` allows ten times that.  A
    triangle is a candidate when float32 could call it a hit: barycentric margin above -tol (1e-4, more for needles, plus pos over the
    triangle's smallest height seen at the ray's angle) and t within (tnear, tfar] up to ut (4 pos seen at the ray's angle to the
    plane, plus 1e-5 of t).  A ray is robust when it has no candidate at all (a miss), or when its closest hit has a margin above
    tol and 1e-4, is not parallel to the plane, is clear of tnear and tfar by ut, and every other candidate is behind it by more than
    both uncertainties."""
    R = rays.shape[0]
    dev = rays.device
    o, d = rays[:, :3].double(), rays[:, 4:7].double()
    tnear, tfar = rays[:, 3].double()[:, None], rays[:, 7].double()[:, None]
    dn = d.norm(dim=1)
    P = geo.P.double()
    tol_all, hmin, vmax = _triangle_tolerance(P)
    omax = o.abs().max(1).values
    flat_all = torch.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0], dim=1).norm(dim=1) == 0
    cc = P.mean(1)
    rr = (P - cc[:, None]).norm(dim=2).max(1).values
    inf = math.inf
    best_t = torch.full((R,), inf, dtype=torch.float64, device=dev)
    best_i = torch.full((R,), -1, dtype=torch.int64, device=dev)
    best_m, best_c, best_u = (torch.zeros(R, dtype=torch.float64, device=dev) for _ in range(3))
    # the two smallest (t - ut) over candidates, and the triangle of the smallest
    k1 = torch.full((R,), inf, dtype=torch.float64, device=dev)
    k2 = torch.full((R,), inf, dtype=torch.float64, device=dev)
    i1 = torch.full((R,), -1, dtype=torch.int64, device=dev)
    for k in range(0, geo.T, chunk):
        t, m, c = _f64_pairs(o, d, P[k:k + chunk])
        pos = 1e-6 * (omax[:, None] + vmax[None, k:k + chunk])
        tol = tol_all[None, k:k + chunk] + pos / (hmin[None, k:k + chunk] * c).clamp_min(1e-300)
        # (a needle's plane is inexact in float32 by an angle of about 1e-2 tol: that moves its hit by that much of its distance)
        needle = 1e-2 * tol_all[None, k:k + chunk] * (P[None, k:k + chunk, 0] - o[:, None]).norm(dim=2)
        ut = (4 * pos + needle) / (c * dn[:, None]).clamp_min(1e-300) + (1e-5 + 1e-2 * tol_all[None, k:k + chunk]) * t.abs()
        cand = (m >= -tol) & (t + ut > tnear) & (t - ut <= tfar)
        # zero-area triangles: float32 evaluates their edges relative to the ray's origin and may call one hit; float64 cannot say, so
        # one near the ray is a candidate
        flat = flat_all[None, k:k + chunk] & (_line_distance(o, d, cc[k:k + chunk]) <= rr[None, k:k + chunk] + 1e-3 * geo.radius)
        cand = cand | flat
        valid = (m >= 0) & (t > tnear) & (t <= tfar)
        key = torch.where(cand, torch.where(flat, -inf, t - ut), torch.full_like(t, inf))
        tv = torch.where(valid, t, torch.full_like(t, inf))
        if key.shape[1] >= 2:
            kv, ki = key.topk(2, dim=1, largest=False)
        else:
            kv = torch.cat([key, torch.full_like(key, inf)], 1)
            ki = torch.zeros_like(kv, dtype=torch.int64)
        allv = torch.stack([k1, k2, kv[:, 0], kv[:, 1]], 1)
        alli = torch.stack([i1, i1, ki[:, 0] + k, ki[:, 1] + k], 1)
        sv, si = allv.sort(1)
        k1, k2, i1 = sv[:, 0], sv[:, 1], alli.gather(1, si[:, :1])[:, 0]
        j = tv.argmin(1)
        tj = tv.gather(1, j[:, None])[:, 0]
        better = tj < best_t
        pick = lambda x: x.gather(1, j[:, None])[:, 0]  # noqa: E731
        best_m = torch.where(better, pick(m) - pick(tol.expand_as(m)), best_m)
        best_c = torch.where(better, pick(c), best_c)
        best_u = torch.where(better, pick(ut), best_u)
        best_i = torch.where(better, j + k, best_i)
        best_t = torch.where(better, tj, best_t)
    hit = best_i >= 0
    tnear, tfar = tnear[:, 0], tfar[:, 0]
    clear = (i1 == best_i) & (k2 > best_t + best_u) & (best_m > 1e-4) & (best_c > 1e-3)
    clear = clear & (best_t - best_u > tnear) & (best_t + best_u < tfar)
    robust = torch.where(hit, clear, k1 == inf)
    # the traversal's early-outs: an empty (tnear, tfar], or |d|^2 <= 1e-3 (a zero / degenerate direction) never hits
    empty = (tfar < tnear) | (dn * dn < 1e-3 * (1 - 1e-4))
    robust = torch.where(empty, True, robust & (dn * dn > 1e-3 * (1 + 1e-4)))
    best_i = torch.where(empty, -1, best_i)
    best_t = torch.where(empty, tfar, best_t)
    return best_i, best_t.float(), robust, best_u


def f64_hit_holds(geo, rays, idx, t32, strict=False):
    """The triangle `idx` of each ray intersects it within (tnear, tfar] in float64, up to float32's placement of the ray and the triangle
    (1e-6 of their coordinates' magnitude, as in f64_closest): barycentric margin above -tol, t within the interval up to ut, and the
    library's t equal to the float64 one up to ut.  This is loose: tol is at least 1e-4 in barycentric terms (0.1 for the 1e4 slivers,
    more seen at a grazing angle or from far away), ut at least 1e-5 of t, and a zero-area triangle always holds, since float64 has no
    intersection to compare with.  It checks that a reported hit is a real one, not the triangle test's last bits; `strict` is the exact
    float64 test without any tolerance."""
    o, d = rays[:, :3].double(), rays[:, 4:7].double()
    tnear, tfar = rays[:, 3].double(), rays[:, 7].double()
    tol_tri, hmin, vmax = _triangle_tolerance(geo.P.double())
    P = geo.P.double()[idx]
    v0, e1, e2 = P[:, 0], P[:, 1] - P[:, 0], P[:, 2] - P[:, 0]
    pv = torch.cross(d, e2, dim=1)
    det = (e1 * pv).sum(1)
    inv = 1.0 / torch.where(det == 0, torch.ones_like(det), det)
    sv = o - v0
    qv = torch.cross(sv, e1, dim=1)
    u, v, t = (sv * pv).sum(1) * inv, (d * qv).sum(1) * inv, (e2 * qv).sum(1) * inv
    margin = torch.minimum(torch.minimum(u, v), 1 - u - v)
    nrm = torch.cross(e1, e2, dim=1).norm(dim=1)
    dn = d.norm(dim=1)
    cos = det.abs() / (nrm * dn).clamp_min(1e-300)
    pos = 1e-6 * (o.abs().max(1).values + vmax[idx])
    tol = tol_tri[idx] + pos / (hmin[idx] * cos).clamp_min(1e-300)
    needle = 1e-2 * tol_tri[idx] * (v0 - o).norm(dim=1)
    ut = (4 * pos + needle) / (cos * dn).clamp_min(1e-300) + (1e-5 + 1e-2 * tol_tri[idx]) * t.abs()
    within = (t + ut > tnear) & (t - ut <= tfar) & ((t - t32.double()).abs() <= ut)
    if strict:  # (the exact float64 test, no tolerance)
        return (nrm > 0) & (margin >= 0) & (t > tnear) & (t <= tfar)
    flat = nrm == 0  # (a zero-area triangle: float64 has no intersection to compare with; see f64_closest)
    return flat | ((margin >= -tol) & within & (det != 0))


# ---------------------------------------------------------------------------------------------------- the query checks
def check_queries(name, scene, shapes, dev, n=4096, n_aim=14000, n_f64=512, seed=0):
    """Every query check on one scene; returns {family: {check: rays compared}} and asserts that no family compared nothing."""
    geo = Geometry(shapes)
    gen = torch.Generator(device=dev).manual_seed(seed)
    fam = primary_families(geo, n, n_aim, gen)
    first = scene.trace_rays(torch.cat([fam["outside"], fam["aimed"]]), brute_force=True)
    fam.update(derived_families(geo, fam, first, gen))
    tol_tri, _, _ = _triangle_tolerance(geo.P.double())
    if bool(((geo.area2 > 0) & (tol_tri <= 1e-3)).any()):
        assert "tfar_at_hit" in fam and "tfar_below_hit" in fam, name + ": no steep hit to set tfar at"
    report = {}
    for fname, rays in fam.items():
        counts = report.setdefault(fname, {})
        assert rays.shape[0] > 0, (name, fname)
        for any_hit in (False, True):
            ids, t = scene.trace_rays(rays, any_hit=any_hit)
            bids, bt = scene.trace_rays(rays, any_hit=any_hit, brute_force=True)
            hit, bhit = ids[:, 0] >= 0, bids[:, 0] >= 0
            mode = "any" if any_hit else "closest"
            # A hit only brute force finds is a lost triangle, unless the exact float64 test does not hit that triangle and float32 cannot
            # decide it either: a zero-area triangle, or a ray whose origin float32 places no better than 1e-3 of the triangle's smallest
            # height (unit triangles seen from 4e6 away).  Such rays are counted and may be at most 1 % of a family.
            only = (bhit & ~hit).nonzero()[:, 0]
            if only.numel():
                bi = geo.index(bids[only])
                pos = 1e-6 * (rays[only, :3].double().abs().max(1).values + geo.vmax[bi])
                unresolved = (geo.area2[bi] == 0) | (pos > 1e-3 * geo.hmin[bi])
                excused = unresolved & ~f64_hit_holds(geo, rays[only], bi, bt[only], strict=True)
                counts[mode + "_unresolved_hits_lost"] = int(excused.sum())
                assert int(excused.sum()) <= 0.01 * rays.shape[0], (name, fname, mode, int(excused.sum()), rays.shape[0])
                hit = hit.clone()
                hit[only[excused]] = True
                ids, t = ids.clone(), t.clone()
                ids[only[excused]], t[only[excused]] = bids[only[excused]], bt[only[excused]]
            bad = (hit != bhit).nonzero()[:, 0]
            assert bad.numel() == 0, "%s/%s any_hit=%d: %d rays hit in one mode only, e.g. ray %s traversal %s brute %s" % (
                name, fname, any_hit, bad.numel(), rays[bad[0]].tolist(), (ids[bad[0]].tolist(), float(t[bad[0]])), (bids[bad[0]].tolist(), float(bt[bad[0]])))
            counts[mode + "_flag"] = rays.shape[0]
            if not any_hit:
                # The same triangle and t bit for bit, except
                # - an exact tie: two triangles whose float64 distances agree to 1e-6 relative, with t at most 2 ulps apart (rays through a
                #   shared vertex or edge; after a hit at t the triangle test, bounding Ts <= |den| * tfar as Embree does, still accepts a
                #   triangle whose rounded t is an ulp larger);
                # - the traversal's answer is the exact one: its triangle is hit by the exact float64 test, and brute force's is either
                #   missed by that test (hit only through the triangle test's one-ulp edge tolerance) or hit no closer in float64 (at a
                #   grazing angle the triangle test's t can fall short of the exact t by more than the leaf box's pad; brute force then
                #   takes that triangle, while the traversal, whose tfar already lies before the box, rightly skips it).
                # A triangle that float64 puts strictly closer than the traversal's answer is a lost triangle and fails.
                diff = ((ids != bids).any(1) | (t.view(torch.int32) != bt.view(torch.int32))).nonzero()[:, 0]
                if diff.numel():
                    same = (ids[diff] == bids[diff]).all(1)
                    assert not bool(same.any()), "%s/%s: the same triangle at two distances" % (name, fname)
                    ti, bi = geo.index(ids[diff]), geo.index(bids[diff])
                    ta, tb = f64_plane_t(geo, rays[diff], ti), f64_plane_t(geo, rays[diff], bi)
                    ulps = (t[diff].view(torch.int32).long() - bt[diff].view(torch.int32).long()).abs()
                    tie = (ulps <= 2) & ((ta - tb).abs() <= 1e-6 * torch.maximum(ta.abs(), tb.abs()))
                    exact = f64_hit_holds(geo, rays[diff], ti, t[diff], strict=True) & (
                        ~f64_hit_holds(geo, rays[diff], bi, bt[diff], strict=True) | (ta <= tb))
                    counts["closest_exact_ties"] = int(tie.sum())
                    counts["closest_traversal_exact"] = int((exact & ~tie).sum())
                    k = diff[~(tie | exact)]
                    assert k.numel() == 0, "%s/%s: traversal and brute force differ beyond a tie: ray %s, traversal %s t %s, brute %s t %s" % (
                        name, fname, rays[k[0]].tolist(), ids[k[0]].tolist(), float(t[k[0]]), bids[k[0]].tolist(), float(bt[k[0]]))
                counts["closest_ids"] = rays.shape[0]
                if fname == "tfar_at_hit":
                    # tfar at the triangle's own t must hit.  The triangle test bounds Ts <= |den| * tfar on its own scale, so a t rounded
                    # down can miss by rounding: count those, and with tfar 4 ulps larger both modes must hit.
                    miss = (~bhit).nonzero()[:, 0]
                    counts["tfar_at_hit_missed_by_rounding"] = int(miss.numel())
                    if miss.numel():
                        again = rays[miss].clone()
                        for _ in range(4):
                            again[:, 7] = torch.nextafter(again[:, 7], torch.full_like(again[:, 7], math.inf))
                        for brute in (False, True):
                            i2, _ = scene.trace_rays(again, brute_force=brute)
                            assert bool((i2[:, 0] >= 0).all()), "%s: a ray misses with tfar 4 ulps above its hit (brute force %s)" % (name, brute)
            else:
                k = hit.nonzero()[:, 0]
                if k.numel():
                    ok = f64_hit_holds(geo, rays[k], geo.index(ids[k]), t[k])
                    assert bool(ok.all()), "%s/%s: any-hit triangle does not intersect the ray in float64: ray %s, ids %s, t %s" % (
                        name, fname, rays[k[~ok][0]].tolist(), ids[k[~ok][0]].tolist(), float(t[k[~ok][0]]))
                counts["any_hit_holds"] = int(k.numel())
                counts["any_miss"] = int((~hit).sum())
        # the plain float64 reference, on the rays whose answer does not depend on rounding (none of the two families whose tfar is at
        # the hit, by construction)
        if fname in ("tfar_at_hit", "tfar_below_hit"):
            continue
        sub = rays[:n_f64] if rays.shape[0] <= n_f64 else rays[torch.randperm(rays.shape[0], generator=gen, device=dev)[:n_f64]]
        ref_i, ref_t, robust, ref_u = f64_closest(geo, sub)
        ids, t = scene.trace_rays(sub)
        r = robust.nonzero()[:, 0]
        lib_i = torch.where(ids[:, 0] >= 0, geo.index(ids), torch.full_like(ref_i, -1))
        wrong = (lib_i[r] != ref_i[r]).nonzero()[:, 0]
        assert wrong.numel() == 0, "%s/%s: %d of %d rays disagree with the float64 closest hit, e.g. ray %s: library %s t %s, float64 %s t %s" % (
            name, fname, wrong.numel(), r.numel(), sub[r[wrong[0]]].tolist(), int(lib_i[r[wrong[0]]]), float(t[r[wrong[0]]]),
            int(ref_i[r[wrong[0]]]), float(ref_t[r[wrong[0]]]))
        h = r[ref_i[r] >= 0]
        # t to 1e-5 relative, or to float32's placement of the ray where that is coarser (an origin close to the surface)
        err = (t[h].double() - ref_t[h].double()).abs() - torch.maximum(1e-5 * ref_t[h].double().abs(), ref_u[h])
        assert not bool((err > 0).any()), (name, fname, float(err.max()))
        counts["f64_reference"] = int(r.numel())
        counts["f64_hits"] = int(h.numel())
    for fname, counts in report.items():
        for check, c in counts.items():
            if check in ("any_hit_holds", "any_miss", "f64_hits", "closest_exact_ties", "closest_traversal_exact", "closest_unresolved_hits_lost",
                         "any_unresolved_hits_lost", "tfar_at_hit_missed_by_rounding"):
                continue  # (whether a family hits anything depends on the scene)
            if check == "f64_reference" and not geo.resolvable:
                continue  # (no ray's answer is independent of rounding)
            if check == "f64_reference" and fname == "shadow":
                continue  # (its target lies 1e-4 beyond tfar by construction: few of these rays are independent of rounding)
            if check == "f64_reference" and fname == "secondary" and geo.magnitude > 100 * geo.radius:
                continue  # (float32 places a surface point far from the origin to more than tnear: leaving it is rounding-dependent)
            assert c > 0, "%s/%s: check %s compared no ray" % (name, fname, check)
    print("%s: %s" % (name, {f: c for f, c in report.items()}))
    return report


def f64_plane_t(geo, rays, idx):
    o, d = rays[:, :3].double(), rays[:, 4:7].double()
    P = geo.P.double()[idx]
    n = torch.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0], dim=1)
    den = (n * d).sum(1)
    return ((P[:, 0] - o) * n).sum(1) / torch.where(den == 0, torch.ones_like(den), den)


# ---------------------------------------------------------------------------------------------------- structure (the LBVH)
def tables(scene):
    nodes = scene.table("bvh_nodes")
    tris = scene.table("bvh_triangles")
    return nodes, tris


def check_structure(name, scene, shapes):
    """The LBVH's tables: see the module docstring.  Returns the tree's height."""
    nodes_b, tris_b = tables(scene)
    T = sum(int(i.shape[0]) for _, i in shapes)
    assert nodes_b.size == 64 * max(T - 1, 0) and tris_b.size == 48 * T, (name, nodes_b.size, tris_b.size, T)
    tri_f = tris_b.view(np.float32).reshape(T, 3, 4)
    tri_i = tris_b.view(np.int32).reshape(T, 3, 4)
    # leaves: a permutation of every (shape, triangle), with the scene's coordinates bit for bit
    sid, tid = tri_i[:, 0, 3].astype(np.int64), tri_i[:, 1, 3].astype(np.int64)
    offs = np.cumsum([0] + [int(i.shape[0]) for _, i in shapes])
    assert (sid >= 0).all() and (sid < len(shapes)).all(), name
    g = offs[sid] + tid
    assert (tid >= 0).all() and (g < offs[sid + 1]).all() and np.array_equal(np.sort(g), np.arange(T)), name + ": leaves are not a permutation"
    P = torch.cat([v.cpu()[i.cpu().long()] for v, i in shapes]).numpy()
    assert np.array_equal(tri_f[:, :, :3].view(np.uint32), P[g].view(np.uint32)), name + ": leaf coordinates differ from vertices[indices]"
    if T == 1:
        return 0
    nd = nodes_b.view(np.float32).reshape(T - 1, 16)
    ni = nodes_b.view(np.int32).reshape(T - 1, 16)
    left, right = ni[:, 12].astype(np.int64), ni[:, 13].astype(np.int64)
    # boxes[node, side] = (lo xyz, hi xyz)
    boxes = np.stack([np.stack([nd[:, 0], nd[:, 4], nd[:, 8], nd[:, 1], nd[:, 5], nd[:, 9]], 1),
                      np.stack([nd[:, 2], nd[:, 6], nd[:, 10], nd[:, 3], nd[:, 7], nd[:, 11]], 1)], 1)
    # the walk from the root (0): every inner node and every leaf slot exactly once, no cycle, at most 63 levels
    seen_inner = np.zeros(T - 1, np.int64)
    seen_leaf = np.zeros(T, np.int64)
    frontier = np.array([0])
    height = 0
    while frontier.size:
        assert height < STACK, name + ": walk deeper than %d levels (cycle?)" % STACK
        np.add.at(seen_inner, frontier, 1)
        ch = np.concatenate([left[frontier], right[frontier]])
        assert (ch < T - 1).all() and (ch >= -T).all(), name + ": child reference out of range"
        np.add.at(seen_leaf, ~ch[ch < 0], 1)
        frontier = ch[ch >= 0]
        height += 1
    assert (seen_inner == 1).all() and (seen_leaf == 1).all(), name + ": nodes not reached exactly once"
    assert height <= STACK - 1, (name, height)
    bits = boxes.view(np.uint32)
    # inner children: the stored box is the min / max of the child's two stored boxes, bit for bit
    for side, child in ((0, left), (1, right)):
        inner = np.nonzero(child >= 0)[0]
        c = child[inner]
        lo = np.minimum(boxes[c, 0, :3], boxes[c, 1, :3])
        hi = np.maximum(boxes[c, 0, 3:], boxes[c, 1, 3:])
        assert np.array_equal(bits[inner, side], np.concatenate([lo, hi], 1).view(np.uint32)), name + ": refit box differs from its children's"
        # leaf children: strictly containing the triangle, with a bounded pad
        leaf = np.nonzero(child < 0)[0]
        slot = ~child[leaf]
        V = tri_f[slot, :, :3].astype(np.float64)
        vlo, vhi = V.min(1), V.max(1)
        b = boxes[leaf, side].astype(np.float64)
        assert (b[:, :3] < vlo).all() and (b[:, 3:] > vhi).all(), name + ": a leaf box does not strictly contain its triangle"
        ext = float((P.reshape(-1, 3).max(0) - P.reshape(-1, 3).min(0)).max())
        bound = 1e-5 * (np.maximum(np.abs(vlo), np.abs(vhi)) + ext)
        assert (vlo - b[:, :3] <= bound).all() and (b[:, 3:] - vhi <= bound).all(), name + ": a leaf box is padded too much"
    return height


# ---------------------------------------------------------------------------------------------------- tests
def _rb():
    from redner_b200 import redner as rb
    return rb


@pytest.fixture(scope="module")
def built():
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()
            shapes = SCENES[name]()
            scene, dev_shapes = make_scene(shapes, DEV, _rb())
            cache[name] = (scene, dev_shapes)
        return cache[name]
    return get


@pytest.mark.parametrize("name", list(SCENES))
def test_lbvh_structure(built, name):
    scene, shapes = built(name)
    height = check_structure(name, scene, shapes)
    again, _ = make_scene([(v.cpu(), i.cpu()) for v, i in shapes], DEV, _rb())
    a, b = tables(scene), tables(again)
    assert all(np.array_equal(x, y) for x, y in zip(a, b)), name + ": two builds differ"
    if name == "depth_63":
        assert height == STACK - 1, height


@pytest.mark.parametrize("name", list(SCENES))
def test_traversal_equals_brute_force_and_float64(built, name):
    scene, shapes = built(name)
    small = name in ("one_triangle", "two_triangles", "three_triangles")
    check_queries(name, scene, shapes, DEV, n=512 if small else 4096)


def test_tree_one_level_too_deep_is_refused():
    with pytest.raises(RuntimeError) as e:
        make_scene(_depth_keys(duplicate=True), DEV, _rb())
    assert "levels deep" in str(e.value), str(e.value)
