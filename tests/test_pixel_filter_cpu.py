"""CPU suite: pixel reconstruction filters (rb_pixel_filter) on the host build of the device headers (tools/cpu_emu).

- The 1-pixel box given explicitly renders what the zero-initialised default renders, bit for bit: images and gradients with both
  edge samplers, Sobol and PCG; primary-edge tables likewise.
- A tent of width 2 and a Gaussian of width 3 give the expected image: an 8x supersampled box render convolved with the filter's
  exact per-cell integrals (expected_image_check).
- Their gradients of a loss with a fixed non-uniform weight image agree with central finite differences (fd_check), including an
  edge that lies outside the image but inside the filter's reach (border_check): zero for the box, the finite difference for the tent.
- An update that changes only the filter equals a new scene with it, table by table; a gloo render_tiles at world size 2 with a tent
  equals world size 1 bit for bit (deterministic mode); every refused combination raises with a message naming the pixel filter.
The device side is tests/test_pixel_filter_gpu.py, which calls the checks below at larger sizes.

Run as a script (`python tests/test_pixel_filter_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import math
import os
import socket
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

FILTERS = {"tent2": ("tent", 2.0), "gauss3": ("gaussian", 3.0)}


# ---------------------------------------------------------------------------------------------------- shared with the GPU suite
def pixel_filter(name):
    from redner_b200 import api
    return None if name is None else api.PixelFilter(*FILTERS[name]) if name in FILTERS else api.PixelFilter(*name)


def filter_cdf(kind, width, t):
    """1-D CDF of the normalised filter at offsets t (pixels) from the pixel centre."""
    t = np.asarray(t, dtype=np.float64)
    r = 0.5 * width
    if kind == "box":
        return np.clip((t + r) / width, 0.0, 1.0)
    if kind == "tent":
        tc = np.clip(t, -r, r)
        return np.where(tc < 0, (tc + r) ** 2 / (2 * r * r), 1.0 - (r - tc) ** 2 / (2 * r * r))
    from scipy.special import erf
    sigma = width / 6.0
    tc = np.clip(t, -r, r)
    return 0.5 * (erf(tc / (sigma * math.sqrt(2))) / erf(r / (sigma * math.sqrt(2))) + 1.0)


def cell_weights(kind, width, n_px, S):
    """[n_px, n_px * S]: integral of pixel c's 1-D filter over sub-cell k (sub-cells of 1/S pixel)."""
    edges = np.arange(n_px * S + 1) / S
    centres = np.arange(n_px) + 0.5
    F = filter_cdf(kind, width, edges[None, :] - centres[:, None])
    return F[:, 1:] - F[:, :-1]


def quadrature_bound(kind, width, S, fine=16):
    """Q = sum over sub-cells k of the integral of |f - mean_k f| (2-D filter, one pixel).  Replacing the radiance L by its sub-cell
    averages changes a pixel by at most Q * (max L - min L) / 2 over its reach: the quadrature error allowed for."""
    r = 0.5 * width
    n = int(math.ceil(r * S)) + 1
    t = (np.arange(-n * S * fine, n * S * fine) + 0.5) / (S * fine)  # fine midpoints over [-n, n) pixels / S
    F = filter_cdf(kind, width, np.concatenate([t - 0.5 / (S * fine), t[-1:] + 0.5 / (S * fine)]))
    f1 = np.diff(F) * (S * fine)
    f2 = np.outer(f1, f1).reshape(2 * n * S, fine, 2 * n * S, fine)
    mean = f2.mean(axis=(1, 3), keepdims=True)
    return float(np.abs(f2 - mean).sum() / (S * fine) ** 2)


def make_scene(dev, name, res, camera="perspective"):
    """'triangle' (C1) or 'room' (the textured glossy room); camera 'perspective', 'ortho' or 'crop' (a viewport inside the image)."""
    import torch
    import scenes
    from redner_b200 import api
    if name == "triangle":
        sc = scenes.single_triangle(dev, resolution=(res, res))
        if camera == "ortho":
            sc.camera = api.Camera(position=torch.tensor([0.0, 0.0, -5.0], requires_grad=True), look_at=torch.tensor([0.0, 0.0, 0.0]),
                                   up=torch.tensor([0.0, 1.0, 0.0]), clip_near=1e-2, resolution=(res, res), camera_type=1,
                                   intrinsic_mat=torch.tensor([[0.45, 0.0, 0.0], [0.0, 0.45, 0.0], [0.0, 0.0, 1.0]]))
    else:
        sc = scenes.glossy_room(dev, resolution=(res, res), camera_type=1 if camera == "ortho" else 0)
    if camera == "crop":
        q = res // 4
        sc.camera.viewport = (q, q + 2, res - q, res - q + 2)
    return sc


def render_image(rb, dev, sc, spp, seed, filt, mb=1, sampler=None):
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=sampler if sampler is not None else rb.SamplerType.independent, device=dev,
                                              backend=rb, pixel_filter=pixel_filter(filt))
    return api.RenderFunction.apply(seed, *args).detach().double().cpu().numpy()


def expected_image_check(rb, dev, name, camera, filt, res, spp, seeds, ss_spp, ss_seeds, S=8):
    """Filtered renders over independent seeds against the S x supersampled box render convolved with the filter's per-cell integrals,
    per 4 x 4 block of the viewport whose reach lies inside the image: |difference| <= 4 combined standard errors (from the seeds)
    + the quadrature bound.  Returns the number of blocks compared."""
    kind, width = FILTERS[filt]
    f = np.stack([render_image(rb, dev, make_scene(dev, name, res, camera), spp, 100 + s, filt) for s in range(seeds)])
    ss = []
    for s in range(ss_seeds):
        sc = make_scene(dev, name, res * S, "ortho" if camera == "ortho" else "perspective")
        ss.append(render_image(rb, dev, sc, ss_spp, 900 + s, None))
    ss = np.stack(ss)  # [seeds, H*S, W*S, 3]: sub-cell averages
    Wy, Wx = cell_weights(kind, width, res, S), cell_weights(kind, width, res, S)
    conv = np.einsum("yk,nklc,xl->nyxc", Wy, ss, Wx)
    inside = np.isclose(Wx.sum(1), 1.0, atol=1e-12)  # pixels whose reach lies inside the image
    Q = quadrature_bound(kind, width, S)
    vp = make_scene(dev, name, res, camera).camera.viewport or (0, 0, res, res)
    y0, x0, y1, x1 = vp
    blocks = 0
    reach = int(math.ceil(0.5 * width))
    for by in range(y0, y1 - 3, 4):
        for bx in range(x0, x1 - 3, 4):
            if not (inside[by:by + 4].all() and inside[bx:bx + 4].all()):
                continue
            a = f[:, by - y0:by - y0 + 4, bx - x0:bx - x0 + 4].sum(axis=(1, 2))  # [seeds, 3]
            b = conv[:, by:by + 4, bx:bx + 4].sum(axis=(1, 2))
            se = np.sqrt(a.var(0, ddof=1) / seeds + b.var(0, ddof=1) / ss_seeds)
            region = ss[:, (by - reach) * S:(by + 4 + reach) * S, (bx - reach) * S:(bx + 4 + reach) * S].mean(0)
            quad = 16 * Q * 0.5 * (region.max() - region.min())
            diff = np.abs(a.mean(0) - b.mean(0))
            assert (diff <= 4 * se + quad + 1e-6).all(), (name, camera, filt, by, bx, diff, se, quad)
            blocks += 1
    assert blocks > 0
    return blocks


def weight_image(shape, seed=11):
    import torch
    g = torch.Generator().manual_seed(seed)
    return 0.2 + 1.6 * torch.rand(shape, generator=g)


def _loss_and_grads(rb, dev, make, filt, spp, seed, mb, grad_of):
    """loss = sum(W * img) with the fixed weight image W; (loss, analytic gradient of grad_of(scene))."""
    import torch
    from redner_b200 import api
    sc = make()
    args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=rb.SamplerType.independent, device=dev, backend=rb,
                                              pixel_filter=pixel_filter(filt))
    img = api.RenderFunction.apply(seed, *args)
    loss = (weight_image(img.shape).to(img.device) * img).sum()
    loss.backward()
    return float(loss.detach()), grad_of(sc)


def fd_check(rb, dev, make, move, grad_of, filt, spp, fd_spp, seeds, eps, mb=1, rel=0.03):
    """Central finite differences (common random numbers) of loss = sum(W * img) under `move(scene, delta)` against the analytic
    gradient, both averaged over `seeds`: |analytic - fd| <= 4 combined standard errors + rel * |fd|.  Returns (analytic, fd)."""
    an = [_loss_and_grads(rb, dev, make, filt, spp, 1 + s, mb, grad_of)[1] for s in range(seeds)]

    def moved(d):
        def mk():
            sc = make()
            move(sc, d)
            return sc
        return mk
    fd = [(_loss_and_grads(rb, dev, moved(eps), filt, fd_spp, 50 + s, mb, lambda sc: 0.0)[0] -
           _loss_and_grads(rb, dev, moved(-eps), filt, fd_spp, 50 + s, mb, lambda sc: 0.0)[0]) / (2 * eps) for s in range(seeds)]
    an, fd = np.array(an), np.array(fd)
    se = math.sqrt(an.var(ddof=1) / seeds + fd.var(ddof=1) / seeds)
    assert abs(an.mean() - fd.mean()) <= 4 * se + rel * abs(fd.mean()), (filt, an, fd, se)
    assert abs(fd.mean()) > 4 * fd.std(ddof=1) / math.sqrt(seeds), (filt, fd)  # (a finite difference that is not noise)
    return an.mean(), fd.mean()


def triangle_moves(dev, res):
    """(make, move, grad_of) for the C1 triangle along x, along y, and the camera position along x."""
    import torch
    import scenes

    def make():
        return scenes.single_triangle(dev, resolution=(res, res))

    def shift(axis):
        def move(sc, d):
            with torch.no_grad():
                sc.shapes[0].vertices[:, axis] += d
        return move

    def cam_move(sc, d):
        with torch.no_grad():
            sc.camera.position[0] += d
    tri = lambda axis: lambda sc: float(sc.shapes[0].vertices.grad[:, axis].sum())  # noqa: E731
    return [(make, shift(0), tri(0)), (make, shift(1), tri(1)), (make, cam_move, lambda sc: float(sc.camera.position.grad[0]))]


def border_scene(dev, res, offset_px=0.25):
    """An emissive quad just outside the image: its inner edge lies offset_px pixels past the image's side, the rest farther out.
    Only samples that leave the image (a filter wider than a pixel) see it, and only its edge moves what they see."""
    import torch
    import scenes
    from redner_b200 import api
    half = 5.0 * math.tan(math.radians(22.5))  # half the image width in world units at the quad's depth (fov 45, distance 5)
    xe = half + offset_px * 2 * half / res
    cam = api.Camera(position=torch.tensor([0.0, 0.0, -5.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([45.0]), clip_near=1e-2, resolution=(res, res))
    v = torch.tensor([[xe, -1.0, 0.0], [xe + 2.0, -1.0, 0.0], [xe, 1.0, 0.0], [xe + 2.0, 1.0, 0.0]], device=dev).requires_grad_(True)
    quad = api.Shape(v, torch.tensor([[0, 1, 2], [1, 3, 2]], dtype=torch.int32, device=dev), 0)
    black = api.Material(diffuse_reflectance=torch.tensor([0.0, 0.0, 0.0], device=dev))
    return api.Scene(cam, [quad], [black], [api.AreaLight(0, torch.tensor([5.0, 5.0, 5.0]), two_sided=True)])


def border_check(rb, dev, res, spp, fd_spp, seeds, eps=0.01):
    """The box: analytic gradient and finite difference both exactly zero.  The tent of width 2 (reach 0.5 pixel): they agree."""
    import torch
    make = lambda: border_scene(dev, res)  # noqa: E731

    def move(sc, d):
        with torch.no_grad():
            sc.shapes[0].vertices[:, 0] += d
    grad_of = lambda sc: float(sc.shapes[0].vertices.grad[:, 0].sum())  # noqa: E731
    for s in range(2):
        _, g = _loss_and_grads(rb, dev, make, None, spp, 1 + s, 0, grad_of)
        assert g == 0.0, g
        lp, _ = _loss_and_grads(rb, dev, lambda: (lambda sc: (move(sc, eps), sc)[1])(make()), None, spp, 1 + s, 0, lambda sc: 0.0)
        assert lp == 0.0, lp
    return fd_check(rb, dev, make, move, grad_of, "tent2", spp, fd_spp, seeds, eps, mb=0)


def scene_tables(scene):
    from redner_b200 import _lib
    return {t: scene.table(t).tobytes() for t in _lib.RB_TABLES}


def native_scene(rb, dev, sc, filt, **kw):
    """The native scene RenderFunction builds for `sc` with pixel filter `filt`."""
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, 1, 1, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb, pixel_filter=pixel_filter(filt), **kw)
    return api.RenderFunction._unpack((1, 2), args)


def box_default_check(rb, dev, cases):
    """{BOX, 1} given explicitly == the zero-initialised default: images, every gradient and the primary-edge tables, bit for bit."""
    import parity_utils as pu
    import scenes
    from redner_b200 import api
    for name, res, spp, mb, sampler in cases:
        outs = []
        for filt in (None, ("box", 1.0)):
            sc = scenes.SCENES[name](dev, resolution=(res, res))
            args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=sampler, device=dev, backend=rb, use_primary_edge_sampling=True,
                                                      use_secondary_edge_sampling=True, pixel_filter=pixel_filter(filt))
            img = api.RenderFunction.apply(3, *args)
            (weight_image(img.shape).to(img.device) * img).sum().backward()
            c = native_scene(rb, dev, scenes.SCENES[name](dev, resolution=(res, res)), filt)
            outs.append((img.detach().cpu().numpy(), pu.collect_grads(sc), scene_tables(c.scene)))
        (i0, g0, t0), (i1, g1, t1) = outs
        assert i0.tobytes() == i1.tobytes(), name
        assert g0.keys() == g1.keys() and g0, name
        for k in g0:
            assert g0[k].numpy().tobytes() == g1[k].numpy().tobytes(), (name, k)
        assert t0 == t1, name


def update_check(rb, dev, make, filters):
    """A Scene.update that changes only the pixel filter == a new scene with that filter, table by table (and back)."""
    c = native_scene(rb, dev, make(), None)
    for filt in list(filters) + [None]:
        ref = native_scene(rb, dev, make(), filt)
        c.scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False, pixel_filter=pixel_filter(filt).native() if filt else None)
        assert scene_tables(c.scene) == scene_tables(ref.scene), filt
    a, b = scene_tables(native_scene(rb, dev, make(), None).scene), scene_tables(native_scene(rb, dev, make(), filters[0]).scene)
    assert a["primary_edge_pmf"] != b["primary_edge_pmf"]  # (the filter does reach the tables)


def refusals_check(rb, dev):
    """Every refused combination raises with a message naming the pixel filter."""
    import pytest
    import torch
    import scenes
    from redner_b200 import api

    def raises(fn):
        with pytest.raises(RuntimeError, match="pixel filter"):
            fn()
    for ct in (2, 3):  # fisheye, panorama
        raises(lambda: native_scene(rb, dev, scenes.glossy_room(dev, resolution=(8, 8), camera_type=ct), "tent2"))
    raises(lambda: native_scene(rb, dev, scenes.glossy_room(dev, resolution=(8, 8), distortion=True), "gauss3"))
    raises(lambda: native_scene(rb, dev, scenes.glossy_room(dev, resolution=(8, 8), camera_type=2), ("box", 2.0)))
    for bad in (("tent", 0.0), ("tent", 4.5), ("gaussian", -1.0), ("box", float("nan"))):
        raises(lambda: native_scene(rb, dev, scenes.single_triangle(dev, resolution=(8, 8)), bad))
    c = native_scene(rb, dev, scenes.single_triangle(dev, resolution=(8, 8)), None)
    raises(lambda: rb.Scene(c.camera, c.shapes, c.materials, c.lights, None, c.scene.use_gpu, c.scene.gpu_index, True, True, pixel_filter=(7, 1.0)))
    # an update to a filtered descriptor with a fisheye camera, and a fisheye camera for a filtered scene
    fish = native_scene(rb, dev, scenes.glossy_room(dev, resolution=(8, 8), camera_type=2), None)
    raises(lambda: fish.scene.update(fish.camera, fish.shapes, fish.materials, fish.lights, None, geometry_changed=False, pixel_filter=(1, 2.0)))
    room = native_scene(rb, dev, scenes.glossy_room(dev, resolution=(8, 8)), "tent2")
    raises(lambda: room.scene.set_camera(fish.camera))
    # rb_render: sample_pixel_center, a screen-gradient image
    sc = scenes.single_triangle(dev, resolution=(8, 8))
    args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev, backend=rb, sample_pixel_center=True, pixel_filter=pixel_filter("tent2"))
    raises(lambda: api.RenderFunction.apply(1, *args))
    c = native_scene(rb, dev, scenes.single_triangle(dev, resolution=(8, 8)), "tent2")
    g = api.RenderFunction.gradient_buffers(c)
    grad_img, sg = torch.ones(8, 8, 3), torch.zeros(8, 8, 2)
    raises(lambda: rb.render(c.scene, c.options, rb.float_ptr(0), rb.float_ptr(grad_img.data_ptr()), g.d_scene, rb.float_ptr(sg.data_ptr()), rb.float_ptr(0)))


# ---------------------------------------------------------------------------------------------------- on the emulator
def _run(checks, timeout=1800):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_explicit_box_is_the_default_bit_for_bit():
    _run(["box_default"])


def test_filtered_image_matches_the_convolved_supersampled_box():
    _run(["expected_image"])


def test_filtered_gradients_match_finite_differences():
    _run(["fd"])


def test_edge_outside_the_image_within_the_filter_reach():
    _run(["border"])


def test_filter_update_equals_a_new_scene():
    _run(["update"])


def test_refused_combinations_name_the_filter():
    _run(["refusals"])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _tile_worker(rank, world, port, emu_so, out_path):
    """One rank of a sharded render with a tent filter under deterministic algorithms, the emulator behind the C ABI."""
    import torch
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import _lib, dist as rdist
    _lib._lib = _lib._bind(ctypes.CDLL(emu_so))  # this process only
    from redner_b200 import redner as rb
    import parity_utils as pu
    import scenes
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cpu")
        sc = scenes.glossy_room(dev, resolution=(22, 18))
        img = rdist.render_tiles(sc, 4, 2, seed=5, rows_per_stripe=4, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                 use_primary_edge_sampling=True, use_secondary_edge_sampling=True, pixel_filter=pixel_filter("tent2"))
        (weight_image(img.shape) * img).sum().backward()
        if rank == 0:
            g = pu.collect_grads(sc)
            np.savez(out_path, image=img.detach().numpy(), **{k: v.numpy() for k, v in g.items()})
    finally:
        dist.destroy_process_group()


def test_gloo_render_tiles_with_a_tent_is_independent_of_world_size(tmp_path):
    import torch.multiprocessing as mp
    import test_device_code_cpu as tdc
    emu = tdc._build()
    outs = {}
    for world in (1, 2):
        path = str(tmp_path / ("w%d.npz" % world))
        mp.spawn(_tile_worker, args=(world, _free_port(), emu, path), nprocs=world, join=True)
        outs[world] = dict(np.load(path))
    assert len(outs[1]) > 5 and any(np.count_nonzero(v) for k, v in outs[1].items() if k != "image")
    assert set(outs[2]) == set(outs[1])
    for k in outs[1]:
        assert outs[2][k].tobytes() == outs[1][k].tobytes(), k


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    dev = torch.device("cpu")
    for name in names:
        if name == "box_default":
            box_default_check(rb, dev, [("single_triangle", 16, 4, 1, rb.SamplerType.sobol), ("single_triangle", 16, 4, 1, rb.SamplerType.independent),
                                        ("glossy_room", 12, 2, 2, rb.SamplerType.sobol)])
        elif name == "expected_image":
            expected_image_check(rb, dev, "triangle", "crop", "tent2", 16, 32, 4, 4, 2)
            expected_image_check(rb, dev, "room", "ortho", "gauss3", 12, 16, 4, 2, 2)
        elif name == "fd":
            for filt in ("tent2", "gauss3"):
                for make, move, grad_of in triangle_moves(dev, 16):
                    fd_check(rb, dev, make, move, grad_of, filt, 64, 1024, 4, 0.05)
        elif name == "border":
            border_check(rb, dev, 12, 256, 1024, 3)
        elif name == "update":
            import scenes
            update_check(rb, dev, lambda: scenes.glossy_room(dev, resolution=(12, 12)), ["tent2", "gauss3"])
        elif name == "refusals":
            refusals_check(rb, dev)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
