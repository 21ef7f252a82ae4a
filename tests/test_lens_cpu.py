"""CPU suite: the thin-lens camera (rb_camera::lens_radius / focus_distance) on the host build of the device headers (tools/cpu_emu).

- An explicit lens_radius of 0 renders what a camera without a lens renders, bit for bit: images, every gradient, the scene tables and
  the exact records; its d(lens_radius) and d(focus_distance) are 0.
- The uv and position channels of a textured plane at the focal distance are those of the pinhole, to float rounding.
- Pinhole-average identity, the main oracle: a lens render is the expectation over the lens point L of a pinhole render whose camera
  moves to L (cam_to_world . translate(L)) and whose principal point moves by K2 L.xy / f.  Those cameras are built as torch functions
  of (lens_radius, focus_distance, u) and rendered through the pinhole path; images, vertex gradients and autograd d/d(lens_radius),
  d/d(focus_distance) agree with the lens render's within 4 standard errors, with primary edges alone and with both edge samplers.
- d/d(lens_radius) and d/d(focus_distance) of a defocused silhouette agree with central differences within 4 standard errors.
- A lens-only update equals a new scene, table by table; set_camera changes the lens; every refused combination raises with a message
  naming the lens; deterministic mode repeats itself bit for bit whatever the band size.
The device side is tests/test_lens_gpu.py, which calls the checks below at larger sizes.

Run as a script (`python tests/test_lens_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the emulator in
place of the library."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------- shared with the GPU suite
def concentric(u):
    """Shirley-Chiu concentric map of u in [0, 1)^2 ([n, 2], float64 tensor) onto the unit disc, as rb_camera.cuh's concentric_disc."""
    import torch
    a, b = 2 * u[:, 0] - 1, 2 * u[:, 1] - 1
    first = a * a > b * b
    r = torch.where(first, a, b)
    safe_a = torch.where(a == 0, torch.ones_like(a), a)
    safe_b = torch.where(b == 0, torch.ones_like(b), b)
    phi = torch.where(first, (math.pi / 4) * (b / safe_a), math.pi / 2 - (math.pi / 4) * (a / safe_b))
    out = torch.stack([r * torch.cos(phi), r * torch.sin(phi)], 1)
    return torch.where(((a == 0) & (b == 0))[:, None], torch.zeros_like(out), out)


def _c2w(eye, target):
    """cam_to_world of a camera at `eye` looking at `target` with up +y (the look-at convention of the renderer: x = normalize(cross(up, z)))."""
    import torch
    eye, target = torch.tensor(eye, dtype=torch.float64), torch.tensor(target, dtype=torch.float64)
    z = (target - eye) / torch.linalg.norm(target - eye)
    x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64), z)
    x = x / torch.linalg.norm(x)
    y = torch.linalg.cross(z, x)
    m = torch.eye(4, dtype=torch.float64)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, z, eye
    return m.float()


def _intrinsic(fov_deg):
    import torch
    f = 1.0 / math.tan(0.5 * math.radians(fov_deg))
    return torch.diag(torch.tensor([f, f, 1.0]))


def lens_camera(res, c2w, K, lens, clip_near=1e-2):
    """api.Camera with cam_to_world `c2w` (4x4) and intrinsic_mat `K`; `lens` = (lens_radius, focus_distance) tensors or None."""
    from redner_b200 import api
    kw = {} if lens is None else dict(lens_radius=lens[0], focus_distance=lens[1])
    return api.Camera(cam_to_world=c2w, intrinsic_mat=K, clip_near=clip_near, resolution=(res, res), **kw)


def pinhole_at(c2w, K, r, f, c):
    """The pinhole camera of lens point L = r c (c on the unit disc): cam_to_world . translate(L), principal point + K2 L.xy / f."""
    import torch
    L = r * c.float()
    T = torch.eye(4).index_put((torch.tensor([0, 1]), torch.tensor([3, 3])), L)
    shift = (K[:2, :2] @ L) / f
    K2 = K.clone()
    K2 = K2.index_put((torch.tensor([0, 1]), torch.tensor([2, 2])), K[:2, 2] + shift)
    return c2w @ T, K2


def glow_scene(dev, res, lens, c2w=None):
    """Primary edges alone: an emissive triangle in front of an emissive quad, seen by a camera at z = -5 (mb 0)."""
    import torch
    from redner_b200 import api
    c2w = _c2w([0.0, 0.0, -5.0], [0.0, 0.0, 0.0]) if c2w is None else c2w
    cam = lens_camera(res, c2w, _intrinsic(45.0), lens)
    black = api.Material(diffuse_reflectance=torch.tensor([0.0, 0.0, 0.0], device=dev))
    tri = api.Shape(torch.tensor([[-1.6, 1.2, 0.3], [1.1, 0.9, -0.3], [-0.3, -1.3, 0.2]], device=dev, requires_grad=True),
                    torch.tensor([[0, 1, 2]], dtype=torch.int32, device=dev), 0)
    quad = api.Shape(torch.tensor([[-1.0, -0.8, 2.5], [1.6, -0.8, 2.5], [-1.0, 1.7, 2.5], [1.6, 1.7, 2.5]], device=dev, requires_grad=True),
                     torch.tensor([[0, 2, 1], [1, 2, 3]], dtype=torch.int32, device=dev), 0)
    lights = [api.AreaLight(0, torch.tensor([3.0, 2.0, 1.0])), api.AreaLight(1, torch.tensor([0.5, 1.0, 2.0]))]
    return api.Scene(cam, [tri, quad], [black], lights)


def room_scene(dev, res, lens, c2w=None):
    """The textured glossy room (both edge samplers, mb 2) seen through cam_to_world / intrinsic_mat."""
    import scenes
    sc = scenes.glossy_room(dev, resolution=(res, res))
    c2w = _c2w([0.3, 1.4, -4.5], [0.0, 0.6, 0.0]) if c2w is None else c2w
    sc.camera = lens_camera(res, c2w, _intrinsic(40.0), lens)
    return sc


SCENES = {"glow": (glow_scene, 0), "room": (room_scene, 2)}


def weight_image(shape, seed=11):
    import torch
    g = torch.Generator().manual_seed(seed)
    return 0.5 + torch.rand(*shape, generator=g)


def _lens_params(r, f):
    import torch
    return torch.tensor([r], requires_grad=True), torch.tensor([f], requires_grad=True)


def _vertex_grads(sc):
    import torch
    return torch.cat([s.vertices.grad.detach().cpu().flatten() for s in sc.shapes if s.vertices.grad is not None])


def render_loss(rb, dev, sc, spp, mb, seed, **kw):
    """(loss, image) of weight_image . image, rendered with RenderFunction (Sobol off: independent samples for the statistics)."""
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, spp, mb, device=dev, backend=rb, use_primary_edge_sampling=True,
                                              use_secondary_edge_sampling=mb > 0, **kw)
    img = api.RenderFunction.apply(seed, *args)
    loss = (weight_image(img.shape).to(img.device) * img).sum()
    return loss, img


def pinhole_average_check(rb, dev, name, res, spp, runs, r=0.25, f=5.0, nontrivial=True):
    """The lens render against the average over lens points of pinhole renders (module docstring): means of the loss, d(loss)/d(lens_radius),
    d(loss)/d(focus_distance) and every vertex-gradient component agree within 4 standard errors.  `nontrivial`: d(loss)/d(lens_radius) or
    d(loss)/d(focus_distance) is also more than 3 standard errors from 0 (the room's are too noisy at affordable sizes for that)."""
    import torch
    make, mb = SCENES[name]
    lens_rows, pin_rows = [], []
    gen = torch.Generator().manual_seed(7)
    for k in range(runs):
        rt, ft = _lens_params(r, f)
        sc = make(dev, res, (rt, ft))
        loss, _ = render_loss(rb, dev, sc, spp, mb, (101 + k, 202 + k))
        loss.backward()
        lens_rows.append(torch.cat([loss.detach().cpu().reshape(1), rt.grad, ft.grad, _vertex_grads(sc)]).double())
        rt, ft = _lens_params(r, f)
        c = concentric(torch.rand(1, 2, generator=gen, dtype=torch.float64))[0]
        base = make(dev, res, None)
        c2w, K = pinhole_at(base.camera.cam_to_world, base.camera.intrinsic_mat, rt, ft, c)
        sc = make(dev, res, None, c2w=c2w)
        sc.camera = lens_camera(res, c2w, K, None)
        loss, _ = render_loss(rb, dev, sc, spp, mb, (303 + k, 404 + k))
        loss.backward()
        pin_rows.append(torch.cat([loss.detach().cpu().reshape(1), rt.grad, ft.grad, _vertex_grads(sc)]).double())
    a, b = torch.stack(lens_rows).numpy(), torch.stack(pin_rows).numpy()
    se = np.sqrt(a.var(axis=0, ddof=1) / runs + b.var(axis=0, ddof=1) / runs)
    diff = np.abs(a.mean(0) - b.mean(0))
    scale = np.abs(b.mean(0)).max()
    bad = diff > 4 * se + 1e-6 * scale
    if os.environ.get("RB_LENS_VERBOSE"):
        print(np.stack([a.mean(0), b.mean(0), se]))
    assert not bad.any(), (name, np.nonzero(bad)[0].tolist(), a.mean(0)[bad], b.mean(0)[bad], se[bad])
    if nontrivial:
        assert (np.abs(a[:, 1:3].mean(0)) > 3 * se[1:3]).any(), (a[:, 1:3].mean(0), se[1:3])
    return a.mean(0), b.mean(0), se


def fd_check(rb, dev, res, spp, runs, eps_r=0.03, eps_f=0.4, r=0.2, f=4.0):
    """d(loss)/d(lens_radius) and d(loss)/d(focus_distance) of the defocused glow scene against central differences over seeds."""
    import torch
    grads, fds = [], []
    for k in range(runs):
        rt, ft = _lens_params(r, f)
        sc = glow_scene(dev, res, (rt, ft))
        loss, _ = render_loss(rb, dev, sc, spp, 0, (11 + k, 12 + k))
        loss.backward()
        grads.append([rt.grad.item(), ft.grad.item()])
        row = []
        for dr, df, eps in ((eps_r, 0.0, eps_r), (0.0, eps_f, eps_f)):
            vals = []
            for sgn in (1, -1):
                with torch.no_grad():
                    sc = glow_scene(dev, res, (torch.tensor([r + sgn * dr]), torch.tensor([f + sgn * df])))
                    vals.append(render_loss(rb, dev, sc, spp, 0, (11 + k, 12 + k))[0].item())
            row.append((vals[0] - vals[1]) / (2 * eps))
        fds.append(row)
    g, d = np.array(grads), np.array(fds)
    se = np.sqrt(g.var(0, ddof=1) / runs + d.var(0, ddof=1) / runs)
    diff = np.abs(g.mean(0) - d.mean(0))
    assert (diff < 4 * se).all(), (g.mean(0), d.mean(0), se)
    assert np.abs(g.mean(0)[1]) > 3 * se[1], (g.mean(0), se)  # (d/d(lens_radius) is too noisy at these sizes to be told from 0)


def scene_tables(scene):
    from redner_b200 import _lib
    return {t: scene.table(t).tobytes() for t in _lib.RB_TABLES}


def native(rb, dev, sc, **kw):
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev, backend=rb, **kw)
    return api.RenderFunction._unpack((1, 2), args)


def zero_radius_check(rb, dev, res, spp):
    """lens_radius 0 == no lens, bit for bit: image, every gradient (the lens's are 0), tables and exact records."""
    import torch
    import parity_utils as pu
    from redner_b200 import api
    outs = []
    for lens in (None, (torch.tensor([0.0], requires_grad=True), torch.tensor([3.0], requires_grad=True))):
        sc = room_scene(dev, res, lens)
        loss, img = render_loss(rb, dev, sc, spp, 2, (5, 6), sampler_type=rb.SamplerType.sobol)
        loss.backward()
        g = pu.collect_grads(sc)
        g["c2w"] = sc.camera.cam_to_world.grad if sc.camera.cam_to_world.grad is not None else torch.zeros(4, 4)
        if lens is not None:
            assert lens[0].grad.item() == 0.0 and lens[1].grad.item() == 0.0
        c = native(rb, dev, room_scene(dev, res, lens), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        gb = api.RenderFunction.gradient_buffers(c)
        count, fp = rb.exact_record_count(c.scene, c.options, gb.d_scene)
        ones = torch.ones(res, res, 3, device=dev)
        rec = rb.render_exact(c.scene, c.options, api._ptr(rb, ones), gb.d_scene)
        outs.append((img.detach().cpu().numpy(), g, scene_tables(c.scene), (count, fp), rec.cpu().numpy()))
    (i0, g0, t0, n0, r0), (i1, g1, t1, n1, r1) = outs
    assert i0.tobytes() == i1.tobytes()
    assert g0.keys() == g1.keys()
    for k in g0:
        assert g0[k].detach().cpu().numpy().tobytes() == g1[k].detach().cpu().numpy().tobytes(), k
    assert t0 == t1
    assert n0 == n1, (n0, n1)
    assert r0.tobytes() == r1.tobytes()
    assert n0[0] > 58


def in_focus_check(rb, dev, res, spp):
    """uv and position of a textured plane at z = focus_distance: the lens render equals the pinhole render to float rounding (at pixel
    centres, so that both draw the same film positions: the lens takes sampler dimensions of its own)."""
    import torch
    from redner_b200 import api
    imgs = []
    for lens in (None, (torch.tensor([0.4]), torch.tensor([6.0]))):
        cam = lens_camera(res, _c2w([0.0, 0.0, -6.0], [0.0, 0.0, 0.0]), _intrinsic(40.0), lens)
        mat = api.Material(diffuse_reflectance=torch.tensor([0.5, 0.5, 0.5], device=dev))
        plane = api.Shape(torch.tensor([[-5.0, -5.0, 0.0], [5.0, -5.0, 0.0], [-5.0, 5.0, 0.0], [5.0, 5.0, 0.0]], device=dev),
                          torch.tensor([[0, 1, 2], [1, 3, 2]], dtype=torch.int32, device=dev), 0,
                          uvs=torch.tensor([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0], [1.0, 1.0]], device=dev))
        sc = api.Scene(cam, [plane], [mat], [])
        args = api.RenderFunction.serialize_scene(sc, spp, 0, channels=[rb.channels.uv, rb.channels.position], device=dev, backend=rb,
                                                  use_primary_edge_sampling=False, use_secondary_edge_sampling=False, sample_pixel_center=True)
        imgs.append(api.RenderFunction.apply(3, *args).cpu().numpy())
    assert np.abs(imgs[0]).max() > 0.1
    assert np.allclose(imgs[0], imgs[1], rtol=0, atol=2e-5 * max(1.0, np.abs(imgs[0]).max())), np.abs(imgs[0] - imgs[1]).max()


def update_check(rb, dev, res):
    """A lens-only update == a new scene, table by table; set_camera with a lens changes the tables likewise."""
    import torch
    c = native(rb, dev, room_scene(dev, res, None), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    pin = scene_tables(c.scene)
    for lens in ((0.2, 4.0), (0.5, 7.0), (0.0, 1.0)):
        lt = (torch.tensor([lens[0]]), torch.tensor([lens[1]]))
        ref = native(rb, dev, room_scene(dev, res, lt), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        new = native(rb, dev, room_scene(dev, res, lt), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        c.scene.update(new.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False)
        assert scene_tables(c.scene) == scene_tables(ref.scene), lens
        if lens[0] > 0:
            assert scene_tables(ref.scene)["primary_edge_pmf"] != pin["primary_edge_pmf"]
    lt = (torch.tensor([0.3]), torch.tensor([5.0]))
    ref = native(rb, dev, room_scene(dev, res, lt), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    c.scene.set_camera(ref.camera)
    assert scene_tables(c.scene)["primary_edge_pmf"] == scene_tables(ref.scene)["primary_edge_pmf"]


def refusals_check(rb, dev):
    """Every refused combination raises with a message naming the lens."""
    import pytest
    import torch
    import scenes
    from redner_b200 import api

    def raises(fn, what="lens"):
        with pytest.raises(RuntimeError, match=what):
            fn()
    lens = (torch.tensor([0.2]), torch.tensor([4.0]))
    for ct in (1, 2, 3):  # orthographic, fisheye, panorama
        sc = scenes.glossy_room(dev, resolution=(8, 8), camera_type=ct)
        sc.camera.lens_radius, sc.camera.focus_distance = lens
        raises(lambda: native(rb, dev, sc))
    sc = scenes.glossy_room(dev, resolution=(8, 8), distortion=True)
    sc.camera.lens_radius, sc.camera.focus_distance = lens
    raises(lambda: native(rb, dev, sc))
    raises(lambda: native(rb, dev, room_scene(dev, 8, lens), pixel_filter=api.PixelFilter("tent", 2.0)))
    # an intrinsic matrix whose last row is not (0, 0, k): the distribution's bound on the circle of confusion assumes it
    sc = room_scene(dev, 8, lens)
    K = _intrinsic(40.0)
    K[2, 0] = 0.05
    sc.camera = lens_camera(8, _c2w([0.3, 1.4, -4.5], [0.0, 0.6, 0.0]), K, lens)
    raises(lambda: native(rb, dev, sc))
    sc.camera = lens_camera(8, _c2w([0.3, 1.4, -4.5], [0.0, 0.6, 0.0]), K, None)
    native(rb, dev, sc)  # (the pinhole takes it)
    for bad in ((-0.1, 4.0), (float("nan"), 4.0), (float("inf"), 4.0), (0.2, 0.0), (0.2, -1.0), (0.2, float("nan")), (0.2, float("inf"))):
        c = native(rb, dev, room_scene(dev, 8, None))
        cam = rb.Camera(8, 8, rb.float_ptr(0), rb.float_ptr(0), rb.float_ptr(0), api._ptr(rb, c.camera_args.cam_to_world),
                        api._ptr(rb, c.camera_args.world_to_cam), api._ptr(rb, c.camera_args.intrinsic_mat_inv), api._ptr(rb, c.camera_args.intrinsic_mat),
                        rb.float_ptr(0), 1e-2, rb.CameraType.perspective, rb.Vector2i(0, 0), rb.Vector2i(8, 8), lens_radius=bad[0], focus_distance=bad[1])
        raises(lambda: rb.Scene(cam, c.shapes, c.materials, c.lights, None, c.scene.use_gpu, c.scene.gpu_index, True, True))
        raises(lambda: c.scene.set_camera(cam))
        raises(lambda: c.scene.update(cam, c.shapes, c.materials, c.lights, None, geometry_changed=False))
    # a filtered scene and set_camera with a lens
    c = native(rb, dev, room_scene(dev, 8, None), pixel_filter=api.PixelFilter("tent", 2.0))
    raises(lambda: c.scene.set_camera(native(rb, dev, room_scene(dev, 8, lens)).camera))
    # rb_render: a screen-gradient image
    c = native(rb, dev, room_scene(dev, 8, lens))
    g = api.RenderFunction.gradient_buffers(c)
    grad_img, sg = torch.ones(8, 8, 3, device=dev), torch.zeros(8, 8, 2, device=dev)
    raises(lambda: rb.render(c.scene, c.options, rb.float_ptr(0), api._ptr(rb, grad_img), g.d_scene, api._ptr(rb, sg), rb.float_ptr(0)))


def deterministic_check(rb, dev, res, spp):
    """Deterministic mode with a lens: two runs and a run in many small bands give the same gradients, bit for bit."""
    import torch
    outs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for band in (None, "4096", None):
            if band:
                os.environ["RB_BAND_BYTES"] = band
            try:
                rt, ft = _lens_params(0.25, 4.0)
                sc = room_scene(dev, res, (rt, ft))
                loss, img = render_loss(rb, dev, sc, spp, 2, (9, 10))
                loss.backward()
                outs.append(torch.cat([rt.grad, ft.grad, _vertex_grads(sc)]).numpy())
            finally:
                os.environ.pop("RB_BAND_BYTES", None)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes()
    assert np.count_nonzero(outs[0][:2]) == 2


# ---------------------------------------------------------------------------------------------------- on the emulator
def _run(checks, timeout=3000):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_zero_radius_is_the_pinhole_bit_for_bit():
    _run(["zero_radius"])


def test_in_focus_plane_is_sharp():
    _run(["in_focus"])


def test_lens_equals_pinhole_average_primary_edges():
    _run(["average_glow"])


def test_lens_equals_pinhole_average_full():
    _run(["average_room"])


def test_lens_gradients_match_finite_differences():
    _run(["fd"])


def test_lens_update_equals_a_new_scene():
    _run(["update"])


def test_refused_combinations_name_the_lens():
    _run(["refusals"])


def test_deterministic_lens_gradients_repeat():
    _run(["deterministic"])


def _free_port():
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def _tile_worker(rank, world, port, emu_so, out_path):
    """One rank of a sharded lens render under deterministic algorithms (exact records summed over the ranks), the emulator behind the
    C ABI."""
    import torch
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import _lib, dist as rdist
    _lib._lib = _lib._bind(ctypes.CDLL(emu_so))  # this process only
    from redner_b200 import redner as rb
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cpu")
        rt, ft = _lens_params(0.25, 4.0)
        sc = room_scene(dev, 14, (rt, ft))
        img = rdist.render_tiles(sc, 2, 2, seed=5, rows_per_stripe=4, device=dev, backend=rb, use_primary_edge_sampling=True,
                                 use_secondary_edge_sampling=True)
        (weight_image(img.shape) * img).sum().backward()
        if rank == 0:
            np.savez(out_path, image=img.detach().numpy(), lens=torch.cat([rt.grad, ft.grad]).numpy(), vertices=_vertex_grads(sc).numpy())
    finally:
        dist.destroy_process_group()


def test_gloo_render_tiles_with_a_lens_is_independent_of_world_size(tmp_path):
    import torch.multiprocessing as mp
    from test_device_code_cpu import _build
    emu = _build()
    outs = {}
    for world in (1, 2):
        path = str(tmp_path / ("w%d.npz" % world))
        mp.spawn(_tile_worker, args=(world, _free_port(), emu, path), nprocs=world, join=True)
        outs[world] = dict(np.load(path))
    assert np.count_nonzero(outs[1]["lens"]) == 2 and np.count_nonzero(outs[1]["vertices"])
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
        if name == "zero_radius":
            zero_radius_check(rb, dev, 10, 2)
        elif name == "in_focus":
            in_focus_check(rb, dev, 12, 2)
        elif name == "average_glow":
            pinhole_average_check(rb, dev, "glow", 32, 16, 300)
        elif name == "average_room":
            pinhole_average_check(rb, dev, "room", 24, 8, 150, nontrivial=False)
        elif name == "fd":
            fd_check(rb, dev, 32, 64, 100)
        elif name == "update":
            update_check(rb, dev, 10)
        elif name == "refusals":
            refusals_check(rb, dev)
        elif name == "deterministic":
            deterministic_check(rb, dev, 8, 2)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
