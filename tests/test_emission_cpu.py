"""CPU suite: emission textures of area lights (rb_area_light::emission, DESIGN.md section "Emission textures"), on the host emulator.

- Identity: a constant emission texture of value 1 renders, bit for bit, the image and the intensity and vertex gradients of the same light
  without a texture (general kernels, deterministic mode, one-sided lights); a constant texture c matches an intensity of intensity * c.
- Closed form: an orthographic camera looks at a textured quad light that fills the image (sample_pixel_center, max_bounces 0).  The
  image is intensity * E(uv) at the uv of every pixel (E bilinear, read at the uv the G-buffer reports there), d(texels) is the
  transposed lookup of d_image * intensity and d(intensity) is sum(d_image * E(uv)), for 1- and 3-channel textures; with a uv_scale that
  requires grad, d(uv_scale) is sum(d_E * (dE/du * u, dE/dv * v)).
- Finite differences (fd_check of the pixel-filter suite) on a textured lamp above a diffuse floor with both edge samplers on: a texel,
  the intensity and the light's uvs; a vertex of the light seen from the front; and the texels of a two-sided lamp whose back face the
  camera sees (the first-hit adjoint under the forward's two-sided condition).
- Adding, changing and removing a texture with rb_scene_update equals a new scene (light tables byte for byte, images bit for bit).
- Every refusal names the emission texture.
- Deterministic mode is bitwise repeatable; the record count and fingerprint change with a texture and are today's without one; a gloo
  render_tiles of a textured scene at world size 2 equals world size 1.

Run as a script (`python tests/test_emission_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the emulator in
place of the library; tests/test_emission_gpu.py calls the same checks on the GPU."""
import ctypes
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


# ---------------------------------------------------------------------------------------------------- scenes
def _quad(z, half, flip=False, cx=0.0, cy=0.0):
    import torch
    v = torch.tensor([[cx - half, cy - half, z], [cx + half, cy - half, z], [cx + half, cy + half, z], [cx - half, cy + half, z]])
    idx = torch.tensor([[0, 2, 1], [0, 3, 2]] if flip else [[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    uvs = torch.tensor([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]])
    return v, idx, uvs


def texture_image(h, w, ch, seed=3):
    import torch
    g = torch.Generator().manual_seed(seed)
    return (0.2 + 1.6 * torch.rand(h, w, ch, generator=g)).contiguous()


def ramp_image(h, w, ch):
    """A smooth texture (ramps in u and v), so that moving the uvs or uv_scale changes the lamp's light by more than the noise."""
    import torch
    x = (torch.arange(w) + 0.5) / w
    y = (torch.arange(h) + 0.5) / h
    c = torch.arange(ch) + 1.0
    return (0.3 + 1.2 * x[None, :, None] * c / ch + 0.4 * y[:, None, None]).expand(h, w, ch).contiguous()


def direct_view(dev, res, ch, tex_size=None, uv_scale=None):
    """An orthographic camera looking down -z at a one-sided textured quad light that fills the image; its texture is tex_size square
    (default: the image's size), with the given uv_scale (default: 1, without a gradient)."""
    import torch
    from redner_b200 import api
    cam = api.Camera(position=torch.tensor([0.0, 0.0, 2.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([90.0]), clip_near=1e-2, resolution=(res, res), camera_type=1)
    v, idx, uvs = _quad(0.0, 1.0)
    mat = api.Material(torch.tensor([0.0, 0.0, 0.0], device=dev))
    shape = api.Shape(v.to(dev), idx.to(dev), 0, uvs=uvs.to(dev).contiguous())
    n = tex_size or res
    tex = texture_image(n, n, ch).to(dev).requires_grad_()
    if uv_scale is not None:
        tex = api.Texture(tex, uv_scale=torch.tensor(uv_scale, device=dev, requires_grad=True))
    light = api.AreaLight(0, torch.tensor([1.5, 0.75, 0.5], requires_grad=True), emission=tex)
    return api.Scene(cam, [shape], [mat], [light])


def lamp(dev, res, emission="image", two_sided=False, faces_camera=False, ch=3):
    """A textured quad lamp above a diffuse floor, seen from above by a perspective camera.  By default the lamp's normal points down: it
    lights the floor with its front face, and the camera sees its back face.  `faces_camera`: the normal points up, to the camera, which
    then sees the front face, and the floor sees the back (lit only when the lamp is two-sided)."""
    import torch
    from redner_b200 import api
    cam = api.Camera(position=torch.tensor([0.0, -2.6, 2.4]), look_at=torch.tensor([0.0, 0.0, 0.5]), up=torch.tensor([0.0, 0.0, 1.0]),
                     fov=torch.tensor([50.0]), clip_near=1e-2, resolution=(res, res))
    fv, fi, fuv = _quad(0.0, 2.0)
    lv, li, luv = _quad(1.0, 0.6, flip=not faces_camera)  # flip: the lamp's normal points down, to the floor
    lv = lv + torch.tensor([0.1, 0.2, 0.0])
    lv.requires_grad_()
    luv = luv.clone().requires_grad_()
    floor = api.Shape(fv.to(dev).requires_grad_(), fi.to(dev), 0, uvs=fuv.to(dev))
    light_shape = api.Shape(lv.to(dev).detach().requires_grad_(), li.to(dev), 1, uvs=luv.to(dev).detach().requires_grad_())
    mats = [api.Material(torch.tensor([0.6, 0.55, 0.5], device=dev)), api.Material(torch.tensor([0.0, 0.0, 0.0], device=dev))]
    if emission == "image":
        tex = api.Texture(ramp_image(8, 8, ch).to(dev).requires_grad_(), uv_scale=torch.tensor([1.0, 1.0], device=dev, requires_grad=True))
    elif emission is None:
        tex = None
    else:
        tex = api.Texture(torch.tensor(emission, device=dev).requires_grad_())
    light = api.AreaLight(1, torch.tensor([4.0, 3.5, 3.0], requires_grad=True), two_sided=two_sided, emission=tex)
    return api.Scene(cam, [floor, light_shape], mats, [light])


def render(rb, dev, sc, spp, seed, mb=1, backward=True, grad_w=None, **kw):
    """(image, gradients) of loss = sum(W * img)."""
    import torch
    from redner_b200 import api
    import test_pixel_filter_cpu as pf
    kw.setdefault("sampler_type", rb.SamplerType.independent)
    args = api.RenderFunction.serialize_scene(sc, spp, mb, device=dev, backend=rb, **kw)
    img = api.RenderFunction.apply(seed, *args)
    grads = {}
    if backward:
        w = grad_w if grad_w is not None else pf.weight_image(img.shape).to(img.device)
        (w * img).sum().backward()
        grads = collect(sc)
    return img.detach().cpu(), grads


def collect(sc):
    out = {}
    for i, s in enumerate(sc.shapes):
        for k in ("vertices", "uvs"):
            t = getattr(s, k)
            if t is not None and t.grad is not None:
                out["shape%d.%s" % (i, k)] = t.grad.detach().cpu().clone()
    for i, l in enumerate(sc.area_lights):
        if l.intensity.grad is not None:
            out["light%d.intensity" % i] = l.intensity.grad.detach().cpu().clone()
        if l.emission is not None:
            if l.emission.texels.grad is not None:
                out["light%d.texels" % i] = l.emission.texels.grad.detach().cpu().clone()
            if l.emission.uv_scale.grad is not None:
                out["light%d.uv_scale" % i] = l.emission.uv_scale.grad.detach().cpu().clone()
    return out


def _bytes_equal(a, b, keys=None):
    for k in keys or a:
        assert a[k].numpy().tobytes() == b[k].numpy().tobytes(), k


# ---------------------------------------------------------------------------------------------------- checks
def identity_check(rb, dev, res=12, spp=8):
    import torch
    os.environ["RB_NO_LEAN"] = "1"
    try:
        torch.use_deterministic_algorithms(True, warn_only=True)
        for mb in (0, 1):
            a_img, a = render(rb, dev, lamp(dev, res, emission=None), spp, 4, mb=mb)
            b_img, b = render(rb, dev, lamp(dev, res, emission=[1.0, 1.0, 1.0]), spp, 4, mb=mb)
            assert a_img.numpy().tobytes() == b_img.numpy().tobytes()
            _bytes_equal(a, b, ["light0.intensity", "shape0.vertices", "shape1.vertices"])
        # a constant c against an intensity of intensity * c
        c = [0.5, 2.0, 1.25]
        sc = lamp(dev, res, emission=c)
        ref = lamp(dev, res, emission=None)
        ref.area_lights[0].intensity = (ref.area_lights[0].intensity.detach() * torch.tensor(c)).requires_grad_()
        x, _ = render(rb, dev, sc, spp, 4, backward=False)
        y, _ = render(rb, dev, ref, spp, 4, backward=False)
        assert torch.allclose(x, y, rtol=1e-5, atol=1e-6), (x - y).abs().max()
    finally:
        torch.use_deterministic_algorithms(False)
        del os.environ["RB_NO_LEAN"]


def _bilinear(tex, uv, grad=False):
    """E(uv) at level 0 (uv already scaled, wrapping) and the taps: [(index (y, x), weight)] per pixel; with `grad` also dE/du and dE/dv."""
    h, w, _ = tex.shape
    x, y = uv[..., 0] * w - 0.5, uv[..., 1] * h - 0.5
    xf, yf = np.floor(x).astype(int), np.floor(y).astype(int)
    fx, fy = x - xf, y - yf
    ff, cf, fc, cc = (yf % h, xf % w), (yf % h, (xf + 1) % w), ((yf + 1) % h, xf % w), ((yf + 1) % h, (xf + 1) % w)
    taps = [(ff, (1 - fx) * (1 - fy)), (cf, fx * (1 - fy)), (fc, (1 - fx) * fy), (cc, fx * fy)]
    val = sum(tex[i][..., :] * wt[..., None] for i, wt in taps)
    if not grad:
        return val, taps
    du = w * ((tex[cf] - tex[ff]) * (1 - fy)[..., None] + (tex[cc] - tex[fc]) * fy[..., None])
    dv = h * ((tex[fc] - tex[ff]) * (1 - fx)[..., None] + (tex[cc] - tex[cf]) * fx[..., None])
    return val, taps, du, dv


def direct_view_check(rb, dev, res=16):
    """Image, intensity and texel gradients for a texture of the image's size (pixel centres on texel centres) and, with a uv_scale that
    requires grad, for a texture of half the size (a footprint below one texel: level 0 alone), whose uv_scale gradient is then
    sum(dE * (dE/du * u, dE/dv * v)) over the pixels."""
    import torch
    for ch, size, scale in ((1, None, None), (3, None, None), (1, res // 2, (0.9, 1.1)), (3, res // 2, (0.9, 1.1))):
        sc = direct_view(dev, res, ch, tex_size=size, uv_scale=scale)
        uvimg, _ = render(rb, dev, sc, 1, 0, mb=0, backward=False, channels=[rb.channels.uv], sample_pixel_center=True)
        uv = uvimg.numpy().astype(np.float64)
        s = np.array(scale if scale is not None else (1.0, 1.0))
        d_img = torch.rand(res, res, 3, generator=torch.Generator().manual_seed(7))
        img, g = render(rb, dev, sc, 1, 0, mb=0, grad_w=d_img.to(dev), sample_pixel_center=True, use_primary_edge_sampling=False,
                        use_secondary_edge_sampling=False)
        tex = sc.area_lights[0].emission.texels.detach().cpu().numpy().astype(np.float64)
        I = np.array([1.5, 0.75, 0.5])
        E, taps, E_u, E_v = _bilinear(tex, uv * s, grad=True)
        E3 = np.broadcast_to(E, (res, res, 3)) if ch == 1 else E
        np.testing.assert_allclose(img.numpy(), I * E3, rtol=1e-5, atol=1e-7)
        dI = (d_img.numpy() * E3).reshape(-1, 3).sum(0)
        np.testing.assert_allclose(g["light0.intensity"].numpy(), dI, rtol=1e-5)
        dE = d_img.numpy() * I
        if ch == 1:
            dE = dE.sum(-1, keepdims=True)
        dtex = np.zeros_like(tex)
        for (iy, ix), wt in taps:
            np.add.at(dtex, (iy, ix), dE * wt[..., None])
        # (a texel of the half-size texture sums the bilinear weights of a dozen pixels, each computed in float from the pixel's uv)
        np.testing.assert_allclose(g["light0.texels"].numpy(), dtex, rtol=1e-5 if size is None else 1e-4, atol=1e-6)
        if scale is not None:
            ds = np.array([((dE * E_u).sum(-1) * uv[..., 0]).sum(), ((dE * E_v).sum(-1) * uv[..., 1]).sum()])
            assert abs(ds).min() > 1e-2, ds
            np.testing.assert_allclose(g["light0.uv_scale"].numpy(), ds, rtol=1e-4)


def fd_checks(rb, dev, res, spp, fd_spp, seeds):
    import torch
    import test_pixel_filter_cpu as pf

    def make_lamp(**kw):
        return lambda: lamp(dev, res, **kw)

    def moves(sc_of, getter, index):
        def move(sc, d):
            with torch.no_grad():
                getter(sc).view(-1)[index] += d
                for light in sc.area_lights:  # (the mip pyramid is built from the texels when they are set)
                    if light.emission is not None:
                        light.emission.texels = light.emission.texels

        def grad_of(sc):
            t = getter(sc)
            return float(t.grad.view(-1)[index]) if t.grad is not None else 0.0
        return move, grad_of

    cases = [
        ("texel", make_lamp(), lambda sc: sc.area_lights[0].emission.texels, 3 * (8 * 3 + 4) + 1, 0.2, 1),
        ("intensity", make_lamp(), lambda sc: sc.area_lights[0].intensity, 1, 0.2, 1),
        ("light uvs", make_lamp(), lambda sc: sc.shapes[1].uvs, 2 * 2, 0.05, 1),
        # (the camera sees the lamp's front face, emission only: the texture slides over the moving surface and its silhouette carries
        # textured radiance.  Under light sampling the light-vertex gradient leaves out the MIS weight's derivative, as the reference does,
        # with or without a texture: DESIGN.md section 7)
        ("light vertex", make_lamp(faces_camera=True), lambda sc: sc.shapes[1].vertices, 3 * 1 + 0, 0.03, 0),
        # (the camera sees the back face of a two-sided lamp, emission only: the first-hit adjoint under the forward's two-sided condition;
        # the reference's gate, dot(wi, n) > 0, would give no gradient at all here)
        ("two-sided texel, from behind", make_lamp(two_sided=True), lambda sc: sc.area_lights[0].emission.texels, 3 * (8 * 4 + 3), 0.2, 0),
    ]
    for name, make, getter, index, eps, mb in cases:
        move, grad_of = moves(make, getter, index)
        pf.fd_check(rb, dev, make, move, grad_of, None, spp, fd_spp, seeds, eps, mb=mb, rel=0.05)
        print("fd", name, flush=True)


def _desc_scene(rb, dev, sc, **kw):
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, 4, 1, device=dev, backend=rb, **kw)
    return api.RenderFunction._unpack((1, 2), args), args


def update_check(rb, dev, res=10):
    """Adding, changing and removing a texture through Scene.update equals a new scene."""
    from redner_b200 import api
    states = [dict(emission=None), dict(emission="image"), dict(emission=[0.5, 1.0, 2.0]), dict(emission=None)]
    c0, keep0 = _desc_scene(rb, dev, lamp(dev, res, **states[0]))
    scene = c0.scene
    for st in states[1:]:
        c, keep = _desc_scene(rb, dev, lamp(dev, res, **st))
        scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False)
        for name in ("lights", "light_pmf", "light_cdf", "light_areas", "area_cdf_pool", "area_cdf_offsets"):
            assert scene.table(name).tobytes() == c.scene.table(name).tobytes(), name
        c.scene, fresh = scene, c.scene
        a = api._render(c)
        c.scene = fresh
        b = api._render(c)
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), st


def refusals_check(rb, dev):
    import torch
    from redner_b200 import _lib as L
    c, keep = _desc_scene(rb, dev, lamp(dev, 8))
    t = torch.ones(4, 4, 3, device=dev)
    uvs = torch.ones(2, device=dev)

    def tex(channels=3, levels=1, width=4, height=4, texels=True, uv=True):
        e = L.rb_texture()
        e.num_levels, e.channels = levels, channels
        for k in range(max(0, min(levels, L.RB_MAX_MIP_LEVELS))):
            e.texels[k] = t.data_ptr() if texels else None
            e.width[k], e.height[k] = width, height
        e.uv_scale = uvs.data_ptr() if uv else None
        return e

    bad = [tex(channels=2), tex(levels=9), tex(levels=-1), tex(width=0, height=4), tex(texels=False), tex(uv=False)]
    for e in bad:
        for build in (True, False):
            c.lights[0]._c.emission = e
            try:
                if build:
                    rb.Scene(c.camera, c.shapes, c.materials, c.lights, None, dev.type == "cuda", -1, True, True)
                else:
                    c.scene.update(c.camera, c.shapes, c.materials, c.lights, None, geometry_changed=False)
            except RuntimeError as err:
                assert "emission texture" in str(err), str(err)
            else:
                raise AssertionError("accepted a bad emission texture")
    # rb_render: a gradient pyramid of another shape
    c, keep = _desc_scene(rb, dev, lamp(dev, 8))
    from redner_b200 import api
    g = api.RenderFunction.gradient_buffers(c)
    g.d_scene._emission[0].width[0] = 5
    img = torch.zeros(8, 8, 3, device=dev)
    try:
        rb.render(c.scene, c.options, rb.float_ptr(0), rb.float_ptr(img.data_ptr()), g.d_scene, rb.float_ptr(0), rb.float_ptr(0))
    except RuntimeError as err:
        assert "emission texture" in str(err), str(err)
    else:
        raise AssertionError("accepted a bad emission gradient")


def deterministic_check(rb, dev, res=12, spp=8):
    import torch
    from redner_b200 import api
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a = render(rb, dev, lamp(dev, res), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        b = render(rb, dev, lamp(dev, res), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        assert a[0].numpy().tobytes() == b[0].numpy().tobytes()
        assert set(a[1]) >= {"light0.texels", "light0.uv_scale", "light0.intensity", "shape1.uvs"}
        _bytes_equal(a[1], b[1])
        if dev.type == "cuda":
            os.environ["RB_BAND_BYTES"] = "65536"
            try:
                c = render(rb, dev, lamp(dev, res), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
            finally:
                del os.environ["RB_BAND_BYTES"]
            _bytes_equal(a[1], c[1])
    finally:
        torch.use_deterministic_algorithms(False)
    # records: a texture adds its levels and uv_scale; without one, the count and fingerprint are the untextured scene's
    counts = {}
    for name, em in (("none", None), ("image", "image")):
        c, keep = _desc_scene(rb, dev, lamp(dev, res, emission=em))
        g = api.RenderFunction.gradient_buffers(c)
        counts[name] = rb.exact_record_count(c.scene, c.options, g.d_scene)
    c, keep = _desc_scene(rb, dev, lamp(dev, res, emission=None))
    g = api.RenderFunction.gradient_buffers(c)
    g.d_scene._c.light_emission = (L_rb_texture_array(1))
    assert rb.exact_record_count(c.scene, c.options, g.d_scene) == counts["none"]
    assert counts["image"][0] == counts["none"][0] + sum(m.numel() for m in lamp(dev, res).area_lights[0].emission.mipmap) + 2
    assert counts["image"][1] != counts["none"][1]


def L_rb_texture_array(n):
    from redner_b200 import _lib as L
    return (L.rb_texture * n)()


def compare_render(rb, dev, res=16, spp=16):
    """Image and texture / light gradients of the textured lamp (both edge samplers), for the GPU-against-emulator comparison."""
    img, g = render(rb, dev, lamp(dev, res), spp, 9, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    out = {"image": img.numpy()}
    out.update({k: v.numpy() for k, v in g.items() if "vertices" not in k})
    return out


# ---------------------------------------------------------------------------------------------------- pytest (emulator in a subprocess)
def _run(checks, timeout=2400):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_constant_texture_of_one_is_no_texture_bit_for_bit():
    _run(["identity"])


def test_direct_view_matches_the_closed_form():
    _run(["direct"])


def test_emission_gradients_match_finite_differences():
    _run(["fd"])


def test_texture_update_equals_a_new_scene():
    _run(["update"])


def test_bad_emission_textures_are_refused():
    _run(["refusals"])


def test_deterministic_repeatable_and_records():
    _run(["deterministic"])


def _free_port():
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def _tile_worker(rank, world, port, emu_so, out_path):
    """One rank of a sharded render of the textured lamp under deterministic algorithms (exact records summed over the ranks), the
    emulator behind the C ABI."""
    import torch
    import torch.distributed as dist
    sys.path.insert(0, HERE)
    from redner_b200 import _lib, dist as rdist
    _lib._lib = _lib._bind(ctypes.CDLL(emu_so))  # this process only
    from redner_b200 import redner as rb
    import test_pixel_filter_cpu as pf
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cpu")
        sc = lamp(dev, 14)
        img = rdist.render_tiles(sc, 2, 1, seed=5, rows_per_stripe=4, device=dev, backend=rb, use_primary_edge_sampling=True,
                                 use_secondary_edge_sampling=True)
        (pf.weight_image(img.shape) * img).sum().backward()
        if rank == 0:
            np.savez(out_path, image=img.detach().numpy(), **{k: v.numpy() for k, v in collect(sc).items()})
    finally:
        dist.destroy_process_group()


def test_gloo_render_tiles_with_an_emission_texture_is_independent_of_world_size(tmp_path):
    import torch.multiprocessing as mp
    from test_device_code_cpu import _build
    emu = _build()
    outs = {}
    for world in (1, 2):
        path = str(tmp_path / ("w%d.npz" % world))
        mp.spawn(_tile_worker, args=(world, _free_port(), emu, path), nprocs=world, join=True)
        outs[world] = dict(np.load(path))
    assert {"light0.texels", "light0.uv_scale", "light0.intensity", "shape1.uvs", "shape1.vertices"} <= set(outs[1])
    assert np.count_nonzero(outs[1]["light0.texels"]) and np.count_nonzero(outs[1]["light0.uv_scale"])
    assert set(outs[2]) == set(outs[1])
    for k in outs[1]:
        assert outs[2][k].tobytes() == outs[1][k].tobytes(), k


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    dev = torch.device("cpu")
    for name in names:
        if name == "identity":
            identity_check(rb, dev)
        elif name == "direct":
            direct_view_check(rb, dev)
        elif name == "fd":
            fd_checks(rb, dev, 12, 16, 128, 4)
        elif name == "update":
            update_check(rb, dev)
        elif name == "refusals":
            refusals_check(rb, dev)
        elif name == "deterministic":
            deterministic_check(rb, dev)
        elif name.startswith("compare:"):
            np.savez(name[len("compare:"):], **compare_render(rb, dev))
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
