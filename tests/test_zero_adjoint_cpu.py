"""CPU suite: the backward pass skips the samples of pixels whose image adjoint is exactly zero, on the host build of the device
headers (tools/cpu_emu).

Every term the backward pass computes for a pixel sample is a product with that pixel's d_image, and every sampler is a pure function
of (pixel, sample, depth), so leaving such samples out (pixel_adjoint_is_zero, edge_point_adjoint_is_zero in rb_render.cuh) must
change no gradient.  Each check renders one scene's backward pass twice, with the skip and with RB_NO_ZERO_CULL=1, and requires the
gradients, the camera gradients and the screen gradient to be bit-identical (on the emulator and in deterministic mode on the GPU).

Scenes: C2 at reduced size (spp 1, 3 and 64: pixels that share a warp with others, and whole-warp pixels), the textured glossy room
(2 bounces, both edge samplers), env_ball (misses that see the environment map), the fisheye room (non-linear primary edges), a tent
filter of width 2 (an edge point reads every pixel in its reach), a G-buffer channel list (radiance first, and radiance last: the
rad_dim offset), a screen_gradient_image, 2-way stripes of the viewport, and a viewport inside the image (edge points outside it read
the clamped border pixel).  d_images: the natural 2 img; a dense one with zeroed
8 x 8 tiles; with a single zero row; zero in only some channels of some pixels (must not be skipped); a NaN pixel (must not be
skipped: its NaN reaches the gradients either way).
The device side is tests/test_zero_adjoint_gpu.py, which calls the checks below.

Run as a script (`python tests/test_zero_adjoint_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# name -> (scene, resolution, spp, max_bounces, edge samplers (1 primary | 2 secondary), options)
CASES = {
    # (at 1 spp the NaN pixel's one sample reaches no differentiable parameter)
    "c2_spp1": ("shadow_blocker", 24, 1, 1, 3, {"nan_unseen": True}),
    "c2_spp3": ("shadow_blocker", 24, 3, 1, 3, {}),
    "c2_spp64": ("shadow_blocker", 16, 64, 1, 3, {}),
    "glossy_room": ("glossy_room", 16, 3, 2, 3, {}),
    "env_ball": ("env_ball", 16, 3, 2, 1, {}),
    "fisheye_room": ("fisheye_room", 16, 2, 1, 1, {}),
    "tent2": ("glossy_room", 16, 3, 1, 3, {"filter": "tent2"}),
    "gbuffer": ("glossy_room", 12, 2, 1, 1, {"channels": ["radiance", "depth", "position", "uv", "diffuse_reflectance", "alpha"]}),
    "gbuffer_radiance_last": ("glossy_room", 12, 2, 1, 1, {"channels": ["depth", "shading_normal", "radiance"]}),
    "screen_gradient": ("single_triangle", 16, 3, 1, 1, {"screen": True}),
    "stripes": ("glossy_room", 16, 3, 1, 3, {"parts": 2}),
    # a viewport inside the image: primary-edge points outside it read the clamped border pixel of the viewport
    "viewport": ("glossy_room", 16, 3, 1, 3, {"viewport": (3, 5, 13, 12)}),
}
D_IMAGES = ["natural", "tiles", "row", "some_channels", "nan_pixel"]


def d_image(kind, img):
    """The image adjoint `kind` for the rendered image `img` ([H, W, C] float32 tensor)."""
    import torch
    h, w, nch = img.shape
    if kind == "natural":  # loss = sum(img^2)
        return (2 * img).contiguous()
    g = torch.Generator().manual_seed(7)
    d = (0.25 + torch.rand(h, w, nch, generator=g)).to(img.device)  # dense: no zero but those put in below
    if kind == "tiles":  # every other 8 x 8 tile, checkerboard
        ty, tx = torch.meshgrid(torch.arange(h) // 8, torch.arange(w) // 8, indexing="ij")
        d[((ty + tx) % 2 == 0).to(img.device)] = 0.0
    elif kind == "row":
        d[h // 2] = 0.0
    elif kind == "some_channels":  # pixels with SOME zero floats still carry an adjoint
        d[::2, :, 0] = 0.0
        d[:, ::3, nch - 1] = -0.0
        d[1::4, 1::4, :] = 0.0  # (and a few wholly zero ones)
    elif kind == "nan_pixel":  # in a pixel of the upper half that sees something lit (the median such pixel), the lower half zero
        lum = img[: h // 2].sum(-1).flatten().cpu()
        lit = torch.nonzero(lum > 0).flatten()
        p = int(lit[torch.argsort(lum[lit])[len(lit) // 2]]) if len(lit) else (h // 4) * w + w // 2
        d[p // w, p % w, 0] = float("nan")
        d[h // 2:] = 0.0
    else:
        raise ValueError(kind)
    return d.contiguous()


def _make_scene(dev, name):
    import scenes
    scene, res = CASES[name][:2]
    sc = scenes.SCENES[scene](dev, resolution=(res, res))
    if "viewport" in CASES[name][5]:
        sc.camera.viewport = CASES[name][5]["viewport"]
    return sc


def backward_outputs(rb, dev, name, kind, seed=3):
    """{output name: numpy array} of one backward pass of case `name` with image adjoint `kind`: every gradient RenderFunction returns
    (camera included) and, for the screen-gradient case, the screen gradient; for the stripes case, those of every part."""
    import torch
    from redner_b200 import api
    from test_pixel_filter_cpu import pixel_filter
    _, _, spp, mb, edges, opt = CASES[name]
    chans = [getattr(rb.channels, c) for c in opt["channels"]] if "channels" in opt else None
    args = api.RenderFunction.serialize_scene(_make_scene(dev, name), spp, mb, channels=chans, sampler_type=rb.SamplerType.sobol, device=dev,
                                              backend=rb, use_primary_edge_sampling=bool(edges & 1), use_secondary_edge_sampling=bool(edges & 2),
                                              pixel_filter=pixel_filter(opt.get("filter")))
    c = api.RenderFunction._unpack((seed, seed + 1000003), args)
    d = d_image(kind, api._render(c))
    out = {}
    parts = opt.get("parts", 1)
    for part in range(parts):
        if parts > 1:
            c.scene.set_partition(part, parts, 4)
        sg = torch.zeros(*d.shape[:2], 2, device=dev) if opt.get("screen") else None
        g = api.RenderFunction.gradient_buffers(c)
        # (rb.render directly: api._backward refuses a d_image that is not finite)
        rc = rb.render(c.scene, api.RenderFunction.backward_options(c), rb.float_ptr(0), api._ptr(rb, d), g.d_scene, api._ptr(rb, sg), rb.float_ptr(0))
        assert rc is None or rc == 0, rc
        for i, t in enumerate(api.RenderFunction.gradient_outputs(c, g)):
            if isinstance(t, torch.Tensor):
                out["part%d.arg%03d" % (part, i)] = t.detach().cpu().numpy().copy()
        if sg is not None:
            out["part%d.screen" % part] = sg.cpu().numpy()
    assert any(np.count_nonzero(v) for v in out.values()), (name, kind)
    return out


def both_ways(rb, dev, name, kind):
    """(outputs with the skip, outputs with RB_NO_ZERO_CULL=1)."""
    os.environ.pop("RB_NO_ZERO_CULL", None)
    skip = backward_outputs(rb, dev, name, kind)
    os.environ["RB_NO_ZERO_CULL"] = "1"
    try:
        full = backward_outputs(rb, dev, name, kind)
    finally:
        os.environ.pop("RB_NO_ZERO_CULL", None)
    assert set(skip) == set(full)
    return skip, full


def assert_bit_identical(skip, full, what):
    for k in full:
        assert skip[k].tobytes() == full[k].tobytes(), (what, k, np.abs(skip[k].astype(np.float64) - full[k]).max(),
                                                        int(np.isnan(skip[k]).sum()), int(np.isnan(full[k]).sum()))


def check_case(rb, dev, name, kinds=D_IMAGES):
    for kind in kinds:
        skip, full = both_ways(rb, dev, name, kind)
        assert_bit_identical(skip, full, (name, kind))
        if kind == "nan_pixel" and not CASES[name][5].get("nan_unseen"):  # its samples were traced: the NaN reached a gradient
            assert any(np.isnan(v).any() for v in full.values()), name


# ---------------------------------------------------------------------------------------------------- on the emulator
def _run(checks, timeout=1800):
    from test_device_code_cpu import _build
    so = _build()
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + checks, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + c for c in checks]


def test_c2_one_sample_per_pixel():
    _run(["c2_spp1"])


def test_c2_three_samples_per_pixel():
    _run(["c2_spp3"])


def test_c2_sixty_four_samples_per_pixel():
    _run(["c2_spp64"])


def test_glossy_room_both_edge_samplers():
    _run(["glossy_room"])


def test_env_ball_misses_see_the_environment_map():
    _run(["env_ball"])


def test_fisheye_room_primary_edges():
    _run(["fisheye_room"])


def test_tent_filter_reach():
    _run(["tent2"])


def test_gbuffer_channels():
    _run(["gbuffer", "gbuffer_radiance_last"])


def test_screen_gradient():
    _run(["screen_gradient"])


def test_two_way_stripes():
    _run(["stripes"])


def test_viewport_inside_the_image():
    _run(["viewport"])


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
        check_case(rb, dev, name)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
