"""GPU suite: emission textures of area lights (the host emulator runs the same checks at small sizes in tests/test_emission_cpu.py).

- Unbiasedness under MIS: an orthographic camera looks down on a Lambertian floor lit by a textured quad light it does not see
  (sample_pixel_center, max_bounces 1, light samples and BSDF samples weighed by MIS).  Per-pixel means over independent renders match a
  float64 quadrature of kd / pi * integral of Le(x') cos cos' / r^2 dA' over the bilinear texture, for one- and two-sided lights and 1- and
  3-channel textures.
- The closed-form direct view, the finite differences and the deterministic checks of the CPU suite at larger sizes.
- The GPU and the emulator agree on the image and every texture and light gradient to 1e-5 relative L2.
- A textured scene renders bit for bit the same with and without RB_NO_LEAN=1: it runs the general kernels.
"""
import math

import numpy as np
import pytest
import torch

import test_emission_cpu as em
from redner_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


KD = 0.7
INTENSITY = np.array([3.0, 2.0, 1.5])
LIGHT = dict(x0=1.4, x1=2.4, y0=-0.5, y1=0.5, z=1.0)


def mis_scene(dev, res, two_sided, ch):
    """The floor z = 0 seen from above by an orthographic camera covering [-1, 1]^2; the light, a quad beside the view at height 1, faces
    the floor (one-sided) or away from it (two-sided: the floor sees its back)."""
    cam = api.Camera(position=torch.tensor([0.0, 0.0, 3.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([90.0]), clip_near=1e-2, resolution=(res, res), camera_type=1)
    fv = torch.tensor([[-4.0, -4.0, 0.0], [4.0, -4.0, 0.0], [4.0, 4.0, 0.0], [-4.0, 4.0, 0.0]])
    fi = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    L = LIGHT
    lv = torch.tensor([[L["x0"], L["y0"], L["z"]], [L["x1"], L["y0"], L["z"]], [L["x1"], L["y1"], L["z"]], [L["x0"], L["y1"], L["z"]]])
    li = torch.tensor([[0, 1, 2], [0, 2, 3]] if two_sided else [[0, 2, 1], [0, 3, 2]], dtype=torch.int32)
    luv = torch.tensor([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]])
    shapes = [api.Shape(fv.to(dev), fi.to(dev), 0), api.Shape(lv.to(dev), li.to(dev), 1, uvs=luv.to(dev))]
    mats = [api.Material(torch.tensor([KD, KD, KD], device=dev)), api.Material(torch.tensor([0.0, 0.0, 0.0], device=dev))]
    tex = em.texture_image(8, 8, ch, seed=5).to(dev)
    light = api.AreaLight(1, torch.tensor(INTENSITY, dtype=torch.float32), two_sided=two_sided, directly_visible=False, emission=tex)
    return api.Scene(cam, shapes, mats, [light]), tex.cpu().numpy().astype(np.float64)


def quadrature(points, tex, n=256):
    """kd / pi * integral of I E(uv) cos cos' / r^2 dA' over the light, per floor point (float64, midpoint rule)."""
    L = LIGHT
    s = (np.arange(n) + 0.5) / n
    u, v = np.meshgrid(s, s, indexing="xy")
    E, _ = em._bilinear(tex, np.stack([u, v], -1))
    if E.shape[-1] == 1:
        E = np.repeat(E, 3, -1)
    xs = L["x0"] + u * (L["x1"] - L["x0"])
    ys = L["y0"] + v * (L["y1"] - L["y0"])
    dA = (L["x1"] - L["x0"]) * (L["y1"] - L["y0"]) / (n * n)
    out = np.zeros(points.shape[:-1] + (3,))
    for idx in np.ndindex(points.shape[:-1]):
        p = points[idx]
        d = np.stack([xs - p[0], ys - p[1], np.full_like(xs, L["z"] - p[2])], -1)
        r2 = (d * d).sum(-1)
        cos_f = d[..., 2] / np.sqrt(r2)  # at the floor (normal +z) and at the light (normal -z): the same
        g = cos_f * cos_f / r2
        out[idx] = KD / math.pi * INTENSITY * (E * g[..., None]).sum((0, 1)) * dA
    return out


@pytest.mark.parametrize("two_sided", [False, True])
@pytest.mark.parametrize("ch", [1, 3])
def test_textured_light_is_unbiased_under_mis(rb, two_sided, ch):
    dev = torch.device("cuda:0")
    res, spp, runs = 16, 256, 24
    sc, tex = mis_scene(dev, res, two_sided, ch)
    args = api.RenderFunction.serialize_scene(sc, spp, 1, device=dev, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False, channels=[rb.channels.position])
    pos = api.RenderFunction.apply(0, *args).cpu().numpy().astype(np.float64)
    ref = quadrature(pos, tex)
    args = api.RenderFunction.serialize_scene(sc, spp, 1, device=dev, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False)
    imgs = np.stack([api.RenderFunction.apply(100 + k, *args).cpu().numpy().astype(np.float64) for k in range(runs)])
    mean, se = imgs.mean(0), imgs.std(0, ddof=1) / math.sqrt(runs)
    assert ref.min() > 0 and mean.min() > 0
    z = (mean - ref) / np.maximum(se, 1e-12)
    # per pixel within 4 standard errors (a few of 768 pixel channels may stray by chance), and the image total within 4 of its own
    assert (np.abs(z) > 4).mean() < 0.01, np.abs(z).max()
    tot = imgs.sum((1, 2, 3))
    assert abs(tot.mean() - ref.sum()) <= 4 * tot.std(ddof=1) / math.sqrt(runs), (tot.mean(), ref.sum())


def test_direct_view_matches_the_closed_form(rb):
    em.direct_view_check(rb, torch.device("cuda:0"), res=64)


def test_emission_gradients_match_finite_differences(rb):
    em.fd_checks(rb, torch.device("cuda:0"), 32, 64, 512, 6)


def test_deterministic_repeatable_band_independent_and_records(rb):
    em.deterministic_check(rb, torch.device("cuda:0"), res=48, spp=8)


def test_texture_update_equals_a_new_scene(rb):
    em.update_check(rb, torch.device("cuda:0"), res=32)


def test_bad_emission_textures_are_refused(rb):
    em.refusals_check(rb, torch.device("cuda:0"))


def test_textured_scene_runs_the_general_kernels(rb, monkeypatch):
    dev = torch.device("cuda:0")
    a = em.render(rb, dev, em.lamp(dev, 64), 4, 7, backward=False)[0].numpy()
    monkeypatch.setenv("RB_NO_LEAN", "1")
    b = em.render(rb, dev, em.lamp(dev, 64), 4, 7, backward=False)[0].numpy()
    assert float(np.abs(a).sum()) > 0
    assert a.tobytes() == b.tobytes()


def test_gpu_matches_the_emulator(rb, tmp_path):
    """The textured lamp on the GPU and on the host build of the same headers (tools/cpu_emu), same seed and samples: the image and every
    texture and light gradient agree to 1e-5 relative L2 (vertex gradients excluded, as for the GGX room)."""
    import subprocess
    import sys
    from test_device_code_cpu import _build
    path = str(tmp_path / "emu.npz")
    r = subprocess.run([sys.executable, em.__file__, _build(), "compare:" + path], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    emu = dict(np.load(path))
    gpu = em.compare_render(rb, torch.device("cuda:0"))
    assert set(gpu) == set(emu) and len(gpu) >= 4

    def rel(a, b):
        return float(np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-30))
    for k in gpu:
        assert rel(gpu[k], emu[k]) < 1e-5, (k, rel(gpu[k], emu[k]))
