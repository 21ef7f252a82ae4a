"""GPU suite: the GGX specular lobe at scene level (the functions are checked on the host build by tests/test_ggx_cpu.py).

- White furnace: a quad with kd = 0, ks = 1 and GGX under a constant environment map of radiance 1, seen by an orthographic camera (one
  view angle for every pixel), one bounce, no edge sampling.  The mean pixel equals the single-scattering directional albedo of the
  lobe, integrated from its float64 restatement, within 4 standard errors.  Sampling, pdf, eval and their MIS with the environment map's
  own sampling all enter.
- A GGX scene renders bit for bit the same with and without RB_NO_LEAN=1: it runs the general kernels.
- The finite-difference and deterministic checks of the CPU suite at larger sizes.
"""
import math

import numpy as np
import pytest
import torch

import test_ggx_cpu as ggx
from redner_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


def albedo(alpha, theta, n_t=3000, n_p=512):
    """Directional albedo of the restated lobe with F = 1: the integral of D G2 / (4 cos(theta_i)) over the directions above the quad
    (bsdf_eval's cut-off |cos(theta_o)| > 1e-3 included), on a grid around the mirror direction."""
    a2 = alpha * alpha
    wi = np.array([math.sin(theta), 0.0, math.cos(theta)])
    m = np.array([-wi[0], 0.0, wi[2]])
    t1 = np.array([0.0, 1.0, 0.0])
    t2 = np.cross(m, t1)
    t = (np.arange(n_t) + 0.5) / n_t
    p = 2 * math.pi * (np.arange(n_p) + 0.5) / n_p
    g = math.pi * t ** 3
    jac = np.sin(g) * 3 * math.pi * t ** 2 * (1.0 / n_t) * (2 * math.pi / n_p)
    wo = (np.cos(g)[:, None, None] * m + np.sin(g)[:, None, None] * (np.cos(p)[None, :, None] * t1 + np.sin(p)[None, :, None] * t2))
    h = wo + wi
    h /= np.linalg.norm(h, axis=-1, keepdims=True)

    def lam(c):
        return (-1.0 + np.sqrt(1.0 + a2 * (1.0 - c * c) / (c * c))) / 2.0
    hz = h[..., 2]
    D = a2 / (math.pi * (hz * hz * (a2 - 1.0) + 1.0) ** 2)
    G2 = 1.0 / (1.0 + lam(wi[2]) + lam(wo[..., 2]))
    val = np.where((wo[..., 2] > 1e-3) & (hz > 0), D * G2 / (4 * wi[2]), 0.0)
    return float((val * jac[:, None]).sum())


# The environment map's sampling tables are piecewise constant per texel row while its pdf is not; at 8 x 16 texels that MIS mismatch
# alone lifts a kd = 1 Lambertian furnace by about 4 %.  At 256 x 512 it is far below the test's standard errors.
ENV_RES = 256


def furnace_scene(dev, alpha, theta, res):
    # The film spans [-2, 2] (intrinsic scale 0.5), so a ray starts d cos(theta) - 2 sin(theta) above the quad at the lowest: positive
    # up to theta = atan(d / 2) = 1.52 rad.  (A film edge below the quad would see the sky directly and lift the mean towards 1.)
    d = 40.0
    cam = api.Camera(position=torch.tensor([d * math.sin(theta), d * math.cos(theta), 0.0]), look_at=torch.tensor([0.0, 0.0, 0.0]),
                     up=torch.tensor([0.0, 0.0, 1.0]), clip_near=1e-2, resolution=(res, res),
                     intrinsic_mat=torch.tensor([[0.5, 0.0, 0.0], [0.0, 0.5, 0.0], [0.0, 0.0, 1.0]]), camera_type=1)
    s = 50.0
    quad = api.Shape(torch.tensor([[-s, 0.0, -s], [-s, 0.0, s], [s, 0.0, -s], [s, 0.0, s]], device=dev),
                     torch.tensor([[0, 1, 2], [1, 3, 2]], device=dev, dtype=torch.int32), 0)
    mat = api.Material(diffuse_reflectance=torch.zeros(3, device=dev), specular_reflectance=torch.ones(3, device=dev),
                       roughness=torch.tensor([alpha * alpha], device=dev), specular_model="ggx")
    env = api.EnvironmentMap(torch.ones(ENV_RES, 2 * ENV_RES, 3, device=dev))
    return api.Scene(cam, [quad], [mat], [], envmap=env)


@pytest.mark.parametrize("alpha", [0.05, 0.3, 0.8])
@pytest.mark.parametrize("theta", [0.3, 1.0, 1.35, 1.45])
def test_white_furnace(rb, alpha, theta):
    dev = torch.device("cuda:0")
    sc = furnace_scene(dev, alpha, theta, 64)
    args = api.RenderFunction.serialize_scene(sc, 16, 1, device=dev, backend=rb, use_primary_edge_sampling=False, use_secondary_edge_sampling=False)
    img = api.RenderFunction.apply(1, *args).detach().double().cpu().numpy()
    px = img[..., 0].ravel()
    assert np.allclose(img[..., 0], img[..., 1]) and np.allclose(img[..., 0], img[..., 2])
    expected = albedo(alpha, theta)
    se = px.std(ddof=1) / math.sqrt(px.size)
    assert 0.3 < expected <= 1.0 + 1e-6
    assert abs(px.mean() - expected) <= 4 * se + 1e-6, (px.mean(), expected, se)


def test_ggx_runs_the_general_kernels(rb, monkeypatch):
    dev = torch.device("cuda:0")
    a = ggx.render(rb, dev, ggx.ggx_room(dev, 64), 4, 7, mb=2, use_secondary_edge_sampling=True)
    monkeypatch.setenv("RB_NO_LEAN", "1")
    b = ggx.render(rb, dev, ggx.ggx_room(dev, 64), 4, 7, mb=2, use_secondary_edge_sampling=True)
    assert float(np.abs(a[0]).sum()) > 0
    assert a[0].tobytes() == b[0].tobytes()


def test_ggx_gradients_match_finite_differences(rb):
    ggx.fd_checks(rb, torch.device("cuda:0"), 48, 64, 512, 6)


def test_ggx_deterministic_repeatable_and_band_independent(rb):
    ggx.deterministic_check(rb, torch.device("cuda:0"), res=48, spp=4)


def test_explicit_blinn_phong_is_the_default(rb):
    # (deterministic mode: float atomics would make even two default runs differ in the last bits)
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        ggx.explicit_default_check(rb, torch.device("cuda:0"), res=32, spp=4)
    finally:
        torch.use_deterministic_algorithms(False)


def test_gpu_matches_the_emulator(rb, tmp_path):
    """The GGX glossy room on the GPU and on the host build of the same headers (tools/cpu_emu), same seed and samples.  Same source, but the
    device build contracts multiply-adds into FMAs and uses approximate division and square root, and the emulator's BVH is a median-split
    tree instead of the LBVH.  The image and every texture and light gradient must agree to 1e-5 relative L2: on an H100 they agree to
    3e-7 and 6e-7, the rounding of float sums in another order.  Vertex gradients are not compared here: they are sums of a few large
    edge-sample terms, and the ball's differs by 0.43 relative L2 at 8 spp (DESIGN.md section 7)."""
    import subprocess
    import sys
    from test_device_code_cpu import _build
    path = str(tmp_path / "emu.npz")
    r = subprocess.run([sys.executable, ggx.__file__, _build(), "compare:" + path], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    emu = dict(np.load(path))
    gpu = ggx.compare_render(rb, torch.device("cuda:0"))
    assert set(gpu) == set(emu) and len(gpu) > 5

    def rel(a, b):
        return float(np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-30))
    errs = {k: rel(gpu[k], emu[k]) for k in gpu}
    print("gpu vs emulator rel L2:", errs)
    for k, e in errs.items():
        assert k.endswith(".vertices") or e <= 1e-5, (k, errs)
