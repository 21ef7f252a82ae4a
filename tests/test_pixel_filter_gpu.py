"""GPU suite: pixel reconstruction filters (rb_pixel_filter) in the CUDA kernels and the device table builders.

- The 1-pixel box given explicitly renders what the zero-initialised default renders, bit for bit: images and gradients (both edge
  samplers, Sobol and PCG; the gradients in deterministic mode) on C1, C2 and the glossy room, and the primary-edge tables of the
  teapot, which are built on the device.
- With a filter the device-built primary-edge PMF equals the host builder's byte for byte (teapot, RB_HOST_TREES=1; the CDFs agree up
  to the order of the scan's additions), and an update
  that changes only the filter equals a new scene with it, table by table.
- A tent of width 2 and a Gaussian of width 3 give the expected image (the convolved 8x supersampled box render) on the single triangle
  and the textured glossy room with a perspective camera, an orthographic camera and a viewport crop; their gradients agree with finite
  differences, the edge just outside the image within the tent's reach included.
- With a tent and torch.use_deterministic_algorithms(True) the gradients are bitwise repeatable and unchanged by the band size.
The checks are those of tests/test_pixel_filter_cpu.py, at sizes the emulator cannot afford."""
import numpy as np
import pytest
import torch

import parity_utils as pu
import scenes
import test_pixel_filter_cpu as pf
from redner_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def test_explicit_box_is_the_default_bit_for_bit(rb, dev):
    # (deterministic mode: the default float atomics add gradients in a run-dependent order, so only exact sums compare bit for bit)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        _box_default(rb, dev)
    finally:
        torch.use_deterministic_algorithms(prev)
    a = pf.scene_tables(pf.native_scene(rb, dev, scenes.teapot(dev, resolution=(256, 256)), None).scene)
    b = pf.scene_tables(pf.native_scene(rb, dev, scenes.teapot(dev, resolution=(256, 256)), ("box", 1.0)).scene)
    assert len(a["primary_edge_pmf"]) > 8000 and a == b


def _box_default(rb, dev):
    pf.box_default_check(rb, dev, [("single_triangle", 64, 16, 1, rb.SamplerType.sobol), ("single_triangle", 64, 16, 1, rb.SamplerType.independent),
                                   ("shadow_blocker", 96, 16, 1, rb.SamplerType.sobol), ("shadow_blocker", 96, 16, 1, rb.SamplerType.independent),
                                   ("glossy_room", 48, 8, 2, rb.SamplerType.sobol), ("glossy_room", 48, 8, 2, rb.SamplerType.independent)])


@pytest.mark.parametrize("filt", ["tent2", "gauss3"])
def test_filtered_tables_device_equal_host(rb, dev, filt, monkeypatch):
    gpu = pf.scene_tables(pf.native_scene(rb, dev, scenes.teapot(dev, resolution=(256, 256)), filt).scene)
    monkeypatch.setenv("RB_HOST_TREES", "1")
    host = pf.scene_tables(pf.native_scene(rb, dev, scenes.teapot(dev, resolution=(256, 256)), filt).scene)
    assert len(gpu["primary_edge_pmf"]) > 8000
    assert gpu["primary_edge_pmf"] == host["primary_edge_pmf"]  # (primary_edge_weight and the normalisation: the same arithmetic)
    # the device CDF is a parallel scan of that PMF (rb_edge_tree.cu), the host's a serial one: equal up to the order of the additions
    cdf_g, cdf_h = (np.frombuffer(t["primary_edge_cdf"], dtype=np.float64) for t in (gpu, host))
    assert np.allclose(cdf_g, cdf_h, rtol=0, atol=1e-13)


@pytest.mark.parametrize("scene", ["teapot", "glossy_room"])
def test_filter_update_equals_a_new_scene(rb, dev, scene):
    pf.update_check(rb, dev, lambda: scenes.SCENES[scene](dev, resolution=(128, 128)), ["tent2", "gauss3"])


@pytest.mark.parametrize("filt", ["tent2", "gauss3"])
@pytest.mark.parametrize("name", ["triangle", "room"])
@pytest.mark.parametrize("camera", ["perspective", "ortho", "crop"])
def test_filtered_image_matches_the_convolved_supersampled_box(rb, dev, name, camera, filt):
    assert pf.expected_image_check(rb, dev, name, camera, filt, 32, 256, 8, 16, 4) >= 4


@pytest.mark.parametrize("filt", ["tent2", "gauss3"])
def test_filtered_gradients_match_finite_differences(rb, dev, filt):
    for make, move, grad_of in pf.triangle_moves(dev, 64):
        pf.fd_check(rb, dev, make, move, grad_of, filt, 256, 4096, 4, 0.02, rel=0.02)


def test_edge_outside_the_image_within_the_filter_reach(rb, dev):
    pf.border_check(rb, dev, 32, 1024, 8192, 4)


def test_deterministic_tent_gradients_repeat_and_ignore_the_band_size(rb, dev, monkeypatch):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        def run():
            sc = scenes.glossy_room(dev, resolution=(64, 64))
            args = api.RenderFunction.serialize_scene(sc, 8, 2, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                                      pixel_filter=api.PixelFilter("tent", 2.0))
            img = api.RenderFunction.apply(5, *args)
            (pf.weight_image(img.shape).to(dev) * img).sum().backward()
            return {k: v.numpy().tobytes() for k, v in pu.collect_grads(sc).items()}
        a, b = run(), run()
        monkeypatch.setenv("RB_BAND_BYTES", str(1 << 20))
        c = run()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert len(a) > 5 and a == b == c
