"""GPU suite: the thin-lens camera in the CUDA kernels and the device table builders.

- lens_radius 0 renders what a camera without a lens renders, bit for bit (gradients in deterministic mode, where sums are exact):
  images, gradients, scene tables and exact records.
- The uv and position channels of a plane at the focal distance equal the pinhole's to float rounding.
- A lens-only update equals a new scene table by table (the teapot's tables are built on the device), and the device primary-edge PMF
  equals the host builder's byte for byte; set_camera changes the lens; the refusals raise.
- With torch.use_deterministic_algorithms(True) lens gradients repeat bit for bit whatever the band size.
- Statistical checks at sizes the emulator cannot afford: the pinhole-average identity and central differences in the lens parameters.
The checks are those of tests/test_lens_cpu.py."""
import os

import numpy as np
import pytest
import torch

import scenes
import test_lens_cpu as lc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _deterministic(fn):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        fn()
    finally:
        torch.use_deterministic_algorithms(prev)


def test_zero_radius_is_the_pinhole_bit_for_bit(rb, dev):
    _deterministic(lambda: lc.zero_radius_check(rb, dev, 32, 4))


def test_in_focus_plane_is_sharp(rb, dev):
    lc.in_focus_check(rb, dev, 64, 4)


def test_lens_update_equals_a_new_scene(rb, dev):
    lc.update_check(rb, dev, 32)


def _teapot_tables(rb, dev, lens, host):
    if host:
        os.environ["RB_HOST_TREES"] = "1"
    try:
        sc = scenes.teapot(dev, resolution=(64, 64))
        cam = sc.camera
        if lens is not None:
            cam.lens_radius, cam.focus_distance = torch.tensor([lens[0]]), torch.tensor([lens[1]])
        c = lc.native(rb, dev, sc, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        return c, lc.scene_tables(c.scene)
    finally:
        os.environ.pop("RB_HOST_TREES", None)


def test_device_distribution_equals_host_and_update(rb, dev):
    _, dev_t = _teapot_tables(rb, dev, (0.3, 4.0), False)
    _, host_t = _teapot_tables(rb, dev, (0.3, 4.0), True)
    assert dev_t["primary_edge_pmf"] == host_t["primary_edge_pmf"]
    d = np.frombuffer(dev_t["primary_edge_cdf"], np.float64)
    h = np.frombuffer(host_t["primary_edge_cdf"], np.float64)
    assert np.abs(d - h).max() < 1e-13
    c, pin = _teapot_tables(rb, dev, None, False)
    assert pin["primary_edge_pmf"] != dev_t["primary_edge_pmf"]
    ref, _ = _teapot_tables(rb, dev, (0.3, 4.0), False)
    c.scene.update(ref.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False)
    assert lc.scene_tables(c.scene) == dev_t


def test_refused_combinations_name_the_lens(rb, dev):
    lc.refusals_check(rb, dev)


def test_deterministic_lens_gradients_repeat(rb, dev):
    lc.deterministic_check(rb, dev, 32, 4)


def test_lens_equals_pinhole_average_primary_edges(rb, dev):
    lc.pinhole_average_check(rb, dev, "glow", 32, 16, 300)


def test_lens_equals_pinhole_average_full(rb, dev):
    lc.pinhole_average_check(rb, dev, "room", 24, 8, 150, nontrivial=False)


def test_lens_gradients_match_finite_differences(rb, dev):
    lc.fd_check(rb, dev, 32, 64, 100)
