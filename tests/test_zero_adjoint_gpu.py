"""GPU suite: the backward pass skips the samples of pixels whose image adjoint is exactly zero (see tests/test_zero_adjoint_cpu.py for
the scenes and image adjoints).  With RB_NO_ZERO_CULL=1 every sample is traced.

- Deterministic mode (exact gradient sums): every gradient, the camera's and the screen gradient are bit-identical with and without the
  skip, for every scene and image adjoint of the CPU suite, and for C2 at 128 x 128 x 64 spp.
- Default mode: the skip changes which samples share a warp and a block, so the gradient atomics add in another order.  Every gradient
  lies within twice what two runs without the skip differ by, plus 1e-4 relative: two runs without the skip keep the same warps and often
  agree bit for bit, while the skip regroups the samples (measured: 1.2e-5 on a 3-float gradient of the stripes case).
- The skip does happen: on C2 the backward pass traces fewer primary hits with it than without.
"""
import numpy as np
import pytest
import torch

import parity_utils as pu
import test_zero_adjoint_cpu as zc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
C2_128 = ("shadow_blocker", 128, 64, 1, 3, {})


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.fixture
def c2_128(monkeypatch):
    monkeypatch.setitem(zc.CASES, "c2_128", C2_128)
    return "c2_128"


@pytest.mark.parametrize("name", sorted(zc.CASES))
def test_skip_is_bit_identical_in_deterministic_mode(rb, deterministic, name):
    zc.check_case(rb, DEV, name)


def test_c2_128_skip_is_bit_identical_in_deterministic_mode(rb, deterministic, c2_128):
    zc.check_case(rb, DEV, c2_128, kinds=["natural", "tiles"])


@pytest.mark.parametrize("name", ["c2_spp3", "c2_spp64", "glossy_room", "env_ball", "fisheye_room", "tent2", "gbuffer", "screen_gradient", "stripes",
                                  "viewport", "c2_128"])
def test_skip_within_the_spread_of_two_runs_without_it(rb, monkeypatch, c2_128, name):
    for kind in ["natural", "tiles", "row", "some_channels"]:
        skip, full = zc.both_ways(rb, DEV, name, kind)
        monkeypatch.setenv("RB_NO_ZERO_CULL", "1")
        full2 = zc.backward_outputs(rb, DEV, name, kind)
        monkeypatch.delenv("RB_NO_ZERO_CULL")
        for k in full:
            noise = pu.rel_l2(full2[k], full[k])
            assert pu.rel_l2(skip[k], full[k]) <= 2 * noise + 1e-4, (name, kind, k, pu.rel_l2(skip[k], full[k]), noise)


def _c2_primary_hits(rb, monkeypatch, skip):
    """Primary hits the backward pass of C2 (128 x 128 x 16 spp, loss sum(img^2)) traced, and the number of pixels with a zero adjoint."""
    import scenes
    from redner_b200 import api
    if skip:
        monkeypatch.delenv("RB_NO_ZERO_CULL", raising=False)
    else:
        monkeypatch.setenv("RB_NO_ZERO_CULL", "1")
    args = api.RenderFunction.serialize_scene(scenes.shadow_blocker(DEV, resolution=(128, 128)), 16, 1, sampler_type=rb.SamplerType.sobol, device=DEV,
                                              backend=rb)
    c = api.RenderFunction._unpack((1, 1000004), args)
    d = (2 * api._render(c)).contiguous()
    api._backward(c, d)
    _, _, hits = c.scene.last_stage_stats()
    return hits, int((d == 0).all(-1).sum())


def test_c2_traces_fewer_samples_with_the_skip(rb, monkeypatch):
    hits_skip, zero_px = _c2_primary_hits(rb, monkeypatch, True)
    hits_full, _ = _c2_primary_hits(rb, monkeypatch, False)
    assert zero_px > 0
    assert 0 < hits_skip < hits_full
    # every skipped sample belongs to a zero pixel: at most zero_px * spp of them
    assert hits_full - hits_skip <= zero_px * 16
