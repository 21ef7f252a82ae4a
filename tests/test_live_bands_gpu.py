"""GPU suite: the backward bands run over the samples of the live pixels only (KernelArgs::live_pixels, rb_scene_last_live_samples).

- The live sample count the library reports is spp times the number of owned pixels whose image adjoint has a float that is not zero,
  counted here in torch, for the whole image and for each part of a 2-way stripe partition; with RB_NO_ZERO_CULL=1 it is every owned
  sample.
- An all-zero image adjoint runs no band and gives zero gradients.
- In deterministic mode, many small bands (RB_BAND_BYTES) give the gradients of one band bit for bit.
"""
import numpy as np
import pytest
import torch

import scenes
import test_zero_adjoint_cpu as zc
from redner_b200 import api
from redner_b200.dist import owned_rows

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
ROWS_PER_STRIPE = 4


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


def backward(rb, scene, res, spp, d_of, parts=1, part=0):
    """(gradients {name: array}, live samples, bands, d_image) of one backward pass of `scene` (both edge samplers, 1 bounce) whose
    image adjoint is d_of(rendered image)."""
    args = api.RenderFunction.serialize_scene(scenes.SCENES[scene](DEV, resolution=(res, res)), spp, 1, sampler_type=rb.SamplerType.sobol, device=DEV, backend=rb)
    c = api.RenderFunction._unpack((3, 1000006), args)
    d = d_of(api._render(c)).contiguous()
    if parts > 1:
        c.scene.set_partition(part, parts, ROWS_PER_STRIPE)
    g = api.RenderFunction.gradient_buffers(c)
    rc = rb.render(c.scene, api.RenderFunction.backward_options(c), rb.float_ptr(0), api._ptr(rb, d), g.d_scene, rb.float_ptr(0), rb.float_ptr(0))
    assert rc is None or rc == 0, rc
    out = {"arg%03d" % i: t.detach().cpu().numpy().copy() for i, t in enumerate(api.RenderFunction.gradient_outputs(c, g)) if isinstance(t, torch.Tensor)}
    live, bands = c.scene.last_live_samples()
    return out, live, bands, d


@pytest.mark.parametrize("kind", ["natural", "tiles", "row"])
@pytest.mark.parametrize("parts", [1, 2])
def test_live_samples_are_the_samples_of_nonzero_pixels(rb, monkeypatch, kind, parts):
    spp = 3
    for part in range(parts):
        monkeypatch.delenv("RB_NO_ZERO_CULL", raising=False)
        _, live, bands, d = backward(rb, "shadow_blocker", 24, spp, lambda img: zc.d_image(kind, img), parts, part)
        rows = owned_rows(d.shape[0], part, parts, ROWS_PER_STRIPE)
        nonzero = int((d[rows] != 0).any(-1).sum())
        assert nonzero > 0, (kind, part)
        assert live == spp * nonzero, (kind, part, live, nonzero)
        assert bands == 1
        monkeypatch.setenv("RB_NO_ZERO_CULL", "1")
        _, live_all, bands_all, _ = backward(rb, "shadow_blocker", 24, spp, lambda img: zc.d_image(kind, img), parts, part)
        assert live_all == spp * len(rows) * d.shape[1] and bands_all == 1


def test_all_zero_adjoint_runs_no_band(rb, monkeypatch):
    monkeypatch.delenv("RB_NO_ZERO_CULL", raising=False)
    out, live, bands, _ = backward(rb, "shadow_blocker", 24, 3, torch.zeros_like)
    assert live == 0 and bands == 0
    assert out and all(not np.any(v) for v in out.values()), [k for k, v in out.items() if np.any(v)]


def test_small_bands_equal_one_band_in_deterministic_mode(rb, monkeypatch, deterministic):
    monkeypatch.delenv("RB_NO_ZERO_CULL", raising=False)
    natural = lambda img: 2 * img  # noqa: E731
    monkeypatch.delenv("RB_BAND_BYTES", raising=False)
    one, live, bands, _ = backward(rb, "shadow_blocker", 128, 16, natural)
    assert bands == 1 and live > 0
    monkeypatch.setenv("RB_BAND_BYTES", str(1 << 20))
    many, live_many, bands_many, _ = backward(rb, "shadow_blocker", 128, 16, natural)
    assert live_many == live and bands_many > 4, (live_many, bands_many)
    assert one.keys() == many.keys()
    for k in one:
        assert one[k].tobytes() == many[k].tobytes(), (k, np.abs(one[k].astype(np.float64) - many[k]).max())
