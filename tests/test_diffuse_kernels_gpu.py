"""GPU suite: the diffuse-only instantiation of the kernels (rb_kernels_diffuse.cu) against the lean one it replaces for scenes whose
materials neither compute specular lighting nor use vertex colours or normal maps.  RB_NO_DIFFUSE=1 forces the lean kernels.  Same
source, same samples: the image must be bit-identical.  The gradients may differ from the lean kernels' by at most twice what two runs
of the lean kernels differ by (the order of the gradient atomics), plus 1e-6 for the device compiler's rounding of the shorter code.
"""
import pytest
import torch

import parity_utils as pu
import scenes
from redner_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


def _bunny_box_diffuse(dev, resolution):
    sc = scenes.bunny_box_shifted(dev, resolution=resolution)
    sc.materials = [api.Material(diffuse_reflectance=m.diffuse_reflectance, two_sided=m.two_sided) for m in sc.materials]
    return sc


def _render(rb, make, res, spp, mb, seed):
    dev = torch.device("cuda:0")
    sc = make(dev, resolution=(res, res))
    args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                              use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    img = api.RenderFunction.apply(seed, *args)
    img.pow(2).sum().backward()
    return img.detach().cpu(), pu.collect_grads(sc)


@pytest.mark.parametrize("make,res,spp,mb", [(scenes.shadow_blocker, 128, 16, 1), (scenes.shadow_blocker_all, 64, 16, 2), (_bunny_box_diffuse, 64, 4, 5)],
                         ids=["c2", "c2_all_vertices", "c4_diffuse"])
def test_diffuse_and_lean_kernels_agree(rb, monkeypatch, make, res, spp, mb):
    img_d, g_d = _render(rb, make, res, spp, mb, 7)
    monkeypatch.setenv("RB_NO_DIFFUSE", "1")
    img_l1, g_l1 = _render(rb, make, res, spp, mb, 7)
    img_l2, g_l2 = _render(rb, make, res, spp, mb, 7)
    assert float(img_d.abs().sum()) > 0
    assert torch.equal(img_d, img_l1) and torch.equal(img_l1, img_l2)
    assert set(g_d) == set(g_l1) and g_d
    for k in g_l1:
        noise = pu.rel_l2(g_l2[k].numpy(), g_l1[k].numpy())
        assert pu.rel_l2(g_d[k].numpy(), g_l1[k].numpy()) <= 2 * noise + 1e-6, (k, noise)
