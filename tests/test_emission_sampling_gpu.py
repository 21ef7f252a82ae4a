"""GPU suite: emission sampling of textured area lights (the host emulator runs the same checks at small sizes in
tests/test_emission_sampling_cpu.py).

- The device tables equal the float64 restatement bit for bit, up to 1024 x 1024 textures; the sampler passes its chi-square, rejection,
  density and quadrature checks with 10^6 samples; the option off, constant and zero textures change nothing; updates equal new scenes;
  refusals name the emission sampling; deterministic mode is repeatable and band-independent.
- Unbiasedness under MIS: the floor lit by a quad light with a window texture (a bright rectangle over 4 % of it) or a smooth one, one- and
  two-sided, 1 and 3 channels: per-pixel means over runs match the float64 quadrature (emission_sampling_ref.quadrature) within 4
  standard errors.  Texels written in place without an update (stale tables) stay unbiased.  On the window texture the image variance
  falls against the area strategy by at least half the ratio that the float64 variance of the MIS estimator predicts.
- Gradients under texture sampling (texel, intensity, uv_scale, floor reflectance) pass finite differences and agree with the area
  strategy's means; exact records are unchanged with the option off and sum over a 2-way partition to one render.
- The GPU and the emulator agree on the textured lamp under texture sampling to 1e-5 relative L2 (image, texture and light gradients).
"""
import math

import numpy as np
import pytest
import torch

import emission_sampling_ref as ref
import test_emission_cpu as em
import test_emission_sampling_cpu as es
from redner_b200 import api

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from redner_b200 import redner
    return redner


DEV = torch.device("cuda:0")


def test_tables_equal_the_restatement(rb):
    es.tables_check(rb, DEV, es.TABLE_CASES + es.TABLE_CASES_LARGE)


def test_sampler_draws_from_its_density(rb):
    es.sampler_check(rb, DEV, n=1000000)


def test_option_off_constant_and_zero_textures_change_nothing(rb):
    es.identity_check(rb, DEV, res=32, spp=8)


def test_updates_equal_a_new_scene(rb):
    es.update_check(rb, DEV)


def test_refusals_name_the_emission_sampling(rb):
    es.refusals_check(rb, DEV)


def test_deterministic_repeatable_and_band_independent(rb):
    es.deterministic_check(rb, DEV, res=32, spp=8)


def test_records_unchanged_when_off_and_partition_sums_equal_one_render(rb):
    es.records_check(rb, DEV, res=32, spp=4)


def test_stale_tables_render_unbiased(rb):
    es.stale_check(rb, DEV, runs=24, spp=256)


def test_gradients_match_finite_differences_and_the_area_strategy(rb):
    es.gradient_checks(rb, DEV, 32, 64, 512, 6)


def _runs(rb, sc, runs, spp):
    args = api.RenderFunction.serialize_scene(sc, spp, 1, device=DEV, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False)
    return np.stack([api.RenderFunction.apply(100 + k, *args).cpu().numpy().astype(np.float64) for k in range(runs)])


def _positions(rb, sc):
    args = api.RenderFunction.serialize_scene(sc, 1, 1, device=DEV, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False, channels=[rb.channels.position])
    return api.RenderFunction.apply(0, *args).cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("two_sided", [False, True])
@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("kind", ["window", "smooth"])
def test_texture_sampling_is_unbiased_under_mis(rb, two_sided, ch, kind):
    tex = es.window_image(16, 16, ch) if kind == "window" else em.ramp_image(16, 16, ch)
    sc = es.light_scene(DEV, tex, two_sided=two_sided, res=16)
    ref_img = ref.quadrature(_positions(rb, sc), tex.numpy().astype(np.float64))
    runs = 24
    imgs = _runs(rb, sc, runs, spp=256)
    mean, se = imgs.mean(0), imgs.std(0, ddof=1) / math.sqrt(runs)
    z = (mean - ref_img) / np.maximum(se, 1e-12)
    assert (np.abs(z) > 4).mean() < 0.01, np.abs(z).max()
    tot = imgs.sum((1, 2, 3))
    assert abs(tot.mean() - ref_img.sum()) <= 4 * tot.std(ddof=1) / math.sqrt(runs), (tot.mean(), ref_img.sum())


def _texture_density_grid(scene, n):
    """The texture strategy's area density (rb_light_sample_test's queries) at the midpoints of the n x n grid of the light's uv square."""
    s = (np.arange(n) + 0.5) / n
    u, v = np.meshgrid(s, s, indexing="xy")
    tri = np.where(u > v, 0, 1)  # (triangles (0, 2, 1) and (0, 3, 2) of the unit square)
    q = torch.tensor(np.stack([tri, u, v], -1).reshape(-1, 3), dtype=torch.float32, device=DEV)
    _, _, pd = scene.light_sample_test(0, torch.zeros(0, 3, dtype=torch.float64, device=DEV), q)
    return pd.cpu().numpy().reshape(n, n)


def test_window_texture_variance_falls_as_the_quadrature_predicts(rb):
    """The variance of the one-sample MIS estimate (light sample + BSDF sample, power heuristic) of every pixel, integrated in float64
    over the light for both strategies (ref.mis_variance), predicts the ratio of the image variances over runs; the measured ratio must
    reach half the predicted one (the variance estimates of 48 runs scatter by a few percent, and the light pdf's cells round against
    the quadrature's grid)."""
    tex = es.window_image(16, 16, 3)
    n = 128
    sc = es.light_scene(DEV, tex, res=16)
    pos = _positions(rb, sc)
    c, keep = es.native(rb, DEV, sc)
    area = float(es._tab(c.scene, "light_areas")[0])
    t64 = tex.numpy().astype(np.float64)
    predicted = ref.mis_variance(pos, t64, np.full((n, n), 1.0 / area), n) / ref.mis_variance(pos, t64, _texture_density_grid(c.scene, n), n)
    v = {}
    for s in ("area", "texture"):
        imgs = _runs(rb, es.light_scene(DEV, tex, sampling=s, res=16), 48, spp=16)
        v[s] = imgs.var(0, ddof=1).sum()
    measured = v["area"] / v["texture"]
    print("image variance, area / texture strategy: measured %.3f, predicted %.3f" % (measured, predicted))
    assert predicted > 2, predicted
    assert measured > 0.5 * predicted, (measured, predicted)


def test_gpu_matches_the_emulator(rb, tmp_path):
    import subprocess
    import sys
    from test_device_code_cpu import _build
    path = str(tmp_path / "emu.npz")
    r = subprocess.run([sys.executable, es.__file__, _build(), "compare:" + path], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    emu = dict(np.load(path))
    gpu = es.compare_render(rb, DEV)
    assert set(gpu) == set(emu) and len(gpu) >= 4

    def rel(a, b):
        return float(np.linalg.norm((a - b).ravel()) / max(np.linalg.norm(b.ravel()), 1e-30))
    for k in gpu:
        assert rel(gpu[k], emu[k]) < 1e-5, (k, rel(gpu[k], emu[k]))
