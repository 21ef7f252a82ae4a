"""CPU suite: emission sampling of textured area lights (rb_area_light::emission_sampling, DESIGN.md "Emission sampling"), on the host
emulator; tests/test_emission_sampling_gpu.py runs the same checks on the GPU at larger sizes.

- Nothing changes when the texture branch is off: the explicit "area" option on the textured lamp, "texture" on a constant texture and
  "texture" on an all-zero texture render the image and gradients of the default bit for bit, with the same light tables.
- The tables (cell weights, summed-area table, per-triangle rectangle, mass, weight, CDF and pdf factor, and the light PMF) equal the float64
  restatement (tests/emission_sampling_ref.py) bit for bit: both perform the same double operations in the same order.  Covered: 1 x 1 to
  64 x 64 textures with 1 and 3 channels, uv_scale (1, 1), (3, 0.5) and a negative one, negative and wrapped uvs, a triangle spanning
  several periods, a zero-uv-area triangle and a shape without uvs.
- The sampler (rb_light_sample_test) draws from its density: counts per (triangle, cell) pass a chi-square test against the restatement's
  polygon-clipped probabilities, the rejection fraction matches, every accepted sample reports the restatement's density at its point, and
  the density integrates over the light to 1 minus the rejection.
- Updates (toggling the option, new texels, a new uv_scale) equal a new scene table for table; refusals name the emission sampling;
  deterministic mode is repeatable with the option on.

Run as a script (`python tests/test_emission_sampling_cpu.py <emulator.so> <check>...`) this file is the subprocess that binds the
emulator in place of the library."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import emission_sampling_ref as ref  # noqa: E402

TABLES = ("lights", "light_pmf", "light_cdf", "light_areas", "area_cdf_pool", "area_cdf_offsets")


# ---------------------------------------------------------------------------------------------------- scenes
def window_image(h, w, ch, peak=40.0, base=0.05):
    """A dark texture with a bright rectangle over about 4 % of it: the case texture sampling is for."""
    import torch
    img = torch.full((h, w, ch), base)
    y0, x0 = int(0.55 * h), int(0.2 * w)
    img[y0:y0 + max(1, h // 5), x0:x0 + max(1, w // 5)] = peak
    if ch == 3:
        img[..., 1] *= 0.8
    return img.contiguous()


def light_scene(dev, tex, sampling="texture", uvs="quad", uv_scale=(1.0, 1.0), extra_tris=False, two_sided=False, second_light=False, res=12):
    """The floor-and-lamp scene of the MIS test: an orthographic camera covering [-1, 1]^2 above a Lambertian floor (kd = ref.KD) lit by
    a quad light beside the view (ref.LIGHT), which faces the floor (one-sided) or away from it (two-sided: the floor sees its back).  `uvs`: "quad" (the unit square), "wrapped" (negative and > 1 uvs), "periods" (the second
    triangle spans several periods) or None (no uvs: the default per-triangle uvs).  `extra_tris`: a third triangle with zero uv area."""
    import torch
    from redner_b200 import api
    cam = api.Camera(position=torch.tensor([0.0, 0.0, 3.0]), look_at=torch.tensor([0.0, 0.0, 0.0]), up=torch.tensor([0.0, 1.0, 0.0]),
                     fov=torch.tensor([90.0]), clip_near=1e-2, resolution=(res, res), camera_type=1)
    fv = torch.tensor([[-4.0, -4.0, 0.0], [4.0, -4.0, 0.0], [4.0, 4.0, 0.0], [-4.0, 4.0, 0.0]])
    fi = torch.tensor([[0, 1, 2], [0, 2, 3]], dtype=torch.int32)
    L = ref.LIGHT
    lv = torch.tensor([[L["x0"], L["y0"], L["z"]], [L["x1"], L["y0"], L["z"]], [L["x1"], L["y1"], L["z"]], [L["x0"], L["y1"], L["z"]]])
    li = [[0, 1, 2], [0, 2, 3]] if two_sided else [[0, 2, 1], [0, 3, 2]]  # (two-sided: the floor sees the back face)
    luv = {"quad": [[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]], "wrapped": [[-0.3, -1.2], [0.9, -1.2], [0.9, 0.1], [-0.3, 0.1]],
           "periods": [[0.0, 0.0], [2.5, -0.5], [3.2, 1.7], [-0.4, 2.1]], None: None}[uvs]
    if extra_tris:  # (a sliver along an edge whose uvs are collinear)
        lv = torch.cat([lv, torch.tensor([[L["x0"], L["y0"] - 0.05, L["z"]]])])
        li.append([0, 1, 4])
        if luv is not None:
            luv = luv + [[0.5 * (luv[0][0] + luv[1][0]), 0.5 * (luv[0][1] + luv[1][1])]]
    shapes = [api.Shape(fv.to(dev), fi.to(dev), 0),
              api.Shape(lv.to(dev), torch.tensor(li, dtype=torch.int32).to(dev), 1, uvs=torch.tensor(luv).to(dev) if luv is not None else None)]
    mats = [api.Material(torch.tensor([ref.KD] * 3, device=dev)), api.Material(torch.tensor([0.0, 0.0, 0.0], device=dev))]
    t = api.Texture(tex.to(dev), uv_scale=torch.tensor(uv_scale, device=dev))
    light = api.AreaLight(1, torch.tensor(ref.INTENSITY, dtype=torch.float32), two_sided=two_sided, directly_visible=False, emission=t,
                          emission_sampling=sampling)
    lights = [light]
    if second_light:  # (an untextured light far off to the side: the light PMF then depends on the textured light's S)
        sv = torch.tensor([[-9.0, -9.0, 4.0], [-8.0, -9.0, 4.0], [-8.0, -8.0, 4.0]])
        shapes.append(api.Shape(sv.to(dev), torch.tensor([[0, 2, 1]], dtype=torch.int32).to(dev), 1))
        lights.append(api.AreaLight(2, torch.tensor([0.5, 0.5, 0.5]), directly_visible=False))
    return api.Scene(cam, shapes, mats, lights)


def light_arrays(sc):
    """(tex, uv_scale, uv corners [T, 3, 2], world corners [T, 3, 3]) of the scene's light, as the restatement takes them."""
    light = sc.area_lights[0]
    shape = sc.shapes[light.shape_id]
    idx = shape.indices.cpu().numpy()
    pos = shape.vertices.detach().cpu().numpy()[idx]
    if shape.uvs is not None:
        uv = shape.uvs.detach().cpu().numpy()[idx]
    else:
        uv = np.broadcast_to(np.float32([[0, 0], [1, 0], [1, 1]]), (len(idx), 3, 2))
    return (light.emission.texels.detach().cpu().numpy(), light.emission.uv_scale.detach().cpu().numpy(), uv.astype(np.float32),
            pos.astype(np.float32))


def native(rb, dev, sc, **kw):
    from redner_b200 import api
    args = api.RenderFunction.serialize_scene(sc, 4, 1, device=dev, backend=rb, **kw)
    return api.RenderFunction._unpack((1, 2), args), args


def _tab(scene, name, dtype=np.float64):
    return scene.table(name).view(dtype)


# ---------------------------------------------------------------------------------------------------- checks
def identity_check(rb, dev, res=12, spp=8):
    """The option off, on with a constant texture and on with an all-zero texture: the default's image, gradients and tables."""
    import torch
    import test_emission_cpu as em
    os.environ["RB_NO_LEAN"] = "1"
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        cases = [("image", "area"), ([0.5, 1.0, 2.0], "texture"), ("zero", "texture")]
        for emission, sampling in cases:
            def make(s):
                sc = em.lamp(dev, res, emission="image" if emission == "zero" else emission)
                if emission == "zero":
                    with torch.no_grad():
                        sc.area_lights[0].emission.texels.zero_()
                    sc.area_lights[0].emission.texels = sc.area_lights[0].emission.texels
                sc.area_lights[0].emission_sampling = s
                return sc
            for mb in (0, 1):
                a_img, a = em.render(rb, dev, make("area"), spp, 4, mb=mb, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
                b_img, b = em.render(rb, dev, make(sampling), spp, 4, mb=mb, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
                assert a_img.numpy().tobytes() == b_img.numpy().tobytes(), (emission, sampling, mb)
                assert set(a) == set(b)
                em._bytes_equal(a, b)
            sc = make("area")  # (one scene, so that both light tables point at the same texels)
            ca, keep_a = native(rb, dev, sc)
            sc.area_lights[0].emission_sampling = sampling
            cb, keep_b = native(rb, dev, sc)
            for name in TABLES:
                assert ca.scene.table(name).tobytes() == cb.scene.table(name).tobytes(), name
            # (the zero texture builds its tables, with S = 0, and keeps the area branch; the others build none)
            extra = _tab(cb.scene, "light_sampling")
            assert (extra.size == 0) if emission != "zero" else extra[0] == 0
    finally:
        torch.use_deterministic_algorithms(False)
        del os.environ["RB_NO_LEAN"]


TABLE_CASES = [  # (texture h, w, channels, uvs, uv_scale, extra triangle)
    (1, 1, 1, "quad", (1.0, 1.0), False),
    (4, 4, 3, "quad", (1.0, 1.0), False),
    (16, 8, 1, "wrapped", (3.0, 0.5), True),
    (8, 16, 3, "periods", (1.0, 1.0), False),
    (32, 32, 3, "quad", (-1.0, 2.0), False),
    (12, 12, 1, None, (1.0, 1.0), False),
    (64, 64, 3, "wrapped", (1.0, 1.0), True),
]
# (the GPU suite adds larger textures)
TABLE_CASES_LARGE = [(256, 256, 1, "periods", (1.0, 1.0), False), (1024, 1024, 3, "quad", (1.0, 1.0), True)]


def tables_check(rb, dev, cases=TABLE_CASES):
    """Every table of the light against the restatement, bit for bit, and the light PMF: the light's weight is S in place of its area."""
    import torch
    for h, w, ch, uvs, scale, extra in cases:
        tex = window_image(h, w, ch) * (0.5 + torch.rand(h, w, ch, generator=torch.Generator().manual_seed(h * w + ch)))
        sc = light_scene(dev, tex, uvs=uvs, uv_scale=scale, extra_tris=extra)
        c, keep = native(rb, dev, sc)
        t, s, uv, pos = light_arrays(sc)
        tab = ref.tables(t, s, uv, pos)
        got = _tab(c.scene, "light_sampling")
        want = ref.flat(tab)
        assert got.shape == want.shape, (got.shape, want.shape)
        assert got.tobytes() == want.tobytes(), (h, w, ch, uvs, scale, np.abs(got - want).max())
        if extra:
            assert tab["recs"][2, 5] == 0  # (zero uv area: no weight)
        assert tab["S"] > 0
        # the light PMF with a second, untextured light: the textured light weighs S (in place of its area) times its luminance
        sc2 = light_scene(dev, tex, uvs=uvs, uv_scale=scale, extra_tris=extra, second_light=True)
        c2, keep2 = native(rb, dev, sc2)
        areas = _tab(c2.scene, "light_areas")
        w = [ref.light_weight(sc2.area_lights[k].intensity.numpy(), tab["S"] if k == 0 else float(areas[k])) for k in range(2)]
        tot = w[0] + w[1]
        want_pmf = np.array([w[0] / tot, w[1] / tot])
        assert _tab(c2.scene, "light_pmf").tobytes() == want_pmf.tobytes(), (_tab(c2.scene, "light_pmf"), want_pmf)
        assert _tab(c2.scene, "light_sampling").tobytes() == want.tobytes()
    print("tables ok", len(cases), flush=True)


def sampler_check(rb, dev, n=200000, cases=((8, 8, 3, "quad", (1.0, 1.0)), (6, 10, 1, "periods", (1.0, 1.0)), (16, 16, 3, "wrapped", (3.0, 0.5)))):
    """Binned counts against the restatement's probabilities (chi-square), the rejection fraction, the density at every accepted sample,
    and the density's integral over the light."""
    import torch
    from scipy import stats
    for h, w, ch, uvs, scale in cases:
        sc = light_scene(dev, window_image(h, w, ch), uvs=uvs, uv_scale=scale)
        c, keep = native(rb, dev, sc)
        t, s, uv, pos = light_arrays(sc)
        tab = ref.tables(t, s, uv, pos)
        area = float(_tab(c.scene, "light_areas")[0])
        probs, p_rej = ref.bin_probabilities(tab, t.shape, s, uv, area)
        g = torch.Generator().manual_seed(h + w)
        smp = torch.rand(n, 3, generator=g, dtype=torch.float64).to(dev)
        ints, dbl, _ = c.scene.light_sample_test(0, smp)
        ints, dbl = ints.cpu().numpy(), dbl.cpu().numpy()
        rej = ints[:, 2] == 1
        assert np.all(ints[rej, 1] >= 0) and np.all(dbl[rej] == 0)
        # the rejection fraction (binomial)
        assert abs(rej.mean() - p_rej) <= 5 * math.sqrt(p_rej * (1 - p_rej) / n) + 1e-9, (rej.mean(), p_rej)
        # bins: the cell of the decoded point, unwrapped, per triangle
        acc = ~rej
        tri = ints[acc, 1]
        b1, b2 = dbl[acc, 0], dbl[acc, 1]
        X, Y = ref.corners(uv, s, w, h)
        px = X[tri, 0] + b1 * (X[tri, 1] - X[tri, 0]) + b2 * (X[tri, 2] - X[tri, 0])
        py = Y[tri, 0] + b1 * (Y[tri, 1] - Y[tri, 0]) + b2 * (Y[tri, 2] - Y[tri, 0])
        keys = list(probs)
        index = {k: i for i, k in enumerate(keys)}
        counts = np.zeros(len(keys) + 1)
        counts[-1] = rej.sum()
        for k, i, j in zip(tri, np.floor(px).astype(int), np.floor(py).astype(int)):
            counts[index[(int(k), int(i), int(j))]] += 1  # (a point outside every cell of its triangle raises)
        expected = np.array([probs[k] for k in keys] + [p_rej]) * n
        assert abs(expected.sum() - n) < 1e-6 * n, expected.sum()
        big = expected >= 5
        obs = np.append(counts[big], counts[~big].sum())
        exp = np.append(expected[big], expected[~big].sum())
        if exp[-1] == 0:
            obs, exp = obs[:-1], exp[:-1]
        p = stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue
        assert p > 1e-4, (h, w, uvs, p)
        # the reported density at each accepted sample: the restatement's at the point's uv (computed in float, as the record gives it)
        uvt = uv[tri].astype(np.float32)
        b1f, b2f = b1.astype(np.float32), b2.astype(np.float32)
        puv = (np.float32(1) - (b1f + b2f))[:, None] * uvt[:, 0] + b1f[:, None] * uvt[:, 1] + b2f[:, None] * uvt[:, 2]
        want = np.array([ref.density(tab, t.shape, s, int(k), q, area) for k, q in zip(tri[:20000], puv[:20000])])
        got = dbl[acc, 2][:20000]
        close = np.isclose(got, want, rtol=1e-12, atol=0)
        assert close.mean() > 0.999, close.mean()  # (a point on a cell boundary may round into its neighbour)
        # quadrature of the density over the light: 1 - rejection
        m = 200
        gu, gv = np.meshgrid((np.arange(m) + 0.5) / m, (np.arange(m) + 0.5) / m)
        inside = gu + gv < 1  # barycentric grid: (b1, b2) = (gu, gv) on the half of the square inside the triangle
        bb1, bb2 = gu[inside], gv[inside]
        total = 0.0
        for k in range(len(uv)):
            q = ((1 - bb1 - bb2)[:, None] * uv[k, 0] + bb1[:, None] * uv[k, 1] + bb2[:, None] * uv[k, 2]).astype(np.float32)
            qs = torch.tensor(np.concatenate([np.full((len(q), 1), k, np.float32), q], 1)).to(dev)
            _, _, pd = c.scene.light_sample_test(0, torch.zeros(0, 3, dtype=torch.float64, device=dev), qs)
            total += float(pd.cpu().numpy().mean()) * tab["areas"][k]
        assert abs(total - (1 - p_rej)) < 0.02, (total, 1 - p_rej)
        print("sampler", h, w, uvs, "rejected %.3f (expected %.3f), chi2 p %.3g, integral %.4f" % (rej.mean(), p_rej, p, total), flush=True)


def update_check(rb, dev):
    """Toggling the option, new texels and a new uv_scale through Scene.update equal a new scene, table for table."""
    import torch
    base = window_image(8, 8, 3)
    states = [dict(tex=base, sampling="area"), dict(tex=base, sampling="texture"), dict(tex=base.flip(0).contiguous(), sampling="texture"),
              dict(tex=base, sampling="texture", uv_scale=(2.0, 0.5)), dict(tex=base, sampling="area")]
    c0, keep0 = native(rb, dev, light_scene(dev, states[0]["tex"], sampling="area"))
    scene = c0.scene
    for st in states[1:]:
        c, keep = native(rb, dev, light_scene(dev, st["tex"], sampling=st["sampling"], uv_scale=st.get("uv_scale", (1.0, 1.0))))
        scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=False)
        for name in TABLES[1:] + ("light_sampling",):
            assert scene.table(name).tobytes() == c.scene.table(name).tobytes(), (name, st["sampling"])
        from redner_b200 import api
        c.scene, fresh = scene, c.scene
        a = api._render(c)
        c.scene = fresh
        b = api._render(c)
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    del torch


def refusals_check(rb, dev):
    """A bad emission_sampling value and texture coordinates too large for the cell indices are refused, naming the emission sampling."""
    c, keep = native(rb, dev, light_scene(dev, window_image(8, 8, 1)))
    for value in (2, -1):
        c.lights[0]._c.emission_sampling = value
        for build in (True, False):
            try:
                if build:
                    rb.Scene(c.camera, c.shapes, c.materials, c.lights, None, dev.type == "cuda", -1, True, True)
                else:
                    c.scene.update(c.camera, c.shapes, c.materials, c.lights, None, geometry_changed=False)
            except RuntimeError as err:
                assert "emission_sampling" in str(err), str(err)
            else:
                raise AssertionError("accepted emission_sampling %d" % value)
    c.lights[0]._c.emission_sampling = 1
    c.scene.update(c.camera, c.shapes, c.materials, c.lights, None, geometry_changed=False)  # (usable again)
    big = light_scene(dev, window_image(8, 8, 1), uv_scale=(3e6, 1.0))
    try:
        native(rb, dev, big)
    except RuntimeError as err:
        assert "emission sampling" in str(err), str(err)
    else:
        raise AssertionError("accepted texture coordinates beyond 2^24 cells")
    # (and by an update: the uv_scale is a device value, so the refusal comes from the table build, and the scene is left incomplete)
    big.area_lights[0].emission_sampling = "area"
    cb, keep_b = native(rb, dev, big)
    cb.lights[0]._c.emission_sampling = 1
    try:
        cb.scene.update(cb.camera, cb.shapes, cb.materials, cb.lights, None, geometry_changed=False)
    except RuntimeError as err:
        assert "emission sampling" in str(err) and "rb_scene_update" in str(err), str(err)
    else:
        raise AssertionError("an update accepted texture coordinates beyond 2^24 cells")


def _lamp(dev, res, sampling, **kw):
    """The textured lamp of test_emission_cpu (a ramp texture with a uv_scale that requires grad, above a diffuse floor) under
    `sampling`, with the floor's diffuse reflectance requiring grad too."""
    import test_emission_cpu as em
    sc = em.lamp(dev, res, **kw)
    sc.area_lights[0].emission_sampling = sampling
    sc.materials[0].diffuse_reflectance.texels.requires_grad_()
    return sc


# (name, getter, index, eps) of the gradients that must not depend on the strategy.  The light's own vertex and uv gradients are left
# out: the adjoint omits the MIS weight's derivative (DESIGN.md section 7), which depends on the light pdf, so those two differ between
# the strategies by design.
GRADIENTS = [
    ("texel", lambda sc: sc.area_lights[0].emission.texels, 3 * (8 * 3 + 4) + 1, 0.2),
    ("intensity", lambda sc: sc.area_lights[0].intensity, 1, 0.2),
    # (uv_scale: means against the area strategy only.  Its finite difference on this lit lamp exceeds the analytic gradient under the
    # area strategy as well -- 3.3 against 1.1 on the emulator's lamp -- so that mismatch is the texture adjoint's under light and BSDF
    # sampling, not the strategy's: DESIGN.md section 7)
    ("uv_scale", lambda sc: sc.area_lights[0].emission.uv_scale, 0, None),
    ("floor reflectance", lambda sc: sc.materials[0].diffuse_reflectance.texels, 0, 0.1),
]


def gradient_checks(rb, dev, res, spp, fd_spp, seeds):
    """Under texture sampling: finite differences (fd_check of the pixel-filter suite, the tolerances of test_emission_cpu.fd_checks) of
    a texel, the intensity and the floor's reflectance; and the means over seeds of the same gradients against the area
    strategy's, within 4 combined standard errors."""
    import torch
    import test_pixel_filter_cpu as pf

    for name, getter, index, eps in GRADIENTS:
        if eps is None:
            continue

        def move(sc, d, getter=getter, index=index):
            with torch.no_grad():
                getter(sc).view(-1)[index] += d
                sc.area_lights[0].emission.texels = sc.area_lights[0].emission.texels  # (rebuild the mip pyramid from the texels)

        def grad_of(sc, getter=getter, index=index):
            t = getter(sc)
            return float(t.grad.view(-1)[index]) if t.grad is not None else 0.0
        pf.fd_check(rb, dev, lambda: _lamp(dev, res, "texture"), move, grad_of, None, spp, fd_spp, seeds, eps, mb=1, rel=0.05)
        print("fd", name, flush=True)
    means = {}
    for sampling in ("area", "texture"):
        per = []
        for k in range(2 * seeds):
            sc = _lamp(dev, res, sampling)
            import test_emission_cpu as em
            em.render(rb, dev, sc, spp, 200 + k, mb=1)
            per.append([float(getter(sc).grad.view(-1)[index]) for _, getter, index, _ in GRADIENTS])
        means[sampling] = np.array(per)
    for g, (name, _, _, _) in enumerate(GRADIENTS):
        a, t = means["area"][:, g], means["texture"][:, g]
        se = math.sqrt(a.var(ddof=1) / len(a) + t.var(ddof=1) / len(t))
        assert abs(a.mean() - t.mean()) <= 4 * se, (name, a.mean(), t.mean(), se)
        print("strategies agree on", name, a.mean(), t.mean(), se, flush=True)


def records_check(rb, dev, res=12, spp=4):
    """Exact records: the option off, on with a constant and on with an all-zero texture give the default's records word for word; with
    the option on, the records of a 2-way partition summed and rounded once equal one deterministic render."""
    import torch
    import test_emission_cpu as em
    from redner_b200 import api
    d_img = torch.rand(res, res, 3, generator=torch.Generator().manual_seed(11)).to(dev)

    def records(sc, part=None):
        c, keep = native(rb, dev, sc, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        g = api.RenderFunction.gradient_buffers(c)
        opts = api.RenderFunction.backward_options(c)
        if part is not None:
            c.scene.set_partition(part, 2, 4)
        return rb.render_exact(c.scene, opts, api._ptr(rb, d_img), g.d_scene).cpu().numpy(), c, g, keep

    for emission, sampling in (("image", "area"), ([0.5, 1.0, 2.0], "texture"), ("zero", "texture")):
        def make(s):
            sc = em.lamp(dev, res, emission="image" if emission == "zero" else emission)
            if emission == "zero":
                with torch.no_grad():
                    sc.area_lights[0].emission.texels.zero_()
            sc.area_lights[0].emission_sampling = s
            return sc
        assert records(make("area"))[0].tobytes() == records(make(sampling))[0].tobytes(), (emission, sampling)
    sc = _lamp(dev, res, "texture")
    whole, c, g, keep = records(sc)
    parts = records(sc, 0)[0] + records(sc, 1)[0]
    out = []
    for rec in (whole, parts):
        g = api.RenderFunction.gradient_buffers(c)
        rb.round_exact(c.scene, api.RenderFunction.backward_options(c), g.d_scene, None, torch.from_numpy(rec).to(dev))
        out.append({k: v.cpu().numpy().copy() for k, v in g.grads.items()})
    assert any(np.count_nonzero(v) for v in out[0].values())
    for k in out[0]:
        assert out[0][k].tobytes() == out[1][k].tobytes(), k


def stale_check(rb, dev, runs=16, spp=64):
    """Texels written in place without an update leave the tables stale: the render stays unbiased (its mean matches the quadrature of
    the new texels), only noisier."""
    import torch
    from redner_b200 import api
    tex = window_image(8, 8, 3)
    sc = light_scene(dev, tex, res=8)
    args = api.RenderFunction.serialize_scene(sc, 1, 1, device=dev, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False, channels=[rb.channels.position])
    pos = api.RenderFunction.apply(0, *args).cpu().numpy().astype(np.float64)
    args = api.RenderFunction.serialize_scene(sc, spp, 1, device=dev, backend=rb, sample_pixel_center=True, use_primary_edge_sampling=False,
                                              use_secondary_edge_sampling=False)
    c = api.RenderFunction._unpack((1, 2), args)  # (one native scene: its tables are those of the old texels)
    with torch.no_grad():
        sc.area_lights[0].emission.texels.copy_(tex.flip(1).to(dev))  # (in place: the scene reads the new texels, the tables stay)
    new = sc.area_lights[0].emission.texels.detach().cpu().numpy().astype(np.float64)
    ref_img = ref.quadrature(pos, new)
    imgs = []
    for k in range(runs):
        c.options.seed = 300 + k
        imgs.append(api._render(c).cpu().numpy().astype(np.float64))
    imgs = np.stack(imgs)
    tot = imgs.sum((1, 2, 3))
    assert abs(tot.mean() - ref_img.sum()) <= 4 * tot.std(ddof=1) / math.sqrt(runs), (tot.mean(), ref_img.sum())


def deterministic_check(rb, dev, res=12, spp=8):
    """Deterministic mode with the option on: repeatable; the record count and fingerprint are the area strategy's."""
    import torch
    import test_emission_cpu as em
    from redner_b200 import api

    def make(s):
        sc = em.lamp(dev, res)
        sc.area_lights[0].emission_sampling = s
        return sc
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a = em.render(rb, dev, make("texture"), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        b = em.render(rb, dev, make("texture"), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
        assert a[0].numpy().tobytes() == b[0].numpy().tobytes()
        em._bytes_equal(a[1], b[1])
        if dev.type == "cuda":
            os.environ["RB_BAND_BYTES"] = "65536"
            try:
                c = em.render(rb, dev, make("texture"), spp, 3, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
            finally:
                del os.environ["RB_BAND_BYTES"]
            em._bytes_equal(a[1], c[1])
    finally:
        torch.use_deterministic_algorithms(False)
    counts = []
    for s in ("area", "texture"):
        c, keep = native(rb, dev, make(s))
        g = api.RenderFunction.gradient_buffers(c)
        counts.append(rb.exact_record_count(c.scene, c.options, g.d_scene))
    assert counts[0] == counts[1]


def compare_render(rb, dev, res=16, spp=16):
    """Image and texture / light gradients of the textured lamp under texture sampling (both edge samplers), for the GPU-against-emulator
    comparison (vertex gradients excluded: see test_emission_cpu.compare_render)."""
    import test_emission_cpu as em
    sc = em.lamp(dev, res)
    sc.area_lights[0].emission_sampling = "texture"
    img, g = em.render(rb, dev, sc, spp, 9, use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
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


def test_option_off_constant_and_zero_textures_change_nothing():
    _run(["identity"])


def test_tables_equal_the_restatement():
    _run(["tables"])


def test_sampler_draws_from_its_density():
    _run(["sampler"])


def test_updates_equal_a_new_scene():
    _run(["update"])


def test_refusals_name_the_emission_sampling():
    _run(["refusals"])


def test_deterministic_repeatable():
    _run(["deterministic"])


def test_records_unchanged_when_off_and_partition_sums_equal_one_render():
    _run(["records"])


def test_stale_tables_render_unbiased():
    _run(["stale"])


def test_gradients_match_finite_differences_and_the_area_strategy():
    _run(["gradients"])


def test_api_rejects_an_unknown_strategy():
    import pytest
    import torch
    from redner_b200 import api
    with pytest.raises(ValueError, match="emission_sampling"):
        api.AreaLight(0, torch.ones(3), emission_sampling="bilinear")


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    dev = torch.device("cpu")
    checks = {"identity": identity_check, "tables": tables_check, "sampler": sampler_check, "update": update_check, "refusals": refusals_check,
              "deterministic": deterministic_check, "records": records_check, "stale": stale_check,
              "gradients": lambda rb, dev: gradient_checks(rb, dev, 12, 16, 128, 4)}
    for name in names:
        if name.startswith("compare:"):
            np.savez(name[len("compare:"):], **compare_render(rb, dev))
        else:
            checks[name](rb, dev)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
