"""GPU suite: updating a scene in place (rb_scene_update, redner.Scene.update, api.SceneRenderer).

After create(A) then update(B), every table of the scene -- BVH nodes and triangles, light PMF / CDF / areas / area-CDF pool and offsets,
edge list, primary-edge PMF / CDF, both secondary-edge trees -- must be what create(B) builds, byte for byte (the trees' weighted lengths
and billboard size with the tolerance of tests/test_scene_build_gpu.py), on the default path and with every table on the device
(RB_GPU_TREES=1).  The light tables built by rb_light_build.cu must also equal a NumPy float64 restatement in the same operation order.
Images rendered after an update are those of a new scene bit for bit; gradients agree up to the order of the atomics."""
import numpy as np
import pytest
import torch

import parity_utils as pu
import scenes
from redner_b200 import _lib as L
from redner_b200 import api

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CASES = ["single_triangle", "shadow_blocker", "glossy_room", "env_ball", "teapot_geometry", "bunny_box_shifted", "hires_room"]


def _rb():
    from redner_b200 import redner as rb
    return rb


def _opts(name):
    return dict(sampler_type=_rb().SamplerType.sobol, device=DEV, backend=_rb(), use_secondary_edge_sampling=name != "env_ball")


def _native(sc, name, scene=None, geometry=None):
    args = api.RenderFunction.serialize_scene(sc, 2, 1, **_opts(name))
    c = api.RenderFunction._unpack((1, 2), args, scene=scene, geometry_changed=geometry)
    c.args = args  # (the native scene holds raw pointers into these)
    return c


def _snapshot(scene):
    t = {n: scene.table(n) for n in L.RB_TABLES}
    t["edges"] = scene.edge_list()
    return t, scene.edge_trees()


def _assert_same_tables(a, b):
    (ta, (ra, csa, ncsa, exa)), (tb, (rb_, csb, ncsb, exb)) = a, b
    for k in ta:
        assert ta[k].shape == tb[k].shape and np.array_equal(ta[k], tb[k]), "%s differs (%s vs %s)" % (k, ta[k].shape, tb[k].shape)
    assert ra.shape == rb_.shape and (csa, ncsa) == (csb, ncsb), (ra.shape, rb_.shape, csa, csb, ncsa, ncsb)
    assert abs(exa - exb) <= 1e-6 * abs(exb)
    words = np.ones(32, dtype=bool)
    words[[12, 26]] = False  # wlen of either child
    words[28:] = False
    assert np.array_equal(ra[:, words], rb_[:, words])
    assert np.allclose(ra[:, [12, 26]].view(np.float32), rb_[:, [12, 26]].view(np.float32), rtol=3e-7, atol=0)


def _perturb(sc, gen, camera=True, in_place=False):
    """Moves every shape (the lights' too) by its own small offset and jitters one shape's vertices, scales every light's intensity and
    moves the camera.  New tensors, or (in_place) writes into the existing vertex tensors."""
    jitter = int(torch.randint(len(sc.shapes), (1,), generator=gen))
    for s, sh in enumerate(sc.shapes):
        v = sh.vertices.detach()
        d = 0.02 * torch.randn(3, generator=gen)
        if s == jitter:
            d = d + 1e-3 * torch.randn(v.shape, generator=gen)
        d = d.to(v.device)
        if in_place:
            with torch.no_grad():
                sh.vertices.add_(d)
        else:
            sh.vertices = (v + d).requires_grad_(sh.vertices.requires_grad)
    for light in sc.area_lights:
        light.intensity = (light.intensity.detach() * (0.5 + torch.rand(3, generator=gen))).requires_grad_(light.intensity.requires_grad)
    if camera:
        p = sc.camera.position
        sc.camera.position = (p.detach() + 0.05 * torch.randn(3, generator=gen)).requires_grad_(p.requires_grad)


def _numpy_light_tables(sc):
    """The light tables restated in NumPy float64 in the operation order of rb_light_build.cuh (np.cumsum is a serial in-order sum)."""
    pool, areas, offsets, pmf = [], [], [], []
    for light in sc.area_lights:
        sh = sc.shapes[light.shape_id]
        V = sh.vertices.detach().cpu().numpy().astype(np.float64)
        i = sh.indices.cpu().numpy()
        e1, e2 = V[i[:, 1]] - V[i[:, 0]], V[i[:, 2]] - V[i[:, 0]]
        cx, cy, cz = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2], e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
        a = 0.5 * np.sqrt(cx * cx + cy * cy + cz * cz)
        run = np.cumsum(a)
        total = run[-1] if len(a) else 0.0
        offsets.append(sum(len(p) for p in pool))
        pool.append(np.concatenate([[0.0], run[:-1]]) / total if len(a) else np.zeros(0))
        areas.append(total)
        it = light.intensity.detach().cpu().numpy().astype(np.float32).astype(np.float64)
        w = [np.float64(np.float32(x)) for x in (0.212671, 0.715160, 0.072169)]
        pmf.append(total * (w[0] * it[0] + w[1] * it[1] + w[2] * it[2]) * np.pi)
    if sc.envmap is not None:
        allv = np.concatenate([s.vertices.detach().cpu().numpy().reshape(-1, 3) for s in sc.shapes]).astype(np.float32)
        lo, hi = allv[:, :2].min(0), allv[:, :2].max(0)
        dx, dy = hi[0] - lo[0], hi[1] - lo[1]
        r = np.float64(np.float32(0.5) * np.sqrt(dx * dx + dy * dy + dy * dy))
        area = 4 * np.pi * r * r
        pmf.append(area / np.float64(np.float32(sc.envmap.pdf_norm)) if area > 0 else 1.0)
    pmf = np.array(pmf, np.float64)
    pmf = pmf / np.cumsum(pmf)[-1]
    cdf = np.concatenate([[0.0], np.cumsum(pmf)[:-1]])
    return {"light_pmf": pmf, "light_cdf": cdf, "light_areas": np.array(areas, np.float64), "area_cdf_pool": np.concatenate(pool).astype(np.float64),
            "area_cdf_offsets": np.array(offsets, np.int32)}


@pytest.mark.parametrize("gpu_trees", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_update_builds_the_tables_of_create(name, gpu_trees, monkeypatch):
    if gpu_trees:
        monkeypatch.setenv("RB_GPU_TREES", "1")
    gen = torch.Generator().manual_seed(11)
    sc = scenes.SCENES[name](DEV, resolution=(32, 32))
    a = _native(sc, name)
    _perturb(sc, gen)
    updated = _native(sc, name, scene=a.scene, geometry=False)  # (new vertex tensors: noticed without the flag)
    assert updated.scene is a.scene
    fresh = _native(sc, name)
    _assert_same_tables(_snapshot(updated.scene), _snapshot(fresh.scene))
    for k, v in _numpy_light_tables(sc).items():
        got = updated.scene.table(k)
        assert got.tobytes() == v.tobytes(), "%s: %s vs %s" % (k, got.view(v.dtype)[:4], v[:4])


def test_update_after_a_failed_update_rebuilds_everything():
    """An update that moved the vertices but failed at the light tables (no light importance left) is refused by rb_render; the next
    update, with the SAME vertex pointers and geometry_changed = 0, must still rebuild the BVH and the edge list the failed call never
    reached."""
    rb = _rb()
    gen = torch.Generator().manual_seed(2)
    sc = scenes.glossy_room(DEV, resolution=(32, 32))
    a = _native(sc, "glossy_room")
    _perturb(sc, gen)
    saved = [l.intensity for l in sc.area_lights]
    for l in sc.area_lights:
        l.intensity = torch.zeros(3)
    with pytest.raises(RuntimeError) as e:
        _native(sc, "glossy_room", scene=a.scene, geometry=True)
    assert "rb_scene_update: total light importance is not positive" in str(e.value), str(e.value)
    img = torch.zeros(32, 32, 3, device=DEV)
    with pytest.raises(RuntimeError) as e:
        rb.render(a.scene, a.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
    assert "last update failed" in str(e.value)
    for l, t in zip(sc.area_lights, saved):
        l.intensity = t
    updated = _native(sc, "glossy_room", scene=a.scene, geometry=False)
    _assert_same_tables(_snapshot(updated.scene), _snapshot(_native(sc, "glossy_room").scene))


def test_update_after_set_camera_restores_the_host_built_tables():
    """rb_scene_set_camera makes the camera tables on the device; an update of a small scene, whose build makes them on the host, makes
    them there again even with an unchanged camera."""
    sc = scenes.shadow_blocker(DEV, resolution=(32, 32))
    a = _native(sc, "shadow_blocker")
    a.scene.set_camera(a.camera)
    updated = _native(sc, "shadow_blocker", scene=a.scene, geometry=False)
    _assert_same_tables(_snapshot(updated.scene), _snapshot(_native(sc, "shadow_blocker").scene))
    assert np.array_equal(updated.scene.edge_trees()[0], _native(sc, "shadow_blocker").scene.edge_trees()[0])


@pytest.mark.parametrize("name", ["glossy_room", "teapot_geometry"])
def test_twenty_random_updates(name):
    gen = torch.Generator().manual_seed(5)
    sc = scenes.SCENES[name](DEV, resolution=(32, 32))
    c = _native(sc, name)
    scene = c.scene
    for step in range(20):
        in_place, camera = bool(torch.randint(2, (1,), generator=gen)), bool(torch.randint(2, (1,), generator=gen))
        if torch.randint(4, (1,), generator=gen) == 0:  # values only: intensities (and maybe the camera)
            for light in sc.area_lights:
                light.intensity = light.intensity.detach() * 1.1
            if camera:
                sc.camera.position = sc.camera.position.detach() + 0.03
            geometry = False
        else:
            _perturb(sc, gen, camera=camera, in_place=in_place)
            geometry = in_place
        c = _native(sc, name, scene=scene, geometry=geometry)
        _assert_same_tables(_snapshot(scene), _snapshot(_native(sc, name).scene))


def _render_both(render, sc, seed, opts):
    """SceneRenderer against RenderFunction with a new scene: image and gradients of sum(img^2)."""
    out = []
    for use_renderer in (True, False):
        for p in _params(sc):
            p.grad = None
        img = render(sc, seed) if use_renderer else api.RenderFunction.apply(seed, *api.RenderFunction.serialize_scene(sc, 4, 1, **opts))
        img.pow(2).sum().backward()
        out.append((img.detach(), [p.grad.detach().clone() if p.grad is not None else None for p in _params(sc)]))
    (ia, ga), (ib, gb) = out
    assert torch.equal(ia, ib)
    for x, y in zip(ga, gb):
        assert (x is None) == (y is None)
        if x is not None:
            assert pu.rel_l2(x.cpu().numpy(), y.cpu().numpy()) < 1e-4, pu.rel_l2(x.cpu().numpy(), y.cpu().numpy())


def _params(sc):
    return [t for s in sc.shapes for t in (s.vertices,) if t.requires_grad] + [l.intensity for l in sc.area_lights if l.intensity.requires_grad]


def test_edge_count_grows_and_shrinks():
    """Lifting one corner of the flat floor quad makes its diagonal an edge; flattening it again removes it."""
    sc = scenes.shadow_blocker(DEV, resolution=(32, 32), grad_all=True)
    opts = _opts("shadow_blocker")
    render = api.SceneRenderer(4, 1, **opts)
    _render_both(render, sc, 1, opts)
    n0 = render._scene.edge_list().shape[0]
    floor = sc.shapes[0].vertices.detach().clone()
    lifted = floor.clone()
    lifted[3, 1] += 0.3
    for k, (v, expect) in enumerate(((lifted, n0 + 1), (floor, n0))):
        sc.shapes[0].vertices = v.clone().requires_grad_(True)
        _render_both(render, sc, 2 + k, opts)
        assert render._scene.edge_list().shape[0] == expect
        _assert_same_tables(_snapshot(render._scene), _snapshot(_native(sc, "shadow_blocker").scene))


@pytest.mark.parametrize("name", ["teapot_geometry", "bunny_box_shifted"])
def test_renders_after_an_update_equal_a_new_scene(name):
    gen = torch.Generator().manual_seed(3)
    sc = scenes.SCENES[name](DEV, resolution=(48, 48))
    opts = dict(_opts(name), use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    render = api.SceneRenderer(4, 1, **opts)
    render(sc, 1)
    first = render._scene
    _perturb(sc, gen)
    _render_both(render, sc, 2, opts)
    assert render._scene is first


def test_device_memory_is_stable_over_many_updates():
    sc = scenes.hires_room(DEV, resolution=(32, 32))
    c = _native(sc, "hires_room")
    v = sc.shapes[3].vertices
    free = {}
    for k in range(200):
        with torch.no_grad():
            v.add_(1e-4)
        c.scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=True)
        if k + 1 in (10, 200):
            torch.cuda.synchronize()
            free[k + 1] = torch.cuda.mem_get_info()[0]
    assert abs(free[200] - free[10]) < 8 << 20, free


def _teapot_params(sc):
    m = sc.materials[-1]
    return [m.diffuse_reflectance.texels, m.specular_reflectance.texels, m.roughness.texels, sc.camera.position]


@pytest.mark.parametrize("name,pick", [("teapot", _teapot_params), ("bunny_box_shifted", lambda sc: [sc.shapes[-1].vertices])])
def test_scene_renderer_adam_loop_equals_a_new_scene_per_step(name, pick):
    """Adam on two copies of the scene in lock step: one rendered with RenderFunction (a new scene per step), the other through one
    SceneRenderer and given the first copy's parameters after every step (the gradients differ by the order of the atomics, and so
    would the trajectories)."""
    kw = dict(sampler_type=_rb().SamplerType.sobol, backend=_rb(), device=DEV)
    sa, sb = scenes.SCENES[name](DEV, resolution=(48, 48)), scenes.SCENES[name](DEV, resolution=(48, 48))
    pa, pb = pick(sa), pick(sb)
    for p in pa + pb:
        p.requires_grad_(True)
    opt = torch.optim.Adam(pa, lr=0.02)
    render = api.SceneRenderer(4, 1, **kw)
    for k in range(4):
        for p in pa + pb:
            p.grad = None
        ia = api.RenderFunction.apply(100 + k, *api.RenderFunction.serialize_scene(sa, 4, 1, **kw))
        ib = render(sb, 100 + k)
        ia.pow(2).sum().backward()
        ib.pow(2).sum().backward()
        assert torch.equal(ia, ib), k
        for x, y in zip(pa, pb):
            assert pu.rel_l2(y.grad.cpu().numpy(), x.grad.cpu().numpy()) < 1e-4, (k, pu.rel_l2(y.grad.cpu().numpy(), x.grad.cpu().numpy()))
        opt.step()
        with torch.no_grad():
            for x, y in zip(pa, pb):
                y.copy_(x)
