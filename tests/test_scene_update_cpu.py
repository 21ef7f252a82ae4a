"""CPU suite: updating a scene in place (rb_scene_update, redner.Scene.update, api.SceneRenderer).

- The decomposition the kernels of rb_light_build.cu use (per-triangle areas found through the pool offsets, one scan per light, bounds
  in another order), run in serial loops, gives the tables of host_build_lights byte for byte (tests/light_tables_check.cpp) on every
  fixture mesh and on random scenes, with and without an environment map.  Both call the arithmetic of rb_light_build.cuh, so this
  checks the decomposition; the arithmetic is compared with a NumPy restatement in tests/test_scene_update_gpu.py.
- On the host build of the device headers (tools/cpu_emu, whose rb_scene_update rebuilds every table from the descriptor): an Adam loop
  through SceneRenderer equals RenderFunction with a fresh scene per step; two renders before one backward() give the fresh-scene
  gradients; a changed index tensor or an added shape builds a new scene; a descriptor of another structure is refused and leaves the
  scene as it was.  The device side is tests/test_scene_update_gpu.py.

Run as a script (`python tests/test_scene_update_cpu.py <emulator.so> <check>...`) this file is also the subprocess that binds the
emulator in place of the library."""
import ctypes
import glob
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------- shared with the GPU suite
def adam_loop(dev, make_scene, pick, steps, spp, mb, use_renderer, **kw):
    """`steps` Adam steps on loss = sum(img^2) over the tensors pick(scene) returns; per step the image and the gradients.  Through one
    api.SceneRenderer, or RenderFunction with a fresh native scene per step."""
    import torch
    from redner_b200 import api
    sc = make_scene()
    params = pick(sc)
    for p in params:
        p.requires_grad_(True)
    opt = torch.optim.Adam(params, lr=0.02)
    render = api.SceneRenderer(spp, mb, device=dev, **kw) if use_renderer else None
    imgs, grads = [], []
    for k in range(steps):
        opt.zero_grad()
        if render is not None:
            img = render(sc, 100 + k)
        else:
            img = api.RenderFunction.apply(100 + k, *api.RenderFunction.serialize_scene(sc, spp, mb, device=dev, **kw))
        img.pow(2).sum().backward()
        imgs.append(img.detach().cpu())
        grads.append([p.grad.detach().cpu().clone() for p in params])
        opt.step()
    return imgs, grads


def assert_same_loop(a, b, grad_tol):
    import parity_utils as pu
    import torch
    (ia, ga), (ib, gb) = a, b
    for k, (x, y) in enumerate(zip(ia, ib)):
        assert torch.equal(x, y), "step %d: images differ" % k
    for k, (x, y) in enumerate(zip(ga, gb)):
        for j, (p, q) in enumerate(zip(x, y)):
            assert pu.rel_l2(p.numpy(), q.numpy()) < grad_tol, (k, j, pu.rel_l2(p.numpy(), q.numpy()))


def glossy_room_params(sc):
    """the sphere's vertices, the floor reflectance, one light's intensity and the camera position"""
    return [sc.shapes[3].vertices, sc.materials[0].diffuse_reflectance.texels, sc.area_lights[0].intensity, sc.camera.position]


# ---------------------------------------------------------------------------------------------------- light tables
@pytest.fixture(scope="module")
def light_checker(tmp_path_factory):
    if shutil.which("g++") is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("needs g++ and the CUDA headers")
    exe = str(tmp_path_factory.mktemp("light_tables") / "light_tables_check")
    cmd = ["g++", "-O2", "-std=c++17", "-w", "-include", os.path.join(ROOT, "tools", "cpu_emu", "emu_shim.h"), "-I/usr/local/cuda/include",
           "-I" + os.path.join(ROOT, "include"), os.path.join(HERE, "light_tables_check.cpp"), "-o", exe]
    subprocess.run(cmd, check=True, timeout=900)
    return exe


def test_light_steps_equal_the_host_builder_on_the_fixture_meshes(light_checker, tmp_path):
    files = []
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "scene_*.npz"))):
        d = np.load(path)
        out = str(tmp_path / (os.path.basename(path)[:-4] + ".bin"))
        with open(out, "wb") as f:
            stem = "shape" if "num_shapes" in d.files else "mesh"
            S = int(d["num_%ss" % ("shape" if stem == "shape" else "meshe")])
            np.array([S], np.int32).tofile(f)
            for s in range(S):
                v, i = d["%s%d.vertices" % (stem, s)].astype(np.float32), d["%s%d.indices" % (stem, s)].astype(np.int32)
                np.array([v.shape[0], i.shape[0]], np.int32).tofile(f)
                v.tofile(f)
                i.tofile(f)
        files.append(out)
    assert len(files) >= 2
    r = subprocess.run([light_checker] + files, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    ok = [l for l in r.stdout.splitlines() if l.startswith("ok ")]
    assert len(ok) == 2 * len(files), r.stdout


def test_light_steps_equal_the_host_builder_on_random_scenes(light_checker):
    r = subprocess.run([light_checker, "--random", "3000"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "random scenes 3000 mismatching 0"


# ---------------------------------------------------------------------------------------------------- on the emulator
@pytest.fixture(scope="module")
def emulator():
    from test_device_code_cpu import _build
    return _build()


def _check(so, names):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), so] + names, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("ok ")] == ["ok " + n for n in names]


def test_scene_renderer_adam_loop_equals_a_fresh_scene_per_step(emulator):
    _check(emulator, ["adam_loop"])


def test_backward_after_a_later_update_renders_its_own_state(emulator):
    _check(emulator, ["two_renders_one_backward"])


def test_changed_topology_builds_a_new_scene(emulator):
    _check(emulator, ["new_scene_on_structure_change"])


def test_update_of_another_structure_is_refused(emulator):
    _check(emulator, ["mismatch_refused"])


def test_failed_update_is_refused_by_render_and_recovered(emulator):
    _check(emulator, ["failed_update_recovers"])


# ---------------------------------------------------------------------------------------------------- the subprocess
def check_adam_loop(rb, dev):
    import scenes
    kw = dict(sampler_type=rb.SamplerType.sobol, backend=rb)

    def make():
        return scenes.glossy_room(dev, resolution=(20, 20), grad=False, textured=False)
    a = adam_loop(dev, make, glossy_room_params, 5, 2, 2, False, **kw)
    b = adam_loop(dev, make, glossy_room_params, 5, 2, 2, True, **kw)
    assert_same_loop(a, b, 1e-5)


def check_two_renders_one_backward(rb, dev):
    import torch
    import parity_utils as pu
    import scenes
    from redner_b200 import api
    kw = dict(sampler_type=rb.SamplerType.sobol, backend=rb, device=dev)

    def run(use_renderer):
        sc = scenes.glossy_room(dev, resolution=(16, 16), grad=False, textured=False)
        v1 = sc.shapes[3].vertices.requires_grad_(True)
        v2 = (v1.detach() + torch.tensor([0.05, -0.02, 0.03])).requires_grad_(True)
        inten = sc.area_lights[0].intensity.requires_grad_(True)
        render = api.SceneRenderer(2, 2, **kw) if use_renderer else (lambda s, seed: api.RenderFunction.apply(seed, *api.RenderFunction.serialize_scene(s, 2, 2, **kw)))
        img1 = render(sc, 5)
        sc.shapes[3].vertices = v2
        img2 = render(sc, 6)
        (img1.pow(2).sum() + 0.5 * img2.pow(2).sum()).backward()
        return [img1.detach(), img2.detach()], [v1.grad.clone(), v2.grad.clone(), inten.grad.clone()]
    (ia, ga), (ib, gb) = run(False), run(True)
    for x, y in zip(ia, ib):
        assert torch.equal(x, y)
    for x, y in zip(ga, gb):
        assert pu.rel_l2(y.numpy(), x.numpy()) < 1e-5, pu.rel_l2(y.numpy(), x.numpy())


def check_new_scene_on_structure_change(rb, dev):
    import torch
    import scenes
    from redner_b200 import api
    kw = dict(sampler_type=rb.SamplerType.sobol, backend=rb, device=dev)
    sc = scenes.shadow_blocker(dev, resolution=(12, 12))
    render = api.SceneRenderer(2, 1, **kw)

    def fresh(seed):
        return api.RenderFunction.apply(seed, *api.RenderFunction.serialize_scene(sc, 2, 1, **kw))
    assert torch.equal(render(sc, 1), fresh(1))
    first = render._scene
    sc.shapes[1].indices = sc.shapes[1].indices.clone()  # a new index tensor with the same contents: still an update
    assert torch.equal(render(sc, 2), fresh(2)) and render._scene is first
    sc.shapes[1].indices = torch.tensor([[0, 2, 1], [1, 2, 3]], dtype=torch.int32)  # other contents: a new scene
    assert torch.equal(render(sc, 3), fresh(3)) and render._scene is not first
    second = render._scene
    with torch.no_grad():
        sc.shapes[1].indices[0, 0] = 3  # written in place
    assert torch.equal(render(sc, 4), fresh(4)) and render._scene is not second
    third = render._scene
    sc.shapes.append(api.Shape(torch.tensor([[0.0, 1.0, 0.0], [0.5, 1.0, 0.0], [0.0, 1.0, 0.5]]), torch.tensor([[0, 1, 2]], dtype=torch.int32), 0))
    assert torch.equal(render(sc, 5), fresh(5)) and render._scene is not third


def check_mismatch_refused(rb, dev):
    import torch
    import scenes
    from redner_b200 import api
    sc = scenes.glossy_room(dev, resolution=(12, 12))
    args = api.RenderFunction.serialize_scene(sc, 2, 1, sampler_type=rb.SamplerType.sobol, backend=rb, device=dev)
    c = api.RenderFunction._unpack((1, 2), args)

    def image():
        img = torch.zeros(12, 12, 3)
        rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
        return img
    before = image()
    for shapes, lights, msg in ((c.shapes + c.shapes[:1], c.lights, "numbers of shapes, materials and lights"),
                                (c.shapes, c.lights[:1], "numbers of shapes, materials and lights"),
                                (c.shapes[:3] + c.shapes[2:3] + c.shapes[4:], c.lights, "vertex, triangle, uv or normal count")):
        with pytest.raises(RuntimeError) as e:
            c.scene.update(c.camera, shapes, c.materials, lights, c.envmap, geometry_changed=True)
        assert msg in str(e.value), str(e.value)
    assert torch.equal(image(), before)


def check_failed_update_recovers(rb, dev):
    """An update that fails after the checks (no light importance left) leaves a scene that rb_render refuses; SceneRenderer drops it and
    its next call builds a new scene, whose image is a fresh scene's."""
    import torch
    import scenes
    from redner_b200 import api
    kw = dict(sampler_type=rb.SamplerType.sobol, backend=rb, device=dev)
    sc = scenes.glossy_room(dev, resolution=(12, 12))
    render = api.SceneRenderer(2, 1, **kw)
    render(sc, 1)
    first = render._scene
    saved = [l.intensity for l in sc.area_lights]
    for l in sc.area_lights:
        l.intensity = torch.zeros(3)
    with pytest.raises(RuntimeError) as e:
        render(sc, 2)
    assert "rb_scene_update: total light importance is not positive" in str(e.value), str(e.value)
    assert render._scene is None
    img = torch.zeros(12, 12, 3)
    with pytest.raises(RuntimeError) as e:
        rb.render(first, rb.RenderOptions(1, 1, 1, [rb.channels.radiance], rb.SamplerType.sobol, False), rb.float_ptr(img.data_ptr()), rb.float_ptr(0),
                  None, rb.float_ptr(0), rb.float_ptr(0))
    assert "last update failed" in str(e.value), str(e.value)
    for l, t in zip(sc.area_lights, saved):
        l.intensity = t
    fresh = api.RenderFunction.apply(3, *api.RenderFunction.serialize_scene(sc, 2, 1, **kw))
    assert torch.equal(render(sc, 3), fresh) and render._scene is not first


def main():
    so, names = sys.argv[1], sys.argv[2:]
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    dev = torch.device("cpu")
    for name in names:
        globals()["check_" + name](rb, dev)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
