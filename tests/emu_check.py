"""Helper of tests/test_device_code_cpu.py (run as a subprocess, never imported by the product).

Binds the Python shim to the host-compiled build of the per-sample device headers (tools/cpu_emu: the same
rb_*.cuh sources the sm_90a kernels are made of, compiled with g++ and driven by plain loops) and checks the named
golden cases with the tolerances of the GPU suite.  This verifies the MATH of the device code on a machine without a GPU;
it says nothing about the kernels' launch structure, compaction, sorting or atomics, which only `-m gpu` covers.

usage: python tests/emu_check.py <emulator.so> <case> [<case> ...]
"""
import ctypes
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))


def check_batch_of_views(rb, dev):
    """api.render_batch (one native scene re-targeted per view with rb_scene_set_camera) == one full Scene per view: images bit for bit,
    gradients to 1e-5 -- the host logic of SURVEY.md section 8f rank 2, on the host build of the device headers."""
    import torch
    import parity_utils as pu
    import scenes
    from redner_b200 import api

    def make():
        views = [scenes.glossy_room(dev, resolution=(24, 24)) for _ in range(3)]
        cams = [([0.3, 1.4, -4.5], [0.0, 0.6, 0.0]), ([1.2, 1.1, -4.0], [0.1, 0.5, 0.1]), ([-0.8, 1.8, -4.2], [0.0, 0.7, 0.2])]
        for v, (p, l) in zip(views, cams):
            v.camera = api.Camera(position=torch.tensor(p, requires_grad=True), look_at=torch.tensor(l, requires_grad=True),
                                  up=torch.tensor([0.0, 1.0, 0.0], requires_grad=True), fov=torch.tensor([40.0]), clip_near=1e-2, resolution=(24, 24))
            v.shapes, v.materials, v.area_lights = views[0].shapes, views[0].materials, views[0].area_lights
        return views
    kw = dict(sampler_type=rb.SamplerType.sobol, device=dev, backend=rb)
    views = make()
    imgs = api.render_batch(views, 4, 2, [11, 12, 13], **kw)
    imgs.pow(2).sum().backward()
    g_batch = pu.collect_grads(views[0])
    cam_batch = [v.camera.position.grad.clone() for v in views]
    views = make()
    singles = [api.RenderFunction.apply(11 + k, *api.RenderFunction.serialize_scene(v, 4, 2, **kw)) for k, v in enumerate(views)]
    sum(s.pow(2).sum() for s in singles).backward()
    g_single = pu.collect_grads(views[0])
    for k in range(3):
        assert torch.equal(imgs[k], singles[k]), k
        assert pu.rel_l2(cam_batch[k].numpy(), views[k].camera.position.grad.numpy()) < 1e-5
    for key in g_single:
        if not key.startswith("cam."):
            assert pu.rel_l2(g_batch[key].numpy(), g_single[key].numpy()) < 1e-5, key


def check_rejected_options(rb, dev):
    """rb_render rejects a duplicated radiance channel, an unknown channel, more than 64 image dimensions and more than 64 bounces with
    secondary edge sampling, with the library's messages.  Called through the C ABI: the Python shim refuses an unknown channel itself."""
    import ctypes as C
    import scenes
    from redner_b200 import _lib as L, api
    sc = scenes.corner_ball(dev, resolution=(8, 8), variant="generic")  # (a 5-channel generic texture; differentiable, so edges are sampled)
    args = api.RenderFunction.serialize_scene(sc, 1, 1, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                              use_primary_edge_sampling=True, use_secondary_edge_sampling=True)
    scene = api.RenderFunction._unpack((1, 2), args).scene
    lib = L._lib
    image = (C.c_float * (8 * 8 * 128))()
    d_image = (C.c_float * (8 * 8 * 3))()
    light_grads = [(C.c_float * 3)() for _ in range(2)]
    d_shapes, d_mats = (L.rb_dshape * 4)(), (L.rb_material * 3)()
    d_lights = (C.c_void_p * 2)(*[C.addressof(g) for g in light_grads])
    d_scene = L.rb_dscene_desc(num_shapes=4, shapes=d_shapes, num_materials=3, materials=d_mats, num_lights=2, light_intensity=d_lights)

    def render(channels, max_bounces=1, backward=False):
        o = L.rb_options(seed=1, num_samples=1, max_bounces=max_bounces, num_channels=len(channels), sampler_type=1, sample_pixel_center=0)
        chs = (C.c_int * len(channels))(*channels)
        o.channels = chs
        rc = lib.rb_render(scene._handle, C.byref(o), None if backward else image, d_image if backward else None, C.byref(d_scene) if backward else None,
                           None, None)
        return rc, L.last_error(lib)

    radiance, generic = int(rb.channels.radiance), int(rb.channels.generic_texture)
    assert render([radiance]) == (0, "")
    assert render([radiance, radiance]) == (1, "Duplicated radiance channel")
    assert render([radiance, 99]) == (1, "rb_render: unknown channel")
    assert render([generic] * 13) == (1, "rb_render: more than 64 image dimensions requested")
    assert render([radiance], max_bounces=65, backward=True) == (1, "rb_render: secondary edge sampling supports at most 64 bounces")


def main():
    so, names = sys.argv[1], sys.argv[2:]
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import redner as rb
    import parity_utils as pu
    dev = torch.device("cpu")
    checks = {"batch_of_views": check_batch_of_views, "rejected_options": check_rejected_options}
    for name in names:
        if name in checks:
            checks[name](rb, dev)
            print("ok", name, flush=True)
            continue
        if name in pu.STAT_CASES:
            pu.assert_stat_matches_golden(name, pu.render_stat_case(rb, dev, name))
        elif name in pu.SCREEN_CASES:
            pu.assert_screen_gradient_matches_golden(name, pu.render_screen_gradient(rb, dev, pu.SCREEN_CASES[name]).numpy())
        elif name in pu.GBUFFER_CASES:
            pu.assert_gbuffer_matches_golden(name, pu.render_gbuffer(rb, dev, pu.GBUFFER_CASES[name]).numpy())
        else:
            cfg = pu.CASES[name] if name in pu.CASES else pu.REFSTREAM_CASES[name]
            img, grads = pu.render_case(rb, dev, cfg, cfg["seed"])
            pu.assert_matches_golden(name, img.numpy(), grads)
        print("ok", name, flush=True)


if __name__ == "__main__":
    main()
