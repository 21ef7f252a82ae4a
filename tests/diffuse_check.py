"""Helper of tests/test_diffuse_kernels_cpu.py (run as a subprocess, never imported by the product).

Binds the Python shim to one host build of the device headers (tools/cpu_emu) and renders the named cases of CASES: image and every
gradient of sum(img^2) are written to an .npz, or, when rb_render refuses the scene, its message.  The test runs it once with the lean
build (-DRB_LEAN) and once with the diffuse-only build (-DRB_LEAN -DRB_DIFFUSE) and compares the two files.

usage: python tests/diffuse_check.py <emulator.so> <out.npz> <case> [<case> ...]
"""
import ctypes
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))


def _diffuse_only(sc, api):
    """The scene with every material reduced to its diffuse reflectance and sidedness (compute_specular_lighting off)."""
    sc.materials = [api.Material(diffuse_reflectance=m.diffuse_reflectance, two_sided=m.two_sided) for m in sc.materials]
    return sc


def _one_feature(feature):
    """C1's triangle with one material feature switched on: each must send the scene back to the lean kernels."""
    def make(dev, resolution):
        import torch
        import scenes
        from redner_b200 import api
        sc = scenes.single_triangle(dev, resolution=resolution)
        m = sc.materials[0]
        kd = m.diffuse_reflectance
        if feature == "specular":
            sc.materials[0] = api.Material(diffuse_reflectance=kd, specular_reflectance=torch.tensor([0.0, 0.0, 0.0], device=dev))
        elif feature == "vertex_color":
            s = sc.shapes[0]
            s.colors = torch.full_like(s.vertices.detach(), 0.5)
            sc.materials[0] = api.Material(diffuse_reflectance=kd, use_vertex_color=True)
        else:
            sc.materials[0] = api.Material(diffuse_reflectance=kd, normal_map=api.Texture(torch.tensor([[[0.5, 0.5, 1.0]]], device=dev)))
        return sc
    return make


def _scene(name):
    import scenes
    from redner_b200 import api
    if name == "bunny_box_diffuse":
        return lambda dev, resolution: _diffuse_only(scenes.bunny_box_shifted(dev, resolution=resolution), api)
    if name.startswith("triangle_with_"):
        return _one_feature(name[len("triangle_with_"):])
    return scenes.SCENES[name]


# (scene, resolution, spp, max_bounces, edge samplers: bit 0 primary, bit 1 secondary, seed)
CASES = {
    "c1": ("single_triangle", 32, 4, 1, 3, 1),
    "c2": ("shadow_blocker", 48, 8, 1, 3, 2),
    "c2_all_vertices": ("shadow_blocker_all", 32, 8, 2, 3, 1),
    "bunny_box_diffuse": ("bunny_box_diffuse", 24, 2, 3, 1, 4),
    "triangle_with_specular": ("triangle_with_specular", 16, 2, 1, 1, 1),
    "triangle_with_vertex_color": ("triangle_with_vertex_color", 16, 2, 1, 1, 1),
    "triangle_with_normal_map": ("triangle_with_normal_map", 16, 2, 1, 1, 1),
}


def main():
    so, out, names = sys.argv[1], sys.argv[2], sys.argv[3:]
    import numpy as np
    import torch
    from redner_b200 import _lib
    _lib._lib = _lib._bind(ctypes.CDLL(so))  # this process only: the emulator exports the same C ABI with host pointers
    from redner_b200 import api
    from redner_b200 import redner as rb
    import parity_utils as pu
    dev = torch.device("cpu")
    res = {}
    for name in names:
        scene, size, spp, mb, edges, seed = CASES[name]
        sc = _scene(scene)(dev, resolution=(size, size))
        args = api.RenderFunction.serialize_scene(sc, spp, mb, sampler_type=rb.SamplerType.sobol, device=dev, backend=rb,
                                                  use_primary_edge_sampling=bool(edges & 1), use_secondary_edge_sampling=bool(edges & 2))
        try:
            img = api.RenderFunction.apply(seed, *args)
            img.pow(2).sum().backward()
        except RuntimeError as e:
            res[name + "/error"] = np.array(str(e))
            continue
        res[name + "/image"] = img.detach().numpy()
        for k, v in pu.collect_grads(sc).items():
            res[name + "/grad." + k] = v.numpy()
    np.savez(out, **res)


if __name__ == "__main__":
    main()
