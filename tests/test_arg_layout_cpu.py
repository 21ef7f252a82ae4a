"""CPU suite: the layout of RenderFunction.serialize_scene's argument list as RenderFunction.read_args reads it.

- For every fixture scene and for variants with a cam_to_world camera, lens distortion, an environment map, generic and normal-map
  textures, uv / normal / colour buffers and a pixel filter, read_args returns the scene's own tensors under their names, and the position
  it records for each is that tensor's index in the list.
- The positions of the gradients RenderFunction.backward returns are pinned for four scenes: bench.py names each gradient it writes
  after that position (grad_argNNN), so a change of the list's layout must show up here.

Pure Python: serialize_scene and gradient_buffers only use the enums and descriptor classes of redner_b200.redner, not its library."""
import math

import pytest
import torch

import scenes
from redner_b200 import api
from redner_b200 import redner as rb

CPU = torch.device("cpu")
RES = (6, 8)


def _cam_to_world_camera(distortion):
    a = 0.3
    c2w = torch.tensor([[math.cos(a), 0.0, math.sin(a), 0.3], [0.0, 1.0, 0.0, 1.4], [-math.sin(a), 0.0, math.cos(a), -4.5], [0.0, 0.0, 0.0, 1.0]])
    d = torch.tensor([0.12, -0.05, 0.01, 0.02, 0.01, -0.004, 0.01, -0.015]) if distortion else None
    return api.Camera(cam_to_world=c2w, fov=torch.tensor([40.0]), clip_near=1e-2, resolution=RES, distortion_params=d)


def _with_camera(make, distortion):
    def scene():
        sc = make()
        sc.camera = _cam_to_world_camera(distortion)
        return sc
    return scene


# name: (scene factory, serialize_scene options)
VARIANTS = {name: (lambda f=f: f(CPU, resolution=RES), {}) for name, f in scenes.SCENES.items()}
VARIANTS.update({
    "glossy_room_cam_to_world": (_with_camera(lambda: scenes.glossy_room(CPU, resolution=RES), False), {}),
    "nmap_room_cam_to_world_distortion": (_with_camera(lambda: scenes.nmap_room(CPU, resolution=RES), True), {}),
    "corner_ball_generic": (lambda: scenes.corner_ball(CPU, resolution=RES, variant="generic"), {}),
    "corner_ball_viewport": (lambda: scenes.corner_ball(CPU, variant="viewport"), {}),
    "glossy_room_tent_filter": (lambda: scenes.glossy_room(CPU, resolution=RES), {"pixel_filter": api.PixelFilter("tent", 2.0)}),
    "env_ball_no_edges": (lambda: scenes.env_ball(CPU, resolution=RES), {"use_primary_edge_sampling": False, "use_secondary_edge_sampling": False}),
})


def _serialize(name):
    make, kw = VARIANTS[name]
    sc = make()
    kw = dict(kw)
    kw.setdefault("use_secondary_edge_sampling", sc.envmap is None)
    args = api.RenderFunction.serialize_scene(sc, (3, 5), 2, sampler_type=rb.SamplerType.sobol, device=CPU, backend=rb, **kw)
    return sc, args


def _index(args, t):
    return next(i for i, x in enumerate(args) if x is t)


def _assert_entry(args, entries, positions, name, expected):
    """entries.<name> is `expected` itself and positions.<name> is where it sits in `args` (for a tensor: its first occurrence)."""
    value, pos = getattr(entries, name), getattr(positions, name)
    assert value is expected, name
    assert args[pos] is expected, name
    if isinstance(expected, torch.Tensor):
        assert pos == _index(args, expected), name


def _assert_texture(args, entry, positions, tex):
    if tex is None:
        assert entry is None and positions is None
        return
    assert len(entry.mips) == len(tex.mipmap) == len(positions.mips)
    for m, p, expected in zip(entry.mips, positions.mips, tex.mipmap):
        assert m is expected and args[p] is expected and p == _index(args, expected)
    _assert_entry(args, entry, positions, "uv_scale", tex.uv_scale)


def _pairs(values, positions):
    """(entry, position) of every entry read_args returned, flattened along its `pos` structure."""
    if positions is None:
        return []
    if isinstance(positions, int):
        return [(values, positions)]
    return [pair for v, p in zip(values, positions) for pair in _pairs(v, p)]


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_read_args_returns_the_scene_tensors_at_their_positions(name):
    sc, args = _serialize(name)
    a = api.RenderFunction.read_args(args)
    p = a.pos
    assert a.args is args
    cam = sc.camera
    for field in ("position", "look_at", "up", "cam_to_world", "world_to_cam", "intrinsic_mat_inv", "intrinsic_mat", "distortion_params"):
        _assert_entry(args, a.camera_args, p.camera_args, field, getattr(cam, field))
    c = a.camera_args
    assert c.clip_near == cam.clip_near and c.resolution == cam.resolution and c.camera_type == cam.camera_type
    assert len(a.shape_args) == len(p.shape_args) == len(sc.shapes)
    for s, q, shape in zip(a.shape_args, p.shape_args, sc.shapes):
        for field in ("vertices", "indices", "uvs", "normals", "uv_indices", "normal_indices", "colors"):
            _assert_entry(args, s, q, field, getattr(shape, field))
        assert (s.material_id, s.light_id) == (shape.material_id, shape.light_id)
    assert len(a.mat_args) == len(p.mat_args) == len(sc.materials)
    for m, q, mat in zip(a.mat_args, p.mat_args, sc.materials):
        for entry, positions, tex in zip(m.textures, q.textures,
                                         (mat.diffuse_reflectance, mat.specular_reflectance, mat.roughness, mat.generic_texture, mat.normal_map)):
            _assert_texture(args, entry, positions, tex)
        assert (m.compute_specular_lighting, m.two_sided, m.use_vertex_color) == (mat.compute_specular_lighting, mat.two_sided, mat.use_vertex_color)
    assert len(a.light_args) == len(p.light_args) == len(sc.area_lights)
    for l, q, light in zip(a.light_args, p.light_args, sc.area_lights):
        _assert_entry(args, l, q, "intensity", light.intensity)
        assert (l.shape_id, l.two_sided, l.directly_visible) == (light.shape_id, light.two_sided, light.directly_visible)
    if sc.envmap is None:
        assert a.env_args is None and p.env_args is None
    else:
        e = sc.envmap
        _assert_texture(args, a.env_args.values, p.env_args.values, e.values)
        for field in ("env_to_world", "world_to_env", "sample_cdf_ys", "sample_cdf_xs"):
            _assert_entry(args, a.env_args, p.env_args, field, getattr(e, field))
        assert (a.env_args.pdf_norm, a.env_args.directly_visible) == (e.pdf_norm, e.directly_visible)
    o = a.option_args
    pixel_filter = VARIANTS[name][1].get("pixel_filter")
    assert (o.num_samples, o.max_bounces, o.channels, o.sampler_type) == ((3, 5), 2, [rb.channels.radiance], rb.SamplerType.sobol)
    assert o.pixel_filter == (pixel_filter.native() if pixel_filter is not None else None)
    assert o.device == CPU and o.backend is rb
    # every entry sits where its position says, and what no position names are the counts: of shapes / materials / lights and of each
    # texture's mip levels (None for no environment map)
    pairs = _pairs([a.camera_args, a.shape_args, a.mat_args, a.light_args, a.env_args, a.option_args],
                   [p.camera_args, p.shape_args, p.mat_args, p.light_args, p.env_args, p.option_args])
    assert all(args[pos] is v for v, pos in pairs)
    named = [pos for _, pos in pairs]
    assert len(named) == len(set(named))
    counts = sorted(set(range(len(args))) - set(named))
    assert counts[:3] == [0, 1, 2] and len(counts) == 3 + 5 * len(a.mat_args) + 1
    assert all(args[i] is None or type(args[i]) is int for i in counts)


# Positions (in RenderFunction.backward's return value: 1 + the index in serialize_scene's list) of the gradients of four scenes.
GRADIENT_POSITIONS = {
    "single_triangle": [4, 5, 6, 9, 10, 16, 25, 35, 36, 38, 39, 41, 42, 49],
    "env_ball": [4, 5, 6, 9, 10, 16, 18, 25, 27, 28, 34, 44, 45, 46, 47, 48, 50, 51, 53, 54, 61, 62, 64, 65, 67, 68, 75, 76, 78, 79, 81, 82, 89, 93,
                 94, 95, 96, 97, 98, 99, 101],
    "corner_ball_generic": [4, 5, 6, 9, 10, 16, 18, 19, 22, 25, 34, 43, 53, 54, 56, 57, 59, 60, 62, 63, 64, 65, 66, 72, 73, 75, 76, 78, 79, 86, 87,
                            89, 90, 92, 93, 100, 104],
    "nmap_room_cam_to_world_distortion": [7, 8, 9, 10, 11, 16, 18, 25, 34, 43, 45, 46, 52, 61, 71, 72, 73, 74, 75, 76, 78, 79, 81, 82, 83, 84, 85, 86,
                                          93, 94, 96, 97, 99, 100, 107, 108, 110, 111, 112, 113, 114, 116, 117, 120, 121, 122, 123, 124, 129, 130,
                                          132, 133, 135, 136, 143, 147],
}


@pytest.mark.parametrize("name", sorted(GRADIENT_POSITIONS))
def test_gradient_positions_are_pinned(name):
    _, args = _serialize(name)
    c = api.RenderFunction.read_args(args)
    out = api.RenderFunction.gradient_outputs(c, api.RenderFunction.gradient_buffers(c))
    assert len(out) == 1 + len(args)
    positions = [i for i, t in enumerate(out) if t is not None]
    assert positions == GRADIENT_POSITIONS[name]
    for i in positions:
        assert out[i].shape == args[i - 1].shape and out[i].dtype == args[i - 1].dtype and out[i].device == args[i - 1].device, i
