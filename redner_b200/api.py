"""Host-side mirror of the pyredner interface for the one hot path (RenderFunction.forward / backward).

Same names, argument meaning and error behaviour as the reference's Python layer, written from scratch:
  Camera      pyredner/camera.py:61-122          Shape      pyredner/shape.py:327-402
  Texture     pyredner/texture.py:10-100         Material   pyredner/material.py:36-100
  AreaLight   pyredner/area_light.py             Scene      pyredner/scene.py:5-68
  RenderFunction.serialize_scene / forward / backward   pyredner/render_pytorch.py:68-269 / :652-707 / :1051-1177

`RenderFunction` drives any module that exposes the `redner` pybind surface (src/redner.cpp:20-272).  The product uses
`redner_b200.redner` (ctypes -> libredner_b200.so -> sm_90a kernels).  The tests additionally pass the compiled,
unmodified reference module (oracle/_ref) through the very same host code to obtain the oracle's images and gradients.
"""
import math
from collections import namedtuple
from types import SimpleNamespace
from typing import List, Optional, Tuple, Union

import torch

_backend = None
_device = None
_use_correlated_random_number = False


def default_backend():
    global _backend
    if _backend is None:
        from . import redner as rb  # raises if libredner_b200.so is not built
        _backend = rb
    return _backend


def set_device(device):
    """pyredner.set_device (pyredner/device.py:26-33)."""
    global _device
    _device = torch.device(device)


def get_device():
    if _device is not None:
        return _device
    if torch.cuda.is_available():
        return torch.device("cuda:%d" % torch.cuda.current_device())
    raise RuntimeError("redner_b200: no CUDA device is visible and there is no CPU fallback for rendering")


def set_use_correlated_random_number(v: bool):
    global _use_correlated_random_number
    _use_correlated_random_number = bool(v)


class Camera:
    def __init__(self, position=None, look_at=None, up=None, fov=None, clip_near: float = 1e-4, resolution: Tuple[int, int] = (256, 256),
                 viewport=None, cam_to_world=None, intrinsic_mat=None, distortion_params=None, camera_type=0):
        if position is None and look_at is None and up is None:
            assert cam_to_world is not None
        for t, n in ((position, 3), (look_at, 3), (up, 3), (fov, 1)):
            if t is not None:
                assert t.dtype == torch.float32 and tuple(t.shape) == (n,)
        assert isinstance(clip_near, float)
        self.position, self.look_at, self.up = position, look_at, up
        self.fov = fov
        self.cam_to_world = cam_to_world
        self.world_to_cam = torch.inverse(cam_to_world).contiguous() if cam_to_world is not None else None
        if intrinsic_mat is None:
            if int(camera_type) == 0:
                f = 1.0 / torch.tan(0.5 * fov * (math.pi / 180.0))
                one = torch.ones([1], dtype=torch.float32, device=f.device)
                intrinsic_mat = torch.diag(torch.cat([f, f, one], 0)).contiguous()
            else:
                intrinsic_mat = torch.eye(3, dtype=torch.float32)
        self.intrinsic_mat = intrinsic_mat
        self.intrinsic_mat_inv = torch.inverse(intrinsic_mat).contiguous()
        self.distortion_params = distortion_params
        self.clip_near = clip_near
        self.resolution = resolution  # (height, width)
        self.viewport = viewport      # (y0, x0, y1, x1) or None
        self.camera_type = camera_type


class Texture:
    """Texture + box-filtered mip pyramid (pyredner/texture.py:34-70)."""

    def __init__(self, texels: torch.Tensor, uv_scale: Optional[torch.Tensor] = None):
        if uv_scale is None:
            uv_scale = torch.tensor([1.0, 1.0], device=texels.device)
        assert texels.dtype == torch.float32 and uv_scale.dtype == torch.float32
        self.uv_scale = uv_scale
        self.texels = texels

    @property
    def texels(self):
        return self._texels

    @texels.setter
    def texels(self, value):
        self._texels = value
        t = value
        if t.dim() >= 2:
            size = max(t.shape[0], t.shape[1])
            levels = min(math.ceil(math.log(size, 2) + 1), 8)
            ch = t.shape[2]
            box = torch.ones(ch, 1, 2, 2, device=t.device) / 4.0
            mip = [t.contiguous()]
            prev = t.unsqueeze(0).permute(0, 3, 1, 2)
            for _ in range(1, levels):
                cur = torch.nn.functional.pad(prev, (0, 1, 0, 1), mode="circular")
                cur = torch.nn.functional.conv2d(cur, box, groups=ch)
                size_next = (max(cur.shape[2] // 2, 1), max(cur.shape[3] // 2, 1))
                cur = torch.nn.functional.interpolate(cur, size=size_next, mode="area")
                mip.append(cur.squeeze(0).permute(1, 2, 0).contiguous())
                prev = cur
        else:
            mip = [t]
        self.mipmap = mip


def _as_texture(x, default=None):
    if x is None:
        return default
    if isinstance(x, Texture):
        return x
    return Texture(x)


class Material:
    def __init__(self, diffuse_reflectance=None, specular_reflectance=None, roughness=None, generic_texture=None, normal_map=None,
                 two_sided: bool = False, use_vertex_color: bool = False):
        if diffuse_reflectance is None:
            diffuse_reflectance = torch.zeros(3)
        dev = diffuse_reflectance.texels.device if isinstance(diffuse_reflectance, Texture) else diffuse_reflectance.device
        compute_specular = specular_reflectance is not None
        if specular_reflectance is None:
            specular_reflectance = torch.zeros(3, device=dev)
        if roughness is None:
            roughness = torch.ones(1, device=dev)
        self.diffuse_reflectance = _as_texture(diffuse_reflectance)
        self.specular_reflectance = _as_texture(specular_reflectance)
        self.roughness = _as_texture(roughness)
        self.generic_texture = _as_texture(generic_texture)
        self.normal_map = _as_texture(normal_map)
        self.compute_specular_lighting = compute_specular
        self.two_sided = two_sided
        self.use_vertex_color = use_vertex_color


class Shape:
    def __init__(self, vertices, indices, material_id: int, uvs=None, normals=None, uv_indices=None, normal_indices=None, colors=None):
        assert vertices.dtype == torch.float32 and vertices.is_contiguous() and vertices.dim() == 2 and vertices.shape[1] == 3
        assert indices.dtype == torch.int32 and indices.is_contiguous() and indices.dim() == 2 and indices.shape[1] == 3
        for t, dt in ((uvs, torch.float32), (normals, torch.float32), (uv_indices, torch.int32), (normal_indices, torch.int32), (colors, torch.float32)):
            if t is not None:
                assert t.dtype == dt and t.is_contiguous()
        self.vertices, self.indices, self.material_id = vertices, indices, material_id
        self.uvs, self.normals, self.uv_indices, self.normal_indices, self.colors = uvs, normals, uv_indices, normal_indices, colors
        self.light_id = -1


class AreaLight:
    def __init__(self, shape_id: int, intensity: torch.Tensor, two_sided: bool = False, directly_visible: bool = True):
        assert intensity.dtype == torch.float32 and tuple(intensity.shape) == (3,)
        self.shape_id, self.intensity, self.two_sided, self.directly_visible = shape_id, intensity, two_sided, directly_visible


class EnvironmentMap:
    """pyredner.EnvironmentMap (pyredner/envmap.py:6-86): latitude-longitude radiance image infinitely far away, with the
    luminance x sin(theta) sampling tables the renderer importance-samples (generate_envmap_pdf, :36-61)."""

    def __init__(self, values, env_to_world: Optional[torch.Tensor] = None, directly_visible: bool = True):
        self.values = values if isinstance(values, Texture) else Texture(values)
        self.env_to_world = env_to_world if env_to_world is not None else torch.eye(4, 4)
        assert self.env_to_world.dtype == torch.float32
        self.world_to_env = torch.inverse(self.env_to_world).contiguous()
        self.directly_visible = directly_visible
        t = self.values.texels.detach()
        assert t.dim() == 3 and t.shape[2] == 3, "the environment map must be an image [height, width, 3]"
        lum = 0.212671 * t[:, :, 0] + 0.715160 * t[:, :, 1] + 0.072169 * t[:, :, 2]
        cdf_xs_ = torch.cumsum(lum, dim=1)
        y_weight = torch.sin(math.pi * (torch.arange(lum.shape[0], dtype=torch.float32, device=lum.device) + 0.5) / float(lum.shape[0]))
        cdf_ys_ = torch.cumsum(cdf_xs_[:, -1] * y_weight, dim=0)
        self.pdf_norm = (lum.shape[0] * lum.shape[1]) / (cdf_ys_[-1].item() * (2 * math.pi * math.pi))
        self.sample_cdf_xs = ((cdf_xs_ - cdf_xs_[:, 0:1]) / torch.clamp(cdf_xs_[:, -1:], min=1e-8)).contiguous()
        self.sample_cdf_ys = ((cdf_ys_ - cdf_ys_[0]) / torch.clamp(cdf_ys_[-1], min=1e-8)).contiguous()


class PixelFilter:
    """Pixel reconstruction filter of a scene (redner_b200 extension; the reference integrates over the 1 x 1 pixel box).  `width` in
    pixels: the box's side, the tent's base width, the Gaussian's truncation interval (sigma = width / 6); at most 4.  Passed as
    `pixel_filter=` to serialize_scene and everything that forwards its options; None keeps the 1-pixel box."""
    KINDS = ("box", "tent", "gaussian")  # rb_filter_type

    def __init__(self, kind: str = "box", width: float = 1.0):
        if kind not in self.KINDS:
            raise ValueError("PixelFilter: kind must be one of %s, not %r" % (", ".join(self.KINDS), kind))
        self.kind, self.width = kind, float(width)

    def native(self):
        """(rb_filter_type, width) as redner.Scene takes it."""
        return self.KINDS.index(self.kind), self.width


class Scene:
    def __init__(self, camera: Camera, shapes: List[Shape], materials: List[Material], area_lights: List[AreaLight], envmap=None):
        self.camera, self.shapes, self.materials, self.area_lights, self.envmap = camera, shapes, materials, area_lights, envmap


# The entries serialize_scene writes for one camera, shape, texture, material, light, environment map and the options, in their order
# (RenderFunction.read_args).
_CameraArgs = namedtuple("_CameraArgs", "position look_at up cam_to_world world_to_cam intrinsic_mat_inv intrinsic_mat distortion_params clip_near "
                                        "resolution viewport camera_type")
_ShapeArgs = namedtuple("_ShapeArgs", "vertices indices uvs normals uv_indices normal_indices colors material_id light_id")
_TextureArgs = namedtuple("_TextureArgs", "mips uv_scale")
_MaterialArgs = namedtuple("_MaterialArgs", "textures compute_specular_lighting two_sided use_vertex_color")
_LightArgs = namedtuple("_LightArgs", "shape_id intensity two_sided directly_visible")
_EnvmapArgs = namedtuple("_EnvmapArgs", "values env_to_world world_to_env sample_cdf_ys sample_cdf_xs pdf_norm directly_visible")
_OptionArgs = namedtuple("_OptionArgs", "num_samples max_bounces channels sampler_type use_primary_edge_sampling use_secondary_edge_sampling "
                                        "sample_pixel_center pixel_filter device backend")


def _ptr(backend, t, kind="float"):
    ctor = backend.float_ptr if kind == "float" else backend.int_ptr
    return ctor(t.data_ptr() if t is not None else 0)


def _native_texture(rb, cls, channels, tex, buffers=None):
    """rb.Texture1 / Texture3 / TextureN of the texture entry `tex` of read_args (None: no texture, of `channels` channels), pointing at
    the texture's own tensors, or at `buffers` = (mips, uv_scale) of the same shapes: its gradient."""
    if tex is None:
        return cls([], [], [], channels, rb.float_ptr(0))
    mips, uv_scale = buffers or (tex.mips, tex.uv_scale)
    first = tex.mips[0]
    if first.dim() == 3:
        return cls([_ptr(rb, m) for m in mips], [int(m.shape[1]) for m in tex.mips], [int(m.shape[0]) for m in tex.mips], int(first.shape[2]),
                   _ptr(rb, uv_scale))
    return cls([_ptr(rb, mips[0])], [0], [0], int(first.shape[0]), _ptr(rb, uv_scale))


def _material_textures(rb):
    """(class, channels of an absent texture) of a material's textures, in the order of read_args: diffuse, specular, roughness,
    generic, normal map."""
    return (rb.Texture3, 3), (rb.Texture3, 3), (rb.Texture1, 1), (rb.TextureN, 0), (rb.Texture3, 3)


def _image_shape(c):
    """(height, width, channels) of the image of the unpacked call `c`."""
    vp = c.viewport
    return vp[2] - vp[0], vp[3] - vp[1], c.backend.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)


def _render(c):
    """The image of the unpacked call `c`, rendered into a new zeroed tensor."""
    rb = c.backend
    img = torch.zeros(*_image_shape(c), device=c.device)
    rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
    return img


def _backward(c, grad_img, screen_grad=None):
    """The backward pass of the unpacked call `c` for d(loss)/d(image) `grad_img`: the gradient of every argument of `c`, at its position
    in RenderFunction.apply's arguments (RenderFunction.backward's return value).  `screen_grad`, an [height, width, 2] tensor, also
    receives d(image)/d(screen position of each pixel)."""
    rb = c.backend
    grad_img = grad_img.contiguous()
    assert torch.isfinite(grad_img).all()
    g = RenderFunction.gradient_buffers(c)
    rb.render(c.scene, RenderFunction.backward_options(c), rb.float_ptr(0), _ptr(rb, grad_img), g.d_scene, _ptr(rb, screen_grad), rb.float_ptr(0))
    return RenderFunction.gradient_outputs(c, g)


def _seeds(seed):
    """The (forward, backward) seeds of RenderFunction.apply's `seed`."""
    assert isinstance(seed, (tuple, int))
    if isinstance(seed, tuple):
        return seed
    return seed, seed if _use_correlated_random_number else seed + 1000003


def _serialize_texture(tex, args, device):
    if tex is None:
        args.append(0)
        return
    args.append(len(tex.mipmap))
    for m in tex.mipmap:
        assert torch.isfinite(m).all()
        assert m.is_contiguous()
        args.append(m.to(device))
    assert torch.isfinite(tex.uv_scale).all()
    args.append(tex.uv_scale.to(device))


class RenderFunction(torch.autograd.Function):
    """torch.autograd.Function around `redner.render` (pyredner/render_pytorch.py:63-1177).

    `RenderFunction.apply(seed, *args)` with `args = RenderFunction.serialize_scene(...)`.  The module implementing the
    `redner` surface is the LAST serialized argument, so the same host code can drive the product and the oracle."""

    @staticmethod
    def serialize_scene(scene: Scene, num_samples: Union[int, Tuple[int, int]], max_bounces: int, channels=None, sampler_type=None,
                        use_primary_edge_sampling: bool = True, use_secondary_edge_sampling: bool = True, sample_pixel_center: bool = False,
                        device: Optional[torch.device] = None, backend=None, pixel_filter: Optional[PixelFilter] = None):
        backend = backend or default_backend()
        if channels is None:
            channels = [backend.channels.radiance]
        if sampler_type is None:
            sampler_type = backend.SamplerType.independent
        if device is None:
            device = get_device()
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda:%d" % torch.cuda.current_device())
        cam = scene.camera
        for light_id, light in enumerate(scene.area_lights):
            scene.shapes[light.shape_id].light_id = light_id
        if max_bounces == 0:
            use_secondary_edge_sampling = False
        vis = False  # does any parameter need discontinuity (edge) sampling? (render_pytorch.py:144-160)
        for t in (cam.position, cam.look_at, cam.up, cam.cam_to_world, cam.world_to_cam, cam.intrinsic_mat, cam.intrinsic_mat_inv, cam.distortion_params):
            if t is not None:
                assert torch.isfinite(t).all()
                vis = vis or t.requires_grad
        args = [len(scene.shapes), len(scene.materials), len(scene.area_lights)]
        args += [cam.position.cpu() if cam.position is not None else None, cam.look_at.cpu() if cam.look_at is not None else None,
                 cam.up.cpu() if cam.up is not None else None]
        args += [cam.cam_to_world.cpu().contiguous() if cam.cam_to_world is not None else None,
                 cam.world_to_cam.cpu().contiguous() if cam.world_to_cam is not None else None]
        args += [cam.intrinsic_mat_inv.cpu().contiguous(), cam.intrinsic_mat.cpu().contiguous()]
        args.append(cam.distortion_params.cpu().contiguous() if cam.distortion_params is not None else None)
        args += [cam.clip_near, cam.resolution]
        vp = cam.viewport if cam.viewport is not None else (0, 0, cam.resolution[0], cam.resolution[1])
        vp = (max(vp[0], 0), max(vp[1], 0), min(vp[2], cam.resolution[0]), min(vp[3], cam.resolution[1]))
        args += [vp, cam.camera_type]
        for s in scene.shapes:
            assert torch.isfinite(s.vertices).all()
            vis = vis or s.vertices.requires_grad
            args += [s.vertices.to(device), s.indices.to(device)]
            for t in (s.uvs, s.normals, s.uv_indices, s.normal_indices, s.colors):
                if t is not None and t.is_floating_point():
                    assert torch.isfinite(t).all()
                args.append(t.to(device) if t is not None else None)
            args += [s.material_id, s.light_id]
        for m in scene.materials:
            for tex in (m.diffuse_reflectance, m.specular_reflectance, m.roughness, m.generic_texture, m.normal_map):
                _serialize_texture(tex, args, device)
            args += [m.compute_specular_lighting, m.two_sided, m.use_vertex_color]
        for light in scene.area_lights:
            args += [light.shape_id, light.intensity.cpu(), light.two_sided, light.directly_visible]
        if scene.envmap is not None:  # pyredner/render_pytorch.py:240-253
            e = scene.envmap
            for t in (e.env_to_world, e.world_to_env, e.sample_cdf_ys, e.sample_cdf_xs):
                assert torch.isfinite(t).all()
            _serialize_texture(e.values, args, device)
            args += [e.env_to_world.cpu().contiguous(), e.world_to_env.cpu().contiguous(), e.sample_cdf_ys.to(device), e.sample_cdf_xs.to(device),
                     e.pdf_norm, e.directly_visible]
        else:
            args.append(None)
        args += [num_samples, max_bounces, channels, sampler_type]
        args += [use_primary_edge_sampling and vis, use_secondary_edge_sampling and vis]
        args += [sample_pixel_center, pixel_filter.native() if pixel_filter is not None else None, device, backend]
        return args

    @staticmethod
    def read_args(args):
        """serialize_scene's argument list, read in one pass.  Besides serialize_scene, this is the only code that knows the list's layout.

        Returns a namespace of `camera_args`, `shape_args`, `mat_args`, `light_args` (lists), `env_args` (None without an environment map)
        and `option_args`: the entries serialize_scene wrote for each, as the named tuples above.  A material's `textures` are five
        _TextureArgs or None (diffuse, specular, roughness, generic, normal map); the environment map's `values` is one.  `pos` holds the
        same structure with the position in `args` of each entry in place of the entry.  `args` is the list itself."""
        k = 3  # (after the numbers of shapes, materials and lights)

        def entries(n):
            nonlocal k
            k += n
            return args[k - n:k], range(k - n, k)

        def take(cls):
            values, positions = entries(len(cls._fields))
            return cls._make(values), cls._make(positions)

        def texture():
            n, _ = entries(1)  # number of mip levels: 0 for a material without this texture, None for a scene without an environment map
            if not n[0]:
                return None, None
            (mips, mip_pos), (uv, uv_pos) = entries(n[0]), entries(1)
            return _TextureArgs(list(mips), uv[0]), _TextureArgs(list(mip_pos), uv_pos[0])

        def material():
            textures = [texture() for _ in range(5)]
            values, positions = entries(3)
            return _MaterialArgs([t for t, _ in textures], *values), _MaterialArgs([p for _, p in textures], *positions)

        def each(n, read):
            pairs = [read() for _ in range(n)]
            return [v for v, _ in pairs], [p for _, p in pairs]

        a = SimpleNamespace(args=args, pos=SimpleNamespace())
        a.camera_args, a.pos.camera_args = take(_CameraArgs)
        a.shape_args, a.pos.shape_args = each(args[0], lambda: take(_ShapeArgs))
        a.mat_args, a.pos.mat_args = each(args[1], material)
        a.light_args, a.pos.light_args = each(args[2], lambda: take(_LightArgs))
        a.env_args = a.pos.env_args = None
        values, positions = texture()
        if values is not None:
            rest, rest_pos = entries(len(_EnvmapArgs._fields) - 1)
            a.env_args, a.pos.env_args = _EnvmapArgs(values, *rest), _EnvmapArgs(positions, *rest_pos)
        a.option_args, a.pos.option_args = take(_OptionArgs)
        assert k == len(args), "serialize_scene's list has %d entries, its layout %d" % (len(args), k)
        return a

    @staticmethod
    def _unpack(seed, args, scene=None, geometry_changed=None):
        """`scene`: an existing native scene of the SAME geometry / materials / lights to re-target at this argument list's camera
        (rb_scene_set_camera) instead of building a new one -- the batch path.  With `geometry_changed` (True / False) the scene only
        needs the same structure and is re-targeted at everything in the argument list (Scene.update) -- the SceneRenderer path.
        Returns read_args(args) with the native objects built from it added."""
        c = RenderFunction.read_args(args)
        cam, opt = c.camera_args, c.option_args
        rb, device, vp = opt.backend, opt.device, cam.viewport
        fp, ip = (lambda t: _ptr(rb, t, "float")), (lambda t: _ptr(rb, t, "int"))
        look_at = cam.cam_to_world is None
        camera = rb.Camera(cam.resolution[1], cam.resolution[0], fp(cam.position if look_at else None), fp(cam.look_at if look_at else None),
                           fp(cam.up if look_at else None), fp(cam.cam_to_world), fp(cam.world_to_cam), fp(cam.intrinsic_mat_inv),
                           fp(cam.intrinsic_mat), fp(cam.distortion_params), cam.clip_near, rb.CameraType(int(cam.camera_type)),
                           rb.Vector2i(vp[1], vp[0]), rb.Vector2i(vp[3], vp[2]))
        shapes = []
        for s in c.shape_args:
            assert s.vertices.is_contiguous() and s.indices.is_contiguous()
            shapes.append(rb.Shape(fp(s.vertices), ip(s.indices), fp(s.uvs), fp(s.normals), ip(s.uv_indices), ip(s.normal_indices), fp(s.colors),
                                   int(s.vertices.shape[0]), int(s.uvs.shape[0]) if s.uvs is not None else 0,
                                   int(s.normals.shape[0]) if s.normals is not None else 0, int(s.indices.shape[0]), s.material_id, s.light_id))
        materials = []
        for m in c.mat_args:
            textures = [_native_texture(rb, cls, nch, t) for (cls, nch), t in zip(_material_textures(rb), m.textures)]
            materials.append(rb.Material(*textures, m.compute_specular_lighting, m.two_sided, m.use_vertex_color))
        lights = [rb.AreaLight(l.shape_id, fp(l.intensity), l.two_sided, l.directly_visible) for l in c.light_args]
        envmap = None
        if c.env_args is not None:
            e = c.env_args
            env_tex = _native_texture(rb, rb.Texture3, 3, e.values)
            envmap = rb.EnvironmentMap(env_tex, fp(e.env_to_world), fp(e.world_to_env), fp(e.sample_cdf_ys), fp(e.sample_cdf_xs), e.pdf_norm,
                                       e.directly_visible)
        c.envmap, c.pixel_filter = envmap, opt.pixel_filter
        if scene is None:
            # (the keyword only when a filter is set: a backend without pixel filters renders the 1-pixel box)
            c.scene = rb.Scene(camera, shapes, materials, lights, envmap, device.type == "cuda", device.index if device.index is not None else -1,
                               opt.use_primary_edge_sampling, opt.use_secondary_edge_sampling,
                               **({} if opt.pixel_filter is None else {"pixel_filter": opt.pixel_filter}))
        elif geometry_changed is not None:
            scene.update(camera, shapes, materials, lights, envmap, geometry_changed=geometry_changed, pixel_filter=opt.pixel_filter)
            c.scene = scene
        else:
            scene.set_camera(camera)
            c.scene = scene
        ns = opt.num_samples if isinstance(opt.num_samples, (tuple, list)) else (opt.num_samples, opt.num_samples)
        channels = [rb.channels(int(ch)) for ch in opt.channels]
        c.options = rb.RenderOptions(seed[0], ns[0], opt.max_bounces, channels, rb.SamplerType(int(opt.sampler_type)), opt.sample_pixel_center)
        c.camera, c.shapes, c.materials, c.lights = camera, shapes, materials, lights
        c.num_samples, c.channels, c.viewport, c.device, c.backend, c.seed = ns, channels, vp, device, rb, seed
        return c

    @staticmethod
    def forward(ctx, seed, *args):
        c = RenderFunction._unpack(_seeds(seed), args)
        ctx.c = c
        ctx.args = args  # keeps the tensors alive (the native side only holds raw pointers)
        return _render(c)

    @staticmethod
    def gradient_buffers(c, zeros=None):
        """Zeroed gradient buffers for every differentiable input of `c` (the unpacked call, or read_args' result alone), and the DScene
        that points at them (`.d_scene`).  `zeros(*shape)` allocates one buffer (default: torch.zeros on the render device).

        The buffers, in the order they are allocated: `camera` (the eight of rb.DCamera, None where there is none), `shapes` ((vertices,
        uvs, normals, colors) per shape), `materials` (per material its five textures, each None or (mips, uv_scale)), `intensities` (per
        light) and `envmap` (None or (mips, uv_scale, world_to_env)).  `grads` maps the position in serialize_scene's list of each argument
        that has a buffer to that buffer."""
        rb, dev, p = c.option_args.backend, c.option_args.device, c.pos
        z = zeros or (lambda *shape: torch.zeros(*shape, device=dev))
        fp = lambda t: _ptr(rb, t, "float")  # noqa: E731
        g = SimpleNamespace(grads={})

        def buf(pos, *shape):
            g.grads[pos] = z(*shape)
            return g.grads[pos]

        def like(t, pos):  # (None for an absent optional tensor)
            return buf(pos, *t.shape) if t is not None else None

        def texture(t, pos):
            return ([buf(q, *m.shape) for q, m in zip(pos.mips, t.mips)], buf(pos.uv_scale, 2)) if t is not None else None

        cam, cp = c.camera_args, p.camera_args
        look_at = cam.cam_to_world is None  # (which pose the native camera uses: _unpack)
        g.camera = (buf(cp.position, 3) if look_at else None, buf(cp.look_at, 3) if look_at else None, buf(cp.up, 3) if look_at else None,
                    None if look_at else buf(cp.cam_to_world, 4, 4), None if look_at else buf(cp.world_to_cam, 4, 4),
                    buf(cp.intrinsic_mat_inv, 3, 3), buf(cp.intrinsic_mat, 3, 3),
                    buf(cp.distortion_params, 8) if cam.distortion_params is not None else None)
        g.shapes = [(like(s.vertices, q.vertices), like(s.uvs, q.uvs), like(s.normals, q.normals), like(s.colors, q.colors))
                    for s, q in zip(c.shape_args, p.shape_args)]
        g.materials = [[texture(t, q) for t, q in zip(m.textures, mp.textures)] for m, mp in zip(c.mat_args, p.mat_args)]
        g.intensities = [buf(q.intensity, 3) for q in p.light_args]
        g.envmap = d_envmap = None
        if c.env_args is not None:  # pyredner/render_pytorch.py:948-968
            values = c.env_args.values
            g.envmap = texture(values, p.env_args.values) + (buf(p.env_args.world_to_env, 4, 4),)
            d_envmap = rb.DEnvironmentMap(_native_texture(rb, rb.Texture3, 3, values, g.envmap[:2]), fp(g.envmap[2]))
        d_materials = [rb.DMaterial(*[_native_texture(rb, cls, nch, t, b) for (cls, nch), t, b in zip(_material_textures(rb), m.textures, bufs)])
                       for m, bufs in zip(c.mat_args, g.materials)]
        g.d_scene = rb.DScene(rb.DCamera(*[fp(t) for t in g.camera]), [rb.DShape(*[fp(t) for t in b]) for b in g.shapes], d_materials,
                              [rb.DAreaLight(fp(t)) for t in g.intensities], d_envmap, dev.type == "cuda", dev.index if dev.index is not None else -1)
        return g

    @staticmethod
    def backward_options(c):
        """The options of the backward pass of `c`: its second seed and sample count."""
        c.options.seed = c.seed[1]
        c.options.num_samples = c.num_samples[1]
        return c.options

    @staticmethod
    def gradient_outputs(c, g):
        """backward's return value: None for the seed, then the buffers of gradient_buffers(c) at the positions of serialize_scene's
        arguments, each on the device of its argument (the host for the camera, the light intensities and world_to_env)."""
        out = [None] * (1 + len(c.args))
        for pos, t in g.grads.items():
            out[1 + pos] = t.to(c.args[pos].device)
        return tuple(out)

    @staticmethod
    def backward(ctx, grad_img):
        return _backward(ctx.c, grad_img)


class BatchRenderFunction(torch.autograd.Function):
    """A batch of views of ONE scene (BASELINE config 5; the pattern of the reference's tests/test_batch.py:10-33, whose Python loop
    builds a full Scene per view).  `args` = the serialize_scene lists of the views, concatenated; the views must share geometry,
    materials and lights (the same tensors) and may differ in camera and options.  The native scene -- BVH, light tables, edge list --
    is built once; per view only the camera-dependent tables are rebuilt, on the device.  Returns [views, height, width, channels]."""

    @staticmethod
    def forward(ctx, seeds, num_views, *args):
        assert num_views >= 1 and len(args) % num_views == 0
        n = len(args) // num_views
        seeds = list(seeds) if isinstance(seeds, (list, tuple)) else [seeds + k for k in range(num_views)]
        views, imgs, scene = [], [], None
        for k in range(num_views):
            sd = seeds[k] if isinstance(seeds[k], tuple) else (seeds[k], seeds[k] + 1000003)
            c = RenderFunction._unpack(sd, args[k * n:(k + 1) * n], scene=scene)
            scene = c.scene
            views.append(c)
            imgs.append(_render(c))
        ctx.views, ctx.args = views, args
        return torch.stack(imgs)

    @staticmethod
    def backward(ctx, grad_imgs):
        out = [None, None]
        for k, c in enumerate(ctx.views):
            c.scene.set_camera(c.camera)
            out += _backward(c, grad_imgs[k])[1:]
        return tuple(out)


class SceneRenderer:
    """Renders one scene over and over -- the steps of an optimisation loop -- through ONE native scene that is updated in place
    (Scene.update / rb_scene_update) instead of built anew for every call the way RenderFunction does.

        render = SceneRenderer(num_samples, max_bounces, **serialize_scene options)
        img = render(scene, seed)   # RenderFunction.apply(seed, *serialize_scene(scene, ...)), with autograd

    The first call builds the native scene.  A later call whose scene has the same structure (shapes, vertex / triangle counts,
    material and light ids, optional buffers, lights, environment map, and the edge-sampling flags, which follow `requires_grad`)
    updates it: the BVH, light areas and edge list are rebuilt only when a vertex tensor was replaced or written to in place (its
    `_version`); a material, light intensity or camera change refreshes the light PMF and the camera tables alone.  An index tensor that
    was replaced or written to is compared with a copy of the one the scene was built from; a change there, or any other change of
    structure, builds a new native scene.  Images are those of RenderFunction; the backward pass renders against the state its forward
    pass saw, even if the scene has been updated since."""

    def __init__(self, num_samples, max_bounces: int, **options):
        self.num_samples, self.max_bounces, self.options = num_samples, max_bounces, options
        self._scene = None       # the native scene
        self._key = None         # structure of its last descriptor
        self._vertices = None    # [(vertex tensor, its _version)] of the last descriptor
        self._indices = None     # [(index tensor, its _version, copy)] of the build

    @staticmethod
    def _structure(a):
        """The parts of a read_args result that rb_scene_update requires to be unchanged, except the contents of index buffers."""
        def shape(t):
            return tuple(t.shape) if t is not None else None

        def texture(t):
            return None if t is None else tuple(shape(m) for m in t.mips) + (shape(t.uv_scale),)
        shapes = tuple((shape(s.vertices), shape(s.indices), shape(s.uvs), shape(s.normals), s.uv_indices is not None, s.normal_indices is not None,
                        s.colors is not None, int(s.material_id), int(s.light_id)) for s in a.shape_args)
        mats = tuple((tuple(texture(t) for t in m.textures), m.compute_specular_lighting, m.two_sided, m.use_vertex_color) for m in a.mat_args)
        lights = tuple(int(l.shape_id) for l in a.light_args)
        env = texture(a.env_args.values) if a.env_args is not None else None
        o = a.option_args
        return shapes, mats, lights, env, (bool(o.use_primary_edge_sampling), bool(o.use_secondary_edge_sampling), str(o.device))

    def _target(self, args):
        """(geometry_changed, state): geometry_changed is None to build a new native scene for `args`, else the flag for an update of the
        current one; `state` is what _commit records once the native call has succeeded."""
        a = RenderFunction.read_args(args)
        key = self._structure(a)
        verts = [s.vertices for s in a.shape_args]
        inds = [s.indices for s in a.shape_args]
        fresh = self._scene is None or key != self._key
        if not fresh:
            for t, (t0, ver0, copy) in zip(inds, self._indices):
                if (t is not t0 or t._version != ver0) and not torch.equal(t, copy):
                    fresh = True
                    break
        if fresh:
            indices = [(t, t._version, t.clone()) for t in inds]
            geometry = None
        else:
            indices = [(t, t._version, copy) for t, (_, _, copy) in zip(inds, self._indices)]
            geometry = any(t is not t0 or t._version != ver0 for t, (t0, ver0) in zip(verts, self._vertices))
        return geometry, (key, [(t, t._version) for t in verts], indices)

    def _commit(self, scene, state):
        self._scene = scene
        self._key, self._vertices, self._indices = state

    def _forget(self):
        """After a failed build or update: the next call builds a new native scene."""
        self._scene = self._key = self._vertices = self._indices = None

    def __call__(self, scene: Scene, seed):
        args = RenderFunction.serialize_scene(scene, self.num_samples, self.max_bounces, **self.options)
        return _SceneRenderFunction.apply(seed, self, *args)


class _SceneRenderFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seed, renderer, *args):
        seed = _seeds(seed)
        geometry, state = renderer._target(args)
        try:
            c = RenderFunction._unpack(seed, args, scene=renderer._scene if geometry is not None else None, geometry_changed=geometry)
        except Exception:
            renderer._forget()
            raise
        renderer._commit(c.scene, state)
        c.scene._generation = getattr(c.scene, "_generation", 0) + 1
        ctx.generation = c.scene._generation
        ctx.c = c
        ctx.args = args  # keeps the tensors alive (the native side only holds raw pointers)
        return _render(c)

    @staticmethod
    def backward(ctx, grad_img):
        c = ctx.c
        if c.scene._generation != ctx.generation:  # updated since this forward pass: back to the state it rendered
            c.scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=True, pixel_filter=c.pixel_filter)
            c.scene._generation += 1
            ctx.generation = c.scene._generation
        return (None,) + _backward(c, grad_img)


def render_batch(scenes, num_samples, max_bounces: int, seeds, **kw) -> torch.Tensor:
    """Views of one scene: `scenes` are Scene objects that share shapes / materials / lights and differ in their camera."""
    args = []
    for sc in scenes:
        args += RenderFunction.serialize_scene(sc, num_samples, max_bounces, **kw)
    return BatchRenderFunction.apply(seeds, len(scenes), *args)


def visualize_screen_gradient(grad_img: Optional[torch.Tensor], seed: int, scene: Scene, num_samples, max_bounces: int, channels=None, sampler_type=None,
                              use_primary_edge_sampling: bool = True, use_secondary_edge_sampling: bool = True, sample_pixel_center: bool = False,
                              device=None, backend=None) -> torch.Tensor:
    """RenderFunction.visualize_screen_gradient (pyredner/render_pytorch.py:982-1048): the derivative of the (weighted) image
    with respect to the screen position of every pixel, [height, width, 2] -- the backward pass with a screen-gradient
    buffer attached (src/primary_intersection.cpp:104-114, src/edge.cpp:765-773).  `grad_img` None means all ones."""
    args = RenderFunction.serialize_scene(scene, num_samples, max_bounces, channels=channels, sampler_type=sampler_type,
                                          use_primary_edge_sampling=use_primary_edge_sampling, use_secondary_edge_sampling=use_secondary_edge_sampling,
                                          sample_pixel_center=sample_pixel_center, device=device, backend=backend)
    c = RenderFunction._unpack((seed, seed), args)
    c.num_samples = (c.num_samples[0], c.num_samples[0])  # (the reference renders this pass with the forward sample count)
    h, w, nch = _image_shape(c)
    if grad_img is None:
        grad_img = torch.ones(h, w, nch, device=c.device)
    assert tuple(grad_img.shape) == (h, w, nch)
    screen_grad = torch.zeros(h, w, 2, device=c.device)
    _backward(c, grad_img.to(c.device), screen_grad)
    return screen_grad


RenderFunction.visualize_screen_gradient = staticmethod(visualize_screen_gradient)  # (where pyredner keeps it)


def render_pathtracing(scene: Scene, num_samples=(4, 4), max_bounces: int = 1, seed: int = 0, sampler_type=None, device=None, backend=None,
                       use_primary_edge_sampling=True, use_secondary_edge_sampling=True, pixel_filter: Optional[PixelFilter] = None):
    """pyredner.render_pathtracing (pyredner/render_utils.py:505-573) for a single scene."""
    args = RenderFunction.serialize_scene(scene, num_samples, max_bounces, sampler_type=sampler_type, device=device, backend=backend,
                                          use_primary_edge_sampling=use_primary_edge_sampling,
                                          use_secondary_edge_sampling=use_secondary_edge_sampling, pixel_filter=pixel_filter)
    return RenderFunction.apply(seed, *args)
