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


class Scene:
    def __init__(self, camera: Camera, shapes: List[Shape], materials: List[Material], area_lights: List[AreaLight], envmap=None):
        self.camera, self.shapes, self.materials, self.area_lights, self.envmap = camera, shapes, materials, area_lights, envmap


class _Ctx:
    pass


def _ptr(backend, t, kind="float"):
    ctor = backend.float_ptr if kind == "float" else backend.int_ptr
    return ctor(t.data_ptr() if t is not None else 0)


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
                        device: Optional[torch.device] = None, backend=None):
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
        args += [sample_pixel_center, device, backend]
        return args

    @staticmethod
    def _unpack(seed, args, scene=None, geometry_changed=None):
        """`scene`: an existing native scene of the SAME geometry / materials / lights to re-target at this argument list's camera
        (rb_scene_set_camera) instead of building a new one -- the batch path.  With `geometry_changed` (True / False) the scene only
        needs the same structure and is re-targeted at everything in the argument list (Scene.update) -- the SceneRenderer path."""
        it = iter(args)
        nxt = lambda: next(it)  # noqa: E731
        c = _Ctx()
        num_shapes, num_materials, num_lights = nxt(), nxt(), nxt()
        cam_pos, cam_look, cam_up, c2w, w2c, intr_inv, intr, dist = nxt(), nxt(), nxt(), nxt(), nxt(), nxt(), nxt(), nxt()
        clip_near, resolution, viewport, camera_type = nxt(), nxt(), nxt(), nxt()
        shape_args, mat_args, light_args = [], [], []
        for _ in range(num_shapes):
            shape_args.append([nxt() for _ in range(9)])
        for _ in range(num_materials):
            texs = []
            for _ in range(5):
                n = nxt()
                if n == 0:
                    texs.append(None)
                else:
                    mips = [nxt() for _ in range(n)]
                    texs.append((mips, nxt()))
            mat_args.append((texs, nxt(), nxt(), nxt()))
        for _ in range(num_lights):
            light_args.append([nxt() for _ in range(4)])
        env_args = None
        n_env = nxt()
        if n_env is not None:
            env_mips = [nxt() for _ in range(n_env)]
            env_args = (env_mips, nxt(), nxt(), nxt(), nxt(), nxt(), nxt(), nxt())  # uv_scale, e2w, w2e, cdf_ys, cdf_xs, pdf_norm, visible
        num_samples, max_bounces, channels, sampler_type = nxt(), nxt(), nxt(), nxt()
        use_prim, use_sec, pixel_center, device, backend = nxt(), nxt(), nxt(), nxt(), nxt()
        rb = backend
        fp, ip = (lambda t: _ptr(rb, t, "float")), (lambda t: _ptr(rb, t, "int"))
        camera = rb.Camera(resolution[1], resolution[0], fp(cam_pos if c2w is None else None), fp(cam_look if c2w is None else None),
                           fp(cam_up if c2w is None else None), fp(c2w), fp(w2c), fp(intr_inv), fp(intr), fp(dist), clip_near,
                           rb.CameraType(int(camera_type)),
                           rb.Vector2i(viewport[1], viewport[0]), rb.Vector2i(viewport[3], viewport[2]))
        shapes = []
        for v, i, uv, n, uvi, ni, col, mid, lid in shape_args:
            assert v.is_contiguous() and i.is_contiguous()
            shapes.append(rb.Shape(fp(v), ip(i), fp(uv), fp(n), ip(uvi), ip(ni), fp(col), int(v.shape[0]), int(uv.shape[0]) if uv is not None else 0,
                                   int(n.shape[0]) if n is not None else 0, int(i.shape[0]), mid, lid))

        def make_tex(cls, t, nch_default):
            if t is None:
                return cls([], [], [], nch_default, rb.float_ptr(0))
            mips, uv_scale = t
            if mips[0].dim() == 3:
                return cls([fp(m) for m in mips], [int(m.shape[1]) for m in mips], [int(m.shape[0]) for m in mips], int(mips[0].shape[2]), fp(uv_scale))
            return cls([fp(mips[0])], [0], [0], int(mips[0].shape[0]), fp(uv_scale))

        materials = []
        for texs, spec, two_sided, vcol in mat_args:
            materials.append(rb.Material(make_tex(rb.Texture3, texs[0], 3), make_tex(rb.Texture3, texs[1], 3), make_tex(rb.Texture1, texs[2], 1),
                                         make_tex(rb.TextureN, texs[3], 0), make_tex(rb.Texture3, texs[4], 3), spec, two_sided, vcol))
        lights = [rb.AreaLight(sid, fp(inten), ts, dv) for sid, inten, ts, dv in light_args]
        use_gpu = device.type == "cuda"
        gpu_index = device.index if device.index is not None else -1
        envmap = None
        if env_args is not None:
            mips, uv_scale, e2w, w2e, cdf_ys, cdf_xs, pdf_norm, visible = env_args
            env_tex = rb.Texture3([fp(m) for m in mips], [int(m.shape[1]) for m in mips], [int(m.shape[0]) for m in mips], 3, fp(uv_scale))
            envmap = rb.EnvironmentMap(env_tex, fp(e2w), fp(w2e), fp(cdf_ys), fp(cdf_xs), pdf_norm, visible)
        c.env_args, c.envmap = env_args, envmap
        if scene is None:
            c.scene = rb.Scene(camera, shapes, materials, lights, envmap, use_gpu, gpu_index, use_prim, use_sec)
        elif geometry_changed is not None:
            scene.update(camera, shapes, materials, lights, envmap, geometry_changed=geometry_changed)
            c.scene = scene
        else:
            scene.set_camera(camera)
            c.scene = scene
        ns = num_samples if isinstance(num_samples, (tuple, list)) else (num_samples, num_samples)
        channels = [rb.channels(int(ch)) for ch in channels]
        c.options = rb.RenderOptions(seed[0], ns[0], max_bounces, channels, rb.SamplerType(int(sampler_type)), pixel_center)
        c.camera, c.shapes, c.materials, c.lights = camera, shapes, materials, lights
        c.shape_args, c.mat_args, c.light_args = shape_args, mat_args, light_args
        c.num_samples, c.channels, c.viewport, c.device, c.backend, c.seed = ns, channels, viewport, device, rb, seed
        c.use_look_at = c2w is None
        c.has_distortion = dist is not None
        return c

    @staticmethod
    def forward(ctx, seed, *args):
        assert isinstance(seed, (tuple, int))
        if not isinstance(seed, tuple):
            seed = (seed, seed if _use_correlated_random_number else seed + 1000003)
        c = RenderFunction._unpack(seed, args)
        rb = c.backend
        nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
        h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
        img = torch.zeros(h, w, nch, device=c.device)
        rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
        ctx.c = c
        ctx.args = args  # keeps the tensors alive (the native side only holds raw pointers)
        return img

    @staticmethod
    def gradient_buffers(c, zeros=None):
        """Zeroed gradient buffers for every differentiable input of the unpacked call `c`, and the DScene that points at them (`.d_scene`).
        `zeros(*shape)` allocates one buffer (default: torch.zeros on c.device)."""
        rb, dev = c.backend, c.device
        z = zeros or (lambda *shape: torch.zeros(*shape, device=dev))
        fp = lambda t: _ptr(rb, t, "float")  # noqa: E731
        g = _Ctx()
        if c.use_look_at:
            d_pos, d_look, d_up, d_c2w, d_w2c = z(3), z(3), z(3), None, None
        else:
            d_pos, d_look, d_up, d_c2w, d_w2c = None, None, None, z(4, 4), z(4, 4)
        d_intr_inv, d_intr = z(3, 3), z(3, 3)
        d_dist = z(8) if c.has_distortion else None
        g.camera = (d_pos, d_look, d_up, d_c2w, d_w2c, d_intr_inv, d_intr, d_dist)
        d_camera = rb.DCamera(*[fp(t) for t in g.camera])
        g.shapes, d_shapes = [], []
        for v, i, uv, n, uvi, ni, col, mid, lid in c.shape_args:
            bufs = (z(*v.shape), z(*uv.shape) if uv is not None else None, z(*n.shape) if n is not None else None, z(*col.shape) if col is not None else None)
            g.shapes.append(bufs)
            d_shapes.append(rb.DShape(fp(bufs[0]), fp(bufs[1]), fp(bufs[2]), fp(bufs[3])))

        def make_dtex(cls, t, nch_default):
            if t is None:
                return None, cls([], [], [], nch_default, rb.float_ptr(0))
            mips, uv_scale = t
            d_mips = [z(*m.shape) for m in mips]
            d_uv = z(2)
            if mips[0].dim() == 3:
                tex = cls([fp(m) for m in d_mips], [int(m.shape[1]) for m in mips], [int(m.shape[0]) for m in mips], int(mips[0].shape[2]), fp(d_uv))
            else:
                tex = cls([fp(d_mips[0])], [0], [0], int(mips[0].shape[0]), fp(d_uv))
            return (d_mips, d_uv), tex

        g.materials, d_materials = [], []
        for texs, spec, two_sided, vcol in c.mat_args:
            classes = (rb.Texture3, rb.Texture3, rb.Texture1, rb.TextureN, rb.Texture3)
            made = [make_dtex(cls, t, nd) for cls, t, nd in zip(classes, texs, (3, 3, 1, 0, 3))]
            g.materials.append([m[0] for m in made])
            d_materials.append(rb.DMaterial(*[m[1] for m in made]))
        g.intensities = [z(3) for _ in c.light_args]
        d_lights = [rb.DAreaLight(fp(t)) for t in g.intensities]
        d_envmap, g.envmap = None, None
        if c.env_args is not None:  # pyredner/render_pytorch.py:948-968
            mips = c.env_args[0]
            g.envmap = ([z(*m.shape) for m in mips], z(2), z(4, 4))
            d_env_tex = rb.Texture3([fp(m) for m in g.envmap[0]], [int(m.shape[1]) for m in mips], [int(m.shape[0]) for m in mips], 3, fp(g.envmap[1]))
            d_envmap = rb.DEnvironmentMap(d_env_tex, fp(g.envmap[2]))
        g.d_scene = rb.DScene(d_camera, d_shapes, d_materials, d_lights, d_envmap, dev.type == "cuda", dev.index if dev.index is not None else -1)
        return g

    @staticmethod
    def backward_options(c):
        """The options of the backward pass of `c`: its second seed and sample count."""
        c.options.seed = c.seed[1]
        c.options.num_samples = c.num_samples[1]
        return c.options

    @staticmethod
    def gradient_outputs(c, g):
        """backward's return value: the buffers of gradient_buffers(c) at the positions of serialize_scene's arguments."""
        out = [None]  # seed
        out += [None, None, None]  # counts
        cpu = lambda t: t.cpu() if t is not None else None  # noqa: E731
        out += [cpu(t) for t in g.camera]
        out += [None, None, None, None]  # clip_near, resolution, viewport, camera_type
        for bufs in g.shapes:
            out += [bufs[0], None, bufs[1], bufs[2], None, None, bufs[3], None, None]
        for mb, (texs, _, _, _) in zip(g.materials, c.mat_args):
            for b, t in zip(mb, texs):
                out.append(None)  # number of levels
                if t is not None:
                    out += list(b[0])
                    out.append(b[1])
            out += [None, None, None]
        for d_i in g.intensities:
            out += [None, d_i.cpu(), None, None]
        if g.envmap is not None:  # pyredner/render_pytorch.py:1154-1164
            out.append(None)  # number of levels
            out += list(g.envmap[0])
            out += [g.envmap[1], None, g.envmap[2].cpu(), None, None, None, None]  # uv_scale, env_to_world, world_to_env, cdfs, pdf_norm, visible
        else:
            out.append(None)  # envmap
        out += [None] * 9  # num_samples .. backend
        return tuple(out)

    @staticmethod
    def backward(ctx, grad_img):
        c = ctx.c
        rb = c.backend
        if not grad_img.is_contiguous():
            grad_img = grad_img.contiguous()
        assert torch.isfinite(grad_img).all()
        g = RenderFunction.gradient_buffers(c)
        screen_grad = getattr(c, "screen_gradient", None)  # (only set by visualize_screen_gradient)
        rb.render(c.scene, RenderFunction.backward_options(c), rb.float_ptr(0), _ptr(rb, grad_img), g.d_scene, _ptr(rb, screen_grad), rb.float_ptr(0))
        return RenderFunction.gradient_outputs(c, g)


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
            rb = c.backend
            nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
            h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
            img = torch.zeros(h, w, nch, device=c.device)
            rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
            views.append(c)
            imgs.append(img)
        ctx.views, ctx.args, ctx.n = views, args, n
        return torch.stack(imgs)

    @staticmethod
    def backward(ctx, grad_imgs):
        out = [None, None]
        for k, c in enumerate(ctx.views):
            c.scene.set_camera(c.camera)
            one = _Ctx()
            one.c, one.args = c, ctx.args[k * ctx.n:(k + 1) * ctx.n]
            out += list(RenderFunction.backward(one, grad_imgs[k]))[1:]
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
    def _structure(args):
        """The parts of a serialize_scene list that rb_scene_update requires to be unchanged, except the contents of index buffers."""
        it = iter(args)
        nxt = lambda: next(it)  # noqa: E731
        num_shapes, num_materials, num_lights = nxt(), nxt(), nxt()
        for _ in range(12):
            nxt()
        shapes, mats, lights = [], [], []
        for _ in range(num_shapes):
            v, i, uv, n, uvi, ni, col, mid, lid = [nxt() for _ in range(9)]
            shapes.append((tuple(v.shape), tuple(i.shape), tuple(uv.shape) if uv is not None else None, tuple(n.shape) if n is not None else None,
                           uvi is not None, ni is not None, col is not None, int(mid), int(lid)))
        for _ in range(num_materials):
            texs = []
            for _ in range(5):
                k = nxt()
                texs.append(None if k == 0 else tuple(tuple(nxt().shape) for _ in range(k + 1)))  # (mip levels, then uv_scale)
            mats.append((tuple(texs), nxt(), nxt(), nxt()))
        for _ in range(num_lights):
            lights.append(int(nxt()))
            nxt(), nxt(), nxt()
        k = nxt()
        env = None if k is None else tuple(tuple(nxt().shape) for _ in range(k + 1))  # (mip levels, then uv_scale)
        if k is not None:
            for _ in range(6):  # matrices, sampling tables, pdf_norm, directly_visible
                nxt()
        rest = [nxt() for _ in range(9)]
        flags = (bool(rest[4]), bool(rest[5]), str(rest[7]))  # edge-sampling flags, device
        return tuple(shapes), tuple(mats), tuple(lights), env, flags

    def _target(self, args):
        """(geometry_changed, state): geometry_changed is None to build a new native scene for `args`, else the flag for an update of the
        current one; `state` is what _commit records once the native call has succeeded."""
        key = self._structure(args)
        n = args[0]
        verts = [args[15 + 9 * s] for s in range(n)]
        inds = [args[16 + 9 * s] for s in range(n)]
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
        assert isinstance(seed, (tuple, int))
        if not isinstance(seed, tuple):
            seed = (seed, seed if _use_correlated_random_number else seed + 1000003)
        geometry, state = renderer._target(args)
        try:
            c = RenderFunction._unpack(seed, args, scene=renderer._scene if geometry is not None else None, geometry_changed=geometry)
        except Exception:
            renderer._forget()
            raise
        renderer._commit(c.scene, state)
        c.scene._generation = getattr(c.scene, "_generation", 0) + 1
        ctx.generation = c.scene._generation
        rb = c.backend
        nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
        h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
        img = torch.zeros(h, w, nch, device=c.device)
        rb.render(c.scene, c.options, rb.float_ptr(img.data_ptr()), rb.float_ptr(0), None, rb.float_ptr(0), rb.float_ptr(0))
        ctx.c = c
        ctx.args = args  # keeps the tensors alive (the native side only holds raw pointers)
        return img

    @staticmethod
    def backward(ctx, grad_img):
        c = ctx.c
        if c.scene._generation != ctx.generation:  # updated since this forward pass: back to the state it rendered
            c.scene.update(c.camera, c.shapes, c.materials, c.lights, c.envmap, geometry_changed=True)
            c.scene._generation += 1
            ctx.generation = c.scene._generation
        return (None,) + RenderFunction.backward(ctx, grad_img)


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
    rb = c.backend
    nch = rb.compute_num_channels(c.channels, c.scene.max_generic_texture_dimension)
    h, w = c.viewport[2] - c.viewport[0], c.viewport[3] - c.viewport[1]
    if grad_img is None:
        grad_img = torch.ones(h, w, nch, device=c.device)
    assert tuple(grad_img.shape) == (h, w, nch)
    c.screen_gradient = torch.zeros(h, w, 2, device=c.device)
    ctx = _Ctx()
    ctx.c, ctx.args = c, args
    RenderFunction.backward(ctx, grad_img.to(c.device))
    return c.screen_gradient


RenderFunction.visualize_screen_gradient = staticmethod(visualize_screen_gradient)  # (where pyredner keeps it)


def render_pathtracing(scene: Scene, num_samples=(4, 4), max_bounces: int = 1, seed: int = 0, sampler_type=None, device=None, backend=None,
                       use_primary_edge_sampling=True, use_secondary_edge_sampling=True):
    """pyredner.render_pathtracing (pyredner/render_utils.py:505-573) for a single scene."""
    args = RenderFunction.serialize_scene(scene, num_samples, max_bounces, sampler_type=sampler_type, device=device, backend=backend,
                                          use_primary_edge_sampling=use_primary_edge_sampling,
                                          use_secondary_edge_sampling=use_secondary_edge_sampling)
    return RenderFunction.apply(seed, *args)
