"""Drop-in replacement for the reference's pybind11 module `redner` (src/redner.cpp:20-272), restricted to the names
`pyredner/render_pytorch.py` uses on the RenderFunction.forward/backward path.  Same class / enum / function names,
same constructor argument order and meaning; objects are thin POD holders that are marshalled into the C ABI of
libredner_b200.so (include/redner_b200.h) when a Scene is constructed or `render` is called.

To run an unmodified pyredner on top of the H100 kernels, put `redner_b200/dropin` in front of `sys.path`
(see INTEGRATION.md); `import redner` then resolves to this module.

Error behaviour: where the reference assert()s / exit(1)s, this module raises RuntimeError carrying rb_last_error().
"""
import ctypes as C
import os
import enum

from . import _lib as L


class float_ptr:  # src/ptr.h:9-23, src/redner.cpp:23-24
    def __init__(self, addr):
        self.addr = int(addr)


class int_ptr:  # src/redner.cpp:25-26
    def __init__(self, addr):
        self.addr = int(addr)


def _addr(p):
    if p is None:
        return 0
    return int(p.addr)


def _read_floats(p, n):
    """Host-read small parameters at construction time (the reference dereferences these pointers on the host:
    src/camera.h:44-62, src/area_light.h:18-20)."""
    a = _addr(p)
    if a == 0:
        return None
    return list((C.c_float * n).from_address(a))


class CameraType(enum.IntEnum):  # src/redner.cpp:28-32
    perspective = 0
    orthographic = 1
    fisheye = 2
    panorama = 3


class SamplerType(enum.IntEnum):  # src/redner.cpp:203-205
    independent = 0
    sobol = 1


class channels(enum.IntEnum):  # src/redner.cpp:183-199
    radiance = 0
    alpha = 1
    depth = 2
    position = 3
    geometry_normal = 4
    shading_normal = 5
    uv = 6
    barycentric_coordinates = 7
    diffuse_reflectance = 8
    specular_reflectance = 9
    roughness = 10
    generic_texture = 11
    vertex_color = 12
    shape_id = 13
    triangle_id = 14
    material_id = 15


class Vector2i:  # src/redner.cpp:218-221
    def __init__(self, x, y):
        self.x = int(x)
        self.y = int(y)


class Camera:  # src/redner.cpp:34-50, src/camera.h:22-66
    def __init__(self, width, height, position, look, up, cam_to_world, world_to_cam, intrinsic_mat_inv, intrinsic_mat,
                 distortion_params, clip_near, camera_type, viewport_beg, viewport_end, lens_radius=0.0, focus_distance=1.0):
        """`lens_radius`, `focus_distance` (redner_b200 extension): a thin lens, in world units; lens_radius 0 is the pinhole."""
        c = L.rb_camera()
        c.width, c.height = int(width), int(height)
        c2w = _read_floats(cam_to_world, 16)
        if c2w is not None:
            w2c = _read_floats(world_to_cam, 16)
            c.cam_to_world[:] = c2w
            c.world_to_cam[:] = w2c
            c.use_look_at = 0
        else:
            c.position[:] = _read_floats(position, 3)
            c.look[:] = _read_floats(look, 3)
            c.up[:] = _read_floats(up, 3)
            c.use_look_at = 1
        c.intrinsic_mat_inv[:] = _read_floats(intrinsic_mat_inv, 9)
        c.intrinsic_mat[:] = _read_floats(intrinsic_mat, 9)
        d = _read_floats(distortion_params, 8)
        c.has_distortion = 0 if d is None else 1
        if d is not None:
            c.distortion[:] = d
        c.clip_near = float(clip_near)
        c.camera_type = int(camera_type)
        c.viewport_beg[:] = [viewport_beg.x, viewport_beg.y]
        c.viewport_end[:] = [viewport_end.x, viewport_end.y]
        c.lens_radius, c.focus_distance = float(lens_radius), float(focus_distance)
        self._c = c
        self.use_look_at = bool(c.use_look_at)

    def has_distortion_params(self):
        return bool(self._c.has_distortion)


class DCamera:  # src/redner.cpp:52-60
    def __init__(self, position, look, up, cam_to_world, world_to_cam, intrinsic_mat_inv, intrinsic_mat, distortion_params, lens=None):
        """`lens` (redner_b200 extension): 2 floats receiving d(lens_radius), d(focus_distance), or None."""
        d = L.rb_dcamera()
        d.position, d.look, d.up = _addr(position) or None, _addr(look) or None, _addr(up) or None
        d.cam_to_world, d.world_to_cam = _addr(cam_to_world) or None, _addr(world_to_cam) or None
        d.intrinsic_mat_inv, d.intrinsic_mat = _addr(intrinsic_mat_inv) or None, _addr(intrinsic_mat) or None
        d.distortion = _addr(distortion_params) or None
        d.lens = _addr(lens) or None
        self._c = d


class Shape:  # src/redner.cpp:84-104, src/shape.h:9-63
    def __init__(self, vertices, indices, uvs, normals, uv_indices, normal_indices, colors, num_vertices, num_uv_vertices,
                 num_normal_vertices, num_triangles, material_id, light_id):
        s = L.rb_shape()
        s.vertices, s.indices = _addr(vertices) or None, _addr(indices) or None
        s.uvs, s.normals = _addr(uvs) or None, _addr(normals) or None
        s.uv_indices, s.normal_indices = _addr(uv_indices) or None, _addr(normal_indices) or None
        s.colors = _addr(colors) or None
        s.num_vertices, s.num_uv_vertices = int(num_vertices), int(num_uv_vertices)
        s.num_normal_vertices, s.num_triangles = int(num_normal_vertices), int(num_triangles)
        s.material_id, s.light_id = int(material_id), int(light_id)
        self._c = s
        self.num_vertices = s.num_vertices
        self.num_uv_vertices = s.num_uv_vertices
        self.num_normal_vertices = s.num_normal_vertices

    def has_uvs(self):
        return bool(self._c.uvs)

    def has_normals(self):
        return bool(self._c.normals)

    def has_colors(self):
        return bool(self._c.colors)


class DShape:  # src/redner.cpp:106-110
    def __init__(self, vertices, uvs, normals, colors):
        d = L.rb_dshape()
        d.vertices, d.uvs = _addr(vertices) or None, _addr(uvs) or None
        d.normals, d.colors = _addr(normals) or None, _addr(colors) or None
        self._c = d


class _Texture:  # src/redner.cpp:112-131, src/texture.h:14-46
    _channels = None

    def __init__(self, texels, width, height, channels, uv_scale):
        assert len(texels) == len(width) == len(height)
        t = L.rb_texture()
        n = min(len(texels), L.RB_MAX_MIP_LEVELS)
        for i in range(n):
            t.texels[i] = _addr(texels[i]) or None
            t.width[i] = int(width[i])
            t.height[i] = int(height[i])
        t.num_levels = n
        t.channels = int(channels) if self._channels is None else self._channels
        t.uv_scale = _addr(uv_scale) or None
        self._c = t


class Texture1(_Texture):
    _channels = 1


class Texture3(_Texture):
    _channels = 3


class TextureN(_Texture):
    _channels = None


class Material:  # src/redner.cpp:133-151, src/material.h:12-91
    def __init__(self, diffuse_reflectance, specular_reflectance, roughness, generic_texture, normal_map, compute_specular_lighting,
                 two_sided, use_vertex_color, specular_model=0):
        """`specular_model` (redner_b200 extension): rb_specular_model, 0 for the reference's Blinn-Phong lobe, 1 for GGX."""
        m = L.rb_material()
        m.diffuse_reflectance = diffuse_reflectance._c
        m.specular_reflectance = specular_reflectance._c
        m.roughness = roughness._c
        m.generic_texture = generic_texture._c
        m.normal_map = normal_map._c
        m.compute_specular_lighting = int(bool(compute_specular_lighting))
        m.two_sided = int(bool(two_sided))
        m.use_vertex_color = int(bool(use_vertex_color))
        m.specular_model = int(specular_model)
        self._c = m

    def _levels(self, t):
        return int(t.num_levels)

    def _size(self, t, i):
        return (int(t.width[i]), int(t.height[i]))

    def get_diffuse_levels(self):
        return self._levels(self._c.diffuse_reflectance)

    def get_diffuse_size(self, i):
        return self._size(self._c.diffuse_reflectance, i)

    def get_specular_levels(self):
        return self._levels(self._c.specular_reflectance)

    def get_specular_size(self, i):
        return self._size(self._c.specular_reflectance, i)

    def get_roughness_levels(self):
        return self._levels(self._c.roughness)

    def get_roughness_size(self, i):
        return self._size(self._c.roughness, i)

    def get_generic_levels(self):
        return self._levels(self._c.generic_texture)

    def get_generic_size(self, i):
        t = self._c.generic_texture
        return (int(t.channels), int(t.width[i]), int(t.height[i]))

    def get_normal_map_levels(self):
        return self._levels(self._c.normal_map)

    def get_normal_map_size(self, i):
        return self._size(self._c.normal_map, i)


class DMaterial:  # src/redner.cpp:153-158
    def __init__(self, diffuse_reflectance, specular_reflectance, roughness, generic_texture, normal_map):
        m = L.rb_material()
        m.diffuse_reflectance = diffuse_reflectance._c
        m.specular_reflectance = specular_reflectance._c
        m.roughness = roughness._c
        m.generic_texture = generic_texture._c
        m.normal_map = normal_map._c
        self._c = m


class AreaLight:  # src/redner.cpp:160-164, src/area_light.h:8-36
    def __init__(self, shape_id, intensity, two_sided, directly_visible, emission=None, emission_sampling=0):
        """`emission` (redner_b200 extension): a Texture1 or Texture3, the light's emission texture (rb_area_light::emission), or None.
        `emission_sampling` (redner_b200 extension): rb_emission_sampling, 0 (by area) or 1 (by the emission texture)."""
        a = L.rb_area_light()
        a.shape_id = int(shape_id)
        a.intensity[:] = _read_floats(intensity, 3)
        a.two_sided = int(bool(two_sided))
        a.directly_visible = int(bool(directly_visible))
        if emission is not None:
            a.emission = emission._c
        a.emission_sampling = int(emission_sampling)
        self._c = a


class DAreaLight:  # src/redner.cpp:166-167
    def __init__(self, intensity, emission=None):
        """`emission` (redner_b200 extension): the gradient pyramid of the light's emission texture (a Texture1 / Texture3 of its shape), or
        None."""
        self.addr = _addr(intensity)
        self.emission = emission


class EnvironmentMap:  # src/redner.cpp:169-178
    def __init__(self, values, env_to_world, world_to_env, sample_cdf_ys, sample_cdf_xs, pdf_norm, directly_visible):
        e = L.rb_envmap()
        e.values = values._c
        e.env_to_world[:] = _read_floats(env_to_world, 16)
        e.world_to_env[:] = _read_floats(world_to_env, 16)
        e.sample_cdf_ys, e.sample_cdf_xs = _addr(sample_cdf_ys) or None, _addr(sample_cdf_xs) or None
        e.pdf_norm = float(pdf_norm)
        e.directly_visible = int(bool(directly_visible))
        self._c = e

    def get_levels(self):
        return int(self._c.values.num_levels)

    def get_size(self, i):
        return (int(self._c.values.width[i]), int(self._c.values.height[i]))


class DEnvironmentMap:  # src/redner.cpp:179-181
    def __init__(self, values, world_to_env):
        e = L.rb_denvmap()
        e.values = values._c
        e.world_to_env = _addr(world_to_env) or None
        self._c = e


class RenderOptions:  # src/redner.cpp:207-216, src/pathtracer.h:16-23
    def __init__(self, seed, num_samples, max_bounces, channels, sampler_type, sample_pixel_center):
        self.seed = int(seed)
        self.num_samples = int(num_samples)
        self.max_bounces = int(max_bounces)
        self.channels = [int(c) for c in channels]
        self.sampler_type = int(sampler_type)
        self.sample_pixel_center = bool(sample_pixel_center)


def compute_num_channels(chs, max_generic_texture_dimension):  # src/redner.cpp:201
    lib = L.load()
    arr = (C.c_int * max(1, len(chs)))(*[int(c) for c in chs])
    n = lib.rb_compute_num_channels(arr, len(chs), int(max_generic_texture_dimension))
    if n < 0:
        raise RuntimeError("compute_num_channels: unknown channel")
    return n


class Scene:  # src/redner.cpp:62-73, src/scene.cpp:63-307
    def __init__(self, camera, shapes, materials, area_lights, envmap, use_gpu, gpu_index, use_primary_edge_sampling,
                 use_secondary_edge_sampling, pixel_filter=None):
        """`pixel_filter` (redner_b200 extension): None for the 1-pixel box of the reference, or (rb_filter_type, width in pixels)."""
        lib = L.load()
        self._lib = lib
        self._handle = None
        if envmap is not None and use_secondary_edge_sampling:
            # The C ABI rejects this combination (the reference differentiates sky-side edge rays at stale hit points, DESIGN.md
            # section 7).  pyredner switches both edge samplers on by default, so an environment-lit scene arrives here with the flag
            # set: fail loudly unless the caller accepts the difference (RB_ENVMAP_WITHOUT_SECONDARY_EDGES=1, or pass
            # use_secondary_edge_sampling=False), in which case the scene is rendered WITHOUT shadow / interreflection boundary terms.
            if os.environ.get("RB_ENVMAP_WITHOUT_SECONDARY_EDGES", "") in ("", "0"):
                raise RuntimeError("redner_b200: secondary edge sampling together with an environment map is not available (DESIGN.md section 7). "
                                   "Pass use_secondary_edge_sampling=False, or set RB_ENVMAP_WITHOUT_SECONDARY_EDGES=1 to have it switched off "
                                   "automatically: such scenes then lose their secondary (shadow / interreflection) boundary gradients compared "
                                   "with the reference.")
            import warnings
            warnings.warn("redner_b200: secondary edge sampling is switched off for this scene (environment map, "
                          "RB_ENVMAP_WITHOUT_SECONDARY_EDGES=1); interior terms and primary edges are rendered and differentiated")
            use_secondary_edge_sampling = False
        self.use_gpu = bool(use_gpu)
        self.gpu_index = int(gpu_index)
        self._flags = (int(bool(use_primary_edge_sampling)), int(bool(use_secondary_edge_sampling)))
        d = self._desc(camera, shapes, materials, area_lights, envmap, pixel_filter)
        h = C.c_void_p()
        stream = self._stream()
        if hasattr(lib, "rb_scene_create_on_stream"):
            rc = lib.rb_scene_create_on_stream(C.byref(d), C.byref(h), C.c_void_p(stream or 0))
        else:
            rc = lib.rb_scene_create(C.byref(d), C.byref(h))
        if rc != 0:
            raise RuntimeError("redner.Scene: " + L.last_error(lib))
        self._handle = h
        self.max_generic_texture_dimension = lib.rb_scene_max_generic_texture_dimension(h)

    def _desc(self, camera, shapes, materials, area_lights, envmap, pixel_filter):
        d = L.rb_scene_desc()
        d.camera = camera._c
        self._shapes = (L.rb_shape * max(1, len(shapes)))(*[s._c for s in shapes])
        self._num_shapes = len(shapes)
        self._materials = (L.rb_material * max(1, len(materials)))(*[m._c for m in materials])
        self._lights = (L.rb_area_light * max(1, len(area_lights)))(*[a._c for a in area_lights])
        d.num_shapes, d.shapes = len(shapes), self._shapes
        d.num_materials, d.materials = len(materials), self._materials
        d.num_lights, d.lights = len(area_lights), self._lights
        self._env = envmap._c if envmap is not None else None
        d.envmap = C.pointer(self._env) if self._env is not None else None
        d.use_gpu = int(self.use_gpu)
        d.gpu_index = self.gpu_index
        d.use_primary_edge_sampling, d.use_secondary_edge_sampling = self._flags
        if pixel_filter is not None:
            d.pixel_filter = L.rb_pixel_filter(int(pixel_filter[0]), float(pixel_filter[1]))
        return d

    def _stream(self):
        # the current PyTorch stream of the scene's device: the geometry tensors were produced there
        try:
            import torch
            if self.use_gpu and torch.cuda.is_available():
                return torch.cuda.current_stream(self.gpu_index if self.gpu_index >= 0 else None).cuda_stream
        except ImportError:
            pass
        return 0

    # --- redner_b200 extensions (no reference counterpart) ---
    def set_partition(self, part, num_parts, rows_per_stripe=16):
        if self._lib.rb_scene_set_partition(self._handle, int(part), int(num_parts), int(rows_per_stripe)) != 0:
            raise RuntimeError("redner.Scene.set_partition: " + L.last_error(self._lib))

    def set_camera(self, camera):
        """Re-target this scene at another camera; only the camera-dependent tables are rebuilt, on the device (rb_scene_set_camera)."""
        if self._lib.rb_scene_set_camera(self._handle, C.byref(camera._c)) != 0:
            raise RuntimeError("redner.Scene.set_camera: " + L.last_error(self._lib))

    def update(self, camera, shapes, materials, area_lights, envmap, geometry_changed=True, pixel_filter=None):
        """Re-target this scene at shapes / materials / lights / environment map / camera / pixel filter of the SAME structure as its build,
        without building a new scene (rb_scene_update): counts, ids and optional buffers as before, index buffers with the same contents.
        Pass geometry_changed=True when vertex positions may have been written in place; a new vertex buffer is noticed by itself."""
        d = self._desc(camera, shapes, materials, area_lights, envmap, pixel_filter)
        if self._lib.rb_scene_update(self._handle, C.byref(d), int(bool(geometry_changed)), C.c_void_p(self._stream() or 0)) != 0:
            raise RuntimeError("redner.Scene.update: " + L.last_error(self._lib))

    def table(self, name):
        """One table of the scene as the kernels see it, as raw bytes (rb_scene_table; names in _lib.RB_TABLES): test hook."""
        import numpy as np
        which = L.RB_TABLES.index(name)
        n = C.c_size_t(0)
        if self._lib.rb_scene_table(self._handle, which, None, 0, C.byref(n)) != 0:
            raise RuntimeError("redner.Scene.table: " + L.last_error(self._lib))
        out = np.zeros(n.value, dtype=np.uint8)
        if n.value > 0 and self._lib.rb_scene_table(self._handle, which, out.ctypes.data_as(C.c_void_p), out.nbytes, C.byref(n)) != 0:
            raise RuntimeError("redner.Scene.table: " + L.last_error(self._lib))
        return out

    def trace_rays(self, rays, any_hit=False, brute_force=False):
        """Ray queries against the scene's triangle BVH (rb_scene_trace_rays): test hook.  `rays` is an [N, 8] float32 tensor on the
        scene's device (the outputs are allocated there too), rows (origin xyz, tnear, direction xyz, tfar).  Returns ([N, 2] int32 (shape id, triangle id), -1 for a miss;
        [N] float32 hit distance, tfar for a miss).  `brute_force` tests every triangle instead of walking the tree."""
        import torch
        rays = rays.to(torch.float32).contiguous()
        if rays.dim() != 2 or rays.shape[1] != 8:
            raise ValueError("redner.Scene.trace_rays: rays must have shape [N, 8]")
        n = rays.shape[0]
        ids = torch.empty((n, 2), dtype=torch.int32, device=rays.device)
        t = torch.empty(n, dtype=torch.float32, device=rays.device)
        flags = (L.RB_TRACE_ANY_HIT if any_hit else 0) | (L.RB_TRACE_BRUTE_FORCE if brute_force else 0)
        if self._lib.rb_scene_trace_rays(self._handle, C.c_void_p(rays.data_ptr()), n, flags, C.c_void_p(ids.data_ptr()), C.c_void_p(t.data_ptr())) != 0:
            raise RuntimeError("redner.Scene.trace_rays: " + L.last_error(self._lib))
        return ids, t

    def light_sample_test(self, light, samples, queries=None):
        """The point-on-light sampler of area light `light` and its density (rb_light_sample_test): test hook.  `samples` is an [N, 3]
        float64 tensor (tri_sel, su, sv) on the scene's device, `queries` None or an [M, 3] float32 tensor (triangle, u, v).  Returns
        ([N, 3] int32 (branch, triangle, rejected), [N, 3] float64 (b1, b2, density), [M] float64 densities or None)."""
        import torch
        samples = samples.to(torch.float64).contiguous()
        if samples.dim() != 2 or samples.shape[1] != 3:
            raise ValueError("redner.Scene.light_sample_test: samples must have shape [N, 3]")
        n, dev = samples.shape[0], samples.device
        ints = torch.empty((n, 3), dtype=torch.int32, device=dev)
        doubles = torch.empty((n, 3), dtype=torch.float64, device=dev)
        m, pdfs = 0, None
        if queries is not None:
            queries = queries.to(device=dev, dtype=torch.float32).contiguous()
            if queries.dim() != 2 or queries.shape[1] != 3:
                raise ValueError("redner.Scene.light_sample_test: queries must have shape [M, 3]")
            m = queries.shape[0]
            pdfs = torch.empty(m, dtype=torch.float64, device=dev)
        stream = 0
        if samples.is_cuda:
            torch.cuda.set_device(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        if self._lib.rb_light_sample_test(self._handle, int(light), ptr(samples), n, ptr(ints), ptr(doubles), ptr(queries), m, ptr(pdfs),
                                          C.c_void_p(stream or 0)) != 0:
            raise RuntimeError("redner.Scene.light_sample_test: " + L.last_error(self._lib))
        return ints, doubles, pdfs

    def surface_test(self, op, inputs, d_shapes=None):
        """Geometry queries through the functions the render kernels call, on this scene's shapes (rb_surface_test): test hook.  `op` is
        one of _lib.RB_SURFTEST_*, `inputs` an [N, <= 96] float64 tensor on the scene's device (rows as in include/redner_b200.h,
        zero-padded).  `d_shapes` is None or one dict per shape of float32 gradient tensors ("vertices", "uvs", "normals", "colors", each
        optional) that the adjoint ops scatter into.  Returns the [N, 96] float64 outputs."""
        import torch
        inputs = inputs.to(torch.float64)
        if inputs.dim() != 2 or inputs.shape[1] > 96:
            raise ValueError("redner.Scene.surface_test: inputs must have shape [N, <= 96]")
        n, dev = inputs.shape[0], inputs.device
        rows = torch.zeros((n, 96), dtype=torch.float64, device=dev)
        rows[:, :inputs.shape[1]] = inputs
        out = torch.zeros((n, 96), dtype=torch.float64, device=dev)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        dsh = None
        if d_shapes is not None:
            if len(d_shapes) != self._num_shapes:
                raise ValueError("redner.Scene.surface_test: d_shapes needs one entry per shape of the scene (%d), not %d" % (self._num_shapes, len(d_shapes)))
            for d in d_shapes:
                for t in d.values():
                    if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or t.device != dev):
                        raise ValueError("redner.Scene.surface_test: gradient buffers must be contiguous float32 tensors on the inputs' device")
            dsh = (L.rb_dshape * max(self._num_shapes, 1))()
            for i, d in enumerate(d_shapes):
                dsh[i] = L.rb_dshape(*(ptr(d.get(k)) for k in ("vertices", "uvs", "normals", "colors")))
        stream = 0
        if rows.is_cuda:
            torch.cuda.set_device(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
        if self._lib.rb_surface_test(self._handle, int(op), ptr(rows), n, ptr(out), dsh, C.c_void_p(stream or 0)) != 0:
            raise RuntimeError("redner.Scene.surface_test: " + L.last_error(self._lib))
        return out

    def camera_test(self, op, inputs, acc=None):
        """Camera queries through the functions the render kernels call, on this scene's camera (rb_camera_test): test hook.  `op` is one
        of _lib.RB_CAMTEST_*, `inputs` an [N, <= 64] float64 tensor on the scene's device (rows as in include/redner_b200.h, zero-padded).
        `acc` is None or the [60, N] float32 accumulator the adjoint ops add to (query i's column is acc[:, i]; a camera without a lens
        uses the first 58 rows); the adjoint ops get a zeroed one when it is None.  Returns ([N, 64] float64 outputs, acc)."""
        import torch
        inputs = inputs.to(torch.float64)
        if inputs.dim() != 2 or inputs.shape[1] > 64:
            raise ValueError("redner.Scene.camera_test: inputs must have shape [N, <= 64]")
        n, dev = inputs.shape[0], inputs.device
        rows = torch.zeros((n, 64), dtype=torch.float64, device=dev)
        rows[:, :inputs.shape[1]] = inputs
        out = torch.zeros((n, 64), dtype=torch.float64, device=dev)
        if acc is None and op in (L.RB_CAMTEST_D_RAY, L.RB_CAMTEST_D_PROJECT):
            acc = torch.zeros((60, n), dtype=torch.float32, device=dev)
        if acc is not None and (acc.dtype != torch.float32 or not acc.is_contiguous() or tuple(acc.shape) != (60, n) or acc.device != dev):
            raise ValueError("redner.Scene.camera_test: acc must be a contiguous float32 [60, N] tensor on the inputs' device")
        stream = 0
        if rows.is_cuda:
            torch.cuda.set_device(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        if self._lib.rb_camera_test(self._handle, int(op), ptr(rows), n, ptr(out), ptr(acc), C.c_void_p(stream or 0)) != 0:
            raise RuntimeError("redner.Scene.camera_test: " + L.last_error(self._lib))
        return out, acc

    def last_stats(self):
        n = C.c_int(0)
        ms = C.c_float(0)
        self._lib.rb_scene_last_stats(self._handle, C.byref(n), C.byref(ms))
        return n.value, ms.value

    def last_exact_bytes(self):
        """Bytes of exact gradient accumulators the last render on this scene used (rb_scene_last_exact_bytes; 0 unless deterministic)."""
        n = C.c_size_t(0)
        self._lib.rb_scene_last_exact_bytes(self._handle, C.byref(n))
        return n.value

    def last_live_samples(self):
        """(live samples, bands) of the last backward pass on this scene (rb_scene_last_live_samples): the samples of the pixels whose
        d_rendered_image is not zero, and the bands the backward pass ran over them."""
        n, b = C.c_longlong(0), C.c_longlong(0)
        self._lib.rb_scene_last_live_samples(self._handle, C.byref(n), C.byref(b))
        return n.value, b.value

    def last_stage_stats(self):
        """({kernel name: ms}, path_vertices, primary_hits) of the last render on this scene."""
        ms = (C.c_float * 4)()
        v, h = C.c_double(0), C.c_double(0)
        self._lib.rb_scene_last_stage_stats(self._handle, ms, C.byref(v), C.byref(h))
        out = dict(zip(("k_forward", "k_backward", "k_primary_edge", "k_finish_camera"), list(ms)))
        if hasattr(self._lib, "rb_scene_last_backward_stats"):
            # "k_backward" is the sum over the backward bands; its three stages follow
            b = (C.c_float * 3)()
            self._lib.rb_scene_last_backward_stats(self._handle, b)
            out.update(dict(zip(("k_bwd_trace", "k_bwd_secondary", "k_bwd_sweep"), list(b))))
        return out, v.value, h.value

    def edge_trees(self):
        """(records [n, 32] as uint32 words, root of the camera-silhouette tree, root of the other tree, billboard size): test hook."""
        import numpy as np
        info = (C.c_int * 3)()
        ex = C.c_float(0)
        self._lib.rb_scene_edge_trees(self._handle, info, C.byref(ex), None, 0)
        rec = np.zeros((max(info[0], 0), 32), dtype=np.uint32)
        if info[0] > 0:
            self._lib.rb_scene_edge_trees(self._handle, info, C.byref(ex), rec.ctypes.data_as(C.c_void_p), rec.nbytes)
        return rec, info[1], info[2], ex.value

    def edge_list(self):
        """[num_edges, 5] int32 rows (shape, v0, v1, f0, f1): test hook."""
        import numpy as np
        n = C.c_int(0)
        self._lib.rb_scene_edge_list(self._handle, C.byref(n), None, 0)
        out = np.zeros((max(n.value, 0), 5), dtype=np.int32)
        if n.value > 0:
            self._lib.rb_scene_edge_list(self._handle, C.byref(n), out.ctypes.data_as(C.POINTER(C.c_int)), out.nbytes)
        return out

    def build_ms(self):
        ms = (C.c_float * 3)()
        self._lib.rb_scene_build_ms(self._handle, ms)
        return dict(zip(("bvh", "lights", "edges"), list(ms)))

    def __del__(self):
        try:
            if self._handle is not None and self._handle.value:
                self._lib.rb_scene_destroy(self._handle)
                self._handle = None
        except Exception:
            pass


def texture_test(tex, queries, d_values=None, d_tex=None):
    """Texture lookups through the lookup and adjoint the render kernels call (rb_texture_test): test hook.  `tex` (and `d_tex`) are
    Texture1 / Texture3 / TextureN; `queries` is an [N, 6] float32 tensor (u, v, du/dx, du/dy, dv/dx, dv/dy) on the textures' device,
    which is made current.  Returns ([N, channels] values, [N, 6] d(queries) or None).  With `d_values` ([N, channels]) the adjoint
    scatters into `d_tex`'s buffers (zeroed by the caller; its uv_scale may be NULL)."""
    import torch
    lib = L.load()
    queries = queries.to(torch.float32).contiguous()
    if queries.dim() != 2 or queries.shape[1] != 6:
        raise ValueError("redner.texture_test: queries must have shape [N, 6]")
    n, nch = queries.shape[0], int(tex._c.channels)
    values = torch.empty((n, nch), dtype=torch.float32, device=queries.device)
    d_queries = None
    if d_values is not None:
        d_values = d_values.to(torch.float32).contiguous()
        if tuple(d_values.shape) != (n, nch):
            raise ValueError("redner.texture_test: d_values must have shape [N, channels]")
        if d_tex is None:
            raise ValueError("redner.texture_test: d_values needs d_tex")
        d_queries = torch.empty((n, 6), dtype=torch.float32, device=queries.device)
    stream = 0
    if queries.is_cuda:
        torch.cuda.set_device(queries.device)
        stream = torch.cuda.current_stream(queries.device).cuda_stream
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    rc = lib.rb_texture_test(C.byref(tex._c), C.byref(d_tex._c) if d_tex is not None else None, ptr(queries), n, ptr(d_values), ptr(values),
                             ptr(d_queries), C.c_void_p(stream or 0))
    if rc != 0:
        raise RuntimeError("redner.texture_test: " + L.last_error(lib))
    return values, d_queries


def envmap_test(envmap, queries, d_out=None, d_values=None, d_w2e=None, samples=None, with_pdf=True):
    """Environment-map lookups, adjoints, samples and pdfs through the functions the render kernels call (rb_envmap_test): test hook.
    `envmap` is an EnvironmentMap, `d_values` a Texture3 gradient pyramid of the map's shape (zeroed by the caller; its uv_scale may be
    NULL) and `d_w2e` a float32 tensor of at least 16 elements or None.  `queries` is an [N, 9] float32 tensor (dir, dir_dx, dir_dy) on
    the map's device, which is made current; `samples` an [M, 2] float64 tensor (sx, sy) or None.  Returns ([N, 3] values, [N] pdfs or
    None, [N, 9] d(queries) or None, [M, 3] sampled directions or None).  With `d_out` ([N, 3]) the adjoint scatters into `d_values`
    and `d_w2e`."""
    import torch
    lib = L.load()
    queries = queries.to(torch.float32).contiguous()
    if queries.dim() != 2 or queries.shape[1] != 9:
        raise ValueError("redner.envmap_test: queries must have shape [N, 9]")
    n, dev = queries.shape[0], queries.device
    values = torch.empty((n, 3), dtype=torch.float32, device=dev)
    pdfs = torch.empty(n, dtype=torch.float32, device=dev) if with_pdf else None
    d_queries = None
    if d_out is not None:
        d_out = d_out.to(torch.float32).contiguous()
        if tuple(d_out.shape) != (n, 3):
            raise ValueError("redner.envmap_test: d_out must have shape [N, 3]")
        if d_values is None:
            raise ValueError("redner.envmap_test: d_out needs d_values")
        if d_w2e is not None and (d_w2e.dtype != torch.float32 or not d_w2e.is_contiguous() or d_w2e.numel() < 16):
            raise ValueError("redner.envmap_test: d_w2e must be a contiguous float32 tensor of at least 16 elements")
        d_queries = torch.empty((n, 9), dtype=torch.float32, device=dev)
    m, sample_dirs = 0, None
    if samples is not None:
        samples = samples.to(device=dev, dtype=torch.float64).contiguous()
        if samples.dim() != 2 or samples.shape[1] != 2:
            raise ValueError("redner.envmap_test: samples must have shape [M, 2]")
        m = samples.shape[0]
        sample_dirs = torch.empty((m, 3), dtype=torch.float32, device=dev)
    stream = 0
    if queries.is_cuda:
        torch.cuda.set_device(dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    rc = lib.rb_envmap_test(C.byref(envmap._c), C.byref(d_values._c) if d_values is not None else None, ptr(d_w2e), ptr(queries), n, ptr(d_out),
                            ptr(values), ptr(pdfs), ptr(d_queries), ptr(samples), m, ptr(sample_dirs), C.c_void_p(stream or 0))
    if rc != 0:
        raise RuntimeError("redner.envmap_test: " + L.last_error(lib))
    return values, pdfs, d_queries, sample_dirs


class DScene:  # src/redner.cpp:75-82
    def __init__(self, camera, shapes, materials, area_lights, envmap, use_gpu, gpu_index):
        d = L.rb_dscene_desc()
        d.camera = camera._c
        self._shapes = (L.rb_dshape * max(1, len(shapes)))(*[s._c for s in shapes])
        self._materials = (L.rb_material * max(1, len(materials)))(*[m._c for m in materials])
        self._lights = (C.c_void_p * max(1, len(area_lights)))(*[a.addr or None for a in area_lights])
        d.num_shapes, d.shapes = len(shapes), self._shapes
        d.num_materials, d.materials = len(materials), self._materials
        d.num_lights, d.light_intensity = len(area_lights), self._lights
        # (the emission gradients only when some light has one: otherwise the descriptor is the one without emission textures)
        emission = [getattr(a, "emission", None) for a in area_lights]
        self._emission = None
        if any(e is not None for e in emission):
            self._emission = (L.rb_texture * len(area_lights))(*[e._c if e is not None else L.rb_texture() for e in emission])
            d.light_emission = self._emission
        self.envmap = envmap
        d.envmap = C.pointer(envmap._c) if envmap is not None else None
        self._c = d


def _options(options, deterministic=None):
    """rb_options of a RenderOptions; the channel array is kept alive by the returned tuple."""
    o = L.rb_options()
    o.seed = options.seed
    o.num_samples = options.num_samples
    o.max_bounces = options.max_bounces
    chs = (C.c_int * max(1, len(options.channels)))(*options.channels)
    o.num_channels = len(options.channels)
    o.channels = chs
    o.sampler_type = options.sampler_type
    o.sample_pixel_center = int(options.sample_pixel_center)
    if deterministic is None:
        try:
            import torch
            deterministic = torch.are_deterministic_algorithms_enabled()
        except ImportError:
            deterministic = False
    o.deterministic = int(bool(deterministic))
    return o, chs


def _render_stream(scene, stream):
    if stream is None:
        try:
            import torch
            # (the stream of the SCENE's device: a stream handle of another device would be invalid there)
            stream = torch.cuda.current_stream(scene.gpu_index if scene.gpu_index >= 0 else None).cuda_stream if torch.cuda.is_available() else 0
        except Exception:
            stream = 0
    return C.c_void_p(stream or 0)


def render(scene, options, rendered_image, d_rendered_image, d_scene, screen_gradient_image, debug_image, stream=None):
    """src/redner.cpp:257 / src/pathtracer.cpp:177-183.  `debug_image` is accepted and ignored (the reference never
    reads it).  `stream` (a cudaStream_t value) is a redner_b200 extension; by default the current PyTorch stream is used
    when torch is importable, else the legacy default stream.

    Under `torch.use_deterministic_algorithms(True)` the backward pass runs in the library's deterministic mode
    (rb_options.deterministic): every gradient is the correctly rounded exact sum of the per-sample contributions, bit for bit the
    same from run to run, at some cost in time and 88 bytes of device scratch per gradient float.  There is no other switch; every
    caller of this function (api.RenderFunction, api.SceneRenderer, api.render_batch, dist and the drop-in) follows PyTorch's."""
    lib = scene._lib
    o, _chs = _options(options)
    rc = lib.rb_render(scene._handle, C.byref(o), _addr(rendered_image) or None, _addr(d_rendered_image) or None,
                       C.byref(d_scene._c) if d_scene is not None else None, _addr(screen_gradient_image) or None, _render_stream(scene, stream))
    if rc != 0:
        raise RuntimeError("redner.render: " + L.last_error(lib))


# --- exact records (redner_b200 extension, no reference counterpart): deterministic gradients summed across calls, devices and processes.
# render_exact hands out the exact accumulators of a deterministic backward pass as an int64 tensor [count, RB_EXACT_RECORD_WORDS];
# records of several calls -- the stripes of one image on several ranks -- are summed as integers (torch.distributed.all_reduce SUM,
# or plain tensor addition), and round_exact turns the sum into gradients once: those of ONE deterministic render over all the
# samples, bit for bit (include/redner_b200.h, rb_render_exact).

def _scene_device(scene):
    import torch
    return torch.device("cuda", scene.gpu_index if scene.gpu_index >= 0 else torch.cuda.current_device()) if scene.use_gpu else torch.device("cpu")


def exact_record_count(scene, options, d_scene, screen_gradient_image=None):
    """(number of records, 64-bit fingerprint of their layout) of a backward pass of `options` into `d_scene` (rb_exact_record_count).
    The fingerprint depends on the structure of the descriptor only; ranks compare it before they sum their records."""
    lib = scene._lib
    o, _chs = _options(options, True)
    n, fp = C.c_size_t(0), C.c_uint64(0)
    if lib.rb_exact_record_count(scene._handle, C.byref(o), C.byref(d_scene._c) if d_scene is not None else None, _addr(screen_gradient_image) or None,
                                 C.byref(n), C.byref(fp)) != 0:
        raise RuntimeError("redner.exact_record_count: " + L.last_error(lib))
    return n.value, fp.value


def _check_records(records, count, device, who):
    import torch
    if records is None:
        raise RuntimeError("redner.%s: records is None" % who)
    if records.dtype != torch.int64 or not records.is_contiguous() or records.device != device:
        raise RuntimeError("redner.%s: records must be a contiguous int64 tensor on %s" % (who, device))
    if records.numel() != count * L.RB_EXACT_RECORD_WORDS:
        raise RuntimeError("redner.%s: records holds %d words, the descriptor needs %d records of %d" % (who, records.numel(), count, L.RB_EXACT_RECORD_WORDS))


def render_exact(scene, options, d_rendered_image, d_scene, screen_gradient_image=None, records=None, stream=None):
    """The deterministic backward pass of `render`, ending in records instead of gradients (rb_render_exact): returns `records` -- an
    int64 tensor [count, RB_EXACT_RECORD_WORDS] on the scene's device, zeros if None -- with this pass's accumulators added.  No buffer of
    `d_scene` is written; its pointers only give the layout."""
    import torch
    lib = scene._lib
    count, _ = exact_record_count(scene, options, d_scene, screen_gradient_image)
    dev = _scene_device(scene)
    if records is None:
        records = torch.zeros((count, L.RB_EXACT_RECORD_WORDS), dtype=torch.int64, device=dev)
    _check_records(records, count, dev, "render_exact")
    o, _chs = _options(options, True)
    rc = lib.rb_render_exact(scene._handle, C.byref(o), _addr(d_rendered_image) or None, C.byref(d_scene._c), _addr(screen_gradient_image) or None,
                             C.c_void_p(records.data_ptr()), count, _render_stream(scene, stream))
    if rc != 0:
        raise RuntimeError("redner.render_exact: " + L.last_error(lib))
    return records


def round_exact(scene, options, d_scene, screen_gradient_image, records, stream=None):
    """The end of a deterministic `render` on `records` (a sum of render_exact results of this layout) (rb_exact_round): every record
    that received something is rounded once and added into d_scene's buffers / the screen-gradient image, and the camera gradients are
    finished with the scene's camera."""
    lib = scene._lib
    count, _ = exact_record_count(scene, options, d_scene, screen_gradient_image)
    _check_records(records, count, _scene_device(scene), "round_exact")
    o, _chs = _options(options, True)
    rc = lib.rb_exact_round(scene._handle, C.byref(o), C.byref(d_scene._c), _addr(screen_gradient_image) or None, C.c_void_p(records.data_ptr()), count,
                            _render_stream(scene, stream))
    if rc != 0:
        raise RuntimeError("redner.round_exact: " + L.last_error(lib))
