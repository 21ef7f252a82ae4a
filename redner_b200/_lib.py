"""ctypes binding of include/redner_b200.h (the C-ABI boundary).

The shared object is built in-tree by `python -m redner_b200.build` (nvcc, sm_90a).  There is NO fallback: if the
library is missing or fails to load, importing this module raises, and every render call goes through the CUDA
kernels in redner_b200/csrc.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libredner_b200.so")
LIB_PATH_F64 = os.path.join(_HERE, "libredner_b200_f64.so")

RB_MAX_MIP_LEVELS = 8

c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int)

# enum rb_scene_table_id
RB_TABLES = ("bvh_nodes", "bvh_triangles", "light_pmf", "light_cdf", "light_areas", "area_cdf_pool", "area_cdf_offsets", "primary_edge_pmf",
             "primary_edge_cdf")
# enum rb_trace_flags
RB_TRACE_ANY_HIT, RB_TRACE_BRUTE_FORCE = 1, 2
# int64 words per record of rb_render_exact / rb_exact_round: 10 limbs, then the counts of +inf, -inf and NaN contributions
RB_EXACT_RECORD_WORDS = 13


class rb_camera(C.Structure):
    _fields_ = [
        ("width", C.c_int), ("height", C.c_int), ("use_look_at", C.c_int),
        ("position", C.c_float * 3), ("look", C.c_float * 3), ("up", C.c_float * 3),
        ("cam_to_world", C.c_float * 16), ("world_to_cam", C.c_float * 16),
        ("intrinsic_mat_inv", C.c_float * 9), ("intrinsic_mat", C.c_float * 9),
        ("has_distortion", C.c_int), ("distortion", C.c_float * 8),
        ("clip_near", C.c_float), ("camera_type", C.c_int),
        ("viewport_beg", C.c_int * 2), ("viewport_end", C.c_int * 2),
    ]


class rb_shape(C.Structure):
    _fields_ = [
        ("vertices", C.c_void_p), ("indices", C.c_void_p), ("uvs", C.c_void_p), ("normals", C.c_void_p),
        ("uv_indices", C.c_void_p), ("normal_indices", C.c_void_p), ("colors", C.c_void_p),
        ("num_vertices", C.c_int), ("num_uv_vertices", C.c_int), ("num_normal_vertices", C.c_int), ("num_triangles", C.c_int),
        ("material_id", C.c_int), ("light_id", C.c_int),
    ]


class rb_texture(C.Structure):
    _fields_ = [
        ("texels", C.c_void_p * RB_MAX_MIP_LEVELS), ("width", C.c_int * RB_MAX_MIP_LEVELS), ("height", C.c_int * RB_MAX_MIP_LEVELS),
        ("channels", C.c_int), ("num_levels", C.c_int), ("uv_scale", C.c_void_p),
    ]


class rb_material(C.Structure):
    _fields_ = [
        ("diffuse_reflectance", rb_texture), ("specular_reflectance", rb_texture), ("roughness", rb_texture),
        ("generic_texture", rb_texture), ("normal_map", rb_texture),
        ("compute_specular_lighting", C.c_int), ("two_sided", C.c_int), ("use_vertex_color", C.c_int),
    ]


class rb_area_light(C.Structure):
    _fields_ = [("shape_id", C.c_int), ("intensity", C.c_float * 3), ("two_sided", C.c_int), ("directly_visible", C.c_int)]


class rb_envmap(C.Structure):
    _fields_ = [
        ("values", rb_texture), ("env_to_world", C.c_float * 16), ("world_to_env", C.c_float * 16),
        ("sample_cdf_ys", C.c_void_p), ("sample_cdf_xs", C.c_void_p), ("pdf_norm", C.c_float), ("directly_visible", C.c_int),
    ]


class rb_scene_desc(C.Structure):
    _fields_ = [
        ("camera", rb_camera),
        ("num_shapes", C.c_int), ("shapes", C.POINTER(rb_shape)),
        ("num_materials", C.c_int), ("materials", C.POINTER(rb_material)),
        ("num_lights", C.c_int), ("lights", C.POINTER(rb_area_light)),
        ("envmap", C.POINTER(rb_envmap)),
        ("use_gpu", C.c_int), ("gpu_index", C.c_int),
        ("use_primary_edge_sampling", C.c_int), ("use_secondary_edge_sampling", C.c_int),
    ]


class rb_options(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64), ("num_samples", C.c_int), ("max_bounces", C.c_int), ("num_channels", C.c_int),
        ("channels", c_int_p), ("sampler_type", C.c_int), ("sample_pixel_center", C.c_int), ("deterministic", C.c_int),
    ]


class rb_dshape(C.Structure):
    _fields_ = [("vertices", C.c_void_p), ("uvs", C.c_void_p), ("normals", C.c_void_p), ("colors", C.c_void_p)]


class rb_dcamera(C.Structure):
    _fields_ = [
        ("position", C.c_void_p), ("look", C.c_void_p), ("up", C.c_void_p), ("cam_to_world", C.c_void_p), ("world_to_cam", C.c_void_p),
        ("intrinsic_mat_inv", C.c_void_p), ("intrinsic_mat", C.c_void_p), ("distortion", C.c_void_p),
    ]


class rb_denvmap(C.Structure):
    _fields_ = [("values", rb_texture), ("world_to_env", C.c_void_p)]


class rb_dscene_desc(C.Structure):
    _fields_ = [
        ("camera", rb_dcamera),
        ("num_shapes", C.c_int), ("shapes", C.POINTER(rb_dshape)),
        ("num_materials", C.c_int), ("materials", C.POINTER(rb_material)),
        ("num_lights", C.c_int), ("light_intensity", C.POINTER(C.c_void_p)),
        ("envmap", C.POINTER(rb_denvmap)),
    ]


EXPORTS = [
    "rb_scene_create", "rb_scene_create_on_stream", "rb_scene_destroy", "rb_scene_max_generic_texture_dimension", "rb_compute_num_channels", "rb_render",
    "rb_scene_set_partition", "rb_scene_last_stats", "rb_scene_last_stage_stats", "rb_scene_last_backward_stats", "rb_scene_last_exact_bytes", "rb_release_scratch", "rb_scene_build_ms", "rb_scene_edge_trees", "rb_scene_edge_list", "rb_scene_table", "rb_scene_trace_rays", "rb_exact_sum_test", "rb_texture_test", "rb_scene_set_camera", "rb_scene_update", "rb_render_batch", "rb_exact_record_count", "rb_render_exact", "rb_exact_round", "rb_last_error", "rb_version",
]


def _bind(lib):
    lib.rb_scene_create.argtypes = [C.POINTER(rb_scene_desc), C.POINTER(C.c_void_p)]
    lib.rb_scene_create.restype = C.c_int
    if hasattr(lib, "rb_scene_create_on_stream"):
        lib.rb_scene_create_on_stream.argtypes = [C.POINTER(rb_scene_desc), C.POINTER(C.c_void_p), C.c_void_p]
        lib.rb_scene_create_on_stream.restype = C.c_int
    if hasattr(lib, "rb_scene_update"):
        lib.rb_scene_update.argtypes = [C.c_void_p, C.POINTER(rb_scene_desc), C.c_int, C.c_void_p]
        lib.rb_scene_update.restype = C.c_int
    lib.rb_scene_destroy.argtypes = [C.c_void_p]
    lib.rb_scene_destroy.restype = None
    lib.rb_scene_max_generic_texture_dimension.argtypes = [C.c_void_p]
    lib.rb_scene_max_generic_texture_dimension.restype = C.c_int
    lib.rb_compute_num_channels.argtypes = [c_int_p, C.c_int, C.c_int]
    lib.rb_compute_num_channels.restype = C.c_int
    lib.rb_render.argtypes = [C.c_void_p, C.POINTER(rb_options), C.c_void_p, C.c_void_p, C.POINTER(rb_dscene_desc), C.c_void_p, C.c_void_p]
    lib.rb_render.restype = C.c_int
    lib.rb_scene_set_partition.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.rb_scene_set_partition.restype = C.c_int
    lib.rb_scene_last_stats.argtypes = [C.c_void_p, c_int_p, c_float_p]
    lib.rb_scene_last_stats.restype = C.c_int
    if hasattr(lib, "rb_scene_last_stage_stats"):
        lib.rb_scene_last_stage_stats.argtypes = [C.c_void_p, c_float_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        lib.rb_scene_last_stage_stats.restype = C.c_int
        lib.rb_scene_build_ms.argtypes = [C.c_void_p, c_float_p]
        lib.rb_scene_build_ms.restype = C.c_int
    if hasattr(lib, "rb_scene_last_backward_stats"):
        lib.rb_scene_last_backward_stats.argtypes = [C.c_void_p, c_float_p]
        lib.rb_scene_last_backward_stats.restype = C.c_int
    if hasattr(lib, "rb_scene_last_exact_bytes"):
        lib.rb_scene_last_exact_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        lib.rb_scene_last_exact_bytes.restype = C.c_int
    if hasattr(lib, "rb_release_scratch"):
        lib.rb_release_scratch.argtypes = []
        lib.rb_release_scratch.restype = None
    if hasattr(lib, "rb_scene_set_camera"):
        lib.rb_scene_set_camera.argtypes = [C.c_void_p, C.POINTER(rb_camera)]
        lib.rb_scene_set_camera.restype = C.c_int
    if hasattr(lib, "rb_render_batch"):
        lib.rb_render_batch.argtypes = [C.c_void_p, C.c_int, C.POINTER(rb_camera), C.POINTER(rb_options), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                        C.POINTER(C.POINTER(rb_dscene_desc)), C.c_void_p]
        lib.rb_render_batch.restype = C.c_int
    if hasattr(lib, "rb_scene_edge_trees"):
        lib.rb_scene_edge_trees.argtypes = [C.c_void_p, c_int_p, c_float_p, C.c_void_p, C.c_size_t]
        lib.rb_scene_edge_trees.restype = C.c_int
    if hasattr(lib, "rb_scene_edge_list"):
        lib.rb_scene_edge_list.argtypes = [C.c_void_p, c_int_p, c_int_p, C.c_size_t]
        lib.rb_scene_edge_list.restype = C.c_int
    if hasattr(lib, "rb_scene_table"):
        lib.rb_scene_table.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        lib.rb_scene_table.restype = C.c_int
    if hasattr(lib, "rb_scene_trace_rays"):
        lib.rb_scene_trace_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        lib.rb_scene_trace_rays.restype = C.c_int
    if hasattr(lib, "rb_exact_sum_test"):
        lib.rb_exact_sum_test.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.rb_exact_sum_test.restype = C.c_int
    if hasattr(lib, "rb_texture_test"):
        lib.rb_texture_test.argtypes = [C.POINTER(rb_texture), C.POINTER(rb_texture), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.rb_texture_test.restype = C.c_int
    if hasattr(lib, "rb_exact_record_count"):
        lib.rb_exact_record_count.argtypes = [C.c_void_p, C.POINTER(rb_options), C.POINTER(rb_dscene_desc), C.c_void_p, C.POINTER(C.c_size_t),
                                              C.POINTER(C.c_uint64)]
        lib.rb_exact_record_count.restype = C.c_int
        lib.rb_render_exact.argtypes = [C.c_void_p, C.POINTER(rb_options), C.c_void_p, C.POINTER(rb_dscene_desc), C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.c_void_p]
        lib.rb_render_exact.restype = C.c_int
        lib.rb_exact_round.argtypes = [C.c_void_p, C.POINTER(rb_options), C.POINTER(rb_dscene_desc), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        lib.rb_exact_round.restype = C.c_int
    lib.rb_last_error.argtypes = []
    lib.rb_last_error.restype = C.c_char_p
    lib.rb_version.argtypes = []
    lib.rb_version.restype = C.c_char_p
    return lib


_lib = None


def load(path=None):
    """Load (once) and return the bound library.  Raises OSError if it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise OSError("redner_b200: %s not found -- build it with `python -m redner_b200.build` "
                      "(there is no CPU or PyTorch fallback for the render path)" % p)
    lib = _bind(C.CDLL(p))
    if path is None:
        _lib = lib
    return lib


def last_error(lib=None):
    lib = lib or load()
    msg = lib.rb_last_error()
    return msg.decode() if msg else ""
