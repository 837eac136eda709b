"""ctypes mirror of include/trb.h (the C ABI) and loaders for the shared libraries.

The product library is ``tray_rust_b200/lib/libtrb.so`` (CUDA kernels + host code,
built by ``__graft_entry__.build()``). There is NO CPU fallback: if the library is
missing, ``load_trb()`` raises.

The parity oracle has its own bindings under ``oracle/pyoracle.py`` (test infrastructure);
nothing in this package imports, loads or links it.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(_HERE)

TRB_ABI_VERSION = 4
TRB_OK, TRB_INVALID_ARG, TRB_CUDA, TRB_OOM, TRB_UNSUPPORTED, TRB_IO, TRB_NO_DEVICE, TRB_NCCL = range(8)
INST_RECEIVER, INST_EMITTER_AREA, INST_EMITTER_POINT = 0, 1, 2
SHAPE_NONE, SHAPE_SPHERE, SHAPE_DISK, SHAPE_RECT, SHAPE_MESH = 0, 1, 2, 3, 4
MAT_MATTE, MAT_PLASTIC, MAT_METAL, MAT_SPECULAR_METAL, MAT_GLASS, MAT_ROUGH_GLASS, MAT_MERL = range(7)
FILTER_MITCHELL_NETRAVALI, FILTER_GAUSSIAN = 0, 1
INTEGRATOR_PATH, INTEGRATOR_WHITTED, INTEGRATOR_NORMALS_DEBUG = 0, 1, 2
RENDER_STATS, RENDER_NO_UPDATE, RENDER_REFERENCE_SHADOW, RENDER_MEGAKERNEL, RENDER_TIME_TRACE = 1, 2, 4, 8, 16
QUERY_CLAMP = 32  # trb_illumination: clamp each sample to [0, 1] before averaging
BXDF_REFLECTION, BXDF_TRANSMISSION, BXDF_DIFFUSE, BXDF_GLOSSY, BXDF_SPECULAR = 1, 2, 4, 8, 16  # bxdf::BxDFType
BXDF_ALL = 31
MISS = 0xFFFFFFFF
BVH_LEAF = 0x80000000
MERL_TABLE_FLOATS = 90 * 90 * 180 * 3

u32, f32 = C.c_uint32, C.c_float


class Keyframe(C.Structure):
    _fields_ = [("translation", f32 * 3), ("rotation", f32 * 4), ("scaling", f32 * 3)]


class Spline(C.Structure):
    _fields_ = [("degree", u32), ("n_ctrl", u32), ("ctrl_first", u32), ("n_knots", u32), ("knot_first", u32)]


class ColorKey(C.Structure):
    _fields_ = [("rgba", f32 * 4), ("time", f32)]


class Instance(C.Structure):
    _fields_ = [("kind", u32), ("shape", u32), ("p0", f32), ("p1", f32), ("mesh", u32), ("material", u32),
                ("spline_first", u32), ("n_splines", u32), ("emission_first", u32), ("n_emission", u32)]


class Mesh(C.Structure):
    _fields_ = [("n_verts", u32), ("n_tris", u32), ("positions", C.POINTER(f32)), ("normals", C.POINTER(f32)),
                ("texcoords", C.POINTER(f32)), ("indices", C.POINTER(u32))]


class Image(C.Structure):
    _fields_ = [("width", u32), ("height", u32), ("rgba8", C.POINTER(C.c_uint8)), ("time", f32), ("pad", u32)]


class Texture(C.Structure):
    _fields_ = [("first_image", u32), ("n_images", u32)]


class Material(C.Structure):
    _fields_ = [("type", u32), ("c0", f32 * 3), ("c1", f32 * 3), ("roughness", f32), ("eta", f32), ("merl", u32), ("tex", u32 * 4)]


class Camera(C.Structure):
    _fields_ = [("spline_first", u32), ("n_splines", u32), ("fov", f32), ("shutter_size", f32), ("active_at", u32),
                ("fov_degree", u32), ("n_fov_ctrl", u32), ("fov_ctrl_first", u32), ("n_fov_knots", u32),
                ("fov_knot_first", u32)]


class Film(C.Structure):
    _fields_ = [("width", u32), ("height", u32), ("samples", u32), ("frames", u32), ("start_frame", u32),
                ("end_frame", u32), ("scene_time", f32), ("filter_type", u32), ("filter_w", f32), ("filter_h", f32),
                ("filter_b", f32), ("filter_c", f32)]


class Integrator(C.Structure):
    _fields_ = [("type", u32), ("min_depth", u32), ("max_depth", u32)]


class SceneDesc(C.Structure):
    _fields_ = [("abi_version", u32), ("film", Film), ("integrator", Integrator),
                ("n_cameras", u32), ("cameras", C.POINTER(Camera)),
                ("n_instances", u32), ("instances", C.POINTER(Instance)),
                ("n_splines", u32), ("splines", C.POINTER(Spline)),
                ("n_keyframes", u32), ("keyframes", C.POINTER(Keyframe)),
                ("n_knots", u32), ("knots", C.POINTER(f32)),
                ("n_color_keys", u32), ("color_keys", C.POINTER(ColorKey)),
                ("n_meshes", u32), ("meshes", C.POINTER(Mesh)),
                ("n_materials", u32), ("materials", C.POINTER(Material)),
                ("n_merl", u32), ("merl_tables", C.POINTER(C.POINTER(f32))),
                ("n_fov_floats", u32), ("fov_floats", C.POINTER(f32)),
                ("n_textures", u32), ("textures", C.POINTER(Texture)),
                ("n_images", u32), ("images", C.POINTER(Image))]


class SceneObjects(C.Structure):
    """trb_scene_objects: the object section of a SceneDesc, with the same field names"""
    _fields_ = [("n_cameras", u32), ("cameras", C.POINTER(Camera)),
                ("n_instances", u32), ("instances", C.POINTER(Instance)),
                ("n_splines", u32), ("splines", C.POINTER(Spline)),
                ("n_keyframes", u32), ("keyframes", C.POINTER(Keyframe)),
                ("n_knots", u32), ("knots", C.POINTER(f32)),
                ("n_color_keys", u32), ("color_keys", C.POINTER(ColorKey)),
                ("n_fov_floats", u32), ("fov_floats", C.POINTER(f32))]


MESH_NEW = 0xFFFFFFFF


class SceneMeshes(C.Structure):
    """trb_scene_meshes: mesh i of the new list is the scene's current mesh keep[i], or meshes[i] where keep[i] is MESH_NEW"""
    _fields_ = [("n_meshes", u32), ("meshes", C.POINTER(Mesh)), ("keep", C.POINTER(u32))]


class SceneMaterials(C.Structure):
    """trb_scene_materials: the material section of a SceneDesc (materials, MERL tables, textures, images), with the same field names"""
    _fields_ = [("n_materials", u32), ("materials", C.POINTER(Material)),
                ("n_merl", u32), ("merl_tables", C.POINTER(C.POINTER(f32))),
                ("n_textures", u32), ("textures", C.POINTER(Texture)),
                ("n_images", u32), ("images", C.POINTER(Image))]


class RenderCfg(C.Structure):
    _fields_ = [("spp", u32), ("sample_first", u32), ("sample_count", u32), ("block_start", u32),
                ("block_count", u32), ("current_frame", u32), ("seed", u32), ("flags", u32),
                ("shard_index", u32), ("shard_count", u32), ("shard_chunk", u32)]


class Stats(C.Structure):
    _fields_ = [("camera_samples", C.c_uint64), ("rays_primary", C.c_uint64), ("rays_shadow", C.c_uint64),
                ("rays_mis", C.c_uint64), ("rays_continuation", C.c_uint64), ("node_tests", C.c_uint64),
                ("tri_tests", C.c_uint64), ("inst_tests", C.c_uint64), ("kernel_ms", f32), ("update_ms", f32)]

    def rays_total(self):
        return self.rays_primary + self.rays_shadow + self.rays_mis + self.rays_continuation

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Adaptive(C.Structure):
    _fields_ = [("min_spp", u32), ("max_spp", u32)]


class Ray(C.Structure):
    _fields_ = [("o", f32 * 3), ("d", f32 * 3), ("min_t", f32), ("max_t", f32)]


class Hit(C.Structure):
    _fields_ = [("t", f32), ("inst", u32), ("prim", u32), ("pad", u32)]


class QueryRay(C.Structure):
    _fields_ = [("o", f32 * 3), ("d", f32 * 3), ("min_t", f32), ("max_t", f32), ("time", f32), ("pad", u32 * 3)]


class Intersection(C.Structure):
    _fields_ = [("t", f32), ("inst", u32), ("prim", u32), ("material", u32), ("p", f32 * 3), ("n", f32 * 3), ("ng", f32 * 3),
                ("u", f32), ("v", f32), ("time", f32), ("dp_du", f32 * 3), ("dp_dv", f32 * 3), ("pad", u32 * 2)]


class IllumRay(C.Structure):
    _fields_ = [("o", f32 * 3), ("d", f32 * 3), ("min_t", f32), ("max_t", f32), ("time", f32), ("key", u32), ("sample", u32), ("pad", u32)]


class BsdfEvalQuery(C.Structure):
    _fields_ = [("wo", f32 * 3), ("bxdf", u32), ("wi", f32 * 3), ("pad", u32)]


class BsdfSampleQuery(C.Structure):
    _fields_ = [("wo", f32 * 3), ("bxdf", u32), ("u", f32 * 2), ("u_comp", f32), ("pad", u32)]


class BsdfSampleResult(C.Structure):
    _fields_ = [("f", f32 * 3), ("pdf", f32), ("wi", f32 * 3), ("sampled", u32)]


class LightQuery(C.Structure):
    _fields_ = [("p", f32 * 3), ("time", f32), ("u", f32 * 2), ("light", u32), ("pad", u32)]


class LightSampleResult(C.Structure):
    _fields_ = [("li", f32 * 3), ("pdf", f32), ("wi", f32 * 3), ("delta", u32), ("shadow", QueryRay)]


class LightPdfQuery(C.Structure):
    _fields_ = [("p", f32 * 3), ("time", f32), ("wi", f32 * 3), ("light", u32)]


class EmitQuery(C.Structure):
    _fields_ = [("w", f32 * 3), ("time", f32), ("n", f32 * 3), ("inst", u32)]


class Sample(C.Structure):
    _fields_ = [("x", f32), ("y", f32), ("r", f32), ("g", f32), ("b", f32)]


class AovFilm(C.Structure):
    """trb_aov_film: the AOV outputs of a film render (any may be NULL)"""
    _fields_ = [("albedo_w", C.c_void_p), ("normal_w", C.c_void_p), ("nearest", C.c_void_p)]


class DenoiseInput(C.Structure):
    """trb_denoise_input: the two half films, the albedo and normal films and the nearest buffer (all required)"""
    _fields_ = [("colour_a", C.c_void_p), ("colour_b", C.c_void_p), ("albedo_w", C.c_void_p), ("normal_w", C.c_void_p),
                ("nearest", C.c_void_p)]


class DenoiseParams(C.Structure):
    """trb_denoise_params (NULL: DENOISE_DEFAULTS)"""
    _fields_ = [("iterations", u32), ("normal_power", u32), ("sigma_luminance", f32), ("sigma_depth", f32)]


DENOISE_DEFAULTS = dict(iterations=5, normal_power=128, sigma_luminance=4.0, sigma_depth=1.0)


class DenoiseTemporalParams(C.Structure):
    """trb_denoise_temporal_params (NULL: DENOISE_DEFAULTS and DENOISE_TEMPORAL_DEFAULTS)"""
    _fields_ = [("spatial", DenoiseParams), ("max_history", u32), ("depth_tolerance", f32), ("normal_threshold", f32), ("pad", u32)]


class DenoiseTemporalOutput(C.Structure):
    """trb_denoise_temporal_output: rgbw (required), motion and history_length (may be NULL)"""
    _fields_ = [("rgbw", C.c_void_p), ("motion", C.c_void_p), ("history_length", C.c_void_p)]


DENOISE_TEMPORAL_DEFAULTS = dict(max_history=8, depth_tolerance=0.05, normal_threshold=0.9)


class DenoiseGradientParams(C.Structure):
    """trb_denoise_gradient_params (NULL: the temporal defaults and DENOISE_GRADIENT_DEFAULTS)"""
    _fields_ = [("temporal", DenoiseTemporalParams), ("iterations", u32), ("pad", u32 * 3)]


class DenoiseGradientOutput(C.Structure):
    """trb_denoise_gradient_output: rgbw (required), motion, history_length and lambda (may be NULL)"""
    _fields_ = [("rgbw", C.c_void_p), ("motion", C.c_void_p), ("history_length", C.c_void_p), ("lambda_", C.c_void_p)]


# Python name of trb_denoise_gradient_params.iterations: `iterations` already names the spatial filter's
DENOISE_GRADIENT_DEFAULTS = dict(gradient_iterations=3)


class DenoiseFrame(C.Structure):
    """trb_denoise_frame: one colour film at any spp, the albedo and normal films and the nearest buffer (all required)"""
    _fields_ = [("colour", C.c_void_p), ("albedo_w", C.c_void_p), ("normal_w", C.c_void_p), ("nearest", C.c_void_p)]


class DenoiseMomentsOutput(C.Structure):
    """trb_denoise_moments_output: rgbw (required), motion, history_length and variance (may be NULL)"""
    _fields_ = [("rgbw", C.c_void_p), ("motion", C.c_void_p), ("history_length", C.c_void_p), ("variance", C.c_void_p)]


class DenoiseMomentsGradientOutput(C.Structure):
    """trb_denoise_moments_gradient_output: rgbw (required), motion, history_length, variance and lambda (may be NULL)"""
    _fields_ = [("rgbw", C.c_void_p), ("motion", C.c_void_p), ("history_length", C.c_void_p), ("variance", C.c_void_p),
                ("lambda_", C.c_void_p)]


# include/trb.h "Moment denoising": the history length from which a pixel's own moments give its variance, and the spatial
# estimate's window radius (7x7)
DENOISE_MOMENTS_MIN_HISTORY = 4
DENOISE_MOMENTS_RADIUS = 3


class BvhNode(C.Structure):
    _fields_ = [("bmin", f32 * 3), ("bmax", f32 * 3), ("a", u32), ("b", u32)]


# numpy dtypes with identical layout
import numpy as np  # noqa: E402

RAY_DTYPE = np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("min_t", "<f4"), ("max_t", "<f4")])
HIT_DTYPE = np.dtype([("t", "<f4"), ("inst", "<u4"), ("prim", "<u4"), ("pad", "<u4")])
SAMPLE_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("r", "<f4"), ("g", "<f4"), ("b", "<f4")])
NODE_DTYPE = np.dtype([("bmin", "<f4", 3), ("bmax", "<f4", 3), ("a", "<u4"), ("b", "<u4")])
QUERY_RAY_DTYPE = np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("min_t", "<f4"), ("max_t", "<f4"), ("time", "<f4"), ("pad", "<u4", 3)])
INTERSECTION_DTYPE = np.dtype([("t", "<f4"), ("inst", "<u4"), ("prim", "<u4"), ("material", "<u4"), ("p", "<f4", 3), ("n", "<f4", 3),
                               ("ng", "<f4", 3), ("u", "<f4"), ("v", "<f4"), ("time", "<f4"), ("dp_du", "<f4", 3), ("dp_dv", "<f4", 3),
                               ("pad", "<u4", 2)])
ILLUM_RAY_DTYPE = np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("min_t", "<f4"), ("max_t", "<f4"), ("time", "<f4"), ("key", "<u4"),
                            ("sample", "<u4"), ("pad", "<u4")])
BSDF_EVAL_QUERY_DTYPE = np.dtype([("wo", "<f4", 3), ("bxdf", "<u4"), ("wi", "<f4", 3), ("pad", "<u4")])
BSDF_SAMPLE_QUERY_DTYPE = np.dtype([("wo", "<f4", 3), ("bxdf", "<u4"), ("u", "<f4", 2), ("u_comp", "<f4"), ("pad", "<u4")])
BSDF_SAMPLE_DTYPE = np.dtype([("f", "<f4", 3), ("pdf", "<f4"), ("wi", "<f4", 3), ("sampled", "<u4")])
LIGHT_QUERY_DTYPE = np.dtype([("p", "<f4", 3), ("time", "<f4"), ("u", "<f4", 2), ("light", "<u4"), ("pad", "<u4")])
LIGHT_SAMPLE_DTYPE = np.dtype([("li", "<f4", 3), ("pdf", "<f4"), ("wi", "<f4", 3), ("delta", "<u4"), ("shadow", QUERY_RAY_DTYPE)])
LIGHT_PDF_QUERY_DTYPE = np.dtype([("p", "<f4", 3), ("time", "<f4"), ("wi", "<f4", 3), ("light", "<u4")])
EMIT_QUERY_DTYPE = np.dtype([("w", "<f4", 3), ("time", "<f4"), ("n", "<f4", 3), ("inst", "<u4")])
KEYFRAME_DTYPE = np.dtype([("translation", "<f4", 3), ("rotation", "<f4", 4), ("scaling", "<f4", 3)])
COLOR_KEY_DTYPE = np.dtype([("rgba", "<f4", 4), ("time", "<f4")])
AOV_SAMPLE_DTYPE = np.dtype([("albedo", "<f4", 3), ("depth", "<f4"), ("n", "<f4", 3), ("inst", "<u4")])  # trb_aov_sample, 32 B
MOTION_SAMPLE_DTYPE = np.dtype([("dx", "<f4"), ("dy", "<f4"), ("valid", "<f4"), ("reserved", "<u4")])  # trb_motion_sample, 16 B
MATERIAL_DTYPE = np.dtype([("type", "<u4"), ("c0", "<f4", 3), ("c1", "<f4", 3), ("roughness", "<f4"), ("eta", "<f4"), ("merl", "<u4"),
                           ("tex", "<u4", 4)])

TRB_SYMBOLS = [
    "trb_scene_create", "trb_scene_load_json", "trb_scene_destroy", "trb_scene_info", "trb_scene_update_frame",
    "trb_render", "trb_render_device", "trb_intersect", "trb_intersect_device", "trb_camera_rays",
    "trb_render_samples", "trb_film_to_srgb8", "trb_block_list", "trb_scene_get_bvh", "trb_scene_get_transform",
    "trb_scene_get_filter_table", "trb_last_error", "trb_abi_version", "trb_desc_load_json", "trb_desc_free",
    "trb_host_build_bvh", "trb_host_keyframe_transform", "trb_host_animated_transform", "trb_host_animated_color", "trb_host_quad_check", "trb_selftest_box", "trb_launch_count", "trb_scene_trace_time", "trb_scene_check_error", "trb_scene_set_option", "trb_write_png",
    "trb_nccl_unique_id", "trb_comm_create", "trb_comm_destroy", "trb_comm_info", "trb_comm_reduce_film", "trb_render_sharded",
    "trb_group_create", "trb_group_load_json", "trb_group_render", "trb_group_scene", "trb_group_destroy",
    "trb_render_adaptive", "trb_render_samples_adaptive", "trb_adaptive_schedule", "trb_host_adaptive_decide",
    "trb_render_adaptive_device", "trb_render_sharded_adaptive", "trb_group_render_adaptive",
    "trb_intersect_records", "trb_intersect_records_device", "trb_occluded", "trb_occluded_device",
    "trb_illumination", "trb_illumination_device",
    "trb_bsdf_eval", "trb_bsdf_eval_device", "trb_bsdf_sample", "trb_bsdf_sample_device", "trb_light_sample", "trb_light_sample_device",
    "trb_light_pdf", "trb_light_pdf_device", "trb_emitted", "trb_emitted_device", "trb_scene_lights",
    "trb_film_write", "trb_film_write_device", "trb_camera_rays_device", "trb_host_film_to_srgb8",
    "trb_build_bvh", "trb_build_bvh_device",
    "trb_scene_update_mesh", "trb_scene_update_mesh_device", "trb_scene_refit_mesh", "trb_scene_refit_mesh_device",
    "trb_scene_update_keyframes", "trb_scene_update_keyframes_device", "trb_scene_update_color_keys", "trb_scene_update_materials",
    "trb_scene_replace_objects", "trb_scene_replace_meshes", "trb_scene_replace_meshes_device",
    "trb_scene_replace_settings", "trb_scene_replace_materials", "trb_scene_replace_materials_device",
    "trb_render_aov", "trb_render_aov_device", "trb_render_samples_aov",
    "trb_denoise", "trb_denoise_device",
    "trb_denoise_history_create", "trb_denoise_history_destroy", "trb_denoise_history_reset", "trb_denoise_temporal",
    "trb_denoise_temporal_device", "trb_denoise_temporal_gradient", "trb_denoise_temporal_gradient_device",
    "trb_denoise_moments", "trb_denoise_moments_device", "trb_denoise_moments_gradient", "trb_denoise_moments_gradient_device",
    "trb_render_adaptive_aov", "trb_render_adaptive_aov_device", "trb_render_samples_adaptive_aov",
    "trb_render_sharded_aov", "trb_render_sharded_adaptive_aov", "trb_group_render_aov", "trb_group_render_adaptive_aov",
    "trb_render_aov_lum", "trb_render_aov_lum_device", "trb_render_adaptive_aov_lum", "trb_render_adaptive_aov_lum_device",
    "trb_denoise_variance", "trb_denoise_variance_device",
    "trb_render_aov_motion", "trb_render_aov_motion_device", "trb_render_adaptive_aov_motion", "trb_render_adaptive_aov_motion_device",
    "trb_render_samples_aov_motion",
    "trb_denoise_variance_temporal", "trb_denoise_variance_temporal_device", "trb_denoise_variance_temporal_gradient",
    "trb_denoise_variance_temporal_gradient_device",
]

_trb = None


def trb_path():
    return os.path.join(_HERE, "lib", "libtrb.so")


def load_trb():
    """Load the product library. Raises if it has not been built — never falls back."""
    global _trb
    if _trb is not None:
        return _trb
    p = trb_path()
    if not os.path.exists(p):
        raise RuntimeError("libtrb.so is missing (%s): run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "tray_rust_b200 has no CPU fallback." % p)
    lib = C.CDLL(p)
    vp, sz = C.c_void_p, C.c_size_t
    lib.trb_last_error.restype = C.c_char_p
    lib.trb_abi_version.restype = u32
    lib.trb_scene_create.argtypes = [C.POINTER(SceneDesc), C.c_int, C.POINTER(vp)]
    lib.trb_scene_load_json.argtypes = [C.c_char_p, u32, u32, u32, C.c_int, C.POINTER(vp)]
    lib.trb_scene_destroy.argtypes = [vp]
    lib.trb_scene_destroy.restype = None
    lib.trb_scene_info.argtypes = [vp] + [C.POINTER(u32)] * 6
    lib.trb_scene_update_frame.argtypes = [vp, u32, f32, f32]
    lib.trb_scene_update_mesh.argtypes = [vp, u32, vp, vp, vp]
    lib.trb_scene_update_mesh_device.argtypes = [vp, u32, vp, vp, vp, vp]
    lib.trb_scene_refit_mesh.argtypes = [vp, u32, vp, vp, vp]
    lib.trb_scene_refit_mesh_device.argtypes = [vp, u32, vp, vp, vp, vp]
    lib.trb_scene_update_keyframes.argtypes = [vp, u32, u32, vp]
    lib.trb_scene_update_keyframes_device.argtypes = [vp, u32, u32, vp, vp]
    lib.trb_scene_update_color_keys.argtypes = [vp, u32, u32, vp]
    lib.trb_scene_update_materials.argtypes = [vp, u32, u32, vp]
    lib.trb_scene_replace_objects.argtypes = [vp, C.POINTER(SceneObjects)]
    lib.trb_scene_replace_meshes.argtypes = [vp, C.POINTER(SceneMeshes), C.POINTER(SceneObjects)]
    lib.trb_scene_replace_meshes_device.argtypes = [vp, C.POINTER(SceneMeshes), C.POINTER(SceneObjects), vp]
    lib.trb_scene_replace_settings.argtypes = [vp, C.POINTER(Film), C.POINTER(Integrator)]
    lib.trb_scene_replace_materials.argtypes = [vp, C.POINTER(SceneMaterials), C.POINTER(SceneObjects)]
    lib.trb_scene_replace_materials_device.argtypes = [vp, C.POINTER(SceneMaterials), C.POINTER(SceneObjects), vp]
    lib.trb_render.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(Stats)]
    lib.trb_render_device.argtypes = [vp, C.POINTER(RenderCfg), vp, vp, vp]
    lib.trb_intersect.argtypes = [vp, sz, vp, vp, C.POINTER(Stats)]
    lib.trb_intersect_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.trb_intersect_records.argtypes = [vp, sz, vp, vp, u32, C.POINTER(Stats)]
    lib.trb_intersect_records_device.argtypes = [vp, sz, vp, vp, u32, vp, vp]
    lib.trb_occluded.argtypes = [vp, sz, vp, vp, u32, C.POINTER(Stats)]
    lib.trb_occluded_device.argtypes = [vp, sz, vp, vp, u32, vp, vp]
    lib.trb_illumination.argtypes = [vp, sz, vp, u32, u32, vp, u32, C.POINTER(Stats)]
    lib.trb_illumination_device.argtypes = [vp, sz, vp, u32, u32, vp, u32, vp, vp]
    lib.trb_bsdf_eval.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_bsdf_eval_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.trb_bsdf_sample.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_bsdf_sample_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.trb_light_sample.argtypes = [vp, sz, vp, vp]
    lib.trb_light_sample_device.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_light_pdf.argtypes = [vp, sz, vp, vp]
    lib.trb_light_pdf_device.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_emitted.argtypes = [vp, sz, vp, vp]
    lib.trb_emitted_device.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_scene_lights.argtypes = [vp, vp]
    lib.trb_camera_rays.argtypes = [vp, C.POINTER(RenderCfg), sz, vp, vp]
    lib.trb_camera_rays_device.argtypes = [vp, C.POINTER(RenderCfg), sz, vp, vp, vp]
    lib.trb_film_write.argtypes = [vp, sz, vp, vp, vp]
    lib.trb_film_write_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.trb_render_samples.argtypes = [vp, C.POINTER(RenderCfg), sz, vp, C.POINTER(Stats)]
    lib.trb_render_aov.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), C.POINTER(Stats)]
    lib.trb_render_aov_device.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), vp, vp]
    lib.trb_render_samples_aov.argtypes = [vp, C.POINTER(RenderCfg), sz, vp, vp, C.POINTER(Stats)]
    lib.trb_denoise.argtypes = [vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseParams), vp]
    lib.trb_denoise_device.argtypes = [vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseParams), vp, vp]
    lib.trb_denoise_history_create.argtypes = [vp, C.POINTER(vp)]
    lib.trb_denoise_history_destroy.argtypes = [vp]
    lib.trb_denoise_history_reset.argtypes = [vp]
    lib.trb_denoise_temporal.argtypes = [vp, vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseTemporalParams), C.POINTER(DenoiseTemporalOutput)]
    lib.trb_denoise_temporal_device.argtypes = [vp, vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseTemporalParams),
                                                C.POINTER(DenoiseTemporalOutput), vp]
    lib.trb_denoise_temporal_gradient.argtypes = [vp, vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseGradientParams), u32,
                                                  C.POINTER(DenoiseGradientOutput)]
    lib.trb_denoise_temporal_gradient_device.argtypes = [vp, vp, C.POINTER(DenoiseInput), C.POINTER(DenoiseGradientParams), u32,
                                                         C.POINTER(DenoiseGradientOutput), vp]
    lib.trb_denoise_moments.argtypes = [vp, vp, C.POINTER(DenoiseFrame), C.POINTER(DenoiseTemporalParams), C.POINTER(DenoiseMomentsOutput)]
    lib.trb_denoise_moments_device.argtypes = [vp, vp, C.POINTER(DenoiseFrame), C.POINTER(DenoiseTemporalParams),
                                               C.POINTER(DenoiseMomentsOutput), vp]
    lib.trb_denoise_moments_gradient.argtypes = [vp, vp, C.POINTER(DenoiseFrame), C.POINTER(DenoiseGradientParams), u32,
                                                 C.POINTER(DenoiseMomentsGradientOutput)]
    lib.trb_denoise_moments_gradient_device.argtypes = [vp, vp, C.POINTER(DenoiseFrame), C.POINTER(DenoiseGradientParams), u32,
                                                        C.POINTER(DenoiseMomentsGradientOutput), vp]
    lib.trb_render_adaptive.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, vp, C.POINTER(Stats)]
    lib.trb_render_samples_adaptive.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), sz, vp, vp, C.POINTER(Stats)]
    lib.trb_render_adaptive_device.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, vp, vp, vp]
    lib.trb_render_adaptive_aov.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, C.POINTER(Stats)]
    lib.trb_render_adaptive_aov_device.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, vp, vp]
    lib.trb_render_samples_adaptive_aov.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), sz, vp, vp, vp, C.POINTER(Stats)]
    lib.trb_render_aov_lum.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), vp, C.POINTER(Stats)]
    lib.trb_render_aov_lum_device.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), vp, vp, vp]
    lib.trb_render_adaptive_aov_lum.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, vp, C.POINTER(Stats)]
    lib.trb_render_adaptive_aov_lum_device.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, vp, vp, vp]
    lib.trb_render_aov_motion.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), vp, vp, f32, C.POINTER(Stats)]
    lib.trb_render_aov_motion_device.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), vp, vp, f32, vp, vp]
    lib.trb_render_adaptive_aov_motion.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, vp, f32, vp,
                                                   C.POINTER(Stats)]
    lib.trb_render_adaptive_aov_motion_device.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, vp, f32, vp,
                                                          vp, vp]
    lib.trb_render_samples_aov_motion.argtypes = [vp, C.POINTER(RenderCfg), sz, vp, vp, vp, f32, C.POINTER(Stats)]
    lib.trb_denoise_variance.argtypes = [vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseParams), vp, vp]
    lib.trb_denoise_variance_device.argtypes = [vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseParams), vp, vp, vp]
    lib.trb_denoise_variance_temporal.argtypes = [vp, vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseTemporalParams),
                                                  C.POINTER(DenoiseMomentsOutput)]
    lib.trb_denoise_variance_temporal_device.argtypes = [vp, vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseTemporalParams),
                                                         C.POINTER(DenoiseMomentsOutput), vp]
    lib.trb_denoise_variance_temporal_gradient.argtypes = [vp, vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseGradientParams), u32,
                                                           C.POINTER(DenoiseMomentsGradientOutput)]
    lib.trb_denoise_variance_temporal_gradient_device.argtypes = [vp, vp, C.POINTER(DenoiseFrame), vp, C.POINTER(DenoiseGradientParams), u32,
                                                                  C.POINTER(DenoiseMomentsGradientOutput), vp]
    lib.trb_adaptive_schedule.argtypes = [C.POINTER(Adaptive)] + [C.POINTER(u32)] * 4
    lib.trb_host_adaptive_decide.argtypes = [C.POINTER(Adaptive), vp, sz, C.POINTER(u32), C.POINTER(f32)]
    lib.trb_film_to_srgb8.argtypes = [vp, vp, vp]
    lib.trb_host_film_to_srgb8.argtypes = [u32, u32, vp, vp]
    lib.trb_block_list.argtypes = [vp, u32, u32, C.POINTER(u32), vp, u32]
    lib.trb_scene_get_bvh.argtypes = [vp, C.c_int, C.POINTER(u32), vp, C.POINTER(u32), vp]
    lib.trb_scene_get_transform.argtypes = [vp, u32, vp, vp]
    lib.trb_scene_get_filter_table.argtypes = [vp, vp]
    lib.trb_desc_load_json.argtypes = [C.c_char_p, u32, u32, u32, C.POINTER(C.POINTER(SceneDesc))]
    lib.trb_desc_free.argtypes = [C.POINTER(SceneDesc)]
    lib.trb_desc_free.restype = None
    lib.trb_host_build_bvh.argtypes = [vp, u32, u32, C.POINTER(u32), vp, vp]
    lib.trb_build_bvh.argtypes = [C.c_int, vp, u32, u32, C.POINTER(u32), vp, vp]
    lib.trb_build_bvh_device.argtypes = [C.c_int, vp, u32, u32, vp, vp, vp, vp]
    lib.trb_host_keyframe_transform.argtypes = [C.POINTER(Keyframe), vp, vp]
    lib.trb_host_animated_transform.argtypes = [C.POINTER(SceneDesc), u32, u32, f32, vp, vp]
    lib.trb_host_animated_color.argtypes = [C.POINTER(SceneDesc), u32, u32, f32, vp]
    lib.trb_host_quad_check.argtypes = [vp, u32, vp, u32, C.POINTER(u32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.trb_selftest_box.argtypes = [u32, u32, C.POINTER(C.c_uint64)]
    lib.trb_launch_count.restype = C.c_uint64
    lib.trb_scene_trace_time.argtypes = [vp, C.POINTER(f32), C.POINTER(u32)]
    lib.trb_write_png.argtypes = [C.c_char_p, vp, u32, u32]
    lib.trb_scene_check_error.argtypes = [vp]
    lib.trb_scene_set_option.argtypes = [vp, C.c_char_p, C.c_longlong]
    lib.trb_nccl_unique_id.argtypes = [vp]
    lib.trb_comm_create.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    lib.trb_comm_destroy.argtypes = [vp]
    lib.trb_comm_destroy.restype = None
    lib.trb_comm_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.trb_comm_reduce_film.argtypes = [vp, vp, sz, C.c_int, vp]
    lib.trb_render_sharded.argtypes = [vp, vp, C.POINTER(RenderCfg), C.c_int, vp, C.POINTER(Stats)]
    lib.trb_group_create.argtypes = [C.POINTER(SceneDesc), C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    lib.trb_group_load_json.argtypes = [C.c_char_p, u32, u32, u32, C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    lib.trb_group_render.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(Stats)]
    lib.trb_render_sharded_adaptive.argtypes = [vp, vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), C.c_int, vp, vp, C.POINTER(Stats)]
    lib.trb_group_render_adaptive.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, vp, C.POINTER(Stats)]
    lib.trb_render_sharded_aov.argtypes = [vp, vp, C.POINTER(RenderCfg), C.c_int, vp, C.POINTER(AovFilm), C.POINTER(Stats)]
    lib.trb_render_sharded_adaptive_aov.argtypes = [vp, vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), C.c_int, vp, C.POINTER(AovFilm), vp,
                                                    C.POINTER(Stats)]
    lib.trb_group_render_aov.argtypes = [vp, C.POINTER(RenderCfg), vp, C.POINTER(AovFilm), C.POINTER(Stats)]
    lib.trb_group_render_adaptive_aov.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(Adaptive), vp, C.POINTER(AovFilm), vp, C.POINTER(Stats)]
    lib.trb_group_scene.argtypes = [vp, C.c_int]
    lib.trb_group_scene.restype = vp
    lib.trb_group_destroy.argtypes = [vp]
    lib.trb_group_destroy.restype = None
    _trb = lib
    return lib


def ptr(a):
    """void* of a contiguous numpy array"""
    return a.ctypes.data_as(C.c_void_p)
