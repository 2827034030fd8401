"""ctypes mirror of include/b200pt.h (the C ABI of the hot path).

Field order and types must match the header exactly; tests/test_abi.py checks
the struct sizes against the compiled library.
"""
import ctypes as C

import numpy as np

MAT_MATTE, MAT_PLASTIC, MAT_METAL, MAT_GLASS = 0, 1, 2, 3
LIGHTS_UNIFORM, LIGHTS_POWER, LIGHTS_SPATIAL = 0, 1, 2


class Material(C.Structure):
    _fields_ = [("type", C.c_int32), ("kd", C.c_float * 3), ("ks", C.c_float * 3),
                ("kt", C.c_float * 3), ("eta", C.c_float * 3), ("k", C.c_float * 3),
                ("alpha_x", C.c_float), ("alpha_y", C.c_float), ("index", C.c_float), ("variant", C.c_int32)]


class AreaLight(C.Structure):
    _fields_ = [("triangle", C.c_int32), ("lemit", C.c_float * 3), ("two_sided", C.c_int32),
                ("sphere", C.c_int32), ("kind", C.c_int32), ("position", C.c_float * 3),
                ("cos_total_width", C.c_float), ("cos_falloff_start", C.c_float), ("world_to_light", C.c_float * 16),
                ("world_radius", C.c_float)]


class Sphere(C.Structure):
    _fields_ = [("object_to_world", C.c_float * 16), ("world_to_object", C.c_float * 16),
                ("radius", C.c_float), ("material_id", C.c_int32), ("light_id", C.c_int32),
                ("reverse_orientation", C.c_uint8), ("transform_swaps_handedness", C.c_uint8),
                ("pad", C.c_uint8 * 2), ("leaf_bounds", C.c_float * 6),
                ("z_min", C.c_float), ("z_max", C.c_float), ("theta_min", C.c_float), ("theta_max", C.c_float),
                ("phi_max", C.c_float)]


class Instance(C.Structure):
    _fields_ = [("first_triangle", C.c_int64), ("n_triangles", C.c_int64), ("instance_to_world", C.c_float * 16),
                ("world_to_instance", C.c_float * 16), ("is_identity", C.c_int32), ("leaf_bounds", C.c_float * 6),
                ("pad", C.c_int32)]


class SceneDesc(C.Structure):
    _fields_ = [("n_triangles", C.c_int64), ("vertices", C.c_void_p), ("material_id", C.c_void_p),
                ("light_id", C.c_void_p), ("flip_normal", C.c_void_p), ("n_materials", C.c_int32),
                ("materials", C.POINTER(Material)), ("n_lights", C.c_int32),
                ("lights", C.POINTER(AreaLight)), ("normals", C.c_void_p), ("uvs", C.c_void_p),
                ("vertex_flags", C.c_void_p), ("n_spheres", C.c_int32), ("spheres", C.POINTER(Sphere)),
                ("n_instances", C.c_int32), ("instances", C.POINTER(Instance)), ("n_toplevel_triangles", C.c_int64),
                ("n_spectrum_samples", C.c_int32), ("reserved_spectral", C.c_int32), ("material_spectra", C.c_void_p),
                ("light_spectra", C.c_void_p), ("cie_xyz", C.c_void_p)]


class CameraDesc(C.Structure):
    _fields_ = [("raster_to_camera", C.c_float * 16), ("camera_to_world", C.c_float * 16),
                ("lens_radius", C.c_float), ("focal_distance", C.c_float),
                ("shutter_open", C.c_float), ("shutter_close", C.c_float)]


class FilmDesc(C.Structure):
    _fields_ = [("full_resolution", C.c_int32 * 2), ("cropped_bounds", C.c_int32 * 4),
                ("filter_radius", C.c_float * 2), ("scale", C.c_float),
                ("max_sample_luminance", C.c_float), ("filter_table", C.c_void_p)]


SAMPLER_SOBOL, SAMPLER_HALTON = 0, 1
SPECTRUM_SAMPLES, MATERIAL_SPECTRA = 60, 5  # B200PT_SPECTRUM_SAMPLES, B200PT_MATERIAL_SPECTRA
LIGHT_AREA, LIGHT_POINT, LIGHT_SPOT, LIGHT_DISTANT, LIGHT_INFINITE = 0, 1, 2, 3, 4


class InfiniteLight(C.Structure):
    """b200pt_infinite_light: level 0 of an InfiniteAreaLight's map and its Distribution2D tables."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("texels", C.c_void_p), ("light_to_world", C.c_float * 16),
                ("nu", C.c_int32), ("nv", C.c_int32), ("cond_func", C.c_void_p), ("cond_cdf", C.c_void_p),
                ("cond_func_int", C.c_void_p), ("marg_func", C.c_void_p), ("marg_cdf", C.c_void_p),
                ("marg_func_int", C.c_float), ("power_rgb", C.c_float * 3)]


WRAP_REPEAT, WRAP_BLACK, WRAP_CLAMP = 0, 1, 2  # B200PT_WRAP_*
MIPMAP_MAX_LEVELS = 16
TEX_KD, TEX_KS, TEX_KT, TEX_ETA, TEX_K, TEX_ROUGHNESS_U, TEX_ROUGHNESS_V, TEX_SLOTS = range(8)


class Mipmap(C.Structure):
    """b200pt_mipmap: an ImageTexture's MIPMap as the host built it (every level, wrap, filter settings, weightLut)."""
    _fields_ = [("n_levels", C.c_int32), ("channels", C.c_int32), ("width", C.c_int32 * MIPMAP_MAX_LEVELS),
                ("height", C.c_int32 * MIPMAP_MAX_LEVELS), ("texels", C.c_void_p * MIPMAP_MAX_LEVELS), ("wrap", C.c_int32),
                ("trilinear", C.c_int32), ("max_anisotropy", C.c_float), ("weight_lut", C.c_float * 128)]


class AlphaMask(C.Structure):
    """b200pt_alpha_mask: level 0 of an alpha / shadowalpha mask's MIPMap under UVMapping2D (0 x 0, no texels: constant 0)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("texels", C.c_void_p), ("wrap", C.c_int32),
                ("su", C.c_float), ("sv", C.c_float), ("du", C.c_float), ("dv", C.c_float)]


class SamplerDesc(C.Structure):
    _fields_ = [("samples_per_pixel", C.c_int32), ("sample_bounds", C.c_int32 * 4),
                ("n_dimensions", C.c_int32), ("matrices32", C.c_void_p), ("vdc", C.c_void_p),
                ("vdc_inv", C.c_void_p), ("type", C.c_int32), ("reserved", C.c_int32),
                ("halton_permutations", C.c_void_p)]


class Medium(C.Structure):
    _fields_ = [("present", C.c_int32), ("sigma_a", C.c_float * 3), ("sigma_s", C.c_float * 3), ("g", C.c_float),
                ("spectra", C.c_void_p)]


class IntegratorDesc(C.Structure):
    _fields_ = [("max_depth", C.c_int32), ("rr_threshold", C.c_float), ("light_strategy", C.c_int32),
                ("pixel_bounds", C.c_int32 * 4), ("volumetric", C.c_int32), ("medium", Medium),
                ("n_bounded_media", C.c_int32), ("reserved", C.c_int32), ("bounded_media", C.c_void_p),
                ("sphere_medium", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [("camera_rays", C.c_uint64), ("regular_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
                ("nodes_visited", C.c_uint64), ("tris_tested", C.c_uint64), ("any_nodes_visited", C.c_uint64),
                ("any_tris_tested", C.c_uint64), ("closest_ms", C.c_double),
                ("any_ms", C.c_double), ("shade_ms", C.c_double), ("launches", C.c_uint64),
                ("closest_launches", C.c_uint64), ("any_launches", C.c_uint64), ("stack_overflows", C.c_uint64),
                ("dimension_overflows", C.c_uint64)]


RAY_DTYPE = np.dtype([("o", np.float32, 3), ("t_max", np.float32), ("d", np.float32, 3),
                      ("pad", np.float32)])
HIT_DTYPE = np.dtype([("triangle", np.int32), ("t", np.float32), ("b0", np.float32), ("b1", np.float32)])


def ptr(a):
    """void* of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)
