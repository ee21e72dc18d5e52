"""ctypes binding of the C ABI in include/bgs.h (libbgs.so).

This is the Python twin of the Rust `bgs_sys` binding shown in INTEGRATION.md: plain structs,
plain pointers, status codes.  There is NO fallback: if libbgs.so is missing or fails to load the
import raises, and if no CUDA device is usable `bgs_context_create` returns BGS_ECUDA.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbgs.so")

BGS_OK, BGS_NOT_READY, BGS_EINVAL, BGS_ECUDA, BGS_ENOMEM, BGS_ENCCL = range(6)
STATUS_NAMES = ["BGS_OK", "BGS_NOT_READY", "BGS_EINVAL", "BGS_ECUDA", "BGS_ENOMEM", "BGS_ENCCL"]

BGS_FORMAT_RGBA8_SRGB, BGS_FORMAT_RGBA16F, BGS_FORMAT_RGBA32F = 0, 1, 2
BGS_FLAG_SORT_ALL = 1
BGS_FLAG_ASYNC = 2
BGS_FLAG_NO_CHUNKS = 4
BGS_FLAG_CHUNKS = 8
BGS_FLAG_PREMULTIPLIED_OUT = 16
BGS_FLAG_BLEND_OVER_TARGET = 32
BGS_FLAG_VISUALIZE_BOUNDING_BOX = 64
BGS_ENTITY_VISUALIZE_BOUNDING_BOX = 1
BGS_SCENE_MAX_CLOUDS = 64
BGS_SELECT_REPLACE, BGS_SELECT_ADD = 0, 1
BGS_TRANSFORM_ALL, BGS_TRANSFORM_SELECTED = 0, 1
BGS_PICK_NONE = 0xFFFFFFFF


class bgs_view(C.Structure):
    _fields_ = [
        ("view_from_world", C.c_float * 16),
        ("clip_from_view", C.c_float * 16),
        ("clip_from_world", C.c_float * 16),
        ("world_position", C.c_float * 3),
        ("viewport", C.c_float * 4),
    ]


class bgs_cloud_uniform(C.Structure):
    _fields_ = [
        ("transform", C.c_float * 16),
        ("global_opacity", C.c_float),
        ("global_scale", C.c_float),
        ("color_space", C.c_uint32),
        ("time", C.c_float),
        ("aabb_min", C.c_float * 4),
        ("aabb_max", C.c_float * 4),
    ]


class bgs_settings(C.Structure):
    _fields_ = [
        ("gaussian_mode", C.c_uint32),
        ("rasterize_mode", C.c_uint32),
        ("aabb", C.c_uint32),
        ("opacity_adaptive_radius", C.c_uint32),
        ("draw_mode", C.c_uint32),
        ("radix_sort_depth_bits", C.c_uint32),
        ("flags", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class bgs_render_extras(C.Structure):
    _fields_ = [
        ("previous_clip_from_world", C.c_float * 16),
        ("delta_time", C.c_float),
        ("num_classes", C.c_uint32),
    ]


class bgs_scene_depth(C.Structure):
    """The scene's Depth32Float depth buffer a frame is depth-tested against (bgs_render_depth_test)."""
    _fields_ = [
        ("depth", C.c_void_p),
        ("pitch_bytes", C.c_uint64),
    ]


class bgs_time_window(C.Structure):
    """CloudSettings.time_start / time_stop of one entity of a bgs_render_scene_4d call."""
    _fields_ = [
        ("time_start", C.c_float),
        ("time_stop", C.c_float),
    ]


class bgs_entity_settings(C.Structure):
    """One entity's own CloudSettings in a bgs_render_entities call."""
    _fields_ = [
        ("gaussian_mode", C.c_uint32),
        ("rasterize_mode", C.c_uint32),
        ("aabb", C.c_uint32),
        ("opacity_adaptive_radius", C.c_uint32),
        ("draw_mode", C.c_uint32),
        ("num_classes", C.c_uint32),
        ("window", bgs_time_window),
    ]


class bgs_frame_stats(C.Structure):
    _fields_ = [
        ("n", C.c_uint32),
        ("n_visible", C.c_uint32),
        ("n_pairs", C.c_uint64),
        ("tiles_x", C.c_uint32),
        ("tiles_y", C.c_uint32),
        ("width", C.c_uint32),
        ("height", C.c_uint32),
        ("rounds", C.c_uint32),
        ("tiles_saturated", C.c_uint32),
    ]


class bgs_particle_behavior(C.Structure):
    """ParticleBehavior (src/morph/particle.rs:349-358), 64 B; the numpy twin is gaussian.PARTICLE_BEHAVIOR_DTYPE."""
    _fields_ = [
        ("indices", C.c_uint32 * 4),
        ("velocity", C.c_float * 4),
        ("acceleration", C.c_float * 4),
        ("jerk", C.c_float * 4),
    ]


class bgs_khr_accessor(C.Structure):
    """One KHR_gaussian_splatting attribute's accessor as bgs_cloud_upload_khr reads it (glTF component codes)."""
    _fields_ = [
        ("data", C.c_void_p),
        ("byte_stride", C.c_uint32),
        ("component_type", C.c_uint32),
        ("normalized", C.c_uint32),
        ("components", C.c_uint32),
    ]


class bgs_khr_primitive(C.Structure):
    """A KHR_gaussian_splatting primitive's accessors; sh[d*d + c] is coefficient c of degree d."""
    _fields_ = [
        ("n", C.c_uint32),
        ("position", bgs_khr_accessor),
        ("rotation", bgs_khr_accessor),
        ("scale", bgs_khr_accessor),
        ("opacity", bgs_khr_accessor),
        ("color_0", bgs_khr_accessor),
        ("sh", bgs_khr_accessor * 16),
        ("sh_degree", C.c_uint32),
    ]


class bgs_pick(C.Structure):
    """One pixel of a pick frame (bgs_render_entities_pick), 16 B; the numpy twin is PICK_DTYPE."""
    _fields_ = [("entity", C.c_uint32), ("index", C.c_uint32), ("weight", C.c_float), ("depth", C.c_float)]


PICK_DTYPE = np.dtype([("entity", "<u4"), ("index", "<u4"), ("weight", "<f4"), ("depth", "<f4")])


# every symbol include/bgs.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("bgs_context_create", C.c_int, [C.c_int, C.POINTER(_P)]),
    ("bgs_context_destroy", None, [_P]),
    ("bgs_cloud_upload_f32", C.c_int, [_P, C.c_uint32, _P, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_upload_f16", C.c_int, [_P, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_upload_f16_cov", C.c_int, [_P, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_upload_f32_sh", C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_upload_f16_sh", C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_upload_f16_cov_sh", C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_download_f32_sh", C.c_int, [_P, _P, _P, _P, _P, _P]),
    ("bgs_cloud_download_f16_sh", C.c_int, [_P, _P, _P, _P, _P]),
    ("bgs_cloud_sh_degree", C.c_int, [_P, C.POINTER(C.c_uint32)]),
    ("bgs_cloud_upload_khr", C.c_int, [_P, C.POINTER(bgs_khr_primitive), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(_P)]),
    ("bgs_cloud_destroy", None, [_P]),
    ("bgs_cloud_select_sparse", C.c_int, [_P, _P, C.c_float, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bgs_cloud_visibility_get", C.c_int, [_P, _P, _P]),
    ("bgs_cloud_visibility_set", C.c_int, [_P, _P, _P]),
    ("bgs_cloud_select_in_mesh", C.c_int, [_P, _P, _P, C.c_uint32, _P, C.c_uint32, _P, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("bgs_cloud_select_in_view", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_view), _P, C.c_int, C.c_uint32,
                                           C.POINTER(C.c_uint32)]),
    ("bgs_cloud_subset", C.c_int, [_P, _P, _P, C.c_uint32, C.POINTER(_P), C.POINTER(C.c_uint32)]),
    ("bgs_cloud_download_f32", C.c_int, [_P, _P, _P, _P, _P, _P]),
    ("bgs_cloud_download_f16", C.c_int, [_P, _P, _P, _P, _P]),
    ("bgs_cloud_upload_4d", C.c_int, [_P, C.c_uint32, _P, _P, _P, _P, _P, C.POINTER(_P)]),
    ("bgs_cloud_download_4d", C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    ("bgs_particles_create", C.c_int, [_P, _P, C.c_uint32, C.POINTER(_P)]),
    ("bgs_particles_get", C.c_int, [_P, _P, _P]),
    ("bgs_particles_destroy", None, [_P]),
    ("bgs_cloud_particles_step", C.c_int, [_P, _P, _P, C.c_float]),
    ("bgs_cloud_positions_get", C.c_int, [_P, _P, _P]),
    ("bgs_cloud_interpolate", C.c_int, [_P, _P, _P, _P, C.c_float, C.c_float, C.c_float]),
    ("bgs_cloud_transform", C.c_int, [_P, _P, _P, C.c_uint32]),
    ("bgs_cloud_bounds", C.c_int, [_P, _P, C.c_uint32, _P, _P, C.POINTER(C.c_uint32)]),
    ("bgs_render", C.c_int, [_P, _P, C.POINTER(bgs_view), C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_settings), _P,
                             C.c_uint32, C.c_int]),
    ("bgs_render_ex", C.c_int, [_P, _P, C.POINTER(bgs_view), C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_settings),
                                C.POINTER(bgs_render_extras), _P, C.c_uint32, C.c_int]),
    ("bgs_render_depth_test", C.c_int, [_P, _P, C.POINTER(bgs_view), C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_settings),
                                        C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int]),
    ("bgs_render_4d", C.c_int, [_P, _P, C.POINTER(bgs_view), C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_settings),
                                C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int, C.c_float,
                                C.c_float]),
    ("bgs_render_scene", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.c_uint32, C.POINTER(bgs_view), C.POINTER(bgs_settings),
                                   C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int]),
    ("bgs_render_scene_4d", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_time_window), C.c_uint32,
                                      C.POINTER(bgs_view), C.POINTER(bgs_settings), C.POINTER(bgs_render_extras),
                                      C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int]),
    ("bgs_render_entities", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), C.c_uint32,
                                      C.POINTER(bgs_view), C.POINTER(bgs_settings), C.POINTER(bgs_render_extras),
                                      C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int]),
    ("bgs_render_entities_ex", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), _P,
                                         C.c_uint32, C.POINTER(bgs_view), C.POINTER(bgs_settings),
                                         C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int]),
    ("bgs_render_entities_aux", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), _P,
                                          C.c_uint32, C.POINTER(bgs_view), C.POINTER(bgs_settings),
                                          C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, _P, _P, C.c_uint32,
                                          C.c_int]),
    ("bgs_render_entities_pick", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), _P,
                                           C.c_uint32, C.POINTER(bgs_view), C.POINTER(bgs_settings),
                                           C.POINTER(bgs_render_extras), C.POINTER(bgs_scene_depth), _P, C.c_uint32, C.c_int,
                                           _P]),
    ("bgs_render_views", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), _P, C.c_uint32,
                                   C.POINTER(bgs_view), C.c_uint32, C.POINTER(bgs_settings), C.POINTER(bgs_scene_depth), _P,
                                   C.c_uint32, C.c_int]),
    ("bgs_render_views_aux", C.c_int, [_P, _P, C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_entity_settings), _P, C.c_uint32,
                                       C.POINTER(bgs_view), C.c_uint32, C.POINTER(bgs_settings), C.POINTER(bgs_scene_depth), _P,
                                       _P, _P, C.c_uint32, C.c_int]),
    ("bgs_render_aux", C.c_int, [_P, _P, C.POINTER(bgs_view), C.POINTER(bgs_cloud_uniform), C.POINTER(bgs_settings), _P, _P, _P,
                                 C.c_uint32, C.c_int]),
    ("bgs_sync", C.c_int, [_P]),
    ("bgs_debug_sorted_entries", C.c_int, [_P, _P]),
    ("bgs_debug_tile_ranges", C.c_int, [_P, _P]),
    ("bgs_debug_tile_entries", C.c_int, [_P, _P, C.c_uint64]),
    ("bgs_debug_projected", C.c_int, [_P, _P, _P]),
    ("bgs_debug_splat_depths", C.c_int, [_P, _P]),
    ("bgs_frame_stats_get", C.c_int, [_P, C.POINTER(bgs_frame_stats)]),
    ("bgs_stage_times_us", C.c_int, [_P, C.POINTER(C.c_float * 6)]),
    ("bgs_last_error", C.c_char_p, [_P]),
    ("bgs_context_stream", _P, [_P]),
    ("bgs_context_copy_stream", _P, [_P]),
    ("bgs_frame_device_ptr", _P, [_P]),
    ("bgs_last_launch_count", C.c_uint32, [_P]),
    ("bgs_frame_export_create", C.c_int, [C.c_int, C.c_size_t, C.POINTER(_P), C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    ("bgs_frame_export_import", C.c_int, [C.c_int, C.c_int, C.c_size_t, C.POINTER(_P)]),
    ("bgs_frame_export_destroy", None, [_P]),
    ("bgs_nccl_unique_id", C.c_int, [_P]),
    ("bgs_nccl_comm_init", C.c_int, [_P, C.c_int, C.c_int, _P, C.POINTER(_P)]),
    ("bgs_nccl_comm_destroy", None, [_P]),
    ("bgs_gather_frames", C.c_int, [_P, _P, C.c_int, _P, _P, C.c_size_t]),
    ("bgs_peer_buffer_create", C.c_int, [C.c_int, C.c_size_t, C.POINTER(_P), _P]),
    ("bgs_peer_buffer_open", C.c_int, [C.c_int, _P, C.POINTER(_P)]),
    ("bgs_peer_buffer_release", None, [_P, C.c_int]),
    ("bgs_push_frame", C.c_int, [_P, _P, _P, C.c_int, C.c_size_t]),
    ("bgs_push_frame_signal", C.c_int, [_P, _P, _P, C.c_int, C.c_size_t, _P, C.c_uint32]),
    ("bgs_wait_frames", C.c_int, [_P, _P, C.c_int, C.c_uint32]),
]

_lib = None


def load() -> C.CDLL:
    """Load libbgs.so (built in-tree by `__graft_entry__.build()` / csrc/Makefile). Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build the CUDA extension first "
            "(python -c 'import __graft_entry__ as g; g.build()').  There is no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


class BgsError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS_NAMES[status] if 0 <= status < 6 else status}: {message}")
        self.status = status
