"""ctypes binding of libaclb200.so (include/aclb200.h). No decode logic lives here."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("ACLB200_LIB", os.path.join(_HERE, "libaclb200.so"))

ROUND_NONE, ROUND_FLOOR, ROUND_CEIL, ROUND_NEAREST, ROUND_PER_TRACK = 0, 1, 2, 3, 4
LOOP_CLAMP, LOOP_WRAP, LOOP_AS_COMPRESSED = 0, 1, 2
NORMALIZE_NEVER, NORMALIZE_LERP_ONLY, NORMALIZE_ALWAYS = 0, 1, 2
DEFAULT_SKIPPED, DEFAULT_CONSTANT, DEFAULT_VARIABLE, DEFAULT_LEGACY = 0, 1, 2, 3
LAYOUT_QVV48, LAYOUT_QVV40 = 0, 1
MATH_EXACT, MATH_FAST = 0, 1
SKIP_ROTATION, SKIP_TRANSLATION, SKIP_SCALE = 1, 2, 4
TRACK_QVVF = 12
TIER_MEDIUM, TIER_LOW = 1, 2

# numpy view of aclb200_request {uint32 clip; float sample_time}
REQUEST_DTYPE = np.dtype([("clip", np.uint32), ("sample_time", np.float32)])
SEEK_STATE_DTYPE = np.dtype([
    ("sample_time", np.float32), ("interpolation_alpha", np.float32),
    ("key_frame_bit_offsets", np.uint32, 2), ("segment_indices", np.uint32, 2), ("animated_offsets", np.uint32, 2),
    ("format_offsets", np.uint32, 2), ("range_offsets", np.uint32, 2),
    ("uses_single_segment", np.uint32), ("looping_policy", np.uint32),
])


# numpy views of aclb200_error_job / aclb200_track_error
ERROR_JOB_DTYPE = np.dtype([("clip", np.uint32), ("num_samples", np.uint32), ("sample_rate", np.float32), ("duration", np.float32),
                            ("num_tracks", np.uint32), ("skeleton_offset", np.uint32), ("first_raw_pose", np.uint64),
                            ("additive_format", np.uint32), ("error_metric", np.uint32), ("first_base_pose", np.uint64)])
METRIC_QVVF, METRIC_QVVF_MATRIX3X4F = 0, 1
ADDITIVE_NONE, ADDITIVE_RELATIVE, ADDITIVE_ADDITIVE0, ADDITIVE_ADDITIVE1 = 0, 1, 2, 3
TRACK_ERROR_DTYPE = np.dtype([("index", np.uint32), ("error", np.float32), ("sample_time", np.float32), ("flags", np.uint32)])
ERROR_FLAG_NEGATIVE_SCALE, ERROR_FLAG_INVALID_SKELETON, ERROR_FLAG_WRAP_CLIP_CYCLE = 1, 2, 4
OBJECT_QVVF, OBJECT_MATRIX3X4F = 0, 1


class AclB200Error(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"aclb200 status {status}: {message}")
        self.status = status


class Options(C.Structure):
    """aclb200_options"""
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("rounding_policy", C.c_uint32), ("looping_policy", C.c_uint32),
        ("normalization", C.c_uint32), ("per_track_rounding", C.c_uint32), ("wrapping", C.c_uint32),
        ("clamp_sample_time", C.c_uint32), ("multiple_rotation_formats", C.c_uint32),
        ("default_rotation_mode", C.c_uint32), ("default_translation_mode", C.c_uint32), ("default_scale_mode", C.c_uint32),
        ("constant_defaults", C.c_float * 12),
        ("d_variable_defaults", C.c_void_p), ("d_per_track_rounding", C.c_void_p),
        ("output_layout", C.c_uint32), ("math_mode", C.c_uint32),
        ("pose_stride_bytes", C.c_uint64),
        ("skip_mask", C.c_uint32), ("d_skip_track_mask", C.c_void_p), ("d_request_policies", C.c_void_p),
    ]

    def __init__(self, **kw):
        super().__init__()
        _lib().aclb200_default_options(C.byref(self))
        for key, value in kw.items():
            if key == "constant_defaults":
                for i, v in enumerate(np.asarray(value, dtype=np.float32).reshape(12)):
                    self.constant_defaults[i] = float(v)
            elif key == "default_modes":
                self.default_rotation_mode, self.default_translation_mode, self.default_scale_mode = value
            else:
                if not hasattr(self, key):
                    raise AttributeError(key)
                setattr(self, key, value)

    @property
    def bone_bytes(self) -> int:
        return 48 if self.output_layout == LAYOUT_QVV48 else 40


class _ClipsetInfo(C.Structure):
    _fields_ = [("num_clips", C.c_uint32), ("track_type", C.c_uint32), ("max_tracks", C.c_uint32), ("min_tracks", C.c_uint32),
                ("blob_bytes", C.c_uint64), ("index_bytes", C.c_uint64)]


class _DatabaseInfo(C.Structure):
    _fields_ = [("num_chunks", C.c_uint32 * 2), ("bulk_data_size", C.c_uint32 * 2), ("max_chunk_size", C.c_uint32), ("num_clips", C.c_uint32),
                ("num_segments", C.c_uint32), ("is_bulk_data_inline", C.c_uint32), ("hash", C.c_uint32), ("size", C.c_uint32)]


KERNEL_NONE, KERNEL_PLAIN, KERNEL_PIPELINE, KERNEL_DATABASE = 0, 1, 2, 3


class LaunchInfo(C.Structure):
    """aclb200_launch_info: the kernel and plan of a context's latest decompress_tracks."""
    _fields_ = [("kernel", C.c_uint32), ("requests_per_block", C.c_uint32), ("grid_blocks", C.c_uint32), ("num_batches", C.c_uint32),
                ("out_bulk", C.c_uint32), ("num_requests", C.c_uint32)]

    @property
    def kernel_name(self) -> str:
        return {KERNEL_NONE: "none", KERNEL_PLAIN: "plain", KERNEL_PIPELINE: "pipeline", KERNEL_DATABASE: "database"}[self.kernel]

    def __repr__(self) -> str:
        return (f"LaunchInfo(kernel={self.kernel_name}, rpb={self.requests_per_block}, grid={self.grid_blocks}, "
                f"batches={self.num_batches}, out_bulk={self.out_bulk}, requests={self.num_requests})")


class _ClipInfo(C.Structure):
    _fields_ = [("num_tracks", C.c_uint32), ("num_samples", C.c_uint32), ("sample_rate", C.c_float), ("duration", C.c_float),
                ("num_segments", C.c_uint32), ("looping_policy", C.c_uint32), ("hash", C.c_uint32), ("size", C.c_uint32)]


_lib_handle = None


def library_path() -> str:
    return _LIB_PATH


def _lib():
    global _lib_handle
    if _lib_handle is None:
        if not os.path.exists(_LIB_PATH):
            raise ImportError(f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(acl_b200/csrc/build.sh). There is no CPU fallback.")
        l = C.CDLL(_LIB_PATH)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        l.aclb200_version_string.restype = C.c_char_p
        l.aclb200_status_string.restype = C.c_char_p
        l.aclb200_status_string.argtypes = [C.c_int]
        l.aclb200_default_options.argtypes = [C.POINTER(Options)]
        l.aclb200_create.argtypes = [C.c_int, C.POINTER(vp)]
        l.aclb200_destroy.argtypes = [vp]
        l.aclb200_last_error.argtypes = [vp]
        l.aclb200_last_error.restype = C.c_char_p
        l.aclb200_upload_clips.argtypes = [vp, vp, vp, u32, u32, C.POINTER(vp), C.POINTER(u32)]
        l.aclb200_upload_clips_packed.argtypes = [vp, vp, vp, vp, u32, u32, C.POINTER(vp), C.POINTER(u32)]
        l.aclb200_release_clipset.argtypes = [vp, vp]
        l.aclb200_clipset_get_info.argtypes = [vp, C.POINTER(_ClipsetInfo)]
        l.aclb200_clipset_get_clip_info.argtypes = [vp, u32, C.POINTER(_ClipInfo)]
        l.aclb200_decompress_tracks.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_decompress_track.argtypes = [vp, vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_scalar_decompress_tracks.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_scalar_decompress_track.argtypes = [vp, vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_decompress_tracks_host.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, C.c_size_t]
        l.aclb200_debug_seek.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_debug_unpack.argtypes = [vp, vp, vp, u32, C.POINTER(Options), u32, u32, vp, vp]
        l.aclb200_debug_set_trace.argtypes = [vp, vp, u32, u32]
        l.aclb200_debug_last_launch.argtypes = [vp, C.POINTER(LaunchInfo)]
        l.aclb200_device_malloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
        l.aclb200_device_free.argtypes = [vp, vp]
        l.aclb200_device_free.restype = None
        l.aclb200_copy_to_device.argtypes = [vp, vp, vp, C.c_size_t]
        l.aclb200_copy_to_host.argtypes = [vp, vp, vp, C.c_size_t]
        l.aclb200_calculate_compression_error.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, C.POINTER(Options), vp, vp, vp]
        l.aclb200_set_error_chunk_bytes.argtypes = [vp, u64]
        l.aclb200_decompress_all_samples.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp]
        l.aclb200_local_to_object_space.argtypes = [vp, vp, vp, u64, u32, u64, vp, vp, vp]
        l.aclb200_decompress_tracks_object_space.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp, u32, vp, vp, vp]
        l.aclb200_decompress_tracks_additive.argtypes = [vp, vp, vp, u32, C.POINTER(Options), u32, vp, vp, vp, u32, vp, vp, vp]
        l.aclb200_apply_additive_to_base.argtypes = [vp, vp, vp, vp, u64, u32, u64, u32, vp, vp]
        l.aclb200_decompress_tracks_blend.argtypes = [vp, vp, vp, u32, C.POINTER(Options), C.c_float, vp, vp, vp, u32, vp, vp, vp]
        l.aclb200_blend_poses.argtypes = [vp, vp, vp, vp, u64, u32, u64, C.c_float, vp, vp]
        l.aclb200_decompress_tracks_skinning.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp, vp, vp, vp, vp]
        l.aclb200_decompress_tracks_additive_skinning.argtypes = [vp, vp, vp, u32, C.POINTER(Options), u32, vp, vp, vp, vp, vp, vp, vp]
        l.aclb200_decompress_tracks_blend_skinning.argtypes = [vp, vp, vp, u32, C.POINTER(Options), C.c_float, vp, vp, vp, vp, vp, vp, vp]
        l.aclb200_local_to_skinning.argtypes = [vp, vp, vp, u64, u32, u64, vp, vp, vp, vp]
        l.aclb200_decompress_tracks_layered.argtypes = [vp, vp, vp, u32, u32, C.POINTER(Options), u32, vp, vp, vp, u32, vp, vp, vp]
        l.aclb200_decompress_tracks_layered_skinning.argtypes = [vp, vp, vp, u32, u32, C.POINTER(Options), u32, vp, vp, vp, vp, vp, vp, vp]
        l.aclb200_decompress_tracks_layered_masked.argtypes = [vp, vp, vp, vp, u32, u32, vp, u32, u32, C.POINTER(Options), u32, vp, vp, vp, u32,
                                                               vp, vp, vp]
        l.aclb200_decompress_tracks_layered_masked_skinning.argtypes = [vp, vp, vp, vp, u32, u32, vp, u32, u32, C.POINTER(Options), u32, vp, vp,
                                                                        vp, vp, vp, vp, vp]
        l.aclb200_decompress_bones.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u32, u32, vp, vp, vp, u32, vp, vp, vp]
        l.aclb200_extract_root_motion.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, vp, vp, vp]
        l.aclb200_extract_pose_features.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u32, vp, u32, u32, vp, vp, vp, vp, vp, vp, vp]
        l.aclb200_pack_pose_features.argtypes = [vp, vp, u32, u32, u32, u64, vp, u32, vp, vp, u32, vp, u32, vp]
        l.aclb200_search_pose_features.argtypes = [vp, vp, u64, u64, vp, vp, vp, u32, u64, u32, vp, vp]
        l.aclb200_begin_inertialization.argtypes = [vp, vp, vp, vp, vp, u64, u32, u64, C.c_float, vp, u64, vp, vp]
        l.aclb200_inertialize_poses.argtypes = [vp, vp, vp, u64, u32, u64, vp, vp, u64, u64, vp]
        l.aclb200_decompress_tracks_inertialized.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u64, u64, vp, vp, u32, vp, vp, vp]
        l.aclb200_decompress_tracks_inertialized_skinning.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u64, u64, vp, vp, vp, vp, vp, vp]
        l.aclb200_mirror_poses.argtypes = [vp, vp, vp, u64, u32, u64, vp, vp, u32, vp, vp]
        l.aclb200_decompress_tracks_mirrored.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u32, vp, vp, u32, vp, vp, vp]
        l.aclb200_decompress_tracks_mirrored_skinning.argtypes = [vp, vp, vp, u32, C.POINTER(Options), vp, u32, vp, vp, vp, vp, vp, vp]
        l.aclb200_upload_database.argtypes = [vp, vp, u32, u32, C.POINTER(vp)]
        l.aclb200_release_database.argtypes = [vp, vp]
        l.aclb200_release_database.restype = None
        l.aclb200_database_get_info.argtypes = [vp, C.POINTER(_DatabaseInfo)]
        l.aclb200_database_get_loaded_chunks.argtypes = [vp, u32, C.POINTER(u32)]
        l.aclb200_database_stream_in.argtypes = [vp, vp, u32, u32, vp, C.POINTER(u32), vp]
        l.aclb200_database_stream_out.argtypes = [vp, vp, u32, u32, C.POINTER(u32), vp]
        l.aclb200_clipset_bind_database.argtypes = [vp, vp, vp, C.POINTER(u32)]
        l.aclb200_launch_count.argtypes = [vp]
        l.aclb200_launch_count.restype = u64
        _lib_handle = l
    return _lib_handle


def exported_symbols() -> list[str]:
    """Every function include/aclb200.h declares (used by the CPU-side symbol test)."""
    return [
        "aclb200_version_string", "aclb200_status_string", "aclb200_default_options", "aclb200_create", "aclb200_destroy",
        "aclb200_last_error", "aclb200_upload_clips", "aclb200_upload_clips_packed", "aclb200_release_clipset",
        "aclb200_clipset_get_info", "aclb200_clipset_get_clip_info", "aclb200_decompress_tracks", "aclb200_decompress_track",
        "aclb200_scalar_decompress_tracks", "aclb200_scalar_decompress_track", "aclb200_decompress_tracks_host",
        "aclb200_debug_seek", "aclb200_debug_unpack", "aclb200_debug_set_trace", "aclb200_debug_last_launch", "aclb200_launch_count",
        "aclb200_device_malloc", "aclb200_device_free", "aclb200_copy_to_device", "aclb200_copy_to_host",
        "aclb200_calculate_compression_error", "aclb200_set_error_chunk_bytes", "aclb200_local_to_object_space",
        "aclb200_decompress_all_samples", "aclb200_upload_database", "aclb200_release_database", "aclb200_database_get_info",
        "aclb200_database_get_loaded_chunks", "aclb200_database_stream_in", "aclb200_database_stream_out", "aclb200_clipset_bind_database",
        "aclb200_decompress_tracks_object_space", "aclb200_decompress_tracks_additive", "aclb200_apply_additive_to_base",
        "aclb200_decompress_tracks_blend", "aclb200_blend_poses", "aclb200_decompress_tracks_skinning",
        "aclb200_decompress_tracks_additive_skinning", "aclb200_decompress_tracks_blend_skinning", "aclb200_local_to_skinning",
        "aclb200_decompress_tracks_layered", "aclb200_decompress_tracks_layered_skinning",
        "aclb200_decompress_tracks_layered_masked", "aclb200_decompress_tracks_layered_masked_skinning", "aclb200_decompress_bones",
        "aclb200_extract_root_motion", "aclb200_extract_pose_features", "aclb200_pack_pose_features", "aclb200_search_pose_features",
        "aclb200_begin_inertialization", "aclb200_inertialize_poses", "aclb200_decompress_tracks_inertialized",
        "aclb200_decompress_tracks_inertialized_skinning", "aclb200_mirror_poses", "aclb200_decompress_tracks_mirrored",
        "aclb200_decompress_tracks_mirrored_skinning",
    ]


def make_requests(clips, times) -> np.ndarray:
    """(clip index, sample time) arrays -> aclb200_request[]"""
    clips = np.asarray(clips, dtype=np.uint32)
    times = np.asarray(times, dtype=np.float32)
    out = np.empty(clips.shape[0], dtype=REQUEST_DTYPE)
    out["clip"] = clips
    out["sample_time"] = times
    return out


ADDITIVE_REQUEST_DTYPE = np.dtype([("base_clip", np.uint32), ("base_time", np.float32), ("additive_clip", np.uint32), ("additive_time", np.float32)])


def make_additive_requests(base_clips, base_times, additive_clips, additive_times) -> np.ndarray:
    """(base clip, base time, additive clip, additive time) arrays -> aclb200_additive_request[]"""
    base_clips = np.asarray(base_clips, dtype=np.uint32)
    out = np.empty(base_clips.shape[0], dtype=ADDITIVE_REQUEST_DTYPE)
    out["base_clip"] = base_clips
    out["base_time"] = np.asarray(base_times, dtype=np.float32)
    out["additive_clip"] = np.asarray(additive_clips, dtype=np.uint32)
    out["additive_time"] = np.asarray(additive_times, dtype=np.float32)
    return out


BLEND_REQUEST_DTYPE = np.dtype([("from_clip", np.uint32), ("from_time", np.float32), ("to_clip", np.uint32), ("to_time", np.float32)])


def make_blend_requests(from_clips, from_times, to_clips, to_times) -> np.ndarray:
    """(from clip, from time, to clip, to time) arrays -> aclb200_blend_request[]"""
    from_clips = np.asarray(from_clips, dtype=np.uint32)
    out = np.empty(from_clips.shape[0], dtype=BLEND_REQUEST_DTYPE)
    out["from_clip"] = from_clips
    out["from_time"] = np.asarray(from_times, dtype=np.float32)
    out["to_clip"] = np.asarray(to_clips, dtype=np.uint32)
    out["to_time"] = np.asarray(to_times, dtype=np.float32)
    return out


LAYER_OFF, LAYER_BLEND, LAYER_ADDITIVE = 0, 1, 2
MAX_LAYERS = 8
LAYER_NO_MASK = 0xFFFFFFFF      # the mask index of a layer without a bone mask (decompress_tracks_layered_masked)
MAX_QUERY_BONES = 32             # bones per list of decompress_bones
NO_BONE = 0xFFFFFFFF             # an unused entry of a bone list (decompress_bones)
LAYER_DTYPE = np.dtype([("clip", np.uint32), ("sample_time", np.float32), ("op", np.uint32), ("weight", np.float32)])
MAX_ROOT_MOTION_CYCLES = 256     # the most loop boundaries one extract_root_motion request may cross
# numpy view of aclb200_root_motion_request {uint32 clip; float from_time; float to_time; int32 cycles}
ROOT_MOTION_REQUEST_DTYPE = np.dtype([("clip", np.uint32), ("from_time", np.float32), ("to_time", np.float32), ("cycles", np.int32)])
FEATURE_CLAMP, FEATURE_LOOP = 0, 1   # extract_pose_features: an offset time beyond the clip's ends is clamped, or wraps into another cycle
MAX_FEATURE_OFFSETS = 8          # the most time offsets of one extract_pose_features launch
# numpy view of aclb200_feature_request {uint32 clip; float time; uint32 looping}
FEATURE_REQUEST_DTYPE = np.dtype([("clip", np.uint32), ("time", np.float32), ("looping", np.uint32)])
FEATURE_POSITION, FEATURE_DIRECTION, FEATURE_VELOCITY = 0, 1, 2   # pack_pose_features term kinds
MAX_FEATURE_DIMS = 64            # the most dimensions of a packed feature vector
NO_ROW = 0xFFFFFFFF              # search_pose_features: the row of a query without a candidate
# numpy views of aclb200_feature_term, aclb200_search_query and aclb200_search_result
FEATURE_TERM_DTYPE = np.dtype([("kind", np.uint32), ("s0", np.uint32), ("s1", np.uint32), ("k", np.uint32), ("axis", np.uint32),
                               ("components", np.uint32), ("inv_dt", np.float32)])
SEARCH_QUERY_DTYPE = np.dtype([("tag_mask", np.uint32), ("exclude_begin", np.uint32), ("exclude_end", np.uint32)])
SEARCH_RESULT_DTYPE = np.dtype([("row", np.uint32), ("cost", np.float32)])
NO_INERTIALIZATION = 0xFFFFFFFF  # an inertialization that reads no record
INERTIALIZATION_DTYPE = np.dtype([("record", np.uint32), ("elapsed", np.float32), ("halflife", np.float32)])
INERTIALIZED_REQUEST_DTYPE = np.dtype([("clip", np.uint32), ("sample_time", np.float32), ("record", np.uint32), ("elapsed", np.float32),
                                       ("halflife", np.float32)])


MIRROR_X, MIRROR_Y, MIRROR_Z = 0, 1, 2  # the normal of the mirror plane
ERROR_FLAG_INVALID_MIRROR = 8  # a mirror table entry without a partner row
MIRROR_ENTRY_DTYPE = np.dtype([("pre", np.float32, 4), ("post", np.float32, 4), ("mirror", np.uint32), ("reserved", np.uint32, 3)])
MIRRORED_REQUEST_DTYPE = np.dtype([("clip", np.uint32), ("sample_time", np.float32), ("mirrored", np.uint32)])


def make_layers(clips, times, ops, weights) -> np.ndarray:
    """[num_poses][num_layers] arrays (or anything that broadcasts to one shape) of clip, sample time, LAYER_* op and blend weight ->
    aclb200_layer[num_poses][num_layers]; pose r's layers are row r."""
    clips, times, ops, weights = np.broadcast_arrays(np.asarray(clips, dtype=np.uint32), np.asarray(times, dtype=np.float32),
                                                     np.asarray(ops, dtype=np.uint32), np.asarray(weights, dtype=np.float32))
    out = np.empty(clips.shape, dtype=LAYER_DTYPE)
    out["clip"] = clips
    out["sample_time"] = times
    out["op"] = ops
    out["weight"] = weights
    return out


def make_root_motion_requests(clips, from_times, to_times, cycles=0) -> np.ndarray:
    """(clip index, previous playback time, current playback time, loop boundaries crossed) arrays, or anything that broadcasts to one
    shape -> aclb200_root_motion_request[]"""
    clips, from_times, to_times, cycles = np.broadcast_arrays(np.asarray(clips, dtype=np.uint32), np.asarray(from_times, dtype=np.float32),
                                                              np.asarray(to_times, dtype=np.float32), np.asarray(cycles, dtype=np.int32))
    out = np.empty(clips.shape, dtype=ROOT_MOTION_REQUEST_DTYPE)
    out["clip"] = clips
    out["from_time"] = from_times
    out["to_time"] = to_times
    out["cycles"] = cycles
    return out.reshape(-1)


def make_feature_requests(clips, times, looping=FEATURE_CLAMP) -> np.ndarray:
    """(clip index, current playback time, FEATURE_CLAMP / FEATURE_LOOP) arrays, or anything that broadcasts to one shape ->
    aclb200_feature_request[]"""
    clips, times, looping = np.broadcast_arrays(np.asarray(clips, dtype=np.uint32), np.asarray(times, dtype=np.float32),
                                                np.asarray(looping, dtype=np.uint32))
    out = np.empty(clips.shape, dtype=FEATURE_REQUEST_DTYPE)
    out["clip"] = clips
    out["time"] = times
    out["looping"] = looping
    return out.reshape(-1)


def make_feature_terms(kinds, s0, k, components=7, s1=0, axis=0, inv_dt=0.0) -> np.ndarray:
    """(FEATURE_* kind, offset s0, bone list entry k, x = 1 | y = 2 | z = 4 component mask, later offset s1 of a velocity, axis of a
    direction, 1 / dt of a velocity) arrays, or anything that broadcasts to one shape -> aclb200_feature_term[]"""
    fields = np.broadcast_arrays(np.asarray(kinds, dtype=np.uint32), np.asarray(s0, dtype=np.uint32), np.asarray(s1, dtype=np.uint32),
                                 np.asarray(k, dtype=np.uint32), np.asarray(axis, dtype=np.uint32), np.asarray(components, dtype=np.uint32),
                                 np.asarray(inv_dt, dtype=np.float32))
    out = np.empty(fields[0].shape, dtype=FEATURE_TERM_DTYPE)
    for name, value in zip(FEATURE_TERM_DTYPE.names, fields):
        out[name] = value
    return out.reshape(-1)


def feature_term_dims(terms: np.ndarray) -> int:
    """D of a term array: the number of components its masks emit"""
    return int(sum(bin(int(c) & 7).count("1") for c in np.asarray(terms)["components"]))


def make_inertializations(records, elapsed, halflife) -> np.ndarray:
    """(record index or NO_INERTIALIZATION, seconds since the capture, halflife in seconds) arrays, or anything that broadcasts to one
    shape -> aclb200_inertialization[]"""
    records, elapsed, halflife = np.broadcast_arrays(np.asarray(records, dtype=np.uint32), np.asarray(elapsed, dtype=np.float32),
                                                     np.asarray(halflife, dtype=np.float32))
    out = np.empty(records.shape, dtype=INERTIALIZATION_DTYPE)
    out["record"], out["elapsed"], out["halflife"] = records, elapsed, halflife
    return out.reshape(-1)


def make_inertialized_requests(clips, times, records, elapsed, halflife) -> np.ndarray:
    """(clip index, sample time, record index or NO_INERTIALIZATION, seconds since the capture, halflife in seconds) arrays, or anything
    that broadcasts to one shape -> aclb200_inertialized_request[]"""
    fields = np.broadcast_arrays(np.asarray(clips, dtype=np.uint32), np.asarray(times, dtype=np.float32), np.asarray(records, dtype=np.uint32),
                                 np.asarray(elapsed, dtype=np.float32), np.asarray(halflife, dtype=np.float32))
    out = np.empty(fields[0].shape, dtype=INERTIALIZED_REQUEST_DTYPE)
    for name, value in zip(INERTIALIZED_REQUEST_DTYPE.names, fields):
        out[name] = value
    return out.reshape(-1)


def make_mirrored_requests(clips, times, mirrored) -> np.ndarray:
    """(clip index, sample time, 0 plain / 1 mirrored) arrays, or anything that broadcasts to one shape -> aclb200_mirrored_request[]"""
    fields = np.broadcast_arrays(np.asarray(clips, dtype=np.uint32), np.asarray(times, dtype=np.float32), np.asarray(mirrored, dtype=np.uint32))
    out = np.empty(fields[0].shape, dtype=MIRRORED_REQUEST_DTYPE)
    for name, value in zip(MIRRORED_REQUEST_DTYPE.names, fields):
        out[name] = value
    return out.reshape(-1)


def _quat_mul64(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """rtm's quat_mul(a, b) (apply a, then b: the Hamilton product b a) on float64 xyzw quaternions, broadcasting"""
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([bw * ax + bx * aw + by * az - bz * ay,
                     bw * ay - bx * az + by * aw + bz * ax,
                     bw * az + bx * ay - by * ax + bz * aw,
                     bw * aw - bx * ax - by * ay - bz * az], axis=-1)


def _conj64(q: np.ndarray) -> np.ndarray:
    return q * np.array([-1.0, -1.0, -1.0, 1.0])


def _reflect_q64(q: np.ndarray, axis: int) -> np.ndarray:
    sign = -np.ones(4)
    sign[axis] = 1.0
    sign[3] = 1.0
    return q * sign


def mirror_table(parents, mirror_bones, bind_object_rotations, axis: int) -> np.ndarray:
    """A skeleton's mirror table for local pose rows (MIRROR_ENTRY_DTYPE[num_bones]), from its parents (0xFFFFFFFF for roots),
    each bone's mirror bone and its bind pose's object space rotations (float [num_bones][4], xyzw). Bone b's correction is
    C_b = quat_mul(Q_b, conj(reflect_q(Q_m(b)))) in float64, normalised, then rounded to float32; pre_b = C_b and post_b =
    conj(C_parent(b)) (identity for roots), so that mirroring the bind pose returns it. Raises ValueError unless mirror_bones is an
    involution (m(m(b)) == b) and the hierarchy is symmetric (parent(m(b)) == m(parent(b)), roots mirror to roots)."""
    parents = np.asarray(parents, dtype=np.int64).reshape(-1)
    mirror = np.asarray(mirror_bones, dtype=np.int64).reshape(-1)
    q = np.asarray(bind_object_rotations, dtype=np.float64).reshape(-1, 4)
    n = parents.shape[0]
    if axis not in (MIRROR_X, MIRROR_Y, MIRROR_Z):
        raise ValueError("axis must be MIRROR_X, MIRROR_Y or MIRROR_Z")
    if mirror.shape[0] != n or q.shape[0] != n:
        raise ValueError("parents, mirror_bones and bind_object_rotations need one entry per bone")
    if ((mirror < 0) | (mirror >= n)).any() or (mirror[mirror] != np.arange(n)).any():
        raise ValueError("mirror_bones is not an involution over the skeleton's bones")
    is_root = (parents < 0) | (parents >= n)
    for b in range(n):
        m = mirror[b]
        if is_root[b] != is_root[m] or (not is_root[b] and parents[m] != mirror[parents[b]]):
            raise ValueError(f"the hierarchy is not symmetric: parent(m({b})) != m(parent({b}))")
    c = _quat_mul64(q, _conj64(_reflect_q64(q[mirror], axis)))
    c = (c / np.linalg.norm(c, axis=-1, keepdims=True)).astype(np.float32)
    table = np.zeros(n, dtype=MIRROR_ENTRY_DTYPE)
    table["pre"] = c
    post = np.tile(np.array([0, 0, 0, 1], np.float32), (n, 1))
    post[~is_root] = _conj64(c[parents[~is_root]].astype(np.float64)).astype(np.float32)
    table["post"] = post
    table["mirror"] = mirror.astype(np.uint32)
    return table


def mirror_rows_table(table: np.ndarray, bones, frame_bone: int) -> np.ndarray:
    """The mirror table of rows that hold the listed bones relative to frame_bone, from a skeleton's table (mirror_table): pose feature
    rows (bones = a bone list, frame_bone = the root) or root motion rows (bones = [root], frame_bone = root). Row k takes pre = C of
    bones[k], post = conj(C of frame_bone) and the row whose bone is bones[k]'s mirror bone. Raises ValueError when a listed bone's mirror
    bone is not listed."""
    table = np.asarray(table)
    bones = [int(b) for b in np.asarray(bones).reshape(-1)]
    row_of = {b: k for k, b in enumerate(bones)}
    out = np.zeros(len(bones), dtype=MIRROR_ENTRY_DTYPE)
    post = _conj64(table["pre"][frame_bone].astype(np.float64)).astype(np.float32)
    for k, b in enumerate(bones):
        m = int(table["mirror"][b])
        if m not in row_of:
            raise ValueError(f"bone {b}'s mirror bone {m} is not among the rows")
        out["pre"][k] = table["pre"][b]
        out["post"][k] = post
        out["mirror"][k] = row_of[m]
    return out


def make_search_queries(tag_masks=0xFFFFFFFF, exclude_begin=0, exclude_end=0) -> np.ndarray:
    """(tag mask, first excluded row, end of the excluded rows) arrays, or anything that broadcasts to one shape -> aclb200_search_query[]"""
    masks, begin, end = np.broadcast_arrays(np.asarray(tag_masks, dtype=np.uint32), np.asarray(exclude_begin, dtype=np.uint32),
                                            np.asarray(exclude_end, dtype=np.uint32))
    out = np.empty(masks.shape, dtype=SEARCH_QUERY_DTYPE)
    out["tag_mask"] = masks
    out["exclude_begin"] = begin
    out["exclude_end"] = end
    return out.reshape(-1)


def _device_ptr(x) -> int:
    """Device pointer of a torch CUDA tensor, or an int passed through."""
    if x is None:
        return 0
    if isinstance(x, int):
        return x
    return x.data_ptr()


def _stream_ptr(stream) -> int:
    if stream is None:
        return 0
    if isinstance(stream, int):
        return stream
    return stream.cuda_stream


class ClipSet:
    def __init__(self, context: "Context", handle: int):
        self._context = context
        self._handle = handle
        info = _ClipsetInfo()
        _lib().aclb200_clipset_get_info(handle, C.byref(info))
        self.num_clips = info.num_clips
        self.track_type = info.track_type
        self.max_tracks = info.max_tracks
        self.min_tracks = info.min_tracks
        self.blob_bytes = info.blob_bytes
        self.index_bytes = info.index_bytes

    @property
    def components(self) -> int:
        """floats per scalar track sample"""
        return self.track_type + 1 if self.track_type <= 3 else 4

    def clip_info(self, clip: int) -> _ClipInfo:
        info = _ClipInfo()
        if _lib().aclb200_clipset_get_clip_info(self._handle, clip, C.byref(info)) != 0:
            raise IndexError(clip)
        return info

    def bind_database(self, database: "Database | None") -> None:
        """decompression_context::initialize(tracks, database) for every clip (None unbinds). A clip the database does not contain
        raises AclB200Error with .failed_clip set."""
        failed = C.c_uint32(0xFFFFFFFF)
        status = _lib().aclb200_clipset_bind_database(self._context._handle, self._handle, database._handle if database else None, C.byref(failed))
        if status != 0:
            error = AclB200Error(status, _lib().aclb200_last_error(self._context._handle).decode())
            error.failed_clip = failed.value
            raise error
        self._database = database       # the database must outlive the binding

    def release(self) -> None:
        if self._handle:
            _lib().aclb200_release_clipset(self._context._handle, self._handle)
            self._handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Database:
    """aclb200_database: a compressed_database on the device, its tiers streamed in and out in chunks."""

    def __init__(self, context: "Context", handle: int):
        self._context = context
        self._handle = handle

    def info(self) -> _DatabaseInfo:
        info = _DatabaseInfo()
        _lib().aclb200_database_get_info(self._handle, C.byref(info))
        return info

    def loaded_chunks(self, tier: int) -> int:
        loaded = C.c_uint32()
        self._context._check(_lib().aclb200_database_get_loaded_chunks(self._handle, tier, C.byref(loaded)))
        return loaded.value

    def is_streamed_in(self, tier: int) -> bool:
        return self.loaded_chunks(tier) == self.info().num_chunks[tier - 1]

    def stream_in(self, tier: int, num_chunks: int = 0xFFFFFFFF, bulk_data: np.ndarray | None = None, stream=None) -> int:
        """database_context::stream_in(tier, num_chunks); bulk_data = the tier's whole bulk data, None for inline bulk data.
        Returns the number of chunks streamed in."""
        if bulk_data is not None:
            bulk_data = np.ascontiguousarray(bulk_data, dtype=np.uint8)
            if bulk_data.nbytes < self.info().bulk_data_size[tier - 1]:
                raise ValueError("bulk_data must hold the tier's whole bulk data")
        count = C.c_uint32()
        self._context._check(_lib().aclb200_database_stream_in(self._context._handle, self._handle, tier, num_chunks,
                                                               None if bulk_data is None else bulk_data.ctypes.data, C.byref(count),
                                                               _stream_ptr(stream)))
        return count.value

    def stream_out(self, tier: int, num_chunks: int = 0xFFFFFFFF, stream=None) -> int:
        count = C.c_uint32()
        self._context._check(_lib().aclb200_database_stream_out(self._context._handle, self._handle, tier, num_chunks, C.byref(count),
                                                                _stream_ptr(stream)))
        return count.value

    def release(self) -> None:
        if self._handle:
            _lib().aclb200_release_database(self._context._handle, self._handle)
            self._handle = 0

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Context:
    """aclb200_context: one per (thread, device)."""

    def __init__(self, device: int = 0):
        handle = C.c_void_p()
        status = _lib().aclb200_create(device, C.byref(handle))
        if status != 0:
            raise AclB200Error(status, _lib().aclb200_status_string(status).decode())
        self._handle = handle.value
        self.device = device

    def close(self) -> None:
        if self._handle:
            _lib().aclb200_destroy(self._handle)
            self._handle = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, status: int) -> None:
        if status != 0:
            raise AclB200Error(status, _lib().aclb200_last_error(self._handle).decode())

    @property
    def launch_count(self) -> int:
        return int(_lib().aclb200_launch_count(self._handle))

    # ---- upload (decompression_context::initialize for many clips) ----
    def upload(self, blobs: list[np.ndarray], check_hash: bool = False) -> ClipSet:
        n = len(blobs)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in blobs])
        sizes = np.array([b.size for b in blobs], dtype=np.uint32)
        handle, failed = C.c_void_p(), C.c_uint32(0xFFFFFFFF)
        status = _lib().aclb200_upload_clips(self._handle, C.cast(ptrs, C.c_void_p), sizes.ctypes.data, n, int(check_hash),
                                             C.byref(handle), C.byref(failed))
        self._check(status)
        return ClipSet(self, handle.value)

    def upload_packed(self, buffer: np.ndarray, offsets: np.ndarray, sizes: np.ndarray, check_hash: bool = False) -> ClipSet:
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        sizes = np.ascontiguousarray(sizes, dtype=np.uint32)
        handle, failed = C.c_void_p(), C.c_uint32(0xFFFFFFFF)
        status = _lib().aclb200_upload_clips_packed(self._handle, buffer.ctypes.data, offsets.ctypes.data, sizes.ctypes.data,
                                                    sizes.size, int(check_hash), C.byref(handle), C.byref(failed))
        self._check(status)
        return ClipSet(self, handle.value)

    def upload_database(self, blob: np.ndarray, check_hash: bool = False) -> Database:
        """Validates and uploads a compressed_database blob (nothing streamed in yet)."""
        handle = C.c_void_p()
        self._check(_lib().aclb200_upload_database(self._handle, blob.ctypes.data, blob.size, int(check_hash), C.byref(handle)))
        return Database(self, handle.value)

    # ---- device entry points: every pointer is a torch CUDA tensor (or a raw device address) ----
    def decompress_tracks(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, stream=None) -> None:
        self._check(_lib().aclb200_decompress_tracks(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                     C.byref(options), _device_ptr(d_out), _stream_ptr(stream)))

    def decompress_tracks_object_space(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices, kind: int,
                                       d_out, d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks followed by the hierarchy walk in one kernel: 48 byte object space bones, rtm::qvvf rows (OBJECT_QVVF) or the
        xyz lanes of a 3x4 matrix's four axes (OBJECT_MATRIX3X4F). Clip c uses the skeleton at d_parent_indices + d_skeleton_offsets[c]
        (None: every clip at offset 0); d_out_flags (optional, uint32) receives the ERROR_FLAG_* met on the way."""
        self._check(_lib().aclb200_decompress_tracks_object_space(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                  C.byref(options), _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                                  kind, _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_tracks_additive(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, additive_format: int = 0,
                                   d_clip_additive_formats=None, d_parent_indices=None, kind: int = 0, d_skeleton_offsets=None,
                                   d_out_flags=None, stream=None) -> None:
        """num_requests additive pairs (make_additive_requests): pose r = apply_additive_to_base(format, decode(base), decode(additive)), the
        additive half with the track_writer defaults. format: d_clip_additive_formats[additive clip] (uint8, None: additive_format for
        every pair). With d_parent_indices the combined pose leaves in object space as `kind` rows (OBJECT_*), the skeleton of the base
        clip c at d_parent_indices + d_skeleton_offsets[c]; without, in options.output_layout. d_out_flags: optional uint32 ERROR_FLAG_*."""
        self._check(_lib().aclb200_decompress_tracks_additive(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                              C.byref(options), additive_format, _device_ptr(d_clip_additive_formats),
                                                              _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets), kind,
                                                              _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_tracks_blend(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, weight: float = 0.5,
                                d_weights=None, d_parent_indices=None, kind: int = 0, d_skeleton_offsets=None, d_out_flags=None,
                                stream=None) -> None:
        """num_requests blend pairs (make_blend_requests): pose r = rtm::qvv_lerp(decode(from), decode(to), w), w = d_weights[r] (float32,
        None: `weight` for every pair), used as given. With d_parent_indices the blended pose leaves in object space as `kind` rows
        (OBJECT_*), the skeleton of the from clip c at d_parent_indices + d_skeleton_offsets[c]; without, in options.output_layout.
        d_out_flags: optional uint32 ERROR_FLAG_* of the walk."""
        self._check(_lib().aclb200_decompress_tracks_blend(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                           C.byref(options), weight, _device_ptr(d_weights), _device_ptr(d_parent_indices),
                                                           _device_ptr(d_skeleton_offsets), kind, _device_ptr(d_out), _device_ptr(d_out_flags),
                                                           _stream_ptr(stream)))

    def decompress_tracks_layered(self, clipset: ClipSet, d_layers, num_poses: int, num_layers: int, options: Options, d_out,
                                  additive_format: int = 0, d_clip_additive_formats=None, d_parent_indices=None, kind: int = 0,
                                  d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """num_poses stacks of num_layers layers (make_layers, 1..8 per pose). The first layer whose op is not LAYER_OFF is the base,
        decoded as decompress_tracks decodes it; each later layer is folded into the running pose in order: LAYER_BLEND =
        rtm::qvv_lerp(running, layer, weight), LAYER_ADDITIVE = apply_additive_to_base(format, running, layer) with the layer decoded with
        the track_writer defaults (format: d_clip_additive_formats[layer clip], uint8, None: additive_format), LAYER_OFF = not read. With
        d_parent_indices the running pose leaves in object space as `kind` rows (OBJECT_*), the base clip c's skeleton at d_parent_indices +
        d_skeleton_offsets[c]; without, in options.output_layout. A pose with an invalid clip, a track count that differs from the base's
        or an unknown op writes nothing. d_out_flags: optional uint32 ERROR_FLAG_*."""
        self._check(_lib().aclb200_decompress_tracks_layered(self._handle, clipset._handle, _device_ptr(d_layers), num_poses, num_layers,
                                                             C.byref(options), additive_format, _device_ptr(d_clip_additive_formats),
                                                             _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets), kind,
                                                             _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_tracks_layered_masked(self, clipset: ClipSet, d_layers, num_poses: int, num_layers: int, options: Options, d_out,
                                         d_layer_masks=None, d_bone_masks=None, num_masks: int = 0, mask_stride: int = 0,
                                         additive_format: int = 0, d_clip_additive_formats=None, d_parent_indices=None, kind: int = 0,
                                         d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_layered with bone masks and weighted additive layers. d_layer_masks: uint32 [num_poses * num_layers] mask
        index per layer (LAYER_NO_MASK: none; None: no layer has a mask); mask m is d_bone_masks[m * mask_stride + b] (float32, one per
        bone of the base clip, mask_stride 0 = max_tracks). At bone b a layer's weight is weight * mask[b]; a mask of +-0 leaves the bone
        untouched. BLEND = qvv_lerp(running, layer, w_b); ADDITIVE = apply_additive_to_base(format, running, layer) when w_b == 1, else
        with qvv_lerp(writer defaults, layer, w_b) as the layer. ADDITIVE weights 1 and no masks give decompress_tracks_layered's bytes."""
        self._check(_lib().aclb200_decompress_tracks_layered_masked(self._handle, clipset._handle, _device_ptr(d_layers), _device_ptr(d_layer_masks),
                                                                    num_poses, num_layers, _device_ptr(d_bone_masks), num_masks, mask_stride,
                                                                    C.byref(options), additive_format, _device_ptr(d_clip_additive_formats),
                                                                    _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets), kind,
                                                                    _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_bones(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_bone_lists, bones_per_list: int, d_out,
                         num_lists: int = 1, d_request_lists=None, d_parent_indices=None, kind: int = 0, d_skeleton_offsets=None,
                         d_out_flags=None, stream=None) -> None:
        """Chosen bones of each request: d_bone_lists holds num_lists lists of bones_per_list (K, 1..32) uint32 bone indices (NO_BONE: a
        hole), request r uses list d_request_lists[r] (uint32, None: list 0 for every request). Entry j of request r's list lands at
        d_out + r * pose_stride + j * bone size (pose_stride: options.pose_stride_bytes, 0 = K rows). Without d_parent_indices, row j is
        row list[j] of decompress_tracks (options.output_layout); with them, row list[j] of decompress_tracks_object_space as `kind` rows,
        clip c's skeleton at d_parent_indices + d_skeleton_offsets[c]. Only the listed bones' ancestor chains are decoded and walked. An
        entry that is NO_BONE or beyond the clip's bones, a list index >= num_lists and an invalid clip leave their rows untouched.
        d_out_flags: optional uint32 ERROR_FLAG_* of the walked bones."""
        self._check(_lib().aclb200_decompress_bones(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                    _device_ptr(d_bone_lists), num_lists, bones_per_list, _device_ptr(d_request_lists),
                                                    _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets), kind,
                                                    _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def extract_root_motion(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, d_root_tracks=None,
                            d_out_flags=None, stream=None) -> None:
        """Root motion of num_requests make_root_motion_requests: M of request r is one 48 byte rtm::qvvf row at d_out + r * 48, the
        delta with T(to) = qvv_mul(M, T(from)) when cycles == 0, composed across `cycles` loop boundaries otherwise (T(t): the root
        track's decompress_tracks row at t with the clamp policy; the root of clip c is d_root_tracks[c], uint32, None: track 0).
        options need the QVV48 layout and LOOP_CLAMP. An invalid clip, a root beyond the clip's tracks or |cycles| >
        MAX_ROOT_MOTION_CYCLES leaves the row untouched. d_out_flags: optional uint32, ERROR_FLAG_NEGATIVE_SCALE (a mirrored root) and
        ERROR_FLAG_WRAP_CLIP_CYCLE (cycles != 0 on a clip compressed with the wrap policy)."""
        self._check(_lib().aclb200_extract_root_motion(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                       _device_ptr(d_root_tracks), _device_ptr(d_out), _device_ptr(d_out_flags),
                                                       _stream_ptr(stream)))

    def extract_pose_features(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, offsets, d_bone_lists,
                              bones_per_list: int, d_parent_indices, d_out, num_lists: int = 1, d_request_lists=None, d_root_tracks=None,
                              d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """Pose features of num_requests make_feature_requests at each time offset of `offsets` (host floats, seconds, 1..8 of them): row
        (s, k) of request r at d_out + r * pose_stride + (s * K + k) * 48 (pose_stride: options.pose_stride_bytes, 0 = S * K rows) is
        qvv_mul(qvv_mul(B, qvv_inverse(T)), M), the object row B of bone list[k] at u' = t + offsets[s] (wrapped into the clip under
        FEATURE_LOOP) carried into the root's frame at t: T is the root's local row at u', M root motion from t to u'. Bone lists as
        decompress_bones; the root of clip c is d_root_tracks[c] (uint32, None: track 0); clip c's skeleton is d_parent_indices +
        d_skeleton_offsets[c]. options need the QVV48 layout and LOOP_CLAMP. d_out_flags: optional uint32 ERROR_FLAG_* of the walk, of M
        and of the rows."""
        values = np.ascontiguousarray(offsets, dtype=np.float32).reshape(-1)
        self._check(_lib().aclb200_extract_pose_features(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                         values.ctypes.data if values.size else None, values.size,
                                                         _device_ptr(d_bone_lists), num_lists, bones_per_list, _device_ptr(d_request_lists),
                                                         _device_ptr(d_root_tracks), _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                         _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def pack_pose_features(self, d_rows, num_requests: int, num_offsets: int, bones_per_list: int, terms: np.ndarray, d_out, out_stride: int,
                           mean=None, scale=None, pose_stride_bytes: int = 0, num_dims: int | None = None, stream=None) -> None:
        """Feature vectors of num_requests requests' extract_pose_features rows (S = num_offsets, K = bones_per_list, pose_stride_bytes 0 =
        S * K rows): the terms (make_feature_terms, host) emit their components in order, out[r][d] = (v_d - mean[d]) * scale[d] (host
        float32 arrays, None: 0 and 1) at d_out + r * out_stride floats. num_dims defaults to the terms' component count."""
        terms = np.ascontiguousarray(terms, dtype=FEATURE_TERM_DTYPE).reshape(-1)
        dims = feature_term_dims(terms) if num_dims is None else num_dims
        stats = [None if a is None else np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in (mean, scale)]
        for a in stats:
            if a is not None and a.size < dims:
                raise ValueError("mean and scale need one float per dimension")
        self._check(_lib().aclb200_pack_pose_features(self._handle, _device_ptr(d_rows), num_requests, num_offsets, bones_per_list,
                                                      pose_stride_bytes, terms.ctypes.data if terms.size else None, terms.size,
                                                      *[None if a is None else a.ctypes.data for a in stats], dims, _device_ptr(d_out),
                                                      out_stride, _stream_ptr(stream)))

    def search_pose_features(self, d_database, num_rows: int, db_stride: int, d_query_vectors, d_queries, num_queries: int, q_stride: int,
                             num_dims: int, d_results, d_row_tags=None, stream=None) -> None:
        """The best row of each query: d_results[q] (SEARCH_RESULT_DTYPE, 8 bytes) = the allowed row with the lowest cost
        sum_d fmaf(q[d] - x[d], ...) (the lowest row on a tie; {NO_ROW, +inf} without one). Row r is allowed for query q
        (make_search_queries) when it is outside [exclude_begin, exclude_end), d_row_tags[r] & tag_mask != 0 (uint32, None: every tag set)
        and its cost is not NaN. Strides are in floats."""
        self._check(_lib().aclb200_search_pose_features(self._handle, _device_ptr(d_database), num_rows, db_stride, _device_ptr(d_row_tags),
                                                        _device_ptr(d_query_vectors), _device_ptr(d_queries), num_queries, q_stride, num_dims,
                                                        _device_ptr(d_results), _stream_ptr(stream)))

    # ---- skinning matrices: the matrix walk, then rtm::matrix_mul(inverse_bind, object) per bone. d_inverse_bind holds 12 floats per
    # skeleton entry (x_axis, y_axis, z_axis, w_axis, xyz each), 16 byte aligned, in parallel with d_parent_indices. Each bone leaves as
    # three float4 rows, row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]) of the skinning matrix: skinned[c] = dot(row c, (p, 1)). ----
    def decompress_tracks_skinning(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices, d_inverse_bind,
                                   d_out, d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_object_space(OBJECT_MATRIX3X4F) followed by the skinning step, in one kernel; clip c uses the skeleton and the
        inverse binds at offset d_skeleton_offsets[c] (None: 0)."""
        self._check(_lib().aclb200_decompress_tracks_skinning(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                              _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                              _device_ptr(d_inverse_bind), _device_ptr(d_out), _device_ptr(d_out_flags),
                                                              _stream_ptr(stream)))

    def decompress_tracks_additive_skinning(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices,
                                            d_inverse_bind, d_out, additive_format: int = 0, d_clip_additive_formats=None,
                                            d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_additive's combined poses as skinning rows, with the base clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_additive_skinning(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                       C.byref(options), additive_format, _device_ptr(d_clip_additive_formats),
                                                                       _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                                       _device_ptr(d_inverse_bind), _device_ptr(d_out), _device_ptr(d_out_flags),
                                                                       _stream_ptr(stream)))

    def decompress_tracks_blend_skinning(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices,
                                         d_inverse_bind, d_out, weight: float = 0.5, d_weights=None, d_skeleton_offsets=None,
                                         d_out_flags=None, stream=None) -> None:
        """decompress_tracks_blend's blended poses as skinning rows, with the from clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_blend_skinning(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                    C.byref(options), weight, _device_ptr(d_weights), _device_ptr(d_parent_indices),
                                                                    _device_ptr(d_skeleton_offsets), _device_ptr(d_inverse_bind), _device_ptr(d_out),
                                                                    _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_tracks_layered_skinning(self, clipset: ClipSet, d_layers, num_poses: int, num_layers: int, options: Options,
                                           d_parent_indices, d_inverse_bind, d_out, additive_format: int = 0, d_clip_additive_formats=None,
                                           d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_layered's running poses as skinning rows, with the base clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_layered_skinning(self._handle, clipset._handle, _device_ptr(d_layers), num_poses, num_layers,
                                                                      C.byref(options), additive_format, _device_ptr(d_clip_additive_formats),
                                                                      _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                                      _device_ptr(d_inverse_bind), _device_ptr(d_out), _device_ptr(d_out_flags),
                                                                      _stream_ptr(stream)))

    def decompress_tracks_layered_masked_skinning(self, clipset: ClipSet, d_layers, num_poses: int, num_layers: int, options: Options,
                                                  d_parent_indices, d_inverse_bind, d_out, d_layer_masks=None, d_bone_masks=None,
                                                  num_masks: int = 0, mask_stride: int = 0, additive_format: int = 0,
                                                  d_clip_additive_formats=None, d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_layered_masked's running poses as skinning rows, with the base clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_layered_masked_skinning(self._handle, clipset._handle, _device_ptr(d_layers),
                                                                             _device_ptr(d_layer_masks), num_poses, num_layers,
                                                                             _device_ptr(d_bone_masks), num_masks, mask_stride, C.byref(options),
                                                                             additive_format, _device_ptr(d_clip_additive_formats),
                                                                             _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                                             _device_ptr(d_inverse_bind), _device_ptr(d_out),
                                                                             _device_ptr(d_out_flags), _stream_ptr(stream)))

    def local_to_skinning(self, d_local_poses, d_out, num_poses: int, num_tracks: int, d_parent_indices, d_inverse_bind,
                          pose_stride_bytes: int = 0, d_out_flags=None, stream=None) -> None:
        """Skinning rows of num_poses QVV48 local poses of one skeleton already on the device (skeleton and inverse binds at offset 0),
        bit-identical to decompress_tracks_skinning; d_out may be d_local_poses."""
        self._check(_lib().aclb200_local_to_skinning(self._handle, _device_ptr(d_local_poses), _device_ptr(d_out), num_poses, num_tracks,
                                                     pose_stride_bytes, _device_ptr(d_parent_indices), _device_ptr(d_inverse_bind),
                                                     _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_track(self, clipset: ClipSet, d_requests, d_track_indices, num_requests: int, options: Options, d_out, stream=None) -> None:
        self._check(_lib().aclb200_decompress_track(self._handle, clipset._handle, _device_ptr(d_requests), _device_ptr(d_track_indices),
                                                    num_requests, C.byref(options), _device_ptr(d_out), _stream_ptr(stream)))

    def scalar_decompress_tracks(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, stream=None) -> None:
        self._check(_lib().aclb200_scalar_decompress_tracks(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                            C.byref(options), _device_ptr(d_out), _stream_ptr(stream)))

    def scalar_decompress_track(self, clipset: ClipSet, d_requests, d_track_indices, num_requests: int, options: Options, d_out, stream=None) -> None:
        self._check(_lib().aclb200_scalar_decompress_track(self._handle, clipset._handle, _device_ptr(d_requests), _device_ptr(d_track_indices),
                                                           num_requests, C.byref(options), _device_ptr(d_out), _stream_ptr(stream)))

    def debug_seek(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, stream=None) -> None:
        self._check(_lib().aclb200_debug_seek(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                              _device_ptr(d_out), _stream_ptr(stream)))

    def debug_unpack(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, which: int, max_sub_tracks: int, d_out, stream=None) -> None:
        self._check(_lib().aclb200_debug_unpack(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                which, max_sub_tracks, _device_ptr(d_out), _stream_ptr(stream)))

    def debug_set_trace(self, d_trace, num_blocks: int, num_iterations: int) -> None:
        self._check(_lib().aclb200_debug_set_trace(self._handle, _device_ptr(d_trace), num_blocks, num_iterations))

    def debug_last_launch(self) -> LaunchInfo:
        """Which kernel the latest decompress_tracks on this context ran, with its requests per block, grid and batch count."""
        info = LaunchInfo()
        self._check(_lib().aclb200_debug_last_launch(self._handle, C.byref(info)))
        return info

    # ---- SURVEY 8(f1) / 8(f3): compression error measurement and the object space walk, poses stay on the device ----
    def calculate_compression_error(self, clipset: ClipSet, jobs: np.ndarray, d_raw_poses, d_parent_indices, d_shell_distances,
                                    options: Options, d_out_errors, d_output_indices=None, d_out_error_matrix=None, d_base_poses=None,
                                    stream=None) -> None:
        jobs = np.ascontiguousarray(jobs)
        assert jobs.dtype == ERROR_JOB_DTYPE
        self._check(_lib().aclb200_calculate_compression_error(
            self._handle, clipset._handle, jobs.ctypes.data, jobs.shape[0], _device_ptr(d_raw_poses), _device_ptr(d_parent_indices),
            _device_ptr(d_shell_distances), _device_ptr(d_output_indices), _device_ptr(d_base_poses), C.byref(options), _device_ptr(d_out_errors),
            _device_ptr(d_out_error_matrix), _stream_ptr(stream)))

    def decompress_all_samples(self, clipset: ClipSet, jobs: np.ndarray, options: Options, d_out, stream=None) -> None:
        jobs = np.ascontiguousarray(jobs)
        assert jobs.dtype == ERROR_JOB_DTYPE
        self._check(_lib().aclb200_decompress_all_samples(self._handle, clipset._handle, jobs.ctypes.data, jobs.shape[0], C.byref(options),
                                                          _device_ptr(d_out), _stream_ptr(stream)))

    def set_error_chunk_bytes(self, num_bytes: int) -> None:
        self._check(_lib().aclb200_set_error_chunk_bytes(self._handle, num_bytes))

    def local_to_object_space(self, d_local_poses, d_object_poses, num_poses: int, num_tracks: int, d_parent_indices,
                              pose_stride_bytes: int = 0, d_out_flags=None, stream=None) -> None:
        self._check(_lib().aclb200_local_to_object_space(self._handle, _device_ptr(d_local_poses), _device_ptr(d_object_poses), num_poses,
                                                         num_tracks, pose_stride_bytes, _device_ptr(d_parent_indices),
                                                         _device_ptr(d_out_flags), _stream_ptr(stream)))

    def apply_additive_to_base(self, d_base_poses, d_additive_poses, d_out, num_poses: int, num_tracks: int, additive_format: int,
                               pose_stride_bytes: int = 0, d_out_flags=None, stream=None) -> None:
        """acl::apply_additive_to_base on every bone of num_poses QVV48 poses; d_out may be either input."""
        self._check(_lib().aclb200_apply_additive_to_base(self._handle, _device_ptr(d_base_poses), _device_ptr(d_additive_poses), _device_ptr(d_out),
                                                          num_poses, num_tracks, pose_stride_bytes, additive_format, _device_ptr(d_out_flags),
                                                          _stream_ptr(stream)))

    def blend_poses(self, d_from_poses, d_to_poses, d_out, num_poses: int, num_tracks: int, weight: float = 0.5, d_weights=None,
                    pose_stride_bytes: int = 0, stream=None) -> None:
        """rtm::qvv_lerp(from, to, w) on every bone of num_poses QVV48 poses, w = d_weights[p] (float32) or `weight`; d_out may be
        either input."""
        self._check(_lib().aclb200_blend_poses(self._handle, _device_ptr(d_from_poses), _device_ptr(d_to_poses), _device_ptr(d_out), num_poses,
                                               num_tracks, pose_stride_bytes, weight, _device_ptr(d_weights), _stream_ptr(stream)))

    def begin_inertialization(self, d_src, d_src_prev, d_dst, d_dst_prev, num_transitions: int, num_tracks: int, inv_dt: float, d_records,
                              d_record_slots=None, pose_stride_bytes: int = 0, record_stride_bytes: int = 0, stream=None) -> None:
        """The inertialization record of each transition: from the displayed QVV48 poses this frame and the frame before (d_src,
        d_src_prev) and the destination poses (d_dst, d_dst_prev), one frame being 1 / inv_dt seconds. Transition j writes the record at
        slot d_record_slots[j] (uint32), or j, of d_records (float32, num_tracks * 16 floats per record unless record_stride_bytes)."""
        self._check(_lib().aclb200_begin_inertialization(self._handle, _device_ptr(d_src), _device_ptr(d_src_prev), _device_ptr(d_dst),
                                                         _device_ptr(d_dst_prev), num_transitions, num_tracks, pose_stride_bytes, inv_dt,
                                                         _device_ptr(d_records), record_stride_bytes, _device_ptr(d_record_slots),
                                                         _stream_ptr(stream)))

    def inertialize_poses(self, d_poses, d_out, num_poses: int, num_tracks: int, d_inertializations, d_records, num_records: int,
                          pose_stride_bytes: int = 0, record_stride_bytes: int = 0, stream=None) -> None:
        """Each QVV48 pose with its record's offset decayed onto it (d_inertializations: INERTIALIZATION_DTYPE bytes, one per pose). A
        pose whose record is NO_INERTIALIZATION is copied unchanged, one whose record is >= num_records is not written; d_out may be
        d_poses."""
        self._check(_lib().aclb200_inertialize_poses(self._handle, _device_ptr(d_poses), _device_ptr(d_out), num_poses, num_tracks,
                                                     pose_stride_bytes, _device_ptr(d_inertializations), _device_ptr(d_records), num_records,
                                                     record_stride_bytes, _stream_ptr(stream)))

    def decompress_tracks_inertialized(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, d_records,
                                       num_records: int, record_stride_bytes: int = 0, d_parent_indices=None, kind: int = 0,
                                       d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """num_requests inertialized requests (make_inertialized_requests): each pose decoded, then its record's offset decayed onto it in
        the same launch (NO_INERTIALIZATION: the plain decode's rows; a record >= num_records: nothing written). With d_parent_indices the
        pose leaves in object space as `kind` rows (OBJECT_*); without, in options.output_layout."""
        self._check(_lib().aclb200_decompress_tracks_inertialized(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                  C.byref(options), _device_ptr(d_records), num_records, record_stride_bytes,
                                                                  _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets), kind,
                                                                  _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def decompress_tracks_inertialized_skinning(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices,
                                                d_inverse_bind, d_out, d_records, num_records: int, record_stride_bytes: int = 0,
                                                d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """decompress_tracks_inertialized's poses as skinning rows, with the clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_inertialized_skinning(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                           C.byref(options), _device_ptr(d_records), num_records,
                                                                           record_stride_bytes, _device_ptr(d_parent_indices),
                                                                           _device_ptr(d_skeleton_offsets), _device_ptr(d_inverse_bind),
                                                                           _device_ptr(d_out), _device_ptr(d_out_flags), _stream_ptr(stream)))

    def mirror_poses(self, d_poses, d_out, num_poses: int, num_rows: int, d_table, axis: int, d_mirrored=None, pose_stride_bytes: int = 0,
                     d_out_flags=None, stream=None) -> None:
        """Each QVV48 pose of num_rows rows mirrored with d_table (MIRROR_ENTRY_DTYPE bytes, one per row) across the plane normal to
        `axis`. d_mirrored (uint32 per pose, optional): 0 copies the pose, 1 mirrors it, anything else leaves it unwritten; without it
        every pose is mirrored. d_out may be d_poses."""
        self._check(_lib().aclb200_mirror_poses(self._handle, _device_ptr(d_poses), _device_ptr(d_out), num_poses, num_rows, pose_stride_bytes,
                                                _device_ptr(d_mirrored), _device_ptr(d_table), axis, _device_ptr(d_out_flags),
                                                _stream_ptr(stream)))

    def decompress_tracks_mirrored(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_out, d_mirror_table, axis: int,
                                   d_parent_indices=None, kind: int = 0, d_skeleton_offsets=None, d_out_flags=None, stream=None) -> None:
        """num_requests mirrored requests (make_mirrored_requests): each pose decoded, then mirrored in the same launch when its request
        says 1 (0: the plain decode's rows; anything else: nothing written). Clip c's table is at d_mirror_table + d_skeleton_offsets[c]
        entries. With d_parent_indices the pose leaves in object space as `kind` rows (OBJECT_*); without, in options.output_layout."""
        self._check(_lib().aclb200_decompress_tracks_mirrored(self._handle, clipset._handle, _device_ptr(d_requests), num_requests, C.byref(options),
                                                              _device_ptr(d_mirror_table), axis, _device_ptr(d_parent_indices),
                                                              _device_ptr(d_skeleton_offsets), kind, _device_ptr(d_out), _device_ptr(d_out_flags),
                                                              _stream_ptr(stream)))

    def decompress_tracks_mirrored_skinning(self, clipset: ClipSet, d_requests, num_requests: int, options: Options, d_parent_indices,
                                            d_inverse_bind, d_out, d_mirror_table, axis: int, d_skeleton_offsets=None, d_out_flags=None,
                                            stream=None) -> None:
        """decompress_tracks_mirrored's poses as skinning rows, with the clip's skeleton and inverse binds."""
        self._check(_lib().aclb200_decompress_tracks_mirrored_skinning(self._handle, clipset._handle, _device_ptr(d_requests), num_requests,
                                                                       C.byref(options), _device_ptr(d_mirror_table), axis,
                                                                       _device_ptr(d_parent_indices), _device_ptr(d_skeleton_offsets),
                                                                       _device_ptr(d_inverse_bind), _device_ptr(d_out), _device_ptr(d_out_flags),
                                                                       _stream_ptr(stream)))

    # ---- host buffers in, host buffers out (the call the C++ header shim uses) ----
    def decompress_tracks_host(self, clipset: ClipSet, requests: np.ndarray, options: Options, out: np.ndarray) -> np.ndarray:
        requests = np.ascontiguousarray(requests)
        assert requests.dtype == REQUEST_DTYPE
        self._check(_lib().aclb200_decompress_tracks_host(self._handle, clipset._handle, requests.ctypes.data, requests.shape[0],
                                                          C.byref(options), out.ctypes.data, out.nbytes))
        return out
