"""ctypes binding of oracle/liboracle.so -- the plain-C restatement of the reference decode path.

TEST INFRASTRUCTURE ONLY (see oracle/acl_oracle.h). The product package never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

ROUND_NONE, ROUND_FLOOR, ROUND_CEIL, ROUND_NEAREST, ROUND_PER_TRACK = 0, 1, 2, 3, 4
LOOP_CLAMP, LOOP_WRAP, LOOP_AS_COMPRESSED = 0, 1, 2
NORMALIZE_NEVER, NORMALIZE_LERP_ONLY, NORMALIZE_ALWAYS = 0, 1, 2
DEFAULT_SKIPPED, DEFAULT_CONSTANT, DEFAULT_VARIABLE, DEFAULT_LEGACY = 0, 1, 2, 3


class Settings(C.Structure):
    _fields_ = [
        ("normalization", C.c_uint32), ("per_track_rounding", C.c_uint32), ("wrapping", C.c_uint32),
        ("clamp_sample_time", C.c_uint32), ("multiple_rotation_formats", C.c_uint32),
        ("default_rotation_mode", C.c_uint32), ("default_translation_mode", C.c_uint32), ("default_scale_mode", C.c_uint32),
        ("constant_defaults", C.c_float * 12),
        ("variable_defaults", C.c_void_p), ("per_track_rounding_policies", C.c_void_p),
    ]


class SeekState(C.Structure):
    _fields_ = [
        ("sample_time", C.c_float), ("interpolation_alpha", C.c_float), ("clip_duration", C.c_float),
        ("looping_policy", C.c_uint32), ("rounding_policy", C.c_uint32),
        ("key_frames", C.c_uint32 * 2), ("segment_indices", C.c_uint32 * 2), ("segment_key_frames", C.c_uint32 * 2),
        ("key_frame_bit_offsets", C.c_uint32 * 2), ("segment_offsets", C.c_uint32 * 2),
        ("format_offsets", C.c_uint32 * 2), ("range_offsets", C.c_uint32 * 2), ("animated_offsets", C.c_uint32 * 2),
        ("uses_single_segment", C.c_uint32),
    ]


class ScalarSeekState(C.Structure):
    _fields_ = [
        ("sample_time", C.c_float), ("interpolation_alpha", C.c_float), ("duration", C.c_float),
        ("looping_policy", C.c_uint32), ("rounding_policy", C.c_uint32),
        ("key_frames", C.c_uint32 * 2), ("key_frame_bit_offsets", C.c_uint32 * 2),
    ]


_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "all"], check=True, capture_output=True)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        l = C.CDLL(_LIB_PATH)
        l.aclo_default_settings.argtypes = [C.POINTER(Settings)]
        l.aclo_validate.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
        l.aclo_hash32.argtypes = [C.c_void_p, C.c_size_t]
        l.aclo_hash32.restype = C.c_uint32
        l.aclo_transform_seek.argtypes = [C.c_void_p, C.POINTER(Settings), C.c_float, C.c_uint32, C.c_uint32, C.POINTER(SeekState)]
        l.aclo_transform_decompress_tracks.argtypes = [C.c_void_p, C.POINTER(Settings), C.POINTER(SeekState), C.c_void_p]
        l.aclo_transform_decompress_track.argtypes = [C.c_void_p, C.POINTER(Settings), C.POINTER(SeekState), C.c_uint32, C.c_void_p]
        l.aclo_transform_extract_key_frame.argtypes = [C.c_void_p, C.POINTER(SeekState), C.c_uint32, C.c_void_p]
        l.aclo_scalar_seek.argtypes = [C.c_void_p, C.POINTER(Settings), C.c_float, C.c_uint32, C.c_uint32, C.POINTER(ScalarSeekState)]
        l.aclo_scalar_decompress_tracks.argtypes = [C.c_void_p, C.POINTER(Settings), C.POINTER(ScalarSeekState), C.c_void_p]
        l.aclo_scalar_decompress_track.argtypes = [C.c_void_p, C.POINTER(Settings), C.POINTER(ScalarSeekState), C.c_uint32, C.c_void_p]
        l.aclo_transform_touched_bytes.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        l.aclo_scalar_touched_bytes.argtypes = [C.c_void_p, C.c_void_p]
        l.aclo_bench_transform.restype = C.c_double
        l.aclo_bench_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        _lib = l
    return _lib


class SettingsBuilder:
    """Keeps the numpy arrays referenced by a Settings struct alive."""

    def __init__(self, normalization=NORMALIZE_LERP_ONLY, per_track_rounding=False, wrapping=True, clamp=True,
                 multiple_rotation_formats=False, default_modes=(DEFAULT_CONSTANT, DEFAULT_CONSTANT, DEFAULT_LEGACY),
                 constant_defaults=None, variable_defaults=None, per_track_policies=None):
        s = Settings()
        lib().aclo_default_settings(C.byref(s))
        s.normalization = normalization
        s.per_track_rounding = int(per_track_rounding)
        s.wrapping = int(wrapping)
        s.clamp_sample_time = int(clamp)
        s.multiple_rotation_formats = int(multiple_rotation_formats)
        s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode = default_modes
        if constant_defaults is not None:
            cd = np.ascontiguousarray(constant_defaults, dtype=np.float32).reshape(12)
            for i in range(12):
                s.constant_defaults[i] = float(cd[i])
        self._variable = None if variable_defaults is None else np.ascontiguousarray(variable_defaults, dtype=np.float32)
        self._policies = None if per_track_policies is None else np.ascontiguousarray(per_track_policies, dtype=np.uint8)
        s.variable_defaults = None if self._variable is None else self._variable.ctypes.data
        s.per_track_rounding_policies = None if self._policies is None else self._policies.ctypes.data
        self.c = s


# The reference settings kinds of oracle/ref_tool.cpp expressed as port settings
def settings_for_kind(kind: int, **kw) -> SettingsBuilder:
    table = {
        0: dict(normalization=NORMALIZE_LERP_ONLY, per_track_rounding=False, multiple_rotation_formats=False),   # default_transform
        1: dict(normalization=NORMALIZE_ALWAYS, per_track_rounding=True, multiple_rotation_formats=True),        # debug_transform
        2: dict(normalization=NORMALIZE_LERP_ONLY, per_track_rounding=False, multiple_rotation_formats=False),   # benchmark
        3: dict(normalization=NORMALIZE_NEVER, per_track_rounding=False, multiple_rotation_formats=True),        # all formats, never
        4: dict(normalization=NORMALIZE_LERP_ONLY, per_track_rounding=False, multiple_rotation_formats=True),    # all formats, lerp_only
        5: dict(normalization=NORMALIZE_ALWAYS, per_track_rounding=False, multiple_rotation_formats=False),      # quatf_full only
    }
    args = dict(table[kind])
    args.update(kw)
    return SettingsBuilder(**args)


def writer_modes(mode: int):
    """ref_tool.cpp writer modes -> (rotation, translation, scale) default sub-track modes."""
    return {0: (DEFAULT_CONSTANT, DEFAULT_CONSTANT, DEFAULT_LEGACY), 1: (DEFAULT_SKIPPED,) * 3,
            2: (DEFAULT_CONSTANT,) * 3, 3: (DEFAULT_VARIABLE,) * 3}[mode]


def num_tracks_of(blob: np.ndarray) -> int:
    return int(blob[16:20].view(np.uint32)[0])


def hash32(data: np.ndarray) -> int:
    """hash32 (FNV-1a 32, core/hash.h) of a byte array: what compressed_tracks stores over bytes [8, size)."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    return int(lib().aclo_hash32(data.ctypes.data, data.size))


def validate(blob: np.ndarray, check_hash: bool = False) -> int:
    return lib().aclo_validate(blob.ctypes.data, blob.size, int(check_hash))


def find_key_frames(num_samples: int, sample_rate: float, sample_time: float, rounding=ROUND_NONE, looping=LOOP_CLAMP):
    """find_linear_interpolation_samples_with_sample_rate: (key frame 0, key frame 1, alpha)."""
    k0, k1, alpha = C.c_uint32(), C.c_uint32(), C.c_float()
    fn = lib().aclo_find_key_frames
    fn.restype = None
    fn.argtypes = [C.c_uint32, C.c_float, C.c_float, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_float)]
    fn(num_samples, sample_rate, sample_time, rounding, looping, C.byref(k0), C.byref(k1), C.byref(alpha))
    return k0.value, k1.value, alpha.value


def transform_seek(blob, settings: SettingsBuilder, t: float, rounding=ROUND_NONE, looping=LOOP_AS_COMPRESSED) -> SeekState:
    st = SeekState()
    rc = lib().aclo_transform_seek(blob.ctypes.data, C.byref(settings.c), t, rounding, looping, C.byref(st))
    if rc != 0:
        raise RuntimeError(f"aclo_transform_seek failed ({rc})")
    return st


def transform_decompress_tracks(blob, settings: SettingsBuilder, t: float, rounding=ROUND_NONE, looping=LOOP_AS_COMPRESSED,
                                out: np.ndarray | None = None) -> np.ndarray:
    st = transform_seek(blob, settings, t, rounding, looping)
    if out is None:
        out = np.zeros((num_tracks_of(blob), 12), dtype=np.float32)
    rc = lib().aclo_transform_decompress_tracks(blob.ctypes.data, C.byref(settings.c), C.byref(st), out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"aclo_transform_decompress_tracks failed ({rc})")
    return out


def transform_decompress_track(blob, settings: SettingsBuilder, t: float, track: int, rounding=ROUND_NONE, looping=LOOP_AS_COMPRESSED,
                               out: np.ndarray | None = None) -> np.ndarray:
    st = transform_seek(blob, settings, t, rounding, looping)
    if out is None:
        out = np.zeros((num_tracks_of(blob), 12), dtype=np.float32)
    rc = lib().aclo_transform_decompress_track(blob.ctypes.data, C.byref(settings.c), C.byref(st), track, out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"aclo_transform_decompress_track failed ({rc})")
    return out


def transform_key_frame_ints(blob, st: SeekState, which: int) -> np.ndarray:
    th = blob[32:32 + 52].view(np.uint32)
    has_scale = int(blob[28:32].view(np.uint32)[0]) & 1
    n = int(th[2]) + int(th[3]) + (int(th[4]) if has_scale else 0)
    out = np.zeros((n, 4), dtype=np.uint32)
    rc = lib().aclo_transform_extract_key_frame(blob.ctypes.data, C.byref(st), which, out.ctypes.data)
    if rc != 0:
        raise RuntimeError("aclo_transform_extract_key_frame failed")
    return out


def scalar_seek(blob, settings: SettingsBuilder, t: float, rounding=ROUND_NONE, looping=LOOP_AS_COMPRESSED) -> ScalarSeekState:
    st = ScalarSeekState()
    rc = lib().aclo_scalar_seek(blob.ctypes.data, C.byref(settings.c), t, rounding, looping, C.byref(st))
    if rc != 0:
        raise RuntimeError(f"aclo_scalar_seek failed ({rc})")
    return st


def scalar_decompress(blob, settings: SettingsBuilder, t: float, rounding=ROUND_NONE, looping=LOOP_AS_COMPRESSED,
                      track: int = -1) -> np.ndarray:
    st = scalar_seek(blob, settings, t, rounding, looping)
    out = np.zeros((num_tracks_of(blob), 4), dtype=np.float32)
    if track < 0:
        rc = lib().aclo_scalar_decompress_tracks(blob.ctypes.data, C.byref(settings.c), C.byref(st), out.ctypes.data)
    else:
        rc = lib().aclo_scalar_decompress_track(blob.ctypes.data, C.byref(settings.c), C.byref(st), track, out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"scalar decode failed ({rc})")
    return out


def transform_touched_bytes(blob, segment_index: int = 0) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    rc = lib().aclo_transform_touched_bytes(blob.ctypes.data, segment_index, out.ctypes.data)
    if rc != 0:
        raise RuntimeError("aclo_transform_touched_bytes failed")
    return out


def scalar_touched_bytes(blob) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    rc = lib().aclo_scalar_touched_bytes(blob.ctypes.data, out.ctypes.data)
    if rc != 0:
        raise RuntimeError("aclo_scalar_touched_bytes failed")
    return out


def bench_transform(blobs, request_clip, request_time, max_tracks: int) -> float:
    ptrs = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    request_clip = np.ascontiguousarray(request_clip, dtype=np.uint32)
    request_time = np.ascontiguousarray(request_time, dtype=np.float32)
    return float(lib().aclo_bench_transform(C.cast(ptrs, C.c_void_p), request_clip.ctypes.data, request_time.ctypes.data,
                                            request_clip.size, max_tracks))


# SURVEY 8(f1): the compression error measurement over already sampled poses (acl_oracle.h)
class TrackError(C.Structure):
    _fields_ = [("index", C.c_uint32), ("error", C.c_float), ("sample_time", C.c_float)]


NORMALIZE_RTM_SSE2, NORMALIZE_IEEE = 0, 1


def local_to_object_space(local_pose: np.ndarray, parents: np.ndarray, normalize_mode: int = NORMALIZE_IEEE) -> np.ndarray:
    """qvvf_transform_error_metric::local_to_object_space of one pose, float32 [num_tracks][12]."""
    local_pose = np.ascontiguousarray(local_pose, dtype=np.float32)
    parents = np.ascontiguousarray(parents, dtype=np.uint32)
    out = np.zeros_like(local_pose)
    fn = lib().aclo_local_to_object_space
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    rc = fn(local_pose.ctypes.data, parents.ctypes.data, local_pose.shape[0], normalize_mode, out.ctypes.data)
    if rc < 0:
        raise RuntimeError("aclo_local_to_object_space: a parent does not precede its child")
    return out


def transform_track_error(raw_poses: np.ndarray, lossy_poses: np.ndarray, sample_rate: float, duration: float, parents: np.ndarray,
                          shell_distances: np.ndarray, normalize_mode: int = NORMALIZE_IEEE, base_poses: np.ndarray | None = None,
                          additive_format: int = 0, metric: int = 0):
    """The loop of calculate_transform_track_error over [num_samples][num_tracks][12] poses.
    Returns (TrackError, errors float32 [num_samples][num_tracks], negative_scale_seen)."""
    raw_poses = np.ascontiguousarray(raw_poses, dtype=np.float32)
    lossy_poses = np.ascontiguousarray(lossy_poses, dtype=np.float32)
    parents = np.ascontiguousarray(parents, dtype=np.uint32)
    shell_distances = np.ascontiguousarray(shell_distances, dtype=np.float32)
    num_samples, num_tracks = raw_poses.shape[0], raw_poses.shape[1]
    assert lossy_poses.shape == raw_poses.shape and raw_poses.shape[2] == 12
    errors = np.zeros((num_samples, num_tracks), dtype=np.float32)
    scratch = np.zeros((4, max(num_tracks, 1), 12), dtype=np.float32)
    if base_poses is not None:
        base_poses = np.ascontiguousarray(base_poses, dtype=np.float32)
        assert base_poses.shape == raw_poses.shape
    result = TrackError()
    fn = lib().aclo_transform_track_error
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_int,
                   C.POINTER(TrackError), C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
    rc = fn(raw_poses.ctypes.data, lossy_poses.ctypes.data, num_samples, num_tracks, sample_rate, duration, parents.ctypes.data,
            shell_distances.ctypes.data, normalize_mode, C.byref(result), errors.ctypes.data, scratch.ctypes.data,
            None if base_poses is None else base_poses.ctypes.data, additive_format, metric)
    if rc < 0:
        raise RuntimeError("aclo_transform_track_error: a parent does not precede its child")
    return result, errors, rc == 1


def apply_additive_to_base(additive_format: int, base_pose: np.ndarray, pose: np.ndarray, normalize_mode: int = NORMALIZE_IEEE) -> np.ndarray:
    """acl::apply_additive_to_base over one pose [num_tracks][12]; returns the combined pose."""
    base_pose = np.ascontiguousarray(base_pose, dtype=np.float32)
    out = np.array(pose, dtype=np.float32, order="C", copy=True)
    fn = lib().aclo_apply_additive_to_base
    fn.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int]
    fn(additive_format, base_pose.ctypes.data, out.ctypes.data, out.shape[0], normalize_mode)
    return out


def scalar_track_error(raw_values: np.ndarray, lossy_values: np.ndarray, components: int, sample_rate: float, duration: float) -> TrackError:
    """calculate_scalar_track_error over [num_samples][num_tracks][4] rows (the first `components` floats of each row count)."""
    raw_values = np.ascontiguousarray(raw_values, dtype=np.float32)
    lossy_values = np.ascontiguousarray(lossy_values, dtype=np.float32)
    assert raw_values.shape == lossy_values.shape and raw_values.shape[2] == 4
    result = TrackError()
    fn = lib().aclo_scalar_track_error
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.POINTER(TrackError)]
    fn(raw_values.ctypes.data, lossy_values.ctypes.data, raw_values.shape[0], raw_values.shape[1], components, sample_rate, duration, C.byref(result))
    return result
