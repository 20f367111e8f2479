"""ctypes binding of the root motion oracles (oracle/root_motion.mk): rtm::qvv_inverse (rtm/qvvf.h:389-395), rtm::qvv_mul and the
composition of aclb200_extract_root_motion from four root samples, as restated by the port (liboracle_root_motion.so) and as the
unmodified reference computes them (_ref/libaclref_root_motion.so, where it was built), plus the reference's whole path from a clip.
Rows are float32 [12] rtm::qvvf rows; the rows returned carry 0 in both w lanes. TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.port import NORMALIZE_IEEE, NORMALIZE_RTM_SSE2  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_root_motion.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_root_motion.so")
_libs: dict = {}


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _lib(path: str):
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "root_motion.mk"), "port"], check=True, capture_output=True)
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _row(row) -> np.ndarray:
    row = np.ascontiguousarray(row, dtype=np.float32)
    assert row.shape == (12,)
    return row


def port_qvv_inverse(row) -> np.ndarray:
    row, out = _row(row), np.zeros(12, np.float32)
    fn = _lib(_PORT_PATH).aclo_qvv_inverse
    fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p], None
    fn(row.ctypes.data, out.ctypes.data)
    return out


def port_qvv_mul(lhs, rhs, normalize_mode: int = NORMALIZE_IEEE) -> np.ndarray:
    lhs, rhs, out = _row(lhs), _row(rhs), np.zeros(12, np.float32)
    fn = _lib(_PORT_PATH).aclo_qvv_mul
    fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p], None
    fn(lhs.ctypes.data, rhs.ctypes.data, normalize_mode, out.ctypes.data)
    return out


def port_root_motion(samples, cycles: int, normalize_mode: int = NORMALIZE_IEEE) -> tuple[np.ndarray, bool]:
    """samples: [4][12] T(from), T(to), T(D), T(0). Returns (M, whether a qvv_mul took the negative scale branch)."""
    samples = np.ascontiguousarray(samples, dtype=np.float32).reshape(4, 12)
    out = np.zeros(12, np.float32)
    fn = _lib(_PORT_PATH).aclo_root_motion
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int, C.c_void_p]
    fn.restype = C.c_int
    base = samples.ctypes.data
    negative = fn(base, base + 48, base + 96, base + 144, cycles, normalize_mode, out.ctypes.data)
    return out, bool(negative)


def reference_qvv_inverse(row) -> np.ndarray:
    row, out = _row(row), np.zeros(12, np.float32)
    fn = _lib(_REF_PATH).aclref_qvv_inverse
    fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p], None
    fn(row.ctypes.data, out.ctypes.data)
    return out


def reference_qvv_mul(lhs, rhs) -> np.ndarray:
    lhs, rhs, out = _row(lhs), _row(rhs), np.zeros(12, np.float32)
    fn = _lib(_REF_PATH).aclref_qvv_mul
    fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p, C.c_void_p], None
    fn(lhs.ctypes.data, rhs.ctypes.data, out.ctypes.data)
    return out


def reference_root_motion(samples, cycles: int) -> np.ndarray:
    samples = np.ascontiguousarray(samples, dtype=np.float32).reshape(4, 12)
    out = np.zeros(12, np.float32)
    fn = _lib(_REF_PATH).aclref_root_motion_compose
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    fn.restype = None
    base = samples.ctypes.data
    fn(base, base + 48, base + 96, base + 144, cycles, out.ctypes.data)
    return out


def reference_extract(blob: np.ndarray, settings_kind: int, writer_mode: int, rounding: int, root: int, from_time: float, to_time: float,
                      cycles: int, per_track_rounding: np.ndarray | None = None, constant_defaults: np.ndarray | None = None,
                      variable_defaults: np.ndarray | None = None) -> tuple[np.ndarray, np.ndarray]:
    """The reference's whole path for one request: decompression_context<settings_kind> with the clamp policy, seek + decompress_tracks
    at from, to, the clamp duration and 0 with a writer that keeps the root's row, then the composition. Returns (M, samples [4][12])."""
    keep = [np.ascontiguousarray(a, dtype=t) if a is not None else None
            for a, t in ((per_track_rounding, np.uint8), (constant_defaults, np.float32), (variable_defaults, np.float32))]
    samples = np.zeros((4, 12), np.float32)
    out = np.zeros(12, np.float32)
    fn = _lib(_REF_PATH).aclref_extract_root_motion
    fn.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_float, C.c_float,
                   C.c_int32, C.c_void_p, C.c_void_p]
    fn.restype = C.c_int
    rc = fn(blob.ctypes.data, settings_kind, writer_mode, rounding, *[None if a is None else a.ctypes.data for a in keep], root, from_time,
            to_time, cycles, samples.ctypes.data, out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"reference extract_root_motion failed ({rc})")
    return out, samples
