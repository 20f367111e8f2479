"""ctypes binding of the blend oracles (oracle/blend.mk): rtm::qvv_lerp (rtm/qvvf.h:439-445) on one pose, as restated by the port
(liboracle_blend.so, in both normalise flavours) and as the unmodified reference computes it (_ref/libaclref_blend.so, where it was built).
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.port import NORMALIZE_IEEE, NORMALIZE_RTM_SSE2  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_blend.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_blend.so")
_libs: dict = {}


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _lib(path: str):
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "blend.mk"), "port"], check=True, capture_output=True)
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _poses(from_pose, to_pose):
    from_pose = np.ascontiguousarray(from_pose, dtype=np.float32)
    to_pose = np.ascontiguousarray(to_pose, dtype=np.float32)
    assert from_pose.shape == to_pose.shape and from_pose.ndim == 2 and from_pose.shape[1] == 12
    return from_pose, to_pose, np.zeros_like(from_pose)


def port_qvv_lerp(from_pose: np.ndarray, to_pose: np.ndarray, weight: float, normalize_mode: int = NORMALIZE_IEEE) -> np.ndarray:
    """The port's: float32 [num_tracks][12] rows in, [num_tracks][12] out, translation and scale w lanes 0."""
    from_pose, to_pose, out = _poses(from_pose, to_pose)
    fn = _lib(_PORT_PATH).aclo_qvv_lerp
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_float, C.c_int, C.c_void_p]
    fn.restype = None
    fn(from_pose.ctypes.data, to_pose.ctypes.data, from_pose.shape[0], weight, normalize_mode, out.ctypes.data)
    return out


def reference_qvv_lerp(from_pose: np.ndarray, to_pose: np.ndarray, weight: float) -> np.ndarray:
    """The unmodified reference's, same layout (w lanes as rtm leaves them)."""
    from_pose, to_pose, out = _poses(from_pose, to_pose)
    fn = _lib(_REF_PATH).aclref_qvv_lerp
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_float, C.c_void_p]
    fn.restype = None
    fn(from_pose.ctypes.data, to_pose.ctypes.data, from_pose.shape[0], weight, out.ctypes.data)
    return out
