"""ctypes binding of the inertialization oracles (oracle/inertialization.mk): the capture of aclb200_begin_inertialization and the apply of
aclb200_inertialize_poses on one pose, restated in C (liboracle_inertialization.so) and as the unmodified reference's rtm computes them
(_ref/libaclref_inertialization.so, where it was built). Poses are float32 [num_tracks][12] QVV48 rows, records float32 [num_tracks][16]
(rot_x, rot_v, pos_x, pos_v, each xyz + 0). TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_inertialization.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_inertialization.so")
_libs: dict = {}


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _lib(path: str):
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "inertialization.mk"), "port"], check=True, capture_output=True)
        l = C.CDLL(path)
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        prefix = "aclo" if path == _PORT_PATH else "aclref"
        for name, args in (("quat_rotation_log", [vp, vp]), ("quat_rotation_exp", [vp, vp]),
                           ("begin_inertialization", [vp, vp, vp, vp, u32, f32, vp]), ("inertialize_pose", [vp, vp, u32, f32, f32, vp])):
            fn = getattr(l, f"{prefix}_{name}")
            fn.argtypes, fn.restype = args, None
        _libs[path] = l
    return _libs[path]


def _fn(reference: bool, name: str):
    path = _REF_PATH if reference else _PORT_PATH
    return getattr(_lib(path), ("aclref_" if reference else "aclo_") + name)


def _rows(pose) -> np.ndarray:
    pose = np.ascontiguousarray(pose, dtype=np.float32)
    assert pose.ndim == 2 and pose.shape[1] == 12
    return pose


def quat_rotation_log(q, reference: bool = False) -> np.ndarray:
    """rtm::quat_rotation_log of one xyzw quaternion (w lane 0)"""
    q, out = np.ascontiguousarray(q, dtype=np.float32).reshape(4), np.zeros(4, np.float32)
    _fn(reference, "quat_rotation_log")(q.ctypes.data, out.ctypes.data)
    return out


def quat_rotation_exp(v, reference: bool = False) -> np.ndarray:
    """rtm::quat_rotation_exp of one xyzw vector (its w is not read)"""
    v, out = np.ascontiguousarray(v, dtype=np.float32).reshape(4), np.zeros(4, np.float32)
    _fn(reference, "quat_rotation_exp")(v.ctypes.data, out.ctypes.data)
    return out


def begin_inertialization(src, src_prev, dst, dst_prev, inv_dt: float, reference: bool = False) -> np.ndarray:
    """The record of one transition: float32 [num_tracks][16]"""
    src, src_prev, dst, dst_prev = (_rows(p) for p in (src, src_prev, dst, dst_prev))
    assert src.shape == src_prev.shape == dst.shape == dst_prev.shape
    record = np.zeros((src.shape[0], 16), np.float32)
    _fn(reference, "begin_inertialization")(src.ctypes.data, src_prev.ctypes.data, dst.ctypes.data, dst_prev.ctypes.data, src.shape[0],
                                             inv_dt, record.ctypes.data)
    return record


def inertialize_pose(pose, record, elapsed: float, halflife: float, reference: bool = False) -> np.ndarray:
    """One pose with its record's offset decayed onto it: float32 [num_tracks][12]"""
    pose = _rows(pose)
    record = np.ascontiguousarray(record, dtype=np.float32).reshape(-1, 16)
    assert record.shape[0] >= pose.shape[0]
    out = np.zeros_like(pose)
    _fn(reference, "inertialize_pose")(pose.ctypes.data, record.ctypes.data, pose.shape[0], elapsed, halflife, out.ctypes.data)
    return out
