"""ctypes binding of the mirror oracles (oracle/mirror.mk): one pose of QVV48 rows mirrored with a mirror table, as aclb200_mirror_poses
mirrors it, restated in C (liboracle_mirror.so) and built from the unmodified reference's rtm (_ref/libaclref_mirror.so, where it was
built). Poses are float32 [num_rows][12]; tables are acl_b200.MIRROR_ENTRY_DTYPE arrays (48 bytes per row). TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_mirror.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_mirror.so")
_libs: dict = {}
INVALID_MIRROR = 8


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _fn(reference: bool):
    path = _REF_PATH if reference else _PORT_PATH
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "mirror.mk"), "port"], check=True, capture_output=True)
        l = C.CDLL(path)
        fn = l.aclref_mirror_pose if reference else l.aclo_mirror_pose
        fn.argtypes, fn.restype = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p], C.c_uint32
        _libs[path] = fn
    return _libs[path]


def mirror_pose(pose, table, axis: int, reference: bool = False) -> tuple[np.ndarray, int]:
    """One pose mirrored: (float32 [num_rows][12] rows with w lanes 0, ACLB200_ERROR_FLAG_INVALID_MIRROR or 0)"""
    pose = np.ascontiguousarray(pose, dtype=np.float32).reshape(-1, 12)
    table = np.ascontiguousarray(table)
    assert table.dtype.itemsize == 48 and table.shape[0] >= pose.shape[0]
    out = np.zeros_like(pose)
    flags = _fn(reference)(pose.ctypes.data, table.ctypes.data, pose.shape[0], axis, out.ctypes.data)
    return out, int(flags)


def mirror_poses(poses, table, axis: int, mirrored=None) -> tuple[np.ndarray, int]:
    """aclb200_mirror_poses over [num_poses][num_rows][12] poses: mirrored[p] 0 copies, 1 mirrors, other values leave the pose's rows as
    they are in the returned copy (the caller puts what the output held there). Returns (poses, flags OR-ed over the mirrored poses)."""
    poses = np.array(poses, dtype=np.float32)
    flags = 0
    for p in range(poses.shape[0]):
        if mirrored is None or mirrored[p] == 1:
            poses[p], f = mirror_pose(poses[p], table, axis)
            flags |= f
    return poses, flags
