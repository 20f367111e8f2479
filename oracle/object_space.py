"""ctypes binding of the matrix object space oracles (oracle/object_space.mk): convert_transforms + local_to_object_space of
qvvf_matrix3x4f_transform_error_metric (compression/transform_error_metrics.h:397-436) on one pose, as restated by the port
(liboracle_object_space.so) and as the unmodified reference computes it (_ref/libaclref_object_space.so, where it was built).
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_object_space.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_object_space.so")
_libs: dict = {}


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _lib(path: str, name: str):
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "object_space.mk"), "port"], check=True, capture_output=True)
        l = C.CDLL(path)
        getattr(l, name).argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        _libs[path] = l
    return getattr(_libs[path], name)


def _matrix(fn, local_pose: np.ndarray, parents: np.ndarray) -> np.ndarray:
    local_pose = np.ascontiguousarray(local_pose, dtype=np.float32)
    parents = np.ascontiguousarray(parents, dtype=np.uint32)
    out = np.zeros((local_pose.shape[0], 12), dtype=np.float32)
    if fn(local_pose.ctypes.data, parents.ctypes.data, local_pose.shape[0], out.ctypes.data) != 0:
        raise RuntimeError("matrix object space: a parent does not precede its child")
    return out


def port_local_to_object_space_matrix(local_pose: np.ndarray, parents: np.ndarray) -> np.ndarray:
    """The port's: float32 [num_tracks][12] qvvf rows in, [num_tracks][12] out (x_axis, y_axis, z_axis, w_axis, xyz each)."""
    return _matrix(_lib(_PORT_PATH, "aclo_local_to_object_space_matrix"), local_pose, parents)


def reference_local_to_object_space_matrix(local_pose: np.ndarray, parents: np.ndarray) -> np.ndarray:
    """The unmodified reference metric's, same layout."""
    return _matrix(_lib(_REF_PATH, "aclref_local_to_object_space_matrix"), local_pose, parents)
