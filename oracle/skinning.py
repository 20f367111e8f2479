"""ctypes binding of the skinning oracles (oracle/skinning.mk): convert_transforms + local_to_object_space of
qvvf_matrix3x4f_transform_error_metric (compression/transform_error_metrics.h:397-436), then rtm::matrix_mul(inverse_bind, object), on one
pose, as restated by the port (liboracle_skinning.so) and as the unmodified reference computes it (_ref/libaclref_skinning.so, where it was
built). Skinning rows are the library's layout: [num_tracks][3][4], row c = (x_axis[c], y_axis[c], z_axis[c], w_axis[c]).
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_PATH = os.path.join(_HERE, "liboracle_skinning.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_skinning.so")
_libs: dict = {}


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def _lib(path: str):
    if path not in _libs:
        if path == _PORT_PATH and not os.path.exists(path):
            subprocess.run(["make", "-f", os.path.join(_HERE, "skinning.mk"), "port"], check=True, capture_output=True)
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _f32(array, columns: int) -> np.ndarray:
    array = np.ascontiguousarray(array, dtype=np.float32)
    assert array.ndim == 2 and array.shape[1] == columns, array.shape
    return array


def _skinning(fn, local_pose, parents, inverse_bind) -> np.ndarray:
    local_pose = _f32(local_pose, 12)
    inverse_bind = _f32(inverse_bind, 12)
    parents = np.ascontiguousarray(parents, dtype=np.uint32)
    assert inverse_bind.shape[0] == parents.shape[0] == local_pose.shape[0]
    out = np.zeros((local_pose.shape[0], 12), dtype=np.float32)
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    if fn(local_pose.ctypes.data, parents.ctypes.data, inverse_bind.ctypes.data, local_pose.shape[0], out.ctypes.data) != 0:
        raise RuntimeError("skinning: a parent does not precede its child")
    return out


def port_local_to_skinning(local_pose: np.ndarray, parents: np.ndarray, inverse_bind: np.ndarray) -> np.ndarray:
    """The port's: float32 [n][12] qvvf rows and [n][12] inverse binds (x_axis, y_axis, z_axis, w_axis, xyz each) in, [n][12] skinning rows out."""
    return _skinning(_lib(_PORT_PATH).aclo_local_to_skinning, local_pose, parents, inverse_bind)


def port_skin_object_matrices(object_pose: np.ndarray, inverse_bind: np.ndarray) -> np.ndarray:
    """The port's skinning step alone: [n][12] object matrices (the rows ACLB200_OBJECT_MATRIX3X4F writes) in, [n][12] skinning rows out."""
    object_pose = _f32(object_pose, 12)
    inverse_bind = _f32(inverse_bind, 12)
    assert object_pose.shape == inverse_bind.shape
    out = np.zeros_like(object_pose)
    fn = _lib(_PORT_PATH).aclo_skin_object_matrices
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    fn.restype = None
    fn(object_pose.ctypes.data, inverse_bind.ctypes.data, object_pose.shape[0], out.ctypes.data)
    return out


def reference_local_to_skinning(local_pose: np.ndarray, parents: np.ndarray, inverse_bind: np.ndarray) -> np.ndarray:
    """The unmodified reference's, same layout."""
    return _skinning(_lib(_REF_PATH).aclref_local_to_skinning, local_pose, parents, inverse_bind)


def reference_skinned_points(local_pose: np.ndarray, parents: np.ndarray, inverse_bind: np.ndarray, points: np.ndarray) -> np.ndarray:
    """rtm::matrix_mul_point3(points[b], skin[b]) of every bone, by the reference: [n][3] float32."""
    local_pose = _f32(local_pose, 12)
    inverse_bind = _f32(inverse_bind, 12)
    points = _f32(points, 3)
    parents = np.ascontiguousarray(parents, dtype=np.uint32)
    out = np.zeros_like(points)
    fn = _lib(_REF_PATH).aclref_skinned_points
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    if fn(local_pose.ctypes.data, parents.ctypes.data, inverse_bind.ctypes.data, local_pose.shape[0], points.ctypes.data, out.ctypes.data) != 0:
        raise RuntimeError("skinning: a parent does not precede its child")
    return out


def rows_to_axes(rows: np.ndarray) -> np.ndarray:
    """The library's skinning rows [..., 12] as the 3x4 matrix's axes [..., 4, 3] (x_axis, y_axis, z_axis, w_axis): one transpose."""
    return np.swapaxes(np.asarray(rows).reshape(rows.shape[:-1] + (3, 4)), -1, -2)
