"""ctypes binding of the motion matching oracle (oracle/feature_search.mk): the pack of aclb200_pack_pose_features and the search of
aclb200_search_pose_features restated in C (liboracle_feature_search.so). Arrays use the numpy views of acl_b200.api. TEST INFRASTRUCTURE
ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from acl_b200.api import FEATURE_TERM_DTYPE, SEARCH_QUERY_DTYPE, SEARCH_RESULT_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "liboracle_feature_search.so")
_handle = None


def _lib():
    global _handle
    if _handle is None:
        if not os.path.exists(_PATH):
            subprocess.run(["make", "-f", os.path.join(_HERE, "feature_search.mk"), "port"], check=True, capture_output=True)
        l = C.CDLL(_PATH)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        l.aclo_feature_direction.argtypes, l.aclo_feature_direction.restype = [vp, u32, vp], None
        l.aclo_pack_pose_features.argtypes = [vp, u32, u32, u64, vp, u32, vp, vp, vp, u64]
        l.aclo_pack_pose_features.restype = u32
        l.aclo_feature_cost.argtypes, l.aclo_feature_cost.restype = [vp, vp, u32], C.c_float
        l.aclo_search_pose_features.argtypes = [vp, u64, u64, vp, vp, vp, u32, u64, u32, vp]
        l.aclo_search_pose_features.restype = None
        _handle = l
    return _handle


def direction(rotation, axis: int) -> np.ndarray:
    """rtm::quat_mul_vector3(e_axis, rotation) of one xyzw rotation"""
    rotation, out = np.ascontiguousarray(rotation, dtype=np.float32).reshape(4), np.zeros(3, np.float32)
    _lib().aclo_feature_direction(rotation.ctypes.data, axis, out.ctypes.data)
    return out


def pack(rows: np.ndarray, num_requests: int, bones_per_list: int, pose_stride: int, terms: np.ndarray, mean=None, scale=None,
         out_stride: int | None = None, out: np.ndarray | None = None) -> np.ndarray:
    """rows: the bytes (or any array) of num_requests poses of extract_pose_features rows, pose_stride bytes apart. Returns float32
    [num_requests][out_stride]; the floats past D keep what `out` held (zeros when it is None)."""
    rows = np.ascontiguousarray(rows).view(np.uint8).reshape(-1)
    terms = np.ascontiguousarray(terms, dtype=FEATURE_TERM_DTYPE).reshape(-1)
    dims = int(sum(bin(int(c) & 7).count("1") for c in terms["components"]))
    stride = dims if out_stride is None else out_stride
    result = np.zeros((num_requests, stride), np.float32) if out is None else np.ascontiguousarray(out, dtype=np.float32).copy()
    assert num_requests == 0 or rows.size >= (num_requests - 1) * pose_stride
    stats = [None if a is None else np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in (mean, scale)]
    _lib().aclo_pack_pose_features(rows.ctypes.data, num_requests, bones_per_list, pose_stride, terms.ctypes.data, terms.size,
                                   *[None if a is None else a.ctypes.data for a in stats], result.ctypes.data, stride)
    return result


def cost(query, row) -> np.float32:
    query = np.ascontiguousarray(query, dtype=np.float32).reshape(-1)
    row = np.ascontiguousarray(row, dtype=np.float32).reshape(-1)
    assert query.size == row.size
    return np.float32(_lib().aclo_feature_cost(query.ctypes.data, row.ctypes.data, query.size))


def search(database: np.ndarray, query_vectors: np.ndarray, queries: np.ndarray, num_dims: int, row_tags=None) -> np.ndarray:
    """database: float32 [N][db_stride], query_vectors: float32 [Q][q_stride], queries: SEARCH_QUERY_DTYPE [Q]. Returns
    SEARCH_RESULT_DTYPE [Q]."""
    database = np.ascontiguousarray(database, dtype=np.float32)
    query_vectors = np.ascontiguousarray(query_vectors, dtype=np.float32)
    queries = np.ascontiguousarray(queries, dtype=SEARCH_QUERY_DTYPE).reshape(-1)
    tags = None if row_tags is None else np.ascontiguousarray(row_tags, dtype=np.uint32).reshape(-1)
    num_rows = database.shape[0] if database.ndim == 2 else 0
    db_stride = database.shape[1] if database.ndim == 2 else num_dims
    results = np.zeros(queries.size, SEARCH_RESULT_DTYPE)
    assert tags is None or tags.size == num_rows
    _lib().aclo_search_pose_features(database.ctypes.data, num_rows, db_stride, None if tags is None else tags.ctypes.data,
                                     query_vectors.ctypes.data, queries.ctypes.data, queries.size, query_vectors.shape[1], num_dims,
                                     results.ctypes.data)
    return results
