"""ctypes binding of the additive oracle (oracle/additive.mk): additive clips compressed by the unmodified reference and its
acl::apply_additive_to_base (core/additive_utils.h:152-162), from _ref/libaclref_additive.so where it was built. TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import ref

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_PATH = os.path.join(_HERE, "_ref", "libaclref_additive.so")
_lib = None


def reference_available() -> bool:
    return os.path.exists(_REF_PATH)


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(_REF_PATH)
        l.aclref_compress_additive.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
        l.aclref_apply_additive_to_base.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        l.aclref_apply_additive_to_base.restype = None
        l.aclref_free.argtypes = [C.c_void_p]
        _lib = l
    return _lib


def compress_additive(base_spec: ref.TransformSpec, spec: ref.TransformSpec, additive_format: int) -> np.ndarray:
    """The additive clip of `spec` over `base_spec` in `additive_format` (1 relative, 2 additive0, 3 additive1), as blob bytes."""
    c_base, c_spec = base_spec.to_c(), spec.to_c()
    ptr, size = C.c_void_p(), C.c_uint32()
    rc = lib().aclref_compress_additive(C.byref(c_base), C.byref(c_spec), additive_format, C.byref(ptr), C.byref(size))
    if rc != 0:
        raise RuntimeError(f"reference additive compression failed ({rc})")
    buf = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(size.value,))
    out = ref.aligned_blob(buf.copy())
    lib().aclref_free(ptr)
    return out


def apply_additive_to_base(additive_format: int, base_pose: np.ndarray, additive_pose: np.ndarray) -> np.ndarray:
    """The reference's apply_additive_to_base on every bone of one pose, float32 [num_tracks][12] each."""
    base_pose = np.ascontiguousarray(base_pose, dtype=np.float32)
    additive_pose = np.ascontiguousarray(additive_pose, dtype=np.float32)
    assert base_pose.shape == additive_pose.shape
    out = np.zeros_like(base_pose)
    lib().aclref_apply_additive_to_base(additive_format, base_pose.ctypes.data, additive_pose.ctypes.data, base_pose.shape[0], out.ctypes.data)
    return out
