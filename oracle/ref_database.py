"""ctypes binding of oracle/_ref/libaclref_db.so (oracle/ref_database.cpp): the reference's streaming database path.
TEST INFRASTRUCTURE ONLY, built by oracle/database.mk where the reference tree exists; the prebuilt library travels with the tree."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import ref

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libaclref_db.so")
STREAM_IN, STREAM_OUT = 0, 1
TIER_MEDIUM, TIER_LOW = 1, 2
_lib = None


def available() -> bool:
    return os.path.exists(_LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(_LIB_PATH)
        l.aclref_build_database.argtypes = [C.c_void_p, C.c_uint32, C.c_float, C.c_float, C.c_uint32, C.c_void_p, C.c_void_p,
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
        l.aclref_decompress_tracks_database.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_float, C.c_uint32, C.c_uint32,
                                                        C.c_int32, C.c_void_p]
        l.aclref_free.argtypes = [C.c_void_p]
        _lib = l
    return _lib


def _take(ptr: int, size: int) -> np.ndarray:
    buf = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(size,))
    out = ref.aligned_blob(buf.copy())
    lib().aclref_free(ptr)
    return out


def build_database(specs: list[ref.TransformSpec], medium_proportion: float = 0.3, low_proportion: float = 0.3,
                   max_chunk_size: int = 4096) -> tuple[list[np.ndarray], np.ndarray]:
    """Compresses the clips of `specs` with database support and splits them with acl::build_database: (bound clips, database blob)."""
    n = len(specs)
    c_specs = (ref._TransformSpec * n)(*[s.to_c() for s in specs])
    clip_ptrs = (C.c_void_p * n)()
    clip_sizes = (C.c_uint32 * n)()
    db_ptr, db_size = C.c_void_p(), C.c_uint32()
    rc = lib().aclref_build_database(C.cast(c_specs, C.c_void_p), n, medium_proportion, low_proportion, max_chunk_size,
                                     C.cast(clip_ptrs, C.c_void_p), C.cast(clip_sizes, C.c_void_p), C.byref(db_ptr), C.byref(db_size))
    if rc != 0:
        raise RuntimeError(f"reference build_database failed ({rc})")
    return [_take(clip_ptrs[i], clip_sizes[i]) for i in range(n)], _take(db_ptr.value, db_size.value)


def decompress(clip: np.ndarray, database: np.ndarray, ops: list[tuple[int, int, int]], t: float, rounding: int = ref.ROUND_NONE,
               looping: int = ref.LOOP_AS_COMPRESSED, track_index: int = -1) -> np.ndarray:
    """decompression_context<debug settings + database>::initialize(tracks, db) after `ops` ((STREAM_IN / STREAM_OUT, tier, num_chunks)
    calls of a database_context with memcpy streamers), seek, decompress_tracks (or decompress_track). float32 [num_tracks, 12]."""
    out = np.zeros((ref.num_tracks_of(clip), 12), dtype=np.float32)
    flat = np.array([v for op in ops for v in op], dtype=np.uint32)
    rc = lib().aclref_decompress_tracks_database(clip.ctypes.data, database.ctypes.data, flat.ctypes.data if flat.size else None, len(ops),
                                                 t, rounding, looping, track_index, out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"reference database decompression failed ({rc})")
    return out
