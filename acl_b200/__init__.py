"""acl_b200 -- H100-native (sm_90a) batched decompression of nfrechette/acl `compressed_tracks`.

The product is the C-ABI shared library `acl_b200/libaclb200.so` (sources in acl_b200/csrc/, interface in
include/aclb200.h, C++ header shim in include/acl_b200/decompress.h). This Python package is only the thin
ctypes binding the tests and bench.py drive it through; it holds no decode logic and has no CPU fallback:
importing it without the built library, or creating a Context without a CUDA device, raises.
"""
from .api import (  # noqa: F401
    AclB200Error, Context, ClipSet, Database, Options, library_path, make_requests, TIER_MEDIUM, TIER_LOW,
    ROUND_NONE, ROUND_FLOOR, ROUND_CEIL, ROUND_NEAREST, ROUND_PER_TRACK,
    LOOP_CLAMP, LOOP_WRAP, LOOP_AS_COMPRESSED,
    NORMALIZE_NEVER, NORMALIZE_LERP_ONLY, NORMALIZE_ALWAYS,
    DEFAULT_SKIPPED, DEFAULT_CONSTANT, DEFAULT_VARIABLE, DEFAULT_LEGACY,
    LAYOUT_QVV48, LAYOUT_QVV40, MATH_EXACT, MATH_FAST, TRACK_QVVF,
    SKIP_ROTATION, SKIP_TRANSLATION, SKIP_SCALE,
    ERROR_JOB_DTYPE, TRACK_ERROR_DTYPE, ERROR_FLAG_NEGATIVE_SCALE, ERROR_FLAG_INVALID_SKELETON, ERROR_FLAG_WRAP_CLIP_CYCLE,
    OBJECT_QVVF, OBJECT_MATRIX3X4F,
    ADDITIVE_NONE, ADDITIVE_RELATIVE, ADDITIVE_ADDITIVE0, ADDITIVE_ADDITIVE1, ADDITIVE_REQUEST_DTYPE, make_additive_requests,
    BLEND_REQUEST_DTYPE, make_blend_requests,
    LAYER_OFF, LAYER_BLEND, LAYER_ADDITIVE, LAYER_NO_MASK, MAX_LAYERS, LAYER_DTYPE, make_layers,
    NO_BONE, MAX_QUERY_BONES,
    MAX_ROOT_MOTION_CYCLES, ROOT_MOTION_REQUEST_DTYPE, make_root_motion_requests,
    FEATURE_CLAMP, FEATURE_LOOP, MAX_FEATURE_OFFSETS, FEATURE_REQUEST_DTYPE, make_feature_requests,
    FEATURE_POSITION, FEATURE_DIRECTION, FEATURE_VELOCITY, MAX_FEATURE_DIMS, NO_ROW, FEATURE_TERM_DTYPE, SEARCH_QUERY_DTYPE,
    SEARCH_RESULT_DTYPE, make_feature_terms, feature_term_dims, make_search_queries,
    NO_INERTIALIZATION, INERTIALIZATION_DTYPE, make_inertializations, INERTIALIZED_REQUEST_DTYPE, make_inertialized_requests,
    MIRROR_X, MIRROR_Y, MIRROR_Z, ERROR_FLAG_INVALID_MIRROR, MIRROR_ENTRY_DTYPE, MIRRORED_REQUEST_DTYPE, make_mirrored_requests, mirror_table,
    mirror_rows_table,
)
