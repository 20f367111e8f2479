"""Additive clips shared by the additive tests: a base clip with animated and mirrored scale, and the relative, additive0 and additive1
clips the reference's compressor writes for a second animation over it (oracle/ref_additive.cpp). The blobs and the reference's
decode-and-apply poses are committed under tests/golden/ (tests/golden/make_additive_golden.py)."""
from __future__ import annotations

import hashlib

import numpy as np

from oracle import ref
from tests import clips

T = ref.TransformSpec
BASE_SPEC = T(num_tracks=24, num_samples=40, seed=4100, rot_default_pct=10, trans_default_pct=10, trans_constant_pct=40,
              scale_default_pct=30, scale_constant_pct=20, negative_scale_pct=8)
FULL_SPEC = T(num_tracks=24, num_samples=31, seed=4101, rot_default_pct=10, trans_default_pct=10, trans_constant_pct=40,
              scale_default_pct=30, scale_constant_pct=20, negative_scale_pct=8)
BASE = "additive_base"
FORMATS = {"additive_relative": 1, "additive_additive0": 2, "additive_additive1": 3}     # acl::additive_clip_format8
NAMES = [BASE] + list(FORMATS)

# sha256 of the committed blobs: the reference's compressor may emit other bytes on another x86 CPU, where regeneration is skipped
BLOB_SHA256 = {
    "additive_base": "43502f373959f4518a12f4942d91610e40d3c791bad6dd3e237a0e6abecf176f",
    "additive_relative": "a48aa14194250417ec2456b2970761a16908fe96480c52a4398e8df1ce2bfb6c",
    "additive_additive0": "e00e77fae31ca55738c9485a11772c82588b5733698c9da0168900fa8ded361a",
    "additive_additive1": "bd1424c2be14972e3d3bff21a1869199d73b979b4b33e65829daa3d6014caeb9",
}

# (settings kind, rounding, looping) triples of the golden poses, and the (base time, additive time) pairs
COMBOS = [(0, 0, 2), (0, 1, 0), (0, 3, 1), (1, 0, 2), (3, 2, 0), (4, 0, 1)]


def time_pairs() -> np.ndarray:
    base_times = clips.sample_times(BASE_SPEC)
    full_times = clips.sample_times(FULL_SPEC)
    rng = np.random.default_rng(4102)
    return np.stack([np.concatenate([base_times, rng.permutation(base_times)]),
                     np.concatenate([np.resize(full_times, base_times.size), np.resize(rng.permutation(full_times), base_times.size)])],
                    axis=1).astype(np.float32)


def blob_sha256(blob: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(blob[:int(blob[0:4].view(np.uint32)[0])]).tobytes()).hexdigest()


def load(name: str) -> np.ndarray:
    return clips.load_blob(name)


def reference_pose(additive_lib, format_, base_blob, additive_blob, base_time, additive_time, kind, rounding, looping) -> np.ndarray:
    """decompress base + decompress additive (track_writer defaults) + apply_additive_to_base, all by the unmodified reference"""
    base = ref.decompress_tracks(base_blob, float(base_time), rounding, looping, settings=kind)
    additive = ref.decompress_tracks(additive_blob, float(additive_time), rounding, looping, settings=kind)
    return additive_lib.apply_additive_to_base(format_, base, additive)


def writer_settings(port, kind: int, **kw):
    """the port's settings of a settings kind with the track_writer defaults (what the additive half of a pair decodes with)"""
    defaults = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)
    return port.settings_for_kind(kind, default_modes=(port.DEFAULT_CONSTANT, port.DEFAULT_CONSTANT, port.DEFAULT_LEGACY),
                                  constant_defaults=defaults, **kw)


def port_pose(port, format_, base_blob, additive_blob, base_time, additive_time, base_settings, additive_settings, rounding, looping,
              normalize_mode) -> np.ndarray:
    """the same through the port (oracle/acl_oracle.c); normalize_mode picks the flavour of the negative scale branch's quat_normalize"""
    base = port.transform_decompress_tracks(base_blob, base_settings, float(base_time), rounding, looping)
    additive = port.transform_decompress_tracks(additive_blob, additive_settings, float(additive_time), rounding, looping)
    return port.apply_additive_to_base(format_, base, additive, normalize_mode)
