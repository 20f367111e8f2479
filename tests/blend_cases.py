"""Blend fixtures shared by the blend tests: two clips of equal track count compressed by the reference (with default bones both clips
share, so identity rotations and unit scales meet themselves, and mirrored-scale bones), fabricated pose pairs that pin the hemisphere
bias of rtm::quat_lerp, and the weights. The blobs and the reference's decode-and-lerp poses are committed under tests/golden/
(tests/golden/make_blend_golden.py)."""
from __future__ import annotations

import hashlib

import numpy as np

from oracle import ref
from tests import clips

T = ref.TransformSpec
FROM_SPEC = T(num_tracks=24, num_samples=40, seed=4200, rot_default_pct=30, rot_constant_pct=20, trans_default_pct=30, trans_constant_pct=30,
              scale_default_pct=40, scale_constant_pct=20, negative_scale_pct=8)
TO_SPEC = T(num_tracks=24, num_samples=31, seed=4201, rot_default_pct=30, rot_constant_pct=20, trans_default_pct=30, trans_constant_pct=30,
            scale_default_pct=40, scale_constant_pct=20, negative_scale_pct=8, rotation_offset=3.14159)     # W near 0: some dots go negative
NAMES = ["blend_from", "blend_to"]
MIRRORED_BONES = [b for b in range(FROM_SPEC.num_tracks) if (b * 7 + 3) % 100 < FROM_SPEC.negative_scale_pct]

# sha256 of the committed blobs: the reference's compressor may emit other bytes on another x86 CPU, where regeneration is skipped
BLOB_SHA256 = {
    "blend_from": "90c646b09fa3051ddf70bb0fb5674ed59c0f602bd95d938cc501702b382c2530",
    "blend_to": "54a8e0b3a2e5edbd3f431e4a502a9e65e20a2306045252be044f6612af859ec0",
}

# (settings kind, rounding, looping) triples of the golden poses, the weights (0 and 1 give the end poses, -0.25 and 1.25 extrapolate)
COMBOS = [(0, 0, 2), (0, 1, 0), (0, 3, 1), (1, 0, 2), (3, 2, 0), (4, 0, 1)]
WEIGHTS = np.array([0.0, 1.0, 0.5, -0.25, 1.25], np.float32)

# rotations are bit-identical to the port's IEEE flavour and within this of the reference (rsqrtss + Newton-Raphson against 1 / sqrt:
# 1 ulp seen); translations and scales are bit-identical to the reference
ROTATION_GATE = 1e-6


def time_pairs() -> np.ndarray:
    """(from time, to time) pairs: every other sample of the from clip and shuffled times of the to clip, plus times past both ends"""
    rng = np.random.default_rng(4202)
    from_times = np.concatenate([clips.sample_times(FROM_SPEC)[::2], [-0.1, 5.0, 0.0, 1.3]])
    to_times = np.resize(rng.permutation(clips.sample_times(TO_SPEC)), from_times.size)
    return np.stack([from_times, to_times], axis=1).astype(np.float32)


def blob_sha256(blob: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(blob[:int(blob[0:4].view(np.uint32)[0])]).tobytes()).hexdigest()


def load(name: str) -> np.ndarray:
    return clips.load_blob(name)


def _row(rotation, translation=(0.0, 0.0, 0.0), scale=(1.0, 1.0, 1.0)) -> np.ndarray:
    return np.array(list(rotation) + list(translation) + [0.0] + list(scale) + [0.0], np.float32)


def fabricated_pairs() -> tuple[list[str], np.ndarray, np.ndarray]:
    """(names, from rows, to rows), float32 [n][12] each: one bone per named case, then random unit pairs
      dot_minus_zero   dot == -0.0: the sign bit flips `to` (the scalar and NEON paths' dot >= 0 would not)
      dpps_order       products 1, -2^-30, -1, 0: (x + y) + (z + w) = +0 keeps `to`, (x + z) + (y + w) = -2^-30 would flip it
      identical        the same unit rotation on both sides (what slerp turns into NaN)
      antipodal        q and -q: the flip makes them the same rotation
      mirrored         a mirrored scale lerped towards an unmirrored one"""
    tiny = np.float32(2.0 ** -15)
    q = np.array([0.1, -0.2, 0.3, 0.927], np.float32)
    q /= np.sqrt(np.sum(q.astype(np.float64) ** 2)).astype(np.float32)
    named = {
        "dot_minus_zero": (_row([1.0, 0.0, 0.0, 0.0], (1.0, 2.0, 3.0)), _row([-0.0, -0.48, -0.6, -0.64], (-1.0, 0.5, 2.0), (2.0, 2.0, 2.0))),
        "dpps_order": (_row([1.0, tiny, 1.0, 0.0], (0.25, 0.0, -3.0)), _row([1.0, -tiny, -1.0, 0.0], (4.0, -1.0, 1e-3), (0.5, 1.0, 3.0))),
        "identical": (_row(q, (1.0, 1.0, 1.0)), _row(q, (1.0, 1.0, 1.0))),
        "antipodal": (_row(q, (0.0, -2.0, 0.0)), _row(-q, (3.0, 2.0, 1.0), (1.0, 0.25, 1.0))),
        "mirrored": (_row(q, scale=(-1.0, 1.0, 1.0)), _row([0.0, 0.0, 0.0, 1.0], scale=(1.0, 1.5, 1.0))),
    }
    rng = np.random.default_rng(4203)
    n = 251
    rot = rng.normal(size=(2, n, 4)).astype(np.float32)
    rot /= np.sqrt(np.sum(rot.astype(np.float64) ** 2, axis=2, keepdims=True)).astype(np.float32)
    rows = np.zeros((2, n, 12), np.float32)
    rows[:, :, 0:4] = rot
    rows[:, :, 4:7] = rng.uniform(-5, 5, (2, n, 3))
    rows[:, :, 8:11] = rng.uniform(-2, 2, (2, n, 3))
    names = list(named) + [f"random_{i}" for i in range(n)]
    from_rows = np.concatenate([np.stack([v[0] for v in named.values()]), rows[0]])
    to_rows = np.concatenate([np.stack([v[1] for v in named.values()]), rows[1]])
    return names, from_rows, to_rows


def reference_pose(blend_lib, from_blob, to_blob, tf, tt, weight, kind, rounding, looping) -> np.ndarray:
    """decompress from + decompress to + rtm::qvv_lerp, all by the unmodified reference"""
    from_pose = ref.decompress_tracks(from_blob, float(tf), rounding, looping, settings=kind)
    to_pose = ref.decompress_tracks(to_blob, float(tt), rounding, looping, settings=kind)
    return blend_lib.reference_qvv_lerp(from_pose, to_pose, float(weight))


def port_pose(port, blend_lib, from_blob, to_blob, tf, tt, weight, settings, rounding, looping, normalize_mode) -> np.ndarray:
    """the same through the port (oracle/acl_oracle.c, oracle/blend_oracle.c): both halves decode with the same settings"""
    from_pose = port.transform_decompress_tracks(from_blob, settings, float(tf), rounding, looping)
    to_pose = port.transform_decompress_tracks(to_blob, settings, float(tt), rounding, looping)
    return blend_lib.port_qvv_lerp(from_pose, to_pose, float(weight), normalize_mode)
