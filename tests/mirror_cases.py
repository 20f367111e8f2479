"""Inputs of the mirror tests, seeded: fabricated QVV48 poses with +-0, +-inf, NaN, subnormal and non-unit lanes under tables with identity
corrections, half turns, general corrections, self-partnered rows and entries without a partner; reference decodes of named clips under a
general table; and a symmetric skeleton with a symmetric bind pose for the table helper. The reference's results on the first two are
pinned in tests/golden/mirror.golden.npz (tests/golden/make_mirror_golden.py)."""
from __future__ import annotations

import os

import numpy as np

from tests import clips

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mirror.golden.npz")
AXES = (0, 1, 2)
NAMED_CLIPS = ("c1_30bones", "mixed_scale", "stripped_loop")
NUM_ROWS = 24
ROOT = 0xFFFFFFFF


def entry_dtype() -> np.dtype:
    return np.dtype([("pre", np.float32, 4), ("post", np.float32, 4), ("mirror", np.uint32), ("reserved", np.uint32, 3)])


def unit(q) -> np.ndarray:
    q = np.asarray(q, np.float64)
    return (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)


def _table(pre, post, mirror) -> np.ndarray:
    t = np.zeros(len(mirror), entry_dtype())
    t["pre"], t["post"], t["mirror"] = pre, post, mirror
    t["reserved"] = 0xDEADBEEF        # ignored
    return t


def fabricated_table() -> np.ndarray:
    """NUM_ROWS entries: pairs (0,1) .. with general corrections, identity and half turn corrections, a self-partnered row (12), a row
    naming a row out of range (13), a row naming a row paired with another (14 -> 15 while 15 and 16 pair), non-unit corrections"""
    rng = np.random.default_rng(21)
    n = NUM_ROWS
    pre = unit(rng.normal(size=(n, 4)))
    post = unit(rng.normal(size=(n, 4)))
    identity = np.array([0, 0, 0, 1], np.float32)
    pre[2:4] = identity
    post[2:4] = identity
    pre[4], post[4] = [1, 0, 0, 0], [0, 0, 0, 1]            # half turn about x
    pre[5], post[5] = [0, 1, 0, 0], [0, 0, -1, 0]           # about y, then z
    pre[20:22] *= np.float32(1.003)                         # non-unit corrections
    post[22:24] *= np.float32(0.97)
    mirror = np.arange(n, dtype=np.uint32) ^ 1
    mirror[12] = 12
    mirror[13] = n + 5
    mirror[14], mirror[15], mirror[16], mirror[17] = 15, 16, 15, 17
    return _table(pre, post, mirror)


def fabricated_poses() -> np.ndarray:
    """float32 [6][NUM_ROWS][12]: unit and non-unit rotations, +-0 and special lanes in every position, w lanes 0"""
    rng = np.random.default_rng(22)
    n = NUM_ROWS
    poses = np.zeros((6, n, 12), np.float32)
    poses[:, :, 0:4] = unit(rng.normal(size=(6, n, 4)))
    poses[:, :, 4:7] = rng.normal(size=(6, n, 3)) * 3
    poses[:, :, 8:11] = rng.uniform(0.2, 2.0, size=(6, n, 3))
    poses[1, :, 0:4] *= np.float32(1.0005)                  # not unit, as a lerp leaves them
    poses[2, :, 8:11] *= -1                                  # negative scale is copied
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0e-40, -1.0e-40, 3.0e38, -0.0, 0.0], np.float32)
    lanes = [0, 1, 2, 3, 4, 5, 6, 8, 9, 10]
    for p in (3, 4, 5):
        for r in range(n):
            for k, lane in enumerate(lanes):
                if (r + k + p) % 4 == 0:
                    poses[p, r, lane] = special[(r * 3 + k + p) % special.size]
    # a NaN with a payload, and signed zeros in whole rows
    poses[5, 7, 4] = np.uint32(0x7FC01234).view(np.float32)
    poses[4, 9, 0:7] = -0.0
    poses[:, :, 7] = 0.0
    poses[:, :, 11] = 0.0
    return poses


def named_table(num_rows: int) -> np.ndarray:
    """bones paired (0,1), (2,3) .. with general corrections; the last bone of an odd count mirrors itself"""
    rng = np.random.default_rng(23 + num_rows)
    mirror = np.arange(num_rows, dtype=np.uint32) ^ 1
    if num_rows % 2:
        mirror[-1] = num_rows - 1
    return _table(unit(rng.normal(size=(num_rows, 4))), unit(rng.normal(size=(num_rows, 4))), mirror)


def named_poses(name: str) -> np.ndarray:
    """the reference decodes pinned for the clip, as float32 [poses][num_tracks][12] QVV48 rows"""
    g = np.load(clips.golden_path(name, "golden.npz"))["poses"]
    rows40 = g.reshape(-1, g.shape[-2], 10).astype(np.float32)
    out = np.zeros(rows40.shape[:2] + (12,), np.float32)
    out[..., 0:7] = rows40[..., 0:7]
    out[..., 8:11] = rows40[..., 7:10]
    return out


# ---- float64 qvv math for the table helper and the tolerance checks (scale 1: rotations and translations) ----
def qmul(a, b) -> np.ndarray:
    """the Hamilton product a b of xyzw quaternions (rtm's quat_mul(b, a)), broadcasting"""
    ax, ay, az, aw = np.moveaxis(np.asarray(a, np.float64), -1, 0)
    bx, by, bz, bw = np.moveaxis(np.asarray(b, np.float64), -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)


def conj(q) -> np.ndarray:
    return np.asarray(q, np.float64) * np.array([-1.0, -1.0, -1.0, 1.0])


def rotate(v, q) -> np.ndarray:
    """v rotated by q"""
    v4 = np.concatenate([np.asarray(v, np.float64), np.zeros(np.shape(v)[:-1] + (1,))], axis=-1)
    return qmul(qmul(q, v4), conj(q))[..., :3]


def to_object(local: np.ndarray, parents) -> np.ndarray:
    """[n][12] local rows (scale 1) to object rows in float64"""
    out = np.array(local, np.float64)
    for b, p in enumerate(parents):
        if p != ROOT:
            out[b, 0:4] = qmul(out[p, 0:4], local[b, 0:4])
            out[b, 4:7] = out[p, 4:7] + rotate(local[b, 4:7], out[p, 0:4])
    return out


def relative_to(rows: np.ndarray, frame: np.ndarray) -> np.ndarray:
    """rows expressed in the frame of the `frame` row (scale 1): rotation conj(F) q, translation conj(F) (t - F.t)"""
    out = np.array(rows, np.float64)
    out[..., 0:4] = qmul(conj(frame[0:4]), rows[..., 0:4])
    out[..., 4:7] = rotate(rows[..., 4:7] - frame[4:7], conj(frame[0:4]))
    return out


def symmetric_skeleton():
    """(parents, mirror bones, bind object rotations, local bind rows [n][12]) of a 12 bone skeleton mirrored across x = 0: root and spine
    on the plane, two arms and two legs. Object rotations are arbitrary (the corrections absorb them); positions are symmetric."""
    parents = np.array([ROOT, 0, 1, 2, 3, 1, 5, 6, 0, 8, 0, 10], np.uint32)
    mirror = np.array([0, 1, 5, 6, 7, 2, 3, 4, 10, 11, 8, 9], np.uint32)
    rng = np.random.default_rng(24)
    n = parents.size
    positions = np.zeros((n, 3))
    positions[0] = [0.0, 1.0, 0.1]
    positions[1] = [0.0, 1.4, 0.0]
    for b in (2, 3, 4, 8, 9):
        positions[b] = rng.uniform(0.1, 1.0, 3) * [1, 1, 1]
    for b in (2, 3, 4, 8, 9):
        positions[mirror[b]] = positions[b] * [-1, 1, 1]
    rotations = unit(rng.normal(size=(n, 4))).astype(np.float64)
    local = np.zeros((n, 12))
    local[:, 8:11] = 1.0
    for b in range(n):
        p = parents[b]
        if p == ROOT:
            local[b, 0:4], local[b, 4:7] = rotations[b], positions[b]
        else:
            local[b, 0:4] = qmul(conj(rotations[p]), rotations[b])
            local[b, 4:7] = rotate(positions[b] - positions[p], conj(rotations[p]))
    return parents, mirror, rotations.astype(np.float32), local.astype(np.float32)


def random_local_poses(num_poses: int, num_bones: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    poses = np.zeros((num_poses, num_bones, 12), np.float32)
    poses[..., 0:4] = unit(rng.normal(size=(num_poses, num_bones, 4)))
    poses[..., 4:7] = rng.normal(size=(num_poses, num_bones, 3))
    poses[..., 8:11] = 1.0
    return poses
