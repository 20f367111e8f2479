"""Skeletons and inverse bind matrices shared by the skinning tests and tests/golden/make_skinning_golden.py.

Inverse binds are [n][12] float32: the xyz lanes of x_axis, y_axis, z_axis, w_axis of an rtm::matrix3x4f, the layout
ACLB200_OBJECT_MATRIX3X4F writes. In rtm's row vector order the full 4x4 matrix has these four axes as its rows and (0, 0, 0, 1) as its
last column, so p' = (p, 1) @ M.
"""
from __future__ import annotations

import numpy as np

from oracle import object_space

ROOT = 0xFFFFFFFF
SKELETONS = ["chain", "tree", "star", "random"]
# clips and sample times of tests/golden/skinning.golden.npz: mixed_scale and c2_100bones have children in a later chunk of 32 bones than
# their parents under every skeleton but the star
GOLDEN_CLIPS = ["c1_30bones", "mixed_scale", "c2_100bones"]
GOLDEN_TIMES = np.array([0.0, 0.41, 1.3], np.float32)


def skeleton(kind: str, n: int, seed: int = 0) -> np.ndarray:
    bones = np.arange(n)
    if kind == "chain":
        return np.where(bones == 0, ROOT, bones - 1).astype(np.uint32)
    if kind == "star":
        return np.where(bones == 0, ROOT, 0).astype(np.uint32)
    if kind == "random":
        rng = np.random.default_rng(seed)
        parents = np.array([ROOT] + [int(rng.integers(0, b)) for b in range(1, n)], np.uint32)
        parents[rng.random(n) < 0.1] = ROOT
        return parents
    return np.where(bones == 0, ROOT, (bones - 1) // 2).astype(np.uint32)


def to_affine(axes: np.ndarray) -> np.ndarray:
    """[..., 12] axes -> [..., 4, 4] float64 row vector matrices"""
    axes = np.asarray(axes, np.float64).reshape(axes.shape[:-1] + (4, 3))
    out = np.zeros(axes.shape[:-2] + (4, 4))
    out[..., :, :3] = axes
    out[..., 3, 3] = 1.0
    return out


def from_affine(m: np.ndarray) -> np.ndarray:
    """[..., 4, 4] row vector matrices -> [..., 12] float32 axes"""
    return np.ascontiguousarray(m[..., :, :3], dtype=np.float32).reshape(m.shape[:-2] + (12,))


def bind_inverse(bind_local: np.ndarray, parents: np.ndarray) -> np.ndarray:
    """The inverse of each bone's bind pose object matrix (the matrix walk of the port), inverted in float64."""
    return from_affine(np.linalg.inv(to_affine(object_space.port_local_to_object_space_matrix(bind_local, parents))))


def random_affine(n: int, seed: int, mirrored: bool = False) -> np.ndarray:
    """Rotation, non-uniform scale in [0.5, 2] and translation in [-3, 3] per bone; `mirrored` negates one scale axis on every other bone."""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    x, y, z, w = q.T
    rotation = np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], -1),
        np.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], -1),
        np.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    scale = rng.uniform(0.5, 2.0, (n, 3))
    if mirrored:
        scale[::2, rng.integers(0, 3)] *= -1.0
    m = np.zeros((n, 4, 4))
    m[:, :3, :3] = rotation * scale[:, :, None]
    m[:, 3, :3] = rng.uniform(-3.0, 3.0, (n, 3))
    m[:, 3, 3] = 1.0
    return from_affine(m)


def inverse_binds(kind: str, n: int, bind_local: np.ndarray, parents: np.ndarray, seed: int = 0) -> np.ndarray:
    if kind == "bind":
        return bind_inverse(bind_local, parents)
    return random_affine(n, seed, mirrored=kind == "mirrored")


INVERSE_BIND_KINDS = ["bind", "random", "mirrored"]
