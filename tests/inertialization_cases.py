"""Inputs of the inertialization tests, seeded: quaternions for rtm's log (near the identity on both sides of the 1 - 1e-6 select, w at +-1
and +-0, half turns, unnormalised), vectors for its exp (lengths on both sides of 1e-6, angles beyond pi where the sin and cos reduction
reflects), and transitions of four QVV48 poses with the signs of one side flipped so that abs() takes both branches. The reference's
results on them are pinned in tests/golden/inertialization.golden.npz (tests/golden/make_inertialization_golden.py)."""
from __future__ import annotations

import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inertialization.golden.npz")
NUM_TRACKS = 19
NUM_TRANSITIONS = 8
INV_DT = 30.0
# (elapsed, halflife) of the apply cases: the spring's start, its body, halflife 0, huge and negative elapsed, NaN in either
DECAYS = np.array([(0.0, 0.2), (0.016666668, 0.2), (0.1, 0.05), (0.35, 0.5), (1.0, 0.1), (0.05, 0.0), (1.0e6, 0.2), (-0.05, 0.2),
                   (0.1, -1.0e-5), (np.nan, 0.2), (0.1, np.nan), (np.inf, 0.2)], dtype=np.float32)


def _unit(q: np.ndarray) -> np.ndarray:
    q = q.astype(np.float64)
    return (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)


def log_inputs(with_nan: bool = True) -> np.ndarray:
    """float32 [n][4] xyzw"""
    rng = np.random.default_rng(11)
    out = [_unit(rng.normal(size=(600, 4)))]
    # near the identity: w on both sides of 1 - 1e-6 (and its float neighbours), small xyz
    edge = np.float32(1.0) - np.float32(1.0e-6)
    ws = [np.nextafter(edge, np.float32(2), dtype=np.float32), edge, np.nextafter(edge, np.float32(0), dtype=np.float32),
          np.float32(1.0), np.nextafter(np.float32(1), np.float32(0), dtype=np.float32), np.float32(1.0000001), np.float32(0.99999)]
    for w in ws:
        xyz = rng.normal(size=(16, 3)).astype(np.float32) * np.float32(np.sqrt(max(1.0 - float(w) ** 2, 1e-14)) / np.sqrt(3))
        out.append(np.concatenate([xyz, np.full((16, 1), w, np.float32)], axis=1))
    # w at -1, +-0 (half turns), near -1, the identity and its negation, zero and tiny xyz
    special = [[0, 0, 0, 1], [0, 0, 0, -1], [1, 0, 0, 0], [0, 1, 0, -0.0], [0, 0, -1, 0], [0.6, 0.8, 0, 0], [0.6, 0.8, 0, -0.0],
               [0, 0, 0, 0], [1e-20, 0, 0, 1], [1e-3, 0, 0, -0.9999995], [0, 0, 0, -0.0], [-0.0, -0.0, -0.0, 1]]
    out.append(np.array(special, np.float32))
    # unnormalised, as a decode's lerp leaves them: scaled by 1 +- a few ulp to 1e-3, and w beyond +-1 (clamped)
    base = _unit(rng.normal(size=(200, 4)))
    out.append(base * rng.uniform(0.999, 1.001, size=(200, 1)).astype(np.float32))
    out.append(np.array([[0.1, 0.0, 0.0, 1.2], [0.0, 0.2, 0.0, -1.5], [0.5, 0.5, 0.5, 0.5 + 1e-3]], np.float32))
    if with_nan:
        out.append(np.array([[0.1, 0.2, 0.3, np.nan], [np.nan, 0.0, 0.0, 0.5]], np.float32))
    return np.concatenate(out).astype(np.float32)


def exp_inputs() -> np.ndarray:
    """float32 [n][4] (xyz, w = 0)"""
    rng = np.random.default_rng(12)
    dirs = _unit(rng.normal(size=(1000, 3)))
    lengths = np.concatenate([rng.uniform(0.0, 3.2, 500), rng.uniform(3.2, 40.0, 300),
                              10.0 ** rng.uniform(-9, -4, 200)]).astype(np.float32)
    v = dirs * lengths[:, None]
    edge = np.float32(1.0e-6)
    around = np.array([np.nextafter(edge, np.float32(0), dtype=np.float32), edge, np.nextafter(edge, np.float32(1), dtype=np.float32)],
                      np.float32)
    extra = np.array([[around[0], 0, 0], [0, around[1], 0], [0, 0, around[2]], [0, 0, 0], [-0.0, 0, 0], [np.pi / 2, 0, 0],
                      [np.pi, 0, 0], [-np.pi, 0, 0], [0, 2 * np.pi, 0], [0, 0, 3 * np.pi / 2]], np.float32)
    v = np.concatenate([v, extra]).astype(np.float32)
    return np.concatenate([v, np.zeros((v.shape[0], 1), np.float32)], axis=1)


def poses(rng: np.random.Generator, num_poses: int, num_tracks: int = NUM_TRACKS) -> np.ndarray:
    """float32 [num_poses][num_tracks][12] QVV48 rows: unit rotations (a few slightly unnormalised), translations, positive scales"""
    p = np.zeros((num_poses, num_tracks, 12), np.float32)
    p[..., 0:4] = _unit(rng.normal(size=(num_poses, num_tracks, 4)))
    p[..., 0:4] *= rng.choice([1.0, 1.0, 1.0, 0.9995, 1.0004], size=(num_poses, num_tracks, 1)).astype(np.float32)
    p[..., 4:7] = rng.normal(size=(num_poses, num_tracks, 3)) * 0.5
    p[..., 8:11] = rng.uniform(0.5, 1.5, size=(num_poses, num_tracks, 3))
    return p


def transitions() -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """(src, src_prev, dst, dst_prev), each float32 [NUM_TRANSITIONS][NUM_TRACKS][12]. Each previous pose is its pose turned a little; the
    destination is either a random pose or the source turned by up to a half turn, and one in three rows is negated so that the double
    cover sends abs() down both branches."""
    rng = np.random.default_rng(13)
    n, b = NUM_TRANSITIONS, NUM_TRACKS
    src = poses(rng, n, b)
    dst = poses(rng, n, b)
    near = rng.random(size=(n, b)) < 0.5
    turned = _turn(src[..., 0:4], rng, rng.uniform(0.0, np.pi, size=(n, b)))
    dst[..., 0:4] = np.where(near[..., None], turned, dst[..., 0:4])
    out = []
    for p in (src, dst):
        prev = p.copy()
        prev[..., 0:4] = _turn(p[..., 0:4], rng, rng.uniform(0.0, 0.2, size=(n, b)))
        prev[..., 4:7] = p[..., 4:7] - rng.normal(size=(n, b, 3)).astype(np.float32) * np.float32(0.03)
        flip = rng.random(size=(n, b)) < 1 / 3
        prev[..., 0:4] = np.where(flip[..., None], -prev[..., 0:4], prev[..., 0:4])
        out.append(prev)
    flip = rng.random(size=(n, b)) < 1 / 3
    dst[..., 0:4] = np.where(flip[..., None], -dst[..., 0:4], dst[..., 0:4])
    return src, out[0], dst, out[1]


def _turn(q: np.ndarray, rng: np.random.Generator, angles: np.ndarray) -> np.ndarray:
    """q turned by `angles` about random axes (Hamilton r q), float32"""
    axis = rng.normal(size=q.shape[:-1] + (3,))
    axis /= np.linalg.norm(axis, axis=-1, keepdims=True)
    r = np.concatenate([axis * np.sin(angles / 2)[..., None], np.cos(angles / 2)[..., None]], axis=-1)
    return hamilton(r, q.astype(np.float64)).astype(np.float32)


def hamilton(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """The Hamilton product a b of xyzw quaternions (float64)"""
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], axis=-1)
