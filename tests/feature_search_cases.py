"""Motion matching cases (aclb200_pack_pose_features, aclb200_search_pose_features): fabricated feature rows and terms, the pack restated
in numpy float32, and the cost and the search restated in exact rational arithmetic. The oracle (oracle/feature_search.py) is checked
against these on the CPU; the GPU tests compare the library with the oracle."""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from acl_b200.api import FEATURE_DIRECTION, FEATURE_POSITION, FEATURE_VELOCITY, make_feature_terms

NO_ROW = 0xFFFFFFFF
KINDS = (FEATURE_POSITION, FEATURE_DIRECTION, FEATURE_VELOCITY)


def fabricated_rows(rng, num_requests: int, num_offsets: int, bones_per_list: int) -> np.ndarray:
    """float32 [R][S * K][12] qvvf rows: unit rotations, translations a few units across, scale 1, both w lanes 0"""
    rows = np.zeros((num_requests, num_offsets * bones_per_list, 12), np.float32)
    q = rng.normal(size=(num_requests, num_offsets * bones_per_list, 4))
    rows[..., 0:4] = (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)
    rows[..., 4:7] = rng.uniform(-3.0, 3.0, size=(num_requests, num_offsets * bones_per_list, 3)).astype(np.float32)
    rows[..., 8:11] = 1.0
    return rows


def every_term(num_offsets: int, bones_per_list: int, inv_dt: float = 30.0) -> np.ndarray:
    """every kind x component mask (1..7) x direction axis, on rows spread over the S x K rows"""
    kinds, s0, s1, k, axis, masks = [], [], [], [], [], []
    i = 0
    for kind in KINDS:
        for mask in range(1, 8):
            for a in (range(3) if kind == FEATURE_DIRECTION else [0]):
                kinds.append(kind)
                s0.append(i % num_offsets)
                s1.append((i + 1) % num_offsets)
                k.append((i // num_offsets) % bones_per_list)
                axis.append(a)
                masks.append(mask)
                i += 1
    return make_feature_terms(kinds, s0, k, masks, s1, axis, inv_dt)


def pinned_direction(rotation, axis: int) -> np.ndarray:
    """rtm::quat_mul_vector3(e_axis, rotation) through the port's qvv_inverse, pinned to the reference's in tests/test_root_motion_oracle.py:
    qvv_inverse({conjugate(rotation), e_axis, scale 1}) has translation -quat_mul_vector3(e_axis * 1, rotation), every step exact but the
    rotation itself (the conjugate's and the negation's sign flips, the multiply by 1 / 1)."""
    from oracle import root_motion as RM
    rotation = np.asarray(rotation, np.float32)
    row = np.zeros(12, np.float32)
    row[0:3] = -rotation[0:3]
    row[3] = rotation[3]
    row[4 + axis] = 1.0
    row[8:11] = 1.0
    return -RM.port_qvv_inverse(row)[4:7]


def numpy_pack(rows: np.ndarray, bones_per_list: int, terms: np.ndarray, mean=None, scale=None) -> np.ndarray:
    """rows: float32 [R][S * K][12]. The pack in numpy float32 (each operation one IEEE rounding), directions from pinned_direction."""
    f32 = np.float32
    out = []
    for r in range(rows.shape[0]):
        vector = []
        for term in terms:
            first = rows[r, int(term["s0"]) * bones_per_list + int(term["k"])]
            second = rows[r, int(term["s1"]) * bones_per_list + int(term["k"])]
            if term["kind"] == FEATURE_POSITION:
                v = first[4:7]
            elif term["kind"] == FEATURE_DIRECTION:
                v = pinned_direction(first[0:4], int(term["axis"]))
            else:
                v = (second[4:7] - first[4:7]) * f32(term["inv_dt"])
            vector += [f32(v[c]) for c in range(3) if int(term["components"]) & (1 << c)]
        out.append(vector)
    out = np.array(out, np.float32)
    m = np.zeros(out.shape[1], np.float32) if mean is None else np.asarray(mean, np.float32)
    s = np.ones(out.shape[1], np.float32) if scale is None else np.asarray(scale, np.float32)
    return ((out - m).astype(np.float32) * s).astype(np.float32)


def round_f32(x: Fraction) -> Fraction:
    """x rounded to the nearest float32, ties to even (subnormals included; beyond the largest float: inf as a float)"""
    if x == 0:
        return Fraction(0)
    sign = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    quantum = Fraction(2) ** (max(e, -126) - 23)
    m = a / quantum
    n = m.numerator // m.denominator
    rest = m - n
    if rest > Fraction(1, 2) or (rest == Fraction(1, 2) and n % 2 == 1):
        n += 1
    result = n * quantum
    if result >= Fraction(2) ** 128:
        return sign * Fraction(10) ** 60        # stands for inf: compared through as_float32
    return sign * result


def as_float32(x: Fraction) -> np.float32:
    return np.float32(np.inf) if abs(x) > Fraction(2) ** 128 else np.float32(float(x))


def exact_cost(query, row) -> np.float32:
    """acc = +0; acc = fmaf(diff, diff, acc) with diff = q[d] - x[d]: each step rounded once, from exact rationals (finite inputs)"""
    acc = Fraction(0)
    for q, x in zip(np.asarray(query, np.float32), np.asarray(row, np.float32)):
        diff = round_f32(Fraction(float(q)) - Fraction(float(x)))
        acc = round_f32(diff * diff + acc)
    return as_float32(acc)


def unfused_cost(query, row) -> np.float32:
    acc = np.float32(0)
    for q, x in zip(np.asarray(query, np.float32), np.asarray(row, np.float32)):
        diff = np.float32(q - x)
        acc = np.float32(acc + np.float32(diff * diff))
    return acc


def reference_search(database, query_vectors, queries, num_dims: int, row_tags=None, cost=None) -> list[tuple[int, np.float32]]:
    """The selection rules written out: (row, cost) per query, by scanning rows in order and keeping a strictly smaller cost"""
    cost = cost or (lambda q, x: np.float32(_float_cost(q, x)))
    out = []
    for q, info in enumerate(queries):
        best = (NO_ROW, np.float32(np.inf))
        for r in range(database.shape[0]):
            tag = 0xFFFFFFFF if row_tags is None else int(row_tags[r])
            if tag & int(info["tag_mask"]) == 0 or int(info["exclude_begin"]) <= r < int(info["exclude_end"]):
                continue
            c = cost(query_vectors[q, :num_dims], database[r, :num_dims])
            if np.isnan(c):
                continue
            if best[0] == NO_ROW or c < best[1]:
                best = (r, c)
        out.append(best)
    return out


def _float_cost(query, row):
    from oracle import feature_search as FS
    return FS.cost(query, row)


def key(row: int, cost) -> int:
    """(cost bits << 32) | row: what the search minimises"""
    return (int(np.float32(cost).view(np.uint32)) << 32) | int(row)
