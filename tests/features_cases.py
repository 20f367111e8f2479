"""Shared cases of the pose features tests (aclb200_extract_pose_features): the offset time u' and loop count c of each (request, offset)
pair, derived once here in numpy float32 as the kernel derives them, the offsets the tests sweep, and the composition of a row from its
three pieces in the port's or the reference's rtm operations.

Row (s, k) of request r is F = qvv_mul(qvv_mul(B, qvv_inverse(T)), M): B the object row of entry k at u', T the root's local row at u',
M root motion's row for {clip, t, u', c}."""
from __future__ import annotations

import numpy as np

CLAMP, LOOP = 0, 1
MAX_CYCLES = 256
# the database build offsets of tools/bench_features.py: one frame back, now, a third and two thirds of a second ahead
BENCH_OFFSETS = np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0], np.float32)


def offset_time(time, offset, looping: int, duration) -> tuple[bool, int, np.float32]:
    """(writes, c, u') of one (request, offset) pair: u = t + o; CLAMP keeps u (the seek clamps it); LOOP wraps it by
    c = floorf(u / D), u' = u - float(c) * D (IEEE divide, multiply, subtract, none fused), D == 0 gives c = 0, u' = 0. A looping value
    other than CLAMP / LOOP, a non-finite u under LOOP and |c| > 256 write nothing."""
    with np.errstate(all="ignore"):
        u = np.float32(np.float32(time) + np.float32(offset))
        if looping == CLAMP:
            return True, 0, u
        if looping != LOOP or not np.isfinite(u):
            return False, 0, u
        duration = np.float32(duration)
        if duration == 0:
            return True, 0, np.float32(0.0)
        cycle = np.floor(np.float32(u / duration))
        if not abs(cycle) <= MAX_CYCLES:
            return False, 0, u
        return True, int(cycle), np.float32(u - np.float32(cycle * duration))


def offsets_for(duration: float) -> list[np.ndarray]:
    """Offset sets (1 to 8 offsets) reaching: negative, zero and positive; exactly k * D; across 0, 1, 3, 256 and 257 loop boundaries"""
    d = np.float32(duration)
    sets = [
        np.array([0.0], np.float32),
        np.array([-0.25, 0.0, 0.1, 0.5], np.float32),
        np.array([-d, d, 2 * d, -3 * d, 0.0], np.float32),
        np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0, d * 1.5, -d * 3.5, d * 256.25, d * 257.5], np.float32),
    ]
    return [np.asarray(s, np.float32) for s in sets]


def request_times(duration: float) -> list[float]:
    """t: 0, D, inside the clip and beyond both ends"""
    d = np.float32(duration)
    return [0.0, float(d), float(np.float32(d * 0.37)), -0.2, float(np.float32(d + 0.3))]


def compose(rm, object_row, root_local, motion, normalize_mode=None, reference: bool = False) -> np.ndarray:
    """F from its pieces with oracle.root_motion's rtm operations: the port's (normalize_mode: its qvv_mul's flavour) or the reference's"""
    if reference:
        return rm.reference_qvv_mul(rm.reference_qvv_mul(object_row, rm.reference_qvv_inverse(root_local)), motion)
    mode = rm.NORMALIZE_IEEE if normalize_mode is None else normalize_mode
    return rm.port_qvv_mul(rm.port_qvv_mul(object_row, rm.port_qvv_inverse(root_local), mode), motion, mode)


def object_rows(port, local: np.ndarray, parents, bones, normalize_mode) -> np.ndarray:
    """The object rows of the listed bones through the bone query's closure: rows outside the closure are NaN before the port walk
    (tests/bones_cases.py; the rows of the listed bones do not depend on them), w lanes 0"""
    from tests import bones_cases
    n = local.shape[0]
    keep = bones_cases.closure(parents, bones, n)
    masked = np.full_like(local, np.nan)
    masked[keep] = local[keep]
    out = port.local_to_object_space(masked, bones_cases.effective_parents(parents), normalize_mode)
    out[:, 7] = 0.0
    out[:, 11] = 0.0
    return out
