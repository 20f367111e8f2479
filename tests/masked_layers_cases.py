"""The masked layered decode's oracle: layers_cases' composition with a per-bone weight on every layer above the base and weighted ADDITIVE
layers, built from the per-operation oracles that are already pinned to the reference (the port's decode, oracle/blend.py's qvv_lerp on
single-bone rows for per-bone weights, the port's and the reference's apply_additive_to_base). A masked stack is a list of (clip, sample
time, op, weight, mask index or None) layers; mask m is masks[m][b] per bone b of the base clip.

At bone b a layer above the base acts with w_b = float32(weight * mask[b]) (its weight without a mask), and not at all where mask[b] is
+0 or -0. BLEND: running = qvv_lerp(running, layer, w_b). ADDITIVE: apply_additive_to_base(format, running, layer) when w_b == 1, else
apply_additive_to_base(format, running, qvv_lerp(writer defaults, layer, w_b)), the writer defaults being the identity rotation, zero
translation and the clip's default scale (1, or 0 for additive1 clips).
tests/golden/masked_layers.golden.npz holds the reference's composition of golden_stacks() (tests/golden/make_masked_layers_golden.py)."""
from __future__ import annotations

import numpy as np

from oracle import ref
from tests import blend_cases
from tests import layers_cases
from tests.layers_cases import ADDITIVE, BLEND, COMBOS, FORMATS, NAMES, OFF, load_blobs  # noqa: F401

NO_MASK = 0xFFFFFFFF
NUM_BONES = 24                                                       # every clip of NAMES


def default_scale_of(blob: np.ndarray) -> float:
    """the clip's default scale, tracks_header::misc_packed bit 1 (1.0, or 0.0 for additive1 clips)"""
    return float((int(blob[28:32].view(np.uint32)[0]) >> 1) & 1)


def writer_default_rows(n: int, scale: float) -> np.ndarray:
    """the track_writer default pose as n QVV48 rows"""
    row = np.array([0, 0, 0, 1, 0, 0, 0, 0, scale, scale, scale, 0], np.float32)
    return np.tile(row, (n, 1))


def bone_weights(layer, masks, n: int):
    """(w_b as float32[n], skipped as bool[n]) of one layer"""
    _, _, _, weight, mask = layer
    w = np.full(n, np.float32(weight), np.float32)
    if mask is None:
        return w, np.zeros(n, bool)
    m = np.asarray(masks[mask][:n], np.float32)
    return (w * m).astype(np.float32), m == 0


def _base(stack):
    for i, layer in enumerate(stack):
        if layer[2] != OFF:
            return i
    return None


def writes_nothing(stack, counts, num_masks: int) -> bool:
    """layers_cases.writes_nothing, or a BLEND / ADDITIVE layer above the base with a mask index at or above num_masks"""
    if layers_cases.writes_nothing([layer[:4] for layer in stack], counts):
        return True
    base = _base(stack)
    return any(layer[2] in (BLEND, ADDITIVE) and layer[4] is not None and layer[4] >= num_masks for layer in stack[base + 1:])


def _format(clip, additive_format, clip_formats):
    if clip_formats is None:
        return additive_format
    f = int(clip_formats[clip])
    return f if f <= 3 else 0


def _fold(acc, stack, masks, blobs, decode_layer, lerp, apply, additive_format, clip_formats):
    """the fold of every layer above the base into acc, bone groups of one weight at a time"""
    n = acc.shape[0]
    acc = acc.copy()
    for i in range(_base(stack) + 1, len(stack)):
        clip, t, op, _, _ = stack[i]
        if op == OFF:
            continue
        layer = decode_layer(clip, t, op)
        w, skipped = bone_weights(stack[i], masks, n)
        bones = np.flatnonzero(~skipped)
        for value in np.unique(w[bones].view(np.uint32)):
            at = bones[w[bones].view(np.uint32) == value]
            wb = float(np.uint32(value).view(np.float32))
            if op == BLEND:
                acc[at] = lerp(acc[at], layer[at], wb)
            else:
                delta = layer[at] if wb == 1.0 else lerp(writer_default_rows(len(at), default_scale_of(blobs[clip])), layer[at], wb)
                acc[at] = apply(_format(clip, additive_format, clip_formats), acc[at], delta)
    return acc


def port_local(port, blend_lib, blobs, stack, masks, settings, writer, rounding, looping, additive_format=0, clip_formats=None,
               normalize_mode=None) -> np.ndarray | None:
    """The port's composition (normalize_mode: port.NORMALIZE_IEEE, what the GPU computes, or NORMALIZE_RTM_SSE2, the reference's
    rsqrtss on this CPU). None: the stack writes nothing."""
    counts = [port.num_tracks_of(b) for b in blobs]
    if writes_nothing(stack, counts, len(masks)):
        return None
    mode = port.NORMALIZE_IEEE if normalize_mode is None else normalize_mode
    clip, t = stack[_base(stack)][:2]
    acc = port.transform_decompress_tracks(blobs[clip], settings, float(t), rounding, looping)

    def decode_layer(c, time, op):
        return port.transform_decompress_tracks(blobs[c], settings if op == BLEND else writer, float(time), rounding, looping)

    return _fold(acc, stack, masks, blobs, decode_layer, lambda a, b, w: blend_lib.port_qvv_lerp(a, b, w, mode),
                 lambda f, a, b: port.apply_additive_to_base(f, a, b, mode), additive_format, clip_formats)


def reference_local(blend_lib, additive_lib, blobs, stack, masks, kind, rounding, looping, additive_format=0, clip_formats=None):
    """The same composition by the unmodified reference: its decode under settings kind `kind`, rtm::qvv_lerp, apply_additive_to_base."""
    counts = [ref.num_tracks_of(b) for b in blobs]
    if writes_nothing(stack, counts, len(masks)):
        return None
    clip, t = stack[_base(stack)][:2]
    acc = ref.decompress_tracks(blobs[clip], float(t), rounding, looping, settings=kind)

    def decode_layer(c, time, op):
        return ref.decompress_tracks(blobs[c], float(time), rounding, looping, settings=kind)

    return _fold(acc, stack, masks, blobs, decode_layer, blend_lib.reference_qvv_lerp, additive_lib.apply_additive_to_base,
                 additive_format, clip_formats)


# ---- how far the port's IEEE composition may be from the reference's, per bone ----
# layers_cases.rotation_gate with each step's own weight w_b, bone by bone; a skipped bone keeps its error. A weighted ADDITIVE step
# (w_b != 1) first lerps the layer's rotation from the identity: that qvv_lerp normalises in the two flavours, so the delta's rotation is
# off by at most ROTATION_GATE per lane; quat_mul(delta, running) then carries it at most twice into each lane (a lane is a dot of the
# delta's four lanes with the unit running rotation's, whose absolute values sum to <= 2): ADDITIVE_LERP_GATE. Format none keeps the
# lerped row itself (<= ROTATION_GATE). The running rotation's earlier error passes as in layers_cases (<= 2 e). The derivation of the
# BLEND step needs w_b in [0, 1], and the lerp from the identity needs it too (|q| >= 1/sqrt(2) for a dot >= 0): a bone where some
# step's w_b leaves [0, 1] gets no gate (inf) and is compared through the rsqrtss flavour only.
ADDITIVE_LERP_GATE = 2.0 * blend_cases.ROTATION_GATE


def rotation_gate(stack, masks, formats, n: int = NUM_BONES) -> np.ndarray:
    """float64[n]: the per bone gate of the IEEE composition's rotations"""
    e = np.zeros(n)
    for clip, t, op, weight, mask in stack[_base(stack) + 1:]:
        if op == OFF:
            continue
        w, skipped = bone_weights((clip, t, op, weight, mask), masks, n)
        w = w.astype(np.float64)
        outside = (w < 0.0) | (w > 1.0) | np.isinf(e)
        finite_e = np.where(np.isinf(e), 0.0, e)
        if op == BLEND:
            step = 4.0 * np.abs(1.0 - w) * finite_e + blend_cases.ROTATION_GATE
        else:
            relative = blend_cases.ROTATION_GATE if formats[clip] == 1 else 0.0
            step = 2.0 * finite_e + relative + np.where(w == 1.0, 0.0, ADDITIVE_LERP_GATE)
        step = np.where(outside, np.inf, step)
        e = np.where(skipped, e, step)
    return e


def vectors_exact(stack, formats) -> bool:
    """layers_cases.vectors_exact, where a weighted ADDITIVE `relative` layer (a weight other than 1 or a mask) also counts as a step that
    moves the rotation, and is itself not exact: qvv_mul's matrix branch (a mirrored bone) reads the additive rotation into the scale"""
    moved = False
    for clip, _, op, weight, mask in stack[_base(stack) + 1:]:
        relative = op == ADDITIVE and formats[clip] == 1
        weighted = relative and (weight != 1.0 or mask is not None)
        if relative and (moved or weighted):
            return False
        if op == BLEND or relative:
            moved = True
    return True


def vector_gate(stack, masks, formats, reference_pose) -> float:
    gate = rotation_gate(stack, masks, formats, reference_pose.shape[0])
    return 8.0 * float(np.max(gate)) * (1.0 + float(np.max(np.abs(reference_pose[:, 4:11])))) ** 2


def golden_masks() -> np.ndarray:
    """[5][24]: upper body (bones 12.. at 1, the rest 0), a feathered spine (0 below bone 8, 0.25 / 0.5 / 0.75 on bones 8..10, 1 from 11),
    mixed values (0, -0, 1, fractions, above 1, negative), all 0, all 1"""
    upper = (np.arange(NUM_BONES) >= 12).astype(np.float32)
    feather = np.clip((np.arange(NUM_BONES) - 7) * 0.25, 0.0, 1.0).astype(np.float32)
    mixed = np.resize(np.array([0.0, -0.0, 1.0, 0.5, 0.3, 1.5, -0.25, 0.75], np.float32), NUM_BONES)
    return np.stack([upper, feather, mixed, np.zeros(NUM_BONES, np.float32), np.ones(NUM_BONES, np.float32)])


def golden_stacks() -> list[list[tuple]]:
    """The stacks of masked_layers.golden.npz over NAMES (clips 0, 1 blend pair, 2 additive base, 3..5 relative / additive0 / additive1)."""
    rng = np.random.default_rng(4700)
    times = np.array([0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    stacks = [
        [(0, 0.2, BLEND, 0.0, None), (1, 0.6, BLEND, 1.0, 0)],
        [(0, 0.2, BLEND, 0.0, None), (1, 0.6, BLEND, 0.8, 1)],
        [(2, 0.25, ADDITIVE, 0.0, None), (4, 0.5, ADDITIVE, 0.5, None)],
        [(2, 0.25, ADDITIVE, 0.0, None), (5, 0.5, ADDITIVE, 0.3, 1), (3, 0.9, ADDITIVE, 1.0, 0)],
        [(0, 0.2, BLEND, 0.0, 2), (1, 0.6, BLEND, 0.5, 2), (4, 0.1, ADDITIVE, 1.0, 2)],
        [(NO_MASK, float("nan"), OFF, 0.0, 3), (2, 0.7, BLEND, 0.0, 3), (1, 0.3, BLEND, 0.4, 3), (3, 0.45, ADDITIVE, 0.6, 4)],
        [(0, 0.2, BLEND, 0.0, None), (1, 0.6, BLEND, 0.25, 0), (0, 0.9, BLEND, 0.4, 1), (4, 0.1, ADDITIVE, 0.5, None)],
    ]
    for depth in (5, 8):
        stack = [(int(rng.choice([0, 1, 2])), float(rng.choice(times)), BLEND, 0.0, None)]
        for _ in range(depth - 1):
            mask = None if rng.random() < 0.3 else int(rng.choice([0, 1, 4]))
            if rng.random() < 0.5:
                stack.append((int(rng.choice([0, 1, 2])), float(rng.choice(times)), BLEND, float(rng.uniform(0.0, 1.0)), mask))
            else:
                stack.append((int(rng.choice([3, 4, 5])), float(rng.choice(times)), ADDITIVE, float(rng.uniform(0.0, 1.0)), mask))
        stacks.append(stack)
    return stacks


def stack_array(stacks) -> np.ndarray:
    """[num_stacks][8][5] float64 (clip, time, op, weight, mask index or NO_MASK), padded with OFF layers"""
    out = np.zeros((len(stacks), 8, 5))
    out[:, :, 0] = NO_MASK
    out[:, :, 4] = NO_MASK
    for i, stack in enumerate(stacks):
        for j, (clip, t, op, weight, mask) in enumerate(stack):
            out[i, j] = (clip, t, op, weight, NO_MASK if mask is None else mask)
    return out


def random_stack(rng, depth: int, num_clips: int, times, num_masks: int, formats_clips=None, allow_off: bool = True,
                 weights=(-0.25, 1.25)) -> list[tuple]:
    """layers_cases.random_stack with a mask (or None) on every layer and ADDITIVE weights from `weights` (1 a quarter of the time)"""
    stack = []
    for clip, t, op, weight in layers_cases.random_stack(rng, depth, num_clips, times, formats_clips, allow_off):
        if op == ADDITIVE:
            weight = 1.0 if rng.random() < 0.25 else float(rng.uniform(*weights))
        elif op == BLEND:
            weight = float(np.clip(weight, *weights))
        mask = None if rng.random() < 0.3 else int(rng.integers(0, num_masks))
        stack.append((clip, t, op, weight, mask))
    return stack
