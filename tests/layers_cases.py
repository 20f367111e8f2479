"""The layered decode's oracle: the composition, in layer order, of the per-operation oracles that are already pinned to the reference
(the port's decode, oracle/blend.py's qvv_lerp, the port's and the reference's apply_additive_to_base, oracle/object_space.py and
oracle/skinning.py). A stack is a list of (clip, sample time, op, weight) layers; the base is its first layer that is not OFF.
tests/golden/layers.golden.npz holds the reference's composition of STACKS (tests/golden/make_layers_golden.py)."""
from __future__ import annotations

import numpy as np

from oracle import ref
from tests import additive_cases, blend_cases, clips

OFF, BLEND, ADDITIVE = 0, 1, 2

# the clips of the golden stacks: the blend pair and the additive base with its three additive formats (24 bones each)
NAMES = blend_cases.NAMES + additive_cases.NAMES
FORMATS = [0, 0, 0] + list(additive_cases.FORMATS.values())         # acl::additive_clip_format8 of each clip
COMBOS = [(0, 0, 2), (1, 0, 2), (3, 2, 0), (4, 0, 1)]


def load_blobs() -> list[np.ndarray]:
    return [clips.load_blob(n) for n in NAMES]


def random_stack(rng, depth: int, num_clips: int, times, formats_clips=None, allow_off: bool = True) -> list[tuple]:
    """A stack of `depth` layers over clips 0..num_clips-1: mixed ops (OFF sometimes, with an invalid clip and a NaN time), weights in
    [-0.25, 1.25]; ADDITIVE layers take the clips of formats_clips when given."""
    stack = []
    for i in range(depth):
        op = int(rng.choice([BLEND, ADDITIVE, OFF] if allow_off else [BLEND, ADDITIVE]))
        if op == OFF:
            stack.append((0xFFFFFFFF, float("nan"), OFF, float("nan")))
            continue
        pool = formats_clips if (op == ADDITIVE and formats_clips) else range(num_clips)
        stack.append((int(rng.choice(list(pool))), float(rng.choice(times)), op, float(rng.uniform(-0.25, 1.25))))
    return stack


def _base(stack):
    for i, layer in enumerate(stack):
        if layer[2] != OFF:
            return i
    return None


def writes_nothing(stack, counts) -> bool:
    """every layer OFF, an op above 2, or a layer that is not OFF with an invalid clip or another track count than the base"""
    base = _base(stack)
    if base is None or any(layer[2] > ADDITIVE for layer in stack):
        return True
    live = [layer for layer in stack if layer[2] != OFF]
    if any(layer[0] >= len(counts) for layer in live):
        return True
    return any(counts[layer[0]] != counts[stack[base][0]] for layer in live)


def base_clip(stack) -> int:
    return stack[_base(stack)][0]


def _format(clip, additive_format, clip_formats):
    if clip_formats is None:
        return additive_format
    f = int(clip_formats[clip])
    return f if f <= 3 else 0


def port_local(port, blend_lib, blobs, stack, settings, writer, rounding, looping, additive_format=0, clip_formats=None,
               normalize_mode=None) -> np.ndarray | None:
    """The port's composition: the base decoded with `settings`, BLEND layers with `settings`, ADDITIVE layers with `writer` (the
    track_writer defaults), folded in order with blend_lib.port_qvv_lerp and port.apply_additive_to_base. None: the stack writes nothing."""
    counts = [port.num_tracks_of(b) for b in blobs]
    if writes_nothing(stack, counts):
        return None
    mode = port.NORMALIZE_IEEE if normalize_mode is None else normalize_mode
    base = _base(stack)
    clip, t, _, _ = stack[base]
    acc = port.transform_decompress_tracks(blobs[clip], settings, float(t), rounding, looping)
    for clip, t, op, weight in stack[base + 1:]:
        if op == BLEND:
            layer = port.transform_decompress_tracks(blobs[clip], settings, float(t), rounding, looping)
            acc = blend_lib.port_qvv_lerp(acc, layer, float(weight), mode)
        elif op == ADDITIVE:
            layer = port.transform_decompress_tracks(blobs[clip], writer, float(t), rounding, looping)
            acc = port.apply_additive_to_base(_format(clip, additive_format, clip_formats), acc, layer, mode)
    return acc


def reference_local(blend_lib, additive_lib, blobs, stack, kind, rounding, looping, additive_format=0, clip_formats=None) -> np.ndarray | None:
    """The same composition by the unmodified reference: its decode under settings kind `kind`, rtm::qvv_lerp, apply_additive_to_base."""
    counts = [ref.num_tracks_of(b) for b in blobs]
    if writes_nothing(stack, counts):
        return None
    base = _base(stack)
    clip, t, _, _ = stack[base]
    acc = ref.decompress_tracks(blobs[clip], float(t), rounding, looping, settings=kind)
    for clip, t, op, weight in stack[base + 1:]:
        if op == OFF:
            continue
        layer = ref.decompress_tracks(blobs[clip], float(t), rounding, looping, settings=kind)
        if op == BLEND:
            acc = blend_lib.reference_qvv_lerp(acc, layer, float(weight))
        else:
            acc = additive_lib.apply_additive_to_base(_format(clip, additive_format, clip_formats), acc, layer)
    return acc


# ---- how far the port's IEEE composition may be from the reference's ----
# One qvv_lerp normalises with an IEEE 1 / sqrt where the reference uses rsqrtss + Newton-Raphson: blend_cases.ROTATION_GATE per
# step. An earlier difference e (max per lane) then passes through the later steps:
#   BLEND     q = (s - w s) + w e' carries at most |1 - w| e per lane into q, then quat_normalize divides by |q| >= 1/sqrt(2) (w in
#             [0, 1], the hemisphere flip makes the dot >= 0; outside [0, 1] |q| >= 1/2 for |w| <= 1.25 is not guaranteed, so the stacks
#             whose gate is used keep w in [0, 1]) and a normalisation moves a lane by at most twice the relative change: <= 4 e, plus
#             the step's own ROTATION_GATE;
#   ADDITIVE  quat_mul(additive, running) with a unit additive rotation: each lane is a dot of 4 products, <= 2 e, plus ROTATION_GATE
#             when a `relative` layer takes qvv_mul's matrix branch (its quat_normalize has the same two flavours).
# Translations and scales never read a rotation in qvv_lerp, additive0 or additive1, so they stay bit for bit unless a `relative` layer
# follows a step that moved the rotation: then qvv_mul rotates t_add * s_running by the running rotation, and rotating v by q + dq moves
# it by at most 4 |dq|_2 |v| <= 8 e |v| (|dq|_2 <= 2 e): vector_gate.
def rotation_gate(stack, formats) -> float:
    e = 0.0
    base = _base(stack)
    for clip, _, op, weight in stack[base + 1:]:
        if op == BLEND:
            e = 4.0 * abs(1.0 - weight) * e + blend_cases.ROTATION_GATE
        elif op == ADDITIVE:
            e = 2.0 * e + (blend_cases.ROTATION_GATE if formats[clip] == 1 else 0.0)
    return e


def vectors_exact(stack, formats) -> bool:
    """no `relative` layer after a step that can move the rotation away from the reference's"""
    moved = False
    base = _base(stack)
    for clip, _, op, _ in stack[base + 1:]:
        if op == ADDITIVE and formats[clip] == 1 and moved:
            return False
        if op == BLEND or (op == ADDITIVE and formats[clip] == 1):
            moved = True
    return True


def vector_gate(stack, formats, reference_pose) -> float:
    return 8.0 * rotation_gate(stack, formats) * (1.0 + float(np.max(np.abs(reference_pose[:, 4:11]))) ** 2)


def golden_stacks() -> list[list[tuple]]:
    """The stacks of layers.golden.npz over NAMES (clips 0, 1 blend pair, 2 additive base, 3..5 relative / additive0 / additive1)."""
    rng = np.random.default_rng(4400)
    times = np.array([0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    stacks = [
        [(2, 0.3, BLEND, 0.0)],
        [(0, 0.2, BLEND, 0.0), (1, 0.6, BLEND, 0.5)],
        [(2, 0.25, ADDITIVE, 0.0), (4, 0.5, ADDITIVE, 0.0)],
        [(0, 0.2, BLEND, 0.0), (1, 0.6, BLEND, 0.25), (0, 0.9, BLEND, 0.4), (4, 0.1, ADDITIVE, 0.0)],
        [(0xFFFFFFFF, float("nan"), OFF, 0.0), (2, 0.7, BLEND, 0.0), (3, 0.3, ADDITIVE, 0.0), (5, 0.45, ADDITIVE, 0.0)],
    ]
    for depth in (5, 8):
        stack = [(int(rng.choice([0, 1, 2])), float(rng.choice(times)), BLEND, 0.0)]
        for _ in range(depth - 1):
            if rng.random() < 0.5:
                stack.append((int(rng.choice([0, 1, 2])), float(rng.choice(times)), BLEND, float(rng.uniform(0.0, 1.0))))
            else:
                stack.append((int(rng.choice([3, 4, 5])), float(rng.choice(times)), ADDITIVE, 0.0))
        stacks.append(stack)
    return stacks


def stack_array(stacks) -> np.ndarray:
    """[num_stacks][8][4] float64 (clip, time, op, weight), padded with OFF layers"""
    out = np.zeros((len(stacks), 8, 4))
    out[:, :, 0] = 0xFFFFFFFF
    for i, stack in enumerate(stacks):
        for j, layer in enumerate(stack):
            out[i, j] = layer
    return out
