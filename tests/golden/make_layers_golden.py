"""Writes the reference's composition of the layer stacks of tests/layers_cases.py.

Run where oracle/_ref/libaclref.so, libaclref_blend.so and libaclref_additive.so exist (the reference tree is present, `make -C oracle`,
`make -f oracle/blend.mk` and `make -f oracle/additive.mk` were run):

    python tests/golden/make_layers_golden.py

It writes layers.golden.npz: for every (settings kind, rounding, looping) triple of layers_cases.COMBOS and stack of
layers_cases.golden_stacks() (over the committed blend and additive clips), the reference's decode of every layer folded in layer order
with its rtm::qvv_lerp and acl::apply_additive_to_base (each clip's own additive format), defined lanes; and the stacks themselves.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import additive, blend  # noqa: E402
from tests import clips, layers_cases as cases  # noqa: E402


def poses() -> np.ndarray:
    blobs = cases.load_blobs()
    stacks = cases.golden_stacks()
    out = np.zeros((len(cases.COMBOS), len(stacks), 24, 10), np.float32)
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        for si, stack in enumerate(stacks):
            pose = cases.reference_local(blend, additive, blobs, stack, kind, rounding, looping, clip_formats=np.array(cases.FORMATS))
            out[ci, si] = pose[:, clips.DEFINED_LANES]
    assert np.isfinite(out).all()
    return out


def main() -> None:
    np.savez_compressed(clips.golden_path("layers", "golden.npz"), combos=np.array(cases.COMBOS, np.int32),
                        stacks=cases.stack_array(cases.golden_stacks()), poses=poses())


if __name__ == "__main__":
    main()
