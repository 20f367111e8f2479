"""Writes the reference's composition of the masked layer stacks of tests/masked_layers_cases.py.

Run where oracle/_ref/libaclref.so, libaclref_blend.so and libaclref_additive.so exist (the reference tree is present, `make -C oracle`,
`make -f oracle/blend.mk` and `make -f oracle/additive.mk` were run):

    python tests/golden/make_masked_layers_golden.py

It writes masked_layers.golden.npz: for every (settings kind, rounding, looping) triple of masked_layers_cases.COMBOS and stack of
masked_layers_cases.golden_stacks() (over the committed blend and additive clips, with golden_masks()), the reference's decode of every
layer folded bone by bone with its rtm::qvv_lerp and acl::apply_additive_to_base (each clip's own additive format), defined lanes; and
the stacks and masks themselves.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import additive, blend  # noqa: E402
from tests import clips, masked_layers_cases as cases  # noqa: E402


def poses() -> np.ndarray:
    blobs = cases.load_blobs()
    stacks = cases.golden_stacks()
    masks = cases.golden_masks()
    out = np.zeros((len(cases.COMBOS), len(stacks), cases.NUM_BONES, 10), np.float32)
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        for si, stack in enumerate(stacks):
            pose = cases.reference_local(blend, additive, blobs, stack, masks, kind, rounding, looping, clip_formats=np.array(cases.FORMATS))
            out[ci, si] = pose[:, clips.DEFINED_LANES]
    assert np.isfinite(out).all()
    return out


def main() -> None:
    np.savez_compressed(clips.golden_path("masked_layers", "golden.npz"), combos=np.array(cases.COMBOS, np.int32),
                        stacks=cases.stack_array(cases.golden_stacks()), masks=cases.golden_masks(), poses=poses())


if __name__ == "__main__":
    main()
