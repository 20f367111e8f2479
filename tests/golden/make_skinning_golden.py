"""Writes the reference's skinning rows for a few named clips' decoded poses.

Run where oracle/_ref/libaclref_skinning.so exists (the reference tree is present and `make -f oracle/skinning.mk` was run):

    python tests/golden/make_skinning_golden.py

It writes skinning.golden.npz: for every clip of skinning_cases.GOLDEN_CLIPS, with the binary tree and the random skeleton,
    <clip>_local                 [times][n][12] the port's decode (settings kind 0) at skinning_cases.GOLDEN_TIMES
    <clip>_<skeleton>_parents    [n] the skeleton
    <clip>_<skeleton>_<kind>     [n][12] the inverse binds of each skinning_cases.INVERSE_BIND_KINDS kind (bind: the inverses of the bind
                                 pose's object matrices, the bind pose being the decode at time 0; random, mirrored: random affine matrices)
    <clip>_<skeleton>_<kind>_skin [times][n][12] the reference's skinning rows (row c = x_axis[c], y_axis[c], z_axis[c], w_axis[c])
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import port, skinning  # noqa: E402
from tests import clips, skinning_cases as cases  # noqa: E402

GOLDEN_SKELETONS = ["tree", "random"]


def main() -> None:
    assert skinning.reference_available(), "needs oracle/_ref/libaclref_skinning.so"
    settings = port.settings_for_kind(0)
    arrays = {"times": cases.GOLDEN_TIMES}
    for ci, name in enumerate(cases.GOLDEN_CLIPS):
        blob = clips.load_blob(name)
        n = clips.TRANSFORM_SPECS[name].num_tracks
        local = np.stack([port.transform_decompress_tracks(blob, settings, float(t)) for t in cases.GOLDEN_TIMES])
        arrays[f"{name}_local"] = local
        for skeleton in GOLDEN_SKELETONS:
            parents = cases.skeleton(skeleton, n, seed=ci)
            arrays[f"{name}_{skeleton}_parents"] = parents
            for kind in cases.INVERSE_BIND_KINDS:
                inverse = cases.inverse_binds(kind, n, local[0], parents, seed=100 + ci)
                arrays[f"{name}_{skeleton}_{kind}"] = inverse
                arrays[f"{name}_{skeleton}_{kind}_skin"] = np.stack([skinning.reference_local_to_skinning(pose, parents, inverse) for pose in local])
    np.savez_compressed(clips.golden_path("skinning", "golden.npz"), **arrays)


if __name__ == "__main__":
    main()
