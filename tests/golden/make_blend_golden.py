"""Writes the blend clips of tests/blend_cases.py and the reference's decode-and-lerp poses for them.

Run where oracle/_ref/libaclref.so and libaclref_blend.so exist (the reference tree is present, `make -C oracle` and
`make -f oracle/blend.mk` were run):

    python tests/golden/make_blend_golden.py

It writes
    blend_from.acl.bin, blend_to.acl.bin   the two clips (24 bones each, shared default bones, mirrored-scale bones)
    blend.golden.npz                       for every (settings kind, rounding, looping) triple of blend_cases.COMBOS, weight of
                                           blend_cases.WEIGHTS and (from time, to time) pair of blend_cases.time_pairs(): the reference's
                                           decompress of both clips followed by rtm::qvv_lerp, defined lanes; and the reference's
                                           qvv_lerp of blend_cases.fabricated_pairs() at every weight, all 12 lanes
and prints the sha256 of each blob for blend_cases.BLOB_SHA256.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import blend, ref  # noqa: E402
from tests import blend_cases as cases, clips  # noqa: E402


def blobs() -> dict:
    return {"blend_from": ref.compress_transform(cases.FROM_SPEC), "blend_to": ref.compress_transform(cases.TO_SPEC)}


def main() -> None:
    made = blobs()
    for name, blob in made.items():
        assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0, name
        size = int(blob[0:4].view(np.uint32)[0])
        with open(clips.golden_path(name, "acl.bin"), "wb") as f:
            f.write(blob[:size].tobytes())
        print(f'    "{name}": "{cases.blob_sha256(blob)}",')
    pairs = cases.time_pairs()
    poses = np.zeros((len(cases.COMBOS), len(cases.WEIGHTS), len(pairs), cases.FROM_SPEC.num_tracks, 10), np.float32)
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        for wi, weight in enumerate(cases.WEIGHTS):
            for pi, (tf, tt) in enumerate(pairs):
                pose = cases.reference_pose(blend, made["blend_from"], made["blend_to"], tf, tt, weight, kind, rounding, looping)
                poses[ci, wi, pi] = pose[:, clips.DEFINED_LANES]
    assert np.isfinite(poses).all()
    _, from_rows, to_rows = cases.fabricated_pairs()
    fabricated = np.stack([blend.reference_qvv_lerp(from_rows, to_rows, float(w)) for w in cases.WEIGHTS])
    np.savez_compressed(clips.golden_path("blend", "golden.npz"), combos=np.array(cases.COMBOS, np.int32), weights=cases.WEIGHTS,
                        pairs=pairs, poses=poses, fabricated_from=from_rows, fabricated_to=to_rows, fabricated=fabricated)


if __name__ == "__main__":
    main()
