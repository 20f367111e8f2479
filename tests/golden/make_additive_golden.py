"""Writes the additive clips of tests/additive_cases.py and the reference's decode-and-apply poses for them.

Run where oracle/_ref/libaclref.so and libaclref_additive.so exist (the reference tree is present, `make -C oracle` and
`make -f oracle/additive.mk` were run):

    python tests/golden/make_additive_golden.py

It writes
    additive_base.acl.bin            the base clip (animated and mirrored scale)
    additive_<format>.acl.bin        the relative, additive0 and additive1 clips of a second animation over that base
    additive.golden.npz              for every format clip, (settings kind, rounding, looping) triple of additive_cases.COMBOS and
                                     (base time, additive time) pair of additive_cases.time_pairs(): the reference's decompress of
                                     both clips (track_writer defaults) followed by apply_additive_to_base, defined lanes
and prints the sha256 of each blob for additive_cases.BLOB_SHA256.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import additive, ref  # noqa: E402
from tests import additive_cases as cases, clips  # noqa: E402


def blobs() -> dict:
    out = {cases.BASE: ref.compress_transform(cases.BASE_SPEC)}
    for name, format_ in cases.FORMATS.items():
        out[name] = additive.compress_additive(cases.BASE_SPEC, cases.FULL_SPEC, format_)
    return out


def main() -> None:
    made = blobs()
    for name, blob in made.items():
        assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0, name
        size = int(blob[0:4].view(np.uint32)[0])
        with open(clips.golden_path(name, "acl.bin"), "wb") as f:
            f.write(blob[:size].tobytes())
        print(f'    "{name}": "{cases.blob_sha256(blob)}",')
    pairs = cases.time_pairs()
    poses = np.zeros((len(cases.FORMATS), len(cases.COMBOS), len(pairs), cases.BASE_SPEC.num_tracks, 10), np.float32)
    for fi, (name, format_) in enumerate(cases.FORMATS.items()):
        for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
            for pi, (tb, ta) in enumerate(pairs):
                pose = cases.reference_pose(additive, format_, made[cases.BASE], made[name], tb, ta, kind, rounding, looping)
                poses[fi, ci, pi] = pose[:, clips.DEFINED_LANES]
    assert np.isfinite(poses).all()
    np.savez_compressed(clips.golden_path("additive", "golden.npz"), formats=np.array(list(cases.FORMATS.values()), np.int32),
                        combos=np.array(cases.COMBOS, np.int32), pairs=pairs, poses=poses)


if __name__ == "__main__":
    main()
