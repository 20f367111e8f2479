"""Writes the fabricated clips of tests/edge_cases.py and the reference's poses for them.

Run where oracle/_ref/libaclref.so exists (the reference tree is present and `make -C oracle` was run):

    python tests/golden/make_edge_golden.py

For every clip of edge_cases.EDGE_SPECS this writes
    <name>.acl.bin          the base clip's blob with the edits of edge_cases.fabricate (deterministic: the same committed base always
                            gives the same bytes, whatever CPU compressed it)
    <name>.manifest.json    one row per edit: kind, sub-track, bone, class, segment, stored key frame, clip key frame
    <name>.golden.npz       the unmodified reference's decompress_tracks at golden_times() for the (settings kind, rounding, looping)
                            triples of golden_combos(), defined lanes of golden_bones()
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import ref  # noqa: E402
from tests import clips, edge_cases  # noqa: E402


def make(name: str) -> None:
    blob, manifest = edge_cases.fabricate(name)
    assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0, name
    with open(clips.golden_path(name, "acl.bin"), "wb") as f:
        f.write(blob.tobytes())
    with open(clips.golden_path(name, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=0)
        f.write("\n")
    times = edge_cases.golden_times(blob)
    bones = edge_cases.golden_bones(blob, manifest)
    combos = edge_cases.golden_combos(name)
    poses = np.zeros((len(combos), len(times), len(bones), 10), dtype=np.float32)
    for ci, (kind, rounding, looping) in enumerate(combos):
        for ti, t in enumerate(times):
            poses[ci, ti] = ref.decompress_tracks(blob, float(t), rounding, looping, settings=kind)[bones][:, clips.DEFINED_LANES]
    assert np.isfinite(poses).all(), name
    np.savez_compressed(clips.golden_path(name, "golden.npz"), times=times, combos=np.array(combos, dtype=np.int32), bones=bones,
                        poses=poses)
    print(f"{name}: {blob.size} byte blob, {len(manifest)} edits, {os.path.getsize(clips.golden_path(name, 'golden.npz'))} byte poses")


def main() -> None:
    for name in edge_cases.EDGE_SPECS:
        make(name)


if __name__ == "__main__":
    main()
