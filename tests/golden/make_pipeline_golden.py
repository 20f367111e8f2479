"""Regenerates the clips of tests/pipeline_cases.py: reference-compressed blobs + the reference's own poses at a few times.

Run where oracle/_ref/libaclref.so exists (the reference tree is present and `make -C oracle` was run):

    python tests/golden/make_pipeline_golden.py

For every clip of pipeline_cases.PIPELINE_SPECS this writes
    <name>.acl.bin        the compressed_tracks blob produced by acl::compress_track_list
    <name>.golden.npz     acl::decompression_context outputs (seek + decompress_tracks) at pipeline_cases.GOLDEN_TIMES for the
                          (settings kind, rounding policy) pairs of pipeline_cases.GOLDEN_COMBOS, defined lanes of the bones
                          pipeline_cases.golden_bones names
The outputs come from the UNMODIFIED reference (oracle/ref_tool.cpp); nothing here involves the port or the CUDA path.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import ref  # noqa: E402
from tests import clips, pipeline_cases  # noqa: E402


def make(name: str, spec) -> None:
    blob = ref.compress_transform(spec)
    with open(clips.golden_path(name, "acl.bin"), "wb") as f:
        f.write(blob.tobytes())
    times = np.array(pipeline_cases.GOLDEN_TIMES[name], dtype=np.float32)
    combos = pipeline_cases.GOLDEN_COMBOS
    bones = pipeline_cases.golden_bones(name)
    poses = np.zeros((len(combos), len(times), len(bones), 10), dtype=np.float32)
    for ci, (kind, rounding) in enumerate(combos):
        for ti, t in enumerate(times):
            poses[ci, ti] = ref.decompress_tracks(blob, float(t), rounding, settings=kind)[bones][:, clips.DEFINED_LANES]
    np.savez_compressed(clips.golden_path(name, "golden.npz"), times=times, combos=np.array(combos, dtype=np.int32), bones=bones,
                        poses=poses)
    print(f"{name}: {blob.size} byte blob, {os.path.getsize(clips.golden_path(name, 'golden.npz'))} byte poses")


def main() -> None:
    for name, spec in pipeline_cases.PIPELINE_SPECS.items():
        make(name, spec)


if __name__ == "__main__":
    main()
