"""Writes the reference's root motion for a fixed request list over several named clips.

Run where oracle/_ref/libaclref_root_motion.so exists (the reference tree is present and `make -f oracle/root_motion.mk` was run):

    python tests/golden/make_root_motion_golden.py

It writes root_motion.golden.npz: the clips (`names`, in clip set order), the root track of each clip (`roots`), the requests (`clip`,
`from_time`, `to_time`, `cycles`) and `motion`, the reference's M of each request (decompression_context<debug settings> with the clamp
policy, rounding none, the library's default sub-tracks; the root is the bone whose translation moves most; rtm::qvv_inverse and rtm::qvv_mul; 12 lanes, w lanes 0).
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import port, root_motion  # noqa: E402
from tests import clips  # noqa: E402

NAMES = ["c1_30bones", "mixed_scale", "looping", "stripped_loop", "full_formats", "ragged_17", "two_samples"]
SETTINGS_KIND = 1
REQUESTS_PER_CLIP = 24


def requests() -> dict:
    """The request list: per clip, steps of 1/30 s forward and backward wrapped at the clamp duration D (cycles set when they wrap),
    multi-cycle jumps, and times at 0, D and beyond both ends"""
    rng = np.random.default_rng(2026)
    settings = port.settings_for_kind(SETTINGS_KIND)
    out = dict(clip=[], from_time=[], to_time=[], cycles=[])
    roots = []
    for c, name in enumerate(NAMES):
        spec = clips.TRANSFORM_SPECS[name]
        blob = clips.load_blob(name)
        duration = float(port.transform_seek(blob, settings, 1.0e9, looping=port.LOOP_CLAMP).clip_duration)
        # the root: the bone whose translation moves most over the clip, so that every component of M carries motion
        poses = np.stack([port.transform_decompress_tracks(blob, settings, t, 0, port.LOOP_CLAMP) for t in (0.0, duration * 0.5, duration)])
        roots.append(int(np.argmax(np.abs(np.diff(poses[:, :, 4:7], axis=0)).sum(axis=(0, 2)))))
        for i in range(REQUESTS_PER_CLIP):
            from_time = float(rng.uniform(0.0, duration))
            step = (1.0 if i % 2 == 0 else -1.0) / 30.0
            cycles = 0
            to_time = from_time + step
            if i % 6 == 4:
                cycles = int(rng.integers(-3, 4))
                to_time = float(rng.uniform(0.0, duration))
            elif duration > 0.0 and to_time > duration:
                to_time, cycles = to_time - duration, 1
            elif duration > 0.0 and to_time < 0.0:
                to_time, cycles = to_time + duration, -1
            if i == 5:
                from_time, to_time = -0.25, duration + 0.25
            if i == 11:
                from_time, to_time = duration, 0.0
            out["clip"].append(c)
            out["from_time"].append(from_time)
            out["to_time"].append(to_time)
            out["cycles"].append(cycles)
    return dict(names=np.array(NAMES), roots=np.array(roots, np.uint32), clip=np.array(out["clip"], np.uint32),
                from_time=np.array(out["from_time"], np.float32), to_time=np.array(out["to_time"], np.float32),
                cycles=np.array(out["cycles"], np.int32))


def compute() -> dict:
    r = requests()
    blobs = [clips.load_blob(name) for name in NAMES]
    motion = np.zeros((r["clip"].size, 12), np.float32)
    for i in range(r["clip"].size):
        c = int(r["clip"][i])
        motion[i], _ = root_motion.reference_extract(blobs[c], SETTINGS_KIND, 0, 0, int(r["roots"][c]), float(r["from_time"][i]),
                                                     float(r["to_time"][i]), int(r["cycles"][i]))
    assert np.isfinite(motion).all()
    r["motion"] = motion
    return r


def main() -> None:
    np.savez_compressed(clips.golden_path("root_motion", "golden.npz"), **compute())


if __name__ == "__main__":
    main()
