"""Writes the reference's pose features rows for a fixed request list over several named clips.

Run where oracle/_ref/libaclref.so and oracle/_ref/libaclref_root_motion.so exist (the reference tree is present and `make -C oracle all`
and `make -f oracle/root_motion.mk` were run):

    python tests/golden/make_features_golden.py

It writes features.golden.npz: the clips (`names`, in clip set order), the root track of each clip (`roots`), the offsets, the bone list
(`bones`, on each clip's binary tree skeleton `tree(num_tracks)`; bones beyond a clip's tracks write nothing), the requests (`clip`,
`time`, `looping`) and `rows` [requests][offsets][bones][12], the reference's rows (decompression_context<debug settings> with the clamp
policy, rounding none, the library's default sub-tracks; rtm::qvv_inverse and rtm::qvv_mul; the object rows by the port walk in the
reference's rsqrtss flavour; w lanes 0), NaN where a row is not written.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import port, ref, root_motion  # noqa: E402
from tests import bones_cases, clips  # noqa: E402
from tests import features_cases as cases  # noqa: E402

NAMES = ["c1_30bones", "mixed_scale", "looping", "ragged_17", "full_formats", "one_sample"]
SETTINGS_KIND = 1
REQUESTS_PER_CLIP = 12
OFFSETS = np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0, -2.5], np.float32)
BONES = [0, 16, 5, 1]


def requests() -> dict:
    rng = np.random.default_rng(2026)
    settings = port.settings_for_kind(SETTINGS_KIND)
    out = dict(clip=[], time=[], looping=[])
    roots = []
    for c, name in enumerate(NAMES):
        spec = clips.TRANSFORM_SPECS[name]
        blob = clips.load_blob(name)
        duration = float(port.transform_seek(blob, settings, 1.0e9, looping=port.LOOP_CLAMP).clip_duration)
        roots.append(0 if c % 2 == 0 else spec.num_tracks - 1)
        for i in range(REQUESTS_PER_CLIP):
            out["clip"].append(c)
            out["time"].append([0.0, duration][i] if i < 2 else float(rng.uniform(-0.1, duration + 0.1)))
            out["looping"].append(i % 2)
    return dict(names=np.array(NAMES), roots=np.array(roots, np.uint32), offsets=OFFSETS, bones=np.array(BONES, np.uint32),
                clip=np.array(out["clip"], np.uint32), time=np.array(out["time"], np.float32), looping=np.array(out["looping"], np.uint32))


def compute() -> dict:
    r = requests()
    blobs = [clips.load_blob(name) for name in NAMES]
    settings = port.settings_for_kind(SETTINGS_KIND)
    rows = np.full((r["clip"].size, OFFSETS.size, len(BONES), 12), np.nan, np.float32)
    for i in range(r["clip"].size):
        c = int(r["clip"][i])
        blob = blobs[c]
        n = clips.TRANSFORM_SPECS[NAMES[c]].num_tracks
        root = int(r["roots"][c])
        duration = float(port.transform_seek(blob, settings, 1.0e9, looping=port.LOOP_CLAMP).clip_duration)
        bones = [b for b in BONES if b < n]
        for s, offset in enumerate(OFFSETS):
            writes, cycles, u = cases.offset_time(r["time"][i], offset, int(r["looping"][i]), duration)
            if not writes:
                continue
            local = ref.decompress_tracks(blob, float(u), 0, ref.LOOP_CLAMP, settings=SETTINGS_KIND)
            local[:, 7] = 0.0
            local[:, 11] = 0.0
            motion, _ = root_motion.reference_extract(blob, SETTINGS_KIND, 0, 0, root, float(r["time"][i]), float(u), cycles)
            objects = cases.object_rows(port, local, bones_cases.tree(n), bones, port.NORMALIZE_RTM_SSE2)
            for k, bone in enumerate(BONES):
                if bone < n:
                    rows[i, s, k] = cases.compose(root_motion, objects[bone], local[root], motion, reference=True)
    r["rows"] = rows
    return r


def main() -> None:
    np.savez_compressed(clips.golden_path("features", "golden.npz"), **compute())


if __name__ == "__main__":
    main()
