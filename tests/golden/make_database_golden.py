"""Regenerates tests/golden/database_tiers.npz: clips bound to a streaming database built by the UNMODIFIED reference
(acl::build_database, 4 KB chunks), the database itself, and what the reference's decompression_context<debug settings + database>
decodes from them in every tier state of tests/test_gpu_database.py (a database_context driven by memcpy streamers through the state's
stream_in / stream_out calls), for every rounding policy with the clips' own looping policy. tests/test_gpu_database.py compares the
CUDA path with these numbers where the compiled reference is absent. Run where oracle/_ref/libaclref_db.so exists:

    python tests/golden/make_database_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref, ref_database  # noqa: E402
from tests import clips  # noqa: E402
from tests.database_cases import ALL_TIMES, PLAIN_CLIP, STATES, build_cases  # noqa: E402


def main() -> None:
    bound, database, other_clip, other_database = build_cases(ref, ref_database)
    plain = clips.load_blob(PLAIN_CLIP)
    arrays = {"database": database, "other_clip": other_clip, "other_database": other_database, "times": ALL_TIMES,
              "num_tracks": np.array([ref.num_tracks_of(b) for b in bound], np.uint32)}
    for i, blob in enumerate(bound):
        arrays[f"clip{i}"] = blob
    for name, ops in STATES.items():
        arrays[f"poses_{name}"] = np.stack([np.stack([np.concatenate(
            [ref_database.decompress(blob, database, ops, float(t), rounding, ref.LOOP_AS_COMPRESSED) for blob in bound])
            for t in ALL_TIMES]) for rounding in range(4)])
    arrays["poses_plain"] = np.stack([np.stack([ref.decompress_tracks(plain, float(t), rounding, ref.LOOP_AS_COMPRESSED, settings=ref.SETTINGS_DEBUG)
                                                for t in ALL_TIMES]) for rounding in range(4)])
    out = clips.golden_path("database_tiers", "npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
