"""Writes tests/golden/scalar_cases.golden.npz: the reference's scalar decode of the fabricated clips of tests/scalar_cases.py at
their golden times, tracks and policy combinations, so that tests/test_scalar_requests.py checks the port without the compiled
reference. Run from the repository root with oracle/_ref built: python -m tests.golden.make_scalar_cases_golden"""
from __future__ import annotations

import numpy as np

from oracle import ref
from tests import clips
from tests import scalar_cases as sc


def main() -> None:
    out = {}
    blobs = sc.all_clips()
    out["names"] = np.array(sorted(blobs))
    for name, blob in blobs.items():
        nc = sc.components(int(blob[15]))
        n = ref.num_tracks_of(blob)
        times, tracks = sc.golden_times(blob), sc.golden_tracks(blob)
        values = np.zeros((len(sc.GOLDEN_COMBOS), len(times), len(tracks), nc), dtype=np.float32)
        for k, (per_track, rounding, looping) in enumerate(sc.GOLDEN_COMBOS):
            for ti, t in enumerate(times.tolist()):
                values[k, ti] = ref.scalar_decompress(blob, t, rounding, looping, settings=int(per_track),
                                                      per_track_rounding=sc.track_policies(n) if per_track else None)[tracks, :nc]
        out[name + "/times"], out[name + "/tracks"], out[name + "/values"] = times, tracks, values
    np.savez_compressed(clips.golden_path("scalar_cases", "golden.npz"), **out)


if __name__ == "__main__":
    main()
