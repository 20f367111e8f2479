"""Regenerates tests/golden/bench_workloads.npz: a fixed sample of the clips and requests bench.py times (workloads c2 and c5, same
seeds), together with what the UNMODIFIED reference decodes for them (acl::decompression_context<benchmark settings>::seek +
decompress_tracks). tests/test_gpu_bench_workloads.py compares the CUDA path with these numbers where the compiled reference is
absent. Run where oracle/_ref/libaclref.so exists:

    python tests/golden/make_bench_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import ref  # noqa: E402
from tests import clips  # noqa: E402

# workload: (clips kept, every n-th of their requests kept)
SAMPLE = {"c2": (1, 30), "c5": (3, 1)}


def main() -> None:
    arrays = {}
    for name, (num_clips, stride) in SAMPLE.items():
        w = bench.make_workload(name, 0, num_clips)
        assert w["distinct"], "needs the reference compressor"
        blobs = [w["buffer"][int(o):int(o) + int(s)] for o, s in zip(w["offsets"], w["sizes"])]
        req_clip, req_time = w["req_clip"][::stride], w["req_time"][::stride]
        want = ref.decode_requests(blobs, req_clip, req_time, w["num_tracks"])
        arrays[f"{name}_blobs"] = np.concatenate(blobs)
        arrays[f"{name}_sizes"] = w["sizes"].astype(np.uint32)
        arrays[f"{name}_req_clip"] = req_clip.astype(np.uint32)
        arrays[f"{name}_req_time"] = req_time.astype(np.float32)
        arrays[f"{name}_want"] = np.ascontiguousarray(want[:, :, clips.DEFINED_LANES])
        print(name, len(blobs), "clips", len(req_clip), "requests", int(w["sizes"].sum()), "bytes")
    np.savez_compressed(clips.golden_path("bench_workloads", "npz"), **arrays)


if __name__ == "__main__":
    main()
