"""Blend decode timings on one GPU: the C2 and C3 workloads of bench.py as blend pairs (request i of the workload is the from half of pair
i, a shuffled request of the same workload its to half; a weight per pair, uniform in [0, 1]; binary tree skeleton parent(b) = (b - 1) / 2),
per launch:
  unfused        aclb200_decompress_tracks (the pipeline kernel) of the from halves, of the to halves, then aclb200_blend_poses
  fused_local    aclb200_decompress_tracks_blend, local QVV48 rows
  unfused_object the unfused route + aclb200_local_to_object_space
  fused_qvvf     aclb200_decompress_tracks_blend with parents, ACLB200_OBJECT_QVVF
  fused_matrix   the same, ACLB200_OBJECT_MATRIX3X4F
Cold data (SURVEY 8d): a 256 MB scratch write precedes every timed launch. Medians of --steps launches after --warmup, for --runs runs.
The algorithmic bytes of each route sit next to its time: the compressed bytes the decodes must read (bench.py's count, twice: two poses
per pair), 48 B per bone-pose written, and for every unfused step 48 B per bone-pose and pose buffer it writes or reads back. The GPU's
name, power limit and SM clock are read in the same run.

    python tools/bench_blend.py --workloads c2 c3 --steps 20 --warmup 5 --runs 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_object_space import _gpu_description, _median_ms  # noqa: E402


def measure(name: str, args, torch, ab, ctx) -> dict:
    import bench
    w = bench.make_workload(name, 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones = w["num_tracks"]
    m = int(w["req_clip"].size)
    rng = np.random.default_rng(7)
    order = rng.permutation(m)
    to_clip, to_time = w["req_clip"][order], w["req_time"][order]
    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    d_parents = torch.from_numpy(parents).cuda()
    d_weights = torch.from_numpy(rng.uniform(0.0, 1.0, m).astype(np.float32)).cuda()
    as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
    d_from_req = as_dev(ab.make_requests(w["req_clip"], w["req_time"]))
    d_to_req = as_dev(ab.make_requests(to_clip, to_time))
    d_pairs = as_dev(ab.make_blend_requests(w["req_clip"], w["req_time"], to_clip, to_time))
    options = ab.Options()
    d_from = torch.empty((m, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    d_to = torch.empty_like(d_from)
    d_out = torch.empty_like(d_from)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def unfused(to_object):
        def launch(events):
            events[0].record()
            ctx.decompress_tracks(clipset, d_from_req, m, options, d_from)
            ctx.decompress_tracks(clipset, d_to_req, m, options, d_to)
            ctx.blend_poses(d_from, d_to, d_from, m, bones, d_weights=d_weights)
            if to_object:
                ctx.local_to_object_space(d_from, d_out, m, bones, d_parents)
            events[1].record()
        return launch

    def fused(kind=None):
        def launch(events):
            events[0].record()
            if kind is None:
                ctx.decompress_tracks_blend(clipset, d_pairs, m, options, d_out, d_weights=d_weights)
            else:
                ctx.decompress_tracks_blend(clipset, d_pairs, m, options, d_out, d_weights=d_weights, d_parent_indices=d_parents, kind=kind)
            events[1].record()
        return launch

    traffic = bench.algorithmic_bytes_transform(w)
    bp = traffic["units"]
    fused_bytes = 2 * traffic["in_bytes"] + 48 * bp
    unfused_bytes = 2 * traffic["in_bytes"] + 48 * bp * (2 + 2 + 1)          # two poses written, both read back, the result written
    runs = []
    for _ in range(args.runs):
        times = {}
        for key, launch in (("unfused", unfused(False)), ("fused_local", fused()), ("unfused_object", unfused(True)),
                            ("fused_qvvf", fused(ab.OBJECT_QVVF)), ("fused_matrix", fused(ab.OBJECT_MATRIX3X4F))):
            times[key + "_ms"] = round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4)
        runs.append(times)
    clipset.release()
    return {"workload": name, "pairs": m, "bones": bones, "bone_poses": bp,
            "algorithmic_bytes": {"unfused": unfused_bytes, "unfused_object": unfused_bytes + 96 * bp, "fused": fused_bytes,
                                  "compressed_in_per_pose": traffic["in_bytes"]},
            "runs": runs}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--workloads", nargs="+", default=["c2", "c3"], choices=["c2", "c3"])
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=3)
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    results = [measure(name, args, torch, ab, ctx) for name in args.workloads]
    print(json.dumps({"gpu": _gpu_description(), "results": results}))


if __name__ == "__main__":
    main()
