"""Skinning decode timings on one GPU: the C2 and C3 workloads of bench.py (binary tree skeleton parent(b) = (b - 1) / 2, random affine
inverse binds), per launch:
  two_step            aclb200_decompress_tracks (the pipeline kernel) into a local pose buffer, then aclb200_local_to_skinning in place
  fused_matrix        aclb200_decompress_tracks_object_space, ACLB200_OBJECT_MATRIX3X4F: the same walk with no skinning step, the floor
  fused_skinning      aclb200_decompress_tracks_skinning
  additive_unfused    request i of the workload as the base of pair i, a shuffled request as its additive half (additive0): two
                      aclb200_decompress_tracks, aclb200_apply_additive_to_base, aclb200_local_to_skinning
  additive_skinning   aclb200_decompress_tracks_additive_skinning of the same pairs
  blend_unfused       the same pairs as blend pairs with a weight each: two aclb200_decompress_tracks, aclb200_blend_poses,
                      aclb200_local_to_skinning
  blend_skinning      aclb200_decompress_tracks_blend_skinning
Cold data and timing as tools/bench_object_space.py: a 256 MB scratch write precedes every timed launch, CUDA event medians of --steps
launches after --warmup, for --runs runs. The algorithmic bytes of each route sit next to its time: the compressed bytes the decodes read
(bench.py's count, twice for pairs), 48 B per bone-pose written, and 48 B per bone-pose for every pose buffer an unfused step writes or
reads back (the inverse binds, 48 B per bone of one skeleton, are left out). The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_skinning.py --workloads c2 c3 --steps 20 --warmup 5 --runs 3
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
    from tests import skinning_cases
    w = bench.make_workload(name, 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones = w["num_tracks"]
    m = int(w["req_clip"].size)
    rng = np.random.default_rng(7)
    order = rng.permutation(m)
    other_clip, other_time = w["req_clip"][order], w["req_time"][order]
    as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
    d_parents = as_dev(skinning_cases.skeleton("tree", bones))
    d_inverse = as_dev(skinning_cases.random_affine(bones, 0))
    d_weights = torch.from_numpy(rng.uniform(0.0, 1.0, m).astype(np.float32)).cuda()
    d_requests = as_dev(ab.make_requests(w["req_clip"], w["req_time"]))
    d_other = as_dev(ab.make_requests(other_clip, other_time))
    d_pairs = as_dev(ab.make_blend_requests(w["req_clip"], w["req_time"], other_clip, other_time))     # same bytes as additive pairs
    options = ab.Options()
    d_first = torch.empty((m, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    d_second = torch.empty_like(d_first)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def timed(body):
        def launch(events):
            events[0].record()
            body()
            events[1].record()
        return launch

    def two_step():
        ctx.decompress_tracks(clipset, d_requests, m, options, d_first)
        ctx.local_to_skinning(d_first, d_first, m, bones, d_parents, d_inverse)

    def unfused(combine):
        def body():
            ctx.decompress_tracks(clipset, d_requests, m, options, d_first)
            ctx.decompress_tracks(clipset, d_other, m, options, d_second)
            combine()
            ctx.local_to_skinning(d_first, d_first, m, bones, d_parents, d_inverse)
        return body

    routes = {
        "two_step": two_step,
        "fused_matrix": lambda: ctx.decompress_tracks_object_space(clipset, d_requests, m, options, d_parents, ab.OBJECT_MATRIX3X4F, d_first),
        "fused_skinning": lambda: ctx.decompress_tracks_skinning(clipset, d_requests, m, options, d_parents, d_inverse, d_first),
        "additive_unfused": unfused(lambda: ctx.apply_additive_to_base(d_first, d_second, d_first, m, bones, ab.ADDITIVE_ADDITIVE0)),
        "additive_skinning": lambda: ctx.decompress_tracks_additive_skinning(clipset, d_pairs, m, options, d_parents, d_inverse, d_first,
                                                                             additive_format=ab.ADDITIVE_ADDITIVE0),
        "blend_unfused": unfused(lambda: ctx.blend_poses(d_first, d_second, d_first, m, bones, d_weights=d_weights)),
        "blend_skinning": lambda: ctx.decompress_tracks_blend_skinning(clipset, d_pairs, m, options, d_parents, d_inverse, d_first,
                                                                       d_weights=d_weights),
    }
    traffic = bench.algorithmic_bytes_transform(w)
    bp = traffic["units"]
    fused = traffic["in_bytes"] + 48 * bp
    pair_fused = 2 * traffic["in_bytes"] + 48 * bp
    algorithmic = {
        "two_step": fused + 96 * bp,                              # the local pose written, then read back
        "fused_matrix": fused, "fused_skinning": fused,
        "additive_unfused": pair_fused + 48 * bp * (2 + 2 + 1 + 1),   # two poses written, both read back, combined written, read back
        "additive_skinning": pair_fused,
        "blend_unfused": pair_fused + 48 * bp * (2 + 2 + 1 + 1),
        "blend_skinning": pair_fused,
    }
    runs = []
    for _ in range(args.runs):
        runs.append({key + "_ms": round(_median_ms(torch, timed(body), flush, args.steps, args.warmup)[1], 4) for key, body in routes.items()})
    clipset.release()
    return {"workload": name, "requests": m, "bones": bones, "bone_poses": bp, "algorithmic_bytes": algorithmic, "runs": runs}


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
