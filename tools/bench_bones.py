"""Bone query timings on one GPU: the C2 and C3 workloads of bench.py (every (clip, sample) request, binary tree skeleton
parent(b) = (b - 1) / 2), K bones per request, by these routes, per launch:
  full_qvvf_gather    aclb200_decompress_tracks_object_space (ACLB200_OBJECT_QVVF) into whole poses, then a gather of the K rows
  full_matrix_gather  the same with ACLB200_OBJECT_MATRIX3X4F
  bones_qvvf          aclb200_decompress_bones with parents, ACLB200_OBJECT_QVVF
  bones_matrix        aclb200_decompress_bones with parents, ACLB200_OBJECT_MATRIX3X4F
  bones_local         aclb200_decompress_bones without parents (local QVV48 rows)
  track_local         aclb200_decompress_track with num_requests * K requests (local rows, decompress_track's own arithmetic): a
                      reference point, not the same result
The lists: root only (K = 1), 4 leaves of different subtrees (on C2: 21 of the 100 bones in the closure), 6 mixed bones, 32 random
bones. Cold data (SURVEY 8d): a 256 MB scratch write precedes every timed launch. Each launch is timed with CUDA events; medians of
--steps launches after --warmup, for --runs runs with the routes alternating. Bytes: what a bone route stores (48 B x K per request)
beside the full decode's algorithmic bytes (bench.py's compressed bytes + 48 B per bone-pose). The compressed bytes a closure touches
are not counted here, so no share of the roofline is claimed for the bone routes. The GPU's name, power limit and SM clock are read in
the same run.

    python tools/bench_bones.py --workloads c2 c3 --steps 20 --warmup 5 --runs 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import bones_cases as cases  # noqa: E402
from tools.bench_object_space import _gpu_description, _median_ms  # noqa: E402


def query_lists(name: str, bones: int) -> dict:
    def leftmost_leaf(b):
        while 2 * b + 1 < bones:
            b = 2 * b + 1
        return b
    leaves = cases.C2_FOUR_LEAVES if bones == 100 else [leftmost_leaf(s) for s in (3, 4, 5, 6)]
    mixed = cases.C2_SIX_MIXED if bones == 100 else [0, bones - 1, 7, bones // 3, leftmost_leaf(3), bones // 4]
    return {"root": [0], "four_leaves": leaves, "six_mixed": mixed,
            "random32": [int(b) for b in np.random.default_rng(7).integers(0, bones, 32)]}


def measure(name: str, args, torch, ab, ctx) -> dict:
    import bench
    w = bench.make_workload(name, 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones = w["num_tracks"]
    num_requests = int(w["req_clip"].size)
    parents = cases.tree(bones)
    d_parents = torch.from_numpy(parents).cuda()
    requests = ab.make_requests(w["req_clip"], w["req_time"])
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    options = ab.Options()
    d_whole = torch.empty((num_requests, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)
    traffic = bench.algorithmic_bytes_transform(w)
    full_bytes = traffic["in_bytes"] + 48 * traffic["units"]

    results = []
    for list_name, bone_list in query_lists(name, bones).items():
        k = len(bone_list)
        d_list = torch.tensor(bone_list, dtype=torch.int32, device="cuda")
        index = d_list.long()
        d_rows = torch.empty((num_requests, k, 12), dtype=torch.float32, device="cuda")
        track_requests = np.repeat(requests, k)
        d_track_requests = torch.from_numpy(track_requests.view(np.uint8)).cuda()
        d_track_indices = torch.from_numpy(np.tile(np.array(bone_list, np.uint32), num_requests)).cuda()

        def full(kind):
            def launch(events):
                events[0].record()
                ctx.decompress_tracks_object_space(clipset, d_requests, num_requests, options, d_parents, kind, d_whole)
                torch.index_select(d_whole, 1, index, out=d_rows)
                events[1].record()
            return launch

        def bone_route(kind, with_parents):
            def launch(events):
                events[0].record()
                ctx.decompress_bones(clipset, d_requests, num_requests, options, d_list, k, d_rows,
                                     d_parent_indices=d_parents if with_parents else None, kind=kind)
                events[1].record()
            return launch

        def track(events):
            events[0].record()
            ctx.decompress_track(clipset, d_track_requests, d_track_indices, num_requests * k, options, d_rows)
            events[1].record()

        routes = {"full_qvvf_gather": full(ab.OBJECT_QVVF), "full_matrix_gather": full(ab.OBJECT_MATRIX3X4F),
                  "bones_qvvf": bone_route(ab.OBJECT_QVVF, True), "bones_matrix": bone_route(ab.OBJECT_MATRIX3X4F, True),
                  "bones_local": bone_route(ab.OBJECT_QVVF, False), "track_local": track}
        runs = []
        for _ in range(args.runs):
            runs.append({route: round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4) for route, launch in routes.items()})
        closure = cases.closure(parents, bone_list, bones).size
        results.append({"list": list_name, "k": k, "closure_bones": int(closure), "stored_bytes": 48 * k * num_requests, "runs": runs})
        del d_rows, d_track_requests, d_track_indices
    clipset.release()
    return {"workload": name, "requests": num_requests, "bones": bones,
            "full_decode_algorithmic_bytes": full_bytes, "full_decode_stored_bytes": 48 * traffic["units"], "lists": results}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--workloads", nargs="+", default=["c2", "c3"], choices=["c2", "c3"])
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    results = [measure(name, args, torch, ab, ctx) for name in args.workloads]
    text = json.dumps({"gpu": _gpu_description(), "results": results})
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
