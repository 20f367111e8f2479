"""Pose features timings on one GPU, S = 4 offsets {-1/30, 0, 1/3, 2/3} s and K = 4 bones (the root, two leaves and a mid bone of a
binary tree skeleton), half the requests FEATURE_LOOP, root = track 0, on two workloads:
  database      the C2 clip set of bench.py, all 600,000 requests (a motion matching database build)
  runtime       C5-shaped: 125,000 clips x 30 bones, one random time per clip (a run time query per character)
by these routes, per launch:
  fused         aclb200_extract_pose_features: one launch
  unfused       the route a caller has without it: each offset's (c, u') worked out on the host (once, outside the timed window), then
                aclb200_decompress_bones for the object rows at the S x N virtual requests, aclb200_decompress_bones again for the root's local
                rows, aclb200_extract_root_motion for {t, u', c}, and F = qvv_mul(qvv_mul(B, qvv_inverse(T)), M) in torch ops (rtm's order,
                positive scale branch): compared on timing only, torch's float order is not the kernel's
Cold data: a 256 MB scratch write precedes every timed launch. Each launch is timed with CUDA events; medians of --steps launches after
--warmup, for --runs runs with the routes alternating. The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_features.py --workloads database runtime --steps 20 --warmup 5 --runs 2
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
from tools.bench_root_motion import _qvv_inverse, _qvv_mul  # noqa: E402

OFFSETS = np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0], np.float32)


def measure(name: str, args, torch, ab, ctx) -> dict:
    import bench
    from tests import bones_cases
    from tests import features_cases as cases
    w = bench.make_workload({"database": "c2", "runtime": "c5"}[name], 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    if name == "database":
        clip, time = w["req_clip"].astype(np.uint32), w["req_time"].astype(np.float32)
    else:
        rng = np.random.default_rng(5)
        clip = np.arange(clipset.num_clips, dtype=np.uint32)
        time = rng.uniform(0.0, 1.0, clip.size).astype(np.float32)
    n, S, K = int(clip.size), OFFSETS.size, 4
    bones = w["num_tracks"]
    tree = bones_cases.tree(bones)
    leaves = [b for b in range(bones) if 2 * b + 1 >= bones]
    bone_list = np.array([0, leaves[0], leaves[-1], bones // 4], np.uint32)
    looping = (np.arange(n) % 2).astype(np.uint32)
    requests = ab.make_feature_requests(clip, time, looping)
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_list = torch.from_numpy(bone_list.view(np.int32)).cuda()
    d_parents = torch.from_numpy(tree.view(np.int32)).cuda()
    options = ab.Options(looping_policy=ab.LOOP_CLAMP)
    d_out = torch.empty((n, S, K, 12), dtype=torch.float32, device="cuda")

    # the unfused route's virtual requests: (c, u') of every (request, offset), on the host
    info = [clipset.clip_info(c) for c in range(clipset.num_clips)]
    duration = np.array([np.float32(i.num_samples - 1) / np.float32(i.sample_rate) if i.num_samples > 1 else 0.0 for i in info], np.float32)
    v_clip = np.repeat(clip, S)
    v_time = np.repeat(time, S)
    # features_cases.offset_time on arrays: every u is finite and every |c| small here, so every pair writes
    v_duration = duration[v_clip]
    u = (v_time + np.tile(OFFSETS, n)).astype(np.float32)
    wraps = (np.repeat(looping, S) == cases.LOOP) & (v_duration > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        cycle = np.where(wraps, np.floor((u / np.where(wraps, v_duration, np.float32(1))).astype(np.float32)), np.float32(0)).astype(np.float32)
    v_cycles = cycle.astype(np.int32)
    v_at = np.where(wraps, (u - (cycle * v_duration).astype(np.float32)).astype(np.float32), u).astype(np.float32)
    v_at[(np.repeat(looping, S) == cases.LOOP) & (v_duration == 0)] = 0.0
    for i in range(0, n * S, max(1, n * S // 1000)):        # spot check against the one rule
        assert cases.offset_time(v_time[i], OFFSETS[i % S], int(looping[i // S]), v_duration[i])[1:] == (v_cycles[i], v_at[i])
    d_v_requests = torch.from_numpy(ab.make_requests(v_clip, v_at).view(np.uint8)).cuda()
    d_motion_requests = torch.from_numpy(ab.make_root_motion_requests(v_clip, v_time, v_at, v_cycles).view(np.uint8)).cuda()
    d_root_list = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_objects = torch.empty((n * S, K, 12), dtype=torch.float32, device="cuda")
    d_local = torch.empty((n * S, 12), dtype=torch.float32, device="cuda")
    d_motion = torch.empty((n * S, 12), dtype=torch.float32, device="cuda")
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def fused(events):
        events[0].record()
        ctx.extract_pose_features(clipset, d_requests, n, options, OFFSETS, d_list, K, d_parents, d_out)
        events[1].record()

    def unfused(events):
        events[0].record()
        ctx.decompress_bones(clipset, d_v_requests, n * S, options, d_list, K, d_objects, d_parent_indices=d_parents, kind=ab.OBJECT_QVVF)
        ctx.decompress_bones(clipset, d_v_requests, n * S, options, d_root_list, 1, d_local)
        ctx.extract_root_motion(clipset, d_motion_requests, n * S, options, d_motion)
        relative = _qvv_inverse(d_local).repeat_interleave(K, 0)
        motion = d_motion.repeat_interleave(K, 0)
        d_out.view(-1, 12).copy_(_qvv_mul(_qvv_mul(d_objects.view(-1, 12), relative), motion))
        events[1].record()

    routes = {"fused": fused, "unfused": unfused}
    runs = []
    for _ in range(args.runs):
        runs.append({route: round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4) for route, launch in routes.items()})
    clipset.release()
    return {"workload": name, "requests": n, "offsets": S, "bones_per_list": K, "bones": bones, "stored_bytes": 48 * n * S * K, "runs": runs}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--workloads", nargs="+", default=["database", "runtime"], choices=["database", "runtime"])
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=2)
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
