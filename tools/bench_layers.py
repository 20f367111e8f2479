"""Layered decode timings on one GPU: the C2 and C3 workloads of bench.py as four layer stacks (request i of the workload is the base of
pose i, two shuffled copies of the workload are BLEND layers with weights uniform in [0, 1], a third shuffled copy is an ADDITIVE layer in
the additive0 format; binary tree skeleton parent(b) = (b - 1) / 2, random affine inverse binds), per launch:
  unfused           aclb200_decompress_tracks (the pipeline kernel) of the base and both blend layers, aclb200_decompress_tracks_additive
                    with format none for the additive layer's track_writer-default pose, 2 x aclb200_blend_poses, aclb200_apply_additive_to_base
  fused_local       aclb200_decompress_tracks_layered, local QVV48 rows
  unfused_skinning  the unfused route + aclb200_local_to_skinning
  fused_skinning    aclb200_decompress_tracks_layered_skinning
  fused_half_off    fused_local with layers 1..3 OFF on every other pose
Cold data: a 256 MB scratch write precedes every timed launch. Medians of --steps launches after --warmup, for --runs runs. The
algorithmic bytes of each route sit next to its time: the compressed bytes the decodes must read (bench.py's count, once per decoded
layer), 48 B per bone-pose written, and for every unfused step 48 B per bone-pose and pose buffer it writes or reads back. The GPU's name,
power limit and SM clock are read in the same run.

    python tools/bench_layers.py --workloads c2 c3 --steps 20 --warmup 5 --runs 2
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
    clip = [w["req_clip"]]
    time = [w["req_time"]]
    for _ in range(3):
        order = rng.permutation(m)
        clip.append(w["req_clip"][order])
        time.append(w["req_time"][order])
    weights = [np.zeros(m, np.float32), rng.uniform(0.0, 1.0, m).astype(np.float32), rng.uniform(0.0, 1.0, m).astype(np.float32)]
    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    d_parents = torch.from_numpy(parents).cuda()
    d_inverse = torch.from_numpy(skinning_cases.random_affine(bones, 8)).cuda()
    d_w1, d_w2 = (torch.from_numpy(x).cuda() for x in weights[1:])
    as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()
    d_req = [as_dev(ab.make_requests(clip[k], time[k])) for k in range(3)]
    d_add_pairs = as_dev(ab.make_additive_requests(clip[0], time[0], clip[3], time[3]))
    ops = np.array([[ab.LAYER_BLEND, ab.LAYER_BLEND, ab.LAYER_BLEND, ab.LAYER_ADDITIVE]], np.uint32)
    stack_w = np.stack(weights + [np.zeros(m, np.float32)], 1)
    d_layers = as_dev(ab.make_layers(np.stack(clip, 1), np.stack(time, 1), ops, stack_w))
    half_ops = np.broadcast_to(ops, (m, 4)).copy()
    half_ops[1::2, 1:] = ab.LAYER_OFF
    d_half = as_dev(ab.make_layers(np.stack(clip, 1), np.stack(time, 1), half_ops, stack_w))
    options = ab.Options()
    poses = [torch.empty((m, clipset.max_tracks, 12), dtype=torch.float32, device="cuda") for _ in range(4)]
    d_out = torch.empty_like(poses[0])
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def unfused(to_skinning):
        def launch(events):
            events[0].record()
            for k in range(3):
                ctx.decompress_tracks(clipset, d_req[k], m, options, poses[k])
            ctx.decompress_tracks_additive(clipset, d_add_pairs, m, options, poses[3], additive_format=ab.ADDITIVE_NONE)
            ctx.blend_poses(poses[0], poses[1], poses[0], m, bones, d_weights=d_w1)
            ctx.blend_poses(poses[0], poses[2], poses[0], m, bones, d_weights=d_w2)
            ctx.apply_additive_to_base(poses[0], poses[3], poses[0], m, bones, ab.ADDITIVE_ADDITIVE0)
            if to_skinning:
                ctx.local_to_skinning(poses[0], d_out, m, bones, d_parents, d_inverse)
            events[1].record()
        return launch

    def fused(layers, to_skinning=False):
        def launch(events):
            events[0].record()
            if to_skinning:
                ctx.decompress_tracks_layered_skinning(clipset, layers, m, 4, options, d_parents, d_inverse, d_out,
                                                       additive_format=ab.ADDITIVE_ADDITIVE0)
            else:
                ctx.decompress_tracks_layered(clipset, layers, m, 4, options, d_out, additive_format=ab.ADDITIVE_ADDITIVE0)
            events[1].record()
        return launch

    traffic = bench.algorithmic_bytes_transform(w)
    bp = traffic["units"]
    fused_bytes = 4 * traffic["in_bytes"] + 48 * bp
    # four decodes written (the additive one through a pair whose base half is decoded too), 2 x blend_poses (2 reads, 1 write each),
    # apply_additive_to_base (2 reads, 1 write)
    unfused_bytes = 5 * traffic["in_bytes"] + 48 * bp * (4 + 3 + 3 + 3)
    runs = []
    for _ in range(args.runs):
        times = {}
        for key, launch in (("unfused", unfused(False)), ("fused_local", fused(d_layers)), ("unfused_skinning", unfused(True)),
                            ("fused_skinning", fused(d_layers, True)), ("fused_half_off", fused(d_half))):
            times[key + "_ms"] = round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4)
        runs.append(times)
    clipset.release()
    return {"workload": name, "poses": m, "bones": bones, "bone_poses": bp,
            "algorithmic_bytes": {"unfused": unfused_bytes, "unfused_skinning": unfused_bytes + 96 * bp, "fused": fused_bytes,
                                  "fused_half_off": int(2.5 * traffic["in_bytes"]) + 48 * bp, "compressed_in_per_pose": traffic["in_bytes"]},
            "runs": runs}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--workloads", nargs="+", default=["c2", "c3"], choices=["c2", "c3"])
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=2)
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    results = [measure(name, args, torch, ab, ctx) for name in args.workloads]
    print(json.dumps({"gpu": _gpu_description(), "results": results}))


if __name__ == "__main__":
    main()
