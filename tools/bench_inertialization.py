"""Inertialization timings on one GPU, on bench.py's C2 workload (its requests are the destination poses; 100 bones; binary tree skeleton
parent(b) = (b - 1) / 2), per launch, with P % of the poses in transition (the rest ACLB200_NO_INERTIALIZATION):
  decode              aclb200_decompress_tracks (the pipeline kernel) alone, the baseline of local rows
  skinning            aclb200_decompress_tracks_skinning alone, the baseline of skinning rows
  fused_local_P       aclb200_decompress_tracks_inertialized, local QVV48 rows
  unfused_local_P     the decode, then aclb200_inertialize_poses in place
  fused_skinning_P    aclb200_decompress_tracks_inertialized_skinning
  unfused_skinning_P  the decode, aclb200_inertialize_poses in place, then aclb200_local_to_skinning in place
  capture             aclb200_begin_inertialization of --transitions transitions of 100 bones
Cold data (SURVEY 8d): a 256 MB scratch write precedes every timed launch. Medians of --steps launches after --warmup, for --runs runs.
Algorithmic bytes beside each route: the decode's compressed bytes and 48 B written per bone-pose; the fused routes add 64 B read per bone
in transition; the unfused apply reads and writes the poses again (and local_to_skinning once more); the capture reads four poses and
writes 64 B per bone. The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_inertialization.py --steps 20 --warmup 5 --runs 3
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


def measure(args, torch, ab, ctx) -> dict:
    import bench
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones = w["num_tracks"]
    m = int(w["req_clip"].size)
    rng = np.random.default_rng(7)
    as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()
    d_req = as_dev(ab.make_requests(w["req_clip"], w["req_time"]))
    options = ab.Options()
    d_out = torch.empty((m, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    # records: one per transition, captured from decoded poses of the workload
    t = args.transitions
    d_poses = [torch.empty((t, bones, 12), dtype=torch.float32, device="cuda") for _ in range(4)]
    for k in range(4):
        pick = rng.integers(0, m, size=t)
        ctx.decompress_tracks(clipset, as_dev(ab.make_requests(w["req_clip"][pick], w["req_time"][pick])), t, options, d_poses[k])
    d_records = torch.empty((t, bones, 16), dtype=torch.float32, device="cuda")
    ctx.begin_inertialization(*d_poses, t, bones, 30.0, d_records)
    torch.cuda.synchronize()

    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    d_parents = torch.from_numpy(parents).cuda()
    d_inverse_bind = torch.from_numpy(rng.normal(size=(bones, 12)).astype(np.float32)).cuda()

    def inertializations(percent):
        record = rng.integers(0, t, size=m).astype(np.uint32)
        record[rng.random(m) >= percent / 100.0] = ab.NO_INERTIALIZATION
        elapsed = rng.uniform(0.0, 0.5, m)
        return (as_dev(ab.make_inertializations(record, elapsed, 0.2)),
                as_dev(ab.make_inertialized_requests(w["req_clip"], w["req_time"], record, elapsed, 0.2)),
                int(np.count_nonzero(record != ab.NO_INERTIALIZATION)))

    def route(kind, d_inert=None, d_fused_req=None):
        def launch(events):
            events[0].record()
            if kind == "fused_local":
                ctx.decompress_tracks_inertialized(clipset, d_fused_req, m, options, d_out, d_records, t)
            elif kind == "fused_skinning":
                ctx.decompress_tracks_inertialized_skinning(clipset, d_fused_req, m, options, d_parents, d_inverse_bind, d_out, d_records, t)
            elif kind == "skinning":
                ctx.decompress_tracks_skinning(clipset, d_req, m, options, d_parents, d_inverse_bind, d_out)
            else:
                ctx.decompress_tracks(clipset, d_req, m, options, d_out)
                if d_inert is not None:
                    ctx.inertialize_poses(d_out, d_out, m, bones, d_inert, d_records, t)
                if kind == "unfused_skinning":
                    ctx.local_to_skinning(d_out, d_out, m, bones, d_parents, d_inverse_bind)
            events[1].record()
        return launch

    def capture(events):
        events[0].record()
        ctx.begin_inertialization(*d_poses, t, bones, 30.0, d_records)
        events[1].record()

    traffic = bench.algorithmic_bytes_transform(w)
    bp = traffic["units"]
    decode_bytes = traffic["in_bytes"] + 48 * bp
    routes = [("decode", route("decode"), decode_bytes), ("skinning", route("skinning"), decode_bytes)]
    for percent in args.percents:
        d_inert, d_fused_req, moving = inertializations(percent)
        record_bytes = 64 * bones * moving
        apply_bytes = 2 * 48 * bp + record_bytes + 12 * m
        routes.append((f"fused_local_{percent}", route("fused_local", d_fused_req=d_fused_req), decode_bytes + record_bytes))
        routes.append((f"unfused_local_{percent}", route("unfused_local", d_inert=d_inert), decode_bytes + apply_bytes))
        routes.append((f"fused_skinning_{percent}", route("fused_skinning", d_fused_req=d_fused_req), decode_bytes + record_bytes))
        routes.append((f"unfused_skinning_{percent}", route("unfused_skinning", d_inert=d_inert), decode_bytes + apply_bytes + 2 * 48 * bp))
    routes.append(("capture", capture, (4 * 48 + 64) * bones * t))
    runs = []
    for _ in range(args.runs):
        runs.append({key + "_ms": round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4) for key, launch, _ in routes})
    clipset.release()
    return {"workload": "c2", "poses": m, "bones": bones, "transitions": t, "algorithmic_bytes": {key: b for key, _, b in routes},
            "runs": runs}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--transitions", type=int, default=4096)
    parser.add_argument("--percents", type=int, nargs="+", default=[0, 25, 100])
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    print(json.dumps({"gpu": _gpu_description(), "result": measure(args, torch, ab, ctx)}))


if __name__ == "__main__":
    main()
