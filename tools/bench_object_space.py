"""Object space decode timings on one GPU: the C2 and C3 workloads of bench.py (every (clip, sample) request, binary tree skeleton
parent(b) = (b - 1) / 2) taken to object space by three routes, per launch:
  two_step     aclb200_decompress_tracks (QVV48, the pipeline kernel) into a local pose buffer, then aclb200_local_to_object_space
  fused_qvvf   aclb200_decompress_tracks_object_space, ACLB200_OBJECT_QVVF
  fused_matrix aclb200_decompress_tracks_object_space, ACLB200_OBJECT_MATRIX3X4F
Cold data (SURVEY 8d): a 256 MB scratch write precedes every timed launch, so no launch finds its inputs in L2. Each launch is timed with
CUDA events (the two-step route also per kernel); medians of --steps launches after --warmup, for --runs runs with the routes alternating.
The algorithmic bytes of each route sit next to its time: the compressed bytes the launch must read (bench.py's count) plus 48 B per
bone-pose written, and for the two-step route 96 B more per bone-pose (the local pose written, then read back). The GPU's name, power
limit and SM clock are read in the same run.

    python tools/bench_object_space.py --workloads c2 c3 --steps 20 --warmup 5 --runs 3
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_description() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def _median_ms(torch, launch, flush, steps: int, warmup: int, marks: int = 1):
    """Median over `steps` cold launches of the time between consecutive events; launch(events) records marks + 1 events."""
    for _ in range(warmup):
        flush()
        launch([torch.cuda.Event(enable_timing=True) for _ in range(marks + 1)])
    samples = []
    for _ in range(steps):
        flush()
        events = [torch.cuda.Event(enable_timing=True) for _ in range(marks + 1)]
        launch(events)
        samples.append(events)
    torch.cuda.synchronize()
    times = np.array([[e[i].elapsed_time(e[i + 1]) for i in range(marks)] for e in samples])
    return [float(np.median(times[:, i])) for i in range(marks)], float(np.median(times.sum(axis=1)))


def measure(name: str, args, torch, ab, ctx) -> dict:
    import bench
    w = bench.make_workload(name, 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones = w["num_tracks"]
    num_requests = int(w["req_clip"].size)
    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    d_parents = torch.from_numpy(parents).cuda()
    d_requests = torch.from_numpy(ab.make_requests(w["req_clip"], w["req_time"]).view(np.uint8)).cuda()
    options = ab.Options()
    d_local = torch.empty((num_requests, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    d_object = torch.empty_like(d_local)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def two_step(events):
        events[0].record()
        ctx.decompress_tracks(clipset, d_requests, num_requests, options, d_local)
        events[1].record()
        ctx.local_to_object_space(d_local, d_object, num_requests, bones, d_parents)
        events[2].record()

    def fused(kind):
        def launch(events):
            events[0].record()
            ctx.decompress_tracks_object_space(clipset, d_requests, num_requests, options, d_parents, kind, d_object)
            events[1].record()
        return launch

    traffic = bench.algorithmic_bytes_transform(w)
    bone_poses = traffic["units"]
    fused_bytes = traffic["in_bytes"] + 48 * bone_poses
    two_step_bytes = fused_bytes + 96 * bone_poses
    runs = []
    for _ in range(args.runs):
        kernels, total = _median_ms(torch, two_step, flush, args.steps, args.warmup, marks=2)
        _, qvvf = _median_ms(torch, fused(ab.OBJECT_QVVF), flush, args.steps, args.warmup)
        _, matrix = _median_ms(torch, fused(ab.OBJECT_MATRIX3X4F), flush, args.steps, args.warmup)
        runs.append(dict(two_step_ms=round(total, 4), decompress_tracks_ms=round(kernels[0], 4), local_to_object_space_ms=round(kernels[1], 4),
                         fused_qvvf_ms=round(qvvf, 4), fused_matrix_ms=round(matrix, 4)))
    clipset.release()
    return {"workload": name, "distinct_clips": bool(w["distinct"]), "requests": num_requests, "bones": bones, "bone_poses": bone_poses,
            "algorithmic_bytes": {"two_step": two_step_bytes, "fused": fused_bytes, "compressed_in": traffic["in_bytes"]},
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
