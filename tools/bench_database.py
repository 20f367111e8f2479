"""Streaming database timings on one GPU: a C2-shaped set of clips bound to one database (100 bones, 60 samples at 30 Hz, compressed
by the reference with database support and split by acl::build_database). Per launch of every (clip, sample) request it reports
  unbound_ms    the clip set without its database: the pipeline kernel (resident key frames only)
  db_ms         the clip set bound, every tier streamed in: the database instances of the plain kernel
and the host-to-device rate of streaming both tiers in (stream_in of every chunk, byte swap on the host included), with the GPU's name
and power limit. Needs oracle/_ref/libaclref_db.so to build the clips.

    python tools/bench_database.py --clips 2000 --steps 20 --warmup 5
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_description() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def _time_launches(torch, launch, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        launch()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        launch()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--clips", type=int, default=2000)
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--medium", type=float, default=0.3)
    parser.add_argument("--low", type=float, default=0.3)
    args = parser.parse_args()

    import torch
    import acl_b200 as ab
    from oracle import ref, ref_database

    specs = [ref.TransformSpec(num_tracks=100, num_samples=60, seed=2000 + i) for i in range(args.clips)]
    t0 = time.perf_counter()
    bound, database_blob = ref_database.build_database(specs, args.medium, args.low, 1 << 20)
    build_s = time.perf_counter() - t0

    ctx = ab.Context(0)
    clipset = ctx.upload(bound)
    database = ctx.upload_database(database_blob)
    info = database.info()
    req_clip = np.repeat(np.arange(args.clips, dtype=np.uint32), 60)
    req_time = np.tile(np.arange(60, dtype=np.float32) / np.float32(30.0), args.clips)
    d_requests = torch.from_numpy(ab.make_requests(req_clip, req_time).view(np.uint8)).cuda()
    options = ab.Options(output_layout=ab.LAYOUT_QVV40)
    d_out = torch.empty((len(req_clip), clipset.max_tracks, 10), dtype=torch.float32, device="cuda")
    launch = lambda: ctx.decompress_tracks(clipset, d_requests, len(req_clip), options, d_out)

    unbound_ms = _time_launches(torch, launch, args.steps, args.warmup)
    clipset.bind_database(database)
    # stream-in rate: every chunk of both tiers, several rounds
    bulk_bytes = int(info.bulk_data_size[0]) + int(info.bulk_data_size[1])
    rates = []
    for _ in range(5):
        for tier in (ab.TIER_MEDIUM, ab.TIER_LOW):
            if info.num_chunks[tier - 1]:
                database.stream_out(tier)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for tier in (ab.TIER_MEDIUM, ab.TIER_LOW):
            if info.num_chunks[tier - 1]:
                database.stream_in(tier)
        torch.cuda.synchronize()
        rates.append(bulk_bytes / (time.perf_counter() - t0) / 1e9)
    db_ms = _time_launches(torch, launch, args.steps, args.warmup)

    print(json.dumps({
        "gpu": _gpu_description(),
        "clips": args.clips, "bones": 100, "requests_per_launch": int(len(req_clip)),
        "database": {"chunks": [int(info.num_chunks[0]), int(info.num_chunks[1])], "bulk_bytes": [int(info.bulk_data_size[0]), int(info.bulk_data_size[1])],
                     "segments": int(info.num_segments), "tier_proportions": [args.medium, args.low], "reference_build_s": round(build_s, 1)},
        "unbound_ms": round(unbound_ms, 4), "db_ms": round(db_ms, 4), "db_over_unbound": round(db_ms / unbound_ms, 3),
        "stream_in_gbs": {"median": round(float(np.median(rates)), 3), "min": round(float(min(rates)), 3), "max": round(float(max(rates)), 3),
                          "what": "stream_in of every chunk of both tiers, host byte swap + pageable H2D copy + metadata, host clock around a device synchronise"},
    }))


if __name__ == "__main__":
    main()
