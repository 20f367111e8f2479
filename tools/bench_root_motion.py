"""Root motion timings on one GPU: the C2 and C3 workloads of bench.py, each (clip, sample) request turned into a root motion request
(clip, from = the request's time, to = from + 1/30 s, wrapped at the clip's clamp duration D with cycles = 1 when it wraps), root = track
0, by these routes, per launch:
  fused         aclb200_extract_root_motion: one launch, M per request
  bones_torch   today's route: aclb200_decompress_bones with the root as the only listed bone at the 2 to 4 sample requests of each request
                (from, to, and D and 0 when it wraps), then the composition with rtm's qvv_inverse / qvv_mul (positive scale branch) in torch
                ops: compared on timing only, torch's float order is not rtm's
  track_floor   aclb200_decompress_track of the root at the same sample requests: seek plus decode alone, a floor and a different result
                (decompress_track's own normalisation), no composition
Cold data: a 256 MB scratch write precedes every timed launch. Each launch is timed with CUDA events; medians of --steps launches after
--warmup, for --runs runs with the routes alternating. The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_root_motion.py --workloads c2 c3 --steps 20 --warmup 5 --runs 3
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


def _quat_mul(l, r):
    """rtm::quat_mul(l, r) on [N, 4] tensors"""
    lx, ly, lz, lw = l.unbind(-1)
    rx, ry, rz, rw = r.unbind(-1)
    import torch
    return torch.stack([(rw * lx + rx * lw) + (ry * lz - rz * ly), (rw * ly - rx * lz) + (ry * lw + rz * lx),
                        (rw * lz + rx * ly) + (rz * lw - ry * lx), (rw * lw - rx * lx) - (ry * ly + rz * lz)], -1)


def _quat_mul_vector3(v, r):
    """rtm::quat_mul_vector3(v, r): quat_mul(quat_mul(conjugate(r), (v, 0)), r), xyz"""
    import torch
    conj = torch.cat([-r[:, :3], r[:, 3:]], -1)
    q = torch.cat([v, torch.zeros_like(v[:, :1])], -1)
    return _quat_mul(_quat_mul(conj, q), r)[:, :3]


def _qvv_mul(lhs, rhs):
    """rtm::qvv_mul's positive scale branch on [N, 12] rows"""
    import torch
    rotation = _quat_mul(lhs[:, 0:4], rhs[:, 0:4])
    translation = _quat_mul_vector3(lhs[:, 4:7] * rhs[:, 8:11], rhs[:, 0:4]) + rhs[:, 4:7]
    zero = torch.zeros_like(lhs[:, :1])
    return torch.cat([rotation, translation, zero, lhs[:, 8:11] * rhs[:, 8:11], zero], -1)


def _qvv_inverse(q):
    import torch
    inv_rotation = torch.cat([-q[:, :3], q[:, 3:4]], -1)
    inv_scale = 1.0 / q[:, 8:11]
    translation = -_quat_mul_vector3(q[:, 4:7] * inv_scale, inv_rotation)
    zero = torch.zeros_like(q[:, :1])
    return torch.cat([inv_rotation, translation, zero, inv_scale, zero], -1)


def measure(name: str, args, torch, ab, ctx) -> dict:
    import bench
    w = bench.make_workload(name, 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    n = int(w["req_clip"].size)
    clip = w["req_clip"].astype(np.uint32)
    info = [clipset.clip_info(c) for c in range(clipset.num_clips)]
    duration = np.array([np.float32(i.num_samples - 1) / np.float32(i.sample_rate) for i in info], np.float32)[clip]
    from_time = w["req_time"].astype(np.float32)
    to_time = (from_time + np.float32(1.0 / 30.0)).astype(np.float32)
    wraps = to_time > duration
    to_time = np.where(wraps, to_time - duration, to_time).astype(np.float32)
    requests = ab.make_root_motion_requests(clip, from_time, to_time, wraps.astype(np.int32))
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    options = ab.Options(looping_policy=ab.LOOP_CLAMP)
    d_out = torch.empty((n, 12), dtype=torch.float32, device="cuda")

    # the sample requests of the two reference routes: from and to of every request, then D and 0 of the wrapping ones
    wrapped = np.flatnonzero(wraps)
    sample_clip = np.concatenate([clip, clip, clip[wrapped], clip[wrapped]])
    sample_time = np.concatenate([from_time, to_time, duration[wrapped], np.zeros(wrapped.size, np.float32)])
    num_samples = int(sample_clip.size)
    d_samples_requests = torch.from_numpy(ab.make_requests(sample_clip, sample_time).view(np.uint8)).cuda()
    d_samples = torch.empty((num_samples, 12), dtype=torch.float32, device="cuda")
    d_root_list = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_track_indices = torch.zeros(num_samples, dtype=torch.int32, device="cuda")
    d_wrapped = torch.from_numpy(wrapped).cuda()
    m = wrapped.size
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)

    def fused(events):
        events[0].record()
        ctx.extract_root_motion(clipset, d_requests, n, options, d_out)
        events[1].record()

    def bones_torch(events):
        events[0].record()
        ctx.decompress_bones(clipset, d_samples_requests, num_samples, options, d_root_list, 1, d_samples)
        f, t = d_samples[:n], d_samples[n:2 * n]
        motion = _qvv_mul(t, _qvv_inverse(f))
        if m:
            end, start = d_samples[2 * n:2 * n + m], d_samples[2 * n + m:]
            crossed = _qvv_mul(_qvv_mul(t[d_wrapped], _qvv_inverse(start)), _qvv_mul(end, _qvv_inverse(f[d_wrapped])))
            motion.index_copy_(0, d_wrapped, crossed)
        d_out.copy_(motion)
        events[1].record()

    def track_floor(events):
        events[0].record()
        ctx.decompress_track(clipset, d_samples_requests, d_track_indices, num_samples, options, d_samples)
        events[1].record()

    routes = {"fused": fused, "bones_torch": bones_torch, "track_floor": track_floor}
    runs = []
    for _ in range(args.runs):
        runs.append({route: round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4) for route, launch in routes.items()})
    clipset.release()
    return {"workload": name, "requests": n, "wrapping_requests": int(m), "sample_requests": num_samples, "bones": w["num_tracks"],
            "stored_bytes": 48 * n, "runs": runs}


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
