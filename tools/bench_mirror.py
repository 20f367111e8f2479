"""Mirroring timings on one GPU, on bench.py's C2 workload (600k requests; 100 bones; binary tree skeleton parent(b) = (b - 1) / 2, bones
paired (1, 2), (3, 4) .. with general corrections and bone 0 its own mirror), per launch, with P % of the requests mirrored:
  decode                        aclb200_decompress_tracks (the pipeline kernel) alone, the baseline of local rows
  skinning                      aclb200_decompress_tracks_skinning alone, the baseline of skinning rows
  fused_local_P                 aclb200_decompress_tracks_mirrored, local QVV48 rows
  unfused_local_P               the decode, then aclb200_mirror_poses in place with the per-request flags
  fused_skinning_P              aclb200_decompress_tracks_mirrored_skinning
  unfused_skinning_P            the decode, aclb200_mirror_poses in place, then aclb200_local_to_skinning in place
  mirror_poses_P                aclb200_mirror_poses alone on the decoded poses, in place
  inertialized_skinning         aclb200_decompress_tracks_inertialized_skinning with no request in transition: the composed mode the fused
                                skinning decode is compared with
  mirrored_inertialized_P       the chain of a mirrored character in transition: aclb200_decompress_tracks_mirrored (local rows), then
                                aclb200_inertialize_poses and aclb200_local_to_skinning in place (every request inertialized)
Cold data (SURVEY 8d): a 256 MB scratch write precedes every timed launch. Medians of --steps launches after --warmup, for --runs runs.
The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_mirror.py --steps 20 --warmup 5 --runs 3
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


def _table(ab, bones: int, rng) -> np.ndarray:
    mirror = np.arange(bones, dtype=np.uint32)
    pairs = np.arange(1, bones - 1, 2)
    mirror[pairs], mirror[pairs + 1] = pairs + 1, pairs
    unit = lambda q: (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    table = np.zeros(bones, dtype=ab.MIRROR_ENTRY_DTYPE)
    table["pre"], table["post"], table["mirror"] = unit(rng.normal(size=(bones, 4))), unit(rng.normal(size=(bones, 4))), mirror
    return table


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

    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    d_parents = torch.from_numpy(parents).cuda()
    d_inverse_bind = torch.from_numpy(rng.normal(size=(bones, 12)).astype(np.float32)).cuda()
    d_table = as_dev(_table(ab, bones, rng))

    # inertialization records for the transition chain, captured from decoded poses of the workload
    t = 4096
    d_poses = [torch.empty((t, bones, 12), dtype=torch.float32, device="cuda") for _ in range(4)]
    for k in range(4):
        pick = rng.integers(0, m, size=t)
        ctx.decompress_tracks(clipset, as_dev(ab.make_requests(w["req_clip"][pick], w["req_time"][pick])), t, options, d_poses[k])
    d_records = torch.empty((t, bones, 16), dtype=torch.float32, device="cuda")
    ctx.begin_inertialization(*d_poses, t, bones, 30.0, d_records)
    d_inert = as_dev(ab.make_inertializations(rng.integers(0, t, size=m), rng.uniform(0.0, 0.5, m), 0.2))
    torch.cuda.synchronize()

    def route(kind, d_flags=None, d_fused_req=None):
        def launch(events):
            events[0].record()
            if kind == "fused_local":
                ctx.decompress_tracks_mirrored(clipset, d_fused_req, m, options, d_out, d_table, ab.MIRROR_X)
            elif kind == "fused_skinning":
                ctx.decompress_tracks_mirrored_skinning(clipset, d_fused_req, m, options, d_parents, d_inverse_bind, d_out, d_table, ab.MIRROR_X)
            elif kind == "skinning":
                ctx.decompress_tracks_skinning(clipset, d_req, m, options, d_parents, d_inverse_bind, d_out)
            elif kind == "inertialized_skinning":
                ctx.decompress_tracks_inertialized_skinning(clipset, d_none_req, m, options, d_parents, d_inverse_bind, d_out, d_records, t)
            elif kind == "mirror_poses":
                ctx.mirror_poses(d_out, d_out, m, bones, d_table, ab.MIRROR_X, d_mirrored=d_flags)
            elif kind == "mirrored_inertialized":
                ctx.decompress_tracks_mirrored(clipset, d_fused_req, m, options, d_out, d_table, ab.MIRROR_X)
                ctx.inertialize_poses(d_out, d_out, m, bones, d_inert, d_records, t)
                ctx.local_to_skinning(d_out, d_out, m, bones, d_parents, d_inverse_bind)
            else:
                ctx.decompress_tracks(clipset, d_req, m, options, d_out)
                if d_flags is not None:
                    ctx.mirror_poses(d_out, d_out, m, bones, d_table, ab.MIRROR_X, d_mirrored=d_flags)
                if kind == "unfused_skinning":
                    ctx.local_to_skinning(d_out, d_out, m, bones, d_parents, d_inverse_bind)
            events[1].record()
        return launch

    d_none_req = as_dev(ab.make_inertialized_requests(w["req_clip"], w["req_time"], ab.NO_INERTIALIZATION, 0.0, 0.2))
    routes = [("decode", route("decode")), ("skinning", route("skinning")), ("inertialized_skinning", route("inertialized_skinning"))]
    ctx.decompress_tracks(clipset, d_req, m, options, d_out)
    for percent in args.percents:
        flags = (rng.random(m) < percent / 100.0).astype(np.uint32)
        d_flags = as_dev(flags)
        d_fused_req = as_dev(ab.make_mirrored_requests(w["req_clip"], w["req_time"], flags))
        routes.append((f"fused_local_{percent}", route("fused_local", d_fused_req=d_fused_req)))
        routes.append((f"unfused_local_{percent}", route("unfused_local", d_flags=d_flags)))
        routes.append((f"fused_skinning_{percent}", route("fused_skinning", d_fused_req=d_fused_req)))
        routes.append((f"unfused_skinning_{percent}", route("unfused_skinning", d_flags=d_flags)))
        routes.append((f"mirror_poses_{percent}", route("mirror_poses", d_flags=d_flags)))
        routes.append((f"mirrored_inertialized_{percent}", route("mirrored_inertialized", d_fused_req=d_fused_req)))
    runs = []
    for _ in range(args.runs):
        runs.append({key + "_ms": round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4) for key, launch in routes})
    clipset.release()
    return {"workload": "c2", "requests": m, "bones": bones, "runs": runs}


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--steps", type=int, default=20)
    parser.add_argument("--warmup", type=int, default=5)
    parser.add_argument("--runs", type=int, default=3)
    parser.add_argument("--percents", type=int, nargs="+", default=[0, 50, 100])
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    print(json.dumps({"gpu": _gpu_description(), "result": measure(args, torch, ab, ctx)}))


if __name__ == "__main__":
    main()
