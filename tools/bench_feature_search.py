"""Motion matching timings on one GPU: the C2 clip set of bench.py, all 600,000 requests, through aclb200_extract_pose_features (S = 4
offsets {-1/30, 0, 1/3, 2/3} s, K = 4 bones: the root, two leaves and a mid bone of a binary tree skeleton, half the requests FEATURE_LOOP,
as tools/bench_features.py), packed into a database of
  D = 23 (stride 24)  two leaf positions at s = 1; the leaf and mid bone velocities between s = 0 and s = 1 (inv_dt = 30); the root's x / z
                      at s = 2 and 3; the root's z axis direction x / z at s = 2 and 3
  D = 64 (stride 64)  every entry's position at every offset, every entry's velocity between s = 0 and 1, the root's z axis x / z at s = 2, 3
then searched by Q in {1, 256, 4096} queries (database rows at random, each excluding its own row +-10), half the rows tagged out, by:
  fused     aclb200_search_pose_features (the results' init kernel and the search)
  chunked   torch: ((q - x)^2).sum(-1) over row chunks of at most 2^28 floats, tags and windows masked to +inf, min / argmin merged across
            chunks
  cdist     torch.cdist(q, x)^2 over row chunks, masked and merged the same way
The torch routes are compared on timing only: their float order is not the search's. Pack times (aclb200_pack_pose_features) of both
databases are in the same table. For each Q the least time is taken from shapes: 3 FLOP per (query, row, dimension) against the H100 SXM's
67 TFLOP/s FP32, and N * D * 4 bytes against 3.35 TB/s; the larger names the bound.
Cold data: a 256 MB scratch write precedes every timed launch. Each launch is timed with CUDA events; medians of --steps launches after
--warmup, for --runs runs with the routes alternating. The GPU's name, power limit and SM clock are read in the same run.

    python tools/bench_feature_search.py --steps 10 --warmup 3 --runs 2
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

OFFSETS = np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0], np.float32)
PEAK_FP32 = 67e12
PEAK_HBM = 3.35e12


def terms_for(ab, dims: int) -> tuple[np.ndarray, int]:
    P, V, Dn = ab.FEATURE_POSITION, ab.FEATURE_VELOCITY, ab.FEATURE_DIRECTION
    if dims == 23:
        terms = ab.make_feature_terms([P, P, V, V, V, P, P, Dn, Dn], [1, 1, 0, 0, 0, 2, 3, 2, 3], [1, 2, 1, 2, 3, 0, 0, 0, 0],
                                      [7, 7, 7, 7, 7, 5, 5, 5, 5], s1=1, axis=2, inv_dt=30.0)
        return terms, 24
    kinds = [P] * 16 + [V] * 4 + [Dn] * 2
    s0 = [s for s in range(4) for _ in range(4)] + [0] * 4 + [2, 3]
    k = [k for _ in range(4) for k in range(4)] + list(range(4)) + [0, 0]
    masks = [7] * 20 + [5, 5]
    return ab.make_feature_terms(kinds, s0, k, masks, s1=1, axis=2, inv_dt=30.0), 64


def torch_search(torch, d_db, dims, d_tags_ok, d_qv, source, window, use_cdist):
    """masked min / argmin over row chunks, merged with a strict < so the earlier chunk keeps a tie"""
    q, n = d_qv.shape[0], d_db.shape[0]
    chunk = max(1, (1 << 28) // (q * (1 if use_cdist else dims)))
    best = torch.full((q,), float("inf"), device="cuda")
    best_row = torch.full((q,), -1, dtype=torch.int64, device="cuda")
    queries = d_qv[:, :dims]
    for first in range(0, n, chunk):
        x = d_db[first:first + chunk, :dims]
        if use_cdist:
            cost = torch.cdist(queries, x).square()
        else:
            cost = (queries[:, None, :] - x[None, :, :]).square().sum(-1)
        rows = torch.arange(first, first + x.shape[0], device="cuda")
        allowed = d_tags_ok[first:first + x.shape[0]][None, :] & ((rows[None, :] - source[:, None]).abs() > window)
        cost = cost.masked_fill(~allowed | cost.isnan(), float("inf"))
        value, index = cost.min(1)
        better = value < best
        best = torch.where(better, value, best)
        best_row = torch.where(better, index + first, best_row)
    return best, best_row


def measure(args, torch, ab, ctx) -> dict:
    import bench
    from tests import bones_cases
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    clip, time = w["req_clip"].astype(np.uint32), w["req_time"].astype(np.float32)
    n, S, K = int(clip.size), OFFSETS.size, 4
    bones = w["num_tracks"]
    leaves = [b for b in range(bones) if 2 * b + 1 >= bones]
    bone_list = np.array([0, leaves[0], leaves[-1], bones // 4], np.uint32)
    requests = ab.make_feature_requests(clip, time, (np.arange(n) % 2).astype(np.uint32))
    d_rows = torch.zeros((n, S, K, 12), dtype=torch.float32, device="cuda")
    ctx.extract_pose_features(clipset, torch.from_numpy(requests.view(np.uint8)).cuda(), n, ab.Options(looping_policy=ab.LOOP_CLAMP), OFFSETS,
                              torch.from_numpy(bone_list.view(np.int32)).cuda(), K,
                              torch.from_numpy(bones_cases.tree(bones).view(np.int32)).cuda(), d_rows)
    clipset.release()
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)
    rng = np.random.default_rng(3)
    tags = (np.arange(n) % 2 + 1).astype(np.uint32)        # odd rows carry tag 2: tagged out of every query (mask 1)
    d_tags = torch.from_numpy(tags.view(np.int32)).cuda()
    d_tags_ok = d_tags == 1
    results = []
    for dims in (23, 64):
        terms, stride = terms_for(ab, dims)
        assert ab.feature_term_dims(terms) == dims
        d_db = torch.zeros((n, stride), dtype=torch.float32, device="cuda")
        pack = lambda events: (events[0].record(), ctx.pack_pose_features(d_rows, n, S, K, terms, d_db, stride), events[1].record())
        pack_ms = [round(_median_ms(torch, pack, flush, args.steps, args.warmup)[1], 4) for _ in range(args.runs)]
        mean, std = d_db[:, :dims].mean(0).cpu().numpy(), d_db[:, :dims].std(0).cpu().numpy()
        scale = np.where(std > 0, 1.0 / np.maximum(std, 1e-12), 1.0).astype(np.float32)
        ctx.pack_pose_features(d_rows, n, S, K, terms, d_db, stride, mean.astype(np.float32), scale)
        for q in args.queries:
            source = np.sort(rng.choice(n, q, replace=False)).astype(np.int64)
            d_qv = d_db[torch.from_numpy(source).cuda()].contiguous()
            d_source = torch.from_numpy(source).cuda()
            queries = ab.make_search_queries(1, np.maximum(source - 10, 0), source + 11)
            d_queries = torch.from_numpy(queries.view(np.uint8)).cuda()
            d_results = torch.empty((q, 2), dtype=torch.int32, device="cuda")

            def fused(events):
                events[0].record()
                ctx.search_pose_features(d_db, n, stride, d_qv, d_queries, q, stride, dims, d_results, d_row_tags=d_tags)
                events[1].record()

            def torch_route(use_cdist):
                def launch(events):
                    events[0].record()
                    torch_search(torch, d_db, dims, d_tags_ok, d_qv, d_source, 10, use_cdist)
                    events[1].record()
                return launch

            routes = {"fused": fused, "chunked": torch_route(False), "cdist": torch_route(True)}
            runs = []
            for _ in range(args.runs):
                runs.append({route: round(_median_ms(torch, launch, flush, args.steps if route == "fused" else args.torch_steps,
                                                     args.warmup if route == "fused" else 1)[1], 4) for route, launch in routes.items()})
            # the fused route's answers, against the torch route's rows where their costs agree (a spot check, not the bit test)
            fused([torch.cuda.Event(), torch.cuda.Event()])
            _, torch_rows = torch_search(torch, d_db, dims, d_tags_ok, d_qv, d_source, 10, False)
            torch.cuda.synchronize()
            agree = float((d_results[:, 0].long() == torch_rows).float().mean())
            flop, bytes_ = 3.0 * q * n * dims, 4.0 * n * dims
            compute_ms, hbm_ms = flop / PEAK_FP32 * 1e3, bytes_ / PEAK_HBM * 1e3
            fused_ms = float(np.median([r["fused"] for r in runs]))
            results.append({"dims": dims, "stride": stride, "rows": n, "queries": q, "runs": runs,
                            "least_ms": {"compute": round(compute_ms, 4), "hbm": round(hbm_ms, 4)},
                            "bound": "compute" if compute_ms > hbm_ms else "hbm",
                            "share_of_least": round(max(compute_ms, hbm_ms) / fused_ms, 3), "rows_equal_to_chunked": round(agree, 4)})
        results.append({"dims": dims, "stride": stride, "rows": n, "pack_ms": pack_ms, "pack_bytes": n * (S * K * 48 + stride * 4)})
    return results


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--queries", nargs="+", type=int, default=[1, 256, 4096])
    parser.add_argument("--steps", type=int, default=10)
    parser.add_argument("--warmup", type=int, default=3)
    parser.add_argument("--torch-steps", type=int, default=3)
    parser.add_argument("--runs", type=int, default=2)
    parser.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = parser.parse_args()

    import torch
    import acl_b200 as ab

    ctx = ab.Context(0)
    text = json.dumps({"gpu": _gpu_description(), "results": measure(args, torch, ab, ctx)})
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
