"""Masked layered decode timings on one GPU: the four layer C2 and C3 stacks of tools/bench_layers.py (base, two BLEND layers with weights
uniform in [0, 1], an ADDITIVE additive0 layer; binary tree skeleton, random affine inverse binds), per launch:
  fused_local        aclb200_decompress_tracks_layered, local QVV48 rows (no masks; the ADDITIVE layer is fully on)
  fused_skinning     aclb200_decompress_tracks_layered_skinning
  masked_local       aclb200_decompress_tracks_layered_masked: both BLEND layers under an upper-body mask (the upper half of the bones 1,
                     the lower half 0, a feather band of 0.25 / 0.5 / 0.75 at the boundary), the ADDITIVE layer at weight 0.5
  masked_skinning    aclb200_decompress_tracks_layered_masked_skinning, same stacks
  masked01_local     the masked route with the 0/1 mask (no feather band) and the ADDITIVE layer fully on: what the route below computes
  two_pass_select    what the 0/1 mask replaces: aclb200_decompress_tracks_layered of the full stack and of the stack with both BLEND layers
                     OFF, then a per-bone select of the two (torch.where) into the output
Cold data: a 256 MB scratch write precedes every timed launch. Medians of --steps launches after --warmup, for --runs runs. The GPU's name,
power limit and SM clock are read in the same run.

    python tools/bench_masked_layers.py --workloads c2 c3 --steps 20 --warmup 5 --runs 2
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
    as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()
    ops = np.array([[ab.LAYER_BLEND, ab.LAYER_BLEND, ab.LAYER_BLEND, ab.LAYER_ADDITIVE]], np.uint32)

    def layers(additive_weight, blend_off=False):
        o = np.broadcast_to(ops, (m, 4)).copy()
        if blend_off:
            o[:, 1:3] = ab.LAYER_OFF
        return as_dev(ab.make_layers(np.stack(clip, 1), np.stack(time, 1), o, np.stack(weights + [np.full(m, additive_weight, np.float32)], 1)))

    d_full, d_half_weight, d_without = layers(1.0), layers(0.5), layers(1.0, blend_off=True)
    upper01 = (np.arange(bones) >= bones // 2).astype(np.float32)
    feather = upper01.copy()
    feather[bones // 2 - 3:bones // 2] = [0.25, 0.5, 0.75]
    d_masks = torch.from_numpy(np.stack([feather, upper01])).cuda()
    d_layer_masks = [as_dev(np.tile(np.array([ab.LAYER_NO_MASK, k, k, ab.LAYER_NO_MASK], np.uint32), m)) for k in (0, 1)]
    d_select = torch.from_numpy(upper01 != 0).cuda()[None, :, None]
    options = ab.Options()
    d_out = torch.empty((m, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    d_other = torch.empty_like(d_out)
    scratch = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    flush = lambda: scratch.fill_(1)
    kw = dict(additive_format=ab.ADDITIVE_ADDITIVE0)

    def plain(to_skinning):
        def launch(events):
            events[0].record()
            if to_skinning:
                ctx.decompress_tracks_layered_skinning(clipset, d_full, m, 4, options, d_parents, d_inverse, d_out, **kw)
            else:
                ctx.decompress_tracks_layered(clipset, d_full, m, 4, options, d_out, **kw)
            events[1].record()
        return launch

    def masked(d_layers, mask, to_skinning=False):
        mkw = dict(d_layer_masks=d_layer_masks[mask], d_bone_masks=d_masks, num_masks=2, **kw)
        def launch(events):
            events[0].record()
            if to_skinning:
                ctx.decompress_tracks_layered_masked_skinning(clipset, d_layers, m, 4, options, d_parents, d_inverse, d_out, **mkw)
            else:
                ctx.decompress_tracks_layered_masked(clipset, d_layers, m, 4, options, d_out, **mkw)
            events[1].record()
        return launch

    def two_pass(events):
        events[0].record()
        ctx.decompress_tracks_layered(clipset, d_full, m, 4, options, d_out, **kw)
        ctx.decompress_tracks_layered(clipset, d_without, m, 4, options, d_other, **kw)
        torch.where(d_select, d_out[:, :bones], d_other[:, :bones], out=d_out[:, :bones])
        events[1].record()

    # the 0/1 masked route computes what the two passes select: checked once before timing
    masked(d_full, 1)([torch.cuda.Event(), torch.cuda.Event()])
    single = d_out.clone()
    two_pass([torch.cuda.Event(), torch.cuda.Event()])
    torch.cuda.synchronize()
    same = bool(torch.equal(single[:, :bones].view(torch.int32), d_out[:, :bones].view(torch.int32)))

    runs = []
    for _ in range(args.runs):
        times = {}
        for key, launch in (("fused_local", plain(False)), ("masked_local", masked(d_half_weight, 0)), ("fused_skinning", plain(True)),
                            ("masked_skinning", masked(d_half_weight, 0, True)), ("masked01_local", masked(d_full, 1)),
                            ("two_pass_select", two_pass)):
            times[key + "_ms"] = round(_median_ms(torch, launch, flush, args.steps, args.warmup)[1], 4)
        runs.append(times)
    clipset.release()
    return {"workload": name, "poses": m, "bones": bones, "masked01_equals_two_pass_select": same, "runs": runs}


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
