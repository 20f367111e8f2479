#!/usr/bin/env python
"""c2_traffic.py -- where the bytes of one pipeline kernel launch go, and how far the kernel is from its store floor.

    python tools/c2_traffic.py [--workload c2] [--clips N] [--requests-per-batch 10 --blocks 264] [--gpu]

Host part (no GPU needed): a model of the bytes the pipeline kernel (pipeline.cu) asks the memory system for, counted from the
layout upload builds (layout.h) and the workload's request list, with the kernel's own batching and grouping rules:
  windows      one TMA copy per group of chained requests (16 B aligned start, 16 B tail, rounded up to 16 B), two per request
               whose key frames sit in two segments
  tables       per group and animated sub-track: AnimDesc (32 B) + the Entry of its segment, loaded once per chain; the crossing
               request of a chain loads the next segment's Entry; requests outside a chain load their own
  base rows    the clip's base pose row, copied unless the pose row still holds the same clip's row (the tag check)
  seek         ClipDesc, start indices and the SegDesc of each key frame (32 B sectors)
`requested` is what the SMs fetch (served by L2 or by DRAM); `distinct` counts every byte once per launch: the DRAM floor if
L2 kept everything until its last use. Both are printed for the 32 B Entry the kernel used to read and the 16 B one it reads now.

GPU part (--gpu): in the same process, the C2 launch time in exact arithmetic (CUDA events, median) next to the floor of the same
number of output bytes written as pure 1-D bulk stores (cp.async.bulk shared -> global of one batch's pose rows, the loop of
tools/experiments/tma_store_floor.cu, compiled into a temporary directory), with the card's name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload synthesis, blob header parsing, clock sampling)

K_GROUP_MAX = 5             # pipeline.cu k_group_max
K_STAGES = 2                # pipeline.cu k_stages
ANIM_DESC_BYTES = 32        # layout.h AnimDesc
CLIP_DESC_BYTES = 128       # layout.h ClipDesc
SEG_DESC_BYTES = 32         # layout.h SegDesc


def clip_tables(w):
    """Per clip: tracks, samples, rate, segments, animated sub-tracks, segment starts and pose bits (from the compressed headers)."""
    buffer, offsets = w["buffer"], w["offsets"].astype(np.int64)
    f = lambda rel: bench.gather_u32(buffer, offsets + rel).astype(np.int64)
    num_tracks, num_samples, misc = f(16), f(20), f(28)
    rate = bench.gather_u32(buffer, offsets + 24).view(np.float32).astype(np.float64)
    nseg = f(32)
    nanim = f(40) + f(44) + f(48)
    seg_headers = f(68)
    stripped = (misc >> 10) & 1
    hsize = np.where(stripped == 1, 20, 16)
    max_seg = int(nseg.max())
    starts = np.full((len(offsets), max_seg + 1), np.iinfo(np.int64).max // 2, dtype=np.int64)
    pose_bits = np.zeros((len(offsets), max_seg), dtype=np.int64)
    for s in range(max_seg):
        valid = nseg > s
        pose_bits[valid, s] = bench.gather_u32(buffer, offsets[valid] + 32 + seg_headers[valid] + s * hsize[valid])
        multi = valid & (nseg > 1)
        starts[multi, s] = bench.gather_u32(buffer, offsets[multi] + 84 + 4 * s)
    starts[nseg == 1, 0] = 0
    return dict(num_tracks=num_tracks, num_samples=num_samples, rate=rate, nseg=nseg, nanim=nanim, starts=starts, pose_bits=pose_bits)


def model(w, requests_per_batch: int, blocks: int, entry_bytes: int, bone_bytes: int = 40) -> dict:
    """Bytes of one launch by kind: requested by the SMs and distinct (see the module docstring). Clamp looping, no rounding, no
    stripped key frames: what the bench workloads request."""
    t = clip_tables(w)
    clip = w["req_clip"].astype(np.int64)
    n = clip.size
    time = np.clip(w["req_time"].astype(np.float64), 0.0, None)
    last = t["num_samples"][clip] - 1
    k0 = np.minimum(np.floor(time * t["rate"][clip]).astype(np.int64), last)
    k1 = np.minimum(k0 + 1, last)
    starts = t["starts"][clip]
    seg0 = np.clip((starts <= k0[:, None]).sum(axis=1) - 1, 0, None)
    seg1 = np.clip((starts <= k1[:, None]).sum(axis=1) - 1, 0, None)
    rows = np.arange(n)
    pb0, pb1 = t["pose_bits"][clip, seg0], t["pose_bits"][clip, seg1]
    kf0 = (k0 - starts[rows, seg0]) * pb0
    kf1 = (k1 - starts[rows, seg1]) * pb1
    nanim = t["nanim"][clip]
    single = seg0 == seg1
    mergeable = single & (kf1 >= kf0) & (nanim > 0)
    crossing = ~single & (nanim > 0)

    # grouping (produce_pass): a request joins its predecessor of the same batch (and seek pass of 32) when both read the same
    # segment's tables and its first key frame is the predecessor's second; runs are cut every K_GROUP_MAX requests
    local = rows % requests_per_batch
    prev = np.maximum(rows - 1, 0)
    join = (local % 32 != 0) & (mergeable | crossing) & mergeable[prev] & (clip == clip[prev]) & (seg0 == seg0[prev]) & (kf0 == kf1[prev])
    join[0] = False
    run_start = np.maximum.accumulate(np.where(~join, rows, 0))
    head = ~join | ((rows - run_start) % K_GROUP_MAX == 0)
    group = np.cumsum(head) - 1
    heads = np.flatnonzero(head)
    count = np.diff(np.append(heads, n))
    tail_crossing = crossing & ~head
    last_is_crossing = tail_crossing[heads + count - 1]
    plain = count - last_is_crossing

    # key frame windows
    win = np.zeros(n, dtype=np.int64)
    tail16 = lambda bits: ((((bits + 7) >> 3) + 16 + 15) // 16) * 16
    merged_head = heads[mergeable[heads]]
    src_byte = ((kf0[merged_head] >> 3) // 16) * 16
    last_plain = merged_head + plain[mergeable[heads]] - 1
    win[merged_head] = tail16(kf1[last_plain] + pb1[last_plain] - src_byte * 8)
    second = tail_crossing | (~mergeable & ~tail_crossing & (nanim > 0))
    first = ~mergeable & ~tail_crossing & (nanim > 0)
    bit0 = kf0 - ((kf0 >> 3) // 16) * 128
    bit1 = kf1 - ((kf1 >> 3) // 16) * 128
    win += np.where(first, tail16(bit0 + pb0), 0) + np.where(second, tail16(bit1 + pb1), 0)

    # tables: chains (2+ requests) load once per group, the rest once per request
    chained = count >= 2
    group_tables = nanim[heads] * (ANIM_DESC_BYTES + entry_bytes)
    tables = int(np.where(chained, group_tables + last_is_crossing * nanim[heads] * entry_bytes, 0).sum())
    alone = ~chained[group]
    tables += int((nanim * (ANIM_DESC_BYTES + entry_bytes * np.where(single, 1, 2)))[alone].sum())

    # base pose rows: a pose row of (block, stage, slot) keeps its clip's base row from batch i - K_STAGES of the same block
    num_batches = (n + requests_per_batch - 1) // requests_per_batch
    share, remainder = divmod(num_batches, blocks)
    batch = rows // requests_per_batch
    block_first = np.arange(blocks) * share + np.minimum(np.arange(blocks), remainder)
    block = np.searchsorted(block_first, batch, side="right") - 1
    iteration = batch - block_first[block]
    earlier = np.maximum(rows - K_STAGES * requests_per_batch, 0)
    copied = (iteration < K_STAGES) | (clip != clip[earlier])
    row_bytes = ((t["num_tracks"][clip] * bone_bytes + 15) // 16) * 16
    base = int(row_bytes[copied].sum())

    seek = int((CLIP_DESC_BYTES + np.where(t["nseg"][clip] > 1, 32, 0) + SEG_DESC_BYTES * np.where(single, 1, 2)).sum())

    # distinct: every touched segment's tables and key frames, every touched clip's AnimDesc, base row and ClipDesc once
    touched_clips = np.unique(clip)
    max_seg = t["pose_bits"].shape[1]
    touched_seg = np.unique(np.concatenate([clip * max_seg + seg0, clip * max_seg + seg1]))
    seg_clip, seg_index = touched_seg // max_seg, touched_seg % max_seg
    keys = np.unique(np.concatenate([clip * 4096 + k0, clip * 4096 + k1]))
    key_clip, key_frame = keys // 4096, keys % 4096
    key_seg = np.clip((t["starts"][key_clip] <= key_frame[:, None]).sum(axis=1) - 1, 0, None)
    distinct = {
        "windows": int(((t["pose_bits"][key_clip, key_seg] + 7) // 8).sum()),
        "entry_tables": int((t["nanim"][seg_clip] * entry_bytes).sum()),
        "anim_desc": int((t["nanim"][touched_clips] * ANIM_DESC_BYTES).sum()),
        "base_rows": int((((t["num_tracks"][touched_clips] * bone_bytes + 15) // 16) * 16).sum()),
        "seek": int(touched_clips.size * CLIP_DESC_BYTES + seg_index.size * SEG_DESC_BYTES),
    }
    requested = {"windows": int(win.sum()), "tables": tables, "base_rows": base, "seek": seek}
    return {"entry_bytes": entry_bytes, "requests": int(n), "groups": int(heads.size), "chained_groups": int(chained.sum()),
            "requested": requested, "requested_total": int(sum(requested.values())),
            "distinct": distinct, "distinct_total": int(sum(distinct.values())),
            "pose_bytes_written": int((t["num_tracks"][clip] * bone_bytes).sum())}


STORE_FLOOR_SOURCE = r"""
#include <cstdint>
#include <cuda_runtime.h>
// Pure 1-D bulk stores: each block owns a contiguous range of the output and loops: fence -> one cp.async.bulk of `chunk` bytes from
// shared memory -> commit; a stage is reused once wait_group.read says the copy has read it (tools/experiments/tma_store_floor.cu).
__global__ void __launch_bounds__(128) store_floor_kernel(uint8_t* out, uint64_t total_bytes, uint32_t chunk)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const uint64_t chunks = total_bytes / chunk;
    const uint64_t share = chunks / gridDim.x, rem = chunks % gridDim.x;
    const uint64_t first = blockIdx.x * share + (blockIdx.x < rem ? blockIdx.x : rem);
    const uint64_t count = share + (blockIdx.x < rem ? 1 : 0);
    for (uint64_t i = 0; i < count; ++i)
    {
        uint8_t* stage = smem + (i % 2) * chunk;
        if (threadIdx.x == 0 && i >= 2)
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        __syncthreads();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (threadIdx.x == 0)
        {
            const uint32_t src = static_cast<uint32_t>(__cvta_generic_to_shared(stage));
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(out + (first + i) * chunk), "r"(src), "r"(chunk) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (threadIdx.x == 0)
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// median of `repeats` launches in ms; `out` holds total_bytes
extern "C" int store_floor_ms(void* out, uint64_t total_bytes, uint32_t chunk, int blocks, int repeats, float* median_ms)
{
    if (cudaFuncSetAttribute(store_floor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * chunk) != cudaSuccess)
        return 1;
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    float times[64];
    repeats = repeats > 64 ? 64 : repeats;
    for (int r = -2; r < repeats; ++r)
    {
        cudaEventRecord(a);
        store_floor_kernel<<<blocks, 128, 2 * chunk>>>(static_cast<uint8_t*>(out), total_bytes, chunk);
        cudaEventRecord(b);
        if (cudaEventSynchronize(b) != cudaSuccess)
            return 2;
        if (r >= 0)
            cudaEventElapsedTime(&times[r], a, b);
    }
    cudaEventDestroy(a); cudaEventDestroy(b);
    for (int i = 1; i < repeats; ++i)
        for (int j = i; j > 0 && times[j] < times[j - 1]; --j) { float t = times[j]; times[j] = times[j - 1]; times[j - 1] = t; }
    *median_ms = times[repeats / 2];
    return 0;
}
"""


def build_store_floor(directory: str) -> ctypes.CDLL:
    source = os.path.join(directory, "store_floor.cu")
    library = os.path.join(directory, "libstore_floor.so")
    with open(source, "w") as f:
        f.write(STORE_FLOOR_SOURCE)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-shared", "-o", library, source],
                   check=True, capture_output=True)
    lib = ctypes.CDLL(library)
    lib.store_floor_ms.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    lib.store_floor_ms.restype = ctypes.c_int
    return lib


def card() -> dict:
    query = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    parts = [p.strip() for p in out.stdout.strip().split(",")] if out.returncode == 0 else []
    return dict(zip(query.split(","), parts)) if len(parts) == 3 else {"nvidia-smi": out.stderr.strip() or "unavailable"}


def gpu_part(w, steps: int, warmup: int) -> dict:
    import torch
    import acl_b200 as ab

    if not torch.cuda.is_available():
        raise SystemExit("--gpu needs a CUDA device")
    torch.cuda.set_device(0)
    ctx = ab.Context(0)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    requests = ab.make_requests(w["req_clip"], w["req_time"])
    num_requests = len(requests)
    options = ab.Options(output_layout=ab.LAYOUT_QVV40, math_mode=ab.MATH_EXACT)
    pose_bytes = clipset.max_tracks * 40
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_out = torch.empty(num_requests * pose_bytes, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()
    launch = lambda: ctx.decompress_tracks(clipset, d_requests, num_requests, options, d_out, stream)
    sampler = bench.ClockSampler(0)
    sampler.start()
    _, kernel_ms = bench.time_launches(torch, launch, stream, steps, warmup, torch.cuda.synchronize, sampler)
    clocks = sampler.stop()
    plan = ctx.debug_last_launch()

    # the floor: the same output bytes as one batch's pose rows per bulk store, from as many blocks as the pipeline kernel runs
    chunk = plan.requests_per_block * pose_bytes
    total = (d_out.numel() // chunk) * chunk
    with tempfile.TemporaryDirectory() as directory:
        lib = build_store_floor(directory)
        floor_ms = ctypes.c_float()
        status = lib.store_floor_ms(ctypes.c_void_p(d_out.data_ptr()), total, chunk, plan.grid_blocks, 20, ctypes.byref(floor_ms))
        if status != 0:
            raise SystemExit(f"store floor kernel failed ({status})")
    floor = float(floor_ms.value) * d_out.numel() / total
    return {"card": card(), "clocks_during_c2": clocks, "plan": {"requests_per_batch": plan.requests_per_block, "blocks": plan.grid_blocks,
            "kernel": plan.kernel_name}, "c2_kernel_ms": kernel_ms, "store_floor_ms": floor, "store_chunk_bytes": chunk,
            "store_floor_gbs": d_out.numel() / floor / 1e6, "c2_over_floor": kernel_ms / floor}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workload", default="c2", choices=["c2", "c3", "c5"])
    ap.add_argument("--clips", type=int, default=None, help="fewer clips (rehearsal)")
    ap.add_argument("--requests-per-batch", type=int, default=10, help="C2 on an H100 (plan_pipeline); --gpu reads the real plan")
    ap.add_argument("--blocks", type=int, default=264, help="2 x the 132 SMs of an H100 SXM; --gpu reads the real plan")
    ap.add_argument("--gpu", action="store_true", help="also time the kernel and the store floor on cuda:0")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    w = bench.make_workload(args.workload, 0, args.clips)
    result = {"workload": args.workload, "clips": int(w["num_clips"]), "distinct_clips": bool(w["distinct"])}
    rpb, blocks = args.requests_per_batch, args.blocks
    if args.gpu:
        result["gpu"] = gpu_part(w, args.steps, args.warmup)
        rpb, blocks = result["gpu"]["plan"]["requests_per_batch"], result["gpu"]["plan"]["blocks"]
    result["model"] = {f"entry_{e}B": model(w, rpb, blocks, e) for e in (32, 16)}

    mb = lambda v: f"{v / 1e6:9.1f} MB"
    for name, m in result["model"].items():
        print(f"{name}: {m['requests']} requests, {m['groups']} groups ({m['chained_groups']} chained), batches of {rpb}, {blocks} blocks", file=sys.stderr)
        for kind, value in m["requested"].items():
            print(f"  requested {kind:<12}{mb(value)}", file=sys.stderr)
        print(f"  requested total     {mb(m['requested_total'])}", file=sys.stderr)
        for kind, value in m["distinct"].items():
            print(f"  distinct  {kind:<12}{mb(value)}", file=sys.stderr)
        print(f"  distinct  total     {mb(m['distinct_total'])}   (pose rows written: {mb(m['pose_bytes_written'])})", file=sys.stderr)
    if args.gpu:
        g = result["gpu"]
        print(f"{g['card']}: C2 exact {g['c2_kernel_ms']:.3f} ms, store floor {g['store_floor_ms']:.3f} ms ({g['store_floor_gbs']:.0f} GB/s), "
              f"C2 / floor = {g['c2_over_floor']:.3f}, SM clock {g['clocks_during_c2'].get('sm_mhz')} MHz", file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
