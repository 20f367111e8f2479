"""Timeline of the pipeline kernel's hand-overs (development helper, GPU box): needs a library built with -DACLB200_PIPE_TRACE=1
(ACLB200_OUT=$PWD/lib_trace.so sh acl_b200/csrc/build.sh -DACLB200_PIPE_TRACE=1, then
ACLB200_LIB=$PWD/lib_trace.so python tools/pipe_trace.py [--clips N] [--math exact|fast]).
Stamps per (block, iteration), SM clock cycles: 0 consumer starts waiting for the stage, 1 stage full, 2 last chunk decoded,
3 consumers' barrier passed, 4 stores handed to the TMA unit, 5 stores have read shared memory, 6 next loads issued, 7 seek done."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import acl_b200 as ab
import bench

ap = argparse.ArgumentParser()
ap.add_argument("--clips", type=int, default=2000)
ap.add_argument("--workload", default="c2")
ap.add_argument("--math", default="exact")
ap.add_argument("--blocks", type=int, default=64)
ap.add_argument("--iterations", type=int, default=24)
args = ap.parse_args()
w = bench.make_workload(args.workload, 0, args.clips)
ctx = ab.Context(0)
cs = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
req = ab.make_requests(w["req_clip"], w["req_time"])
d_req = torch.from_numpy(req.view(np.uint8)).cuda()
opts = ab.Options(output_layout=ab.LAYOUT_QVV40, math_mode=ab.MATH_FAST if args.math == "fast" else ab.MATH_EXACT)
out = torch.empty(len(req) * cs.max_tracks * 40, dtype=torch.uint8, device="cuda")
for _ in range(3):
    ctx.decompress_tracks(cs, d_req, len(req), opts, out)
trace = torch.zeros(args.blocks * args.iterations * 8, dtype=torch.int64, device="cuda")
ctx.debug_set_trace(trace, args.blocks, args.iterations)
ctx.decompress_tracks(cs, d_req, len(req), opts, out)
torch.cuda.synchronize()
ctx.debug_set_trace(None, 0, 0)
t = trace.cpu().numpy().reshape(args.blocks, args.iterations, 8).astype(np.float64)
ok = (t[:, :, :7] > 0).all(axis=2)
names = ["wait_full(1-0)", "decode(2-1)", "barrier(3-2)", "store_issue(4-3)", "store_read(5-4)", "load_issue(6-5)"]
res = {}
for k, name in enumerate(names):
    d = (t[:, 2:, k + 1] - t[:, 2:, k])[ok[:, 2:]]
    res[name] = {"median": float(np.median(d)), "p90": float(np.percentile(d, 90)), "mean": float(d.mean())}
cyc = (t[:, 3:, 0] - t[:, 2:-1, 0])[ok[:, 3:] & ok[:, 2:-1]]
res["iteration(0 to next 0)"] = {"median": float(np.median(cyc)), "p90": float(np.percentile(cyc, 90)), "mean": float(cyc.mean())}
lead = (t[:, 2:, 1] - t[:, 2:, 7])[ok[:, 2:]]
res["seek_lead(full - seek done)"] = {"median": float(np.median(lead))}
print(json.dumps({"unit": "SM clock cycles", "blocks": args.blocks, "iterations": args.iterations, "stats": res}, indent=1))
b0 = t[0] - t[0, 0, 0]
print("block 0 stamps relative to its first:")
for i in range(min(args.iterations, 12)):
    print("  it", i, [int(x) for x in b0[i]])
