"""Small workload for compute-sanitizer (tools/sanitize.sh): every kernel of the library once or twice, checked against the oracle --
chained playback through the pipeline kernel (groups, tail crossing, base row reuse), ragged random requests, per track rounding,
skipped defaults (plain kernels), decompress_track, the object space decode (both kinds, a skeleton per clip), the additive decode (local and
object space, per clip formats) and aclb200_apply_additive_to_base, the blend decode (local and object space, a weight per pair) and
aclb200_blend_poses, the skinning decodes, the layered decode (local, object space and skinning rows), the chained scalar kernel."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import acl_b200 as ab
from oracle import object_space, port
from tests import clips

L = clips.DEFINED_LANES
ctx = ab.Context(0)
names = ["c2_100bones", "mixed_scale", "stripped_loop", "c1_30bones", "ragged_17", "full_formats"]
blobs = [clips.load_blob(n) for n in names]
cs = ctx.upload(blobs, check_hash=True)
settings = port.settings_for_kind(0)
# sequential playback of every clip (chains + segment crossings), then random requests
req_clip, req_time = [], []
for c, n in enumerate(names):
    spec = clips.TRANSFORM_SPECS[n]
    for s in range(spec.num_samples):
        req_clip.append(c); req_time.append((s + 0.37) / spec.sample_rate)
rng = np.random.default_rng(0)
for _ in range(200):
    c = int(rng.integers(0, len(names))); req_clip.append(c); req_time.append(float(rng.uniform(-0.1, 2.5)))
req_clip = np.array(req_clip, np.uint32); req_time = np.array(req_time, np.float32)
req = ab.make_requests(req_clip, req_time)
d_req = torch.from_numpy(req.view(np.uint8)).cuda()
bad = 0
for layout, width in ((ab.LAYOUT_QVV48, 12), (ab.LAYOUT_QVV40, 10)):
    for math in (ab.MATH_EXACT, ab.MATH_FAST):
        out = torch.zeros((len(req), cs.max_tracks, width), dtype=torch.float32, device="cuda")
        ctx.decompress_tracks(cs, d_req, len(req), ab.Options(output_layout=layout, math_mode=math), out)
        torch.cuda.synchronize()
        if math == ab.MATH_EXACT and layout == ab.LAYOUT_QVV48:
            got = out.cpu().numpy()
            for i in range(0, len(req), 3):
                want = port.transform_decompress_tracks(blobs[req_clip[i]], settings, float(req_time[i]))
                bad += not clips.bit_equal(got[i, :want.shape[0]][:, L], want[:, L])
# per track rounding + always normalisation (generic consumers), skipped defaults (plain kernels), decompress_track
debug = port.settings_for_kind(1)
policies = torch.from_numpy(rng.integers(0, 4, cs.max_tracks).astype(np.uint8)).cuda()
out = torch.zeros((len(req), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
ctx.decompress_tracks(cs, d_req, len(req), ab.Options(normalization=ab.NORMALIZE_ALWAYS, per_track_rounding=1, rounding_policy=ab.ROUND_PER_TRACK,
                                                      d_per_track_rounding=policies.data_ptr(), multiple_rotation_formats=1), out)
ctx.decompress_tracks(cs, d_req, len(req), ab.Options(default_modes=(ab.DEFAULT_SKIPPED, ab.DEFAULT_SKIPPED, ab.DEFAULT_SKIPPED), skip_mask=ab.SKIP_SCALE), out)
tracks = torch.from_numpy(rng.integers(0, 17, len(req)).astype(np.uint32)).cuda()
one = torch.zeros((len(req), 12), dtype=torch.float32, device="cuda")
ctx.decompress_track(cs, d_req, tracks, len(req), ab.Options(), one)
torch.cuda.synchronize()
# object space decode: the OBJECT = true instances of the plain kernel, a binary tree skeleton per clip
counts = [clips.TRANSFORM_SPECS[n].num_tracks for n in names]
trees = [np.array([0xFFFFFFFF] + [(b - 1) // 2 for b in range(1, n)], np.uint32) for n in counts]
d_parents = torch.from_numpy(np.concatenate(trees)).cuda()
d_offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)).cuda()
for kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
    out = torch.zeros((len(req), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_object_space(cs, d_req, len(req), ab.Options(), d_parents, kind, out, d_skeleton_offsets=d_offsets)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(0, len(req), 7):
        c = req_clip[i]
        local = port.transform_decompress_tracks(blobs[c], settings, float(req_time[i]))
        if kind == ab.OBJECT_MATRIX3X4F:
            bad += not clips.bit_equal(got[i, :counts[c]], object_space.port_local_to_object_space_matrix(local, trees[c]))
        else:
            bad += not clips.bit_equal(got[i, :counts[c]][:, L], port.local_to_object_space(local, trees[c], port.NORMALIZE_IEEE)[:, L])
# additive decode: the ADDITIVE = true instances (pairs of clips with equal bone counts, every format, local then object space) and the
# standalone apply_additive_kernel, in place
pair_clip = np.array([c for c in range(len(names)) for _ in range(8)], np.uint32)
pair_time = rng.uniform(-0.1, 2.5, (len(pair_clip), 2)).astype(np.float32)
pairs = ab.make_additive_requests(pair_clip, pair_time[:, 0], pair_clip, pair_time[:, 1])
d_pairs = torch.from_numpy(pairs.view(np.uint8)).cuda()
d_formats = torch.from_numpy(np.arange(len(names), dtype=np.uint8) % 5).cuda()
writer = port.settings_for_kind(0, constant_defaults=np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32))
for parents in (None, d_parents):
    out = torch.zeros((len(pairs), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_additive(cs, d_pairs, len(pairs), ab.Options(), out, d_clip_additive_formats=d_formats, d_parent_indices=parents,
                                   d_skeleton_offsets=d_offsets)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(0, len(pairs), 5):
        c = pair_clip[i]
        base = port.transform_decompress_tracks(blobs[c], settings, float(pair_time[i, 0]))
        additive = port.transform_decompress_tracks(blobs[c], writer, float(pair_time[i, 1]))
        want = port.apply_additive_to_base(int(c % 5) if c % 5 <= 3 else 0, base, additive, port.NORMALIZE_IEEE)
        if parents is not None:
            want = port.local_to_object_space(want, trees[c], port.NORMALIZE_IEEE)
        bad += not clips.bit_equal(got[i, :counts[c]][:, L], want[:, L])
ctx.apply_additive_to_base(out, out, out, len(pairs), cs.max_tracks, ab.ADDITIVE_ADDITIVE0)
torch.cuda.synchronize()
# blend decode: the PAIR = blend instances (pairs of clips with equal bone counts, a weight per pair, local then object space) and the
# standalone blend_poses_kernel, in place
from oracle import blend
blend_pairs = ab.make_blend_requests(pair_clip, pair_time[:, 0], pair_clip, pair_time[:, 1])
d_blend_pairs = torch.from_numpy(blend_pairs.view(np.uint8)).cuda()
blend_weights = rng.uniform(-0.25, 1.25, len(blend_pairs)).astype(np.float32)
d_blend_weights = torch.from_numpy(blend_weights).cuda()
for parents in (None, d_parents):
    out = torch.zeros((len(blend_pairs), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_blend(cs, d_blend_pairs, len(blend_pairs), ab.Options(), out, d_weights=d_blend_weights, d_parent_indices=parents,
                                d_skeleton_offsets=d_offsets)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(0, len(blend_pairs), 5):
        c = pair_clip[i]
        want = blend.port_qvv_lerp(port.transform_decompress_tracks(blobs[c], settings, float(pair_time[i, 0])),
                                   port.transform_decompress_tracks(blobs[c], settings, float(pair_time[i, 1])), float(blend_weights[i]))
        if parents is not None:
            want = port.local_to_object_space(want, trees[c], port.NORMALIZE_IEEE)
        bad += not clips.bit_equal(got[i, :counts[c]][:, L], want[:, L])
ctx.blend_poses(out, out, out, len(blend_pairs), cs.max_tracks, d_weights=d_blend_weights)
torch.cuda.synchronize()
# skinning decodes: the object, additive and blend instances with the skinning step (per clip skeletons and inverse binds), and the
# standalone local_to_skinning_kernel, in place
from oracle import skinning
from tests import skinning_cases
inverses = [skinning_cases.random_affine(int(counts[c]), c, mirrored=True) for c in range(len(names))]
d_inverse = torch.from_numpy(np.concatenate(inverses)).cuda()
out = torch.zeros((len(req), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
ctx.decompress_tracks_skinning(cs, d_req, len(req), ab.Options(), d_parents, d_inverse, out, d_skeleton_offsets=d_offsets)
torch.cuda.synchronize()
got = out.cpu().numpy()
for i in range(0, len(req), 7):
    c = req_clip[i]
    local = port.transform_decompress_tracks(blobs[c], settings, float(req_time[i]))
    bad += not clips.bit_equal(got[i, :counts[c]], skinning.port_local_to_skinning(local, trees[c], inverses[c]))
out = torch.zeros((len(pairs), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
ctx.decompress_tracks_additive_skinning(cs, d_pairs, len(pairs), ab.Options(), d_parents, d_inverse, out, d_clip_additive_formats=d_formats,
                                        d_skeleton_offsets=d_offsets)
ctx.decompress_tracks_blend_skinning(cs, d_blend_pairs, len(blend_pairs), ab.Options(), d_parents, d_inverse, out, d_weights=d_blend_weights,
                                     d_skeleton_offsets=d_offsets)
one = ctx.upload([blobs[0]])
local = torch.zeros((64, one.max_tracks, 12), dtype=torch.float32, device="cuda")
ctx.decompress_tracks(one, torch.from_numpy(ab.make_requests(np.zeros(64), np.linspace(0, 1, 64)).view(np.uint8)).cuda(), 64, ab.Options(), local)
ctx.local_to_skinning(local, local, 64, one.max_tracks, d_parents, d_inverse)
torch.cuda.synchronize()
one.release()
# layered decode: the layers instances (three layer stacks of one clip each: base, BLEND, ADDITIVE with the per clip formats, the middle
# layer OFF on every other stack), local, object space and skinning rows
from tests import layers_cases
stacks = [[(c, float(pair_time[i, 0]), layers_cases.BLEND, 0.0),
           (c, float(pair_time[i, 1]), layers_cases.BLEND if i % 2 else layers_cases.OFF, float(blend_weights[i])),
           (c, float(pair_time[i, 0]) * 0.5, layers_cases.ADDITIVE, 0.0)] for i, c in enumerate(pair_clip)]
stack_values = np.array(stacks, np.float64)
d_layers = torch.from_numpy(ab.make_layers(stack_values[..., 0].astype(np.uint32), stack_values[..., 1], stack_values[..., 2].astype(np.uint32),
                                           stack_values[..., 3]).reshape(-1).view(np.uint8)).cuda()
for parents in (None, d_parents):
    out = torch.zeros((len(stacks), cs.max_tracks, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_layered(cs, d_layers, len(stacks), 3, ab.Options(), out, d_clip_additive_formats=d_formats, d_parent_indices=parents,
                                  d_skeleton_offsets=d_offsets)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(0, len(stacks), 5):
        c = pair_clip[i]
        want = layers_cases.port_local(port, blend, blobs, stacks[i], settings, writer, 0, 2, clip_formats=np.arange(len(names)) % 5)
        if parents is not None:
            want = port.local_to_object_space(want, trees[c], port.NORMALIZE_IEEE)
        bad += not clips.bit_equal(got[i, :counts[c]][:, L], want[:, L])
ctx.decompress_tracks_layered_skinning(cs, d_layers, len(stacks), 3, ab.Options(), d_parents, d_inverse, out, d_clip_additive_formats=d_formats,
                                       d_skeleton_offsets=d_offsets)
torch.cuda.synchronize()
# scalar clips
for name in ("float1", "float3", "vector4", "float1_c4_small"):
    blob = clips.load_blob(name); spec = clips.SCALAR_SPECS[name]
    scs = ctx.upload([blob])
    times = np.concatenate([(np.arange(spec.num_samples) + 0.4) / spec.sample_rate, rng.uniform(-0.1, 3.0, 40)]).astype(np.float32)
    sreq = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_sreq = torch.from_numpy(sreq.view(np.uint8)).cuda()
    sout = torch.zeros((len(times), scs.max_tracks, scs.components), dtype=torch.float32, device="cuda")
    ctx.scalar_decompress_tracks(scs, d_sreq, len(times), ab.Options(), sout)
    torch.cuda.synchronize()
    got = sout.cpu().numpy()
    scs.release()
print("driver done, mismatches vs oracle:", bad)
sys.exit(1 if bad else 0)
