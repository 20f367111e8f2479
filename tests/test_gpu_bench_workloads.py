"""GPU parity of the BENCHMARKED workloads, exhaustively: the exact request lists `bench.py` times (BASELINE.json configs
C2, C3, C4, C5 at full size, same seeds) are decoded in one launch through the C ABI and EVERY request is compared with the
unmodified reference (oracle/_ref: acl::decompression_context<benchmark settings>::seek + decompress_tracks into a
debug_track_writer style pose, oracle/ref_tool.cpp aclref_bench_transform / aclref_bench_scalar with an output buffer).
Mirrors what the reference's own validation walks (tools/acl_compressor/sources/validate_tracks.cpp:92-260,328-511).

Bar: ACLB200_MATH_EXACT bit-identical on every defined lane; ACLB200_MATH_FAST rotations <= 1e-5 absolute, translations and
scales bit-identical. The exhaustive tests need the compiled reference and are skipped without it; a fixed sample of the
same clips and requests is compared with the reference's stored output (tests/golden/bench_workloads.npz) everywhere.
"""
import numpy as np
import pytest

from tests import clips

pytestmark = pytest.mark.gpu

LANES = clips.DEFINED_LANES
FAST_MATH_TOLERANCE = 1e-5


@pytest.fixture(scope="module")
def env():
    import torch
    import acl_b200 as ab
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref/libaclref.so not built (needs /root/reference at build time)")
    ref.lib()
    return dict(torch=torch, ab=ab, ref=ref, ctx=ab.Context(0))


def _blobs(w):
    return [w["buffer"][int(o):int(o) + int(s)] for o, s in zip(w["offsets"], w["sizes"])]


def _compare_transform(env, w, clipset, slice_requests):
    """Decodes the whole request list in ONE launch per arithmetic mode (the launch bench.py times), then walks it slice by
    slice against the reference. Returns (requests compared, worst fast-math rotation error)."""
    torch, ab, ref, ctx = env["torch"], env["ab"], env["ref"], env["ctx"]
    n_req, tracks = len(w["req_clip"]), clipset.max_tracks
    requests = ab.make_requests(w["req_clip"], w["req_time"])
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_exact = torch.full((n_req, tracks, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n_req, ab.Options(output_layout=ab.LAYOUT_QVV48, math_mode=ab.MATH_EXACT), d_exact)
    d_fast = torch.full((n_req, tracks, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n_req, ab.Options(output_layout=ab.LAYOUT_QVV48, math_mode=ab.MATH_FAST), d_fast)
    # the 40 byte layout the bench measures carries the same bits
    d_40 = torch.full((n_req, tracks, 10), float("nan"), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n_req, ab.Options(output_layout=ab.LAYOUT_QVV40, math_mode=ab.MATH_EXACT), d_40)
    torch.cuda.synchronize()
    assert torch.equal(d_40.view(torch.int32), d_exact[:, :, LANES].contiguous().view(torch.int32))
    del d_40

    blobs = _blobs(w)
    lanes = torch.tensor(LANES, device="cuda")
    vector_lanes = torch.tensor([4, 5, 6, 8, 9, 10], device="cuda")
    worst_fast = 0.0
    for begin in range(0, n_req, slice_requests):
        end = min(begin + slice_requests, n_req)
        want = ref.decode_requests(blobs, w["req_clip"][begin:end], w["req_time"][begin:end], tracks)
        d_want = torch.from_numpy(want).cuda()
        got = d_exact[begin:end]
        same = torch.equal(got.index_select(2, lanes).view(torch.int32), d_want.index_select(2, lanes).view(torch.int32))
        if not same:
            diff = (got.index_select(2, lanes).view(torch.int32) != d_want.index_select(2, lanes).view(torch.int32)).nonzero()
            r, bone, lane = (int(v) for v in diff[0])
            raise AssertionError(f"request {begin + r} (clip {int(w['req_clip'][begin + r])}, t={float(w['req_time'][begin + r])}) bone {bone} lane {LANES[lane]}: "
                                 f"got {got[r, bone].tolist()} want {d_want[r, bone].tolist()} ({diff.shape[0]} differing values in this slice)")
        fast = d_fast[begin:end]
        worst_fast = max(worst_fast, float((fast[:, :, :4] - d_want[:, :, :4]).abs().max()))
        assert torch.equal(fast.index_select(2, vector_lanes).view(torch.int32), d_want.index_select(2, vector_lanes).view(torch.int32))
        del d_want
    assert worst_fast <= FAST_MATH_TOLERANCE, worst_fast
    return n_req, worst_fast


@pytest.mark.parametrize("name, slice_requests", [("c2", 60000), ("c3", 6000), ("c5", 125000)])
def test_bench_workload_every_request_vs_reference(env, name, slice_requests):
    import bench
    w = bench.make_workload(name, 0, None)
    assert w["distinct"], "the reference compressor is needed for the bench clips"
    clipset = env["ctx"].upload_packed(w["buffer"], w["offsets"], w["sizes"], check_hash=True)
    assert clipset.max_tracks == w["num_tracks"]
    compared, worst_fast = _compare_transform(env, w, clipset, slice_requests)
    assert compared == len(w["req_clip"])
    print(f"{name}: {compared} requests x {w['num_tracks']} bones bit-identical to the reference; fast math worst rotation error {worst_fast:.2e}")
    clipset.release()


@pytest.mark.parametrize("name", ["c2", "c5"])
def test_bench_workload_sample_vs_stored_reference(name):
    """A fixed sample of the benchmarked clips and requests (tests/golden/make_bench_golden.py) against what the reference decoded for
    them, stored with the clips: the same bar as above without the compiled reference. The sample must also still be what bench.py
    builds when the reference compressor is at hand."""
    import torch
    import acl_b200 as ab
    from oracle import ref
    golden = np.load(clips.golden_path("bench_workloads", "npz"))
    sizes = golden[f"{name}_sizes"]
    ends = np.cumsum(sizes.astype(np.int64))
    blobs = [ref.aligned_blob(golden[f"{name}_blobs"][end - size:end]) for size, end in zip(sizes, ends)]
    req_clip, req_time, want = golden[f"{name}_req_clip"], golden[f"{name}_req_time"], golden[f"{name}_want"]
    if ref.available():
        import bench
        w = bench.make_workload(name, 0, len(blobs))
        assert np.array_equal(np.concatenate([w["buffer"][int(o):int(o) + int(s)] for o, s in zip(w["offsets"], w["sizes"])]), golden[f"{name}_blobs"])
    ctx = ab.Context(0)
    clipset = ctx.upload(blobs, check_hash=True)
    n = len(req_clip)
    d_requests = torch.from_numpy(ab.make_requests(req_clip, req_time).view(np.uint8)).cuda()
    got = {}
    for mode in (ab.MATH_EXACT, ab.MATH_FAST):
        d_out = torch.full((n, clipset.max_tracks, 12), float("nan"), dtype=torch.float32, device="cuda")
        ctx.decompress_tracks(clipset, d_requests, n, ab.Options(output_layout=ab.LAYOUT_QVV48, math_mode=mode), d_out)
        torch.cuda.synchronize()
        got[mode] = d_out.cpu().numpy()[:, :, LANES]
    assert clips.bit_equal(got[ab.MATH_EXACT], want)
    assert clips.bit_equal(got[ab.MATH_FAST][:, :, 4:], want[:, :, 4:])
    assert float(np.abs(got[ab.MATH_FAST][:, :, :4] - want[:, :, :4]).max()) <= FAST_MATH_TOLERANCE
    clipset.release()


def test_bench_workload_c4_every_request_vs_reference(env):
    """C4: scalar float1f 4096 tracks x 1024 samples replicated x64, the 65 536 requests bench.py times."""
    import bench
    torch, ab, ref, ctx = env["torch"], env["ab"], env["ref"], env["ctx"]
    w = bench.make_workload("c4", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"], check_hash=True)
    n_req, tracks = len(w["req_clip"]), clipset.max_tracks
    assert tracks == 4096 and clipset.components == 1
    requests = ab.make_requests(w["req_clip"], w["req_time"])
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_out = torch.full((n_req, tracks), float("nan"), dtype=torch.float32, device="cuda")
    ctx.scalar_decompress_tracks(clipset, d_requests, n_req, ab.Options(), d_out)
    torch.cuda.synchronize()
    blobs = _blobs(w)
    for begin in range(0, n_req, 4096):
        end = min(begin + 4096, n_req)
        want = ref.decode_requests(blobs, w["req_clip"][begin:end], w["req_time"][begin:end], tracks, scalar=True)[:, :, 0]
        d_want = torch.from_numpy(np.ascontiguousarray(want)).cuda()
        assert torch.equal(d_out[begin:end].view(torch.int32), d_want.view(torch.int32)), f"requests {begin}..{end}"
    clipset.release()


# ------------------------------------------------------------------------------------------------------------------
# v02_00_00 clips: the raw bit rate marker is 32 instead of 31 (animated_track_cache.transform.h:523), scalar tracks use the 19 entry
# bit rate table (decompression.scalar.h:259-263), the wrap flag does not exist (compressed_tracks.impl.h:127-134). The compressor
# here only writes the latest version: the fixtures are golden blobs re-labelled on the host (version field, markers / table
# indices re-mapped so that the payload means the same, hash recomputed) and decoded by the unmodified reference. A scalar track
# whose bit rate the v02_00_00 table lacks (1, 2 or 20-23 bits) is re-quantized to the nearest rate it has (3 or 19 bits) and the
# key frame stream repacked: the payload then means something slightly different, which is fine, because the reference decodes the
# very same re-labelled clip.
# ------------------------------------------------------------------------------------------------------------------
def _fnv1a32(data: np.ndarray) -> int:
    acc = 2166136261
    for byte in data.tobytes():
        acc = ((acc ^ byte) * 16777619) & 0xFFFFFFFF
    return acc


def _as_version_7(blob: np.ndarray):
    """Returns (re-labelled blob, number of raw / re-mapped entries), or None when the clip cannot be expressed in v02_00_00."""
    b = blob.copy() if int(blob[15]) == 12 else _requantize_scalar_for_version_7(blob)
    u32 = lambda off: int(b[off:off + 4].view(np.uint32)[0])
    size = u32(0)
    track_type, misc = int(b[15]), u32(28)
    touched = 0
    if track_type == 12:
        if (misc >> 10) & 1 or (misc >> 30) & 1:
            return None                                  # stripped key frames / wrap optimised loops do not exist in v02_00_00
        num_segments, num_variable = u32(32), u32(36)
        headers = 32 + u32(32 + 36)
        for s in range(num_segments):
            data = 32 + u32(headers + 16 * s + 12)
            fmt = b[data:data + num_variable]
            touched += int((fmt == 31).sum())
            fmt[fmt == 31] = 32
    else:
        v10, v7 = V10_SCALAR_BITS, V7_SCALAR_BITS
        num_tracks = u32(16)
        meta = 32 + u32(32 + 4)
        rates = b[meta:meta + num_tracks]
        rates[:] = [v7.index(v10[r]) for r in rates]
        touched = num_tracks
    b[12:14] = np.array([7], dtype=np.uint16).view(np.uint8)
    b[4:8] = np.array([_fnv1a32(b[8:size])], dtype=np.uint32).view(np.uint8)
    return b, touched


V10_SCALAR_BITS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 32]
V7_SCALAR_BITS = [0, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 32]


def _requantize_scalar_for_version_7(blob: np.ndarray) -> np.ndarray:
    """A copy of a (latest version) scalar clip whose variable bit rates all exist in the v02_00_00 table: a 1 or 2 bit track becomes
    3 bits, a 20-23 bit track 19 bits (values shifted by the difference). The key frame stream is the clip's last section: frames of
    num_bits_per_frame bits, tracks in order, each animated track's components MSB first (decompression.scalar.h:212-481)."""
    u32 = lambda off: int(blob[off:off + 4].view(np.uint32)[0])
    size, num_tracks, num_samples = u32(0), u32(16), u32(20)
    components = int(blob[15]) + 1 if int(blob[15]) <= 3 else 4
    bits_per_frame, meta, animated = u32(32), 32 + u32(36), 32 + u32(48)
    old_bits = [V10_SCALAR_BITS[r] for r in blob[meta:meta + num_tracks]]
    new_bits = [x if x in V7_SCALAR_BITS else (3 if x < 3 else 19) for x in old_bits]
    if new_bits == old_bits:
        return blob.copy()
    old_bytes = (num_samples * bits_per_frame + 7) // 8
    stream = np.unpackbits(blob[animated:animated + old_bytes])
    new_bits_per_frame = components * sum(new_bits)
    out_stream = np.zeros(num_samples * new_bits_per_frame, dtype=np.uint8)
    weights = lambda n: (1 << np.arange(n - 1, -1, -1, dtype=np.uint64))
    for frame in range(num_samples):
        src, dst = frame * bits_per_frame, frame * new_bits_per_frame
        for old, new in zip(old_bits, new_bits):
            for _ in range(components if old else 0):
                value = int(stream[src:src + old].astype(np.uint64) @ weights(old))
                value = value >> (old - new) if old > new else value << (new - old)
                out_stream[dst:dst + new] = (value >> np.arange(new - 1, -1, -1)) & 1
                src, dst = src + old, dst + new
    tail = size - animated - old_bytes
    packed = np.packbits(out_stream)
    b = np.concatenate([blob[:animated], packed, np.zeros(tail, np.uint8)])
    b[0:4] = np.array([b.size], dtype=np.uint32).view(np.uint8)
    b[32:36] = np.array([new_bits_per_frame], dtype=np.uint32).view(np.uint8)
    b[meta:meta + num_tracks] = [V10_SCALAR_BITS.index(x) for x in new_bits]
    return b


@pytest.mark.parametrize("name", ["noisy_raw", "mixed_scale", "c1_30bones", "full_formats"])
def test_v02_00_00_transform_clip_vs_reference(env, name):
    torch, ab, ref, ctx = env["torch"], env["ab"], env["ref"], env["ctx"]
    made = _as_version_7(clips.load_blob(name))
    assert made is not None
    blob, raw_entries = made
    blob = ref.aligned_blob(blob)
    assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0, "the reference itself must accept the re-labelled clip (hash checked)"
    if name == "noisy_raw":
        assert raw_entries > 0, "this clip is here for its raw bit rate sub-tracks"
    clipset = ctx.upload([blob], check_hash=True)
    spec = clips.TRANSFORM_SPECS[name]
    times = clips.sample_times(spec)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_out = torch.full((len(times), clipset.max_tracks, 12), float("nan"), dtype=torch.float32, device="cuda")
    # debug settings: every format, version `any`, rotations always normalised
    options = ab.Options(normalization=ab.NORMALIZE_ALWAYS, per_track_rounding=1, multiple_rotation_formats=1,
                         default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_CONSTANT, ab.DEFAULT_LEGACY))
    ctx.decompress_tracks(clipset, d_requests, len(times), options, d_out)
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    for i, t in enumerate(times):
        want = ref.decompress_tracks(blob, float(t), settings=ref.SETTINGS_DEBUG, writer=ref.WRITER_LEGACY)
        assert clips.bit_equal(got[i][:, LANES], want[:, LANES]), (name, float(t))
    clipset.release()


@pytest.mark.parametrize("name", ["float1", "float2", "float3", "vector4"])
def test_v02_00_00_scalar_clip_vs_reference(env, name):
    torch, ab, ref, ctx = env["torch"], env["ab"], env["ref"], env["ctx"]
    made = _as_version_7(clips.load_blob(name))
    assert made is not None
    blob = ref.aligned_blob(made[0])
    assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0
    clipset = ctx.upload([blob], check_hash=True)
    spec = clips.SCALAR_SPECS[name]
    times = clips.sample_times(spec)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
    d_out = torch.full((len(times), clipset.max_tracks, clipset.components), float("nan"), dtype=torch.float32, device="cuda")
    ctx.scalar_decompress_tracks(clipset, d_requests, len(times), ab.Options(), d_out)
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    for i, t in enumerate(times):
        want = ref.scalar_decompress(blob, float(t))
        assert clips.bit_equal(got[i], want[:, :clipset.components]), (name, float(t))
    clipset.release()


def test_routed_c5_job_matches_reference_per_shard(env):
    """bench.py's routed C5 job (SURVEY 8e) on one GPU: the clip table is split with partition_clips, every shard becomes its own clip
    set, the global request list is bucketed with route_requests, each shard decodes its requests, and every pose is compared with
    the reference decoding the ORIGINAL (global) request. What N ranks do, shard after shard."""
    import bench
    from acl_b200 import sharding
    torch, ab, ref, ctx = env["torch"], env["ab"], env["ref"], env["ctx"]
    w = bench.make_workload("c5", 0, 3000)
    sizes = w["sizes"].astype(np.int64)
    blobs = _blobs(w)
    world = 3
    owner, local_index, bounds = sharding.partition_clips(sizes, world)
    rng = np.random.default_rng(11)
    req_clip = rng.permutation(len(blobs)).astype(np.uint32)
    req_time = (rng.random(len(blobs)) * (31 / 30.0)).astype(np.float32)
    want = ref.decode_requests(blobs, req_clip, req_time, 30)
    seen = 0
    for rank in range(world):
        lo, hi = bounds[rank]
        clipset = ctx.upload(blobs[lo:hi], check_hash=True)
        positions, local_clip, times = sharding.route_requests(req_clip, req_time, owner, local_index, rank)
        requests = ab.make_requests(local_clip, times)
        d_requests = torch.from_numpy(requests.view(np.uint8)).cuda()
        d_out = torch.zeros((len(requests), 30, 12), dtype=torch.float32, device="cuda")
        ctx.decompress_tracks(clipset, d_requests, len(requests), ab.Options(), d_out)
        torch.cuda.synchronize()
        got = d_out.cpu().numpy()
        assert clips.bit_equal(got[:, :, LANES], want[positions][:, :, LANES]), rank
        seen += len(positions)
        clipset.release()
    assert seen == len(req_clip)
