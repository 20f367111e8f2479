"""The chained scalar kernel (scalar_tracks_pipeline_kernel) and scalar_decompress_track_kernel on the fabricated clip sets of
tests/scalar_cases.py: every plan shape and pool state, every track type, every bit width, raw specials and edge seek times, each launch
compared with the port's decode request by request, bit for bit (NaN where the port gives NaN, whatever the payload), with the bytes a
launch must not write checked against a sentinel."""
from __future__ import annotations

import numpy as np
import pytest

from tests import scalar_cases as sc

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT = 1
SENTINEL = int(np.uint32(sc.SENTINEL).view(np.int32))


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    return dict(torch=torch, ab=ab, port=port, ctx=ab.Context(0))


def _to_device(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).view(np.uint8).reshape(-1)).cuda()


def _expected(oracle, req_clip, req_time, req_policy, row_words, policies=sc.policy_pair):
    """uint32 [requests][row_words]: the oracle's rows, the sentinel wherever a request writes nothing; and where the oracle is NaN.
    `policies` maps a request's policy pair to the (rounding, looping) it seeks with."""
    want = np.full((len(req_clip), row_words), sc.SENTINEL, dtype=np.uint32)
    nan = np.zeros(want.shape, dtype=bool)
    for r, (c, t, p) in enumerate(zip(req_clip.tolist(), req_time.tolist(), req_policy.tolist())):
        if c >= len(oracle.blobs):
            continue
        row = oracle.row(c, np.float32(t), *policies(p)).reshape(-1)
        want[r, :row.size] = row.view(np.uint32)
        nan[r, :row.size] = np.isnan(row)
    return want, nan


def _check(got, want, nan, what):
    ok = np.where(nan, np.isnan(got.view(np.float32)), got == want)
    if not ok.all():
        r, lane = np.argwhere(~ok)[0]
        raise AssertionError(f"{what}: request {r} lane {lane}: got {got[r, lane]:#010x}, want {want[r, lane]:#010x} "
                             f"({int((~ok.all(axis=1)).sum())} requests differ)")


def _launch(gpu, call, num_rows, row_bytes, offset):
    """Runs call(d_out) on a sentinel filled allocation with d_out `offset` bytes in; returns uint32 [num_rows][row_bytes / 4] and checks
    the bytes around the rows kept the sentinel."""
    torch = gpu["torch"]
    words = num_rows * row_bytes // 4
    buffer = torch.full((offset // 4 + words + 4,), SENTINEL, dtype=torch.int32, device="cuda")
    call(buffer.data_ptr() + offset)
    torch.cuda.synchronize()
    host = buffer.cpu().numpy().view(np.uint32)
    assert (host[:offset // 4] == sc.SENTINEL).all() and (host[offset // 4 + words:] == sc.SENTINEL).all(), "a write outside the rows"
    return host[offset // 4:offset // 4 + words].reshape(num_rows, row_bytes // 4)


@pytest.mark.parametrize("name", list(sc.CLIP_SETS))
def test_scalar_tracks_launch(gpu, name):
    """One launch per list with per request policies and a padded stride, its shuffled copy, a second launch of it (every bit again,
    NaN payloads included), and a per track rounding launch; outputs 4, 8, 12 and 0 bytes past an allocation."""
    ab, ctx = gpu["ab"], gpu["ctx"]
    track_type, blobs = sc.clip_set(name)
    clipset = ctx.upload(blobs, check_hash=True)
    nc, max_tracks = clipset.components, clipset.max_tracks
    req_clip, req_time, req_policy = sc.request_list(name)
    count = len(req_clip)
    oracle = sc.Oracle(blobs, track_type)
    stride = max_tracks * nc * 4 + 12

    def run(clip_, time_, policy_, offset):
        d_requests = _to_device(gpu, ab.make_requests(clip_, time_))
        d_policies = _to_device(gpu, policy_.astype(np.uint16))
        options = ab.Options(pose_stride_bytes=stride, d_request_policies=d_policies.data_ptr())
        return _launch(gpu, lambda out: ctx.scalar_decompress_tracks(clipset, d_requests, count, options, out), count, stride, offset)

    want, nan = _expected(oracle, req_clip, req_time, req_policy, stride // 4)
    first = run(req_clip, req_time, req_policy, 4)
    _check(first, want, nan, f"{name}: list")
    perm = np.random.default_rng(1).permutation(count)
    _check(run(req_clip[perm], req_time[perm], req_policy[perm], 8), want[perm], nan[perm], f"{name}: shuffled list")
    again = run(req_clip, req_time, req_policy, 12)
    assert np.array_equal(again, first), f"{name}: a second launch of the list differs"

    # per track rounding: the batch seeks with the per_track policy, each track rounds its own way
    policies = sc.track_policies(max_tracks)
    d_track_policies = _to_device(gpu, policies)
    per_track = sc.Oracle(blobs, track_type, per_track_policies=policies)
    want, nan = _expected(per_track, req_clip, req_time, np.zeros(count, dtype=np.int64), max_tracks * nc,
                          policies=lambda p: (sc.port.ROUND_PER_TRACK, sc.port.LOOP_AS_COMPRESSED))
    d_requests = _to_device(gpu, ab.make_requests(req_clip, req_time))
    options = ab.Options(rounding_policy=ab.ROUND_PER_TRACK, per_track_rounding=1, d_per_track_rounding=d_track_policies.data_ptr())
    got = _launch(gpu, lambda out: ctx.scalar_decompress_tracks(clipset, d_requests, count, options, out), count, max_tracks * nc * 4, 0)
    _check(got, want, nan, f"{name}: per track rounding")
    clipset.release()


@pytest.mark.parametrize("name", list(sc.CLIP_SETS))
def test_scalar_decompress_track(gpu, name):
    """One track per request: every track of every clip up to 1000 tracks (every 37th of wider ones) and the last, at a few times and
    policies; track indices at or past a clip's track count and invalid clips leave the sentinel."""
    ab, ctx, port = gpu["ab"], gpu["ctx"], gpu["port"]
    track_type, blobs = sc.clip_set(name)
    clipset = ctx.upload(blobs, check_hash=True)
    nc = clipset.components
    rng = np.random.default_rng(3)
    settings = port.SettingsBuilder()
    rows = []       # clip, time, policy pair, track
    for c, blob in enumerate(blobs):
        n = port.num_tracks_of(blob)
        tracks = list(range(n)) if n <= 1000 else list(range(0, n, 37)) + [n - 1]
        times = sc.vocabulary_times(blob)
        for t in times[rng.integers(0, len(times), 3)].tolist():
            p = sc.pair(int(rng.integers(0, 4)), int(rng.integers(0, 3)))
            rows += [(c, t, p, k) for k in tracks + [n, n + 1, clipset.max_tracks, 0xFFFFFFFF]]
    rows += [(len(blobs) + 1, 0.25, 0, 0), (0xFFFFFFFF, 0.5, 0, 1)]
    req_clip = np.array([r[0] for r in rows], dtype=np.uint32)
    req_time = np.array([r[1] for r in rows], dtype=np.float32)
    req_policy = np.array([r[2] for r in rows], dtype=np.uint16)
    req_track = np.array([r[3] for r in rows], dtype=np.uint32)
    want = np.full((len(rows), nc), sc.SENTINEL, dtype=np.uint32)
    nan = np.zeros(want.shape, dtype=bool)
    cache = {}
    for i, (c, t, p, k) in enumerate(rows):
        if c >= len(blobs) or k >= port.num_tracks_of(blobs[c]):
            continue
        key = (c, t, p, k)
        if key not in cache:
            cache[key] = port.scalar_decompress(blobs[c], settings, t, *sc.policy_pair(p), track=k)[k, :nc]
        want[i] = cache[key].view(np.uint32)
        nan[i] = np.isnan(cache[key])
    d_requests = _to_device(gpu, ab.make_requests(req_clip, req_time))
    d_tracks = _to_device(gpu, req_track)
    d_policies = _to_device(gpu, req_policy)
    options = ab.Options(d_request_policies=d_policies.data_ptr())
    got = _launch(gpu, lambda out: ctx.scalar_decompress_track(clipset, d_requests, d_tracks, len(rows), options, out), len(rows), nc * 4, 4)
    _check(got, want, nan, f"{name}: decompress_track")
    clipset.release()


def test_host_path_chunks_equal_one_launch(gpu):
    """decompress_tracks_host over 65,541 requests (eight chunks) of a ragged clip set with a padded stride and per request policies:
    the same bytes as one device launch into a zeroed buffer."""
    ab, ctx, torch = gpu["ab"], gpu["ctx"], gpu["torch"]
    track_type, blobs = sc.clip_set("float1_r32")
    clipset = ctx.upload(blobs, check_hash=True)
    assert clipset.min_tracks != clipset.max_tracks
    req_clip, req_time, req_policy = (np.resize(x, 65541) for x in sc.request_list("float1_r32"))
    stride = clipset.max_tracks * 4 + 8
    d_policies = _to_device(gpu, req_policy.astype(np.uint16))
    options = ab.Options(pose_stride_bytes=stride, d_request_policies=d_policies.data_ptr())
    requests = ab.make_requests(req_clip, req_time)
    host = np.full(len(requests) * stride // 4, sc.SENTINEL, dtype=np.uint32)
    ctx.decompress_tracks_host(clipset, requests, options, host)
    d_out = torch.zeros(len(requests) * stride // 4, dtype=torch.int32, device="cuda")
    ctx.scalar_decompress_tracks(clipset, _to_device(gpu, requests), len(requests), options, d_out)
    torch.cuda.synchronize()
    device = d_out.cpu().numpy().view(np.uint32)
    same = host == device
    assert same.all(), f"host path differs from one launch at request {int(np.argmin(same)) * 4 // stride}"
    clipset.release()


def test_misaligned_scalar_outputs_are_refused(gpu):
    """A pose stride or output pointer that is not a multiple of 4 would make the kernels' 4 byte stores fault: both entry points and the
    host path refuse it before anything is launched or written."""
    ab, ctx, torch = gpu["ab"], gpu["ctx"], gpu["torch"]
    track_type, blobs = sc.clip_set("float2_r32")
    clipset = ctx.upload(blobs, check_hash=True)
    row = clipset.max_tracks * clipset.components * 4
    count = 40
    requests = ab.make_requests(np.arange(count) % len(blobs), np.linspace(0.0, 1.0, count))
    d_requests = _to_device(gpu, requests)
    d_tracks = _to_device(gpu, np.zeros(count, dtype=np.uint32))
    buffer = torch.full((count * (row + 16) // 4 + 16,), SENTINEL, dtype=torch.int32, device="cuda")
    base = buffer.data_ptr()
    cases = [
        ("tracks, stride + 2", lambda: ctx.scalar_decompress_tracks(clipset, d_requests, count, ab.Options(pose_stride_bytes=row + 2), base)),
        ("tracks, stride + 6", lambda: ctx.scalar_decompress_tracks(clipset, d_requests, count, ab.Options(pose_stride_bytes=row + 6), base)),
        ("tracks, output + 2", lambda: ctx.scalar_decompress_tracks(clipset, d_requests, count, ab.Options(), base + 2)),
        ("tracks, output + 1, stride + 1", lambda: ctx.scalar_decompress_tracks(clipset, d_requests, count, ab.Options(pose_stride_bytes=row + 1), base + 1)),
        ("track, output + 2", lambda: ctx.scalar_decompress_track(clipset, d_requests, d_tracks, count, ab.Options(), base + 2)),
        ("track, output + 3", lambda: ctx.scalar_decompress_track(clipset, d_requests, d_tracks, count, ab.Options(), base + 3)),
    ]
    for what, call in cases:
        launches = ctx.launch_count
        with pytest.raises(ab.AclB200Error) as error:
            call()
        torch.cuda.synchronize()
        assert error.value.status == ERR_INVALID_ARGUMENT, what
        assert ctx.launch_count == launches, what
        assert (buffer.cpu().numpy() == SENTINEL).all(), what
    host = np.full(count * (row + 2) // 4 + 4, sc.SENTINEL, dtype=np.uint32)
    launches = ctx.launch_count
    with pytest.raises(ab.AclB200Error) as error:
        ctx.decompress_tracks_host(clipset, requests, ab.Options(pose_stride_bytes=row + 2), host)
    assert error.value.status == ERR_INVALID_ARGUMENT and ctx.launch_count == launches
    assert (host == sc.SENTINEL).all()
    # a stride and an output that are multiples of 4 but not of 16 decode
    got = _launch(gpu, lambda out: ctx.scalar_decompress_tracks(clipset, d_requests, count, ab.Options(pose_stride_bytes=row + 4), out),
                  count, row + 4, 4)
    want, nan = _expected(sc.Oracle(blobs, track_type), requests["clip"], requests["sample_time"],
                          np.full(count, sc.pair(0, 2)), (row + 4) // 4)
    _check(got, want, nan, "stride + 4, output + 4")
    clipset.release()
