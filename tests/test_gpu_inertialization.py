"""aclb200_begin_inertialization and aclb200_inertialize_poses against the C oracle (oracle/inertialization_oracle.c, pinned to the
reference's rtm by tests/test_inertialization_oracle.py): bit for bit (a NaN matches any NaN), on fabricated transitions, on poses the
decode wrote, at every decay edge, with record slots, padded strides, records that are missing or out of range, in place, on two streams
and at the C2 launch size; and every refusal of the C ABI."""
import numpy as np
import pytest

from oracle import inertialization as oracle
from tests import clips
from tests import inertialization_cases as cases

pytestmark = pytest.mark.gpu
SENTINEL = np.uint32(0x7FBADBAD)
NO_INERTIALIZATION = 0xFFFFFFFF


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    return dict(torch=torch, ab=ab, ctx=ab.Context(0))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8).copy()).cuda()


def _host(tensor, dtype=np.float32):
    return tensor.cpu().numpy().view(dtype)


def _same(got, want) -> bool:
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    both_nan = np.isnan(got) & np.isnan(want)
    return got.shape == want.shape and bool(np.all((got.view(np.uint32) == want.view(np.uint32)) | both_nan))


def _padded(poses: np.ndarray, stride_floats: int) -> np.ndarray:
    """[n][tracks][12] poses at stride_floats floats apart, the padding holding the sentinel"""
    n = poses.shape[0]
    out = np.full((n, stride_floats), SENTINEL, np.uint32).view(np.float32)
    out[:, : poses.shape[1] * 12] = poses.reshape(n, -1)
    return out


def _capture(gpu, src, src_prev, dst, dst_prev, slots=None, num_records=None, pose_stride=0, record_stride_floats=None):
    n, tracks = src.shape[0], src.shape[1]
    stride_floats = pose_stride // 4 if pose_stride else tracks * 12
    record_floats = record_stride_floats or tracks * 16
    records = _dev(gpu, np.full(((num_records or n) * record_floats,), SENTINEL, np.uint32))
    buffers = [_dev(gpu, _padded(p, stride_floats)) for p in (src, src_prev, dst, dst_prev)]
    d_slots = None if slots is None else _dev(gpu, np.asarray(slots, np.uint32))
    gpu["ctx"].begin_inertialization(*buffers, n, tracks, cases.INV_DT, records, d_record_slots=d_slots, pose_stride_bytes=pose_stride,
                                     record_stride_bytes=0 if record_stride_floats is None else record_stride_floats * 4)
    gpu["torch"].cuda.synchronize()
    return records, _host(records).reshape(-1, record_floats)


def test_capture_equals_the_oracle_with_slots_and_padded_strides(gpu):
    src, src_prev, dst, dst_prev = cases.transitions()
    n, tracks = src.shape[0], src.shape[1]
    want = np.stack([oracle.begin_inertialization(src[j], src_prev[j], dst[j], dst_prev[j], cases.INV_DT) for j in range(n)])
    # default strides, slot j
    _, got = _capture(gpu, src, src_prev, dst, dst_prev)
    assert _same(got.reshape(want.shape), want)
    # slots in a shuffled order into a larger record array, padded pose and record strides: slots not named keep the sentinel
    slots = np.random.default_rng(2).permutation(2 * n)[:n]
    record_floats = tracks * 16 + 8
    _, got = _capture(gpu, src, src_prev, dst, dst_prev, slots=slots, num_records=2 * n, pose_stride=(tracks * 12 + 4) * 4,
                      record_stride_floats=record_floats)
    for j in range(n):
        assert _same(got[slots[j], : tracks * 16].reshape(tracks, 16), want[j]), j
        assert (got[slots[j], tracks * 16:].view(np.uint32) == SENTINEL).all()
    untouched = np.setdiff1d(np.arange(2 * n), slots)
    assert (got[untouched].view(np.uint32) == SENTINEL).all()


def _apply_case(gpu, poses, records, inertializations, num_records, in_place=False, pose_stride_floats=None, stream=None):
    torch = gpu["torch"]
    n, tracks = poses.shape[0], poses.shape[1]
    stride = pose_stride_floats or tracks * 12
    d_poses = _dev(gpu, _padded(poses, stride))
    d_out = d_poses if in_place else _dev(gpu, np.full((n * stride,), SENTINEL, np.uint32))
    d_inert = _dev(gpu, inertializations)
    gpu["ctx"].inertialize_poses(d_poses, d_out, n, tracks, d_inert, records, num_records, pose_stride_bytes=stride * 4 if pose_stride_floats else 0,
                                 stream=stream)
    torch.cuda.synchronize()
    return _host(d_out).reshape(n, stride)


def _want_apply(poses, record_rows, inertializations, num_records, stride, before):
    """what the apply leaves in each pose's `stride` floats, `before` being what the output buffer held"""
    n, tracks = poses.shape[0], poses.shape[1]
    want = before.copy()
    for p in range(n):
        record, elapsed, halflife = inertializations[p]
        if record == NO_INERTIALIZATION:
            want[p, : tracks * 12] = poses[p].reshape(-1)
        elif record < num_records:
            want[p, : tracks * 12] = oracle.inertialize_pose(poses[p], record_rows[record][: tracks * 16].reshape(tracks, 16), float(elapsed),
                                                             float(halflife)).reshape(-1)
    return want


@pytest.mark.parametrize("in_place", [False, True])
def test_apply_equals_the_oracle_at_every_decay(gpu, in_place):
    """Every (elapsed, halflife) edge of the cases on every transition's record, records named in a shuffled order, with poses that take
    no record (copied) and poses whose record is out of range (not written) mixed in, padded strides"""
    ab = gpu["ab"]
    src, src_prev, dst, dst_prev = cases.transitions()
    n, tracks = src.shape[0], src.shape[1]
    d_records, record_rows = _capture(gpu, src, src_prev, dst, dst_prev)
    rng = np.random.default_rng(4)
    num_poses = len(cases.DECAYS) * n + 6
    poses = cases.poses(rng, num_poses, tracks)
    record_of = rng.integers(0, n, size=num_poses).astype(np.uint32)
    record_of[-6:-3] = ab.NO_INERTIALIZATION
    record_of[-3:] = [n, n + 7, 0xFFFFFFFE]
    decays = np.concatenate([np.repeat(cases.DECAYS, n, axis=0), np.full((6, 2), 0.1, np.float32)])
    inert = ab.make_inertializations(record_of, decays[:, 0], decays[:, 1])
    stride = tracks * 12 + 4
    got = _apply_case(gpu, poses, d_records, inert, n, in_place=in_place, pose_stride_floats=stride)
    before = _padded(poses, stride) if in_place else np.full((num_poses, stride), SENTINEL, np.uint32).view(np.float32)
    with np.errstate(all="ignore"):
        want = _want_apply(poses, record_rows, [tuple(r) for r in inert.tolist()], n, stride, before)
    assert _same(got, want)


def test_decoded_poses(gpu):
    """The displayed and destination poses a decode writes (unnormalised rotations as the decode leaves them): capture from them, decay
    onto the destination, against the oracle"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    names = ["c1_30bones", "mixed_scale", "stripped_loop"]
    blobs = [clips.load_blob(n) for n in names]
    clipset = ctx.upload(blobs, check_hash=True)
    rng = np.random.default_rng(6)
    n = 96
    clip = rng.integers(0, len(blobs), size=(2, n)).astype(np.uint32)
    tracks = clipset.max_tracks
    # one skeleton per launch of the capture: transitions between clips of one bone count (pad with the same clip)
    counts = np.array([int(b[16:20].view(np.uint32)[0]) for b in blobs])
    clip[1] = np.where(counts[clip[1]] == counts[clip[0]], clip[1], clip[0])
    t = rng.uniform(0.0, 2.0, size=(2, n)).astype(np.float32)
    dt = np.float32(1.0 / cases.INV_DT)
    times = [t[0], t[0] - dt, t[1], t[1] - dt]
    poses = []
    for k, tt in enumerate(times):
        out = torch.zeros((n, tracks, 12), dtype=torch.float32, device="cuda")
        ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(clip[k // 2], tt)), n, ab.Options(), out)
        poses.append(out)
    torch.cuda.synchronize()
    for b in sorted(set(counts.tolist())):
        sel = np.nonzero(counts[clip[0]] == b)[0]
        if sel.size == 0:
            continue
        sub = [p.cpu().numpy()[sel][:, :b] for p in poses]
        d_records, rows = _capture(gpu, *sub)
        for j in range(sel.size):
            want = oracle.begin_inertialization(sub[0][j], sub[1][j], sub[2][j], sub[3][j], cases.INV_DT)
            assert _same(rows[j].reshape(b, 16), want), (b, j)
        inert = ab.make_inertializations(np.arange(sel.size), rng.uniform(0, 0.5, sel.size), 0.15)
        got = _apply_case(gpu, sub[2], d_records, inert, sel.size)
        for j in range(sel.size):
            want = oracle.inertialize_pose(sub[2][j], rows[j].reshape(b, 16), float(inert["elapsed"][j]), 0.15)
            assert _same(got[j].reshape(b, 12), want), (b, j)


def test_two_streams(gpu):
    """Two halves of the poses decayed on two streams at once: each half as one launch on the default stream writes it"""
    torch, ab = gpu["torch"], gpu["ab"]
    src, src_prev, dst, dst_prev = cases.transitions()
    n, tracks = src.shape[0], src.shape[1]
    d_records, _ = _capture(gpu, src, src_prev, dst, dst_prev)
    rng = np.random.default_rng(8)
    m = 20000
    poses = cases.poses(rng, m, tracks)
    inert = ab.make_inertializations(rng.integers(0, n, size=m), rng.uniform(0, 0.4, m), 0.2)
    whole = _apply_case(gpu, poses, d_records, inert, n)
    d_poses, d_out, d_inert = _dev(gpu, poses), _dev(gpu, np.zeros(poses.size, np.float32)), _dev(gpu, inert)
    half = m // 2
    pose_bytes, inert_bytes = tracks * 48, ab.INERTIALIZATION_DTYPE.itemsize
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for k, s in enumerate(streams):
        with torch.cuda.stream(s):
            gpu["ctx"].inertialize_poses(d_poses[k * half * pose_bytes:], d_out[k * half * pose_bytes:], half, tracks,
                                         d_inert[k * half * inert_bytes:], d_records, n, stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(_host(d_out).view(np.uint32), whole.reshape(-1).view(np.uint32))


def test_c2_launch_size(gpu):
    """600k poses of 100 bones in one launch (the C2 shape; 2.9 GB per pose buffer): sampled poses, the first and the last, against the
    oracle, and poses without a record copied byte for byte"""
    torch, ab = gpu["torch"], gpu["ab"]
    rng = np.random.default_rng(9)
    tracks, n_records, m = 100, 64, 600_000
    small = [cases.poses(rng, n_records, tracks) for _ in range(4)]
    d_records, rows = _capture(gpu, *small)
    base = cases.poses(rng, 997, tracks)
    d_base = _dev(gpu, base)
    reps = -(-m // 997)
    d_poses = d_base.view(torch.float32).reshape(997, tracks * 12).repeat(reps, 1)[:m].contiguous()
    record_of = rng.integers(0, n_records, size=m).astype(np.uint32)
    record_of[::5] = ab.NO_INERTIALIZATION
    inert = ab.make_inertializations(record_of, rng.uniform(0, 0.5, m), 0.2)
    d_out = torch.empty_like(d_poses)
    gpu["ctx"].inertialize_poses(d_poses, d_out, m, tracks, _dev(gpu, inert), d_records, n_records)
    torch.cuda.synchronize()
    sample = np.concatenate([[0, 5, m - 1], rng.integers(0, m, size=200)])
    got = d_out[torch.from_numpy(sample).cuda()].cpu().numpy()
    for i, p in enumerate(sample):
        pose = base[p % 997]
        if record_of[p] == ab.NO_INERTIALIZATION:
            want = pose
        else:
            want = oracle.inertialize_pose(pose, rows[record_of[p]].reshape(tracks, 16), float(inert["elapsed"][p]), 0.2)
        assert _same(got[i].reshape(tracks, 12), want), p
    del d_poses, d_out


def test_refusals(gpu):
    """Each refusal launches nothing (the records and poses keep their bytes) and raises"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    tracks, n = 5, 3
    poses = _dev(gpu, cases.poses(np.random.default_rng(1), n, tracks))
    records = _dev(gpu, np.full(n * tracks * 16, SENTINEL, np.uint32))
    inert = _dev(gpu, ab.make_inertializations(np.arange(n), 0.1, 0.2))
    launches = ctx.launch_count
    bad_capture = [
        dict(inv_dt=0.0), dict(inv_dt=float("inf")), dict(inv_dt=float("nan")),
        dict(d_records=records.data_ptr() + 4), dict(record_stride_bytes=tracks * 64 - 16), dict(record_stride_bytes=tracks * 64 + 8),
        dict(pose_stride_bytes=tracks * 48 - 16), dict(pose_stride_bytes=tracks * 48 + 4), dict(d_src=poses.data_ptr() + 8),
        dict(d_record_slots=_dev(gpu, np.zeros(n + 1, np.uint32)).data_ptr() + 2), dict(d_dst=0), dict(d_records=0),
    ]
    for bad in bad_capture:
        args = dict(d_src=poses, d_src_prev=poses, d_dst=poses, d_dst_prev=poses, num_transitions=n, num_tracks=tracks, inv_dt=30.0,
                    d_records=records)
        args.update(bad)
        with pytest.raises(ab.AclB200Error):
            ctx.begin_inertialization(**args)
    bad_apply = [
        dict(num_records=0xFFFFFFFF), dict(num_records=1 << 40), dict(d_records=records.data_ptr() + 4),
        dict(record_stride_bytes=tracks * 64 - 16), dict(record_stride_bytes=tracks * 64 + 4), dict(d_records=0),
        dict(d_inertializations=inert.data_ptr() + 2), dict(d_inertializations=0), dict(d_out=0), dict(d_poses=poses.data_ptr() + 8),
        dict(pose_stride_bytes=tracks * 48 + 8),
    ]
    for bad in bad_apply:
        args = dict(d_poses=poses, d_out=poses, num_poses=n, num_tracks=tracks, d_inertializations=inert, d_records=records, num_records=n)
        args.update(bad)
        with pytest.raises(ab.AclB200Error):
            ctx.inertialize_poses(**args)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches
    assert (_host(records, np.uint32) == SENTINEL).all()
    # nothing to do is not an error: zero transitions, zero poses, zero records with every pose NO_INERTIALIZATION
    ctx.begin_inertialization(0, 0, 0, 0, 0, tracks, 30.0, 0)
    ctx.inertialize_poses(0, 0, 0, tracks, 0, 0, 0)
    ctx.inertialize_poses(poses, poses, n, tracks, _dev(gpu, ab.make_inertializations(np.full(n, ab.NO_INERTIALIZATION), 0.0, 0.2)), 0, 0)


# ---- the inertialized decode (aclb200_decompress_tracks_inertialized and _skinning): against the unfused route and the plain decodes ----
@pytest.fixture(scope="module")
def c2(gpu):
    """The C2 bench clips (10k clips of 100 bones) and a launch of 600k inertialized requests over them: records from fabricated
    transitions, 25 % of the requests without a record, a few with an out of range record or an invalid clip."""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    bones, m, n_records = w["num_tracks"], 600_000, 64
    rng = np.random.default_rng(31)
    d_records, _ = _capture(gpu, *[cases.poses(rng, n_records, bones) for _ in range(4)])
    clip, time = w["req_clip"][:m].copy(), w["req_time"][:m].copy()
    record = rng.integers(0, n_records, size=m).astype(np.uint32)
    record[rng.random(m) < 0.25] = ab.NO_INERTIALIZATION
    record[rng.integers(0, m, size=50)] = n_records + rng.integers(0, 1000, size=50).astype(np.uint32)
    bad_clip = rng.integers(0, m, size=50)
    clip[bad_clip] = 1 << 30
    elapsed = rng.uniform(0.0, 0.6, m).astype(np.float32)
    halflife = rng.uniform(0.05, 0.3, m).astype(np.float32)
    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, bones) - 1) // 2]).astype(np.uint32)
    inverse_bind = rng.normal(size=(bones, 12)).astype(np.float32)
    data = dict(w=w, clipset=clipset, bones=bones, m=m, n_records=n_records, d_records=d_records, clip=clip, time=time, record=record,
                elapsed=elapsed, halflife=halflife, d_parents=torch.from_numpy(parents).cuda(),
                d_inverse_bind=torch.from_numpy(inverse_bind).cuda(),
                d_requests=_dev(gpu, ab.make_inertialized_requests(clip, time, record, elapsed, halflife)),
                d_plain_requests=_dev(gpu, ab.make_requests(clip, time)),
                d_inertializations=_dev(gpu, ab.make_inertializations(record, elapsed, halflife)),
                unwritten=torch.from_numpy(np.union1d(bad_clip, np.nonzero((record != ab.NO_INERTIALIZATION) & (record >= n_records))[0])).cuda())
    yield data
    clipset.release()


def _filled(torch, like, stride_floats=None):
    out = torch.empty(like if stride_floats is None else (like[0], stride_floats), dtype=torch.float32, device="cuda")
    out.view(torch.int32).fill_(int(SENTINEL))
    return out


def _unfused_local(gpu, c2):
    """decompress_tracks, then inertialize_poses; the requests the fused decode does not write keep the sentinel"""
    torch, ctx = gpu["torch"], gpu["ctx"]
    m, bones = c2["m"], c2["bones"]
    d_plain = _filled(torch, (m, bones * 12))
    ctx.decompress_tracks(c2["clipset"], c2["d_plain_requests"], m, gpu["ab"].Options(), d_plain)
    d_unfused = _filled(torch, (m, bones * 12))
    ctx.inertialize_poses(d_plain, d_unfused, m, bones, c2["d_inertializations"], c2["d_records"], c2["n_records"])
    d_unfused[c2["unwritten"]] = _filled(torch, (1, bones * 12))
    return d_unfused


def _equal(torch, a, b) -> bool:
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def test_fused_local_equals_the_unfused_route(gpu, c2):
    """600k requests: local QVV48 rows byte for byte those of decompress_tracks + inertialize_poses; with a padded pose stride the padding
    is not written; QVV40 rows are the QVV48 rows without their w lanes"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    m, bones = c2["m"], c2["bones"]
    want = _unfused_local(gpu, c2)
    d_fused = _filled(torch, (m, bones * 12))
    ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(), d_fused, c2["d_records"], c2["n_records"])
    torch.cuda.synchronize()
    assert _equal(torch, d_fused, want)
    stride = bones * 12 + 4
    d_padded = _filled(torch, (m, stride))
    ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(pose_stride_bytes=stride * 4), d_padded, c2["d_records"],
                                       c2["n_records"])
    torch.cuda.synchronize()
    assert _equal(torch, d_padded[:, : bones * 12], want)
    assert bool((d_padded[:, bones * 12:].view(torch.int32) == int(SENTINEL)).all())
    d_qvv40 = _filled(torch, (m, bones * 10))
    ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(output_layout=ab.LAYOUT_QVV40), d_qvv40, c2["d_records"],
                                       c2["n_records"])
    torch.cuda.synchronize()
    rows48 = want.view(m, bones, 12)
    want40 = torch.cat([rows48[:, :, 0:7], rows48[:, :, 8:11]], dim=2).reshape(m, bones * 10)
    assert _equal(torch, d_qvv40, want40)


def test_fused_object_and_skinning_equal_the_unfused_route(gpu, c2):
    """With parents: qvvf object rows are those of decompress_tracks + inertialize_poses + local_to_object_space, skinning rows those of
    ... + local_to_skinning; matrix rows of requests without a record are those of decompress_tracks_object_space"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    m, bones = c2["m"], c2["bones"]
    local = _unfused_local(gpu, c2)
    written = torch.ones(m, dtype=torch.bool, device="cuda")
    written[c2["unwritten"]] = False
    for route in ("qvvf", "skinning"):
        want = _filled(torch, (m, bones * 12))
        if route == "qvvf":
            ctx.local_to_object_space(local, want, m, bones, c2["d_parents"])
        else:
            ctx.local_to_skinning(local, want, m, bones, c2["d_parents"], c2["d_inverse_bind"])
        want[~written] = _filled(torch, (1, bones * 12))
        got = _filled(torch, (m, bones * 12))
        if route == "qvvf":
            ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(), got, c2["d_records"], c2["n_records"],
                                               d_parent_indices=c2["d_parents"], kind=ab.OBJECT_QVVF)
        else:
            ctx.decompress_tracks_inertialized_skinning(c2["clipset"], c2["d_requests"], m, ab.Options(), c2["d_parents"], c2["d_inverse_bind"],
                                                        got, c2["d_records"], c2["n_records"])
        torch.cuda.synchronize()
        assert _equal(torch, got, want), route
    none = torch.from_numpy(np.nonzero(c2["record"] == ab.NO_INERTIALIZATION)[0]).cuda()
    got = _filled(torch, (m, bones * 12))
    ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(), got, c2["d_records"], c2["n_records"],
                                       d_parent_indices=c2["d_parents"], kind=ab.OBJECT_MATRIX3X4F)
    want = _filled(torch, (m, bones * 12))
    ctx.decompress_tracks_object_space(c2["clipset"], c2["d_plain_requests"], m, ab.Options(), c2["d_parents"], ab.OBJECT_MATRIX3X4F, want)
    torch.cuda.synchronize()
    assert _equal(torch, got[none], want[none])


def test_no_inertialization_requests_are_the_plain_decodes(gpu, c2):
    """Every request without a record: local, object (qvvf and matrix) and skinning rows byte for byte those of decompress_tracks,
    decompress_tracks_object_space and decompress_tracks_skinning"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    m, bones, cs = c2["m"], c2["bones"], c2["clipset"]
    ok = c2["clip"] < (1 << 30)
    d_requests = _dev(gpu, ab.make_inertialized_requests(c2["clip"][ok], c2["time"][ok], ab.NO_INERTIALIZATION, 0.0, 0.2))
    d_plain = _dev(gpu, ab.make_requests(c2["clip"][ok], c2["time"][ok]))
    n = int(ok.sum())
    routes = {
        "local": (lambda out: ctx.decompress_tracks_inertialized(cs, d_requests, n, ab.Options(), out, None, 0),
                  lambda out: ctx.decompress_tracks(cs, d_plain, n, ab.Options(), out)),
        "qvvf": (lambda out: ctx.decompress_tracks_inertialized(cs, d_requests, n, ab.Options(), out, None, 0, d_parent_indices=c2["d_parents"],
                                                               kind=ab.OBJECT_QVVF),
                 lambda out: ctx.decompress_tracks_object_space(cs, d_plain, n, ab.Options(), c2["d_parents"], ab.OBJECT_QVVF, out)),
        "matrix": (lambda out: ctx.decompress_tracks_inertialized(cs, d_requests, n, ab.Options(), out, None, 0, d_parent_indices=c2["d_parents"],
                                                                 kind=ab.OBJECT_MATRIX3X4F),
                   lambda out: ctx.decompress_tracks_object_space(cs, d_plain, n, ab.Options(), c2["d_parents"], ab.OBJECT_MATRIX3X4F, out)),
        "skinning": (lambda out: ctx.decompress_tracks_inertialized_skinning(cs, d_requests, n, ab.Options(), c2["d_parents"],
                                                                             c2["d_inverse_bind"], out, None, 0),
                     lambda out: ctx.decompress_tracks_skinning(cs, d_plain, n, ab.Options(), c2["d_parents"], c2["d_inverse_bind"], out)),
    }
    for name, (fused, plain) in routes.items():
        got, want = _filled(torch, (n, bones * 12)), _filled(torch, (n, bones * 12))
        fused(got)
        plain(want)
        torch.cuda.synchronize()
        assert _equal(torch, got, want), name


def test_fused_on_two_streams(gpu, c2):
    """The launch split in two halves on two streams writes what the whole launch writes"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    m, bones = c2["m"], c2["bones"]
    whole = _filled(torch, (m, bones * 12))
    ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"], m, ab.Options(), whole, c2["d_records"], c2["n_records"])
    halves = _filled(torch, (m, bones * 12))
    half = m // 2
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for k, s in enumerate(streams):
        with torch.cuda.stream(s):
            ctx.decompress_tracks_inertialized(c2["clipset"], c2["d_requests"][k * half * 20:], half, ab.Options(), halves[k * half:],
                                               c2["d_records"], c2["n_records"], stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert _equal(torch, halves, whole)


def test_fused_refusals(gpu, c2):
    """Each refusal raises and launches nothing"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    bones, cs = c2["bones"], c2["clipset"]
    out = _filled(torch, (4, bones * 12))
    launches = ctx.launch_count
    records = c2["d_records"]
    bad = [
        dict(num_records=0xFFFFFFFF), dict(d_records=records.data_ptr() + 4), dict(d_records=0), dict(record_stride_bytes=bones * 64 - 16),
        dict(record_stride_bytes=bones * 64 + 8), dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40), d_parent_indices=c2["d_parents"]), dict(d_parent_indices=c2["d_parents"], kind=7),
        dict(d_requests=0),
    ]
    for b in bad:
        args = dict(clipset=cs, d_requests=c2["d_requests"], num_requests=4, options=ab.Options(), d_out=out, d_records=records,
                    num_records=c2["n_records"])
        args.update(b)
        with pytest.raises(ab.AclB200Error):
            ctx.decompress_tracks_inertialized(**args)
    with pytest.raises(ab.AclB200Error):
        ctx.decompress_tracks_inertialized_skinning(cs, c2["d_requests"], 4, ab.Options(), c2["d_parents"], None, out, records, c2["n_records"])
    torch.cuda.synchronize()
    assert ctx.launch_count == launches
    assert bool((out.view(torch.int32) == int(SENTINEL)).all())
