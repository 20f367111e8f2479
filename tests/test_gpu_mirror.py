"""aclb200_mirror_poses and aclb200_decompress_tracks_mirrored / _skinning, all bytes compared: the fused decode against the C oracle
(oracle/mirror_oracle.c, pinned to the reference's rtm by tests/test_mirror_oracle.py) applied to the library's own decompress_tracks rows,
then the library's walk and skinning; unmirrored requests against the plain decodes; flags, skeleton offsets, rows left unwritten;
mirror_poses in place and out of place on decodes, feature rows and root motion rows; and every refusal of the C ABI."""
import numpy as np
import pytest

from oracle import mirror as oracle
from oracle import object_space
from tests import clips
from tests import mirror_cases as cases

pytestmark = pytest.mark.gpu
SENTINEL = np.uint32(0x7FBADBAD)
NUM_REQUESTS = 96


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    return dict(torch=torch, ab=ab, ctx=ab.Context(0))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8).copy()).cuda()


def _host(tensor, dtype=np.float32):
    return tensor.cpu().numpy().view(dtype)


def _filled(gpu, floats):
    return _dev(gpu, np.full(floats, SENTINEL, np.uint32))


def _same(got, want) -> bool:
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    both_nan = np.isnan(got) & np.isnan(want)
    return got.shape == want.shape and bool(np.all((got.view(np.uint32) == want.view(np.uint32)) | both_nan))


def _tree(n):
    return np.concatenate([[0xFFFFFFFF], (np.arange(1, n) - 1) // 2]).astype(np.uint32)


def _requests(n_clips, seed):
    """times over the clip, flags 0 and 1 mixed, a few 2 and 7 (not written) and invalid clips"""
    rng = np.random.default_rng(seed)
    clip = rng.integers(0, n_clips, NUM_REQUESTS).astype(np.uint32)
    time = rng.uniform(-0.1, 2.0, NUM_REQUESTS).astype(np.float32)
    flag = rng.integers(0, 2, NUM_REQUESTS).astype(np.uint32)
    flag[[5, 17]] = [2, 7]
    clip[[9, 40]] = [n_clips, 1 << 30]
    return clip, time, flag


def _want_local(plain, clip, flag, table_of, tracks_of, n_clips, axis):
    """[requests][max_tracks][12] what the fused local decode writes: the plain rows, mirrored by the oracle where flag == 1; None where
    nothing is written"""
    want = []
    for r in range(plain.shape[0]):
        if flag[r] > 1 or clip[r] >= n_clips:
            want.append(None)
            continue
        rows = plain[r].copy()
        if flag[r] == 1:
            n = tracks_of[clip[r]]
            rows[:n], _ = oracle.mirror_pose(rows[:n], table_of[clip[r]], axis)
        want.append(rows)
    return want


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("name", cases.NAMED_CLIPS)
def test_named_clip_every_route(gpu, name, axis):
    """QVV48 and QVV40 local rows, qvvf and matrix object rows and skinning rows of mixed mirrored and plain requests"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob(name)], check_hash=True)
    n = clipset.max_tracks
    table = cases.named_table(n)
    parents = _tree(n)
    inverse_bind = np.random.default_rng(3).normal(size=(n, 12)).astype(np.float32)
    d_table, d_parents, d_inverse_bind = _dev(gpu, table), _dev(gpu, parents), _dev(gpu, inverse_bind)
    clip, time, flag = _requests(1, 10 + axis)
    d_req = _dev(gpu, ab.make_mirrored_requests(clip, time, flag))
    ok = (flag <= 1) & (clip < 1)
    d_plain_req = _dev(gpu, ab.make_requests(np.where(ok, clip, 0), time))
    m = NUM_REQUESTS
    d_plain = _filled(gpu, m * n * 12)
    ctx.decompress_tracks(clipset, d_plain_req, m, ab.Options(), d_plain)
    torch.cuda.synchronize()
    plain = _host(d_plain).reshape(m, n, 12)
    want = _want_local(plain, clip, flag, [table], [n], 1, axis)
    sentinel = np.full((n, 12), SENTINEL, np.uint32).view(np.float32)
    want48 = np.stack([w if w is not None else sentinel for w in want])
    d_flags = _dev(gpu, np.array([0xFFFF], np.uint32))

    got = _filled(gpu, m * n * 12)
    ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), got, d_table, axis, d_out_flags=d_flags)
    torch.cuda.synchronize()
    assert _same(_host(got).reshape(m, n, 12), want48)
    assert int(_host(d_flags, np.uint32)[0]) == 0

    got40 = _filled(gpu, m * n * 10)
    ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(output_layout=ab.LAYOUT_QVV40), got40, d_table, axis)
    torch.cuda.synchronize()
    want40 = np.concatenate([want48[:, :, 0:7], want48[:, :, 8:11]], axis=2)
    assert _same(_host(got40).reshape(m, n, 10), want40)

    # the library's walk and skinning of the oracle's local rows
    d_want_local = _dev(gpu, want48)
    d_qvvf, d_skin = _filled(gpu, m * n * 12), _filled(gpu, m * n * 12)
    ctx.local_to_object_space(d_want_local, d_qvvf, m, n, d_parents)
    ctx.local_to_skinning(d_want_local, d_skin, m, n, d_parents, d_inverse_bind)
    torch.cuda.synchronize()
    routes = {"qvvf": _host(d_qvvf).reshape(m, n, 12), "skinning": _host(d_skin).reshape(m, n, 12),
              "matrix": np.stack([object_space.port_local_to_object_space_matrix(w, parents) if w is not None else sentinel for w in want])}
    for route, expected in routes.items():
        out = _filled(gpu, m * n * 12)
        if route == "skinning":
            ctx.decompress_tracks_mirrored_skinning(clipset, d_req, m, ab.Options(), d_parents, d_inverse_bind, out, d_table, axis)
        else:
            kind = ab.OBJECT_QVVF if route == "qvvf" else ab.OBJECT_MATRIX3X4F
            ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), out, d_table, axis, d_parent_indices=d_parents, kind=kind)
        torch.cuda.synchronize()
        got_rows = _host(out).reshape(m, n, 12)
        written = np.array([w is not None for w in want])
        assert _same(got_rows[written], expected[written]), route
        assert (got_rows[~written].view(np.uint32) == SENTINEL).all(), route
    clipset.release()


def test_unmirrored_requests_are_the_plain_decodes(gpu):
    """In a launch mixed with mirrored requests, the requests with mirrored == 0 are byte for byte those of decompress_tracks,
    decompress_tracks_object_space (qvvf and matrix) and decompress_tracks_skinning"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blobs = [clips.load_blob(n) for n in cases.NAMED_CLIPS]
    clipset = ctx.upload(blobs, check_hash=True)
    n = clipset.max_tracks
    rng = np.random.default_rng(5)
    m = 4096
    clip = rng.integers(0, len(blobs), m).astype(np.uint32)
    time = rng.uniform(0, 2, m).astype(np.float32)
    flag = (rng.random(m) < 0.5).astype(np.uint32)
    d_table, d_parents = _dev(gpu, cases.named_table(n)), _dev(gpu, _tree(n))
    d_inverse_bind = _dev(gpu, rng.normal(size=(n, 12)).astype(np.float32))
    d_req, d_plain = _dev(gpu, ab.make_mirrored_requests(clip, time, flag)), _dev(gpu, ab.make_requests(clip, time))
    plain_rows = torch.from_numpy(np.nonzero(flag == 0)[0]).cuda()
    routes = {
        "local": (lambda out: ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), out, d_table, 0),
                  lambda out: ctx.decompress_tracks(clipset, d_plain, m, ab.Options(), out)),
        "qvvf": (lambda out: ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), out, d_table, 1, d_parent_indices=d_parents,
                                                            kind=ab.OBJECT_QVVF),
                 lambda out: ctx.decompress_tracks_object_space(clipset, d_plain, m, ab.Options(), d_parents, ab.OBJECT_QVVF, out)),
        "matrix": (lambda out: ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), out, d_table, 2, d_parent_indices=d_parents,
                                                              kind=ab.OBJECT_MATRIX3X4F),
                   lambda out: ctx.decompress_tracks_object_space(clipset, d_plain, m, ab.Options(), d_parents, ab.OBJECT_MATRIX3X4F, out)),
        "skinning": (lambda out: ctx.decompress_tracks_mirrored_skinning(clipset, d_req, m, ab.Options(), d_parents, d_inverse_bind, out,
                                                                         d_table, 0),
                     lambda out: ctx.decompress_tracks_skinning(clipset, d_plain, m, ab.Options(), d_parents, d_inverse_bind, out)),
    }
    for name, (fused, reference) in routes.items():
        got, want = _filled(gpu, m * n * 12), _filled(gpu, m * n * 12)
        fused(got)
        reference(want)
        torch.cuda.synchronize()
        got, want = got.view(torch.int32).reshape(m, -1), want.view(torch.int32).reshape(m, -1)
        assert torch.equal(got[plain_rows], want[plain_rows]), name
        assert not torch.equal(got, want), name
    clipset.release()


def test_two_skeletons(gpu):
    """Two clips of different bone counts in one clip set, each with its own skeleton and table through d_skeleton_offsets"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    names = ["c1_30bones", "mixed_scale"]
    clipset = ctx.upload([clips.load_blob(nm) for nm in names], check_hash=True)
    counts = [30, 57]
    n = clipset.max_tracks
    offsets = np.array([0, counts[0]], np.uint32)
    tables = [cases.named_table(c) for c in counts]
    parents = [_tree(c) for c in counts]
    d_table, d_parents = _dev(gpu, np.concatenate(tables)), _dev(gpu, np.concatenate(parents))
    d_offsets = _dev(gpu, offsets)
    clip, time, flag = _requests(2, 30)
    m = NUM_REQUESTS
    d_req = _dev(gpu, ab.make_mirrored_requests(clip, time, flag))
    ok = (flag <= 1) & (clip < 2)
    d_plain = _filled(gpu, m * n * 12)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(np.where(ok, clip, 0), time)), m, ab.Options(), d_plain)
    got_local, got_obj = _filled(gpu, m * n * 12), _filled(gpu, m * n * 12)
    ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), got_local, d_table, 0, d_skeleton_offsets=d_offsets)
    ctx.decompress_tracks_mirrored(clipset, d_req, m, ab.Options(), got_obj, d_table, 0, d_parent_indices=d_parents, kind=ab.OBJECT_MATRIX3X4F,
                                   d_skeleton_offsets=d_offsets)
    torch.cuda.synchronize()
    plain = _host(d_plain).reshape(m, n, 12)
    want = _want_local(plain, clip, flag, tables, counts, 2, 0)
    got_local, got_obj = _host(got_local).reshape(m, n, 12), _host(got_obj).reshape(m, n, 12)
    for r in range(m):
        if want[r] is None:
            assert (got_local[r].view(np.uint32) == SENTINEL).all() and (got_obj[r].view(np.uint32) == SENTINEL).all(), r
            continue
        c = counts[clip[r]]
        assert _same(got_local[r, :c], want[r][:c]), r
        assert (got_local[r, c:].view(np.uint32) == SENTINEL).all(), r
        assert _same(got_obj[r, :c], object_space.port_local_to_object_space_matrix(want[r][:c], parents[clip[r]])), r
    clipset.release()


def test_non_involutive_table_flags_and_self_partners(gpu):
    """Entries without a partner take their own row and raise ACLB200_ERROR_FLAG_INVALID_MIRROR, in the decode and in mirror_poses; a
    request that is not mirrored raises nothing"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")], check_hash=True)
    n = clipset.max_tracks
    table = cases.named_table(n)
    table["mirror"][3] = 7              # 3 -> 7 while 7 and 6 pair: 3 is its own partner
    table["mirror"][10] = n + 100       # out of range
    d_table = _dev(gpu, table)
    time = np.linspace(0, 1, 32).astype(np.float32)
    d_plain = _filled(gpu, 32 * n * 12)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(np.zeros(32, np.uint32), time)), 32, ab.Options(), d_plain)
    d_flags = _dev(gpu, np.zeros(1, np.uint32))
    for mirrored, want_flag in ((0, 0), (1, ab.ERROR_FLAG_INVALID_MIRROR)):
        got = _filled(gpu, 32 * n * 12)
        ctx.decompress_tracks_mirrored(clipset, _dev(gpu, ab.make_mirrored_requests(0, time, mirrored)), 32, ab.Options(), got, d_table, 1,
                                       d_out_flags=d_flags)
        torch.cuda.synchronize()
        assert int(_host(d_flags, np.uint32)[0]) == want_flag
        plain = _host(d_plain).reshape(32, n, 12)
        for p in range(32):
            want = oracle.mirror_pose(plain[p], table, 1)[0] if mirrored else plain[p]
            assert _same(_host(got).reshape(32, n, 12)[p], want), p
    out = _filled(gpu, 32 * n * 12)
    ctx.mirror_poses(d_plain, out, 32, n, d_table, 1, d_out_flags=d_flags)
    torch.cuda.synchronize()
    assert int(_host(d_flags, np.uint32)[0]) == ab.ERROR_FLAG_INVALID_MIRROR
    clipset.release()


@pytest.mark.parametrize("in_place", [False, True])
def test_mirror_poses_with_flags_and_padded_strides(gpu, in_place):
    """Fabricated poses (special lanes, non-unit rotations) at a padded stride under the fabricated table, every axis: flag 0 copies, 1
    mirrors, 2 and above leave the pose and the padding unwritten; without flags every pose is mirrored"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    table = cases.fabricated_table()
    poses = np.tile(cases.fabricated_poses(), (4, 1, 1))
    p, n = poses.shape[0], poses.shape[1]
    stride = n * 12 + 8
    padded = np.full((p, stride), SENTINEL, np.uint32).view(np.float32)
    padded[:, : n * 12] = poses.reshape(p, -1)
    flag = np.array([0, 1, 2, 1, 0xFFFFFFFF, 1] * 4, np.uint32)
    d_table = _dev(gpu, table)
    for axis in cases.AXES:
        for flags in (flag, None):
            d_poses = _dev(gpu, padded)
            d_out = d_poses if in_place else _filled(gpu, p * stride)
            ctx.mirror_poses(d_poses, d_out, p, n, d_table, axis, d_mirrored=None if flags is None else _dev(gpu, flags),
                             pose_stride_bytes=stride * 4)
            torch.cuda.synchronize()
            got = _host(d_out).reshape(p, stride)
            before = padded if in_place else np.full((p, stride), SENTINEL, np.uint32).view(np.float32)
            want = before.copy()
            with np.errstate(all="ignore"):
                for k in range(p):
                    f = 1 if flags is None else flags[k]
                    if f == 0:
                        want[k, : n * 12] = poses[k].reshape(-1)
                    elif f == 1:
                        want[k, : n * 12] = oracle.mirror_pose(poses[k], table, axis)[0].reshape(-1)
            assert _same(got, want), (axis, flags is None)


def test_mirror_poses_on_feature_and_root_motion_rows(gpu):
    """Rows of extract_pose_features (one pose per (request, offset)) with a mirror_rows_table, and rows of extract_root_motion with the
    one-row table, mirrored by mirror_poses: the oracle's rows"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")], check_hash=True)
    n = clipset.max_tracks
    parents = _tree(n)
    skeleton = cases.named_table(n)
    skeleton["mirror"][[0, 1]] = [0, 1]         # the root and bone 1 on the mirror plane
    bones = [2, 3, 4, 5, 0, 1]
    rows_table = ab.mirror_rows_table(skeleton, bones, 0)
    root_table = ab.mirror_rows_table(skeleton, [0], 0)
    rng = np.random.default_rng(12)
    r = 64
    time = rng.uniform(0, 1.5, r).astype(np.float32)
    offsets = [0.0, 0.2, 0.4]
    d_features = _filled(gpu, r * len(offsets) * len(bones) * 12)
    clamp = ab.Options(looping_policy=ab.LOOP_CLAMP)
    ctx.extract_pose_features(clipset, _dev(gpu, ab.make_feature_requests(0, time)), r, clamp, offsets,
                              _dev(gpu, np.array(bones, np.uint32)), len(bones), _dev(gpu, parents), d_features)
    d_motion = _filled(gpu, r * 12)
    ctx.extract_root_motion(clipset, _dev(gpu, ab.make_root_motion_requests(0, time, time + np.float32(0.1))), r, clamp, d_motion)
    torch.cuda.synchronize()
    for d_rows, table, rows in ((d_features, rows_table, len(bones)), (d_motion, root_table, 1)):
        source = _host(d_rows).reshape(-1, rows, 12).copy()
        num_poses = source.shape[0]
        out = _filled(gpu, source.size)
        ctx.mirror_poses(d_rows, out, num_poses, rows, _dev(gpu, table), ab.MIRROR_Z)
        torch.cuda.synchronize()
        want = np.stack([oracle.mirror_pose(s, table, ab.MIRROR_Z)[0] for s in source])
        assert _same(_host(out).reshape(num_poses, rows, 12), want), rows
    clipset.release()


def test_refusals(gpu):
    """Each refusal raises and launches nothing; nothing to do is not an error"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")], check_hash=True)
    n = clipset.max_tracks
    table = _dev(gpu, cases.named_table(n))
    poses = _filled(gpu, 4 * n * 12)
    flags = _dev(gpu, np.ones(5, np.uint32))
    parents = _dev(gpu, _tree(n))
    req = _dev(gpu, ab.make_mirrored_requests(0, [0.1, 0.2, 0.3, 0.4], 1))
    out = _filled(gpu, 4 * n * 12)
    launches = ctx.launch_count
    bad_mirror = [dict(axis=3), dict(axis=0xFFFFFFFF), dict(d_table=0), dict(d_table=table.data_ptr() + 8), dict(d_poses=0), dict(d_out=0),
                  dict(d_poses=poses.data_ptr() + 4), dict(pose_stride_bytes=n * 48 - 16), dict(pose_stride_bytes=n * 48 + 8),
                  dict(d_mirrored=flags.data_ptr() + 2)]
    for bad in bad_mirror:
        args = dict(d_poses=poses, d_out=poses, num_poses=4, num_rows=n, d_table=table, axis=0)
        args.update(bad)
        with pytest.raises(ab.AclB200Error):
            ctx.mirror_poses(**args)
    bad_decode = [dict(axis=3), dict(d_mirror_table=0), dict(d_mirror_table=table.data_ptr() + 4), dict(d_requests=0), dict(d_out=0),
                  dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)), dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40), d_parent_indices=parents),
                  dict(d_parent_indices=parents, kind=7), dict(d_out=out.data_ptr() + 8)]
    for bad in bad_decode:
        args = dict(clipset=clipset, d_requests=req, num_requests=4, options=ab.Options(), d_out=out, d_mirror_table=table, axis=0)
        args.update(bad)
        with pytest.raises(ab.AclB200Error):
            ctx.decompress_tracks_mirrored(**args)
    for bad in (dict(d_inverse_bind=None), dict(d_parent_indices=None), dict(axis=5), dict(d_mirror_table=None)):
        args = dict(clipset=clipset, d_requests=req, num_requests=4, options=ab.Options(), d_parent_indices=parents,
                    d_inverse_bind=_dev(gpu, np.zeros(n * 12, np.float32)), d_out=out, d_mirror_table=table, axis=0)
        args.update(bad)
        with pytest.raises(ab.AclB200Error):
            ctx.decompress_tracks_mirrored_skinning(**args)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches
    assert (_host(out, np.uint32) == SENTINEL).all() and (_host(poses, np.uint32) == SENTINEL).all()
    ctx.mirror_poses(0, 0, 0, n, 0, 0)
    ctx.mirror_poses(0, 0, 4, 0, 0, 2)
    ctx.decompress_tracks_mirrored(clipset, 0, 0, ab.Options(), 0, 0, 1)
    assert ctx.launch_count == launches
    clipset.release()
