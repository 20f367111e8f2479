"""aclb200_decompress_tracks_blend (decompress from + decompress to + rtm::qvv_lerp in one kernel) and aclb200_blend_poses, against
  * the port's decode of both clips and its qvv_lerp with the IEEE quat_normalize (oracle/acl_oracle.c, oracle/blend_oracle.c, pinned to
    the reference by tests/test_blend_oracle.py): BIT FOR BIT;
  * blend.golden.npz, the reference's own poses: translations and scales bit for bit, rotations within blend_cases.ROTATION_GATE (the
    reference normalises with rsqrtss + Newton-Raphson);
  * the unfused route (two decompress_tracks launches + aclb200_blend_poses) at the C2 launch size: byte for byte.
"""
import numpy as np
import pytest

from oracle import blend, object_space
from tests import blend_cases as cases
from tests import clips
from tests import database_cases as dbcases

pytestmark = pytest.mark.gpu
LANES = clips.DEFINED_LANES
ROOT = 0xFFFFFFFF
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    ctx = ab.Context(0)
    blobs = [cases.load(n) for n in cases.NAMES]
    return dict(torch=torch, ab=ab, port=port, ctx=ctx, blobs=blobs, clipset=ctx.upload(blobs, check_hash=True))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8)).cuda()


def _options(gpu, kind, **kw):
    s = gpu["port"].settings_for_kind(kind).c
    fields = dict(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                  clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                  default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                  constant_defaults=list(s.constant_defaults))
    fields.update(kw)
    return gpu["ab"].Options(**fields)


def tree(n):
    bones = np.arange(n)
    return np.where(bones == 0, ROOT, (bones - 1) // 2).astype(np.uint32)


def ref_tracks(blob):
    return int(blob[16:20].view(np.uint32)[0])


def expected(gpu, from_blob, to_blob, tf, tt, weight, kind, rounding, looping, settings=None):
    port = gpu["port"]
    return cases.port_pose(port, blend, from_blob, to_blob, tf, tt, weight, settings or port.settings_for_kind(kind), rounding, looping,
                           blend.NORMALIZE_IEEE)


def _rows_equal(got, want, layout_40=False):
    """defined lanes bit for bit; QVV48 rows carry 0 in the translation and scale w lanes"""
    if layout_40:
        return clips.bit_equal(got, want[:, LANES])
    return clips.bit_equal(got[:, LANES], want[:, LANES]) and not got[:, [7, 11]].view(np.uint32).any()


def _run(gpu, requests, options, clipset=None, fill=0x7FC00001, width=None, **kw):
    torch, ctx = gpu["torch"], gpu["ctx"]
    clipset = clipset or gpu["clipset"]
    n = len(requests)
    d_out = torch.full((n, width or clipset.max_tracks * 12), fill, dtype=torch.int32, device="cuda")
    ctx.decompress_tracks_blend(clipset, _dev(gpu, requests), n, options, d_out, **kw)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.float32)


def _pair_weights(m):
    return np.resize(cases.WEIGHTS, m).astype(np.float32)


def test_settings_match_the_oracle(gpu):
    """Every golden combo (settings kind, rounding, looping), QVV48 and QVV40, with a weight per pair and with the scalar weight; then per
    request policies in one launch and a variable bind pose that both halves decode with (neither takes the track_writer defaults)."""
    ab, port, torch = gpu["ab"], gpu["port"], gpu["torch"]
    from_blob, to_blob = gpu["blobs"]
    pairs = cases.time_pairs()
    m, n = len(pairs), cases.FROM_SPEC.num_tracks
    weights = _pair_weights(m)
    d_weights = torch.from_numpy(weights).cuda()
    requests = ab.make_blend_requests(np.zeros(m), pairs[:, 0], np.ones(m), pairs[:, 1])
    for kind, rounding, looping in cases.COMBOS:
        for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
            options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping, output_layout=layout, pose_stride_bytes=n * 48)
            for scalar in (None, -0.25):
                got = _run(gpu, requests, options, d_weights=None if scalar is not None else d_weights, weight=scalar or 0.0)
                for i, (tf, tt) in enumerate(pairs):
                    w = scalar if scalar is not None else weights[i]
                    want = expected(gpu, from_blob, to_blob, tf, tt, w, kind, rounding, looping)
                    row = got[i, :n * 12].reshape(n, 12) if layout == ab.LAYOUT_QVV48 else got[i, :n * 10].reshape(n, 10)
                    assert _rows_equal(row, want, layout == ab.LAYOUT_QVV40), (kind, rounding, looping, layout, scalar, i)

    policies = np.resize(np.array([(r, l) for r in range(4) for l in range(3)], np.uint8), (m, 2))
    variable = np.tile(IDENTITY, (n, 1))
    rng = np.random.default_rng(5)
    variable[:, 4:7] = rng.uniform(-2, 2, (n, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (n, 3))
    d_variable = torch.from_numpy(variable).cuda()
    settings = port.settings_for_kind(0, default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable)
    d_policies = _dev(gpu, policies)
    options = _options(gpu, 0, d_request_policies=d_policies.data_ptr(), default_modes=(ab.DEFAULT_VARIABLE,) * 3,
                       d_variable_defaults=d_variable.data_ptr())
    got = _run(gpu, requests, options, d_weights=d_weights)
    for i, (tf, tt) in enumerate(pairs):
        rounding, looping = int(policies[i][0]), int(policies[i][1])
        want = expected(gpu, from_blob, to_blob, tf, tt, weights[i], 0, rounding, looping, settings)
        assert _rows_equal(got[i, :n * 12].reshape(n, 12), want), ("policies + variable", i)


def test_reference_poses(gpu):
    """blend.golden.npz: the reference's decode-and-lerp at every combo and weight: translations and scales bit for bit, rotations within
    the gate."""
    ab = gpu["ab"]
    golden = np.load(clips.golden_path("blend", "golden.npz"))
    pairs = golden["pairs"]
    m, n = len(pairs), cases.FROM_SPEC.num_tracks
    requests = ab.make_blend_requests(np.zeros(m), pairs[:, 0], np.ones(m), pairs[:, 1])
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        for wi, weight in enumerate(golden["weights"]):
            got = _run(gpu, requests, _options(gpu, kind, rounding_policy=rounding, looping_policy=looping), weight=float(weight))
            got = got[:, :n * 12].reshape(m, n, 12)[..., LANES]
            want = golden["poses"][ci, wi]
            assert clips.bit_equal(got[..., 4:], want[..., 4:]), (kind, rounding, looping, float(weight))
            assert float(np.max(np.abs(got[..., 0:4] - want[..., 0:4]))) <= cases.ROTATION_GATE, (kind, rounding, looping, float(weight))


@pytest.mark.parametrize("layout", ["qvv48", "qvv40"])
def test_invalid_pairs_and_untouched_bytes(gpu, layout):
    """A clip set with the two clips and a 30 bone clip: invalid clip indices on either side, track count mismatches, a weight per pair,
    a padded stride and an output 16 (QVV48) or 8 (QVV40) bytes into its allocation: every byte nobody may write keeps its sentinel."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blobs = gpu["blobs"] + [clips.load_blob("c1_30bones")]
    clipset = ctx.upload(blobs, check_hash=True)
    qvv40 = layout == "qvv40"
    bone = 40 if qvv40 else 48
    rng = np.random.default_rng(12)
    m = 400
    from_clip = rng.choice([0, 0, 1, 1, 2, 3, 0xFFFFFFFF], m).astype(np.uint32)
    to_clip = rng.choice([0, 1, 1, 2, 2, 5], m).astype(np.uint32)
    tf = rng.uniform(-0.2, 1.6, m).astype(np.float32)
    tt = rng.uniform(-0.2, 1.2, m).astype(np.float32)
    weights = rng.uniform(-0.5, 1.5, m).astype(np.float32)
    requests = ab.make_blend_requests(from_clip, tf, to_clip, tt)
    stride = clipset.max_tracks * bone + 32
    lead = 8 if qvv40 else 16
    buffer = torch.full((lead + stride * m + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d_flags = torch.full((1,), 0x7F, dtype=torch.int32, device="cuda")
    options = ab.Options(pose_stride_bytes=stride, output_layout=ab.LAYOUT_QVV40 if qvv40 else ab.LAYOUT_QVV48)
    ctx.decompress_tracks_blend(clipset, _dev(gpu, requests), m, options, buffer.data_ptr() + lead, d_weights=torch.from_numpy(weights).cuda(),
                                d_out_flags=d_flags)
    torch.cuda.synchronize()
    raw = buffer.cpu().numpy()
    assert (raw[:lead] == 0xA5).all() and (raw[lead + stride * m:] == 0xA5).all()
    assert int(d_flags.item()) == 0
    counts = [ref_tracks(b) for b in blobs]
    written = 0
    for i in range(m):
        row = raw[lead + i * stride:lead + (i + 1) * stride]
        f, t = int(from_clip[i]), int(to_clip[i])
        if f >= len(blobs) or t >= len(blobs) or counts[f] != counts[t]:
            assert (row == 0xA5).all(), i
            continue
        n = counts[f]
        assert (row[n * bone:] == 0xA5).all(), i
        want = expected(gpu, blobs[f], blobs[t], tf[i], tt[i], weights[i], 0, 0, ab.LOOP_AS_COMPRESSED)
        assert _rows_equal(row[:n * bone].copy().view(np.float32).reshape(n, bone // 4), want, qvv40), (i, f, t)
        written += 1
    assert written > m // 4
    clipset.release()


def test_object_space(gpu):
    """With parents the blended pose leaves in object space, the skeleton of each pair's from clip: qvvf rows and 3x4 matrices against the
    oracle's walk of the oracle's blended pose; flags from the qvvf walk over the mirrored bones (the matrix walk has no branch to flag)
    and from a parent after its child."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    blobs = gpu["blobs"] + [clips.load_blob("c1_30bones"), clips.load_blob("c5_30x32")]
    clipset = ctx.upload(blobs)
    counts = [ref_tracks(b) for b in blobs]
    skeletons = [tree(c) for c in counts]
    skeletons[2] = np.where(np.arange(30) == 0, ROOT, np.arange(30) - 1).astype(np.uint32)     # a chain
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    parents = np.concatenate(skeletons)
    rng = np.random.default_rng(13)
    m = 120
    choice = [(0, 1), (1, 0), (0, 0), (2, 3), (3, 2)]
    picks = rng.integers(0, len(choice), m)
    from_clip = np.array([choice[p][0] for p in picks], np.uint32)
    to_clip = np.array([choice[p][1] for p in picks], np.uint32)
    tf = rng.uniform(0, 1.3, m).astype(np.float32)
    tt = rng.uniform(0, 1.0, m).astype(np.float32)
    weights = rng.uniform(-0.25, 1.25, m).astype(np.float32)
    d_weights = torch.from_numpy(weights).cuda()
    requests = ab.make_blend_requests(from_clip, tf, to_clip, tt)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for object_kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        got = _run(gpu, requests, ab.Options(), clipset=clipset, d_weights=d_weights, d_parent_indices=_dev(gpu, parents),
                   d_skeleton_offsets=_dev(gpu, offsets), kind=object_kind, d_out_flags=d_flags)
        assert int(d_flags.item()) == (ab.ERROR_FLAG_NEGATIVE_SCALE if object_kind == ab.OBJECT_QVVF else 0)
        for i in range(m):
            f, t = int(from_clip[i]), int(to_clip[i])
            n = counts[f]
            local = expected(gpu, blobs[f], blobs[t], tf[i], tt[i], weights[i], 0, 0, ab.LOOP_AS_COMPRESSED)
            row = got[i, :n * 12].reshape(n, 12)
            if object_kind == ab.OBJECT_MATRIX3X4F:
                assert clips.bit_equal(row, object_space.port_local_to_object_space_matrix(local, skeletons[f])), (i, object_kind)
            else:
                want = port.local_to_object_space(local, skeletons[f], port.NORMALIZE_IEEE)
                assert _rows_equal(row, want), (i, object_kind)
    bad = parents.copy()
    bad[offsets[2] + 3] = 7
    _run(gpu, requests, ab.Options(), clipset=clipset, d_weights=d_weights, d_parent_indices=_dev(gpu, bad),
         d_skeleton_offsets=_dev(gpu, offsets), kind=ab.OBJECT_QVVF, d_out_flags=d_flags)
    assert int(d_flags.item()) == ab.ERROR_FLAG_NEGATIVE_SCALE | ab.ERROR_FLAG_INVALID_SKELETON
    clipset.release()


def test_database_tiers(gpu):
    """A clip set bound to a database, in every tier state of tests/database_cases.py: each bound clip blended with each clip of the same
    track count (both halves decode from what is streamed in) against the reference's poses of those states."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    reference = _Reference(ref, ref_database)
    clipset = ctx.upload(reference.bound + [reference.plain], check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in reference.bound + [reference.plain]]
    pairs = [(f, t) for f in range(5) for t in range(5) if counts[f] == counts[t]]
    times = dbcases.ALL_TIMES
    from_clip = np.repeat([p[0] for p in pairs], len(times)).astype(np.uint32)
    to_clip = np.repeat([p[1] for p in pairs], len(times)).astype(np.uint32)
    tf = np.tile(times, len(pairs)).astype(np.float32)
    tt = np.tile(times[::-1], len(pairs)).astype(np.float32)
    weights = _pair_weights(len(from_clip))
    requests = ab.make_blend_requests(from_clip, tf, to_clip, tt)
    done = []
    for state, ops in dbcases.STATES.items():
        for op, tier, count in ops[len(done):]:
            (database.stream_in if op == dbcases.IN else database.stream_out)(tier, count)
        done = ops
        got = _run(gpu, requests, _options(gpu, 1), clipset=clipset, d_weights=torch.from_numpy(weights).cuda())
        for i in range(len(requests)):
            f, t = int(from_clip[i]), int(to_clip[i])
            n = counts[f]
            from_pose = reference.poses(state, f, tf[i], 0, ab.LOOP_AS_COMPRESSED)
            to_pose = reference.poses(state, t, tt[i], 0, ab.LOOP_AS_COMPRESSED)
            want = blend.port_qvv_lerp(from_pose, to_pose, float(weights[i]), blend.NORMALIZE_IEEE)
            assert _rows_equal(got[i, :n * 12].reshape(n, 12), want), (state, f, t, i)
    clipset.release()


def test_wide_pose_limits(gpu):
    """wide_2500 (2500 bones): two QVV48 poses (2 x 120,000 bytes) do not fit one block and are refused; two QVV40 poses (2 x 100,000)
    fit and decode."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blob = clips.load_blob("wide_2500")
    clipset = ctx.upload([blob])
    times = [0.05, 0.1333, 0.27]
    requests = ab.make_blend_requests([0, 0, 0], times, [0, 0, 0], times[::-1])
    buffer = torch.full((3 * 2500 * 12,), 0x7FC00001, dtype=torch.int32, device="cuda")
    with pytest.raises(ab.api.AclB200Error) as error:
        ctx.decompress_tracks_blend(clipset, _dev(gpu, requests), 3, ab.Options(), buffer, weight=0.5)
    assert error.value.status == 3                   # ACLB200_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (buffer.cpu().numpy() == 0x7FC00001).all()
    got = _run(gpu, requests, _options(gpu, 0, output_layout=ab.LAYOUT_QVV40, pose_stride_bytes=2500 * 48), clipset=clipset, weight=0.3)
    for i, t in enumerate(times):
        want = expected(gpu, blob, blob, t, times[::-1][i], 0.3, 0, 0, ab.LOOP_AS_COMPRESSED)
        assert _rows_equal(got[i, :2500 * 10].reshape(2500, 10), want, True), i
    clipset.release()


def test_refusals_write_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_blend_requests(np.zeros(8), np.linspace(0, 1, 8), np.ones(8), np.linspace(0, 1, 8)))
    parents = _dev(gpu, tree(24))
    skip_tracks = torch.zeros(24, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(clipset=scalar),
        dict(parents=parents, kind=2),
        dict(parents=parents, options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(offset=8),                                 # QVV48 rows must stay 16 byte aligned
        dict(offset=4, options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(options=ab.Options(pose_stride_bytes=24 * 48 + 8)),
    ]
    for case in refusals:
        buffer = torch.full((8 * 24 * 48 + 64 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.decompress_tracks_blend(case.get("clipset", gpu["clipset"]), requests, 8, case.get("options", ab.Options()),
                                        buffer.data_ptr() + case.get("offset", 0), weight=0.5, d_parent_indices=case.get("parents"),
                                        kind=case.get("kind", 0), d_out_flags=d_flags)
        assert error.value.status == 1, case             # ACLB200_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    pose = torch.full((2, 24, 12), 7.0, dtype=torch.float32, device="cuda")
    raw = pose.view(torch.uint8).reshape(-1)
    for args, kw in (((pose, pose, 0), {}), ((raw[8:], pose, pose), {}), ((pose, pose, pose), dict(pose_stride_bytes=24 * 48 + 8))):
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.blend_poses(*args, 1, 24, 0.5, **kw)
        assert error.value.status == 1
    torch.cuda.synchronize()
    assert (pose.cpu().numpy() == 7.0).all()
    scalar.release()


def test_standalone_blend_poses(gpu):
    """aclb200_blend_poses on the fabricated pairs (dot == -0.0, the dpps order, identical, antipodal, mirrored, random) at every weight,
    as one pose of many bones and as many one-bone poses with a weight each, into a third buffer and in place over either input: bit for
    bit against the port, and against the reference's stored lerps within the gate."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    golden = np.load(clips.golden_path("blend", "golden.npz"))
    names, from_rows, to_rows = cases.fabricated_pairs()
    n = len(names)
    stride = n * 48 + 32

    def padded(rows, poses=1):
        out = np.zeros((poses, stride // 4), np.float32)
        out[:, :n * 12] = np.broadcast_to(rows.reshape(1, -1), (poses, n * 12))
        return torch.from_numpy(out).cuda()

    for wi, weight in enumerate(cases.WEIGHTS):
        want = blend.port_qvv_lerp(from_rows, to_rows, float(weight), blend.NORMALIZE_IEEE)
        stored = golden["fabricated"][wi]
        assert clips.bit_equal(want[:, [4, 5, 6, 8, 9, 10]], stored[:, [4, 5, 6, 8, 9, 10]])
        assert float(np.max(np.abs(want[:, 0:4] - stored[:, 0:4]))) <= cases.ROTATION_GATE
        for target in ("third", "from", "to"):
            d_from, d_to = padded(from_rows), padded(to_rows)
            d_out = {"third": torch.full_like(d_from, float("nan")), "from": d_from, "to": d_to}[target]
            ctx.blend_poses(d_from, d_to, d_out, 1, n, float(weight), pose_stride_bytes=stride)
            torch.cuda.synchronize()
            got = d_out.cpu().numpy()
            assert _rows_equal(got[0, :n * 12].reshape(n, 12), want), (float(weight), target)
            if target == "third":
                assert np.isnan(got[:, n * 12:]).all()

    # one bone per pose, a weight per pose from d_weights
    weights = np.resize(cases.WEIGHTS, n).astype(np.float32)
    d_from = torch.from_numpy(from_rows.copy()).cuda()
    d_to = torch.from_numpy(to_rows.copy()).cuda()
    d_out = torch.full_like(d_from, float("nan"))
    ctx.blend_poses(d_from, d_to, d_out, n, 1, 0.0, d_weights=torch.from_numpy(weights).cuda())
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    for i in range(n):
        want = blend.port_qvv_lerp(from_rows[i:i + 1], to_rows[i:i + 1], float(weights[i]), blend.NORMALIZE_IEEE)
        assert _rows_equal(got[i:i + 1], want), (names[i], float(weights[i]))


def test_c2_launch_equals_the_unfused_route(gpu):
    """300,000 pairs over the C2 bench clips (100 bones): the fused call writes byte for byte what decompress_tracks(from) +
    decompress_tracks(to) + aclb200_blend_poses write, with a weight per pair and with the scalar weight, checked on the device."""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    m, bones = 300000, w["num_tracks"]
    rng = np.random.default_rng(21)
    from_clip, from_time = w["req_clip"][:m], w["req_time"][:m]
    to_clip = rng.permutation(w["req_clip"])[:m]
    to_time = rng.permutation(w["req_time"])[:m]
    weights = torch.from_numpy(rng.uniform(-0.25, 1.25, m).astype(np.float32)).cuda()
    options = ab.Options()
    d_from = torch.empty((m, bones, 12), dtype=torch.float32, device="cuda")
    d_to = torch.empty_like(d_from)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(from_clip, from_time)), m, options, d_from)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(to_clip, to_time)), m, options, d_to)
    d_pairs = _dev(gpu, ab.make_blend_requests(from_clip, from_time, to_clip, to_time))
    d_unfused = torch.empty_like(d_from)
    d_fused = torch.empty_like(d_from)
    for kw in (dict(d_weights=weights), dict(weight=0.375)):
        ctx.blend_poses(d_from, d_to, d_unfused, m, bones, **kw)
        d_fused.fill_(float("nan"))
        ctx.decompress_tracks_blend(clipset, d_pairs, m, options, d_fused, **kw)
        torch.cuda.synchronize()
        assert torch.equal(d_fused.view(torch.int32), d_unfused.view(torch.int32)), list(kw)
    clipset.release()
