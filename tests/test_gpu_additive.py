"""aclb200_decompress_tracks_additive (decompress base + decompress additive + apply_additive_to_base in one kernel) and
aclb200_apply_additive_to_base, against
  * the port's decode of both clips (the additive one with the track_writer defaults) and its apply_additive_to_base (oracle/acl_oracle.c,
    pinned to the reference by tests/test_additive_oracle.py): BIT FOR BIT, with the IEEE quat_normalize in the negative scale branch;
  * additive.golden.npz, the reference's own poses: bit for bit on every bone that does not take the negative scale branch;
  * the unfused route (two decompress_tracks launches + aclb200_apply_additive_to_base) at the C2 launch size: byte for byte.
"""
import numpy as np
import pytest

from oracle import object_space
from tests import additive_cases as cases
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


def expected(gpu, format_, base_blob, additive_blob, tb, ta, kind, rounding, looping, base_settings=None):
    port = gpu["port"]
    return cases.port_pose(port, format_, base_blob, additive_blob, tb, ta, base_settings or port.settings_for_kind(kind),
                           cases.writer_settings(port, kind), rounding, looping, port.NORMALIZE_IEEE)


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
    ctx.decompress_tracks_additive(clipset, _dev(gpu, requests), n, options, d_out, **kw)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.float32)


@pytest.mark.parametrize("name", list(cases.FORMATS))
def test_formats_match_the_oracle(gpu, name):
    """Every golden combo (settings kind, rounding, looping) of each format clip, QVV48 and QVV40, then per request policies in one launch and
    a variable bind pose on the base (the additive half keeps the track_writer defaults)."""
    ab, port = gpu["ab"], gpu["port"]
    format_ = cases.FORMATS[name]
    ci = cases.NAMES.index(name)
    base_blob, additive_blob = gpu["blobs"][0], gpu["blobs"][ci]
    pairs = cases.time_pairs()
    n = cases.BASE_SPEC.num_tracks
    requests = ab.make_additive_requests(np.zeros(len(pairs)), pairs[:, 0], np.full(len(pairs), ci), pairs[:, 1])
    for kind, rounding, looping in cases.COMBOS:
        for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
            options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping, output_layout=layout, pose_stride_bytes=n * 48)
            got = _run(gpu, requests, options, additive_format=format_)
            for i, (tb, ta) in enumerate(pairs):
                want = expected(gpu, format_, base_blob, additive_blob, tb, ta, kind, rounding, looping)
                row = got[i, :n * 12].reshape(n, 12) if layout == ab.LAYOUT_QVV48 else got[i, :n * 10].reshape(n, 10)
                assert _rows_equal(row, want, layout == ab.LAYOUT_QVV40), (name, kind, rounding, looping, layout, i)

    policies = np.resize(np.array([(r, l) for r in range(4) for l in range(3)], np.uint8), (len(pairs), 2))
    d_policies = _dev(gpu, policies)
    variable = np.tile(IDENTITY, (n, 1))
    rng = np.random.default_rng(5)
    variable[:, 4:7] = rng.uniform(-2, 2, (n, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (n, 3))
    d_variable = gpu["torch"].from_numpy(variable).cuda()
    base_settings = port.settings_for_kind(0, default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable)
    options = _options(gpu, 0, d_request_policies=d_policies.data_ptr(), default_modes=(ab.DEFAULT_VARIABLE,) * 3,
                       d_variable_defaults=d_variable.data_ptr())
    got = _run(gpu, requests, options, additive_format=format_)
    for i, (tb, ta) in enumerate(pairs):
        rounding, looping = int(policies[i][0]), int(policies[i][1])
        want = expected(gpu, format_, base_blob, additive_blob, tb, ta, 0, rounding, looping, base_settings)
        assert _rows_equal(got[i, :n * 12].reshape(n, 12), want), (name, "policies + variable", i)


def test_reference_poses(gpu):
    """additive.golden.npz: the reference's decode-and-apply, bit for bit except the bones whose `relative` product takes rtm::qvv_mul's
    matrix branch (the reference normalises with rsqrtss there): those within 1e-5."""
    ab = gpu["ab"]
    golden = np.load(clips.golden_path("additive", "golden.npz"))
    pairs = golden["pairs"]
    n = cases.BASE_SPEC.num_tracks
    for fi, (name, format_) in enumerate(cases.FORMATS.items()):
        ci = cases.NAMES.index(name)
        requests = ab.make_additive_requests(np.zeros(len(pairs)), pairs[:, 0], np.full(len(pairs), ci), pairs[:, 1])
        for k, (kind, rounding, looping) in enumerate(cases.COMBOS):
            got = _run(gpu, requests, _options(gpu, kind, rounding_policy=rounding, looping_policy=looping), additive_format=format_)
            got = got[:, :n * 12].reshape(len(pairs), n, 12)[..., LANES]
            want = golden["poses"][fi, k]
            exact = np.ones(n, bool)
            if format_ == ab.ADDITIVE_RELATIVE:
                exact = ~((np.arange(n) * 7 + 3) % 100 < cases.BASE_SPEC.negative_scale_pct)     # the mirrored bones of the base
            assert clips.bit_equal(got[:, exact], want[:, exact]), (name, kind, rounding, looping)
            assert float(np.max(np.abs(got - want))) <= 1e-5, (name, kind, rounding, looping)


def test_additive1_default_scale_reads_zero(gpu):
    """The additive1 clip's default scale sub-tracks decode as 0 (its own default scale), not as a bind pose or a constant 1: with a
    constant default scale of 1 they would give 2 x base scale."""
    ab = gpu["ab"]
    ci = cases.NAMES.index("additive_additive1")
    n = cases.BASE_SPEC.num_tracks
    requests = ab.make_additive_requests([0], [0.1], [ci], [0.1])
    base = gpu["port"].transform_decompress_tracks(gpu["blobs"][0], gpu["port"].settings_for_kind(0), 0.1)
    additive = gpu["port"].transform_decompress_tracks(gpu["blobs"][ci], cases.writer_settings(gpu["port"], 0), 0.1)
    zero = (additive[:, 8:11] == 0.0).all(axis=1)
    assert zero.any()
    options = _options(gpu, 0, constant_defaults=[0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 1], default_modes=(ab.DEFAULT_CONSTANT,) * 3)
    got = _run(gpu, requests, options, additive_format=ab.ADDITIVE_ADDITIVE1)[0, :n * 12].reshape(n, 12)
    assert clips.bit_equal(got[zero][:, 8:11], base[zero][:, 8:11])


def test_per_clip_formats_and_untouched_bytes(gpu):
    """A clip set with the four clips and a 30 bone clip: per clip formats (a byte above 3 reads as none), invalid clip indices and track
    count mismatches, a padded stride and an output 16 bytes into its allocation: every byte nobody may write keeps its sentinel."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blobs = gpu["blobs"] + [clips.load_blob("c1_30bones")]
    clipset = ctx.upload(blobs, check_hash=True)
    formats = np.array([9, 1, 2, 3, 0], np.uint8)       # byte of the additive clip; the base's 9 reads as none
    rng = np.random.default_rng(12)
    m = 400
    base_clip = rng.choice([0, 0, 0, 1, 2, 4, 5, 0xFFFFFFFF], m).astype(np.uint32)
    additive_clip = rng.choice([0, 1, 2, 3, 3, 4, 6], m).astype(np.uint32)
    tb = rng.uniform(-0.2, 1.6, m).astype(np.float32)
    ta = rng.uniform(-0.2, 1.2, m).astype(np.float32)
    requests = ab.make_additive_requests(base_clip, tb, additive_clip, ta)
    stride = clipset.max_tracks * 48 + 32
    lead = 16
    buffer = torch.full((lead + stride * m + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d_flags = torch.full((1,), 0x7F, dtype=torch.int32, device="cuda")
    ctx.decompress_tracks_additive(clipset, _dev(gpu, requests), m, ab.Options(pose_stride_bytes=stride), buffer.data_ptr() + lead,
                                   additive_format=ab.ADDITIVE_RELATIVE, d_clip_additive_formats=_dev(gpu, formats), d_out_flags=d_flags)
    torch.cuda.synchronize()
    raw = buffer.cpu().numpy()
    assert (raw[:lead] == 0xA5).all() and (raw[lead + stride * m:] == 0xA5).all()
    counts = [ref_tracks(b) for b in blobs]
    written = 0
    for i in range(m):
        row = raw[lead + i * stride:lead + (i + 1) * stride]
        b, a = int(base_clip[i]), int(additive_clip[i])
        if b >= len(blobs) or a >= len(blobs) or counts[b] != counts[a]:
            assert (row == 0xA5).all(), i
            continue
        n = counts[b]
        assert (row[n * 48:] == 0xA5).all(), i
        format_ = int(formats[a]) if formats[a] <= 3 else 0
        want = expected(gpu, format_, blobs[b], blobs[a], tb[i], ta[i], 0, 0, ab.LOOP_AS_COMPRESSED)
        assert _rows_equal(row[:n * 48].copy().view(np.float32).reshape(n, 12), want), (i, b, a)
        written += 1
    assert written > m // 3
    assert int(d_flags.item()) == ab.ERROR_FLAG_NEGATIVE_SCALE      # relative pairs over the mirrored base bones
    clipset.release()


def ref_tracks(blob):
    return int(blob[16:20].view(np.uint32)[0])


def test_object_space(gpu):
    """With parents the combined pose leaves in object space, the skeleton of each pair's base clip: qvvf rows and 3x4 matrices against
    the oracle's walk of the oracle's combined pose; flags from the mirrored bones and from a parent after its child."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    blobs = gpu["blobs"] + [clips.load_blob("c1_30bones"), clips.load_blob("c5_30x32")]
    clipset = ctx.upload(blobs)
    counts = [ref_tracks(b) for b in blobs]
    skeletons = [tree(c) for c in counts]
    skeletons[4] = np.where(np.arange(30) == 0, ROOT, np.arange(30) - 1).astype(np.uint32)     # a chain
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    parents = np.concatenate(skeletons)
    rng = np.random.default_rng(13)
    m = 120
    choice = [(0, 1, 1), (0, 2, 2), (0, 3, 3), (4, 5, 2), (5, 4, 3)]
    picks = rng.integers(0, len(choice), m)
    base_clip = np.array([choice[p][0] for p in picks], np.uint32)
    additive_clip = np.array([choice[p][1] for p in picks], np.uint32)
    formats = np.array([0, 1, 2, 3, 2, 3], np.uint8)
    tb = rng.uniform(0, 1.3, m).astype(np.float32)
    ta = rng.uniform(0, 1.0, m).astype(np.float32)
    requests = ab.make_additive_requests(base_clip, tb, additive_clip, ta)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for object_kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        got = _run(gpu, requests, ab.Options(), clipset=clipset, d_clip_additive_formats=_dev(gpu, formats), d_parent_indices=_dev(gpu, parents),
                   d_skeleton_offsets=_dev(gpu, offsets), kind=object_kind, d_out_flags=d_flags)
        assert int(d_flags.item()) == ab.ERROR_FLAG_NEGATIVE_SCALE
        for i in range(m):
            b, a = int(base_clip[i]), int(additive_clip[i])
            n = counts[b]
            local = expected(gpu, int(formats[a]), blobs[b], blobs[a], tb[i], ta[i], 0, 0, ab.LOOP_AS_COMPRESSED)
            row = got[i, :n * 12].reshape(n, 12)
            if object_kind == ab.OBJECT_MATRIX3X4F:
                assert clips.bit_equal(row, object_space.port_local_to_object_space_matrix(local, skeletons[b])), (i, object_kind)
            else:
                want = port.local_to_object_space(local, skeletons[b], port.NORMALIZE_IEEE)
                assert _rows_equal(row, want), (i, object_kind)
    bad = parents.copy()
    bad[offsets[4] + 3] = 7
    _run(gpu, requests, ab.Options(), clipset=clipset, d_clip_additive_formats=_dev(gpu, formats), d_parent_indices=_dev(gpu, bad),
         d_skeleton_offsets=_dev(gpu, offsets), kind=ab.OBJECT_QVVF, d_out_flags=d_flags)
    assert int(d_flags.item()) == ab.ERROR_FLAG_NEGATIVE_SCALE | ab.ERROR_FLAG_INVALID_SKELETON
    clipset.release()


def test_database_tiers(gpu):
    """A clip set bound to a database, in every tier state of tests/database_cases.py: each bound clip layered on the plain clip of the same
    database spec (both halves decode from what is streamed in) against the reference's poses of those states."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    reference = _Reference(ref, ref_database)
    clipset = ctx.upload(reference.bound + [reference.plain], check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in reference.bound + [reference.plain]]
    pairs = [(b, a) for b in range(5) for a in range(5) if counts[a] == counts[b]]
    times = dbcases.ALL_TIMES
    base_clip = np.repeat([p[0] for p in pairs], len(times)).astype(np.uint32)
    additive_clip = np.repeat([p[1] for p in pairs], len(times)).astype(np.uint32)
    tb = np.tile(times, len(pairs)).astype(np.float32)
    ta = np.tile(times[::-1], len(pairs)).astype(np.float32)
    requests = ab.make_additive_requests(base_clip, tb, additive_clip, ta)
    done = []
    for state, ops in dbcases.STATES.items():
        for op, tier, count in ops[len(done):]:
            (database.stream_in if op == dbcases.IN else database.stream_out)(tier, count)
        done = ops
        got = _run(gpu, requests, _options(gpu, 1), clipset=clipset, additive_format=ab.ADDITIVE_ADDITIVE0)
        for i in range(len(requests)):
            b, a = int(base_clip[i]), int(additive_clip[i])
            n = counts[b]
            base = reference.poses(state, b, tb[i], 0, ab.LOOP_AS_COMPRESSED)
            additive = reference.poses(state, a, ta[i], 0, ab.LOOP_AS_COMPRESSED)
            want = port.apply_additive_to_base(ab.ADDITIVE_ADDITIVE0, base, additive, port.NORMALIZE_IEEE)
            assert _rows_equal(got[i, :n * 12].reshape(n, 12), want), (state, b, a, i)
    clipset.release()


def test_wide_pose_limits(gpu):
    """wide_2500 (2500 bones): two QVV48 poses (2 x 120,000 bytes) do not fit one block and are refused; two QVV40 poses (2 x 100,000)
    fit and decode."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blob = clips.load_blob("wide_2500")
    clipset = ctx.upload([blob])
    times = [0.05, 0.1333, 0.27]
    requests = ab.make_additive_requests([0, 0, 0], times, [0, 0, 0], times[::-1])
    buffer = torch.full((3 * 2500 * 12,), 0x7FC00001, dtype=torch.int32, device="cuda")
    with pytest.raises(ab.api.AclB200Error) as error:
        ctx.decompress_tracks_additive(clipset, _dev(gpu, requests), 3, ab.Options(), buffer, additive_format=ab.ADDITIVE_ADDITIVE0)
    assert error.value.status == 3                   # ACLB200_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (buffer.cpu().numpy() == 0x7FC00001).all()
    got = _run(gpu, requests, _options(gpu, 0, output_layout=ab.LAYOUT_QVV40, pose_stride_bytes=2500 * 48), clipset=clipset,
               additive_format=ab.ADDITIVE_ADDITIVE0)
    for i, t in enumerate(times):
        want = expected(gpu, ab.ADDITIVE_ADDITIVE0, blob, blob, t, times[::-1][i], 0, 0, ab.LOOP_AS_COMPRESSED)
        assert _rows_equal(got[i, :2500 * 10].reshape(2500, 10), want, True), i
    clipset.release()


def test_refusals_write_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_additive_requests(np.zeros(8), np.linspace(0, 1, 8), np.ones(8), np.linspace(0, 1, 8)))
    parents = _dev(gpu, tree(24))
    skip_tracks = torch.zeros(24, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(format=4),
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
            ctx.decompress_tracks_additive(case.get("clipset", gpu["clipset"]), requests, 8, case.get("options", ab.Options()),
                                           buffer.data_ptr() + case.get("offset", 0), additive_format=case.get("format", 1),
                                           d_parent_indices=case.get("parents"), kind=case.get("kind", 0), d_out_flags=d_flags)
        assert error.value.status == 1, case             # ACLB200_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    pose = torch.zeros((2, 24, 12), dtype=torch.float32, device="cuda")
    for kw in (dict(additive_format=4), dict(additive_format=1, pose_stride_bytes=24 * 48 + 8)):
        with pytest.raises(ab.api.AclB200Error):
            ctx.apply_additive_to_base(pose, pose, pose, 2, 24, **kw)
    scalar.release()


def test_standalone_apply(gpu):
    """aclb200_apply_additive_to_base over decoded poses in every format, into a third buffer and in place over either input (flags
    from the mirrored bones of `relative`)."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    pairs = cases.time_pairs()
    m, n = len(pairs), cases.BASE_SPEC.num_tracks
    base = np.stack([port.transform_decompress_tracks(gpu["blobs"][0], port.settings_for_kind(0), float(t)) for t in pairs[:, 0]])
    base[..., [7, 11]] = 0.0
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    stride = n * 48 + 16
    for name, format_ in [("additive_relative", 1), ("additive_additive0", 2), ("additive_additive1", 3), ("additive_relative", 0)]:
        blob = gpu["blobs"][cases.NAMES.index(name)]
        additive = np.stack([port.transform_decompress_tracks(blob, cases.writer_settings(port, 0), float(t)) for t in pairs[:, 1]])
        want = np.stack([port.apply_additive_to_base(format_, base[i], additive[i], port.NORMALIZE_IEEE) for i in range(m)])

        def padded(a):
            out = np.zeros((m, stride // 4), np.float32)
            out[:, :n * 12] = a.reshape(m, -1)
            return torch.from_numpy(out).cuda()
        for target in ("third", "base", "additive"):
            d_base, d_add = padded(base), padded(additive)
            d_out = {"third": torch.full_like(d_base, float("nan")), "base": d_base, "additive": d_add}[target]
            ctx.apply_additive_to_base(d_base, d_add, d_out, m, n, format_, pose_stride_bytes=stride, d_out_flags=d_flags)
            torch.cuda.synchronize()
            got = d_out.cpu().numpy()
            assert int(d_flags.item()) == (ab.ERROR_FLAG_NEGATIVE_SCALE if format_ == 1 else 0), (name, format_, target)
            for i in range(m):
                assert _rows_equal(got[i, :n * 12].reshape(n, 12), want[i]), (name, format_, target, i)
            if target == "third":
                assert np.isnan(got[:, n * 12:]).all()


def test_c2_launch_equals_the_unfused_route(gpu):
    """300,000 pairs over the C2 bench clips (100 bones; every pair's clips from the same clip set): the fused call writes byte for byte
    what decompress_tracks(base) + decompress_tracks(additive, track_writer defaults) + aclb200_apply_additive_to_base write, checked
    on the device for every pair and format."""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    m, bones = 300000, w["num_tracks"]
    rng = np.random.default_rng(21)
    base_clip, base_time = w["req_clip"][:m], w["req_time"][:m]
    additive_clip = rng.permutation(w["req_clip"])[:m]
    additive_time = rng.permutation(w["req_time"])[:m]
    options = ab.Options()
    writer = ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_CONSTANT, ab.DEFAULT_LEGACY),
                        constant_defaults=[0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0])
    d_base = torch.empty((m, bones, 12), dtype=torch.float32, device="cuda")
    d_add = torch.empty_like(d_base)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(base_clip, base_time)), m, options, d_base)
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(additive_clip, additive_time)), m, writer, d_add)
    d_pairs = _dev(gpu, ab.make_additive_requests(base_clip, base_time, additive_clip, additive_time))
    d_unfused = torch.empty_like(d_base)
    d_fused = torch.empty_like(d_base)
    for format_ in (0, 1, 2, 3):
        ctx.apply_additive_to_base(d_base, d_add, d_unfused, m, bones, format_)
        d_fused.fill_(float("nan"))
        ctx.decompress_tracks_additive(clipset, d_pairs, m, options, d_fused, additive_format=format_)
        torch.cuda.synchronize()
        assert torch.equal(d_fused.view(torch.int32), d_unfused.view(torch.int32)), format_
    clipset.release()
