"""aclb200_decompress_tracks_object_space: decompress_tracks and the hierarchy walk in one kernel, against
  * the oracle's decode followed by its object space (oracle/acl_oracle.c, pinned to the reference by tests/test_oracle_vs_reference.py,
    tests/test_error_metric_oracle.py and tests/test_object_space_oracle.py): BIT FOR BIT, IEEE normalisation for qvvf rows, the matrix
    metric's convert_transforms + local_to_object_space for matrices;
  * decompress_tracks followed by aclb200_local_to_object_space at the C2 launch size: bit for bit;
  * the reference itself where oracle/_ref/libaclref.so and libaclref_object_space.so exist: qvvf within the normalisation tolerance, matrices bit for bit.
"""
import numpy as np
import pytest

from oracle import object_space
from tests import clips
from tests import database_cases as cases
from tests.test_error_metric_oracle import ERROR_TOLERANCE

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
    return dict(torch=torch, ab=ab, port=port, ctx=ab.Context(0))


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


def skeleton(kind, n, rng=None):
    bones = np.arange(n)
    if kind == "chain":
        return np.where(bones == 0, ROOT, bones - 1).astype(np.uint32)
    if kind == "star":
        return np.where(bones == 0, ROOT, 0).astype(np.uint32)
    if kind == "random":
        parents = np.array([ROOT] + [int(rng.integers(0, b)) for b in range(1, n)], np.uint32)
        parents[rng.random(n) < 0.1] = ROOT          # a few more roots
        return parents
    return tree(n)


def expected(gpu, local, parents, object_kind):
    """the oracle's object space of one local pose, as the 48 byte rows the call writes ([n][12] float32)"""
    port, ab = gpu["port"], gpu["ab"]
    if object_kind == ab.OBJECT_MATRIX3X4F:
        return object_space.port_local_to_object_space_matrix(local, parents)
    out = port.local_to_object_space(local, parents, port.NORMALIZE_IEEE)
    out[:, 7] = 0.0
    out[:, 11] = 0.0
    return out


def _run(gpu, clipset, requests, options, parents, object_kind, offsets=None, flags=None, stride_floats=None, fill=float("nan")):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    n = len(requests)
    width = stride_floats or clipset.max_tracks * 12
    d_out = torch.full((n, width), fill, dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_object_space(clipset, _dev(gpu, requests), n, options, _dev(gpu, parents), object_kind, d_out,
                                       d_skeleton_offsets=None if offsets is None else _dev(gpu, offsets), d_out_flags=flags)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def _same_rows(got, want, object_kind, ab):
    lanes = slice(None) if object_kind == ab.OBJECT_MATRIX3X4F else LANES
    return clips.bit_equal(got[:, lanes], want[:, lanes]) and (object_kind == ab.OBJECT_MATRIX3X4F or not got[:, [7, 11]].any())


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_named_clips_match_the_oracle(gpu, name):
    """Every settings kind, every rounding and looping policy (per request where the settings allow it, batch wide with per track
    rounding), variable defaults, both object kinds."""
    ab, port = gpu["ab"], gpu["port"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = gpu["ctx"].upload([blob], check_hash=True)
    parents = tree(spec.num_tracks)
    times = clips.sample_times(spec)[::2]
    pairs = [(r, l) for r in range(4) for l in range(3)]
    rng = np.random.default_rng(spec.seed)
    variable = np.tile(IDENTITY, (spec.num_tracks, 1))
    variable[:, 4:7] = rng.uniform(-2, 2, (spec.num_tracks, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (spec.num_tracks, 3))
    d_variable = gpu["torch"].from_numpy(variable).cuda()
    cases_ = [(kind, {}) for kind in range(6)] + [(0, dict(variable=True))]
    for kind, extra in cases_:
        settings = port.settings_for_kind(kind, **(dict(default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable) if extra else {}))
        fields = dict(default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr()) if extra else {}
        per_track = settings.c.per_track_rounding != 0
        launches = []
        if per_track:
            for rounding, looping in pairs:
                launches.append((_options(gpu, kind, rounding_policy=rounding, looping_policy=looping, **fields), [(rounding, looping)] * len(times)))
        else:
            policies = np.array([p for p in pairs for _ in times], np.uint8)
            d_policies = _dev(gpu, policies)
            launches.append((_options(gpu, kind, d_request_policies=d_policies.data_ptr(), **fields), [tuple(p) for p in policies], d_policies))
        for launch in launches:
            options, policy_list = launch[0], launch[1]
            request_times = np.resize(times, len(policy_list))
            requests = ab.make_requests(np.zeros(len(policy_list), np.uint32), request_times)
            got = {k: _run(gpu, clipset, requests, options, parents, k).reshape(len(requests), -1, 12)
                   for k in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F)}
            for i, ((rounding, looping), t) in enumerate(zip(policy_list, request_times)):
                local = port.transform_decompress_tracks(blob, settings, float(t), int(rounding), int(looping))
                for k, out in got.items():
                    assert _same_rows(out[i], expected(gpu, local, parents, k), k, ab), (name, kind, extra, rounding, looping, float(t), k)
    clipset.release()


@pytest.mark.parametrize("name", ["c1_30bones", "mixed_scale", "stripped_single", "ragged_17", "paragon_like"])
def test_live_reference(gpu, name):
    """The reference's own object space: calculate_compression_error's decode (debug settings, identity bind pose) taken to object
    space by qvvf_transform_error_metric (within ERROR_TOLERANCE: rsqrtss) and by the matrix metric (bit for bit)."""
    from oracle import ref
    if not ref.available() or not object_space.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so and libaclref_object_space.so")
    torch, ab = gpu["torch"], gpu["ab"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    r = ref.transform_error(spec, blob, 1)
    clipset = gpu["ctx"].upload([blob])
    times = np.array([min(np.float32(s) / np.float32(r["sample_rate"]), np.float32(r["duration"])) for s in range(spec.num_samples)], np.float32)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_identity = torch.from_numpy(np.tile(IDENTITY, (spec.num_tracks, 1))).cuda()
    options = _options(gpu, 1, rounding_policy=r["rounding"], default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_identity.data_ptr())
    qvvf = _run(gpu, clipset, requests, options, r["parents"], ab.OBJECT_QVVF).reshape(len(times), -1, 12)
    matrix = _run(gpu, clipset, requests, options, r["parents"], ab.OBJECT_MATRIX3X4F).reshape(len(times), -1, 12)
    assert float(np.max(np.abs(qvvf[..., LANES] - r["object_poses"][1][..., LANES]))) <= ERROR_TOLERANCE
    for s in range(spec.num_samples):
        assert clips.bit_equal(matrix[s], object_space.reference_local_to_object_space_matrix(r["lossy_poses"][s], r["parents"])), (name, s)
    clipset.release()


def test_c2_launch_composes_the_two_calls(gpu):
    """The C2 bench workload in one launch (600,000 requests x 100 bones, binary tree skeleton): qvvf rows equal decompress_tracks
    followed by local_to_object_space for every request; matrices equal the oracle on a seeded sample that holds the first and last request."""
    import bench
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    from oracle import ref
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    n, bones = int(w["req_clip"].size), w["num_tracks"]
    assert n == 600000 and bones == 100
    parents = tree(bones)
    d_parents = _dev(gpu, parents)
    d_requests = _dev(gpu, ab.make_requests(w["req_clip"], w["req_time"]))
    options = ab.Options()
    d_local = torch.empty((n, bones, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n, options, d_local)
    d_two_step = torch.full_like(d_local, float("nan"))
    ctx.local_to_object_space(d_local, d_two_step, n, bones, d_parents)
    del d_local
    d_fused = torch.full_like(d_two_step, float("nan"))
    ctx.decompress_tracks_object_space(clipset, d_requests, n, options, d_parents, ab.OBJECT_QVVF, d_fused)
    torch.cuda.synchronize()
    assert torch.equal(d_fused.view(torch.int32), d_two_step.view(torch.int32))
    del d_two_step
    ctx.decompress_tracks_object_space(clipset, d_requests, n, options, d_parents, ab.OBJECT_MATRIX3X4F, d_fused)
    torch.cuda.synchronize()
    sample = np.unique(np.concatenate([[0, n - 1], np.random.default_rng(1).choice(n, 5000, replace=False)]))
    got = d_fused[torch.from_numpy(sample).cuda()].cpu().numpy()
    del d_fused
    settings = port.settings_for_kind(0)
    blobs = {}
    for row, i in enumerate(sample):
        c = int(w["req_clip"][i])
        if c not in blobs:
            start = int(w["offsets"][c])
            blobs[c] = ref.aligned_blob(w["buffer"][start:start + int(w["sizes"][c])].tobytes())
        local = port.transform_decompress_tracks(blobs[c], settings, float(w["req_time"][i]))
        assert clips.bit_equal(got[row], object_space.port_local_to_object_space_matrix(local, parents)), int(i)
    clipset.release()


def test_mixed_rigs_and_untouched_bytes(gpu):
    """One ragged clip set with a skeleton per clip (chain, tree, star, random), invalid clip indices, a padded stride and an output
    pointer 16 bytes into its allocation: every byte no request may write keeps its sentinel."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    names = ["c1_30bones", "ragged_17", "mixed_scale", "one_bone", "c2_100bones", "single_segment"]
    kinds = ["chain", "tree", "star", "random", "random", "chain"]
    rng = np.random.default_rng(11)
    blobs = [clips.load_blob(n) for n in names]
    specs = [clips.TRANSFORM_SPECS[n] for n in names]
    skeletons = [skeleton(k, s.num_tracks, rng) for k, s in zip(kinds, specs)]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in skeletons])[:-1]]).astype(np.uint32)
    parents = np.concatenate(skeletons)
    clipset = ctx.upload(blobs, check_hash=True)
    num_requests = 300
    req_clip = rng.integers(0, len(names), num_requests).astype(np.uint32)
    req_clip[rng.random(num_requests) < 0.08] = len(names)
    req_clip[7] = 0xFFFFFFFF
    req_time = rng.uniform(-0.2, 2.5, num_requests).astype(np.float32)
    requests = ab.make_requests(req_clip, req_time)
    stride = clipset.max_tracks * 48 + 32
    lead = 16
    settings = port.settings_for_kind(0)
    for object_kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        buffer = torch.full((lead + stride * num_requests + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        options = ab.Options(pose_stride_bytes=stride)
        d_flags = torch.full((1,), 0x7F, dtype=torch.int32, device="cuda")
        ctx.decompress_tracks_object_space(clipset, _dev(gpu, requests), num_requests, options, _dev(gpu, parents), object_kind,
                                           buffer.data_ptr() + lead, d_skeleton_offsets=_dev(gpu, offsets), d_out_flags=d_flags)
        torch.cuda.synchronize()
        raw = buffer.cpu().numpy()
        assert int(d_flags.item()) == 0
        assert (raw[:lead] == 0xA5).all() and (raw[lead + stride * num_requests:] == 0xA5).all()
        for i in range(num_requests):
            row = raw[lead + i * stride:lead + (i + 1) * stride]
            c = int(req_clip[i])
            if c >= len(names):
                assert (row == 0xA5).all(), i
                continue
            n = specs[c].num_tracks
            assert (row[n * 48:] == 0xA5).all(), i
            local = port.transform_decompress_tracks(blobs[c], settings, float(req_time[i]))
            got = row[:n * 48].copy().view(np.float32).reshape(n, 12)
            assert _same_rows(got, expected(gpu, local, skeletons[c], object_kind), object_kind, ab), (names[c], kinds[c], i, object_kind)
    clipset.release()


def test_flags(gpu):
    """A parent after its child is reported and the bone taken as a root; mirrored bones (a negative default scale) take rtm::qvv_mul's
    matrix branch, are reported, and still match the oracle bit for bit."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = ctx.upload([blob])
    times = clips.sample_times(spec)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    parents = tree(spec.num_tracks)
    bad = parents.copy()
    bad[7] = 9
    as_root = parents.copy()
    as_root[7] = ROOT
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    settings = port.settings_for_kind(0)
    for object_kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        got = _run(gpu, clipset, requests, ab.Options(), bad, object_kind, flags=d_flags).reshape(len(times), -1, 12)
        assert int(d_flags.item()) == ab.ERROR_FLAG_INVALID_SKELETON
        for i, t in enumerate(times):
            assert _same_rows(got[i], expected(gpu, port.transform_decompress_tracks(blob, settings, float(t)), as_root, object_kind), object_kind, ab)

    variable = np.tile(IDENTITY, (spec.num_tracks, 1))
    variable[::3, 8] = -1.0                          # bones whose scale is a default sub-track become mirrored
    d_variable = torch.from_numpy(variable).cuda()
    mirrored = port.settings_for_kind(0, default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable)
    options = ab.Options(default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
    for object_kind, flag in ((ab.OBJECT_QVVF, ab.ERROR_FLAG_NEGATIVE_SCALE), (ab.OBJECT_MATRIX3X4F, 0)):
        got = _run(gpu, clipset, requests, options, parents, object_kind, flags=d_flags).reshape(len(times), -1, 12)
        assert int(d_flags.item()) == flag
        for i, t in enumerate(times):
            local = port.transform_decompress_tracks(blob, mirrored, float(t))
            assert local[:, 8].min() < 0.0
            assert _same_rows(got[i], expected(gpu, local, parents, object_kind), object_kind, ab), (object_kind, float(t))
    clipset.release()


def test_database_tiers(gpu):
    """Every tier state of tests/golden/database_tiers.npz (or the live reference): the object space of the reference's poses."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    reference = _Reference(ref, ref_database)
    clipset = ctx.upload(reference.bound + [reference.plain], check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in reference.bound + [reference.plain]]
    skeletons = [tree(n) for n in counts]
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    parents = np.concatenate(skeletons)
    req_clip = np.repeat(np.arange(5, dtype=np.uint32), len(cases.ALL_TIMES))
    req_time = np.tile(cases.ALL_TIMES, 5)
    requests = ab.make_requests(req_clip, req_time)
    done = []
    for state, ops in cases.STATES.items():
        for op, tier, n in ops[len(done):]:
            (database.stream_in if op == cases.IN else database.stream_out)(tier, n)
        done = ops
        for object_kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
            got = _run(gpu, clipset, requests, _options(gpu, 1), parents, object_kind, offsets=offsets).reshape(len(requests), -1, 12)
            for i, (c, t) in enumerate(zip(req_clip, req_time)):
                local = reference.poses(state, int(c), t, 0, ab.LOOP_AS_COMPRESSED)
                n = local.shape[0]
                assert _same_rows(got[i, :n], expected(gpu, local, skeletons[c], object_kind), object_kind, ab), (state, int(c), float(t), object_kind)
    clipset.release()


def test_refusals_write_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blob = clips.load_blob("c1_30bones")
    clipset = ctx.upload([blob])
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_requests(np.zeros(8, np.uint32), np.linspace(0, 1, 8).astype(np.float32)))
    parents = _dev(gpu, tree(30))
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(kind=2),
        dict(parents=None),
        dict(clipset=scalar),
        dict(offset=8),         # QVV48 rows must stay 16 byte aligned
    ]
    for case in refusals:
        buffer = torch.full((8 * 30 * 48 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.decompress_tracks_object_space(case.get("clipset", clipset), requests, 8, case.get("options", ab.Options()),
                                               case["parents"] if "parents" in case else parents, case.get("kind", ab.OBJECT_QVVF),
                                               buffer.data_ptr() + case.get("offset", 0), d_out_flags=d_flags)
        assert error.value.status == 1, case             # ACLB200_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    clipset.release()
    scalar.release()
