"""aclb200_decompress_tracks_skinning, _additive_skinning, _blend_skinning and aclb200_local_to_skinning: the matrix walk of the object
space decodes, then rtm::matrix_mul(inverse_bind, object) per bone, stored as three float4 rows (row c = x_axis[c], y_axis[c], z_axis[c],
w_axis[c]). Against
  * the port (oracle/skinning_oracle.c, pinned to the reference by tests/test_skinning_oracle.py): BIT FOR BIT;
  * the port's skinning step applied to the ACLB200_OBJECT_MATRIX3X4F rows the existing entry points write for the same requests: BIT FOR
    BIT, for all three composed routes (this checks the skinning step independently of any reference);
  * the reference itself where oracle/_ref exists: bit for bit on the plain decode and on the additive bones whose chain takes no negative
    scale `relative` product, within gates elsewhere;
  * decompress_tracks followed by aclb200_local_to_skinning at the C2 launch size: byte for byte.
Skeletons with more than 32 bones put children in a later chunk of 32 than their parents, so skinning a chunk before the whole walk ends
shows up as a mismatch.
"""
import numpy as np
import pytest

from oracle import object_space, skinning
from tests import additive_cases, blend_cases, clips
from tests import database_cases as dbcases
from tests import skinning_cases as cases

pytestmark = pytest.mark.gpu
LANES = clips.DEFINED_LANES
ROOT = cases.ROOT
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)
SENTINEL = 0x7FC00001


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


def _out(gpu, n, width):
    return gpu["torch"].full((n, width), SENTINEL, dtype=gpu["torch"].int32, device="cuda")


def _host(gpu, d_out):
    gpu["torch"].cuda.synchronize()
    return d_out.cpu().numpy().view(np.float32)


def _skin(gpu, clipset, requests, options, parents, inverse, offsets=None, flags=None, route="plain", **kw):
    """one skinning launch of `route` (plain, additive, blend) into a sentinel filled buffer, rows [n][max_tracks * 12] float32"""
    ctx = gpu["ctx"]
    n = len(requests)
    d_out = _out(gpu, n, clipset.max_tracks * 12)
    call = dict(plain=ctx.decompress_tracks_skinning, additive=ctx.decompress_tracks_additive_skinning, blend=ctx.decompress_tracks_blend_skinning)[route]
    call(clipset, _dev(gpu, requests), n, options, _dev(gpu, parents), _dev(gpu, inverse), d_out,
         d_skeleton_offsets=None if offsets is None else _dev(gpu, offsets), d_out_flags=flags, **kw)
    return _host(gpu, d_out)


def _matrix(gpu, clipset, requests, options, parents, offsets=None, flags=None, route="plain", **kw):
    """the same requests through the existing entry point with ACLB200_OBJECT_MATRIX3X4F"""
    ab, ctx = gpu["ab"], gpu["ctx"]
    n = len(requests)
    d_out = _out(gpu, n, clipset.max_tracks * 12)
    d_parents = _dev(gpu, parents)
    d_offsets = None if offsets is None else _dev(gpu, offsets)
    if route == "plain":
        ctx.decompress_tracks_object_space(clipset, _dev(gpu, requests), n, options, d_parents, ab.OBJECT_MATRIX3X4F, d_out,
                                           d_skeleton_offsets=d_offsets, d_out_flags=flags)
    else:
        call = ctx.decompress_tracks_additive if route == "additive" else ctx.decompress_tracks_blend
        call(clipset, _dev(gpu, requests), n, options, d_out, d_parent_indices=d_parents, kind=ab.OBJECT_MATRIX3X4F,
             d_skeleton_offsets=d_offsets, d_out_flags=flags, **kw)
    return _host(gpu, d_out)


def _rigs(names, kinds, seed):
    """a skeleton and random (every other clip: mirrored) inverse binds per clip, concatenated, with their offsets"""
    counts = [clips.TRANSFORM_SPECS[n].num_tracks if n in clips.TRANSFORM_SPECS else n for n in names]
    skeletons = [cases.skeleton(k, c, seed=seed + i) for i, (k, c) in enumerate(zip(kinds, counts))]
    inverses = [cases.random_affine(c, seed + 50 + i, mirrored=i % 2 == 1) for i, c in enumerate(counts)]
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    return skeletons, inverses, offsets, np.concatenate(skeletons), np.concatenate(inverses)


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_plain_decode_matches_the_port(gpu, name):
    """Every settings kind, every rounding and looping policy (per request where the settings allow it, batch wide with per track
    rounding), a variable bind pose; the random skeleton with mirrored inverse binds. The rows also equal the port's skinning step on the
    MATRIX3X4F rows of aclb200_decompress_tracks_object_space."""
    ab, port = gpu["ab"], gpu["port"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = gpu["ctx"].upload([blob], check_hash=True)
    parents = cases.skeleton("random", spec.num_tracks, seed=spec.seed)
    inverse = cases.random_affine(spec.num_tracks, spec.seed, mirrored=True)
    times = clips.sample_times(spec)[::2]
    pairs = [(r, l) for r in range(4) for l in range(3)]
    rng = np.random.default_rng(spec.seed)
    variable = np.tile(IDENTITY, (spec.num_tracks, 1))
    variable[:, 4:7] = rng.uniform(-2, 2, (spec.num_tracks, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (spec.num_tracks, 3))
    d_variable = gpu["torch"].from_numpy(variable).cuda()
    for kind, extra in [(kind, False) for kind in range(6)] + [(0, True)]:
        settings = port.settings_for_kind(kind, **(dict(default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable) if extra else {}))
        fields = dict(default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr()) if extra else {}
        launches = []
        if settings.c.per_track_rounding != 0:
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
            got = _skin(gpu, clipset, requests, options, parents, inverse).reshape(len(requests), -1, 12)
            matrix = _matrix(gpu, clipset, requests, options, parents).reshape(len(requests), -1, 12)
            for i, ((rounding, looping), t) in enumerate(zip(policy_list, request_times)):
                local = port.transform_decompress_tracks(blob, settings, float(t), int(rounding), int(looping))
                want = skinning.port_local_to_skinning(local, parents, inverse)
                assert clips.bit_equal(got[i], want), (name, kind, extra, rounding, looping, float(t))
                assert clips.bit_equal(skinning.port_skin_object_matrices(matrix[i], inverse), want), (name, kind, rounding, looping)
    clipset.release()


@pytest.mark.parametrize("name", ["c1_30bones", "mixed_scale", "stripped_single", "ragged_17", "paragon_like"])
def test_live_reference(gpu, name):
    """The reference's decode (debug settings, identity bind pose) taken through the reference metric's matrix walk and
    rtm::matrix_mul(inverse_bind, object): bit for bit, with bind pose inverses and mirrored random inverse binds."""
    from oracle import ref
    if not ref.available() or not skinning.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so and libaclref_skinning.so")
    torch, ab = gpu["torch"], gpu["ab"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    r = ref.transform_error(spec, blob, 1)
    clipset = gpu["ctx"].upload([blob])
    times = np.array([min(np.float32(s) / np.float32(r["sample_rate"]), np.float32(r["duration"])) for s in range(spec.num_samples)], np.float32)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_identity = torch.from_numpy(np.tile(IDENTITY, (spec.num_tracks, 1))).cuda()
    options = _options(gpu, 1, rounding_policy=r["rounding"], default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_identity.data_ptr())
    for kind in ("bind", "mirrored"):
        inverse = cases.inverse_binds(kind, spec.num_tracks, r["lossy_poses"][0], r["parents"], seed=spec.seed)
        got = _skin(gpu, clipset, requests, options, r["parents"], inverse).reshape(len(times), -1, 12)
        for s in range(spec.num_samples):
            assert clips.bit_equal(got[s], skinning.reference_local_to_skinning(r["lossy_poses"][s], r["parents"], inverse)), (name, kind, s)
    clipset.release()


def test_additive_route(gpu):
    """Every additive format and golden combo: bit for bit against the port's apply_additive_to_base + skinning and against the port's
    skinning step on the MATRIX3X4F rows of aclb200_decompress_tracks_additive (same flags); against the reference bit for bit on every
    bone whose chain takes no negative scale `relative` product, elsewhere within the additive tests' 1e-5 gate carried through the walk
    (times 8) and scaled by the rows' magnitude."""
    from oracle import additive, port as port_module, ref
    ab, torch, ctx, port = gpu["ab"], gpu["torch"], gpu["ctx"], gpu["port"]
    blobs = [additive_cases.load(n) for n in additive_cases.NAMES]
    clipset = ctx.upload(blobs, check_hash=True)
    n = additive_cases.BASE_SPEC.num_tracks
    parents = cases.skeleton("random", n, seed=3)
    inverse = cases.random_affine(n, 7, mirrored=True)
    pairs = additive_cases.time_pairs()[::3]
    live = ref.available() and skinning.reference_available() and additive.reference_available()
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_matrix_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for additive_name, format_ in additive_cases.FORMATS.items():
        additive_clip = additive_cases.NAMES.index(additive_name)
        requests = ab.make_additive_requests(np.zeros(len(pairs)), pairs[:, 0], np.full(len(pairs), additive_clip), pairs[:, 1])
        for kind, rounding, looping in additive_cases.COMBOS:
            options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping)
            got = _skin(gpu, clipset, requests, options, parents, inverse, flags=d_flags, route="additive", additive_format=format_).reshape(len(pairs), -1, 12)
            matrix = _matrix(gpu, clipset, requests, options, parents, flags=d_matrix_flags, route="additive", additive_format=format_).reshape(len(pairs), -1, 12)
            assert int(d_flags.item()) == int(d_matrix_flags.item()), (additive_name, kind)
            base_settings = port.settings_for_kind(kind)
            additive_settings = additive_cases.writer_settings(port, kind)
            for i, (tb, ta) in enumerate(pairs):
                local = additive_cases.port_pose(port, format_, blobs[0], blobs[additive_clip], tb, ta, base_settings, additive_settings, rounding,
                                                 looping, port_module.NORMALIZE_IEEE)
                want = skinning.port_local_to_skinning(local, parents, inverse)
                assert clips.bit_equal(got[i, :n], want), (additive_name, kind, rounding, looping, i)
                assert clips.bit_equal(skinning.port_skin_object_matrices(matrix[i, :n], inverse), want), (additive_name, kind, i)
                if not live:
                    continue
                reference = skinning.reference_local_to_skinning(
                    additive_cases.reference_pose(additive, format_, blobs[0], blobs[additive_clip], tb, ta, kind, rounding, looping), parents, inverse)
                base = port.transform_decompress_tracks(blobs[0], base_settings, float(tb), rounding, looping)
                extra = port.transform_decompress_tracks(blobs[additive_clip], additive_settings, float(ta), rounding, looping)
                negative = (format_ == ab.ADDITIVE_RELATIVE) & (np.minimum(base[:, 8:11], extra[:, 8:11]) < 0).any(axis=1)
                for bone in range(n):             # a bone inherits its ancestors' negative products
                    if parents[bone] != ROOT:
                        negative[bone] |= negative[parents[bone]]
                assert clips.bit_equal(got[i, :n][~negative], reference[~negative]), (additive_name, kind, i)
                gate = 8 * 1e-5 * (1.0 + np.abs(reference).max())
                assert float(np.max(np.abs(got[i, :n] - reference), initial=0.0)) <= gate, (additive_name, kind, i)
    clipset.release()


def test_blend_route(gpu):
    """Per pair weights over the golden combos: bit for bit against the port's IEEE qvv_lerp + skinning and against the port's skinning
    step on the MATRIX3X4F rows of aclb200_decompress_tracks_blend; against the reference within the blend tests' 1e-6 rotation gate,
    carried through a 24 bone walk (times 64) and scaled by the rows' magnitude."""
    from oracle import blend, ref
    ab, torch, ctx, port = gpu["ab"], gpu["torch"], gpu["ctx"], gpu["port"]
    blobs = [blend_cases.load(n) for n in blend_cases.NAMES]
    clipset = ctx.upload(blobs, check_hash=True)
    n = blend_cases.FROM_SPEC.num_tracks
    parents = cases.skeleton("chain", n)
    inverse = cases.random_affine(n, 8, mirrored=True)
    pairs = blend_cases.time_pairs()
    weights = np.resize(blend_cases.WEIGHTS, len(pairs)).astype(np.float32)
    d_weights = torch.from_numpy(weights).cuda()
    requests = ab.make_blend_requests(np.zeros(len(pairs)), pairs[:, 0], np.ones(len(pairs)), pairs[:, 1])
    live = ref.available() and skinning.reference_available() and blend.reference_available()
    for kind, rounding, looping in blend_cases.COMBOS:
        options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping)
        got = _skin(gpu, clipset, requests, options, parents, inverse, route="blend", d_weights=d_weights).reshape(len(pairs), -1, 12)
        matrix = _matrix(gpu, clipset, requests, options, parents, route="blend", d_weights=d_weights).reshape(len(pairs), -1, 12)
        for i, (tf, tt) in enumerate(pairs):
            local = blend_cases.port_pose(port, blend, blobs[0], blobs[1], tf, tt, weights[i], port.settings_for_kind(kind), rounding, looping,
                                          blend.NORMALIZE_IEEE)
            want = skinning.port_local_to_skinning(local, parents, inverse)
            assert clips.bit_equal(got[i, :n], want), (kind, rounding, looping, i)
            assert clips.bit_equal(skinning.port_skin_object_matrices(matrix[i, :n], inverse), want), (kind, i)
            if live:
                reference = skinning.reference_local_to_skinning(
                    blend_cases.reference_pose(blend, blobs[0], blobs[1], tf, tt, weights[i], kind, rounding, looping), parents, inverse)
                gate = 64 * blend_cases.ROTATION_GATE * (1.0 + np.abs(reference).max())
                assert float(np.max(np.abs(got[i, :n] - reference))) <= gate, (kind, rounding, looping, i)
    clipset.release()


def test_mixed_rigs_and_untouched_bytes(gpu):
    """One ragged clip set with a skeleton and inverse binds per clip (d_skeleton_offsets), invalid clip indices, a padded stride and an
    output pointer 16 bytes into its allocation: rows equal the port, every byte no request may write keeps its sentinel."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    names = ["c1_30bones", "ragged_17", "mixed_scale", "one_bone", "c2_100bones", "single_segment"]
    kinds = ["chain", "tree", "star", "random", "random", "chain"]
    skeletons, inverses, offsets, parents, inverse = _rigs(names, kinds, 11)
    blobs = [clips.load_blob(n) for n in names]
    clipset = ctx.upload(blobs, check_hash=True)
    rng = np.random.default_rng(11)
    num_requests = 300
    req_clip = rng.integers(0, len(names), num_requests).astype(np.uint32)
    req_clip[rng.random(num_requests) < 0.08] = len(names)
    req_clip[7] = 0xFFFFFFFF
    req_time = rng.uniform(-0.2, 2.5, num_requests).astype(np.float32)
    requests = ab.make_requests(req_clip, req_time)
    stride = clipset.max_tracks * 48 + 32
    lead = 16
    buffer = torch.full((lead + stride * num_requests + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    d_flags = torch.full((1,), 0x7F, dtype=torch.int32, device="cuda")
    ctx.decompress_tracks_skinning(clipset, _dev(gpu, requests), num_requests, ab.Options(pose_stride_bytes=stride), _dev(gpu, parents),
                                   _dev(gpu, inverse), buffer.data_ptr() + lead, d_skeleton_offsets=_dev(gpu, offsets), d_out_flags=d_flags)
    torch.cuda.synchronize()
    raw = buffer.cpu().numpy()
    assert int(d_flags.item()) == 0
    assert (raw[:lead] == 0xA5).all() and (raw[lead + stride * num_requests:] == 0xA5).all()
    settings = port.settings_for_kind(0)
    for i in range(num_requests):
        row = raw[lead + i * stride:lead + (i + 1) * stride]
        c = int(req_clip[i])
        if c >= len(names):
            assert (row == 0xA5).all(), i
            continue
        n = clips.TRANSFORM_SPECS[names[c]].num_tracks
        assert (row[n * 48:] == 0xA5).all(), i
        local = port.transform_decompress_tracks(blobs[c], settings, float(req_time[i]))
        got = row[:n * 48].copy().view(np.float32).reshape(n, 12)
        assert clips.bit_equal(got, skinning.port_local_to_skinning(local, skeletons[c], inverses[c])), (names[c], kinds[c], i)
    clipset.release()


def test_invalid_pairs_write_nothing(gpu):
    """Additive and blend pairs naming an invalid clip or clips of different track counts write nothing; the others their rows only."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    names = ["c1_30bones", "c2_100bones", "ragged_17"]
    blobs = [clips.load_blob(n) for n in names]
    clipset = ctx.upload(blobs)
    skeletons, inverses, offsets, parents, inverse = _rigs(names, ["tree", "random", "chain"], 21)
    clip_pairs = [(0, 0), (1, 1), (0, 1), (2, 9), (9, 2), (2, 2), (1, 0)]
    times = [(0.1 * i, 0.05 * i + 0.02) for i in range(len(clip_pairs))]
    settings = port.settings_for_kind(0)
    writer = additive_cases.writer_settings(port, 0)
    for route in ("additive", "blend"):
        make = ab.make_additive_requests if route == "additive" else ab.make_blend_requests
        requests = make([a for a, _ in clip_pairs], [t for t, _ in times], [b for _, b in clip_pairs], [t for _, t in times])
        extra = dict(additive_format=ab.ADDITIVE_ADDITIVE0) if route == "additive" else dict(weight=0.3)
        got = _skin(gpu, clipset, requests, ab.Options(), parents, inverse, offsets=offsets, route=route, **extra)
        for i, (a, b) in enumerate(clip_pairs):
            row = got[i].view(np.uint32)
            if a != b:
                assert (row == SENTINEL).all(), (route, i)
                continue
            n = clips.TRANSFORM_SPECS[names[a]].num_tracks
            first = port.transform_decompress_tracks(blobs[a], settings, float(times[i][0]))
            if route == "additive":
                local = port.apply_additive_to_base(ab.ADDITIVE_ADDITIVE0, first,
                                                    port.transform_decompress_tracks(blobs[b], writer, float(times[i][1])), port.NORMALIZE_IEEE)
            else:
                from oracle import blend
                local = blend.port_qvv_lerp(first, port.transform_decompress_tracks(blobs[b], settings, float(times[i][1])), 0.3)
            assert clips.bit_equal(got[i, :n * 12].reshape(n, 12), skinning.port_local_to_skinning(local, skeletons[a], inverses[a])), (route, i)
            assert (row[n * 12:] == SENTINEL).all(), (route, i)
    clipset.release()


def test_flags(gpu):
    """A parent after its child is reported and the bone taken as a root; mirrored bind pose scales take no branch of the matrix walk
    and raise nothing."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = ctx.upload([blob])
    times = clips.sample_times(spec)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    parents = cases.skeleton("tree", spec.num_tracks)
    inverse = cases.random_affine(spec.num_tracks, 4)
    bad, as_root = parents.copy(), parents.copy()
    bad[40], as_root[40] = 45, ROOT
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    settings = port.settings_for_kind(0)
    got = _skin(gpu, clipset, requests, ab.Options(), bad, inverse, flags=d_flags).reshape(len(times), -1, 12)
    assert int(d_flags.item()) == ab.ERROR_FLAG_INVALID_SKELETON
    for i, t in enumerate(times):
        assert clips.bit_equal(got[i], skinning.port_local_to_skinning(port.transform_decompress_tracks(blob, settings, float(t)), as_root, inverse))

    variable = np.tile(IDENTITY, (spec.num_tracks, 1))
    variable[::3, 8] = -1.0
    d_variable = torch.from_numpy(variable).cuda()
    mirrored = port.settings_for_kind(0, default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable)
    options = ab.Options(default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
    got = _skin(gpu, clipset, requests, options, parents, inverse, flags=d_flags).reshape(len(times), -1, 12)
    assert int(d_flags.item()) == 0
    for i, t in enumerate(times):
        local = port.transform_decompress_tracks(blob, mirrored, float(t))
        assert local[:, 8].min() < 0.0
        assert clips.bit_equal(got[i], skinning.port_local_to_skinning(local, parents, inverse)), float(t)
    clipset.release()


def test_database_tiers(gpu):
    """Every tier state of tests/golden/database_tiers.npz (or the live reference): the skinning rows of the reference's poses."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    ab, ctx = gpu["ab"], gpu["ctx"]
    reference = _Reference(ref, ref_database)
    clipset = ctx.upload(reference.bound + [reference.plain], check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in reference.bound + [reference.plain]]
    skeletons, inverses, offsets, parents, inverse = _rigs(counts, ["tree", "random", "chain", "random", "tree"], 31)
    req_clip = np.repeat(np.arange(5, dtype=np.uint32), len(dbcases.ALL_TIMES))
    req_time = np.tile(dbcases.ALL_TIMES, 5)
    requests = ab.make_requests(req_clip, req_time)
    done = []
    for state, ops in dbcases.STATES.items():
        for op, tier, count in ops[len(done):]:
            (database.stream_in if op == dbcases.IN else database.stream_out)(tier, count)
        done = ops
        got = _skin(gpu, clipset, requests, _options(gpu, 1), parents, inverse, offsets=offsets).reshape(len(requests), -1, 12)
        for i, (c, t) in enumerate(zip(req_clip, req_time)):
            local = reference.poses(state, int(c), t, 0, ab.LOOP_AS_COMPRESSED)
            n = local.shape[0]
            assert clips.bit_equal(got[i, :n], skinning.port_local_to_skinning(local, skeletons[c], inverses[c])), (state, int(c), float(t))
    clipset.release()


def test_wide_pose_limits(gpu):
    """wide_2500 (2500 bones, 120,000 bytes per QVV48 pose): one pose fits a block, so the plain skinning decode and the standalone call
    run and agree with the port; the two poses of an additive or blend pair do not fit and are refused, writing nothing."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    blob = clips.load_blob("wide_2500")
    clipset = ctx.upload([blob])
    n = 2500
    parents = cases.skeleton("random", n, seed=2)
    inverse = cases.random_affine(n, 2, mirrored=True)
    times = [0.05, 0.1333, 0.27]
    got = _skin(gpu, clipset, ab.make_requests([0, 0, 0], times), ab.Options(), parents, inverse).reshape(3, n, 12)
    d_local = torch.empty((3, n, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests([0, 0, 0], times)), 3, ab.Options(), d_local)
    ctx.local_to_skinning(d_local, d_local, 3, n, _dev(gpu, parents), _dev(gpu, inverse))
    standalone = _host(gpu, d_local.view(torch.int32)).reshape(3, n, 12)
    settings = port.settings_for_kind(0)
    for i, t in enumerate(times):
        want = skinning.port_local_to_skinning(port.transform_decompress_tracks(blob, settings, t), parents, inverse)
        assert clips.bit_equal(got[i], want) and clips.bit_equal(standalone[i], want), t
    for route, make in (("additive", ab.make_additive_requests), ("blend", ab.make_blend_requests)):
        d_out = _out(gpu, 3, n * 12)
        call = ctx.decompress_tracks_additive_skinning if route == "additive" else ctx.decompress_tracks_blend_skinning
        with pytest.raises(ab.api.AclB200Error) as error:
            call(clipset, _dev(gpu, make([0, 0, 0], times, [0, 0, 0], times[::-1])), 3, ab.Options(), _dev(gpu, parents), _dev(gpu, inverse), d_out)
        assert error.value.status == 3, route            # ACLB200_ERR_UNSUPPORTED
        assert (_host(gpu, d_out).view(np.uint32) == SENTINEL).all(), route
    clipset.release()


def test_refusals_write_nothing(gpu):
    """Every refusal of the four entry points returns before the flags are cleared: neither the output nor the flags change. A launch that
    would keep the caller's bytes (skip masks, a `skipped` default mode) is refused with a message that names the entry point called."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")])
    scalar = ctx.upload([clips.load_blob("float1")])
    plain_requests = _dev(gpu, ab.make_requests(np.zeros(8, np.uint32), np.linspace(0, 1, 8).astype(np.float32)))
    pair_requests = _dev(gpu, ab.make_blend_requests(np.zeros(8), np.linspace(0, 1, 8), np.zeros(8), np.linspace(1, 0, 8)))
    parents = _dev(gpu, cases.skeleton("tree", 30))
    inverse = _dev(gpu, np.concatenate([cases.random_affine(30, 1).reshape(-1), np.zeros(4, np.float32)]))
    aligned = inverse.data_ptr()
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    keeps_bytes = "the composed poses need every decoded sub-track (no skip masks, no `skipped` default mode)"
    decode_refusals = [
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE), message=keeps_bytes),
        dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr()), message=keeps_bytes),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY)), message=keeps_bytes),
        dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(parents=0),
        dict(inverse=0),
        dict(inverse=inverse.data_ptr() + 8),
        dict(clipset=scalar),
        dict(offset=8),
    ]
    routes = [("decompress_tracks_skinning", ctx.decompress_tracks_skinning, plain_requests, {}),
              ("decompress_tracks_additive_skinning", ctx.decompress_tracks_additive_skinning, pair_requests, dict(additive_format=1)),
              ("decompress_tracks_blend_skinning", ctx.decompress_tracks_blend_skinning, pair_requests, dict(weight=0.5))]
    cases_ = [(route, case) for route in routes for case in decode_refusals]
    cases_.append((routes[1][:3] + (dict(additive_format=4),), {}))
    for (route, call, requests, extra), case in cases_:
        buffer = torch.full((8 * 30 * 48 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            call(case.get("clipset", clipset), requests, 8, case.get("options", ab.Options()), case.get("parents", parents),
                 case.get("inverse", aligned), buffer.data_ptr() + case.get("offset", 0), d_out_flags=d_flags, **extra)
        assert error.value.status == 1, (route, case, extra)      # ACLB200_ERR_INVALID_ARGUMENT
        if "message" in case:
            assert str(error.value).endswith(f"{route}: {case['message']}"), (route, str(error.value))
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), (route, case)
        assert int(d_flags.item()) == 0x5A5A5A5A, (route, case)

    local = torch.zeros((8, 30, 12), dtype=torch.float32, device="cuda")
    standalone_refusals = [dict(local=0), dict(out=0), dict(parents=0), dict(inverse=0), dict(inverse=inverse.data_ptr() + 8),
                           dict(out=local.data_ptr() + 8), dict(stride=30 * 48 + 8), dict(stride=29 * 48)]
    for case in standalone_refusals:
        out = torch.full((8 * 30 * 48 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.local_to_skinning(case.get("local", local.data_ptr()), case.get("out", out.data_ptr()), 2, 30, case.get("parents", parents),
                                  case.get("inverse", aligned), pose_stride_bytes=case.get("stride", 0), d_out_flags=d_flags)
        assert error.value.status == 1, case
        torch.cuda.synchronize()
        assert (out.cpu().numpy() == 0x5A).all() and not local.any(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    clipset.release()
    scalar.release()


def test_standalone_equals_the_fused_route(gpu):
    """decompress_tracks + aclb200_local_to_skinning, into another buffer with a padded stride and in place, equals the fused call byte for
    byte on a > 32 bone clip with a random skeleton, and reports the same flags."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = ctx.upload([clips.load_blob(name)])
    n = spec.num_tracks
    parents = cases.skeleton("random", n, seed=8)
    parents[50] = 52                      # reported, taken as a root by both routes
    inverse = cases.random_affine(n, 8, mirrored=True)
    times = np.resize(clips.sample_times(spec), 333).astype(np.float32)
    requests = ab.make_requests(np.zeros(times.size, np.uint32), times)
    stride = n * 48 + 48
    options = ab.Options(pose_stride_bytes=stride)
    d_flags = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(3)]
    fused = torch.full((times.size, stride // 4), SENTINEL, dtype=torch.int32, device="cuda")
    ctx.decompress_tracks_skinning(clipset, _dev(gpu, requests), times.size, options, _dev(gpu, parents), _dev(gpu, inverse), fused,
                                   d_out_flags=d_flags[0])
    local = torch.full_like(fused, SENTINEL)
    ctx.decompress_tracks(clipset, _dev(gpu, requests), times.size, options, local)
    other = torch.full_like(fused, SENTINEL)
    ctx.local_to_skinning(local, other, times.size, n, _dev(gpu, parents), _dev(gpu, inverse), pose_stride_bytes=stride, d_out_flags=d_flags[1])
    ctx.local_to_skinning(local, local, times.size, n, _dev(gpu, parents), _dev(gpu, inverse), pose_stride_bytes=stride, d_out_flags=d_flags[2])
    torch.cuda.synchronize()
    assert torch.equal(fused, other) and torch.equal(fused, local)
    assert [int(f.item()) for f in d_flags] == [ab.ERROR_FLAG_INVALID_SKELETON] * 3
    clipset.release()


def test_c2_launch_composes_the_two_calls(gpu):
    """The C2 bench workload in one launch (600,000 requests x 100 bones, binary tree skeleton, bind pose inverses): byte for byte what
    decompress_tracks followed by aclb200_local_to_skinning writes."""
    import bench
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    from oracle import ref
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    n, bones = int(w["req_clip"].size), w["num_tracks"]
    assert n == 600000 and bones == 100
    parents = cases.skeleton("tree", bones)
    first = int(w["offsets"][0])
    blob = ref.aligned_blob(w["buffer"][first:first + int(w["sizes"][0])].tobytes())
    inverse = cases.bind_inverse(port.transform_decompress_tracks(blob, port.settings_for_kind(0), 0.0), parents)
    d_parents, d_inverse = _dev(gpu, parents), _dev(gpu, inverse)
    d_requests = _dev(gpu, ab.make_requests(w["req_clip"], w["req_time"]))
    options = ab.Options()
    d_two_step = torch.empty((n, bones, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n, options, d_two_step)
    ctx.local_to_skinning(d_two_step, d_two_step, n, bones, d_parents, d_inverse)
    d_fused = torch.full_like(d_two_step, float("nan"))
    ctx.decompress_tracks_skinning(clipset, d_requests, n, options, d_parents, d_inverse, d_fused)
    torch.cuda.synchronize()
    assert torch.equal(d_fused.view(torch.int32), d_two_step.view(torch.int32))
    clipset.release()
