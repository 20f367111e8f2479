"""aclb200_decompress_bones: chosen bones of each pose, against the library's own whole-pose decodes gathered at the listed bones.

  * local rows: byte for byte the rows of aclb200_decompress_tracks (the lanes of clips.DEFINED_LANES for QVV48, all 40 bytes for QVV40);
  * object rows: all 48 bytes of the rows of aclb200_decompress_tracks_object_space, qvvf and matrix;
  * every row a query may not write (NO_BONE entries, bones beyond the clip, requests with an invalid clip or list, padding, the bytes
    around the output) keeps its sentinel.
Both whole-pose decodes are pinned to the oracle and the reference by their own tests (test_gpu_parity.py, test_gpu_object_space.py);
tests/test_bones_oracle.py pins the closure rule to the oracle.
"""
import numpy as np
import pytest

from tests import bones_cases as cases
from tests import clips

pytestmark = pytest.mark.gpu
LANES = clips.DEFINED_LANES
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)
SENTINEL = 0xA5
LOCAL48, LOCAL40, QVVF, MATRIX = "local48", "local40", "qvvf", "matrix"
MODES = [LOCAL48, LOCAL40, QVVF, MATRIX]


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    return dict(torch=torch, ab=ab, port=port, ctx=ab.Context(0))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8)).cuda()


def _options(gpu, kind, mode, **kw):
    ab = gpu["ab"]
    s = gpu["port"].settings_for_kind(kind).c
    fields = dict(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                  clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                  default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                  constant_defaults=list(s.constant_defaults), output_layout=ab.LAYOUT_QVV40 if mode == LOCAL40 else ab.LAYOUT_QVV48)
    fields.update(kw)
    return ab.Options(**fields)


def _bone_bytes(mode):
    return 40 if mode == LOCAL40 else 48


def _object_kind(gpu, mode):
    return gpu["ab"].OBJECT_MATRIX3X4F if mode == MATRIX else gpu["ab"].OBJECT_QVVF


def full_rows(gpu, clipset, d_requests, num_requests, options, mode, d_parents=None, d_offsets=None, d_flags=None):
    """[num_requests][max_tracks][bone bytes] uint8: the whole-pose decode the query gathers from"""
    torch, ctx = gpu["torch"], gpu["ctx"]
    bone = _bone_bytes(mode)
    d_out = torch.zeros((num_requests, clipset.max_tracks * bone), dtype=torch.uint8, device="cuda")
    full_options = gpu["ab"].Options()
    for field, _ in type(options)._fields_:
        setattr(full_options, field, getattr(options, field))
    full_options.pose_stride_bytes = 0
    if mode in (LOCAL48, LOCAL40):
        ctx.decompress_tracks(clipset, d_requests, num_requests, full_options, d_out)
    else:
        ctx.decompress_tracks_object_space(clipset, d_requests, num_requests, full_options, d_parents, _object_kind(gpu, mode), d_out,
                                           d_skeleton_offsets=d_offsets, d_out_flags=d_flags)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().reshape(num_requests, clipset.max_tracks, bone)


def query(gpu, clipset, d_requests, num_requests, options, mode, lists, request_lists=None, d_parents=None, d_offsets=None, d_flags=None,
          stride=0, lead=0, num_lists=None):
    """Runs the query into a sentinel-filled buffer; returns (the buffer's bytes, the stride used)"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    lists = np.asarray(lists, np.uint32).reshape(len(lists), -1)
    k = lists.shape[1]
    pose_stride = stride or k * _bone_bytes(mode)
    buffer = torch.full((lead + pose_stride * num_requests + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    options.pose_stride_bytes = stride
    ctx.decompress_bones(clipset, d_requests, num_requests, options, _dev(gpu, lists), k, buffer.data_ptr() + lead,
                         num_lists=len(lists) if num_lists is None else num_lists,
                         d_request_lists=None if request_lists is None else _dev(gpu, np.asarray(request_lists, np.uint32)),
                         d_parent_indices=None if mode in (LOCAL48, LOCAL40) else d_parents,
                         kind=_object_kind(gpu, mode), d_skeleton_offsets=d_offsets, d_out_flags=d_flags)
    torch.cuda.synchronize()
    return buffer.cpu().numpy(), pose_stride


def check(got_bytes, pose_stride, full, mode, lists, request_lists, num_tracks_of, lead=0, num_lists=None, context=()):
    """Every row of every request: the gathered whole-pose row, or the sentinel; every other byte of the buffer the sentinel"""
    lists = np.asarray(lists, np.uint32).reshape(len(lists), -1)
    num_lists = len(lists) if num_lists is None else num_lists
    k = lists.shape[1]
    bone = _bone_bytes(mode)
    n = full.shape[0]
    assert (got_bytes[:lead] == SENTINEL).all() and (got_bytes[lead + pose_stride * n:] == SENTINEL).all(), context
    for r in range(n):
        row = got_bytes[lead + r * pose_stride:lead + (r + 1) * pose_stride]
        assert (row[k * bone:] == SENTINEL).all(), (context, r)
        li = 0 if request_lists is None else int(request_lists[r])
        tracks = num_tracks_of(r)
        for j in range(k):
            got = row[j * bone:(j + 1) * bone]
            bone_index = int(lists[li, j]) if li < num_lists else 0xFFFFFFFF
            if li >= num_lists or tracks == 0 or bone_index >= tracks:
                assert (got == SENTINEL).all(), (context, r, j)
                continue
            want = full[r, bone_index]
            if mode == LOCAL48:
                assert clips.bit_equal(got.view(np.float32)[LANES], want.view(np.float32)[LANES]), (context, r, j, bone_index)
            else:
                assert (got == want).all(), (context, r, j, bone_index)


def _single_clip_tracks(n):
    return lambda r: n


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_named_clips_every_setting(gpu, name):
    """Every named clip x every settings kind x rounding and looping (per request, or batch wide with per track rounding) x variable
    defaults, local QVV48 and QVV40 rows, qvvf and matrix rows on a binary tree; three lists in one launch, picked per request."""
    ab, torch = gpu["ab"], gpu["torch"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = gpu["ctx"].upload([blob], check_hash=True)
    n = spec.num_tracks
    d_parents = _dev(gpu, cases.tree(n))
    named = cases.bone_lists(n, seed=spec.seed)
    lists = cases.pad_lists([named["leaves"], named["duplicates_reversed"], named["holes"]], 5)
    times = clips.sample_times(spec)[::2]
    pairs = [(r, l) for r in range(4) for l in range(3)]
    rng = np.random.default_rng(spec.seed)
    variable = np.tile(IDENTITY, (n, 1))
    variable[:, 4:7] = rng.uniform(-2, 2, (n, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (n, 3))
    d_variable = torch.from_numpy(variable).cuda()
    for kind, extra in [(kind, False) for kind in range(6)] + [(0, True)]:
        fields = dict(default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr()) if extra else {}
        per_track = gpu["port"].settings_for_kind(kind).c.per_track_rounding != 0
        if per_track:
            launches = [(dict(rounding_policy=r, looping_policy=l), None) for r, l in pairs]
        else:
            policies = np.array([p for p in pairs for _ in times], np.uint8)
            d_policies = _dev(gpu, policies)
            launches = [(dict(d_request_policies=d_policies.data_ptr()), d_policies)]
        for policy_fields, keep_alive in launches:
            num_requests = len(times) * (1 if per_track else len(pairs))
            requests = ab.make_requests(np.zeros(num_requests, np.uint32), np.resize(times, num_requests))
            d_requests = _dev(gpu, requests)
            request_lists = np.arange(num_requests, dtype=np.uint32) % len(lists)
            for mode in MODES:
                options = _options(gpu, kind, mode, **policy_fields, **fields)
                full = full_rows(gpu, clipset, d_requests, num_requests, options, mode, d_parents)
                got, stride = query(gpu, clipset, d_requests, num_requests, options, mode, lists, request_lists, d_parents)
                check(got, stride, full, mode, lists, request_lists, _single_clip_tracks(n), context=(name, kind, extra, policy_fields, mode))
            del keep_alive
    clipset.release()


@pytest.mark.parametrize("name", ["c1_30bones", "c2_100bones", "mixed_scale", "paragon_like"])
@pytest.mark.parametrize("skeleton", cases.SKELETONS)
def test_lists_and_skeletons(gpu, name, skeleton):
    """Each named list on its own (root only, one deep leaf, 4 leaves, K = 32, every bone of a clip of at most 32 bones, duplicates and
    reversed order, NO_BONE holes, bones beyond the clip) on a chain, star, tree, random multi-root skeleton and one with parents after
    their children: the flags are those of the walked bones."""
    ab, torch = gpu["ab"], gpu["torch"]
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = spec.num_tracks
    parents = cases.skeleton(skeleton, n, seed=spec.seed)
    d_parents = _dev(gpu, parents)
    times = clips.sample_times(spec)
    requests = ab.make_requests(np.zeros(len(times), np.uint32), times)
    d_requests = _dev(gpu, requests)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for list_name, bones in cases.bone_lists(n, seed=spec.seed).items():
        walked = cases.closure(parents, bones, n)
        bad = any(parents[b] != cases.ROOT and parents[b] >= b for b in walked)
        for mode in MODES:
            options = _options(gpu, 0, mode)
            full = full_rows(gpu, clipset, d_requests, len(times), options, mode, d_parents)
            got, stride = query(gpu, clipset, d_requests, len(times), options, mode, [bones], None, d_parents, d_flags=d_flags)
            check(got, stride, full, mode, [bones], None, _single_clip_tracks(n), context=(name, skeleton, list_name, mode))
            want_flags = ab.ERROR_FLAG_INVALID_SKELETON if bad and mode in (QVVF, MATRIX) else 0
            assert int(d_flags.item()) == want_flags, (name, skeleton, list_name, mode)
    clipset.release()


def test_mirrored_bones(gpu):
    """A mirrored bone (a negative default scale) takes qvv_mul's matrix branch: NEGATIVE_SCALE is reported when a chain holds it and
    not when only a bone outside every chain does; the rows equal the whole decode's either way."""
    ab, torch = gpu["ab"], gpu["torch"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = spec.num_tracks
    parents = cases.tree(n)
    d_parents = _dev(gpu, parents)
    times = clips.sample_times(spec)
    d_requests = _dev(gpu, ab.make_requests(np.zeros(len(times), np.uint32), times))
    leaves = [b for b in range(n) if 2 * b + 1 >= n]
    variable = np.tile(IDENTITY, (n, 1))
    variable[leaves, 8] = -1.0
    d_variable = torch.from_numpy(variable).cuda()
    probe = _options(gpu, 0, LOCAL48, default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
    local = full_rows(gpu, clipset, d_requests, len(times), probe, LOCAL48).view(np.float32)
    mirrored = [b for b in leaves if (local[:, b, 8] < 0).all()]
    plain = [b for b in leaves if (local[:, b, 8] > 0).all()]
    assert mirrored and plain
    variable = np.tile(IDENTITY, (n, 1))
    variable[mirrored[0], 8] = -1.0
    d_variable = torch.from_numpy(variable).cuda()
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for mode in (QVVF, MATRIX):
        options = _options(gpu, 0, mode, default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
        full = full_rows(gpu, clipset, d_requests, len(times), options, mode, d_parents, d_flags=d_flags)
        assert int(d_flags.item()) == (ab.ERROR_FLAG_NEGATIVE_SCALE if mode == QVVF else 0)
        for bones, flag in (([mirrored[0], plain[0]], ab.ERROR_FLAG_NEGATIVE_SCALE), ([plain[0], 0], 0)):
            got, stride = query(gpu, clipset, d_requests, len(times), options, mode, [bones], None, d_parents, d_flags=d_flags)
            check(got, stride, full, mode, [bones], None, _single_clip_tracks(n), context=(mode, bones))
            assert int(d_flags.item()) == (flag if mode == QVVF else 0), (mode, bones)
    clipset.release()


def test_mixed_rigs_lists_and_untouched_bytes(gpu):
    """A ragged clip set with a skeleton per clip (d_skeleton_offsets), a list per request (some list indices >= num_lists), invalid
    clips, a padded stride and an output 16 bytes into its allocation; 301 requests leave a partial last block."""
    ab, torch = gpu["ab"], gpu["torch"]
    names = ["c1_30bones", "ragged_17", "mixed_scale", "one_bone", "c2_100bones", "single_segment"]
    kinds = ["chain", "tree", "star", "random", "late", "chain"]
    specs = [clips.TRANSFORM_SPECS[n] for n in names]
    skeletons = [cases.skeleton(k, s.num_tracks, seed=i) for i, (k, s) in enumerate(zip(kinds, specs))]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in skeletons])[:-1]]).astype(np.uint32)
    clipset = gpu["ctx"].upload([clips.load_blob(n) for n in names], check_hash=True)
    rng = np.random.default_rng(11)
    num_requests = 301
    req_clip = rng.integers(0, len(names), num_requests).astype(np.uint32)
    req_clip[rng.random(num_requests) < 0.08] = len(names)
    req_clip[7] = 0xFFFFFFFF
    requests = ab.make_requests(req_clip, rng.uniform(-0.2, 2.5, num_requests).astype(np.float32))
    d_requests = _dev(gpu, requests)
    lists = cases.pad_lists([[0], [99, 16, 5, 56, 29], [3, cases.NO_BONE, 3, 40, 0], list(range(0, 64, 2))], 32)
    request_lists = rng.integers(0, len(lists) + 2, num_requests).astype(np.uint32)     # some beyond num_lists
    request_lists[3] = 0xFFFFFFFF
    tracks = [specs[c].num_tracks if c < len(names) else 0 for c in req_clip]
    d_parents, d_offsets = _dev(gpu, np.concatenate(skeletons)), _dev(gpu, offsets)
    for mode in MODES:
        options = _options(gpu, 0, mode)
        full = full_rows(gpu, clipset, d_requests, num_requests, options, mode, d_parents, d_offsets)
        stride = 32 * _bone_bytes(mode) + 64
        got, stride = query(gpu, clipset, d_requests, num_requests, options, mode, lists, request_lists, d_parents, d_offsets, stride=stride,
                            lead=16)
        check(got, stride, full, mode, lists, request_lists, lambda r: tracks[r], lead=16, context=mode)
    clipset.release()


def test_wide_clip_and_partial_blocks(gpu):
    """wide_2500: one 2500-bone QVV48 pose per block still fits; a chain walk through every chunk of 32 bones; request counts around
    the block size."""
    ab = gpu["ab"]
    blob = clips.load_blob("wide_2500")
    clipset = gpu["ctx"].upload([blob])
    n = 2500
    for skeleton in ("tree", "chain", "random"):
        parents = cases.skeleton(skeleton, n, seed=3)
        d_parents = _dev(gpu, parents)
        lists = cases.pad_lists([[n - 1, 0, 1234, 2047], [17, 2499, cases.NO_BONE, 640]], 4)
        for num_requests in (1, 3, 10):
            times = np.linspace(0.0, 0.3, num_requests).astype(np.float32)
            d_requests = _dev(gpu, ab.make_requests(np.zeros(num_requests, np.uint32), times))
            request_lists = np.arange(num_requests, dtype=np.uint32) % 2
            for mode in MODES:
                options = _options(gpu, 0, mode)
                full = full_rows(gpu, clipset, d_requests, num_requests, options, mode, d_parents)
                got, stride = query(gpu, clipset, d_requests, num_requests, options, mode, lists, request_lists, d_parents)
                check(got, stride, full, mode, lists, request_lists, _single_clip_tracks(n), context=(skeleton, num_requests, mode))
    clipset.release()


def test_database_tiers(gpu):
    """Clip sets bound to a database, in every tier state of tests/database_cases.py: the rows of the whole decodes, which read the
    same streamed tiers."""
    from tests.test_gpu_database import _Reference
    from tests import database_cases as db_cases
    from oracle import ref, ref_database
    ab, ctx = gpu["ab"], gpu["ctx"]
    reference = _Reference(ref, ref_database)
    blobs = reference.bound + [reference.plain]
    clipset = ctx.upload(blobs, check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in blobs]
    skeletons = [cases.tree(c) for c in counts]
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    d_parents, d_offsets = _dev(gpu, np.concatenate(skeletons)), _dev(gpu, offsets)
    req_clip = np.repeat(np.arange(len(blobs), dtype=np.uint32), len(db_cases.ALL_TIMES))
    d_requests = _dev(gpu, ab.make_requests(req_clip, np.tile(db_cases.ALL_TIMES, len(blobs))))
    lists = cases.pad_lists([[min(counts) - 1, 0, 5], [1, 2, 3]], 3)
    request_lists = np.arange(req_clip.size, dtype=np.uint32) % 2
    done = []
    for state, ops in db_cases.STATES.items():
        for op, tier, n in ops[len(done):]:
            (database.stream_in if op == db_cases.IN else database.stream_out)(tier, n)
        done = ops
        for mode in MODES:
            options = _options(gpu, 1, mode)
            full = full_rows(gpu, clipset, d_requests, req_clip.size, options, mode, d_parents, d_offsets)
            got, stride = query(gpu, clipset, d_requests, req_clip.size, options, mode, lists, request_lists, d_parents, d_offsets)
            check(got, stride, full, mode, lists, request_lists, lambda r: counts[req_clip[r]], context=(state, mode))
    clipset.release()


def test_c2_full_size(gpu):
    """The C2 bench request list (600,000 requests, binary tree skeleton) with the 4-leaf list and a 32-bone list: the rows of the whole
    object space decode (qvvf, matrix) and of decompress_tracks, gathered and compared on the device."""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    n, bones = int(w["req_clip"].size), w["num_tracks"]
    assert n == 600000 and bones == 100
    d_parents = _dev(gpu, cases.tree(bones))
    d_requests = _dev(gpu, ab.make_requests(w["req_clip"], w["req_time"]))
    random32 = np.random.default_rng(5).integers(0, bones, 32).astype(np.uint32)
    for bone_list in (np.array(cases.C2_FOUR_LEAVES, np.uint32), random32):
        index = torch.from_numpy(bone_list.astype(np.int64)).cuda()
        d_list = _dev(gpu, bone_list)
        for mode in (QVVF, MATRIX, LOCAL48):
            d_full = torch.empty((n, bones, 12), dtype=torch.float32, device="cuda")
            if mode == LOCAL48:
                ctx.decompress_tracks(clipset, d_requests, n, ab.Options(), d_full)
            else:
                ctx.decompress_tracks_object_space(clipset, d_requests, n, ab.Options(), d_parents, _object_kind(gpu, mode), d_full)
            want = d_full[:, index].contiguous()
            del d_full
            d_got = torch.full((n, bone_list.size, 12), float("nan"), dtype=torch.float32, device="cuda")
            ctx.decompress_bones(clipset, d_requests, n, ab.Options(), d_list, bone_list.size, d_got,
                                 d_parent_indices=None if mode == LOCAL48 else d_parents, kind=_object_kind(gpu, mode))
            torch.cuda.synchronize()
            if mode == LOCAL48:
                lanes = torch.tensor(LANES, device="cuda")
                assert torch.equal(d_got[..., lanes].view(torch.int32), want[..., lanes].view(torch.int32)), (mode, bone_list.size)
            else:
                assert torch.equal(d_got.view(torch.int32), want.view(torch.int32)), (mode, bone_list.size)
            del want, d_got
    clipset.release()


def test_refusals_write_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")])
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_requests(np.zeros(8, np.uint32), np.linspace(0, 1, 8).astype(np.float32)))
    parents = _dev(gpu, cases.tree(30))
    lists = _dev(gpu, np.arange(32, dtype=np.uint32))
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    refusals = [
        (dict(k=0), 1), (dict(k=33), 1), (dict(num_lists=0), 1), (dict(lists=None), 1),
        (dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)), 1),
        (dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr())), 1),
        (dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))), 1),
        (dict(clipset=scalar), 1),
        (dict(kind=2), 1),
        (dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40)), 1),
        (dict(options=ab.Options(pose_stride_bytes=4 * 48 - 16)), 1),
        (dict(options=ab.Options(pose_stride_bytes=4 * 48 + 8)), 1),
        (dict(offset=8), 1),
        (dict(options=ab.Options(output_layout=ab.LAYOUT_QVV40), parents=None, offset=4), 1),
    ]
    for case, status in refusals:
        buffer = torch.full((8 * 32 * 48 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.decompress_bones(case.get("clipset", clipset), requests, 8, case.get("options", ab.Options()),
                                 case["lists"] if "lists" in case else lists, case.get("k", 4), buffer.data_ptr() + case.get("offset", 0),
                                 num_lists=case.get("num_lists", 1), d_parent_indices=case["parents"] if "parents" in case else parents,
                                 kind=case.get("kind", ab.OBJECT_QVVF), d_out_flags=d_flags)
        assert error.value.status == status, case
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    clipset.release()
    scalar.release()

