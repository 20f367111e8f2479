"""aclb200_extract_pose_features: all 48 bytes of every row against the port's composition (tests/features_cases.py, the IEEE flavour of
the CUDA path) of the library's own pieces for each (request, offset) pair with u' and c derived by features_cases.offset_time:
  B  the object rows of aclb200_decompress_bones at u' (the same parents, ACLB200_OBJECT_QVVF);
  T  the root's local row of aclb200_decompress_bones at u' (the root as the only listed bone, no parents);
  M  the row of aclb200_extract_root_motion for {clip, t, u', c}.
Those entry points are pinned by tests/test_gpu_bones.py and tests/test_gpu_root_motion.py; tests/test_features_oracle.py pins the
composition to the reference. Rows the launch may not write keep their sentinel, and so do the bytes around and between the rows."""
import numpy as np
import pytest

from oracle import root_motion as RM
from tests import bones_cases
from tests import clips
from tests import features_cases as cases
from tests.test_gpu_root_motion import durations

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5
NO_BONE = bones_cases.NO_BONE
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
    ab = gpu["ab"]
    s = gpu["port"].settings_for_kind(kind).c
    fields = dict(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                  clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                  default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                  constant_defaults=list(s.constant_defaults), looping_policy=ab.LOOP_CLAMP)
    fields.update(kw)
    return ab.Options(**fields)


class Launch:
    """One extract_pose_features launch and everything its expected rows need"""

    def __init__(self, gpu, clipset, requests, offsets, lists, parents, request_lists=None, roots=None, skeleton_offsets=None):
        self.gpu, self.clipset, self.requests = gpu, clipset, requests
        self.offsets = np.asarray(offsets, np.float32)
        self.lists = np.asarray(lists, np.uint32)
        self.parents, self.request_lists, self.roots, self.skeleton_offsets = parents, request_lists, roots, skeleton_offsets
        self.d_lists = _dev(gpu, self.lists)
        self.d_parents = _dev(gpu, parents)
        self.d_request_lists = None if request_lists is None else _dev(gpu, request_lists)
        self.d_roots = None if roots is None else _dev(gpu, roots)
        self.d_skeleton_offsets = None if skeleton_offsets is None else _dev(gpu, skeleton_offsets)

    def run(self, options, stride=0, lead=16, d_flags=None, d_requests=None):
        """The output buffer's bytes: lead bytes, n poses of `stride` bytes (0: S * K * 48), 64 tail bytes"""
        torch, ctx = self.gpu["torch"], self.gpu["ctx"]
        n, S, K = self.requests.size, self.offsets.size, self.lists.shape[1]
        pose = stride or S * K * 48
        buffer = torch.full((lead + pose * n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        options.pose_stride_bytes = stride
        ctx.extract_pose_features(self.clipset, _dev(self.gpu, self.requests) if d_requests is None else d_requests, n, options, self.offsets,
                                  self.d_lists, K, self.d_parents, buffer.data_ptr() + lead, num_lists=self.lists.shape[0],
                                  d_request_lists=self.d_request_lists, d_root_tracks=self.d_roots, d_skeleton_offsets=self.d_skeleton_offsets,
                                  d_out_flags=d_flags)
        torch.cuda.synchronize()
        options.pose_stride_bytes = 0
        return buffer.cpu().numpy()

    def pieces(self, options):
        """The (request, offset) pairs that write, their (c, u') and the library's B [V][K][12], T [V][12] and M [V][12]"""
        ab, torch, ctx = self.gpu["ab"], self.gpu["torch"], self.gpu["ctx"]
        clipset = self.clipset
        n, S, K = self.requests.size, self.offsets.size, self.lists.shape[1]
        duration = durations(self.gpu, clipset)
        tracks = np.array([clipset.clip_info(c).num_tracks for c in range(clipset.num_clips)], np.uint32)
        roots = self.roots if self.roots is not None else np.zeros(clipset.num_clips, np.uint32)
        request_lists = self.request_lists if self.request_lists is not None else np.zeros(n, np.uint32)
        pairs = []
        for r in range(n):
            clip, looping = int(self.requests["clip"][r]), int(self.requests["looping"][r])
            if clip >= clipset.num_clips or request_lists[r] >= self.lists.shape[0] or roots[clip] >= tracks[clip] or looping > 1:
                continue
            for s in range(S):
                writes, c, u = cases.offset_time(self.requests["time"][r], self.offsets[s], looping, duration[clip])
                if writes:
                    pairs.append((r, s, clip, c, u))
        v = len(pairs)
        if v == 0:
            return pairs, None, None, None
        clip = np.array([p[2] for p in pairs], np.uint32)
        u = np.array([p[4] for p in pairs], np.float32)
        d_requests = _dev(self.gpu, ab.make_requests(clip, u))
        d_objects = torch.zeros((v, K, 12), dtype=torch.float32, device="cuda")
        ctx.decompress_bones(clipset, d_requests, v, options, self.d_lists, K, d_objects, num_lists=self.lists.shape[0],
                             d_request_lists=_dev(self.gpu, request_lists[[p[0] for p in pairs]]), d_parent_indices=self.d_parents,
                             kind=ab.OBJECT_QVVF, d_skeleton_offsets=self.d_skeleton_offsets)
        d_local = torch.zeros((v, 12), dtype=torch.float32, device="cuda")
        ctx.decompress_bones(clipset, d_requests, v, options, _dev(self.gpu, roots), 1, d_local, num_lists=clipset.num_clips,
                             d_request_lists=_dev(self.gpu, clip))
        motion_requests = ab.make_root_motion_requests(clip, self.requests["time"][[p[0] for p in pairs]], u, [p[3] for p in pairs])
        d_motion = torch.zeros((v, 12), dtype=torch.float32, device="cuda")
        ctx.extract_root_motion(clipset, _dev(self.gpu, motion_requests), v, options, d_motion, d_root_tracks=self.d_roots)
        torch.cuda.synchronize()
        return pairs, d_objects.cpu().numpy(), d_local.cpu().numpy(), d_motion.cpu().numpy()

    def expected(self, options, sample=None):
        """{(r, s, k): the expected 12 floats} for the rows that are written (sample: a fraction of them, at random)"""
        pairs, objects, local, motion = self.pieces(options)
        tracks = [self.clipset.clip_info(c).num_tracks for c in range(self.clipset.num_clips)]
        request_lists = self.request_lists if self.request_lists is not None else np.zeros(self.requests.size, np.uint32)
        rng = np.random.default_rng(0)
        out = {}
        for i, (r, s, clip, c, u) in enumerate(pairs):
            for k, bone in enumerate(self.lists[request_lists[r]]):
                if bone >= tracks[clip] or (sample is not None and rng.random() >= sample):
                    continue
                out[(r, s, k)] = cases.compose(RM, objects[i, k], local[i], motion[i], RM.NORMALIZE_IEEE)
        return out

    def check(self, options, got_bytes, stride=0, lead=16, context=()):
        n, S, K = self.requests.size, self.offsets.size, self.lists.shape[1]
        pose = stride or S * K * 48
        want = self.expected(options)
        assert (got_bytes[:lead] == SENTINEL).all() and (got_bytes[lead + pose * n:] == SENTINEL).all(), context
        body = got_bytes[lead:lead + pose * n].reshape(n, pose)
        expected = np.full((n, pose), SENTINEL, np.uint8)
        for (r, s, k), row in want.items():
            expected[r, (s * K + k) * 48:(s * K + k + 1) * 48] = row.view(np.uint8)
        bad = np.argwhere((body != expected).any(axis=1))
        assert bad.size == 0, (context, int(bad[0][0]), self.requests[int(bad[0][0])], body[int(bad[0][0])].view(np.float32)[:S * K * 12],
                               expected[int(bad[0][0])].view(np.float32)[:S * K * 12])
        return len(want)


def _requests(gpu, num_clips, duration, seed, n=None):
    """Per clip: t at 0, D, inside and beyond both ends, CLAMP and LOOP, and one looping = 2 request"""
    rng = np.random.default_rng(seed)
    clip, time, looping = [], [], []
    for c in range(num_clips):
        d = float(duration[c])
        for t in [0.0, d, d * 0.37, -0.2, d + 0.3] + list(rng.uniform(-0.1, d + 0.1, 3)):
            for loop in (0, 1):
                clip.append(c)
                time.append(t)
                looping.append(loop)
        clip.append(c)
        time.append(d * 0.5)
        looping.append(2)
    return gpu["ab"].make_feature_requests(clip, time, looping)


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_named_clips_bit_for_bit(gpu, name):
    """Every named clip x settings kind x rounding (none, floor, ceil, nearest, per track): eight offsets across 0, 1, 3, 256 and 257
    boundaries and on k * D; a list with a hole and a duplicate; the root at track 0 (a skeleton root) and at the last track (not one)"""
    from tests import root_motion_cases as rm_cases
    ab = gpu["ab"]
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)], check_hash=True)
    n = spec.num_tracks
    duration = durations(gpu, clipset)
    requests = _requests(gpu, 1, duration, spec.seed)
    offsets = cases.offsets_for(float(duration[0]))[3]
    lists = bones_cases.pad_lists([[n - 1, NO_BONE, n // 2, n - 1]], 4)
    d_policies = _dev(gpu, (np.arange(n) % 4).astype(np.uint8))
    for kind in rm_cases.kinds_for(spec):
        roundings = [dict(rounding_policy=r) for r in range(4)]
        if kind == 1:
            roundings.append(dict(rounding_policy=ab.ROUND_PER_TRACK, d_per_track_rounding=d_policies.data_ptr()))
        for fields in roundings:
            options = _options(gpu, kind, **fields)
            for root in sorted({0, n - 1}):
                launch = Launch(gpu, clipset, requests, offsets, lists, bones_cases.tree(n), roots=np.array([root], np.uint32))
                assert launch.check(options, launch.run(options), context=(name, kind, fields, root)) > 0
    clipset.release()


def test_golden_fixture(gpu):
    """The reference's rows (tests/golden/make_features_golden.py) within tests/test_features_oracle.py's gate (the walk's normalisation
    flavour), scale lanes bit for bit; the rows it does not write keep the sentinel"""
    from tests.test_features_oracle import _gate
    ab = gpu["ab"]
    g = np.load(clips.golden_path("features", "golden.npz"))
    names = [str(x) for x in g["names"]]
    specs = [clips.TRANSFORM_SPECS[x] for x in names]
    clipset = gpu["ctx"].upload([clips.load_blob(x) for x in names], check_hash=True)
    skeletons = [bones_cases.tree(s.num_tracks) for s in specs]
    skeleton_offsets = np.concatenate([[0], np.cumsum([s.num_tracks for s in specs])[:-1]]).astype(np.uint32)
    requests = ab.make_feature_requests(g["clip"], g["time"], g["looping"])
    launch = Launch(gpu, clipset, requests, g["offsets"], g["bones"][None, :], np.concatenate(skeletons), roots=g["roots"],
                    skeleton_offsets=skeleton_offsets)
    options = _options(gpu, 1)
    got = launch.run(options)
    launch.check(options, got, context="golden")
    S, K = g["offsets"].size, g["bones"].size
    rows = got[16:16 + requests.size * S * K * 48].view(np.float32).reshape(requests.size, S, K, 12)
    written = ~np.isnan(g["rows"][..., 0])
    assert written.any() and not written.all()
    for r, s, k in np.argwhere(written):
        depth = int(np.log2(specs[int(g["clip"][r])].num_tracks)) + 1
        assert _gate(g["rows"][r, s, k], rows[r, s, k], depth), (r, s, k)
    clipset.release()


@pytest.mark.parametrize("num_offsets", range(1, 9))
def test_lists_and_offset_counts(gpu, num_offsets):
    """S from 1 to 8 with K of 1, 4 and 32 (holes, duplicates, bones beyond the clip), a list per request (some beyond num_lists)"""
    ab = gpu["ab"]
    name = "c2_100bones"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = spec.num_tracks
    duration = durations(gpu, clipset)
    rng = np.random.default_rng(num_offsets)
    offsets = np.concatenate([[0.0], rng.uniform(-1.5, 1.5, num_offsets - 1)]).astype(np.float32)
    requests = _requests(gpu, 1, duration, num_offsets)
    options = _options(gpu, 0)
    for k in (1, 4, 32):
        raw = [list(rng.integers(0, n, k)), [NO_BONE] + [n - 1] * (k - 1), list(bones_cases.C2_FOUR_LEAVES * 8)[:k], [n + 3] + [0] * (k - 1)]
        lists = bones_cases.pad_lists(raw, k)
        request_lists = rng.integers(0, len(raw) + 1, requests.size).astype(np.uint32)
        launch = Launch(gpu, clipset, requests, offsets, lists, bones_cases.tree(n), request_lists=request_lists,
                        roots=np.array([3], np.uint32))
        launch.check(options, launch.run(options), context=(num_offsets, k))
    clipset.release()


def test_mixed_rigs_untouched_rows_strides_and_request_offsets(gpu):
    """A ragged clip set with a skeleton and a root per clip (one root is not a skeleton root, one beyond its clip's tracks), invalid
    clips and lists, looping = 2, a padded stride, an output 16 bytes into its allocation, and the request array at byte offsets 4 and 8"""
    ab, torch = gpu["ab"], gpu["torch"]
    names = ["c1_30bones", "ragged_17", "mixed_scale", "one_bone", "c2_100bones", "looping", "one_sample"]
    kinds = ["chain", "tree", "star", "random", "late", "tree", "tree"]
    specs = [clips.TRANSFORM_SPECS[x] for x in names]
    skeletons = [bones_cases.skeleton(k, s.num_tracks, seed=i) for i, (k, s) in enumerate(zip(kinds, specs))]
    skeleton_offsets = np.concatenate([[0], np.cumsum([len(s) for s in skeletons])[:-1]]).astype(np.uint32)
    clipset = gpu["ctx"].upload([clips.load_blob(x) for x in names], check_hash=True)
    roots = np.array([5, 0, 0, 0, 99, 40, 0], np.uint32)          # looping has 40 tracks: its root is out of range
    rng = np.random.default_rng(7)
    num_requests = 301
    clip = rng.integers(0, len(names), num_requests).astype(np.uint32)
    clip[rng.random(num_requests) < 0.08] = len(names)
    clip[3] = 0xFFFFFFFF
    looping = rng.integers(0, 2, num_requests).astype(np.uint32)
    looping[::23] = 2
    requests = ab.make_feature_requests(clip, rng.uniform(-0.2, 2.5, num_requests), looping)
    lists = bones_cases.pad_lists([[0], [99, 16, 5, 56, 29], [3, NO_BONE, 3, 40, 0], list(range(0, 64, 2))], 32)
    request_lists = rng.integers(0, len(lists) + 2, num_requests).astype(np.uint32)
    request_lists[4] = 0xFFFFFFFF
    offsets = np.array([-0.4, 0.0, 0.25, 1.7, -3.1], np.float32)
    launch = Launch(gpu, clipset, requests, offsets, lists, np.concatenate(skeletons), request_lists=request_lists, roots=roots,
                    skeleton_offsets=skeleton_offsets)
    options = _options(gpu, 1)
    stride = offsets.size * 32 * 48 + 64
    want = launch.run(options, stride=stride)
    launch.check(options, want, stride=stride, context="mixed")
    raw = np.ascontiguousarray(requests).view(np.uint8)
    for offset in (4, 8):
        packed = torch.zeros(raw.size + 16, dtype=torch.uint8, device="cuda")
        packed[offset:offset + raw.size] = torch.from_numpy(raw).cuda()
        got = launch.run(options, stride=stride, d_requests=packed.data_ptr() + offset)
        assert (got == want).all(), offset
    clipset.release()


def test_flags(gpu):
    """NEGATIVE_SCALE for a mirrored listed bone and for a mirrored root (only then), WRAP_CLIP_CYCLE for a loop crossing on a wrap-compressed
    clip (only with c != 0), INVALID_SKELETON for a bad parent on a chain; the rows match the port's composition each time"""
    ab, torch = gpu["ab"], gpu["torch"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = spec.num_tracks
    parents = bones_cases.tree(n)
    leaves = [b for b in range(n) if 2 * b + 1 >= n]
    requests = ab.make_feature_requests(0, np.linspace(0.0, 1.0, 9), [0, 1] * 4 + [0])
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    # which sub-tracks a negative variable default scale reaches: bones whose scale is a default sub-track
    variable = np.tile(IDENTITY, (n, 1))
    variable[:, 8] = -1.0
    d_variable = torch.from_numpy(variable).cuda()
    probe = _options(gpu, 0, default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
    d_pose = torch.zeros((1, n, 12), dtype=torch.float32, device="cuda")
    gpu["ctx"].decompress_tracks(clipset, _dev(gpu, ab.make_requests([0], [0.3])), 1, probe, d_pose)
    scale = d_pose.cpu().numpy()[0, :, 8]
    mirrored_leaf = [b for b in leaves if scale[b] < 0][0]
    plain_leaf = [b for b in leaves if scale[b] > 0][0]
    for bones, root, flag in (([plain_leaf], 0, ab.ERROR_FLAG_NEGATIVE_SCALE if scale[0] < 0 else 0),
                              ([mirrored_leaf], 1, ab.ERROR_FLAG_NEGATIVE_SCALE), ([plain_leaf, 0], 2, None)):
        variable = np.tile(IDENTITY, (n, 1))
        variable[mirrored_leaf, 8] = -1.0
        if flag is None:                # a mirrored root, the listed bones plain
            variable[root, 8] = -1.0
            flag = ab.ERROR_FLAG_NEGATIVE_SCALE if scale[root] < 0 else 0
        d_variable = torch.from_numpy(variable).cuda()
        options = _options(gpu, 0, default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
        launch = Launch(gpu, clipset, requests, [0.0, 0.4], bones_cases.pad_lists([bones], len(bones)), parents,
                        roots=np.array([root], np.uint32))
        launch.check(options, launch.run(options, d_flags=d_flags), context=("mirrored", bones, root))
        assert int(d_flags.item()) == flag, (bones, root)
    # a bad parent on the listed bone's chain
    late = parents.copy()
    late[1] = 1
    launch = Launch(gpu, clipset, requests, [0.0], bones_cases.pad_lists([[3]], 1), late)
    options = _options(gpu, 0)
    launch.check(options, launch.run(options, d_flags=d_flags), context="bad parent")
    assert int(d_flags.item()) == ab.ERROR_FLAG_INVALID_SKELETON
    clipset.release()
    # loop crossings on wrap-compressed clips
    names = ["looping", "c1_30bones"]
    clipset = gpu["ctx"].upload([clips.load_blob(x) for x in names])
    assert clipset.clip_info(0).looping_policy == ab.LOOP_WRAP and clipset.clip_info(1).looping_policy != ab.LOOP_WRAP
    options = _options(gpu, 1)
    for c in range(2):
        for looping, offset in ((1, 5.0), (0, 5.0), (1, 0.1)):
            launch = Launch(gpu, clipset, ab.make_feature_requests(c, [0.2], looping), [offset], bones_cases.pad_lists([[0, 7]], 2),
                            bones_cases.tree(40 if c == 0 else 30))
            launch.check(options, launch.run(options, d_flags=d_flags), context=("wrap", c, looping, offset))
            want = ab.ERROR_FLAG_WRAP_CLIP_CYCLE if c == 0 and looping == 1 and offset > 1.0 else 0
            assert int(d_flags.item()) == want, (c, looping, offset)
    clipset.release()


def test_database_tiers(gpu):
    """Clip sets bound to a database, in every tier state of tests/database_cases.py: the pieces the library decodes from the same tiers"""
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
    skeletons = [bones_cases.tree(c) for c in counts]
    skeleton_offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    t = db_cases.ALL_TIMES
    requests = ab.make_feature_requests(np.repeat(np.arange(len(blobs), dtype=np.uint32), t.size), np.tile(t, len(blobs)),
                                        np.tile([0, 1], (t.size * len(blobs) + 1) // 2)[:t.size * len(blobs)])
    launch = Launch(gpu, clipset, requests, [-0.3, 0.0, 0.5, 1.25], bones_cases.pad_lists([[min(counts) - 1, 0, 5]], 3), np.concatenate(skeletons),
                    roots=np.array([min(counts) - 1] * len(blobs), np.uint32), skeleton_offsets=skeleton_offsets)
    done = []
    for state, ops in db_cases.STATES.items():
        for op, tier, k in ops[len(done):]:
            (database.stream_in if op == db_cases.IN else database.stream_out)(tier, k)
        done = ops
        options = _options(gpu, 1)
        launch.check(options, launch.run(options), context=state)
    clipset.release()


def test_wide_clip(gpu):
    """wide_2500: one 2500-bone pose per block still fits; a chain through every chunk of 32 bones"""
    ab = gpu["ab"]
    clipset = gpu["ctx"].upload([clips.load_blob("wide_2500")])
    n = 2500
    for skeleton in ("tree", "chain"):
        requests = ab.make_feature_requests(0, np.linspace(0.0, 0.3, 3), [0, 1, 1])
        launch = Launch(gpu, clipset, requests, [-0.1, 0.0, 0.2], bones_cases.pad_lists([[n - 1, 0, 1234, NO_BONE]], 4),
                        bones_cases.skeleton(skeleton, n, seed=3), roots=np.array([700], np.uint32))
        options = _options(gpu, 0)
        launch.check(options, launch.run(options), context=skeleton)
    clipset.release()


def test_c2_sized_launch(gpu):
    """The C2 bench clips and request count (600,000), S = 4 offsets, K = 4 on a binary tree, half the requests LOOP, a random root per
    clip; a random tenth of the rows is composed by the port"""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    n = int(w["req_clip"].size)
    assert n == 600000
    rng = np.random.default_rng(3)
    roots = rng.integers(0, w["num_tracks"], clipset.num_clips).astype(np.uint32)
    duration = durations(gpu, clipset)
    clip = w["req_clip"].astype(np.uint32)
    requests = ab.make_feature_requests(clip, rng.uniform(-0.1, 1.1, n) * duration[clip], rng.integers(0, 2, n))
    lists = bones_cases.pad_lists([[0, 63, 99, 7]], 4)
    launch = Launch(gpu, clipset, requests, cases.BENCH_OFFSETS, lists, bones_cases.tree(w["num_tracks"]), roots=roots)
    options = _options(gpu, 0)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_out = torch.full((n, 4, 4, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.extract_pose_features(clipset, _dev(gpu, requests), n, options, cases.BENCH_OFFSETS, launch.d_lists, 4, launch.d_parents, d_out,
                              d_root_tracks=launch.d_roots, d_out_flags=d_flags)
    torch.cuda.synchronize()
    assert int(d_flags.item()) == 0
    got = d_out.cpu().numpy()
    want = launch.expected(options, sample=0.1)
    assert len(want) > n
    for (r, s, k), row in want.items():
        assert clips.bit_equal(got[r, s, k], row), (r, s, k, requests[r])
    clipset.release()


def test_refusals_launch_nothing(gpu):
    import ctypes as C
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")])
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_feature_requests(0, np.linspace(0, 1, 8), 1))
    d_lists = _dev(gpu, np.array([0, 5, 29, 3], np.uint32))
    d_parents = _dev(gpu, bones_cases.tree(30))
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    policies = torch.zeros(16, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(offsets=None), dict(offsets=np.zeros(0, np.float32)), dict(offsets=np.zeros(9, np.float32)),
        dict(offsets=np.array([0.0, np.nan], np.float32)), dict(offsets=np.array([np.inf], np.float32)),
        dict(parents=None), dict(k=0), dict(k=33), dict(num_lists=0), dict(lists=None),
        dict(requests=None), dict(out=None), dict(offset=8), dict(stride=4 * 2 * 48 - 16), dict(stride=4 * 2 * 48 + 8),
        dict(options=_options(gpu, 0, output_layout=ab.LAYOUT_QVV40)),
        dict(options=_options(gpu, 0, looping_policy=ab.LOOP_WRAP)),
        dict(options=_options(gpu, 0, looping_policy=ab.LOOP_AS_COMPRESSED)),
        dict(options=_options(gpu, 0, d_request_policies=policies.data_ptr())),
        dict(options=_options(gpu, 0, skip_mask=ab.SKIP_SCALE)),
        dict(options=_options(gpu, 0, d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=_options(gpu, 0, default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(clipset=scalar),
        dict(options=_options(gpu, 0, struct_size=8)),
    ]
    lib = ab.api._lib()
    for case in refusals:
        buffer = torch.full((8 * 4 * 2 * 48 + 256,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        launches = ctx.launch_count
        options = case.get("options", _options(gpu, 0))
        options.pose_stride_bytes = case.get("stride", 0)
        offsets = case.get("offsets", np.array([0.0, 0.5], np.float32))
        out = 0 if "out" in case else buffer.data_ptr() + case.get("offset", 0)
        status = lib.aclb200_extract_pose_features(
            ctx._handle, case.get("clipset", clipset)._handle, None if case.get("requests", 1) is None else requests.data_ptr(), 8,
            C.byref(options), None if offsets is None else offsets.ctypes.data, 2 if offsets is None else offsets.size,
            None if case.get("lists", 1) is None else d_lists.data_ptr(), case.get("num_lists", 1), case.get("k", 4), None, None,
            None if case.get("parents", 1) is None else d_parents.data_ptr(), None, out or None, d_flags.data_ptr(), None)
        assert status == 1, case
        torch.cuda.synchronize()
        assert ctx.launch_count == launches, case
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    clipset.release()
    scalar.release()
