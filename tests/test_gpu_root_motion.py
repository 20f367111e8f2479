"""aclb200_extract_root_motion: every 48 byte row against the port's composition (oracle/root_motion_oracle.c, the IEEE normalise flavour
of the CUDA path) of the library's own root samples, the root rows aclb200_decompress_tracks writes at from_time, to_time, D and 0 with
the clamp policy. Those rows are pinned to the oracle and the reference by tests/test_gpu_parity.py; tests/test_root_motion_oracle.py pins
the port's composition to the reference. Rows a request may not write keep their sentinel, and so do the bytes around the output."""
import numpy as np
import pytest

from oracle import root_motion as RM
from tests import clips
from tests import root_motion_cases as cases

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5
CYCLES = [0, 1, -1, 2, -2, 256, -256]


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


def durations(gpu, clipset):
    """D of each clip: the clip info's duration for clamp-compressed clips, recomputed for the wrap-compressed ones"""
    out = []
    for c in range(clipset.num_clips):
        info = clipset.clip_info(c)
        out.append(np.float32(info.num_samples - 1) / np.float32(info.sample_rate) if info.num_samples > 1 else np.float32(0.0))
    return np.array(out, np.float32)


def library_samples(gpu, clipset, requests, roots, options):
    """[n][4][12] the root rows of aclb200_decompress_tracks at from, to, D and 0 (zeros for requests without a valid root)"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    n = requests.size
    duration = durations(gpu, clipset)
    clip = requests["clip"]
    valid = clip < clipset.num_clips
    safe = np.where(valid, clip, 0)
    times = np.stack([requests["from_time"], requests["to_time"], duration[safe], np.zeros(n, np.float32)], axis=1)
    d_requests = _dev(gpu, ab.make_requests(np.repeat(clip, 4), times.reshape(-1)))
    d_out = torch.zeros((n * 4, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, d_requests, n * 4, options, d_out)
    torch.cuda.synchronize()
    poses = d_out.cpu().numpy().reshape(n, 4, clipset.max_tracks, 12)
    root = np.where(valid, roots[safe], 0)
    return poses[np.arange(n), :, np.minimum(root, clipset.max_tracks - 1)]


def extract(gpu, clipset, requests, options, d_roots=None, d_flags=None, lead=16):
    """Runs the extraction into a sentinel-filled buffer; returns the buffer's bytes (lead bytes, n rows of 48 bytes, 64 tail bytes)"""
    torch, ctx = gpu["torch"], gpu["ctx"]
    n = requests.size
    buffer = torch.full((lead + 48 * n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.extract_root_motion(clipset, _dev(gpu, requests), n, options, buffer.data_ptr() + lead, d_root_tracks=d_roots, d_out_flags=d_flags)
    torch.cuda.synchronize()
    return buffer.cpu().numpy()


def check(got_bytes, requests, samples, writes, lead=16, context=()):
    """Every row: the port's composition of the library's samples, all 48 bytes, or the sentinel; the bytes around it the sentinel"""
    n = requests.size
    assert (got_bytes[:lead] == SENTINEL).all() and (got_bytes[lead + 48 * n:] == SENTINEL).all(), context
    rows = got_bytes[lead:lead + 48 * n].reshape(n, 48)
    for r in range(n):
        if not writes[r]:
            assert (rows[r] == SENTINEL).all(), (context, r)
            continue
        want, _ = RM.port_root_motion(samples[r], int(requests["cycles"][r]), RM.NORMALIZE_IEEE)
        assert (rows[r] == want.view(np.uint8)).all(), (context, r, requests[r], rows[r].view(np.float32), want)


def _named_requests(gpu, spec, duration):
    """Every time pair of root_motion_cases plus +-1 ulp around key frames and the NaN / inf times, at each cycle count of CYCLES"""
    pairs = cases.time_pairs(spec, duration)
    key_frames = [np.float32(k / spec.sample_rate) for k in (1, 7, 20) if k < spec.num_samples]
    for t in key_frames:
        pairs += [(float(np.nextafter(t, np.float32(-1))), float(np.nextafter(t, np.float32(9)))), (float(t), float(np.nextafter(t, np.float32(9))))]
    for special in (np.nan, np.inf, -np.inf):
        pairs += [(special, float(duration) * 0.5), (0.1, special)]
    froms = np.array([p[0] for p in pairs], np.float32)
    tos = np.array([p[1] for p in pairs], np.float32)
    return gpu["ab"].make_root_motion_requests(0, np.repeat(froms, len(CYCLES)), np.repeat(tos, len(CYCLES)), np.tile(CYCLES, len(pairs)))


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_named_clips_bit_for_bit(gpu, name):
    """Every named clip x settings kind x rounding (none, floor, ceil, nearest, per track) x time pair x cycles; the root at track 0 and at
    the clip's last track"""
    ab, torch = gpu["ab"], gpu["torch"]
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = gpu["ctx"].upload([blob], check_hash=True)
    requests = _named_requests(gpu, spec, durations(gpu, clipset)[0])
    writes = np.abs(requests["cycles"]) <= ab.MAX_ROOT_MOTION_CYCLES
    policies = (np.arange(spec.num_tracks) % 4).astype(np.uint8)
    d_policies = _dev(gpu, policies)
    for kind in cases.kinds_for(spec):
        roundings = [dict(rounding_policy=r) for r in range(4)]
        if kind == 1:
            roundings.append(dict(rounding_policy=ab.ROUND_PER_TRACK, d_per_track_rounding=d_policies.data_ptr()))
        for fields in roundings:
            options = _options(gpu, kind, **fields)
            for root in sorted({0, spec.num_tracks - 1}):
                roots = np.array([root], np.uint32)
                samples = library_samples(gpu, clipset, requests, roots, options)
                got = extract(gpu, clipset, requests, options, d_roots=_dev(gpu, roots) if root else None)
                check(got, requests, samples, writes, context=(name, kind, fields, root))
    del d_policies, torch
    clipset.release()


def test_golden_fixture(gpu):
    """The reference's M (tests/golden/make_root_motion_golden.py), all 48 bytes"""
    ab, torch = gpu["ab"], gpu["torch"]
    g = np.load(clips.golden_path("root_motion", "golden.npz"))
    clipset = gpu["ctx"].upload([clips.load_blob(str(n)) for n in g["names"]], check_hash=True)
    requests = ab.make_root_motion_requests(g["clip"], g["from_time"], g["to_time"], g["cycles"])
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = extract(gpu, clipset, requests, _options(gpu, 1), d_roots=_dev(gpu, g["roots"]), d_flags=d_flags)
    rows = got[16:16 + 48 * requests.size].reshape(-1, 48)
    assert (rows == np.ascontiguousarray(g["motion"]).view(np.uint8)).all()
    clipset.release()


def test_mixed_rigs_and_untouched_rows(gpu):
    """A ragged clip set with a root per clip (some not track 0, one beyond its clip's tracks), invalid clips and |cycles| = MAX + 1;
    301 requests leave a partial last block"""
    ab = gpu["ab"]
    names = ["c1_30bones", "ragged_17", "mixed_scale", "one_bone", "c2_100bones", "looping", "single_segment"]
    specs = [clips.TRANSFORM_SPECS[n] for n in names]
    clipset = gpu["ctx"].upload([clips.load_blob(n) for n in names], check_hash=True)
    roots = np.array([5, 16, 0, 0, 99, 40, 7], np.uint32)          # looping has 40 tracks: its root is out of range
    rng = np.random.default_rng(7)
    n = 301
    clip = rng.integers(0, len(names), n).astype(np.uint32)
    clip[rng.random(n) < 0.08] = len(names)
    clip[3] = 0xFFFFFFFF
    cycles = rng.integers(-3, 4, n).astype(np.int32)
    cycles[::17] = ab.MAX_ROOT_MOTION_CYCLES + 1
    cycles[5::17] = -ab.MAX_ROOT_MOTION_CYCLES - 1
    cycles[7::17] = ab.MAX_ROOT_MOTION_CYCLES
    requests = ab.make_root_motion_requests(clip, rng.uniform(-0.2, 2.5, n), rng.uniform(-0.2, 2.5, n), cycles)
    tracks = np.array([s.num_tracks for s in specs] + [0], np.uint32)
    safe = np.minimum(clip, len(names))
    writes = (clip < len(names)) & (np.append(roots, 0)[safe] < tracks[safe]) & (np.abs(cycles) <= ab.MAX_ROOT_MOTION_CYCLES)
    assert writes.any() and not writes.all()
    options = _options(gpu, 1)
    samples = library_samples(gpu, clipset, requests, roots, options)
    check(extract(gpu, clipset, requests, options, d_roots=_dev(gpu, roots)), requests, samples, writes, context="mixed")
    clipset.release()


def test_negative_scale_flag(gpu):
    """A mirrored root (a negative variable default scale on a root whose scale is a default sub-track) takes qvv_mul's matrix branch:
    NEGATIVE_SCALE is reported, and only then; the rows match the port either way"""
    ab, torch = gpu["ab"], gpu["torch"]
    name = "mixed_scale"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = spec.num_tracks
    times = clips.sample_times(spec)
    variable = np.tile(cases.IDENTITY, (n, 1))
    variable[:, 8] = -1.0
    d_variable = torch.from_numpy(variable).cuda()
    probe = _options(gpu, 0, default_modes=(ab.DEFAULT_VARIABLE,) * 3, d_variable_defaults=d_variable.data_ptr())
    d_pose = torch.zeros((times.size, n, 12), dtype=torch.float32, device="cuda")
    gpu["ctx"].decompress_tracks(clipset, _dev(gpu, ab.make_requests(np.zeros(times.size, np.uint32), times)), times.size, probe, d_pose)
    local = d_pose.cpu().numpy()
    mirrored = [b for b in range(n) if (local[:, b, 8] < 0).all()]
    plain = [b for b in range(n) if (local[:, b, 8] > 0).all()]
    assert mirrored and plain
    requests = ab.make_root_motion_requests(0, np.repeat(times, 3), np.repeat(times[::-1], 3), np.tile([0, 2, -1], times.size))
    writes = np.ones(requests.size, bool)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    for root, flag in ((mirrored[0], ab.ERROR_FLAG_NEGATIVE_SCALE), (plain[0], 0)):
        roots = np.array([root], np.uint32)
        samples = library_samples(gpu, clipset, requests, roots, probe)
        got = extract(gpu, clipset, requests, probe, d_roots=_dev(gpu, roots), d_flags=d_flags)
        check(got, requests, samples, writes, context=("mirrored", root))
        assert int(d_flags.item()) == flag, root
    clipset.release()


def test_wrap_clip_cycle_flag(gpu):
    """WRAP_CLIP_CYCLE appears only on clips compressed with the wrap policy, and only with cycles != 0. looping and stripped_loop are
    built from loop optimised content; all_default's sub-tracks are all defaults, so its first and last samples are equal and the
    compressor keeps it as a loop too"""
    ab, torch = gpu["ab"], gpu["torch"]
    names = list(clips.TRANSFORM_SPECS)
    clipset = gpu["ctx"].upload([clips.load_blob(n) for n in names])
    wrap = {n for c, n in enumerate(names) if clipset.clip_info(c).looping_policy == ab.LOOP_WRAP}
    assert wrap == {"looping", "stripped_loop", "all_default"}
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    options = _options(gpu, 1)
    for c, name in enumerate(names):
        for cycles in (0, 1, -2):
            requests = ab.make_root_motion_requests(c, [0.1, 1.2], [0.5, 0.3], cycles)
            extract(gpu, clipset, requests, options, d_flags=d_flags)
            want = ab.ERROR_FLAG_WRAP_CLIP_CYCLE if name in wrap and cycles != 0 else 0
            assert int(d_flags.item()) == want, (name, cycles)
    # a request that leaves its row untouched reports nothing
    c = names.index("looping")
    extract(gpu, clipset, ab.make_root_motion_requests(c, 0.1, 0.5, ab.MAX_ROOT_MOTION_CYCLES + 1), options, d_flags=d_flags)
    assert int(d_flags.item()) == 0
    clipset.release()


def test_database_tiers(gpu):
    """Clip sets bound to a database, in every tier state of tests/database_cases.py: the samples the library decodes from the same
    streamed tiers"""
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
    roots = np.array([min(counts) - 1] * len(blobs), np.uint32)
    t = db_cases.ALL_TIMES
    clip = np.repeat(np.arange(len(blobs), dtype=np.uint32), t.size * 3)
    requests = ab.make_root_motion_requests(clip, np.tile(np.repeat(t, 3), len(blobs)), np.tile(np.repeat(t[::-1], 3), len(blobs)),
                                            np.tile([0, 1, -2], t.size * len(blobs)))
    writes = np.ones(requests.size, bool)
    done = []
    for state, ops in db_cases.STATES.items():
        for op, tier, k in ops[len(done):]:
            (database.stream_in if op == db_cases.IN else database.stream_out)(tier, k)
        done = ops
        options = _options(gpu, 1)
        samples = library_samples(gpu, clipset, requests, roots, options)
        check(extract(gpu, clipset, requests, options, d_roots=_dev(gpu, roots)), requests, samples, writes, context=state)
    clipset.release()


@pytest.mark.parametrize("num_requests", [1, 13])
def test_small_launches(gpu, num_requests):
    """One request, and a partial warp"""
    ab = gpu["ab"]
    spec = clips.TRANSFORM_SPECS["c1_30bones"]
    clipset = gpu["ctx"].upload([clips.load_blob("c1_30bones")])
    rng = np.random.default_rng(num_requests)
    requests = ab.make_root_motion_requests(0, rng.uniform(0, 2, num_requests), rng.uniform(0, 2, num_requests),
                                            rng.integers(-2, 3, num_requests))
    options = _options(gpu, 0)
    roots = np.array([spec.num_tracks - 1], np.uint32)
    samples = library_samples(gpu, clipset, requests, roots, options)
    check(extract(gpu, clipset, requests, options, d_roots=_dev(gpu, roots)), requests, samples, np.ones(num_requests, bool))
    clipset.release()


def test_c2_sized_launch(gpu):
    """The C2 bench clips and request count (600,000) with random from / to / cycles and a random root per clip; the library's samples
    come from decompress_bones with the root as the only listed bone (byte for byte decompress_tracks's root row, tests/test_gpu_bones.py),
    and a random tenth of the rows is composed by the port"""
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
    requests = ab.make_root_motion_requests(clip, rng.uniform(-0.1, 1.1, n) * duration[clip], rng.uniform(-0.1, 1.1, n) * duration[clip],
                                            rng.integers(-3, 4, n))
    options = _options(gpu, 0)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_out = torch.full((n, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.extract_root_motion(clipset, _dev(gpu, requests), n, options, d_out, d_root_tracks=_dev(gpu, roots), d_out_flags=d_flags)
    times = np.stack([requests["from_time"], requests["to_time"], duration[clip], np.zeros(n, np.float32)], axis=1).reshape(-1)
    d_samples = torch.zeros((n * 4, 12), dtype=torch.float32, device="cuda")
    ctx.decompress_bones(clipset, _dev(gpu, ab.make_requests(np.repeat(clip, 4), times)), n * 4, options, _dev(gpu, roots), 1, d_samples,
                         num_lists=clipset.num_clips, d_request_lists=_dev(gpu, np.repeat(clip, 4)))
    torch.cuda.synchronize()
    assert int(d_flags.item()) == 0
    got = d_out.cpu().numpy()
    samples = d_samples.cpu().numpy().reshape(n, 4, 12)
    for r in rng.choice(n, n // 10, replace=False):
        want, _ = RM.port_root_motion(samples[r], int(requests["cycles"][r]), RM.NORMALIZE_IEEE)
        assert clips.bit_equal(got[r], want), (r, requests[r])
    clipset.release()


def test_refusals_launch_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")])
    scalar = ctx.upload([clips.load_blob("float1")])
    requests = _dev(gpu, ab.make_root_motion_requests(0, np.linspace(0, 1, 8), np.linspace(1, 0, 8), 1))
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    policies = torch.zeros(16, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(requests=None), dict(out=None), dict(offset=8),
        dict(options=_options(gpu, 0, output_layout=ab.LAYOUT_QVV40)),
        dict(options=_options(gpu, 0, looping_policy=ab.LOOP_WRAP)),
        dict(options=_options(gpu, 0, looping_policy=ab.LOOP_AS_COMPRESSED)),
        dict(options=_options(gpu, 0, d_request_policies=policies.data_ptr())),
        dict(options=_options(gpu, 0, skip_mask=ab.SKIP_SCALE)),
        dict(options=_options(gpu, 0, d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=_options(gpu, 0, default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(clipset=scalar),
        dict(options=_options(gpu, 0, struct_size=8)),          # an options struct of another size: refused before any option is read
    ]
    for case in refusals:
        buffer = torch.full((8 * 48 + 64,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        launches = ctx.launch_count
        out = 0 if "out" in case else buffer.data_ptr() + case.get("offset", 0)
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.extract_root_motion(case.get("clipset", clipset), case["requests"] if "requests" in case else requests, 8,
                                    case.get("options", _options(gpu, 0)), out, d_out_flags=d_flags)
        assert error.value.status == 1, case
        torch.cuda.synchronize()
        assert ctx.launch_count == launches, case
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    clipset.release()
    scalar.release()


def test_requests_at_any_4_byte_offset(gpu):
    """The request array only needs its fields' 4 byte alignment: requests packed at byte offsets 4, 8 and 12 of a larger device buffer
    give the rows of the same requests at offset 0"""
    torch, ab = gpu["torch"], gpu["ab"]
    spec = clips.TRANSFORM_SPECS["mixed_scale"]
    clipset = gpu["ctx"].upload([clips.load_blob("mixed_scale")])
    rng = np.random.default_rng(17)
    n = 77
    requests = ab.make_root_motion_requests(0, rng.uniform(-0.1, 2.6, n), rng.uniform(-0.1, 2.6, n), rng.integers(-3, 4, n))
    options = _options(gpu, 1)
    roots = np.array([spec.num_tracks - 1], np.uint32)
    samples = library_samples(gpu, clipset, requests, roots, options)
    d_roots = _dev(gpu, roots)
    want = extract(gpu, clipset, requests, options, d_roots=d_roots)
    check(want, requests, samples, np.ones(n, bool), context="offset 0")
    raw = np.ascontiguousarray(requests).view(np.uint8)
    for offset in (4, 8, 12):
        packed = torch.zeros(raw.size + 16, dtype=torch.uint8, device="cuda")
        packed[offset:offset + raw.size] = torch.from_numpy(raw).cuda()
        buffer = torch.full((16 + 48 * n + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        gpu["ctx"].extract_root_motion(clipset, packed.data_ptr() + offset, n, options, buffer.data_ptr() + 16, d_root_tracks=d_roots)
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == want).all(), offset
    clipset.release()
