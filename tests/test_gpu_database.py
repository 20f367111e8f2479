"""Clip sets bound to a streaming database (acl::compressed_database), decoded on the device from the tiers streamed in: bit for bit
against the reference's decompression_context initialised with a database_context driven through the same stream_in / stream_out calls
(oracle/ref_database.cpp, or its stored outputs in tests/golden/database_tiers.npz). decompress_track rotations are gated at 1e-5 as in test_gpu_parity.py."""
import numpy as np
import pytest

from tests import clips
from tests import database_cases as cases

pytestmark = pytest.mark.gpu
IN, OUT, MEDIUM, LOW, ALL = cases.IN, cases.OUT, cases.MEDIUM, cases.LOW, cases.ALL
LANES = clips.DEFINED_LANES
SINGLE_TRACK_TOLERANCE = 1e-5
ROUNDINGS = range(4)


class _Reference:
    """What the reference decodes: the compiled reference (oracle/_ref/libaclref_db.so) where it exists, else the stored outputs of
    tests/golden/database_tiers.npz (every rounding policy with the clips' own looping policy)."""

    def __init__(self, ref, rd):
        self.ref, self.rd = ref, rd
        self.live = rd.available()
        if self.live:
            self.bound, self.database, self.other_clip, self.other_database = cases.build_cases(ref, rd)
            self.plain = clips.load_blob(cases.PLAIN_CLIP)
        else:
            g = np.load(clips.golden_path("database_tiers", "npz"))
            self.golden = g
            self.bound = [ref.aligned_blob(g[f"clip{i}"]) for i in range(len(g["num_tracks"]))]
            self.database = ref.aligned_blob(g["database"])
            self.other_clip, self.other_database = ref.aligned_blob(g["other_clip"]), ref.aligned_blob(g["other_database"])
            self.first_track = np.concatenate([[0], np.cumsum(g["num_tracks"])]).astype(int)
            self.plain = clips.load_blob(cases.PLAIN_CLIP)

    def has(self, looping):
        return self.live or looping == self.ref.LOOP_AS_COMPRESSED

    def poses(self, state, clip, t, rounding, looping):
        """float32 [num_tracks, 12]; clip 4 is the plain clip"""
        if self.live:
            if clip == 4:
                return self.ref.decompress_tracks(self.plain, float(t), rounding, looping, settings=self.ref.SETTINGS_DEBUG)
            return self.rd.decompress(self.bound[clip], self.database, cases.STATES[state], float(t), rounding, looping)
        time_index = int(np.nonzero(cases.ALL_TIMES == np.float32(t))[0][0])
        if clip == 4:
            return self.golden["poses_plain"][rounding, time_index]
        rows = self.golden[f"poses_{state}"][rounding, time_index]
        return rows[self.first_track[clip]:self.first_track[clip + 1]]


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port, ref, ref_database
    return dict(torch=torch, ab=ab, port=port, ref=ref, ctx=ab.Context(0), reference=_Reference(ref, ref_database))


def _to_device(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).view(np.uint8).reshape(-1)).cuda()


def _options(gpu, kind=1, **kw):
    s = gpu["port"].settings_for_kind(kind).c        # kind 1: debug settings, the reference's settings_database
    fields = dict(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                  clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                  default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                  constant_defaults=list(s.constant_defaults))
    fields.update(kw)
    return gpu["ab"].Options(**fields)


def _requests():
    # every database clip and the plain clip (index 4) in one launch, times past both ends
    return np.repeat(np.arange(5, dtype=np.uint32), len(cases.ALL_TIMES)), np.tile(cases.ALL_TIMES, 5)


def _decode(gpu, clipset, options, stream=None, prefill=None):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    req_clip, req_time = _requests()
    width = 12 if options.output_layout == ab.LAYOUT_QVV48 else 10
    if prefill is None:
        d_out = torch.full((len(req_clip), clipset.max_tracks, width), float("nan"), dtype=torch.float32, device="cuda")
    else:
        d_out = torch.full((len(req_clip), clipset.max_tracks, width), prefill, dtype=torch.float32, device="cuda")
    ctx.decompress_tracks(clipset, _to_device(gpu, ab.make_requests(req_clip, req_time)), len(req_clip), options, d_out, stream)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    if width == 10:     # QVV40 -> the 12 float rows of the reference writer
        wide = np.zeros(out.shape[:2] + (12,), np.float32)
        wide[..., [0, 1, 2, 3, 4, 5, 6, 8, 9, 10]] = out
        out = wide
    return out


def _want(gpu, state, clip, t, rounding, looping):
    return gpu["reference"].poses(state, clip, t, rounding, looping)


def _check_state(gpu, clipset, state, layouts=(0,), roundings=ROUNDINGS, loopings=None):
    ab, reference = gpu["ab"], gpu["reference"]
    req_clip, req_time = _requests()
    loopings = loopings or (ab.LOOP_CLAMP, ab.LOOP_WRAP, ab.LOOP_AS_COMPRESSED)
    for layout in layouts:
        for rounding in roundings:
            for looping in loopings:
                if not reference.has(looping):
                    continue
                got = _decode(gpu, clipset, _options(gpu, rounding_policy=rounding, looping_policy=looping, output_layout=layout))
                for i, (clip, t) in enumerate(zip(req_clip, req_time)):
                    want = _want(gpu, state, int(clip), t, rounding, looping)
                    n = want.shape[0]
                    assert clips.bit_equal(got[i, :n][:, LANES], want[:, LANES]), (state, layout, rounding, looping, int(clip), float(t))


def _upload(gpu, database_blob=None):
    ctx, reference = gpu["ctx"], gpu["reference"]
    clipset = ctx.upload(reference.bound + [reference.plain], check_hash=True)
    database = ctx.upload_database(reference.database if database_blob is None else database_blob, check_hash=True)
    clipset.bind_database(database)
    return clipset, database


def _apply(database, ops):
    for op, tier, n in ops:
        (database.stream_in if op == IN else database.stream_out)(tier, n)


def test_parity_in_every_tier_state(gpu):
    clipset, database = _upload(gpu)
    info = database.info()
    assert info.num_chunks[0] >= 2 and info.num_chunks[1] >= 1, "the fixture must give several chunks"
    done = []
    for name, ops in cases.STATES.items():
        _apply(database, ops[len(done):])
        done = ops
        _check_state(gpu, clipset, name, layouts=(0, 1) if name in ("some_medium", "all_medium_low") else (0,))


def test_decompress_track_and_request_policies(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset, database = _upload(gpu)
    _apply(database, cases.STATES["all_medium_low"])
    req_clip, req_time = _requests()
    for bone in (0, 5, 7):
        requests = ab.make_requests(req_clip, req_time)
        d_out = torch.zeros((len(req_clip), 12), dtype=torch.float32, device="cuda")
        ctx.decompress_track(clipset, _to_device(gpu, requests), _to_device(gpu, np.full(len(req_clip), bone, np.uint32)), len(req_clip),
                             _options(gpu), d_out)
        torch.cuda.synchronize()
        single = d_out.cpu().numpy()
        for i, (clip, t) in enumerate(zip(req_clip, req_time)):
            want = _want(gpu, "all_medium_low", int(clip), t, 0, ab.LOOP_AS_COMPRESSED)[bone]
            assert np.max(np.abs(single[i, :4] - want[:4])) <= SINGLE_TRACK_TOLERANCE, (bone, int(clip), float(t))
            assert clips.bit_equal(single[i, [4, 5, 6, 8, 9, 10]], want[[4, 5, 6, 8, 9, 10]]), (bone, int(clip), float(t))
    # per request (rounding, looping) pairs need per_track_rounding == 0, a decode the reference's per track settings do not make: each
    # row must equal the same launch with that pair batch wide
    rng = np.random.default_rng(5)
    pairs = np.stack([rng.integers(0, 4, len(req_clip)), rng.integers(0, 3, len(req_clip))], axis=1).astype(np.uint8)
    d_pairs = _to_device(gpu, pairs)
    options = _options(gpu, d_request_policies=d_pairs.data_ptr())
    options.per_track_rounding = 0
    got = _decode(gpu, clipset, options)
    for rounding in range(4):
        for looping in range(3):
            batch = _options(gpu, rounding_policy=rounding, looping_policy=looping)
            batch.per_track_rounding = 0
            want = _decode(gpu, clipset, batch)
            rows = (pairs[:, 0] == rounding) & (pairs[:, 1] == looping)
            assert got[rows].tobytes() == want[rows].tobytes(), (rounding, looping)


def test_database_kernels_follow_the_plain_kernels_options(gpu):
    """Every option the plain kernels take (normalisation, per track rounding, default modes and values, skip masks, math mode, layout)
    on the database kernels. A launch with tiers streamed in takes the database kernels for every clip of the set: the rows of the clip
    without a database must match, byte for byte, the plain kernels on an unbound clip set, over the whole option matrix. The database
    clips' rows are compared with the reference (debug settings) in both layouts."""
    torch, ab, ctx, reference = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["reference"]
    unbound = ctx.upload(reference.bound + [reference.plain])
    clipset, database = _upload(gpu)
    database.stream_in(MEDIUM)
    database.stream_in(LOW)
    skip_mask = torch.from_numpy(np.tile(np.array([0, 1, 2, 4, 6], np.uint8), 8)).cuda()
    variable = torch.from_numpy(np.random.default_rng(3).standard_normal((40, 12)).astype(np.float32)).cuda()
    per_track = torch.from_numpy(np.tile(np.array([0, 1, 2, 3], np.uint8), 10)).cuda()
    matrix = []
    for kind in (0, 1, 3, 4):
        matrix.append(dict(kind=kind))
    matrix += [dict(kind=1, math_mode=ab.MATH_FAST), dict(kind=4, math_mode=ab.MATH_FAST),
               dict(kind=1, default_modes=(ab.DEFAULT_SKIPPED, ab.DEFAULT_SKIPPED, ab.DEFAULT_SKIPPED)),
               dict(kind=1, default_modes=(ab.DEFAULT_VARIABLE, ab.DEFAULT_VARIABLE, ab.DEFAULT_VARIABLE), d_variable_defaults=variable.data_ptr()),
               dict(kind=1, default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_CONSTANT, ab.DEFAULT_CONSTANT), constant_defaults=np.arange(12, dtype=np.float32)),
               dict(kind=1, skip_mask=ab.SKIP_TRANSLATION), dict(kind=1, d_skip_track_mask=skip_mask.data_ptr()),
               dict(kind=1, rounding_policy=ab.ROUND_PER_TRACK, d_per_track_rounding=per_track.data_ptr())]
    for entry in matrix:
        entry = dict(entry)
        kind = entry.pop("kind")
        for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
            options = _options(gpu, kind, output_layout=layout, **entry)
            got = _decode(gpu, clipset, options, prefill=7.0)
            plain = _decode(gpu, unbound, options, prefill=7.0)
            req_clip, _ = _requests()
            if options.math_mode == ab.MATH_FAST:
                # the unbound launch takes the pipeline kernel, whose fast math rotations sit within 1e-5 of the exact ones
                assert np.allclose(got[req_clip == 4], plain[req_clip == 4], rtol=0, atol=1e-5), (kind, entry, layout)
            else:
                assert got[req_clip == 4].tobytes() == plain[req_clip == 4].tobytes(), (kind, entry, layout)
    _check_state(gpu, clipset, "all_medium_low", layouts=(0, 1), loopings=(ab.LOOP_AS_COMPRESSED,))


def test_nothing_streamed_in_matches_the_unbound_clip_set(gpu):
    ctx, reference = gpu["ctx"], gpu["reference"]
    unbound = ctx.upload(reference.bound + [reference.plain])
    clipset, database = _upload(gpu)
    for rounding in range(4):
        options = _options(gpu, rounding_policy=rounding)
        assert _decode(gpu, unbound, options).tobytes() == _decode(gpu, clipset, options).tobytes()
    database.stream_in(MEDIUM, 1)
    database.stream_out(MEDIUM, ALL)
    assert database.loaded_chunks(MEDIUM) == 0
    assert _decode(gpu, unbound, _options(gpu)).tobytes() == _decode(gpu, clipset, _options(gpu)).tobytes()


def test_stream_order_on_one_stream(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset, database = _upload(gpu)
    stream = torch.cuda.Stream()
    req_clip, req_time = _requests()
    d_requests = _to_device(gpu, ab.make_requests(req_clip, req_time))
    options = _options(gpu)
    outs = [torch.zeros((len(req_clip), clipset.max_tracks, 12), dtype=torch.float32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    ctx.decompress_tracks(clipset, d_requests, len(req_clip), options, outs[0], stream)
    database.stream_in(MEDIUM, ALL, stream=stream)
    database.stream_in(LOW, ALL, stream=stream)
    ctx.decompress_tracks(clipset, d_requests, len(req_clip), options, outs[1], stream)
    stream.synchronize()
    before, after = outs[0].cpu().numpy(), outs[1].cpu().numpy()
    for i, (clip, t) in enumerate(zip(req_clip, req_time)):
        for got, state in ((before, "nothing"), (after, "all_medium_low")):
            want = _want(gpu, state, int(clip), t, 0, ab.LOOP_AS_COMPRESSED)
            assert clips.bit_equal(got[i, :want.shape[0]][:, LANES], want[:, LANES]), (state, int(clip), float(t))


def test_lifetime_stream_out_and_in_again(gpu):
    clipset, database = _upload(gpu)
    info = database.info()
    assert database.stream_in(MEDIUM) == info.num_chunks[0] and database.is_streamed_in(MEDIUM)
    assert database.stream_in(MEDIUM) == 0          # nothing left to stream
    assert database.stream_out(MEDIUM) == info.num_chunks[0] and database.loaded_chunks(MEDIUM) == 0
    assert database.stream_out(MEDIUM) == 0
    database.stream_in(MEDIUM, 1)
    database.stream_in(MEDIUM)
    _check_state(gpu, clipset, "all_medium")


def test_rejections(gpu):
    torch, ab, ctx, reference = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["reference"]
    blob = reference.database

    def status_of(data, check_hash=True):
        try:
            ctx.upload_database(gpu["ref"].aligned_blob(data), check_hash=check_hash).release()
            return 0
        except ab.AclB200Error as err:
            return err.status

    assert status_of(blob) == 0
    bad = blob.copy(); bad[8] ^= 0xFF                                   # tag
    assert status_of(bad) == 2
    bad = blob.copy(); bad[12:14] = np.frombuffer(np.uint16(99).tobytes(), np.uint8)   # version
    assert status_of(bad, check_hash=False) == 2
    bad = blob.copy(); bad[-70] ^= 0x40                                  # hash
    assert status_of(bad) == 2 and status_of(bad, check_hash=False) == 0
    assert status_of(blob[:blob.size // 2], check_hash=False) == 2         # truncated
    bad = blob.copy(); bad[68:72] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)   # first medium chunk offset
    assert status_of(bad, check_hash=False) == 2
    bad = blob.copy(); bad[32:36] = np.frombuffer(np.uint32(1 << 28).tobytes(), np.uint8)      # num_segments
    assert status_of(bad, check_hash=False) == 2

    # a clip the database does not contain (another database's clip), reported by index
    clipset = ctx.upload([reference.plain, reference.bound[0], reference.other_clip])
    database = ctx.upload_database(blob)
    with pytest.raises(ab.AclB200Error) as err:
        clipset.bind_database(database)
    assert err.value.status == 2 and err.value.failed_clip == 2

    # a tier with no chunks (the other database has a medium tier only), a tier that does not exist, a short bulk data array
    other = ctx.upload_database(reference.other_database)
    assert other.info().num_chunks[1] == 0
    with pytest.raises(ab.AclB200Error) as err:
        other.stream_in(LOW)
    assert err.value.status == 1
    with pytest.raises(ab.AclB200Error) as err:
        other.stream_out(LOW)
    assert err.value.status == 1
    clipset, database = _upload(gpu)
    with pytest.raises(ab.AclB200Error) as err:
        database.stream_in(0)
    assert err.value.status == 1
    with pytest.raises(ValueError):
        database.stream_in(MEDIUM, bulk_data=np.zeros(16, np.uint8))

    # measurement and debug entry points refuse a clip set with tiers streamed in, and accept it again once they are out
    req_clip, req_time = _requests()
    d_requests = _to_device(gpu, ab.make_requests(req_clip, req_time))
    d_seek = torch.zeros((len(req_clip), 14), dtype=torch.int32, device="cuda")
    jobs = np.zeros(1, ab.ERROR_JOB_DTYPE)
    jobs["clip"], jobs["num_samples"], jobs["sample_rate"], jobs["duration"], jobs["num_tracks"] = 0, 2, 30.0, 1.0 / 30.0, 12
    d_raw = torch.zeros((2, clipset.max_tracks, 12), dtype=torch.float32, device="cuda")
    d_parents = torch.from_numpy(np.full(clipset.max_tracks, 0xFFFFFFFF, np.uint32).view(np.int32)).cuda()
    d_shell = torch.ones(clipset.max_tracks, dtype=torch.float32, device="cuda")
    d_errors = torch.zeros(4, dtype=torch.int32, device="cuda")
    database.stream_in(MEDIUM, 1)
    for call in (lambda: ctx.debug_seek(clipset, d_requests, len(req_clip), _options(gpu), d_seek),
                 lambda: ctx.debug_unpack(clipset, d_requests, len(req_clip), _options(gpu), 0, 4, d_seek),
                 lambda: ctx.decompress_all_samples(clipset, jobs, _options(gpu), d_seek),
                 lambda: ctx.calculate_compression_error(clipset, jobs, d_raw, d_parents, d_shell, _options(gpu), d_errors)):
        with pytest.raises(ab.AclB200Error) as err:
            call()
        assert err.value.status == 3
    database.stream_out(MEDIUM)
    ctx.debug_seek(clipset, d_requests, len(req_clip), _options(gpu), d_seek)
    ctx.calculate_compression_error(clipset, jobs, d_raw, d_parents, d_shell, _options(gpu), d_errors)
    torch.cuda.synchronize()
