"""aclb200_calculate_compression_error, aclb200_local_to_object_space and aclb200_decompress_all_samples (error_metric.cu) at the skeleton
shapes, launch sizes, ties, NaN, strides and streams where its own hierarchy walk, plane reuse and arg max keys can go wrong, BIT FOR BIT
against the port (the IEEE flavour, pinned to the reference by tests/test_error_metric_oracle.py): every per bone error of the error
matrix, and the index, error, sample time and flags of every job. NaN errors compare by NaN-ness (the device's NaN bit patterns are not
the CPU's). Fixtures: tests/error_shapes_cases.py, checked on the CPU by tests/test_error_shapes_cases.py."""
import math

import numpy as np
import pytest

from tests import bones_cases, clips
from tests import error_shapes_cases as E

pytestmark = pytest.mark.gpu

LANES = clips.DEFINED_LANES
DEFAULT_CHUNK_BYTES = 1024 << 20


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    props = torch.cuda.get_device_properties(0)
    ctx = ab.Context(0)
    yield dict(torch=torch, ab=ab, port=port, ctx=ctx, num_sms=props.multi_processor_count, optin=props.shared_memory_per_block_optin)
    ctx.set_error_chunk_bytes(DEFAULT_CHUNK_BYTES)


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array)).cuda()


def _options(gpu, pose_stride_bytes=0):
    """The settings calculate_compression_error is handed (the port's decode: tests/error_shapes_cases.decoded), the bind pose as defaults"""
    ab = gpu["ab"]
    s = gpu["port"].settings_for_kind(1).c
    return ab.Options(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                      clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                      default_modes=(ab.DEFAULT_CONSTANT,) * 3, constant_defaults=E.IDENTITY.tolist(), pose_stride_bytes=pose_stride_bytes)


class Call:
    """One calculate_compression_error call of packed jobs, its device buffers allocated (and filled) up front"""

    def __init__(self, gpu, clipset, jobs, pose_floats=None, zero_sample_jobs=()):
        torch = gpu["torch"]
        self.gpu, self.clipset, self.jobs = gpu, clipset, jobs
        self.max_tracks = clipset.max_tracks
        self.p = E.pack(jobs, gpu["ab"].ERROR_JOB_DTYPE, self.max_tracks, pose_floats, zero_sample_jobs)
        self.pose_floats = self.p["raw"].shape[1]
        self.row_floats = self.pose_floats * 4 // 48            # the error matrix row: tracks a pose row holds
        p = self.p
        self.d_raw = _dev(gpu, p["raw"])
        self.d_base = None if p["base"] is None else _dev(gpu, p["base"])
        self.d_parents, self.d_shells = _dev(gpu, p["parents"]), _dev(gpu, p["shells"])
        self.d_outputs = None if p["output_indices"] is None else _dev(gpu, p["output_indices"])
        self.d_errors = torch.full((len(p["jobs"]) * 4,), -7, dtype=torch.int32, device="cuda")
        self.d_matrix = torch.full((max(p["total_rows"], 1), self.row_floats), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

    def enqueue(self, stream=None):
        options = _options(self.gpu, 0 if self.pose_floats == self.max_tracks * 12 else self.pose_floats * 4)
        self.gpu["ctx"].calculate_compression_error(self.clipset, self.p["jobs"], self.d_raw, self.d_parents, self.d_shells, options,
                                                    self.d_errors, d_output_indices=self.d_outputs, d_out_error_matrix=self.d_matrix,
                                                    d_base_poses=self.d_base, stream=stream)

    def run(self):
        self.enqueue()
        self.gpu["torch"].cuda.synchronize()
        return self

    def check(self, label):
        """Every job against the port; jobs without samples give track_error() with no flags; nothing is written beyond a job's tracks"""
        port = self.gpu["port"]
        records = self.d_errors.cpu().numpy().view(self.gpu["ab"].TRACK_ERROR_DTYPE)
        matrix = self.d_matrix.cpu().numpy()
        for job, slot, row in zip(self.jobs, self.p["slots"], self.p["rows"]):
            index, error, sample_time, flags, want = job.expected(port)
            got = matrix[row:row + job.num_samples]
            where = (label, slot)
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(got[:, :job.num_tracks]), nan), where
            assert clips.bit_equal(np.where(nan, 0, got[:, :job.num_tracks]), np.where(nan, 0, want)), where
            assert np.isnan(got[:, job.num_tracks:]).all(), where
            r = records[slot]
            assert (int(r["index"]), _bits(r["error"]), _bits(r["sample_time"]), int(r["flags"])) == \
                (index, _bits(error), _bits(sample_time), flags), (where, (int(r["index"]), float(r["error"]), float(r["sample_time"])), (index, error, sample_time))
        for slot in sorted(set(range(len(records))) - set(self.p["slots"])):
            r = records[slot]
            assert (int(r["index"]), _bits(r["error"]), _bits(r["sample_time"]), int(r["flags"])) == (E.NO_INDEX, 0, 0, 0), (label, slot)
        return records


def _bits(value) -> int:
    return int(np.float32(value).view(np.uint32))


@pytest.mark.parametrize("name", ["c1_30bones", "c2_100bones", "paragon_like"])
def test_every_skeleton_shape(gpu, name):
    """Tree, chain, star, random (extra roots) and late parents (made roots, ERROR_FLAG_INVALID_SKELETON), each with both metrics, in one
    call; at 540 bones the warps of a block drop to 2 (qvvf) and 1 (matrix)"""
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    n = clipset.max_tracks
    if name == "paragon_like":
        assert [E.warps_for(n, E.PLANE_FLOATS[m], gpu["optin"]) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)] == [2, 1]
    rng = np.random.default_rng(10)
    jobs = [E.clip_job(name, 0, bones_cases.skeleton(kind, n, seed), rng, metric)
            for seed, kind in enumerate(bones_cases.SKELETONS) for metric in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    records = Call(gpu, clipset, jobs).run().check(name)
    assert {int(r["flags"]) for r in records} == {0, E.FLAG_INVALID_SKELETON}
    clipset.release()


def test_additive_formats_on_skeletons(gpu):
    """additive_qvvf_transform_error_metric<format> for formats 1-3 on a tree, a chain and a random skeleton (the matrix metric takes no
    additive base)"""
    clipset = gpu["ctx"].upload([clips.load_blob("c1_30bones")])
    rng = np.random.default_rng(11)
    jobs = [E.additive_job("c1_30bones", 0, bones_cases.skeleton(kind, 30, 2), fmt, rng) for kind in ("tree", "chain", "random") for fmt in (1, 2, 3)]
    Call(gpu, clipset, jobs).run().check("additive")
    clipset.release()


def test_mirrored_bones_on_a_chain_across_chunks(gpu):
    """Negative scales on a 100 bone chain: object_transform_slow per stream (raw only, and both streams where the clip does not output
    the bone), in every 32 bone chunk; the matrix metric needs no branch (and raises no flag)"""
    clipset = gpu["ctx"].upload([clips.load_blob("c2_100bones")])
    rng = np.random.default_rng(12)
    jobs = [E.mirrored_chain_job("c2_100bones", 0, rng, metric) for metric in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    records = Call(gpu, clipset, jobs).run().check("mirrored")
    assert [int(r["flags"]) for r in records] == [E.FLAG_NEGATIVE_SCALE, 0]
    clipset.release()


@pytest.mark.parametrize("chunk_poses", [None, 70])
def test_mixed_rigs_in_one_call(gpu, chunk_poses):
    """Jobs of 1, 17, 40 (stripped: sought with `none`), 100 and 540 bones in one call, each with a skeleton of its own, both metrics,
    duplicated, shuffled, and jobs without samples: every job runs at the widest job's plane stride and warp count. With a chunk budget of
    70 poses every job is a launch of its own."""
    ctx = gpu["ctx"]
    names = ["one_bone", "ragged_17", "stripped_single", "c2_100bones", "paragon_like"]
    kinds = ["tree", "late", "chain", "star", "random"]
    clipset = ctx.upload([clips.load_blob(n) for n in names])
    rng = np.random.default_rng(13)
    jobs = []
    for clip, (name, kind) in enumerate(zip(names, kinds)):
        n = clips.TRANSFORM_SPECS[name].num_tracks
        jobs += [E.clip_job(name, clip, bones_cases.skeleton(kind, n, clip), rng, metric) for metric in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    jobs += [jobs[3], jobs[8]]
    jobs = [jobs[i] for i in rng.permutation(len(jobs))]
    if chunk_poses is not None:
        ctx.set_error_chunk_bytes(chunk_poses * clipset.max_tracks * 48)
    try:
        Call(gpu, clipset, jobs, zero_sample_jobs={0: (3, 100), 5: (1, 17)}).run().check(("mixed", chunk_poses))
    finally:
        ctx.set_error_chunk_bytes(DEFAULT_CHUNK_BYTES)
    clipset.release()


def test_grid_stride_sweeps(gpu):
    """At least two passes of the grid-strided kernel for both metrics: one clip, a perturbation of its own per job, the jobs of the two
    metrics interleaved; then local_to_object_space in place over as many poses"""
    torch, ctx, port = gpu["torch"], gpu["ctx"], gpu["port"]
    name = "c1_30bones"
    clipset = ctx.upload([clips.load_blob(name)])
    n, s = clipset.max_tracks, clips.TRANSFORM_SPECS[name].num_samples
    sweep = {m: E.poses_per_sweep(n, E.PLANE_FLOATS[m], gpu["num_sms"], gpu["optin"]) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)}
    jobs_per_metric = math.ceil(2 * max(sweep.values()) / s)
    qvvf = E.strided_sweep_jobs(name, 0, jobs_per_metric, E.METRIC_QVVF, 14)
    matrix = E.strided_sweep_jobs(name, 0, jobs_per_metric, E.METRIC_MATRIX, 15)
    jobs = [job for pair in zip(qvvf, matrix) for job in pair]
    for metric, poses in sweep.items():
        assert sum(j.num_samples for j in jobs if j.metric == metric) >= 2 * poses > 0
    Call(gpu, clipset, jobs).run().check("sweeps")
    clipset.release()

    poses_per_sweep = E.poses_per_sweep(n, E.LOCAL_TO_OBJECT_FLOATS, gpu["num_sms"], gpu["optin"])
    num_poses = 2 * poses_per_sweep + 17
    decoded = np.asarray(E.decoded(name))
    local = E.perturb(np.tile(decoded, (math.ceil(num_poses / s), 1, 1))[:num_poses], np.random.default_rng(16), 0.01)
    parents = bones_cases.skeleton("random", n, 16)
    d_poses = _dev(gpu, local)
    d_flags = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    ctx.local_to_object_space(d_poses, d_poses, num_poses, n, _dev(gpu, parents), d_out_flags=d_flags)
    torch.cuda.synchronize()
    got = d_poses.cpu().numpy()
    assert int(d_flags.item()) == 0
    for pose in range(num_poses):
        assert clips.bit_equal(got[pose][:, LANES], port.local_to_object_space(local[pose], parents, port.NORMALIZE_IEEE)[:, LANES]), pose


def test_exact_ties_keep_the_first_in_sample_then_bone_order(gpu):
    """(a) raw == decoded: every error is +0, the result is sample 0, bone 0. (b) Equal largest errors on bones in different lanes and 32
    bone chunks (raw tracks aliased onto one decoded track through output_indices) and on every sample sought at the clamped duration:
    the first sample, then the first bone, wins."""
    clipset = gpu["ctx"].upload([clips.load_blob("c2_100bones"), clips.load_blob("c1_30bones")])
    jobs = [E.tie_job("c2_100bones", 0, m) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)] + \
           [E.unchanged_job("c1_30bones", 1, m) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    records = Call(gpu, clipset, jobs).run().check("ties")
    for r, job in zip(records[:2], jobs):
        assert (int(r["index"]), np.float32(r["sample_time"])) == (E.TIE_BONES[0], np.float32(job.duration))
    for r in records[2:]:
        assert (int(r["index"]), _bits(r["error"]), _bits(r["sample_time"])) == (0, 0, 0)
    clipset.release()


def test_nan_raw_poses_are_never_kept(gpu):
    """NaN in one bone's rotation (it and its descendants measure NaN), in one sample's root translation (the whole sample), and in every
    raw pose (index 0xFFFFFFFF, error -1): a NaN never wins the arg max, both metrics"""
    clipset = gpu["ctx"].upload([clips.load_blob("c2_100bones")])
    jobs = E.nan_jobs("c2_100bones", 0, E.METRIC_QVVF) + E.nan_jobs("c2_100bones", 0, E.METRIC_MATRIX)
    records = Call(gpu, clipset, jobs).run().check("nan")
    for r in (records[2], records[5]):
        assert (int(r["index"]), float(r["error"]), float(r["sample_time"])) == (E.NO_INDEX, -1.0, 0.0)
    clipset.release()


def test_nan_raw_scalar_values_are_never_kept(gpu):
    """The scalar kernel's `error >= 0` guard: NaN at the clean worst track (the next worst wins), and NaN everywhere (index 0xFFFFFFFF,
    error -1); the error matrix is |raw - decoded| per track"""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    name = "float1"
    clipset = ctx.upload([clips.load_blob(name)])
    assert clipset.components == 1
    raw, lossy, rate, duration = E.scalar_values(name, np.random.default_rng(17))
    clean = port.scalar_track_error(raw, lossy, 1, rate, duration)
    dirty = raw.copy()
    dirty[int(round(clean.sample_time * rate)), clean.index, 0] = np.nan
    everything = raw.copy()
    everything[..., 0] = np.nan
    cases = [raw, dirty, everything]
    s, t = raw.shape[:2]
    jobs = np.zeros(len(cases), ab.ERROR_JOB_DTYPE)
    for i in range(len(cases)):
        jobs[i]["clip"], jobs[i]["num_samples"], jobs[i]["sample_rate"], jobs[i]["duration"] = 0, s, rate, duration
        jobs[i]["num_tracks"], jobs[i]["first_raw_pose"] = t, 1 + i * s
    values = np.concatenate([np.full((1, t), np.nan, np.float32)] + [c[..., 0] for c in cases])
    d_errors = torch.zeros(len(cases) * 4, dtype=torch.int32, device="cuda")
    d_matrix = torch.full((len(cases) * s, t), -3.0, dtype=torch.float32, device="cuda")
    ctx.calculate_compression_error(clipset, jobs, _dev(gpu, values), None, None, ab.Options(), d_errors, d_out_error_matrix=d_matrix)
    torch.cuda.synchronize()
    records = d_errors.cpu().numpy().view(ab.TRACK_ERROR_DTYPE)
    matrix = d_matrix.cpu().numpy()
    for i, values_i in enumerate(cases):
        want = port.scalar_track_error(values_i, lossy, 1, rate, duration)
        r = records[i]
        assert (int(r["index"]), _bits(r["error"]), _bits(r["sample_time"]), int(r["flags"])) == \
            (want.index, _bits(want.error), _bits(want.sample_time), 0), i
        errors = np.abs(values_i[..., 0] - lossy[..., 0])
        got = matrix[i * s:(i + 1) * s]
        assert np.array_equal(np.isnan(got), np.isnan(errors)) and clips.bit_equal(np.nan_to_num(got), np.nan_to_num(errors)), i
    assert (int(records[2]["index"]), float(records[2]["error"])) == (E.NO_INDEX, -1.0)
    clipset.release()


def test_padded_strides_and_permuted_outputs(gpu):
    """A pose stride of 101 tracks and 16 bytes for 100 track rows: raw poses, base poses and the error matrix rows (101 floats) follow
    it; output_indices a permutation; an additive job reads its base at that stride"""
    clipset = gpu["ctx"].upload([clips.load_blob(n) for n in ("c2_100bones", "ragged_17", "c1_30bones")])
    rng = np.random.default_rng(18)
    jobs = [E.permuted_job("c2_100bones", 0, rng, m) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    jobs += [E.additive_job("ragged_17", 1, bones_cases.skeleton("random", 17, 3), 2, rng)]
    jobs += [E.clip_job("c1_30bones", 2, bones_cases.tree(30), rng, m) for m in (E.METRIC_QVVF, E.METRIC_MATRIX)]
    call = Call(gpu, clipset, jobs, pose_floats=101 * 12 + 4)
    assert call.row_floats == 101
    call.run().check("strides")
    clipset.release()


def _all_samples_expected(gpu, blob, job, rounding):
    port = gpu["port"]
    settings = port.settings_for_kind(1, default_modes=(port.DEFAULT_CONSTANT,) * 3, constant_defaults=E.IDENTITY)
    rate, duration = np.float32(job["sample_rate"]), np.float32(job["duration"])
    out = []
    for sample in range(int(job["num_samples"])):
        t = np.float32(sample) / rate
        out.append(port.transform_decompress_tracks(blob, settings, float(min(t, duration)), rounding))
    return out


@pytest.mark.parametrize("rounding", [E.ROUND_NEAREST, E.ROUND_NONE])
def test_decompress_all_samples_clamped_and_fractional_rates(gpu, rounding):
    """Sample i of a job at min(i / sample_rate, duration) with a non-integer rate, durations that clamp the last samples, more samples
    than the clip has, a job without samples, into padded pose rows"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    names = ["c1_30bones", "ragged_17", "stripped_single"]
    blobs = [clips.load_blob(n) for n in names]
    clipset = ctx.upload(blobs)
    rows = [(0, 80, 23.7, 1.5), (1, 47, 29.97, E.clip_duration("ragged_17")), (2, 25, 12.5, 0.9), (0, 0, 30.0, 1.0), (0, 7, 1000.0 / 3.0, 0.01)]
    jobs = np.zeros(len(rows), ab.ERROR_JOB_DTYPE)
    for i, (clip, num_samples, rate, duration) in enumerate(rows):
        jobs[i]["clip"], jobs[i]["num_samples"], jobs[i]["sample_rate"], jobs[i]["duration"] = clip, num_samples, rate, duration
    pose_floats = clipset.max_tracks * 12 + 8
    total = int(jobs["num_samples"].sum())
    d_out = torch.full((total, pose_floats), float("nan"), dtype=torch.float32, device="cuda")
    options = _options(gpu, pose_floats * 4)
    options.rounding_policy = rounding
    ctx.decompress_all_samples(clipset, jobs, options, d_out)
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    pose = 0
    for job in jobs:
        blob = blobs[int(job["clip"])]
        n = gpu["port"].num_tracks_of(blob)
        for want in _all_samples_expected(gpu, blob, job, rounding):
            assert clips.bit_equal(got[pose, :n * 12].reshape(n, 12)[:, LANES], want[:, LANES]), (rounding, int(job["clip"]), pose)
            pose += 1
    assert pose == total
    clipset.release()


def test_two_streams_one_context_measure(gpu):
    """Two calls on two streams, enqueued back to back without synchronising, with the same clips, jobs and buffer sizes (so the same
    scratch layout) and different raw poses: each must give its own results. The context's scratch orders the second after the first."""
    torch, ctx = gpu["torch"], gpu["ctx"]
    name = "c1_30bones"
    clipset = ctx.upload([clips.load_blob(name)])
    calls = []
    for seed, amount in ((20, 0.002), (21, 0.02)):
        jobs = [job for pair in zip(E.strided_sweep_jobs(name, 0, 300, E.METRIC_QVVF, seed, amount),
                                    E.strided_sweep_jobs(name, 0, 300, E.METRIC_MATRIX, seed + 10, amount)) for job in pair]
        calls.append(Call(gpu, clipset, jobs))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for call, stream in zip(calls, streams):
        call.enqueue(stream)
    torch.cuda.synchronize()
    for i, call in enumerate(calls):
        call.check(("stream", i))
    clipset.release()


def test_two_streams_one_context_all_samples(gpu):
    """decompress_all_samples on two streams back to back without synchronising: same clips, jobs, sample counts and buffer sizes, only
    the sample rates differ; each call must decode its own sample times"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    name = "c2_100bones"
    blob = clips.load_blob(name)
    clipset = ctx.upload([blob])
    num_jobs, num_samples = 16, 1000
    options = _options(gpu)
    options.rounding_policy = E.ROUND_NEAREST
    tables, outs = [], []
    for first_rate in (600.0, 500.0):
        jobs = np.zeros(num_jobs, ab.ERROR_JOB_DTYPE)
        jobs["clip"], jobs["num_samples"], jobs["duration"] = 0, num_samples, E.clip_duration(name)
        jobs["sample_rate"] = first_rate + np.arange(num_jobs, dtype=np.float32)
        tables.append(jobs)
        outs.append(torch.full((num_jobs * num_samples, clipset.max_tracks, 12), float("nan"), dtype=torch.float32, device="cuda"))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for jobs, out, stream in zip(tables, outs, streams):
        ctx.decompress_all_samples(clipset, jobs, options, out, stream=stream)
    torch.cuda.synchronize()
    for i, (jobs, out) in enumerate(zip(tables, outs)):
        got = out.cpu().numpy()
        pose = 0
        for job in jobs:
            for want in _all_samples_expected(gpu, blob, job, E.ROUND_NEAREST):
                assert clips.bit_equal(got[pose][:, LANES], want[:, LANES]), (i, pose)
                pose += 1
    clipset.release()
