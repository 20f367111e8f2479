"""CPU checks of the fixtures of tests/test_gpu_error_shapes.py (tests/error_shapes_cases.py): each builds the case it claims to build,
as the port sees it."""
import numpy as np
import pytest

from tests import bones_cases, clips
from tests import error_shapes_cases as E


@pytest.mark.parametrize("name", [n for n in clips.TRANSFORM_SPECS if n in ("c1_30bones", "ragged_17", "one_bone", "stripped_single", "mixed_scale")])
def test_rounding_is_the_one_the_reference_measured_with(name):
    assert E.rounding_of(clips.load_blob(name)) == int(np.load(clips.golden_path(name, "error.npz"))["rounding"])


def test_scalar_clips_are_sought_with_nearest():
    for name in ("float1", "float4"):
        assert int(np.load(clips.golden_path(name, "error.npz"))["rounding"]) == E.ROUND_NEAREST


def test_warps_and_sweeps_follow_the_launch_rule():
    optin = 227 * 1024          # sharedMemPerBlockOptin of an H100
    qvvf, matrix = E.PLANE_FLOATS[E.METRIC_QVVF], E.PLANE_FLOATS[E.METRIC_MATRIX]
    assert (E.warps_for(540, qvvf, optin), E.warps_for(540, matrix, optin)) == (2, 1)
    assert (E.warps_for(30, qvvf, optin), E.warps_for(100, matrix, optin), E.warps_for(540, E.LOCAL_TO_OBJECT_FLOATS, optin)) == (8, 8, 4)
    assert E.poses_per_sweep(30, qvvf, 132, optin) == 132 * 32 * 8
    assert E.warps_for(3000, matrix, optin) == 0


@pytest.mark.parametrize("kind", bones_cases.SKELETONS)
def test_skeleton_jobs_run_through_the_port(oracle_port, kind):
    rng = np.random.default_rng(1)
    for name in ("c1_30bones", "c2_100bones"):
        n = E.decoded(name).shape[1]
        for metric in (E.METRIC_QVVF, E.METRIC_MATRIX):
            job = E.clip_job(name, 0, bones_cases.skeleton(kind, n, 3), rng, metric)
            index, error, sample_time, flags, errors = job.expected(oracle_port)
            assert flags == (E.FLAG_INVALID_SKELETON if kind == "late" else 0)
            assert np.isfinite(errors).all() and error > 0 and index < n
            assert error == errors.max() and errors[int(round(float(sample_time) * 30)), index] == error


def test_mirrored_chain_takes_the_matrix_branch(oracle_port):
    job = E.mirrored_chain_job("c2_100bones", 0, np.random.default_rng(2))
    assert job.expected(oracle_port)[3] == E.FLAG_NEGATIVE_SCALE
    # a bone the clip does not output is compared with its raw value: mirrored in both streams
    assert job.lossy[0, 31, 8] < 0 and job.raw[0, 32, 8] < 0 < job.lossy[0, 32, 8]
    assert E.invalid_order(job.parents) is False and job.parents[99] == 98


@pytest.mark.parametrize("additive_format", [1, 2, 3])
def test_additive_jobs_measure_finite_errors(oracle_port, additive_format):
    job = E.additive_job("c1_30bones", 0, bones_cases.skeleton("random", 30, 4), additive_format, np.random.default_rng(3))
    index, error, _, flags, errors = job.expected(oracle_port)
    assert flags == 0 and np.isfinite(errors).all() and error > 0
    # the device measures against what it decodes: the fixture may change raw and base poses only
    assert np.array_equal(job.lossy, E.decoded("c1_30bones"))


@pytest.mark.parametrize("metric", [E.METRIC_QVVF, E.METRIC_MATRIX])
def test_tie_job_is_exactly_the_intended_tie(oracle_port, metric):
    job = E.tie_job("c2_100bones", 0, metric)
    index, error, sample_time, flags, errors = job.expected(oracle_port)
    ties = set(zip(*np.nonzero(errors == errors.max())))
    assert ties == E.tie_positions(job.num_samples)
    # across lanes and 32 bone chunks, and across samples sought at the same (clamped) time
    assert len({b % 32 for b in E.TIE_BONES}) == len(E.TIE_BONES) and len({b // 32 for b in E.TIE_BONES}) == 3
    assert E.TIE_DURATION_SAMPLES < job.num_samples - 1 and job.duration < (job.num_samples - 1) / job.sample_rate
    assert (index, sample_time, flags) == (E.TIE_BONES[0], np.float32(job.duration), 0) and error == errors.max() > 0
    # the tie is at the largest error only: the bones' errors before the clamped samples are not
    assert errors[:E.TIE_DURATION_SAMPLES].max() < error


@pytest.mark.parametrize("metric", [E.METRIC_QVVF, E.METRIC_MATRIX])
def test_unchanged_job_measures_plus_zero_everywhere(oracle_port, metric):
    job = E.unchanged_job("c1_30bones", 0, metric)
    index, error, sample_time, flags, errors = job.expected(oracle_port)
    assert np.array_equal(errors.view(np.uint32), np.zeros_like(errors).view(np.uint32))
    assert (index, error.view(np.uint32), sample_time, flags) == (0, 0, 0.0, 0)


@pytest.mark.parametrize("metric", [E.METRIC_QVVF, E.METRIC_MATRIX])
def test_nan_jobs_spread_to_descendants_and_are_never_kept(oracle_port, metric):
    one_bone, one_sample, everything = E.nan_jobs("c2_100bones", 0, metric)
    _, _, _, _, errors = one_bone.expected(oracle_port)
    nan = np.zeros_like(errors, bool)
    nan[E.NAN_BONE_SAMPLE, sorted(E.descendants(one_bone.parents, E.NAN_BONE))] = True
    assert np.array_equal(np.isnan(errors), nan) and nan.sum() > 1
    _, _, _, _, errors = one_sample.expected(oracle_port)
    assert np.isnan(errors[E.NAN_SAMPLE]).all() and np.isnan(errors).sum() == errors.shape[1]
    index, error, sample_time, _, errors = everything.expected(oracle_port)
    assert np.isnan(errors).all() and (index, error, sample_time) == (E.NO_INDEX, -1.0, 0.0)


def test_scalar_nan_is_never_kept(oracle_port):
    raw, lossy, rate, duration = E.scalar_values("float1", np.random.default_rng(4))
    components = 1
    clean = oracle_port.scalar_track_error(raw, lossy, components, rate, duration)
    worst = int(round(clean.sample_time * rate)), clean.index
    raw[worst[0], worst[1], 0] = np.nan
    dirty = oracle_port.scalar_track_error(raw, lossy, components, rate, duration)
    assert (dirty.index, dirty.sample_time) != (clean.index, clean.sample_time) and dirty.error < clean.error
    raw[..., 0] = np.nan
    nothing = oracle_port.scalar_track_error(raw, lossy, components, rate, duration)
    assert (nothing.index, nothing.error, nothing.sample_time) == (E.NO_INDEX, -1.0, 0.0)


def test_sweep_jobs_each_have_their_own_worst_track(oracle_port):
    jobs = E.strided_sweep_jobs("c1_30bones", 0, 12, E.METRIC_QVVF, 9)
    worst = [job.expected(oracle_port)[:3] for job in jobs]
    assert len({(w[0], float(w[2])) for w in worst}) >= 10 and len({float(w[1]) for w in worst}) == len(jobs)


def test_permuted_job_compares_each_raw_track_with_its_output(oracle_port):
    job = E.permuted_job("c2_100bones", 0, np.random.default_rng(6))
    perm = job.output_indices.astype(np.int64)
    assert sorted(perm) == list(range(100)) and np.count_nonzero(perm == np.arange(100)) < 10
    assert np.array_equal(job.lossy, np.asarray(E.decoded("c2_100bones"))[:, perm])
    assert 0 < job.expected(oracle_port)[1] < 100


def test_pack_lays_jobs_out_with_gaps_and_offsets():
    from acl_b200.api import ERROR_JOB_DTYPE
    rng = np.random.default_rng(5)
    jobs = [E.clip_job("ragged_17", 1, bones_cases.tree(17), rng), E.clip_job("one_bone", 0, [E.ROOT], rng, E.METRIC_MATRIX)]
    p = E.pack(jobs, ERROR_JOB_DTYPE, 17, pose_floats=17 * 12 + 8, zero_sample_jobs={1: (0, 1)})
    assert p["slots"] == [0, 2] and p["rows"] == [0, 47] and p["total_rows"] == 87 and p["output_indices"] is None
    for job, slot in zip(jobs, p["slots"]):
        e = p["jobs"][slot]
        first = int(e["first_raw_pose"])
        assert np.array_equal(p["raw"][first:first + job.num_samples, :job.num_tracks * 12], job.raw.reshape(job.num_samples, -1))
        assert np.array_equal(p["parents"][e["skeleton_offset"]:e["skeleton_offset"] + job.num_tracks], job.parents)
        assert np.isnan(p["raw"][first - 1]).all() and np.isnan(p["raw"][first:first + job.num_samples, job.num_tracks * 12:]).all()
    assert p["jobs"][1]["num_samples"] == 0
