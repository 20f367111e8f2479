"""Pins the port's root motion (oracle/root_motion_oracle.c: rtm::qvv_inverse, and the composition of aclb200_extract_root_motion over
rtm::qvv_mul) to the unmodified reference (oracle/_ref/libaclref_root_motion.so, oracle/root_motion.mk), bit for bit:
  * rtm::qvv_inverse and rel(a, b) = qvv_mul(T(b), qvv_inverse(T(a))) on the root rows of every named clip, and on mirrored rows, whose
    qvv_mul takes the matrix branch (the normalise flavour of the reference's rsqrtss, as the other mirrored tests);
  * the whole path: the port's decompress_tracks root rows composed by the port against the reference's decompression_context with the
    clamp policy and a root-only track_writer, composed with rtm, over every named clip, settings kind, rounding policy, cycles -3..3 and
    time pairs inside, at and beyond both ends and on key frames;
  * the committed golden fixture (tests/golden/root_motion.golden.npz) reproduces;
  * the convention: for cycles == 0, qvv_mul(M, T(from)) is T(to).
The GPU tests (tests/test_gpu_root_motion.py) pin the library to the port's composition."""
import numpy as np
import pytest

from oracle import root_motion as RM
from tests import clips
from tests import root_motion_cases as cases
from tests.test_error_metric_oracle import MIRRORED_CASES, mirrored_spec

LANES = clips.DEFINED_LANES


@pytest.fixture(scope="module")
def rm_reference(reference):
    if not RM.reference_available():
        pytest.skip("oracle/_ref/libaclref_root_motion.so not built (needs the reference tree at build time)")
    return RM


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_port_inverse_and_composition_match_rtm(rm_reference, oracle_port, name):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    settings = oracle_port.settings_for_kind(cases.kinds_for(spec)[0])
    times = clips.sample_times(spec)
    rows = [oracle_port.transform_decompress_tracks(blob, settings, float(t), 0, oracle_port.LOOP_CLAMP) for t in times]
    bones = sorted({0, spec.num_tracks // 2, spec.num_tracks - 1})
    for bone in bones:
        samples = [r[bone] for r in rows]
        for a, row in enumerate(samples):
            assert clips.bit_equal(RM.port_qvv_inverse(row), RM.reference_qvv_inverse(row)), (name, bone, a)
            b = samples[(a + 5) % len(samples)]
            got = RM.port_qvv_mul(b, RM.port_qvv_inverse(row), RM.NORMALIZE_RTM_SSE2)
            assert clips.bit_equal(got, RM.reference_qvv_mul(b, RM.reference_qvv_inverse(row))), (name, bone, a)
        for i in range(0, len(samples) - 3, 2):
            four = np.stack(samples[i:i + 4])
            for cycles in cases.CYCLES + [cases.CYCLES[-1] * 10]:
                got, negative = RM.port_root_motion(four, cycles, RM.NORMALIZE_RTM_SSE2)
                assert not negative
                assert clips.bit_equal(got, RM.reference_root_motion(four, cycles)), (name, bone, i, cycles)


@pytest.mark.parametrize("name,negative_scale_pct", MIRRORED_CASES)
def test_port_composition_mirrored(reference, rm_reference, name, negative_scale_pct):
    """Rows with a negative scale, compressed and decoded by the reference: every qvv_mul takes the matrix branch"""
    spec = mirrored_spec(name, negative_scale_pct)
    r = reference.transform_error(spec, reference.compress_transform(spec), 1)
    poses = r["lossy_poses"]
    mirrored = [b for b in range(spec.num_tracks) if (poses[:, b, 8:11] < 0).any()]
    assert mirrored
    for bone in mirrored[:6]:
        samples = poses[:, bone]
        for i in range(0, spec.num_samples - 3, 5):
            four = samples[i:i + 4]
            for cycles in cases.CYCLES:
                got, negative = RM.port_root_motion(four, cycles, RM.NORMALIZE_RTM_SSE2)
                assert negative == bool((four[:, 8:11] < 0).any()), (name, bone, i, cycles)
                assert clips.bit_equal(got, RM.reference_root_motion(four, cycles)), (name, bone, i, cycles)


def _roundings(kind):
    return [(r, None) for r in range(4)] + ([(4, np.arange(64, dtype=np.uint8) % 4)] if kind == 1 else [])


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_end_to_end_matches_reference_harness(rm_reference, oracle_port, name):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    roots = sorted({0, spec.num_tracks - 1})
    for kind in cases.kinds_for(spec):
        for rounding, per_track in _roundings(kind):
            policies = None if per_track is None else np.resize(per_track, spec.num_tracks).astype(np.uint8)
            settings = oracle_port.settings_for_kind(kind, per_track_policies=policies)
            duration = cases.clamp_duration(oracle_port, blob, settings)
            for root in roots:
                for from_time, to_time in cases.time_pairs(spec, duration)[::2 if kind != 1 else 1]:
                    samples = cases.port_samples(oracle_port, blob, settings, rounding, root, from_time, to_time, duration)
                    for cycles in cases.CYCLES:
                        want, ref_samples = RM.reference_extract(blob, kind, 0, rounding, root, from_time, to_time, cycles, per_track_rounding=policies)
                        context = (name, kind, rounding, root, from_time, to_time, cycles)
                        assert clips.bit_equal(samples[:, LANES], ref_samples[:, LANES]), context
                        got, _ = RM.port_root_motion(samples, cycles, RM.NORMALIZE_RTM_SSE2)
                        assert clips.bit_equal(got, want), context


@pytest.mark.parametrize("name", ["mixed_scale", "ragged_17", "full_formats"])
def test_end_to_end_with_writer_defaults(rm_reference, oracle_port, name):
    """Constant and variable default sub-tracks of the writer (the root's default sub-tracks take them)"""
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    rng = np.random.default_rng(5)
    constant = cases.IDENTITY.copy()
    constant[4:7] = rng.uniform(-1, 1, 3)
    constant[8:11] = rng.uniform(0.5, 1.5, 3)
    variable = np.tile(cases.IDENTITY, (spec.num_tracks, 1))
    variable[:, 4:7] = rng.uniform(-2, 2, (spec.num_tracks, 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (spec.num_tracks, 3))
    for writer in (2, 3):
        settings = oracle_port.settings_for_kind(1, default_modes=oracle_port.writer_modes(writer), constant_defaults=constant,
                                                 variable_defaults=variable)
        duration = cases.clamp_duration(oracle_port, blob, settings)
        for root in range(spec.num_tracks):
            for from_time, to_time in cases.time_pairs(spec, duration)[::4]:
                samples = cases.port_samples(oracle_port, blob, settings, 0, root, from_time, to_time, duration)
                for cycles in (-2, 0, 1):
                    want, _ = RM.reference_extract(blob, 1, writer, 0, root, from_time, to_time, cycles, constant_defaults=constant,
                                                   variable_defaults=variable)
                    got, _ = RM.port_root_motion(samples, cycles, RM.NORMALIZE_RTM_SSE2)
                    assert clips.bit_equal(got, want), (name, writer, root, from_time, to_time, cycles)


def test_golden_fixture_reproduces(rm_reference):
    """tests/golden/make_root_motion_golden.py wrote the reference's M for its request list: the reference built here still gives it"""
    from tests.golden import make_root_motion_golden as make
    g = np.load(clips.golden_path("root_motion", "golden.npz"))
    want = make.compute()
    assert set(g.files) == set(want)
    for key in g.files:
        assert np.array_equal(g[key].view(np.uint8), np.ascontiguousarray(want[key]).view(np.uint8)), key


@pytest.mark.parametrize("name", ["c1_30bones", "noisy_raw", "half_turn", "looping", "stripped_loop"])
def test_delta_convention(oracle_port, name):
    """cycles == 0: T(to) = qvv_mul(M, T(from)), the engine's M <- qvv_mul(delta, M), within 1e-5. qvv products compose exactly only
    with a uniform scale (a non-uniform one would need shear, rtm/qvvf.h:310-314): these roots have scale 1."""
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    settings = oracle_port.settings_for_kind(1)
    duration = cases.clamp_duration(oracle_port, blob, settings)
    for root in sorted({0, spec.num_tracks - 1}):
        for from_time, to_time in cases.time_pairs(spec, duration):
            samples = cases.port_samples(oracle_port, blob, settings, 0, root, from_time, to_time, duration)
            assert (samples[:, 8:11] == 1.0).all(), (name, root)
            motion, _ = RM.port_root_motion(samples, 0)
            reached = RM.port_qvv_mul(motion, samples[0])
            assert np.allclose(reached[LANES], samples[1][LANES], rtol=1e-5, atol=1e-5), (name, root, from_time, to_time)
