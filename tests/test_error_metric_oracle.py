"""Pins the oracle's restatement of the reference's compression error measurement (SURVEY 8(f1): calculate_compression_error,
includes/acl/compression/impl/track_error.impl.h:166-392 + qvvf_transform_error_metric, compression/transform_error_metrics.h:281-385).

  * against the reference run live (oracle/_ref/libaclref.so), BIT FOR BIT: object space poses, every per bone error, the track_error.
    The port then repeats rtm::quat_normalize's rsqrtss + 2 Newton-Raphson steps (normalize mode 0): same CPU, same estimate.
  * against the committed golden numbers (tests/golden/*.error.npz) with a tolerance: they carry the estimate of the CPU that made them.
  * the IEEE 1 / sqrt flavour (normalize mode 1, what the CUDA path computes) stays within ERROR_TOLERANCE of the reference.
"""
import os

import numpy as np
import pytest

from tests import clips
from oracle import port as P

# |error(IEEE normalize) - error(reference)| on the test clips: <= 1.8e-5 measured (object space translations reach ~50 units through 7
# levels of hierarchy, i.e. ~3e-7 relative); the gate leaves a factor of ~3
ERROR_TOLERANCE = 5e-5
LANES = clips.DEFINED_LANES


def error_tolerance(oracle_port, poses, parents) -> float:
    """The gate scaled to the size of the poses: ERROR_TOLERANCE for object space positions up to 50 units from the root, 1e-6 of the
    largest distance beyond (additive clips compound scales: positions reach thousands of units there)."""
    reach = 0.0
    for sample in range(0, poses.shape[0], max(1, poses.shape[0] // 8)):
        obj = oracle_port.local_to_object_space(poses[sample], parents, P.NORMALIZE_IEEE)
        reach = max(reach, float(np.max(np.abs(obj[:, 4:7]))) if obj.size else 0.0)
    return ERROR_TOLERANCE * max(1.0, reach / 50.0)


ADDITIVE_CASES = [("c1_30bones", 1, 60), ("c1_30bones", 2, 17), ("c1_30bones", 3, 1), ("mixed_scale", 1, 17), ("mixed_scale", 2, 1), ("mixed_scale", 3, 75),
                  ("stripped_single", 1, 25), ("stripped_single", 3, 17), ("ragged_17", 2, 47)]


def additive_base_spec(spec, base_samples: int):
    import dataclasses
    return dataclasses.replace(spec, seed=spec.seed + 777, num_samples=base_samples, scale_default_pct=40, scale_constant_pct=30)

GOLDEN_TRANSFORM = [n for n in clips.TRANSFORM_SPECS if os.path.exists(clips.golden_path(n, "error.npz"))]
GOLDEN_SCALAR = [n for n in clips.SCALAR_SPECS if os.path.exists(clips.golden_path(n, "error.npz"))]


def bind_pose_settings(kind: int, num_tracks: int):
    """The settings / writer calculate_compression_error decodes with: debug_track_writer skips default sub-tracks over a buffer that
    initialize_with_defaults() filled with track_desc_transformf::default_value = identity (debug_track_writer.h:75-101)."""
    identity = np.tile(np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], dtype=np.float32), (num_tracks, 1))
    return P.settings_for_kind(kind, default_modes=(P.DEFAULT_VARIABLE,) * 3, variable_defaults=identity)


def lossy_poses_from_port(blob, kind, num_samples, sample_rate, duration, rounding):
    settings = bind_pose_settings(kind, P.num_tracks_of(blob))
    poses = []
    for sample in range(num_samples):
        t = min(np.float32(sample) / np.float32(sample_rate), np.float32(duration))
        poses.append(P.transform_decompress_tracks(blob, settings, float(t), int(rounding)))
    return np.stack(poses) if poses else np.zeros((0, P.num_tracks_of(blob), 12), np.float32)


def kinds_for(spec):
    from oracle import ref
    default_ok = spec.rotation_format == ref.QUATF_DROP_W_VARIABLE and spec.translation_format == ref.VECTOR3F_VARIABLE \
        and spec.scale_format == ref.VECTOR3F_VARIABLE
    return [1] + ([0] if default_ok else [])


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_port_matches_live_reference_bit_for_bit(reference, oracle_port, name):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    for kind in kinds_for(spec):
        r = reference.transform_error(spec, blob, kind)
        # the port's own decode feeds the measurement, as it does for the CUDA path
        lossy = lossy_poses_from_port(blob, kind, spec.num_samples, r["sample_rate"], r["duration"], r["rounding"])
        assert clips.bit_equal(lossy[..., LANES], r["lossy_poses"][..., LANES]), (name, kind)
        got, errors, negative = oracle_port.transform_track_error(r["raw_poses"], lossy, r["sample_rate"], r["duration"], r["parents"],
                                                                  r["shell_distances"], P.NORMALIZE_RTM_SSE2)
        assert not negative
        for stream, poses in ((0, r["raw_poses"]), (1, lossy)):
            for sample in range(spec.num_samples):
                obj = oracle_port.local_to_object_space(poses[sample], r["parents"], P.NORMALIZE_RTM_SSE2)
                assert clips.bit_equal(obj[:, LANES], r["object_poses"][stream, sample][:, LANES]), (name, kind, stream, sample)
        assert clips.bit_equal(errors, r["errors"]), (name, kind)
        assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (r["index"], np.float32(r["error"]), np.float32(r["sample_time"])), (name, kind)

        # the flavour the CUDA path computes
        ieee, ieee_errors, _ = oracle_port.transform_track_error(r["raw_poses"], lossy, r["sample_rate"], r["duration"], r["parents"],
                                                                 r["shell_distances"], P.NORMALIZE_IEEE)
        if errors.size:
            assert float(np.max(np.abs(ieee_errors - r["errors"]))) <= ERROR_TOLERANCE, (name, kind)
        assert abs(ieee.error - r["error"]) <= ERROR_TOLERANCE, (name, kind)
        if ieee.index != 0xFFFFFFFF:
            # the same worst bone, or one the reference puts within the tolerance of its worst
            sample = int(round(ieee.sample_time * r["sample_rate"]))
            assert r["errors"][sample, ieee.index] >= r["error"] - 2 * ERROR_TOLERANCE, (name, kind)


@pytest.mark.parametrize("name,additive_format,base_samples", ADDITIVE_CASES)
def test_port_matches_live_reference_additive(reference, oracle_port, name, additive_format, base_samples):
    """calculate_compression_error with an additive base (track_error.impl.h:573-680) + additive_qvvf_transform_error_metric<format>:
    the clip measured on top of a base clip of another length, all three additive formats."""
    spec = clips.TRANSFORM_SPECS[name]
    r = reference.transform_error_additive(spec, clips.load_blob(name), additive_base_spec(spec, base_samples), additive_format)
    got, errors, negative = oracle_port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                              r["shell_distances"], P.NORMALIZE_RTM_SSE2, r["base_poses"], additive_format)
    assert not negative
    assert clips.bit_equal(errors, r["errors"])
    assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (r["index"], np.float32(r["error"]), np.float32(r["sample_time"]))
    applied = np.stack([oracle_port.apply_additive_to_base(additive_format, r["base_poses"][s], r["raw_poses"][s]) for s in range(spec.num_samples)])
    tolerance = error_tolerance(oracle_port, applied, r["parents"])
    ieee, ieee_errors, _ = oracle_port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                             r["shell_distances"], P.NORMALIZE_IEEE, r["base_poses"], additive_format)
    assert float(np.max(np.abs(ieee_errors - r["errors"]))) <= tolerance
    assert abs(ieee.error - r["error"]) <= tolerance


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS) + ["mirrored"])
def test_port_matrix_metric_matches_live_reference_bit_for_bit(reference, oracle_port, name):
    """qvvf_matrix3x4f_transform_error_metric (transform_error_metrics.h:389-464): matrix_from_qvv, matrix_mul down the hierarchy,
    matrix_mul_point3 of the shell points. No CPU specific step: one flavour, bit for bit."""
    spec = mirrored_spec("mixed_scale", 30) if name == "mirrored" else clips.TRANSFORM_SPECS[name]
    blob = reference.compress_transform(spec) if name == "mirrored" else clips.load_blob(name)
    r = reference.transform_error(spec, blob, 1)
    m = reference.transform_error_matrix(spec, blob)
    for mode in (P.NORMALIZE_RTM_SSE2, P.NORMALIZE_IEEE):       # the normalisation flavour must not matter to this metric
        got, errors, _ = oracle_port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                           r["shell_distances"], mode, metric=1)
        assert clips.bit_equal(errors, m["errors"]), name
        assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (m["index"], np.float32(m["error"]), np.float32(m["sample_time"])), name


MIRRORED_CASES = [("mixed_scale", 30), ("c1_30bones", 20), ("ragged_17", 50), ("single_segment", 100)]


def mirrored_spec(name: str, negative_scale_pct: int):
    """A named clip with scale.x mirrored on some bones: their children go through rtm::qvv_mul's matrix branch (qvvf.h:320-345)."""
    import dataclasses
    spec = clips.TRANSFORM_SPECS[name]
    return dataclasses.replace(spec, negative_scale_pct=negative_scale_pct, scale_default_pct=min(spec.scale_default_pct, 60))


@pytest.mark.parametrize("name,negative_scale_pct", MIRRORED_CASES)
def test_port_matches_live_reference_negative_scale(reference, oracle_port, name, negative_scale_pct):
    spec = mirrored_spec(name, negative_scale_pct)
    blob = reference.compress_transform(spec)
    r = reference.transform_error(spec, blob, 1)
    assert r["raw_poses"][..., 8:11].min() < 0.0
    got, errors, negative = oracle_port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                              r["shell_distances"], P.NORMALIZE_RTM_SSE2)
    assert negative
    for sample in range(0, spec.num_samples, 7):
        obj = oracle_port.local_to_object_space(r["lossy_poses"][sample], r["parents"], P.NORMALIZE_RTM_SSE2)
        assert clips.bit_equal(obj[:, LANES], r["object_poses"][1, sample][:, LANES]), (name, sample)
    assert clips.bit_equal(errors, r["errors"])
    assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (r["index"], np.float32(r["error"]), np.float32(r["sample_time"]))
    ieee, ieee_errors, _ = oracle_port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                             r["shell_distances"], P.NORMALIZE_IEEE)
    assert float(np.max(np.abs(ieee_errors - r["errors"]))) <= error_tolerance(oracle_port, r["raw_poses"], r["parents"])
    # the relative additive format multiplies through rtm::qvv_mul as well
    ra = reference.transform_error_additive(spec, blob, additive_base_spec(spec, 17), 1)
    got, errors, negative = oracle_port.transform_track_error(ra["raw_poses"], ra["lossy_poses"], ra["sample_rate"], ra["duration"], ra["parents"],
                                                              ra["shell_distances"], P.NORMALIZE_RTM_SSE2, ra["base_poses"], 1)
    assert negative and clips.bit_equal(errors, ra["errors"])


@pytest.mark.parametrize("name", GOLDEN_TRANSFORM)
def test_port_matches_golden_errors(oracle_port, name):
    blob = clips.load_blob(name)
    g = np.load(clips.golden_path(name, "error.npz"))
    num_samples = g["raw_poses"].shape[0]
    lossy = lossy_poses_from_port(blob, 1, num_samples, float(g["sample_rate"]), float(g["duration"]), int(g["rounding"]))
    for mode in (P.NORMALIZE_RTM_SSE2, P.NORMALIZE_IEEE):
        got, errors, negative = oracle_port.transform_track_error(g["raw_poses"], lossy, float(g["sample_rate"]), float(g["duration"]),
                                                                  g["parents"], g["shell_distances"], mode)
        assert not negative
        assert float(np.max(np.abs(errors - g["errors"]))) <= ERROR_TOLERANCE, (name, mode)
        assert abs(got.error - float(g["error"])) <= ERROR_TOLERANCE, (name, mode)
        sample = int(round(got.sample_time * float(g["sample_rate"])))
        assert g["errors"][sample, got.index] >= float(g["error"]) - 2 * ERROR_TOLERANCE, (name, mode)


@pytest.mark.parametrize("name", GOLDEN_TRANSFORM)
def test_port_matrix_metric_matches_golden(oracle_port, name):
    """The reference's qvvf_matrix3x4f_transform_error_metric numbers committed with the clip: no CPU specific step, bit for bit."""
    blob = clips.load_blob(name)
    g = np.load(clips.golden_path(name, "error.npz"))
    m = np.load(clips.golden_path(name, "matrix_error.npz"))
    lossy = lossy_poses_from_port(blob, 1, g["raw_poses"].shape[0], float(g["sample_rate"]), float(g["duration"]), int(g["rounding"]))
    got, errors, _ = oracle_port.transform_track_error(g["raw_poses"], lossy, float(g["sample_rate"]), float(g["duration"]), g["parents"],
                                                       g["shell_distances"], P.NORMALIZE_IEEE, metric=1)
    assert clips.bit_equal(errors, m["errors"]), name
    assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (int(m["index"]), np.float32(m["error"]), np.float32(m["sample_time"])), name


def lossy_scalar_from_port(blob, num_samples, sample_rate, duration, rounding):
    settings = P.settings_for_kind(0)
    rows = []
    for sample in range(num_samples):
        t = min(np.float32(sample) / np.float32(sample_rate), np.float32(duration))
        rows.append(P.scalar_decompress(blob, settings, float(t), int(rounding)))
    return np.stack(rows)


@pytest.mark.parametrize("name", list(clips.SCALAR_SPECS))
def test_scalar_port_matches_live_reference(reference, oracle_port, name):
    spec = clips.SCALAR_SPECS[name]
    blob = clips.load_blob(name)
    r = reference.scalar_error(spec, blob)
    lossy = lossy_scalar_from_port(blob, spec.num_samples, r["sample_rate"], r["duration"], r["rounding"])
    components = min(spec.track_type + 1, 4)
    got = oracle_port.scalar_track_error(r["raw_values"], lossy, components, r["sample_rate"], r["duration"])
    assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (r["index"], np.float32(r["error"]), np.float32(r["sample_time"])), name


@pytest.mark.parametrize("name", GOLDEN_SCALAR)
def test_scalar_port_matches_golden(oracle_port, name):
    spec = clips.SCALAR_SPECS[name]
    blob = clips.load_blob(name)
    g = np.load(clips.golden_path(name, "error.npz"))
    lossy = lossy_scalar_from_port(blob, spec.num_samples, float(g["sample_rate"]), float(g["duration"]), int(g["rounding"]))
    got = oracle_port.scalar_track_error(g["raw_values"], lossy, min(spec.track_type + 1, 4), float(g["sample_rate"]), float(g["duration"]))
    # no CPU specific estimate on this path: bit for bit
    assert (got.index, np.float32(got.error), np.float32(got.sample_time)) == (int(g["index"]), np.float32(g["error"]), np.float32(g["sample_time"])), name


def test_object_space_rejects_a_parent_after_its_child(oracle_port):
    pose = np.tile(np.array([0, 0, 0, 1, 1, 2, 3, 0, 1, 1, 1, 0], dtype=np.float32), (3, 1))
    with pytest.raises(RuntimeError):
        oracle_port.local_to_object_space(pose, np.array([0xFFFFFFFF, 2, 0], dtype=np.uint32))
