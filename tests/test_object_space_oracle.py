"""Pins the oracle's matrix object space (aclo_local_to_object_space_matrix: convert_transforms + local_to_object_space of
qvvf_matrix3x4f_transform_error_metric, compression/transform_error_metrics.h:397-436) to the unmodified reference metric run live
(oracle/_ref/libaclref_object_space.so, oracle/object_space.mk), BIT FOR BIT: the metric has no CPU specific step. Poses are the named
clips decoded by the port, plus mirrored clips (scale.x negative on some bones); skeletons are a binary tree, a chain and a star."""
import numpy as np
import pytest

from oracle import object_space as OS
from tests import clips
from tests.test_error_metric_oracle import MIRRORED_CASES, mirrored_spec

ROOT = 0xFFFFFFFF


@pytest.fixture(scope="module")
def matrix_reference(reference):
    if not OS.reference_available():
        pytest.skip("oracle/_ref/libaclref_object_space.so not built (needs the reference tree at build time)")
    return OS.reference_local_to_object_space_matrix


def skeletons(num_tracks: int) -> dict:
    bones = np.arange(num_tracks)
    return dict(tree=np.where(bones == 0, ROOT, (bones - 1) // 2).astype(np.uint32),
                chain=np.where(bones == 0, ROOT, bones - 1).astype(np.uint32),
                star=np.where(bones == 0, ROOT, 0).astype(np.uint32))


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_port_matrix_object_space_matches_live_reference(matrix_reference, oracle_port, name):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    settings = oracle_port.settings_for_kind(1)
    for t in clips.sample_times(spec)[::3]:
        local = oracle_port.transform_decompress_tracks(blob, settings, float(t))
        for skeleton, parents in skeletons(spec.num_tracks).items():
            want = matrix_reference(local, parents)
            got = OS.port_local_to_object_space_matrix(local, parents)
            assert clips.bit_equal(got, want), (name, skeleton, float(t))


@pytest.mark.parametrize("name,negative_scale_pct", MIRRORED_CASES)
def test_port_matrix_object_space_mirrored(reference, matrix_reference, oracle_port, name, negative_scale_pct):
    spec = mirrored_spec(name, negative_scale_pct)
    r = reference.transform_error(spec, reference.compress_transform(spec), 1)
    assert r["lossy_poses"][..., 8:11].min() < 0.0
    for sample in range(0, spec.num_samples, 7):
        for parents in [r["parents"]] + list(skeletons(spec.num_tracks).values()):
            local = r["lossy_poses"][sample]
            assert clips.bit_equal(OS.port_local_to_object_space_matrix(local, parents), matrix_reference(local, parents)), \
                (name, sample)


def test_bad_parent_is_refused(matrix_reference):
    local = np.tile(np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32), (4, 1))
    parents = np.array([ROOT, 0, 3, 0], np.uint32)
    with pytest.raises(RuntimeError):
        OS.port_local_to_object_space_matrix(local, parents)
    with pytest.raises(RuntimeError):
        matrix_reference(local, parents)
