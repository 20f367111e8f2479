"""Pins the oracle's skinning rows (oracle/skinning_oracle.c: the matrix walk of qvvf_matrix3x4f_transform_error_metric, then
rtm::matrix_mul(inverse_bind, object)) to the unmodified reference run live (oracle/_ref/libaclref_skinning.so) BIT FOR BIT: every step is
an IEEE multiply or add in a fixed order. Where the reference is absent, tests/golden/skinning.golden.npz pins the port instead. The order
and layout tests check what the rows mean, in float64, independently of both."""
import numpy as np
import pytest

from oracle import skinning
from tests import clips, skinning_cases as cases

GOLDEN = clips.golden_path("skinning", "golden.npz")


@pytest.fixture(scope="module")
def skinning_reference():
    if not skinning.reference_available():
        pytest.skip("oracle/_ref/libaclref_skinning.so not built (needs the reference tree at build time)")
    return skinning.reference_local_to_skinning


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_port_matches_live_reference(skinning_reference, oracle_port, name):
    """Every named clip's decoded poses, chain / tree / star / random skeletons, bind pose, random and mirrored inverse binds."""
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    settings = oracle_port.settings_for_kind(1)
    times = clips.sample_times(spec)[::4]
    poses = [oracle_port.transform_decompress_tracks(blob, settings, float(t)) for t in times]
    for si, skeleton in enumerate(cases.SKELETONS):
        parents = cases.skeleton(skeleton, spec.num_tracks, seed=si)
        for kind in cases.INVERSE_BIND_KINDS:
            inverse = cases.inverse_binds(kind, spec.num_tracks, poses[0], parents, seed=spec.seed)
            for t, local in zip(times, poses):
                got = skinning.port_local_to_skinning(local, parents, inverse)
                assert np.isfinite(got).all()
                assert clips.bit_equal(got, skinning_reference(local, parents, inverse)), (name, skeleton, kind, float(t))


def test_port_matches_the_golden_rows(oracle_port):
    """The reference's rows stored in skinning.golden.npz, for the port on the stored poses and inverse binds."""
    golden = np.load(GOLDEN)
    count = 0
    for name in cases.GOLDEN_CLIPS:
        local = golden[f"{name}_local"]
        for skeleton in ("tree", "random"):
            parents = golden[f"{name}_{skeleton}_parents"]
            for kind in cases.INVERSE_BIND_KINDS:
                inverse = golden[f"{name}_{skeleton}_{kind}"]
                want = golden[f"{name}_{skeleton}_{kind}_skin"]
                for t in range(local.shape[0]):
                    assert clips.bit_equal(skinning.port_local_to_skinning(local[t], parents, inverse), want[t]), (name, skeleton, kind, t)
                    count += 1
    assert count == len(cases.GOLDEN_CLIPS) * 2 * len(cases.INVERSE_BIND_KINDS) * len(cases.GOLDEN_TIMES)


def test_golden_inputs_are_the_port_decode(oracle_port):
    """The stored poses are the port's decode (itself pinned to the reference), the stored bind inverses those of the first pose."""
    golden = np.load(GOLDEN)
    settings = oracle_port.settings_for_kind(0)
    for name in cases.GOLDEN_CLIPS:
        blob = clips.load_blob(name)
        for t, pose in zip(golden["times"], golden[f"{name}_local"]):
            assert clips.bit_equal(pose, oracle_port.transform_decompress_tracks(blob, settings, float(t)))
        parents = golden[f"{name}_tree_parents"]
        assert clips.bit_equal(golden[f"{name}_tree_bind"], cases.bind_inverse(golden[f"{name}_local"][0], parents))


def _skinned_f64(object_rows, inverse, points):
    """(p, 1) @ inverse_bind @ object in float64: the point a bind pose vertex p moves to"""
    p = np.concatenate([points, np.ones((points.shape[0], 1))], 1)[:, None, :]
    return (p @ cases.to_affine(inverse) @ cases.to_affine(object_rows))[:, 0, :3]


def test_order(oracle_port):
    """The bind pose skinned with its own inverse binds is the identity; another pose skinned with them moves a bind pose vertex p to
    p @ inverse_bind @ object (rtm's row vector order), which object @ inverse_bind does not."""
    from oracle import object_space
    spec = clips.TRANSFORM_SPECS["mixed_scale"]
    blob = clips.load_blob("mixed_scale")
    settings = oracle_port.settings_for_kind(0)
    bind = oracle_port.transform_decompress_tracks(blob, settings, 0.2)
    other = oracle_port.transform_decompress_tracks(blob, settings, 1.1)
    identity_rows = np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32), (spec.num_tracks, 1))
    for skeleton in cases.SKELETONS:
        parents = cases.skeleton(skeleton, spec.num_tracks)
        inverse = cases.bind_inverse(bind, parents)
        rows = skinning.port_local_to_skinning(bind, parents, inverse)
        # float32 rounding grows with the object translations (a 57 bone chain reaches far from its root)
        magnitude = 1.0 + np.abs(object_space.port_local_to_object_space_matrix(bind, parents)).max()
        np.testing.assert_allclose(rows, identity_rows, atol=4e-6 * magnitude, err_msg=skeleton)

        rows = skinning.port_local_to_skinning(other, parents, inverse).reshape(-1, 3, 4)
        points = np.random.default_rng(3).uniform(-1.0, 1.0, (spec.num_tracks, 3))
        got = np.einsum("bcj,bj->bc", rows.astype(np.float64), np.concatenate([points, np.ones((spec.num_tracks, 1))], 1))
        object_rows = object_space.port_local_to_object_space_matrix(other, parents)
        want = _skinned_f64(object_rows, inverse, points)
        scale = 1.0 + np.abs(want).max()
        assert np.abs(got - want).max() <= 1e-4 * scale, skeleton
        p = np.concatenate([points, np.ones((spec.num_tracks, 1))], 1)[:, None, :]
        swapped = (p @ cases.to_affine(object_rows) @ cases.to_affine(inverse))[:, 0, :3]
        assert np.abs(got - swapped).max() > 1e-2 * scale, skeleton


@pytest.mark.parametrize("kind", cases.INVERSE_BIND_KINDS)
def test_layout(oracle_port, kind):
    """dot(row c, (p, 1)) of the rows is component c of the skinned point: against float64 arithmetic always, and against the reference's
    rtm::matrix_mul_point3(p, skin) where it was built."""
    from oracle import object_space
    spec = clips.TRANSFORM_SPECS["c2_100bones"]
    blob = clips.load_blob("c2_100bones")
    settings = oracle_port.settings_for_kind(0)
    local = oracle_port.transform_decompress_tracks(blob, settings, 0.7)
    parents = cases.skeleton("random", spec.num_tracks, seed=5)
    inverse = cases.inverse_binds(kind, spec.num_tracks, oracle_port.transform_decompress_tracks(blob, settings, 0.0), parents, seed=9)
    points = np.random.default_rng(4).uniform(-2.0, 2.0, (spec.num_tracks, 3)).astype(np.float32)
    rows = skinning.port_local_to_skinning(local, parents, inverse).reshape(-1, 3, 4)
    got = np.einsum("bcj,bj->bc", rows.astype(np.float64), np.concatenate([points, np.ones((spec.num_tracks, 1), np.float32)], 1))
    want = _skinned_f64(object_space.port_local_to_object_space_matrix(local, parents), inverse, points.astype(np.float64))
    scale = 1.0 + np.abs(want).max()
    assert np.abs(got - want).max() <= 1e-4 * scale
    assert clips.bit_equal(skinning.rows_to_axes(rows.reshape(-1, 12)).reshape(-1, 12)[:, 9:12], rows[:, :, 3])
    if skinning.reference_available():
        reference_points = skinning.reference_skinned_points(local, parents, inverse, points)
        assert np.abs(got - reference_points).max() <= 1e-4 * scale


def test_bad_parent_is_refused():
    local = np.tile(np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32), (4, 1))
    parents = np.array([cases.ROOT, 0, 3, 0], np.uint32)
    inverse = cases.random_affine(4, 0)
    with pytest.raises(RuntimeError):
        skinning.port_local_to_skinning(local, parents, inverse)
    if skinning.reference_available():
        with pytest.raises(RuntimeError):
            skinning.reference_local_to_skinning(local, parents, inverse)
