"""The mirror oracle: the C restatement (oracle/mirror_oracle.c) against the unmodified reference's rtm::quat_mul and quat_mul_vector3
(oracle/ref_mirror.cpp, pinned in tests/golden/mirror.golden.npz) bit for bit; the table helpers of acl_b200.api on a symmetric skeleton;
and mirrored feature and root motion rows against the same compositions run on mirrored local poses, in float64."""
import numpy as np
import pytest

from oracle import mirror as oracle
from tests import mirror_cases as cases


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same(got, want) -> bool:
    """bit for bit, except that a NaN matches any NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    both_nan = np.isnan(got) & np.isnan(want)
    return got.shape == want.shape and bool(np.all((_bits(got) == _bits(want)) | both_nan))


def _port_results():
    from tests.golden import make_mirror_golden
    with np.errstate(all="ignore"):
        return make_mirror_golden.results(reference=False)


@pytest.mark.parametrize("what", ["fabricated", "fabricated_flags", *cases.NAMED_CLIPS])
def test_port_equals_the_pinned_reference(what):
    """Every axis on fabricated poses (+-0, +-inf, NaN, subnormals, non-unit rotations, identity, half turn and general corrections,
    self-partnered rows and entries without a partner) and on the reference decodes of named clips"""
    want = np.load(cases.GOLDEN)[what]
    got = _port_results()[what]
    if what == "fabricated_flags":
        assert np.array_equal(got, want) and (want == oracle.INVALID_MIRROR).all()
        return
    assert _same(got, want), np.argwhere((_bits(got) != _bits(want)) & ~(np.isnan(got) & np.isnan(want)))[:8]


def test_pinned_reference_is_the_live_reference():
    if not oracle.reference_available():
        pytest.skip("needs oracle/_ref/libaclref_mirror.so (the reference tree)")
    from tests.golden import make_mirror_golden
    with np.errstate(all="ignore"):
        live = make_mirror_golden.results(reference=True)
    golden = np.load(cases.GOLDEN)
    for what in golden.files:
        assert _same(live[what], golden[what]), what


def test_row_rules_on_fabricated_rows():
    """The partner rule (a self-partnered row is not flagged; entries without a partner take their own row), the sign flips (+-0 swap,
    the NaN payload of a copied lane kept), the scale bits copied and the w lanes written as 0"""
    table = cases.fabricated_table()
    poses = cases.fabricated_poses()
    for axis in cases.AXES:
        for pose in poses:
            with np.errstate(all="ignore"):
                out, flags = oracle.mirror_pose(pose, table, axis)
            assert flags == oracle.INVALID_MIRROR
            partner = [1, 0, 3, 2, 5, 4, 7, 6, 9, 8, 11, 10, 12, 13, 14, 16, 15, 17, 19, 18, 21, 20, 23, 22]
            for i, m in enumerate(partner):
                assert np.array_equal(_bits(out[i, 8:11]), _bits(pose[m, 8:11])), (axis, i)
            assert (_bits(out[:, [7, 11]]) == 0).all()
            # rows 2 and 3 have identity corrections: the result is the reflection itself, sign bit for sign bit
            for i in (2, 3):
                src = pose[partner[i]]
                want_q = _bits(src[0:4]) ^ np.array([0 if k == axis or k == 3 else 0x80000000 for k in range(4)], np.uint32)
                finite = np.isfinite(src[0:4]).all() and np.isfinite(src[4:7]).all()
                if finite and not (np.abs(src[0:7]) < 1e-30).any():
                    np.testing.assert_allclose(out[i, 0:4], want_q.view(np.float32), rtol=1e-6)
                    want_t = src[4:7] * np.array([-1 if k == axis else 1 for k in range(3)], np.float32)
                    np.testing.assert_allclose(out[i, 4:7], want_t, rtol=1e-6, atol=1e-6)
    # a NaN payload in a scale lane is copied with the lane
    pose = cases.fabricated_poses()[5]
    pose[2, 9] = np.uint32(0x7FC0BEEF).view(np.float32)
    with np.errstate(all="ignore"):
        out, _ = oracle.mirror_pose(pose, table, 0)
    assert _bits(out[3, 9]) == 0x7FC0BEEF


def test_table_helper_mirrors_the_bind_pose_onto_itself():
    import acl_b200 as ab
    parents, mirror, rotations, bind = cases.symmetric_skeleton()
    table = ab.mirror_table(parents, mirror, rotations, ab.MIRROR_X)
    assert table.dtype == ab.MIRROR_ENTRY_DTYPE and table.shape == (parents.size,)
    out, flags = oracle.mirror_pose(bind, table, ab.MIRROR_X)
    assert flags == 0
    # q and -q are the same rotation
    sign = np.sign(np.sum(out[:, 0:4] * bind[:, 0:4], axis=1, keepdims=True))
    np.testing.assert_allclose(out[:, 0:4] * sign, bind[:, 0:4], atol=1e-5)
    np.testing.assert_allclose(out[:, 4:7], bind[:, 4:7], atol=1e-5)
    np.testing.assert_array_equal(out[:, 8:11], bind[:, 8:11])


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_table_helper_mirror_twice_is_the_identity(axis):
    import acl_b200 as ab
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    table = ab.mirror_table(parents, mirror, rotations, axis)
    for pose in cases.random_local_poses(20, parents.size, seed=40 + axis):
        twice, flags = oracle.mirror_pose(oracle.mirror_pose(pose, table, axis)[0], table, axis)
        assert flags == 0
        np.testing.assert_allclose(twice[:, 0:7], pose[:, 0:7], atol=1e-5)


def test_mirrored_object_pose_is_the_reflected_object_pose():
    """Walked to object space, the mirrored pose of bone b is the reflection of bone m(b)'s object transform times b's correction: its
    position is exactly the reflected position"""
    import acl_b200 as ab
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    table = ab.mirror_table(parents, mirror, rotations, ab.MIRROR_X)
    for pose in cases.random_local_poses(10, parents.size, seed=50):
        mirrored, _ = oracle.mirror_pose(pose, table, ab.MIRROR_X)
        obj = cases.to_object(pose, parents)
        obj_m = cases.to_object(mirrored, parents)
        np.testing.assert_allclose(obj_m[:, 4:7], obj[mirror, 4:7] * [-1, 1, 1], atol=1e-5)


def test_table_helper_refusals():
    import acl_b200 as ab
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    bad_mirror = mirror.copy()
    bad_mirror[2] = 6                                        # 2 -> 6 -> 3: not an involution
    with pytest.raises(ValueError):
        ab.mirror_table(parents, bad_mirror, rotations, ab.MIRROR_X)
    out_of_range = mirror.copy()
    out_of_range[0] = parents.size
    with pytest.raises(ValueError):
        ab.mirror_table(parents, out_of_range, rotations, ab.MIRROR_X)
    asymmetric = parents.copy()
    asymmetric[6] = 1                                        # the right forearm hangs from the spine, the left one from the upper arm
    with pytest.raises(ValueError):
        ab.mirror_table(asymmetric, mirror, rotations, ab.MIRROR_X)
    with pytest.raises(ValueError):
        ab.mirror_table(parents, mirror, rotations, 3)
    table = ab.mirror_table(parents, mirror, rotations, ab.MIRROR_X)
    with pytest.raises(ValueError):
        ab.mirror_rows_table(table, [0, 2, 3], 0)            # bone 2's mirror bone 5 is not among the rows


def test_feature_rows_mirror_like_the_local_poses():
    """Feature rows (chosen bones in the root's frame) mirrored by mirror_poses with mirror_rows_table equal, within float32 tolerance,
    the feature rows of the mirrored local poses"""
    import acl_b200 as ab
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    for axis in cases.AXES:
        table = ab.mirror_table(parents, mirror, rotations, axis)
        bones = [4, 7, 9, 11, 1, 0]
        rows_table = ab.mirror_rows_table(table, bones, 0)
        assert rows_table["mirror"].tolist() == [1, 0, 3, 2, 4, 5]
        for pose in cases.random_local_poses(10, parents.size, seed=60 + axis):
            obj = cases.to_object(pose, parents)
            features = cases.relative_to(obj[bones], obj[0]).astype(np.float32)
            got, flags = oracle.mirror_pose(features, rows_table, axis)
            assert flags == 0
            mirrored_local, _ = oracle.mirror_pose(pose, table, axis)
            obj_m = cases.to_object(mirrored_local, parents)
            want = cases.relative_to(obj_m[bones], obj_m[0])
            sign = np.sign(np.sum(got[:, 0:4] * want[:, 0:4], axis=1, keepdims=True))
            np.testing.assert_allclose(got[:, 0:4] * sign, want[:, 0:4], atol=2e-5)
            np.testing.assert_allclose(got[:, 4:7], want[:, 4:7], atol=2e-5)


def test_root_motion_rows_mirror_like_the_local_poses():
    """The root's displacement between two poses, in the first pose's root frame, mirrored with the one-row table equals the displacement
    between the two mirrored poses"""
    import acl_b200 as ab
    parents, mirror, rotations, _ = cases.symmetric_skeleton()
    for axis in cases.AXES:
        table = ab.mirror_table(parents, mirror, rotations, axis)
        root_table = ab.mirror_rows_table(table, [0], 0)
        assert root_table["mirror"].tolist() == [0]
        np.testing.assert_array_equal(root_table["pre"][0], table["pre"][0])
        np.testing.assert_allclose(root_table["post"][0], table["pre"][0] * [-1, -1, -1, 1])
        poses = cases.random_local_poses(16, parents.size, seed=70 + axis)
        for a, b in zip(poses[0::2], poses[1::2]):
            motion = cases.relative_to(b[0:1], a[0]).astype(np.float32)
            got, _ = oracle.mirror_pose(motion, root_table, axis)
            ma, mb = oracle.mirror_pose(a, table, axis)[0], oracle.mirror_pose(b, table, axis)[0]
            want = cases.relative_to(mb[0:1], ma[0])
            sign = np.sign(np.sum(got[:, 0:4] * want[:, 0:4]))
            np.testing.assert_allclose(got[:, 0:4] * sign, want[:, 0:4], atol=2e-5)
            np.testing.assert_allclose(got[:, 4:7], want[:, 4:7], atol=2e-5)
