"""The blend decode's oracle: the port's rtm::qvv_lerp (oracle/blend_oracle.c) against the unmodified reference's (oracle/ref_blend.cpp),
on the fabricated pairs and on the decoded poses of the fixture clips, and the committed fixtures of tests/blend_cases.py."""
import numpy as np
import pytest

from oracle import blend, port, ref
from tests import blend_cases as cases
from tests import clips

LANES = clips.DEFINED_LANES
VECTOR_LANES = [4, 5, 6, 8, 9, 10]


def _needs_reference():
    if not ref.available() or not blend.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so and libaclref_blend.so (the reference tree)")


def _check_flavours(from_rows, to_rows, weight, what):
    """SSE2 flavour bit for bit; IEEE flavour: vectors bit for bit, rotations within the gate"""
    want = blend.reference_qvv_lerp(from_rows, to_rows, weight)
    sse2 = blend.port_qvv_lerp(from_rows, to_rows, weight, blend.NORMALIZE_RTM_SSE2)
    ieee = blend.port_qvv_lerp(from_rows, to_rows, weight, blend.NORMALIZE_IEEE)
    assert clips.bit_equal(sse2[:, LANES], want[:, LANES]), what
    assert clips.bit_equal(ieee[:, VECTOR_LANES], want[:, VECTOR_LANES]), what
    assert float(np.max(np.abs(ieee[:, 0:4] - want[:, 0:4]))) <= cases.ROTATION_GATE, what
    return want


def test_fixtures_rebuild():
    """The committed blobs are what the reference's compressor writes for the specs (on a CPU whose compressor emits other bytes, the
    committed blobs must still be the pinned ones)."""
    _needs_reference()
    from tests.golden import make_blend_golden
    made = make_blend_golden.blobs()
    differs = []
    for name in cases.NAMES:
        committed = cases.load(name)
        assert cases.blob_sha256(committed) == cases.BLOB_SHA256[name], name
        assert ref.lib().aclref_is_valid(made[name].ctypes.data, 1) == 0, name
        if cases.blob_sha256(made[name]) != cases.BLOB_SHA256[name]:
            differs.append(name)
    if differs:
        pytest.skip(f"this CPU's reference compressor writes other bytes for {differs}; the committed blobs are pinned by hash")


def test_fixture_clips_share_default_bones_and_mirror_scales():
    """Both clips have bones whose rotation is the identity in both (a rotation blended with itself) and mirrored-scale bones."""
    settings = port.settings_for_kind(0)
    a = port.transform_decompress_tracks(cases.load("blend_from"), settings, 0.3)
    b = port.transform_decompress_tracks(cases.load("blend_to"), settings, 0.7)
    identity = np.array([0, 0, 0, 1], np.float32)
    assert ((a[:, 0:4] == identity).all(axis=1) & (b[:, 0:4] == identity).all(axis=1)).any()
    assert (a[cases.MIRRORED_BONES, 8] < 0).all() and (b[cases.MIRRORED_BONES, 8] < 0).all()


@pytest.mark.parametrize("weight", cases.WEIGHTS.tolist())
def test_fabricated_pairs_match_live_reference(weight):
    _needs_reference()
    names, from_rows, to_rows = cases.fabricated_pairs()
    _check_flavours(from_rows, to_rows, weight, weight)


def test_hemisphere_bias_is_the_sign_bit_of_the_dpps_dot():
    """The live reference flips `to` on dot == -0.0 and sums the dot in dpps order: the two named pairs come out as the port predicts, and
    not as the scalar path's dot >= 0 or the SSE2 fallback's (x + z) + (y + w) would have them."""
    _needs_reference()
    names, from_rows, to_rows = cases.fabricated_pairs()
    want = blend.reference_qvv_lerp(from_rows, to_rows, 0.5)
    for name, flips in (("dot_minus_zero", True), ("dpps_order", False)):
        i = names.index(name)
        s, e = from_rows[i, 0:4], to_rows[i, 0:4]
        q = (s - np.float32(0.5) * s) + np.float32(0.5) * (-e if flips else e)
        q_other = (s - np.float32(0.5) * s) + np.float32(0.5) * (e if flips else -e)
        got = want[i, 0:4]
        assert np.allclose(got, q / np.linalg.norm(q), atol=1e-6), name
        assert not np.allclose(got, q_other / np.linalg.norm(q_other), atol=1e-3), name


def test_fixture_clips_match_live_reference():
    """Decoded poses of the fixture clips at every pair, combo and weight: port flavours against the reference's qvv_lerp."""
    _needs_reference()
    from_blob, to_blob = cases.load("blend_from"), cases.load("blend_to")
    flipped = 0
    for kind, rounding, looping in cases.COMBOS:
        settings = port.settings_for_kind(kind)
        for tf, tt in cases.time_pairs():
            from_pose = ref.decompress_tracks(from_blob, float(tf), rounding, looping, settings=kind)
            to_pose = ref.decompress_tracks(to_blob, float(tt), rounding, looping, settings=kind)
            assert clips.bit_equal(port.transform_decompress_tracks(from_blob, settings, float(tf), rounding, looping)[:, LANES], from_pose[:, LANES])
            flipped += int(np.sum(np.sum(from_pose[:, 0:4] * to_pose[:, 0:4], axis=1) < 0))
            for weight in cases.WEIGHTS:
                _check_flavours(from_pose, to_pose, float(weight), (kind, rounding, looping, float(tf), float(tt), float(weight)))
    assert flipped > 0


def test_stored_poses_match_live_reference_and_port():
    """blend.golden.npz against the live reference where it exists, and always against the port's IEEE flavour (vectors bit for bit,
    rotations within the gate). The stored rotations carry the rsqrtss estimate of the CPU that wrote them, and that estimate differs
    between CPU models: against the live reference they are bit for bit only where this CPU's estimate reproduces the stored fabricated
    lerps, else within the gate; translations and scales are bit for bit everywhere."""
    golden = np.load(clips.golden_path("blend", "golden.npz"))
    assert golden["combos"].tolist() == [list(c) for c in cases.COMBOS]
    assert np.array_equal(golden["pairs"], cases.time_pairs())
    assert np.array_equal(golden["weights"], cases.WEIGHTS)
    _, from_rows, to_rows = cases.fabricated_pairs()
    assert np.array_equal(golden["fabricated_from"], from_rows) and np.array_equal(golden["fabricated_to"], to_rows)
    same_estimate = all(clips.bit_equal(blend.port_qvv_lerp(from_rows, to_rows, float(w), blend.NORMALIZE_RTM_SSE2)[:, 0:4],
                                        golden["fabricated"][wi][:, 0:4]) for wi, w in enumerate(cases.WEIGHTS))

    def matches(got, stored):
        if not clips.bit_equal(got[..., 4:], stored[..., 4:]):
            return False
        if same_estimate:
            return clips.bit_equal(got[..., 0:4], stored[..., 0:4])
        return float(np.max(np.abs(got[..., 0:4] - stored[..., 0:4]))) <= cases.ROTATION_GATE

    live = ref.available() and blend.reference_available()
    from_blob, to_blob = cases.load("blend_from"), cases.load("blend_to")
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        settings = port.settings_for_kind(kind)
        for wi, weight in enumerate(cases.WEIGHTS):
            for pi, (tf, tt) in enumerate(golden["pairs"]):
                stored = golden["poses"][ci, wi, pi]
                got = cases.port_pose(port, blend, from_blob, to_blob, tf, tt, weight, settings, rounding, looping, blend.NORMALIZE_IEEE)[:, LANES]
                assert clips.bit_equal(got[:, 4:], stored[:, 4:]), (kind, rounding, looping, float(weight), pi)
                assert float(np.max(np.abs(got[:, 0:4] - stored[:, 0:4]))) <= cases.ROTATION_GATE
                if live:
                    want = cases.reference_pose(blend, from_blob, to_blob, tf, tt, weight, kind, rounding, looping)
                    assert matches(want[:, LANES], stored), (kind, rounding, looping, float(weight), pi, same_estimate)
    if live:
        for wi, weight in enumerate(cases.WEIGHTS):
            assert matches(blend.reference_qvv_lerp(from_rows, to_rows, float(weight))[:, LANES], golden["fabricated"][wi][:, LANES])
