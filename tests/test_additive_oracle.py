"""The additive decode's oracle: the port's decompress of a base and an additive clip followed by its apply_additive_to_base
(oracle/acl_oracle.c) against the unmodified reference (oracle/ref_additive.cpp), and the committed fixtures of tests/additive_cases.py."""
import numpy as np
import pytest

from oracle import additive, port, ref
from tests import additive_cases as cases
from tests import clips

LANES = clips.DEFINED_LANES


def _needs_reference():
    if not ref.available() or not additive.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so and libaclref_additive.so (the reference tree)")


def test_fixtures_rebuild():
    """The committed blobs are what the reference's compressor writes for the specs (on a CPU whose compressor emits other bytes, the
    committed blobs must still be the pinned ones)."""
    _needs_reference()
    from tests.golden import make_additive_golden
    made = make_additive_golden.blobs()
    differs = []
    for name in cases.NAMES:
        committed = cases.load(name)
        assert cases.blob_sha256(committed) == cases.BLOB_SHA256[name], name
        assert ref.lib().aclref_is_valid(made[name].ctypes.data, 1) == 0, name
        if cases.blob_sha256(made[name]) != cases.BLOB_SHA256[name]:
            differs.append(name)
    if differs:
        pytest.skip(f"this CPU's reference compressor writes other bytes for {differs}; the committed blobs are pinned by hash")


def test_additive1_clip_reads_zero_default_scale():
    """The compressor gives additive1 clips a default scale of 0 (compress.transform.impl.h: set_default_scale), and this one has default
    scale sub-tracks that a track_writer-default decode reads as 0."""
    blob = cases.load("additive_additive1")
    pose = port.transform_decompress_tracks(blob, cases.writer_settings(port, 0), 0.1)
    assert (pose[:, 8:11] == 0.0).all(axis=1).any()


@pytest.mark.parametrize("name", list(cases.FORMATS))
def test_port_matches_live_reference(name):
    """Every format clip at every golden pair and combo: bit for bit, with the port's rsqrtss flavour of quat_normalize."""
    _needs_reference()
    format_ = cases.FORMATS[name]
    base_blob, additive_blob = cases.load(cases.BASE), cases.load(name)
    for kind, rounding, looping in cases.COMBOS:
        base_settings, additive_settings = port.settings_for_kind(kind), cases.writer_settings(port, kind)
        for tb, ta in cases.time_pairs():
            want = cases.reference_pose(additive, format_, base_blob, additive_blob, tb, ta, kind, rounding, looping)
            got = cases.port_pose(port, format_, base_blob, additive_blob, tb, ta, base_settings, additive_settings, rounding, looping,
                                  port.NORMALIZE_RTM_SSE2)
            assert clips.bit_equal(got[:, LANES], want[:, LANES]), (name, kind, rounding, looping, float(tb), float(ta))


@pytest.mark.parametrize("pair", [("c1_30bones", "c5_30x32"), ("full_formats", "mixed_formats"), ("drop_w_full", "full_formats")])
@pytest.mark.parametrize("format_", [0, 1, 2, 3])
def test_named_clips_paired(pair, format_):
    """Named clips of equal bone counts layered on each other in every format (none included), under the settings kinds that decode
    every rotation format: port against the live reference."""
    _needs_reference()
    base_blob, additive_blob = clips.load_blob(pair[0]), clips.load_blob(pair[1])
    times = clips.sample_times(clips.TRANSFORM_SPECS[pair[0]])
    other = np.resize(clips.sample_times(clips.TRANSFORM_SPECS[pair[1]]), times.size)
    for kind, rounding, looping in [(1, 0, 2), (3, 2, 0), (4, 0, 1)]:
        base_settings, additive_settings = port.settings_for_kind(kind), cases.writer_settings(port, kind)
        for tb, ta in zip(times, other):
            want = cases.reference_pose(additive, format_, base_blob, additive_blob, tb, ta, kind, rounding, looping)
            got = cases.port_pose(port, format_, base_blob, additive_blob, tb, ta, base_settings, additive_settings, rounding, looping,
                                  port.NORMALIZE_RTM_SSE2)
            assert clips.bit_equal(got[:, LANES], want[:, LANES]), (pair, format_, kind, float(tb), float(ta))


def test_stored_poses_match_the_port():
    """additive.golden.npz (the reference's poses) against the port, every format, combo and pair: bit for bit."""
    golden = np.load(clips.golden_path("additive", "golden.npz"))
    assert golden["combos"].tolist() == [list(c) for c in cases.COMBOS]
    assert np.array_equal(golden["pairs"], cases.time_pairs())
    base_blob = cases.load(cases.BASE)
    for fi, (name, format_) in enumerate(cases.FORMATS.items()):
        assert int(golden["formats"][fi]) == format_
        additive_blob = cases.load(name)
        for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
            base_settings, additive_settings = port.settings_for_kind(kind), cases.writer_settings(port, kind)
            for pi, (tb, ta) in enumerate(golden["pairs"]):
                got = cases.port_pose(port, format_, base_blob, additive_blob, tb, ta, base_settings, additive_settings, rounding, looping,
                                      port.NORMALIZE_RTM_SSE2)
                assert clips.bit_equal(got[:, LANES], golden["poses"][fi, ci, pi]), (name, kind, rounding, looping, pi)
