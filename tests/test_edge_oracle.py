"""CPU checks of the fabricated edge clips (tests/edge_cases.py): they are what their recipe makes, valid with their hash, decoded by
the port exactly as the unmodified reference decodes them at every edge time, and the GPU request lists put every W input class at
every position of the pipeline's rotation chain."""
import numpy as np
import pytest

from tests import clips
from tests import edge_cases as ec
from tests import pipeline_cases as pc

LANES = clips.DEFINED_LANES
NAMES = list(ec.EDGE_SPECS)


@pytest.mark.parametrize("name", NAMES)
def test_fabricated_blob_is_reproducible(oracle_port, name):
    blob, manifest = ec.fabricate(name)
    assert np.array_equal(blob, ec.load_blob(name)), "the recipe no longer makes the committed blob"
    assert manifest == ec.load_manifest(name)


@pytest.mark.parametrize("name", NAMES)
def test_fabricated_blob_hash_and_edits(oracle_port, name):
    blob = ec.load_blob(name)
    assert oracle_port.validate(blob, check_hash=True) == 0
    broken = blob.copy()
    broken[200] ^= 1
    assert oracle_port.validate(broken, check_hash=True) != 0
    # every edited key frame holds the integers the recipe wrote, as the port's bit stream reader sees them
    lay = ec.Layout(blob)
    settings = oracle_port.settings_for_kind(3)
    for row in ec.load_manifest(name):
        if row["stored"] < 0:
            continue
        t = (row["key_frame"] + 0.25) / lay.rate
        st = oracle_port.transform_seek(blob, settings, t, oracle_port.ROUND_FLOOR, oracle_port.LOOP_CLAMP)
        assert st.segment_indices[0] == row["segment"] and st.key_frame_bit_offsets[0] == row["stored"] * lay.segments[row["segment"]]["pose_bits"]
        ints = oracle_port.transform_key_frame_ints(blob, st, 0)
        flat = row["sub_track"] + sum(lay.num_animated[:row["kind"]])
        bits = int(ints[flat, 3])
        want = (1 << bits) - 1 if row["cls"] == "int_max" else 0
        assert list(ints[flat, :3]) == [want] * 3, row
        if row["kind"] == 0 and row["cls"] in ec.W_CLASSES:
            pose = oracle_port.transform_decompress_tracks(blob, settings, t, oracle_port.ROUND_FLOOR, oracle_port.LOOP_CLAMP)
            assert ec.classify(*pose[row["bone"], :3]) == row["cls"], row
            assert clips.bit_equal(pose[row["bone"], :3], np.array(ec.W_CLASSES[row["cls"]], dtype=np.float32)), row


@pytest.mark.parametrize("name", NAMES + ["seg_200"] + list(clips.TRANSFORM_SPECS))
def test_port_equals_live_reference_at_edge_times(oracle_port, reference, name):
    blob = ec.load_blob(name)
    times = ec.edge_times(blob)
    for kind in ec.settings_kinds(name):
        settings = oracle_port.settings_for_kind(kind)
        for rounding in range(4):
            for looping in range(3):
                for t in times.tolist():
                    want = reference.decompress_tracks(blob, t, rounding, looping, settings=kind)
                    got = oracle_port.transform_decompress_tracks(blob, settings, t, rounding, looping)
                    assert clips.bit_equal(got[:, LANES], want[:, LANES]), (name, kind, rounding, looping, t)
                    if name in ec.EDGE_SPECS:
                        assert np.isfinite(want[:, LANES]).all(), (name, kind, rounding, looping, t)


@pytest.mark.parametrize("name", NAMES)
def test_port_equals_stored_reference_poses(oracle_port, name):
    blob = ec.load_blob(name)
    g = np.load(clips.golden_path(name, "golden.npz"))
    for ci, (kind, rounding, looping) in enumerate(g["combos"]):
        settings = oracle_port.settings_for_kind(int(kind))
        for ti, t in enumerate(g["times"]):
            got = oracle_port.transform_decompress_tracks(blob, settings, float(t), int(rounding), int(looping))[g["bones"]][:, LANES]
            assert clips.bit_equal(got, g["poses"][ci, ti]), (name, kind, rounding, looping, float(t))


@pytest.mark.parametrize("unit", [True, False])
def test_every_class_reaches_every_chain_position(oracle_port, unit):
    """Each W input (or squared length) class at each position of the chained rotation loop, in the request lists the GPU tests
    decode, at the batch shapes they reach."""
    names = ec.UNIT_SET if unit else ec.HUGE_SET
    blobs = [ec.load_blob(n) for n in names]
    req = ec.request_list(blobs, seed=ec.SEED)
    rows = pc.seek_rows(oracle_port, blobs, oracle_port.settings_for_kind(0), *req)
    classes = {}
    for c, name in enumerate(names):
        if name not in ec.EDGE_SPECS:
            continue
        manifest = ec.load_manifest(name)
        bones = sorted({row["bone"] for row in manifest if row["kind"] == 0 and row["segment"] >= 0 and row["cls"] not in ("int_max", "int_zero")})
        frames = ec.key_frame_rotations(blobs[c], bones)
        classes[c] = {key: {ec.classify(*xyz) for xyz in value} for key, value in frames.items()}
    wanted = list(ec.W_CLASSES) + ["outside_unit"] if unit else list(ec.LEN2_CLASSES)
    for rpb in ec.BATCH_SHAPES["unit" if unit else "huge"]:
        counts = {(cls, pos): 0 for cls in wanted for pos in ec.CHAIN_POSITIONS}
        for r, pos, seg, kf in ec.chain_positions(rows, rpb):
            for cls in classes.get(int(req[0][r]), {}).get((seg, kf), ()):
                if (cls, pos) in counts:
                    counts[(cls, pos)] += 1
        missing = [key for key, count in counts.items() if count == 0]
        print(rpb, counts)
        assert not missing, (rpb, missing)
