"""CPU checks behind tests/test_gpu_pipeline.py: the two wide clips of tests/pipeline_cases.py are pinned to the reference, and the
request lists offer the grouping every case it was written for, whatever the batch size."""
import numpy as np
import pytest

from tests import clips
from tests import pipeline_cases as pc

LANES = clips.DEFINED_LANES


@pytest.mark.parametrize("name", list(pc.PIPELINE_SPECS))
def test_port_matches_stored_reference_poses(oracle_port, name):
    blob = pc.load_blob(name)
    assert oracle_port.validate(blob, check_hash=True) == 0
    assert oracle_port.num_tracks_of(blob) == pc.PIPELINE_SPECS[name].num_tracks
    g = np.load(clips.golden_path(name, "golden.npz"))
    for ci, (kind, rounding) in enumerate(g["combos"]):
        settings = oracle_port.settings_for_kind(int(kind))
        for ti, t in enumerate(g["times"]):
            got = oracle_port.transform_decompress_tracks(blob, settings, float(t), int(rounding))[g["bones"]][:, LANES]
            assert clips.bit_equal(got, g["poses"][ci, ti]), (name, kind, rounding, float(t))


@pytest.mark.parametrize("name", list(pc.PIPELINE_SPECS))
def test_pipeline_blobs_are_reproducible(reference, name):
    live = reference.compress_transform(pc.PIPELINE_SPECS[name])
    assert np.array_equal(live, pc.load_blob(name)), "the reference no longer produces the committed blob"


# (clip names, clips whose runs wrap) of the GPU cases that decode sequential runs
LISTS = {
    "ragged": (["c1_30bones", "c5_30x32", "ragged_17", "one_bone", "two_samples", "one_sample", "all_default"], []),
    "raw_loops": (["noisy_raw", "looping", "stripped_loop"], ["looping", "stripped_loop"]),
    "seg200": (["seg_200", "c2_100bones"], ["seg_200"]),
}


@pytest.mark.parametrize("case", list(LISTS))
def test_request_lists_offer_every_grouping_case(oracle_port, case):
    names, wrap_names = LISTS[case]
    blobs = [pc.load_blob(n) for n in names]
    req = pc.request_list(names, wrap_names, 20000, seed=200)
    rows = pc.seek_rows(oracle_port, blobs, oracle_port.settings_for_kind(0), *req)
    s = pc.pair_stats(rows)
    assert s["invalid"] >= 100, s
    assert s["chained_pairs"] >= 1000 and s["longest_run"] > pc.K_GROUP_MAX, s           # runs long enough to be cut at k_group_max
    assert all(count >= 10 for count in s["runs_reaching"][2:12]), s                    # chains of every length up to 11
    assert s["chain_then_crossing"] >= 20 and s["crossings"] >= 50, s                   # chains that end on a segment crossing
    assert s["repeats"] >= 100 and s["clamped_repeats"] >= 20, s
    if wrap_names:
        assert s["wraps_into_segment_0"] >= 10 and s["chained_wrap_crossings"] >= 5, s
    if len(names) > 1:
        clip = req[0]
        changes = int(((clip[1:] != clip[:-1]) & (clip[1:] < len(names)) & (clip[:-1] < len(names))).sum())
        assert changes >= 1000, changes                                                 # clips interleaved request by request


def test_group_model_cuts_and_crossings():
    """pc.groups on a hand-made list: one 7 request run of one segment that ends on a crossing, at 8 requests per batch."""
    # valid, clip, seg0, seg1, kf0, kf1, single, animated
    rows = [(1, 0, 0, 0, k, k + 1, 1, 1) for k in range(7)] + [(1, 0, 0, 1, 7, 0, 0, 1)]
    g = pc.groups(np.array(rows, dtype=np.int64), 8)
    assert g["groups"] == 2 and g["cuts"] == 1 and g["groups_of_5"] == 1 and g["groups_of_3"] == 1, g
    assert g["tail_crossings"] == 1 and g["tail_crossings_at_last_lane"] == 1, g
    g = pc.groups(np.array(rows, dtype=np.int64), 4)        # batch starts cut the run too
    assert g["groups_of_4"] == 2 and g["cuts"] == 0 and g["tail_crossings_at_last_lane"] == 1, g
