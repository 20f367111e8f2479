"""CPU checks of the streaming database test data: tests/golden/database_tiers.npz is what the unmodified reference decodes (pinned
against the compiled reference where it exists), and its tier states really change the decoded poses."""
import numpy as np
import pytest

from tests import clips
from tests import database_cases as cases


@pytest.fixture(scope="module")
def golden():
    return np.load(clips.golden_path("database_tiers", "npz"))


def test_golden_matches_the_live_reference(golden):
    from oracle import ref, ref_database
    if not ref_database.available():
        pytest.skip("the compiled reference (oracle/_ref/libaclref_db.so) is absent")
    bound, database, other_clip, other_database = cases.build_cases(ref, ref_database)
    assert database.tobytes() == golden["database"].tobytes()
    assert other_clip.tobytes() == golden["other_clip"].tobytes() and other_database.tobytes() == golden["other_database"].tobytes()
    for i, blob in enumerate(bound):
        assert blob.tobytes() == golden[f"clip{i}"].tobytes()
    first = np.concatenate([[0], np.cumsum(golden["num_tracks"])]).astype(int)
    for state, ops in cases.STATES.items():
        for rounding in (0, 3):
            for k, t in enumerate(cases.ALL_TIMES):
                for i, blob in enumerate(bound):
                    want = ref_database.decompress(blob, database, ops, float(t), rounding, ref.LOOP_AS_COMPRESSED)
                    assert clips.bit_equal(golden[f"poses_{state}"][rounding, k, first[i]:first[i + 1]], want), (state, rounding, float(t), i)


def test_tier_states_change_the_poses(golden):
    """every tier state of the fixture decodes differently from the resident key frames alone for some clip and time"""
    nothing = golden["poses_nothing"]
    for state in ("some_medium", "all_medium", "all_medium_low", "medium_out"):
        assert not np.array_equal(golden[f"poses_{state}"], nothing), state
    assert not np.array_equal(golden["poses_all_medium_low"], golden["poses_all_medium"])


def test_fixture_database_layout(golden):
    """the header fields the device validation reads: tag, version, chunk counts of both tiers, inline bulk data"""
    blob = golden["database"]
    header = blob[8:64].view(np.uint32)
    assert int(header[0]) == 0xAC11DB01
    assert 7 <= int(blob[12:14].view(np.uint16)[0]) <= 10
    assert header[2] >= 2 and header[3] >= 1 and (blob[14] & 1) == 1
    other = golden["other_database"][8:64].view(np.uint32)
    assert other[2] >= 1 and other[3] == 0
