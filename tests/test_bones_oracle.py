"""The bone query's closure (tests/bones_cases.py) against the pinned port: the rows of the listed bones depend on the local rows of
their ancestor closure and on nothing else.

  * the closure rule itself: chains end at roots and at parents that do not precede their child, on any parent table;
  * sufficient: a local pose whose rows outside the closure are NaN gives the listed object rows bit for bit equal to the whole pose's
    (port.local_to_object_space, IEEE normalisation, and object_space.port_local_to_object_space_matrix), for every named clip and
    every skeleton kind;
  * necessary: making any one closure bone's local row NaN changes a listed row.
"""
import numpy as np
import pytest

from oracle import object_space
from tests import bones_cases as cases
from tests import clips

ROOT = cases.ROOT


def test_closure_rule():
    n = 100
    tree = cases.tree(n)
    assert cases.closure(tree, [0], n).tolist() == [0]
    assert cases.closure(tree, cases.C2_FOUR_LEAVES, n).size == 21
    assert cases.closure(tree, [63], n).tolist() == [0, 1, 3, 7, 15, 31, 63]
    chain = cases.skeleton("chain", n)
    assert cases.closure(chain, [n - 1], n).tolist() == list(range(n))
    star = cases.skeleton("star", n)
    assert cases.closure(star, [5, 9, 5], n).tolist() == [0, 5, 9]
    # without parents: the listed bones below num_tracks, holes and out of range bones dropped
    assert cases.closure(tree, [63, cases.NO_BONE, 63, n, 2], n, with_parents=False).tolist() == [2, 63]
    # a parent at or above its child ends the chain; a cyclic or garbage table cannot make the walk loop
    late = tree.copy()
    late[31] = 80
    assert cases.closure(late, [63], n).tolist() == [31, 63]
    cyclic = np.array([1, 0, 3, 2, 2], np.uint32)
    assert cases.closure(cyclic, [4], 5).tolist() == [2, 4]
    assert cases.closure(np.full(8, 7, np.uint32), [7, 6], 8).tolist() == [6, 7]
    assert cases.effective_parents(late)[31] == ROOT and cases.effective_parents(cyclic).tolist() == [ROOT, 0, ROOT, 2, 2]


def _poses(oracle_port, name, count=2):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    settings = oracle_port.settings_for_kind(1)
    times = clips.sample_times(spec)
    return spec, [oracle_port.transform_decompress_tracks(blob, settings, float(t)) for t in times[:: max(1, len(times) // count)][:count]]


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_closure_is_sufficient(oracle_port, name):
    spec, poses = _poses(oracle_port, name)
    n = spec.num_tracks
    for kind in cases.SKELETONS:
        parents = cases.skeleton(kind, n, seed=spec.seed)
        for list_name, bones in cases.bone_lists(n, seed=spec.seed).items():
            keep = cases.closure(parents, bones, n)
            valid = [b for b in bones if b < n]
            for local in poses:
                masked = np.full_like(local, np.nan)
                masked[keep] = local[keep]
                for matrix in (False, True):
                    want = cases.object_rows(oracle_port, object_space, local, parents, matrix)[valid]
                    got = cases.object_rows(oracle_port, object_space, masked, parents, matrix)[valid]
                    assert clips.bit_equal(got, want), (name, kind, list_name, matrix)


@pytest.mark.parametrize("name", ["c2_100bones", "mixed_scale", "ragged_17", "paragon_like"])
def test_closure_is_necessary(oracle_port, name):
    spec, poses = _poses(oracle_port, name, count=1)
    n = spec.num_tracks
    local = poses[0]
    for kind in ("tree", "random", "late"):
        parents = cases.skeleton(kind, n, seed=spec.seed)
        for list_name in ("leaves", "deep_leaf", "duplicates_reversed"):
            bones = [b for b in cases.bone_lists(n, seed=spec.seed)[list_name] if b < n]
            keep = cases.closure(parents, bones, n)
            for matrix in (False, True):
                want = cases.object_rows(oracle_port, object_space, local, parents, matrix)[bones]
                for dropped in keep:
                    masked = local.copy()
                    masked[dropped] = np.nan
                    got = cases.object_rows(oracle_port, object_space, masked, parents, matrix)[bones]
                    assert not clips.bit_equal(got, want), (name, kind, list_name, matrix, int(dropped))
