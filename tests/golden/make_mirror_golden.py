"""Writes tests/golden/mirror.golden.npz: the mirrored poses the unmodified reference's rtm::quat_mul and quat_mul_vector3 give
(oracle/ref_mirror.cpp) on tests/mirror_cases.py's fabricated poses and on the reference decodes of its named clips, on every axis.
Needs oracle/_ref/libaclref_mirror.so. Run from the repository root: python -m tests.golden.make_mirror_golden"""
from __future__ import annotations

import numpy as np

from oracle import mirror as oracle
from tests import mirror_cases as cases


def results(reference: bool) -> dict[str, np.ndarray]:
    out = {}
    table = cases.fabricated_table()
    poses = cases.fabricated_poses()
    mirrored = [[oracle.mirror_pose(p, table, axis, reference=reference) for p in poses] for axis in cases.AXES]
    out["fabricated"] = np.array([[m[0] for m in row] for row in mirrored])
    out["fabricated_flags"] = np.array([[m[1] for m in row] for row in mirrored], np.uint32)
    for name in cases.NAMED_CLIPS:
        named = cases.named_poses(name)
        named_table = cases.named_table(named.shape[1])
        out[name] = np.array([[oracle.mirror_pose(p, named_table, axis, reference=reference)[0] for p in named] for axis in cases.AXES])
    return out


if __name__ == "__main__":
    assert oracle.reference_available(), "needs oracle/_ref/libaclref_mirror.so"
    with np.errstate(all="ignore"):
        np.savez_compressed(cases.GOLDEN, **results(reference=True))
    print("wrote", cases.GOLDEN)
