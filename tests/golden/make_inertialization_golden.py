"""Writes tests/golden/inertialization.golden.npz: the unmodified reference's rtm::quat_rotation_log and quat_rotation_exp on
tests/inertialization_cases.py's inputs, and the capture and apply built from them (oracle/ref_inertialization.cpp) on its transitions.
Needs oracle/_ref/libaclref_inertialization.so. Run from the repository root: python -m tests.golden.make_inertialization_golden"""
from __future__ import annotations

import numpy as np

from oracle import inertialization as oracle
from tests import inertialization_cases as cases


def reference_results() -> dict[str, np.ndarray]:
    logs = cases.log_inputs()
    exps = cases.exp_inputs()
    src, src_prev, dst, dst_prev = cases.transitions()
    records = np.stack([oracle.begin_inertialization(src[j], src_prev[j], dst[j], dst_prev[j], cases.INV_DT, reference=True)
                        for j in range(cases.NUM_TRANSITIONS)])
    applied = np.stack([np.stack([oracle.inertialize_pose(dst[j], records[j], float(e), float(h), reference=True)
                                  for j in range(cases.NUM_TRANSITIONS)]) for e, h in cases.DECAYS])
    return {
        "log": np.stack([oracle.quat_rotation_log(q, reference=True) for q in logs]),
        "exp": np.stack([oracle.quat_rotation_exp(v, reference=True) for v in exps]),
        "records": records,
        "applied": applied,
    }


if __name__ == "__main__":
    assert oracle.reference_available(), "needs oracle/_ref/libaclref_inertialization.so"
    np.savez_compressed(cases.GOLDEN, **reference_results())
    print("wrote", cases.GOLDEN)
