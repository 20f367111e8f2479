"""The inertialization oracle: the C restatement (oracle/inertialization_oracle.c) against the unmodified reference's rtm
(oracle/ref_inertialization.cpp, pinned in tests/golden/inertialization.golden.npz) bit for bit, and the spring's properties in float64
numpy against the oracle's float32 results."""
import numpy as np
import pytest

from oracle import inertialization as oracle
from tests import inertialization_cases as cases


def _golden():
    return np.load(cases.GOLDEN)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same(got, want) -> bool:
    """bit for bit, except that a NaN matches any NaN (the sign and payload of a NaN are not specified)"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    both_nan = np.isnan(got) & np.isnan(want)
    return got.shape == want.shape and bool(np.all((_bits(got) == _bits(want)) | both_nan))


def _port_results():
    src, src_prev, dst, dst_prev = cases.transitions()
    records = np.stack([oracle.begin_inertialization(src[j], src_prev[j], dst[j], dst_prev[j], cases.INV_DT)
                        for j in range(cases.NUM_TRANSITIONS)])
    applied = np.stack([np.stack([oracle.inertialize_pose(dst[j], records[j], float(e), float(h)) for j in range(cases.NUM_TRANSITIONS)])
                        for e, h in cases.DECAYS])
    return {"log": np.stack([oracle.quat_rotation_log(q) for q in cases.log_inputs()]),
            "exp": np.stack([oracle.quat_rotation_exp(v) for v in cases.exp_inputs()]), "records": records, "applied": applied}


@pytest.mark.parametrize("what", ["log", "exp", "records", "applied"])
def test_port_equals_the_pinned_reference(what):
    """log and exp on adversarial inputs, the capture of every transition and the apply at every (elapsed, halflife) edge: bit for bit"""
    want = _golden()[what]
    got = _port_results()[what]
    assert _same(got, want), np.argwhere((_bits(got) != _bits(want)) & ~(np.isnan(got) & np.isnan(want)))[:8]


def test_pinned_reference_is_the_live_reference():
    if not oracle.reference_available():
        pytest.skip("needs oracle/_ref/libaclref_inertialization.so (the reference tree)")
    from tests.golden import make_inertialization_golden
    live = make_inertialization_golden.reference_results()
    golden = _golden()
    for what in ("log", "exp", "records", "applied"):
        assert np.array_equal(_bits(live[what]), _bits(golden[what])), what


def test_log_and_exp_take_every_select():
    """The inputs reach both sides of log's near identity select (on w after the clamp), exp's near zero select, and the sin / cos
    reflection"""
    logs = cases.log_inputs(with_nan=False)
    w = np.clip(logs[:, 3], -1, 1)
    assert (w > np.float32(1) - np.float32(1e-6)).any() and (w <= np.float32(1) - np.float32(1e-6)).any()
    lengths = np.sqrt(np.sum(cases.exp_inputs()[:, :3].astype(np.float64) ** 2, axis=1))
    assert (lengths < 1e-6).any() and (lengths >= 1e-6).any() and (lengths > np.pi).any()
    # the log of a unit quaternion is half its angle about its axis, exp inverts it
    for q in cases._unit(np.random.default_rng(3).normal(size=(200, 4))):
        q = q if q[3] >= 0 else -q
        back = oracle.quat_rotation_exp(oracle.quat_rotation_log(q))
        assert np.allclose(back, q, atol=2e-6), (q, back)


def _decay64(x0, v0, t, halflife):
    """the specified spring in float64: fast_negexp, not exp (it is up to 9 % of x0 away from exp's spring)"""
    y = 4 * np.log(2) / (halflife + 1e-5) / 2
    u = y * t
    return (x0 + (v0 + x0 * y) * t) / (1 + u + 0.48 * u * u + 0.235 * u ** 3)


def _transition():
    """transition 0 with its rotations normalised: the properties below are those of rotations (an unnormalised rotation's log is not its
    angle)"""
    poses = [p[0].copy() for p in cases.transitions()]
    for p in poses:
        p[:, 0:4] = cases._unit(p[:, 0:4])
    return poses


def _same_rotation(a, b, atol):
    """a and b are the same rotation (either cover) within atol per lane"""
    sign = np.where(np.sum(a.astype(np.float64) * b, axis=-1) < 0, -1.0, 1.0)[..., None]
    return np.abs(a * sign - b).max() <= atol


def test_elapsed_zero_gives_the_source_pose():
    src, src_prev, dst, dst_prev = _transition()
    record = oracle.begin_inertialization(src, src_prev, dst, dst_prev, cases.INV_DT)
    out = oracle.inertialize_pose(dst, record, 0.0, 0.3)
    assert _same_rotation(out[:, 0:4], src[:, 0:4], 2e-6)
    assert np.abs(out[:, 4:7] - src[:, 4:7]).max() <= 4 * np.finfo(np.float32).eps * max(1.0, float(np.abs(src[:, 4:7]).max()))
    assert np.array_equal(out[:, 8:11], dst[:, 8:11]) and not out[:, [7, 11]].any()


def test_velocity_at_zero_approaches_the_source_velocity():
    """The displayed pose's finite difference over a short step after the jump is the source's velocity plus the destination's: the offset
    carries rot_v = w(src) - w(dst), so the output moves as the source did"""
    src, src_prev, dst, dst_prev = _transition()
    record = oracle.begin_inertialization(src, src_prev, dst, dst_prev, cases.INV_DT)
    h = 1e-3
    # the destination advances at its own velocity over h: its translation by v(dst) h; its rotation held, so the output's rotation
    # velocity is the offset's rot_v (checked on the record), translation velocity v(src) - v(dst) + v(dst)
    dst_h = dst.copy()
    v_dst = (dst[:, 4:7].astype(np.float64) - dst_prev[:, 4:7]) * cases.INV_DT
    dst_h[:, 4:7] = dst[:, 4:7] + v_dst * h
    a = oracle.inertialize_pose(dst, record, 0.0, 0.3).astype(np.float64)
    b = oracle.inertialize_pose(dst_h, record, h, 0.3).astype(np.float64)
    v_src = (src[:, 4:7].astype(np.float64) - src_prev[:, 4:7]) * cases.INV_DT
    assert np.abs((b[:, 4:7] - a[:, 4:7]) / h - v_src).max() <= 0.02 * max(1.0, np.abs(v_src).max())
    # rotation: the output's angular velocity about the held destination is the offset's, d/dt (2 log(out dst^-1)) at 0 = rot_v
    b_held = oracle.inertialize_pose(dst, record, h, 0.3).astype(np.float64)
    rot_b = np.stack([2 * oracle.quat_rotation_log(_canonical(cases.hamilton(b_held[i, 0:4], _conj(dst[i, 0:4]))).astype(np.float32))[:3]
                      for i in range(a.shape[0])])
    rot_a = np.stack([2 * oracle.quat_rotation_log(_canonical(cases.hamilton(a[i, 0:4], _conj(dst[i, 0:4]))).astype(np.float32))[:3]
                      for i in range(a.shape[0])])
    assert np.abs((rot_b - rot_a) / h - record[:, 4:7]).max() <= 0.02 * max(1.0, np.abs(record[:, 4:7]).max())


def _conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]], np.float64)


def _canonical(q):
    return q if q[3] >= 0 else -q


@pytest.mark.parametrize("halflife", [0.05, 0.2, 1.0])
def test_offset_decays_monotonically(halflife):
    """With no velocity offset the spring never overshoots: |offset| falls at every step, as the float64 spring does"""
    src, src_prev, dst, dst_prev = _transition()
    record = oracle.begin_inertialization(src, src, dst, dst, cases.INV_DT)
    assert not record[:, 4:8].any() and not record[:, 12:16].any()
    previous = None
    for t in np.linspace(0.0, 5 * halflife, 60, dtype=np.float32):
        out = oracle.inertialize_pose(dst, record, float(t), halflife).astype(np.float64)
        offset = np.linalg.norm(out[:, 4:7] - dst[:, 4:7], axis=1)
        want = np.linalg.norm(_decay64(record[:, 8:11].astype(np.float64), 0.0, float(t), halflife), axis=1)
        assert np.abs(offset - want).max() <= 1e-6 * np.linalg.norm(record[:, 8:11], axis=1).max() + 1e-7
        if previous is not None:
            assert (offset <= previous * (1 + 1e-6) + 1e-7).all()
        previous = offset


def test_chained_capture_continues_without_a_jump():
    """A second jump during the first transition: its capture starts from the displayed (inertialized) poses, so at elapsed 0 the new
    decay shows what was displayed"""
    rng = np.random.default_rng(5)
    src, src_prev, dst, dst_prev = _transition()
    record = oracle.begin_inertialization(src, src_prev, dst, dst_prev, cases.INV_DT)
    t, dt = np.float32(0.1), np.float32(1 / cases.INV_DT)
    displayed = oracle.inertialize_pose(dst, record, float(t), 0.2)
    displayed_prev = oracle.inertialize_pose(dst_prev, record, float(t - dt), 0.2)
    third = cases.poses(rng, 2, src.shape[0])
    third[..., 0:4] = cases._unit(third[..., 0:4])
    record2 = oracle.begin_inertialization(displayed, displayed_prev, third[0], third[1], cases.INV_DT)
    out = oracle.inertialize_pose(third[0], record2, 0.0, 0.2)
    assert _same_rotation(out[:, 0:4], displayed[:, 0:4], 2e-6)
    assert np.abs(out[:, 4:7] - displayed[:, 4:7]).max() <= 1e-6 * max(1.0, float(np.abs(displayed[:, 4:7]).max()))


def test_edge_decays_are_computed_as_specified():
    """halflife 0, huge, negative and NaN elapsed, NaN halflife: y and e step by step in numpy float32, and the translation they give"""
    src, src_prev, dst, dst_prev = _transition()
    record = oracle.begin_inertialization(src, src_prev, dst, dst_prev, cases.INV_DT)
    f = np.float32
    with np.errstate(all="ignore"):
        for elapsed, halflife in cases.DECAYS:
            y = (f(2.7725887) / (halflife + f(1e-5))) * f(0.5)
            u = y * elapsed
            e = f(1) / (((f(1) + u) + (f(0.48) * u) * u) + ((f(0.235) * u) * u) * u)
            x0, v0 = record[:, 8:11], record[:, 12:15]
            want = dst[:, 4:7] + e * (x0 + (v0 + x0 * y) * elapsed)
            got = oracle.inertialize_pose(dst, record, float(elapsed), float(halflife))
            assert _same(got[:, 4:7], want), (elapsed, halflife)
            if np.isfinite(elapsed) and elapsed > 1e3:
                # the spring has run out: the destination itself
                assert np.array_equal(got[:, 4:7], dst[:, 4:7]) and _same_rotation(got[:, 0:4], dst[:, 0:4], 0.0)
