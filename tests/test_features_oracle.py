"""Pins the port's pose features composition (tests/features_cases.py) to the unmodified reference, from oracle pieces already pinned:

  * port side: the port decode at u' (clamp policy), the port walk (oracle.port.local_to_object_space) through the bone query's closure,
    oracle.root_motion.port_root_motion and port_qvv_mul / port_qvv_inverse;
  * reference side: oracle.ref.decompress_tracks at u' with the clamp policy, reference_root_motion's whole path (reference_extract) and
    reference_qvv_mul / reference_qvv_inverse. No harness exposes the reference's qvvf walk, so its object rows are the port walk in the
    rsqrtss flavour, which tests/test_error_metric_oracle.py pins bit for bit to the reference's.

With every normalisation in the rsqrtss flavour the two compositions are equal bit for bit. In the IEEE flavour the GPU runs, the scale
lanes are still equal bit for bit (no normalisation touches them); rotations and translations differ by the walk's normalisations:
each quat_normalize differs by at most a few ulps between the flavours, and a bone's rotation and translation carry those of every
ancestor (at most depth ~ 7 for the named clips' binary trees), then two more qvv_mul. The gate is 4e-6 per level of that chain on unit
quaternions, and the same relative to the row's translation magnitude.
Every named clip x settings kind x rounding policy, S up to 8, offsets negative, zero, positive, on k * D, across 0, 1, 3, 256 and 257
boundaries, t = 0 and t = D, and the one-sample clip (D = 0)."""
import numpy as np
import pytest

from oracle import root_motion as RM
from tests import bones_cases
from tests import clips
from tests import features_cases as cases
from tests import root_motion_cases as rm_cases

ROTATION, TRANSLATION, SCALE = slice(0, 4), slice(4, 7), slice(8, 11)


@pytest.fixture(scope="module")
def rm_reference(reference):
    if not RM.reference_available():
        pytest.skip("oracle/_ref/libaclref_root_motion.so not built (needs the reference tree at build time)")
    return RM


def test_offset_time_rule():
    d = np.float32(1.0)
    assert cases.offset_time(0.5, 0.25, cases.CLAMP, d) == (True, 0, np.float32(0.75))
    assert cases.offset_time(0.5, 0.75, cases.LOOP, d) == (True, 1, np.float32(0.25))
    assert cases.offset_time(0.5, -0.75, cases.LOOP, d) == (True, -1, np.float32(0.75))
    assert cases.offset_time(0.0, 3.0, cases.LOOP, d) == (True, 3, np.float32(0.0))          # exactly on k * D: the next cycle's start
    assert cases.offset_time(0.5, 256.0, cases.LOOP, d)[:2] == (True, 256)
    assert not cases.offset_time(0.5, 257.0, cases.LOOP, d)[0]
    assert not cases.offset_time(np.inf, 0.0, cases.LOOP, d)[0] and cases.offset_time(np.inf, 0.0, cases.CLAMP, d)[0]
    assert cases.offset_time(0.7, 5.0, cases.LOOP, 0.0) == (True, 0, np.float32(0.0))
    assert not cases.offset_time(0.5, 0.0, 2, d)[0]


def _roundings(kind, n):
    return [(r, None) for r in range(4)] + ([(4, (np.arange(n) % 4).astype(np.uint8))] if kind == 1 else [])


def _zero_pads(rows):
    rows = np.array(rows, np.float32)
    rows[..., 7] = 0.0
    rows[..., 11] = 0.0
    return rows


def _gate(want, got, depth):
    rotation = 4e-6 * (depth + 2)
    magnitude = max(1.0, float(np.abs(want[TRANSLATION]).max()))
    return (np.abs(got[ROTATION] - want[ROTATION]) <= rotation).all() and \
        (np.abs(got[TRANSLATION] - want[TRANSLATION]) <= rotation * magnitude).all() and clips.bit_equal(got[SCALE], want[SCALE])


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_port_composition_matches_reference(rm_reference, reference, oracle_port, name):
    port = oracle_port
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    n = spec.num_tracks
    parents = bones_cases.tree(n)
    bones = sorted({0, n - 1, n // 2, (n - 1) // 2})
    depth = int(np.log2(n)) + 1
    step = 0
    for kind in rm_cases.kinds_for(spec):
        for rounding, per_track in _roundings(kind, n):
            settings = port.settings_for_kind(kind, per_track_policies=per_track)
            duration = rm_cases.clamp_duration(port, blob, settings)
            times = cases.request_times(duration)
            time = times[step % len(times)]
            step += 1
            for root in sorted({0, n - 1}):
                for offsets in cases.offsets_for(duration):
                    for looping in (cases.CLAMP, cases.LOOP):
                        for offset in offsets:
                            writes, c, u = cases.offset_time(time, offset, looping, duration)
                            if not writes:
                                continue
                            context = (name, kind, rounding, root, time, float(offset), looping, c, float(u))
                            # port side
                            local = _zero_pads(port.transform_decompress_tracks(blob, settings, float(u), rounding, port.LOOP_CLAMP))
                            samples = _zero_pads(rm_cases.port_samples(port, blob, settings, rounding, root, time, float(u), duration))
                            # reference side
                            ref_local = _zero_pads(reference.decompress_tracks(blob, float(u), rounding, reference.LOOP_CLAMP, settings=kind,
                                                                               per_track_rounding=per_track))
                            ref_motion, _ = RM.reference_extract(blob, kind, 0, rounding, root, time, float(u), c, per_track_rounding=per_track)
                            ref_objects = cases.object_rows(port, ref_local, parents, bones, port.NORMALIZE_RTM_SSE2)
                            sse_objects = cases.object_rows(port, local, parents, bones, port.NORMALIZE_RTM_SSE2)
                            ieee_objects = cases.object_rows(port, local, parents, bones, port.NORMALIZE_IEEE)
                            sse_motion, _ = RM.port_root_motion(samples, c, RM.NORMALIZE_RTM_SSE2)
                            ieee_motion, _ = RM.port_root_motion(samples, c, RM.NORMALIZE_IEEE)
                            for bone in bones:
                                want = cases.compose(RM, ref_objects[bone], ref_local[root], ref_motion, reference=True)
                                got = cases.compose(RM, sse_objects[bone], local[root], sse_motion, RM.NORMALIZE_RTM_SSE2)
                                assert clips.bit_equal(got, want), context + (bone,)
                                ieee = cases.compose(RM, ieee_objects[bone], local[root], ieee_motion, RM.NORMALIZE_IEEE)
                                assert _gate(want, ieee, depth), context + (bone, ieee, want)


def test_trajectory_entry(oracle_port):
    """With the root a root of the skeleton, its own entry is M up to rounding (qvv_mul(qvv_mul(T, qvv_inverse(T)), M)), for clips whose
    root has scale 1"""
    port = oracle_port
    for name in ("c1_30bones", "looping", "half_turn"):
        spec = clips.TRANSFORM_SPECS[name]
        blob = clips.load_blob(name)
        settings = port.settings_for_kind(1)
        duration = rm_cases.clamp_duration(port, blob, settings)
        parents = bones_cases.tree(spec.num_tracks)
        for offset in cases.offsets_for(duration)[3]:
            writes, c, u = cases.offset_time(0.1, offset, cases.LOOP, duration)
            if not writes:
                continue
            local = _zero_pads(port.transform_decompress_tracks(blob, settings, float(u), 0, port.LOOP_CLAMP))
            samples = _zero_pads(rm_cases.port_samples(port, blob, settings, 0, 0, 0.1, float(u), duration))
            motion, _ = RM.port_root_motion(samples, c)
            row = cases.compose(RM, cases.object_rows(port, local, parents, [0], port.NORMALIZE_IEEE)[0], local[0], motion)
            assert np.allclose(row, motion, atol=1e-5), (name, float(offset))


def test_golden_fixture_reproduces(rm_reference, reference):
    """tests/golden/make_features_golden.py wrote the reference's rows: the reference built here still gives them"""
    from tests.golden import make_features_golden as make
    g = np.load(clips.golden_path("features", "golden.npz"))
    want = make.compute()
    assert set(g.files) == set(want)
    for key in g.files:
        assert np.array_equal(g[key].view(np.uint8), np.ascontiguousarray(want[key]).view(np.uint8)), key
