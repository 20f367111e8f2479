"""The layered decode's oracle (tests/layers_cases.py): the port's composition of decode, qvv_lerp and apply_additive_to_base against the
unmodified reference's composition of the same steps, and against the committed golden rows (layers.golden.npz).

The port's rsqrtss flavour of quat_normalize reproduces the reference bit for bit on one CPU, so that composition must match the live
reference in every lane. The IEEE flavour is what the GPU computes: its translations and scales match bit for bit wherever no `relative`
layer follows a step that moved the rotation (layers_cases.vectors_exact), and its rotations stay within layers_cases.rotation_gate, the
per step blend gate carried through the later steps (the derivation is beside rotation_gate)."""
import numpy as np
import pytest

from oracle import additive, blend, port, ref
from tests import additive_cases, clips
from tests import layers_cases as cases

LANES = clips.DEFINED_LANES
NAMED = list(clips.TRANSFORM_SPECS)


def _needs_reference():
    if not ref.available() or not blend.reference_available() or not additive.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so, libaclref_blend.so and libaclref_additive.so (the reference tree)")


def _compare(blobs, stack, kind, rounding, looping, formats, clip_formats=None, additive_format=0):
    settings, writer = port.settings_for_kind(kind), additive_cases.writer_settings(port, kind)
    want = cases.reference_local(blend, additive, blobs, stack, kind, rounding, looping, additive_format, clip_formats)
    sse2 = cases.port_local(port, blend, blobs, stack, settings, writer, rounding, looping, additive_format, clip_formats, port.NORMALIZE_RTM_SSE2)
    ieee = cases.port_local(port, blend, blobs, stack, settings, writer, rounding, looping, additive_format, clip_formats, port.NORMALIZE_IEEE)
    if want is None:
        assert sse2 is None and ieee is None
        return False
    assert clips.bit_equal(sse2[:, LANES], want[:, LANES]), (kind, stack)
    assert float(np.max(np.abs(ieee[:, 0:4] - want[:, 0:4]))) <= cases.rotation_gate(stack, formats), (kind, stack)
    if cases.vectors_exact(stack, formats):
        assert clips.bit_equal(ieee[:, [4, 5, 6, 8, 9, 10]], want[:, [4, 5, 6, 8, 9, 10]]), (kind, stack)
    else:
        assert float(np.max(np.abs(ieee[:, 4:11] - want[:, 4:11]))) <= cases.vector_gate(stack, formats, want), (kind, stack)
    return True


@pytest.mark.parametrize("depth", list(range(1, 9)))
def test_fixture_stacks_match_live_reference(depth):
    """Mixed ops over the blend and additive clips (all three additive formats through the per clip table, OFF anywhere), weights in
    [0, 1] where the gate's derivation holds: every combo."""
    _needs_reference()
    blobs = cases.load_blobs()
    formats = cases.FORMATS
    rng = np.random.default_rng(4600 + depth)
    times = np.array([0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    checked = 0
    for kind, rounding, looping in cases.COMBOS:
        for _ in range(12):
            stack = cases.random_stack(rng, depth, len(blobs), times, formats_clips=[3, 4, 5])
            stack = [(c, t, op, min(max(w, 0.0), 1.0)) for c, t, op, w in stack]
            checked += _compare(blobs, stack, kind, rounding, looping, formats, clip_formats=np.array(formats))
    assert checked > 0


@pytest.mark.parametrize("name", NAMED)
def test_named_clips(name):
    """Each named clip stacked on itself at different times: blends and every additive format (one format per call), depths 1 to 8."""
    _needs_reference()
    blob = clips.load_blob(name)
    times = clips.sample_times(clips.TRANSFORM_SPECS[name])
    rng = np.random.default_rng(sum(name.encode()))
    for additive_format in (0, 1, 2, 3):
        formats = [additive_format]
        for depth in (1, 2, 3, 5, 8):
            stack = cases.random_stack(rng, depth, 1, times, allow_off=depth > 1)
            stack = [(c, t, op, min(max(w, 0.0), 1.0)) for c, t, op, w in stack]
            _compare([blob], stack, 1, 0, 2, formats, additive_format=additive_format)


def test_golden_rows_match_the_port():
    """layers.golden.npz (the reference's rows) against the port's IEEE composition, on any machine: translations and scales bit for bit
    where vectors_exact holds, rotations within the gate; where the live reference exists, it still writes the stored rows (vectors bit for
    bit, rotations within the gate: the stored rotations carry the rsqrtss estimate of the CPU that wrote them)."""
    golden = np.load(clips.golden_path("layers", "golden.npz"))
    stacks = cases.golden_stacks()
    assert golden["combos"].tolist() == [list(c) for c in cases.COMBOS]
    assert np.array_equal(golden["stacks"], cases.stack_array(stacks), equal_nan=True)
    blobs = cases.load_blobs()
    formats = np.array(cases.FORMATS)
    live = ref.available() and blend.reference_available() and additive.reference_available()
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        settings, writer = port.settings_for_kind(kind), additive_cases.writer_settings(port, kind)
        for si, stack in enumerate(stacks):
            stored = golden["poses"][ci, si]
            got = cases.port_local(port, blend, blobs, stack, settings, writer, rounding, looping, clip_formats=formats)[:, LANES]
            gate = cases.rotation_gate(stack, cases.FORMATS)
            assert float(np.max(np.abs(got[:, 0:4] - stored[:, 0:4]))) <= gate, (kind, si)
            if cases.vectors_exact(stack, cases.FORMATS):
                assert clips.bit_equal(got[:, 4:], stored[:, 4:]), (kind, si)
            if live:
                want = cases.reference_local(blend, additive, blobs, stack, kind, rounding, looping, clip_formats=formats)[:, LANES]
                assert clips.bit_equal(want[:, 4:], stored[:, 4:]) or not cases.vectors_exact(stack, cases.FORMATS), (kind, si)
                assert float(np.max(np.abs(want[:, 0:4] - stored[:, 0:4]))) <= 2 * gate + 1e-7, (kind, si)


def test_blend_space_step_weights():
    """The header's rule for a normalised blend space: step weights w_i = a_i / (a_0 + ... + a_i) make the chain of lerps give sum a_i x_i
    (checked on translations, which qvv_lerp lerps without normalising)."""
    rng = np.random.default_rng(4610)
    a = rng.uniform(0.1, 1.0, 5)
    a /= a.sum()
    x = rng.uniform(-3, 3, (5, 3))
    acc = x[0]
    for i in range(1, 5):
        w = a[i] / a[:i + 1].sum()
        acc = (1 - w) * acc + w * x[i]
    assert np.allclose(acc, (a[:, None] * x).sum(0), atol=1e-12)
