"""The masked layered decode's oracle (tests/masked_layers_cases.py): the port's composition of decode, per-bone qvv_lerp and
apply_additive_to_base against the unmodified reference's composition of the same steps, and against the committed golden rows
(masked_layers.golden.npz).

The port's rsqrtss flavour reproduces the reference bit for bit on one CPU, whatever the masks and weights. The IEEE flavour is what the GPU
computes: its rotations stay within masked_layers_cases.rotation_gate bone by bone (where every step's weight is in [0, 1], the gate's
derivation), and its translations and scales match bit for bit wherever masked_layers_cases.vectors_exact holds."""
import numpy as np
import pytest

from oracle import additive, blend, port, ref
from tests import additive_cases, clips
from tests import masked_layers_cases as cases

LANES = clips.DEFINED_LANES
NAMED = list(clips.TRANSFORM_SPECS)
BLEND, ADDITIVE, OFF = cases.BLEND, cases.ADDITIVE, cases.OFF


def _needs_reference():
    if not ref.available() or not blend.reference_available() or not additive.reference_available():
        pytest.skip("needs oracle/_ref/libaclref.so, libaclref_blend.so and libaclref_additive.so (the reference tree)")


def _check_ieee(ieee, want, stack, masks, formats, what):
    gate = cases.rotation_gate(stack, masks, formats, want.shape[0])
    finite = np.isfinite(gate)
    error = np.max(np.abs(ieee[:, 0:4] - want[:, 0:4]), axis=1)
    assert (error[finite] <= gate[finite]).all(), what
    if cases.vectors_exact(stack, formats):
        assert clips.bit_equal(ieee[:, [4, 5, 6, 8, 9, 10]], want[:, [4, 5, 6, 8, 9, 10]]), what
    elif finite.all():
        assert float(np.max(np.abs(ieee[:, 4:11] - want[:, 4:11]))) <= cases.vector_gate(stack, masks, formats, want), what


def _compare(blobs, stack, masks, kind, rounding, looping, formats, clip_formats=None, additive_format=0):
    settings, writer = port.settings_for_kind(kind), additive_cases.writer_settings(port, kind)
    want = cases.reference_local(blend, additive, blobs, stack, masks, kind, rounding, looping, additive_format, clip_formats)
    sse2 = cases.port_local(port, blend, blobs, stack, masks, settings, writer, rounding, looping, additive_format, clip_formats,
                            port.NORMALIZE_RTM_SSE2)
    ieee = cases.port_local(port, blend, blobs, stack, masks, settings, writer, rounding, looping, additive_format, clip_formats,
                            port.NORMALIZE_IEEE)
    if want is None:
        assert sse2 is None and ieee is None
        return False
    assert clips.bit_equal(sse2[:, LANES], want[:, LANES]), (kind, stack)
    _check_ieee(ieee, want, stack, masks, formats, (kind, stack))
    return True


@pytest.mark.parametrize("depth", [1, 2, 3, 5, 8])
def test_fixture_stacks_match_live_reference(depth):
    """Mixed ops over the blend and additive clips (every additive format through the per clip table, OFF anywhere), the golden masks
    (0, -0, 1, fractions, above 1, negative) on most layers, weights in [-0.25, 1.25] (rsqrtss flavour bit for bit) and in [0, 1] (IEEE
    flavour within the gate)."""
    _needs_reference()
    blobs = cases.load_blobs()
    masks = cases.golden_masks()
    rng = np.random.default_rng(4800 + depth)
    times = np.array([0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    checked = 0
    for kind, rounding, looping in cases.COMBOS:
        for weights in ((-0.25, 1.25), (0.0, 1.0)):
            for _ in range(6):
                stack = cases.random_stack(rng, depth, len(blobs), times, len(masks), formats_clips=[3, 4, 5], weights=weights)
                checked += _compare(blobs, stack, masks, kind, rounding, looping, cases.FORMATS, clip_formats=np.array(cases.FORMATS))
    assert checked > 0


@pytest.mark.parametrize("name", NAMED)
def test_named_clips(name):
    """Each named clip stacked on itself at different times under masks of its own bone count: blends and every additive format (one
    format per call), depths 1 to 8."""
    _needs_reference()
    blob = clips.load_blob(name)
    n = port.num_tracks_of(blob)
    times = clips.sample_times(clips.TRANSFORM_SPECS[name])
    rng = np.random.default_rng(sum(name.encode()) + 48)
    masks = np.stack([(np.arange(n) >= n // 2).astype(np.float32), np.linspace(0, 1, n, dtype=np.float32),
                      np.resize(np.array([0.0, -0.0, 1.0, 0.5, 1.5, -0.25], np.float32), n)])
    for additive_format in (0, 1, 2, 3):
        for depth in (1, 2, 3, 5, 8):
            stack = cases.random_stack(rng, depth, 1, times, len(masks), allow_off=depth > 1, weights=(0.0, 1.0))
            _compare([blob], stack, masks, 1, 0, 2, [additive_format], additive_format=additive_format)


def test_fixture_clips_every_format_weighted():
    """The blend pair and the additive clips: [base, BLEND under each mask, ADDITIVE of each format at weights 0, 0.5, 1 under each mask]."""
    _needs_reference()
    blobs = cases.load_blobs()
    masks = cases.golden_masks()
    for kind, rounding, looping in cases.COMBOS:
        for m in list(range(len(masks))) + [None]:
            for clip in (3, 4, 5):
                for weight in (0.0, 0.5, 1.0):
                    stack = [(2, 0.3, BLEND, 0.0, None), (0, 0.7, BLEND, 0.6, m), (clip, 0.45, ADDITIVE, weight, m)]
                    assert _compare(blobs, stack, masks, kind, rounding, looping, cases.FORMATS, clip_formats=np.array(cases.FORMATS))


def test_golden_rows_match_the_port():
    """masked_layers.golden.npz (the reference's rows) against the port's IEEE composition, on any machine: rotations within the gate,
    translations and scales bit for bit where vectors_exact holds; where the live reference exists, it still writes the stored rows."""
    golden = np.load(clips.golden_path("masked_layers", "golden.npz"))
    stacks = cases.golden_stacks()
    masks = cases.golden_masks()
    assert golden["combos"].tolist() == [list(c) for c in cases.COMBOS]
    assert np.array_equal(golden["stacks"], cases.stack_array(stacks), equal_nan=True)
    assert clips.bit_equal(golden["masks"], masks)
    blobs = cases.load_blobs()
    formats = np.array(cases.FORMATS)
    live = ref.available() and blend.reference_available() and additive.reference_available()
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        settings, writer = port.settings_for_kind(kind), additive_cases.writer_settings(port, kind)
        for si, stack in enumerate(stacks):
            stored = golden["poses"][ci, si]
            got = cases.port_local(port, blend, blobs, stack, masks, settings, writer, rounding, looping, clip_formats=formats)[:, LANES]
            gate = cases.rotation_gate(stack, masks, cases.FORMATS)
            finite = np.isfinite(gate)
            assert (np.max(np.abs(got[:, 0:4] - stored[:, 0:4]), axis=1)[finite] <= gate[finite]).all(), (kind, si)
            if cases.vectors_exact(stack, cases.FORMATS):
                assert clips.bit_equal(got[:, 4:], stored[:, 4:]), (kind, si)
            if live:
                want = cases.reference_local(blend, additive, blobs, stack, masks, kind, rounding, looping, clip_formats=formats)[:, LANES]
                assert clips.bit_equal(want[:, 4:], stored[:, 4:]), (kind, si)
                assert (np.max(np.abs(want[:, 0:4] - stored[:, 0:4]), axis=1)[finite] <= 2 * gate[finite] + 1e-7).all(), (kind, si)


def test_the_rules_themselves():
    """Weight 1 is the plain apply; a mask of +-0 keeps the running row byte for byte; the weight-0 lerp from the writer defaults gives
    the writer defaults exactly (both flavours, both default scales); unmasked layers with ADDITIVE weight 1 are layers_cases' stack."""
    from tests import layers_cases
    blobs = cases.load_blobs()
    settings, writer = port.settings_for_kind(0), additive_cases.writer_settings(port, 0)
    formats = np.array(cases.FORMATS)
    rng = np.random.default_rng(4810)
    for scale in (0.0, 1.0):
        layer = port.transform_decompress_tracks(blobs[5 if scale == 0.0 else 4], writer, 0.4, 0, 2)
        for mode in (port.NORMALIZE_IEEE, port.NORMALIZE_RTM_SSE2):
            lerped = blend.port_qvv_lerp(cases.writer_default_rows(24, scale), layer, 0.0, mode)
            assert clips.bit_equal(lerped, cases.writer_default_rows(24, scale))
    for clip in (3, 4, 5):
        base = [(2, 0.3, BLEND, 0.0, None)]
        plain = layers_cases.port_local(port, blend, blobs, [layer[:4] for layer in base] + [(clip, 0.5, ADDITIVE, 0.0)], settings, writer,
                                        0, 2, clip_formats=formats)
        weighted = cases.port_local(port, blend, blobs, base + [(clip, 0.5, ADDITIVE, 1.0, None)], cases.golden_masks(), settings, writer, 0, 2,
                                    clip_formats=formats)
        assert clips.bit_equal(plain, weighted)
        masks = np.stack([np.zeros(24, np.float32), np.full(24, -0.0, np.float32)])
        for m in (0, 1):
            kept = cases.port_local(port, blend, blobs, base + [(clip, 0.5, ADDITIVE, 0.5, m), (0, 0.2, BLEND, 0.3, m)], masks, settings,
                                    writer, 0, 2, clip_formats=formats)
            alone = port.transform_decompress_tracks(blobs[2], settings, 0.3, 0, 2)
            assert clips.bit_equal(kept, alone)
    times = np.array([0.0, 0.3, 0.9], np.float32)
    for _ in range(20):
        stack = layers_cases.random_stack(rng, 4, 6, times)
        stack = [(c, t, op, 1.0 if op == ADDITIVE else w) for c, t, op, w in stack]
        plain = layers_cases.port_local(port, blend, blobs, stack, settings, writer, 0, 2, clip_formats=formats)
        masked = cases.port_local(port, blend, blobs, [layer + (None,) for layer in stack], cases.golden_masks(), settings, writer, 0, 2,
                                  clip_formats=formats)
        assert (plain is None and masked is None) or clips.bit_equal(plain, masked)
