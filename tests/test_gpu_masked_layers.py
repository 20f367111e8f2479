"""aclb200_decompress_tracks_layered_masked and _layered_masked_skinning (bone masks on any layer, weighted ADDITIVE layers, folded in one
kernel) against
  * the port's composition of its pinned per-operation oracles (tests/masked_layers_cases.py): BIT FOR BIT, local, object (qvvf, matrix)
    and skinning rows;
  * the existing entry points, byte for byte: no masks with ADDITIVE weights 1 and all-ones masks equal decompress_tracks_layered
    (_layered_skinning); a layer whose mask is 0 everywhere equals the stack with that layer OFF; a 0/1 mask gives each bone the row of
    the full stack or of the stack without the layer;
  * masked_layers.golden.npz, the reference's composition: rotations within masked_layers_cases.rotation_gate, translations and scales
    bit for bit where masked_layers_cases.vectors_exact holds.
"""
import numpy as np
import pytest

from oracle import blend, object_space, skinning
from tests import additive_cases, clips
from tests import database_cases as dbcases
from tests import masked_layers_cases as cases
from tests import skinning_cases

pytestmark = pytest.mark.gpu
LANES = clips.DEFINED_LANES
ROOT = 0xFFFFFFFF
SENTINEL = 0x7FC00001
OFF, BLEND, ADDITIVE = cases.OFF, cases.BLEND, cases.ADDITIVE
NO_MASK = cases.NO_MASK


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    ctx = ab.Context(0)
    # the six 24 bone clips of tests/layers_cases.py, then a 30 bone clip (a track count mismatch for the others)
    blobs = cases.load_blobs() + [clips.load_blob("c1_30bones")]
    formats = np.array(cases.FORMATS + [7], np.uint8)       # a byte above 3 reads as none
    clipset = ctx.upload(blobs, check_hash=True)
    # masks of 30 floats (the clip set's max_tracks): the golden masks (24 bone rig) padded with 9, then two masks of the 30 bone rig
    masks = np.full((7, 30), 9.0, np.float32)
    masks[:5, :24] = cases.golden_masks()
    masks[5] = (np.arange(30) >= 15).astype(np.float32)
    masks[6] = np.clip((np.arange(30) - 10) * 0.25, 0.0, 1.0)
    return dict(torch=torch, ab=ab, port=port, ctx=ctx, blobs=blobs, formats=formats, clipset=clipset, masks=masks)


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8)).cuda()


def _options(gpu, kind, **kw):
    s = gpu["port"].settings_for_kind(kind).c
    fields = dict(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                  clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                  default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                  constant_defaults=list(s.constant_defaults))
    fields.update(kw)
    return gpu["ab"].Options(**fields)


def _layers(gpu, stacks):
    """list of equal depth masked stacks -> (aclb200_layer[num_poses][num_layers], uint32 mask indices)"""
    a = np.array([[layer[:4] for layer in stack] for stack in stacks], np.float64)
    masks = np.array([[NO_MASK if layer[4] is None else layer[4] for layer in stack] for stack in stacks], np.uint32)
    return gpu["ab"].make_layers(a[..., 0].astype(np.uint32), a[..., 1], a[..., 2].astype(np.uint32), a[..., 3]), masks


def _run(gpu, stacks, options, clipset=None, width=None, skinning_call=False, masks=None, no_layer_masks=False, **kw):
    torch, ctx = gpu["torch"], gpu["ctx"]
    clipset = clipset or gpu["clipset"]
    masks = gpu["masks"] if masks is None else masks
    n, depth = len(stacks), len(stacks[0])
    d_out = torch.full((n, width or clipset.max_tracks * 12), SENTINEL, dtype=torch.int32, device="cuda")
    layers, layer_masks = _layers(gpu, stacks)
    mask_kw = dict(d_bone_masks=_dev(gpu, masks), num_masks=masks.shape[0], mask_stride=masks.shape[1])
    if not no_layer_masks:
        mask_kw["d_layer_masks"] = _dev(gpu, layer_masks)
    if skinning_call:
        ctx.decompress_tracks_layered_masked_skinning(clipset, _dev(gpu, layers), n, depth, options, kw.pop("d_parent_indices"),
                                                      kw.pop("d_inverse_bind"), d_out, **mask_kw, **kw)
    else:
        ctx.decompress_tracks_layered_masked(clipset, _dev(gpu, layers), n, depth, options, d_out, **mask_kw, **kw)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def _rows_equal(got, want, layout_40=False):
    """defined lanes bit for bit; QVV48 rows carry 0 in the translation and scale w lanes"""
    if layout_40:
        return clips.bit_equal(got, want[:, LANES])
    return clips.bit_equal(got[:, LANES], want[:, LANES]) and not got[:, [7, 11]].view(np.uint32).any()


def _counts(gpu):
    return [gpu["port"].num_tracks_of(b) for b in gpu["blobs"]]


def _expected(gpu, stack, kind, rounding=0, looping=2, settings=None, writer=None, clip_formats=True, additive_format=0, masks=None):
    port = gpu["port"]
    return cases.port_local(port, blend, gpu["blobs"], stack, gpu["masks"] if masks is None else masks, settings or port.settings_for_kind(kind),
                            writer or additive_cases.writer_settings(port, kind), rounding, looping, additive_format=additive_format,
                            clip_formats=gpu["formats"] if clip_formats else None)


def _random_stacks(rng, count, depth, num_clips=7, off_first=False, num_masks=7):
    times = np.array([-0.1, 0.0, 0.13, 0.41, 0.77, 1.2, 5.0], np.float32)
    stacks = [cases.random_stack(rng, depth, num_clips, times, num_masks) for _ in range(count)]
    if off_first:
        for stack in stacks[::3]:
            stack[0] = (ROOT, float("nan"), OFF, float("nan"), 1000)
    for stack in stacks[5::11]:
        stack[-1] = (40, 0.2, BLEND, 0.5, 0)                # an invalid clip on a layer that is not OFF
    for stack in stacks[7::13]:
        stack[-1] = stack[-1][:4] + (num_masks,)            # a mask index at num_masks: written nothing when the layer is live
    return stacks


def _check_local(gpu, got, stacks, kind, rounding=0, looping=2, layout_40=False, policies=None, **kw):
    bone = 10 if layout_40 else 12
    counts = _counts(gpu)
    written = 0
    for i, stack in enumerate(stacks):
        r, l = (int(policies[i][0]), int(policies[i][1])) if policies is not None else (rounding, looping)
        want = _expected(gpu, stack, kind, r, l, **kw)
        if want is None:
            assert (got[i].view(np.int32) == SENTINEL).all(), (i, stack)
            continue
        n = counts[stack[cases._base(stack)][0]]
        assert (got[i, n * bone:].view(np.int32) == SENTINEL).all(), (i, stack)
        assert _rows_equal(got[i, :n * bone].view(np.float32).reshape(n, bone), want, layout_40), (kind, r, l, i, stack)
        written += 1
    return written


@pytest.mark.parametrize("depth", [1, 2, 3, 5, 8])
def test_against_the_port(gpu, depth):
    """Every clip, every settings kind combo, both layouts, masks with 0, -0, 1, fractions, values above 1 and negative ones on most layers,
    ADDITIVE weights in [-0.25, 1.25] (1 a quarter of the time), OFF anywhere, invalid clips, out of range mask indices, the per clip
    format table and one format for all: bit for bit against the port's IEEE composition."""
    ab = gpu["ab"]
    rng = np.random.default_rng(4900 + depth)
    stacks = _random_stacks(rng, 160, depth, off_first=depth > 1)
    written = 0
    for kind, rounding, looping in cases.COMBOS:
        for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
            options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping, output_layout=layout,
                               pose_stride_bytes=gpu["clipset"].max_tracks * 48)
            got = _run(gpu, stacks, options, d_clip_additive_formats=_dev(gpu, gpu["formats"]))
            width = 12 if layout == ab.LAYOUT_QVV48 else 10
            got = got[:, :gpu["clipset"].max_tracks * width].view(np.float32)
            written += _check_local(gpu, got, stacks, kind, rounding, looping, layout == ab.LAYOUT_QVV40)
    assert written > len(stacks)
    for additive_format in (0, 1, 2, 3):
        got = _run(gpu, stacks, _options(gpu, 0), additive_format=additive_format)
        _check_local(gpu, got.view(np.float32), stacks, 0, clip_formats=False, additive_format=additive_format)


def test_per_request_policies_and_variable_defaults(gpu):
    """d_request_policies[r] applies to every layer of pose r; a variable bind pose reaches the base and the BLEND layers, while ADDITIVE
    layers keep the track_writer defaults (and lerp from them)."""
    torch, port, ab = gpu["torch"], gpu["port"], gpu["ab"]
    rng = np.random.default_rng(4910)
    stacks = _random_stacks(rng, 120, 4, num_clips=6, off_first=True)
    policies = np.resize(np.array([(r, l) for r in range(4) for l in range(3)], np.uint8), (len(stacks), 2))
    n = 24
    variable = np.tile(np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32), (gpu["clipset"].max_tracks, 1))
    variable[:, 4:7] = rng.uniform(-2, 2, (variable.shape[0], 3))
    variable[:, 8:11] = rng.uniform(0.5, 1.5, (variable.shape[0], 3))
    d_variable = torch.from_numpy(variable).cuda()
    settings = port.settings_for_kind(0, default_modes=(port.DEFAULT_VARIABLE,) * 3, variable_defaults=variable[:n])
    d_policies = _dev(gpu, policies)
    options = _options(gpu, 0, d_request_policies=d_policies.data_ptr(), default_modes=(ab.DEFAULT_VARIABLE,) * 3,
                       d_variable_defaults=d_variable.data_ptr())
    got = _run(gpu, stacks, options, d_clip_additive_formats=_dev(gpu, gpu["formats"]))
    assert _check_local(gpu, got.view(np.float32), stacks, 0, policies=policies, settings=settings) > 50


def _skeletons(gpu):
    counts = _counts(gpu)
    skeletons = [skinning_cases.skeleton(["tree", "chain", "random"][c % 3], n, seed=c) for c, n in enumerate(counts)]
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    return skeletons, offsets, np.concatenate(skeletons)


def _rig_stacks(rng, count, depth):
    """stacks over both rigs (clips 0..5 with 24 bones, clip 6 with 30), each layer's mask from its stack's rig (0..4: 24 bones, 5, 6: 30)"""
    times = np.array([0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    stacks = []
    for i in range(count):
        if i % 4 == 3:
            stack = [(6, float(rng.choice(times)), BLEND, float(rng.uniform(0, 1)), int(rng.choice([5, 6]))) for _ in range(depth)]
            stack[-1] = (6, stack[-1][1], ADDITIVE, 0.5, 6)
        else:
            stack = cases.random_stack(rng, depth, 6, times, 5, formats_clips=[3, 4, 5])
        stacks.append(stack)
    return stacks


def test_object_space_and_skinning_mixed_rigs(gpu):
    """With parents the running pose walks the BASE clip's skeleton (mixed rigs through skeleton offsets, each layer masked with a mask of
    its stack's rig): qvvf rows, 3x4 matrices and skinning rows against the port's walk of the port's composition."""
    torch, ab, port = gpu["torch"], gpu["ab"], gpu["port"]
    rng = np.random.default_rng(4920)
    stacks = _rig_stacks(rng, 150, 5)
    skeletons, offsets, parents = _skeletons(gpu)
    inverse = skinning_cases.random_affine(len(parents), 4921, mirrored=True)
    d_parents, d_offsets = _dev(gpu, parents), _dev(gpu, offsets)
    d_formats = _dev(gpu, gpu["formats"])
    counts = _counts(gpu)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    checked = 0
    for route in ("qvvf", "matrix", "skinning"):
        kw = dict(d_skeleton_offsets=d_offsets, d_clip_additive_formats=d_formats, d_out_flags=d_flags)
        if route == "skinning":
            got = _run(gpu, stacks, ab.Options(), skinning_call=True, d_parent_indices=d_parents, d_inverse_bind=_dev(gpu, inverse), **kw)
        else:
            got = _run(gpu, stacks, ab.Options(), d_parent_indices=d_parents, kind=ab.OBJECT_QVVF if route == "qvvf" else ab.OBJECT_MATRIX3X4F, **kw)
        got = got.view(np.float32)
        for i, stack in enumerate(stacks):
            local = _expected(gpu, stack, 0)
            if local is None:
                assert (got[i].view(np.int32) == SENTINEL).all(), (route, i)
                continue
            c = stack[cases._base(stack)][0]
            n = counts[c]
            row = got[i, :n * 12].reshape(n, 12)
            assert (got[i, n * 12:].view(np.int32) == SENTINEL).all(), (route, i)
            if route == "qvvf":
                assert _rows_equal(row, port.local_to_object_space(local, skeletons[c], port.NORMALIZE_IEEE)), (route, i, stack)
            elif route == "matrix":
                assert clips.bit_equal(row, object_space.port_local_to_object_space_matrix(local, skeletons[c])), (route, i, stack)
            else:
                want = skinning.port_local_to_skinning(local, skeletons[c], inverse[offsets[c]:offsets[c] + n])
                assert clips.bit_equal(row, want), (route, i, stack)
            checked += c == 6
    assert checked > 0


def test_equivalences_with_the_plain_layered_decode(gpu):
    """Byte for byte, buffers filled with one sentinel: no masks (NULL, and every index NO_MASK) with ADDITIVE weights 1, and all-ones masks,
    equal decompress_tracks_layered (local, object, skinning, flags); a layer whose mask is 0 on every bone equals that layer OFF; an
    upper/lower 0/1 mask gives each bone the row of the full stack or of the stack with the layer OFF, and local_to_skinning of that local
    pose equals the masked skinning route."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = gpu["clipset"]
    rng = np.random.default_rng(4930)
    times = np.array([-0.1, 0.0, 0.13, 0.41, 0.77, 1.2], np.float32)
    stacks = [cases.random_stack(rng, 4, 6, times, 5, formats_clips=[3, 4, 5]) for _ in range(240)]
    stacks = [[(c, t, op, 1.0 if op == ADDITIVE else w, m) for c, t, op, w, m in stack] for stack in stacks]
    skeletons, offsets, parents = _skeletons(gpu)
    inverse = skinning_cases.random_affine(len(parents), 4931)
    d_parents, d_offsets, d_inverse = _dev(gpu, parents), _dev(gpu, offsets), _dev(gpu, inverse)
    d_formats = _dev(gpu, gpu["formats"])
    m, width = len(stacks), clipset.max_tracks * 12

    def plain(stack_list, route, options):
        layers, _ = _layers(gpu, stack_list)
        out = torch.full((len(stack_list), width), SENTINEL, dtype=torch.int32, device="cuda")
        flags = torch.full((1,), 7, dtype=torch.int32, device="cuda")
        kw = dict(d_clip_additive_formats=d_formats, d_skeleton_offsets=d_offsets, d_out_flags=flags)
        if route == "skinning":
            ctx.decompress_tracks_layered_skinning(clipset, _dev(gpu, layers), len(stack_list), 4, options, d_parents, d_inverse, out, **kw)
        elif route == "local":
            ctx.decompress_tracks_layered(clipset, _dev(gpu, layers), len(stack_list), 4, options, out, **kw)
        else:
            ctx.decompress_tracks_layered(clipset, _dev(gpu, layers), len(stack_list), 4, options, out, d_parent_indices=d_parents,
                                          kind=ab.OBJECT_MATRIX3X4F, **kw)
        torch.cuda.synchronize()
        return out.cpu().numpy(), int(flags.item())

    def masked(stack_list, route, options, **kw):
        flags = torch.full((1,), 9, dtype=torch.int32, device="cuda")
        common = dict(d_clip_additive_formats=d_formats, d_skeleton_offsets=d_offsets, d_out_flags=flags)
        if route == "skinning":
            out = _run(gpu, stack_list, options, skinning_call=True, d_parent_indices=d_parents, d_inverse_bind=d_inverse, **common, **kw)
        elif route == "local":
            out = _run(gpu, stack_list, options, **common, **kw)
        else:
            out = _run(gpu, stack_list, options, d_parent_indices=d_parents, kind=ab.OBJECT_MATRIX3X4F, **common, **kw)
        return out, int(flags.item())

    unmasked = [[layer[:4] + (None,) for layer in stack] for stack in stacks]
    ones = [[layer[:4] + (4,) for layer in stack] for stack in stacks]
    for route in ("local", "object", "skinning"):
        for layout in ((ab.LAYOUT_QVV48, ab.LAYOUT_QVV40) if route == "local" else (ab.LAYOUT_QVV48,)):
            options = ab.Options(output_layout=layout)
            want = plain(stacks, route, options)
            got = [masked(unmasked, route, options, no_layer_masks=True), masked(unmasked, route, options), masked(ones, route, options)]
            for g, what in zip(got, ("NULL", "NO_MASK", "all ones")):
                assert np.array_equal(g[0], want[0]) and g[1] == want[1], (route, layout, what)

    # a mask of 0 (mask 3) on layer 2: the layer OFF; the upper/lower mask (mask 0) on layer 2: per bone, one or the other
    zero = [stack[:2] + [stack[2][:4] + (3,)] + stack[3:] for stack in unmasked]
    off = [stack[:2] + [(ROOT, float("nan"), OFF, 0.0, None)] + stack[3:] for stack in unmasked]
    half = [stack[:2] + [stack[2][:4] + (0,)] + stack[3:] for stack in unmasked]
    options = ab.Options()
    without, _ = masked(off, "local", options)
    zeroed, _ = masked(zero, "local", options)
    layer2_above_base = [cases._base(stack) is not None and cases._base(stack) < 2 for stack in unmasked]
    assert sum(layer2_above_base) > m // 2
    for i in range(m):
        if layer2_above_base[i]:
            assert np.array_equal(zeroed[i], without[i]), (i, unmasked[i])
    full, _ = masked(unmasked, "local", options)
    got, _ = masked(half, "local", options)
    upper = np.repeat(np.arange(clipset.max_tracks) >= 12, 12)
    lower_ok = [np.array_equal(got[i, :width][~upper], without[i, :width][~upper]) for i in range(m)]
    upper_ok = [np.array_equal(got[i, :width][upper], full[i, :width][upper]) for i in range(m)]
    counts = _counts(gpu)
    for i, stack in enumerate(half):
        if cases.writes_nothing(stack, counts, 5) or cases.writes_nothing(off[i], counts, 5):
            continue
        if not layer2_above_base[i]:
            continue                                          # layer 2 is the base there: the mask is not read
        assert lower_ok[i] and upper_ok[i], (i, stack)
    # local_to_skinning of the masked local pose of 24 bone stacks equals the masked skinning route
    rig = [i for i, stack in enumerate(half) if not cases.writes_nothing(stack, counts, 5) and stack[cases._base(stack)][0] == 0]
    local = torch.from_numpy(np.ascontiguousarray(got[rig, :24 * 12])).cuda()
    ctx.local_to_skinning(local, local, len(rig), 24, d_parents, d_inverse)          # clip 0's skeleton and inverse binds are at offset 0
    fused, _ = masked([half[i] for i in rig], "skinning", options)
    torch.cuda.synchronize()
    assert np.array_equal(local.cpu().numpy(), fused[:, :24 * 12])


def test_c2_stacks(gpu):
    """300,000 four layer stacks over the C2 bench clips (base, BLEND, BLEND, ADDITIVE additive0): all-ones masks with ADDITIVE weight 1 write
    byte for byte what decompress_tracks_layered writes; an upper-body mask on the BLEND layers with a feather band and ADDITIVE weight 0.5
    matches the port's composition bit for bit on a seeded sample of 200 poses."""
    import bench
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    m, bones = 300000, w["num_tracks"]
    rng = np.random.default_rng(4940)
    clip = [w["req_clip"][:m]] + [rng.permutation(w["req_clip"])[:m] for _ in range(3)]
    time = [w["req_time"][:m]] + [rng.permutation(w["req_time"])[:m] for _ in range(3)]
    weight = [np.zeros(m, np.float32), rng.uniform(0, 1, m).astype(np.float32), rng.uniform(-0.25, 1.25, m).astype(np.float32)]
    ops = np.array([[BLEND, BLEND, BLEND, ADDITIVE]], np.uint32)
    options = ab.Options()
    upper = np.zeros(bones, np.float32)
    upper[bones // 2:] = 1.0
    upper[bones // 2 - 3:bones // 2] = [0.25, 0.5, 0.75]
    masks = np.stack([np.ones(bones, np.float32), upper])
    d_masks = _dev(gpu, masks)
    outs = []
    for additive_weight, mask in ((1.0, 0), (0.5, 1)):
        layers = _dev(gpu, ab.make_layers(np.stack(clip, 1), np.stack(time, 1), ops,
                                          np.stack(weight + [np.full(m, additive_weight, np.float32)], 1)))
        layer_masks = _dev(gpu, np.tile(np.array([NO_MASK, mask, mask, NO_MASK], np.uint32), m))
        out = torch.full((m, bones, 12), float("nan"), dtype=torch.float32, device="cuda")
        ctx.decompress_tracks_layered_masked(clipset, layers, m, 4, options, out, d_layer_masks=layer_masks, d_bone_masks=d_masks, num_masks=2,
                                             additive_format=ab.ADDITIVE_ADDITIVE0)
        outs.append((layers, out))
    plain = torch.full((m, bones, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.decompress_tracks_layered(clipset, outs[0][0], m, 4, options, plain, additive_format=ab.ADDITIVE_ADDITIVE0)
    torch.cuda.synchronize()
    assert torch.equal(plain.view(torch.int32), outs[0][1].view(torch.int32))
    got = outs[1][1].cpu().numpy()
    settings, writer = port.settings_for_kind(0), additive_cases.writer_settings(port, 0)
    buffer = np.asarray(w["buffer"])
    for r in np.random.default_rng(4941).choice(m, 200, replace=False):
        blobs = [buffer[int(w["offsets"][c]):int(w["offsets"][c]) + int(w["sizes"][c])] for c in (clip[k][r] for k in range(4))]
        stack = [(0, float(time[0][r]), BLEND, 0.0, None), (1, float(time[1][r]), BLEND, float(weight[1][r]), 1),
                 (2, float(time[2][r]), BLEND, float(weight[2][r]), 1), (3, float(time[3][r]), ADDITIVE, 0.5, None)]
        want = cases.port_local(port, blend, blobs, stack, masks, settings, writer, 0, ab.LOOP_AS_COMPRESSED,
                                additive_format=ab.ADDITIVE_ADDITIVE0)
        assert _rows_equal(got[r], want), r
    clipset.release()


def test_poses_that_write_nothing_and_refusals(gpu):
    """An out of range mask index, an invalid clip on a masked layer (and everything _layered writes nothing for) write nothing; a mask
    index on the base or an OFF layer is not read; every refusal writes nothing and leaves the flags untouched."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    good = [(0, 0.3, BLEND, 0.0, None), (1, 0.2, BLEND, 0.5, 0), (4, 0.1, ADDITIVE, 0.5, 1)]
    stacks = [
        good,
        [(0, 0.3, BLEND, 0.0, None), (1, 0.2, BLEND, 0.5, 7), (4, 0.1, ADDITIVE, 0.0, None)],          # mask index == num_masks
        [(0, 0.3, BLEND, 0.0, None), (1, 0.2, BLEND, 0.5, None), (4, 0.1, ADDITIVE, 0.5, 0x7FFFFFFF)],  # far out of range
        [(0, 0.3, BLEND, 0.0, None), (9, 0.2, BLEND, 0.5, 0), (4, 0.1, ADDITIVE, 0.5, 1)],             # invalid clip on a masked layer
        [(0, 0.3, BLEND, 0.0, None), (6, 0.2, BLEND, 0.5, 2), (4, 0.1, ADDITIVE, 0.0, None)],          # 30 bones under a 24 bone base
        [(0, 0.3, BLEND, 0.0, None), (1, 0.2, 3, 0.5, 0), (4, 0.1, ADDITIVE, 0.0, None)],              # unknown op
        [(0, 0.3, BLEND, 0.0, 1000), (1, 0.2, BLEND, 0.5, 0), (4, 0.1, ADDITIVE, 0.5, 1)],             # the base's mask: not read
        [(0, 0.3, OFF, 0.0, 1000), (1, 0.2, BLEND, 0.5, 1000), (4, 0.1, ADDITIVE, 0.5, 1)],            # OFF and base masks: not read
    ]
    got = _run(gpu, stacks, ab.Options())
    for i in (0, 6, 7):
        assert not (got[i].view(np.int32) == SENTINEL).all(), i
    assert (got[0, 24 * 12:] == SENTINEL).all()
    for i in range(1, 6):
        assert (got[i] == SENTINEL).all(), i
    _check_local(gpu, got.view(np.float32), stacks, 0, clip_formats=False)

    layers, layer_masks = _layers(gpu, [good] * 8)
    layers, layer_masks = _dev(gpu, layers), _dev(gpu, layer_masks)
    masks = torch.zeros(64 * 30 + 4, dtype=torch.float32, device="cuda")
    parents = _dev(gpu, np.where(np.arange(30) == 0, ROOT, np.arange(30) - 1).astype(np.uint32))
    inverse = torch.zeros((30, 12), dtype=torch.float32, device="cuda")
    scalar = ctx.upload([clips.load_blob("float1")])
    m = masks.data_ptr()
    refusals = [
        # the mask table's own refusals
        dict(bone_masks=0), dict(num_masks=0), dict(bone_masks=m + 2), dict(num_masks=1 << 29), dict(mask_stride=29),
        dict(num_masks=0x10000, mask_stride=0x10000), dict(skin=True, parents=parents, inverse=inverse, bone_masks=m + 1),
        # _layered's refusals, through the masked entry points
        dict(num_layers=0), dict(num_layers=9), dict(num_poses=0x20000000, num_layers=8),
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(additive_format=4), dict(clipset=scalar),
        dict(parents=parents, kind=2),
        dict(parents=parents, options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(offset=8), dict(options=ab.Options(pose_stride_bytes=30 * 48 + 8)),
        dict(skin=True), dict(skin=True, parents=parents), dict(skin=True, parents=parents, inverse=inverse.data_ptr() + 4),
    ]
    for case in refusals:
        buffer = torch.full((8 * 30 * 48 + 128,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        args = (case.get("clipset", gpu["clipset"]), layers, case.get("num_poses", 8), case.get("num_layers", 3), case.get("options", ab.Options()))
        mask_kw = dict(d_layer_masks=layer_masks, d_bone_masks=case.get("bone_masks", m), num_masks=case.get("num_masks", 2),
                       mask_stride=case.get("mask_stride", 0))
        out = buffer.data_ptr() + case.get("offset", 0)
        with pytest.raises(ab.api.AclB200Error) as error:
            if case.get("skin"):
                ctx.decompress_tracks_layered_masked_skinning(*args, case.get("parents"), case.get("inverse"), out, d_out_flags=d_flags, **mask_kw)
            else:
                ctx.decompress_tracks_layered_masked(*args, out, additive_format=case.get("additive_format", 0),
                                                     d_parent_indices=case.get("parents"), kind=case.get("kind", 0), d_out_flags=d_flags,
                                                     **mask_kw)
        assert error.value.status == 1, case             # ACLB200_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    scalar.release()


def test_wide_pose_limits(gpu):
    """wide_2500 (2500 bones) keeps the _layered limits: one QVV48 pose fits one block and two do not (ACLB200_ERR_UNSUPPORTED, nothing
    written); the one layer stacks that fit are the port's poses."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    blob = clips.load_blob("wide_2500")
    clipset = ctx.upload([blob])
    masks = np.linspace(0, 1, 2500, dtype=np.float32)[None, :]
    options = ab.Options(pose_stride_bytes=2500 * 48)
    stacks = [[(0, 0.05 * (i + 1), BLEND, 0.0, None), (0, 0.27, BLEND, 0.5, 0)] for i in range(3)]
    buffer = torch.full((3, 2500 * 12), SENTINEL, dtype=torch.int32, device="cuda")
    layers, layer_masks = _layers(gpu, stacks)
    with pytest.raises(ab.api.AclB200Error) as error:
        ctx.decompress_tracks_layered_masked(clipset, _dev(gpu, layers), 3, 2, options, buffer, d_layer_masks=_dev(gpu, layer_masks),
                                             d_bone_masks=_dev(gpu, masks), num_masks=1)
    assert error.value.status == 3                       # ACLB200_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (buffer.cpu().numpy() == SENTINEL).all()
    stacks = [stack[:1] for stack in stacks]
    got = _run(gpu, stacks, options, clipset=clipset, width=2500 * 12, masks=masks).view(np.float32)
    settings, writer = port.settings_for_kind(0), additive_cases.writer_settings(port, 0)
    for i, stack in enumerate(stacks):
        want = cases.port_local(port, blend, [blob], stack, masks, settings, writer, 0, ab.LOOP_AS_COMPRESSED)
        assert _rows_equal(got[i].reshape(2500, 12), want), i
    clipset.release()


def test_database_tiers(gpu):
    """A clip set bound to a database, in every tier state of tests/database_cases.py: [base, BLEND 0.375 under a feathered mask, OFF]
    stacks decode every layer from what is streamed in, against the reference's poses of those states lerped bone by bone."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    reference = _Reference(ref, ref_database)
    blobs = reference.bound + [reference.plain]
    clipset = ctx.upload(blobs, check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in blobs]
    pairs = [(a, b) for a in range(5) for b in range(5) if counts[a] == counts[b]][:40]
    times = dbcases.ALL_TIMES
    masks = np.clip(np.arange(clipset.max_tracks, dtype=np.float32) / 8.0 - 0.5, 0.0, 1.0)[None, :]
    stacks = [[(a, float(times[i % len(times)]), BLEND, 0.0, None), (b, float(times[(i + 3) % len(times)]), BLEND, 0.375, 0),
               (a, float(times[(i + 5) % len(times)]), OFF, 0.0, None)] for i, (a, b) in enumerate(pairs)]
    done = []
    for state, ops in dbcases.STATES.items():
        for op, tier, count in ops[len(done):]:
            (database.stream_in if op == dbcases.IN else database.stream_out)(tier, count)
        done = ops
        got = _run(gpu, stacks, _options(gpu, 1), clipset=clipset, masks=masks).view(np.float32)
        for i, stack in enumerate(stacks):
            (a, ta, _, _, _), (b, tb, _, w, _), _ = stack
            n = counts[a]
            acc = reference.poses(state, a, ta, 0, ab.LOOP_AS_COMPRESSED).copy()
            layer = reference.poses(state, b, tb, 0, ab.LOOP_AS_COMPRESSED)
            for bone in range(n):
                if masks[0, bone] != 0:
                    wb = float(np.float32(w) * masks[0, bone])
                    acc[bone:bone + 1] = blend.port_qvv_lerp(acc[bone:bone + 1], layer[bone:bone + 1], wb, blend.NORMALIZE_IEEE)
            assert _rows_equal(got[i, :n * 12].reshape(n, 12), acc), (state, i)
    clipset.release()


def test_reference_composition(gpu):
    """masked_layers.golden.npz, the reference's composition of masked_layers_cases.golden_stacks(): rotations within rotation_gate bone by
    bone, translations and scales bit for bit where vectors_exact holds (within vector_gate elsewhere, where the gate is finite)."""
    golden = np.load(clips.golden_path("masked_layers", "golden.npz"))
    stacks = cases.golden_stacks()
    masks = cases.golden_masks()
    assert np.array_equal(golden["stacks"], cases.stack_array(stacks), equal_nan=True)
    blobs_clipset = gpu["ctx"].upload(cases.load_blobs())
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping)
        for si, stack in enumerate(stacks):
            padded = [stack + [(ROOT, float("nan"), OFF, 0.0, None)] * (8 - len(stack))]
            got = _run(gpu, padded, options, clipset=blobs_clipset, masks=masks,
                       d_clip_additive_formats=_dev(gpu, np.array(cases.FORMATS, np.uint8)))
            got = got.view(np.float32)[0, :24 * 12].reshape(24, 12)[:, LANES]
            want = golden["poses"][ci, si]
            gate = cases.rotation_gate(stack, masks, cases.FORMATS)
            finite = np.isfinite(gate)
            assert (np.max(np.abs(got[:, 0:4] - want[:, 0:4]), axis=1)[finite] <= gate[finite]).all(), (kind, si)
            if cases.vectors_exact(stack, cases.FORMATS):
                assert clips.bit_equal(got[:, 4:], want[:, 4:]), (kind, si)
            elif finite.all():
                assert float(np.max(np.abs(got[:, 4:] - want[:, 4:]))) <= cases.vector_gate(stack, masks, cases.FORMATS, want), (kind, si)
    blobs_clipset.release()
