"""aclb200_decompress_tracks_layered and _layered_skinning (up to eight layers per pose, folded in one kernel) against
  * the port's composition of its pinned per-operation oracles (tests/layers_cases.py): BIT FOR BIT, local, object (qvvf, matrix) and
    skinning rows;
  * the existing entry points: one layer equals decompress_tracks / _object_space / _skinning, [base, BLEND w] equals
    decompress_tracks_blend, [base, ADDITIVE] equals decompress_tracks_additive, and a four layer stack at the C2 launch size equals the
    unfused chain of decodes, blend_poses, apply_additive_to_base and local_to_skinning: byte for byte;
  * layers.golden.npz, the reference's composition: translations and scales bit for bit where no `relative` layer follows a step that
    moved the rotation, rotations within layers_cases.rotation_gate.
"""
import numpy as np
import pytest

from oracle import blend, object_space, skinning
from tests import additive_cases, clips
from tests import database_cases as dbcases
from tests import layers_cases as cases
from tests import skinning_cases

pytestmark = pytest.mark.gpu
LANES = clips.DEFINED_LANES
ROOT = 0xFFFFFFFF
SENTINEL = 0x7FC00001
OFF, BLEND, ADDITIVE = cases.OFF, cases.BLEND, cases.ADDITIVE


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
    return dict(torch=torch, ab=ab, port=port, ctx=ctx, blobs=blobs, formats=formats, clipset=ctx.upload(blobs, check_hash=True))


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
    """list of equal depth stacks -> aclb200_layer[num_poses][num_layers]"""
    a = np.array([[layer for layer in stack] for stack in stacks], np.float64)
    return gpu["ab"].make_layers(a[..., 0].astype(np.uint32), a[..., 1], a[..., 2].astype(np.uint32), a[..., 3])


def _run(gpu, stacks, options, clipset=None, width=None, skinning_call=False, **kw):
    torch, ctx = gpu["torch"], gpu["ctx"]
    clipset = clipset or gpu["clipset"]
    n, depth = len(stacks), len(stacks[0])
    d_out = torch.full((n, width or clipset.max_tracks * 12), SENTINEL, dtype=torch.int32, device="cuda")
    call = ctx.decompress_tracks_layered_skinning if skinning_call else ctx.decompress_tracks_layered
    if skinning_call:
        call(clipset, _dev(gpu, _layers(gpu, stacks)), n, depth, options, kw.pop("d_parent_indices"), kw.pop("d_inverse_bind"), d_out, **kw)
    else:
        call(clipset, _dev(gpu, _layers(gpu, stacks)), n, depth, options, d_out, **kw)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def _rows_equal(got, want, layout_40=False):
    """defined lanes bit for bit; QVV48 rows carry 0 in the translation and scale w lanes"""
    if layout_40:
        return clips.bit_equal(got, want[:, LANES])
    return clips.bit_equal(got[:, LANES], want[:, LANES]) and not got[:, [7, 11]].view(np.uint32).any()


def _counts(gpu):
    return [gpu["port"].num_tracks_of(b) for b in gpu["blobs"]]


def _expected(gpu, stack, kind, rounding=0, looping=2, settings=None, writer=None, clip_formats=True, additive_format=0):
    port = gpu["port"]
    return cases.port_local(port, blend, gpu["blobs"], stack, settings or port.settings_for_kind(kind),
                            writer or additive_cases.writer_settings(port, kind), rounding, looping, additive_format=additive_format,
                            clip_formats=gpu["formats"] if clip_formats else None)


def _random_stacks(rng, count, depth, num_clips=7, off_first=False):
    times = np.array([-0.1, 0.0, 0.13, 0.41, 0.77, 1.2, 5.0], np.float32)
    stacks = [cases.random_stack(rng, depth, num_clips, times) for _ in range(count)]
    if off_first:
        for stack in stacks[::3]:
            stack[0] = (ROOT, float("nan"), OFF, float("nan"))
    for stack in stacks[5::11]:
        stack[-1] = (40, 0.2, BLEND, 0.5)                   # an invalid clip on a layer that is not OFF
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
        n = counts[cases.base_clip(stack)]
        assert (got[i, n * bone:].view(np.int32) == SENTINEL).all(), (i, stack)
        assert _rows_equal(got[i, :n * bone].view(np.float32).reshape(n, bone), want, layout_40), (kind, r, l, i, stack)
        written += 1
    return written


@pytest.mark.parametrize("depth", [1, 2, 3, 5, 8])
def test_against_the_port(gpu, depth):
    """Every clip, every settings kind combo, both layouts, mixed ops with OFF anywhere (layer 0 included, so the base is a later
    layer), invalid clips and track count mismatches, the per clip format table: bit for bit against the port's composition."""
    ab = gpu["ab"]
    rng = np.random.default_rng(4500 + depth)
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
    # one additive format for every layer, no table
    for additive_format in (0, 1, 2, 3):
        got = _run(gpu, stacks, _options(gpu, 0), additive_format=additive_format)
        _check_local(gpu, got.view(np.float32), stacks, 0, clip_formats=False, additive_format=additive_format)


def test_per_request_policies_and_variable_defaults(gpu):
    """d_request_policies[r] applies to every layer of pose r; a variable bind pose reaches the base and the BLEND layers, while ADDITIVE
    layers keep the track_writer defaults."""
    torch, port, ab = gpu["torch"], gpu["port"], gpu["ab"]
    rng = np.random.default_rng(4510)
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
    assert _check_local(gpu, got.view(np.float32), stacks, 0, policies=policies, settings=settings) > 60


def _skeletons(gpu):
    counts = _counts(gpu)
    skeletons = [skinning_cases.skeleton(["tree", "chain", "random"][c % 3], n, seed=c) for c, n in enumerate(counts)]
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint32)
    return skeletons, offsets, np.concatenate(skeletons)


def test_object_space_and_skinning(gpu):
    """With parents the running pose walks the BASE clip's skeleton (mixed rigs through skeleton offsets): qvvf rows, 3x4 matrices and
    skinning rows against the port's walk of the port's composition; flags from the relative layers and from a parent after its child."""
    torch, ab, port = gpu["torch"], gpu["ab"], gpu["port"]
    rng = np.random.default_rng(4520)
    stacks = _random_stacks(rng, 150, 5, off_first=True)
    skeletons, offsets, parents = _skeletons(gpu)
    inverse = skinning_cases.random_affine(len(parents), 4521, mirrored=True)
    d_parents, d_offsets = _dev(gpu, parents), _dev(gpu, offsets)
    d_formats = _dev(gpu, gpu["formats"])
    counts = _counts(gpu)
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
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
            c = cases.base_clip(stack)
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
    bad = parents.copy()
    bad[offsets[2] + 3] = 9
    _run(gpu, stacks, ab.Options(), d_parent_indices=_dev(gpu, bad), kind=ab.OBJECT_MATRIX3X4F, d_skeleton_offsets=d_offsets,
         d_clip_additive_formats=d_formats, d_out_flags=d_flags)
    assert int(d_flags.item()) & ab.ERROR_FLAG_INVALID_SKELETON


def test_equivalences_with_the_existing_entry_points(gpu):
    """L = 1 is decompress_tracks (and its object space and skinning forms); [base, BLEND w] is decompress_tracks_blend; [base, ADDITIVE]
    is decompress_tracks_additive: byte for byte, the buffers filled with the same sentinel."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    clipset = gpu["clipset"]
    rng = np.random.default_rng(4530)
    m = 300
    a =rng.integers(0, 6, m).astype(np.uint32)
    b = rng.integers(0, 6, m).astype(np.uint32)
    ta = rng.uniform(-0.1, 1.4, m).astype(np.float32)
    tb = rng.uniform(-0.1, 1.4, m).astype(np.float32)
    w = rng.uniform(-0.25, 1.25, m).astype(np.float32)
    skeletons, offsets, parents = _skeletons(gpu)
    inverse = skinning_cases.random_affine(len(parents), 4531)
    d_parents, d_offsets, d_inverse = _dev(gpu, parents), _dev(gpu, offsets), _dev(gpu, inverse)
    d_formats = _dev(gpu, gpu["formats"])
    options = ab.Options()
    width = clipset.max_tracks * 12

    def fresh():
        return torch.full((m, width), SENTINEL, dtype=torch.int32, device="cuda")

    def same(x, y, what):
        torch.cuda.synchronize()
        assert torch.equal(x, y), what

    single = _dev(gpu, ab.make_layers(a[:, None], ta[:, None], BLEND, 0.0))
    requests = _dev(gpu, ab.make_requests(a, ta))
    x, y = fresh(), fresh()
    ctx.decompress_tracks(clipset, requests, m, options, x)
    ctx.decompress_tracks_layered(clipset, single, m, 1, options, y)
    same(x, y, "L = 1 local")
    for kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        x, y = fresh(), fresh()
        ctx.decompress_tracks_object_space(clipset, requests, m, options, d_parents, kind, x, d_skeleton_offsets=d_offsets)
        ctx.decompress_tracks_layered(clipset, single, m, 1, options, y, d_parent_indices=d_parents, kind=kind, d_skeleton_offsets=d_offsets)
        same(x, y, ("L = 1 object", kind))
    x, y = fresh(), fresh()
    ctx.decompress_tracks_skinning(clipset, requests, m, options, d_parents, d_inverse, x, d_skeleton_offsets=d_offsets)
    ctx.decompress_tracks_layered_skinning(clipset, single, m, 1, options, d_parents, d_inverse, y, d_skeleton_offsets=d_offsets)
    same(x, y, "L = 1 skinning")

    pairs_blend = _dev(gpu, ab.make_blend_requests(a, ta, b, tb))
    layers_blend = _dev(gpu, ab.make_layers(np.stack([a, b], 1), np.stack([ta, tb], 1), [[BLEND, BLEND]], np.stack([np.zeros(m), w], 1)))
    d_w = torch.from_numpy(w).cuda()
    for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
        x, y = fresh(), fresh()
        opts = ab.Options(output_layout=layout)
        ctx.decompress_tracks_blend(clipset, pairs_blend, m, opts, x, d_weights=d_w)
        ctx.decompress_tracks_layered(clipset, layers_blend, m, 2, opts, y)
        same(x, y, ("blend", layout))
    for kind in (ab.OBJECT_QVVF, ab.OBJECT_MATRIX3X4F):
        x, y = fresh(), fresh()
        ctx.decompress_tracks_blend(clipset, pairs_blend, m, options, x, d_weights=d_w, d_parent_indices=d_parents, kind=kind,
                                    d_skeleton_offsets=d_offsets)
        ctx.decompress_tracks_layered(clipset, layers_blend, m, 2, options, y, d_parent_indices=d_parents, kind=kind, d_skeleton_offsets=d_offsets)
        same(x, y, ("blend object", kind))
    x, y = fresh(), fresh()
    ctx.decompress_tracks_blend_skinning(clipset, pairs_blend, m, options, d_parents, d_inverse, x, d_weights=d_w, d_skeleton_offsets=d_offsets)
    ctx.decompress_tracks_layered_skinning(clipset, layers_blend, m, 2, options, d_parents, d_inverse, y, d_skeleton_offsets=d_offsets)
    same(x, y, "blend skinning")

    c = rng.choice([3, 4, 5], m).astype(np.uint32)
    pairs_add = _dev(gpu, ab.make_additive_requests(a, ta, c, tb))
    layers_add = _dev(gpu, ab.make_layers(np.stack([a, c], 1), np.stack([ta, tb], 1), [[ADDITIVE, ADDITIVE]], 0.0))
    d_flags_x = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_flags_y = torch.ones(1, dtype=torch.int32, device="cuda")
    for kw in (dict(d_clip_additive_formats=d_formats), dict(additive_format=ab.ADDITIVE_RELATIVE)):
        for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
            x, y = fresh(), fresh()
            opts = ab.Options(output_layout=layout)
            ctx.decompress_tracks_additive(clipset, pairs_add, m, opts, x, d_out_flags=d_flags_x, **kw)
            ctx.decompress_tracks_layered(clipset, layers_add, m, 2, opts, y, d_out_flags=d_flags_y, **kw)
            same(x, y, ("additive", layout, list(kw)))
            assert int(d_flags_x.item()) == int(d_flags_y.item())
        x, y = fresh(), fresh()
        ctx.decompress_tracks_additive(clipset, pairs_add, m, options, x, d_parent_indices=d_parents, kind=ab.OBJECT_QVVF,
                                       d_skeleton_offsets=d_offsets, **kw)
        ctx.decompress_tracks_layered(clipset, layers_add, m, 2, options, y, d_parent_indices=d_parents, kind=ab.OBJECT_QVVF,
                                      d_skeleton_offsets=d_offsets, **kw)
        same(x, y, ("additive object", list(kw)))
        x, y = fresh(), fresh()
        ctx.decompress_tracks_additive_skinning(clipset, pairs_add, m, options, d_parents, d_inverse, x, d_skeleton_offsets=d_offsets, **kw)
        ctx.decompress_tracks_layered_skinning(clipset, layers_add, m, 2, options, d_parents, d_inverse, y, d_skeleton_offsets=d_offsets, **kw)
        same(x, y, ("additive skinning", list(kw)))


def test_c2_stack_equals_the_unfused_chain(gpu):
    """300,000 four layer stacks over the C2 bench clips (base, BLEND, BLEND, ADDITIVE additive0): the fused call writes byte for byte what
    decompress_tracks (base and blend layers) + decompress_tracks_additive with format none (the additive layer's writer-default pose) +
    2 x blend_poses + apply_additive_to_base write, and the skinning call what local_to_skinning then writes; checked pose by pose on the
    device."""
    import bench
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    w = bench.make_workload("c2", 0, None)
    clipset = ctx.upload_packed(w["buffer"], w["offsets"], w["sizes"])
    m, bones = 300000, w["num_tracks"]
    rng = np.random.default_rng(4540)
    clip = [w["req_clip"][:m]] + [rng.permutation(w["req_clip"])[:m] for _ in range(3)]
    time = [w["req_time"][:m]] + [rng.permutation(w["req_time"])[:m] for _ in range(3)]
    weight = [np.zeros(m, np.float32), rng.uniform(0, 1, m).astype(np.float32), rng.uniform(-0.25, 1.25, m).astype(np.float32)]
    options = ab.Options()
    poses = [torch.empty((m, bones, 12), dtype=torch.float32, device="cuda") for _ in range(4)]
    for k in range(3):
        ctx.decompress_tracks(clipset, _dev(gpu, ab.make_requests(clip[k], time[k])), m, options, poses[k])
    ctx.decompress_tracks_additive(clipset, _dev(gpu, ab.make_additive_requests(clip[0], time[0], clip[3], time[3])), m, options, poses[3],
                                   additive_format=ab.ADDITIVE_NONE)
    chain = poses[0]
    ctx.blend_poses(chain, poses[1], chain, m, bones, d_weights=torch.from_numpy(weight[1]).cuda())
    ctx.blend_poses(chain, poses[2], chain, m, bones, d_weights=torch.from_numpy(weight[2]).cuda())
    ctx.apply_additive_to_base(chain, poses[3], chain, m, bones, ab.ADDITIVE_ADDITIVE0)
    ops = np.array([[BLEND, BLEND, BLEND, ADDITIVE]], np.uint32)
    layers = _dev(gpu, ab.make_layers(np.stack(clip, 1), np.stack(time, 1), ops, np.stack(weight + [np.zeros(m, np.float32)], 1)))
    fused = torch.full_like(chain, float("nan"))
    ctx.decompress_tracks_layered(clipset, layers, m, 4, options, fused, additive_format=ab.ADDITIVE_ADDITIVE0)
    torch.cuda.synchronize()
    assert torch.equal(fused.view(torch.int32), chain.view(torch.int32))
    parents = np.where(np.arange(bones) == 0, ROOT, (np.arange(bones) - 1) // 2).astype(np.uint32)
    inverse = torch.from_numpy(skinning_cases.random_affine(bones, 4541)).cuda()
    d_parents = _dev(gpu, parents)
    ctx.local_to_skinning(chain, chain, m, bones, d_parents, inverse)
    fused.fill_(float("nan"))
    ctx.decompress_tracks_layered_skinning(clipset, layers, m, 4, options, d_parents, inverse, fused, additive_format=ab.ADDITIVE_ADDITIVE0)
    torch.cuda.synchronize()
    assert torch.equal(fused.view(torch.int32), chain.view(torch.int32))
    clipset.release()


def test_off_layers_change_nothing(gpu):
    """OFF layers with invalid clip indices and NaN times inserted anywhere (first, middle, last) leave every output byte unchanged."""
    ab = gpu["ab"]
    rng = np.random.default_rng(4550)
    stacks = [cases.random_stack(rng, 3, 6, np.array([0.0, 0.3, 0.9], np.float32), allow_off=False) for _ in range(200)]
    d_formats = _dev(gpu, gpu["formats"])
    want = _run(gpu, stacks, ab.Options(), d_clip_additive_formats=d_formats)
    off = (0xFFFFFFF0, float("nan"), OFF, float("nan"))
    for where in ([0], [1], [3], [0, 2, 5]):
        padded = []
        for stack in stacks:
            s = list(stack)
            for position in where:
                s.insert(position, off)
            padded.append(s)
        got = _run(gpu, padded, ab.Options(), d_clip_additive_formats=d_formats)
        assert np.array_equal(got, want), where


def test_poses_that_write_nothing_and_refusals(gpu):
    """Invalid clips, track count mismatches, unknown ops and all-OFF stacks write nothing (bytes past num_tracks included); every refusal
    writes nothing and leaves the flags untouched."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    good = [(0, 0.3, BLEND, 0.0), (1, 0.2, BLEND, 0.5), (4, 0.1, ADDITIVE, 0.0)]
    stacks = [
        good,
        [(0, 0.3, BLEND, 0.0), (9, 0.2, BLEND, 0.5), (4, 0.1, ADDITIVE, 0.0)],         # invalid clip
        [(0, 0.3, BLEND, 0.0), (6, 0.2, BLEND, 0.5), (4, 0.1, ADDITIVE, 0.0)],         # 30 bones under a 24 bone base
        [(0, 0.3, BLEND, 0.0), (1, 0.2, 3, 0.5), (4, 0.1, ADDITIVE, 0.0)],             # unknown op
        [(0, 0.3, 7, 0.0), (1, 0.2, BLEND, 0.5), (4, 0.1, ADDITIVE, 0.0)],             # unknown op on the first layer
        [(0, 0.3, OFF, 0.0), (1, 0.2, OFF, 0.5), (4, 0.1, OFF, 0.0)],                  # all OFF
        [(6, 0.3, OFF, 0.0), (6, 0.2, ADDITIVE, 0.5), (6, 0.1, BLEND, 0.0)],           # a 30 bone stack whose base is layer 1
    ]
    got = _run(gpu, stacks, ab.Options())
    assert not (got[0].view(np.int32) == SENTINEL).all() and not (got[6].view(np.int32) == SENTINEL).all()
    assert (got[0, 24 * 12:] == SENTINEL).all()
    for i in range(1, 6):
        assert (got[i] == SENTINEL).all(), i
    _check_local(gpu, got.view(np.float32), stacks, 0, clip_formats=False)

    layers = _dev(gpu, _layers(gpu, [good] * 8))
    parents = _dev(gpu, np.where(np.arange(30) == 0, ROOT, np.arange(30) - 1).astype(np.uint32))
    inverse = torch.zeros((30, 12), dtype=torch.float32, device="cuda")
    scalar = ctx.upload([clips.load_blob("float1")])
    skip_tracks = torch.zeros(30, dtype=torch.uint8, device="cuda")
    refusals = [
        dict(num_layers=0), dict(num_layers=9), dict(num_poses=0x20000000, num_layers=8),
        dict(options=ab.Options(skip_mask=ab.SKIP_SCALE)),
        dict(options=ab.Options(d_skip_track_mask=skip_tracks.data_ptr())),
        dict(options=ab.Options(default_modes=(ab.DEFAULT_CONSTANT, ab.DEFAULT_SKIPPED, ab.DEFAULT_LEGACY))),
        dict(additive_format=4), dict(clipset=scalar),
        dict(parents=parents, kind=2),
        dict(parents=parents, options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(offset=8), dict(offset=4, options=ab.Options(output_layout=ab.LAYOUT_QVV40)),
        dict(options=ab.Options(pose_stride_bytes=30 * 48 + 8)),
        dict(skin=True), dict(skin=True, parents=parents), dict(skin=True, parents=parents, inverse=inverse.data_ptr() + 4),
        dict(skin=True, parents=parents, inverse=inverse, num_layers=0),
    ]
    for case in refusals:
        buffer = torch.full((8 * 30 * 48 + 128,), 0x5A, dtype=torch.uint8, device="cuda")
        d_flags = torch.full((1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        args = (case.get("clipset", gpu["clipset"]), layers, case.get("num_poses", 8), case.get("num_layers", 3), case.get("options", ab.Options()))
        out = buffer.data_ptr() + case.get("offset", 0)
        with pytest.raises(ab.api.AclB200Error) as error:
            if case.get("skin"):
                ctx.decompress_tracks_layered_skinning(*args, case.get("parents"), case.get("inverse"), out, d_out_flags=d_flags)
            else:
                ctx.decompress_tracks_layered(*args, out, additive_format=case.get("additive_format", 0), d_parent_indices=case.get("parents"),
                                              kind=case.get("kind", 0), d_out_flags=d_flags)
        assert error.value.status == 1, case             # ACLB200_ERR_INVALID_ARGUMENT
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == 0x5A).all(), case
        assert int(d_flags.item()) == 0x5A5A5A5A, case
    scalar.release()


def test_wide_pose_limits(gpu):
    """wide_2500 (2500 bones) follows the pair limits: one QVV48 pose (120,000 bytes) fits one block and two do not; in QVV40 two poses
    (2 x 100,000 bytes) just fit and three just fail. A refusal is ACLB200_ERR_UNSUPPORTED and writes nothing."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blob = clips.load_blob("wide_2500")
    clipset = ctx.upload([blob])
    times = [0.05, 0.1333, 0.27]
    weights = [0.0, 0.3, 0.8]
    port = gpu["port"]
    settings, writer = port.settings_for_kind(0), additive_cases.writer_settings(port, 0)
    for layout, fits, fails in ((ab.LAYOUT_QVV48, 1, 2), (ab.LAYOUT_QVV40, 2, 3)):
        bone = 12 if layout == ab.LAYOUT_QVV48 else 10
        options = ab.Options(output_layout=layout, pose_stride_bytes=2500 * 48)
        stacks = [[(0, times[(i + k) % 3], BLEND, weights[k]) for k in range(fails)] for i in range(3)]
        buffer = torch.full((3, 2500 * 12), SENTINEL, dtype=torch.int32, device="cuda")
        with pytest.raises(ab.api.AclB200Error) as error:
            ctx.decompress_tracks_layered(clipset, _dev(gpu, _layers(gpu, stacks)), 3, fails, options, buffer)
        assert error.value.status == 3                   # ACLB200_ERR_UNSUPPORTED
        torch.cuda.synchronize()
        assert (buffer.cpu().numpy() == SENTINEL).all()
        stacks = [stack[:fits] for stack in stacks]
        got = _run(gpu, stacks, options, clipset=clipset, width=2500 * 12).view(np.float32)
        for i, stack in enumerate(stacks):
            want = cases.port_local(port, blend, [blob], stack, settings, writer, 0, ab.LOOP_AS_COMPRESSED)
            assert _rows_equal(got[i, :2500 * bone].reshape(2500, bone), want, layout == ab.LAYOUT_QVV40), (layout, i)
    clipset.release()


def test_database_tiers(gpu):
    """A clip set bound to a database, in every tier state of tests/database_cases.py: three layer stacks of equal track count clips
    (base, BLEND, ADDITIVE none) decode every layer from what is streamed in, against the reference's poses of those states."""
    from tests.test_gpu_database import _Reference
    from oracle import ref, ref_database
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    reference = _Reference(ref, ref_database)
    blobs = reference.bound + [reference.plain]
    clipset = ctx.upload(blobs, check_hash=True)
    database = ctx.upload_database(reference.database, check_hash=True)
    clipset.bind_database(database)
    counts = [int(ref.num_tracks_of(b)) for b in blobs]
    triples = [(a, b, c) for a in range(5) for b in range(5) for c in range(5) if counts[a] == counts[b] == counts[c]][:40]
    times = dbcases.ALL_TIMES
    stacks = [[(a, float(times[i % len(times)]), BLEND, 0.0), (b, float(times[(i + 3) % len(times)]), BLEND, 0.375),
               (c, float(times[(i + 5) % len(times)]), OFF, 0.0)] for i, (a, b, c) in enumerate(triples)]
    done = []
    for state, ops in dbcases.STATES.items():
        for op, tier, count in ops[len(done):]:
            (database.stream_in if op == dbcases.IN else database.stream_out)(tier, count)
        done = ops
        got = _run(gpu, stacks, _options(gpu, 1), clipset=clipset).view(np.float32)
        for i, stack in enumerate(stacks):
            (a, ta, _, _), (b, tb, _, w), _ = stack
            n = counts[a]
            want = blend.port_qvv_lerp(reference.poses(state, a, ta, 0, ab.LOOP_AS_COMPRESSED),
                                       reference.poses(state, b, tb, 0, ab.LOOP_AS_COMPRESSED), w, blend.NORMALIZE_IEEE)
            assert _rows_equal(got[i, :n * 12].reshape(n, 12), want), (state, i)
    clipset.release()


def test_reference_composition(gpu):
    """layers.golden.npz, the reference's composition of layers_cases.golden_stacks(): translations and scales bit for bit where
    layers_cases.vectors_exact holds (within vector_gate elsewhere), rotations within layers_cases.rotation_gate."""
    golden = np.load(clips.golden_path("layers", "golden.npz"))
    stacks = cases.golden_stacks()
    assert np.array_equal(golden["stacks"], cases.stack_array(stacks), equal_nan=True)
    ab = gpu["ab"]
    blobs_clipset = gpu["ctx"].upload(cases.load_blobs())
    for ci, (kind, rounding, looping) in enumerate(cases.COMBOS):
        options = _options(gpu, kind, rounding_policy=rounding, looping_policy=looping)
        for si, stack in enumerate(stacks):
            padded = [stack + [(ROOT, float("nan"), OFF, 0.0)] * (8 - len(stack))]
            got = _run(gpu, padded, options, clipset=blobs_clipset, d_clip_additive_formats=_dev(gpu, np.array(cases.FORMATS, np.uint8)))
            got = got.view(np.float32)[0, :24 * 12].reshape(24, 12)[:, LANES]
            want = golden["poses"][ci, si]
            gate = cases.rotation_gate(stack, cases.FORMATS)
            assert float(np.max(np.abs(got[:, 0:4] - want[:, 0:4]))) <= gate, (kind, si)
            if cases.vectors_exact(stack, cases.FORMATS):
                assert clips.bit_equal(got[:, 4:], want[:, 4:]), (kind, si)
            else:
                assert float(np.max(np.abs(got[:, 4:] - want[:, 4:]))) <= cases.vector_gate(stack, cases.FORMATS, want), (kind, si)
    blobs_clipset.release()
    assert ab.MAX_LAYERS == 8
