"""GPU parity of SURVEY 8(f1) / 8(f3): aclb200_calculate_compression_error and aclb200_local_to_object_space (acl_b200/csrc/error_metric.cu)
through the C ABI, against

  * the oracle's restatement with IEEE normalisation (oracle/acl_oracle.c, pinned to the reference by tests/test_error_metric_oracle.py):
    BIT FOR BIT -- every per bone error, the worst track, its error and its sample time, object space poses;
  * the unmodified reference's calculate_compression_error (oracle/_ref/libaclref.so): within ERROR_TOLERANCE (rtm::quat_normalize starts
    from the CPU's rsqrtss estimate, external/rtm/includes/rtm/quatf.h:917-953: no two CPU models agree bit for bit either);
    scalar clips have no such step and match the reference exactly;
  * the committed golden numbers (tests/golden/*.error.npz) when the compiled reference is absent.
"""
import numpy as np
import pytest

from tests import clips
from tests.test_error_metric_oracle import (ADDITIVE_CASES, ERROR_TOLERANCE, GOLDEN_SCALAR, GOLDEN_TRANSFORM, MIRRORED_CASES, additive_base_spec,
                                            error_tolerance, kinds_for, mirrored_spec)

pytestmark = pytest.mark.gpu

LANES = clips.DEFINED_LANES
IDENTITY = [0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0]


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    return dict(torch=torch, ab=ab, port=port, ctx=ab.Context(0))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array)).cuda()


def _options(gpu, kind):
    """The context calculate_compression_error is handed + the bind pose its debug_track_writer starts from (identity)."""
    ab, port = gpu["ab"], gpu["port"]
    s = port.settings_for_kind(kind).c
    return ab.Options(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                      clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                      default_modes=(ab.DEFAULT_CONSTANT,) * 3, constant_defaults=IDENTITY)


def _jobs(gpu, rows):
    jobs = np.zeros(len(rows), dtype=gpu["ab"].ERROR_JOB_DTYPE)
    for i, row in enumerate(rows):
        for key, value in row.items():
            jobs[i][key] = value
    return jobs


def _measure(gpu, clipset, jobs, raw_poses, parents, shells, options, output_indices=None, base_poses=None):
    """Runs the call and returns (track errors structured array, error matrix [total poses][max_tracks])."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    total = int(jobs["num_samples"].sum())
    d_errors = torch.zeros(len(jobs) * 4, dtype=torch.int32, device="cuda")
    d_matrix = torch.full((max(total, 1), clipset.max_tracks), float("nan"), dtype=torch.float32, device="cuda")
    ctx.calculate_compression_error(clipset, jobs, _dev(gpu, raw_poses), None if parents is None else _dev(gpu, parents),
                                    None if shells is None else _dev(gpu, shells), options, d_errors,
                                    d_output_indices=None if output_indices is None else _dev(gpu, output_indices), d_out_error_matrix=d_matrix,
                                    d_base_poses=None if base_poses is None else _dev(gpu, base_poses))
    torch.cuda.synchronize()
    return d_errors.cpu().numpy().view(ab.TRACK_ERROR_DTYPE), d_matrix.cpu().numpy()


def _check_against(gpu, got, matrix_rows, raw, lossy, sample_rate, duration, parents, shells, reference_numbers, label):
    """got: one TRACK_ERROR record; matrix_rows: [num_samples][num_tracks] of the GPU; reference_numbers: dict(errors, index, error, sample_time)."""
    port = gpu["port"]
    want, want_errors, negative = port.transform_track_error(raw, lossy, sample_rate, duration, parents, shells, port.NORMALIZE_IEEE)
    assert not negative and got["flags"] == 0, label
    assert clips.bit_equal(matrix_rows, want_errors), label
    assert (int(got["index"]), np.float32(got["error"]), np.float32(got["sample_time"])) == (want.index, np.float32(want.error), np.float32(want.sample_time)), label
    if reference_numbers is not None:
        r = reference_numbers
        if r["errors"].size:
            assert float(np.max(np.abs(matrix_rows - r["errors"]))) <= ERROR_TOLERANCE, label
        assert abs(float(got["error"]) - float(r["error"])) <= ERROR_TOLERANCE, label
        if int(got["index"]) != 0xFFFFFFFF:
            sample = int(round(float(got["sample_time"]) * sample_rate))
            assert r["errors"][sample, int(got["index"])] >= float(r["error"]) - 2 * ERROR_TOLERANCE, label


def _reference_case(name, kind):
    """Inputs + the reference's numbers: live when oracle/_ref is built, else the committed golden file (debug settings only)."""
    from oracle import ref
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    if ref.available():
        return ref.transform_error(spec, blob, kind)
    if kind != 1 or name not in GOLDEN_TRANSFORM:
        pytest.skip("needs oracle/_ref/libaclref.so")
    g = np.load(clips.golden_path(name, "error.npz"))
    from tests.test_error_metric_oracle import lossy_poses_from_port
    out = {k: g[k] for k in ("raw_poses", "errors", "parents", "shell_distances")}
    out.update(index=int(g["index"]), error=float(g["error"]), sample_time=float(g["sample_time"]), rounding=int(g["rounding"]),
               sample_rate=float(g["sample_rate"]), duration=float(g["duration"]))
    out["lossy_poses"] = lossy_poses_from_port(blob, 1, g["raw_poses"].shape[0], out["sample_rate"], out["duration"], out["rounding"])
    return out


@pytest.mark.parametrize("name", list(clips.TRANSFORM_SPECS))
def test_compression_error_one_clip(gpu, name):
    spec = clips.TRANSFORM_SPECS[name]
    blob = clips.load_blob(name)
    clipset = gpu["ctx"].upload([blob], check_hash=True)
    for kind in kinds_for(spec):
        r = _reference_case(name, kind)
        jobs = _jobs(gpu, [dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"],
                                num_tracks=spec.num_tracks, skeleton_offset=0, first_raw_pose=0)])
        got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, kind))
        _check_against(gpu, got[0], matrix[:spec.num_samples, :spec.num_tracks], r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"],
                       r["parents"], r["shell_distances"], r, (name, kind))
    clipset.release()


def test_compression_error_many_clips_ragged_chunked(gpu):
    """Clips of different widths, stripped (sought with `none`) and not (`nearest`), jobs out of order, one clip measured twice, raw poses
    and skeletons at arbitrary offsets, and a chunk budget small enough to cut the job list into several launches."""
    ab, ctx = gpu["ab"], gpu["ctx"]
    names = ["mixed_scale", "stripped_single", "c1_30bones", "stripped_loop", "ragged_17", "one_bone", "two_samples", "c2_100bones", "one_sample"]
    blobs = [clips.load_blob(n) for n in names]
    clipset = ctx.upload(blobs, check_hash=True)
    max_tracks = clipset.max_tracks
    cases = [_reference_case(n, 1) for n in names]

    order = [3, 0, 7, 1, 5, 0, 8, 2, 6, 4]
    raw_rows, parents, shells, rows = [np.zeros((3, max_tracks, 12), np.float32)], [np.zeros(5, np.uint32)], [np.zeros(5, np.float32)], []
    skeleton_offset, pose_offset = 5, 3
    for clip in order:
        r, spec = cases[clip], clips.TRANSFORM_SPECS[names[clip]]
        padded = np.zeros((spec.num_samples, max_tracks, 12), np.float32)
        padded[:, :spec.num_tracks] = r["raw_poses"]
        raw_rows.append(padded)
        parents.append(r["parents"])
        shells.append(r["shell_distances"])
        rows.append(dict(clip=clip, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"],
                         num_tracks=spec.num_tracks, skeleton_offset=skeleton_offset, first_raw_pose=pose_offset))
        skeleton_offset += spec.num_tracks
        pose_offset += spec.num_samples
    jobs = _jobs(gpu, rows)
    raw = np.concatenate(raw_rows)
    for chunk_bytes in (1024 << 20, 100 * max_tracks * 48):
        ctx.set_error_chunk_bytes(chunk_bytes)
        got, matrix = _measure(gpu, clipset, jobs, raw, np.concatenate(parents), np.concatenate(shells), _options(gpu, 1))
        row = 0
        for slot, clip in enumerate(order):
            r, spec = cases[clip], clips.TRANSFORM_SPECS[names[clip]]
            _check_against(gpu, got[slot], matrix[row:row + spec.num_samples, :spec.num_tracks], r["raw_poses"], r["lossy_poses"], r["sample_rate"],
                           r["duration"], r["parents"], r["shell_distances"], r, (names[clip], slot, chunk_bytes))
            row += spec.num_samples
    ctx.set_error_chunk_bytes(1024 << 20)
    clipset.release()


def test_compression_error_fast_math_within_gate(gpu):
    """ACLB200_MATH_FAST decode (rotations <= 1e-5 from exact) moves the measured error by no more than the metric's own tolerance."""
    ab = gpu["ab"]
    name = "c2_100bones"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    r = _reference_case(name, 1)
    jobs = _jobs(gpu, [dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks)])
    options = _options(gpu, 1)
    options.math_mode = ab.MATH_FAST
    got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], options)
    assert float(np.max(np.abs(matrix[:spec.num_samples, :spec.num_tracks] - r["errors"]))) <= 1e-3
    assert abs(float(got[0]["error"]) - r["error"]) <= 1e-3
    clipset.release()


@pytest.mark.parametrize("name,additive_format,base_samples", ADDITIVE_CASES)
def test_compression_error_with_additive_base(gpu, name, additive_format, base_samples):
    """The additive base overload (track_error.impl.h:573-680) + additive_qvvf_transform_error_metric<format>: bit for bit against the
    oracle, within the (pose size scaled) tolerance of the live reference; measured next to a plain job of the same clip in one call."""
    from oracle import ref
    if not ref.available():
        pytest.skip("needs oracle/_ref/libaclref.so")
    port = gpu["port"]
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    r = ref.transform_error_additive(spec, clips.load_blob(name), additive_base_spec(spec, base_samples), additive_format)
    plain = _reference_case(name, 1)
    common = dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks)
    # base poses behind 2 unrelated rows; the plain job carries no additive format and must ignore them
    base = np.concatenate([np.full((2, spec.num_tracks, 12), 7.0, np.float32), r["base_poses"]])
    jobs = _jobs(gpu, [dict(common, additive_format=additive_format, first_base_pose=2), dict(common)])
    got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, 1), base_poses=base)
    want, want_errors, negative = port.transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                             r["shell_distances"], port.NORMALIZE_IEEE, r["base_poses"], additive_format)
    assert not negative and got[0]["flags"] == 0
    assert clips.bit_equal(matrix[:spec.num_samples, :spec.num_tracks], want_errors)
    assert (int(got[0]["index"]), np.float32(got[0]["error"]), np.float32(got[0]["sample_time"])) == (want.index, np.float32(want.error), np.float32(want.sample_time))
    applied = np.stack([port.apply_additive_to_base(additive_format, r["base_poses"][s], r["raw_poses"][s]) for s in range(spec.num_samples)])
    tolerance = error_tolerance(port, applied, r["parents"])
    assert float(np.max(np.abs(matrix[:spec.num_samples, :spec.num_tracks] - r["errors"]))) <= tolerance
    assert abs(float(got[0]["error"]) - r["error"]) <= tolerance
    _check_against(gpu, got[1], matrix[spec.num_samples:2 * spec.num_samples, :spec.num_tracks], plain["raw_poses"], plain["lossy_poses"], plain["sample_rate"],
                   plain["duration"], plain["parents"], plain["shell_distances"], plain, (name, "plain job next to the additive one"))
    clipset.release()


@pytest.mark.parametrize("name,negative_scale_pct", MIRRORED_CASES)
def test_compression_error_with_negative_scales(gpu, name, negative_scale_pct):
    """Mirrored bones: rtm::qvv_mul's matrix branch (matrix_from_qvv, matrix_mul, matrix_remove_scale, quat_from_matrix) on the device,
    per stream, bit for bit against the oracle; also under the relative additive format, and through aclb200_local_to_object_space."""
    from oracle import ref
    if not ref.available():
        pytest.skip("needs oracle/_ref/libaclref.so")
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    spec = mirrored_spec(name, negative_scale_pct)
    blob = ref.compress_transform(spec)
    clipset = ctx.upload([blob], check_hash=True)
    r = ref.transform_error(spec, blob, 1)
    ra = ref.transform_error_additive(spec, blob, additive_base_spec(spec, 17), 1)
    common = dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks)
    jobs = _jobs(gpu, [dict(common), dict(common, additive_format=1)])
    got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, 1), base_poses=ra["base_poses"])
    for slot, (case, base, fmt) in enumerate(((r, None, 0), (ra, ra["base_poses"], 1))):
        want, want_errors, negative = port.transform_track_error(case["raw_poses"], case["lossy_poses"], case["sample_rate"], case["duration"], case["parents"],
                                                                 case["shell_distances"], port.NORMALIZE_IEEE, base, fmt)
        rows = matrix[slot * spec.num_samples:(slot + 1) * spec.num_samples, :spec.num_tracks]
        assert negative and int(got[slot]["flags"]) == ab.ERROR_FLAG_NEGATIVE_SCALE
        assert clips.bit_equal(rows, want_errors), (name, slot)
        assert (int(got[slot]["index"]), np.float32(got[slot]["error"]), np.float32(got[slot]["sample_time"])) == (want.index, np.float32(want.error), np.float32(want.sample_time))
        applied = case["raw_poses"] if base is None else np.stack([port.apply_additive_to_base(fmt, base[s], case["raw_poses"][s]) for s in range(spec.num_samples)])
        assert float(np.max(np.abs(rows - case["errors"]))) <= error_tolerance(port, applied, case["parents"]), (name, slot)

    d_local = _dev(gpu, r["lossy_poses"])
    d_object = torch.empty_like(d_local)
    ctx.local_to_object_space(d_local, d_object, spec.num_samples, spec.num_tracks, _dev(gpu, r["parents"]))
    torch.cuda.synchronize()
    got_object = d_object.cpu().numpy()
    for sample in range(0, spec.num_samples, 5):
        assert clips.bit_equal(got_object[sample][:, LANES], port.local_to_object_space(r["lossy_poses"][sample], r["parents"], port.NORMALIZE_IEEE)[:, LANES])
    clipset.release()


@pytest.mark.parametrize("name", ["c1_30bones", "c2_100bones", "mixed_scale", "stripped_single", "paragon_like", "ragged_17", "one_bone", "mirrored",
                                  "single_segment", "two_samples"])
def test_matrix_metric_matches_the_reference_exactly(gpu, name):
    """ACLB200_METRIC_QVVF_MATRIX3X4F == qvvf_matrix3x4f_transform_error_metric: no CPU specific step, so the device must give the
    reference's numbers bit for bit (every per bone error, the worst track, its error and sample time); measured next to a job of the
    same clip with the default metric in one call. Without the compiled reference its committed numbers stand in
    (tests/golden/*.matrix_error.npz, machine independent: the metric has no CPU specific step)."""
    from oracle import ref
    ab = gpu["ab"]
    spec = mirrored_spec("mixed_scale", 30) if name == "mirrored" else clips.TRANSFORM_SPECS[name]
    if ref.available():
        blob = ref.compress_transform(spec) if name == "mirrored" else clips.load_blob(name)
        r = ref.transform_error(spec, blob, 1)
        m = ref.transform_error_matrix(spec, blob)
    elif name in GOLDEN_TRANSFORM:
        blob = clips.load_blob(name)
        r = _reference_case(name, 1)
        g = np.load(clips.golden_path(name, "matrix_error.npz"))
        m = dict(errors=g["errors"], index=int(g["index"]), error=float(g["error"]), sample_time=float(g["sample_time"]))
    else:
        pytest.skip("needs oracle/_ref/libaclref.so")
    clipset = gpu["ctx"].upload([blob])
    common = dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks)
    jobs = _jobs(gpu, [dict(common), dict(common, error_metric=ab.api.METRIC_QVVF_MATRIX3X4F)])
    got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, 1))
    rows = matrix[spec.num_samples:2 * spec.num_samples, :spec.num_tracks]
    assert clips.bit_equal(rows, m["errors"]), name
    assert (int(got[1]["index"]), np.float32(got[1]["error"]), np.float32(got[1]["sample_time"]), int(got[1]["flags"])) == \
        (m["index"], np.float32(m["error"]), np.float32(m["sample_time"]), 0), name
    want, want_errors, _ = gpu["port"].transform_track_error(r["raw_poses"], r["lossy_poses"], r["sample_rate"], r["duration"], r["parents"],
                                                             r["shell_distances"], gpu["port"].NORMALIZE_IEEE)
    assert clips.bit_equal(matrix[:spec.num_samples, :spec.num_tracks], want_errors), (name, "default metric job next to it")
    # the reference does not implement an additive base for this metric: refused, not guessed
    with pytest.raises(ab.AclB200Error):
        _measure(gpu, clipset, _jobs(gpu, [dict(common, error_metric=1, additive_format=2)]), r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, 1),
                 base_poses=r["raw_poses"])
    clipset.release()


def test_output_indices_remap(gpu):
    """remap_output (track_error.impl.h:522-532): a raw track the compressed clip does not output is measured with its raw value."""
    port = gpu["port"]
    name = "c1_30bones"
    spec = clips.TRANSFORM_SPECS[name]
    clipset = gpu["ctx"].upload([clips.load_blob(name)])
    r = _reference_case(name, 1)
    output_indices = np.arange(spec.num_tracks, dtype=np.uint32)
    dropped = [4, 17]
    output_indices[dropped] = 0xFFFFFFFF
    lossy = r["lossy_poses"].copy()
    lossy[:, dropped] = r["raw_poses"][:, dropped]
    jobs = _jobs(gpu, [dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks)])
    got, matrix = _measure(gpu, clipset, jobs, r["raw_poses"], r["parents"], r["shell_distances"], _options(gpu, 1), output_indices=output_indices)
    _check_against(gpu, got[0], matrix[:spec.num_samples, :spec.num_tracks], r["raw_poses"], lossy, r["sample_rate"], r["duration"], r["parents"],
                   r["shell_distances"], None, name)
    clipset.release()


@pytest.mark.parametrize("name", ["c2_100bones", "paragon_like", "mixed_scale", "one_bone"])
def test_local_to_object_space(gpu, name):
    torch, ctx, port = gpu["torch"], gpu["ctx"], gpu["port"]
    spec = clips.TRANSFORM_SPECS[name]
    r = _reference_case(name, 1)
    poses = r["lossy_poses"]
    d_local = _dev(gpu, poses)
    d_object = torch.full_like(d_local, float("nan"))
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.local_to_object_space(d_local, d_object, poses.shape[0], spec.num_tracks, _dev(gpu, r["parents"]), d_out_flags=d_flags)
    ctx.local_to_object_space(d_local, d_local, poses.shape[0], spec.num_tracks, _dev(gpu, r["parents"]))      # in place
    torch.cuda.synchronize()
    got, in_place = d_object.cpu().numpy(), d_local.cpu().numpy()
    assert int(d_flags.item()) == 0
    for sample in range(poses.shape[0]):
        want = port.local_to_object_space(poses[sample], r["parents"], port.NORMALIZE_IEEE)
        assert clips.bit_equal(got[sample][:, LANES], want[:, LANES]), (name, sample)
        assert clips.bit_equal(in_place[sample][:, LANES], want[:, LANES]), (name, sample)
    if "object_poses" in r:        # live reference: its own object space poses, within the normalisation tolerance
        assert float(np.max(np.abs(got[..., LANES] - r["object_poses"][1][..., LANES]))) <= ERROR_TOLERANCE
    # a chain: every bone the child of the previous one (32 wavefronts per chunk of bones)
    chain = np.concatenate([[0xFFFFFFFF], np.arange(spec.num_tracks - 1)]).astype(np.uint32)
    d_local = _dev(gpu, poses)
    ctx.local_to_object_space(d_local, d_object, poses.shape[0], spec.num_tracks, _dev(gpu, chain))
    torch.cuda.synchronize()
    got = d_object.cpu().numpy()
    for sample in (0, poses.shape[0] - 1):
        assert clips.bit_equal(got[sample][:, LANES], port.local_to_object_space(poses[sample], chain, port.NORMALIZE_IEEE)[:, LANES]), (name, "chain")


def test_flags_invalid_skeleton_and_negative_scale(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    rng = np.random.default_rng(3)
    poses = np.tile(np.array(IDENTITY, dtype=np.float32), (4, 40, 1))
    poses[..., 4:7] = rng.uniform(-1, 1, size=(4, 40, 3)).astype(np.float32)
    parents = np.concatenate([[0xFFFFFFFF], (np.arange(1, 40) - 1) // 2]).astype(np.uint32)
    d_object = torch.zeros((4, 40, 12), dtype=torch.float32, device="cuda")
    d_flags = torch.zeros(1, dtype=torch.int32, device="cuda")

    bad_parents = parents.copy()
    bad_parents[7] = 9          # a parent after its child
    ctx.local_to_object_space(_dev(gpu, poses), d_object, 4, 40, _dev(gpu, bad_parents), d_out_flags=d_flags)
    torch.cuda.synchronize()
    assert int(d_flags.item()) == ab.ERROR_FLAG_INVALID_SKELETON

    mirrored = poses.copy()
    mirrored[2, 5, 8] = -1.0     # rtm::qvv_mul takes its matrix branch for this bone's children
    ctx.local_to_object_space(_dev(gpu, mirrored), d_object, 4, 40, _dev(gpu, parents), d_out_flags=d_flags)
    torch.cuda.synchronize()
    assert int(d_flags.item()) == ab.ERROR_FLAG_NEGATIVE_SCALE        # informational: the matrix branch ran
    got = d_object.cpu().numpy()
    for sample in range(4):
        assert clips.bit_equal(got[sample][:, LANES], gpu["port"].local_to_object_space(mirrored[sample], parents, gpu["port"].NORMALIZE_IEEE)[:, LANES])


@pytest.mark.parametrize("name", list(clips.SCALAR_SPECS))
def test_scalar_compression_error_matches_reference_exactly(gpu, name):
    from oracle import ref
    ab, ctx, port = gpu["ab"], gpu["ctx"], gpu["port"]
    spec = clips.SCALAR_SPECS[name]
    blob = clips.load_blob(name)
    if ref.available():
        r = ref.scalar_error(spec, blob)
    elif name in GOLDEN_SCALAR:
        g = np.load(clips.golden_path(name, "error.npz"))
        r = dict(raw_values=g["raw_values"], index=int(g["index"]), error=float(g["error"]), sample_time=float(g["sample_time"]),
                 sample_rate=float(g["sample_rate"]), duration=float(g["duration"]))
    else:
        pytest.skip("needs oracle/_ref/libaclref.so")
    clipset = ctx.upload([blob, blob], check_hash=True)
    components = clipset.components
    raw = np.ascontiguousarray(r["raw_values"][:, :, :components])
    # the clip twice: the second job reads its raw values behind the first one's
    jobs = _jobs(gpu, [dict(clip=1, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks),
                       dict(clip=0, num_samples=spec.num_samples, sample_rate=r["sample_rate"], duration=r["duration"], num_tracks=spec.num_tracks,
                            first_raw_pose=spec.num_samples)])
    got, _ = _measure(gpu, clipset, jobs, np.concatenate([raw, raw]), None, None, ab.Options())
    for record in got:
        assert (int(record["index"]), np.float32(record["error"]), np.float32(record["sample_time"]), int(record["flags"])) == \
            (r["index"], np.float32(r["error"]), np.float32(r["sample_time"]), 0), name
    clipset.release()


def test_rejects_what_it_cannot_measure(gpu):
    ab, ctx = gpu["ab"], gpu["ctx"]
    spec = clips.TRANSFORM_SPECS["c1_30bones"]
    clipset = ctx.upload([clips.load_blob("c1_30bones")])
    raw = np.zeros((spec.num_samples, spec.num_tracks, 12), np.float32)
    parents = np.full(spec.num_tracks, 0xFFFFFFFF, np.uint32)
    shells = np.ones(spec.num_tracks, np.float32)
    good = dict(clip=0, num_samples=spec.num_samples, sample_rate=30.0, duration=1.0, num_tracks=spec.num_tracks)
    for row, options in ((dict(good, clip=3), ab.Options()), (dict(good, num_tracks=spec.num_tracks + 1), ab.Options()),
                         (good, ab.Options(default_modes=(ab.DEFAULT_SKIPPED,) * 3)), (good, ab.Options(skip_mask=ab.SKIP_SCALE)),
                         (good, ab.Options(rounding_policy=ab.ROUND_PER_TRACK, per_track_rounding=1))):
        with pytest.raises(ab.AclB200Error) as err:
            _measure(gpu, clipset, _jobs(gpu, [row]), raw, parents, shells, options)
        assert err.value.status == 1
    # no samples / nothing to do
    got, _ = _measure(gpu, clipset, _jobs(gpu, [dict(good, num_samples=0)]), raw, parents, shells, ab.Options())
    assert (int(got[0]["index"]), float(got[0]["error"]), float(got[0]["sample_time"])) == (0xFFFFFFFF, 0.0, 0.0)
    clipset.release()


def test_decompress_all_samples_is_the_reference_sampling_loop(gpu):
    """aclb200_decompress_all_samples == the loop of convert_track_list / calculate_compression_error (convert.impl.h:164-171,
    track_error.impl.h:337-339): every sample of several clips in one call, bit for bit what the reference decoded sample by sample."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    names = ["mixed_scale", "c1_30bones", "ragged_17", "looping", "one_sample"]
    clipset = ctx.upload([clips.load_blob(n) for n in names], check_hash=True)
    cases = [_reference_case(n, 1) for n in names]
    order = [2, 0, 4, 3, 1, 0]
    rows = [dict(clip=c, num_samples=clips.TRANSFORM_SPECS[names[c]].num_samples, sample_rate=cases[c]["sample_rate"], duration=cases[c]["duration"]) for c in order]
    total = sum(r["num_samples"] for r in rows)
    options = _options(gpu, 1)
    options.rounding_policy = ab.ROUND_NEAREST
    d_out = torch.full((total, clipset.max_tracks, 12), float("nan"), dtype=torch.float32, device="cuda")
    ctx.decompress_all_samples(clipset, _jobs(gpu, rows), options, d_out)
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    row = 0
    for c in order:
        spec = clips.TRANSFORM_SPECS[names[c]]
        assert cases[c]["rounding"] == ab.ROUND_NEAREST
        assert clips.bit_equal(got[row:row + spec.num_samples, :spec.num_tracks][..., LANES], cases[c]["lossy_poses"][..., LANES]), names[c]
        row += spec.num_samples
    clipset.release()
