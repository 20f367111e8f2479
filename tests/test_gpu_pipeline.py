"""The pipeline kernel (acl_b200/csrc/pipeline.cu) at real launch sizes, request by request against the oracle.

Every case picks a clip set whose widest clip gives one batch shape (requests per batch, batches per seek pass), asserts through
Context.debug_last_launch() that the launches really take that kernel and plan, and decodes request lists built from sequential
playback runs (chains of every length, cuts at k_group_max, segment crossings, wraps, repeats, reversed runs), clips interleaved
request by request and in blocks, invalid clip indices, and all of it shuffled. Launch sizes go from one request to more than ten
batches per block, so that every block walks its ring of ReqHot slots several times.

Every request of every launch is compared with oracle/port: bit for bit in exact mode on the defined lanes; in fast mode rotations
within 1e-5 and vectors bit for bit. Bytes nobody may write (invalid requests, bones past a clip's bone count, stride padding, the bytes
before an offset output pointer) keep their sentinel. The oracle runs once per distinct (clip, time, policy); a launch's expected
output is a gather.
"""
import numpy as np
import pytest

from tests import clips
from tests import pipeline_cases as pc

pytestmark = pytest.mark.gpu

LANES = clips.DEFINED_LANES
FAST_MATH_TOLERANCE = 1e-5
SENTINEL = np.uint32(0x7FBADBAD)        # a NaN no decode produces


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    from oracle import port
    port.lib()
    return dict(torch=torch, ab=ab, port=port, ctx=ab.Context(0), sms=torch.cuda.get_device_properties(0).multi_processor_count)


# (clip names, clips whose request runs wrap, the requests per batch the widest clip gives: (low, high)). Measured on an H100 in
# QVV48: 24 for the 30 bone set (one batch per seek pass), 13 and 15 for 57 and 40 bones (two per pass).
CASES = {
    "ragged_30": (["c1_30bones", "c5_30x32", "ragged_17", "one_bone", "two_samples", "one_sample", "all_default"], [], (17, 32)),
    "mixed_scale_57": (["mixed_scale"], [], (11, 20)),
    "raw_loops_40": (["noisy_raw", "looping", "stripped_loop"], ["looping", "stripped_loop"], (11, 20)),
    "half_turn_64": (["half_turn"], [], (11, 16)),
    "c2_100": (["c2_100bones"], [], (9, 10)),
    "seg_200": (["seg_200", "c2_100bones"], ["seg_200"], (3, 8)),
    "paragon_540": (["paragon_like"], [], None),
    "wide_2500": (["wide_2500", "c1_30bones"], [], None),
}

# (settings kind, layout, math): the grouped instances (kinds 0, 4: lerp_only; 3: never) in both layouts and in fast math, the
# ungrouped ones (kind 1: per track rounding, normalise always)
COMBOS = [(0, 0, 0), (3, 1, 0), (1, 0, 0), (0, 1, 0), (4, 0, 1), (3, 1, 1), (1, 1, 0)]
BIG_COMBOS = 3          # the first three also decode the launches of ten and more batches per block


def _options(gpu, kind, layout, math, **kw):
    ab = gpu["ab"]
    s = gpu["port"].settings_for_kind(kind).c
    return ab.Options(normalization=s.normalization, per_track_rounding=s.per_track_rounding, wrapping=s.wrapping,
                      clamp_sample_time=s.clamp_sample_time, multiple_rotation_formats=s.multiple_rotation_formats,
                      default_modes=(s.default_rotation_mode, s.default_translation_mode, s.default_scale_mode),
                      constant_defaults=list(s.constant_defaults), output_layout=layout, math_mode=math, **kw)


class Oracle:
    """The oracle's poses per (clip, time, policy pair), computed on first use."""

    def __init__(self, port, blobs, kind):
        self.port, self.blobs, self.settings = port, blobs, port.settings_for_kind(kind)
        self.rows = {}

    def pose(self, clip, t, policy):
        key = (clip, t, policy)
        if key not in self.rows:
            rounding, looping = pc.POLICY_PAIRS[policy]
            self.rows[key] = self.port.transform_decompress_tracks(self.blobs[clip], self.settings, t, rounding, looping)
        return self.rows[key]


def _launch(gpu, clipset, blobs, oracle, req_clip, req_time, req_policy, kind, layout, math, uniform=None, stride_pad=0, offset=0):
    """One decompress_tracks over an output buffer full of sentinels; checks every byte of it. Returns the launch info."""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    n = len(req_clip)
    width = 12 if layout == ab.LAYOUT_QVV48 else 10
    max_tracks = clipset.max_tracks
    pose_words = max_tracks * width
    stride_words = pose_words + stride_pad // 4
    total_words = offset // 4 + n * stride_words + 4
    d_out = torch.full((total_words,), int(SENTINEL.view(np.int32)), dtype=torch.int32, device="cuda")
    d_requests = torch.from_numpy(ab.make_requests(req_clip, req_time).view(np.uint8)).cuda()
    policy_bytes = np.array([pc.POLICY_PAIRS[p] for p in req_policy.tolist()], dtype=np.uint8).reshape(n, 2)
    if uniform is None:
        d_policies = torch.from_numpy(policy_bytes).cuda()
        options = _options(gpu, kind, layout, math, d_request_policies=d_policies.data_ptr())
    else:
        rounding, looping = pc.POLICY_PAIRS[uniform]
        req_policy = np.full(n, uniform)
        options = _options(gpu, kind, layout, math, rounding_policy=rounding, looping_policy=looping)
    options.pose_stride_bytes = stride_words * 4 if stride_pad else 0
    ctx.decompress_tracks(clipset, d_requests, n, options, d_out.data_ptr() + offset)
    torch.cuda.synchronize()
    info = ctx.debug_last_launch()
    got = d_out.cpu().numpy().view(np.uint32)

    # expected: sentinels everywhere, the oracle's rows where a request writes
    want = np.full(total_words, SENTINEL, dtype=np.uint32)
    rows = want[offset // 4: offset // 4 + n * stride_words].reshape(n, stride_words)
    check = np.ones_like(rows, dtype=bool)          # lanes compared bit for bit
    rot = np.zeros_like(rows, dtype=bool)           # rotation lanes (fast math: compared within the tolerance)
    lanes = LANES if layout == ab.LAYOUT_QVV48 else list(range(10))
    for i in range(n):
        c = int(req_clip[i])
        if c >= len(blobs):
            continue
        pose = oracle.pose(c, float(req_time[i]), int(req_policy[i]))
        nt = pose.shape[0]
        block = np.zeros((nt, width), dtype=np.float32)
        block[:, lanes] = pose[:, LANES]
        rows[i, :nt * width] = block.view(np.uint32).reshape(-1)
        if layout == ab.LAYOUT_QVV48:       # translation.w / scale.w are not defined by the reference
            check[i, :nt * width].reshape(nt, width)[:, [7, 11]] = False
        rot[i, :nt * width].reshape(nt, width)[:, :4] = True
    got_rows = got[offset // 4: offset // 4 + n * stride_words].reshape(n, stride_words)
    assert np.array_equal(got[:offset // 4], want[:offset // 4]) and np.array_equal(got[offset // 4 + n * stride_words:], want[offset // 4 + n * stride_words:]), \
        "bytes outside the poses were written"
    exact = check & ~rot if math == ab.MATH_FAST else check
    bad = exact & (got_rows != rows)
    if math == ab.MATH_FAST:
        diff = np.abs(got_rows.view(np.float32) - rows.view(np.float32))
        bad |= rot & check & ~(diff <= FAST_MATH_TOLERANCE)
    if bad.any():
        r, w = np.argwhere(bad)[0]
        rpb = max(info.requests_per_block, 1)
        c = int(req_clip[r])
        raise AssertionError(
            f"{int(bad.any(axis=1).sum())} of {n} requests differ; first: request {r} (batch {r // rpb}, lane {r % rpb}), clip {c}, "
            f"time {float(req_time[r])!r}, policy {pc.POLICY_PAIRS[int(req_policy[r])]}, bone {w // width}, lane {w % width}: "
            f"got {got_rows[r, w].view(np.float32)!r} want {rows[r, w].view(np.float32)!r}; {info}")
    return info


def _sizes(rpb, grid):
    whole = grid * rpb
    return sorted({s for s in (1, rpb - 1, rpb + 1, whole - 1, whole + 1) if s >= 1})


@pytest.mark.parametrize("case", list(CASES))
def test_pipeline_batch_shapes_vs_oracle(gpu, case):
    ab, ctx, port = gpu["ab"], gpu["ctx"], gpu["port"]
    names, wrap_names, expected_rpb = CASES[case]
    blobs = [pc.load_blob(n) for n in names]
    clipset = ctx.upload(blobs, check_hash=True)
    all_even = all(int(pc.spec_of(n).num_tracks) % 2 == 0 for n in names)
    report = []
    for ci, (kind, layout, math) in enumerate(COMBOS):
        if case == "wide_2500" and layout == ab.LAYOUT_QVV48 and ci >= BIG_COMBOS:
            continue
        oracle = Oracle(port, blobs, kind)
        # per request policies exist for the batch wide rounding only: per track rounding (kind 1) takes one policy per launch
        per_launch = (lambda i: None) if kind != 1 else (lambda i: (5 * i + 1) % len(pc.POLICY_PAIRS))
        probe = pc.request_list(names, wrap_names, 8, seed=ci)
        info = _launch(gpu, clipset, blobs, oracle, *probe, kind, layout, math, uniform=per_launch(0))
        rpb = info.requests_per_block
        # the launch shape this case exists for
        if case == "wide_2500" and layout == ab.LAYOUT_QVV48:
            assert info.kernel == ab.api.KERNEL_PLAIN, info         # a 2500 bone QVV48 pose does not fit in shared memory
        else:
            assert info.kernel == ab.api.KERNEL_PIPELINE, info
        if case == "paragon_540":
            assert rpb == (1 if layout == ab.LAYOUT_QVV48 else 2), info
        elif case == "wide_2500":
            assert layout == ab.LAYOUT_QVV48 or rpb == 1, info
        else:
            assert expected_rpb[0] <= rpb <= expected_rpb[1], info
        # the resident grid: from a launch of more batches than the device holds blocks
        big = pc.request_list(names, wrap_names, 2 * 2 * gpu["sms"] * rpb + 3, seed=100 + ci)
        info = _launch(gpu, clipset, blobs, oracle, *big, kind, layout, math, uniform=per_launch(1))
        grid = info.grid_blocks
        if info.kernel == ab.api.KERNEL_PIPELINE:
            assert grid in (gpu["sms"], 2 * gpu["sms"]), info
            if case == "wide_2500":
                assert grid == gpu["sms"], info             # one block per SM
        pipeline = info.kernel == ab.api.KERNEL_PIPELINE
        sizes = _sizes(rpb, grid) if pipeline else [1, 2, 7, 33]
        if ci < BIG_COMBOS and pipeline:
            sizes.append(10 * grid * rpb + rpb // 2 + 1)
        master = pc.request_list(names, wrap_names, max(sizes) + 64, seed=200 + ci)
        for si, size in enumerate(sizes):
            start = (si * 37) % 64
            part = tuple(x[start:start + size] for x in master)
            # addressing: plain, padded stride, an output pointer 8 (QVV40) or 16 (QVV48) bytes past an allocation
            variant = si % 3
            stride_pad = (16 if layout == ab.LAYOUT_QVV48 else 24) if variant == 1 else 0
            offset = (16 if layout == ab.LAYOUT_QVV48 else 8) if variant == 2 else 0
            info = _launch(gpu, clipset, blobs, oracle, *part, kind, layout, math, uniform=per_launch(si), stride_pad=stride_pad, offset=offset)
            assert info.num_requests == size and info.num_batches == -(-size // max(info.requests_per_block, 1)), info
            if info.kernel == ab.api.KERNEL_PIPELINE:
                rows_16 = layout == ab.LAYOUT_QVV48 or all_even
                assert info.out_bulk == int(rows_16 and stride_pad % 16 == 0 and offset % 16 == 0), (info, stride_pad, offset)
            if size > 10 * grid * rpb:
                assert info.num_batches // info.grid_blocks >= 10, info
                rows = pc.seek_rows(port, blobs, port.settings_for_kind(kind), *part)
                cover = pc.groups(rows, info.requests_per_block, grouped=kind != 1)
                report.append((kind, layout, math, repr(info), cover))
                if kind != 1 and info.kernel == ab.api.KERNEL_PIPELINE:
                    _assert_coverage(case, names, wrap_names, blobs, info.requests_per_block, cover)
                # the same requests shuffled: order must not matter
                perm = np.random.default_rng(size).permutation(size)
                _launch(gpu, clipset, blobs, oracle, *(x[perm] for x in part), kind, layout, math, uniform=per_launch(si + 1))
        # one policy for the whole launch
        _launch(gpu, clipset, blobs, oracle, *master, kind, layout, math, uniform=3 * 3 + (1 if wrap_names else 0))
    for line in report:
        print(case, *line)
    clipset.release()


def _assert_coverage(case, names, wrap_names, blobs, rpb, cover):
    segmented = any(port_segments(b) > 1 for b in blobs)
    for length in range(2, min(pc.K_GROUP_MAX, rpb) + 1):
        assert cover[f"groups_of_{length}"] >= 3, (case, length, cover)
    if rpb > pc.K_GROUP_MAX:
        assert cover["cuts"] >= 3, (case, cover)
    if segmented and rpb >= 2:
        assert cover["tail_crossings"] >= 3 and cover["tail_crossings_at_last_lane"] >= 1, (case, cover)
        assert cover["crossings_at_lane_0"] >= 1, (case, cover)
    if wrap_names and rpb >= 2:
        assert cover["tail_crossings_into_segment_0"] >= 1, (case, cover)
    if rpb >= 2:
        assert cover["chained_clamped_repeats"] >= 3, (case, cover)


def port_segments(blob):
    from oracle import port
    s = port.settings_for_kind(0)
    return len({port.transform_seek(blob, s, float(t), 0, 0).segment_indices[0] for t in np.linspace(0, 10, 200)})


def test_host_call_in_chunks_matches_device(gpu):
    """decompress_tracks_host splits 65 536 requests or more into 8 chunks whose boundaries fall inside batches; with a padded stride
    the result equals one device launch."""
    torch, ab, ctx, port = gpu["torch"], gpu["ab"], gpu["ctx"], gpu["port"]
    names, wrap_names, _ = CASES["ragged_30"]
    blobs = [pc.load_blob(n) for n in names]
    clipset = ctx.upload(blobs)
    count = 65536 + 77
    req_clip, req_time, _ = pc.request_list(names, wrap_names, count, seed=9)
    width = 12
    stride = clipset.max_tracks * 48 + 32
    options = _options(gpu, 0, ab.LAYOUT_QVV48, 0)
    options.pose_stride_bytes = stride
    requests = ab.make_requests(req_clip, req_time)
    d_out = torch.zeros(count * stride // 4, dtype=torch.int32, device="cuda")
    ctx.decompress_tracks(clipset, torch.from_numpy(requests.view(np.uint8)).cuda(), count, options, d_out)
    torch.cuda.synchronize()
    device = d_out.cpu().numpy().view(np.uint32)
    host = np.full(count * stride // 4, 7, dtype=np.uint32)
    ctx.decompress_tracks_host(clipset, requests, options, host)
    info = ctx.debug_last_launch()
    assert info.kernel == ab.api.KERNEL_PIPELINE and info.num_requests in (count // 8, count // 8 + 1), info
    assert np.array_equal(host, device)
    # and a sample against the oracle
    settings = port.settings_for_kind(0)
    rows = host.view(np.float32).reshape(count, stride // 4)
    for i in np.random.default_rng(1).integers(0, count, 300):
        c = int(req_clip[i])
        if c >= len(blobs):
            continue
        want = port.transform_decompress_tracks(blobs[c], settings, float(req_time[i]))
        nt = want.shape[0]
        assert clips.bit_equal(rows[i, :nt * width].reshape(nt, width)[:, LANES], want[:, LANES]), i
    clipset.release()
