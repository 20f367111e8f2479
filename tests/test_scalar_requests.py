"""The fabricated scalar clips of tests/scalar_cases.py against the reference, and what their request lists make the chained scalar
kernel's plan and warp 0 do (the model in tests/scalar_cases.py). CPU only; tests/test_gpu_scalar.py decodes the same lists on the
device."""
from __future__ import annotations

import hashlib

import numpy as np
import pytest

from tests import clips
from tests import scalar_cases as sc

GOLDEN = "scalar_cases"

# sha256 of every fabricated clip: a change in the writer, the recipes or numpy's generators shows here first
PINNED_SHA256 = {
    "float1_constant_20": "72dff5cbc0cceac070331f81816e4c146da6196ea80ae5f8db4e7cfac3f8838f",
    "float1_content_1000_12_24.0_False_5": "d7b7a6d9ecc9bfb6b2b4631b43f5d39babff5400d2ce3d3aadb159fa38b498d8",
    "float1_content_257_40_30.0_False_1": "04c090c1da993fa463d29a4a5487f31eb9fb72926c6a0635150c4def0ad7fed5",
    "float1_content_257_40_30.0_False_2": "f18fba9ff364fff20015f540e8b330cb2edab2cfea5c07d240fc114557049f78",
    "float1_content_300_25_32.0_True_3": "1c1f95c13650ba6afbab7de7352cef79fa092b4a43f4fdf3f86f70c5d0fb4410",
    "float1_content_513_30_30.0_False_4": "40d2d36f609cc5e541407c6e3c0d3d975861c9ff11ff52f0ae2ebaf17637b31f",
    "float1_filler_1400_6": "4de19cec443cccae448d18166c6b809e2a01957d31ee976915f4fdc0d50644a8",
    "float1_filler_1460_5": "b2130cfd56d9f4b31f899e64c04c1f3550c9e69d923ab0cc176e43ecdef1911e",
    "float1_filler_2700_5": "48edbebc5194da90db519c779ee77f19cc94ad66e24b433a307954d426a546a7",
    "float1_one_sample_9": "a6fa298d73338d987a448f4ff881dc72b33ba61ae5cc729b08d225382abca6ec",
    "float2_constant_20": "2f3be1e23d4a0301aa743f62a6052f7b8ca590590a23b5ed4dd06b373515df52",
    "float2_content_1000_12_24.0_False_5": "e6207eb02ae46cb2642ca3758c998ee21dc1813ea5f0dc6860a5aaf54c4a422d",
    "float2_content_257_40_30.0_False_1": "a638848402be891962547077b62eb4cad958053d03a277b68932af2f011f4137",
    "float2_content_257_40_30.0_False_2": "9a2152d2f0ac5bc352283f1232d57e26ad84f7505b0f7d11aacb28fd7c3ad109",
    "float2_content_300_25_32.0_True_3": "c344b6d0f1fbe31fa55bc5dd74f74cd0a80dc2dd1950f29546555dd36b2d0bf4",
    "float2_content_513_30_30.0_False_4": "423eb387230cc7e035e53f0b6987ef3e57253fdc9a4438461cc30cbd6195e481",
    "float2_filler_5000_5": "bd02ff78a069af866de390bd2e612062b1c93b7977a4816216b286f0ca28dbae",
    "float2_filler_9000_4": "58c27b1c84d80d1837c0574122b80a8da48ac5f509af18eb5f88df7a68fd7328",
    "float2_one_sample_9": "a34d6b70283f2fe1ec72c86fa10dd74575fc90e7150df0946d9c9075bd0edc6f",
    "float3_constant_20": "4bc2bf9e272b96645a9c43f826e1dfc655b44b2eabdeda97534a0608bae07188",
    "float3_content_1000_12_24.0_False_5": "ad08841ad58fd2ffdab0b36badc99cda176d317fbb35882f8bbfa45c3042ad85",
    "float3_content_257_40_30.0_False_1": "6d9beaeb2f148dfc472b3f6599ce8367e540bf28ab6fd68c64e486732b16ab88",
    "float3_content_257_40_30.0_False_2": "aa7ad9b66c4d40d1f80777946bb1bb82a977d69a563b0539f86b96fbd8b50f7f",
    "float3_content_300_25_32.0_True_3": "dd665957020e883539a9468b31ae6777be6f44565104acc3fe11f6512a53c00a",
    "float3_content_513_30_30.0_False_4": "94558485539c66be9ff0074c72509aab4465e1f74284156ced8486b4b57871fc",
    "float3_filler_14000_4": "ae3a283736e166dd506f846f9f80491c8bfe207bf6fe43b41e6d38b9711c40c4",
    "float3_filler_20000_4": "b2890a3b457545c27b90ba45199134cd64770cffcc909c9b20656a01cbe736cc",
    "float3_one_sample_9": "24ae30304d9ff72c71aa146f34e410663b08e0d64a97935b4de010ff7b384237",
    "float4_constant_20": "cf81fa35f6e75824377e3d5d577be183387646a3215b3fae07e0a50e4ce384c3",
    "float4_content_1000_12_24.0_False_5": "66703d6c1e2e95300dc79affd7f1cfd5a4ac5e29535b655ac685f95aac63d447",
    "float4_content_257_40_30.0_False_1": "dc885a1d0c058ba23ea8093a621e55ba848d3d2acf4b40e5bd6539c53e441dd6",
    "float4_content_257_40_30.0_False_2": "994d0732174bd534b25d0ae09ebe08ac5b22a6325010e4f1598b723522afe77b",
    "float4_content_300_25_32.0_True_3": "4638fac6b7a093289b4e7d17830c9ad198b6be8bfa9acc6f9f79815af4ca0df7",
    "float4_content_513_30_30.0_False_4": "8e217401dd1fd7dc72c7f8f9a1e7a39cef8f755604bc1f8d699aa4d893768221",
    "float4_filler_30000_3": "16db3754000fff111e77d3f30c19c1d70af0f24d0822facd734127859ccb007a",
    "float4_one_sample_9": "8aee1cc41ca191257513d3db14650aefd591d1f558fe6bd664ee27098da57f09",
    "vector4_constant_20": "1eb6a897decdf43ba66fb2dd088c2df5c9ef52ab6e38ea1d6f74d1610e3426f6",
    "vector4_content_1000_12_24.0_False_5": "2d0e76937bdb73aa93980cd5541a517e4a1fca0d14a2b5e17cc69129cc7a5331",
    "vector4_content_257_40_30.0_False_1": "0cb7b8c0ef69d40b994f7b650d9ccf2ce9115d62f18a0965a478827f27a95b8a",
    "vector4_content_257_40_30.0_False_2": "84f4c706e9d0e2fc301f4df58de3d78765bbda8aea017331bcb1a73c7ddeaf48",
    "vector4_content_300_25_32.0_True_3": "26ed823b6d49a537b67af6b0e673ba4e3d59c05cc5d12c3da9d3fb9f6f8c8a38",
    "vector4_content_513_30_30.0_False_4": "9133e79e437b38aad3306e3aba4be3cd9104888bf7397cdf795093e794609bcf",
    "vector4_filler_50000_3": "f76b15f5e0427ef33705cd5d9c210d609f37a071615c9f460dfc106a13a6a25a",
    "vector4_one_sample_9": "8fb0b4ce8356a304798682d97ce6f29c108a7d46c1b7c19a2e4608ff6dab168c",
}

# requests per block by key frame bytes of the widest clip (plan_scalar_launch): each row's bounds and, for one request per block,
# whether a request's two key frames fit the pool and whether one key frame alone does
PLAN_TABLE = [(32, 0, 1441), (31, 1442, 1488), (16, 2683, 2843), (8, 4868, 5413), (4, 8145, 9782), (2, 12241, 16336),
              (1, 16337, 24528), (1, 24529, 49104), (1, 49105, 200000)]


def test_plan_table():
    for rpb, lo, hi in PLAN_TABLE:
        assert sc.plan(lo) == rpb and sc.plan(hi) == rpb, (rpb, lo, hi)
    for rpb, lo, hi in PLAN_TABLE[:6]:
        assert sc.plan(lo - 1) > rpb or lo == 0, (rpb, lo)
        assert sc.plan(hi + 1) < rpb, (rpb, hi)
    # one request per block: below 24529 bytes its two key frames fit the pool wherever they start; at 50000 not even one does
    assert max(sc.window_bytes(at, at + 8 * 24528, 8 * 24528) for at in range(128)) <= sc.POOL_BYTES
    assert min(sc.window_bytes(at, at, 8 * 50000) for at in range(128)) > sc.POOL_BYTES


def test_clip_sets_reach_every_plan_shape():
    reached = set()
    for name, (track_type, recipes, rpb) in sc.CLIP_SETS.items():
        _, blobs = sc.clip_set(name)
        kfb = max(sc.key_frame_bytes(b) for b in blobs)
        assert sc.plan(kfb) == rpb, (name, kfb)
        reached.update(i for i, (r, lo, hi) in enumerate(PLAN_TABLE) if r == rpb and lo <= kfb <= hi)
    assert reached == set(range(len(PLAN_TABLE)))
    shapes = {}
    for name, (track_type, _, rpb) in sc.CLIP_SETS.items():
        shapes.setdefault(track_type, set()).add(rpb)
    assert all(len(s) >= 3 for s in shapes.values()) and len(shapes) == 5, shapes
    # 257, 300, 513 and 1000 tracks at every component count
    for nc in (1, 2, 3, 4):
        counts = {recipe[1] for (track_type, recipes, _) in sc.CLIP_SETS.values() if sc.components(track_type) == nc
                  for recipe in recipes if recipe[0] == "content"}
        assert {257, 300, 513, 1000} <= counts, (nc, counts)


def test_blobs_are_valid_and_pinned(oracle_port):
    from oracle import ref
    blobs = sc.all_clips()
    assert set(blobs) == set(PINNED_SHA256)
    for name, blob in blobs.items():
        assert oracle_port.validate(blob, check_hash=True) == 0, name
        assert hashlib.sha256(blob.tobytes()).hexdigest() == PINNED_SHA256[name], name
        if ref.available():
            assert ref.lib().aclref_is_valid(blob.ctypes.data, 1) == 0, name


def _stream_layout(blob):
    """(bit offset in the frame, bits, components) of every animated track."""
    nc = sc.components(int(blob[15]))
    n = clips_num_tracks(blob)
    metadata = blob[52:52 + n]
    out, offset = [], 0
    for rate in metadata.tolist():
        bits = 32 if rate == 24 else rate
        if bits:
            out.append((offset, bits, nc))
        offset += bits * nc
    return out


def clips_num_tracks(blob) -> int:
    return int(blob[16:20].view(np.uint32)[0])


def test_blob_content():
    """Every bit width, integers at 0 and 2^bits - 1, components straddling a 32 bit word of the stream, constant tracks where the
    kernel's track loop turns, raw specials, a wrap clip and an all constant clip."""
    blobs = sc.all_clips()
    straddle, widths, types = set(), set(), set()
    for name, blob in blobs.items():
        types.add(int(blob[15]))
        bpf, samples = sc.bits_per_frame(blob), int(blob[20:24].view(np.uint32)[0])
        for offset, bits, nc in _stream_layout(blob):
            widths.add(bits)
            for k in range(samples):
                for c in range(nc):
                    at = k * bpf + offset + bits * c
                    if at % 32 + bits > 32:
                        straddle.add(bits)
    assert widths == set(sc.BIT_WIDTHS) and straddle == set(sc.BIT_WIDTHS) - {1}
    assert types == {0, 1, 2, 3, 4}
    assert any(int(b[28:32].view(np.uint32)[0]) >> 30 & 1 for b in blobs.values())
    assert any(sc.bits_per_frame(b) == 0 for b in blobs.values())
    tracks = sc.content_tracks(1, 300, 6, 1)
    assert all(tracks[t]["bits"] == 0 for t in (0, 255, 256, 257, 299))
    quantised = [t for t in tracks if 0 < t["bits"] < 32]
    assert all((t["ints"] == 0).any() and (t["ints"] == (1 << t["bits"]) - 1).any() for t in quantised)
    ranges = np.concatenate([np.concatenate([t["min"], t["extent"]]) for t in quantised])
    assert (np.abs(ranges[ranges != 0]) < np.float32(2.0 ** -126)).any() and (ranges == 0).any() and (ranges < 0).any()
    raw = np.concatenate([t["raw"].reshape(-1) for t in tracks if t["bits"] == 32])
    assert set(sc.RAW_SPECIALS.tolist()) <= set(raw.tolist())


@pytest.mark.parametrize("name", list(sc.CLIP_SETS))
def test_request_lists_cover_the_grouping(oracle_port, name):
    """The warp 0 model over the clip set's request list: groups of every length up to the batch, a group filling a batch, blocks
    whose pool runs out after some groups were staged, blocks staging nothing, chains broken by each cause, a final partial block.
    Where the plan rules a case out, the model must never meet it."""
    _, blobs = sc.clip_set(name)
    kfb = max(sc.key_frame_bytes(b) for b in blobs)
    rpb = sc.plan(kfb)
    req_clip, req_time, req_policy = sc.request_list(name)
    rows = sc.seek_rows(blobs, req_clip, req_time, req_policy)
    cov = sc.coverage(blobs, rows, rpb)
    assert cov["group_lengths"] == list(range(1, rpb + 1)), cov
    assert cov["full_batch"] > 0
    assert (cov["staged_then_global"] > 0) == sc.pool_can_run_out_mid_block(rpb, kfb), cov
    assert (cov["none_staged"] > 0) == sc.first_group_can_miss_pool(rpb, kfb), cov
    if rpb > 1:
        assert all(v > 0 for v in cov["breaks"].values()), cov["breaks"]
        assert cov["final_partial"]
    valid, clip_index, bpf, kf0, kf1 = rows.T
    staged = [g for groups in sc.block_groups(rows, rpb) for g in groups if g["staged"]]
    if rpb == 1 and 2 * kfb + 47 > sc.POOL_BYTES:
        # only a request whose two key frames are one (clamped, kf0 == kf1) can be staged, and none if one frame is over the pool
        widest = int(np.argmax([sc.key_frame_bytes(b) for b in blobs]))
        wide_staged = [g for g in staged if clip_index[g["first"]] == widest]
        assert all(kf0[g["first"]] == kf1[g["first"]] for g in wide_staged)
        assert (len(wide_staged) > 0) == (kfb + 47 <= sc.POOL_BYTES)


def _vocabulary(blob):
    return sc.vocabulary_times(blob)


@pytest.mark.parametrize("name", sorted(sc.all_clips()))
def test_port_equals_reference(reference, oracle_port, name):
    """The port against the live reference on every vocabulary time under every policy pair, decompress_tracks and decompress_track,
    per track rounding off (default_scalar settings) and on (debug_scalar, rounding per_track and none)."""
    blob = sc.all_clips()[name]
    nc = sc.components(int(blob[15]))
    n = clips_num_tracks(blob)
    policies = sc.track_policies(n)
    for per_track in (False, True):
        settings = oracle_port.SettingsBuilder(per_track_rounding=per_track, per_track_policies=policies if per_track else None)
        roundings = (0, 4) if per_track else (0, 1, 2, 3)
        for ti, t in enumerate(_vocabulary(blob).tolist()):
            for rounding in roundings:
                for looping in (0, 1, 2):
                    kw = dict(settings=int(per_track), per_track_rounding=policies if per_track else None)
                    want = reference.scalar_decompress(blob, t, rounding, looping, **kw)[:, :nc]
                    got = oracle_port.scalar_decompress(blob, settings, t, rounding, looping)[:, :nc]
                    assert sc.nan_rule_equal(got, want).all(), (name, per_track, t, rounding, looping)
                    for track in {(ti * 7 + rounding + looping) % n, n - 1}:
                        want1 = reference.scalar_decompress(blob, t, rounding, looping, track_index=track, **kw)[:, :nc]
                        got1 = oracle_port.scalar_decompress(blob, settings, t, rounding, looping, track=track)[:, :nc]
                        assert sc.nan_rule_equal(got1, want1).all(), (name, per_track, t, rounding, looping, track)


def test_port_equals_golden(oracle_port):
    """The reference's values stored by tests/golden/make_scalar_cases_golden.py, for machines without the compiled reference."""
    g = np.load(clips.golden_path(GOLDEN, "golden.npz"))
    blobs = sc.all_clips()
    assert sorted(blobs) == sorted(str(x) for x in g["names"])
    for name, blob in blobs.items():
        nc = sc.components(int(blob[15]))
        n = clips_num_tracks(blob)
        times, tracks = g[name + "/times"], g[name + "/tracks"]
        values = g[name + "/values"]
        for k, (per_track, rounding, looping) in enumerate(sc.GOLDEN_COMBOS):
            settings = oracle_port.SettingsBuilder(per_track_rounding=per_track, per_track_policies=sc.track_policies(n) if per_track else None)
            for ti, t in enumerate(times.tolist()):
                got = oracle_port.scalar_decompress(blob, settings, t, rounding, looping)[tracks, :nc]
                assert sc.nan_rule_equal(got, values[k, ti]).all(), (name, k, t)
