"""Fabricated scalar clips, request lists and a model of the chained scalar kernel's plan and grouping (tests/test_scalar_requests.py,
tests/test_gpu_scalar.py, tests/golden/make_scalar_cases_golden.py).

The reference's compressor picks bit widths and frame sizes itself, and never stores -0.0, subnormals, +-FLT_MAX or +-inf in a raw
track. A writer can. `write_blob` lays out a compressed_tracks v02_01_00 scalar clip the way compress.scalar.impl.h does (headers,
one bit rate byte per track, constant values, range values, the animated bit stream, 15 bytes of padding, the FNV-1a hash over bytes
[8, size)), so that the unmodified reference, the port and the library all decode it. Clips are built from recipes at test time; their
bytes are pinned by sha256 in tests/test_scalar_requests.py.

Each clip set puts small clips beside one wide clip, whose key frame size sets the requests per block of every launch on the set
(plan_scalar_launch in acl_b200/csrc/kernels.cu), and so the pressure on the 48 KB key frame pool. `plan` and `block_groups` mirror
that plan and warp 0 of scalar_tracks_pipeline_kernel: which requests chain into groups, the window each group stages and whether it
fits the pool.

Request lists index a per clip vocabulary of (time, policy) pairs, so the oracle runs once per entry and the expected output of a
launch is a gather.
"""
from __future__ import annotations

import functools

import numpy as np

from oracle import port, ref
from tests import edge_cases

TAG = 0xAC11AC11
VERSION = 10                    # v02_01_00
POOL_BYTES = 48 * 1024          # kernels.cu: k_scalar_pool_bytes
MAX_BATCH = 32                  # k_scalar_max_batch
BIT_WIDTHS = list(range(1, 24)) + [32]
TYPE_NAMES = {0: "float1", 1: "float2", 2: "float3", 3: "float4", 4: "vector4"}
F32_MAX = float(np.finfo(np.float32).max)
# raw 32 bit values no compressor stores: signed zero, subnormals, the largest finite values and infinities
RAW_SPECIALS = np.array([-0.0, 1e-45, -1e-45, 2.0 ** -130, F32_MAX, -F32_MAX, np.inf, -np.inf], dtype=np.float32).view(np.uint32)
SENTINEL = 0xDEADBEEF           # -6.26e18: not a NaN, so a lane holding it is compared bit for bit


def components(track_type: int) -> int:
    return track_type + 1 if track_type <= 3 else 4


# ---- the writer ----

def write_blob(track_type: int, sample_rate: float, num_samples: int, tracks: list[dict], wrap: bool = False) -> np.ndarray:
    """A compressed_tracks v02_01_00 scalar clip. Each track is a dict with `bits` (0, 1..23 or 32) and:
    bits 0: `value` float32[nc]; 1..23: `min`, `extent` float32[nc] and `ints` uint[num_samples][nc]; 32: `raw` uint32[num_samples][nc]
    (float bit patterns)."""
    nc = components(track_type)
    metadata = np.array([t["bits"] if t["bits"] <= 23 else 24 for t in tracks], dtype=np.uint8)
    constants = [np.asarray(t["value"], dtype=np.float32) for t in tracks if t["bits"] == 0]
    ranges = [np.concatenate([np.asarray(t["min"], np.float32), np.asarray(t["extent"], np.float32)]) for t in tracks if 0 < t["bits"] < 32]
    columns = []        # [num_samples, width] bits of one component, in stream order
    for t in tracks:
        b = t["bits"]
        if b == 0:
            continue
        values = np.asarray(t["raw"] if b == 32 else t["ints"], dtype=np.uint64).reshape(num_samples, nc)
        assert int(values.max(initial=0)) < (1 << b)
        shifts = np.arange(b - 1, -1, -1, dtype=np.uint64)
        for c in range(nc):
            columns.append(((values[:, c:c + 1] >> shifts) & 1).astype(np.uint8))
    bits_per_frame = sum(t["bits"] * nc for t in tracks)
    stream = np.packbits(np.concatenate(columns, axis=1).reshape(-1)) if columns else np.zeros(0, np.uint8)

    def align4(n):
        return (n + 3) & ~3
    metadata_at = 52
    constant_at = align4(metadata_at + len(tracks))
    range_at = constant_at + 4 * nc * len(constants)
    animated_at = range_at + 8 * nc * len(ranges)
    size = animated_at + stream.size + 15
    blob = np.zeros(size, dtype=np.uint8)
    blob[0:4] = np.array([size], np.uint32).view(np.uint8)
    blob[8:12] = np.array([TAG], np.uint32).view(np.uint8)
    blob[12:14] = np.array([VERSION], np.uint16).view(np.uint8)
    blob[15] = track_type
    header = np.array([len(tracks), num_samples], np.uint32).view(np.uint8)
    blob[16:24] = header
    blob[24:28] = np.array([sample_rate], np.float32).view(np.uint8)
    blob[28:32] = np.array([(1 << 30) if wrap else 0], np.uint32).view(np.uint8)
    offsets = np.array([bits_per_frame, metadata_at - 32, constant_at - 32, range_at - 32, animated_at - 32], np.uint32)
    blob[32:52] = offsets.view(np.uint8)
    blob[metadata_at:metadata_at + len(tracks)] = metadata
    if constants:
        blob[constant_at:range_at] = np.concatenate(constants).view(np.uint8)
    if ranges:
        blob[range_at:animated_at] = np.concatenate(ranges).view(np.uint8)
    blob[animated_at:animated_at + stream.size] = stream
    blob[4:8] = np.array([port.hash32(blob[8:size])], np.uint32).view(np.uint8)
    return ref.aligned_blob(blob)


def bits_per_frame(blob: np.ndarray) -> int:
    return int(blob[32:36].view(np.uint32)[0])


def key_frame_bytes(blob: np.ndarray) -> int:
    return (bits_per_frame(blob) + 7) // 8


# ---- clip recipes ----

# Constant tracks first, last and at 255, 256 and 257 (the second pass of the kernel's 256 thread track loop begins at 256)
CONSTANT_AT = (0, 255, 256, 257)


def _quantised(rng, nc, num_samples, b, kind):
    """Range and integers of a quantised track. Integers at 0 and 2^bits - 1 in every fifth key frame; `kind` picks a subnormal,
    zero or negative range, or a plain one."""
    top = (1 << b) - 1
    ints = rng.integers(0, top + 1, size=(num_samples, nc), dtype=np.int64)
    ints[1::5] = 0
    ints[3::5] = top
    if kind == 0:
        lo, ext = rng.uniform(-2.0 ** -128, 2.0 ** -128, nc), rng.uniform(2.0 ** -135, 2.0 ** -127, nc)     # subnormal
    elif kind == 1:
        lo, ext = rng.uniform(-50, 50, nc), np.zeros(nc)                                                # zero extent
    elif kind == 2:
        lo, ext = rng.uniform(-1e6, -1, nc), -rng.uniform(0.5, 1e3, nc)                                 # negative min and extent
    else:
        lo, ext = rng.uniform(-10, 10, nc), rng.uniform(0.01, 20, nc)
    return dict(bits=b, min=lo.astype(np.float32), extent=ext.astype(np.float32), ints=ints)


def _raw(rng, nc, num_samples, track, specials: bool):
    raw = rng.uniform(-1e4, 1e4, size=(num_samples, nc)).astype(np.float32).view(np.uint32)
    if specials:
        for k in range(0, num_samples, 3):
            for c in range(nc):
                raw[k, c] = RAW_SPECIALS[(track + k + c) % len(RAW_SPECIALS)]
    return dict(bits=32, raw=raw)


def content_tracks(nc: int, num_tracks: int, num_samples: int, seed: int) -> list[dict]:
    """Tracks cycling through every bit width (1..23, 32), constant at CONSTANT_AT and the last track; the widths depend on the track
    index only, so clips of one track count share their frame layout whatever the seed."""
    rng = np.random.default_rng(seed)
    tracks = []
    width = 0
    for track in range(num_tracks):
        if track in CONSTANT_AT or track == num_tracks - 1 or track % 11 == 5:
            value = rng.uniform(-100, 100, nc).astype(np.float32)
            if track % 3 == 0:
                value[0] = -0.0
            tracks.append(dict(bits=0, value=value))
            continue
        b = BIT_WIDTHS[width % len(BIT_WIDTHS)]
        width += 1
        tracks.append(_raw(rng, nc, num_samples, track, specials=track % 2 == 1) if b == 32 else _quantised(rng, nc, num_samples, b, track % 7))
    return tracks


def filler_tracks(nc: int, kfb: int, num_samples: int, seed: int) -> list[dict]:
    """Raw tracks, then one or two quantised ones, so that (bits per frame + 7) // 8 == kfb exactly."""
    rng = np.random.default_rng(seed)
    target = (8 * kfb) // nc * nc
    assert (target + 7) // 8 == kfb
    raw_tracks = (target - 24 * nc) // (32 * nc)
    tracks = [_raw(rng, nc, num_samples, t, specials=False) for t in range(raw_tracks)]
    rest = (target - raw_tracks * 32 * nc) // nc
    while rest > 0:
        b = min(rest, 23)
        tracks.append(_quantised(rng, nc, num_samples, b, 3))
        rest -= b
    return tracks


@functools.lru_cache(maxsize=None)
def clip(track_type: int, recipe: tuple) -> np.ndarray:
    """The blob of one recipe: ("content", tracks, samples, rate, wrap, seed), ("constant", tracks), ("one_sample", tracks) or
    ("filler", key frame bytes, samples)."""
    nc = components(track_type)
    kind = recipe[0]
    if kind == "content":
        _, num_tracks, num_samples, rate, wrap, seed = recipe
        return write_blob(track_type, rate, num_samples, content_tracks(nc, num_tracks, num_samples, seed), wrap)
    if kind == "constant":
        rng = np.random.default_rng(recipe[1])
        tracks = [dict(bits=0, value=rng.uniform(-5, 5, nc).astype(np.float32)) for _ in range(recipe[1])]
        return write_blob(track_type, 30.0, 10, tracks)
    if kind == "one_sample":
        return write_blob(track_type, 30.0, 1, content_tracks(nc, recipe[1], 1, 77))
    if kind == "filler":
        _, kfb, num_samples = recipe
        return write_blob(track_type, 30.0, num_samples, filler_tracks(nc, kfb, num_samples, kfb))
    raise ValueError(recipe)


C257 = ("content", 257, 40, 30.0, False, 1)
TWIN257 = ("content", 257, 40, 30.0, False, 2)          # C257's frame layout with other values: chains break on the clip alone
C300W = ("content", 300, 25, 32.0, True, 3)             # wrap flag; t * 32 is exact, so alpha = 0.5 ties exist
C513 = ("content", 513, 30, 30.0, False, 4)
C1000 = ("content", 1000, 12, 24.0, False, 5)
CONST = ("constant", 20)
ONE = ("one_sample", 9)

# name: track type, clips, the requests per block the plan gives
CLIP_SETS = {
    "float1_r32": (0, [C257, TWIN257, C300W, CONST, ONE, ("filler", 1400, 6)], 32),
    "float1_r31": (0, [C513, C257, TWIN257, CONST, ("filler", 1460, 5)], 31),
    "float1_r16": (0, [C1000, C257, TWIN257, CONST, ("filler", 2700, 5)], 16),
    "float2_r32": (1, [C257, TWIN257, C300W, CONST, ONE], 32),
    "float2_r8": (1, [C257, TWIN257, C300W, CONST, ("filler", 5000, 5)], 8),
    "float2_r4": (1, [C513, C1000, TWIN257, C257, CONST, ("filler", 9000, 4)], 4),
    "float3_r2": (2, [C257, TWIN257, C300W, CONST, ("filler", 14000, 4)], 2),
    "float3_r1_two_frames_fit": (2, [C513, C1000, C257, TWIN257, CONST, ("filler", 20000, 4)], 1),
    "float3_r32": (2, [C257, TWIN257, CONST, ONE], 32),
    "float4_r1_two_frames_do_not_fit": (3, [C257, TWIN257, C300W, CONST, ("filler", 30000, 3)], 1),
    "float4_r7": (3, [C513, C1000, C257, TWIN257, CONST], 7),
    "float4_r31": (3, [C257, TWIN257, CONST, ONE], 31),
    "vector4_r1_frame_over_pool": (4, [C257, TWIN257, C300W, CONST, ("filler", 50000, 3)], 1),
    "vector4_r7": (4, [C513, C1000, C257, TWIN257, CONST], 7),
    "vector4_r27": (4, [C300W, C257, TWIN257, CONST, ONE], 27),
}


def clip_set(name: str) -> tuple[int, list[np.ndarray]]:
    track_type, recipes, _ = CLIP_SETS[name]
    return track_type, [clip(track_type, r) for r in recipes]


def clip_name(track_type: int, recipe: tuple) -> str:
    return TYPE_NAMES[track_type] + "_" + "_".join(str(x) for x in recipe)


def all_clips() -> dict[str, np.ndarray]:
    """Every distinct clip of the clip sets, by name."""
    out = {}
    for track_type, recipes, _ in CLIP_SETS.values():
        for r in recipes:
            out[clip_name(track_type, r)] = clip(track_type, r)
    return out


# ---- the plan and warp 0 of scalar_tracks_pipeline_kernel ----

def plan(max_key_frame_bytes: int) -> int:
    """Requests per block of a scalar decompress_tracks launch (plan_scalar_launch)."""
    r = POOL_BYTES // (max_key_frame_bytes + 48)
    if r > 1:
        r -= 1
    return min(max(r, 1), MAX_BATCH)


def window_bytes(head_kf0: int, last_kf1: int, bits_per_frame: int) -> int:
    src_byte = (head_kf0 >> 3) & ~15
    return ((((last_kf1 + bits_per_frame - src_byte * 8) + 7) >> 3) + 16 + 15) & ~15


def seek_rows(blobs, req_clip, req_time, req_policy) -> np.ndarray:
    """What warp 0 reads of each request: valid, clip, bits per frame, key frame 0 and 1 bit offsets."""
    rows = np.zeros((len(req_clip), 5), dtype=np.int64)
    settings = port.SettingsBuilder()
    cache = {}
    for i, (c, t, p) in enumerate(zip(req_clip.tolist(), req_time.astype(np.float32).view(np.uint32).tolist(), req_policy.tolist())):
        if c >= len(blobs):
            continue
        key = (c, t, p)
        if key not in cache:
            rounding, looping = policy_pair(p)
            st = port.scalar_seek(blobs[c], settings, float(np.uint32(t).view(np.float32)), rounding, looping)
            cache[key] = (1, c, bits_per_frame(blobs[c]), st.key_frame_bit_offsets[0], st.key_frame_bit_offsets[1])
        rows[i] = cache[key]
    return rows


def block_groups(rows: np.ndarray, rpb: int) -> list[list[dict]]:
    """Per block, its groups as warp 0 forms them: first request, count, mergeable, window bytes, pool offset, staged."""
    valid, clip_index, bpf, kf0, kf1 = rows.T
    mergeable = (valid == 1) & (kf1 >= kf0) & (bpf != 0)
    blocks = []
    for first in range(0, len(rows), rpb):
        last = min(first + rpb, len(rows))
        heads = [i for i in range(first, last)
                 if not (i > first and mergeable[i] and mergeable[i - 1] and clip_index[i] == clip_index[i - 1] and kf0[i] == kf1[i - 1])]
        groups, offset = [], 0
        for h, end in zip(heads, heads[1:] + [last]):
            window = window_bytes(int(kf0[h]), int(kf1[end - 1]), int(bpf[h])) if mergeable[h] else 0
            staged = bool(mergeable[h] and window != 0 and offset + window <= POOL_BYTES)
            groups.append(dict(first=h, count=end - h, mergeable=bool(mergeable[h]), window=window, offset=offset, staged=staged))
            offset += window
        blocks.append(groups)
    return blocks


BREAK_CAUSES = ("clip", "invalid", "wrap", "backward", "constant")


def coverage(blobs, rows: np.ndarray, rpb: int) -> dict:
    """What a request list makes warp 0 do: group lengths, whole batch groups, blocks whose staged groups are followed by groups read
    from global memory, blocks with mergeable groups none of which is staged, the causes of broken chains, a final partial block."""
    valid, clip_index, bpf, kf0, kf1 = rows.T
    mergeable = (valid == 1) & (kf1 >= kf0) & (bpf != 0)
    blocks = block_groups(rows, rpb)
    lengths = set()
    out = dict(full_batch=0, staged_then_global=0, none_staged=0, final_partial=int(len(rows) % rpb != 0))
    for groups in blocks:
        staged = [g["staged"] for g in groups if g["mergeable"]]
        lengths.update(g["count"] for g in groups if g["mergeable"])
        out["full_batch"] += int(any(g["mergeable"] and g["count"] == rpb for g in groups))
        out["staged_then_global"] += int(any(staged[i] and not staged[j] for i in range(len(staged)) for j in range(i + 1, len(staged))))
        out["none_staged"] += int(len(staged) > 0 and not any(staged))
    out["group_lengths"] = sorted(lengths)
    causes = dict.fromkeys(BREAK_CAUSES, 0)
    for i in range(1, len(rows)):
        if i % rpb == 0:
            continue
        a, b = i - 1, i
        if not valid[a] or not valid[b]:
            causes["invalid"] += 1
        elif bpf[a] == 0 or bpf[b] == 0:
            causes["constant"] += 1
        elif kf1[a] < kf0[a] or kf1[b] < kf0[b]:
            causes["wrap"] += 1
        elif clip_index[a] != clip_index[b]:
            causes["clip"] += int(kf0[b] == kf1[a])        # the key frames chain: only the clip check keeps them apart
        elif kf0[b] < kf1[a]:
            causes["backward"] += 1
    out["breaks"] = causes
    return out


def pool_can_run_out_mid_block(rpb: int, kfb: int) -> bool:
    """False when no block can stage some groups and not a later one whatever the requests: a block of one request has one group,
    and a group of n requests stages at most (n + 1) * kfb + 47 bytes, so a block's groups stage at most rpb * (2 kfb + 47)."""
    return rpb > 1 and rpb * (2 * kfb + 47) > POOL_BYTES


def first_group_can_miss_pool(rpb: int, kfb: int) -> bool:
    """False when a block's first group always fits the pool: a chain of rpb requests stages at most (rpb + 1) * kfb + 47 bytes."""
    return (rpb + 1) * kfb + 47 > POOL_BYTES


# ---- vocabularies and request lists ----

def policy_pair(byte_pair: int) -> tuple[int, int]:
    """(rounding, looping) of a per request policy pair (rounding byte | looping byte << 8): values out of range read as none /
    as_compressed."""
    rounding, looping = byte_pair & 0xFF, byte_pair >> 8
    return (rounding if rounding <= port.ROUND_NEAREST else port.ROUND_NONE, looping if looping <= port.LOOP_AS_COMPRESSED else port.LOOP_AS_COMPRESSED)


def pair(rounding: int, looping: int) -> int:
    return rounding | (looping << 8)


OUT_OF_RANGE_PAIRS = [pair(4, 0), pair(200, 1), pair(1, 3), pair(255, 255), pair(3, 17)]


def vocabulary_times(blob: np.ndarray) -> np.ndarray:
    """The edge times of tests/edge_cases.py: every key frame and one ulp either side, both durations and their neighbours, the
    ties of a 32 Hz clip, -0.0, the smallest subnormal, +-inf, NaN and 1e30."""
    return edge_cases.edge_times(blob)


def _runs(blob: np.ndarray, rng, wrap: bool, count: int) -> list[np.ndarray]:
    """Playback runs of 1..40 requests one frame apart from every key frame at four fractions of a frame, runs past the end (clamped)
    or across it (wrapped), repeats of one time, reversed runs, and runs of the edge times."""
    rate, n = edge_cases.sample_rate(blob), edge_cases.num_samples(blob)
    end = np.float32((n - 1) / rate)
    fractions = (0.0, 0.25, 0.5, 0.999)
    runs, total, length, start = [], 0, 1, 0
    while total < count:
        fraction = fractions[(start // n) % 4]
        first = start % n
        kind = len(runs) % 9
        if kind == 7:
            t = (first + fraction) / rate if rng.integers(0, 2) else float(end) * (1 + rng.integers(1, 4))
            run = [t] * length
        else:
            run = []
            for k in range(first, first + length):
                if wrap:
                    run.append(((k % n) + fraction) / rate)
                else:
                    run.append((k + fraction) / rate if k < n else (float(end) if k == n else float(end) + (k - n) / rate))
            if kind == 8:
                run = run[::-1]
        runs.append(np.array(run, dtype=np.float32))
        total += length
        length = length % 40 + 1
        start += 7 if length == 1 else 1
    times = vocabulary_times(blob)
    for s in range(0, len(times), 5):
        runs.append(times[s:s + 5])
    return runs


def request_list(name: str, seed: int = 0, count: int = 1500):
    """Clip indices, times and policy pairs of a clip set's launch:
    - aligned blocks: a chain of every length L from rpb down to 1 starting a block, the rest of the block a chain of the twin clip;
    - pressure blocks: the widest clip played backwards, one group per request, so that the pool runs out within a block;
    - a run across the end of the first clip under the wrap policy, and one broken by a request of the all constant clip;
    - playback runs of every clip under one policy pair per run (a policy pair per request in some, out of range pairs among them),
      runs interleaved in random order, ABAB and AAAABBBB between the first clip and its twin, invalid clip indices inside runs;
    then a final partial block."""
    track_type, blobs = clip_set(name)
    rpb = plan(max(key_frame_bytes(b) for b in blobs))
    rng = np.random.default_rng(seed)
    recipes = CLIP_SETS[name][1]
    twin = recipes.index(TWIN257) if TWIN257 in recipes else 0
    base = recipes.index(C257) if C257 in recipes else 0
    widest = int(np.argmax([key_frame_bytes(b) for b in blobs]))
    clip_l, time_l, policy_l = [], [], []

    def add(c, times, policies):
        clip_l.append(np.full(len(times), c))
        time_l.append(np.asarray(times, dtype=np.float32))
        policy_l.append(np.broadcast_to(np.asarray(policies), (len(times),)))

    rate = 30.0
    for length in range(rpb, 0, -1):
        add(base, [(k + 0.5) / rate for k in range(length)], pair(0, 0))
        if rpb - length:
            add(twin, [(k + 0.25) / rate for k in range(length, rpb)], pair(0, 0))
    wide = blobs[widest]
    wide_n, wide_rate = edge_cases.num_samples(wide), edge_cases.sample_rate(wide)
    for _ in range(3):
        add(widest, [((wide_n - 2 - (k % max(wide_n - 1, 1))) % max(wide_n - 1, 1) + 0.5) / wide_rate for k in range(rpb)], pair(0, 0))
    # ABAB and AAAABBBB: requests of two clips with one frame layout, their key frames chaining across the clip change
    for block in (1, 4):
        times = [(k + 0.5) / rate for k in range(32)]
        for k, t in enumerate(times):
            add(base if (k // block) % 2 == 0 else twin, [t], pair(0, 0))
    n_base = edge_cases.num_samples(blobs[base])
    add(base, [(k % n_base + 0.5) / rate for k in range(n_base - 3, n_base + 3)], pair(0, port.LOOP_WRAP))
    constant = recipes.index(CONST)
    add(base, [0.5 / rate, 1.5 / rate], pair(0, 0))
    add(constant, [2.5 / rate], pair(0, 0))
    add(base, [2.5 / rate, 3.5 / rate], pair(0, 0))
    fixed = sum(len(x) for x in clip_l)
    runs = []
    for c, blob in enumerate(blobs):
        wrap = recipes[c][0] == "content" and recipes[c][4]
        for w in (False, True) if wrap else (False,):
            for r in _runs(blob, rng, w, count // len(blobs)):
                if rng.random() < 0.75:
                    looping = port.LOOP_WRAP if w else int(rng.choice([0, 2]))
                    policies = np.full(len(r), pair(int(rng.integers(0, 4)), looping))
                else:
                    choices = [pair(ro, lo) for ro in range(4) for lo in range(3)] + OUT_OF_RANGE_PAIRS
                    policies = np.array(choices)[rng.integers(0, len(choices), len(r))]
                runs.append((c, r, policies))
    for i in rng.permutation(len(runs)):
        c, r, policies = runs[i]
        add(c, r, policies)
    req_clip = np.concatenate(clip_l).astype(np.uint32)
    req_time = np.concatenate(time_l).astype(np.float32)
    req_policy = np.concatenate(policy_l).astype(np.int64)
    invalid = (rng.random(len(req_clip)) < 0.02) & (np.arange(len(req_clip)) >= fixed)
    req_clip = np.where(invalid, np.uint32(len(blobs) + 3), req_clip).astype(np.uint32)
    if rpb > 1 and len(req_clip) % rpb == 0:
        req_clip, req_time, req_policy = req_clip[:-1], req_time[:-1], req_policy[:-1]
    return req_clip, req_time, req_policy


# ---- the oracle ----

def track_policies(num_tracks: int) -> np.ndarray:
    """Rounding policy per track (none, floor, ceil, nearest) for the per track rounding decodes."""
    return (np.arange(num_tracks) * 7 // 3 % 4).astype(np.uint8)


# (per track rounding, rounding, looping) of the reference values tests/golden/make_scalar_cases_golden.py stores, at every fourth
# vocabulary time and the special times, for the constant tracks, the last one, every fifth of the first 300 and every 97th after
GOLDEN_COMBOS = [(False, port.ROUND_NONE, port.LOOP_AS_COMPRESSED), (False, port.ROUND_NEAREST, port.LOOP_CLAMP),
                 (True, port.ROUND_PER_TRACK, port.LOOP_WRAP)]


def golden_times(blob: np.ndarray) -> np.ndarray:
    return edge_cases.golden_times(blob)


def golden_tracks(blob: np.ndarray) -> np.ndarray:
    n = port.num_tracks_of(blob)
    return np.unique(np.array([t for t in CONSTANT_AT if t < n] + [n - 1] + list(range(0, min(n, 300), 5)) + list(range(300, n, 97)),
                               dtype=np.int64))


def nan_rule_equal(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Lane by lane: NaN where the oracle gives NaN (any payload: x86 and CUDA make different default NaNs), else the same bits."""
    g = np.ascontiguousarray(got, dtype=np.float32)
    w = np.ascontiguousarray(want, dtype=np.float32)
    return np.where(np.isnan(w), np.isnan(g), g.view(np.uint32) == w.view(np.uint32))


class Oracle:
    """The port's decode of every (clip, time, policy pair) a launch asks for, cached."""

    def __init__(self, blobs, track_type: int, per_track_policies: np.ndarray | None = None):
        self.blobs, self.nc = blobs, components(track_type)
        self.settings = port.SettingsBuilder(per_track_rounding=per_track_policies is not None, per_track_policies=per_track_policies)
        self.cache = {}

    def row(self, c: int, t: np.float32, rounding: int, looping: int) -> np.ndarray:
        key = (c, int(np.float32(t).view(np.uint32)), rounding, looping)
        if key not in self.cache:
            self.cache[key] = port.scalar_decompress(self.blobs[c], self.settings, float(t), rounding, looping)[:, :self.nc].copy()
        return self.cache[key]
