"""Clips and request lists for the pipeline kernel tests (tests/test_gpu_pipeline.py, tests/test_pipeline_requests.py,
tests/golden/make_pipeline_golden.py).

The two clips here are sized for batch shapes the clips of tests/clips.py do not reach. They stay out of clips.TRANSFORM_SPECS so
that the tests parametrized over that dict do not grow.

Request lists are index sequences into a per-clip vocabulary of sample times, so that the oracle runs once per (clip, time, policy)
and the expected output of a whole launch is a gather.
"""
from __future__ import annotations

import numpy as np

from oracle import ref
from tests import clips

T = ref.TransformSpec

PIPELINE_SPECS: dict[str, ref.TransformSpec] = {
    # about 200 bones: 3 to 8 requests per batch, several batches per seek pass; many segments, stripped key frames, a wrap loop,
    # raw (noisy) and animated scale tracks. The reference compresses most seeds of this recipe to slightly different blobs on different
    # x86 CPUs (as it does mixed_scale, noisy_raw and paragon_like); this seed gives the same bytes on every CPU it was tried on, so
    # the blob can be regenerated and compared anywhere
    "seg_200": T(num_tracks=200, num_samples=130, seed=41,rot_constant_pct=55, trans_constant_pct=85, scale_default_pct=80,
                 scale_constant_pct=5, noisy_pct=4, partial_activity_pct=20, looping_content=1, strip_proportion=0.25),
    # about 2500 bones, few samples, mostly constant tracks: one request per batch and one block per SM in QVV40, a pose too large for
    # shared memory in QVV48 (the plain kernels then serve the launch)
    "wide_2500": T(num_tracks=2500, num_samples=9, seed=32, rot_constant_pct=96, trans_constant_pct=98, scale_default_pct=100),
}

# the times at which tests/golden/make_pipeline_golden.py stores the reference's poses, and the bones it keeps (every fifth of the
# wide clip: its constant bones cost as much to store as its animated ones)
GOLDEN_TIMES = {"seg_200": [-0.1, 0.0, 0.51, 1.0, 2.345, 4.3], "wide_2500": [0.05, 0.1333, 0.27]}
GOLDEN_COMBOS = [(0, 0), (1, 3), (3, 1)]        # (settings kind, rounding policy)


def golden_bones(name: str) -> np.ndarray:
    n = PIPELINE_SPECS[name].num_tracks
    return np.arange(n) if n <= 256 else np.unique(np.concatenate([np.arange(0, n, 5), [n - 1]]))

K_GROUP_MAX = 5         # pipeline.cu: k_group_max, the longest group one consumer thread walks


def load_blob(name: str) -> np.ndarray:
    return clips.load_blob(name)


def spec_of(name: str) -> ref.TransformSpec:
    return PIPELINE_SPECS[name] if name in PIPELINE_SPECS else clips.TRANSFORM_SPECS[name]


def num_animated(blob: np.ndarray) -> int:
    """Animated sub-tracks of a clip (the pipeline groups nothing for a clip without any)."""
    header = blob[32:84].view(np.uint32)
    has_scale = int(blob[28:32].view(np.uint32)[0]) & 1
    return int(header[2]) + int(header[3]) + (int(header[4]) if has_scale else 0)


FRACTIONS = (0.0, 0.25, 0.5, 0.999)
POLICY_PAIRS = [(r, l) for r in range(4) for l in range(3)]     # (rounding, looping) pairs a request may carry
LOOP_WRAP = 1


def playback_lists(spec, rng, count: int, wrap: bool) -> list[np.ndarray]:
    """Sequential playback runs of one clip as lists of times: runs of 1..12 requests one frame apart (request i + 1 starts on the key
    frame request i ends on), starting at every frame and every fraction of a frame. Clamped runs that pass the end continue with times
    past it (every one of them seeks kf0 == kf1 == the last frame); wrapped runs (`wrap`) go on from frame 0. Some runs are repeated
    requests of one time, some are played backwards."""
    rate = np.float64(spec.sample_rate)
    n = spec.num_samples
    duration = max(n - 1, 0) / rate
    past_end = [duration + 0.25 / rate, duration * 2.0, duration * 3.0 + 0.3 / rate, duration * 7.5 + 1.0]
    runs, total, length, start = [], 0, 1, 0
    while total < count:
        fraction = FRACTIONS[(start // max(n, 1)) % len(FRACTIONS)]
        first = start % max(n, 1)
        kind = len(runs) % 9
        if kind == 7:           # one time repeated
            t = (first + fraction) / rate if rng.integers(0, 2) else past_end[int(rng.integers(0, len(past_end)))]
            run = [t] * length
        else:
            frames = [first + j for j in range(length)]
            if wrap:
                run = [((k % n) + fraction) / rate for k in frames]
            else:
                run = [(k + fraction) / rate if k < n else past_end[min(k - n, len(past_end) - 1)] for k in frames]
            if kind == 8:       # reversed playback
                run = run[::-1]
        runs.append(np.array(run, dtype=np.float32))
        total += length
        length = length % 12 + 1
        start += 7 if length == 1 else 1
    return runs


def seek_rows(port, blobs, settings, req_clip, req_time, req_policy) -> np.ndarray:
    """The seek the pipeline's grouping reads, per request: valid, clip, segment of key frame 0 and 1, key frame bit offsets, single
    segment flag, whether the clip has animated sub-tracks."""
    rows = np.zeros((len(req_clip), 8), dtype=np.int64)
    cache = {}
    animated = [num_animated(b) for b in blobs]
    for i, (c, t, p) in enumerate(zip(req_clip.tolist(), req_time.tolist(), req_policy.tolist())):
        if c >= len(blobs):
            continue
        key = (c, t, p)
        if key not in cache:
            rounding, looping = POLICY_PAIRS[p]
            st = port.transform_seek(blobs[c], settings, t, rounding, looping)
            cache[key] = (1, c, st.segment_indices[0], st.segment_indices[1], st.key_frame_bit_offsets[0], st.key_frame_bit_offsets[1],
                          st.uses_single_segment, int(animated[c] != 0))
        rows[i] = cache[key]
    return rows


def pair_stats(rows: np.ndarray) -> dict:
    """What a request list offers the grouping, whatever the batch size: consecutive pairs that chain, crossings, wraps, repeats."""
    valid, clip, seg0, seg1, kf0, kf1, single, animated = rows.T
    mergeable = (valid == 1) & (animated == 1) & (single == 1) & (kf1 >= kf0)
    crossing = (valid == 1) & (animated == 1) & (single == 0)
    same_table = (clip[1:] == clip[:-1]) & (seg0[1:] == seg0[:-1])
    chains = mergeable[:-1] & same_table & (kf0[1:] == kf1[:-1])
    joins_mergeable = chains & mergeable[1:]
    joins_crossing = chains & crossing[1:]
    run, longest, lengths = 1, 1, np.zeros(13, dtype=np.int64)
    for j in joins_mergeable:
        run = run + 1 if j else 1
        longest = max(longest, run)
        if run <= 12:
            lengths[run] += 1
    repeats = (valid[1:] == 1) & (clip[1:] == clip[:-1]) & (seg0[1:] == seg0[:-1]) & (kf0[1:] == kf0[:-1]) & (kf1[1:] == kf1[:-1])
    return dict(chained_pairs=int(joins_mergeable.sum()), chain_then_crossing=int(joins_crossing.sum()), crossings=int(crossing.sum()),
                wrapped_single=int(((valid == 1) & (single == 1) & (kf1 < kf0)).sum()),
                wraps_into_segment_0=int((crossing & (seg1 == 0) & (seg0 > 0)).sum()),
                chained_wrap_crossings=int((joins_crossing & (seg1[1:] == 0)).sum()),
                repeats=int(repeats.sum()), clamped_repeats=int((repeats & (kf0[1:] == kf1[1:])).sum()),
                invalid=int((valid == 0).sum()), longest_run=int(longest), runs_reaching=lengths.tolist())


def groups(rows: np.ndarray, rpb: int, grouped: bool = True) -> dict:
    """The groups the seek warp forms (pipeline.cu, produce_pass), batch by batch: request i joins request i - 1 of the same batch when
    i - 1 reads one segment, both read the same segment of the same clip and i starts on the key frame i - 1 ends on; runs are cut every
    K_GROUP_MAX requests (k_group_max); a request whose key frames sit in two segments can only end a chain (a tail crossing)."""
    valid, clip, seg0, seg1, kf0, kf1, single, animated = rows.T
    mergeable = (valid == 1) & (animated == 1) & (single == 1) & (kf1 >= kf0)
    crossing = (valid == 1) & (animated == 1) & (single == 0)
    has_table = mergeable | crossing
    n = len(rows)
    lane = np.arange(n) % rpb
    join = np.zeros(n, dtype=bool)
    join[1:] = grouped & (lane[1:] > 0) & has_table[1:] & mergeable[:-1] & (clip[1:] == clip[:-1]) & (seg0[1:] == seg0[:-1]) \
        & (kf0[1:] == kf1[:-1])
    head = np.ones(n, dtype=bool)
    cuts = 0
    run_start = 0
    for i in range(n):
        if not join[i]:
            run_start = i
        elif (i - run_start) % K_GROUP_MAX == 0:
            cuts += 1
        else:
            head[i] = False
    starts = np.nonzero(head)[0]
    sizes = np.diff(np.append(starts, n))
    tail = crossing & ~head
    last = (starts + sizes - 1)
    stats = dict(groups=len(starts), cuts=cuts, tail_crossings=int(tail.sum()),
                 tail_crossings_at_last_lane=int((tail & (lane == rpb - 1)).sum()),
                 tail_crossings_into_segment_0=int((tail & (seg1 == 0) & (seg0 > 0)).sum()),
                 crossings_at_lane_0=int((crossing & (lane == 0)).sum()),
                 chained_clamped_repeats=int((~head & (kf0 == kf1) & (valid == 1)).sum()))
    for length in range(1, K_GROUP_MAX + 1):
        stats[f"groups_of_{length}"] = int(((sizes == length) & valid[starts].astype(bool)).sum())
    stats["chains_with_tail"] = int(tail[last].sum())
    return stats


def request_list(names, wrap_names, count, seed):
    """clip indices, times and policy pair indices of `count` requests: per clip playback runs (under the clip's own policy pairs,
    wrapped for the clips of `wrap_names`), then those runs interleaved request by request and in blocks of four between clips, with
    invalid clip indices inside runs."""
    rng = np.random.default_rng(seed)
    specs = [spec_of(n) for n in names]
    per_clip = max(count // len(names), 16)
    runs = []       # (clip, times, policy pair) per run
    for c, spec in enumerate(specs):
        wrap = names[c] in wrap_names
        for r in playback_lists(spec, rng, per_clip, wrap):
            if rng.random() < 0.75:     # one policy for a whole run (its requests still chain), else a policy per request
                rounding = 0 if rng.random() < 0.5 else int(rng.integers(0, 4))
                looping = LOOP_WRAP if wrap else int(rng.choice([0, 2]))
                policy = np.full(len(r), rounding * 3 + looping)
            else:
                policy = rng.integers(0, 12, len(r))
            runs.append((np.full(len(r), c), r, policy))
    order = rng.permutation(len(runs))
    clip = np.concatenate([runs[i][0] for i in order])
    time = np.concatenate([runs[i][1] for i in order])
    policy = np.concatenate([runs[i][2] for i in order])
    if len(names) > 1:
        # ABAB and AAAABBBB: consecutive requests of different clips, so that base row tags both hit and miss
        half = len(clip) // 2
        for block in (1, 4):
            lo = half if block == 1 else half + half // 2
            span = min(len(clip) - lo, 2048)
            sel = np.arange(lo, lo + span)
            key = (sel - lo) // block % 2
            other = (clip[sel] + 1) % len(names)
            clip[sel] = np.where(key == 1, other, clip[sel])
    invalid = rng.random(len(clip)) < 0.02
    clip = np.where(invalid, len(names) + 3, clip)
    clip, time, policy = (np.resize(x, count) for x in (clip, time, policy))
    return clip.astype(np.uint32), time.astype(np.float32), policy.astype(np.int64)
