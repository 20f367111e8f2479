"""Fixtures of the compression error tests at every skeleton shape, launch size, tie and NaN (tests/test_gpu_error_shapes.py).

Everything is built from the committed clips and the port alone: the lossy poses are the port's decode of a clip at the times
calculate_compression_error seeks, and the raw poses are those plus seeded perturbations, so no reference is needed. The expected
result of a job is the port's IEEE flavour (port.transform_track_error, port.scalar_track_error), which
tests/test_error_metric_oracle.py pins to the reference bit for bit. The port walks bone by bone whatever the skeleton's shape; a
parent at or after its child, which it refuses, is made a root (what the device walk does, and flags ERROR_FLAG_INVALID_SKELETON)."""
from __future__ import annotations

import dataclasses
import functools

import numpy as np

from tests import bones_cases, clips

ROOT = 0xFFFFFFFF
NO_OUTPUT = 0xFFFFFFFF
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)
METRIC_QVVF, METRIC_MATRIX = 0, 1
ROUND_NONE, ROUND_NEAREST = 0, 3
FLAG_NEGATIVE_SCALE, FLAG_INVALID_SKELETON = 1, 2
NO_INDEX = 0xFFFFFFFF

# floats of a bone in a warp's object transform planes (error_metric.cu): the measurement keeps two streams (raw, lossy) of qvvf or of
# 3x4 matrices, local_to_object_space one stream of qvvf
PLANE_FLOATS = {METRIC_QVVF: 2 * 10, METRIC_MATRIX: 2 * 12}
LOCAL_TO_OBJECT_FLOATS = 10


def plane_stride(num_tracks: int) -> int:
    return (max(num_tracks, 1) + 31) & ~31


def warps_for(widest_tracks: int, floats_per_bone: int, max_dynamic_smem: int) -> int:
    """error_metric.cu's warps_for: warps per block of the object space kernel, set by the widest job of the call"""
    per_warp = floats_per_bone * plane_stride(widest_tracks) * 4
    if per_warp > max_dynamic_smem:
        return 0
    return min(8, max(per_warp, min(max_dynamic_smem, 100 * 1024)) // per_warp)


def poses_per_sweep(widest_tracks: int, floats_per_bone: int, num_sms: int, max_dynamic_smem: int) -> int:
    """Poses one pass of the grid-strided object space kernel covers: at most num_sms * 32 blocks of warps_for warps, one pose per warp"""
    return num_sms * 32 * warps_for(widest_tracks, floats_per_bone, max_dynamic_smem)


def rounding_of(blob) -> int:
    """The rounding calculate_compression_error seeks a clip with: none when it has stripped key frames, else nearest"""
    misc = int(np.asarray(blob[28:32]).view(np.uint32)[0])
    return ROUND_NONE if (misc >> 10) & 1 else ROUND_NEAREST


def clip_duration(name: str, sample_rate: float | None = None) -> float:
    spec = clips.TRANSFORM_SPECS[name]
    rate = np.float32(spec.sample_rate if sample_rate is None else sample_rate)
    return float(np.float32(max(spec.num_samples - 1, 0)) / rate)


@functools.lru_cache(maxsize=None)
def _decoded(name: str, num_samples: int, sample_rate: float, duration: float) -> np.ndarray:
    from tests.test_error_metric_oracle import lossy_poses_from_port
    blob = clips.load_blob(name)
    out = lossy_poses_from_port(blob, 1, num_samples, sample_rate, duration, rounding_of(blob))
    out.setflags(write=False)
    return out


def decoded(name: str, num_samples: int | None = None, sample_rate: float | None = None, duration: float | None = None) -> np.ndarray:
    """[num_samples][clip tracks][12]: what the device decodes for a job of the clip, sample s at min(s / sample_rate, duration), with the
    bind pose as defaults (the port's decode, pinned to the reference)"""
    spec = clips.TRANSFORM_SPECS[name]
    rate = float(spec.sample_rate if sample_rate is None else sample_rate)
    return _decoded(name, spec.num_samples if num_samples is None else num_samples, rate,
                    clip_duration(name, rate) if duration is None else float(duration))


def perturb(poses: np.ndarray, rng, amount: float) -> np.ndarray:
    """Raw poses near `poses`: rotations turned and renormalised, translations moved by ~amount, scales by ~amount / 10 (signs kept)"""
    out = np.array(poses, np.float32, copy=True)
    shape = out.shape[:-1]
    rotation = out[..., 0:4] + rng.normal(0.0, amount, shape + (4,)).astype(np.float32)
    out[..., 0:4] = rotation / np.linalg.norm(rotation, axis=-1, keepdims=True).astype(np.float32)
    out[..., 4:7] += rng.normal(0.0, amount, shape + (3,)).astype(np.float32)
    out[..., 8:11] *= (1.0 + rng.normal(0.0, amount / 10, shape + (3,))).astype(np.float32)
    return out


def shells(num_tracks: int, rng) -> np.ndarray:
    return rng.uniform(0.5, 4.0, num_tracks).astype(np.float32)


def invalid_order(parents) -> bool:
    parents = np.asarray(parents, np.uint64)
    return bool(np.any((parents != ROOT) & (parents >= np.arange(parents.size, dtype=np.uint64))))


@dataclasses.dataclass
class Job:
    """One aclb200_error_job with everything the port needs to say what it must give"""
    clip: int                       # index in the clip set
    raw: np.ndarray                 # [num_samples][num_tracks][12]
    lossy: np.ndarray               # [num_samples][num_tracks][12] the decoded poses seen through output_indices
    sample_rate: float
    duration: float
    parents: np.ndarray             # as handed to the device (may hold late parents)
    shells: np.ndarray
    output_indices: np.ndarray | None = None
    base: np.ndarray | None = None  # [num_samples][num_tracks][12] additive base
    additive_format: int = 0
    metric: int = METRIC_QVVF

    @property
    def num_samples(self) -> int:
        return self.raw.shape[0]

    @property
    def num_tracks(self) -> int:
        return self.raw.shape[1]

    def expected(self, port):
        """(index, error, sample_time, flags, errors [num_samples][num_tracks]) of the port"""
        result, errors, negative = port.transform_track_error(self.raw, self.lossy, self.sample_rate, self.duration,
                                                              bones_cases.effective_parents(self.parents), self.shells, port.NORMALIZE_IEEE,
                                                              self.base, self.additive_format, self.metric)
        flags = (FLAG_NEGATIVE_SCALE if negative else 0) | (FLAG_INVALID_SKELETON if invalid_order(self.parents) else 0)
        return int(result.index), np.float32(result.error), np.float32(result.sample_time), flags, errors


def clip_job(name: str, clip: int, parents, rng, metric=METRIC_QVVF, amount=0.02, **kw) -> Job:
    """A job of a whole clip: raw = the clip's decoded poses, perturbed"""
    lossy = decoded(name)
    return Job(clip=clip, raw=perturb(lossy, rng, amount), lossy=np.array(lossy), sample_rate=float(clips.TRANSFORM_SPECS[name].sample_rate),
               duration=clip_duration(name), parents=np.asarray(parents, np.uint32), shells=shells(lossy.shape[1], rng), metric=metric, **kw)


def permuted_job(name: str, clip: int, rng, metric=METRIC_QVVF) -> Job:
    """Raw track i is decoded track perm[i] (a permutation through output_indices), perturbed"""
    lossy = decoded(name)
    n = lossy.shape[1]
    output_indices = rng.permutation(n).astype(np.uint32)
    raw = perturb(lossy[:, output_indices], rng, 0.02)
    return Job(clip=clip, raw=raw, lossy=remapped(lossy, raw, output_indices), sample_rate=float(clips.TRANSFORM_SPECS[name].sample_rate),
               duration=clip_duration(name), parents=bones_cases.skeleton("random", n, 7), shells=shells(n, rng), output_indices=output_indices,
               metric=metric)


def remapped(decoded_poses: np.ndarray, raw: np.ndarray, output_indices) -> np.ndarray:
    """remap_output (track_error.impl.h:522-532): raw track i is compared with decoded output_indices[i], or with itself when stripped"""
    out = np.array(raw, np.float32, copy=True)
    for track, output in enumerate(np.asarray(output_indices, np.uint64)):
        if output != NO_OUTPUT:
            out[:, track] = decoded_poses[:, int(output)]
    return out


def mirrored_chain_job(name: str, clip: int, rng, metric=METRIC_QVVF) -> Job:
    """A chain through every bone (so through every 32 bone chunk) with mirrored raw bones: their children take rtm::qvv_mul's matrix
    branch in the raw stream only; bones the clip does not output (raw value compared with itself) are mirrored in both streams."""
    lossy = decoded(name)
    n = lossy.shape[1]
    raw = perturb(lossy, rng, 0.02)
    mirrored = [3, 31, 32, 47, 64, n - 2]
    raw[:, mirrored, 8] *= -1.0
    output_indices = np.arange(n, dtype=np.uint32)
    output_indices[[31, 64]] = NO_OUTPUT
    return Job(clip=clip, raw=raw, lossy=remapped(lossy, raw, output_indices), sample_rate=float(clips.TRANSFORM_SPECS[name].sample_rate),
               duration=clip_duration(name), parents=bones_cases.skeleton("chain", n), shells=shells(n, rng), output_indices=output_indices,
               metric=metric)


def additive_job(name: str, clip: int, parents, additive_format: int, rng) -> Job:
    """The clip's poses as the additive layer over a base made of the same poses one sample on, perturbed. The decoded poses are the
    clip's whatever the format (additive1 doubles their scales near 1)."""
    job = clip_job(name, clip, parents, rng)
    job.base, job.additive_format = perturb(np.roll(decoded(name), 1, axis=0), rng, 0.05), additive_format
    return job


def strided_sweep_jobs(name: str, clip: int, num_jobs: int, metric: int, seed: int, amount: float = 0.005) -> list:
    """num_jobs jobs of one clip and skeleton, each with a perturbation of its own and one bone of one sample moved further: every job has
    its own worst track, so a pose measured for the wrong job, or a job slot's arg max mixed with another, changes a result"""
    rng = np.random.default_rng(seed)
    lossy = np.array(decoded(name))
    s, n = lossy.shape[:2]
    parents = bones_cases.skeleton("random", n, seed)
    shell = shells(n, rng)
    rate, duration = float(clips.TRANSFORM_SPECS[name].sample_rate), clip_duration(name)
    jobs = []
    for _ in range(num_jobs):
        raw = perturb(lossy, rng, amount)
        raw[int(rng.integers(0, s)), int(rng.integers(0, n)), 4:7] += rng.uniform(10 * amount, 100 * amount, 3).astype(np.float32)
        jobs.append(Job(clip=clip, raw=raw, lossy=lossy, sample_rate=rate, duration=duration, parents=parents, shells=shell, metric=metric))
    return jobs


# ---- exact ties ----------------------------------------------------------------------------------------------------------------------
TIE_BONES = [37, 40, 70, 99]         # chunks 1, 1, 2, 3 at lanes 5, 8, 6, 3: raw tracks aliased onto decoded track 37
TIE_PARENT = 3
TIE_DURATION_SAMPLES = 45            # duration = 45 / 30 s: samples 45 .. 59 are all sought at the duration


def tie_job(name: str, clip: int, metric: int, seed: int = 5) -> Job:
    """Exact non-zero ties, in (sample, bone) order first at (TIE_DURATION_SAMPLES, TIE_BONES[0]):
      * bones: the TIE_BONES raw tracks share a parent, a raw transform, a shell distance and (through output_indices) a decoded track,
        and have no children: their errors are equal in every sample;
      * samples: every sample from TIE_DURATION_SAMPLES on is sought at the duration (same decoded pose) and has the same raw pose.
    Those bones carry a large error from that sample on and a small one before; every other bone a small one."""
    rng = np.random.default_rng(seed)
    spec = clips.TRANSFORM_SPECS[name]
    rate = float(spec.sample_rate)
    duration = float(np.float32(TIE_DURATION_SAMPLES) / np.float32(rate))
    lossy = decoded(name, spec.num_samples, rate, duration)
    s, n = lossy.shape[:2]
    parents = bones_cases.skeleton("random", n, seed)
    for bone in range(n):
        if parents[bone] in TIE_BONES or bone in TIE_BONES:
            parents[bone] = TIE_PARENT if bone > TIE_PARENT else ROOT
    output_indices = np.arange(n, dtype=np.uint32)
    output_indices[TIE_BONES] = TIE_BONES[0]
    raw = perturb(lossy, rng, 0.001)
    raw[:, TIE_BONES] = raw[:, TIE_BONES[0]][:, None]
    raw[TIE_DURATION_SAMPLES:, TIE_BONES[0], 4:7] += np.float32(0.75)
    raw[TIE_DURATION_SAMPLES:, TIE_BONES] = raw[TIE_DURATION_SAMPLES:, TIE_BONES[0]][:, None]
    raw[TIE_DURATION_SAMPLES + 1:] = raw[TIE_DURATION_SAMPLES]
    shell = shells(n, rng)
    shell[TIE_BONES] = 2.5
    return Job(clip=clip, raw=raw, lossy=remapped(lossy, raw, output_indices), sample_rate=rate, duration=duration, parents=parents,
               shells=shell, output_indices=output_indices, metric=metric)


def tie_positions(num_samples: int):
    """(sample, bone) of every error equal to the tie job's largest"""
    return {(sample, bone) for sample in range(TIE_DURATION_SAMPLES, num_samples) for bone in TIE_BONES}


def unchanged_job(name: str, clip: int, metric: int, seed: int = 6) -> Job:
    """raw == decoded: every error is +0, the first (sample 0, bone 0) is the worst"""
    rng = np.random.default_rng(seed)
    lossy = decoded(name)
    n = lossy.shape[1]
    return Job(clip=clip, raw=np.array(lossy), lossy=np.array(lossy), sample_rate=float(clips.TRANSFORM_SPECS[name].sample_rate),
               duration=clip_duration(name), parents=bones_cases.skeleton("random", n, seed), shells=shells(n, rng), metric=metric)


# ---- NaN in raw poses ----------------------------------------------------------------------------------------------------------------
NAN_BONE_SAMPLE, NAN_BONE = 7, 5     # bone 5 of sample 7: its rotation
NAN_SAMPLE = 20                      # every bone of sample 20: the root's translation


def nan_jobs(name: str, clip: int, metric: int, seed: int = 8) -> list:
    """Three jobs of the clip on a tree: NaN in one bone's rotation (it and its descendants measure NaN in that sample), in the root
    translation of one sample (the whole sample), and in every raw pose (no error is ever kept: index NO_INDEX, error -1)"""
    n = decoded(name).shape[1]
    jobs = [clip_job(name, clip, bones_cases.tree(n), np.random.default_rng(seed + i), metric) for i in range(3)]
    jobs[0].raw[NAN_BONE_SAMPLE, NAN_BONE, 1] = np.nan
    jobs[1].raw[NAN_SAMPLE, 0, 5] = np.nan
    jobs[2].raw[:, :, 0] = np.nan
    return jobs


def descendants(parents, bone: int) -> set:
    out = {bone}
    for child in range(bone + 1, len(parents)):
        if int(parents[child]) in out:
            out.add(child)
    return out


def scalar_values(name: str, rng, amount: float = 0.01):
    """(raw, decoded) [num_samples][num_tracks][4] of a scalar clip, raw = decoded perturbed, sampled like calculate_compression_error
    (nearest, at min(s / sample_rate, duration)); plus sample_rate and duration"""
    from tests.test_error_metric_oracle import lossy_scalar_from_port
    spec = clips.SCALAR_SPECS[name]
    rate = float(spec.sample_rate)
    duration = float(np.float32(max(spec.num_samples - 1, 0)) / np.float32(rate))
    lossy = lossy_scalar_from_port(clips.load_blob(name), spec.num_samples, rate, duration, ROUND_NEAREST)
    raw = (lossy + rng.normal(0.0, amount, lossy.shape)).astype(np.float32)
    return raw, lossy, rate, duration


# ---- the device call's inputs --------------------------------------------------------------------------------------------------------
def pack(jobs, job_dtype, max_tracks: int, pose_floats: int | None = None, zero_sample_jobs=()):
    """The buffers of one calculate_compression_error call for `jobs` (plus jobs without samples, zero_sample_jobs = {slot: (clip,
    num_tracks)}, inserted at those slots). pose_floats: floats per raw / base pose row (default max_tracks * 12; more pads every row with NaN). Each job's
    raw poses and skeleton start behind a gap. Returns dict(jobs=table, raw, base or None, parents, shells, output_indices or None,
    slots=[slot of each of `jobs`], rows=[first error matrix row of each of `jobs`])."""
    pose_floats = max_tracks * 12 if pose_floats is None else pose_floats
    skeleton_gap, pose_gap = 3, 2
    total_poses = sum(j.num_samples + pose_gap for j in jobs) + pose_gap
    raw = np.full((total_poses, pose_floats), np.nan, np.float32)
    base = np.full_like(raw, np.nan) if any(j.base is not None for j in jobs) else None
    parents, shell, outputs = [np.full(skeleton_gap, 7, np.uint32)], [np.full(skeleton_gap, np.nan, np.float32)], [np.full(skeleton_gap, 7, np.uint32)]
    remap = any(j.output_indices is not None for j in jobs)
    extra = dict(zero_sample_jobs)
    table = np.zeros(len(jobs) + len(extra), job_dtype)
    slots, rows = [], []
    pose, skeleton, row, it = pose_gap, skeleton_gap, 0, iter(jobs)
    for slot in range(len(table)):
        if slot in extra:
            e = table[slot]
            e["clip"], e["num_tracks"] = extra[slot]
            e["num_samples"], e["sample_rate"], e["duration"] = 0, 30.0, 1.0
            continue
        j = next(it)
        raw[pose:pose + j.num_samples, :j.num_tracks * 12] = j.raw.reshape(j.num_samples, -1)
        if j.base is not None:
            base[pose:pose + j.num_samples, :j.num_tracks * 12] = j.base.reshape(j.num_samples, -1)
        parents.append(j.parents)
        shell.append(j.shells)
        outputs.append(j.output_indices if j.output_indices is not None else np.arange(j.num_tracks, dtype=np.uint32))
        e = table[slot]
        e["clip"], e["num_samples"], e["sample_rate"], e["duration"] = j.clip, j.num_samples, j.sample_rate, j.duration
        e["num_tracks"], e["skeleton_offset"], e["first_raw_pose"] = j.num_tracks, skeleton, pose
        e["additive_format"], e["error_metric"], e["first_base_pose"] = j.additive_format, j.metric, pose
        slots.append(slot)
        rows.append(row)
        pose += j.num_samples + pose_gap
        skeleton += j.num_tracks + skeleton_gap
        row += j.num_samples
        parents.append(np.full(skeleton_gap, 7, np.uint32))
        shell.append(np.full(skeleton_gap, np.nan, np.float32))
        outputs.append(np.full(skeleton_gap, 7, np.uint32))
    return dict(jobs=table, raw=raw, base=base, parents=np.concatenate(parents), shells=np.concatenate(shell),
                output_indices=np.concatenate(outputs) if remap else None, slots=slots, rows=rows, total_rows=row)
