"""Shared cases of the root motion tests (aclb200_extract_root_motion): settings kinds per clip, playback time pairs and the port's
samples and composition."""
from __future__ import annotations

import numpy as np

from tests import clips

CYCLES = list(range(-3, 4))
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 1, 0], np.float32)


def kinds_for(spec) -> list[int]:
    """The settings kinds (oracle.port.settings_for_kind) whose decompression settings accept the clip's formats"""
    from oracle import ref
    is_full = spec.rotation_format == ref.QUATF_FULL
    default_ok = spec.rotation_format == ref.QUATF_DROP_W_VARIABLE and spec.translation_format == ref.VECTOR3F_VARIABLE \
        and spec.scale_format == ref.VECTOR3F_VARIABLE
    return [1, 3, 4] + ([0, 2] if default_ok else []) + ([5] if is_full else [])


def clamp_duration(port, blob, settings) -> float:
    """D, the clip's clamp duration (num_samples - 1) / sample_rate in float, as the port's seek computes it"""
    return float(port.transform_seek(blob, settings, 1.0e9, looping=port.LOOP_CLAMP).clip_duration)


def time_pairs(spec, duration: float) -> list[tuple[float, float]]:
    """(from, to) playback times: steps forward and backward inside the clip, at 0 and D, beyond both ends, on key frames and equal"""
    times = [float(t) for t in clips.sample_times(spec)]
    pairs = [(times[i], times[i + 1]) for i in range(len(times) - 1)]
    pairs += [(b, a) for a, b in pairs[::3]]
    pairs += [(0.0, duration), (duration, 0.0), (0.0, 0.0), (duration, duration), (times[3], times[3]), (-0.5, duration + 0.5),
              (duration + 0.25, -0.25)]
    return [(float(np.float32(a)), float(np.float32(b))) for a, b in pairs]


def port_samples(port, blob, settings, rounding: int, root: int, from_time: float, to_time: float, duration: float) -> np.ndarray:
    """[4][12] T(from), T(to), T(D), T(0): the port's decompress_tracks root rows with the clamp policy"""
    return np.stack([port.transform_decompress_tracks(blob, settings, t, rounding, port.LOOP_CLAMP)[root]
                     for t in (from_time, to_time, duration, 0.0)])
