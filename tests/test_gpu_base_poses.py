"""The pipeline kernel's cached base pose rows (acquire_base_poses in acl_b200/csrc/pipeline.cu): the constant and default sub-tracks
of every clip, laid out once per (output layout, normalisation, default modes, constant default values) and copied into each pose
before its animated sub-tracks are decoded. A clip set keeps a handful of these variants and evicts the least recently used one.

Every launch here is asserted through Context.debug_last_launch() to take the pipeline kernel, and every pose is compared bit for bit
with oracle/port under the launch's own settings (fast math: rotations within 1e-5). A key that left out a field, a variant served
stale or before its build finished, or phase A run without the right normalisation shows as a wrong row:

* mixed_scale has 3 constant rotations whose NORMALIZE_ALWAYS copy differs in bits, 20 rows that change with the constant default
  values and 26 that change between the LEGACY and CONSTANT scale defaults; in the ragged set all 16 rows of all_default are
  defaults and one_sample has a constant rotation that NORMALIZE_ALWAYS changes.
* The key sweep walks eight distinct keys so that each is a miss, a hit, evicted and rebuilt with the cache's four variants, and
  decodes in between settings whose rows are those of one of the keys (NORMALIZE_NEVER / LERP_ONLY, fast / exact math, per track /
  plain rounding). Their output is checked; whether they hit their key's entry or built one of their own is not observable from
  here, since nothing exposes the cache's entries.
"""
import dataclasses

import numpy as np
import pytest

import acl_b200 as ab
from tests import clips

pytestmark = pytest.mark.gpu

LANES = clips.DEFINED_LANES
FAST_MATH_TOLERANCE = 1e-5
SENTINEL = np.uint32(0x7FBADBAD)        # a NaN no decode produces

CLIP_SETS = {
    "mixed_scale": ["mixed_scale"],
    "ragged": ["c1_30bones", "all_default", "one_sample", "ragged_17"],
}

C, V, L = ab.DEFAULT_CONSTANT, ab.DEFAULT_VARIABLE, ab.DEFAULT_LEGACY
# constant default values: rotation xyzw, translation xyz_, scale xyz_ (a scale that is not 1, so LEGACY and CONSTANT scales differ)
DEFAULTS_A = (0.1, -0.2, 0.3, 0.9, 1.5, -2.5, 3.25, 0.0, 0.5, 2.0, 1.25, 0.0)
DEFAULTS_B = (-0.3, 0.4, 0.1, 0.85, -4.0, 0.75, 1.5, 0.0, 1.75, 0.25, 3.0, 0.0)


@dataclasses.dataclass(frozen=True)
class Variant:
    layout: int
    normalization: int
    modes: tuple
    defaults: tuple
    math: int = ab.MATH_EXACT
    per_track: bool = False
    variable: bool = False      # pass a device array of variable default values (the kernel's own phase A serves them)


# Distinct keys: both layouts, LERP_ONLY and ALWAYS, four default mode triples (VARIABLE without a defaults pointer is cached like
# CONSTANT), two sets of constant default values under the same modes. The pairs 0/1 (default modes), 1/2 (normalisation), 2/3
# (constant defaults), 4/5 and 6/7 (normalisation) differ in one field of the key.
KEYS = [
    Variant(ab.LAYOUT_QVV48, ab.NORMALIZE_LERP_ONLY, (C, C, L), DEFAULTS_A),
    Variant(ab.LAYOUT_QVV48, ab.NORMALIZE_LERP_ONLY, (C, C, C), DEFAULTS_A),
    Variant(ab.LAYOUT_QVV48, ab.NORMALIZE_ALWAYS, (C, C, C), DEFAULTS_A),
    Variant(ab.LAYOUT_QVV48, ab.NORMALIZE_ALWAYS, (C, C, C), DEFAULTS_B),
    Variant(ab.LAYOUT_QVV40, ab.NORMALIZE_ALWAYS, (C, V, L), DEFAULTS_B),
    Variant(ab.LAYOUT_QVV40, ab.NORMALIZE_LERP_ONLY, (C, V, L), DEFAULTS_B),
    Variant(ab.LAYOUT_QVV40, ab.NORMALIZE_LERP_ONLY, (V, V, V), DEFAULTS_A),
    Variant(ab.LAYOUT_QVV40, ab.NORMALIZE_ALWAYS, (V, V, V), DEFAULTS_A),
]

# Settings whose rows are those of KEYS[i], decoded right after it (their output is checked, not which entry served them)
SHARING = {
    0: [dataclasses.replace(KEYS[0], normalization=ab.NORMALIZE_NEVER)],
    1: [dataclasses.replace(KEYS[1], math=ab.MATH_FAST)],
    5: [dataclasses.replace(KEYS[5], per_track=True)],
    6: [dataclasses.replace(KEYS[6], math=ab.MATH_FAST), dataclasses.replace(KEYS[6], normalization=ab.NORMALIZE_NEVER)],
}

# With four variants cached: forward (each key a miss, then a hit; the last four evict the first four), reversed (the last four hit,
# the first four are rebuilt and evict them), interleaved (the last four are rebuilt)
FORWARD = [i for i in range(len(KEYS)) for _ in range(2)]
REVERSED = list(reversed(range(len(KEYS))))
INTERLEAVED = [i for pair in zip(range(4), range(4, 8)) for i in pair]


@pytest.fixture(scope="module")
def gpu():
    import torch
    from oracle import port
    port.lib()
    rng = np.random.default_rng(5)
    return dict(torch=torch, port=port, ctx=ab.Context(0), policies=rng.integers(0, 4, 2048).astype(np.uint8),
                variable_defaults=rng.normal(size=(2048, 12)).astype(np.float32))


class Launch:
    """One decompress_tracks of a variant into its own sentinel-filled buffer, checked after the stream is synchronised."""

    def __init__(self, gpu, case, variant, stream=None):
        torch, ctx = gpu["torch"], gpu["ctx"]
        self.case, self.variant = case, variant
        self.width = 12 if variant.layout == ab.LAYOUT_QVV48 else 10
        n, max_tracks = len(case.req_clip), case.clipset.max_tracks
        stream = stream if stream is not None else torch.cuda.current_stream()
        with torch.cuda.stream(stream):     # the sentinels land before the decode
            self.d_out = torch.full((n * max_tracks * self.width,), int(SENTINEL.view(np.int32)), dtype=torch.int32, device="cuda")
        options = ab.Options(normalization=variant.normalization, default_modes=variant.modes, constant_defaults=variant.defaults,
                             output_layout=variant.layout, math_mode=variant.math)
        if variant.per_track:
            options.per_track_rounding = 1
            options.rounding_policy = ab.ROUND_PER_TRACK
            options.d_per_track_rounding = case.d_policies.data_ptr()
        if variant.variable:
            options.d_variable_defaults = case.d_variable.data_ptr()
        ctx.decompress_tracks(case.clipset, case.d_requests, n, options, self.d_out, stream=stream)
        self.info = ctx.debug_last_launch()
        assert self.info.kernel == ab.api.KERNEL_PIPELINE, (variant, self.info)

    def check(self):
        case, variant, width = self.case, self.variant, self.width
        n, max_tracks = len(case.req_clip), case.clipset.max_tracks
        got = self.d_out.cpu().numpy().view(np.uint32).reshape(n, max_tracks, width)
        want = np.full_like(got, SENTINEL)
        compared = np.ones(got.shape, dtype=bool)
        lanes = LANES if width == 12 else list(range(10))
        for r in range(n):
            c = int(case.req_clip[r])
            if c >= len(case.blobs):
                continue                # a clip outside the set: the request writes nothing
            pose = case.oracle(variant, c, float(case.req_time[r]))
            want[r, :pose.shape[0]][:, lanes] = pose[:, LANES].view(np.uint32)
            if width == 12:             # translation.w and scale.w are not defined by the reference
                compared[r, :pose.shape[0], 7] = compared[r, :pose.shape[0], 11] = False
        bad = compared & (got != want)
        if variant.math == ab.MATH_FAST:
            rot = np.zeros_like(compared)
            rot[..., :4] = True
            with np.errstate(invalid="ignore"):     # sentinels are NaN
                close = np.abs(got.view(np.float32) - want.view(np.float32)) <= FAST_MATH_TOLERANCE
            bad &= ~(rot & close)
        if bad.any():
            r, bone, lane = np.argwhere(bad)[0]
            raise AssertionError(f"{int(bad.any(axis=(1, 2)).sum())} of {n} poses differ; first: request {r} (clip {int(case.req_clip[r])}, "
                                 f"time {float(case.req_time[r])!r}), bone {bone}, lane {lane}: got {got[r, bone, lane].view(np.float32)!r} "
                                 f"want {want[r, bone, lane].view(np.float32)!r}; {variant} {self.info}")


class Case:
    """A clip set, its request list (every clip at clips.sample_times, two requests naming clips outside the set, shuffled) and the
    oracle's poses per (settings, clip, time)."""

    def __init__(self, gpu, names):
        torch, port = gpu["torch"], gpu["port"]
        self.gpu, self.port = gpu, port
        self.blobs = [clips.load_blob(n) for n in names]
        self.clipset = gpu["ctx"].upload(self.blobs)
        req_clip, req_time = [], []
        for c, name in enumerate(names):
            times = clips.sample_times(clips.TRANSFORM_SPECS[name])
            req_clip += [c] * len(times)
            req_time += list(times)
        req_clip += [len(names), len(names) + 7]
        req_time += [0.0, 0.5]
        perm = np.random.default_rng(len(req_clip)).permutation(len(req_clip))
        self.req_clip = np.array(req_clip, dtype=np.uint32)[perm]
        self.req_time = np.array(req_time, dtype=np.float32)[perm]
        self.d_requests = torch.from_numpy(ab.make_requests(self.req_clip, self.req_time).view(np.uint8)).cuda()
        max_tracks = self.clipset.max_tracks
        self.policies = gpu["policies"][:max_tracks]
        self.variable = gpu["variable_defaults"][:max_tracks]
        self.d_policies = torch.from_numpy(self.policies.copy()).cuda()
        self.d_variable = torch.from_numpy(self.variable.copy()).cuda()
        self.settings, self.poses = {}, {}

    def oracle(self, variant, clip, t):
        if variant not in self.settings:
            # VARIABLE without a defaults pointer takes the constant default values for every bone
            variable = self.variable if variant.variable else np.tile(np.float32(variant.defaults), (len(self.variable), 1))
            self.settings[variant] = self.port.SettingsBuilder(
                normalization=variant.normalization, per_track_rounding=variant.per_track, default_modes=variant.modes,
                constant_defaults=variant.defaults, variable_defaults=variable,
                per_track_policies=self.policies if variant.per_track else None)
        key = (variant, clip, t)
        if key not in self.poses:
            rounding = self.port.ROUND_PER_TRACK if variant.per_track else self.port.ROUND_NONE
            self.poses[key] = self.port.transform_decompress_tracks(self.blobs[clip], self.settings[variant], t, rounding)
        return self.poses[key]


@pytest.mark.parametrize("clip_set", list(CLIP_SETS))
def test_key_sweep_with_eviction_and_rebuild(gpu, clip_set):
    """Forward, reversed and interleaved walks over the distinct keys with the settings whose rows are those of a key decoded next to
    it, back to back on one stream, one output buffer each, synchronised once at the end."""
    case = Case(gpu, CLIP_SETS[clip_set])
    launches = []
    for walk in (FORWARD, REVERSED, INTERLEAVED):
        for i in walk:
            for variant in [KEYS[i]] + SHARING.get(i, []):
                launches.append(Launch(gpu, case, variant))
    gpu["torch"].cuda.synchronize()
    for launch in launches:
        launch.check()
    case.clipset.release()


@pytest.mark.parametrize("clip_set", list(CLIP_SETS))
def test_phase_a_in_the_kernel(gpu, clip_set):
    """Variable default values come from caller memory and are never cached: with one VARIABLE kind and a defaults array, the
    kernel runs phase A itself, here under NORMALIZE_ALWAYS with CONSTANT and LEGACY on the other kinds, in both layouts."""
    case = Case(gpu, CLIP_SETS[clip_set])
    launches = []
    for layout in (ab.LAYOUT_QVV48, ab.LAYOUT_QVV40):
        for modes in ((V, C, L), (C, V, L), (C, C, V), (V, C, C)):
            launches.append(Launch(gpu, case, Variant(layout, ab.NORMALIZE_ALWAYS, modes, DEFAULTS_A, variable=True)))
    gpu["torch"].cuda.synchronize()
    for launch in launches:
        launch.check()
    case.clipset.release()


def test_variant_built_on_a_delayed_stream(gpu):
    """Stream 1 sleeps, then decodes a key the clip set never saw: a miss whose build is queued behind the sleep. Stream 2 decodes the
    same key at once: a hit that must wait for the build, or it reads rows that are allocated but not yet written."""
    torch = gpu["torch"]
    variant = Variant(ab.LAYOUT_QVV48, ab.NORMALIZE_ALWAYS, (C, C, C), (0.6, 0.0, -0.8, 0.0, 7.0, -7.0, 0.5, 0.0, 3.5, 0.75, 2.5, 0.0))
    # The same kernels on another clip set first, so that no first launch loads a module (and waits for the device) below. Its
    # constant defaults differ: the rows it frees hold the wrong default sub-tracks for `variant`, so a miss handed that memory back
    # still shows a hit that did not wait. No other test builds rows with `variant`'s defaults.
    warm = Case(gpu, CLIP_SETS["mixed_scale"])
    Launch(gpu, warm, dataclasses.replace(variant, defaults=DEFAULTS_A)).check()
    warm.clipset.release()

    case = Case(gpu, CLIP_SETS["mixed_scale"])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    slept = torch.cuda.Event()
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(100_000_000)      # about 50 ms
    slept.record(s1)
    built = Launch(gpu, case, variant, stream=s1)
    hit = Launch(gpu, case, variant, stream=s2)
    assert not slept.query(), "the sleep ended before the second launch was enqueued: the hit did not race the build"
    torch.cuda.synchronize()
    built.check()
    hit.check()
    case.clipset.release()
