"""The streaming database cases shared by tests/test_gpu_database.py, tests/test_database_oracle.py and
tests/golden/make_database_golden.py: the clips, the tier states and the sample times."""
import numpy as np

IN, OUT, MEDIUM, LOW = 0, 1, 1, 2
ALL = 0xFFFFFFFF
PLAIN_CLIP = "c1_30bones"           # a clip without a database, decoded in the same launches
# tier states, each the stream_in / stream_out calls that lead to it from nothing streamed in
STATES = {
    "nothing": [],
    "some_medium": [(IN, MEDIUM, 1)],
    "all_medium": [(IN, MEDIUM, 1), (IN, MEDIUM, ALL)],
    "all_medium_low": [(IN, MEDIUM, 1), (IN, MEDIUM, ALL), (IN, LOW, ALL)],
    "medium_out": [(IN, MEDIUM, 1), (IN, MEDIUM, ALL), (IN, LOW, ALL), (OUT, MEDIUM, ALL)],
}
ALL_TIMES = np.array([-0.1, 0.0, 0.13, 0.5, 0.77, 1.01, 1.5, 2.2, 3.5], np.float32)


def _specs(ref):
    return [
        ref.TransformSpec(num_tracks=12, num_samples=28, seed=11),                                  # single segment
        ref.TransformSpec(num_tracks=10, num_samples=120, seed=12, scale_default_pct=0),            # several segments, with scale
        ref.TransformSpec(num_tracks=16, num_samples=100, seed=13, trans_constant_pct=50),          # several segments, no scale
        ref.TransformSpec(num_tracks=8, num_samples=90, seed=14, strip_proportion=0.3),             # stripped key frames
    ]


def build_cases(ref, ref_database):
    """(bound clips, database, a clip of another database, that medium-only database) from the reference compressor."""
    bound, database = ref_database.build_database(_specs(ref), 0.3, 0.3, 4096)
    others, other_database = ref_database.build_database([ref.TransformSpec(num_tracks=12, num_samples=50, seed=99)], 0.5, 0.0, 4096)
    return bound, database, others[0], other_database
