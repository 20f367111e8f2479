"""Regenerates tests/golden/*.error.npz: what the UNMODIFIED reference's calculate_compression_error
(includes/acl/compression/impl/track_error.impl.h:400-571) returns for a few of the named clips of tests/clips.py, together with the
raw poses it sampled (its input) and the per bone errors it measured. Run where oracle/_ref/libaclref.so exists:

    python tests/golden/make_error_golden.py

The numbers carry the rsqrtss estimate of the CPU that ran this script (rtm::quat_normalize, external/rtm/includes/rtm/quatf.h:917-953):
another CPU's reference agrees within a few 1e-6, so the tests compare them with a tolerance and compare bit for bit only against the
reference run live on the machine at hand.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import ref  # noqa: E402
from tests import clips  # noqa: E402

TRANSFORM = ["c1_30bones", "mixed_scale", "single_segment", "stripped_single", "two_samples", "one_bone", "ragged_17"]
SCALAR = ["float1", "float2", "float3", "float4", "vector4", "float1_one_sample"]
SETTINGS_KIND = 1       # debug_transform_decompression_settings, what tools/acl_compressor measures with


def main() -> None:
    for name in TRANSFORM:
        spec = clips.TRANSFORM_SPECS[name]
        r = ref.transform_error(spec, clips.load_blob(name), SETTINGS_KIND)
        np.savez_compressed(clips.golden_path(name, "error.npz"), raw_poses=r["raw_poses"], errors=r["errors"], parents=r["parents"],
                            shell_distances=r["shell_distances"], index=np.uint32(r["index"]), error=np.float32(r["error"]),
                            sample_time=np.float32(r["sample_time"]), rounding=np.uint32(r["rounding"]),
                            sample_rate=np.float32(r["sample_rate"]), duration=np.float32(r["duration"]))
        print("transform", name, r["index"], r["error"], r["sample_time"])
    for name in SCALAR:
        spec = clips.SCALAR_SPECS[name]
        r = ref.scalar_error(spec, clips.load_blob(name))
        np.savez_compressed(clips.golden_path(name, "error.npz"), raw_values=r["raw_values"], index=np.uint32(r["index"]),
                            error=np.float32(r["error"]), sample_time=np.float32(r["sample_time"]), rounding=np.uint32(r["rounding"]),
                            sample_rate=np.float32(r["sample_rate"]), duration=np.float32(r["duration"]))
        print("scalar", name, r["index"], r["error"], r["sample_time"])
    write_matrix_golden()


def write_matrix_golden() -> None:
    """tests/golden/*.matrix_error.npz: qvvf_matrix3x4f_transform_error_metric over the same raw poses. That metric has no CPU specific
    step, so these numbers are the reference's on any machine and the tests compare them bit for bit."""
    for name in TRANSFORM:
        m = ref.transform_error_matrix(clips.TRANSFORM_SPECS[name], clips.load_blob(name))
        np.savez_compressed(clips.golden_path(name, "matrix_error.npz"), errors=m["errors"], index=np.uint32(m["index"]),
                            error=np.float32(m["error"]), sample_time=np.float32(m["sample_time"]))
        print("matrix", name, m["index"], m["error"], m["sample_time"])


if __name__ == "__main__":
    main()
