"""include/acl_b200/decompress.h: batch_decompressor::extract_pose_features is a thin member over the C call (tests/cpp/shim_features.cpp
runs both on the same inputs and compares the bytes and the flags)."""
import os
import subprocess

import pytest

from tests.test_cpp_shim import ROOT, build_shim_program


def test_features_shim_compiles_and_has_no_cpu_fallback(tmp_path):
    import torch
    exe = build_shim_program(tmp_path, "shim_features", cuda_runtime=True)
    if not torch.cuda.is_available():
        result = subprocess.run([exe, os.path.join(ROOT, "tests", "golden", "c1_30bones.acl.bin")], capture_output=True, text=True)
        assert result.returncode == 3, (result.returncode, result.stdout, result.stderr)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c1_30bones", "mixed_scale", "looping"])
def test_features_shim_equals_the_c_call(tmp_path, name):
    exe = build_shim_program(tmp_path, "shim_features", cuda_runtime=True)
    result = subprocess.run([exe, os.path.join(ROOT, "tests", "golden", name + ".acl.bin")], capture_output=True, text=True)
    assert result.returncode == 0 and "PASS" in result.stdout, (result.stdout, result.stderr)
