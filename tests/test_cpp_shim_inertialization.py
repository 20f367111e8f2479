"""include/acl_b200/decompress.h: batch_decompressor::begin_inertialization and inertialize_poses are thin members over the C calls
(tests/cpp/shim_inertialization.cpp runs both on the same inputs and compares the bytes)."""
import subprocess

import pytest

from tests.test_cpp_shim import build_shim_program


def test_inertialization_shim_compiles_and_has_no_cpu_fallback(tmp_path):
    import torch
    exe = build_shim_program(tmp_path, "shim_inertialization", cuda_runtime=True)
    if not torch.cuda.is_available():
        result = subprocess.run([exe], capture_output=True, text=True)
        assert result.returncode == 3, (result.returncode, result.stdout, result.stderr)


@pytest.mark.gpu
def test_inertialization_shim_equals_the_c_calls(tmp_path):
    exe = build_shim_program(tmp_path, "shim_inertialization", cuda_runtime=True)
    result = subprocess.run([exe], capture_output=True, text=True)
    assert result.returncode == 0 and "PASS" in result.stdout, (result.stdout, result.stderr)
