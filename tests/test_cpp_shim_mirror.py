"""include/acl_b200/decompress.h: batch_decompressor::mirror_poses, decompress_tracks_mirrored and decompress_tracks_mirrored_skinning are
thin members over the C calls (tests/cpp/shim_mirror.cpp runs both on the same inputs and compares the bytes)."""
import os
import subprocess

import pytest

from tests.test_cpp_shim import ROOT, build_shim_program

CLIP = os.path.join(ROOT, "tests", "golden", "c1_30bones.acl.bin")


def test_mirror_shim_compiles_and_has_no_cpu_fallback(tmp_path):
    import torch
    exe = build_shim_program(tmp_path, "shim_mirror", cuda_runtime=True)
    if not torch.cuda.is_available():
        result = subprocess.run([exe, CLIP], capture_output=True, text=True)
        assert result.returncode == 3, (result.returncode, result.stdout, result.stderr)


@pytest.mark.gpu
def test_mirror_shim_equals_the_c_calls(tmp_path):
    exe = build_shim_program(tmp_path, "shim_mirror", cuda_runtime=True)
    result = subprocess.run([exe, CLIP], capture_output=True, text=True)
    assert result.returncode == 0 and "PASS" in result.stdout, (result.stdout, result.stderr)
