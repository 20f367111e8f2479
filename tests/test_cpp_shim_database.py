"""The streaming database API of the C++ header shim (include/acl_b200/decompress.h: database_context, decompression_context::
initialize(tracks, database)): tests/cpp/shim_database.cpp is a reference call site compiled against acl:: and acl_b200::."""
import os
import subprocess

import numpy as np
import pytest

from tests import clips

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE_INCLUDES = ["/root/reference/includes", "/root/reference/external/rtm/includes"]
SHIM_DATABASE_EXE = os.path.join(ROOT, "tests", "cpp", "_build", "shim_database")


def build_shim_database():
    """Needs the reference's headers: built where they exist (__graft_entry__.build() does it too) and shipped prebuilt."""
    os.makedirs(os.path.dirname(SHIM_DATABASE_EXE), exist_ok=True)
    cmd = ["g++", "-std=c++14", "-O2", "-msse4.1", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror"] + ["-I" + d for d in REFERENCE_INCLUDES] + [
        "-o", SHIM_DATABASE_EXE, os.path.join(ROOT, "tests", "cpp", "shim_database.cpp"),
        "-L" + os.path.join(ROOT, "acl_b200"), "-laclb200", "-Wl,-rpath,$ORIGIN/../../../acl_b200"]
    subprocess.run(cmd, check=True, capture_output=True, text=True)


def _inputs(tmp_path, clip):
    g = np.load(clips.golden_path("database_tiers", "npz"))
    clip_path, database_path = tmp_path / "clip.bin", tmp_path / "database.bin"
    clip_path.write_bytes(g[f"clip{clip}"].tobytes())
    database_path.write_bytes(g["database"].tobytes())
    return str(clip_path), str(database_path)


@pytest.mark.skipif(not all(os.path.isdir(d) for d in REFERENCE_INCLUDES), reason="needs the reference's headers")
def test_database_callsite_compiles_against_the_shim(tmp_path):
    import torch
    build_shim_database()
    result = subprocess.run([SHIM_DATABASE_EXE, *_inputs(tmp_path, 1)], capture_output=True, text=True)
    if not torch.cuda.is_available():
        assert result.returncode == 3, (result.returncode, result.stdout, result.stderr)


@pytest.mark.gpu
@pytest.mark.parametrize("clip", [0, 1, 2, 3])
def test_database_callsite_matches_the_reference(tmp_path, clip):
    if not os.path.exists(SHIM_DATABASE_EXE):
        pytest.skip("tests/cpp/_build/shim_database was not built (needs /root/reference at build time)")
    result = subprocess.run([SHIM_DATABASE_EXE, *_inputs(tmp_path, clip)], capture_output=True, text=True)
    assert result.returncode == 0 and "PASS" in result.stdout, (result.stdout, result.stderr)
