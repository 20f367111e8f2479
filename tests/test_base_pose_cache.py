"""acl_b200/csrc/base_pose_cache.h: the bookkeeping behind the pipeline kernel's cached base pose rows, compiled on the host and
driven through the interleavings that threads sharing a clip set can produce (tests/cpp/base_pose_cache.cpp): a variant handed to a
launch being set up, by a hit or by the miss that built it, is never evicted under it; a full cache of pinned variants grows past
its cap; unpinned variants go in least recently used order; every key field tells variants apart."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_base_pose_cache_bookkeeping(tmp_path):
    exe = str(tmp_path / "base_pose_cache")
    subprocess.run(["g++", "-std=c++14", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "acl_b200", "csrc"), "-o", exe,
                    os.path.join(ROOT, "tests", "cpp", "base_pose_cache.cpp")], check=True, capture_output=True, text=True)
    result = subprocess.run([exe], capture_output=True, text=True)
    assert result.returncode == 0 and result.stdout.strip().endswith("PASS"), result.stdout + result.stderr
