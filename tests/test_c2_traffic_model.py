"""tools/c2_traffic.py's host model on a few C2 clips: the kernel's grouping rules and the Entry size show up where they should."""
import importlib.util
import os

import numpy as np

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load_tool():
    # tools/ is not a package: load the script by path, without putting tools/ on sys.path for the rest of the session
    spec = importlib.util.spec_from_file_location("c2_traffic", os.path.join(ROOT, "tools", "c2_traffic.py"))
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module


c2_traffic = _load_tool()


def test_model_counts_chains_tables_and_base_rows():
    w = bench.make_workload("c2", 0, 12)
    # 72 batches over 4 blocks: each block walks 18 consecutive batches, as the blocks of a full C2 launch walk about 230
    old, new = (c2_traffic.model(w, 10, 4, entry) for entry in (32, 16))
    requests = w["req_clip"].size
    assert old["requests"] == new["requests"] == requests
    # sequential playback in batches of 10: chains of at most five, at least two per batch, whatever the Entry size
    assert old["groups"] == new["groups"] >= requests // 5
    assert old["chained_groups"] == new["chained_groups"] > 0
    assert old["requested"]["windows"] == new["requested"]["windows"] > 0
    assert old["requested"]["base_rows"] == new["requested"]["base_rows"]
    # only the Entry part of the tables shrinks: AnimDesc (32 B) stays
    t = c2_traffic.clip_tables(w)
    assert new["distinct"]["entry_tables"] * 2 == old["distinct"]["entry_tables"]
    assert old["distinct"]["anim_desc"] == new["distinct"]["anim_desc"] == int(t["nanim"].sum()) * 32
    assert new["requested"]["tables"] < old["requested"]["tables"]
    # a pose row keeps its clip's base row across the block's batches: far fewer copies than requests
    row = int(((t["num_tracks"][0] * 40 + 15) // 16) * 16)
    assert 0 < new["requested"]["base_rows"] < requests * row
    assert new["pose_bytes_written"] == int((t["num_tracks"][w["req_clip"]] * 40).sum())
    assert np.isfinite(new["distinct_total"])
