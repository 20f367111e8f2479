"""Bone queries (aclb200_decompress_bones): the ancestor closure of a bone list, the skeletons and bone lists the tests and
tools/bench_bones.py use, and the rows a query must give, gathered from a whole pose.

The closure rule is the kernel's: from each listed bone below the clip's num_tracks, walk to the parent while the parent precedes the
bone (a root, 0xFFFFFFFF, or a parent at or above its child ends the chain; such a bone is a root for the walk, as in the whole walk).
A walk only ever moves to a lower bone index, so it ends on any parent table."""
from __future__ import annotations

import numpy as np

ROOT = 0xFFFFFFFF
NO_BONE = 0xFFFFFFFF


def closure(parents, bones, num_tracks: int, with_parents: bool = True) -> np.ndarray:
    """Sorted bone indices the query of `bones` decodes (with_parents: and walks)."""
    parents = np.asarray(parents, dtype=np.uint64)
    marked = set()
    for bone in bones:
        bone = int(bone)
        while bone < num_tracks and bone not in marked:
            marked.add(bone)
            if not with_parents:
                break
            parent = int(parents[bone])
            bone = parent if parent < bone else ROOT
    return np.array(sorted(marked), dtype=np.int64)


def effective_parents(parents) -> np.ndarray:
    """The skeleton the walk uses: a parent that does not precede its child becomes a root."""
    parents = np.asarray(parents, dtype=np.uint32).copy()
    bones = np.arange(parents.size, dtype=np.uint64)
    parents[(parents != ROOT) & (parents.astype(np.uint64) >= bones)] = ROOT
    return parents


def tree(n: int) -> np.ndarray:
    bones = np.arange(n)
    return np.where(bones == 0, ROOT, (bones - 1) // 2).astype(np.uint32)


def skeleton(kind: str, n: int, seed: int = 0) -> np.ndarray:
    """tree (binary), chain (the deepest walk), star, random (extra roots), late (a tree with a parent after its child)"""
    bones = np.arange(n)
    if kind == "chain":
        return np.where(bones == 0, ROOT, bones - 1).astype(np.uint32)
    if kind == "star":
        return np.where(bones == 0, ROOT, 0).astype(np.uint32)
    if kind == "random":
        rng = np.random.default_rng(seed)
        parents = np.array([ROOT] + [int(rng.integers(0, b)) for b in range(1, n)], np.uint32)
        parents[rng.random(n) < 0.1] = ROOT
        return parents
    parents = tree(n)
    if kind == "late" and n > 3:
        parents[n // 2] = n - 1          # a parent after its child: that bone is a root for the walk
        parents[1] = 1                   # a bone that is its own parent
    return parents


SKELETONS = ["tree", "chain", "star", "random", "late"]

# C2's binary tree: one leaf under each of bones 3, 4, 5 and 6 (two at depth 6, two at depth 5): 21 of the 100 bones are in the closure
C2_FOUR_LEAVES = [63, 79, 50, 55]
C2_SIX_MIXED = [0, 99, 7, 40, 63, 26]


def bone_lists(num_tracks: int, seed: int = 0) -> dict:
    """Named bone lists for a clip of num_tracks bones (entries may be NO_BONE or beyond num_tracks: those rows stay untouched)"""
    rng = np.random.default_rng(seed)
    n = num_tracks
    leaves = [b for b in range(n) if 2 * b + 1 >= n] or [0]
    lists = {
        "root": [0],
        "deep_leaf": [n - 1],
        "leaves": [leaves[0], leaves[len(leaves) // 3], leaves[(2 * len(leaves)) // 3], leaves[-1]],
        "k32": [int(b) for b in rng.integers(0, n, 32)],
        "duplicates_reversed": [n - 1, n // 2, n - 1, 0, n // 2][::-1],
        "holes": [NO_BONE, n - 1, NO_BONE, 0],
        "out_of_range": [n, 0, n + 7, n - 1, 0x7FFFFFFF],
    }
    if n <= 32:
        lists["all_bones"] = list(range(n))
    return lists


def pad_lists(lists, k: int) -> np.ndarray:
    """[num_lists][k] uint32, short lists padded with NO_BONE"""
    out = np.full((len(lists), k), NO_BONE, np.uint32)
    for i, bones in enumerate(lists):
        out[i, :len(bones)] = bones
    return out


def gather(pose_rows: np.ndarray, bones, num_tracks: int, sentinel_row: np.ndarray) -> np.ndarray:
    """The K rows a query writes from a whole pose's rows: row list[j], or the sentinel where the entry is NO_BONE or out of range"""
    out = np.empty((len(bones),) + pose_rows.shape[1:], pose_rows.dtype)
    for j, bone in enumerate(bones):
        out[j] = pose_rows[int(bone)] if int(bone) < num_tracks else sentinel_row
    return out


def object_rows(port, object_space, local: np.ndarray, parents, matrix: bool) -> np.ndarray:
    """The 48 byte object space rows of aclb200_decompress_tracks_object_space for one local pose ([n][12] float32)"""
    parents = effective_parents(parents)
    if matrix:
        return object_space.port_local_to_object_space_matrix(local, parents)
    out = port.local_to_object_space(local, parents, port.NORMALIZE_IEEE)
    out[:, 7] = 0.0
    out[:, 11] = 0.0
    return out
