"""Loader of tests/islands/collect_island.cpp, the CPU restatement of IslandSleeper.CollectIsland that bepucuda_find_sleepable_islands is held to.
Compiled with g++ on first use into the temporary directory (tests/harness.py), so the tree stays as it is."""
import ctypes as C
import os

import numpy as np

from tests import harness

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "islands", "collect_island.cpp")


class IslandTypeBatch(C.Structure):
    _fields_ = [("bodies", C.c_int32), ("constraint_count", C.c_int32), ("body_references", C.c_void_p)]


def load():
    lib = harness.load("collect_island", [SRC], ["-O2", "-std=c++17", "-Wall", "-shared", "-fPIC"])
    lib.collect_sleepable_islands.argtypes = [C.POINTER(IslandTypeBatch), C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def find_sleepable_islands(type_batches, body_count, bundle_width, sleep_candidates):
    """CollectIsland run from every body no earlier traversal reached. `type_batches`: objects with constraint_count and
    body_references[bundles, bodies, bundle_width] (a Simulation's type_batches(), or hand-made ones); `sleep_candidates`: one flag per body.
    Returns (island_of_body, roots, counts) in the form of bepucuda_find_sleepable_islands."""
    lib = load()
    tbs = list(type_batches)
    refs = [np.ascontiguousarray(tb.body_references, dtype=np.int32) for tb in tbs]
    arr = (IslandTypeBatch * max(len(tbs), 1))()
    for i, (tb, r) in enumerate(zip(tbs, refs)):
        assert r.ndim == 3 and r.shape[2] == bundle_width
        arr[i].bodies = r.shape[1]
        arr[i].constraint_count = tb.constraint_count
        arr[i].body_references = r.ctypes.data
    candidates = np.ascontiguousarray(sleep_candidates, dtype=np.uint8).reshape(-1)
    assert candidates.shape[0] == body_count
    labels = np.zeros(max(body_count, 1), dtype=np.int32)
    roots = np.zeros(max(body_count, 1), dtype=np.int32)
    counts = np.zeros(max(body_count, 1), dtype=np.int32)
    count = lib.collect_sleepable_islands(arr, len(tbs), bundle_width, body_count, candidates.ctypes.data, labels.ctypes.data, roots.ctypes.data, counts.ctypes.data)
    if count < 0:
        raise ValueError("collect_sleepable_islands failed: %d" % count)
    return labels[:body_count], roots[:count].copy(), counts[:count].copy()
