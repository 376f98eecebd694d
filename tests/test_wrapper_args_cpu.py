"""The Python wrapper's argument conversions (hnsw.py), without a GPU: what each turns a search argument into, as the C
calls take it, and the ValueError or TypeError, with its message, it raises for a malformed one."""
from importlib import import_module

import numpy as np
import pytest

hnsw = import_module("hnswlib-rs_b200.hnsw")


def same(a, values, dtype):
    assert a.dtype == dtype and a.flags.c_contiguous and a.tolist() == values


def test_label_sets_from_lists():
    off, vals = hnsw._label_sets([[3, 1], [], np.array([7], np.int64), (2, 2, hnsw.LABEL_NONE)], 4)
    same(off, [0, 2, 2, 3, 6], np.uint64)
    same(vals, [3, 1, 7, 2, 2, hnsw.LABEL_NONE], np.uint32)


def test_label_sets_from_offsets_and_values():
    off, vals = hnsw._label_sets(([0, 1, 3], np.array([5, 6, 7], np.int32)), 2)
    same(off, [0, 1, 3], np.uint64)
    same(vals, [5, 6, 7], np.uint32)
    off, vals = hnsw._label_sets((np.array([[0], [0]], np.uint64), []), 1)   # offsets of any shape, flattened
    same(off, [0, 0], np.uint64)


@pytest.mark.parametrize("sets", [[[], []], ([0, 0, 0], [])])
def test_label_sets_never_a_null_values_pointer(sets):
    off, vals = hnsw._label_sets(sets, 2)
    same(off, [0, 0, 0], np.uint64)
    assert vals.dtype == np.uint32 and vals.size == 1


def test_label_sets_of_no_queries():
    off, vals = hnsw._label_sets([], 0)
    same(off, [0], np.uint64)
    assert vals.size == 1


@pytest.mark.parametrize("sets, nq, msg", [
    (([0, 1, 2, 2], [1, 2]), 2, "sets: 4 offsets for 2 queries, expected 3"),
    (([0, 1], [1]), 2, "sets: 2 offsets for 2 queries, expected 3"),
    (([0, 1, 3], [1, 2]), 2, r"sets: offsets must be integers in \[0, 2\], the number of values"),
    (([0, -1, 2], [1, 2]), 2, r"sets: offsets must be integers in \[0, 2\], the number of values"),
    (([0.0, 1.0, 2.0], [1, 2]), 2, r"sets: offsets must be integers in \[0, 2\], the number of values"),
    (([0, 1, 2], [1, -2]), 2, "sets: labels are unsigned 32-bit integers"),
    (([0, 1, 2], [1, 1 << 32]), 2, "sets: labels are unsigned 32-bit integers"),
    ([[1], [2], [3]], 2, "sets has 3 entries for 2 queries"),
    ([[1]], 2, "sets has 1 entries for 2 queries"),
    ([[1], [-5]], 2, "sets: labels are unsigned 32-bit integers"),
])
def test_label_sets_refusals(sets, nq, msg):
    with pytest.raises(ValueError, match=f"^{msg}$"):
        hnsw._label_sets(sets, nq)


def test_excluded_from_lists():
    off, ids = hnsw._excluded([[9, 4, 9], [], np.array([0], np.uint64)], 3)
    same(off, [0, 3, 3, 4], np.uint64)
    same(ids, [9, 4, 9, 0], np.uint64)


def test_excluded_from_offsets_and_ranks():
    off, ids = hnsw._excluded((np.array([0, 2, 2], np.int64), [11, 12]), 2)
    same(off, [0, 2, 2], np.uint64)
    same(ids, [11, 12], np.uint64)
    off, ids = hnsw._excluded(([0, 5, 9], [1]), 2)   # offsets past the ranks are the C call's to refuse
    same(off, [0, 5, 9], np.uint64)


@pytest.mark.parametrize("excluded", [[[], []], ([0, 0, 0], [])])
def test_excluded_never_a_null_ranks_pointer(excluded):
    off, ids = hnsw._excluded(excluded, 2)
    same(off, [0, 0, 0], np.uint64)
    assert ids.dtype == np.uint64 and ids.size == 1


@pytest.mark.parametrize("excluded, nq, msg", [
    (([0, 1, 2, 2], [1, 2]), 2, "excluded: 4 offsets for 2 queries, expected 3"),
    (([0, 1], [1]), 2, "excluded: 2 offsets for 2 queries, expected 3"),
    (([0, -1, 2], [1, 2]), 2, "excluded: offsets must be non-negative integers"),
    (([0.0, 1.0, 2.0], [1, 2]), 2, "excluded: offsets must be non-negative integers"),
    (([0, 1, 2], [1, -2]), 2, "excluded: ranks must be non-negative integers"),
    (([0, 1, 2], [1.0, 2.0]), 2, "excluded: ranks must be non-negative integers"),
    ([[1], [2], [3]], 2, "excluded has 3 entries for 2 queries"),
    ([[1], [-1]], 2, "excluded: ranks must be non-negative integers"),
])
def test_excluded_refusals(excluded, nq, msg):
    with pytest.raises(ValueError, match=f"^{msg}$"):
        hnsw._excluded(excluded, nq)


def test_ranges():
    same(hnsw._ranges([(1, 2), (-5, 7)], 2), [1, 2, -5, 7], np.int64)
    same(hnsw._ranges(np.array([[0, 9]], np.uint32), 1), [0, 9], np.int64)
    same(hnsw._ranges([hnsw.RANGE_ALL], 1), list(hnsw.RANGE_ALL), np.int64)
    r = hnsw._ranges([], 0)   # never a NULL pointer
    assert r.dtype == np.int64 and r.size == 2


@pytest.mark.parametrize("ranges, nq, msg", [
    ([(1, 2)], 2, r"ranges has shape \(1, 2\), expected \(2, 2\)"),
    ([1, 2], 1, r"ranges has shape \(2,\), expected \(1, 2\)"),
    ([(1, 2, 3)], 1, r"ranges has shape \(1, 3\), expected \(1, 2\)"),
    ([(0.5, 2.0)], 1, r"ranges: bounds are 64-bit integers \(attr_of_float maps floats\)"),
    (np.array([[0, 1 << 63]], np.uint64), 1, "ranges: bounds are signed 64-bit integers"),
])
def test_ranges_refusals(ranges, nq, msg):
    with pytest.raises(ValueError, match=f"^{msg}$"):
        hnsw._ranges(ranges, nq)


def test_filter_ids():
    same(hnsw._filter_ids([None, hnsw.ResidentFilter(None, 5), None], 3), [-1, 5, -1], np.int64)
    same(hnsw._filter_ids([], 0), [], np.int64)


def test_filter_ids_refusals():
    with pytest.raises(ValueError, match="^filters has 1 entries for 2 queries$"):
        hnsw._filter_ids([None], 2)
    with pytest.raises(TypeError, match=r"^the exact searches take a ResidentFilter \(Hnsw.make_filter\) or None as "
                                        r"their filter$"):
        hnsw._filter_ids([None, [1, 2]], 2)
