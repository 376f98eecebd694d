"""The argument checks of every search entry point (include/hnsw_b200.h), table-driven: each row calls one entry point
through the raw C ABI with one defect, or with two to fix which one is answered first, and asserts the return value,
the last_error() wording and that every output array still holds its sentinel."""
import ctypes as C
from importlib import import_module

import numpy as np
import pytest
import torch  # imported first, so that torch's own NCCL is the one the library binds at run time

pytestmark = pytest.mark.gpu

N, D, NQ, K, EF = 300, 16, 3, 5, 32
SENTINEL = 7
ANS = ["ids", "dist", "internal", "pid", "counts"]
DEV = ["d_out", "d_counts", "sync", "kms"]
ROWS = ["filter", "qrange", "qset_off", "qset"]

# every search entry point, by its parameters in order (names as the defaults below give them)
ENTRIES = {
    "search_flat": ["h", "q", "nq", "dim", "k", "ef", "mode", "fids", "nf", "fn", "ctx", *ANS],
    "search_flat_filtered": ["h", "filter", "q", "nq", "dim", "k", "ef", *ANS],
    "search_flat_submit": ["h", "q", "nq", "dim", "k", "ef", *ANS],
    "search_flat_submit_filtered": ["h", "filter", "q", "nq", "dim", "k", "ef", *ANS],
    "search_device": ["h", "dq", "nq", "k", "ef", *DEV],
    "search_device_filtered": ["h", "filter", "dq", "nq", "k", "ef", *DEV],
    "search_exact": ["h", "filter", "q", "nq", "dim", "k", *ANS],
    "search_flat_per_query": ["h", "filters", "q", "nq", "dim", "k", "ef", *ANS],
    "search_exact_per_query": ["h", "filters", "q", "nq", "dim", "k", *ANS],
    "search_flat_labeled": ["h", "qlabels", "q", "nq", "dim", "k", "ef", *ANS],
    "search_exact_labeled": ["h", "qlabels", "q", "nq", "dim", "k", *ANS],
    "search_flat_label_sets": ["h", "qset_off", "qset", "q", "nq", "dim", "k", "ef", *ANS],
    "search_exact_label_sets": ["h", "qset_off", "qset", "q", "nq", "dim", "k", *ANS],
    "search_flat_ranges": ["h", "qrange", "qset_off", "qset", "q", "nq", "dim", "k", "ef", *ANS],
    "search_exact_ranges": ["h", "qrange", "qset_off", "qset", "q", "nq", "dim", "k", *ANS],
    "search_exact_device": ["h", "filter", "dq", "nq", "k", *DEV],
    "search_flat_by_id": ["h", "qids", "nq", "k", "ef", "excl", *ROWS, *ANS],
    "search_exact_by_id": ["h", "qids", "nq", "k", "excl", *ROWS, *ANS],
    "search_device_by_id": ["h", "exact", "filter", "dqids", "nq", "k", "ef", "excl", *DEV],
    "search_flat_excluding": ["h", "qx_off", "qx", *ROWS, "q", "nq", "dim", "k", "ef", *ANS],
    "search_exact_excluding": ["h", "qx_off", "qx", *ROWS, "q", "nq", "dim", "k", *ANS],
    "count_admitted": ["h", *ROWS, "nq", "out_count"],
    "search_planned": ["h", "qx_off", "qx", *ROWS, "q", "nq", "dim", "k", "ef", *ANS, "out_exact"],
    "search_planned_by_id": ["h", "qids", "nq", "k", "ef", "excl", *ROWS, *ANS, "out_exact"],
    "search_exact_radius": ["h", *ROWS, "q", "nq", "dim", "radius", "k", *ANS, "out_total"],
    "search_exact_radius_by_id": ["h", "qids", "nq", "radius", "k", "excl", *ROWS, *ANS, "out_total"],
}
# the arguments an entry point must be given (the others default to NULL, or -1 for a filter)
REQUIRED = {
    "search_flat_filtered": {"filter"}, "search_flat_submit_filtered": {"filter"}, "search_device_filtered": {"filter"},
    "search_flat_label_sets": {"qset_off", "qset"}, "search_exact_label_sets": {"qset_off", "qset"},
    "search_flat_ranges": {"qrange"}, "search_exact_ranges": {"qrange"},
    "search_flat_excluding": {"qx_off", "qx"}, "search_exact_excluding": {"qx_off", "qx"},
}
OPTIONAL = {"filter", "qrange", "qset_off", "qset", "qx_off", "qx"}
INPUTS = ["q", "dq", "qids", "dqids", "filters", "qlabels", "qrange", "qset_off", "qset", "qx_off", "qx", "radius"]
CONFLICT = {"filter": "rf", "qset_off": "set_off", "qset": "set_vals"}   # a resident filter together with sets
BY_ID = ["search_flat_by_id", "search_exact_by_id", "search_planned_by_id", "search_exact_radius_by_id"]
RADIUS = ["search_exact_radius", "search_exact_radius_by_id"]
EXCLUDING = ["search_flat_excluding", "search_exact_excluding"]
DEVICE = ["search_device", "search_device_filtered", "search_exact_device", "search_device_by_id"]
FILTER_FN = import_module("hnswlib-rs_b200.hnsw").FILTER_FN
COMBINE = "a resident filter cannot be combined with label sets or ranges"


def rows():
    """(entry point, handle, argument overrides, return value, message) per case; an override names an argument and
    gives its value, None for NULL or one of the valid arrays by name; the handle is "h", "null" or "part" (the
    partitioned handle)"""
    out = []
    for e, params in ENTRIES.items():
        nulls = {a: None for a in params if a in INPUTS}
        out.append((e, "null", nulls, -1, "NULL handle"))
        if e.startswith("search_flat_submit"):
            out.append((e, "h", {**nulls, "nq": 0}, -1, "bad argument"))
        else:
            out.append((e, "h", {**nulls, "nq": 0, "out_count": None}, 0, None))
    for e in ("search_flat_submit", "search_flat_submit_filtered", *DEVICE):
        out.append((e, "part", {}, -1, f"{e} is not available on a partitioned handle"))
    out += [
        ("search_device_by_id", "part", {"nq": 0}, 0, None),
        ("search_device_by_id", "part", {"dqids": None}, -1, "search_device_by_id: qids is NULL"),
        ("search_device_by_id", "h", {"dqids": "dqids_far"}, -1, f"qids[1] = {N} is not below nb_point = {N}"),
        ("search_flat", "h", {"counts": None}, -1, "bad argument"),
        ("search_flat", "h", {"k": 0}, -1, "bad argument"),
        ("search_flat", "h", {"q": None}, -1, "bad argument"),
        ("search_flat_submit", "h", {"q": None}, -1, "bad argument"),
        ("search_flat_per_query", "h", {"filters": None}, -1, "filters is NULL"),
        ("search_exact_per_query", "h", {"filters": None, "dist": None}, -1, "filters is NULL"),
        ("search_flat_labeled", "h", {"qlabels": None}, -1, "qlabels is NULL"),
        ("search_exact_labeled", "h", {"qlabels": None, "ids": None}, -1, "qlabels is NULL"),
        ("search_flat_label_sets", "h", {"qset_off": None, "qset": None}, -1, "qset_off is NULL"),
        ("search_exact_label_sets", "h", {"qset": None, "counts": None}, -1, "qset is NULL"),
        ("search_flat_ranges", "h", {"qrange": None, "qset_off": "set_off"}, -1, "qrange is NULL"),
        ("search_exact_ranges", "h", {"qset_off": "set_off"}, -1, "qset is NULL"),
        ("search_exact_ranges", "h", {"qset": "set_vals"}, -1, "qset_off is NULL"),
        ("count_admitted", "h", {"filter": "rf", "qrange": "ranges"}, -1, f"count_admitted: {COMBINE}"),
        ("count_admitted", "h", {**CONFLICT, "qset": None}, -1, f"count_admitted: {COMBINE}"),
        ("count_admitted", "h", {"qset_off": "set_off"}, -1, "qset is NULL"),
        ("count_admitted", "h", {"qset": "set_vals", "out_count": None}, -1, "qset_off is NULL"),
        ("count_admitted", "h", {"out_count": None}, -1, "count_admitted: out_count is NULL"),
        ("search_planned", "h", {"qx": "xs"}, -1, "search_planned: qx_off is NULL"),
        ("search_planned", "h", {"qx_off": "x_off", **CONFLICT}, -1, "search_planned: qx is NULL"),
        ("search_planned", "h", {"qx_off": "x_off", "qx": "xs", **CONFLICT}, -1, f"search_planned: {COMBINE}"),
    ]
    for e in BY_ID:
        out += [
            (e, "h", {"qids": None, **CONFLICT}, -1, f"{e}: qids is NULL"),
            (e, "h", {"qids": "qids_far", **CONFLICT}, -1, f"{e}: {COMBINE}"),
            (e, "h", {"qids": "qids_far", "qset_off": "set_off"}, -1, f"{e}: qids[1] = {N} is not below nb_point = {N}"),
            (e, "h", {"qids": "qids_far"}, -1, f"{e}: qids[1] = {N} is not below nb_point = {N}"),
            (e, "h", {"filter": "rf", "qrange": "ranges"}, -1, f"{e}: {COMBINE}"),
            (e, "h", {"qset_off": "set_off"}, -1, "qset is NULL"),
        ]
    for e in RADIUS:
        out += [
            (e, "h", {"radius": None, **CONFLICT}, -1, f"{e}: radius is NULL"),
            (e, "h", {"radius": "radius_nan", **CONFLICT}, -1, (f"{e}: radius[1] = ", " is NaN")),
            (e, "h", {"radius": "radius_neg"}, -1, (f"{e}: radius[1] = ", " is negative")),
            (e, "h", {**CONFLICT}, -1, f"{e}: {COMBINE}"),
        ]
    out.append(("search_exact_radius_by_id", "h", {"qids": None, "radius": None}, -1,
                "search_exact_radius_by_id: qids is NULL"))
    for e in EXCLUDING:
        out += [
            (e, "h", {"qx_off": None, "qx": None}, -1, f"{e}: qx_off is NULL"),
            (e, "h", {"qx": None, **CONFLICT}, -1, f"{e}: qx is NULL"),
            (e, "h", {**CONFLICT}, -1, f"{e}: {COMBINE}"),
        ]
    return out


@pytest.fixture(scope="module")
def env(pkg):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((N, D)).astype(np.float32)
    h = pkg.Hnsw(16, N, 16, 64, "DistL2", device=0)
    h.insert_flat(X)
    hp = pkg.Hnsw(16, N, 16, 64, "DistL2", device=0)
    hp.partition([0, 0])
    hp.insert_flat(X)
    rf = h.make_filter(np.arange(0, N, 2, dtype=np.uint64))
    Q = np.ascontiguousarray(X[:NQ] + 0.01)
    arrays = {
        "q": Q, "qids": np.array([0, 1, 2], np.uint64), "qids_far": np.array([0, N, 1], np.uint64),
        "filters": np.array([-1, rf.id, -1], np.int64), "qlabels": np.array([1, 2, 0xFFFFFFFF], np.uint32),
        "ranges": np.array([0, 10, -5, 5, 0, 0], np.int64), "set_off": np.array([0, 1, 2, 3], np.uint64),
        "set_vals": np.array([1, 2, 0xFFFFFFFF], np.uint32), "x_off": np.array([0, 1, 1, 2], np.uint64),
        "xs": np.array([4, 9], np.uint64), "radius": np.array([1.0, 2.0, np.inf], np.float32),
        "radius_nan": np.array([1.0, np.nan, 1.0], np.float32), "radius_neg": np.array([1.0, -1.0, 1.0], np.float32),
    }
    dev = {"dq": torch.from_numpy(Q).cuda(), "dqids": torch.tensor([0, 1, 2], dtype=torch.int64, device="cuda"),
           "dqids_far": torch.tensor([0, N, 1], dtype=torch.int64, device="cuda")}
    yield h, hp, rf, arrays, dev
    rf.free()
    hp.close()
    h.close()


def call(pkg, env, entry, handle="h", overrides=None):
    """the raw C call of `entry` on outputs that hold SENTINEL; returns (return value, last_error(), whether every
    output still holds SENTINEL, the outputs)"""
    h, hp, rf, arrays, dev = env
    named = {"rf": rf.id, **arrays, **dev}
    outs = {"ids": np.full((NQ, K), SENTINEL, np.uint64), "dist": np.full((NQ, K), SENTINEL, np.float32),
            "internal": np.full((NQ, K), SENTINEL, np.uint32), "pid": np.full((NQ, K, 2), SENTINEL, np.int32),
            "counts": np.full(NQ, SENTINEL, np.int32), "out_count": np.full(NQ, SENTINEL, np.uint64),
            "out_exact": np.full(NQ, SENTINEL, np.int32), "out_total": np.full(NQ, SENTINEL, np.uint64),
            "d_out": torch.full((NQ * K * 16,), SENTINEL, dtype=torch.uint8, device="cuda"),
            "d_counts": torch.full((NQ,), SENTINEL, dtype=torch.int32, device="cuda")}
    given = {"h": {"h": h._h, "null": None, "part": hp._h}[handle], "nq": NQ, "dim": D, "k": K, "ef": EF, "mode": 0,
             "fids": None, "nf": 0, "fn": FILTER_FN(0), "ctx": None, "excl": 0, "exact": 0, "sync": 1,
             "kms": None, "filter": -1, "q": "q", "qids": "qids", "filters": "filters", "qlabels": "qlabels",
             "radius": "radius", "dq": "dq", "dqids": "dqids", **{o: o for o in outs}}
    need = REQUIRED.get(entry, set())
    given.update({"filter": "rf"} if "filter" in need else {})
    given.update({"qrange": "ranges"} if "qrange" in need else {})
    given.update({"qset_off": "set_off", "qset": "set_vals"} if "qset" in need else {})
    given.update({"qx_off": "x_off", "qx": "xs"} if "qx" in need else {})
    for a in OPTIONAL - need - {"filter"}:
        given[a] = None
    given.update(overrides or {})

    def value(v):
        if isinstance(v, str) and v in outs:
            v = outs[v]
        elif isinstance(v, str):
            v = named[v]
        if isinstance(v, np.ndarray):
            return v.ctypes.data_as(C.c_void_p)
        if isinstance(v, torch.Tensor):
            return C.c_void_p(v.data_ptr())
        return v

    h._L.hnsw_b200_set_visited_stages(h._h, 9)   # a refusal, so that no message of an earlier call is read
    rc = getattr(h._L, "hnsw_b200_" + entry)(*[value(given[a]) for a in ENTRIES[entry]])
    torch.cuda.synchronize()
    kept = all(np.all(a == SENTINEL) if isinstance(a, np.ndarray) else bool(torch.all(a == SENTINEL))
               for a in outs.values())
    return rc, pkg.last_error(), kept, outs


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_defaults_are_a_valid_call(pkg, env, entry):
    rc, msg, _, _ = call(pkg, env, entry)
    if entry.startswith("search_flat_submit"):
        assert rc >= 0, msg
        assert env[0]._L.hnsw_b200_search_flat_wait(env[0]._h, rc) == 0, pkg.last_error()
    else:
        assert rc == 0, msg


@pytest.mark.parametrize("entry, handle, overrides, rc, msg", rows(),
                         ids=lambda v: v if isinstance(v, str) else None)
def test_entry_checks(pkg, env, entry, handle, overrides, rc, msg):
    got, err, kept, _ = call(pkg, env, entry, handle, overrides)
    assert got == rc, (got, err)
    for part in ([msg] if isinstance(msg, str) else msg or []):
        assert part in err, err
    assert kept


@pytest.mark.parametrize("entry", RADIUS)
def test_radius_counts_only(pkg, env, entry):
    """knbn == 0: the row arrays may be NULL, every count is 0 and the totals are written"""
    got, err, _, outs = call(pkg, env, entry, overrides={"k": 0, "ids": None, "dist": None, "internal": None, "pid": None})
    assert got == 0, err
    assert np.all(outs["counts"] == 0) and np.all(outs["out_total"] != SENTINEL)
