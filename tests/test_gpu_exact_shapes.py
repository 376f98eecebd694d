"""The exact k-NN scan (exact_knn_kernel, csrc/aux.cu) at every tile, ring and split shape its host side can choose.

One kernel answers every exact search and hnsw_b200_bruteforce, the recall ground truth, so a shape where it is wrong
would go unnoticed by any check that takes its ground truth from the same kernel.  Two host choices decide how it runs:
exact_shape picks the tile (tq queries per CTA), the ring (`rows` per block x `stages`) and the shared memory, and
exact_on_ctx picks S, the CTAs that split one tile's points and merge their lists in the kernel.  tests/exactref.py
restates both choices (exact_layout, exact_shape and the slice-count rule), and this module for every launch:
  * checks that the kernel was an exact_knn_kernel instantiation with the shared memory the restatement predicts;
  * predicts S from the SM count and the CTAs per SM the runtime grants (the grid is not reported);
  * compares every answer with the oracle's brute force (ids, distance bits, internal ids, PointIds, counts, padding)
    and with float64 distances (tests/distref.py's formulas and bounds): each returned distance within its bound, and
    no returned point farther than the float64 k-th nearest admitted point plus both bounds.
Each launch adds its (pass, tq, rows, stages, S > 1) to a ledger; test_zz_every_exact_shape_was_reached fails when the
module missed a shape the host can choose."""
import time

import numpy as np
import pytest
import torch  # device buffers; imported first, so that torch's own NCCL is the one the library binds at run time

from answers import device_answers, same, same_host_device
from exactref import (F64, SHAPE_CASES, check_f64, d4_of, exact_shape, exact_slices, expected, handle, origin_ids, points,
                      shape_case_id, stored_queries, tile_points)
from graphs import data

pytestmark = pytest.mark.gpu

T0 = time.time()
LEDGER = set()    # (pass, tq, rows, stages, S > 1) of every launch
EMPTY_SPLIT = []  # tiled launches with S > 1, an empty tile and a tile of fewer points than S
LOG = []          # one line per launch
DONE = []         # cases that ran to the end
NONE = 0xFFFFFFFF  # LABEL_NONE
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FULL = (I64_MIN, I64_MAX)


# ---------------------------------------------------------------- the host's shape choices (exactref), checked
def largest_k(d4, nq):
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if exact_shape(d4, mid, nq) else (lo, mid - 1)
    return lo


def check_launch(pkg, d4, k, groups, what):
    """the launch just made ran exact_knn_kernel with the predicted shared memory; into the ledger with its S"""
    ps, tq, rows, stages, smem = exact_shape(d4, k, max(r for r, _ in groups))
    kern = pkg.last_kernel()
    assert "exact_knn_kernel" in kern, f"{what}: the last kernel was {kern}"
    got, threads, bps = pkg.last_kernel_shape()
    assert (got, threads) == (smem, 256), f"{what}: {got} bytes x {threads} threads, the mirror says {smem} x 256"
    pts = tile_points(groups, tq)
    S = exact_slices(pts, torch.cuda.get_device_properties(0).multi_processor_count * bps)
    LEDGER.add((ps, tq, rows, stages, S > 1))
    if len(groups) > 1 and S > 1 and 0 in pts and any(0 < p < S for p in pts):
        EMPTY_SPLIT.append(what)
    LOG.append(f"{what}: pass {ps} tq {tq} rows {rows} stages {stages} S {S} ({bps} CTA/SM, {smem} B)")


def row_groups(keys, npts):
    """(rows, points) per group of a batch: the unrestricted rows (key None) scan every point, each other distinct key
    is one group over its admitted points"""
    out = {}
    for key, p in zip(keys, npts):
        out.setdefault(key, [0, p])[0] += 1
    return [tuple(v) for v in out.values()]


def half(n, seed):
    return np.sort(np.random.default_rng(seed).choice(n, max(1, n // 2), replace=False))


def exact_call(pkg, po, h, F, X, Q, k, metric, adm, rf, what):
    """search_exact over adm (resident filter rf, or None for every point) against the oracle and float64"""
    got = h.search_exact(Q, k, filter=rf)
    check_launch(pkg, d4_of(X.shape[1], X.dtype), k, [(len(Q), len(adm))], what)
    same(got, expected(po, h, X, Q, k, metric, adm), what)
    check_f64(F, Q, got, k, [adm] * len(Q), what)
    return got


# ---------------------------------------------------------------- shape cases (exactref.SHAPE_CASES)
@pytest.mark.parametrize("dtype,metric,d,n,nq,k", SHAPE_CASES, ids=[shape_case_id(c) for c in SHAPE_CASES])
def test_shape(pkg, po, dtype, metric, d, n, nq, k):
    """every point and ~half of them through search_exact, and every point through bruteforce"""
    X = points(dtype, metric, n, d, d + n)
    Q = stored_queries(X, dtype, metric, nq, d + n + 1)
    h = handle(pkg, X, metric)
    F = F64(X, metric)
    every = np.arange(n)
    want = exact_call(pkg, po, h, F, X, Q, k, metric, every, None, "every point")
    adm = half(n, d)
    with h.make_filter(origin_ids(n)[adm]) as rf:
        exact_call(pkg, po, h, F, X, Q, k, metric, adm, rf, "half the points")
    bi, bd = h.bruteforce(Q, k)
    check_launch(pkg, d4_of(d, dtype), k, [(nq, n)], "bruteforce")
    assert np.array_equal(bi, want[2]) and np.array_equal(bd.view(np.uint32), want[1].view(np.uint32)), "bruteforce"
    DONE.append(shape_case_id((dtype, metric, d, n, nq, k)))


# ---------------------------------------------------------------- split launches: few queries over many points
SPLIT_CASES = [(784, 100), (1024, 1000)]


@pytest.mark.parametrize("d,k", SPLIT_CASES, ids=[f"d{d}-k{k}" for d, k in SPLIT_CASES])
def test_split_launches(pkg, po, d, k):
    """1, 4 and 33 queries over 60 000 points (d = 784: pass 1 at 33 queries; k = 1000: each of the S lists offers k
    keys to the merge), every point and ~half of them"""
    n = 60000
    X = points(np.float32, "DistL2", n, d, d + 5)
    Q = stored_queries(X, np.float32, "DistL2", 33, d + 6)
    h = handle(pkg, X, "DistL2")
    F = F64(X, "DistL2")
    adm = half(n, d + 7)
    with h.make_filter(origin_ids(n)[adm]) as rf:
        for nq in (1, 4, 33):
            exact_call(pkg, po, h, F, X, Q[:nq], k, "DistL2", np.arange(n), None, f"{nq} queries, every point")
            exact_call(pkg, po, h, F, X, Q[:nq], k, "DistL2", adm, rf, f"{nq} queries, half the points")
    DONE.append(f"split d{d} k{k}")


# ---------------------------------------------------------------- tiled launches: a restriction per row
SIZES = [1, 3, 1023, 1024, 1025, 2047, 2049]   # points of labels 1 .. 7; label 8 holds the rest, label 9 none


def labelled(n, seed):
    """labels (1 .. 7 on SIZES random points, 8 on the rest) and attributes (a permutation of -n/2 .. n/2 - 1)"""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n)
    lab = np.full(n, 8, np.uint32)
    at = 0
    for L, s in enumerate(SIZES, 1):
        lab[perm[at:at + s]] = L
        at += s
    return lab, rng.permutation(n).astype(np.int64) - n // 2


def rows_per_query(h, n, lab, attr):
    """three unrestricted rows, then filters of 0, 1, 3, 1023, 1024 (twice), 1025, 2047 and 2049 points"""
    og = origin_ids(n)
    adms = [np.arange(n)] * 3 + [np.zeros(0, np.int64)] + [np.flatnonzero(lab == L) for L in (1, 2, 3, 4, 4, 5, 6, 7)]
    keys = [None] * 3 + [len(a) for a in adms[3:]]   # the sizes differ, but for the two rows of label 4
    made = {key: h.make_filter(og[a]) for key, a in zip(keys[3:], adms[3:])}
    filters = [None if key is None else made[key] for key in keys]
    return (lambda Q, k: h.search_exact_per_query(Q, k, filters)), adms, keys, list(made.values())


def rows_label_sets(h, n, lab, attr):
    """three unrestricted rows, the empty set, a label of no points, each label alone, and sets of several labels that
    are not adjacent (scanned as their slices joined)"""
    sets = [[NONE]] * 3 + [[], [9]] + [[L] for L in range(1, 8)] + [[1, 3, 5], [2, 6, 9], [7, 3, 3], [8]]
    adms = [np.arange(n) if s == [NONE] else np.flatnonzero(np.isin(lab, np.array(s, np.uint32))) for s in sets]
    keys = [None if s == [NONE] else tuple(sorted(set(s))) for s in sets]
    return (lambda Q, k: h.search_exact_label_sets(Q, k, sets)), adms, keys, []


def rows_ranges(h, n, lab, attr):
    """three unrestricted rows, ranges of 0, 1, 3, 1023, 1024, 1025, 2047 and 2049 values, ranges within sets of labels
    that are not adjacent, and a set with the full range"""
    a0 = int(attr.min())
    rg = [FULL] * 3 + [(5, 4)] + [(a0 + 100, a0 + 99 + s) for s in SIZES + [1024]]
    sets = [[NONE]] * len(rg)
    rg += [(-n // 4, n // 4), (0, I64_MAX), FULL]
    sets += [[1, 3, 5], [2, 4, 6, 8], [7]]
    adms, keys = [], []
    for s, r in zip(sets, rg):
        m = np.ones(n, bool) if s == [NONE] else np.isin(lab, np.array(s, np.uint32))
        m &= (attr >= r[0]) & (attr <= r[1])
        adms.append(np.flatnonzero(m))
        plain = s == [NONE] and r == FULL
        keys.append(None if plain else (tuple(s), r if r[0] <= r[1] else "empty"))
    return (lambda Q, k: h.search_exact_ranges(Q, k, np.array(rg, np.int64), sets=sets)), adms, keys, []


TILED_CASES = [(d, kind) for d in (24, 784) for kind in ("per_query", "label_sets", "ranges")]
BIG = {}   # the 60 000 points of one dimension, shared by its three kinds


@pytest.mark.parametrize("d,kind", TILED_CASES, ids=[f"d{d}-{kind}" for d, kind in TILED_CASES])
def test_tiled_and_split(pkg, po, d, kind):
    """one batch of rows with their own restrictions over 60 000 points: unrestricted rows make the widest tile (split),
    the others tiles of 0 .. 2049 points; k = 10 and k = 1100 (padding past the smaller sets).  Each row's admitted
    points come from the labels and attributes set here, and each row must equal the oracle over them."""
    n = 60000
    if d not in BIG:
        BIG.clear()
        X = points(np.float32, "DistL2", n, d, d + 11)
        BIG[d] = X, stored_queries(X, np.float32, "DistL2", 30, d + 12), F64(X, "DistL2"), labelled(n, d)
    X, Q0, F, (lab, attr) = BIG[d]
    h = handle(pkg, X, "DistL2")
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    call, adms, keys, owned = {"per_query": rows_per_query, "label_sets": rows_label_sets,
                               "ranges": rows_ranges}[kind](h, n, lab, attr)
    Q = Q0[:len(adms)]
    groups = row_groups(keys, [len(a) for a in adms])
    for k in (10, 1100):
        got = call(Q, k)
        check_launch(pkg, d4_of(d, np.float32), k, groups, f"{kind} k={k}")
        for i, a in enumerate(adms):
            same(tuple(x[i:i + 1] for x in got), expected(po, h, X, Q[i:i + 1], k, "DistL2", a), f"{kind} k={k} row {i}")
        check_f64(F, Q, got, k, adms, f"{kind} k={k}")
    for f in owned:
        f.free()
    DONE.append(f"tiled d{d} {kind}")


# ---------------------------------------------------------------- limits and other entry points
@pytest.mark.parametrize("d,n", [(784, 30000), (12000, 10500)])
def test_largest_k_and_refusal(pkg, po, d, n):
    """the largest k the restatement admits answers as the oracle does; k + 1 is refused by search_exact and
    bruteforce, and the handle answers as before"""
    nq = 2
    X = points(np.float32, "DistL2", n, d, d + 21)
    Q = stored_queries(X, np.float32, "DistL2", nq, d + 22)
    h = handle(pkg, X, "DistL2")
    k = largest_k(d4_of(d, np.float32), nq)
    got = exact_call(pkg, po, h, F64(X, "DistL2"), X, Q, k, "DistL2", np.arange(n), None, f"largest k = {k}")
    for call in (lambda: h.search_exact(Q, k + 1), lambda: h.bruteforce(Q, k + 1)):
        with pytest.raises(pkg.HnswError, match="k / dimension too large for the exact search kernel"):
            call()
    same(h.search_exact(Q, k), got, "after a refused call")
    bi, bd = h.bruteforce(Q, k)
    assert np.array_equal(bi, got[2]) and np.array_equal(bd.view(np.uint32), got[1].view(np.uint32))
    DONE.append(f"largest k d{d}")


def test_device_variant_at_a_pass1_shape(pkg, po):
    """search_exact_device at (1, 16, 4, 2), synchronous and two asynchronous launches in flight, equals the host call"""
    n, d, nq, k = 3000, 2048, 33, 10
    X = points(np.float32, "DistL2", n, d, 31)
    Q = stored_queries(X, np.float32, "DistL2", nq, 32)
    h = handle(pkg, X, "DistL2")
    adm = half(n, 33)
    with h.make_filter(origin_ids(n)[adm]) as rf:
        for f, a in ((None, np.arange(n)), (rf, adm)):
            want = h.search_exact(Q, k, filter=f, with_pid=False)
            q_dev = torch.from_numpy(Q).cuda()
            outs = [torch.empty((nq, k, 16), dtype=torch.uint8, device="cuda") for _ in range(3)]
            cnts = [torch.empty((nq,), dtype=torch.int32, device="cuda") for _ in range(3)]
            torch.cuda.synchronize()
            h.search_exact_device(q_dev.data_ptr(), nq, k, outs[0].data_ptr(), cnts[0].data_ptr(), sync=True, filter=f)
            check_launch(pkg, d4_of(d, np.float32), k, [(nq, len(a))], "device, sync")
            same_host_device(want, device_answers(outs[0], cnts[0]), "sync")
            for i in (1, 2):
                h.search_exact_device(q_dev.data_ptr(), nq, k, outs[i].data_ptr(), cnts[i].data_ptr(), sync=False, filter=f)
                check_launch(pkg, d4_of(d, np.float32), k, [(nq, len(a))], f"device, async {i}")
            h.join()
            assert h.check_status() == 0
            for i in (1, 2):
                same_host_device(want, device_answers(outs[i], cnts[i]), f"async {i}")
    DONE.append("device")


def test_partitioned_handle_at_a_pass1_shape(pkg, po):
    """two partitions at (1, 16, 4, 2) answer as the unpartitioned handle does (data without ties)"""
    n, d, nq, k = 2000, 2048, 33, 10
    X = data(np.float32, "DistL2", n, d, 41)
    Q = stored_queries(X, np.float32, "DistL2", nq, 42)
    ids = origin_ids(n)
    plain = pkg.Hnsw(8, n, 16, 48, "DistL2")
    plain.insert_flat(X, ids=ids)
    ph = pkg.Hnsw(8, n, 16, 48, "DistL2")
    ph.partition([0, 0])
    ph.insert_flat(X, ids=ids)
    for kk in (1, k, 100):
        a = plain.search_exact(Q, kk, with_pid=False)
        check_launch(pkg, d4_of(d, np.float32), kk, [(nq, n)], f"unpartitioned k={kk}")
        b = ph.search_exact(Q, kk, with_pid=False)
        check_launch(pkg, d4_of(d, np.float32), kk, [(nq, n // 2)], f"partition k={kk}")
        for x, y, what in zip(a, b, ("origin", "dist", "internal", "pid", "counts")):
            if x is not None:
                assert np.array_equal(x, y), (kk, what)
    DONE.append("partitioned")


# ---------------------------------------------------------------- the ledger
def test_zz_every_exact_shape_was_reached():
    want = len(SHAPE_CASES) + len(SPLIT_CASES) + len(TILED_CASES) + 2 + 1 + 1
    if len(DONE) != want:
        pytest.fail(f"the shape ledger needs every case of this module to pass: {len(DONE)} of {want} did")
    print("\nexact shapes (pass, tq, rows, stages, S > 1):\n" + "\n".join(map(str, sorted(LEDGER))))
    print("\n".join(LOG))
    print(f"module wall time {time.time() - T0:.0f} s")
    missing = [f"rows {r}" for r in (32, 16, 8, 4, 2, 1) if not any(s[2] == r for s in LEDGER)]
    missing += [f"{st} stages" for st in (3, 2) if not any(s[3] == st for s in LEDGER)]
    missing += [f"pass {p}" for p in (0, 1) if not any(s[0] == p for s in LEDGER)]
    missing += [f"tq {t}" for t in (32, 16, 8, 4, 3, 2, 1) if not any(s[1] == t for s in LEDGER)]
    if not any(s[0] == 1 and s[4] for s in LEDGER):
        missing.append("S > 1 at a pass-1 shape")
    if not EMPTY_SPLIT:
        missing.append("S > 1 in a tiled launch with an empty tile and a tile of fewer points than S")
    assert not missing, "shapes never launched: " + ", ".join(missing)
