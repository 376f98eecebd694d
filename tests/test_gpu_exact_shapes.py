"""The exact k-NN scan (exact_knn_kernel, csrc/aux.cu) at every tile, ring and split shape its host side can choose.

One kernel answers every exact search and hnsw_b200_bruteforce, the recall ground truth, so a shape where it is wrong
would go unnoticed by any check that takes its ground truth from the same kernel.  Two host choices decide how it runs:
exact_shape picks the tile (tq queries per CTA), the ring (`rows` per block x `stages`) and the shared memory, and
exact_on_ctx picks S, the CTAs that split one tile's points and merge their lists in the kernel.  This module restates
both choices (exact_layout, exact_shape and the slice-count rule) and for every launch:
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

import distref
from test_gpu_exact import expected, handle, origin_ids
from test_gpu_matrix import data, same
from test_gpu_resident_filter import device_answers, same_host_device

pytestmark = pytest.mark.gpu

T0 = time.time()
LEDGER = set()    # (pass, tq, rows, stages, S > 1) of every launch
EMPTY_SPLIT = []  # tiled launches with S > 1, an empty tile and a tile of fewer points than S
LOG = []          # one line per launch
DONE = []         # cases that ran to the end
NONE = 0xFFFFFFFF  # LABEL_NONE
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FULL = (I64_MIN, I64_MAX)

# ---------------------------------------------------------------- the host's shape choices, restated
SMEM_BUDGET = 220 * 1024   # kernels.h
RING = [(32, 3), (32, 2), (16, 2), (8, 2), (4, 2), (2, 2), (1, 2)]   # aux.cu exact_shape: (rows, stages)


def d4_of(d, dtype):
    """16-byte units of a stored row: dim * element size rounded up to whole 128-byte lines"""
    return (d * np.dtype(dtype).itemsize + 127) // 128 * 8


def layout_bytes(d4, k, tq, rows, stages):
    """exact_layout(...).bytes: [query tile][ring][tq queues of k keys][tq x rows candidates][thresholds][candidate
    counts][queue lengths][stages mbarriers], 128-byte rounded"""
    queue = tq * d4 * 16 + stages * rows * d4 * 16
    cand = queue + tq * k * 8
    qn = cand + tq * rows * 8 + tq * 8 + tq * 4
    bar = (qn + tq * 4 + 15) & ~15
    return (bar + stages * 8 + 127) // 128 * 128


def exact_shape(d4, k, nq):
    """(pass, tq, rows, stages, bytes): the whole tile (up to 32 queries) with a ring of >= 8 rows within half the
    budget, else the largest tile (halving) and ring within the whole budget; None: refused"""
    for ps, budget in ((0, SMEM_BUDGET // 2), (1, SMEM_BUDGET)):
        tq = min(32, nq)
        while tq >= 1:
            for rows, stages in RING:
                if ps == 0 and rows < 8:
                    break
                b = layout_bytes(d4, k, tq, rows, stages)
                if b <= budget:
                    return ps, tq, rows, stages, b
            tq = 0 if ps == 0 else tq // 2
    return None


def largest_k(d4, nq):
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if exact_shape(d4, mid, nq) else (lo, mid - 1)
    return lo


def exact_slices(pts, slots):
    """S for tiles scanning pts points each: the smallest S within 2 % of the least
    cost(S) = max(ceil(tiles * S / slots) * mean, widest) / (S * widest), S <= max(1, min(widest / 1024, 4 slots))"""
    tiles, widest = len(pts), float(max(pts))
    mean = sum(pts) / tiles
    smax = max(1, min(int(widest) // 1024, 4 * slots))

    def cost(S):
        return 1.0 / S if widest <= 0 else max(((tiles * S + slots - 1) // slots) * mean, widest) / (S * widest)
    best = min(cost(S) for S in range(1, smax + 1))
    S = 1
    while cost(S) > best * 1.02:
        S += 1
    return S


def tile_points(groups, tq):
    """points each tile scans, for groups [(rows, points)]: one group is the untiled launch over equal tiles"""
    return [p for r, p in groups for _ in range(-(-r // tq))]


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


# ---------------------------------------------------------------- float64 reference
U = distref.U


class F64:
    """float64 distances of stored points to a query, with tests/distref.py's formulas and bounds (L2 squared)"""

    def __init__(self, X, metric):
        self.X, self.metric, self.d = X, metric, X.shape[1]
        self.step = max(1, (1 << 23) // self.d)   # rows per float64 block (64 MB)
        if metric in ("DistL2", "DistCosine"):
            self.xx = self._rows(np.arange(len(X)), lambda x: (x * x).sum(1))

    def _rows(self, ids, f):
        """f over the float64 rows ids, block by block"""
        s = self.step
        return np.concatenate([f(self.X[ids[b:b + s]].astype(np.float64)) for b in range(0, len(ids), s)] or [np.zeros(0)])

    def exact(self, ids, q):
        d, q64 = self.d, q.astype(np.float64)
        if self.metric == "DistL2":
            s = self._rows(ids, lambda x: ((x - q64) ** 2).sum(1))
            return s, (d + 7) * U * s
        if self.metric == "DistCosine":
            ab, aa, bb = self._rows(ids, lambda x: x @ q64), self.xx[ids], q64 @ q64
            v = np.where((aa > 0) & (bb > 0), np.maximum(0.0, 1.0 - ab / np.sqrt(np.maximum(aa * bb, 1e-300))), 0.0)
            return v, U * v + (d + 8) * 2.0 ** -50
        if self.metric == "DistHamming":
            c = np.count_nonzero(self.X[ids] != q, axis=1).astype(np.float32)
            return (c / np.float32(d)).astype(np.float64), np.zeros(len(ids))
        if self.metric == "DistJaccard":
            mn = np.minimum(self.X[ids], q).sum(1, dtype=np.int64)
            mx = np.maximum(self.X[ids], q).sum(1, dtype=np.int64)
            v = (1.0 - mn / np.maximum(mx, 1)).astype(np.float32).astype(np.float64)
            return np.where(mx == 0, 0.0, v), np.zeros(len(ids))
        raise ValueError(self.metric)

    def kth(self, adm, q, c):
        """(value, bound) of the c-th nearest point of adm"""
        cand = adm
        if self.metric == "DistL2" and len(adm) > 4 * c + 256:   # preselect on |x|^2 - 2 x.q, exact on the survivors
            q64 = q.astype(np.float64)
            a = self.xx[adm] - 2.0 * self._rows(adm, lambda x: x @ q64)
            cut = np.partition(a, c - 1)[c - 1]
            cand = adm[a <= cut + 1e-9 * (self.xx[adm].max() + q64 @ q64)]
        v, b = self.exact(cand, q)
        j = np.argsort(v, kind="stable")[c - 1]
        return v[j], b[j]


def check_f64(F, Q, got, k, adms, what):
    """row i of got against the float64 distances of the points adms[i]"""
    dist, it, cnt = got[1], got[2], got[4]
    for i, adm in enumerate(adms):
        c = min(k, len(adm))
        assert cnt[i] == c, f"{what}, row {i}: count {cnt[i]}, {c} admitted"
        if c == 0:
            continue
        ids = it[i, :c].astype(np.int64)
        assert len(np.unique(ids)) == c and np.isin(ids, adm).all(), f"{what}, row {i}: ids not distinct admitted points"
        v, b = F.exact(ids, Q[i])
        # the block formulas are distref.reference's, applied to many rows at once
        rv, rb, sq = distref.reference(F.X[ids[0]], Q[i], F.metric)
        assert np.isclose(rv * rv if sq else rv, v[0], rtol=1e-9, atol=1e-12) and np.isclose(rb, b[0], rtol=1e-9, atol=1e-12)
        g = dist[i, :c].astype(np.float64)
        if F.metric == "DistL2":
            g = g * g
        bad = np.flatnonzero(np.abs(g - v) > b)
        assert not len(bad), f"{what}, row {i}, slot {bad[0]}: got {g[bad[0]]!r}, float64 {v[bad[0]]!r} +- {b[bad[0]]:.3g}"
        kv, kb = F.kth(adm, Q[i], c)
        far = np.flatnonzero(v > kv + b + kb)
        assert not len(far), f"{what}, row {i}, slot {far[0]}: {v[far[0]]!r} is beyond the {c}-th nearest {kv!r}"


def stored_queries(X, dtype, metric, nq, seed):
    """nq queries, a tenth (at least one) of them stored points: the first is row 10, whose copy is row n - 10"""
    Q = data(dtype, metric, nq, X.shape[1], seed)
    n = len(X)
    for j in range(max(1, nq // 10)):
        Q[j] = X[(10 + 7 * j) % n]
    return Q


def points(dtype, metric, n, d, seed):
    """n points; rows 10 and n - 10 identical, so that a split launch merges equal keys from its first and last slices"""
    X = data(dtype, metric, n, d, seed)
    if n >= 30:
        X[n - 10] = X[10]
    return X


def half(n, seed):
    return np.sort(np.random.default_rng(seed).choice(n, max(1, n // 2), replace=False))


def exact_call(pkg, po, h, F, X, Q, k, metric, adm, rf, what):
    """search_exact over adm (resident filter rf, or None for every point) against the oracle and float64"""
    got = h.search_exact(Q, k, filter=rf)
    check_launch(pkg, d4_of(X.shape[1], X.dtype), k, [(len(Q), len(adm))], what)
    same(got, expected(po, h, X, Q, k, metric, adm), what)
    check_f64(F, Q, got, k, [adm] * len(Q), what)
    return got


# ---------------------------------------------------------------- shape cases
# (dtype, metric, d, n, nq, k); the restatement's (pass, tq, rows, stages) for each
SHAPE_CASES = [
    (np.float32, "DistL2", 24, 3000, 200, 10),       # (0, 32, 32, 3)
    (np.float32, "DistL2", 24, 6000, 3, 5000),       # (1, 3, 32, 3): k of several thousand
    (np.float32, "DistL2", 784, 20000, 32, 10),      # (1, 32, 16, 2): c4's brute force, split
    (np.float32, "DistL2", 784, 15, 4, 100),         # (0, 4, 8, 2), n = rows x stages - 1
    (np.float32, "DistL2", 784, 17, 4, 100),         # n = rows x stages + 1
    (np.float32, "DistL2", 1024, 5, 1, 100),         # (0, 1, 8, 2): fewer points than one ring block
    (np.float32, "DistL2", 1024, 3000, 33, 1000),    # (1, 16, 2, 2)
    (np.float32, "DistL2", 2048, 3000, 33, 1),       # (1, 16, 4, 2)
    (np.float32, "DistL2", 4096, 3000, 3, 10),       # (1, 3, 4, 2)
    (np.float32, "DistL2", 7000, 2000, 33, 10),      # (1, 4, 2, 2)
    (np.float32, "DistL2", 7000, 1400, 200, 100),    # (1, 4, 1, 2)
    (np.float32, "DistL2", 11000, 3000, 1, 10),      # (1, 1, 2, 2)
    (np.float32, "DistL2", 11000, 3000, 2, 10),      # (1, 2, 1, 2)
    (np.float32, "DistL2", 12000, 3000, 3, 10),      # (1, 1, 1, 2)
    (np.float32, "DistCosine", 3000, 3000, 33, 100),  # generic row loop (CH = 0), f64 accumulation
    (np.uint8, "DistHamming", 16384, 3000, 33, 10),   # (1, 8, 2, 2), integer ops on 16 KB rows
    (np.uint8, "DistJaccard", 16384, 3000, 33, 10),
    (np.uint16, "DistL2", 8192, 3000, 33, 10),
]


def case_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}-n{c[3]}-nq{c[4]}-k{c[5]}"


@pytest.mark.parametrize("dtype,metric,d,n,nq,k", SHAPE_CASES, ids=[case_id(c) for c in SHAPE_CASES])
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
    DONE.append(case_id((dtype, metric, d, n, nq, k)))


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
