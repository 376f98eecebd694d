"""The exact-scan reference: a handle holding points without a graph, the oracle's exact answers over the points a
restriction admits, float64 distances with their bounds, and the host's choice of exact_knn_kernel's shape (exact_layout,
exact_shape and the slice count S in csrc/aux.cu) restated.

pytest shows the compared values only for asserts in test modules, so every assert here says in its message what it
compared."""
import numpy as np

import distref
from graphs import data

INVALID = 0xFFFFFFFF

# (dtype, metric, d, ties) of the exact searches' oracle parity; their ids are graphs.case_id's
EXACT_CASES = ([(np.float32, m, d, False) for m in ("DistL1", "DistL2", "DistDot", "DistCosine")
                for d in (24, 48, 100, 150)]
               + [(np.uint8, m, 100, False) for m in ("DistL1", "DistL2", "DistHamming", "DistJaccard")]
               + [(np.uint16, m, 200, False) for m in ("DistL1", "DistL2", "DistHamming", "DistJaccard")]
               + [(np.uint32, "DistJaccard", 24, False), (np.int32, "DistL2", 24, False)]
               + [(np.float32, "DistL2", 24, True), (np.float32, "DistCosine", 100, True)])


def origin_ids(n):
    return np.arange(n, dtype=np.uint64) * 5 + 2   # distinct from the internal ids, so a mix-up shows


def handle(pkg, X, metric, ids=None):
    """the points X stored in internal-id order (no graph: the exact search does not read one)"""
    n = len(X)
    h = pkg.Hnsw(8, n, 16, 48, metric, dtype=X.dtype)
    h.import_graph(X, origin_ids(n) if ids is None else ids, np.zeros(n, np.uint8), 0,
                   [(np.zeros(n + 1, np.uint64), np.zeros(0, np.uint32), None)])
    return h


def expected(po, h, X, Q, k, metric, adm):
    """the oracle's exact k nearest among X[adm], as search_exact reports them on handle h"""
    lv, rk, og, _ = h.export_points()
    nq = len(Q)
    o = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    d = np.full((nq, k), np.inf, np.float32)
    it = np.full((nq, k), INVALID, np.uint32)
    pid = np.full((nq, k, 2), -1, np.int32)
    c = min(k, len(adm))
    if c:
        ti, td = po.bruteforce(X[adm], Q, k, metric, po.ORDER_GPU)
        g = adm[ti[:, :c].astype(np.int64)]
        it[:, :c], o[:, :c], d[:, :c] = g, og[g], td[:, :c]
        pid[:, :c, 0], pid[:, :c, 1] = lv[g], rk[g]
    return o, d, it, pid, np.full(nq, c, np.int32)


def filter_sets(n, seed):
    """internal ids admitted: none, one, three, ~5 %, ~50 %, all"""
    rng = np.random.default_rng(seed)
    return {"0": np.zeros(0, np.int64), "1": np.array([n // 2]), "3": np.array([0, n // 3, n - 1]),
            "5%": np.sort(rng.choice(n, n // 20, replace=False)), "50%": np.sort(rng.choice(n, n // 2, replace=False)),
            "all": np.arange(n)}


# ---------------------------------------------------------------- the host's shape choices, restated
SMEM_BUDGET = 220 * 1024   # kernels.h
RING = [(32, 3), (32, 2), (16, 2), (8, 2), (4, 2), (2, 2), (1, 2)]   # aux.cu exact_shape: (rows, stages)


def d4_of(d, dtype):
    """16-byte units of a stored row: dim * element size rounded up to whole 128-byte lines (Index::row_bytes / 16)"""
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


def shape_case_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}-n{c[3]}-nq{c[4]}-k{c[5]}"


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
        assert np.isclose(rv * rv if sq else rv, v[0], rtol=1e-9, atol=1e-12) and np.isclose(rb, b[0], rtol=1e-9, atol=1e-12), \
            f"{what}, row {i}: the block formula gives {v[0]!r} +- {b[0]!r}, distref.reference {rv!r} +- {rb!r} (squared: {sq})"
        g = dist[i, :c].astype(np.float64)
        if F.metric == "DistL2":
            g = g * g
        bad = np.flatnonzero(np.abs(g - v) > b)
        assert not len(bad), f"{what}, row {i}, slot {bad[0]}: got {g[bad[0]]!r}, float64 {v[bad[0]]!r} +- {b[bad[0]]:.3g}"
        kv, kb = F.kth(adm, Q[i], c)
        far = np.flatnonzero(v > kv + b + kb)
        assert not len(far), f"{what}, row {i}, slot {far[0]}: {v[far[0]]!r} is beyond the {c}-th nearest {kv!r}"
