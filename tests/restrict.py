"""Fixtures of the restricted searches (a filter per query, labels, label sets, attribute ranges, excluded lists, deleted
points, search by stored point): the oracle graph they search, the point labels and attributes they assign, the rows of
the ranged searches, the excluded lists and deleted sets they use, the exclude_self rule, and their resident filters."""
import numpy as np

from exactref import INVALID, origin_ids
from graphs import data
from util import oracle_layers

N, M, EFC = 2000, 8, 48
NONE = 0xFFFFFFFF   # LABEL_NONE

GRAPH_CASES = [(np.float32, "DistL2", 128), (np.float32, "DistL2", 100), (np.uint8, "DistHamming", 100),
               (np.uint16, "DistL1", 100), (np.int32, "DistL2", 24)]


def build(pkg, po, dtype, metric, d, nq=300, seed=1, n=N):
    """an oracle graph of n points imported into the engine.  Points 0..399 come in identical pairs, so that a filter
    admitting them has an equal-distance twin for every answer."""
    X = data(dtype, metric, n, d, seed)
    X[1:400:2] = X[0:400:2]
    o = po.Oracle(M, n, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, ids=origin_ids(n))
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    Q = data(dtype, metric, nq, d, seed + 100)
    Q[:20] = X[:40:2]   # stored points with a twin: distance-0 ties
    return X, Q, o, h


def point_labels(n, seed):
    """large labels (0: ~40 %, 1: ~30 %), tiny ones (7: one point, 8: three), the rest without a label"""
    rng = np.random.default_rng(seed)
    lab = rng.choice(np.array([0, 0, 0, 0, 1, 1, 1, 2, NONE, NONE], np.uint32), n)
    lab[lab == 7] = NONE
    lab[rng.choice(n, 4, replace=False)] = [7, 8, 8, 8]
    return lab


I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FULL = (I64_MIN, I64_MAX)   # RANGE_ALL


def point_attrs(n, seed):
    """values in [-1000, 1000) (~20 % of the points without one), one point at INT64_MIN + 1, one at INT64_MAX and one
    at 4242, the only value outside [-1000, 1000)"""
    rng = np.random.default_rng(seed)
    a = rng.integers(-1000, 1000, n, dtype=np.int64)
    a[rng.random(n) < 0.2] = I64_MIN
    i = rng.choice(n, 3, replace=False)
    a[i] = [I64_MIN + 1, I64_MAX, 4242]
    return a


# (label set, range) rows over point_labels and point_attrs: a range alone, with a one-label and a several-label set,
# with an empty set; full ranges with a set and with [LABEL_NONE]; lo > hi; ranges admitting no point, one point (4242)
# and every point with an attribute; bounds at INT64_MIN + 1 and INT64_MAX
ROWS = [([NONE], (-100, 300)), ([0], (0, 500)), ([1, 2, 8], (-500, 499)), ([0, 1], FULL), ([NONE], FULL),
        ([NONE], (10, 5)), ([NONE], (2000, 4000)), ([NONE], (4242, 4242)), ([NONE], (I64_MIN + 1, I64_MAX)),
        ([NONE], (I64_MAX, I64_MAX)), ([NONE], (I64_MIN, I64_MIN + 1)), ([7, 8], (-1000, 999)), ([], (0, 100)),
        ([2], (I64_MIN, 0)), ([NONE], (I64_MIN, I64_MIN))]


def lists_for(po, X, Q, metric, entry, n, seed):
    """excluded lists (insertion ranks): row i's, by kind i % 7, is empty, one id, the query's brute-force top 20, the
    entry point, half of the points, every point, or a random third of the points unsorted with repeats"""
    rng = np.random.default_rng(seed)
    top, _ = po.bruteforce(X, Q, 20, metric, po.ORDER_GPU)
    out = []
    for i in range(len(Q)):
        kind = i % 7
        out.append([np.zeros(0, np.int64), np.array([int(rng.integers(n))]), top[i].astype(np.int64),
                    np.array([entry]), np.sort(rng.choice(n, n // 2, replace=False)), np.arange(n),
                    np.concatenate([x := rng.choice(n, n // 3, replace=False), x[: n // 10]])][kind])
    return out


def deleted_set(po, kind, X, Q, metric, entry, seed=11):
    """insertion ranks to delete: one point, the entry point, the queries' brute-force top 5, a tenth, half, all but
    one, or every point"""
    rng = np.random.default_rng(seed)
    n = len(X)
    if kind == "one":
        return np.array([int(rng.integers(n))])
    if kind == "entry":
        return np.array([entry])
    if kind == "top5":
        return np.unique(po.bruteforce(X, Q, 5, metric, po.ORDER_GPU)[0])
    if kind == "tenth":
        return np.sort(rng.choice(n, n // 10, replace=False))
    if kind == "half":
        return np.sort(rng.choice(n, n // 2, replace=False))
    if kind == "all_but_one":
        return np.delete(np.arange(n), int(rng.integers(n)))
    return np.arange(n)


def minus_self(rows, qids, k):
    """the (k + 1)-wide rows `rows` under the exclude_self rule, k wide"""
    o, d, it, pid, c = rows
    nq = len(qids)
    ro = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    rd = np.full((nq, k), np.inf, np.float32)
    ri = np.full((nq, k), INVALID, np.uint32)
    rp = np.full((nq, k, 2), -1, np.int32)
    rc = np.zeros(nq, np.int32)
    for i in range(nq):
        keep = [j for j in range(c[i]) if it[i, j] != qids[i]][:k]
        n = len(keep)
        ro[i, :n], rd[i, :n], ri[i, :n], rp[i, :n], rc[i] = o[i, keep], d[i, keep], it[i, keep], pid[i, keep], n
    return ro, rd, ri, rp, rc


def unrestricted(s):
    return len(s) > 0 and set(s) == {NONE}


def admitted(lab, attr, s, r):
    """the points a (label set, range) row admits, as a bool mask"""
    m = np.ones(len(attr), bool)
    if not unrestricted(s):
        m &= np.isin(lab, np.array(s, np.uint32))
    if tuple(r) != FULL:
        m &= (attr != I64_MIN) & (attr >= r[0]) & (attr <= r[1])
    return m


def free(rfs):
    for rf in rfs:
        if rf is not None:
            rf.free()
