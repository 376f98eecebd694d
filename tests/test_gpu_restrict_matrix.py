"""Every search restriction at every filtered and exact kernel instantiation, row for row against the oracle.

search_filter_kernel (csrc/filter.cu) and exact_knn_kernel (csrc/aux.cu) are templates over the distance op and the row
chunks CH, and filter.cu picks per op how a row looks up its label set and its excluded list: inlined, or through the
out-of-line in_sorted_call.  One graph per (element type, metric, dimension) reaches every compiled instantiation of
both: f32 L1 / L2 / Dot / Cosine at d = 24 (exact CH = 1, filtered CH = 0), 100 (CH = 4 in both) and 150 (CH = 0, a
partial last chunk column), the f32 probability metrics at d = 150, u8 and u16 at d = 100, u32 and i32 at d = 24.

Each graph is built by the oracle (MODE_DET, ORDER_GPU) with origin ids that differ from the insertion ranks, and
imported (restrict.build: points 0..399 in identical pairs, so that an admitted point can have an equal-distance twin
that is not admitted).  Every restriction then runs on it: a resident filter and a FilterT list, labels, label sets (also
with every point relabelled, and sets of up to 1500 labels), attribute ranges alone and within sets, excluded lists
alone and on top of the others, a filter per query, search by stored point, planned search, and deleted points under
all of them.  Each row must equal, bit for bit, the oracle's over the points it admits: the oracle's graph search under
that filter, or its brute force (exactref.expected); with statistics on, the graph launch's traversal counters must
equal the oracle's.  An unrestricted graph row of an index with deleted points follows the live stop rule, which the
oracle does not model; it is compared with liveref.LiveRef.  Exact rows of the float metrics exactref.F64 has formulas
for are also checked against float64.

Each single-launch call records (last kernel, restriction part).  test_zz_every_restricted_kernel_part_was_reached
compares that ledger with the entry points `cuobjdump -symbols` lists: every search_filter_kernel must have run under
each filtered part, and every exact_knn_kernel under each exact part."""
import re
import subprocess
import time

import numpy as np
import pytest

from answers import same
from exactref import F64, check_f64, expected, origin_ids
from graphs import cuobjdump
from liveref import LiveRef
from restrict import (FULL, NONE, ROWS, admitted, build, deleted_set, free, lists_for, minus_self, point_attrs,
                      point_labels, unrestricted)

pytestmark = pytest.mark.gpu

T0 = time.time()
N, NQ = 1500, 35
LIVE = np.arange(12, 28)   # the rows a live reference runs on: 8 stored points with a twin, 8 others
GRID = [(1, 1), (10, 32), (10, 65), (40, 129), (10, 257)]
LIVE_GRID = GRID[:3]
KS = (1, 10, 40)
INT_OPS = ["DistL1", "DistL2", "DistHamming", "DistJaccard"]
CASES = ([(np.float32, m, d) for m in ("DistL1", "DistL2", "DistDot", "DistCosine") for d in (24, 100, 150)]
         + [(np.float32, m, 150) for m in ("DistHellinger", "DistJeffreys", "DistJensenShannon")]
         + [(dt, m, d) for dt, d in ((np.uint8, 100), (np.uint16, 100), (np.uint32, 24)) for m in INT_OPS]
         + [(np.int32, m, 24) for m in INT_OPS[:3]])
F64_METRICS = ("DistL2", "DistCosine", "DistHellinger", "DistJeffreys", "DistJensenShannon")   # f32: exactref.F64's
FILTERED, EXACT = "search_filter_kernel", "exact_knn_kernel"
FILTERED_PARTS = ("bitmap", "label", "set", "range", "excluded", "deleted", "live")
EXACT_PARTS = ("list", "excluded", "deleted")
LEDGER = set()   # (mangled kernel name, part)
DONE = []        # ids of the cases that ran to the end
# label sets by row: empty, one label (large, tiny, absent), several, unsorted with repeats, [LABEL_NONE]
SETS = [[], [0], [1, 2, 8], [8, 7, 8, 1, 7], [NONE], [5], [2, 5, 6], [7], [0, 1, 2, 7, 8]]
LABELS = [0, 1, 7, 8, 5, NONE]


def case_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}"


def groups(adms):
    """(rows, admitted ids or None) per distinct admitted set of adms, None (unrestricted) included"""
    at = {}
    for i, a in enumerate(adms):
        at.setdefault(None if a is None else np.asarray(a, np.int64).tobytes(), (a, []))[1].append(i)
    return [(np.array(rows), None if a is None else np.asarray(a, np.int64)) for a, rows in at.values()]


def empty_rows(nq, k):
    return [np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32), np.empty((nq, k), np.uint32),
            np.empty((nq, k, 2), np.int32), np.empty(nq, np.int32)]


def set_adm(lab, s):
    return None if unrestricted(s) else np.flatnonzero(np.isin(lab, np.asarray(s, np.int64)))


def minus(adm, lst, n=N):
    """adm (None: every point) without the ranks lst; None when that leaves the row unrestricted"""
    lst = np.asarray(lst, np.int64)
    if adm is None and lst.size == 0:
        return None
    return np.setdiff1d(np.arange(n) if adm is None else adm, lst)


def pick(ex, x, g):
    """row i of x where ex[i], else of g"""
    return tuple(np.where(ex.reshape((-1,) + (1,) * (a.ndim - 1)) != 0, b, a) for a, b in zip(g, x))


class Case:
    """one oracle graph imported into the engine, its labels and attributes, and the oracle's rows over any admitted
    sets, minus the points deleted at the time"""

    def __init__(self, pkg, po, dtype, metric, d):
        seed = d + 31 * CASES.index((dtype, metric, d))
        self.pkg, self.po, self.metric = pkg, po, metric
        self.X, self.Q, self.o, self.h = build(pkg, po, dtype, metric, d, nq=NQ, seed=seed, n=N)
        self.og = origin_ids(N)
        self.lab, self.attr = point_labels(N, seed), point_attrs(N, seed)
        self.h.set_labels(0, self.lab)
        self.h.set_attributes(0, self.attr)
        self.h.enable_stats(True)
        self.F = F64(self.X, metric) if np.dtype(dtype) == np.float32 and metric in F64_METRICS else None
        self.ref = LiveRef(po, self.o, self.X, metric)
        self.dead = np.zeros(0, np.int64)
        self.live_rows = {}
        self.seed = seed

    def delete(self, dead):
        self.h.delete_points(dead)
        self.dead = np.asarray(dead, np.int64)
        self.live_rows = {}

    def restore(self):
        self.h.restore_points(self.dead)
        assert self.h.nb_deleted() == 0
        self.dead = np.zeros(0, np.int64)
        self.live_rows = {}

    def live(self, q, k, ef):
        """LiveRef's live row of query q over the points not deleted, and its counters, computed once"""
        key = (q.tobytes(), k, ef)
        if key not in self.live_rows:
            keep = np.ones(N, bool)
            keep[self.dead] = False
            self.live_rows[key] = self.ref.batch(q[None], k, ef, keep, live=True)
        return self.live_rows[key]

    def graph_want(self, Q, k, ef, adms):
        """the oracle's rows of Q under adms (None: unrestricted) and their summed traversal counters"""
        out = empty_rows(len(Q), k)
        tot = {"evals": 0, "expansions": 0, "adj_read": 0}
        for rows, adm in groups(adms):
            if adm is None and len(self.dead):
                parts = [self.live(Q[r], k, ef) for r in rows]
                res = tuple(np.concatenate([p[0][j] for p in parts]) for j in range(5))
                cnt = {key: sum(p[1][key] for p in parts) for key in tot}
            else:
                self.o.counters()
                res = (self.o.search_batch(Q[rows], k, ef) if adm is None else
                       self.o.search_batch(Q[rows], k, ef, filter_ids=self.og[np.setdiff1d(adm, self.dead)]))
                cnt = self.o.counters()
            for a, r in zip(out, res):
                a[rows] = r
            for key in tot:
                tot[key] += cnt[key]
        return tuple(out), tot

    def exact_adms(self, adms):
        return [np.setdiff1d(np.arange(N) if a is None else a, self.dead) for a in adms]

    def exact_want(self, Q, k, adms):
        out = empty_rows(len(Q), k)
        for rows, adm in groups(self.exact_adms(adms)):
            for a, r in zip(out, expected(self.po, self.h, self.X, Q[rows], k, self.metric, adm)):
                a[rows] = r
        return tuple(out)

    def record(self, family, parts):
        kern = self.pkg.last_kernel()
        if family in kern:
            LEDGER.update((kern, p) for p in parts + (("deleted",) if len(self.dead) else ()))

    def graph(self, what, call, adms, parts, Q=None, grid=GRID, width=0, qids=None):
        """call(k, ef) against the oracle over adms, with its counters; width 1 with qids: the exclude_self rule"""
        Q = self.Q if Q is None else Q
        for k, ef in grid:
            tag = f"{what} k={k} ef={ef}"
            self.h.get_stats()
            got = call(k, ef)
            self.record(FILTERED, parts)
            st = self.h.get_stats()
            want, cnt = self.graph_want(Q, k + width, ef, adms)
            same(got, want if qids is None else minus_self(want, qids, k), tag)
            if st["queries"] == len(Q):   # a launch re-run after a visited-table overflow counts its work twice
                for key in cnt:
                    assert st[key] == cnt[key], (tag, key, st, cnt)

    def exact(self, what, call, adms, parts, Q=None, ks=KS, width=0, qids=None):
        Q = self.Q if Q is None else Q
        for k in ks:
            tag = f"{what} exact k={k}"
            got = call(k)
            self.record(EXACT, parts)
            want = self.exact_want(Q, k + width, adms)
            same(got, want if qids is None else minus_self(want, qids, k), tag)
            if self.F is not None and qids is None:
                check_f64(self.F, Q, got, k, self.exact_adms(adms), tag)


def restricted(c):
    """every restriction on an index without deleted points"""
    h, Q, lab, attr, og = c.h, c.Q, c.lab, c.attr, c.og
    nq = len(Q)
    rng = np.random.default_rng(c.seed)
    third = np.sort(rng.choice(N, N // 3, replace=False))
    tiny = np.array([0, 1, 777])   # a twin pair and one more point
    half = np.sort(rng.choice(N, N // 2, replace=False))
    rf, rf_tiny, rf_half = (h.make_filter(og[a]) for a in (third, tiny, half))
    # 1. a bitmap: a resident filter and the same set as a FilterT list of origin ids
    c.graph("resident filter", lambda k, ef: h.search_flat(Q, k, ef, filter=rf), [third] * nq, ("bitmap",))
    c.graph("FilterT", lambda k, ef: h.search_flat(Q, k, ef, filter=og[third]), [third] * nq, ("bitmap",))
    c.exact("resident filter", lambda k: h.search_exact(Q, k, filter=rf), [third] * nq, ("list",))
    # 2. labels: large, tiny, absent, LABEL_NONE
    labels = np.array([LABELS[i % len(LABELS)] for i in range(nq)], np.uint32)
    adms = [set_adm(lab, [x]) for x in labels]
    c.graph("labels", lambda k, ef: h.search_flat_labeled(Q, k, ef, labels), adms, ("label",))
    c.exact("labels", lambda k: h.search_exact_labeled(Q, k, labels), adms, ("list",))
    # 3. label sets, then every point its own label and sets of 37, 1000 and 1500 labels with absent values
    sets = [SETS[i % len(SETS)] for i in range(nq)]
    adms = [set_adm(lab, s) for s in sets]
    c.graph("label sets", lambda k, ef: h.search_flat_label_sets(Q, k, ef, sets), adms, ("set", "label"))
    c.exact("label sets", lambda k: h.search_exact_label_sets(Q, k, sets), adms, ("list",))
    own = (0xFFFFFFFE - 3 * np.arange(N, dtype=np.int64)).astype(np.uint32)   # rank 0: the largest valid label
    h.set_labels(0, own)

    def wide(size):
        present = rng.choice(own, size * 2 // 3, replace=False)
        absent = rng.choice(own.astype(np.int64) - 1, size - len(present), replace=False)
        return rng.permutation(np.concatenate([present.astype(np.int64), absent]))
    big = [wide(37), wide(1000), wide(1500), [int(own[0])], [int(own[5]), int(own[700]), int(own[5])], [],
           np.concatenate([wide(37), [int(own[0])]])]
    wsets = [big[i % len(big)] for i in range(nq)]
    adms = [set_adm(own, s) for s in wsets]
    c.graph("own labels", lambda k, ef: h.search_flat_label_sets(Q, k, ef, wsets), adms, ("set", "label"))
    c.exact("own labels", lambda k: h.search_exact_label_sets(Q, k, wsets), adms, ("list",))
    h.set_labels(0, lab)
    # 4. ranges, alone and within label sets
    rows = [ROWS[i % len(ROWS)] for i in range(nq)]
    rg = np.array([r for _, r in rows], np.int64)
    alone = [None if tuple(r) == FULL else np.flatnonzero(admitted(lab, attr, [NONE], r)) for _, r in rows]
    c.graph("ranges", lambda k, ef: h.search_flat_ranges(Q, k, ef, rg), alone, ("range",))
    c.exact("ranges", lambda k: h.search_exact_ranges(Q, k, rg), alone, ("list",))
    rsets = [s for s, _ in rows]
    within = [None if unrestricted(s) and tuple(r) == FULL else np.flatnonzero(admitted(lab, attr, s, r))
              for s, r in rows]
    c.graph("ranges in sets", lambda k, ef: h.search_flat_ranges(Q, k, ef, rg, rsets), within, ("range", "set", "label"))
    c.exact("ranges in sets", lambda k: h.search_exact_ranges(Q, k, rg, rsets), within, ("list",))
    # 5. excluded lists: alone, on sets, on ranges within sets, on a resident filter
    lists = lists_for(c.po, c.X, Q, c.metric, c.o.entry, N, c.seed + 1)
    for name, kw, base, parts in (("alone", {}, [None] * nq, ()),
                                  ("sets", {"sets": sets}, [set_adm(lab, s) for s in sets], ("set", "label")),
                                  ("ranges in sets", {"sets": rsets, "ranges": rg}, within, ("range", "set", "label")),
                                  ("filter", {"filter": rf}, [third] * nq, ("bitmap",))):
        adms = [minus(a, x) for a, x in zip(base, lists)]
        c.graph(f"excluded, {name}", lambda k, ef: h.search_flat_excluding(Q, k, ef, lists, **kw), adms,
                ("excluded",) + parts)
        c.exact(f"excluded, {name}", lambda k: h.search_exact_excluding(Q, k, lists, **kw), adms,
                ("excluded",) + (("list",) if parts else ()))
    # 6. a filter per query, None rows mixed in
    filters = [[rf, None, rf_tiny, rf_half][i % 4] for i in range(nq)]
    fadm = {id(rf): third, id(rf_tiny): tiny, id(rf_half): half}
    adms = [None if f is None else fadm[id(f)] for f in filters]
    c.graph("per query", lambda k, ef: h.search_flat_per_query(Q, k, ef, filters), adms, ("bitmap",))
    c.exact("per query", lambda k: h.search_exact_per_query(Q, k, filters), adms, ("list",))
    # 8. by stored point under a set, with and without exclude_self: the oracle's row of X[qid] (k + 1 wide, without
    # the point, for exclude_self)
    qids = np.concatenate([[0, 1, 2, 3, c.o.entry, N - 1], rng.choice(N, nq - 6, replace=False)]).astype(np.uint64)
    QX = c.X[qids.astype(np.int64)]
    adms = [set_adm(lab, s) for s in sets]
    for xs in (False, True):
        c.graph(f"by id, exclude_self={xs}",
                lambda k, ef: h.search_by_id(qids, k, ef, sets=sets, exclude_self=xs), adms, ("set", "label"), Q=QX,
                width=int(xs), qids=qids if xs else None)
        c.exact(f"by id, exclude_self={xs}", lambda k: h.search_exact_by_id(qids, k, sets=sets, exclude_self=xs), adms,
                ("list",), Q=QX, width=int(xs), qids=qids if xs else None)
    # 9. planned, with sets and lists: each row the oracle's graph row or its exact row, as out_exact says
    adms = [minus(set_adm(lab, s), x) for s, x in zip(sets, lists)]
    for k, ef in GRID:
        got = h.search_planned(Q, k, ef, lists, sets=sets)
        want = pick(got[5], c.exact_want(Q, k, adms), c.graph_want(Q, k, ef, adms)[0])
        same(got[:5], want, f"planned k={k} ef={ef}")
    free([rf, rf_tiny, rf_half])


def deleted(c):
    """three deleted sets in turn (the entry point, the queries' top 5, half of the points) under the restrictions"""
    h, Q, lab, attr, og = c.h, c.Q, c.lab, c.attr, c.og
    nq = len(Q)
    QL = Q[LIVE]
    rng = np.random.default_rng(c.seed + 2)
    third = np.sort(rng.choice(N, N // 3, replace=False))
    rf = h.make_filter(og[third])
    lists = lists_for(c.po, c.X, Q, c.metric, c.o.entry, N, c.seed + 3)
    sets = [SETS[i % len(SETS)] for i in range(nq)]
    rows = [r for r in ROWS if not (unrestricted(r[0]) and tuple(r[1]) == FULL)]
    rows = [rows[i % len(rows)] for i in range(nq)]
    rg, rsets = np.array([r for _, r in rows], np.int64), [s for s, _ in rows]
    within = [np.flatnonzero(admitted(lab, attr, s, r)) for s, r in rows]
    for kind in ("entry", "top5", "half"):
        c.delete(deleted_set(c.po, kind, c.X, QL, c.metric, c.o.entry))
        # unrestricted rows: live rows; then one launch of live rows and restricted ones (sets, a filter per query)
        c.graph(f"{kind}: live", lambda k, ef: h.search_flat(QL, k, ef), [None] * len(QL), ("live",), Q=QL,
                grid=LIVE_GRID)
        ls = [sets[i] for i in LIVE]
        c.graph(f"{kind}: live and sets", lambda k, ef: h.search_flat_label_sets(QL, k, ef, ls),
                [set_adm(lab, s) for s in ls], ("live", "set", "label"), Q=QL, grid=LIVE_GRID)
        lf = [rf if i % 2 else None for i in range(len(QL))]
        c.graph(f"{kind}: live and per query", lambda k, ef: h.search_flat_per_query(QL, k, ef, lf),
                [third if f is not None else None for f in lf], ("live", "bitmap"), Q=QL, grid=LIVE_GRID)
        # restricted rows: the oracle over the admitted points minus the deleted ones
        adms = [minus(third, x) for x in lists]
        c.graph(f"{kind}: filter, excluded", lambda k, ef: h.search_flat_excluding(Q, k, ef, lists, filter=rf), adms,
                ("bitmap", "excluded"))
        c.graph(f"{kind}: ranges in sets", lambda k, ef: h.search_flat_ranges(Q, k, ef, rg, rsets), within,
                ("range", "set", "label"))
        labels = np.array([LABELS[i % (len(LABELS) - 1)] for i in range(nq)], np.uint32)
        c.graph(f"{kind}: labels", lambda k, ef: h.search_flat_labeled(Q, k, ef, labels),
                [set_adm(lab, [x]) for x in labels], ("label",))
        # exact rows: unrestricted, with lists on sets, and ranges in sets
        c.exact(f"{kind}: unrestricted", lambda k: h.search_exact(Q, k), [None] * nq, ())
        c.exact(f"{kind}: excluded, sets", lambda k: h.search_exact_excluding(Q, k, lists, sets=sets),
                [minus(set_adm(lab, s), x) for s, x in zip(sets, lists)], ("excluded", "list"))
        c.exact(f"{kind}: ranges in sets", lambda k: h.search_exact_ranges(Q, k, rg, rsets), within, ("list",))
        c.restore()
    rf.free()


@pytest.mark.parametrize("dtype,metric,d", CASES, ids=[case_id(c) for c in CASES])
def test_restrictions_against_the_oracle(pkg, po, dtype, metric, d):
    c = Case(pkg, po, dtype, metric, d)
    restricted(c)
    deleted(c)
    DONE.append(case_id((dtype, metric, d)))


def test_zz_every_restricted_kernel_part_was_reached(pkg):
    if len(DONE) != len(CASES):
        pytest.fail(f"the ledger needs every case of this module to pass: {len(DONE)} of {len(CASES)} did")
    exe = cuobjdump()
    if exe is None:
        pytest.fail("cuobjdump (CUDA toolkit) not found: the compiled kernel list cannot be read")
    out = subprocess.run([exe, "-symbols", pkg.lib_path()], capture_output=True, text=True, check=True).stdout
    compiled = set(re.findall(r"STO_ENTRY\s+(\S+)", out))
    filtered = sorted(k for k in compiled if FILTERED in k)
    exact = sorted(k for k in compiled if EXACT in k)
    assert len(filtered) >= 26 and len(exact) >= 30, f"{len(filtered)} filtered and {len(exact)} exact entry points"
    stray = {k for k, _ in LEDGER} - compiled
    assert not stray, f"recorded kernels that cuobjdump does not list: {sorted(stray)}"
    missed = [f"{k} {p}" for family, parts in ((filtered, FILTERED_PARTS), (exact, EXACT_PARTS))
              for k in family for p in parts if (k, p) not in LEDGER]
    print(f"\nrestriction ledger: {len(filtered)} search_filter_kernel entry points under {len(FILTERED_PARTS)} parts, "
          f"{len(exact)} exact_knn_kernel entry points under {len(EXACT_PARTS)} parts, {len(missed)} pairs missed; "
          f"module wall time {time.time() - T0:.0f} s")
    assert not missed, f"{len(missed)} (kernel, part) pairs never ran:\n" + "\n".join(missed)
