"""Host search paths: every host entry point writes the same answers.

search_flat (with and without the internal / PointId columns), search_flat with a sorted-list, a callback and a resident
filter, submit / wait with several batches in flight, parallel_search_neighbours and search_neighbours all plan, run and
write a batch through one driver.  On unpartitioned handles and on handles with P = 1, 2 and 3 partitions (on one
device) they must agree bit for bit: all k slots of the flat arrays, padding included, the counts, the first `count`
entries of the Neighbour_api answers, and the traversal counters of get_stats."""
import numpy as np
import pytest

from test_gpu_matrix import data, same

pytestmark = pytest.mark.gpu

N, NQ, M, EFC = 2000, 60, 8, 48
INV = 0xFFFFFFFF
CASES = [(np.float32, "DistL2", 24), (np.uint8, "DistHamming", 100)]


def origin_ids(n):
    return np.arange(n, dtype=np.uint64) * 5 + 2   # distinct from the internal ids, so a mix-up shows


def handle(pkg, dtype, metric, d, P):
    X = data(dtype, metric, N, d, d + P)
    h = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
    if P:
        h.partition([0] * P)
    h.insert_flat(X, ids=origin_ids(N))
    Q = data(dtype, metric, NQ, d, d + 100)
    Q[: NQ // 10] = X[: NQ // 10]   # stored points: distance-0 answers
    return h, Q


def same_columns(got, want, what):
    """search_flat without the optional columns against the full answer"""
    go, gd, gi, gpid, gc = got
    assert gi is None and gpid is None
    assert np.array_equal(gc, want[4]), f"{what}: counts differ"
    assert np.array_equal(go, want[0]), f"{what}: origin ids differ"
    assert np.array_equal(gd.view(np.uint32), want[1].view(np.uint32)), f"{what}: distances are not bit-identical"


def same_nb(lists, want, what):
    """Neighbour_api answers (first count entries) against search_flat's arrays"""
    o, d, _, _, c = want
    assert len(lists) == len(c)
    for q, nb in enumerate(lists):
        assert len(nb) == c[q], f"{what}: count of query {q}"
        assert [n.d_id for n in nb] == o[q, :c[q]].tolist(), f"{what}: ids of query {q}"
        dist = np.array([n.distance for n in nb], np.float32)
        assert np.array_equal(dist.view(np.uint32), d[q, :c[q]].view(np.uint32)), f"{what}: distances of query {q}"


def all_padding(a, what):
    o, d, it, pid, c = a
    assert np.all(c == 0), what
    assert np.all(o == np.iinfo(np.uint64).max) and np.all(np.isinf(d)) and np.all(it == INV) and np.all(pid == -1), what


def submitted(h, Q, k, ef, inflight, filter=None):
    """Q in six batches, `inflight` of them outstanding at a time, the answers concatenated"""
    parts, tickets, got = np.array_split(np.arange(NQ), 6), [], []
    for idx in parts:
        tickets.append(h.submit_flat(Q[idx], k, ef, filter=filter))
        if len(tickets) == inflight:
            got.append(h.wait_flat(tickets.pop(0)))
    got += [h.wait_flat(t) for t in tickets]
    return tuple(np.concatenate([g[i] for g in got]) for i in range(5))


def twice(h, call):
    """call() run twice; the answers and the counters of the second run.  The first run of a shape on a search context
    may overflow its visited table and be re-run on a grown one, and the counters include both runs; the second never
    overflows, so its counters depend on the queries alone."""
    call()
    h.get_stats()
    got = call()
    return got, h.get_stats()


@pytest.mark.parametrize("P", [0, 1, 2, 3], ids=["unpartitioned", "P1", "P2", "P3"])
@pytest.mark.parametrize("dtype,metric,d", CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in CASES])
def test_host_paths_agree(pkg, dtype, metric, d, P):
    h, Q = handle(pkg, dtype, metric, d, P)
    ids = origin_ids(N)
    allow = ids[1::3]
    allowed = set(allow.tolist())
    h.enable_stats(True)
    with h.make_filter(allow) as by_list, h.make_filter(lambda i: i in allowed) as by_fn, \
            h.make_filter([]) as none_list, h.make_filter(lambda i: False) as none_fn:
        for k in (1, 10, 40):
            for ef in sorted({k, 64, 257}):
                at = f"P={P} k={k} ef={ef}"
                want, s = twice(h, lambda: h.search_flat(Q, k, ef))
                calls = [("no columns", lambda: h.search_flat(Q, k, ef, with_internal=False, with_pid=False), same_columns),
                         ("parallel_search_neighbours", lambda: h.parallel_search(list(Q), k, ef), same_nb),
                         ("search_neighbours", lambda: [h.search(q, k, ef) for q in Q], same_nb)]
                if not P:
                    calls += [(f"submit, {n} in flight", lambda n=n: submitted(h, Q, k, ef, n), same) for n in (2, 3, 4)]
                for what, call, check in calls:
                    got, gs = twice(h, call)
                    check(got, want, f"{at} {what}")
                    assert gs == s, f"{at} {what}: stats"
                for fl, fn, fr, what in ((allow, lambda i: i in allowed, (by_list, by_fn), "filter"),
                                         ([], lambda i: False, (none_list, none_fn), "always-false filter")):
                    fw, fs = twice(h, lambda: h.search_flat(Q, k, ef, filter=fl))
                    if fl is not allow:
                        all_padding(fw, f"{at} {what}")
                    calls = [("callback", lambda: h.search_flat(Q, k, ef, filter=fn))]
                    for rf, form in zip(fr, ("list", "callback")):
                        calls.append((f"resident ({form})", lambda rf=rf: h.search_flat(Q, k, ef, filter=rf)))
                        if not P:
                            calls.append((f"submitted, resident ({form})", lambda rf=rf: submitted(h, Q, k, ef, 3, filter=rf)))
                    for form, call in calls:
                        got, gs = twice(h, call)
                        same(got, fw, f"{at} {what}, {form}")
                        assert gs == fs, f"{at} {what}, {form}: stats"
    h.enable_stats(False)
