"""Resident filters (include/hnsw_b200.h "Resident filters"): a FilterT materialised once with Hnsw.make_filter and passed
by id to search_flat, submit_flat / wait_flat and search_device.

A search with a resident filter must return, bit for bit, what search_flat returns with the filter arguments it was made
from (ids, distance bits, internal ids, PointIds, counts and traversal counters), and so equal the oracle's filtered
search on the same graph.  Every refusal (stale filter, freed or foreign id, view, partitioned submit / device search)
must leave the handle answering as before."""
import threading
import time

import numpy as np
import pytest
import torch  # device buffers; imported first, so that torch's own NCCL is the one the library binds at run time

from answers import device_answers, same, same_host_device
from exactref import origin_ids
from graphs import data
from util import oracle_layers

pytestmark = pytest.mark.gpu

N, NQ, M, EFC = 2000, 60, 8, 48


def build(pkg, po, dtype, metric, d, n=N, seed=1):
    """an oracle graph (MODE_DET, ORDER_GPU) imported into the engine: the same graph on both sides"""
    X = data(dtype, metric, n, d, seed)
    o = po.Oracle(M, n, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, ids=origin_ids(n))
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    Q = data(dtype, metric, NQ, d, seed + 100)
    Q[: NQ // 10] = X[: NQ // 10]   # stored points: distance-0 answers
    return X, Q, o, h


CASES = [(np.float32, "DistL2", 24), (np.float32, "DistL2", 100), (np.uint8, "DistHamming", 100)]


@pytest.mark.parametrize("dtype,metric,d", CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in CASES])
def test_resident_equals_per_call_and_oracle(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d, seed=d)
    ids = origin_ids(N)
    allow = ids[1::3]
    allowed = set(allow.tolist())
    calls = []

    def fn(i):
        calls.append(i)
        return i in allowed
    by_list = h.make_filter(allow)
    by_fn = h.make_filter(fn)
    assert len(calls) == N and sorted(calls) == sorted(ids.tolist())   # once per stored point, in make_filter
    calls.clear()
    for k in (1, 10, 40):
        for ef in sorted({1, k, 64, 257}):
            want_o = o.search_batch(Q, k, ef, filter_ids=allow)
            for stats in (False, True):
                h.enable_stats(stats)
                h.get_stats()
                per_call = h.search_flat(Q, k, ef, filter=allow)
                s_call = h.get_stats()
                for rf, form in ((by_list, "list"), (by_fn, "callback")):
                    got = h.search_flat(Q, k, ef, filter=rf)
                    s_res = h.get_stats()
                    what = f"{form} k={k} ef={ef} stats={stats}"
                    same(got, per_call, what)
                    if stats:
                        assert s_res == s_call, (what, s_res, s_call)
                go, gd, gi, _, gc = per_call
                assert np.array_equal(gc, want_o[4]) and np.array_equal(gi, want_o[2]), f"oracle k={k} ef={ef}"
                assert np.array_equal(gd.view(np.uint32), want_o[1].view(np.uint32))
    h.enable_stats(False)
    assert calls == []   # no callback during the searches
    # the mirrored single-query API takes it too
    res = h.search_filter(Q[0], 10, 64, filter=by_list)
    go, _, _, _, gc = h.search_flat(Q[:1], 10, 64, filter=allow)
    assert [r.d_id for r in res] == go[0, :gc[0]].tolist()
    by_list.free()
    by_fn.free()


def test_always_false_single_id_and_empty_index(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24)
    with h.make_filter(lambda i: False) as none:
        z = h.search_flat(Q, 10, 64, filter=none)
        assert np.all(z[4] == 0)
        same(z, h.search_flat(Q, 10, 64, filter=lambda i: False), "always false")
    one_id = [int(origin_ids(N)[1234])]
    with h.make_filter(one_id) as one:
        for k, ef in ((10, 4), (1, 1)):
            got = h.search_flat(Q, k, ef, filter=one)
            oo = o.search_batch(Q, k, ef, filter_ids=one_id)
            assert np.all(got[4] <= 1) and np.array_equal(got[4], oo[4]) and np.array_equal(got[2], oo[2])
            same(got, h.search_flat(Q, k, ef, filter=one_id), f"single id k={k} ef={ef}")
    empty = pkg.Hnsw(M, 100, 16, EFC, "DistL2")
    with empty.make_filter([1, 2, 3]) as rf:
        got = empty.search_flat(Q[:, :8], 4, 16, filter=rf)
        assert np.all(got[4] == 0)
        same(got, empty.search_flat(Q[:, :8], 4, 16, filter=[1, 2, 3]), "empty index")
        t = empty.submit_flat(Q[:, :8], 4, 16, filter=rf)
        same(empty.wait_flat(t), got, "empty index, submit")


def test_submit_wait_batches_in_flight(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=3)
    allow = origin_ids(N)[::2]
    batches = [data(np.float32, "DistL2", 200, 24, 50 + b) for b in range(6)]
    with h.make_filter(allow) as rf:
        want = [h.search_flat(B, 10, 64, filter=allow) for B in batches]
        for inflight in (2, 3, 4):
            tickets, got = [], []
            for b, B in enumerate(batches):
                tickets.append(h.submit_flat(B, 10, 64, filter=rf))
                if len(tickets) == inflight:
                    got.append(h.wait_flat(tickets.pop(0)))
            got += [h.wait_flat(t) for t in tickets]
            for b in range(len(batches)):
                same(got[b], want[b], f"{inflight} in flight, batch {b}")


def test_search_device_sync_and_async(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 100, seed=4)
    allow = origin_ids(N)[1::4]
    k, ef = 10, 64
    with h.make_filter(allow) as rf:
        want = h.search_flat(Q, k, ef, filter=allow, with_pid=False)
        q_dev = torch.from_numpy(Q).cuda()
        outs = [torch.empty((NQ, k, 16), dtype=torch.uint8, device="cuda") for _ in range(3)]
        cnts = [torch.empty((NQ,), dtype=torch.int32, device="cuda") for _ in range(3)]
        torch.cuda.synchronize()
        h.search_device(q_dev.data_ptr(), NQ, k, ef, outs[0].data_ptr(), cnts[0].data_ptr(), sync=True, filter=rf)
        same_host_device(want, device_answers(outs[0], cnts[0]), "sync")
        for i in (1, 2):   # two asynchronous launches in flight together, on distinct outputs
            h.search_device(q_dev.data_ptr(), NQ, k, ef, outs[i].data_ptr(), cnts[i].data_ptr(), sync=False, filter=rf)
        h.join()
        assert h.check_status() == 0
        for i in (1, 2):
            same_host_device(want, device_answers(outs[i], cnts[i]), f"async {i}")


def test_refusals_leave_the_handle_unchanged(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, n=1500, seed=5)
    E = pkg.HnswError
    allow = origin_ids(1500)[::3]
    stale = h.make_filter(allow)
    h.insert_flat(data(np.float32, "DistL2", 10, 24, 77), ids=np.arange(10, dtype=np.uint64) + 10 ** 6)
    want = h.search_flat(Q, 10, 64)
    want_f = h.search_flat(Q, 10, 64, filter=allow)
    q_dev = torch.from_numpy(Q).cuda()
    out = torch.empty((NQ, 10, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.empty((NQ,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def unchanged():
        assert h.get_nb_point() == 1510
        same(h.search_flat(Q, 10, 64), want, "after a refused call")
        same(h.search_flat(Q, 10, 64, filter=allow), want_f, "after a refused call, filtered")

    def refused(rf, why):
        for call in (lambda: h.search_flat(Q, 10, 64, filter=rf),
                     lambda: h.search_filter(Q[0], 10, 64, filter=rf),
                     lambda: h.submit_flat(Q, 10, 64, filter=rf),
                     lambda: h.search_device(q_dev.data_ptr(), NQ, 10, 64, out.data_ptr(), cnt.data_ptr(), filter=rf),
                     lambda: h.search_device(q_dev.data_ptr(), NQ, 10, 64, out.data_ptr(), cnt.data_ptr(), sync=False,
                                             filter=rf)):
            with pytest.raises(E, match=why):
                call()
            unchanged()
    refused(stale, "stale")
    fresh = h.make_filter(allow)   # a filter made now covers the new points
    same(h.search_flat(Q, 10, 64, filter=fresh), want_f, "fresh filter")
    fresh.free()
    refused(fresh, "not a live filter")
    L = pkg.load_library()
    assert L.hnsw_b200_filter_free(h._h, fresh.id) < 0   # a second free
    for bad in (-1, 10 ** 12):
        assert L.hnsw_b200_filter_free(h._h, bad) < 0
        refused(pkg.ResidentFilter(h, bad), "not a live filter")
    unchanged()
    other = pkg.Hnsw(M, 1500, 16, EFC, "DistL2")
    other.insert_flat(X, ids=origin_ids(1500))
    foreign = other.make_filter(allow)
    refused(foreign, "not a live filter")
    assert L.hnsw_b200_filter_free(h._h, foreign.id) < 0
    other.search_flat(Q, 10, 64, filter=foreign)   # still alive on its own handle
    foreign.free()
    stale.free()   # a stale filter is still freed
    unchanged()
    assert L.hnsw_b200_filter_new(h._h, 3, None, 0, pkg.hnsw.FILTER_FN(0), None) < 0   # no such filter mode
    assert "filter_mode" in pkg.last_error()
    # a partition view refuses make_filter; a partitioned handle refuses the submit and device variants
    ph = pkg.Hnsw(M, 600, 16, EFC, "DistL2")
    ph.partition([0, 0])
    ph.insert_flat(X[:600], ids=origin_ids(600))
    with pytest.raises(E, match="read-only"):
        ph.partition_view(1).make_filter(allow)
    prf = ph.make_filter(allow)
    pwant = ph.search_flat(Q, 10, 64)
    for call in (lambda: ph.submit_flat(Q, 10, 64, filter=prf),
                 lambda: ph.search_device(q_dev.data_ptr(), NQ, 10, 64, out.data_ptr(), cnt.data_ptr(), filter=prf)):
        with pytest.raises(E, match="partitioned"):
            call()
        same(ph.search_flat(Q, 10, 64), pwant, "partitioned handle after a refused call")
    with pytest.raises(E, match="not a live filter"):   # the view does not know its handle's filters
        ph.partition_view(0).search_flat(Q, 10, 64, filter=prf)
    prf.free()


def test_free_waits_for_the_owners_ticket(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=6)
    allow = origin_ids(N)[::3]
    want = h.search_flat(Q, 10, 64, filter=allow)
    rf = h.make_filter(allow)
    t = h.submit_flat(Q, 10, 64, filter=rf)
    done = threading.Event()
    errs = []

    def free():
        try:
            rf.free()
        except Exception as e:   # noqa: BLE001  (reported below, on the test's thread)
            errs.append(e)
        done.set()
    th = threading.Thread(target=free)
    th.start()
    time.sleep(0.5)
    assert not done.is_set(), "filter_free returned while a submitted batch with the filter was outstanding"
    got = h.wait_flat(t)
    th.join(timeout=30)
    assert done.is_set() and not errs, errs
    same(got, want, "the batch collected while a free was waiting")
    with pytest.raises(pkg.HnswError):
        h.search_flat(Q, 10, 64, filter=pkg.ResidentFilter(h, rf.id))


@pytest.mark.parametrize("P", [1, 2, 3])
def test_partitioned_handle(pkg, po, P):
    X = data(np.float32, "DistL2", N, 24, 8)
    Q = data(np.float32, "DistL2", NQ, 24, 108)
    ids = origin_ids(N)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X, ids=ids)
    allow = ids[1::3]
    allowed = set(allow.tolist())
    calls, threads = [], set()

    def fn(i):
        calls.append(i)
        threads.add(threading.get_ident())
        return i in allowed
    with h.make_filter(allow) as by_list, h.make_filter(fn) as by_fn:
        assert len(calls) == N and sorted(calls) == sorted(ids.tolist()) and threads == {threading.get_ident()}
        calls.clear()
        for k, ef in ((1, 1), (10, 64), (40, 257)):
            want = h.search_flat(Q, k, ef, filter=allow)
            same(h.search_flat(Q, k, ef, filter=by_list), want, f"P={P} list k={k} ef={ef}")
            same(h.search_flat(Q, k, ef, filter=by_fn), want, f"P={P} callback k={k} ef={ef}")
        assert calls == []
        h.insert_flat(X[:P], ids=np.arange(P, dtype=np.uint64) + 10 ** 6)   # every partition grows by one point
        with pytest.raises(pkg.HnswError, match="stale"):
            h.search_flat(Q, 10, 64, filter=by_list)


def test_two_gpus_match_one_with_replicate_after_make_filter(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X, _, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=9)
    Q = data(np.float32, "DistL2", 1000, 24, 109)   # >= 64 per device: sharded
    allow = origin_ids(N)[::3]
    with h.make_filter(allow) as rf:
        one = h.search_flat(Q, 10, 64, filter=rf)
        same(one, h.search_flat(Q, 10, 64, filter=allow), "one GPU")
        h.replicate([0, 1])
        assert h.replica_count() == 1
        same(h.search_flat(Q, 10, 64, filter=rf), one, "two GPUs, search_flat")
        same(h.wait_flat(h.submit_flat(Q, 10, 64, filter=rf)), one, "two GPUs, submit")
