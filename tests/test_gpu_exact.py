"""Exact search (include/hnsw_b200.h "Exact search"): Hnsw.search_exact / search_exact_device, the exact k nearest
neighbours among the points a resident filter admits, or among every point.

Every answer must equal the oracle's brute force over the admitted points (ORDER_GPU sums) mapped back to the handle's
ids: origin ids, distance bits, internal ids, PointIds and counts, with (~0, +inf, INVALID_ID, (-1, -1)) past the count.
The kernel may split a batch's points over several CTAs and merge their lists in the kernel; both shapes must agree.
hnsw_b200_bruteforce runs the same kernel, so its answers and its instantiation must match too."""
import numpy as np
import pytest
import torch  # device buffers; imported first, so that torch's own NCCL is the one the library binds at run time

from answers import device_answers, same, same_host_device
from exactref import EXACT_CASES, INVALID, expected, filter_sets, handle, origin_ids
from graphs import case_id, data

pytestmark = pytest.mark.gpu

N, NQ, M = 1500, 40, 8


@pytest.mark.parametrize("dtype,metric,d,ties", EXACT_CASES, ids=[case_id(c) for c in EXACT_CASES])
def test_exact_equals_oracle(pkg, po, dtype, metric, d, ties):
    X = data(dtype, metric, N, d, d + 3, ties)
    Q = data(dtype, metric, NQ, d, d + 103)
    Q[: NQ // 10] = X[: NQ // 10]   # stored points: distance-0 answers
    h = handle(pkg, X, metric)
    og = origin_ids(N)
    for name, adm in filter_sets(N, d).items():
        with h.make_filter(og[adm]) as rf:
            for k in sorted({1, 10, 40, 128, len(adm) + 2}):
                same(h.search_exact(Q, k, filter=rf), expected(po, h, X, Q, k, metric, adm), f"filter {name} k={k}")
    for k in (1, 10, 40, 128, N + 5):
        same(h.search_exact(Q, k), expected(po, h, X, Q, k, metric, np.arange(N)), f"every point k={k}")


@pytest.mark.parametrize("metric", ["DistHellinger", "DistJeffreys", "DistJensenShannon"])
def test_probability_metrics(pkg, po, metric):
    """the device's logf and the oracle's std::log may differ in the last bit: 1e-5 relative on distances and >= 99 %
    identical ids, as the kernel matrix allows"""
    rng = np.random.default_rng(5)
    X = rng.random((N, 32), dtype=np.float32) + np.float32(1e-3)
    X /= X.sum(1, keepdims=True)
    Q = rng.random((NQ, 32), dtype=np.float32) + np.float32(1e-3)
    Q /= Q.sum(1, keepdims=True)
    h = handle(pkg, X, metric)
    adm = filter_sets(N, 1)["50%"]
    with h.make_filter(origin_ids(N)[adm]) as rf:
        got, want = h.search_exact(Q, 10, filter=rf), expected(po, h, X, Q, 10, metric, adm)
    ok = got[2] == want[2]
    assert ok.mean() >= 0.99
    assert np.allclose(got[1][ok], want[1][ok], rtol=1e-5, atol=1e-7)
    assert np.array_equal(got[4], want[4])


def test_split_and_unsplit_launches_agree(pkg, po):
    """A few queries over 60 000 points split the points over many CTAs and merge their lists in the kernel; a filter
    that admits fewer than 2 048 points is never split (a slice keeps >= 1 024 points).  Both must equal the oracle,
    and a 9 000-query batch (many query tiles, split only to even out its last wave) must give the few queries' answers."""
    n, d = 60000, 24
    X = data(np.float32, "DistL2", n, d, 21)
    Q = data(np.float32, "DistL2", 9000, d, 22)
    h = handle(pkg, X, "DistL2")
    sets = filter_sets(n, 2)
    small = sets["5%"][:1500]
    with h.make_filter(origin_ids(n)[sets["50%"]]) as half, h.make_filter(origin_ids(n)[small]) as few_pts:
        for k in (10, 100):
            for f, a in ((None, np.arange(n)), (half, sets["50%"]), (few_pts, small)):
                few = h.search_exact(Q[:4], k, filter=f)
                same(few, expected(po, h, X, Q[:4], k, "DistL2", a), f"{len(a)} points, 4 queries, k={k}")
                many = h.search_exact(Q, k, filter=f)
                same(tuple(x[:4] for x in many), few, f"{len(a)} points, 9000 queries, k={k}")


def test_bruteforce_runs_the_same_kernel(pkg, po):
    """hnsw_b200_bruteforce at the largest k the earlier brute-force kernel accepted at d = 24
    (((d4 * 16 + 256 + 8k + 15) & ~15) * 8 <= 220 KB: k = 3472), against the oracle; and search_exact runs the
    instantiation bruteforce runs"""
    n, d, k = 5000, 24, 3472
    X = data(np.float32, "DistL2", n, d, 31)
    Q = data(np.float32, "DistL2", 8, d, 32)
    h = handle(pkg, X, "DistL2")
    bi, bd = h.bruteforce(Q, k)
    ti, td = po.bruteforce(X, Q, k, "DistL2", po.ORDER_GPU)
    assert np.array_equal(bi, ti) and np.array_equal(bd.view(np.uint32), td.view(np.uint32))
    h.bruteforce(Q, 10)
    kern = pkg.last_kernel()
    assert "exact_knn_kernel" in kern
    h.search_exact(Q, 10)
    assert pkg.last_kernel() == kern


def test_device_variant_sync_and_async(pkg, po):
    n, d, k = 20000, 100, 10
    X = data(np.float32, "DistL2", n, d, 41)
    Q = data(np.float32, "DistL2", 300, d, 42)
    h = handle(pkg, X, "DistL2")
    nq = len(Q)
    with h.make_filter(origin_ids(n)[filter_sets(n, 3)["5%"]]) as rf:
        for f in (None, rf):
            want = h.search_exact(Q, k, filter=f, with_pid=False)
            q_dev = torch.from_numpy(Q).cuda()
            outs = [torch.empty((nq, k, 16), dtype=torch.uint8, device="cuda") for _ in range(3)]
            cnts = [torch.empty((nq,), dtype=torch.int32, device="cuda") for _ in range(3)]
            torch.cuda.synchronize()
            h.search_exact_device(q_dev.data_ptr(), nq, k, outs[0].data_ptr(), cnts[0].data_ptr(), sync=True, filter=f)
            same_host_device(want, device_answers(outs[0], cnts[0]), "sync")
            for i in (1, 2):   # two asynchronous launches in flight together, on distinct outputs
                h.search_exact_device(q_dev.data_ptr(), nq, k, outs[i].data_ptr(), cnts[i].data_ptr(), sync=False, filter=f)
            h.join()
            assert h.check_status() == 0
            for i in (1, 2):
                same_host_device(want, device_answers(outs[i], cnts[i]), f"async {i}")


def test_empty_index(pkg, po):
    h = pkg.Hnsw(M, 100, 16, 48, "DistL2")
    Q = data(np.float32, "DistL2", 5, 24, 1)
    o, d, it, pid, cnt = h.search_exact(Q, 10)
    assert np.all(cnt == 0) and np.all(it == INVALID) and np.all(np.isinf(d))


@pytest.mark.parametrize("P", [1, 2, 3])
def test_partitioned_handle(pkg, po, P):
    """partitions merged by (distance, partition, position) with global ranks: on data without ties, the answers of the
    unpartitioned handle; a partition view answers over its own points with its local ids"""
    X = data(np.float32, "DistL2", N, 24, 51)
    Q = data(np.float32, "DistL2", NQ, 24, 52)
    ids = origin_ids(N)
    plain = pkg.Hnsw(M, N, 16, 48, "DistL2")
    plain.insert_flat(X, ids=ids)
    ph = pkg.Hnsw(M, N, 16, 48, "DistL2")
    ph.partition([0] * P)
    ph.insert_flat(X, ids=ids)
    adm = filter_sets(N, 4)["50%"]
    with plain.make_filter(ids[adm]) as rp, ph.make_filter(ids[adm]) as rq:
        for k in (1, 10, 40):
            for fp, fq in ((None, None), (rp, rq)):
                a = plain.search_exact(Q, k, filter=fp, with_pid=False)
                b = ph.search_exact(Q, k, filter=fq, with_pid=False)
                for x, y, what in zip(a, b, ("origin", "dist", "internal", "pid", "counts")):
                    if x is not None:
                        assert np.array_equal(x, y), (P, k, what)
    v = ph.partition_view(0)
    Xp = X[0::P]
    got = v.search_exact(Q, 10)
    ti, td = po.bruteforce(Xp, Q, 10, "DistL2", po.ORDER_GPU)
    assert np.array_equal(got[2], ti) and np.array_equal(got[1].view(np.uint32), td.view(np.uint32))
    assert np.array_equal(got[0], ids[0::P][ti])


def test_two_gpus_match_one(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X = data(np.float32, "DistL2", N, 24, 61)
    Q = data(np.float32, "DistL2", 1000, 24, 62)   # >= 64 per device: sharded
    h = handle(pkg, X, "DistL2")
    with h.make_filter(origin_ids(N)[::3]) as rf:
        one = [h.search_exact(Q, 10, filter=f) for f in (None, rf)]
        h.replicate([0, 1])
        for f, want in zip((None, rf), one):
            same(h.search_exact(Q, 10, filter=f), want, "two GPUs")


def test_refusals_leave_the_handle_unchanged(pkg, po):
    n = 1500
    X = data(np.float32, "DistL2", n, 24, 71)
    Q = data(np.float32, "DistL2", NQ, 24, 72)
    E = pkg.HnswError
    ids = origin_ids(n)
    h = pkg.Hnsw(M, n + 10, 16, 48, "DistL2")
    h.insert_flat(X, ids=ids)
    stale = h.make_filter(ids[::3])
    h.insert_flat(data(np.float32, "DistL2", 10, 24, 77), ids=np.arange(10, dtype=np.uint64) + 10 ** 6)
    q_dev = torch.from_numpy(Q).cuda()
    out = torch.empty((NQ, 10, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.empty((NQ,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    want = h.search_exact(Q, 10)
    fresh = h.make_filter(ids[::3])
    want_f = h.search_exact(Q, 10, filter=fresh)

    def unchanged():
        same(h.search_exact(Q, 10), want, "after a refused call")
        same(h.search_exact(Q, 10, filter=fresh), want_f, "after a refused call, filtered")

    def refused(rf, why):
        for call in (lambda: h.search_exact(Q, 10, filter=rf),
                     lambda: h.search_exact_device(q_dev.data_ptr(), NQ, 10, out.data_ptr(), cnt.data_ptr(), filter=rf),
                     lambda: h.search_exact_device(q_dev.data_ptr(), NQ, 10, out.data_ptr(), cnt.data_ptr(), sync=False,
                                                   filter=rf)):
            with pytest.raises(E, match=why):
                call()
            unchanged()
    refused(stale, "stale")
    gone = h.make_filter(ids[::2])
    gone.free()
    refused(gone, "not a live filter")
    refused(pkg.ResidentFilter(h, 10 ** 12), "not a live filter")
    other = handle(pkg, X, "DistL2")
    foreign = other.make_filter(ids[::3])
    refused(foreign, "not a live filter")
    foreign.free()
    with pytest.raises(E, match="dimension"):
        h.search_exact(Q[:, :20], 10)
    unchanged()
    ph = pkg.Hnsw(M, 600, 16, 48, "DistL2")
    ph.partition([0, 0])
    ph.insert_flat(X[:600], ids=ids[:600])
    pwant = ph.search_exact(Q, 10)
    with pytest.raises(E, match="partitioned"):
        ph.search_exact_device(q_dev.data_ptr(), NQ, 10, out.data_ptr(), cnt.data_ptr())
    same(ph.search_exact(Q, 10), pwant, "partitioned handle after a refused call")
    fresh.free()
    stale.free()


def test_free_waits_for_an_async_exact_launch(pkg, po):
    """filter_free synchronises the asynchronous launches that may read the filter's id list: once it returns, the
    launch's answers are complete"""
    n, d, k = 60000, 100, 10
    X = data(np.float32, "DistL2", n, d, 81)
    Q = data(np.float32, "DistL2", 2000, d, 82)
    h = handle(pkg, X, "DistL2")
    rf = h.make_filter(origin_ids(n)[filter_sets(n, 5)["50%"]])
    want = h.search_exact(Q, k, filter=rf, with_pid=False)
    q_dev = torch.from_numpy(Q).cuda()
    out = torch.zeros((len(Q), k, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.zeros((len(Q),), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    h.search_exact_device(q_dev.data_ptr(), len(Q), k, out.data_ptr(), cnt.data_ptr(), sync=False, filter=rf)
    rf.free()
    same_host_device(want, device_answers(out, cnt), "async launch, read after filter_free")
