"""A handle's settings are one value on the handle, read by every Index that serves it: its partitions (and their views)
and its replicas, whether the setting was made before or after partition / replicate.

The data is u8 Hamming over {0, 1, 2}: nearly every comparison meets equal distances, so the two tie modes return
different answers, and a device that searched in the wrong mode shows in the ids.  With N + EXTRA points below 3/4 of a
search's visited table (2 * (EF + 16) * 2M entries, rounded up to 2048) no table can overflow, so no batch is re-run and
the traversal counters of a batch do not depend on which device's tables answered it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, EXTRA, D, M, EFC, K, EF, NQ = 1400, 100, 32, 8, 64, 10, 32, 600


def tie_data(n, seed):
    return np.random.default_rng(seed).integers(0, 3, (n, D)).astype(np.uint8)


def build(pkg):
    h = pkg.Hnsw(M, N + EXTRA, 16, EFC, "DistHamming", dtype=np.uint8)
    h.set_level_seed(7)
    return h


def same(got, want, what):
    for name, a, b in zip(("origin", "dist", "internal", "pid", "counts"), got, want):
        assert np.array_equal(a, b), f"{what}: {name} differs"


@pytest.mark.parametrize("when", ["before", "after"])
def test_partitions_read_the_handles_settings(pkg, when):
    """tie mode 1 and statistics, set on the handle before partition([0, 0]) or after it, reach both partitions: a view
    searches with search_std_kernel, and the handle's counters are the sum of the views'"""
    X, Q = tie_data(N, 1), tie_data(NQ, 2)
    h = build(pkg)

    def settings():
        h.set_tie_mode(1)
        h.enable_stats(True)
    if when == "before":
        settings()
    h.partition([0, 0])
    if when == "after":
        settings()
    h.insert_flat(X)
    views = [h.partition_view(p) for p in range(2)]
    h.get_stats()
    h.search_flat(Q, K, EF)
    total = h.get_stats(reset=False)
    each = [v.get_stats(reset=False) for v in views]
    assert total == {key: sum(s[key] for s in each) for key in total}, (total, each)
    assert [s["queries"] for s in each] == [NQ, NQ]
    assert total["evals"] > 0 and all(s["evals"] > 0 for s in each)
    for p, v in enumerate(views):
        v.search_flat(Q, K, EF)
        assert "search_std_kernel" in pkg.last_kernel(), f"partition {p}: {pkg.last_kernel()}"
    h.set_tie_mode(0)
    for p, v in enumerate(views):
        v.search_flat(Q, K, EF)
        assert "search_std_kernel" not in pkg.last_kernel(), f"partition {p}: {pkg.last_kernel()}"


@pytest.mark.parametrize("when", ["before", "after"])
def test_replicas_read_the_handles_settings(pkg, when):
    """tie mode 1 on a replicated handle, set before or after replicate: a sharded batch returns, bit for bit, what the
    unreplicated handle returns, also after an insert forces a re-broadcast, and get_stats sums every device's counters"""
    L = pkg.load_library()
    if L.hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    ndev = min(4, L.hnsw_b200_device_count())
    assert NQ >= 64 * ndev   # the batch is sharded
    X, Q, extra = tie_data(N, 3), tie_data(NQ, 4), tie_data(EXTRA, 5)
    one, rep = build(pkg), build(pkg)
    for h in (one, rep):
        h.insert_flat(X)

    def same_graph(what):
        for layer in range(int(one.export_points()[0].max()) + 1):
            for a, b in zip(one.export_layer(layer), rep.export_layer(layer)):
                assert np.array_equal(a, b), f"{what}: the two builds differ at layer {layer}"
    same_graph("built")
    # on this data the tie modes differ on one GPU
    ties_by_id = one.search_flat(Q, K, EF)
    one.set_tie_mode(1)
    one.enable_stats(True)
    one.get_stats()
    want = one.search_flat(Q, K, EF)
    assert not np.array_equal(ties_by_id[2], want[2]), "the tie modes agree on this data"

    def settings():
        rep.set_tie_mode(1)
        rep.enable_stats(True)
        rep.get_stats()
    if when == "before":
        settings()
    rep.replicate(list(range(ndev)))
    assert rep.replica_count() == ndev - 1
    if when == "after":
        settings()
    same(rep.search_flat(Q, K, EF), want, "sharded")
    # the inserts' own counters are left out: only the searches' are compared
    for h in (one, rep):
        h.enable_stats(False)
        h.insert_flat(extra, ids=np.arange(N, N + EXTRA, dtype=np.uint64))
        h.enable_stats(True)
    same_graph("after the insert")
    want = one.search_flat(Q, K, EF)
    same(rep.search_flat(Q, K, EF), want, "sharded after a re-broadcast")
    got, single = rep.get_stats(), one.get_stats()
    assert got == single, (got, single)
    assert got["queries"] == 2 * NQ
