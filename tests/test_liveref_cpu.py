"""The live-search reference (liveref.py) against the oracle: its unfiltered and filtered rules must give the oracle's
rows and traversal counters bit for bit, on the graphs and data of test_gpu_deletions.py, so that its live rule, one
branch away from the filtered one, can stand for the oracle in the GPU tests.  CPU only."""
import numpy as np
import pytest

from answers import same
from graphs import data
from liveref import LiveRef

N, M, EFC, NQ = 600, 8, 64, 12
GRAPHS = [(np.float32, "DistL2", 48), (np.float32, "DistCosine", 100), (np.uint8, "DistHamming", 100)]


@pytest.mark.parametrize("dtype,metric,d", GRAPHS, ids=[g[1] for g in GRAPHS])
def test_reference_matches_oracle(po, dtype, metric, d):
    X = data(dtype, metric, N, d, 5)
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    ref = LiveRef(po, o, X, metric)
    Q = data(dtype, metric, NQ, d, 6)
    rng = np.random.default_rng(7)
    for k, ef in ((1, 1), (10, 10), (10, 64), (64, 200)):
        for allow in (None, np.sort(rng.choice(N, N // 2, replace=False)), np.array([ref.entry])):
            admit = None
            if allow is not None:
                admit = np.zeros(N, bool)
                admit[allow] = True
            o.counters()
            want = o.search_batch(Q, k, ef, filter_ids=None if allow is None else allow.astype(np.uint64))
            co = o.counters()
            got, cg = ref.batch(Q, k, ef, admit)
            what = f"{metric} k={k} ef={ef} filter={'none' if allow is None else len(allow)}"
            same(got, want, what)
            for key in ("evals", "expansions", "adj_read"):
                assert cg[key] == co[key], (what, key, cg, co)


@pytest.mark.parametrize("dtype,metric,d", GRAPHS[:2], ids=[g[1] for g in GRAPHS[:2]])
def test_live_rule_matches_oracle_without_deletions(po, dtype, metric, d):
    """The live branch itself against the oracle: with every point live, a live search makes the unfiltered search's
    decisions except on equal distances at the stop test, which continuous f32 data does not produce, so its rows and
    counters must be the oracle's unfiltered ones."""
    X = data(dtype, metric, N, d, 8)
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    ref = LiveRef(po, o, X, metric)
    Q = data(dtype, metric, NQ, d, 9)
    for k, ef in ((1, 1), (10, 10), (10, 64), (64, 200)):
        o.counters()
        want = o.search_batch(Q, k, ef)
        co = o.counters()
        got, cg = ref.batch(Q, k, ef, np.ones(N, bool), live=True)
        same(got, want, f"{metric} live k={k} ef={ef}")
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == co[key], (metric, k, ef, key, cg, co)
