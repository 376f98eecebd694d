"""Building one graph on the GPU and in the oracle and comparing the two: the test data, the serial and batched builds,
the graph comparison, and the cases of the kernel instantiation matrix (test_gpu_matrix), which the batched builds
(test_gpu_batched_insert) repeat.

pytest shows the compared values only for asserts in test modules, so every assert here says in its message what it
compared."""
import importlib
import os
import shutil

import numpy as np

import distref
from batched import engine_batches, entry_level_after
from util import csr_lists, oracle_layers

NTH = os.cpu_count() or 8   # oracle threads of insert_both

# ---------------------------------------------------------------- the instantiation matrix's cases
F32_OPS = ["DistL1", "DistL2", "DistDot", "DistCosine"]
F32_DIMS = [24, 48, 100, 150]          # rows of 128 / 256 / 512 / 640 bytes: CH = 1, 2, 4, generic
PROB_OPS = ["DistHellinger", "DistJeffreys", "DistJensenShannon"]   # generic row loop only, at every dimension
PROB_DIMS = [24, 100, 150]             # one 128-byte chunk column, four, and five with a partial last one
U8_DIMS = [100, 200, 400, 600]
U16_DIMS = [50, 100, 200, 300]
CASES = ([(np.float32, m, d, False) for m in F32_OPS for d in F32_DIMS]
         + [(np.float32, m, d, False) for m in PROB_OPS for d in PROB_DIMS]
         + [(np.float32, "DistL2", 24, True), (np.float32, "DistCosine", 100, True), (np.float32, "DistJeffreys", 24, True)]
         + [(np.uint8, m, d, False) for m in distref.INT_METRICS for d in U8_DIMS]
         + [(np.uint16, m, d, False) for m in distref.INT_METRICS for d in U16_DIMS]
         + [(np.uint32, m, 24, False) for m in distref.INT_METRICS]
         + [(np.int32, m, 24, False) for m in ("DistL1", "DistL2", "DistHamming")])
INSERT_CASES = ([(m, d, efc) for m in F32_OPS for d in F32_DIMS for efc in (48, 300)]
                + [(m, 100, efc) for m in PROB_OPS for efc in (48, 300)])


def case_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" + ("-ties" if c[3] else "")


def data(dtype, metric, n, d, seed, ties=False):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt == np.float32 and metric in PROB_OPS:
        return probabilities(n, d, seed, ties)
    if dt == np.float32:
        kind = "unit" if metric == "DistDot" else "uniform"
        dg = importlib.import_module("hnswlib-rs_b200").datagen
        if ties:   # every vector stored 4 times: the kernels must order equal distances by id
            base = dg.make(kind, (n + 3) // 4, d, seed)
            return np.repeat(base, 4, axis=0)[:n].copy()
        return dg.make(kind, n, d, seed)
    hi = {"DistHamming": 3, "DistJaccard": 16 if dt == np.uint8 else 1000}.get(metric)
    if hi is None:
        hi = {np.dtype(np.uint8): 256, np.dtype(np.uint16): 5000, np.dtype(np.uint32): 100000}.get(dt, 2000)
    lo = -hi if dt == np.int32 and metric != "DistHamming" else 0
    return rng.integers(lo, hi, (n, d)).astype(dt)


def probabilities(n, d, seed, ties=False):
    """n probability rows normalised in f32; every other row has about a third of its entries exactly 0, which Jeffreys'
    1e-30 clamp and Jensen-Shannon's zero terms meet.  With ties, every row is stored 4 times."""
    rng = np.random.default_rng(seed)
    m = (n + 3) // 4 if ties else n
    X = rng.random((m, d), dtype=np.float32)
    odd = X[1::2]
    odd[rng.random(odd.shape) < 1 / 3] = 0
    X[X.sum(1) == 0, 0] = 1
    X /= X.sum(1, keepdims=True)
    return np.repeat(X, 4, axis=0)[:n].copy() if ties else X


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
            if root and os.path.exists(os.path.join(root, "bin", "cuobjdump")):
                return os.path.join(root, "bin", "cuobjdump")
    return exe


# ---------------------------------------------------------------- graphs
def assert_same_graph(h, o, n):
    lv, rk, og, entry = h.export_points()
    olv, ork, oog = o.export_points()
    assert entry == o.entry, f"entry point {entry}, the oracle's {o.entry}"
    for what, a, b in (("levels", lv, olv), ("ranks", rk, ork), ("origin ids", og, oog)):
        assert np.array_equal(a, b), f"{what} differ"
    for layer in range(0, int(olv.max()) + 1):
        goff, gids, gds = h.export_layer(layer)
        ooff, oids, ods = o.export_layer(layer)
        if layer == 0:
            assert np.array_equal(goff, ooff) and np.array_equal(gids, oids), "layer 0 differs"
            assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32)), "layer-0 link distances differ"
            continue
        gl, ol = csr_lists(goff, gids), csr_lists(ooff, oids)
        for p in range(n):
            if not gl[p] and olv[p] < layer:   # a list no search can reach, which the engine does not store
                continue
            assert gl[p] == ol[p], (layer, p, gl[p], ol[p])


def build_both(pkg, po, dtype, metric, n, d, M, efc, seed, ties=False, max_elements=None, ledger=None):
    """the same graph serially on the GPU (one insert in flight) and in the oracle (MODE_DET, ORDER_GPU), asserted
    equal; the insert kernel goes into `ledger` unless it is None"""
    X = data(dtype, metric, n, d, seed, ties)
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, max_elements or n, 16, efc, metric, dtype=dtype)
    h.set_insert_batching(1 << 30, 1)   # one insert in flight: a deterministic serial build
    h.insert_flat(X, levels=levels)
    if ledger is not None:
        ledger.add(pkg.last_kernel())
    assert_same_graph(h, o, n)
    return X, o, h


def build_pair(pkg, po, n, d, M, efc, metric, kind="uniform", max_layer=16, seed=1):
    """an oracle graph (MODE_DET, ORDER_GPU) of datagen rows imported into the engine"""
    X = pkg.datagen.make(kind, n, d, seed)
    o = po.Oracle(M, n, max_layer, efc, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, max_layer, efc, metric)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return X, o, h


# ---------------------------------------------------------------- batched builds
def make_oracle(po, dtype, metric, d, M, efc, n, extend=False, keep_pruned=False):
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.set_extend_candidates(extend)
    o.set_keeping_pruned(keep_pruned)
    return o


def make_engine(pkg, dtype, metric, M, efc, n, sched=None, extend=False, keep_pruned=False, link_mode=0):
    h = pkg.Hnsw(M, n, 16, efc, metric, dtype=dtype)
    h.set_extend_candidates(extend)
    h.set_keeping_pruned(keep_pruned)
    h.set_link_mode(link_mode)
    if sched is not None:
        h.set_insert_batching(*sched)
    return h


class State:
    """the handle's point count and entry level, which the next call's schedule starts from"""

    def __init__(self):
        self.n, self.top = 0, -1

    def batches(self, levels, sched=None):
        out = engine_batches(self.n, self.top, levels, *(sched or ()))
        self.top = entry_level_after(self.n, self.top, levels)
        self.n += len(levels)
        return out


def insert_both(pkg, h, o, X, levels, st, sched=None, ids=None, link_mode=0, ledger=None):
    """one insert call on the engine (stats on) and the same call, batch for batch, on the oracle; the counters equal.
    The insert kernel goes into `ledger` unless it is None."""
    o.counters()
    o.insert_batched(X, ids=ids, levels=levels, batches=st.batches(levels, sched), nthreads=NTH, link_mode=link_mode)
    co = o.counters()
    h.enable_stats(True)
    h.get_stats()
    h.insert_flat(X, ids=ids, levels=levels)
    if ledger is not None:
        ledger.add(pkg.last_kernel())
    cg = h.get_stats()
    h.enable_stats(False)
    for key in ("expansions", "adj_read"):
        assert cg[key] == co[key], ("insert", key, cg, co)
