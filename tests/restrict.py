"""Fixtures of the restricted searches (a filter per query, labels, label sets, attribute ranges): the oracle graph they
search, the point labels they assign, and their resident filters."""
import numpy as np

from exactref import origin_ids
from graphs import data
from util import oracle_layers

N, M, EFC = 2000, 8, 48
NONE = 0xFFFFFFFF   # LABEL_NONE

GRAPH_CASES = [(np.float32, "DistL2", 128), (np.float32, "DistL2", 100), (np.uint8, "DistHamming", 100),
               (np.uint16, "DistL1", 100), (np.int32, "DistL2", 24)]


def build(pkg, po, dtype, metric, d, nq=300, seed=1):
    """an oracle graph imported into the engine.  Points 0..399 come in identical pairs, so that a filter admitting
    them has an equal-distance twin for every answer."""
    X = data(dtype, metric, N, d, seed)
    X[1:400:2] = X[0:400:2]
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, ids=origin_ids(N))
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
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


def unrestricted(s):
    return len(s) > 0 and set(s) == {NONE}


def free(rfs):
    for rf in rfs:
        if rf is not None:
            rf.free()
