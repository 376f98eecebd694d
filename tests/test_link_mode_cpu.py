"""Link mode 1 (per-layer reverse links) in the oracle, without a GPU.

One seeded serial build of 10 000 x 25 uniform points, M = 16, ef_construction = 200, made twice from the same levels:
link mode 0 (the reference's rule, every back-link under the new point's level, hnsw.rs:1257) and link mode 1 (each
back-link in the layer it was made in).  Mode 1 must leave (almost) no upper-level point without a layer-0 in-link,
search better at the same ef, and keep no list above a point's level except the lists of former entry points.
"""
import numpy as np
import pytest

from linkgraph import entry_history, insert_link_mode1, lists_above_level, without_layer0_inlink
from util import recall_ids

N, D, M, EFC = 10000, 25, 16, 200


@pytest.fixture(scope="module")
def builds(pkg, po):
    X = pkg.datagen.uniform(N, D, 31)
    Q = pkg.datagen.uniform(1000, D, 32)
    levels = po.Oracle(M, N, 16, EFC, "DistL2", D, mode=po.MODE_DET, order=po.ORDER_GPU).draw_levels(N)
    out = {}
    for mode in (0, 1):
        o = po.Oracle(M, N, 16, EFC, "DistL2", D, mode=po.MODE_DET, order=po.ORDER_GPU)
        if mode == 0:
            o.insert_batch(X, levels=levels)
        else:
            insert_link_mode1(o, X, levels)
        out[mode] = o
    return X, Q, levels, out


def test_upper_points_keep_layer0_inlinks(builds):
    X, Q, levels, o = builds
    count = {m: len(without_layer0_inlink(o[m].export_layer(0), levels, o[m].entry)) for m in (0, 1)}
    print(f"level >= 1 points without a layer-0 in-link: mode 0 {count[0]}, mode 1 {count[1]} "
          f"(of {int((levels >= 1).sum())})")
    assert count[0] > 0
    assert count[1] <= count[0] / 10


def test_per_layer_links_raise_recall(builds, po):
    X, Q, levels, o = builds
    truth, _ = po.bruteforce(X, Q, 10, "DistL2")
    for ef in (24, 64):
        r = {}
        for m in (0, 1):
            _, _, it, _, cnt = o[m].search_batch(Q, 10, ef)
            r[m] = recall_ids(it, cnt, truth)
        print(f"recall@10 at ef = {ef}: mode 0 {r[0]:.4f}, mode 1 {r[1]:.4f}")
        assert r[1] > r[0]


def test_no_list_above_level_except_former_entry_points(builds):
    X, Q, levels, o = builds
    lv, _, _ = o[1].export_points()
    assert np.array_equal(lv, levels)
    nl = int(levels.max()) + 1
    entries = set(entry_history(levels))
    above = {m: lists_above_level([o[m].export_layer(l) for l in range(nl)], levels) for m in (0, 1)}
    assert [(l, p) for l, p in above[1] if p not in entries] == []
    # the reference's rule (and its stray push, hnsw.rs:1140-1144) writes such lists for ordinary points
    assert any(p not in entries for _, p in above[0])
