"""Search by stored point against the host-query calls it replaces, at the c2 size.

  python scripts/measure_search_by_id.py [--runs R]

c2 size: clustered 1 M x 128 f32, M = 16, ef_construction = 200, k = 10, ef = 64.  Three measurements, each after a check
that both sides give the same answers bit for bit, then R runs alternating the two sides, host clock around calls that
end in a synchronisation:
  * 10 000 random ranks: search_by_id against search_flat on the same rows, held in pinned host memory;
  * the k-NN graph of all 1 M points (exclude_self, batches of 65 536): knn_graph against export_vectors, then search_flat
    with k + 1 on the same batches and each point's own entry removed in numpy (the rule of exclude_self);
  * a 100 000-point prefix: knn_graph(exact=True), knn_graph(ef=64), and the recall@10 of the second against the first.
Prints the card and its power limit first, then one JSON line per measurement."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return time.perf_counter() - t, r


def minus_self(it, d, c, qids, k):
    """(k + 1)-wide rows without each query's own id, or without their last entry, cut to k (vectorised)"""
    hit = (it == qids[:, None].astype(np.uint32)) & (np.arange(it.shape[1])[None, :] < c[:, None])
    has = hit.any(1)
    pos = np.where(has, hit.argmax(1), k + 1)
    src = np.arange(k)[None, :] + (np.arange(k)[None, :] >= pos[:, None])
    rows = np.arange(len(qids))[:, None]
    cnt = np.where(has, c - 1, np.minimum(c, k))
    oi, od = it[rows, src].copy(), d[rows, src].copy()
    pad = np.arange(k)[None, :] >= cnt[:, None]
    oi[pad], od[pad] = 0xFFFFFFFF, np.inf
    return oi, od


def stats(ts):
    return {"min_ms": round(1e3 * min(ts), 3), "median_ms": round(1e3 * float(np.median(ts)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    n, d, k, ef, nq, B = 1_000_000, 128, 10, 64, 10_000, 65536
    print(json.dumps({"gpu": gpu_info(), "lib": pkg.lib_path(), "n": n, "dim": d, "k": k, "ef": ef}), flush=True)
    X = pkg.datagen.clustered(n, d, 1)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)

    # ---- 10 000 random ranks
    qids = np.random.default_rng(3).choice(n, nq, replace=False).astype(np.uint64)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = h.get_vectors(qids)
    by_id = lambda: h.search_by_id(qids, k, ef, with_pid=False)
    flat = lambda: h.search_flat(Q, k, ef, with_pid=False)
    a, b = by_id(), flat()
    assert all(np.array_equal(x, y) for x, y in zip(a, b) if x is not None), "by-id rows differ from search_flat's"
    ta, tb = [], []
    for _ in range(args.runs):
        ta.append(timed(by_id)[0])
        tb.append(timed(flat)[0])
    print(json.dumps({"what": "10000 random ranks", "search_by_id": stats(ta), "search_flat_pinned": stats(tb)}), flush=True)

    # ---- the k-NN graph of every point
    def host_graph():
        t0 = time.perf_counter()
        V = h.export_vectors()
        t1 = time.perf_counter()
        ids, ds = np.empty((n, k), np.uint32), np.empty((n, k), np.float32)
        search = strip = 0.0
        for s in range(0, n, B):
            q = np.arange(s, min(n, s + B), dtype=np.uint64)
            dt, (_, dd, it, _, c) = timed(lambda: h.search_flat(V[s:s + q.size], k + 1, ef, with_pid=False))
            search += dt
            dt, (ids[s:s + q.size], ds[s:s + q.size]) = timed(lambda: minus_self(it, dd, c, q, k))
            strip += dt
        return (ids, ds), {"export_ms": 1e3 * (t1 - t0), "search_ms": 1e3 * search, "strip_ms": 1e3 * strip}
    (gi, gd), (hi, hd) = h.knn_graph(k, ef=ef, batch=B), host_graph()[0]
    assert np.array_equal(gi, hi) and np.array_equal(gd.view(np.uint32), hd.view(np.uint32)), "k-NN graphs differ"
    ta, tb, parts = [], [], []
    for _ in range(max(1, args.runs // 2)):
        ta.append(timed(lambda: h.knn_graph(k, ef=ef, batch=B))[0])
        dt, (_, p) = timed(host_graph)
        tb.append(dt)
        parts.append({key: round(v, 1) for key, v in p.items()})
    print(json.dumps({"what": "k-NN graph of 1M points", "knn_graph": stats(ta), "export_then_search_flat": stats(tb),
                      "host_parts": parts}), flush=True)

    # ---- exact k-NN graph of a 100 000-point prefix, and the graph version's recall against it
    m = 100_000
    hp = pkg.Hnsw(16, m, 16, 200, "DistL2")
    hp.insert_flat(X[:m])
    (eids, _), (gids, _) = hp.knn_graph(k, exact=True), hp.knn_graph(k, ef=ef)
    te, tg = [], []
    for _ in range(max(1, args.runs // 2)):
        te.append(timed(lambda: hp.knn_graph(k, exact=True))[0])
        tg.append(timed(lambda: hp.knn_graph(k, ef=ef))[0])
    recall = float(np.mean([len(np.intersect1d(gids[i], eids[i])) for i in range(m)]) / k)
    print(json.dumps({"what": "k-NN graph of a 100000-point prefix", "exact": stats(te), "graph_ef64": stats(tg),
                      "recall_at_10": round(recall, 4)}), flush=True)


if __name__ == "__main__":
    main()
