"""Label sets against one resident filter per distinct set, and against one labelled exact call per label.

  python scripts/measure_label_sets.py [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10, ef = 64.  Points are
labelled round robin (point g carries label g % T), T = 20 and 1 000.  For s = 1, 4 and 16 labels per set, 20 distinct
sets are drawn (set j: s distinct labels), and query i is restricted to set i % 20.  The other sides:
  * per-query filters: one resident filter per distinct set, admitting the same points (filter_new over id lists,
    timed as setup), and one search_flat_per_query / search_exact_per_query call;
  * exact only, per label: one search_exact_labeled call per label some set names, over the queries whose set names it,
    merged on the host by (distance, internal id), the exact scan's order.
Graph searches run at T = 20, and at T = 1 000 for s = 4 and 16 (s = 1 there is a labelled search, measure_labels.py);
--kinds picks graph, exact or both.  The label-set side is timed twice: with the sets as Python lists (converted at
every call) and as a prebuilt (offsets, values) pair, which is what the library itself costs.  The answers are checked equal before anything is timed; the sides alternate within each of R runs, each timed with the
host clock around calls that end in a synchronisation.  Prints the card and its power limit first, then one JSON line
per measurement."""
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

NSETS = 20


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def equal(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[:3] + a[4:], b[:3] + b[4:])) and np.array_equal(
        a[1].view(np.uint32), b[1].view(np.uint32))


def rows_by_label(sets, sel):
    """label -> the rows whose set names it"""
    return {L: np.flatnonzero([L in sets[g] for g in sel]) for L in sorted({L for s in sets for L in s})}


def per_label_exact(h, Q, k, by_label):
    """one search_exact_labeled call per label, over the rows whose set names it, merged per row"""
    nq = len(Q)
    cand_d, cand_i, cand_o = [[] for _ in range(nq)], [[] for _ in range(nq)], [[] for _ in range(nq)]
    for L, rows in by_label.items():
        o, d, it, _, c = h.search_exact_labeled(Q[rows], k, np.full(len(rows), L, np.uint32), with_pid=False)
        for r, row in enumerate(rows):
            cand_d[row].append(d[r, :c[r]])
            cand_i[row].append(it[r, :c[r]])
            cand_o[row].append(o[r, :c[r]])
    ids = np.full((nq, k), ~np.uint64(0), np.uint64)
    dist = np.full((nq, k), np.inf, np.float32)
    internal = np.full((nq, k), 0xFFFFFFFF, np.uint32)
    counts = np.zeros(nq, np.int32)
    for q in range(nq):
        d, it, o = np.concatenate(cand_d[q]), np.concatenate(cand_i[q]), np.concatenate(cand_o[q])
        top = np.lexsort((it, d))[:k]
        n = len(top)
        ids[q, :n], dist[q, :n], internal[q, :n], counts[q] = o[top], d[top], it[top], n
    return ids, dist, internal, None, counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--kinds", default="graph,exact")
    args = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    n, d, nq, k, ef = 1_000_000, 128, 10_000, 10, 64
    X = pkg.datagen.clustered(n, d, 1)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = pkg.datagen.clustered(nq, d, 2)
    print(json.dumps({"gpu": gpu_info(), "shape": "c2", "n": n, "dim": d, "nq": nq, "k": k, "ef": ef,
                      "distinct_sets": NSETS}), flush=True)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    ids = np.arange(n, dtype=np.uint64)
    sel = np.arange(nq) % NSETS
    rng = np.random.default_rng(5)
    for T in (20, 1000):
        lab = (np.arange(n) % T).astype(np.uint32)
        h.set_labels(0, lab)
        for s in (1, 4, 16):
            sets = [sorted(rng.choice(T, s, replace=False).tolist()) for _ in range(NSETS)]
            qs = [sets[g] for g in sel]
            pair = (np.concatenate([[0], np.cumsum([len(sets[g]) for g in sel])]).astype(np.uint64),
                    np.array([L for g in sel for L in sets[g]], np.uint32))
            rfs = []
            t_fil = timed(lambda: rfs.extend(h.make_filter(np.ascontiguousarray(ids[np.isin(lab, st)])) for st in sets))
            filters = [rfs[g] for g in sel]
            by_label = rows_by_label(sets, sel)
            admitted = s / T
            kinds = ("graph", "exact") if T == 20 or s > 1 else ("exact",)
            for kind in (x for x in kinds if x in args.kinds.split(",")):
                if kind == "graph":
                    sides = {"label_sets_s": lambda: h.search_flat_label_sets(Q, k, ef, qs, with_pid=False),
                             "label_sets_pair_s": lambda: h.search_flat_label_sets(Q, k, ef, pair, with_pid=False),
                             "per_query_s": lambda: h.search_flat_per_query(Q, k, ef, filters, with_pid=False)}
                else:
                    sides = {"label_sets_s": lambda: h.search_exact_label_sets(Q, k, qs, with_pid=False),
                             "label_sets_pair_s": lambda: h.search_exact_label_sets(Q, k, pair, with_pid=False),
                             "per_query_s": lambda: h.search_exact_per_query(Q, k, filters, with_pid=False),
                             "per_label_merged_s": lambda: per_label_exact(h, Q, k, by_label)}
                a = sides["label_sets_s"]()
                for name, call in sides.items():
                    assert equal(a, call()), (T, s, kind, name, "answers differ")
                ts = {name: [] for name in sides}
                for _ in range(args.runs):
                    for name, call in sides.items():
                        ts[name].append(timed(call))
                print(json.dumps({"T": T, "labels_per_set": s, "admitted": admitted, "search": kind, **ts,
                                  "setup_filter_new_s": t_fil}), flush=True)
            for rf in rfs:
                rf.free()


if __name__ == "__main__":
    main()
