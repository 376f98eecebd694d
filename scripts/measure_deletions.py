"""Searches of an index with deleted points, against a resident filter of the live points.

  python scripts/measure_deletions.py [--n N] [--nq NQ] [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10, ef = 64.  The deleted
points are a random 0, 0.1 %, 1 %, 10 % and 50 % of the index (each fraction a fresh draw, the previous one restored).
Per fraction:
  * search_flat: queries/s, and recall@10 against search_exact over the live points (with deleted points the rows run
    the filtered kernel by the live stop rule, at 0 % the lean kernel);
  * the same batch through a resident filter of the live points (search_flat_filtered, the filtered kernel's
    fall-through rule), queries/s and recall@10;
  * search_exact: queries/s.
Each call is timed with the host clock around calls that end in a synchronisation, the three alternating within each of
R runs; the best run is reported.  Prints the card and its power limit first, then one JSON line per fraction."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def recall(got, truth):
    ids, cnt = got[2], got[4]
    tids, tcnt = truth[2], truth[4]
    hit = sum(len(set(ids[i, :cnt[i]].tolist()) & set(tids[i, :tcnt[i]].tolist())) for i in range(len(cnt)))
    return hit / max(1, int(tcnt.sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    pkg = importlib.import_module("hnswlib-rs_b200")
    n, d, k, ef = a.n, 128, 10, 64
    X = pkg.datagen.clustered(n, d, 1)
    Q = torch.from_numpy(pkg.datagen.clustered(a.nq, d, 2)).pin_memory().numpy()
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    rng = np.random.default_rng(3)
    prev = np.zeros(0, np.int64)
    for frac in (0.0, 0.001, 0.01, 0.1, 0.5):
        h.restore_points(prev)
        dead = np.sort(rng.choice(n, int(round(frac * n)), replace=False))
        h.delete_points(dead)
        prev = dead
        live = np.setdiff1d(np.arange(n), dead).astype(np.uint64)
        rf = h.make_filter(live)
        truth = h.search_exact(Q, k)
        h.search_flat(Q, k, ef)
        kernel = pkg.last_kernel()
        h.search_flat(Q, k, ef, filter=rf)
        best = {"flat": 1e30, "filter": 1e30, "exact": 1e30}
        for _ in range(a.runs):
            t, flat = timed(lambda: h.search_flat(Q, k, ef))
            best["flat"] = min(best["flat"], t)
            t, filt = timed(lambda: h.search_flat(Q, k, ef, filter=rf))
            best["filter"] = min(best["filter"], t)
            t, _ = timed(lambda: h.search_exact(Q, k))
            best["exact"] = min(best["exact"], t)
        rf.free()
        print(json.dumps({"deleted_fraction": frac, "deleted": int(len(dead)), "flat_kernel": kernel,
                          "flat_qps": a.nq / best["flat"], "flat_recall": recall(flat, truth),
                          "live_filter_qps": a.nq / best["filter"], "live_filter_recall": recall(filt, truth),
                          "exact_qps": a.nq / best["exact"]}), flush=True)


if __name__ == "__main__":
    main()
