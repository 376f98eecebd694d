"""Radius search against the exact k-NN search of the same k, at the c2 size.

  python scripts/measure_radius.py [--runs R]

c2 shape: clustered 1 M x 128 f32 (datagen.clustered, seed 1), the points imported without a graph (the exact scan reads
none).  For 1 000 and 10 000 queries (clustered, seed 2), radii at each query's distance to its 10th, 100th and 1 000th
exact neighbour, and knbn in {0, 16, 128, 1024}: ms per warmed call of search_exact_radius and of search_exact with
k = max(knbn, 1), R runs alternating the two, host clock around calls that end in a synchronisation.  Before timing,
each radius row is checked against the k-NN row cut at the radius where the k-NN row reaches past it.  Prints the card,
its power limit and max SM clock first, then one JSON line per (nq, radius, knbn)."""
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
    fn()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    n, d = 1_000_000, 128
    print(json.dumps({"gpu": gpu_info(), "lib": pkg.lib_path(), "n": n, "dim": d}), flush=True)
    X = pkg.datagen.clustered(n, d, 1)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.import_graph(X, np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), 0,
                   [(np.zeros(n + 1, np.uint64), np.zeros(0, np.uint32), None)])
    Qall = pkg.datagen.clustered(10_000, d, 2)
    for nq in (1000, 10_000):
        Q = Qall[:nq]
        ref = h.search_exact(Q, 1000, with_pid=False)
        for at in (10, 100, 1000):
            r = ref[1][:, at - 1].copy()
            for knbn in (0, 16, 128, 1024):
                k = max(knbn, 1)
                rad = lambda: h.search_exact_radius(Q, r, knbn, with_pid=False)
                knn = lambda: h.search_exact(Q, k, with_pid=False)
                got, want = rad(), knn()
                if knbn:
                    c = np.minimum(got[4], want[4])
                    assert all(np.array_equal(got[2][i, :c[i]], want[2][i, :c[i]]) for i in range(nq))
                assert np.all(got[5] >= min(at, n))
                tr, tk = [], []
                for _ in range(args.runs):
                    tr.append(timed(rad))
                    tk.append(timed(knn))
                print(json.dumps({"nq": nq, "radius_at": at, "knbn": knbn, "k": k,
                                  "radius_ms": [round(1e3 * t, 3) for t in tr],
                                  "exact_ms": [round(1e3 * t, 3) for t in tk],
                                  "median_total": float(np.median(got[5]))}), flush=True)


if __name__ == "__main__":
    main()
