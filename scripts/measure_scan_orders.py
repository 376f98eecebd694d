"""The host cost of the exact scan's orders: the first exact call after set_labels / set_attributes, against the next.

  python scripts/measure_scan_orders.py [--runs R]

c2 size: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10.  Point g carries label
g % 20 and, as attribute, a random permutation of 0 .. n - 1; query i is restricted to label i % 20, and a ranged query
to the window [0, n / 10), alone or within the set {i % 20}.  Each of R runs first calls set_labels, which makes the
orders keyed on labels stale, and times search_exact_labeled twice (the first call builds the order by label); then
calls set_attributes, which makes the orders keyed on values stale, and times search_exact_ranges twice without sets
(the first builds the order by value) and twice with them (the first builds the order by label and value).  Host clock
around calls that end in a synchronisation, after one warm-up call of each kind.  The library is the package's, or
HNSW_B200_LIB's, so that two builds can be compared by alternating processes.  Prints the card and its power limit
first, then one JSON line per run."""
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
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
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
    import torch
    n, d, nq, k, T = 1_000_000, 128, 10_000, 10, 20
    X = pkg.datagen.clustered(n, d, 1)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = pkg.datagen.clustered(nq, d, 2)
    print(json.dumps({"gpu": gpu_info(), "lib": pkg.lib_path(), "n": n, "dim": d, "nq": nq, "k": k, "T": T}), flush=True)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    lab = (np.arange(n) % T).astype(np.uint32)
    attr = np.random.default_rng(7).permutation(n).astype(np.int64)
    qlab = (np.arange(nq) % T).astype(np.uint32)
    window = np.tile(np.array([0, n // 10 - 1], np.int64), (nq, 1))
    sets = [[int(x)] for x in qlab]
    labeled = lambda: h.search_exact_labeled(Q, k, qlab, with_pid=False)
    ranged = lambda: h.search_exact_ranges(Q, k, window, with_pid=False)
    ranged_sets = lambda: h.search_exact_ranges(Q, k, window, sets, with_pid=False)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    for call in (labeled, ranged, ranged_sets):   # warm-up: modules, scratch and the orders' device buffers
        call()
    for run in range(args.runs):
        out = {"run": run}
        h.set_labels(0, lab)
        out["labeled_first_s"], out["labeled_next_s"] = timed(labeled), timed(labeled)
        h.set_attributes(0, attr)
        out["ranged_first_s"], out["ranged_next_s"] = timed(ranged), timed(ranged)
        out["ranged_sets_first_s"], out["ranged_sets_next_s"] = timed(ranged_sets), timed(ranged_sets)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
