"""Filtered and labelled graph search on the generic filtered kernels (CH = 0: rows of other than 32 float4 chunks, e.g.
f32 at d = 100 or 768, and every integer type), where measure_filters.py and measure_labels.py, at d = 128, run the CH = 4 kernels.

  python scripts/measure_filters_generic.py [--runs R]

200 000 points, M = 16, ef_construction = 100: clustered f32 DistL2 at d = 100 and 768, and uniform u32 DistHamming
(values 0..3) at d = 64, whose filtered kernel spills since label sets were added; 10 000 pinned queries, k = 10,
ef = 64.  Per shape, one 10 000-query call of: search_flat_filtered with a resident filter admitting origin ids
g % 100 < 50 (50 %) and < 5 (5 %), and search_flat_labeled with point g labelled g % 20 and query i restricted to
label i % 20 (5 %).  Host clock around warmed calls that end in a synchronisation, R runs each.  Runs with whichever
library HNSW_B200_LIB names, so that two builds can be compared alternately.  Prints the card and its power limit first,
then one JSON line per shape."""
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


def timed(fn, runs):
    fn()
    ts = []
    for _ in range(runs):
        t = time.perf_counter()
        fn()
        ts.append(round((time.perf_counter() - t) * 1e3, 3))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default=None, help="run the shapes of this metric only")
    args = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    n, nq, k, ef = 200_000, 10_000, 10, 64
    print(json.dumps({"gpu": gpu_info(), "n": n, "nq": nq, "k": k, "ef": ef}), flush=True)
    for dtype, metric, d in ((np.float32, "DistL2", 100), (np.float32, "DistL2", 768), (np.uint32, "DistHamming", 64)):
        if args.only and metric != args.only:
            continue
        if dtype == np.float32:
            X, Q0 = pkg.datagen.clustered(n, d, 1), pkg.datagen.clustered(nq, d, 2)
        else:
            rng = np.random.default_rng(1)
            X, Q0 = rng.integers(0, 4, (n, d)).astype(dtype), rng.integers(0, 4, (nq, d)).astype(dtype)
        bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
        Q = bq.numpy().view(dtype).reshape(nq, d)
        Q[:] = Q0
        h = pkg.Hnsw(16, n, 16, 100, metric, dtype=dtype)
        h.insert_flat(X)
        ids = np.arange(n, dtype=np.uint64)
        h.set_labels(0, (np.arange(n) % 20).astype(np.uint32))
        ql = (np.arange(nq) % 20).astype(np.uint32)
        out = {"dtype": np.dtype(dtype).name, "metric": metric, "dim": d}
        for name, share in (("filtered_50pct_ms", 50), ("filtered_5pct_ms", 5)):
            with h.make_filter(np.ascontiguousarray(ids[ids % 100 < share])) as rf:
                out[name] = timed(lambda: h.search_flat(Q, k, ef, filter=rf, with_pid=False), args.runs)
        out["labeled_5pct_ms"] = timed(lambda: h.search_flat_labeled(Q, k, ef, ql, with_pid=False), args.runs)
        print(json.dumps(out), flush=True)
        del h


if __name__ == "__main__":
    main()
