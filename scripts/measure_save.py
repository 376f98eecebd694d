"""Saving and restoring an index, against a plain dump / load and a rebuild from the raw vectors.

  python scripts/measure_save.py [--n N] [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200, every point with a label and an attribute.  Reports
the GPU build time from the raw vectors (insert_flat), save and restore wall times, file_dump and load wall times, and
the sizes of the files each writes.  Files go to a fresh temporary directory (the page cache is warm: the times are of
the library's work, not of the disk).  Each time is the best of R runs.  Prints the card and its power limit first, then
one JSON line."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def best(runs, fn):
    """(best wall time of `runs` calls of fn, fn's last result)"""
    ts, out = [], None
    for _ in range(runs):
        t = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t)
    return min(ts), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    print(gpu_info(), flush=True)
    n, d = a.n, 128
    X = pkg.datagen.clustered(n, d, 1)
    rng = np.random.default_rng(3)

    def build():
        h = pkg.Hnsw(16, n, 16, 200, "DistL2")
        h.insert_flat(X)
        return h
    t_build, h = best(a.runs, build)
    h.set_labels(0, rng.integers(0, 1000, n).astype(np.uint32))
    h.set_attributes(0, rng.integers(-10 ** 9, 10 ** 9, n))
    res = {"n": n, "dim": d, "build_s": round(t_build, 3)}
    with tempfile.TemporaryDirectory() as td:
        t_save, _ = best(a.runs, lambda: h.save(td, "s"))
        t_restore, r = best(a.runs, lambda: pkg.Hnsw.restore(td, "s"))
        t_dump, _ = best(a.runs, lambda: h.file_dump(td, "d"))
        t_load, _ = best(a.runs, lambda: pkg.Hnsw.load(td, "d", "DistL2"))
        size = lambda name: os.path.getsize(os.path.join(td, name))
        res.update(save_s=round(t_save, 3), restore_s=round(t_restore, 3), dump_s=round(t_dump, 3),
                   load_s=round(t_load, 3), graph_mb=round(size("s.hnsw.graph") / 2 ** 20, 1),
                   data_mb=round(size("s.hnsw.data") / 2 ** 20, 1), manifest_mb=round(size("s.hnsw.b200") / 2 ** 20, 1))
        Q = pkg.datagen.clustered(1000, d, 2)
        a1, a2 = h.search_flat(Q, 10, 64), r.search_flat(Q, 10, 64)
        res["restored_answers_equal"] = bool(np.array_equal(a1[2], a2[2]) and np.array_equal(a1[1].view(np.uint32),
                                                                                            a2[1].view(np.uint32)))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
