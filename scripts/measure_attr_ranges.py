"""Attribute ranges against resident filters over the same points.

  python scripts/measure_attr_ranges.py [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10, ef = 64.  Point p's
attribute is a random permutation of 0 .. n - 1, so that a window of w n values admits a fraction w of the points,
scattered over the graph and over the internal ids.  Measured:
  * one window shared by every row, admitting 0.1, 1, 5, 20 and 50 %: search_flat_ranges / search_exact_ranges against
    search_flat / search_exact with one resident filter admitting the same points (filter_new timed as setup).  The
    graph search runs at 5 % and above only: below, a filtered search expands most of the graph (tens of seconds per
    call, DESIGN.md §4.2b), whichever form the filter takes;
  * the same fraction with a different window per row (10 000 runs): against the shared window;
  * a 50 % window within a label set of s = 1 and 4 labels (T = 20 labels round robin, 20 distinct sets): against
    search_flat_per_query / search_exact_per_query with one resident filter per distinct (set, window);
  * set_attributes over every point, and the first exact ranged call after it (which sorts the points by value, and
    by label and value, on the host) against the next one.
The answers are checked equal before anything is timed; the sides alternate within each of R runs, each timed with the
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


def compare(sides, runs, **tags):
    """checks every side's answers against the first side's, then times them alternating"""
    names = list(sides)
    a = sides[names[0]]()
    for name in names[1:]:
        assert equal(a, sides[name]()), (tags, name, "answers differ")
    ts = {name: [] for name in names}
    for _ in range(runs):
        for name in names:
            ts[name].append(timed(sides[name]))
    print(json.dumps({**tags, **ts}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    n, d, nq, k, ef = 1_000_000, 128, 10_000, 10, 64
    X = pkg.datagen.clustered(n, d, 1)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = pkg.datagen.clustered(nq, d, 2)
    print(json.dumps({"gpu": gpu_info(), "shape": "c2", "n": n, "dim": d, "nq": nq, "k": k, "ef": ef}), flush=True)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    ids = np.arange(n, dtype=np.uint64)
    rng = np.random.default_rng(7)
    attr = rng.permutation(n).astype(np.int64)
    t_set = timed(lambda: h.set_attributes(0, attr))
    one = np.tile(np.array([0, n // 10], np.int64), (nq, 1))
    t_first = timed(lambda: h.search_exact_ranges(Q, k, one, with_pid=False))
    t_next = timed(lambda: h.search_exact_ranges(Q, k, one, with_pid=False))
    T = 20
    lab = (np.arange(n) % T).astype(np.uint32)
    h.set_labels(0, lab)
    sets1 = [[0]] * nq
    t_first_l = timed(lambda: h.search_exact_ranges(Q, k, one, sets1, with_pid=False))
    t_next_l = timed(lambda: h.search_exact_ranges(Q, k, one, sets1, with_pid=False))
    print(json.dumps({"set_attributes_s": t_set, "exact_first_by_value_s": t_first, "exact_next_by_value_s": t_next,
                      "exact_first_by_label_value_s": t_first_l, "exact_next_by_label_value_s": t_next_l}), flush=True)

    for frac in (0.001, 0.01, 0.05, 0.2, 0.5):
        w = int(n * frac)
        lo = int(rng.integers(0, n - w))
        shared = np.tile(np.array([lo, lo + w - 1], np.int64), (nq, 1))
        starts = rng.integers(0, n - w, nq)
        own = np.stack([starts, starts + w - 1], 1).astype(np.int64)
        rf = []
        t_fil = timed(lambda: rf.append(h.make_filter(np.ascontiguousarray(ids[(attr >= lo) & (attr < lo + w)]))))
        graph = frac >= 0.05
        if graph:
            compare({"ranges_s": lambda: h.search_flat_ranges(Q, k, ef, shared, with_pid=False),
                     "filter_s": lambda: h.search_flat(Q, k, ef, filter=rf[0], with_pid=False)},
                    args.runs, admitted=frac, search="graph", window="shared", setup_filter_new_s=t_fil)
        compare({"ranges_s": lambda: h.search_exact_ranges(Q, k, shared, with_pid=False),
                 "filter_s": lambda: h.search_exact(Q, k, filter=rf[0], with_pid=False)},
                args.runs, admitted=frac, search="exact", window="shared", setup_filter_new_s=t_fil)
        rf[0].free()
        for kind, call in (("graph", lambda r: h.search_flat_ranges(Q, k, ef, r, with_pid=False)),
                           ("exact", lambda r: h.search_exact_ranges(Q, k, r, with_pid=False)))[0 if graph else 1:]:
            ts = {"shared_s": [], "per_row_s": []}
            for _ in range(args.runs):
                ts["shared_s"].append(timed(lambda: call(shared)))
                ts["per_row_s"].append(timed(lambda: call(own)))
            print(json.dumps({"admitted": frac, "search": kind, "window": "shared vs one per row", **ts}), flush=True)

    w = n // 2
    lo = int(rng.integers(0, n - w))
    win = np.tile(np.array([lo, lo + w - 1], np.int64), (nq, 1))
    sel = np.arange(nq) % 20
    in_win = (attr >= lo) & (attr < lo + w)
    for s in (1, 4):
        sets = [sorted(rng.choice(T, s, replace=False).tolist()) for _ in range(20)]
        qs = [sets[g] for g in sel]
        rfs = []
        t_fil = timed(lambda: rfs.extend(h.make_filter(np.ascontiguousarray(ids[in_win & np.isin(lab, st)])) for st in sets))
        filters = [rfs[g] for g in sel]
        compare({"ranges_s": lambda: h.search_flat_ranges(Q, k, ef, win, qs, with_pid=False),
                 "per_query_s": lambda: h.search_flat_per_query(Q, k, ef, filters, with_pid=False)},
                args.runs, T=T, labels_per_set=s, admitted=0.5 * s / T, search="graph", setup_filter_new_s=t_fil)
        compare({"ranges_s": lambda: h.search_exact_ranges(Q, k, win, qs, with_pid=False),
                 "per_query_s": lambda: h.search_exact_per_query(Q, k, filters, with_pid=False)},
                args.runs, T=T, labels_per_set=s, admitted=0.5 * s / T, search="exact")
        for rf in rfs:
            rf.free()


if __name__ == "__main__":
    main()
