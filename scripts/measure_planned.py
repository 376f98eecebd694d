"""Planned search against the two calls it chooses between.

  python scripts/measure_planned.py [--n N] [--nq NQ] [--sweep-nq NQ] [--runs R] [--parts sweep,mix]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; k = 10.
  * Crossover sweep: label 0 on a share s of the points (2 % to 60 %), label 1 on the rest; --sweep-nq queries each
    restricted to label 0, through search_flat_label_sets and search_exact_label_sets, at ef = 64 and ef = 128.  The
    measured crossover c* is where the two times meet (log-log interpolation between the bracketing shares), and the
    measured GAMMA is c*^2 / (n e D); the rule's own crossover is sqrt(GAMMA n e D) at the library's GAMMA.
  * Tenant mix: 1 000 tenants whose sizes follow a Zipf law (size of rank r proportional to 1 / r), each point in one
    tenant; each query asks within a tenant drawn in proportion to its size, and 0 % or 20 % of the rows are
    unrestricted.  search_planned against search_exact_label_sets on the same batch at ef = 64; the planned rows are
    checked first against the exact rows and, on their own, the graph rows the rule picked.
Each side is timed with the host clock around a call that ends in a synchronisation; the sides alternate within each
of R runs and the median is reported, in ms per batch.  The tenant mix's pure graph call is not timed: its rows of the
smallest tenants (about 130 points) search most of the graph, and neither the whole batch nor its first 200 rows
finished within 6 minutes on an H100.  Prints the card and its power limit first, then one JSON line per measurement."""
import argparse
import importlib
import json
import math
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GAMMA = int(re.search(r"#define HNSW_B200_PLANNED_GAMMA (\d+)",
                      open(os.path.join(ROOT, "include", "hnsw_b200.h")).read()).group(1))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def median_ms(sides, runs):
    """{name: median ms} of the callables, alternating within each run"""
    t = {name: [] for name in sides}
    for _ in range(runs):
        for name, fn in sides.items():
            s = time.perf_counter()
            fn()
            t[name].append((time.perf_counter() - s) * 1e3)
    return {name: round(float(np.median(v)), 2) for name, v in t.items()}


def same_rows(a, b, rows):
    return all(np.array_equal(x[rows], y[rows]) for x, y in zip((a[2], a[1].view(np.uint32), a[4]),
                                                                 (b[2], b[1].view(np.uint32), b[4])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--sweep-nq", type=int, default=2_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parts", default="sweep,mix")
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "gamma": GAMMA}), flush=True)
    pkg = importlib.import_module("hnswlib-rs_b200")
    n, d, M, k = a.n, 128, 16, 10
    X = pkg.datagen.clustered(n, d, 1)
    h = pkg.Hnsw(M, n, 16, 200, "DistL2")
    s = time.perf_counter()
    h.insert_flat(X)
    print(json.dumps({"build_s": round(time.perf_counter() - s, 1), "n": n}), flush=True)
    rng = np.random.default_rng(7)

    # crossover sweep
    Qs = pkg.datagen.clustered(a.sweep_nq, d, 2)
    one = [[0]] * a.sweep_nq
    order = rng.permutation(n)
    for ef in (64, 128) if "sweep" in a.parts else ():
        pts = []
        for share in (0.02, 0.05, 0.1, 0.2, 0.3, 0.4, 0.6):
            c = int(n * share)
            lab = np.ones(n, np.uint32)
            lab[order[:c]] = 0
            h.set_labels(0, lab)
            h.search_exact_label_sets(Qs[:64], k, one[:64])   # the scan order is built once per label change
            ms = median_ms({"graph": lambda: h.search_flat_label_sets(Qs, k, ef, one, with_pid=False),
                            "exact": lambda: h.search_exact_label_sets(Qs, k, one, with_pid=False)}, a.runs)
            pts.append((c, ms["graph"], ms["exact"]))
            print(json.dumps({"sweep": "c2", "ef": ef, "nq": a.sweep_nq, "share": share, "admitted": c,
                              "graph_ms": ms["graph"], "exact_ms": ms["exact"],
                              "rule_picks": "exact" if c * c <= GAMMA * n * ef * 2 * M else "graph"}), flush=True)
        cross = None
        for (c0, g0, e0), (c1, g1, e1) in zip(pts, pts[1:]):
            r0, r1 = math.log(g0 / e0), math.log(g1 / e1)
            if r0 > 0 >= r1:   # the graph turns faster between c0 and c1
                cross = math.exp(math.log(c0) + (math.log(c1) - math.log(c0)) * r0 / (r0 - r1))
        rule = math.sqrt(GAMMA * n * ef * 2 * M)
        print(json.dumps({"crossover": "c2", "ef": ef, "measured_admitted": None if cross is None else round(cross),
                          "measured_gamma": None if cross is None else round(cross * cross / (n * ef * 2 * M), 2),
                          "rule_admitted": round(rule),
                          "rule_over_measured": None if cross is None else round(rule / cross, 2)}), flush=True)

    if "mix" not in a.parts:
        return
    # tenant mix
    T = 1000
    w = 1.0 / np.arange(1, T + 1)
    sizes = np.maximum(1, np.floor(w / w.sum() * n)).astype(np.int64)
    sizes[0] += n - sizes.sum()
    lab = np.repeat(np.arange(T, dtype=np.uint32), sizes)[np.argsort(order)]
    h.set_labels(0, lab)
    Q = pkg.datagen.clustered(a.nq, d, 3)
    tenant = rng.choice(T, a.nq, p=sizes / n)
    ef = 64
    for free in (0.0, 0.2):
        sets = [[pkg.LABEL_NONE] if rng.random() < free else [int(t)] for t in tenant]
        off, vals = pkg.hnsw._label_sets(sets, a.nq)   # the (offsets, values) pair the C calls take, made once
        packed = (off, vals)
        got = h.search_planned(Q, k, ef, sets=packed, with_pid=False)
        ex = got[5].astype(bool)
        gr = np.flatnonzero(~ex)   # the graph rows, checked on their own: the whole graph call is too slow
        g = h.search_flat_label_sets(Q[gr], k, ef, [sets[i] for i in gr], with_pid=False)
        x = h.search_exact_label_sets(Q, k, packed, with_pid=False)
        assert same_rows(got, x, ex), "planned rows differ from the exact rows the rule picked"
        assert all(np.array_equal(u[gr], v) for u, v in zip((got[2], got[1].view(np.uint32), got[4]),
                                                            (g[2], g[1].view(np.uint32), g[4]))), "graph rows differ"
        ms = median_ms({"planned": lambda: h.search_planned(Q, k, ef, sets=packed, with_pid=False),
                        "exact": lambda: h.search_exact_label_sets(Q, k, packed, with_pid=False)}, a.runs)
        print(json.dumps({"mix": "zipf", "tenants": T, "nq": a.nq, "ef": ef, "unrestricted": free,
                          "exact_rows": int(ex.sum()), "planned_ms": ms["planned"], "exact_ms": ms["exact"]}), flush=True)


if __name__ == "__main__":
    main()
