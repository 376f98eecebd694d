"""Excluded points per query against what a caller can do without them.

  python scripts/measure_exclusions.py [--n N] [--nq NQ] [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 queries, k = 10, ef = 64.  Each query's list E
(|E| = 0, 16, 256, 4096) is drawn half from its true 50 nearest (at most all 50) and the rest at random.  Per |E|:
  * search_flat_excluding and search_exact_excluding: queries/s, and recall@10 against the exact rows (the exact call
    is the truth, so its recall is 1 by construction);
  * over-fetch and drop: search_flat with k + |E| (ef = max(64, k + |E|)), then E dropped in numpy (vectorised) and
    the rows cut to k; the search and the drop are timed apart, and a k + |E| the kernel refuses is reported as such;
  * one resident filter per query (filter_new over the query's admitted ids, then search_flat_filtered), on the first
    100 queries only, filter set-up included.
Each side is timed with the host clock around calls that end in a synchronisation, the sides alternating within each
of R runs; the best run is reported.  Prints the card and its power limit first, then one JSON line per measurement."""
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
    out = fn()
    return time.perf_counter() - t, out


def recall(got, truth, k):
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
    Q = pkg.datagen.clustered(a.nq, d, 2)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    t, _ = timed(lambda: h.insert_flat(X))
    print(json.dumps({"build_s": round(t, 1), "n": n}), flush=True)
    top50 = h.search_exact(Q, 50, with_pid=False)[2].astype(np.int64)
    rng = np.random.default_rng(3)
    for size in (0, 16, 256, 4096):
        near = min(size // 2, 50)
        E = [np.concatenate([top50[i, :near], rng.choice(n, size - near, replace=False)]) for i in range(a.nq)]
        packed = pkg.hnsw._excluded(E, a.nq)   # the (offsets, ranks) pair the C calls take, made once
        truth = h.search_exact_excluding(Q, k, packed, with_pid=False)
        # E as one sorted array of row * n + rank keys, so that the over-fetch side drops it with one np.isin
        rows = np.arange(a.nq, dtype=np.int64)[:, None] * n
        Ekeys = (np.stack(E) + rows).ravel() if size else np.zeros(0, np.int64)

        def overfetch_search():
            kk = k + size
            return h.search_flat(Q, kk, max(ef, kk), with_pid=False)

        def overfetch_drop(r):
            ids, cnt = r[2].astype(np.int64), r[4]
            live = np.arange(ids.shape[1])[None, :] < cnt[:, None]
            keep = live & ~np.isin(ids + rows, Ekeys)
            order = np.argsort(~keep, axis=1, kind="stable")[:, :k]   # the kept slots first, in their order
            out_ids = np.take_along_axis(np.where(keep, ids, 0xFFFFFFFF), order, 1)
            return None, None, out_ids, None, np.minimum(keep.sum(1), k).astype(np.int32)

        small = min(100, a.nq)

        def per_query_filters():
            for i in range(small):
                rf = h.make_filter(np.setdiff1d(np.arange(n), E[i]).astype(np.uint64))
                h.search_flat(Q[i:i + 1], k, ef, filter=rf, with_pid=False)
                rf.free()

        sides = {"flat_excluding": lambda: h.search_flat_excluding(Q, k, ef, packed, with_pid=False),
                 "exact_excluding": lambda: h.search_exact_excluding(Q, k, packed, with_pid=False)}
        best, res = {}, {}
        over_ok = True
        for _ in range(a.runs):
            for name, fn in sides.items():
                t, res[name] = timed(fn)
                best[name] = min(best.get(name, t), t)
            if over_ok:
                try:
                    t, r = timed(overfetch_search)
                except pkg.HnswError as e:   # k + |E| beyond what one query's shared memory holds
                    over_ok = False
                    print(json.dumps({"E": size, "side": "overfetch", "refused": str(e)}), flush=True)
                else:
                    best["overfetch_search"] = min(best.get("overfetch_search", t), t)
                    t, res["overfetch"] = timed(lambda: overfetch_drop(r))
                    best["overfetch_drop"] = min(best.get("overfetch_drop", t), t)
            t, _ = timed(per_query_filters)
            best["filter_per_query"] = min(best.get("filter_per_query", t), t)
        for name in sides:
            print(json.dumps({"E": size, "side": name, "qps": round(a.nq / best[name]),
                              "recall@10": round(recall(res[name], truth, k), 4)}), flush=True)
        if over_ok:
            print(json.dumps({"E": size, "side": "overfetch", "search_s": round(best["overfetch_search"], 4),
                              "drop_s": round(best["overfetch_drop"], 4),
                              "qps_search_only": round(a.nq / best["overfetch_search"]),
                              "qps_with_drop": round(a.nq / (best["overfetch_search"] + best["overfetch_drop"])),
                              "recall@10": round(recall(res["overfetch"], truth, k), 4)}), flush=True)
        print(json.dumps({"E": size, "side": "filter_per_query", "nq": small, "qps": round(small / best["filter_per_query"], 1)}),
              flush=True)


if __name__ == "__main__":
    main()
