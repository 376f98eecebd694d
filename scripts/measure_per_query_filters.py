"""One per-query call against one call per distinct filter.

  python scripts/measure_per_query_filters.py [--runs R] [--tenants 1,10,100,1000]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10, ef = 64.  Query i
belongs to tenant i % T.  Tenant t's resident filter admits origin id g when (g + 7919 t) % 100 < 5 (about 5 %) or
< 50 (about 50 %), a different subset per tenant.  The "mix" variant leaves every fifth query (20 %) unfiltered (-1).
Per (T, admitted, mix), timed with the host clock around calls that end in a synchronisation, after one warm-up of each:
  * graph: one search_flat_per_query call; T sequential search_flat_filtered calls (plus one unfiltered call for the
    -1 rows); T submit_filtered calls with up to 4 in flight;
  * exact: one search_exact_per_query call; T search_exact calls (plus one with -1).
The methods alternate within each of R runs.  Before timing, the per-query answers are checked equal to the per-group
calls'.  Prints the card and its power limit first, then one JSON line per (T, admitted, mix) with the per-run seconds."""
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
    ap.add_argument("--tenants", default="1,10,100,1000")
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
    for T in [int(t) for t in args.tenants.split(",")]:
        for pct in (5, 50):
            rfs = [h.make_filter(np.ascontiguousarray(ids[(ids + 7919 * t) % 100 < pct])) for t in range(T)]
            for mix in (False, True):
                tenant = np.arange(nq) % T
                plain = (np.arange(nq) % 5 == 4) if mix else np.zeros(nq, bool)
                filters = [None if plain[i] else rfs[tenant[i]] for i in range(nq)]
                groups = [(rfs[t], np.flatnonzero((tenant == t) & ~plain)) for t in range(T)]
                groups = [(rf, rows) for rf, rows in groups if len(rows)]
                prows = np.flatnonzero(plain)
                # contiguous per-group copies of the pinned queries, as a caller that splits its batch would hold them
                gq = [(rf, torch.empty(len(r) * d * 4, dtype=torch.uint8, pin_memory=True).numpy().view(np.float32)
                       .reshape(len(r), d), r) for rf, r in groups]
                for _, buf, r in gq:
                    buf[:] = Q[r]
                pq_buf = Q[prows] if len(prows) else None

                def per_query():
                    return h.search_flat_per_query(Q, k, ef, filters, with_pid=False)

                def sequential():
                    out = [h.search_flat(buf, k, ef, filter=rf, with_pid=False) for rf, buf, _ in gq]
                    if pq_buf is not None:
                        out.append(h.search_flat(pq_buf, k, ef, with_pid=False))
                    return out

                def submitted():
                    tickets, out = [], []
                    for rf, buf, _ in gq:
                        tickets.append(h.submit_flat(buf, k, ef, with_pid=False, filter=rf))
                        if len(tickets) == 4:
                            out.append(h.wait_flat(tickets.pop(0)))
                    out += [h.wait_flat(t) for t in tickets]
                    if pq_buf is not None:
                        out.append(h.search_flat(pq_buf, k, ef, with_pid=False))
                    return out

                def exact_per_query():
                    return h.search_exact_per_query(Q, k, filters, with_pid=False)

                def exact_sequential():
                    out = [h.search_exact(buf, k, filter=rf, with_pid=False) for rf, buf, _ in gq]
                    if pq_buf is not None:
                        out.append(h.search_exact(pq_buf, k, with_pid=False))
                    return out

                # equal answers before timing (also the warm-up of every method)
                for one, many in ((per_query, sequential), (per_query, submitted), (exact_per_query, exact_sequential)):
                    a, b = one(), many()
                    rows = [r for _, _, r in gq] + ([prows] if len(prows) else [])
                    for r, got in zip(rows, b):
                        assert np.array_equal(a[0][r], got[0]) and np.array_equal(a[4][r], got[4])
                        assert np.array_equal(a[1][r].view(np.uint32), got[1].view(np.uint32))
                res = {m: [] for m in ("per_query", "sequential", "submit4", "exact_per_query", "exact_sequential")}
                for _ in range(args.runs):
                    res["per_query"].append(timed(per_query))
                    res["sequential"].append(timed(sequential))
                    res["submit4"].append(timed(submitted))
                    res["exact_per_query"].append(timed(exact_per_query))
                    res["exact_sequential"].append(timed(exact_sequential))
                print(json.dumps({"tenants": T, "admitted_pct": pct, "unfiltered_pct": 20 if mix else 0,
                                  **{m: [round(s, 4) for s in v] for m, v in res.items()}}), flush=True)
            for rf in rfs:
                rf.free()
    h.close()


if __name__ == "__main__":
    main()
