"""Point labels against one resident filter per tenant.

  python scripts/measure_labels.py [--runs R]

c2 shape: clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10, ef = 64.  Points are
labelled round robin (point g carries label g % T) and query i is restricted to label i % T, so one label admits 1/T of
the points.  The per-query side gives tenant t the resident filter admitting the same points (origin ids g with
g % T == t).  Timed with the host clock around calls that end in a synchronisation, after one warm-up of each:
  * setup: one set_labels call over 1 M points, against T filter_new calls (id lists);
  * search: one search_flat_labeled call against one search_flat_per_query call (graph, T = 2 and 20), and
    search_exact_labeled against search_exact_per_query (T = 20, 1 000 and 100 000; at 100 000 the per-query side is
    not run, its memory is computed).  The answers are checked equal before anything is timed; the two alternate
    within each of R runs;
  * churn: 10 000 new points inserted, then one set_labels of their 10 000 labels, against T filter rebuilds (free and
    filter_new over the grown index), followed by one search of each kind, checked equal.
Memory is computed from the layouts: labels 4 bytes per point on the device and 4 on the host, plus the exact path's
CSR, 4 bytes per labelled point per device; a filter n / 8 bytes on the device and n / 8 on the host per tenant, plus
its exact id list, 4 bytes per admitted point per device.  Prints the card and its power limit first, then one JSON
line per measurement."""
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


def memory(n, T, exact):
    """bytes on the device and on the host: labels, and one filter per tenant (round robin: every point admitted once)"""
    lab_dev = 4 * n + (4 * n if exact else 0)
    fil_dev = T * ((n + 31) // 32 + 1) * 4 + (4 * n if exact else 0)
    return {"labels_device_bytes": lab_dev, "labels_host_bytes": 4 * n,
            "filters_device_bytes": fil_dev, "filters_host_bytes": T * ((n + 31) // 32 + 1) * 4}


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
    h = pkg.Hnsw(16, n + nq, 16, 200, "DistL2")
    h.insert_flat(X)
    ids = np.arange(n, dtype=np.uint64)
    iq = np.arange(nq)

    def filters(T, count):
        return [h.make_filter(np.ascontiguousarray(ids[t::T])) for t in range(T)] if count else []

    for T, kinds in ((2, ("graph",)), (20, ("graph", "exact")), (1000, ("exact",)), (100000, ("exact",))):
        lab = (np.arange(n) % T).astype(np.uint32)
        ql = (iq % T).astype(np.uint32)
        t_lab = timed(lambda: h.set_labels(0, lab))
        run_pq = T <= 1000
        rfs = []
        t_fil = timed(lambda: rfs.extend(filters(T, run_pq))) if run_pq else None
        for kind in kinds:
            if kind == "graph":
                lab_call = lambda: h.search_flat_labeled(Q, k, ef, ql, with_pid=False)   # noqa: E731
                pq_call = lambda: h.search_flat_per_query(Q, k, ef, [rfs[i % T] for i in iq], with_pid=False)   # noqa: E731
            else:
                lab_call = lambda: h.search_exact_labeled(Q, k, ql, with_pid=False)   # noqa: E731
                pq_call = lambda: h.search_exact_per_query(Q, k, [rfs[i % T] for i in iq], with_pid=False)   # noqa: E731
            a = lab_call()
            if run_pq:
                assert equal(a, pq_call()), (T, kind, "labelled rows differ from the per-query filters'")
            ts_lab, ts_pq = [], []
            for _ in range(args.runs):
                ts_lab.append(timed(lab_call))
                if run_pq:
                    ts_pq.append(timed(pq_call))
            print(json.dumps({"T": T, "search": kind, "labeled_s": ts_lab, "per_query_s": ts_pq if run_pq else "not run",
                              "setup_set_labels_s": t_lab, "setup_filter_new_s": t_fil if run_pq else "not run",
                              **memory(n, T, kind == "exact")}), flush=True)
        for rf in rfs:
            rf.free()

    # churn at T = 20: insert 10 000 labelled points, then search
    T = 20
    h.set_labels(0, (np.arange(n) % T).astype(np.uint32))
    rfs = filters(T, True)
    ql = (iq % T).astype(np.uint32)
    Xn = pkg.datagen.clustered(nq, d, 3)
    t_ins = timed(lambda: h.insert_flat(Xn, ids=np.arange(n, n + nq, dtype=np.uint64)))
    new_lab = (np.arange(n, n + nq) % T).astype(np.uint32)
    t_lab = timed(lambda: h.set_labels(n, new_lab))
    n2 = n + nq
    ids2 = np.arange(n2, dtype=np.uint64)

    def rebuild():
        for rf in rfs:
            rf.free()
        rfs[:] = [h.make_filter(np.ascontiguousarray(ids2[t::T])) for t in range(T)]
    t_fil = timed(rebuild)
    a = h.search_flat_labeled(Q, k, ef, ql, with_pid=False)
    b = h.search_flat_per_query(Q, k, ef, [rfs[i % T] for i in iq], with_pid=False)
    assert equal(a, b), "after the churn, labelled rows differ from the rebuilt filters'"
    print(json.dumps({"churn": "insert 10 000 then search", "T": T, "insert_s": t_ins, "set_labels_s": t_lab,
                      "filter_rebuild_s": t_fil}), flush=True)


if __name__ == "__main__":
    main()
