"""Link mode 0 (the reference's back-links, filed under the new point's level) against link mode 1 (filed per layer).

  python scripts/measure_link_mode.py [--n N] [--nq NQ]
      c2 shape by default: clustered 1 M x 128 f32, M = 16, ef_construction = 200, 10 000 queries, k = 10.  Both modes
      are built from the same levels (drawn once from the reference's law).  Per mode: build seconds; level >= 1 points
      (the entry point excepted) that no layer-0 list names; then for each ef, recall@10 against hnsw_b200_bruteforce's
      exact answers, queries/s of warmed synchronous search_flat calls on pinned queries (host clock around calls that
      end in a synchronisation, median of 5) and search_device's kernel milliseconds (CUDA events, median of 5).
      Last, the lowest ef at which each mode reaches recall 0.90 and 0.95.
Prints the card and its power limit first.  One JSON line per result."""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

M, EFC, K = 16, 200, 10
EFS = (10, 16, 24, 32, 48, 64, 96, 128)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def median_call_s(fn, reps=5):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def recall(found, counts, truth):
    return float(np.mean([len(set(found[i, :counts[i]].tolist()) & set(truth[i].tolist())) / truth.shape[1]
                          for i in range(len(truth))]))


def without_layer0_inlink(h, levels):
    _, ids, _ = h.export_layer(0)
    linked = np.zeros(len(levels), bool)
    linked[ids.astype(np.int64)] = True
    entry = h.export_points()[3]
    miss = (levels >= 1) & ~linked
    miss[entry] = False
    return int(miss.sum())


def main(n, nq):
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    d = 128
    X = pkg.datagen.clustered(n, d, 1)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = pkg.datagen.clustered(nq, d, 2)
    # LayerGenerator::generate (hnsw.rs:363-374) with scale 1 / ln(M), drawn once for both builds
    u = np.random.default_rng(7).random(n)
    levels = np.minimum(np.floor(-np.log(np.maximum(u, 1e-300)) / np.log(M)), 15).astype(np.int32)
    print(json.dumps({"gpu": gpu_info(), "n": n, "dim": d, "nq": nq, "k": K, "M": M, "ef_construction": EFC}), flush=True)
    qd = torch.from_numpy(np.asarray(Q)).cuda()
    dout = torch.empty((nq, K, 16), dtype=torch.uint8, device="cuda")
    dcnt = torch.empty((nq,), dtype=torch.int32, device="cuda")
    truth = None
    reach = {}
    for mode in (0, 1):
        h = pkg.Hnsw(M, n, 16, EFC, "DistL2")
        h.set_link_mode(mode)
        torch.cuda.synchronize()
        t = time.perf_counter()
        h.insert_flat(X, levels=levels)
        build_s = time.perf_counter() - t
        if truth is None:
            truth, _ = h.bruteforce(Q, K)
        print(json.dumps({"mode": mode, "build_s": round(build_s, 3),
                          "level_ge1_without_layer0_inlink": without_layer0_inlink(h, levels),
                          "level_ge1_points": int((levels >= 1).sum())}), flush=True)
        reach[mode] = {}
        for ef in EFS:
            got = h.search_flat(Q, K, ef)
            r = recall(got[2], got[4], truth)
            t_call = median_call_s(lambda: h.search_flat(Q, K, ef, with_pid=False))
            h.search_device(qd.data_ptr(), nq, K, ef, dout.data_ptr(), dcnt.data_ptr())
            kern = float(np.median([h.search_device(qd.data_ptr(), nq, K, ef, dout.data_ptr(), dcnt.data_ptr())
                                    for _ in range(5)]))
            print(json.dumps({"mode": mode, "ef": ef, "recall10": round(r, 4), "search_flat_qps": round(nq / t_call),
                              "search_device_kernel_ms": round(kern, 3)}), flush=True)
            for bar in (0.90, 0.95):
                if r >= bar and bar not in reach[mode]:
                    reach[mode][bar] = ef
        h.close()
    print(json.dumps({"lowest_ef_reaching": {f"mode{m}": {str(b): reach[m].get(b) for b in (0.90, 0.95)}
                                             for m in (0, 1)}}), flush=True)


if __name__ == "__main__":
    a = sys.argv
    main(int(a[a.index("--n") + 1]) if "--n" in a else 1_000_000, int(a[a.index("--nq") + 1]) if "--nq" in a else 10_000)
