"""Exact search against filtered HNSW, and hnsw_b200_bruteforce against another build of the library.

  python scripts/measure_exact.py exact
      c2 shape (clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10).  Filters admit
      origin id g when g % 1000 < 1, 10, 50, 200, 500, 1000 (0.1 ... 100 %).  Per filter: ms per warmed call of
      search_exact (host clock around calls that end in a synchronisation) and search_exact_device's kernel time (CUDA
      events); search_flat_filtered with the same resident filter at ef = 64 (below 5 % admitted timed on the first
      HNSW_NQ queries and scaled to 10 000); the recall@10 of the latter against the
      former; and the kernel's share of its bound, the larger of 2 * nq * admitted * d flop at the data sheet's
      67 TFLOP/s FP32 and the bytes it must read (every query tile reads the admitted rows once) at 3.35 TB/s.
  python scripts/measure_exact.py ab OTHER_TREE [--reps R]
      hnsw_b200_bruteforce with this tree's library and another tree's (OTHER_TREE/hnswlib-rs_b200 with its lib/, e.g.
      an earlier commit's, run with its own hnsw.py and selected by HNSW_B200_LIB), alternating, R runs each, one process
      per run: nq = 20, 1 000, 10 000 over the c2 points and 1 000 queries at the c4 shape (60 000 x 784 f32), k = 10 and
      100.  Prints ms per call of every run and whether the two builds' outputs are identical.
Prints the card and its power limit first.  One JSON line per result."""
import hashlib
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

C2 = dict(n=1_000_000, d=128, nq=10_000)
FRACTIONS = (1, 10, 50, 200, 500, 1000)   # per mille admitted
PEAK_FLOPS, PEAK_BYTES = 67e12, 3.35e12
HNSW_NQ = 200


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def per_call_s(fn, reps, warm=1):
    for _ in range(warm):
        fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def recall(found, counts, truth, tcounts):
    tot, k = 0.0, truth.shape[1]
    for i in range(len(truth)):
        want = set(truth[i, :tcounts[i]].tolist())
        if want:
            tot += len(set(found[i, :counts[i]].tolist()) & want) / min(k, len(want))
        else:
            tot += 1.0
    return tot / len(truth)


def exact():
    pkg = importlib.import_module("hnswlib-rs_b200")
    import torch
    n, d, nq, k, ef = C2["n"], C2["d"], C2["nq"], 10, 64
    X = pkg.datagen.clustered(n, d, 1)
    bq = torch.empty(nq * d * 4, dtype=torch.uint8, pin_memory=True)
    Q = bq.numpy().view(np.float32).reshape(nq, d)
    Q[:] = pkg.datagen.clustered(nq, d, 2)
    print(json.dumps({"gpu": gpu_info(), "shape": "c2", "n": n, "dim": d, "nq": nq, "k": k, "ef": ef}), flush=True)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    qd = torch.from_numpy(np.asarray(Q)).cuda()
    dout = torch.empty((nq, k, 16), dtype=torch.uint8, device="cuda")
    dcnt = torch.empty((nq,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ids = np.arange(n, dtype=np.uint64)
    for pm in FRACTIONS:
        allow = np.ascontiguousarray(ids[ids % 1000 < pm])
        a = len(allow)
        with h.make_filter(allow) as rf:
            row = {"admitted_pct": pm / 10, "admitted": a}
            ex = h.search_exact(Q, k, filter=rf)
            t_ex = per_call_s(lambda: h.search_exact(Q, k, filter=rf, with_pid=False), reps=5)
            ms = [h.search_exact_device(qd.data_ptr(), nq, k, dout.data_ptr(), dcnt.data_ptr(), filter=rf) for _ in range(6)][1:]
            kern = float(np.median(ms)) * 1e-3
            print(json.dumps(dict(row, exact_ms=round(t_ex * 1e3, 3), exact_kernel_ms=round(kern * 1e3, 3))), flush=True)
            # a selective filter makes every graph search expand until its candidate queue is empty: below 5 % a
            # 10 000-query call takes minutes, so the graph search is timed on the first HNSW_NQ queries there and
            # reported per 10 000 queries; one timed call after the first (which also grows the visited tables)
            hq = nq if pm >= 50 else HNSW_NQ
            hn = h.search_flat(Q[:hq], k, ef, filter=rf)
            t_hn = per_call_s(lambda: h.search_flat(Q[:hq], k, ef, filter=rf, with_pid=False), reps=5 if pm >= 50 else 1,
                              warm=0) * nq / hq
            row["hnsw_timed_queries"] = hq
            flop_s = 2.0 * nq * a * d / PEAK_FLOPS
            byte_s = (-(-nq // 32) * a * d * 4 + nq * d * 4) / PEAK_BYTES
            row.update(exact_ms=round(t_ex * 1e3, 3), exact_kernel_ms=round(kern * 1e3, 3), hnsw_ef64_ms=round(t_hn * 1e3, 3),
                       hnsw_recall10=round(recall(hn[0], hn[4], ex[0][:hq], ex[4][:hq]), 4),
                       kernel_bound="fp32" if flop_s >= byte_s else "bytes",
                       kernel_share_of_bound=round(max(flop_s, byte_s) / kern, 3) if kern > 0 else None,
                       exact_faster=bool(t_ex < t_hn))
            print(json.dumps(row), flush=True)
    h.close()


def ab_data(tmp, shape, nq):
    """the points and queries of a shape, made once and saved under tmp for every run"""
    pkg = importlib.import_module("hnswlib-rs_b200")
    if shape == "c2":
        X, Q = pkg.datagen.clustered(C2["n"], C2["d"], 1), pkg.datagen.clustered(nq, C2["d"], 2)
    else:
        X, Q = pkg.datagen.uniform(60_000, 784, 3), pkg.datagen.uniform(nq, 784, 4)
    np.save(os.path.join(tmp, "X.npy"), X)
    np.save(os.path.join(tmp, "Q.npy"), Q)


def ab_child(tree, tmp, k, reps):
    """one run in this process, on the package of `tree`: ms per call of bruteforce, and a digest of the outputs"""
    sys.path.insert(0, tree)
    pkg = importlib.import_module("hnswlib-rs_b200")
    X, Q = np.load(os.path.join(tmp, "X.npy")), np.load(os.path.join(tmp, "Q.npy"))
    n = len(X)
    h = pkg.Hnsw(16, n, 16, 48, "DistL2")
    h.import_graph(X, np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), 0,
                   [(np.zeros(n + 1, np.uint64), np.zeros(0, np.uint32), None)])
    out = h.bruteforce(Q, k)
    t = per_call_s(lambda: h.bruteforce(Q, k), reps=reps, warm=0)
    dig = hashlib.sha256(out[0].tobytes() + out[1].tobytes()).hexdigest()[:16]
    print(json.dumps({"ms": round(t * 1e3, 3), "digest": dig}), flush=True)


def ab(other, runs):
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    shapes = [("c2", 20), ("c2", 1000), ("c2", 10_000), ("c4", 1000)]
    trees = {"this": ROOT, "other": os.path.abspath(other)}
    tmp = tempfile.mkdtemp(prefix="hnsw_ab_")
    for shape, nq in shapes:
        ab_data(tmp, shape, nq)
        for k in (10, 100):
            res = {"this": [], "other": []}
            digests = {"this": set(), "other": set()}
            for _ in range(runs):
                for name, tree in trees.items():
                    env = dict(os.environ, HNSW_B200_LIB=os.path.join(tree, "hnswlib-rs_b200", "lib", "libhnsw_b200.so"))
                    reps = 3 if nq >= 10_000 else 10
                    r = subprocess.run([sys.executable, __file__, "ab-child", tree, tmp, str(k), str(reps)], env=env,
                                       capture_output=True, text=True, check=True)
                    j = json.loads(r.stdout.strip().splitlines()[-1])
                    res[name].append(j["ms"])
                    digests[name].add(j["digest"])
            print(json.dumps({"shape": shape, "nq": nq, "k": k, "this_ms": res["this"], "other_ms": res["other"],
                              "identical": len(digests["this"] | digests["other"]) == 1}), flush=True)


if __name__ == "__main__":
    if sys.argv[1] == "exact":
        exact()
    elif sys.argv[1] == "ab":
        ab(sys.argv[2], int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3)
    elif sys.argv[1] == "ab-child":
        ab_child(sys.argv[2], sys.argv[3], int(sys.argv[4]), int(sys.argv[5]))
