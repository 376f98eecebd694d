"""Partitioned index at the c2 shape (clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 queries, k = 10,
ef = 64): unpartitioned, P = 2 and 4 on device 0, and P = every GPU when there are several.

Per configuration: build seconds; search_flat queries/s from pinned buffers (host clock over 20 warmed synchronous calls);
the merge's share of a call; recall@10 against the handle's own bruteforce.  The merge share is estimated: the same P
searches run on the partition views from P host threads at once (kernels, synchronisation and the ordinary unpack, no
merge), and the share is 1 - t(views) / t(partitioned call).  Prints one JSON line per configuration."""
import ctypes as C
import importlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("hnswlib-rs_b200")
import torch  # noqa: E402  (pinned host buffers)

N, D, M, EFC, NQ, K, EF, CALLS = 1_000_000, 128, 16, 200, 10_000, 10, 64, 20


def pinned(shape, dtype):
    t = torch.empty(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8, pin_memory=True)
    return t, t.numpy().view(dtype).reshape(shape)


def gpu_info():
    out = []
    for i in range(torch.cuda.device_count()):
        q = subprocess.run(["nvidia-smi", "-i", str(i), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True)
        out.append(q.stdout.strip() or torch.cuda.get_device_name(i))
    return out


def timed_calls(fn):
    for _ in range(3):
        fn()
    t = time.perf_counter()
    for _ in range(CALLS):
        fn()
    return (time.perf_counter() - t) / CALLS


def main():
    L = pkg.load_library()
    X = pkg.datagen.clustered(N, D, 1)
    keep = []
    bq, Q = pinned((NQ, D), np.float32)
    Q[:] = pkg.datagen.clustered(NQ, D, 2)
    outs = [pinned((NQ, K), np.uint64), pinned((NQ, K), np.float32), pinned((NQ, K), np.uint32), pinned((NQ,), np.int32)]
    keep += [bq] + [o[0] for o in outs]
    o_ids, o_d, o_it, o_c = [o[1] for o in outs]
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    ngpu = torch.cuda.device_count()
    configs = [("unpartitioned", None), ("P=2 on device 0", [0, 0]), ("P=4 on device 0", [0, 0, 0, 0])]
    if ngpu > 1:
        configs.append((f"P={ngpu} on {ngpu} GPUs", list(range(ngpu))))
    info = gpu_info()
    print(json.dumps({"gpus": info}), flush=True)
    for name, devs in configs:
        h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
        if devs:
            h.partition(devs)
        t = time.perf_counter()
        h.insert_flat(X)
        build_s = time.perf_counter() - t

        def call(hh=h):
            r = L.hnsw_b200_search_flat(hh._h, p(Q), NQ, D, K, EF, 0, None, 0, pkg.hnsw.FILTER_FN(0), None,
                                        p(o_ids), p(o_d), p(o_it), None, p(o_c))
            assert r == 0, pkg.last_error()
        t_call = timed_calls(call)
        it, c = o_it.copy(), o_c.copy()
        ti, _ = h.bruteforce(np.asarray(Q), K)
        rec = float(np.mean([len(set(it[i, :c[i]].tolist()) & set(ti[i].tolist())) / K for i in range(NQ)]))
        row = {"config": name, "build_s": round(build_s, 2), "qps": round(NQ / t_call, 1), "call_ms": round(t_call * 1e3, 3),
               "recall@10": round(rec, 4)}
        if devs:
            views = [h.partition_view(i) for i in range(len(devs))]
            bufs = [[pinned((NQ, K), np.uint64), pinned((NQ, K), np.float32), pinned((NQ,), np.int32)] for _ in views]
            keep += [b[0] for bb in bufs for b in bb]

            def one(v, b):
                r = L.hnsw_b200_search_flat(v._h, p(Q), NQ, D, K, EF, 0, None, 0, pkg.hnsw.FILTER_FN(0), None,
                                            p(b[0][1]), p(b[1][1]), None, None, p(b[2][1]))
                assert r == 0, pkg.last_error()

            def all_views():
                th = [threading.Thread(target=one, args=(v, b)) for v, b in zip(views, bufs)]
                for x in th:
                    x.start()
                for x in th:
                    x.join()
            t_views = timed_calls(all_views)
            row["views_ms"] = round(t_views * 1e3, 3)
            row["merge_share_est"] = round(max(0.0, 1 - t_views / t_call), 3)
        print(json.dumps(row), flush=True)
        h.close()


if __name__ == "__main__":
    main()
