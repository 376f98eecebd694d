"""Filtered search at the c2 shape (clustered 1 M x 128 f32, M = 16, ef_construction = 200; 10 000 pinned queries, k = 10,
ef = 64): what a per-call FilterT costs next to the kernel, and what a resident filter (hnsw_b200_filter_new) saves.

Two filters: origin id g admitted when g % 100 < 50 (50 %) or < 5 (5 %).  Per filter, queries/s of one 10 000-query call
(host clock over warmed calls that end in a synchronisation), for
  * the per-call path (hnsw_b200_search_flat): sorted id list, a C callback, a Python callback (ctypes);
  * the resident path: search_flat_filtered; submit_filtered / wait with 2, 3 and 4 batches in flight; and
    search_device_filtered on device buffers (synchronous calls, and asynchronous pairs closed by join + check_status,
    whose overflow flag is reported: an asynchronous launch does not grow its visited tables);
  * the one-time hnsw_b200_filter_new (list, C callback, Python callback).
The C callback is compiled into a temporary directory with the host's C compiler.  Unfiltered search_flat is the
yardstick.  Prints the card and its power limit, then one JSON line per filter."""
import ctypes as C
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
pkg = importlib.import_module("hnswlib-rs_b200")
import torch  # noqa: E402  (pinned host buffers, device buffers)

N, D, M, EFC, NQ, K, EF = 1_000_000, 128, 16, 200, 10_000, 10, 64
WARM, REPS, REPS_PY = 2, 5, 2

C_FILTER = r"""
#include <stdint.h>
int admit(uint64_t id, void* ctx) { return (int)(id % 100) < *(const int*)ctx; }
"""


def c_callback():
    d = tempfile.mkdtemp(prefix="hnsw_filter_")
    src, so = os.path.join(d, "admit.c"), os.path.join(d, "libadmit.so")
    open(src, "w").write(C_FILTER)
    subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", so, src])
    return pkg.hnsw.FILTER_FN(("admit", C.CDLL(so)))


def pinned(shape, dtype):
    t = torch.empty(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8, pin_memory=True)
    return t, t.numpy().view(dtype).reshape(shape)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def per_call_s(fn, reps=REPS, warm=WARM):
    for _ in range(warm):
        fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def main():
    L = pkg.load_library()
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    chk = lambda r: r == 0 or sys.exit(pkg.last_error())  # noqa: E731
    X = pkg.datagen.clustered(N, D, 1)
    keep = []
    bq, Q = pinned((NQ, D), np.float32)
    Q[:] = pkg.datagen.clustered(NQ, D, 2)
    keep.append(bq)

    def out_set():
        o = [pinned((NQ, K), np.uint64), pinned((NQ, K), np.float32), pinned((NQ, K), np.uint32), pinned((NQ,), np.int32)]
        keep.extend(x[0] for x in o)
        return [x[1] for x in o]
    outs = [out_set() for _ in range(4)]
    o0 = outs[0]
    print(json.dumps({"gpu": gpu_info(), "shape": "c2", "n": N, "dim": D, "nq": NQ, "k": K, "ef": EF}), flush=True)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    t = time.perf_counter()
    h.insert_flat(X)
    print(json.dumps({"build_s": round(time.perf_counter() - t, 2)}), flush=True)
    ids = np.arange(N, dtype=np.uint64)
    none_cb = pkg.hnsw.FILTER_FN(0)
    admit = c_callback()
    qd = torch.from_numpy(np.asarray(Q)).cuda()
    dout = [torch.empty((NQ, K, 16), dtype=torch.uint8, device="cuda") for _ in range(2)]
    dcnt = [torch.empty((NQ,), dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()

    def flat(mode, fids, nf, cb, ctx):
        chk(L.hnsw_b200_search_flat(h._h, p(Q), NQ, D, K, EF, mode, fids, nf, cb, ctx, p(o0[0]), p(o0[1]), p(o0[2]), None,
                                    p(o0[3])))
    t_unf = per_call_s(lambda: flat(0, None, 0, none_cb, None))
    print(json.dumps({"unfiltered_qps": round(NQ / t_unf, 1)}), flush=True)
    for pct in (50, 5):
        allow = np.ascontiguousarray(ids[ids % 100 < pct])
        ctx = C.c_int(pct)
        py_fn = pkg.hnsw.FILTER_FN(lambda i, _c, pct=pct: 1 if i % 100 < pct else 0)
        row = {"filter": f"{pct}%"}
        rows = {}
        # ---- per call
        t_list = per_call_s(lambda: flat(1, p(allow), len(allow), none_cb, None))
        ref = [a.copy() for a in o0]
        t_c = per_call_s(lambda: flat(2, None, 0, admit, C.byref(ctx)))
        assert all(np.array_equal(a, b) for a, b in zip(o0, ref))
        t_py = per_call_s(lambda: flat(2, None, 0, py_fn, None), reps=REPS_PY, warm=1)
        rows.update(per_call_list=t_list, per_call_c_callback=t_c, per_call_py_callback=t_py)
        # ---- one-time filter_new
        new = {}
        for name, args in (("list", (1, p(allow), len(allow), none_cb, None)), ("c_callback", (2, None, 0, admit, C.byref(ctx))),
                           ("py_callback", (2, None, 0, py_fn, None))):
            t = time.perf_counter()
            fid = L.hnsw_b200_filter_new(h._h, *args)
            new[name] = time.perf_counter() - t
            assert fid >= 0, pkg.last_error()
            if name != "list":
                chk(L.hnsw_b200_filter_free(h._h, fid))
            else:
                rf = fid
        row["filter_new_ms"] = {k: round(v * 1e3, 2) for k, v in new.items()}
        # ---- resident: sync, submit/wait, device

        def res_flat(o=o0):
            chk(L.hnsw_b200_search_flat_filtered(h._h, rf, p(Q), NQ, D, K, EF, p(o[0]), p(o[1]), p(o[2]), None, p(o[3])))
        rows["resident_sync"] = per_call_s(res_flat)
        assert all(np.array_equal(a, b) for a, b in zip(o0, ref)), "resident answers differ from the per-call answers"
        for depth in (2, 3, 4):
            def pipelined(depth=depth, nb=4 * depth):
                tickets = []
                for b in range(nb):
                    o = outs[b % depth]
                    t = L.hnsw_b200_search_flat_submit_filtered(h._h, rf, p(Q), NQ, D, K, EF, p(o[0]), p(o[1]), p(o[2]), None,
                                                                p(o[3]))
                    assert t >= 0, pkg.last_error()
                    tickets.append(t)
                    if len(tickets) == depth:
                        chk(L.hnsw_b200_search_flat_wait(h._h, tickets.pop(0)))
                for t in tickets:
                    chk(L.hnsw_b200_search_flat_wait(h._h, t))
            rows[f"resident_submit_{depth}_in_flight"] = per_call_s(pipelined, reps=2, warm=1) / (4 * depth)
        ms = C.c_float()

        def dev_sync():
            chk(L.hnsw_b200_search_device_filtered(h._h, rf, C.c_void_p(qd.data_ptr()), NQ, K, EF, C.c_void_p(dout[0].data_ptr()),
                                                   C.c_void_p(dcnt[0].data_ptr()), 1, C.byref(ms)))
        rows["resident_device_sync"] = per_call_s(dev_sync)

        def dev_async_pair():
            for i in (0, 1):
                chk(L.hnsw_b200_search_device_filtered(h._h, rf, C.c_void_p(qd.data_ptr()), NQ, K, EF,
                                                       C.c_void_p(dout[i].data_ptr()), C.c_void_p(dcnt[i].data_ptr()), 0, None))
            chk(L.hnsw_b200_join(h._h))
            overflow.append(L.hnsw_b200_check_status(h._h))
        overflow = []
        rows["resident_device_async"] = per_call_s(dev_async_pair) / 2
        # an asynchronous launch does not grow its visited tables: 1 = some answers are empty and need a synchronous re-run
        row["device_async_overflow"] = max(overflow)
        if not row["device_async_overflow"]:
            got = dout[1].cpu().numpy()
            assert np.array_equal(got[..., 0:8].copy().view(np.uint64)[..., 0], ref[0])
        chk(L.hnsw_b200_filter_free(h._h, rf))
        row["kernel_ms_device_sync"] = round(ms.value, 3)
        row["qps"] = {k: round(NQ / v, 1) for k, v in rows.items()}
        row["call_ms"] = {k: round(v * 1e3, 3) for k, v in rows.items()}
        row["per_call_host_share"] = {k: round(max(0.0, 1 - rows["resident_sync"] / rows[k]), 3)
                                      for k in ("per_call_list", "per_call_c_callback", "per_call_py_callback")}
        print(json.dumps(row), flush=True)
    h.close()


if __name__ == "__main__":
    main()
