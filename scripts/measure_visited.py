"""Visited tables at the c2 shape (1 M x 128 f32 L2, M = 16, ef_c = 200, k = 10, ef = 64): per-launch kernel ms of the
lean search for 10 000 and 100 000 queries (search_device, best of 5 after a warm-up launch), the launch's dynamic shared
memory per CTA (with the first stage in shared memory when the launch is staged) and the CTAs per SM the runtime grants
it (cudaOccupancyMaxActiveBlocksPerMultiprocessor), and how many queries outgrow a first stage of cap / 8, cap / 4 and
cap / 2 entries (cap / 4 is the one the searches use).  A search moves when its layer-0 insertions (one per
layer-0 evaluation, the entry included) reach 3/4 of the first stage; the counters give evaluations per query including
the descent's (at most 1 + max_level * M), so the moved count is given as a range.  HNSW_B200_LIB selects a build."""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("hnswlib-rs_b200")

n, d, M, efc, k, ef = 1000000, 128, 16, 200, 10, 64
print(torch.cuda.get_device_name(0), flush=True)
h = pkg.Hnsw(M, n, 16, efc, "DistL2")
h.insert_flat(pkg.datagen.make("clustered", n, d, 1))
for nq in (10000, 100000):
    q = torch.from_numpy(pkg.datagen.make("clustered", nq, d, 2)).cuda()
    out = torch.empty((nq, k, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.empty((nq,), dtype=torch.int32, device="cuda")
    h.search_device(q.data_ptr(), nq, k, ef, out.data_ptr(), cnt.data_ptr(), sync=True)
    ms = [h.search_device(q.data_ptr(), nq, k, ef, out.data_ptr(), cnt.data_ptr(), sync=True) for _ in range(5)]
    print(f"{nq} queries per launch: kernel {min(ms):.3f} ms (best of 5), {nq / min(ms) / 1e3:.2f} M queries/s", flush=True)
    smem, threads, bps = pkg.last_kernel_shape()
    print(f"  {pkg.last_kernel()}: {smem} bytes of dynamic shared memory per {threads}-thread CTA, {bps} CTAs per SM",
          flush=True)

Q = pkg.datagen.make("clustered", 500, d, 3)
h.enable_stats(True)
h.get_stats()
ev = []
for i in range(len(Q)):
    h.search_flat(Q[i:i + 1], k, ef)
    ev.append(h.get_stats()["evals"])
h.enable_stats(False)
ev = np.array(ev)
descent = 1 + h.get_max_level_observed() * M
cap = 1 << max(10, (2 * (ef + 16) * 2 * M - 1).bit_length())
print(f"evaluations per query over {len(Q)}: mean {ev.mean():.0f}, p50 {np.percentile(ev, 50):.0f}, "
      f"p99 {np.percentile(ev, 99):.0f}, max {ev.max()}; descent <= {descent}; full stage {cap} entries")
for div in (8, 4, 2):
    at = (cap // div) * 3 // 4
    lo, hi = int((ev >= at + descent).sum()), int((ev >= at).sum())
    print(f"first stage cap/{div} = {cap // div}: moves at {at} insertions: {lo}..{hi} of {len(Q)} queries moved")
