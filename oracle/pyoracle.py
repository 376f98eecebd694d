"""ctypes wrapper around oracle/liboracle.so.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
PARITY UNPINNED (see hnsw_oracle.cpp header): the reference cannot be built here.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

METRICS = {"DistL1": 0, "DistL2": 1, "DistDot": 2, "DistCosine": 3, "DistHamming": 4, "DistJaccard": 5,
           "DistHellinger": 6, "DistJeffreys": 7, "DistJensenShannon": 8}
DTYPES = {np.dtype(np.float32): 0, np.dtype(np.uint8): 1, np.dtype(np.uint16): 2, np.dtype(np.uint32): 3,
          np.dtype(np.int32): 4}
MODE_STD, MODE_DET = 0, 1
ORDER_REF, ORDER_GPU = 0, 1

FILTER_FN = C.CFUNCTYPE(C.c_int, C.c_uint64, C.c_void_p)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("hnsw_oracle.cpp", "rheap.h", "distances.h", "Makefile")]
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs if os.path.exists(s))
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        vp, u64, i32, i64, f64 = C.c_void_p, C.c_uint64, C.c_int, C.c_int64, C.c_double
        L.oracle_new.restype = vp
        L.oracle_new.argtypes = [i32, i32, u64, i32, i32, i32, i32]
        L.oracle_free.argtypes = [vp]
        L.oracle_set_option.argtypes = [vp, i32, f64]
        L.oracle_size.restype = u64
        L.oracle_size.argtypes = [vp]
        L.oracle_entry.restype = i64
        L.oracle_entry.argtypes = [vp]
        L.oracle_insert_batch.argtypes = [vp, vp, vp, vp, u64, i32]
        L.oracle_insert_batched.argtypes = [vp, vp, vp, vp, u64, vp, u64, i32, i32, u64]
        L.oracle_draw_levels.argtypes = [vp, vp, u64]
        L.oracle_search_batch.argtypes = [vp, vp, u64, u64, u64, i32, vp, u64, FILTER_FN, vp, i32, vp, vp, vp, vp, vp]
        L.oracle_counters.argtypes = [vp, vp, i32]
        L.oracle_export_points.argtypes = [vp, vp, vp, vp]
        L.oracle_layer_edges.restype = u64
        L.oracle_layer_edges.argtypes = [vp, i32]
        L.oracle_export_layer.argtypes = [vp, i32, vp, vp, vp]
        L.oracle_export_vectors.argtypes = [vp, vp]
        L.oracle_import_points.argtypes = [vp, vp, vp, vp, u64, i64]
        L.oracle_import_layer.argtypes = [vp, i32, vp, vp, vp, u64]
        L.oracle_dist.restype = C.c_float
        L.oracle_dist.argtypes = [i32, i32, i32, vp, vp, u64]
        L.oracle_logf.argtypes = [i32, vp, vp, u64]
        L.oracle_bruteforce.argtypes = [i32, i32, i32, vp, u64, vp, u64, u64, u64, i32, vp, vp]
        L.oracle_numa_interleave.restype = i32
        L.oracle_numa_interleave.argtypes = [i32]
        L.oracle_rheap_script.restype = u64
        L.oracle_rheap_script.argtypes = [vp, vp, u64, i32, i32, vp]
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def numa_interleave(on=True):
    """interleave this thread's future allocations over all NUMA nodes (CPU-baseline fairness); 0 ok, -1 refused"""
    return int(lib().oracle_numa_interleave(int(bool(on))))


def dist(a, b, metric, order=ORDER_REF):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b, dtype=a.dtype)
    return float(lib().oracle_dist(DTYPES[a.dtype], METRICS[metric], order, _p(a), _p(b), a.size))


def logf(x, order=ORDER_REF):
    """float32 natural logarithm of every element of x as `order` computes it: the device's logf (ORDER_GPU) or the C
    library's (ORDER_REF)"""
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    lib().oracle_logf(int(order), _p(x), _p(out), x.size)
    return out


def bruteforce(base, queries, k, metric, order=ORDER_REF, nthreads=None):
    base = np.ascontiguousarray(base)
    queries = np.ascontiguousarray(queries, dtype=base.dtype)
    nq, d = queries.shape
    ids = np.empty((nq, k), np.uint32)
    ds = np.empty((nq, k), np.float32)
    lib().oracle_bruteforce(DTYPES[base.dtype], METRICS[metric], order, _p(base), base.shape[0], _p(queries), nq, d, k,
                            nthreads or os.cpu_count(), _p(ids), _p(ds))
    return ids, ds


def rheap_script(ops, vals, mode=MODE_STD, neg=False):
    ops = np.ascontiguousarray(ops, np.int64)
    vals = np.ascontiguousarray(vals, np.float32)
    out = np.empty(2 * len(ops) + 4, np.int64)
    n = lib().oracle_rheap_script(_p(ops), _p(vals), len(ops), mode, int(neg), _p(out))
    return out[:n]


class Oracle:
    """CPU restatement of Hnsw<T,D> (reference src/hnsw.rs:739-1635)."""

    def __init__(self, max_nb_connection, max_elements, max_layer, ef_construction, metric, dim, dtype=np.float32,
                 mode=MODE_STD, order=ORDER_REF, seed=None):
        self.L = lib()
        self.dtype = np.dtype(dtype)
        self.dim = int(dim)
        self.metric = metric
        self.M = int(max_nb_connection)
        self.h = self.L.oracle_new(DTYPES[self.dtype], self.M, int(max_elements), int(max_layer), int(ef_construction),
                                   METRICS[metric], self.dim)
        if not self.h:
            raise ValueError("oracle_new failed")
        self.set_mode(mode)
        self.set_order(order)
        if seed is not None:
            self.L.oracle_set_option(self.h, 5, float(seed))

    def __del__(self):
        try:
            if self.h:
                self.L.oracle_free(self.h)
                self.h = None
        except Exception:
            pass

    def set_mode(self, m):
        self.L.oracle_set_option(self.h, 0, float(m))

    def set_order(self, o):
        self.L.oracle_set_option(self.h, 1, float(o))

    def set_extend_candidates(self, f):
        self.L.oracle_set_option(self.h, 2, float(bool(f)))

    def set_keeping_pruned(self, f):
        self.L.oracle_set_option(self.h, 3, float(bool(f)))

    def modify_level_scale(self, s):
        self.L.oracle_set_option(self.h, 4, float(s))

    def __len__(self):
        return int(self.L.oracle_size(self.h))

    @property
    def entry(self):
        return int(self.L.oracle_entry(self.h))

    def draw_levels(self, n):
        out = np.empty(n, np.int32)
        self.L.oracle_draw_levels(self.h, _p(out), n)
        return out

    def insert_batch(self, vecs, ids=None, levels=None, nthreads=1):
        vecs = np.ascontiguousarray(vecs, dtype=self.dtype).reshape(-1, self.dim)
        n = vecs.shape[0]
        if ids is None:
            ids = np.arange(len(self), len(self) + n)
        ids = np.ascontiguousarray(ids, np.uint64)
        lv = None if levels is None else np.ascontiguousarray(levels, np.int32)
        self.L.oracle_insert_batch(self.h, _p(vecs), _p(ids), _p(lv), n, int(nthreads))

    def insert_batched(self, vecs, ids=None, levels=None, *, batches, nthreads=1, link_mode=0, order_seed=0):
        """The engine's batch-synchronous insert (hnsw_oracle.cpp Index::insert_batched): `batches` are the sizes of
        consecutive batches covering all of vecs (tests/batched.py engine_batches gives the engine's own).  The graph and
        the counters do not depend on nthreads or order_seed."""
        vecs = np.ascontiguousarray(vecs, dtype=self.dtype).reshape(-1, self.dim)
        n = vecs.shape[0]
        if ids is None:
            ids = np.arange(len(self), len(self) + n)
        ids = np.ascontiguousarray(ids, np.uint64)
        lv = self.draw_levels(n) if levels is None else np.ascontiguousarray(levels, np.int32)
        sizes = np.ascontiguousarray(batches, np.uint64)
        if len(ids) != n or len(lv) != n or int(sizes.sum()) != n or (len(sizes) and int(sizes.min()) == 0):
            raise ValueError("insert_batched: ids, levels and the batch sizes must cover the points exactly")
        self.L.oracle_insert_batched(self.h, _p(vecs), _p(ids), _p(lv), n, _p(sizes), len(sizes), int(nthreads),
                                     int(link_mode), int(order_seed))

    def search_batch(self, queries, k, ef, filter_ids=None, filter_fn=None, nthreads=1):
        """Returns (origin_ids[nq,k] u64, dists[nq,k] f32, internal[nq,k] u32, pid[nq,k,2] i32, counts[nq])."""
        q = np.ascontiguousarray(queries, dtype=self.dtype).reshape(-1, self.dim)
        nq = q.shape[0]
        o = np.empty((nq, k), np.uint64)
        d = np.empty((nq, k), np.float32)
        it = np.empty((nq, k), np.uint32)
        pid = np.empty((nq, k, 2), np.int32)
        cnt = np.empty(nq, np.int32)
        use = 0
        fids = None
        nf = 0
        cb = FILTER_FN(0)
        if filter_ids is not None:
            fids = np.ascontiguousarray(np.sort(np.asarray(filter_ids, np.uint64)))
            nf = len(fids)
            use = 1
        if filter_fn is not None:
            cb = FILTER_FN(lambda i, _ctx: 1 if filter_fn(int(i)) else 0)
            use = 1
        self.L.oracle_search_batch(self.h, _p(q), nq, k, ef, use, _p(fids), nf, cb, None, int(nthreads), _p(o), _p(d),
                                   _p(it), _p(pid), _p(cnt))
        return o, d, it, pid, cnt

    def counters(self, reset=True):
        out = np.zeros(4, np.uint64)
        self.L.oracle_counters(self.h, _p(out), int(reset))
        return {"evals": int(out[0]), "expansions": int(out[1]), "adj_read": int(out[2]), "queries": int(out[3])}

    def export_points(self):
        n = len(self)
        lv = np.empty(n, np.uint8)
        rk = np.empty(n, np.int32)
        og = np.empty(n, np.uint64)
        self.L.oracle_export_points(self.h, _p(lv), _p(rk), _p(og))
        return lv, rk, og

    def export_layer(self, layer, with_dists=True):
        n = len(self)
        ne = int(self.L.oracle_layer_edges(self.h, layer))
        off = np.empty(n + 1, np.uint64)
        ids = np.empty(ne, np.uint32)
        ds = np.empty(ne, np.float32) if with_dists else None
        self.L.oracle_export_layer(self.h, layer, _p(off), _p(ids), _p(ds))
        return off, ids, ds

    def export_vectors(self):
        out = np.empty((len(self), self.dim), self.dtype)
        self.L.oracle_export_vectors(self.h, _p(out))
        return out

    def import_graph(self, vecs, origin, levels, entry, layers):
        """layers: dict layer -> (offsets u64[N+1], ids u32, dists f32|None)."""
        vecs = np.ascontiguousarray(vecs, dtype=self.dtype).reshape(-1, self.dim)
        n = vecs.shape[0]
        origin = np.ascontiguousarray(origin, np.uint64)
        levels = np.ascontiguousarray(levels, np.uint8)
        self.L.oracle_import_points(self.h, _p(vecs), _p(origin), _p(levels), n, int(entry))
        for l, (off, ids, ds) in layers.items():
            off = np.ascontiguousarray(off, np.uint64)
            ids = np.ascontiguousarray(ids, np.uint32)
            ds = None if ds is None else np.ascontiguousarray(ds, np.float32)
            self.L.oracle_import_layer(self.h, int(l), _p(off), _p(ids), _p(ds), n)
