"""A Python restatement of the oracle's deterministic search (oracle/hnsw_oracle.cpp search / search_layer, MODE_DET,
distances by pyoracle.dist in ORDER_GPU) on a graph exported from an oracle, with one more rule: the live stop of a
search over the live points of an index with deleted points (include/hnsw_b200.h "Deleted points").  A filtered search
that finds its nearest candidate farther than W's farthest point drops W's non-admitted points and expands on; a live
search returns W there, as an unfiltered search does.  Everything else is the filtered search's.

Test infrastructure only.  test_liveref_cpu.py checks that the filtered and unfiltered rules here give the oracle's
rows and counters bit for bit, and that the live rule with every point live gives the oracle's unfiltered rows and
counters on continuous data (where no two distances tie at the stop test)."""
import bisect
import heapq

import numpy as np


class LiveRef:
    def __init__(self, po, o, X, metric):
        self.po, self.X, self.metric = po, X, metric
        lv, rk, og = o.export_points()
        self.level, self.rank, self.origin = lv.astype(np.int64), rk, og
        self.entry = o.entry
        self.adj = []
        for layer in range(int(lv.max()) + 1):
            off, ids, _ = o.export_layer(layer, with_dists=False)
            self.adj.append((off.astype(np.int64), ids.astype(np.int64)))
        counts = np.bincount(lv, minlength=16)
        self.layer0 = int(np.nonzero(counts)[0][0])

    def _nbrs(self, p, layer):
        off, ids = self.adj[layer]
        return ids[off[p]:off[p + 1]]

    def search(self, q, k, ef, admit=None, live=False):
        """one query: (rows [(origin, dist f32, internal)], counters {evals, expansions, adj_read}).  admit: bool per
        internal id (None: unfiltered); live: the live stop rule (with admit)."""
        po, X, metric = self.po, self.X, self.metric
        c = {"evals": 0, "expansions": 0, "adj_read": 0}

        def dist(i):
            c["evals"] += 1
            return float(np.float32(po.dist(q, X[i], metric, po.ORDER_GPU)))

        ep = self.entry
        best = dist(ep)
        pivot = ep
        for layer in range(int(self.level[ep]), 0, -1):
            nbs = self._nbrs(pivot, layer)
            c["adj_read"] += len(nbs)
            new = pivot
            for n in nbs:
                t = dist(n)
                if t < best:
                    new, best = int(n), t
            pivot = new
        ef = max(ef, k)
        W = self._layer(q, pivot, ef, admit, live, dist, c)
        out = []
        for d, i in W[:min(k, ef, len(W))]:
            if admit is None or admit[i]:
                out.append((int(self.origin[i]), d, i))
        return out, c

    def _layer(self, q, ep, ef, admit, live, dist, c):
        layer = self.layer0
        filt = admit is not None
        d0 = dist(ep)
        visited = {ep}
        C = [(d0, ep)]           # nearest first, ties by smaller id
        W = [(d0, ep)]           # ascending (distance, id): W[-1] is the farthest
        while C:
            cd, ci = heapq.heappop(C)
            if not W:
                return W
            fd, fi = W[-1]
            stop = cd > fd if filt else (cd, ci) > (fd, fi)
            if stop:
                if not filt or live:
                    return W
                if len(W) >= ef:
                    W = [w for w in W if admit[w[1]]]
            nbs = self._nbrs(ci, layer)
            c["expansions"] += 1
            c["adj_read"] += len(nbs)
            for e in nbs:
                e = int(e)
                if e in visited:
                    continue
                visited.add(e)
                if not W:
                    return W
                f2 = W[-1]
                de = dist(e)
                if (de, e) < f2 or len(W) < ef:
                    heapq.heappush(C, (de, e))
                    if not filt:
                        bisect.insort(W, (de, e))
                    elif admit[e]:
                        if len(W) == 1 and not admit[W[0][1]]:
                            W = []
                        bisect.insort(W, (de, e))
                    if len(W) > ef:
                        W.pop()
        return W

    def batch(self, Q, k, ef, admit=None, live=False):
        """search_flat's (origin u64, dist f32, internal u32, pid i32 [.,.,2], counts) and the summed counters"""
        nq = len(Q)
        o = np.full((nq, k), ~np.uint64(0), np.uint64)
        d = np.full((nq, k), np.inf, np.float32)
        it = np.full((nq, k), 0xFFFFFFFF, np.uint32)
        pid = np.full((nq, k, 2), -1, np.int32)
        cnt = np.zeros(nq, np.int32)
        tot = {"evals": 0, "expansions": 0, "adj_read": 0}
        for r in range(nq):
            rows, c = self.search(Q[r], k, ef, admit, live)
            for key in tot:
                tot[key] += c[key]
            cnt[r] = len(rows)
            for j, (og, dd, i) in enumerate(rows):
                o[r, j], d[r, j], it[r, j] = og, dd, i
                pid[r, j] = (self.level[i], self.rank[i])
        return (o, d, it, pid, cnt), tot
