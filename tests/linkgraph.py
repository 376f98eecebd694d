"""Helpers of the link-mode tests: the oracle's serial build in link mode 1, and graph facts computed from exported CSR
layers.

The oracle restates the reference, whose reverse links go to the new point's level (hnsw.rs:1257).  insert_link_mode1
drives it one point at a time and rewrites what link mode 1 does differently, through the oracle's own export / import
of layers:
  * phase B: for a point x of level L >= 1, the lists of layers 0..L are rebuilt from their state before the insert
    plus x's own lists (phase A, which both modes share), and every own link (q, d) of layer l adds (x, d) to q's layer-l
    list with the reference's duplicate check, (distance, id) order (MODE_DET), 2M / M capacity and truncation of the
    farthest (hnsw.rs:1258-1284).  For L = 0 both rules file every link in layer 0, so the oracle's own phase B stands.
  * the ef = 1 descent's push into x's own lists above its level (hnsw.rs:1140-1144) is removed.
"""
import ctypes as C

import numpy as np


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _replace_rows(layer, n, rows):
    """the CSR `layer` (offsets, ids, dists) grown to n rows, with rows[p] = [(id, dist), ...] replacing row p"""
    off, ids, ds = np.asarray(layer[0], np.int64), layer[1], layer[2]
    counts = np.zeros(n, np.int64)
    counts[:len(off) - 1] = np.diff(off)
    changed = np.zeros(n, bool)
    for p, r in rows.items():
        counts[p] = len(r)
        changed[p] = True
    new_off = np.zeros(n + 1, np.int64)
    np.cumsum(counts, out=new_off[1:])
    rid = np.repeat(np.arange(len(off) - 1), np.diff(off))
    keep = ~changed[rid]
    pos = new_off[rid[keep]] + (np.arange(len(ids))[keep] - off[rid[keep]])
    new_ids = np.empty(int(new_off[-1]), np.uint32)
    new_ds = np.empty(int(new_off[-1]), np.float32)
    new_ids[pos], new_ds[pos] = ids[keep], ds[keep]
    for p, r in rows.items():
        b = int(new_off[p])
        new_ids[b:b + len(r)] = [e[0] for e in r]
        new_ds[b:b + len(r)] = [e[1] for e in r]
    return new_off.astype(np.uint64), new_ids, new_ds


def _import_layer(o, layer, csr, n):
    off, ids, ds = csr
    o.L.oracle_import_layer(o.h, int(layer), _ptr(off), _ptr(ids), _ptr(ds), int(n))


def _row(layer, p):
    off = layer[0]
    b, e = int(off[p]), int(off[p + 1])
    return list(zip(layer[1][b:e].tolist(), layer[2][b:e].tolist()))


def insert_link_mode1(o, vecs, levels, ids=None):
    """insert vecs one at a time into the MODE_DET oracle `o` as link mode 1 does (see the module docstring)"""
    vecs = np.ascontiguousarray(vecs, o.dtype).reshape(-1, o.dim)
    if ids is None:
        ids = np.arange(len(o), len(o) + len(vecs))
    ids = np.asarray(ids, np.uint64)
    top = int(o.export_points()[0][o.entry]) if o.entry >= 0 else -1
    for i in range(len(vecs)):
        L, x = int(levels[i]), len(o)
        before = {l: o.export_layer(l) for l in range(L + 1)} if L >= 1 else {}
        o.insert_batch(vecs[i:i + 1], ids=ids[i:i + 1], levels=[L])
        n = x + 1
        for l in range(L + 1, top + 1):   # the descent's push above x's level (hnsw.rs:1140-1144)
            after = o.export_layer(l)
            if after[0][x + 1] > after[0][x]:
                _import_layer(o, l, _replace_rows(after, n, {x: []}), n)
        for l in range(L + 1) if L >= 1 else ():   # phase B per layer (link mode 1)
            own = _row(o.export_layer(l), x)
            cap = 2 * o.M if l == 0 else o.M
            rows = {x: own}
            for q, d in own:
                if q == x:
                    continue
                row = rows[q] if q in rows else _row(before[l], q)
                if any(e[0] == x for e in row):
                    continue
                row.append((x, d))
                row.sort(key=lambda e: (e[1], e[0]))
                if len(row) > cap:
                    row.pop()
                rows[q] = row
            _import_layer(o, l, _replace_rows(before[l], n, rows), n)
        top = max(top, L)


def entry_history(levels):
    """the points that were the entry point at some time during a serial build with these levels, in insertion order
    (the first point, then every point whose level exceeds the entry's, hnsw.rs:534-557)"""
    out, top = [], -1
    for p, lv in enumerate(np.asarray(levels).tolist()):
        if lv > top:
            out.append(p)
            top = lv
    return out


def without_layer0_inlink(layer0, levels, entry):
    """ids of the points of level >= 1, the entry point excepted, that no layer-0 list names"""
    off, ids = layer0[0], layer0[1]
    n = len(off) - 1
    linked = np.zeros(n, bool)
    linked[np.asarray(ids, np.int64)] = True
    levels = np.asarray(levels)
    return [p for p in range(n) if levels[p] >= 1 and p != entry and not linked[p]]


def lists_above_level(layers, levels):
    """(layer, point) of every non-empty list above its point's level; layers[l] = (offsets, ids, dists)"""
    levels = np.asarray(levels)
    out = []
    for l in range(1, len(layers)):
        off = np.asarray(layers[l][0], np.int64)
        sizes = off[1:] - off[:-1]
        out += [(l, int(p)) for p in np.nonzero((sizes > 0) & (levels < l))[0]]
    return out
