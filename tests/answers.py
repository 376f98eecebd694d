"""Comparing search answers: the (origin ids, distances, internal ids, PointIds, counts) tuples the host calls return,
the Neighbour_api rows the device calls write, and the per-group reference of a batch whose rows carry their own
restriction.

pytest shows the compared values only for asserts in test modules, so every assert here says in its message what it
compared."""
import numpy as np


def same(got, want, what):
    go, gd, gi, gpid, gc = got
    oo, od, oi, opid, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ"
    assert np.array_equal(gi, oi), f"{what}: internal ids differ"
    assert np.array_equal(go, oo), f"{what}: origin ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distances are not bit-identical"
    assert np.array_equal(gpid, opid), f"{what}: PointIds differ"


def device_answers(raw, cnt):
    """Neighbour_api[nq][k] (origin u64, dist f32, internal id in the tail padding) + counts, as search_flat's arrays"""
    a = raw.cpu().numpy()
    o = a[..., 0:8].copy().view(np.uint64)[..., 0]
    d = a[..., 8:12].copy().view(np.float32)[..., 0]
    it = a[..., 12:16].copy().view(np.uint32)[..., 0]
    return o, d, it, cnt.cpu().numpy()


def same_host_device(host, dev, what):
    o, d, it, c = dev
    assert np.array_equal(c, host[4]), f"{what}: counts differ"
    assert np.array_equal(it, host[2]), f"{what}: internal ids differ"
    assert np.array_equal(o, host[0]), f"{what}: origin ids differ"
    assert np.array_equal(d.view(np.uint32), host[1].view(np.uint32)), f"{what}: distances are not bit-identical"


def rows_of(sel, g):
    return np.flatnonzero(sel == g)


def per_group(call, Q, sel, rfs):
    """the single-filter call on each group's rows, assembled in the batch's row order; sel[i] = -1 or an index of rfs"""
    out = None
    for g in np.unique(sel):
        rows = rows_of(sel, g)
        res = call(Q[rows], None if g < 0 else rfs[g])
        if out is None:
            out = tuple(None if x is None else np.empty((len(Q),) + x.shape[1:], x.dtype) for x in res)
        for o, x in zip(out, res):
            if o is not None:
                o[rows] = x
    return out


def stats_sum(dicts):
    return {key: sum(d[key] for d in dicts) for key in dicts[0]}


def same_as_single_filter_calls(h, Q, sel, rfs, flat, exact=None):
    """Each row of the restricted batch call equals the single-filter call on its group (per_group), in tie modes 0 and 1
    at (k, ef) = (1, 1), (10, 64), (40, 257); with statistics on, the batch call's counters equal the sum over the
    groups' calls.  flat(k, ef) and exact(k) make the batch's graph and exact calls; without exact the exact rows are
    not compared.  Tie mode 1 is left set."""
    for tie in (0, 1):
        h.set_tie_mode(tie)
        for k, ef in ((1, 1), (10, 64), (40, 257)):
            what = f"tie={tie} k={k} ef={ef}"
            single = lambda q, rf: h.search_flat(q, k, ef, filter=rf)   # noqa: E731
            want = per_group(single, Q, sel, rfs)
            same(flat(k, ef), want, what)
            # statistics: every run above grew the contexts' tables, so none of these overflows and re-runs
            h.enable_stats(True)
            h.get_stats()
            got = flat(k, ef)
            s_batch = h.get_stats()
            parts = []
            for g in np.unique(sel):
                single(Q[rows_of(sel, g)], None if g < 0 else rfs[g])
                parts.append(h.get_stats())
            h.enable_stats(False)
            same(got, want, what + " stats on")
            assert s_batch == stats_sum(parts), (what, s_batch, parts)
        if exact is not None:
            for k in (1, 10):
                same(exact(k), per_group(lambda q, rf: h.search_exact(q, k, filter=rf), Q, sel, rfs),
                     f"tie={tie} exact k={k}")
