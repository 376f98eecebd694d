"""The batch schedule of the engine's insert (Index::insert_batch in csrc/index.cu), restated once for the tests that
compare a batched GPU build with the oracle's batch-synchronous one (pyoracle.Oracle.insert_batched).

One insert call cuts its points into batches:
  * the first point into an empty index goes alone (it becomes the entry point);
  * otherwise the next batch holds nb = min(max(linked // ratio, 1), max_batch, remaining) points, where linked is the
    number of points stored before the batch;
  * the batch is cut before a point whose level exceeds the current entry level, and such a point goes alone;
  * the entry level moves to that point's level after its batch.
A call's schedule starts from the handle's point count and entry level, so the state carries across calls.
"""
import numpy as np

RATIO, MAX_BATCH = 16, 16384   # the engine's defaults (Index::batch_ratio, batch_max)


def engine_batches(n_before, entry_level, levels, ratio=RATIO, max_batch=MAX_BATCH):
    """the batch sizes Index::insert_batch uses for one call inserting points of these levels into an index of n_before
    points whose entry point has level entry_level (ignored when n_before == 0)"""
    lv = np.asarray(levels).tolist()
    n, done, sizes = len(lv), 0, []
    empty = n_before == 0
    while done < n:
        if empty:
            sizes.append(1)
            entry_level, empty = lv[done], False
            done += 1
            continue
        nb = min(max((n_before + done) // ratio, 1), max_batch, n - done)
        for j in range(nb):
            if lv[done + j] > entry_level:
                nb = max(j, 1)
                if j == 0:
                    entry_level = lv[done]
                break
        sizes.append(nb)
        done += nb
    return sizes


def promoting_levels(po, n, seed, M=8):
    """drawn levels, capped so that the entry point is promoted at points 3, 40, 200 and 600 (the last by two layers),
    as in test_gpu_link_mode.py; points past n are dropped"""
    lv = po.Oracle(M, n, 16, 48, "DistL2", 4, seed=seed).draw_levels(n)
    i = np.arange(n)
    lv = np.minimum(lv, np.select([i < 3, i < 40, i < 200, i < 600], [0, 1, 2, 3], 5))
    for p, l in ((3, 1), (40, 2), (200, 3), (600, 5)):
        if p < n:
            lv[p] = l
    return lv.astype(np.int32)


def entry_level_after(n_before, entry_level, levels):
    """the entry level once a call with these levels is done (the state the next call's schedule starts from)"""
    top = -1 if n_before == 0 else entry_level
    return max([top] + np.asarray(levels).tolist())
