"""The oracle's distance functions (oracle/distances.h, both summation orders) against a float64 statement of each of the
nine definitions, on edge inputs and on dimensions that leave partial 16-byte chunks (tests/distref.py states the formulas
and the error bound).  Every GPU kernel is compared bit for bit with the oracle's ORDER_GPU sums, so this pins the kernels
to the formulas too; tests/test_gpu_matrix.py checks the device's dist_batch against the same bound directly."""
import numpy as np
import pytest

import distref

DTYPES = [np.float32, np.uint8, np.uint16, np.uint32, np.int32]
CASES = [(dt, m) for dt in DTYPES for m in distref.F32_METRICS + ["DistHamming", "DistJaccard"] if distref.supported(dt, m)]


@pytest.mark.parametrize("dtype,metric", CASES, ids=[f"{np.dtype(d).name}-{m}" for d, m in CASES])
def test_oracle_distance_matches_float64_formula(po, dtype, metric):
    checked = 0
    for d in distref.DIMS:
        for name, a, b in distref.edge_pairs(dtype, metric, d):
            for order in (po.ORDER_REF, po.ORDER_GPU):
                for x, y in ((a, b), (b, a)):
                    got = po.dist(x, y, metric, order)
                    ok, msg = distref.within(got, metric, x, y)
                    assert ok, f"{name}, order {order}: {msg}"
                    if (metric, name) in distref.EXACT_ZERO:
                        assert got == 0.0, f"{name}, order {order}: {metric} must be exactly 0, got {got!r}"
                    checked += 1
    assert checked >= 4 * len(distref.DIMS) * 5


def test_bound_is_tight_enough_to_catch_a_wrong_term():
    """the bound must reject an implementation that drops or duplicates one element"""
    rng = np.random.default_rng(1)
    for metric in ("DistL1", "DistL2", "DistDot", "DistHellinger", "DistJeffreys", "DistJensenShannon"):
        for d in (17, 129):
            a, b = distref.edge_pairs(np.float32, metric, d)[0][1:]
            v = distref.reference(a, b, metric)[0]
            wrong = distref.reference(a[:-1].copy(), b[:-1].copy(), metric)[0]
            if abs(wrong - v) < 1e-6:
                continue
            assert not distref.within(np.float32(wrong), metric, a, b)[0], (metric, d)
    u = rng.integers(0, 4, 33).astype(np.uint16)
    v = rng.integers(0, 4, 33).astype(np.uint16)
    h = distref.reference(u, v, "DistHamming")[0]
    assert not distref.within(np.float32(h * 33 / 40), "DistHamming", u, v)[0]   # count / (d4 * 8) instead of / d
