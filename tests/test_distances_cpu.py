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


def test_device_logf_restatement_within_one_ulp(po):
    """ORDER_GPU's logf (oracle/distances.h device_logf, the sequence nvcc emits for the device's logf) against the
    float64 log: every float of [0.5, 2), every 64th subnormal and every 61st positive finite float, each within 1 ulp of
    the result; the special values exactly; and on some input it rounds differently from the C library's logf, which
    ORDER_REF keeps"""
    bits = np.concatenate([np.arange(0x3F000000, 0x40000000, dtype=np.uint32),   # [0.5, 1) and [1, 2)
                           np.arange(1, 0x00800000, 64, dtype=np.uint32),          # subnormals
                           np.arange(1, 0x7F800000, 61, dtype=np.uint32)])         # every 61st positive finite float
    differs_from_libm = 0
    for part in np.array_split(bits, 16):
        x = part.view(np.float32)
        got = po.logf(x, po.ORDER_GPU)
        exact = np.log(x.astype(np.float64))
        ulp = np.ldexp(1.0, np.frexp(exact)[1] - 24)   # ulp of a float32 with the exponent of the exact result
        err = np.abs(got.astype(np.float64) - exact) / ulp
        nonzero = exact != 0
        worst = int(np.argmax(np.where(nonzero, err, 0)))
        assert err[nonzero].max() <= 1.0, \
            f"logf(0x{part[worst]:08X}) = {got[worst]!r}, float64 log {exact[worst]!r}: {err[worst]:.3f} ulp"
        assert np.all(got[~nonzero] == 0), "logf(1) must be exactly 0"
        differs_from_libm += int(np.count_nonzero(got.view(np.uint32) != po.logf(x, po.ORDER_REF).view(np.uint32)))
    assert differs_from_libm > 0, "ORDER_GPU's logf rounds every swept input as the C library does"
    sp = np.array([1.0, 0.0, -0.0, np.inf, -1.0, -np.inf, -1e-40, np.nan], np.float32)
    got = po.logf(sp, po.ORDER_GPU)
    assert got[0] == 0 and not np.signbit(got[0]), f"logf(1) = {got[0]!r}"
    assert got[1] == -np.inf and got[2] == -np.inf, f"logf(+-0) = {got[1:3]}"
    assert got[3] == np.inf, f"logf(inf) = {got[3]!r}"
    assert np.all(np.isnan(got[4:])), f"logf of negative inputs and NaN = {got[4:]}"
