"""attr_of_float (hnsw.py): the order-preserving map from float64 to int64 attributes, checked without a GPU."""
import numpy as np
import pytest


def test_monotone_and_never_none(pkg):
    tiny = np.finfo(np.float64).smallest_subnormal
    big = np.finfo(np.float64).max
    xs = np.array([-np.inf, -big, -1e300, -2.5, -1.0, -np.finfo(np.float64).tiny, -2 * tiny, -tiny, -0.0, 0.0, tiny, 2 * tiny,
                   np.finfo(np.float64).tiny, 1.0, 2.5, 1e300, big, np.inf])
    rng = np.random.default_rng(0)
    xs = np.sort(np.concatenate([xs, rng.standard_normal(2000) * 10.0 ** rng.integers(-300, 300, 2000)]))
    a = pkg.attr_of_float(xs)
    assert a.dtype == np.int64 and a.shape == xs.shape
    assert np.all(np.diff(a) >= 0)
    assert np.all((np.diff(a) > 0) == (np.diff(xs) > 0))   # equal only for equal floats (-0.0 and +0.0 among them)
    assert not np.any(a == pkg.ATTR_NONE)
    assert pkg.attr_of_float(-0.0) == pkg.attr_of_float(0.0) == 0
    assert pkg.attr_of_float(1.0) == int(np.float64(1.0).view(np.int64))
    assert pkg.attr_of_float(-1.0) < pkg.attr_of_float(-tiny) < 0 < pkg.attr_of_float(tiny)
    assert pkg.attr_of_float(-np.inf) > pkg.ATTR_NONE


@pytest.mark.parametrize("x", [np.nan, [1.0, np.nan], -np.nan])
def test_nan_is_refused(pkg, x):
    with pytest.raises(ValueError, match="NaN"):
        pkg.attr_of_float(x)
