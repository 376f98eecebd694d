"""Float64 statement of the nine distance definitions, the edge inputs that test them, and the forward-error bound an f32
implementation must meet (shared by tests/test_distances_cpu.py and the GPU twin in tests/test_gpu_matrix.py).

The formulas (the anndists semantics the engine and the oracle implement):
  L1 = sum |a-b|          L2 = sqrt(sum (a-b)^2)              Dot = max(0, 1 - sum a*b)
  Cosine = max(0, 1 - ab / sqrt(aa*bb)), 0 when a norm is 0   Hamming = #{a_i != b_i} / d
  Jaccard = 1 - sum min / sum max, 0 when sum max is 0        Hellinger = sqrt(max(0, 1 - sum sqrt(a*b)))
  Jeffreys = sum (a-b) ln(max(a,1e-30) / max(b,1e-30))        JensenShannon = sqrt(0.5 sum [a ln(a/m) + b ln(b/m)]), m = (a+b)/2
Integer elements are cast to f32 for L1 / L2 (exactly for u8 / u16, rounded for u32 / i32 beyond 2^24).

Bound: with u = 2^-24 and d elements, an f32 sum of d terms computed in any order (fused or not) is within
(d+4) * u * T of the exact sum, T = sum |terms| (Higham, Accuracy and Stability of Numerical Algorithms, §4.2; the +4 covers
the rounding of each term, of the input casts and of the final 1 - s).  Metrics that end in a square root are compared
squared; logarithms contribute an absolute error of about u per term, which the T of Jeffreys and Jensen-Shannon carries.
Cosine accumulates in f64 and rounds once to f32.  Hamming and Jaccard have integer sums: exact.
"""
import numpy as np

U = 2.0 ** -24
EPS_CLAMP = float(np.float32(1e-30))   # Jeffreys' clamp, as the f32 constant it is

F32_METRICS = ["DistL1", "DistL2", "DistDot", "DistCosine", "DistHellinger", "DistJeffreys", "DistJensenShannon"]
INT_METRICS = ["DistL1", "DistL2", "DistHamming", "DistJaccard"]
DIMS = [1, 3, 15, 17, 33, 129, 257]


def supported(dtype, metric):
    if np.dtype(dtype) == np.float32:
        return metric in F32_METRICS
    return metric in INT_METRICS and not (np.dtype(dtype) == np.int32 and metric == "DistJaccard")


def as_f32_exact(dtype):
    """integer values this type holds are all exactly representable in f32"""
    return np.dtype(dtype) in (np.dtype(np.float32), np.dtype(np.uint8), np.dtype(np.uint16))


def reference(a, b, metric):
    """(value, bound, compare_squared): float64 value of the formula and the permitted |got - value| (or |got^2 - value^2|
    when compare_squared)."""
    dt = a.dtype
    x, y = a.astype(np.float64), b.astype(np.float64)
    d = len(x)
    g = (d + 4) * U
    inexact_in = not as_f32_exact(dt)
    if metric == "DistL1":
        t = (np.abs(x) + np.abs(y)) if inexact_in else np.abs(x - y)
        return np.abs(x - y).sum(), g * t.sum(), False
    if metric == "DistL2":
        t = (np.abs(x) + np.abs(y)) ** 2 if inexact_in else (x - y) ** 2
        s = ((x - y) ** 2).sum()
        return np.sqrt(s), (g + 3 * U) * t.sum(), True
    if metric == "DistDot":
        s = (x * y).sum()
        return max(0.0, 1.0 - s), g * (np.abs(x * y).sum() + 1.0), False
    if metric == "DistCosine":
        ab, aa, bb = x @ y, x @ x, y @ y
        v = max(0.0, 1.0 - ab / np.sqrt(aa * bb)) if aa > 0 and bb > 0 else 0.0
        return v, U * v + (d + 8) * 2.0 ** -50, False
    if metric == "DistHamming":
        c = np.float32(np.count_nonzero(a != b))
        return float(c / np.float32(d)), 0.0, False
    if metric == "DistJaccard":
        mn = int(np.minimum(a.astype(np.int64), b.astype(np.int64)).sum())
        mx = int(np.maximum(a.astype(np.int64), b.astype(np.int64)).sum())
        return (0.0 if mx == 0 else float(np.float32(1.0 - mn / mx))), 0.0, False
    if metric == "DistHellinger":
        t = np.sqrt(x * y)
        return np.sqrt(max(0.0, 1.0 - t.sum())), (g + 3 * U) * (t.sum() + 1.0), True
    if metric == "DistJeffreys":
        lr = np.log(np.maximum(x, EPS_CLAMP) / np.maximum(y, EPS_CLAMP))
        return ((x - y) * lr).sum(), g * (np.abs(x - y) * (1.0 + np.abs(lr))).sum(), False
    if metric == "DistJensenShannon":
        m = 0.5 * (x + y)
        with np.errstate(divide="ignore", invalid="ignore"):
            la = np.where(x > 0, np.log(np.where(x > 0, x, 1.0) / np.where(m > 0, m, 1.0)), 0.0)
            lb = np.where(y > 0, np.log(np.where(y > 0, y, 1.0) / np.where(m > 0, m, 1.0)), 0.0)
        s = (x * la + y * lb).sum()
        t = ((x + y) * (1.0 + np.abs(la) + np.abs(lb))).sum()
        return np.sqrt(max(0.0, 0.5 * s)), (g + 3 * U) * t, True
    raise ValueError(metric)


def within(got, metric, a, b):
    """(ok, message) for one computed distance"""
    v, bound, sq = reference(a, b, metric)
    err = abs(float(got) ** 2 - v * v) if sq else abs(float(got) - v)
    return err <= bound, f"{metric} {a.dtype} d={len(a)}: got {float(got)!r} want {v!r} err {err:.3g} > bound {bound:.3g}"


def _prob(rng, d, zeros):
    p = rng.random(d)
    if zeros:
        p[rng.random(d) < 0.4] = 0.0
        if not p.any():
            p[0] = 1.0
    return (p / p.sum()).astype(np.float32)


def edge_pairs(dtype, metric, d, seed=0):
    """[(name, a, b)]: random pairs plus the edge inputs where an implementation goes wrong.  `exact_zero` pairs carry a
    distance that must come out as exactly 0."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(seed * 1000 + d)
    out = []
    if dt == np.float32:
        if metric in ("DistHellinger", "DistJeffreys", "DistJensenShannon"):
            for i in range(3):
                out.append(("random", _prob(rng, d, False), _prob(rng, d, False)))
            out.append(("zeros in both", _prob(rng, d, True), _prob(rng, d, True)))
            p = _prob(rng, d, True)
            out.append(("identical", p, p.copy()))
            one = np.zeros(d, np.float32)
            one[d // 2] = 1.0
            out.append(("one-hot vs spread", one, _prob(rng, d, False)))
            out.append(("one-hot vs itself", one, one.copy()))
            return out
        if metric == "DistDot":
            def unit(v):
                return (v / np.linalg.norm(v.astype(np.float64))).astype(np.float32)
            for i in range(3):
                out.append(("random", unit(rng.standard_normal(d)), unit(rng.standard_normal(d))))
            v = unit(rng.standard_normal(d))
            out.append(("identical", v, v.copy()))
            out.append(("opposite", v, -v))
            one = np.zeros(d, np.float32)
            one[0] = 1.0
            out.append(("one-hot", one, unit(rng.standard_normal(d))))
            out.append(("zero vector", np.zeros(d, np.float32), v))
            return out
        for i in range(3):
            out.append(("random", rng.standard_normal(d).astype(np.float32) * 10, rng.random(d, dtype=np.float32)))
        v = rng.standard_normal(d).astype(np.float32)
        out.append(("identical", v, v.copy()))
        out.append(("zero vs x", np.zeros(d, np.float32), v))
        out.append(("zero vs zero", np.zeros(d, np.float32), np.zeros(d, np.float32)))
        one = np.zeros(d, np.float32)
        one[d - 1] = 3.0
        out.append(("one-hot", one, v))
        out.append(("large", np.full(d, 1e15, np.float32), np.full(d, -1e15, np.float32)))
        return out
    info = np.iinfo(dt)
    top = int(info.max) + 1
    for i in range(3):
        out.append(("random", rng.integers(info.min, top, d).astype(dt), rng.integers(info.min, top, d).astype(dt)))
    out.append(("few values", rng.integers(0, 3, d).astype(dt), rng.integers(0, 3, d).astype(dt)))
    v = rng.integers(0, top, d).astype(dt)
    out.append(("identical", v, v.copy()))
    out.append(("zero vs zero", np.zeros(d, dt), np.zeros(d, dt)))
    out.append(("zero vs x", np.zeros(d, dt), v))
    out.append(("max vs min", np.full(d, info.max, dt), np.full(d, info.min, dt)))
    out.append(("max vs max", np.full(d, info.max, dt), np.full(d, info.max, dt)))
    mixed = np.where(np.arange(d) % 2 == 0, info.max, info.min).astype(dt)
    out.append(("alternating ends", mixed, mixed[::-1].copy()))
    one = np.zeros(d, dt)
    one[d // 3] = info.max
    out.append(("one-hot max", one, np.zeros(d, dt)))
    return out


EXACT_ZERO = {  # (metric, pair name) whose distance is exactly 0 in every correct implementation
    ("DistL1", "identical"), ("DistL2", "identical"), ("DistCosine", "identical"), ("DistHamming", "identical"),
    ("DistJaccard", "identical"), ("DistJeffreys", "identical"), ("DistJensenShannon", "identical"),
    ("DistJeffreys", "one-hot vs itself"), ("DistJensenShannon", "one-hot vs itself"),
    ("DistCosine", "zero vs x"), ("DistCosine", "zero vs zero"), ("DistJaccard", "zero vs zero"),
    ("DistL1", "zero vs zero"), ("DistL2", "zero vs zero"), ("DistHamming", "zero vs zero"),
    ("DistL1", "max vs max"), ("DistL2", "max vs max"), ("DistHamming", "max vs max"), ("DistJaccard", "max vs max"),
}
