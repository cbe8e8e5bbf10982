"""The exact float32 mode of tests/adaptive_ref.py, which the GPU tests hold the device's stopping rule to bit for bit: its fma and
flush-to-zero helpers against libm, its errors against hand computations, the pinned luminance order, and the scale invariance of
the rule (multiplying every sample by 2^k leaves the err bits alone while nothing underflows, overflows or reaches the mean floor)."""
import ctypes
import ctypes.util

import numpy as np
import pytest

import adaptive_ref as A

F32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)


@pytest.fixture(scope="module")
def libm():
    m = ctypes.CDLL(ctypes.util.find_library("m"))
    m.fmaf.restype = ctypes.c_float
    m.fmaf.argtypes = [ctypes.c_float] * 3
    return m


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def edge_operands():
    """Operand triples where a double-rounded or an unfused fma goes wrong: exact cancellation, ties, overflow, underflow, non-finite."""
    rng = np.random.default_rng(1)
    n = 4000
    a = (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    with np.errstate(over="ignore"):
        c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * 1e-7)).astype(np.float32)   # near-cancellation
    one_ulp = np.float32(1 + 2.0 ** -23)
    special = [(one_ulp, one_ulp, F32(-1)), (F32(1 + 2.0 ** -12), F32(1 + 2.0 ** -12), F32(2.0 ** -48)),   # sums at a tie
               (F32(FLT_MAX), F32(2), F32(-FLT_MAX)), (F32(FLT_MAX), F32(1.5), F32(0)), (F32(1e-30), F32(1e-10), F32(0)),
               (F32(1e-20), F32(1e-19), F32(-1e-39)), (F32(np.inf), F32(0), F32(1)), (F32(np.inf), F32(1), F32(-np.inf)),
               (F32(np.nan), F32(1), F32(1)), (F32(-0.0), F32(1), F32(0.0)), (F32(3), F32(1e-45), F32(0)), (F32(0.1), F32(10), F32(-1))]
    sa, sb, sc = (np.array(v, np.float32) for v in zip(*special))
    return np.concatenate([a, sa]), np.concatenate([b, sb]), np.concatenate([c, sc])


def test_fma_is_libm_fmaf(libm):
    a, b, c = edge_operands()
    with np.errstate(over="ignore"):
        want = np.array([libm.fmaf(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], np.float32)
    got = A.fma_rn(a, b, c)
    same = (bits(got) == bits(want)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), list(zip(a[~same][:5], b[~same][:5], c[~same][:5]))
    # and the unfused product-then-sum differs somewhere, so the comparison has teeth
    with np.errstate(over="ignore", invalid="ignore"):
        unfused = (a * b + c).astype(np.float32)
    assert (bits(unfused) != bits(want)).sum() > 100


def test_flush_to_zero_helpers(libm):
    sub = np.array([1e-45, -1e-45, 1e-39, -1.1e-38, np.nextafter(F32(FLT_MIN), F32(0))], np.float32)
    assert (bits(A.ftz(sub)) == bits(np.copysign(F32(0), sub))).all()
    keep = np.array([FLT_MIN, -FLT_MIN, 0.0, -0.0, 1.0, FLT_MAX, np.inf, -np.inf], np.float32)
    assert (bits(A.ftz(keep)) == bits(keep)).all()
    assert np.isnan(A.ftz(np.float32(np.nan)))
    # a subnormal operand is flushed before the operation, a subnormal result after it
    assert bits(A.pfma(F32(1e-39), F32(1e30), F32(0))) == bits(F32(0))                 # libm would give ~1e-9
    assert libm.fmaf(1e-39, 1e30, 0.0) > 0
    assert bits(A.pmul(F32(1e-20), F32(1e-20))) == bits(F32(0))
    assert bits(A.pmul(F32(-1e-20), F32(1e-20))) == bits(F32(-0.0))
    assert bits(A.pdiv(F32(1e-30), F32(1e10))) == bits(F32(0))
    assert bits(A.padd(F32(1.5e-38), F32(-1.2e-38))) == bits(F32(0))                   # exact difference is subnormal
    # every result that is normal is libm's correctly rounded one
    a, b, c = edge_operands()
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        want = np.array([libm.fmaf(x, y, z) for x, y, z in zip(A.ftz(a).tolist(), A.ftz(b).tolist(), A.ftz(c).tolist())], np.float32)
    got = A.pfma(a, b, c)
    normal = np.isfinite(want) & (np.abs(want) >= FLT_MIN)
    assert (bits(got[normal]) == bits(want[normal])).all()
    assert (got[np.isfinite(want) & (np.abs(want) < FLT_MIN)] == 0).all()


def err_of(ys):
    n = mean = m2 = np.zeros(1, np.float32)
    for y in ys:
        n, mean, m2 = A.welford_exact(n, mean, m2, np.array([y], np.float32))
    return A.rel_error_exact(n, mean, m2)[0], (n[0], mean[0], m2[0])


def test_errors_match_hand_computations():
    # 1, 3: n 2, mean 2, M2 = 0 + 2 (3 - 2) = 2, err = sqrt(2 / 2) / 2
    e, st = err_of([1, 3])
    assert st == (2, 2, 2) and e == F32(0.5)
    # 2, 4, 6, 8: mean 5, M2 20 (exact in float32 at every step), err = sqrt(20 / 12) / 5
    e, st = err_of([2, 4, 6, 8])
    assert st == (4, 5, 20) and bits(e) == bits(F32(np.sqrt(F32(20) / F32(12))) / F32(5))
    # constant samples: err exactly 0, also at zero mean (the floor)
    assert err_of([0.25] * 9)[0] == 0 and err_of([0.0] * 3)[0] == 0
    # -1, 1: mean 0 takes the floor: sqrt(2 / 2) / 1e-3
    assert bits(err_of([-1, 1])[0]) == bits(F32(1) / F32(1e-3))
    # a negative mean takes the floor too
    assert bits(err_of([-3, -1])[0]) == bits(F32(1) / F32(1e-3))
    # one sample: +Inf; a NaN sample: NaN err (the mean takes the floor, M2 is NaN)
    assert err_of([5])[0] == np.inf
    assert np.isnan(err_of([1, np.nan, 1])[0])
    # large samples of one sign: M2 overflows to +Inf, err +Inf
    e, st = err_of([1e38, 3e38])
    assert e == np.inf and st[1] == F32(F32(1e38) + F32(F32(F32(3e38) - F32(1e38)) / F32(2))) and st[2] == np.inf
    # opposite signs of large magnitude: Y - mean overflows, the mean becomes -Inf, M2 = -Inf * Inf, err NaN
    e, st = err_of([3e38, -3e38])
    assert np.isnan(e) and st[1] == -np.inf
    # an Inf sample: d = Inf, mean Inf, M2 = Inf * (Inf - Inf) = NaN
    assert np.isnan(err_of([1, np.inf])[0])


def test_luminance_is_the_pinned_fma_chain():
    from fractions import Fraction as Fr
    rng = np.random.default_rng(3)
    rgb = rng.uniform(0, 4, (5000, 3)).astype(np.float32)
    got = A.luminance_exact(rgb)
    w = [F32(c) for c in A.LUMA]

    def rn(x):                                          # Fraction -> nearest float32 (the values here are normal)
        f = np.float32(float(x))                        # nearest double, then float32: exact enough to pick a candidate
        cands = [np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))]
        return min(cands, key=lambda c: (abs(Fr(float(c)) - x), int(np.float32(c).view(np.uint32)) & 1))
    for k in range(200):
        r, g, b = (Fr(float(v)) for v in rgb[k])
        t = rn(Fr(float(w[1])) * g)                                   # pmul(0.7152, g)
        t = rn(Fr(float(w[0])) * r + Fr(float(t)))                     # pfma(0.2126, r, .)
        t = rn(Fr(float(w[2])) * b + Fr(float(t)))                     # pfma(0.0722, b, .)
        assert bits(got[k]) == bits(t), k
    # the order matters: a contraction in another order gives other bits on some samples
    other = A.pfma(w[1], rgb[:, 1], A.pfma(w[2], rgb[:, 2], A.pmul(w[0], rgb[:, 0])))
    assert (bits(other) != bits(got)).sum() > 50


def noisy(P, H, W, seed):
    rng = np.random.default_rng(seed)
    level = rng.uniform(0.5, 2.0, (1, H, W, 1))
    sigma = rng.uniform(0.0, 0.6, (1, H, W, 1))
    return (level * (1 + sigma * rng.standard_normal((P, H, W, 3)))).astype(np.float32)


@pytest.mark.parametrize("k", [-6, -2, 1, 5, 20, 55])
def test_scale_invariance_of_the_exact_rule(k):
    """Samples times 2^k: every intermediate scales exactly, so err bits and counts are unchanged while mean 2^k stays above the floor
    at every test and M2 4^k stays finite (and nothing becomes subnormal)."""
    P, H, W, mn, iv = 40, 9, 13, 4, 3
    s = noisy(P, H, W, 5)
    s[:, 2:4, 5:8] = np.abs(s[:, 2:4, 5:8])                     # keep every mean positive
    s = np.abs(s)
    base = A.simulate(s, mn, iv, FLT_MAX, exact=True)["tests"][0]["err"]
    thr = float(np.quantile(A.max3x3(base), 0.5))
    ref = A.simulate(s, mn, iv, thr, exact=True)
    assert len(np.unique(ref["counts"])) >= 2
    scaled = (s * np.float32(2.0 ** k)).astype(np.float32)
    assert (scaled == s.astype(np.float64) * 2.0 ** k).all()
    got = A.simulate(scaled, mn, iv, thr, exact=True)
    # the conditions of the claim on the scaled samples: every running mean from the first test on above the floor, M2 finite
    Y = A.luminance_exact(scaled).astype(np.float64)
    run = np.cumsum(Y, axis=0) / np.arange(1, P + 1)[:, None, None]
    assert run[mn - 1:].min() > 2e-3 and (Y ** 2).sum(axis=0).max() < 1e37
    assert np.array_equal(got["counts"], ref["counts"]) and got["passes_run"] == ref["passes_run"]
    assert (bits(got["err"]) == bits(ref["err"])).all()
    for a, b in zip(got["tests"], ref["tests"]):
        assert (bits(a["err"]) == bits(b["err"])).all()


def test_past_overflow_the_error_is_infinite_or_nan():
    P, H, W = 12, 4, 5
    s = noisy(P, H, W, 8)
    s = np.abs(s) + 0.1
    big = (s * np.float32(2.0 ** 126)).astype(np.float32)       # ~1e38: luminance finite, d * d overflows
    got = A.simulate(big, 2, 2, FLT_MAX, exact=True)["tests"][0]["err"]
    assert (np.isinf(got) | np.isnan(got) | (got >= A.simulate(s, 2, 2, FLT_MAX, exact=True)["tests"][0]["err"])).all()


def test_max3x3_counts_nan_as_infinity():
    a = np.zeros((4, 5), np.float32); a[1, 2] = np.nan
    m = A.max3x3(a)
    assert (m[0:3, 1:4] == np.inf).all() and m[3].max() == 0 and m[:, 0].max() == 0
    # a pixel with a NaN err and its 8 neighbours never stop; the rest stop at the first test
    s = np.ones((10, 4, 5, 3), np.float32); s[0, 1, 2] = np.nan
    out = A.simulate(s, 2, 2, 0.5, exact=True)
    want = np.full((4, 5), 2); want[0:3, 1:4] = 10
    assert np.array_equal(out["counts"], want)
