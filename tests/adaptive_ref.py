"""NumPy restatement of the adaptive-sampling rule of vpt_render_adaptive (include/vpt_b200.h), for the tests.

Per pixel a Welford state of the sample luminance Y = 0.2126 r + 0.7152 g + 0.0722 b is updated by every pass the pixel takes:

    n += 1;  d = Y - mean;  mean += d / n;  M2 += d * (Y - mean)
    err = sqrt(M2 / (n (n-1))) / max(mean, MEAN_FLOOR)          (infinite while n < 2)

After `min_passes` passes and then every `check_interval` passes, an active pixel stops when the largest err over its 3x3
neighbourhood (clipped at the frame edge; a stopped neighbour counts with the err it stopped with; a NaN err counts as +Inf) is
strictly below the threshold.  The frame ends after the last pass or when no pixel is active.  The state is float32 by default, as on
the device.

exact=True follows the device's pinned arithmetic (DESIGN.md section 8a) bit for bit: Y = fma(0.0722, b, fma(0.2126, r, 0.7152 g)),
every operation float32 round-to-nearest with subnormal inputs and results flushed to zero (as the .rn.ftz instructions do), M2's update
a product then a sum, and max(mean, floor) returning the floor for a NaN mean (fmaxf).
"""
import numpy as np

MEAN_FLOOR = 1e-3
LUMA = (0.2126, 0.7152, 0.0722)
F32 = np.float32
FLT_MIN = np.finfo(np.float32).tiny


def luminance(rgb, dtype=np.float32):
    """(..., 3) radiance -> (...) luminance, evaluated in `dtype`."""
    rgb = np.asarray(rgb, dtype=dtype)
    w = [dtype(c) for c in LUMA]
    return w[0] * rgb[..., 0] + w[1] * rgb[..., 1] + w[2] * rgb[..., 2]


def rel_error(n, mean, m2):
    """err of a Welford state (arrays of one dtype); infinite where n < 2."""
    n = np.asarray(n); dt = n.dtype.type
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.sqrt(m2 / (n * (n - dt(1)))) / np.maximum(mean, dt(MEAN_FLOOR))
    return np.where(n >= 2, e, dt(np.inf)).astype(n.dtype)


# ---- exact float32 arithmetic with flush-to-zero ---------------------------------------------------------------------------------
def ftz(x):
    """float32 with every subnormal replaced by a zero of its sign."""
    x = np.asarray(x, np.float32)
    return np.where(np.abs(x) < FLT_MIN, np.copysign(F32(0), x), x).astype(np.float32)


def fma_rn(a, b, c):
    """Correctly rounded float32 fma of float32 operands (no flushing).  The product is exact in float64; the sum is rounded to odd in
    float64 (round to nearest, then the odd neighbour toward the exact sum when inexact), which the final rounding to float32 turns into
    the correctly rounded result (53 >= 24 + 2 bits)."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)                      # exact error of s (TwoSum), NaN when s is not finite
        fix = np.isfinite(s) & (e != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def pfma(a, b, c):
    return ftz(fma_rn(ftz(a), ftz(b), ftz(c)))


def padd(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ftz(ftz(a) + ftz(b))


def psub(a, b):
    with np.errstate(over="ignore", invalid="ignore"):
        return ftz(ftz(a) - ftz(b))


def pmul(a, b):
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        return ftz(ftz(a) * ftz(b))


def pdiv(a, b):
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        return ftz(ftz(a) / ftz(b))


def psqrt(a):
    with np.errstate(invalid="ignore"):
        return ftz(np.sqrt(ftz(a)))


def luminance_exact(rgb):
    """(..., 3) float32 radiance -> the device's luminance bits: fma(0.0722, b, fma(0.2126, r, 0.7152 g))."""
    rgb = np.asarray(rgb, np.float32)
    return pfma(F32(LUMA[2]), rgb[..., 2], pfma(F32(LUMA[0]), rgb[..., 0], pmul(F32(LUMA[1]), rgb[..., 1])))


def welford_exact(n, mean, m2, y):
    """One pass of the device's Welford step on float32 arrays; returns the new (n, mean, m2)."""
    n = padd(n, F32(1))
    d = psub(y, mean)
    mean = padd(mean, pdiv(d, n))
    m2 = padd(m2, pmul(d, psub(y, mean)))
    return n, mean, m2


def rel_error_exact(n, mean, m2):
    """The device's err bits: sqrt(M2 / (n (n-1))) / fmaxf(mean, 1e-3), +Inf where n < 2."""
    floor = np.fmax(ftz(mean), F32(MEAN_FLOOR)).astype(np.float32)
    e = pdiv(psqrt(pdiv(m2, pmul(n, psub(n, F32(1))))), floor)
    return np.where(np.asarray(n) >= 2, e, F32(np.inf)).astype(np.float32)


def max3x3(a):
    """Largest value over each element's 3x3 neighbourhood, clipped at the edge of the 2-D array; a NaN counts as +Inf."""
    a = np.where(np.isnan(a), np.inf, a).astype(a.dtype)
    h, w = a.shape
    p = np.full((h + 2, w + 2), -np.inf, dtype=a.dtype)
    p[1:-1, 1:-1] = a
    return np.max([p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w] for dy in (-1, 0, 1) for dx in (-1, 0, 1)], axis=0)


def simulate(samples, min_passes, check_interval, threshold, dtype=np.float32, exact=False):
    """samples: (P, H, W) luminance of each pass (P = the frame's pass budget), or (P, H, W, 3) radiance.  exact: the device's pinned
    float32 arithmetic (the luminance too, for radiance), compared with the threshold as a float32.

    Returns dict(counts (H, W) int64 passes taken, err (H, W) last err, passes_run, tests: one dict per convergence test with
    `passes` (the test point), `err` (every pixel's err at the test) and `active` (pixels active before the test))."""
    s = np.asarray(samples)
    if exact:
        dtype = np.float32
        Y = luminance_exact(s) if s.ndim == 4 else s.astype(np.float32)
        step, err_of = welford_exact, rel_error_exact
    else:
        Y = luminance(s, dtype) if s.ndim == 4 else s.astype(dtype)
        step, err_of = None, rel_error
    P, H, W = Y.shape
    dt = np.dtype(dtype).type
    n = np.zeros((H, W), dtype); mean = np.zeros((H, W), dtype); m2 = np.zeros((H, W), dtype)
    err = np.full((H, W), np.inf, dtype)
    active = np.ones((H, W), bool)
    counts = np.zeros((H, W), np.int64)
    tests = []
    next_test, done = int(min_passes), 0
    while done < P and active.any():
        y = Y[done]; a = active
        if step is not None:
            n[a], mean[a], m2[a] = step(n[a], mean[a], m2[a], y[a])
        else:
            n[a] += dt(1)
            d = y[a] - mean[a]
            mean[a] += d / n[a]
            m2[a] += d * (y[a] - mean[a])
        counts[a] += 1
        done += 1
        if done == next_test and done < P:
            err[a] = err_of(n[a], mean[a], m2[a])
            tests.append(dict(passes=done, err=err.copy(), active=active.copy()))
            active = active & ~(max3x3(err) < dt(threshold))
            next_test += int(check_interval)
    err[active] = err_of(n[active], mean[active], m2[active])
    return dict(counts=counts, err=err, passes_run=done, tests=tests)
