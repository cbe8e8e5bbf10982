"""NumPy restatement of the adaptive-sampling rule of vpt_render_adaptive (include/vpt_b200.h), for the tests.

Per pixel a Welford state of the sample luminance Y = 0.2126 r + 0.7152 g + 0.0722 b is updated by every pass the pixel takes:

    n += 1;  d = Y - mean;  mean += d / n;  M2 += d * (Y - mean)
    err = sqrt(M2 / (n (n-1))) / max(mean, MEAN_FLOOR)          (infinite while n < 2)

After `min_passes` passes and then every `check_interval` passes, an active pixel stops when the largest err over its 3x3
neighbourhood (clipped at the frame edge; a stopped neighbour counts with the err it stopped with) is strictly below the
threshold.  The frame ends after the last pass or when no pixel is active.  The state is float32 by default, as on the device.
"""
import numpy as np

MEAN_FLOOR = 1e-3
LUMA = (0.2126, 0.7152, 0.0722)


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


def max3x3(a):
    """Largest value over each element's 3x3 neighbourhood, clipped at the edge of the 2-D array."""
    h, w = a.shape
    p = np.full((h + 2, w + 2), -np.inf, dtype=a.dtype)
    p[1:-1, 1:-1] = a
    return np.max([p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w] for dy in (-1, 0, 1) for dx in (-1, 0, 1)], axis=0)


def simulate(samples, min_passes, check_interval, threshold, dtype=np.float32):
    """samples: (P, H, W) luminance of each pass (P = the frame's pass budget), or (P, H, W, 3) radiance.

    Returns dict(counts (H, W) int64 passes taken, err (H, W) last err, passes_run, tests: one dict per convergence test with
    `passes` (the test point), `err` (every pixel's err at the test) and `active` (pixels active before the test))."""
    s = np.asarray(samples)
    Y = luminance(s, dtype) if s.ndim == 4 else s.astype(dtype)
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
        n[a] += dt(1)
        d = y[a] - mean[a]
        mean[a] += d / n[a]
        m2[a] += d * (y[a] - mean[a])
        counts[a] += 1
        done += 1
        if done == next_test and done < P:
            err[a] = rel_error(n[a], mean[a], m2[a])
            tests.append(dict(passes=done, err=err.copy(), active=active.copy()))
            active = active & ~(max3x3(err) < dt(threshold))
            next_test += int(check_interval)
    err[active] = rel_error(n[active], mean[active], m2[active])
    return dict(counts=counts, err=err, passes_run=done, tests=tests)
