"""NumPy restatement of the deep-slice binning rule (include/vpt_b200.h, vpt_set_deep_buffers).

A sample of depth d falls in slice k of bounds z_0 < ... < z_K when d > 0, z_k <= d, and d < z_{k+1} or z_{k+1} = +inf.  A NaN, a miss
(d = 0) and a depth outside [z_0, z_K) fall in no slice."""
import numpy as np


def slice_of(depth, bounds):
    """-> int array shaped like `depth`: the slice of each depth, -1 for none (float32 comparisons, as the kernel makes them)"""
    d = np.asarray(depth, dtype=np.float32)
    z = np.asarray(bounds, dtype=np.float32)
    out = np.full(d.shape, -1, dtype=np.int64)
    with np.errstate(invalid="ignore"):
        for k in range(len(z) - 1):
            inside = (d > 0) & (z[k] <= d) & ((d < z[k + 1]) | np.isposinf(z[k + 1]))
            out[inside] = k
    return out


def in_slice(depth, bounds, k):
    return slice_of(depth, bounds) == k
