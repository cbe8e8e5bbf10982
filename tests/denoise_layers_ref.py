"""NumPy restatement of vpt_denoise_layers (include/vpt_b200.h), for the tests: the beauty as tests/denoise_ref.py filters it, and every
layer filtered at every level with the beauty's weights of that level,

    x' = sum(h w x_q) / sum(h w)

over the same taps, with the same copy rule (a pixel the beauty copies keeps its layer values).  Each level is evaluated in float64 and
stored in float32 (flushed with ftz), as the device keeps its planes; the weights are tests/denoise_ref.py's level_taps.
"""
import numpy as np

from denoise_ref import apply_level, filter_levels


def denoise_layers(color, layers, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, ftz=True):
    """(H, W, 3) frame and a list of (H, W, C) or (H, W) float32 layers -> (denoised frame, [denoised layers]) in float32."""
    flat = [np.asarray(x, np.float32) for x in layers]
    xs = [x[..., None] if x.ndim == 2 else x.copy() for x in flat]
    for c, filt, taps in filter_levels(color, depth, rel_error, iterations, sigma_luminance, sigma_depth, ftz):
        xs = [apply_level(x, filt, taps, ftz) for x in xs]
    return c, [x[..., 0] if f.ndim == 2 else x for x, f in zip(xs, flat)]
