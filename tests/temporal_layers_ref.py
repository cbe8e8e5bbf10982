"""NumPy restatement of vpt_temporal_layers' layers (include/vpt_b200.h, DESIGN.md section 8r) on top of tests/temporal_ref.py.

beauty_taps() (temporal_ref.beauty_taps) finds, per pixel, the taps vpt_temporal's step 2 uses for the beauty -- the same motion
(temporal_ref.pixel_motion), the same bilinear footprint, the same drop rules (outside the frame, weight 0, a non-finite beauty history
colour) -- with their weights, the weight sum and the beauty's L_new.  blend_layer() blends one layer with them:
    h_x = sum(w H_x) / sum(w)  (fma in tap order),   out_x = h_x + (x - h_x) / L_new,
and copies x where the beauty has no history.  The layer is not clipped.  blend_layer_loop() is its per-pixel form, kept to check it.

dtype=np.float32 follows the kernel's order of operations with correctly rounded division, as temporal_ref does; the kernel's blend divides
with accum's fast-math division, so float32 results are exact only where that division needs no rounding.  np.float64 is the reference
for everything else, with temporal_ref's diff32 (x - h_x formed in float32) and ftz (denormals flushed in arithmetic, not in copies).
layer_reach() gives the M of the pass rule (temporal_ref.compare).
"""
import numpy as np

import temporal_ref as T
from temporal_ref import beauty_taps, layer_reach  # noqa: F401  (part of this module's interface)


def blend_layer(bt, src, history, channels, count=1, dt=np.float64, diff32=True, ftz=True):
    """One layer of `count` planes of `channels` channels blended with the beauty's taps `bt` (beauty_taps); (count, N, channels)."""
    N = len(bt["used"])
    X32 = np.asarray(src, np.float32).reshape(count, N, channels)
    out = X32.astype(dt)
    if history is None:
        return out
    used = bt["used"]
    Hh = T.flush(np.asarray(history, np.float32).reshape(count, N, channels), ftz).astype(dt)
    fma, _ = T._ops(dt)
    with np.errstate(all="ignore"):
        s = np.zeros((count, N, channels), dt)
        for k in range(4):
            t = bt["taps"][:, k]
            s = np.where((t >= 0)[None, :, None], T.flush(fma(bt["w"][:, k].astype(dt)[None, :, None], Hh[:, np.maximum(t, 0)], s), ftz),
                         s).astype(dt)
        h = T.flush((s / np.where(used, bt["sw"], 1).astype(dt)[None, :, None]).astype(dt), ftz)
        o = T.blend(h, T.flush(X32, ftz), bt["L"].astype(dt)[None, :, None], dt, diff32, ftz)
    return np.where(used[None, :, None], T.flush(o, ftz), out).astype(dt)


def blend_layer_loop(bt, src, history, channels, count=1, dt=np.float64):
    """blend_layer() pixel by pixel, without the diff32 / ftz decisions"""
    N = len(bt["used"])
    X = np.asarray(src, np.float32).reshape(count, N, channels).astype(dt)
    out = X.copy()
    if history is None:
        return out
    Hh = np.asarray(history, np.float32).reshape(count, N, channels).astype(dt)
    fma, _ = T._ops(dt)
    with np.errstate(all="ignore"):
        for p in np.flatnonzero(bt["used"]):
            s = np.zeros((count, channels), dt)
            for k in range(4):
                t = bt["taps"][p, k]
                if t < 0:
                    continue
                s = fma(bt["w"][p, k], Hh[:, t], s).astype(dt)
            h = (s / bt["sw"][p]).astype(dt)
            out[:, p] = (h + (X[:, p] - h) / bt["L"][p]).astype(dt)
    return out
