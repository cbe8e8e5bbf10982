"""NumPy restatement of vpt_temporal_layers' layers (include/vpt_b200.h, DESIGN.md section 8r) on top of tests/temporal_ref.py.

beauty_taps() finds, per pixel, the taps vpt_temporal's step 2 uses for the beauty -- the same motion (temporal_ref.pixel_motion), the
same bilinear footprint, the same drop rules (outside the frame, weight 0, a non-finite beauty history colour) -- with their weights, the
weight sum and the beauty's L_new.  blend_layer() blends one layer with them:
    h_x = sum(w H_x) / sum(w)  (fma in tap order),   out_x = h_x + (x - h_x) / L_new,
and copies x where the beauty has no history.  The layer is not clipped.

dtype=np.float32 follows the kernel's order of operations with correctly rounded division, as temporal_ref does; the kernel's blend divides
with accum's fast-math division, so float32 results are exact only where that division needs no rounding.  np.float64 is the reference
for everything else.
"""
import numpy as np

import temporal_ref as T


def beauty_taps(W, H, color, vectors, cam_a, cam_b, history, history_len, max_history=16, dt=np.float64, motion_dt=None):
    """The beauty's taps: a dict of used (N,) bool (the pixel has a history), taps (N, 4) int (pixel index of each tap, -1 when not used,
    in the order (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)), w (N, 4) their weights (0 when not used), sw (N,) the weight
    sum in tap order and L (N,) the beauty's L_new (1 without history)."""
    N = W * H
    C = np.asarray(color, np.float32).reshape(N, 3)
    res = dict(used=np.zeros(N, bool), taps=np.full((N, 4), -1, np.int64), w=np.zeros((N, 4), dt), sw=np.zeros(N, dt), L=np.ones(N, dt))
    if history is None:
        return res
    Hh = np.asarray(history, np.float32).reshape(N, 3)
    Lh = np.asarray(history_len, np.float32).reshape(N).astype(dt)
    fma, mul = T._ops(dt)
    v, ok = T.pixel_motion(W, H, vectors, cam_a, cam_b, motion_dt or dt)
    v = v.astype(dt)
    cfin = np.isfinite(C).all(1)
    hfin = np.isfinite(Hh).all(1)
    y, x = np.divmod(np.arange(N), W)
    for p in np.flatnonzero(ok & cfin & np.isfinite(v).all(1)):
        qx, qy = dt(dt(x[p]) + dt(0.5)) + dt(v[p, 0]), dt(dt(y[p]) + dt(0.5)) + dt(v[p, 1])
        if not (0 <= qx <= W and 0 <= qy <= H):
            continue
        px, py = dt(qx - dt(0.5)), dt(qy - dt(0.5))
        x0, y0 = np.floor(px), np.floor(py)
        fx, fy = dt(px - x0), dt(py - y0)
        sw, lmin = dt(0), None
        taps, ws = [-1] * 4, [dt(0)] * 4
        for j in (0, 1):
            for i in (0, 1):
                tx, ty = int(x0) + i, int(y0) + j
                w = mul(fx if i else dt(dt(1) - fx), fy if j else dt(dt(1) - fy))
                if not w > 0 or tx < 0 or ty < 0 or tx >= W or ty >= H:
                    continue
                t = ty * W + tx
                if not hfin[t]:
                    continue
                lmin = Lh[t] if lmin is None else min(lmin, Lh[t])
                sw = dt(sw + w)
                taps[2 * j + i], ws[2 * j + i] = t, w
        if not sw > 0:
            continue
        res["used"][p] = True
        res["taps"][p] = taps
        res["w"][p] = ws
        res["sw"][p] = sw
        res["L"][p] = min(dt(lmin + 1), dt(max_history))
    return res


def blend_layer(bt, src, history, channels, count=1, dt=np.float64):
    """One layer of `count` planes of `channels` channels blended with the beauty's taps `bt` (beauty_taps); (count, N, channels)."""
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
