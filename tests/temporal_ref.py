"""NumPy restatement of vpt_temporal (include/vpt_b200.h, DESIGN.md section 8p).

Per pixel (x, y) of a W x H frame, with C the colour, M = (c vx, c vy, c) the premultiplied motion vectors towards the history's camera B,
A the frame camera, H / L the history and its lengths:
  1. v = M.xy, and when M.z < 1: v = fma(1 - M.z, pi_B(d) - pi_A(d), M.xy), d = fma(t, v_A, fma(s, h_A, e_A)) the direction through the
     pixel centre (s = (x + 1/2) / W, t = (y + 1/2) / H); no history if either projection fails.
  2. q = (x + 1/2, y + 1/2) + v; no history if v is not finite or q is outside [0, W] x [0, H]; else the bilinear taps around q - 1/2 in
     the order (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1), dropping taps outside the frame, of weight 0 or with a non-finite
     colour, renormalised; L_hist the least L of the taps used.
  3. h' = clamp(h, mu - gamma sigma, mu + gamma sigma), mu / sigma the mean and population deviation of C's finite 3x3 window.
  4. L_new = min(L_hist + 1, max_history), out = h' + (C - h') / L_new; no history or a non-finite C: out = C, L_new = 1.

dtype=np.float32 follows the kernel's operation order (each fma rounded once, through float64), for the cases the tests compare bit for
bit: zero motion, integer shifts, no history.  Its division is correctly rounded, while the kernel's blend divides with accum's fast-math
division, so a float32 blend is exact where L_new is a power of two or the quotient needs no rounding.  dtype=np.float64 is the reference
for everything else.
"""
import numpy as np


def cam_fields(cam):
    """(origin, lower_left_corner, horizontal, vertical) of a vpt_camera (ctypes) or a dict, as float32 arrays"""
    if isinstance(cam, dict):
        return tuple(np.asarray(cam[k], np.float32) for k in ("origin", "lower_left_corner", "horizontal", "vertical"))
    f = lambda v: np.array([v.x, v.y, v.z], np.float32)
    return f(cam.origin), f(cam.lower_left_corner), f(cam.horizontal), f(cam.vertical)


def _ops(dt):
    if dt == np.float64:
        return (lambda a, b, c: a * b + c), (lambda a, b: a * b)
    f64 = np.float64
    fma = lambda a, b, c: (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(np.float32)
    mul = lambda a, b: (np.asarray(a, np.float32) * np.asarray(b, np.float32)).astype(np.float32)
    return fma, mul


def film_cam(cam, dt=np.float64):
    o, llc, h, v = (a.astype(dt) for a in cam_fields(cam))
    fma, mul = _ops(dt)
    dot = lambda a, b: fma(a[..., 2], b[..., 2], fma(a[..., 0], b[..., 0], mul(a[..., 1], b[..., 1])))
    cross = lambda a, b: np.stack([fma(a[..., 1], b[..., 2], -mul(a[..., 2], b[..., 1])), fma(a[..., 2], b[..., 0], -mul(a[..., 0], b[..., 2])),
                                   fma(a[..., 0], b[..., 1], -mul(a[..., 1], b[..., 0]))], -1)
    e = (llc - o).astype(dt)
    K = dict(o=o, e=e, h=h, v=v, hh=dot(h, h), hv=dot(h, v), vv=dot(v, v), dot=dot, cross=cross, fma=fma, mul=mul, dt=dt)
    K["en"] = dot(e, cross(h, v))
    K["det"] = fma(K["hh"], K["vv"], -mul(K["hv"], K["hv"]))
    return K


def film_project_dir(K, d, W, H):
    """pi_K with d in place of P - origin: ((N, 2) film positions, (N,) ok)"""
    dt, fma, mul, dot = K["dt"], K["fma"], K["mul"], K["dot"]
    with np.errstate(all="ignore"):
        k = (K["en"] / dot(d, K["cross"](K["h"], K["v"]))).astype(dt)
        q = np.stack([fma(k, d[:, i], -K["e"][i]) for i in range(3)], -1)
        qh, qv = dot(q, K["h"]), dot(q, K["v"])
        if K["hv"] == 0:
            s, t = (qh / K["hh"]).astype(dt), (qv / K["vv"]).astype(dt)
        else:
            s = (fma(K["vv"], qh, -mul(K["hv"], qv)) / K["det"]).astype(dt)
            t = (fma(K["hh"], qv, -mul(K["hv"], qh)) / K["det"]).astype(dt)
        st = np.stack([mul(s, dt(W)), mul(t, dt(H))], -1)
    return st, (k > 0) & np.isfinite(st).all(-1)


def pixel_motion(W, H, vectors, cam_a, cam_b, dt=np.float64):
    """((N, 2) v, (N,) ok) for the row-major pixels of the frame; vectors (N, 3)"""
    M = np.asarray(vectors, np.float32).reshape(-1, 3).astype(dt)
    v = M[:, :2].copy()
    ok = np.ones(len(M), bool)
    env = M[:, 2] < 1
    if env.any():
        A, B = film_cam(cam_a, dt), film_cam(cam_b, dt)
        fma = A["fma"]
        y, x = np.divmod(np.arange(W * H), W)
        s = ((x.astype(dt) + dt(0.5)) / dt(W)).astype(dt)
        t = ((y.astype(dt) + dt(0.5)) / dt(H)).astype(dt)
        d = np.stack([fma(t, A["v"][i], fma(s, A["h"][i], A["e"][i])) for i in range(3)], -1)[env]
        pa, oka = film_project_dir(A, d, W, H)
        pb, okb = film_project_dir(B, d, W, H)
        w = (dt(1) - M[env, 2]).astype(dt)
        with np.errstate(all="ignore"):
            ve = np.stack([fma(w, (pb[:, i] - pa[:, i]).astype(dt), M[env, i]) for i in range(2)], -1)
        v[env] = ve
        ok[env] = oka & okb
    return v, ok


def accum_step(acc, value, n):
    """accum's running mean in float32: acc + (value - acc) / (float)n (correctly rounded division)"""
    acc, value = np.asarray(acc, np.float32), np.asarray(value, np.float32)
    return (acc + (value - acc) / np.float32(n)).astype(np.float32)


def temporal(W, H, color, vectors, cam_a, cam_b, history=None, history_len=None, max_history=16, clip_sigma=np.inf, dt=np.float64,
             motion_dt=None):
    """vpt_temporal computed in dtype dt: a dict of out (N, 3), L (N,), used (N,) bool (the pixel had a history), h (N, 3) the fetched
    history and hc (N, 3) the clipped one (NaN where unused).  motion_dt: the dtype of step 1 (None: dt); np.float32 puts the kernel's
    rounding of the motion into a float64 computation of the rest, for inputs whose history is not smooth"""
    N = W * H
    C = np.asarray(color, np.float32).reshape(N, 3).astype(dt)
    out, L = C.copy(), np.ones(N, dt)
    used = np.zeros(N, bool)
    hf, hcl = np.full((N, 3), np.nan, dt), np.full((N, 3), np.nan, dt)
    res = dict(out=out, L=L, used=used, h=hf, hc=hcl)
    if history is None:
        return res
    Hh = np.asarray(history, np.float32).reshape(N, 3).astype(dt)
    Lh = np.asarray(history_len, np.float32).reshape(N).astype(dt)
    fma, mul = _ops(dt)
    v, ok = pixel_motion(W, H, vectors, cam_a, cam_b, motion_dt or dt)
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
        sw, sh, lmin = dt(0), np.zeros(3, dt), None
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
                sh = np.array([fma(w, Hh[t, c], sh[c]) for c in range(3)], dt)
        if not sw > 0:
            continue
        h = (sh / sw).astype(dt)
        hf[p] = h
        if np.isfinite(clip_sigma):
            win = [C[yy * W + xx] for yy in range(y[p] - 1, y[p] + 2) for xx in range(x[p] - 1, x[p] + 2)
                   if 0 <= xx < W and 0 <= yy < H and cfin[yy * W + xx]]
            n = dt(len(win))
            s = np.zeros(3, dt)
            for c in win:
                s = (s + c).astype(dt)
            mu = (s / n).astype(dt)
            ss = np.zeros(3, dt)
            for c in win:
                d = (c - mu).astype(dt)
                ss = np.array([fma(d[k], d[k], ss[k]) for k in range(3)], dt)
            r = mul(dt(clip_sigma), np.sqrt((ss / n).astype(dt)).astype(dt))
            h = np.minimum(np.maximum(h, (mu - r).astype(dt)), (mu + r).astype(dt))
        hcl[p] = h
        Ln = min(dt(lmin + 1), dt(max_history))
        out[p] = (h + (C[p] - h) / Ln).astype(dt)
        L[p] = Ln
        used[p] = True
    return res
