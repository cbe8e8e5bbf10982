"""NumPy restatement of vpt_temporal (include/vpt_b200.h, DESIGN.md section 8p).

Per pixel (x, y) of a W x H frame, with C the colour, M = (c vx, c vy, c) the premultiplied motion vectors towards the history's camera B,
A the frame camera, H / L the history and its lengths:
  1. v = M.xy, and when M.z < 1: v = fma(1 - M.z, pi_B(d) - pi_A(d), M.xy), d = fma(t, v_A, fma(s, h_A, e_A)) the direction through the
     pixel centre (s = (x + 1/2) / W, t = (y + 1/2) / H); no history if either projection fails.
  2. q = (x + 1/2, y + 1/2) + v; no history if v is not finite or q is outside [0, W] x [0, H]; else the bilinear taps around q - 1/2 in
     the order (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1), dropping taps outside the frame, of weight 0 or with a non-finite
     colour, renormalised; L_hist the least L of the taps used, a NaN length ignored (fminf), NaN when every used tap's is.
  3. h' = clamp(h, mu - gamma sigma, mu + gamma sigma), mu / sigma the mean and population deviation of C's finite 3x3 window; fmaxf /
     fminf, so a NaN bound leaves h as it is.
  4. L_new = fminf(L_hist + 1, max_history) in float32 (NaN L_hist: max_history), out = h' + (C - h') / L_new; no history or a
     non-finite C: out = C, L_new = 1.

temporal() is vectorised over the pixels; temporal_loop() is the per-pixel form it was written from, kept to check it on small frames.
dtype=np.float32 follows the kernel's operation order (each fma rounded once, through float64), for the cases the tests compare bit for
bit: zero motion, integer shifts, no history.  Its division is correctly rounded, while the kernel's blend divides with accum's fast-math
division, so a float32 blend is exact where L_new is a power of two or the quotient needs no rounding.  dtype=np.float64 is the reference
for everything else, with the float32 decisions the device makes switched on by flags:
  footprint_dt=np.float32  q, px, floor, fx, the tap weights and their sum in the kernel's float32 order, so the taps used, L and `used`
                           are decided as on the device (the history mean, clip and blend stay in dt);
  diff32                   C - h' formed in float32 from float32 operands: +-inf when C and h' lie near +-FLT_MAX with opposite signs;
  clip32                   the clip's window sum, mean, deviation and bounds in float32 in the kernel's order: a window sum that overflows
                           gives mu = +-inf, mu - r NaN, and the clip does nothing on that channel;
  ftz                      denormals flushed to zero in arithmetic (C, H, the layer values, clip_sigma, every float32 result), as the
                           library's --use_fast_math build does; copied pixels keep theirs.

compare() is the pass rule of the GPU tests: a pixel without history equals its input bit for bit, non-finite values match in kind, and
every finite value is within ATOL + R M, M the largest finite |value| the pixel read (the "M" of temporal(), layer_reach()).
"""
import numpy as np

import denoise_ref as D

F32 = np.float32
FLT_MIN = D.FLT_MIN
ATOL, RTOL = D.ATOL, D.RTOL
kind = D.kind


def flush(a, ftz=True):
    """`a` with its float32 denormals flushed to zero (sign kept), in a's dtype"""
    a = np.asarray(a)
    if not ftz:
        return a
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(a) < FLT_MIN, a * 0, a).astype(a.dtype)


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


def footprint(W, H, v, dt=np.float64):
    """Step 2's footprint of every pixel in dtype dt (np.float32: the kernel's __fadd_rn order): (inside (N,) bool -- v finite and q in
    [0, W] x [0, H] --, x0, y0 (N,) int the first tap, fx, fy (N,) the fractions); x0 = y0 = 0 where not inside."""
    N = len(v)
    y, x = np.divmod(np.arange(N), W)
    with np.errstate(all="ignore"):
        vv = np.asarray(v).astype(dt)
        qx = (x.astype(dt) + dt(0.5)).astype(dt) + vv[:, 0]
        qy = (y.astype(dt) + dt(0.5)).astype(dt) + vv[:, 1]
        inside = np.isfinite(vv).all(1) & (qx >= 0) & (qx <= dt(W)) & (qy >= 0) & (qy <= dt(H))
        px, py = np.where(inside, qx - dt(0.5), 0).astype(dt), np.where(inside, qy - dt(0.5), 0).astype(dt)
        fx0, fy0 = np.floor(px), np.floor(py)
        fx, fy = (px - fx0).astype(dt), (py - fy0).astype(dt)
    return inside, fx0.astype(np.int64), fy0.astype(np.int64), fx, fy


def tap_weight(fx, fy, i, j, dt=np.float64):
    """(i ? fx : 1 - fx) * (j ? fy : 1 - fy), each operation rounded in dt"""
    a = fx if i else (dt(1) - fx).astype(dt)
    b = fy if j else (dt(1) - fy).astype(dt)
    return (a * b).astype(dt)


def beauty_taps(W, H, color, vectors, cam_a, cam_b, history, history_len, max_history=16, dt=np.float64, motion_dt=None,
                footprint_dt=None, ftz=True):
    """Steps 1 and 2: a dict of used (N,) bool (the pixel has a history), taps (N, 4) int (pixel index of each tap, -1 when not used, in
    the order (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)), w (N, 4) their weights (0 when not used), sw (N,) the weight sum in
    tap order, h (N, 3) the history mean sum(w H) / sw (fma in tap order, NaN where unused), Lh (N,) L_hist and L (N,) L_new (1 without
    history), v (N, 2) the motion.  Weights, sw and the tap choice are computed in footprint_dt (None: dt), the mean in dt."""
    N = W * H
    fdt = footprint_dt or dt
    C = np.asarray(color, np.float32).reshape(N, 3)
    res = dict(used=np.zeros(N, bool), taps=np.full((N, 4), -1, np.int64), w=np.zeros((N, 4), dt), sw=np.zeros(N, dt),
               h=np.full((N, 3), np.nan, dt), Lh=np.full(N, np.nan, dt), L=np.ones(N, dt), v=np.full((N, 2), np.nan, dt))
    if history is None:
        return res
    Hh = flush(np.asarray(history, np.float32).reshape(N, 3), ftz).astype(dt)
    Lh = np.asarray(history_len, np.float32).reshape(N)
    hfin = np.isfinite(np.asarray(history, np.float32).reshape(N, 3)).all(1)
    v, ok = pixel_motion(W, H, vectors, cam_a, cam_b, motion_dt or dt)
    res["v"] = v.astype(dt)
    inside, x0, y0, fx, fy = footprint(W, H, v, fdt)
    cand = ok & np.isfinite(C).all(1) & inside
    fma, _ = _ops(dt)
    sw = np.zeros(N, fdt)
    sh = np.zeros((N, 3), dt)
    l = np.full(N, np.nan, np.float32)
    have = np.zeros(N, bool)
    with np.errstate(all="ignore"):
        for k in range(4):
            i, j = k & 1, k >> 1
            tx, ty = x0 + i, y0 + j
            w = tap_weight(fx, fy, i, j, fdt)
            use = cand & (w > 0) & (tx >= 0) & (ty >= 0) & (tx < W) & (ty < H)
            t = np.where(use, ty * W + tx, 0)
            use &= hfin[t]
            l = np.where(use, np.where(have, np.fmin(l, Lh[t]), Lh[t]), l)     # l = sw > 0 ? fminf(l, tl) : tl
            sw = np.where(use, (sw + w).astype(fdt), sw)
            sh = np.where(use[:, None], fma(w.astype(dt)[:, None], Hh[t], sh), sh).astype(dt)
            sh = flush(sh, ftz)
            have |= use
            res["taps"][:, k] = np.where(use, t, -1)
            res["w"][:, k] = np.where(use, w, 0)
        used = cand & (sw > 0)
        res["taps"][~used] = -1
        res["w"][~used] = 0
        res["used"] = used
        res["sw"] = np.where(used, sw, 0).astype(dt)
        res["h"] = np.where(used[:, None], flush(sh / np.where(used, sw, 1).astype(dt)[:, None], ftz), np.nan).astype(dt)
        res["Lh"] = np.where(used, l, np.nan).astype(dt)
        Ln = np.fmin((l + F32(1)).astype(F32), F32(max_history))                # fminf(L_hist + 1, max_history) in float32
        res["L"] = np.where(used, Ln, 1).astype(dt)
    return res


def _window(W, H, ok):
    """The 3x3 window of every pixel in the kernel's order: [(index (N,), in (N,) bool: inside the frame and ok)]"""
    N = W * H
    y, x = np.divmod(np.arange(N), W)
    out = []
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            tx, ty = x + dx, y + dy
            m = (tx >= 0) & (ty >= 0) & (tx < W) & (ty < H)
            t = np.where(m, ty * W + tx, 0)
            out.append((t, m & ok[t]))
    return out


def clip_bounds(W, H, color, clip_sigma, dt=np.float64, clip32=True, ftz=True):
    """(lo, hi, wmax): mu -+ clip_sigma sigma of every pixel's finite 3x3 window (N, 3), and the largest finite |value| in the window (N,).
    clip32: in float32 in the kernel's order (__fadd_rn sum, __fdiv_rn mean, fmaf deviations, __fsqrt_rn), each result flushed with ftz."""
    N = W * H
    C32 = np.asarray(color, np.float32).reshape(N, 3)
    cfin = np.isfinite(C32).all(1)
    win = _window(W, H, cfin)
    a = np.where(cfin[:, None], np.abs(C32.astype(np.float64)), 0).max(1)
    wmax = np.max([np.where(m, a[t], 0) for t, m in win], axis=0)
    cdt = np.float32 if clip32 else dt
    fl = (lambda z: flush(z, ftz)) if clip32 else (lambda z: z)
    Cw = fl(C32).astype(cdt)
    with np.errstate(all="ignore"):
        s = np.zeros((N, 3), cdt)
        n = np.zeros(N, cdt)
        for t, m in win:
            s = np.where(m[:, None], fl((s + Cw[t]).astype(cdt)), s)
            n = n + m
        mu = fl((s / n[:, None]).astype(cdt))
        ss = np.zeros((N, 3), cdt)
        for t, m in win:
            d = fl((Cw[t] - mu).astype(cdt))
            ss = np.where(m[:, None], fl((d.astype(np.float64) * d + ss).astype(cdt)), ss)
        g = fl(np.asarray(clip_sigma, np.float32)).astype(cdt)
        r = fl((g * fl(np.sqrt(fl((ss / n[:, None]).astype(cdt))).astype(cdt))).astype(cdt))
        lo, hi = fl((mu - r).astype(cdt)), fl((mu + r).astype(cdt))
    return lo.astype(dt), hi.astype(dt), wmax


def blend(h, x, L, dt=np.float64, diff32=True, ftz=True):
    """h + (x - h) / L, with x - h formed in float32 (diff32) and float32 results flushed (ftz)"""
    with np.errstate(all="ignore"):
        if diff32:
            d = flush((flush(np.asarray(x, F32), ftz) - np.asarray(h).astype(F32)).astype(F32), ftz).astype(dt)
        else:
            d = (np.asarray(x).astype(dt) - h).astype(dt)
        return (h + (d / L).astype(dt)).astype(dt)


def temporal(W, H, color, vectors, cam_a, cam_b, history=None, history_len=None, max_history=16, clip_sigma=np.inf, dt=np.float64,
             motion_dt=None, footprint_dt=None, diff32=True, clip32=True, ftz=True):
    """vpt_temporal computed in dtype dt: a dict of out (N, 3), L (N,), used (N,) bool (the pixel had a history), h (N, 3) the fetched
    history, hc (N, 3) the clipped one (NaN where unused), M (N,) the largest finite |value| the pixel read (C, its window when clipped,
    the history taps used) and the taps of beauty_taps().  motion_dt: the dtype of step 1 (None: dt); np.float32 puts the kernel's
    rounding of the motion into a float64 computation of the rest, for inputs whose history is not smooth.  footprint_dt, diff32, clip32,
    ftz: see the module's docstring."""
    N = W * H
    C32 = np.asarray(color, np.float32).reshape(N, 3)
    C = C32.astype(dt)
    with np.errstate(invalid="ignore"):
        M = np.where(np.isfinite(C32), np.abs(C32.astype(np.float64)), 0).max(1)
    bt = beauty_taps(W, H, color, vectors, cam_a, cam_b, history, history_len, max_history, dt, motion_dt, footprint_dt, ftz)
    used = bt["used"]
    out = C.copy()
    res = dict(bt, out=out, M=M, hc=np.full((N, 3), np.nan, dt))
    if history is None or not used.any():
        return res
    Hh = np.asarray(history, np.float32).reshape(N, 3).astype(np.float64)
    for k in range(4):
        t = bt["taps"][:, k]
        M = np.maximum(M, np.where(t >= 0, np.abs(Hh[np.maximum(t, 0)]).max(1), 0))
    h = bt["h"]
    if np.isfinite(clip_sigma):
        lo, hi, wmax = clip_bounds(W, H, color, clip_sigma, dt, clip32, ftz)
        M = np.where(used, np.maximum(M, wmax), M)
        h = np.fmin(np.fmax(h, lo), hi)
    res["hc"] = np.where(used[:, None], h, np.nan).astype(dt)
    Cb = flush(C32, ftz).astype(dt)
    with np.errstate(all="ignore"):
        o = blend(h, Cb, bt["L"][:, None], dt, diff32, ftz)
    res["out"] = np.where(used[:, None], flush(o, ftz), C).astype(dt)
    res["M"] = M
    return res


def layer_reach(bt, src, history, channels, count=1):
    """M of every value of a layer: the largest finite |value| among its src and the history taps the beauty used, per plane and pixel
    (count, N)."""
    N = len(bt["used"])
    X = np.abs(np.asarray(src, np.float32).reshape(count, N, channels).astype(np.float64))
    M = np.where(np.isfinite(X), X, 0).max(-1)
    if history is None:
        return M
    Hh = np.abs(np.asarray(history, np.float32).reshape(count, N, channels).astype(np.float64))
    Hh = np.where(np.isfinite(Hh), Hh, 0).max(-1)
    for k in range(4):
        t = bt["taps"][:, k]
        M = np.maximum(M, np.where(t >= 0, Hh[:, np.maximum(t, 0)], 0))
    return M


def tolerance(M, rtol=RTOL, atol=ATOL):
    """The bound atol + rtol M on |device - restatement|: a weighted mean is off by a share of the values it averages, so the bound scales
    with the largest of them, not with the result (which may cancel)."""
    return atol + rtol * np.asarray(M, np.float64)


def compare(got, want, src, copied, M, rtol=RTOL):
    """Every value of a device result `got` against the restatement's `want` for the input `src` (all (N, C) or (N,)): a row in `copied`
    equals its input bit for bit, non-finite values match in kind (want taken to float32, as the device stores it), and every finite value
    is within tolerance(M).  -> (list of failures, stats: the largest |d| / bound, the largest |d| / (atol + M), the share of rows equal to
    the restatement bit for bit, the number of copied rows)."""
    x2 = lambda a, t: np.asarray(a, t)[:, None] if np.ndim(a) == 1 else np.asarray(a, t)
    with np.errstate(all="ignore"):
        g, s, w = x2(got, np.float32), x2(src, np.float32), x2(want, np.float64)
        w32 = w.astype(np.float32)
    M = np.asarray(M, np.float64)
    bound = tolerance(M, rtol)
    fails = []
    bad = copied & ~(g.view(np.uint32) == s.view(np.uint32)).all(-1)
    if bad.any():
        p = np.flatnonzero(bad)[0]
        fails.append(f"{int(bad.sum())} pixels without history differ from their input, first {p}: {g[p]} vs {s[p]}")
    bad = ~copied & (kind(g) != kind(w32)).any(-1)
    if bad.any():
        p = np.flatnonzero(bad)[0]
        fails.append(f"{int(bad.sum())} pixels differ in kind (NaN / +inf / -inf), first {p}: {g[p]} vs {w[p]}")
    both = np.isfinite(g) & np.isfinite(w32)
    with np.errstate(all="ignore"):
        d = np.where(both, np.abs(g.astype(np.float64) - w), 0.0).max(-1)
    bad = ~copied & (d > bound)
    if bad.any():
        p = int(np.argmax(np.where(bad, d / bound, 0)))
        fails.append(f"{int(bad.sum())} pixels outside {ATOL} + {rtol} M, worst {p}: {g[p]} vs {w[p]} (M {M[p]:.4g})")
    stats = {"worst": float((d / bound).max(initial=0)), "ratio": float((np.where(copied, 0, d) / (ATOL + M)).max(initial=0)),
             "bit_equal": float((g.view(np.uint32) == w32.view(np.uint32)).all(-1).mean()), "copied": int(copied.sum())}
    return fails, stats


def display_words(rgb, exposure_scale=1.0):
    """k_resolve's display words (ACES fit, exposure, gamma 2.2, 0xffRRGGBB) of an (..., 3) frame in float32 -> uint32, for every value:
    fmaxf(NaN, 0) = 0 and fminf(NaN, 1) = 1, as on the device, so a NaN channel packs 0 and an infinite one 255."""
    with np.errstate(all="ignore"):
        v = np.asarray(rgb, np.float32) @ D.ACES_IN.T
        a = v * (v + np.float32(0.0245786)) - np.float32(0.000090537)
        b = v * (np.float32(0.983729) * v + np.float32(0.4329510)) + np.float32(0.238081)
        val = ((a / b) @ D.ACES_OUT.T) * np.float32(exposure_scale)
        ch = (255.0 * np.fmin(np.power(np.fmax(val, np.float32(0)), np.float32(1.0 / 2.2)), np.float32(1))).astype(np.uint32)
    return np.uint32(0xff000000) | (ch[..., 0] << 16) | (ch[..., 1] << 8) | ch[..., 2]


def temporal_loop(W, H, color, vectors, cam_a, cam_b, history=None, history_len=None, max_history=16, clip_sigma=np.inf, dt=np.float64,
                  motion_dt=None, footprint_dt=None):
    """temporal() pixel by pixel, without the diff32 / clip32 / ftz decisions: the form the vectorised one is checked against"""
    N = W * H
    C = np.asarray(color, np.float32).reshape(N, 3).astype(dt)
    out, L = C.copy(), np.ones(N, dt)
    used = np.zeros(N, bool)
    hf, hcl = np.full((N, 3), np.nan, dt), np.full((N, 3), np.nan, dt)
    res = dict(out=out, L=L, used=used, h=hf, hc=hcl)
    if history is None:
        return res
    Hh = np.asarray(history, np.float32).reshape(N, 3).astype(dt)
    Lh = np.asarray(history_len, np.float32).reshape(N)
    fma, mul = _ops(dt)
    v, ok = pixel_motion(W, H, vectors, cam_a, cam_b, motion_dt or dt)
    v = v.astype(dt)
    cfin = np.isfinite(C).all(1)
    hfin = np.isfinite(Hh).all(1)
    y, x = np.divmod(np.arange(N), W)
    fdt = footprint_dt or dt
    fmul = _ops(fdt)[1]
    for p in np.flatnonzero(ok & cfin & np.isfinite(v).all(1)):
        qx, qy = fdt(fdt(x[p]) + fdt(0.5)) + fdt(v[p, 0]), fdt(fdt(y[p]) + fdt(0.5)) + fdt(v[p, 1])
        if not (0 <= qx <= W and 0 <= qy <= H):
            continue
        px, py = fdt(qx - fdt(0.5)), fdt(qy - fdt(0.5))
        x0, y0 = np.floor(px), np.floor(py)
        fx, fy = fdt(px - x0), fdt(py - y0)
        sw, sh, lmin = fdt(0), np.zeros(3, dt), None
        for j in (0, 1):
            for i in (0, 1):
                tx, ty = int(x0) + i, int(y0) + j
                w = fmul(fx if i else fdt(fdt(1) - fx), fy if j else fdt(fdt(1) - fy))
                if not w > 0 or tx < 0 or ty < 0 or tx >= W or ty >= H:
                    continue
                t = ty * W + tx
                if not hfin[t]:
                    continue
                lmin = Lh[t] if lmin is None else np.fmin(lmin, Lh[t])     # fminf: a NaN length is ignored
                sw = fdt(sw + w)
                sh = np.array([fma(dt(w), Hh[t, c], sh[c]) for c in range(3)], dt)
        if not sw > 0:
            continue
        h = (sh / dt(sw)).astype(dt)
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
            h = np.fmin(np.fmax(h, (mu - r).astype(dt)), (mu + r).astype(dt))
        hcl[p] = h
        Ln = dt(np.fmin(F32(F32(lmin) + F32(1)), F32(max_history)))     # in float32; NaN L_hist: max_history
        with np.errstate(all="ignore"):
            out[p] = (h + (C[p] - h) / Ln).astype(dt)
        L[p] = Ln
        used[p] = True
    return res
