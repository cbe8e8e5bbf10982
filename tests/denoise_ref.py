"""NumPy restatement of vpt_denoise (include/vpt_b200.h), for the tests.

Y = 0.2126 r + 0.7152 g + 0.0722 b.  The noise variance of each pixel's mean luminance is

    v = (err * max(Y, 1e-3))^2          with vpt_render_adaptive's error map (err NaN or <= 0 -> 0, +inf -> +inf), or
    v = population variance of Y over the 5x5 window (clipped at the frame edge, finite pixels only) without it.

Level i (step s = 2^i): g = 3x3 Gaussian (1/4, 1/2, 1/4)^2 of v, renormalised over the taps inside the frame.  A pixel with g == 0, or
whose colour or luminance is not finite, is copied.  Otherwise the taps q at s * (-2..2)^2 inside the frame, with B3-spline weights h,
weigh w = exp(-|Y_p - Y_q| / (sigma_l sqrt(g) + 1e-10) - |z_p - z_q| / (sigma_z max(|z_p|, |z_q|) + 1e-6)) (the centre exactly 1, a
non-finite neighbour 0; a tap whose h w is not > 0 drops out), and

    c' = sum(h w c_q) / sum(h w),   v' = sum((h w)^2 v_q) / sum(h w)^2.

Each level is evaluated in float64 and stored in float32, as the device keeps its planes, except where float32 decides the outcome:
|Y_p - Y_q| is formed in float32 (inf for luminances near FLT_MAX of opposite sign), and with ftz (the default) the values the device's
--use_fast_math arithmetic flushes to zero are flushed here too: v, the stored planes of each level, g's partial sums, and h w and
(h w)^2 below 2^-126.  Without ftz every level is float64 throughout, which filters pixels whose 3x3 window of v is all denormal.

compare() is the pass rule of the GPU tests: copied pixels bit for bit, non-finite values in kind, and every finite value within
1e-5 + R M, with M the largest finite |value| of the input within the filter's reach of the pixel (tolerance()).
"""
import numpy as np
from scipy.ndimage import maximum_filter

MEAN_FLOOR = 1e-3
FLT_MIN = 2.0 ** -126          # the smallest normal float32: the device flushes anything smaller to 0
ATOL = 1e-5
RTOL = 1e-4                    # R of the GPU tests' bound 1e-5 + R M (see compare())
LUMA = (0.2126, 0.7152, 0.0722)
B3 = (1 / 16, 1 / 4, 3 / 8, 1 / 4, 1 / 16)
G3 = (0.25, 0.5, 0.25)
ACES_IN = np.array([0.59719, 0.35458, 0.04823, 0.07600, 0.90834, 0.01566, 0.02840, 0.13383, 0.83777], np.float32).reshape(3, 3)
ACES_OUT = np.array([1.60475, -0.53108, -0.07367, -0.10208, 1.10813, -0.00605, -0.00327, -0.07276, 1.07602], np.float32).reshape(3, 3)


def luminance(rgb):
    """(..., 3) -> (...) in float32, the device's arithmetic type."""
    rgb = np.asarray(rgb, np.float32)
    w = [np.float32(c) for c in LUMA]
    return w[0] * rgb[..., 0] + w[1] * rgb[..., 1] + w[2] * rgb[..., 2]


def shifted(a, dy, dx, fill):
    """b[y, x] = a[y + dy, x + dx], `fill` outside the frame; and the mask of taps inside it."""
    h, w = a.shape[:2]
    b = np.full_like(a, fill)
    m = np.zeros((h, w), bool)
    if abs(dy) >= h or abs(dx) >= w:
        return b, m
    ys, yd = (slice(dy, h), slice(0, h - dy)) if dy >= 0 else (slice(0, h + dy), slice(-dy, h))
    xs, xd = (slice(dx, w), slice(0, w - dx)) if dx >= 0 else (slice(0, w + dx), slice(-dx, w))
    b[yd, xd] = a[ys, xs]
    m[yd, xd] = True
    return b, m


def finite_pixels(color):
    c = np.asarray(color, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.isfinite(c).all(axis=-1) & np.isfinite(luminance(c))


def noise_variance(color, rel_error=None, ftz=True):
    """v of every pixel (float32, flushed with ftz: a v below 2^-126 is 0 on the device); 0 for non-finite pixels."""
    c = np.asarray(color, np.float32)
    ok = finite_pixels(c)
    with np.errstate(over="ignore", invalid="ignore"):
        Y = luminance(c).astype(np.float64)
    if rel_error is not None:
        e = np.asarray(rel_error, np.float32).astype(np.float64)
        with np.errstate(over="ignore", invalid="ignore"):
            v = np.where(e > 0, (e * np.maximum(Y, MEAN_FLOOR)) ** 2, 0.0)
    else:
        Yf = np.where(ok, Y, 0.0)
        s = np.zeros_like(Yf); n = np.zeros_like(Yf)
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                y2, m = shifted(Yf, dy, dx, 0.0); o2, _ = shifted(ok, dy, dx, False)
                use = m & o2
                s += np.where(use, y2, 0.0); n += use
        mean = s / np.maximum(n, 1)
        ss = np.zeros_like(Yf)
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                y2, m = shifted(Yf, dy, dx, 0.0); o2, _ = shifted(ok, dy, dx, False)
                ss += np.where(m & o2, (y2 - mean) ** 2, 0.0)
        v = ss / np.maximum(n, 1)
    with np.errstate(over="ignore"):
        return flush(np.where(ok, v, 0.0), ftz)


def flush(a, ftz=True):
    """float32 `a` with its denormals flushed to zero (keeping the sign), as the library's --use_fast_math arithmetic stores them."""
    a = np.asarray(a, np.float32)
    if not ftz:
        return a
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(a) < FLT_MIN, a * np.float32(0), a).astype(np.float32)


def gaussian_v(v, ftz=True):
    """g: the 3x3 Gaussian of v, renormalised over the taps inside the frame.  With ftz it is summed in float32 in the device's order, each
    partial sum rounded and flushed, so that g == 0 (the copy decision) is decided as on the device."""
    h, w = v.shape
    gs = np.zeros((h, w), np.float32 if ftz else np.float64); gw = np.zeros((h, w))
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            v2, m = shifted(v.astype(np.float64), dy, dx, 0.0)
            k = G3[dy + 1] * G3[dx + 1]
            with np.errstate(invalid="ignore"):
                s = gs.astype(np.float64) + k * v2
            gs = np.where(m, flush(s) if ftz else s, gs)
            gw += np.where(m, k, 0.0)
    return gs.astype(np.float64) / gw


def level_taps(v, Y, z, ok, step, sigma_l, sigma_z, use_depth, ftz=True):
    """The weights of one level: (filt, taps) with filt the pixels it filters and taps = [(dy, dx, hw, use)], hw 0 where the tap is not
    used.  |Y_p - Y_q| is formed in float32 as on the device, so luminances of opposite sign near FLT_MAX give inf (and inf * 0 = NaN
    drops the tap when g is infinite).  With ftz an h w below FLT_MIN drops out, as __expf and the product flush it on the device."""
    h, w = v.shape
    g = gaussian_v(v, ftz)
    filt = ok & (g > 0)
    taps = []
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        inv_l = 1.0 / (sigma_l * np.sqrt(g) + 1e-10)
        Y32 = np.asarray(Y, np.float32); zp = z.astype(np.float64)
        for j in range(5):
            for i in range(5):
                dy, dx = (j - 2) * step, (i - 2) * step
                Yq, m = shifted(Y32, dy, dx, np.float32(np.nan))
                zq, _ = shifted(zp, dy, dx, 0.0)
                if dy == 0 and dx == 0:
                    wq = np.ones((h, w))
                else:
                    e = np.abs(Y32 - Yq).astype(np.float64) * inv_l
                    if use_depth:
                        e = e + np.abs(zp - zq) / (sigma_z * np.maximum(np.abs(zp), np.abs(zq)) + 1e-6)
                    wq = np.where(m & np.isfinite(Yq), np.exp(-e), 0.0)
                hw = B3[j] * B3[i] * wq
                if ftz:
                    hw = np.where(hw < FLT_MIN, 0.0, hw)
                use = filt & m & (hw > 0)
                taps.append((dy, dx, np.where(use, hw, 0.0), use))
    return filt, taps


def apply_level(x, filt, taps, ftz=True):
    """x' = sum(h w x_q) / sum(h w) of an (H, W, C) float32 plane with one level's weights (a pixel not in filt keeps x) -> float32."""
    x64 = x.astype(np.float64)
    sw = np.zeros(x.shape[:2]); sx = np.zeros(x.shape)
    with np.errstate(over="ignore", invalid="ignore"):
        for dy, dx, hw, use in taps:
            xq, _ = shifted(x64, dy, dx, 0.0)
            sw += hw; sx += hw[..., None] * np.where(use[..., None], xq, 0.0)
        return flush(np.where(filt[..., None], sx / np.where(filt, sw, 1.0)[..., None], x), ftz)


def next_variance(v, filt, taps, ftz=True):
    """v' = sum((h w)^2 v_q) / sum(h w)^2 (a pixel not in filt keeps v) -> float32.  With ftz a (h w)^2 below FLT_MIN is 0, as the device
    squares h w in float32: against an infinite v_q that makes the sum NaN, and the pixels whose g then sees it are copied."""
    sw = np.zeros(v.shape); sv = np.zeros(v.shape)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        for dy, dx, hw, use in taps:
            vq, _ = shifted(v.astype(np.float64), dy, dx, 0.0)
            hw2 = hw * hw
            if ftz:
                hw2 = np.where(hw2 < FLT_MIN, 0.0, hw2)
            sw += hw; sv += np.where(use, hw2 * vq, 0.0)
        return flush(np.where(filt, sv / np.where(filt, sw, 1.0) ** 2, v), ftz)


def filter_levels(color, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, ftz=True):
    """The beauty level by level: yields (c, filt, taps) of each level, c its float32 output and (filt, taps) its weights."""
    c = np.array(color, np.float32, copy=True)
    ok = finite_pixels(c)
    v = noise_variance(c, rel_error, ftz)
    with np.errstate(over="ignore", invalid="ignore"):
        Y = flush(np.where(ok, luminance(c), np.float32(np.nan)), ftz)
    z = np.zeros(v.shape, np.float32) if depth is None else np.asarray(depth, np.float32)
    for i in range(iterations):
        filt, taps = level_taps(v, Y, z, ok, 1 << i, sigma_luminance, sigma_depth, depth is not None, ftz)
        c = apply_level(c, filt, taps, ftz)
        v = next_variance(v, filt, taps, ftz)
        with np.errstate(over="ignore", invalid="ignore"):
            Y = flush(np.where(filt, luminance(c), Y), ftz)
        yield c, filt, taps


def denoise_and_copies(color, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, ftz=True):
    """-> (the filtered (H, W, 3) float32 frame, the (H, W) mask of pixels every level copied: the device keeps those bit for bit)."""
    copied = np.ones(np.shape(color)[:2], bool)
    for c, filt, _ in filter_levels(color, depth, rel_error, iterations, sigma_luminance, sigma_depth, ftz):
        copied &= ~filt
    return c, copied


def denoise(color, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, ftz=True):
    """(H, W, 3) float32 frame -> the filtered (H, W, 3) float32 frame."""
    return denoise_and_copies(color, depth, rel_error, iterations, sigma_luminance, sigma_depth, ftz)[0]


def copied_pixels(color, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, ftz=True):
    """The (H, W) mask of pixels the restatement copies at every level."""
    return denoise_and_copies(color, depth, rel_error, iterations, sigma_luminance, sigma_depth, ftz)[1]


def reach_max(src, iterations):
    """M: the largest finite |value| of `src` ((H, W) or (H, W, C)) within the filter's total tap reach of each pixel, 2 (2^n - 1) in
    Chebyshev distance for n levels (0 where there is none)."""
    a = np.abs(np.asarray(src, np.float64))
    a = np.where(np.isfinite(a), a, 0.0)
    if a.ndim == 3:
        a = a.max(axis=-1)
    reach = 2 * ((1 << iterations) - 1)
    return maximum_filter(a, size=2 * reach + 1, mode="constant", cval=0.0)


def tolerance(src, iterations, rtol, atol=ATOL):
    """The bound atol + rtol M on |device - restatement| of each pixel.  A weighted mean can only be off by a share of the values it
    averages, so the bound scales with the largest of them, not with the result (which may cancel)."""
    return atol + rtol * reach_max(src, iterations)


def kind(a):
    """0 finite, 1 NaN, 2 +inf, 3 -inf."""
    a = np.asarray(a)
    return np.where(np.isnan(a), 1, np.where(a == np.inf, 2, np.where(a == -np.inf, 3, 0)))


def compare(got, want, src, copied, iterations, rtol):
    """Every pixel of a device result `got` against the restatement's `want` for the input `src` (all (H, W) or (H, W, C) float32):
    a pixel in `copied` equals its input bit for bit, non-finite values match in kind, and every finite value is within
    tolerance(src, ...).  -> (list of failures, stats: the largest |d| / bound, the largest |d| / (atol + M), the share of pixels equal
    to the restatement bit for bit, the number of copied pixels)."""
    x3 = lambda a: np.asarray(a, np.float32)[..., None] if np.ndim(a) == 2 else np.asarray(a, np.float32)
    g, w, s = x3(got), x3(want), x3(src)
    M = reach_max(s, iterations)
    bound = ATOL + rtol * M
    fails = []
    bad = copied & ~(g.view(np.uint32) == s.view(np.uint32)).all(axis=-1)
    if bad.any():
        fails.append(f"{int(bad.sum())} copied pixels moved, first at {tuple(np.argwhere(bad)[0])}")
    bad = ~copied & (kind(g) != kind(w)).any(axis=-1)
    if bad.any():
        y, x = np.argwhere(bad)[0]
        fails.append(f"{int(bad.sum())} pixels differ in kind (NaN / +inf / -inf), first at {(y, x)}: {g[y, x]} vs {w[y, x]}")
    both = np.isfinite(g) & np.isfinite(w)
    with np.errstate(over="ignore", invalid="ignore"):
        d = np.where(both, np.abs(g.astype(np.float64) - w.astype(np.float64)), 0.0).max(axis=-1)
    bad = ~copied & (d > bound)
    if bad.any():
        y, x = np.unravel_index(np.argmax(np.where(bad, d / bound, 0)), d.shape)
        fails.append(f"{int(bad.sum())} pixels outside {ATOL} + {rtol} M, worst at {(y, x)}: {g[y, x]} vs {w[y, x]} (M {M[y, x]:.4g})")
    stats = {"worst": float((d / bound).max()), "ratio": float((d / (ATOL + M)).max()),
             "bit_equal": float((g.view(np.uint32) == w.view(np.uint32)).all(axis=-1).mean()), "copied": int(copied.sum())}
    return fails, stats


def display_words(rgb, exposure_scale=1.0):
    """k_resolve's display words (ACES fit, exposure, gamma 2.2, 0xffRRGGBB) of an (..., 3) frame, in float32 -> uint32."""
    v = np.asarray(rgb, np.float32) @ ACES_IN.T
    a = v * (v + np.float32(0.0245786)) - np.float32(0.000090537)
    b = v * (np.float32(0.983729) * v + np.float32(0.4329510)) + np.float32(0.238081)
    val = ((a / b) @ ACES_OUT.T) * np.float32(exposure_scale)
    ch = (255.0 * np.minimum(np.power(np.maximum(val, 0.0), 1.0 / 2.2), 1.0)).astype(np.uint32)
    return np.uint32(0xff000000) | (ch[..., 0] << 16) | (ch[..., 1] << 8) | ch[..., 2]
