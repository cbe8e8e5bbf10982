"""NumPy restatement of vpt_denoise (include/vpt_b200.h), for the tests.

Y = 0.2126 r + 0.7152 g + 0.0722 b.  The noise variance of each pixel's mean luminance is

    v = (err * max(Y, 1e-3))^2          with vpt_render_adaptive's error map (err NaN or <= 0 -> 0, +inf -> +inf), or
    v = population variance of Y over the 5x5 window (clipped at the frame edge, finite pixels only) without it.

Level i (step s = 2^i): g = 3x3 Gaussian (1/4, 1/2, 1/4)^2 of v, renormalised over the taps inside the frame.  A pixel with g == 0, or
whose colour or luminance is not finite, is copied.  Otherwise the taps q at s * (-2..2)^2 inside the frame, with B3-spline weights h,
weigh w = exp(-|Y_p - Y_q| / (sigma_l sqrt(g) + 1e-10) - |z_p - z_q| / (sigma_z max(|z_p|, |z_q|) + 1e-6)) (the centre exactly 1, a
non-finite neighbour 0; a tap whose h w is not > 0 drops out), and

    c' = sum(h w c_q) / sum(h w),   v' = sum((h w)^2 v_q) / sum(h w)^2.

Each level is evaluated in float64 and stored in float32, as the device keeps its planes.
"""
import numpy as np

MEAN_FLOOR = 1e-3
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


def noise_variance(color, rel_error=None):
    """v of every pixel (float32); 0 for non-finite pixels."""
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
        return np.where(ok, v, 0.0).astype(np.float32)


def atrous_level(c, v, Y, z, ok, step, sigma_l, sigma_z, use_depth):
    """One level on float32 planes -> (c', v', Y') in float32."""
    h, w = v.shape
    gs = np.zeros((h, w)); gw = np.zeros((h, w))
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            v2, m = shifted(v.astype(np.float64), dy, dx, 0.0)
            k = G3[dy + 1] * G3[dx + 1]
            gs += np.where(m, k * v2, 0.0); gw += np.where(m, k, 0.0)
    g = gs / gw
    filt = ok & (g > 0)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        inv_l = 1.0 / (sigma_l * np.sqrt(g) + 1e-10)
        Yp = Y.astype(np.float64); zp = z.astype(np.float64)
        sw = np.zeros((h, w)); sc = np.zeros((h, w, 3)); sv = np.zeros((h, w))
        for j in range(5):
            for i in range(5):
                dy, dx = (j - 2) * step, (i - 2) * step
                Yq, m = shifted(Yp, dy, dx, np.nan)
                zq, _ = shifted(zp, dy, dx, 0.0)
                cq, _ = shifted(c.astype(np.float64), dy, dx, 0.0)
                vq, _ = shifted(v.astype(np.float64), dy, dx, 0.0)
                if dy == 0 and dx == 0:
                    wq = np.ones((h, w))
                else:
                    e = np.abs(Yp - Yq) * inv_l
                    if use_depth:
                        e = e + np.abs(zp - zq) / (sigma_z * np.maximum(np.abs(zp), np.abs(zq)) + 1e-6)
                    wq = np.where(m & np.isfinite(Yq), np.exp(-e), 0.0)
                hw = B3[j] * B3[i] * wq
                use = filt & m & (hw > 0)
                hw = np.where(use, hw, 0.0)
                sw += hw; sc += hw[..., None] * np.where(use[..., None], cq, 0.0); sv += np.where(use, hw * hw * vq, 0.0)
        c_new = np.where(filt[..., None], sc / np.where(filt, sw, 1.0)[..., None], c).astype(np.float32)
        v_new = np.where(filt, sv / np.where(filt, sw, 1.0) ** 2, v).astype(np.float32)
    Y_new = np.where(filt, luminance(c_new), Y).astype(np.float32)
    return c_new, v_new, Y_new


def denoise(color, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2):
    """(H, W, 3) float32 frame -> the filtered (H, W, 3) float32 frame."""
    c = np.array(color, np.float32, copy=True)
    ok = finite_pixels(c)
    v = noise_variance(c, rel_error)
    with np.errstate(over="ignore", invalid="ignore"):
        Y = np.where(ok, luminance(c), np.float32(np.nan)).astype(np.float32)
    z = np.zeros(v.shape, np.float32) if depth is None else np.asarray(depth, np.float32)
    for i in range(iterations):
        c, v, Y = atrous_level(c, v, Y, z, ok, 1 << i, sigma_luminance, sigma_depth, depth is not None)
    return c


def display_words(rgb, exposure_scale=1.0):
    """k_resolve's display words (ACES fit, exposure, gamma 2.2, 0xffRRGGBB) of an (..., 3) frame, in float32 -> uint32."""
    v = np.asarray(rgb, np.float32) @ ACES_IN.T
    a = v * (v + np.float32(0.0245786)) - np.float32(0.000090537)
    b = v * (np.float32(0.983729) * v + np.float32(0.4329510)) + np.float32(0.238081)
    val = ((a / b) @ ACES_OUT.T) * np.float32(exposure_scale)
    ch = (255.0 * np.minimum(np.power(np.maximum(val, 0.0), 1.0 / 2.2), 1.0)).astype(np.uint32)
    return np.uint32(0xff000000) | (ch[..., 0] << 16) | (ch[..., 1] << 8) | ch[..., 2]
