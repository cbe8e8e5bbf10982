"""NumPy restatement of vpt_denoise_layers (include/vpt_b200.h), for the tests: the beauty as tests/denoise_ref.py filters it, and every
layer filtered at every level with the beauty's weights of that level,

    x' = sum(h w x_q) / sum(h w)

over the same taps, with the same copy rule (a pixel the beauty copies keeps its layer values).  Each level is evaluated in float64 and
stored in float32, as the device keeps its planes.
"""
import numpy as np

from denoise_ref import B3, G3, finite_pixels, luminance, noise_variance, shifted


def level_weights(v, Y, z, ok, step, sigma_l, sigma_z, use_depth):
    """The beauty's weights of one level: (filt, [(dy, dx, hw)]) with hw 0 where the tap is not used."""
    h, w = v.shape
    gs = np.zeros((h, w)); gw = np.zeros((h, w))
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            v2, m = shifted(v.astype(np.float64), dy, dx, 0.0)
            k = G3[dy + 1] * G3[dx + 1]
            gs += np.where(m, k * v2, 0.0); gw += np.where(m, k, 0.0)
    g = gs / gw
    filt = ok & (g > 0)
    taps = []
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        inv_l = 1.0 / (sigma_l * np.sqrt(g) + 1e-10)
        Yp = Y.astype(np.float64); zp = z.astype(np.float64)
        for j in range(5):
            for i in range(5):
                dy, dx = (j - 2) * step, (i - 2) * step
                Yq, m = shifted(Yp, dy, dx, np.nan)
                zq, _ = shifted(zp, dy, dx, 0.0)
                if dy == 0 and dx == 0:
                    wq = np.ones((h, w))
                else:
                    e = np.abs(Yp - Yq) * inv_l
                    if use_depth:
                        e = e + np.abs(zp - zq) / (sigma_z * np.maximum(np.abs(zp), np.abs(zq)) + 1e-6)
                    wq = np.where(m & np.isfinite(Yq), np.exp(-e), 0.0)
                hw = B3[j] * B3[i] * wq
                use = filt & m & (hw > 0)
                taps.append((dy, dx, np.where(use, hw, 0.0), use))
    return filt, taps


def apply_level(x, filt, taps):
    """One level of an (H, W, C) float32 plane with the beauty's weights -> float32."""
    x64 = x.astype(np.float64)
    sw = np.zeros(x.shape[:2]); sx = np.zeros(x.shape)
    with np.errstate(over="ignore", invalid="ignore"):
        for dy, dx, hw, use in taps:
            xq, _ = shifted(x64, dy, dx, 0.0)
            sw += hw; sx += hw[..., None] * np.where(use[..., None], xq, 0.0)
        return np.where(filt[..., None], sx / np.where(filt, sw, 1.0)[..., None], x).astype(np.float32)


def denoise_layers(color, layers, depth=None, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2):
    """(H, W, 3) frame and a list of (H, W, C) or (H, W) float32 layers -> (denoised frame, [denoised layers]) in float32."""
    c = np.array(color, np.float32, copy=True)
    ok = finite_pixels(c)
    v = noise_variance(c, rel_error)
    with np.errstate(over="ignore", invalid="ignore"):
        Y = np.where(ok, luminance(c), np.float32(np.nan)).astype(np.float32)
    z = np.zeros(v.shape, np.float32) if depth is None else np.asarray(depth, np.float32)
    flat = [np.asarray(x, np.float32) for x in layers]
    xs = [x[..., None] if x.ndim == 2 else x.copy() for x in flat]
    for i in range(iterations):
        filt, taps = level_weights(v, Y, z, ok, 1 << i, sigma_luminance, sigma_depth, depth is not None)
        xs = [apply_level(x, filt, taps) for x in xs]
        c = apply_level(c, filt, taps)
        sw = sum(t[2] for t in taps)
        sv = np.zeros(v.shape)
        for dy, dx, hw, use in taps:
            vq, _ = shifted(v.astype(np.float64), dy, dx, 0.0)
            sv += np.where(use, hw * hw * vq, 0.0)
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            v = np.where(filt, sv / np.where(filt, sw, 1.0) ** 2, v).astype(np.float32)
        Y = np.where(filt, luminance(c), Y).astype(np.float32)
    return c, [x[..., 0] if f.ndim == 2 else x for x, f in zip(xs, flat)]
