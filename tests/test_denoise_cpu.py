"""The denoiser without a GPU: the NumPy restatement of vpt_denoise (tests/denoise_ref.py) on synthetic frames, and the host-only parts
of the C entry points."""
import ctypes as C

import numpy as np

import denoise_ref as D


def grey(a):
    """(H, W) -> (H, W, 3) with r = g = b, so Y equals the value (the luminance weights sum to 1)."""
    return np.repeat(np.asarray(a, np.float32)[..., None], 3, axis=-1)


def test_zero_error_map_is_the_identity_bit_for_bit():
    rng = np.random.RandomState(0)
    c = (rng.rand(23, 31, 3) * 4).astype(np.float32)
    z = (rng.rand(23, 31) * 10).astype(np.float32)
    out = D.denoise(c, depth=z, rel_error=np.zeros((23, 31), np.float32))
    assert out.dtype == np.float32 and np.array_equal(out.view(np.uint32), c.view(np.uint32))


def test_constant_image_stays_within_two_ulp():
    c = np.full((40, 37, 3), 0.7311, np.float32)
    c[..., 1] = 1.25; c[..., 2] = 0.0625
    out = D.denoise(c, rel_error=np.full((40, 37), 0.05, np.float32))
    ulp = np.spacing(c)
    assert (np.abs(out - c) <= 2 * ulp).all(), float(np.max(np.abs(out - c) / ulp))
    spatial = D.denoise(c + np.float32(0))            # a constant frame has spatial variance 0: copied
    assert np.array_equal(spatial, c)


def step_frame(sigma=0.05, lo=1.0, h=64, w=64, seed=3):
    hi = lo + 20 * sigma
    truth = np.where(np.arange(w)[None, :] < w // 2, lo, hi) * np.ones((h, 1))
    noisy = (truth + sigma * np.random.RandomState(seed).randn(h, w)).astype(np.float32)
    err = (sigma / np.maximum(noisy.astype(np.float64), D.MEAN_FLOOR)).astype(np.float32)   # v = sigma^2 for every pixel
    return truth, noisy, err, lo, hi


def test_step_edge_noise_drops_and_the_edge_stays_sharp():
    sigma = 0.05
    truth, noisy, err, lo, hi = step_frame(sigma)
    out = D.denoise(grey(noisy), rel_error=err)[..., 0].astype(np.float64)
    w = truth.shape[1]
    inner = np.ones(w, bool); inner[w // 2 - 4:w // 2 + 4] = False                     # the regions, away from the edge
    rmse_in = np.sqrt(np.mean((noisy[:, inner] - truth[:, inner]) ** 2))
    rmse_out = np.sqrt(np.mean((out[:, inner] - truth[:, inner]) ** 2))
    print(f"RMSE inside the regions: {rmse_in:.4f} -> {rmse_out:.4f} ({rmse_in / rmse_out:.1f}x)")
    assert rmse_in / rmse_out >= 3.0
    left = out[:, w // 2 - 2:w // 2].mean(); right = out[:, w // 2:w // 2 + 2].mean()
    assert abs(left - lo) <= 0.5 * sigma and abs(right - hi) <= 0.5 * sigma, (left, right)


def test_spatial_estimate_smooths_more_at_the_edge():
    """Without an error map the 5x5 variance at the edge includes the step itself, so the edge leaks more than with the error map
    (about 2 sigma here), but stays far closer to its own level than to the other side's."""
    sigma = 0.05
    truth, noisy, _, lo, hi = step_frame(sigma, seed=5)
    out = D.denoise(grey(noisy))[..., 0].astype(np.float64)
    w = truth.shape[1]
    inner = np.ones(w, bool); inner[w // 2 - 4:w // 2 + 4] = False
    assert np.sqrt(np.mean((out[:, inner] - truth[:, inner]) ** 2)) * 3 <= np.sqrt(np.mean((noisy[:, inner] - truth[:, inner]) ** 2))
    assert abs(out[:, w // 2 - 2:w // 2].mean() - lo) <= 5 * sigma and abs(out[:, w // 2:w // 2 + 2].mean() - hi) <= 5 * sigma


def test_a_nan_pixel_is_copied_and_does_not_leak():
    rng = np.random.RandomState(7)
    c = (1.0 + 0.05 * rng.randn(20, 20, 3)).astype(np.float32)
    c[9, 11, 1] = np.nan
    c[3, 4, 0] = np.inf
    err = np.full((20, 20), 0.05, np.float32)
    for rel in (err, None):
        out = D.denoise(c, depth=np.ones((20, 20), np.float32), rel_error=rel)
        assert np.array_equal(out[9, 11].view(np.uint32), c[9, 11].view(np.uint32))
        assert np.array_equal(out[3, 4].view(np.uint32), c[3, 4].view(np.uint32))
        others = np.ones((20, 20), bool); others[9, 11] = others[3, 4] = False
        assert np.isfinite(out[others]).all()
        assert not np.array_equal(out[others], c[others])                          # the rest was filtered


def test_error_map_edge_cases_give_the_documented_variance():
    c = grey(np.array([[0.5, 2.0, 1e-5, 1.0, 1.0]], np.float32))
    err = np.array([[0.1, np.nan, 0.2, -1.0, np.inf]], np.float32)
    v = D.noise_variance(c, err)
    assert np.allclose(v[0, :3], [(0.1 * 0.5) ** 2, 0.0, (0.2 * 1e-3) ** 2], rtol=1e-6)
    assert v[0, 3] == 0 and np.isinf(v[0, 4])


def test_depth_term_stops_at_a_depth_edge():
    """Same luminance statistics on both sides, different depth: with depth the two sides stay apart."""
    sigma = 0.05
    truth, noisy, err, lo, hi = step_frame(sigma, seed=9)
    z = np.where(np.arange(64)[None, :] < 32, 2.0, 10.0) * np.ones((64, 1), np.float32)
    with_z = D.denoise(grey(noisy), depth=z, rel_error=err, sigma_luminance=1e6)[..., 0]   # luminance term off
    without = D.denoise(grey(noisy), rel_error=err, sigma_luminance=1e6)[..., 0]
    edge = lambda o: max(abs(float(o[:, 30:32].mean()) - lo), abs(float(o[:, 32:34].mean()) - hi))
    assert edge(with_z) <= 0.5 * sigma and edge(without) >= 5 * sigma


def test_display_words_restatement_matches_a_hand_value():
    assert D.display_words(np.zeros(3, np.float32)) == 0xff000000
    w = int(D.display_words(np.full(3, 1e6, np.float32)))
    assert w == 0xffffffff


def test_options_defaults_and_null_context_fail_loudly():
    from vpt_b200 import _native as N
    o = N.denoise_options(0, 0.0, 0.0)
    N.lib.vpt_denoise_options_defaults(C.byref(o))
    assert o.iterations == 5 and abs(o.sigma_luminance - 4.0) < 1e-9 and abs(o.sigma_depth - 0.2) < 1e-7
    assert C.sizeof(N.denoise_options) == 12
    rc = N.lib.vpt_denoise(None, 4, 4, C.c_void_p(16), None, None, None, 1.0, C.c_void_p(64), None, None)
    assert rc == -1 and b"vpt_denoise" in N.lib.vpt_last_error(None)
