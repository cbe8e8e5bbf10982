"""The denoiser without a GPU: the NumPy restatement of vpt_denoise (tests/denoise_ref.py) on synthetic frames, its float32 rules (the
flush to zero and the float32 luminance difference), its pass rule, and the host-only parts of the C entry points."""
import ctypes as C

import numpy as np
import pytest

import denoise_ref as D


def grey(a):
    """(H, W) -> (H, W, 3) with r = g = b, so Y equals the value (the luminance weights sum to 1)."""
    return np.repeat(np.asarray(a, np.float32)[..., None], 3, axis=-1)


def noisy_ramp(h, w, seed, noise=0.1):
    """A tinted ramp along x and y with `noise` relative Gaussian noise per channel -> (colour, depth, error map), float32."""
    rng = np.random.RandomState(seed)
    x = np.arange(w)[None, :] / max(w - 1, 1); y = np.arange(h)[:, None] / max(h - 1, 1)
    base = 0.5 + 1.0 * x + 0.5 * y
    c = (base[..., None] * np.array([0.8, 1.0, 1.2]) * (1 + noise * rng.randn(h, w, 3))).astype(np.float32)
    z = (2 + 3 * x + 0.5 * y + 0.05 * rng.randn(h, w)).astype(np.float32)
    err = (noise * (0.5 + rng.rand(h, w))).astype(np.float32)
    return c, z, err


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


def test_a_denormal_variance_is_flushed_and_its_window_copied():
    """err = 1e-20 at Y ~ 0.5 gives v ~ 2.5e-41, a float32 denormal the device flushes to 0: a pixel whose whole 3x3 window is like that
    has g == 0 and is copied.  Without the flush the restatement filters it."""
    rng = np.random.RandomState(11)
    c = grey(0.5 + 0.01 * rng.rand(3, 3))
    err = np.full((3, 3), 1e-20, np.float32)
    assert (D.noise_variance(c, err) == 0).all()
    assert 0 < D.noise_variance(c, err, ftz=False).min() < D.FLT_MIN
    out, copied = D.denoise_and_copies(c, rel_error=err)
    assert copied.all() and np.array_equal(out.view(np.uint32), c.view(np.uint32))
    out64, copied64 = D.denoise_and_copies(c, rel_error=err, ftz=False)
    assert not copied64.any()
    # one normal v in the window: every pixel next to it is filtered again
    err[1, 1] = 0.05
    assert not D.copied_pixels(c, rel_error=err).any()
    assert D.flush(np.array([1e-40, -1e-40, 2e-38, np.nan, -np.inf], np.float32)).tolist()[:3] == [0.0, 0.0, np.float32(2e-38)]
    assert np.signbit(D.flush(np.float32(-1e-40)))


def test_the_luminance_difference_overflows_in_float32():
    """Grey +-3e38 side by side in a 5x1 frame with an infinite error map: g = inf makes inv_l 0, |Y_p - Y_q| is inf in float32, and
    inf * 0 = NaN drops the tap, so each sign averages only with itself.  In float64 the difference is finite and every tap weighs 1."""
    c = grey(np.array([[3e38, 3e38, -3e38, -3e38, 3e38]], np.float32))
    err = np.full((1, 5), np.inf, np.float32)
    out = D.denoise(c, rel_error=err, iterations=1)[0, :, 0]
    assert np.isinf(D.noise_variance(c, err)).all()
    assert (np.sign(out) == np.sign(c[0, :, 0])).all() and (np.abs(out) > 2.9e38).all(), out
    mixed = D.denoise(c, rel_error=err, iterations=1, ftz=False)[0, :, 0]   # the float32 difference in either mode
    assert np.array_equal(mixed, out)
    # the same frame at 1e37: no overflow, every tap weighs 1, so the two signs mix
    small = D.denoise(c * np.float32(1 / 30), rel_error=err, iterations=1)[0, :, 0]
    assert abs(small[1]) < 1e37 and abs(small[2]) < 1e37


def test_an_infinite_variance_behind_a_tiny_tap_weight_turns_nan():
    """A tap whose h w squares below 2^-126 weighs 0 in the variance on the device; against an infinite v that is 0 * inf = NaN, and a
    pixel whose g sees a NaN v is copied.  Pixel 6 (Y 2, finite g, inv_l 12.5) reaches pixel 8 (Y 7, v = inf) with e = 62.5."""
    c = grey(np.array([[2.0] * 8 + [7.0]], np.float32))
    err = np.array([[0.01] * 8 + [np.inf]], np.float32)
    v, ok = D.noise_variance(c, err), D.finite_pixels(c)
    filt, taps = D.level_taps(v, D.luminance(c), np.zeros(v.shape, np.float32), ok, 1, 4.0, 0.2, False)
    hw = {dx: t[0, 6] for dy, dx, t, _ in taps if dy == 0}
    assert D.FLT_MIN < hw[2] and hw[2] ** 2 < D.FLT_MIN, hw
    v1, v1_64 = D.next_variance(v, filt, taps), D.next_variance(v, filt, taps, ftz=False)
    assert np.isnan(v1[0, 6]) and np.isinf(v1_64[0, 6])
    assert np.isinf(v1[0, 7]) and np.isinf(v1[0, 8]) and np.isfinite(v1[0, :6]).all()
    # at the next level every pixel whose 3x3 window holds that NaN is copied
    nxt = list(D.filter_levels(c, rel_error=err, iterations=2))[1][1]
    assert not nxt[0, 5:8].any() and nxt[0, :4].all()


@pytest.mark.parametrize("option", ["iterations", "sigma_luminance", "sigma_depth"])
def test_every_option_changes_the_output_on_a_noisy_ramp(option):
    """Each value the GPU tests give an option moves the restatement's output away from the default-option output by far more than the
    GPU tolerance, so an option the device ignored could not pass them."""
    values = {"iterations": (1, 2, 3, 6, 10), "sigma_luminance": (0.25, 64.0), "sigma_depth": (0.01, 5.0)}[option]
    for w, h in ((67, 45), (1100, 7), (1, 300), (300, 1)):
        c, z, err = noisy_ramp(h, w, 1)
        base = D.denoise(c, z, err)
        for v in values:
            out = D.denoise(c, z, err, **{option: v})
            moved = float((np.abs(out.astype(np.float64) - base).max(axis=-1) / D.tolerance(c, max(5, v if option == "iterations" else 5), 1e-4)).max())
            assert moved > 5, (w, h, option, v, moved)


def test_the_pass_rule():
    """compare(): the bound scales with the largest input value within reach, copied pixels must be bit for bit, kinds must match."""
    c, z, err = noisy_ramp(9, 40, 2)
    assert D.reach_max(c, 1).shape == (9, 40)
    spike = np.zeros((9, 40), np.float32); spike[4, 20] = 100.0; spike[0, 0] = np.nan
    M = D.reach_max(spike, 2)                                        # reach 6
    assert M[4, 26] == 100 and M[4, 27] == 0 and M[0, 0] == 0 and M[0, 14] == 100
    want, copied = D.denoise_and_copies(c, z, err)
    assert not copied.any()
    fails, stats = D.compare(want, want, c, copied, 5, 1e-4)
    assert not fails and stats["worst"] == 0 and stats["bit_equal"] == 1
    got = want.copy(); got[3, 7, 1] += np.float32(1e-3)                 # M ~ 2.2: 1e-3 is ~4x the bound
    fails, stats = D.compare(got, want, c, copied, 5, 1e-4)
    assert len(fails) == 1 and "outside" in fails[0] and 3 < stats["worst"] < 6
    got = want.copy(); got[0, 0, 2] = np.inf
    assert "kind" in D.compare(got, want, c, copied, 5, 1e-4)[0][0]
    cp = copied.copy(); cp[5, 5] = True                               # a copied pixel must equal its input, not the restatement
    assert "copied" in D.compare(want, want, c, cp, 5, 1e-4)[0][0]
