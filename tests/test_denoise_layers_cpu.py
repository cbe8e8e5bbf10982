"""Layer denoising without a GPU: the NumPy restatement of vpt_denoise_layers (tests/denoise_layers_ref.py) against vpt_denoise's
(tests/denoise_ref.py) on synthetic frames, the identities it keeps, and the host-only parts of the C entry point."""
import ctypes as C

import numpy as np

import denoise_ref as D
import denoise_layers_ref as DL


def frame(seed=0, h=29, w=37):
    rng = np.random.RandomState(seed)
    c = (0.5 + rng.rand(h, w, 3) * 2).astype(np.float32)
    z = (1 + rng.rand(h, w) * 10).astype(np.float32)
    err = (0.02 + 0.2 * rng.rand(h, w)).astype(np.float32)
    return rng, c, z, err


def test_a_layer_equal_to_the_colour_reproduces_the_denoiser_exactly():
    _, c, z, err = frame()
    for depth, rel in ((z, err), (None, err), (z, None), (None, None)):
        want = D.denoise(c, depth=depth, rel_error=rel)
        beauty, (same, r) = DL.denoise_layers(c, [c, c[..., 0]], depth=depth, rel_error=rel)
        assert np.array_equal(beauty.view(np.uint32), want.view(np.uint32))
        assert np.array_equal(same.view(np.uint32), want.view(np.uint32))
        assert np.array_equal(r.view(np.uint32), want[..., 0].view(np.uint32))


def test_the_filter_is_additive_to_float32_rounding():
    rng, c, z, err = frame(1)
    a = (rng.rand(*c.shape) * 3).astype(np.float32)
    b = (rng.rand(*c.shape) * 0.5).astype(np.float32)
    _, (fa, fb, fab) = DL.denoise_layers(c, [a, b, a + b], depth=z, rel_error=err)
    tol = 4 * np.spacing(np.abs(fab).astype(np.float32))
    assert (np.abs(fa.astype(np.float64) + fb - fab) <= tol).all()


def test_copied_pixels_keep_their_layers_bit_for_bit():
    rng, c, z, err = frame(2)
    c[5, 7, 1] = np.nan
    layer = (rng.rand(*c.shape[:2], 4) * 2).astype(np.float32)
    _, (out,) = DL.denoise_layers(c, [layer], depth=z, rel_error=err)
    assert np.array_equal(out[5, 7].view(np.uint32), layer[5, 7].view(np.uint32))
    others = np.ones(c.shape[:2], bool); others[5, 7] = False
    assert np.isfinite(out[others]).all() and not np.array_equal(out[others], layer[others])
    _, (zero,) = DL.denoise_layers(c, [layer], depth=z, rel_error=np.zeros(c.shape[:2], np.float32))   # g == 0 everywhere
    assert np.array_equal(zero.view(np.uint32), layer.view(np.uint32))


def test_an_alpha_in_the_unit_interval_stays_there():
    rng, c, z, err = frame(3)
    alpha = rng.rand(*c.shape[:2]).astype(np.float32)
    alpha[:, :5] = 1.0; alpha[:3] = 0.0
    _, (out,) = DL.denoise_layers(c, [alpha], depth=z, rel_error=err)
    ulp = np.spacing(np.float32(1.0))
    assert out.min() >= -4 * ulp and out.max() <= 1 + 4 * ulp


def test_null_context_fails_loudly():
    from vpt_b200 import _native as N
    assert C.sizeof(N.denoise_layer) == 24
    lay = (N.denoise_layer * 1)(N.denoise_layer(128, 256, 1, 1))
    rc = N.lib.vpt_denoise_layers(None, 4, 4, C.c_void_p(16), None, None, None, 1.0, C.c_void_p(64), None, lay, 1, None)
    assert rc == -1 and b"vpt_denoise_layers" in N.lib.vpt_last_error(None)
