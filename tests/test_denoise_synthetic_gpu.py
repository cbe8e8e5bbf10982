"""The denoiser and the layer denoiser on the GPU against the NumPy restatement (tests/denoise_ref.py, tests/denoise_layers_ref.py), on
synthetic frames passed in through the C ABI (vpt_denoise, vpt_denoise_layers): every value of every option on frames from 1x1 to the
65535-pixel width cap, non-finite and extreme colours, error maps and depths, every launch grouping of the layer planes, and one context
reused across frame sizes and plane counts.

Every pixel is checked (denoise_ref.compare): a pixel the restatement copies at every level equals its input bit for bit, non-finite
values match in kind, and every finite value is within 1e-5 + RTOL M, with M the largest finite |value| of the input within the
filter's reach of the pixel.  Display words are within 1 LSB of the packing of the device's own colour."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
import denoise_layers_ref as DL
import denoise_ref as D
from test_denoise_cpu import grey, noisy_ramp

pytestmark = pytest.mark.gpu
DEFAULTS = (5, 4.0, 0.2)
GUIDES = [("err+depth", True, True), ("err", True, False), ("depth", False, True), ("spatial", False, False)]
ITERATIONS, SIGMA_L, SIGMA_Z = (1, 2, 3, 6, 10), (0.25, 4.0, 64.0), (0.01, 0.2, 5.0)


def new_context():
    """A bare context: the denoiser needs no scene, and takes the frame size per call."""
    ctx = C.c_void_p(0)
    assert V.lib.vpt_create(C.byref(ctx)) == 0
    return ctx


@pytest.fixture(scope="module")
def ctx():
    c = new_context()
    yield c
    torch.cuda.synchronize()
    V.lib.vpt_destroy(c)


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def run_denoise(ctx, color, depth=None, err=None, opt=DEFAULTS, exposure=1.0):
    """vpt_denoise of NumPy inputs -> (colour, display words) in NumPy."""
    H, W = color.shape[:2]
    c, z, e = dev(color), dev(depth), dev(err)
    out = torch.empty(H, W, 3, dtype=torch.float32, device="cuda")
    words = torch.empty(H, W, dtype=torch.int32, device="cuda")
    rc = V.lib.vpt_denoise(ctx, W, H, ptr(c), ptr(z), ptr(e), C.byref(V._native.denoise_options(*opt)), exposure, ptr(out), ptr(words), None)
    assert rc == 0, V.lib.vpt_last_error(ctx).decode()
    torch.cuda.synchronize()
    return out.cpu().numpy(), words.cpu().numpy().view(np.uint32)


def run_layers(ctx, color, depth, err, layers, opt=DEFAULTS, exposure=1.0):
    """vpt_denoise_layers of NumPy inputs.  layers = [(src, channels, count, mode)]: src (count, H, W, channels) float32 or None for the
    colour itself; mode "out" (a new dst), "in" (dst == src).  -> (beauty, display words, [dst per layer]) in NumPy."""
    H, W = color.shape[:2]
    c, z, e = dev(color), dev(depth), dev(err)
    out = torch.empty(H, W, 3, dtype=torch.float32, device="cuda")
    words = torch.empty(H, W, dtype=torch.int32, device="cuda")
    srcs, keep, descs = [], [], []                  # srcs holds the sources until the call is done
    for src, ch, k, mode in layers:
        s = c if src is None else dev(src)
        d = s if mode == "in" else torch.empty(k * H * W * ch, dtype=torch.float32, device="cuda")
        srcs.append(s); keep.append(d)
        descs.append(V._native.denoise_layer(s.data_ptr(), d.data_ptr(), ch, k))
    arr = (V._native.denoise_layer * max(1, len(descs)))(*descs)
    rc = V.lib.vpt_denoise_layers(ctx, W, H, ptr(c), ptr(z), ptr(e), C.byref(V._native.denoise_options(*opt)), exposure, ptr(out),
                                  ptr(words), arr, len(descs), None)
    assert rc == 0, V.lib.vpt_last_error(ctx).decode()
    torch.cuda.synchronize()
    return out.cpu().numpy(), words.cpu().numpy().view(np.uint32), [d.cpu().numpy().reshape(k, H, W, ch) for d, (_, ch, k, _) in zip(keep, layers)]


def assert_display(label, got, words, exposure=1.0):
    """Display words within 1 LSB of the packing of the device's colour, where that colour is finite and small enough to tone-map."""
    fine = (np.isfinite(got) & (np.abs(got) < 1e15)).all(axis=-1)
    want = D.display_words(np.where(fine[..., None], got, 0), exposure)
    lsb = max(int(np.max(np.abs(((words >> s) & 0xff).astype(int) - ((want >> s) & 0xff).astype(int))[fine], initial=0)) for s in (0, 8, 16))
    assert lsb <= 1 and (words >> 24 == 0xff).all(), f"{label}: display words {lsb} LSB away"


def assert_matches(label, got, words, color, depth, err, opt, exposure=1.0):
    """The device's colour against the restatement, every pixel -> the device's colour."""
    want, copied = D.denoise_and_copies(color, depth, err, *opt)
    fails, st = D.compare(got, want, color, copied, opt[0], D.RTOL)
    print(f"{label}: worst |d|/bound {st['worst']:.3g}, |d|/(1e-5 + M) {st['ratio']:.3g}, {100 * st['bit_equal']:.2f} % bit-equal, "
          f"{st['copied']} copied")
    assert not fails, f"{label}: " + "; ".join(fails)
    assert_display(label, got, words, exposure)


def option_sets(gi):
    """Five option triples for guide setting gi: every value of each option appears once or more for each guide setting."""
    return [(ITERATIONS[k], SIGMA_L[(k + gi) % 3], SIGMA_Z[(k + 2 * gi) % 3]) for k in range(5)]


# ---- 1. the options ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wh", [(67, 45), (1, 300), (300, 1), (1100, 7), (1, 1)])
def test_every_option_value_against_the_restatement(ctx, wh):
    """1x300 and 300x1 have every step past the frame on one axis; 1100x7 at 10 levels has in-frame taps at +-512 and +-1024 along x."""
    W, H = wh
    color, depth, err = noisy_ramp(H, W, seed=W + 7 * H)
    for gi, (g, use_err, use_depth) in enumerate(GUIDES):
        z, e = depth if use_depth else None, err if use_err else None
        for opt in option_sets(gi):
            got, words = run_denoise(ctx, color, z, e, opt)
            assert_matches(f"{W}x{H} {g} {opt}", got, words, color, z, e, opt)


@pytest.mark.parametrize("wh", [(67, 45), (1, 300), (300, 1), (1100, 7)])
def test_every_option_moves_the_device_output(ctx, wh):
    """Each non-default value of each option, the others at their defaults, changes the device's output and matches the restatement:
    an option the host ignored, or two sigmas swapped, cannot pass."""
    W, H = wh
    color, depth, err = noisy_ramp(H, W, seed=3 * W + H)
    base, _ = run_denoise(ctx, color, depth, err, DEFAULTS)
    changes = [(k, v) for k, vals in enumerate((ITERATIONS, SIGMA_L, SIGMA_Z)) for v in vals if v != DEFAULTS[k]]
    for k, v in changes:
        opt = tuple(v if m == k else DEFAULTS[m] for m in range(3))
        got, words = run_denoise(ctx, color, depth, err, opt)
        assert not np.array_equal(got, base), f"{W}x{H}: {opt} gives the default options' output"
        assert_matches(f"{W}x{H} err+depth {opt}", got, words, color, depth, err, opt)


def test_the_width_cap(ctx):
    """65535x2 at 10 levels: taps at up to +-1024 along x, every step past the frame along y."""
    W, H = 65535, 2
    color, depth, err = noisy_ramp(H, W, seed=5)
    for opt, z, e in (((10, 64.0, 5.0), depth, err), ((10, 4.0, 0.2), None, None)):
        got, words = run_denoise(ctx, color, z, e, opt)
        assert_matches(f"{W}x{H} {'err+depth' if z is not None else 'spatial'} {opt}", got, words, color, z, e, opt)


# ---- 2. non-finite and extreme inputs ------------------------------------------------------------------------------------------------

def hostile_frame(h, w, seed, extreme):
    """A noisy ramp with a step, then: NaN / +inf / -inf in single channels of ~3 % of the pixels and in clusters on the corners and
    edges; moderate negative colours; an error map holding NaN, -1, 0, +inf, 1e20 and 1e-20 (scattered where Y < 1, and a 5x5 block:
    v is a float32 denormal there, 0 on the device); a depth holding 0, negative values, NaN, +inf and a sharp edge; and with `extreme` a
    3x3 block of grey +-3e38 (checkerboard signs) whose error map is +inf."""
    rng = np.random.RandomState(seed)
    c, z, err = noisy_ramp(h, w, seed)
    c[:, 2 * w // 3:] *= np.float32(4)                                                    # a luminance step
    pick = lambda frac: rng.rand(h, w) < frac
    neg = pick(0.03)
    c[neg, rng.randint(0, 3)] = -(0.05 + 0.5 * rng.rand(int(neg.sum()))).astype(np.float32)
    for val, frac in ((np.nan, 0.012), (np.inf, 0.009), (-np.inf, 0.009)):
        m = np.argwhere(pick(frac))
        c[m[:, 0], m[:, 1], rng.randint(0, 3, len(m))] = val
    for (y, x), val in zip(((0, 0), (0, w - 2), (h - 2, 0), (h - 2, w - 2)), (np.nan, np.inf, -np.inf, np.nan)):
        c[y:y + 2, x:x + 2, (y + x) % 3] = val                                             # 2x2 clusters on the corners
    c[0, w // 2:w // 2 + 3, 1] = np.nan; c[h // 2:h // 2 + 3, 0, 2] = np.inf; c[h - 1, w // 3, 0] = -np.inf   # runs on the edges
    c[h // 3:h // 3 + 5, 4:9] = grey(0.5 + 0.05 * rng.rand(5, 5))
    err[h // 3:h // 3 + 5, 4:9] = 1e-20
    with np.errstate(invalid="ignore"):
        err[pick(0.03) & (np.abs(D.luminance(c)) < 1)] = 1e-20
    for val in (np.nan, -1.0, 0.0, np.inf, 1e20):
        err[pick(0.015)] = val
    for val in (0.0, np.nan, np.inf):
        z[pick(0.02)] = val
    z[pick(0.03)] *= -1
    z[h // 2:, :] *= np.float32(8)                                                         # a sharp depth edge
    if extreme:
        y0, x0 = h // 2 - 1, w // 2 - 1
        sign = np.where((np.arange(3)[:, None] + np.arange(3)[None, :]) % 2 == 0, 1.0, -1.0)
        c[y0:y0 + 3, x0:x0 + 3] = grey(3e38 * sign * (1 - 0.01 * rng.rand(3, 3)))
        err[y0:y0 + 3, x0:x0 + 3] = np.inf
    return c, z, err


@pytest.mark.parametrize("wh", [(96, 64), (37, 23)])
def test_non_finite_and_extreme_inputs_against_the_restatement(ctx, wh):
    W, H = wh
    for extreme in (False, True):
        color, depth, err = hostile_frame(H, W, seed=W + H + extreme, extreme=extreme)
        for g, use_err, use_depth in GUIDES:
            if extreme and not use_err:
                continue                                    # the +-3e38 block comes with its infinite error map
            z, e = depth if use_depth else None, err if use_err else None
            for opt in (DEFAULTS, (3, 0.25, 0.01), (10, 64.0, 5.0)):
                got, words = run_denoise(ctx, color, z, e, opt)
                label = f"{W}x{H} {'extreme ' if extreme else ''}{g} {opt}"
                assert_matches(label, got, words, color, z, e, opt)


def test_a_frame_of_denormal_variances_is_copied_bit_for_bit(ctx):
    """err = 1e-20 at Y < 1 gives v = (err Y)^2 below 2^-126, which the device flushes to 0: every g is 0, and every level copies every
    pixel (a float64 v would filter them all)."""
    rng = np.random.RandomState(4)
    color = (0.3 + 0.6 * rng.rand(17, 23, 3)).astype(np.float32)
    err = np.full((17, 23), 1e-20, np.float32)
    for opt in (DEFAULTS, (10, 0.25, 5.0)):
        assert D.copied_pixels(color, None, err, *opt).all() and not D.copied_pixels(color, None, err, *opt, ftz=False).any()
        got, words = run_denoise(ctx, color, None, err, opt)
        assert_matches(f"23x17 err 1e-20 {opt}", got, words, color, None, err, opt)


# ---- 3. layers at every launch grouping ----------------------------------------------------------------------------------------------

def layer_specs(total, seed):
    """[(channels, count)] adding up to `total` planes: channels cycle through 1..4 and counts through 1..3, so the channel counts mix
    inside every launch group of 8 / 4 / 2 / 1 planes and layer boundaries fall inside groups."""
    specs, k = [], seed
    while total:
        n = min(total, 1 + k % 3)
        specs.append((1 + k % 4, n)); total -= n; k += 1
    return specs


@pytest.mark.parametrize("planes", [1, 2, 3, 5, 7, 8, 9, 13, 15, 17])
def test_layers_at_every_plane_count(ctx, planes):
    """Every layer against the restatement, every pixel; the beauty equal to vpt_denoise's bit for bit; NaN in some layer taps; every
    other layer in place; from 3 planes on, the colour itself as the first layer (equal to the beauty bit for bit)."""
    W, H = 67, 45
    rng = np.random.RandomState(planes)
    color, depth, err = noisy_ramp(H, W, seed=100 + planes)
    color[rng.rand(H, W) < 0.01, 1] = np.nan
    opt = [DEFAULTS, (6, 0.25, 5.0), (3, 64.0, 0.01), (10, 4.0, 0.2), (1, 4.0, 0.2)][planes % 5]
    specs = layer_specs(planes - (planes >= 3), seed=planes)
    layers = [(None, 3, 1, "out")] if planes >= 3 else []
    for i, (ch, k) in enumerate(specs):
        src = (rng.randn(k, H, W, ch) * 2).astype(np.float32)
        src[rng.rand(k, H, W, ch) < 0.003] = np.nan
        layers.append((src, ch, k, "in" if i % 2 else "out"))
    assert sum(k for _, _, k, _ in layers) == planes
    beauty, words, outs = run_layers(ctx, color, depth, err, layers, opt)
    alone, alone_words = run_denoise(ctx, color, depth, err, opt)
    assert np.array_equal(beauty.view(np.uint32), alone.view(np.uint32)) and np.array_equal(words, alone_words), "beauty != vpt_denoise"
    assert_matches(f"{planes} planes beauty {opt}", beauty, words, color, depth, err, opt)
    srcs = [color[None] if s is None else s for s, _, _, _ in layers]
    _, copied = D.denoise_and_copies(color, depth, err, *opt)
    _, want = DL.denoise_layers(color, [p for s in srcs for p in s], depth, err, *opt)
    want = iter(want)
    for l, (src, out) in enumerate(zip(srcs, outs)):
        if layers[l][0] is None:
            assert np.array_equal(out[0].view(np.uint32), beauty.view(np.uint32)), "the colour as a layer != the beauty"
        for k in range(src.shape[0]):
            fails, st = D.compare(out[k], next(want), src[k], copied, opt[0], D.RTOL)
            print(f"{planes} planes, layer {l} ({layers[l][1]} ch, {layers[l][3]}) plane {k}: worst |d|/bound {st['worst']:.3g}, "
                  f"|d|/(1e-5 + M) {st['ratio']:.3g}, {100 * st['bit_equal']:.2f} % bit-equal, {st['copied']} copied")
            assert not fails, f"{planes} planes, layer {l} plane {k}: " + "; ".join(fails)


# ---- 4. one context across sizes and plane counts ------------------------------------------------------------------------------------

def test_a_context_reused_across_sizes_equals_fresh_contexts():
    """The scratch planes grow with the frame and the layer planes with the plane count: 16x9, then 333x197, then 333x197 with 9 and with
    3 layer planes, then 16x9 again on one context give the bits of the same calls on fresh contexts."""
    frames = {wh: noisy_ramp(wh[1], wh[0], seed=wh[0]) for wh in ((16, 9), (333, 197))}

    def layers_of(wh, specs):
        rng = np.random.RandomState(len(specs))
        return [((rng.rand(k, wh[1], wh[0], ch) * 3).astype(np.float32), ch, k, "out") for ch, k in specs]
    calls = [((16, 9), None), ((333, 197), None), ((333, 197), layers_of((333, 197), layer_specs(9, 1))),
             ((333, 197), layers_of((333, 197), layer_specs(3, 2))), ((16, 9), layers_of((16, 9), layer_specs(2, 3)))]
    opt = (6, 4.0, 0.2)
    shared = new_context()
    try:
        for wh, layers in calls:
            c, z, e = frames[wh]
            fresh = new_context()
            try:
                if layers is None:
                    got, want = run_denoise(shared, c, z, e, opt), run_denoise(fresh, c, z, e, opt)
                else:
                    b, w, o = run_layers(shared, c, z, e, layers, opt)
                    fb, fw, fo = run_layers(fresh, c, z, e, layers, opt)
                    got, want = (b, w, *o), (fb, fw, *fo)
                for a, b in zip(got, want):
                    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{wh} with {0 if layers is None else len(layers)} layers"
            finally:
                torch.cuda.synchronize()
                V.lib.vpt_destroy(fresh)
    finally:
        torch.cuda.synchronize()
        V.lib.vpt_destroy(shared)
