"""Layer denoising on the GPU (vpt_denoise_layers): the beauty is vpt_denoise's bit for bit, a layer equal to the beauty comes out equal
to it, the layers match the NumPy restatement (tests/denoise_layers_ref.py), the additive identities of the layers survive denoising, a
sharded frame denoises to the single context's bits, and every refusal."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
import denoise_layers_ref as DL
import denoise_ref as D
from test_adaptive_gpu import make_case
from test_aov_gpu import constant_env_renderer
from test_denoise_gpu import MODES, noisy_frame
from test_exchange_binned_gpu import ALL, Case, Shards, atmosphere, dragon, emissive, same  # noqa: F401 (fixtures)
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
NAMES = ("alpha", "volume", *V.LIGHT_GROUPS, "deep", "mattes")


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def call_layers(r, color, depth, err, layers, words=None, opt=None):
    """vpt_denoise_layers through the C ABI: layers = [(src, dst, channels, count)] -> (rc, message, beauty)."""
    out = torch.empty(r.height, r.width, 3, dtype=torch.float32, device=color.device)
    descs = (V._native.denoise_layer * max(1, len(layers)))(*[V._native.denoise_layer(s.data_ptr(), d.data_ptr(), ch, k)
                                                              for s, d, ch, k in layers])
    rc = V.lib.vpt_denoise_layers(r.ctx, r.width, r.height, ptr(color), ptr(depth), ptr(err), opt, float(r.kp.exposure_scale), ptr(out),
                                  ptr(words), descs, len(layers), None)
    return rc, V.lib.vpt_last_error(r.ctx).decode(), out


def check_beauty_and_same_weights(r, color, depth, err, label):
    """(1) the beauty and display words equal Renderer.denoise with and without layers; (2) the colour as a 3-channel layer, and each of
    its channels as a 1-channel layer, equals the denoised beauty bit for bit."""
    want, want_words = r.denoise(color=color, depth=depth, rel_error=err, display=True)
    got = r.denoise_layers([], color=color, depth=depth if depth is not None else False, rel_error=err, display=True)
    H, W = r.height, r.width
    c3 = torch.empty_like(color)
    ch = [torch.empty(H, W, dtype=torch.float32, device=color.device) for _ in range(3)]
    planes = [color[..., k].contiguous() for k in range(3)]
    words = torch.empty(H, W, dtype=torch.int32, device=color.device)
    rc, msg, beauty = call_layers(r, color, depth, err, [(color, c3, 3, 1)] + [(planes[k], ch[k], 1, 1) for k in range(3)], words)
    torch.cuda.synchronize()
    assert rc == 0, msg
    assert same(got["beauty"], want) and torch.equal(got["display"], want_words), f"{label}: beauty without layers"
    assert same(beauty, want) and torch.equal(words, want_words), f"{label}: beauty with layers"
    assert same(c3, want), f"{label}: the colour as a 3-channel layer"
    for k in range(3):
        assert same(ch[k], want[..., k]), f"{label}: channel {k} as a 1-channel layer"


@pytest.mark.parametrize("name", ["headline", "vol_sky_table", "lights_sphere"])
def test_beauty_unchanged_and_same_weights_on_rendered_frames(dragon, name):
    scene, mk, keep = make_case(name, dragon, None)
    r = mk()
    color, depth, err = noisy_frame(scene, r)
    for label, use_err, use_depth in MODES:
        check_beauty_and_same_weights(r, color, depth if use_depth else None, err if use_err else None, f"{name} {label}")


@pytest.mark.parametrize("wh", [(333, 197), (7, 3), (1, 1)])
def test_beauty_unchanged_and_same_weights_on_ragged_and_tiny_frames(dragon, wh):
    W, H = wh
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=100))
    color, depth, err = noisy_frame(scene, r)
    for label, use_err, use_depth in MODES:
        check_beauty_and_same_weights(r, color, depth if use_depth else None, err if use_err else None, f"{W}x{H} {label}")


def layered(case, K_deep=8, K_mattes=3):
    r = case.renderer(case.scene())
    r.enable_aovs(); r.enable_light_groups(); r.enable_deep(case.bounds(K_deep))
    sets, sphere = case.sets(K_mattes)
    r.enable_mattes(sets, sphere)
    return r


def test_layers_against_the_restatement(dragon, emissive, atmosphere):
    """(3) the vol_emit frame (every light group non-zero) with its AOVs, groups, 8 deep slices and 3 mattes."""
    case = Case("vol_emit", dragon, emissive, atmosphere)
    r = layered(case)
    color, depth, err = noisy_frame(r.scene, r)
    out = r.denoise_layers(NAMES, rel_error=err)
    torch.cuda.synchronize()
    srcs = {"alpha": r.alpha_image(), "volume": r.volume_image(), **{g: r.light_group_image(g) for g in V.LIGHT_GROUPS}}
    for g in V.LIGHT_GROUPS:
        assert float(srcs[g].abs().max()) > 0, f"light group {g} is empty"
    flat = [srcs[n].cpu().numpy() for n in srcs] + list(r.deep_image().cpu().numpy()) + list(r.matte_image().cpu().numpy())
    args = (color.cpu().numpy(), depth.cpu().numpy(), err.cpu().numpy())
    beauty, want = DL.denoise_layers(args[0], flat, *args[1:])
    _, copied = D.denoise_and_copies(*args)
    got = [out[n].cpu().numpy() for n in srcs] + list(out["deep"].cpu().numpy()) + list(out["mattes"].cpu().numpy())
    labels = list(srcs) + [f"deep {k}" for k in range(8)] + [f"matte {k}" for k in range(3)]
    for label, g, w, s in zip(labels, got, want, flat):
        fails, st = D.compare(g, w, s, copied, 5, D.RTOL)
        print(f"{label}: worst |d|/bound {st['worst']:.3g}, |d|/(1e-5 + M) {st['ratio']:.3g}, {100 * st['bit_equal']:.2f} % bit-equal, "
              f"{st['copied']} copied")
        assert not fails, f"{label}: " + "; ".join(fails)


def test_identities_survive_denoising(dragon, emissive, atmosphere):
    """(4) Sum of groups' = beauty' and Sum_k deep'_k = (volume', alpha'); and under a constant
    environment k, beauty' = volume' + (1 - alpha') k.  Each bound: the identity's worst error before denoising plus a few ulps."""
    case = Case("vol_emit", dragon, emissive, atmosphere)
    r = layered(case, K_deep=8, K_mattes=3)
    color, depth, err = noisy_frame(r.scene, r)
    out = r.denoise_layers(NAMES, rel_error=err)
    torch.cuda.synchronize()
    f64 = lambda t: t.double().cpu().numpy()
    ulps = lambda x: 8 * np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)

    def check(lhs0, rhs0, lhs1, rhs1, what):
        before = float(np.max(np.abs(lhs0 - rhs0)))
        after = np.abs(lhs1 - rhs1)
        assert (after <= before + ulps(rhs1) + 1e-30).all(), f"{what}: {float(after.max())} after, {before} before"
        print(f"{what}: worst error {before:.3g} before, {float(after.max()):.3g} after")
    groups0 = sum(f64(r.light_group_image(g)) for g in V.LIGHT_GROUPS)
    groups1 = sum(f64(out[g]) for g in V.LIGHT_GROUPS)
    check(groups0, f64(color), groups1, f64(out["beauty"]), "sum of the light groups")
    deep0, deep1 = f64(r.deep_image()).sum(0), f64(out["deep"]).sum(0)
    check(deep0[..., :3], f64(r.volume_image()), deep1[..., :3], f64(out["volume"]), "sum of the deep slices (colour)")
    check(deep0[..., 3], f64(r.alpha_image()), deep1[..., 3], f64(out["alpha"]), "sum of the deep slices (coverage)")

    E = 2.0
    scene, rc = constant_env_renderer(dragon, E)
    color, depth, err = noisy_frame(scene, rc)
    o = rc.denoise_layers(["alpha", "volume"], rel_error=err)
    torch.cuda.synchronize()
    k = (np.float32(E) * np.array([rc.kp.sky_color.x, rc.kp.sky_color.y, rc.kp.sky_color.z], np.float32) *
         np.float32(1.0 / (4.0 * np.pi))).astype(np.float64)
    comp0 = f64(rc.volume_image()) + (1.0 - f64(rc.alpha_image()))[..., None] * k
    comp1 = f64(o["volume"]) + (1.0 - f64(o["alpha"]))[..., None] * k
    check(comp0, f64(color), comp1, f64(o["beauty"]), "volume + (1 - alpha) k")


def test_one_matte_of_the_full_map_stays_the_aovs(dragon, emissive, atmosphere):
    """(4) a K = 1 matte of the full map is (volume, alpha) bit for bit in a fixed-count frame, and stays so after denoising."""
    case = Case("instances", dragon, emissive, atmosphere)
    r = layered(case, K_deep=1, K_mattes=1)
    r.scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(8); torch.cuda.synchronize()
    m = r.matte_image()[0]
    assert same(m[..., :3].contiguous(), r.volume_image()) and same(m[..., 3].contiguous(), r.alpha_image())
    for rel in (None, torch.full((r.height, r.width), 0.05, dtype=torch.float32, device=m.device)):
        out = r.denoise_layers(["alpha", "volume", "mattes"], rel_error=rel)
        torch.cuda.synchronize()
        m = out["mattes"][0]
        assert not same(out["volume"], r.volume_image()), "the filter must move the volume"
        assert same(m[..., :3].contiguous(), out["volume"]) and same(m[..., 3].contiguous(), out["alpha"]), "K = 1 matte of the full map"


def test_in_place_equals_out_of_place(dragon, emissive, atmosphere):
    """(5) dst == src gives the out-of-place bits; the inputs stay untouched; two calls give the same bits."""
    case = Case("vol_emit", dragon, emissive, atmosphere)
    r = layered(case)
    color, depth, err = noisy_frame(r.scene, r)
    c0, d0, e0 = color.clone(), depth.clone(), err.clone()
    a = r.denoise_layers(NAMES, color=color, rel_error=err)
    b = r.denoise_layers(NAMES, color=color, rel_error=err)
    torch.cuda.synchronize()
    for n in ("beauty",) + NAMES:
        assert same(a[n], b[n]), f"two calls differ in {n}"
    srcs = {"alpha": r.buffers.alpha, "volume": r.buffers.volume, **r.buffers.groups, "deep": r.buffers.deep, "mattes": r.buffers.mattes}
    keep = {n: t.clone() for n, t in srcs.items()}
    chs = {"alpha": 1, "deep": 4, "mattes": 4}
    work = {n: t.clone() for n, t in srcs.items()}
    layers = [(work[n], work[n], chs.get(n, 3), work[n].shape[0] if n in ("deep", "mattes") else 1) for n in work]
    rc, msg, beauty = call_layers(r, color, depth, err, layers)
    torch.cuda.synchronize()
    assert rc == 0, msg
    assert torch.equal(color, c0) and torch.equal(depth, d0) and torch.equal(err, e0)
    for n in srcs:
        assert same(srcs[n], keep[n]), f"{n}: the renderer's buffer was written"
        assert same(work[n], a[n]), f"{n}: in place differs from out of place"
    assert same(beauty, a["beauty"])


def shard_frames(dragon, emissive, atmosphere, adaptive):
    sh = Shards(Case("instances", dragon, emissive, atmosphere), 3, 5, ALL, 8, 3)
    sh.enable(8, 3, layers=True)
    res = {}

    def fn(k, r, stream):
        r.kp.iteration = 0
        if adaptive:
            if k < 0:
                res["ref"] = r.render_adaptive(24, threshold=0.05, min_passes=4, check_interval=4, error_map=True)
            else:
                sh.d[k].render_adaptive(24, threshold=0.05, min_passes=4, check_interval=4, stream=stream)
        else:
            r.render(6, stream=stream) if k < 0 else sh.d[k].render(6, stream=stream)
    sh.all(fn)
    return sh, res


@pytest.mark.parametrize("adaptive", [False, True])
def test_sharded_frames_denoise_to_the_single_context(dragon, emissive, atmosphere, adaptive):
    """(6) three shards on one GPU over the peer-memory exchange: every shard's DistributedRenderer.denoise_layers equals the single
    context's Renderer.denoise_layers bit for bit, for every layer."""
    sh, res = shard_frames(dragon, emissive, atmosphere, adaptive)
    err = res["ref"][2] if adaptive else None
    want = sh.ref.denoise_layers(NAMES, rel_error=err, display=True)
    got = sh.all(lambda k, r, stream: None if k < 0 else sh.d[k].denoise_layers(NAMES, display=True, stream=stream))
    torch.cuda.synchronize()
    for k, g in enumerate(got):
        for n in ("beauty", "display") + NAMES:
            assert same(g[n], want[n]), f"shard {k}: {n}"
    sh.close()


def test_refusals_say_why_and_enqueue_nothing(dragon):
    """(7) every refusal returns VPT_ERR_INVALID with a message naming vpt_denoise, and writes nothing."""
    W, H = 64, 48
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=2))
    dev = r.buffers.accum.device
    n = W * H
    big = torch.arange(16 * n, dtype=torch.float32, device=dev)
    col, out = big[:3 * n], big[3 * n:6 * n]
    z, e = big[6 * n:7 * n], big[7 * n:8 * n]
    s1, d1 = big[8 * n:11 * n], big[11 * n:14 * n]
    s2, d2 = big[14 * n:15 * n], big[15 * n:16 * n]
    before = big.clone()
    opt = lambda *a: C.byref(V._native.denoise_options(*a))
    lib = V.lib
    L = V._native.denoise_layer

    def call(layers, *, color=col, n_layers=None, o=None, out_f3=out, depth=z, err=e):
        arr = (L * max(1, len(layers)))(*[L(a, b, c, k) for a, b, c, k in layers]) if layers is not None else None
        rc = lib.vpt_denoise_layers(r.ctx, W, H, ptr(color) if color is not None else None, ptr(depth), ptr(err), o, 1.0,
                                    ptr(out_f3) if out_f3 is not None else None, None, arr,
                                    len(layers or []) if n_layers is None else n_layers, None)
        return rc, lib.vpt_last_error(r.ctx).decode()
    a = lambda t, off=0: t.data_ptr() + 4 * off
    good = [(a(s1), a(d1), 3, 1), (a(s2), a(d2), 1, 1)]
    refused = {
        "null colour": call(good, color=None), "null output": call(good, out_f3=None),
        "iterations 0": call(good, o=opt(0, 4.0, 0.2)), "sigma_l nan": call(good, o=opt(5, float("nan"), 0.2)),
        "output partially over colour": call(good, out_f3=big[3:]),
        "null layers": call(None, n_layers=2),
        "null src": call([(0, a(d1), 3, 1)]), "null dst": call([(a(s1), 0, 3, 1)]),
        "channels 0": call([(a(s1), a(d1), 0, 1)]), "channels 5": call([(a(s1), a(d1), 5, 1)]),
        "count 0": call([(a(s1), a(d1), 3, 0)]),
        "dst partially over its src": call([(a(s1), a(s1, 1), 3, 1)]),
        "dst over another layer's src": call([(a(s1), a(d1), 3, 1), (a(d1, 5), a(d2), 1, 1)]),
        "dst over another layer's dst": call([(a(s1), a(d1), 3, 1), (a(s2), a(d1, 2 * n), 1, 1)]),
        "dst over the colour": call([(a(s1), a(col), 3, 1)]),
        "dst over the output": call([(a(s1), a(out, 7), 1, 1)]),
        "dst over the depth": call([(a(s1), a(z, -3), 1, 1)]),
        "dst over the error map": call([(a(s2), a(e), 1, 1)]),
    }
    torch.cuda.synchronize()
    for what, (rc, msg) in refused.items():
        assert rc == -1 and "vpt_denoise" in msg, (what, rc, msg)
    assert torch.equal(big, before), "a refused call wrote"
    assert call(good)[0] == 0 and call([(a(s1), a(s1), 3, 1)])[0] == 0 and call([(a(col), a(d1), 3, 1)])[0] == 0
    torch.cuda.synchronize()
    with pytest.raises(V.VptError, match="unknown layer"):
        r.denoise_layers(["nope"])
    with pytest.raises(V.VptError, match="enable_aovs"):
        r.denoise_layers(["alpha"])
    with pytest.raises(V.VptError, match="enable_deep"):
        r.denoise_layers(["deep"])
    part = V.Renderer(scene, W, H, kp=make_kp(ray_depth=2), cam=r.cam, rank=0, n_ranks=2, stripe_rows=8)
    with pytest.raises(V.VptError, match="partitioned"):
        part.denoise_layers(["alpha"], color=col.view(H, W, 3))
    part.close()
