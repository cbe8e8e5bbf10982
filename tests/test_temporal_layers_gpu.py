"""Temporal layers on the GPU (vpt_temporal_layers; DESIGN.md section 8r).

1. The beauty, its lengths and display words equal vpt_temporal's bit for bit, with and without history and clip, on orbit frames of the
   headline scene (dragon, sun + HDRI) with every layer enabled.
2. The colour as one 3-channel layer and as three 1-channel layers equals the beauty bit for bit (no clip).
3. The layers against tests/temporal_layers_ref.py on synthetic inputs with every drop rule, 1 to 4 channels and NaNs in layer taps.
4. The still-camera guarantee: 8 one-pass frames through render_temporal give every layer of the 8-pass progressive frame bit for bit.
5. After a moving-camera sequence the layers still add up: position.w is alpha bit for bit, the light groups sum to the beauty, the deep
   coverage to alpha, and volume + (1 - alpha) k to the beauty under a constant environment, each within its unfiltered rounding level.
6. Refusals, each leaving every dst untouched and enqueuing nothing.
7. render_temporal returns the same beauty with and without layers."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp
from test_aov_gpu import constant_env_renderer
from test_temporal_gpu import bits, same, copy_cam, pan_cameras, look_at, synthetic, dragon  # noqa: F401 (fixture)
import temporal_layers_ref as TL
import temporal_ref as T

pytestmark = pytest.mark.gpu
INF = float("inf")
ALL = ("alpha", "volume", *V.LIGHT_GROUPS, "position", "normal", "albedo", "deep", "mattes")


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def headline(dragon, w, h, ray_depth=100):
    """The headline scene (dragon, sun + HDRI) with every layer enabled: AOVs, light groups, collision AOVs, deep K = 2, mattes K = 2."""
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, w, h, kp=make_kp(ray_depth=ray_depth))
    r.enable_aovs(); r.enable_light_groups(); r.enable_collision_aovs()
    lo, hi = scene.world_bounds()
    r.enable_deep([0.0, float(np.linalg.norm(hi - lo)), INF])
    r.enable_mattes([[0], []])
    return scene, r


def call(r, prev, color, vectors, history, history_len, layers, clip=INF, max_history=16, words=None):
    """vpt_temporal_layers through the C ABI: layers = [(src, history, dst, channels, count)] -> (rc, message, out, out_len)."""
    dev = color.device
    out = torch.empty(r.height, r.width, 3, dtype=torch.float32, device=dev)
    out_len = torch.empty(r.height, r.width, dtype=torch.float32, device=dev)
    descs = (N.temporal_layer * max(1, len(layers)))(*[N.temporal_layer(s.data_ptr(), h.data_ptr() if h is not None else None,
                                                                        d.data_ptr() if d is not None else None, ch, k)
                                                       for s, h, d, ch, k in layers])
    opt = N.temporal_options(max_history, clip)
    rc = V.lib.vpt_temporal_layers(r.ctx, r.width, r.height, ptr(color), ptr(vectors), C.byref(r.cam), C.byref(prev), ptr(history),
                                   ptr(history_len), C.byref(opt), float(r.kp.exposure_scale), ptr(out), ptr(out_len), ptr(words), descs,
                                   len(layers), None)
    return rc, V.lib.vpt_last_error(r.ctx).decode(), out, out_len


def render_frame(r, cam, prev, passes, offset):
    V.lib.vpt_set_motion_vectors(r.ctx, ptr(r.buffers.motion), C.byref(prev))
    r.set_sample_offset(offset)
    C.memmove(C.byref(r.cam), C.byref(cam), C.sizeof(r.cam))
    r.kp.iteration = 0
    r.render(passes)


# ---- 1, 2: the beauty is vpt_temporal's; the colour as a layer is the beauty ------------------------------------------------------------
@pytest.mark.parametrize("clip", [INF, 1.5])
def test_the_beauty_is_vpt_temporal_and_the_colour_as_a_layer_is_the_beauty(dragon, clip):
    w, h = 320, 180
    scene, r = headline(dragon, w, h)
    r.buffers.motion = torch.zeros(w * h, 3, dtype=torch.float32, device=r.buffers.accum.device)
    cams = pan_cameras(scene, w, h, 4, 1.0)
    scene.reset_blue_noise()
    hist = ln = None
    lh = None
    for f, cam in enumerate(cams):
        prev = cams[max(f - 1, 0)]
        render_frame(r, cam, prev, 2, 2 * f)
        want, want_len, want_words = r.temporal(prev, history=hist, history_len=ln, clip_sigma=clip, display=True)
        got = r.temporal_layers(prev, ALL, layer_history=lh, history=hist, history_len=ln, clip_sigma=clip, display=True)
        color = r.buffers.accum.view(h, w, 3)
        c3 = torch.empty_like(color)
        planes = [color[..., k].contiguous() for k in range(3)]
        hplanes = [hist[..., k].contiguous() if hist is not None else None for k in range(3)]
        c1 = [torch.empty(h, w, dtype=torch.float32, device=color.device) for _ in range(3)]
        words = torch.empty(h, w, dtype=torch.int32, device=color.device)
        rc, msg, out, out_len = call(r, prev, color, r.buffers.motion, hist, ln,
                                     [(color, hist, c3, 3, 1)] + [(planes[k], hplanes[k], c1[k], 1, 1) for k in range(3)], clip, words=words)
        torch.cuda.synchronize()
        assert rc == 0, msg
        label = f"frame {f}, clip {clip}"
        assert same(got["beauty"], want) and same(got["len"], want_len) and same(got["display"], want_words), f"{label}: Renderer.temporal_layers"
        assert same(out, want) and same(out_len, want_len) and same(words, want_words), f"{label}: C ABI with the colour as layers"
        if f > 0:
            assert bool((want_len > 1).any()), label
        if clip == INF:
            assert same(c3, want), f"{label}: the colour as a 3-channel layer"
            for k in range(3):
                assert same(c1[k], want[..., k]), f"{label}: channel {k} as a 1-channel layer"
        hist, ln = want, want_len
        lh = {n: got[n] for n in ALL}
    r.close()


# ---- 3: the layers against the restatement ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(7, 3), (61, 37)])
@pytest.mark.parametrize("motion", ["fractional", "integer"])
@pytest.mark.parametrize("clip", [INF, 1.5])
def test_the_layers_match_the_restatement(dragon, w, h, motion, clip):
    scene = V.Scene([dragon.instance()], env=synthetic_env(64, 32))
    a = look_at((3.0, 2.0, 9.0), (0.2, 0.1, 0.0), w, h)
    b = look_at((3.1, 2.0, 8.9), (0.25, 0.1, 0.0), w, h)
    r = V.Renderer(scene, w, h, cam=a)
    c, m, hist, ln = synthetic(w, h, w * 100 + h, motion)
    n = w * h
    rng = np.random.default_rng(w + h)
    hist[rng.random(n) < 0.05, 2] = -np.inf                     # non-finite beauty taps, one channel only
    specs = [(1, 1), (2, 1), (3, 2), (4, 3)]                    # (channels, count)
    srcs = [rng.uniform(-2.0, 2.0, (k, n, ch)).astype(np.float32) for ch, k in specs]
    hists = [rng.uniform(-2.0, 2.0, (k, n, ch)).astype(np.float32) for ch, k in specs]
    hists[2][0, rng.random(n) < 0.04, 1] = np.nan               # NaNs in layer taps
    dev = r.buffers.accum.device
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)
    dsts = [torch.empty(k * n * ch, dtype=torch.float32, device=dev) for ch, k in specs]
    ts, th = [t(x) for x in srcs], [t(x) for x in hists]
    rc, msg, out, out_len = call(r, b, t(c), t(m), t(hist), t(ln), [(ts[i], th[i], dsts[i], ch, k) for i, (ch, k) in enumerate(specs)],
                                 clip, max_history=8)
    torch.cuda.synchronize()
    assert rc == 0, msg
    bt = TL.beauty_taps(w, h, c, m, a, b, hist, ln, max_history=8, motion_dt=np.float32, footprint_dt=np.float32)
    assert np.array_equal(out_len.cpu().numpy().reshape(-1).view(np.uint32), bt["L"].astype(np.float32).view(np.uint32)), "history lengths"
    used = bt["used"]
    if n > 100:
        assert used.any() and (~used).any()
    for i, (ch, k) in enumerate(specs):
        got = dsts[i].cpu().numpy().reshape(k, n, ch)
        want = TL.blend_layer(bt, srcs[i], hists[i], ch, k)
        M = TL.layer_reach(bt, srcs[i], hists[i], ch, k)
        for p in range(k):
            # every value: no history => the value bit for bit, non-finite in kind, finite within 1e-5 + 1e-4 M
            fails, _ = T.compare(got[p], want[p], srcs[i][p], ~used, M[p])
            assert not fails, f"{ch} channels x {k}, plane {p}: " + "; ".join(fails)
    if n > 100:
        assert np.isnan(dsts[2].cpu().numpy()).any(), "a NaN in a used tap spreads"
    r.close()


# ---- 4: the still-camera guarantee -----------------------------------------------------------------------------------------------------
def layer_frames(r):
    b = r.buffers
    return {"alpha": b.alpha, "volume": b.volume, **(b.groups or {}), "position": b.position, "normal": b.normal, "albedo": b.albedo,
            "deep": b.deep, "mattes": b.mattes, "beauty": b.accum}


def test_eight_offset_frames_give_every_layer_of_the_eight_pass_frame(dragon):
    w, h, F = 240, 136, 8
    scene, r = headline(dragon, w, h)
    r.enable_temporal(max_history=F, layers=ALL)
    scene.reset_blue_noise()
    cam = copy_cam(r.cam)
    for _ in range(F):
        out, L = r.render_temporal(cam, 1)
    torch.cuda.synchronize()
    assert bool((L == F).all())
    got = r.temporal_layer_images()
    _, ref = headline(dragon, w, h)
    scene.reset_blue_noise(); ref.kp.iteration = 0
    for _ in range(F): ref.render_pass()
    torch.cuda.synchronize()
    want = layer_frames(ref)
    assert same(out.reshape(-1, 3), want["beauty"]), "beauty"
    for name in ALL:
        assert same(got[name].reshape(want[name].shape), want[name]), name
        if name not in ("point", "emission"):                   # the headline scene has neither point lights nor emission
            assert float(want[name].abs().max()) > 0, f"{name} is empty"
    r.disable_temporal(); r.close(); ref.close()


# ---- 5: the identities after a moving-camera sequence ----------------------------------------------------------------------------------
def orbit(r, scene, names, frames=8, passes=2, step=0.5):
    cams = pan_cameras(scene, r.width, r.height, frames, step)
    r.enable_temporal(layers=names)
    scene.reset_blue_noise()
    before = []
    for cam in cams:
        out, L = r.render_temporal(cam, passes)
        before.append({n: t.clone() for n, t in layer_frames(r).items() if t is not None})
    torch.cuda.synchronize()
    return out, L, r.temporal_layer_images(), before


def check(lhs0, rhs0, lhs1, rhs1, what):
    """the identity's worst error over the unfiltered frames plus a few ulps bounds it after filtering"""
    ulps = 16 * np.spacing(np.abs(rhs1).astype(np.float32)).astype(np.float64)
    before = max(float(np.max(np.abs(a - b))) for a, b in zip(lhs0, rhs0))
    after = np.abs(lhs1 - rhs1)
    print(f"[temporal layers] {what}: worst error {before:.3g} unfiltered, {float(after.max()):.3g} filtered")
    assert (after <= before + ulps + 1e-30).all(), f"{what}: {float(after.max())} after, {before} before"


def test_the_identities_survive_a_moving_camera(dragon):
    w, h = 320, 180
    scene, r = headline(dragon, w, h)
    out, L, got, before = orbit(r, scene, ALL)
    assert float(L.max()) > 2
    f64 = lambda t: t.double().cpu().numpy()
    assert same(got["position"][..., 3].contiguous(), got["alpha"]), "position.w is alpha"
    groups0 = [sum(f64(b[g]) for g in V.LIGHT_GROUPS) for b in before]
    check(groups0, [f64(b["beauty"]) for b in before], sum(f64(got[g]) for g in V.LIGHT_GROUPS).reshape(-1, 3), f64(out).reshape(-1, 3),
          "sum of the light groups")
    check([f64(b["deep"])[..., 3].sum(0) for b in before], [f64(b["alpha"]) for b in before], f64(got["deep"])[..., 3].sum(0).reshape(-1),
          f64(got["alpha"]).reshape(-1), "sum of the deep coverage")
    r.disable_temporal(); r.close()

    E = 2.0
    scene, rc = constant_env_renderer(dragon, E, W=w, H=h)
    out, L, got, before = orbit(rc, scene, ("alpha", "volume"))
    k = (np.float32(E) * np.array([rc.kp.sky_color.x, rc.kp.sky_color.y, rc.kp.sky_color.z], np.float32) *
         np.float32(1.0 / (4.0 * np.pi))).astype(np.float64)
    comp = lambda vol, alpha: vol.reshape(-1, 3) + (1.0 - alpha.reshape(-1))[:, None] * k
    check([comp(f64(b["volume"]), f64(b["alpha"])) for b in before], [f64(b["beauty"]) for b in before],
          comp(f64(got["volume"]), f64(got["alpha"])), f64(out).reshape(-1, 3), "volume + (1 - alpha) k")
    rc.disable_temporal(); rc.close()


# ---- 6: refusals -----------------------------------------------------------------------------------------------------------------------
def test_refusals(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(64, 32))
    w, h = 16, 8
    n = w * h
    r = V.Renderer(scene, w, h)
    dev = r.buffers.accum.device
    z = lambda *s: torch.zeros(*s, device=dev)
    c, m, hist, ln = z(n, 3), z(n, 3), z(n, 3), torch.ones(n, device=dev)
    src, lhist = z(2, n, 4), z(2, n, 4)
    dst, dst2 = torch.full((2, n, 4), 7.0, device=dev), torch.full((n,), 7.0, device=dev)
    src1, lhist1 = z(n), z(n)
    launches = r.stats()[0]

    def refused(match, layers, history=hist, history_len=ln, n_layers=None):
        descs = (N.temporal_layer * max(1, len(layers)))(*layers)
        opt = N.temporal_options(16, INF)
        out, out_len = z(n, 3), z(n)
        rc = V.lib.vpt_temporal_layers(r.ctx, w, h, ptr(c), ptr(m), C.byref(r.cam), C.byref(r.cam), ptr(history), ptr(history_len),
                                       C.byref(opt), 1.0, ptr(out), ptr(out_len), None, descs if layers else None,
                                       len(layers) if n_layers is None else n_layers, None)
        assert rc == -1, match
        assert match in V.lib.vpt_last_error(r.ctx).decode(), (match, V.lib.vpt_last_error(r.ctx))
    L = lambda s=src, hh=lhist, d=dst, ch=4, k=2: N.temporal_layer(s.data_ptr() if s is not None else None,
                                                                   hh.data_ptr() if hh is not None else None,
                                                                   d.data_ptr() if d is not None else None, ch, k)
    good = L(src1, lhist1, dst2, 1, 1)
    refused("null layers array", [], n_layers=1)
    refused("at most 16 layers", [good] * 17)
    refused("null src or dst", [L(s=None)])
    refused("null src or dst", [L(d=None)])
    refused("history must be set exactly when", [L(hh=None)])
    refused("history must be set exactly when", [L()], history=None, history_len=None)
    refused("channels must be 1..4", [L(ch=0)])
    refused("channels must be 1..4", [L(ch=5)])
    refused("count must be >= 1", [L(k=0)])
    refused("layer 0 dst overlaps d_color_f3", [L(d=c, ch=3, k=1)])
    refused("layer 0 dst overlaps d_history_len", [L(d=ln, ch=1, k=1)])
    refused("layer 0 dst overlaps layer 0 src", [L(d=src)])
    refused("layer 0 dst overlaps layer 0 history", [L(d=lhist)])
    refused("layer 1 dst overlaps layer 0 src", [good, L(src1, lhist1, src1, 1, 1)])
    refused("layer 0 dst overlaps layer 1 dst", [L(), L(src1, lhist1, dst[1], 1, 1)])
    out = z(n, 3)
    descs = (N.temporal_layer * 1)(L(s=out, hh=lhist1, d=dst2, ch=1, k=1))
    rc = V.lib.vpt_temporal_layers(r.ctx, w, h, ptr(c), ptr(m), C.byref(r.cam), C.byref(r.cam), ptr(hist), ptr(ln), None, 1.0, ptr(out),
                                   ptr(z(n)), None, descs, 1, None)
    assert rc == -1 and "d_out_f3 overlaps layer 0 src" in V.lib.vpt_last_error(r.ctx).decode()
    with pytest.raises(V.VptError, match="layer_history must be given exactly when history is"):
        r.temporal_layers(r.cam, {"alpha": src1}, vectors=m, color=c, history=hist, history_len=ln)
    with pytest.raises(V.VptError, match="needs the AOVs"):
        r.enable_temporal(layers=("alpha",))
    torch.cuda.synchronize()
    assert r.stats()[0] == launches, "a refused call enqueued work"
    assert bool((dst == 7.0).all()) and bool((dst2 == 7.0).all()), "a refused call wrote a dst"
    rc, msg, _, _ = call(r, r.cam, c, m, hist, ln, [(src1, lhist1, dst2, 1, 1)])
    assert rc == 0, msg
    assert r.stats()[0] == launches + 1
    r.close()


# ---- 7: render_temporal's return value -------------------------------------------------------------------------------------------------
def test_render_temporal_returns_the_same_beauty_with_and_without_layers(dragon):
    w, h = 240, 136
    outs = []
    for names in ((), ALL):
        scene, r = headline(dragon, w, h)
        cams = pan_cameras(scene, w, h, 4, 0.5)
        r.enable_temporal(layers=names)
        scene.reset_blue_noise()
        frames = []
        for cam in cams:
            frames.append([t.clone() for t in r.render_temporal(cam, 2, display=True)])
        torch.cuda.synchronize()
        outs.append(frames)
        if names:
            assert set(r.temporal_layer_images()) == set(ALL)
        r.disable_temporal(); r.close()
    for f, (a, b) in enumerate(zip(*outs)):
        for x, y in zip(a, b):
            assert same(x, y), f"frame {f}"
