"""Temporal accumulation (vpt_set_sample_offset, vpt_temporal; DESIGN.md section 8p) on the GPU.

1. The sample offset, bit for bit: a one-pass frame at iteration 0 and offset k is pass k of the progressive frame -- accum's rule applied
   to the progressive accum after k passes with it as the sample gives the accum after k + 1 passes, and the same for depth; raw.w (the
   pass's tr) is equal.  The accum rule is applied by vpt_temporal with B == A, no clip and history length k, which is accum's own
   expression compiled with k_resolve's flags (NumPy's correctly rounded division is not the fast-math division).  A guarded sample would
   break the identity at its pixel, so the exact equality also asserts the scenes have none.  Offset 0 set explicitly changes nothing; the
   three-shard peer exchange at offset k equals the single context.
2. The central guarantee: 8 one-pass frames at offsets 0..7 through vpt_temporal (B == A, no clip) give accum and display of the 8-pass
   progressive frame bit for bit.
3. k_temporal against the float64 restatement (tests/temporal_ref.py) on synthetic inputs, and "no history => out = C, L = 1, display =
   k_resolve's word" bit for bit.
4. A slow pan through render_temporal ends closer to a converged frame of its last pose than the unfiltered frame.
5. Refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp
from test_aov_gpu import make_aov_case
from test_adaptive_gpu import make_case
from test_exchange_layers_gpu import Case as LayerCase, Shards as LayerShards, enable_all
import temporal_ref as T

pytestmark = pytest.mark.gpu
INF = float("inf")


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


@pytest.fixture(scope="module")
def emissive():
    n = 48
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    c = (n - 1) / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) / c
    return V.Volume.from_dense((np.clip(1.1 - r, 0.0, None) ** 1.5).astype(np.float32), bbox_min=(-c, -c, -c),
                               emission=(3.0 * np.clip(0.8 - r, 0.0, None)).astype(np.float32))


@pytest.fixture(scope="module")
def atmosphere():
    atm = V.Atmosphere()
    yield atm
    atm.destroy()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def copy_cam(cam):
    return N.camera.from_buffer_copy(bytes(cam))


def moved(cam, d_origin, d_llc):
    c = copy_cam(cam)
    def add(v, d): return N.f3(*[float(np.float32(getattr(v, a)) + np.float32(x)) for a, x in zip("xyz", d)])
    c.origin = add(cam.origin, d_origin)
    c.lower_left_corner = add(cam.lower_left_corner, d_llc)
    return c


def scale_of(scene):
    lo, hi = scene.world_bounds()
    return float(np.linalg.norm(hi - lo))


def accum_rule(r, acc, value, k):
    """acc + (value - acc) / (float)(k + 1) in k_resolve's arithmetic: vpt_temporal with B == A, no clip, history length k"""
    n = acc.shape[0]
    still = torch.zeros(n, 3, dtype=torch.float32, device=acc.device)
    still[:, 2] = 1.0
    out, _ = r.temporal(r.cam, color=value.contiguous(), vectors=still, history=acc.contiguous(),
                        history_len=torch.full((n,), float(k), device=acc.device), max_history=1 << 24, clip_sigma=INF)
    return out.reshape(n, 3)


def f3(t):
    return t.reshape(-1, 1).expand(-1, 3).contiguous()


# ---- 1: the sample offset --------------------------------------------------------------------------------------------------------------
OFFSET_CASES = ["headline", "lights_sphere", "vol_sky_table", "motion", "brick"]


def offset_renderer(name, dragon, perlin):
    if name == "motion":
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        cam = scene.frame_camera(192, 96)
        s = scale_of(scene)
        def mk():
            r = V.Renderer(scene, 192, 96, kp=make_kp(ray_depth=2), cam=cam)
            r.set_camera_motion(moved(cam, (0.03 * s, 0.0, -0.02 * s), (0.03 * s, 0.01 * s, -0.02 * s)))
            return r
        return scene, mk, []
    scene, mk, keep = make_aov_case(name, dragon, perlin)
    return scene, (lambda: mk(aovs=False)), keep


@pytest.mark.parametrize("name", OFFSET_CASES)
def test_a_one_pass_frame_at_offset_k_is_pass_k_of_the_progressive_frame(dragon, perlin, name):
    scene, mk, keep = offset_renderer(name, dragon, perlin)
    r = mk()
    for k in (1, 3):
        scene.reset_blue_noise(); r.set_sample_offset(0); r.kp.iteration = 0; r.buffers.zero_()
        for _ in range(k): r.render_pass()
        torch.cuda.synchronize()
        acc_k, dep_k = r.buffers.accum.clone(), r.buffers.depth.clone()
        r.render_pass(); torch.cuda.synchronize()
        acc_k1, dep_k1, raw_k1 = r.buffers.accum.clone(), r.buffers.depth.clone(), r.buffers.raw.clone()
        scene.reset_blue_noise(); r.kp.iteration = 0
        for _ in range(k): r.render_pass()                   # the blue noise of pass k: one advance per launch
        r.set_sample_offset(k); r.kp.iteration = 0
        r.render_pass(); torch.cuda.synchronize()
        sample, dsample, raw = r.buffers.accum.clone(), r.buffers.depth.clone(), r.buffers.raw.clone()
        assert same(accum_rule(r, acc_k, sample, k), acc_k1), f"{name}, k = {k}: accum"
        assert same(accum_rule(r, f3(dep_k), f3(dsample), k)[:, 0], dep_k1), f"{name}, k = {k}: depth"
        assert same(raw[:, 3], raw_k1[:, 3]), f"{name}, k = {k}: raw.w (the pass's tr)"
        assert not same(sample, acc_k1)
    r.set_sample_offset(0)


def test_offset_zero_set_explicitly_changes_nothing(dragon, perlin):
    scene, mk, keep = offset_renderer("lights_sphere", dragon, perlin)
    outs = []
    for explicit in (False, True):
        r = mk()
        if explicit: r.set_sample_offset(0)
        scene.reset_blue_noise(); r.kp.iteration = 0
        r.render(4); r.render(2); torch.cuda.synchronize()
        outs.append({k: getattr(r.buffers, k).clone() for k in ("accum", "depth", "cost", "raw", "display")})
        r.close()
    for k in outs[0]:
        assert same(outs[0][k], outs[1][k]), k


def test_the_offset_takes_effect_at_iteration_zero(dragon, perlin):
    scene, mk, keep = offset_renderer("headline", dragon, perlin)
    r, ref = mk(), mk()
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(2)
    r.set_sample_offset(5); r.render(2)                     # a continued frame keeps offset 0
    scene.reset_blue_noise(); ref.kp.iteration = 0; ref.render(4); torch.cuda.synchronize()
    assert same(r.buffers.accum, ref.buffers.accum)
    r.set_sample_offset(0)


def test_three_shards_at_an_offset_equal_the_single_context(dragon, emissive, atmosphere):
    case = LayerCase("hdri", dragon, emissive, atmosphere)
    sh = LayerShards(case, 3, 7)
    try:
        sh.each(enable_all)
        sh.each(lambda r: r.set_sample_offset(5))
        sh.ref_scene.reset_blue_noise()
        for s in sh.scenes: s.reset_blue_noise()
        sh.render(3, iteration=0); sh.check("offset 5", layers=())
        zero = case.renderer(case.scene())
        zero.kp.iteration = 0; zero.render(3); torch.cuda.synchronize()
        assert not same(zero.buffers.accum, sh.ref.buffers.accum)
        zero.close()
    finally:
        sh.close()


# ---- 2: the central guarantee ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["headline", "lights_sphere"])
def test_eight_offset_frames_through_the_filter_are_the_eight_pass_frame(dragon, perlin, name):
    scene, mk, keep = make_case(name, dragon, perlin)
    F = 8
    r = mk()
    r.enable_motion_vectors(r.cam)                          # B == A
    scene.reset_blue_noise()
    hist = ln = None
    for f in range(F):
        r.set_sample_offset(f); r.kp.iteration = 0
        r.render_pass()
        hist, ln, words = r.temporal(r.cam, history=hist, history_len=ln, max_history=F, clip_sigma=INF, display=True)
    torch.cuda.synchronize()
    assert not bool(r.buffers.motion[:, :2].abs().max()) and bool((r.buffers.motion[:, 2] > 0).any())
    assert bool((ln == F).all())
    ref = mk()
    scene.reset_blue_noise(); ref.kp.iteration = 0
    for _ in range(F): ref.render_pass()
    torch.cuda.synchronize()
    assert same(hist.reshape(-1, 3), ref.buffers.accum), name
    assert same(words.reshape(-1), ref.buffers.display.view(torch.int32).reshape(-1)), name


# ---- 3: the kernel against the restatement ---------------------------------------------------------------------------------------------
def look_at(frm, at, w, h, fov=35.0):
    cam = N.camera()
    V.lib.vpt_camera_look_at(C.byref(cam), N.fvec(frm), N.fvec(at), N.fvec((0, 1, 0)), fov, w / h, 0.0)
    return cam


def synthetic(w, h, seed, motion):
    rng = np.random.default_rng(seed)
    n = w * h
    c = rng.uniform(0.0, 2.0, (n, 3)).astype(np.float32)
    hist = rng.uniform(0.0, 2.0, (n, 3)).astype(np.float32)
    ln = rng.integers(1, 12, n).astype(np.float32)
    m = np.zeros((n, 3), np.float32)
    m[:, 2] = rng.choice([0.0, 0.3, 1.0], n)
    if motion == "integer":
        m[:, :2] = rng.integers(-3, 4, (n, 2))
    else:
        m[:, :2] = rng.uniform(-3.0, 3.0, (n, 2))
    m[:, :2] *= m[:, 2:3]                                       # premultiplied
    far = rng.random(n) < 0.05
    m[far, :2] = 1e4                                            # q off the frame
    m[far, 2] = 1.0
    c[rng.random(n) < 0.03] = np.nan
    c[rng.random(n) < 0.02, 1] = np.inf
    hist[rng.random(n) < 0.05] = np.nan
    return c, m, hist, ln


@pytest.mark.parametrize("w,h", [(1, 1), (7, 3), (61, 37)])
@pytest.mark.parametrize("motion", ["fractional", "integer"])
@pytest.mark.parametrize("clip", [INF, 1.5])
def test_the_kernel_matches_the_restatement(dragon, w, h, motion, clip):
    scene = V.Scene([dragon.instance()], env=synthetic_env(64, 32))
    a = look_at((3.0, 2.0, 9.0), (0.2, 0.1, 0.0), w, h)
    b = look_at((3.1, 2.0, 8.9), (0.25, 0.1, 0.0), w, h)
    r = V.Renderer(scene, w, h, cam=a)
    c, m, hist, ln = synthetic(w, h, w * 100 + h, motion)
    dev = r.buffers.accum.device
    t = lambda x: torch.as_tensor(x, device=dev).contiguous()
    out, L, words = r.temporal(b, color=t(c), vectors=t(m), history=t(hist), history_len=t(ln), max_history=8, clip_sigma=clip, display=True)
    torch.cuda.synchronize()
    out, L, words = out.cpu().numpy().reshape(-1, 3), L.cpu().numpy().reshape(-1), words.cpu().numpy().reshape(-1).view(np.uint32)
    # the history is white noise, so a rounding of the motion by 1e-4 pixels moves out by 1e-4: the motion and the footprint in the
    # kernel's float32 order
    ref = T.temporal(w, h, c, m, a, b, hist, ln, max_history=8, clip_sigma=clip, motion_dt=np.float32, footprint_dt=np.float32)
    assert np.array_equal(L.view(np.uint32), ref["L"].astype(np.float32).view(np.uint32)), "history lengths"
    used = ref["used"]
    fails, _ = T.compare(out, ref["out"], c, ~used, ref["M"])       # every pixel: no history => out = C bit for bit
    assert not fails, "; ".join(fails)
    want = T.display_words(out, float(r.kp.exposure_scale))
    for s in (0, 8, 16):
        d = np.abs(((words >> s) & 0xFF).astype(int) - ((want >> s) & 0xFF).astype(int))
        assert d.max() <= 1, s
    if w * h > 100:
        assert used.any() and (~used).any()
    r.close()


def test_no_history_is_the_frame_and_k_resolves_display_word(dragon, perlin):
    scene, mk, keep = make_aov_case("lights_sphere", dragon, perlin)
    r = mk(aovs=False)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(3); torch.cuda.synchronize()
    still = torch.zeros_like(r.buffers.accum)
    out, L, words = r.temporal(r.cam, vectors=still, display=True)
    torch.cuda.synchronize()
    assert same(out.reshape(-1, 3), r.buffers.accum) and bool((L == 1).all())
    assert same(words.reshape(-1), r.buffers.display.view(torch.int32).reshape(-1))


# ---- 4: a moving camera, end to end ----------------------------------------------------------------------------------------------------
def pan_cameras(scene, w, h, n, step_deg):
    lo, hi = scene.world_bounds()
    centre = (hi + lo) / 2
    dist = float(np.linalg.norm(hi - lo))
    cams = []
    for i in range(n):
        ang = np.radians(step_deg * i)
        frm = centre + dist * np.array([np.cos(ang), 0.6, np.sin(ang)])
        cam = N.camera()
        V.lib.vpt_camera_look_at(C.byref(cam), N.fvec(frm.astype(np.float32)), N.fvec(centre.astype(np.float32)), N.fvec((0, 1, 0)), 30.0,
                                 w / h, 0.0)
        cams.append(cam)
    return cams


def test_a_slow_pan_converges_better_than_the_unfiltered_frame(dragon, perlin):
    scene, _, keep = make_case("headline", dragon, perlin)
    w, h, P = 480, 270, 2
    cams = pan_cameras(scene, w, h, 12, 0.5)
    r = V.Renderer(scene, w, h, kp=make_kp(ray_depth=100), cam=copy_cam(cams[0]))
    r.enable_temporal()
    scene.reset_blue_noise()
    for cam in cams:
        out, L = r.render_temporal(cam, P)
    torch.cuda.synchronize()
    raw = r.buffers.accum.reshape(h, w, 3).clone()
    ref = V.Renderer(scene, w, h, kp=make_kp(ray_depth=100), cam=copy_cam(cams[-1]))
    ref.set_sample_offset(1 << 20); ref.kp.iteration = 0; ref.render(512); torch.cuda.synchronize()
    want = ref.buffers.accum.reshape(h, w, 3)
    rmse = lambda x: float(torch.sqrt(((x - want) ** 2).mean()))
    e_t, e_raw = rmse(out), rmse(raw)
    print(f"[temporal pan] RMSE filtered {e_t:.5f} unfiltered {e_raw:.5f} ratio {e_raw / e_t:.3f}, mean L {float(L.mean()):.2f}")
    assert e_t < e_raw
    r.disable_temporal()


# ---- 5: refusals -----------------------------------------------------------------------------------------------------------------------
def test_refusals(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(64, 32))
    w, h = 16, 8
    r = V.Renderer(scene, w, h)
    dev = r.buffers.accum.device
    c = torch.zeros(w * h, 3, device=dev); m = torch.zeros(w * h, 3, device=dev)
    hist = torch.zeros(w * h, 3, device=dev); ln = torch.ones(w * h, device=dev)
    launches = r.stats()[0]

    def refused(match, **kw):
        args = dict(color=c, vectors=m, history=hist, history_len=ln)
        args.update(kw)
        with pytest.raises(V.VptError, match=match):
            r.temporal(r.cam, **args)
    refused("both be set", history_len=None)
    refused("both be set", history=None)
    refused("max_history", max_history=0)
    refused("max_history", max_history=(1 << 24) + 1)
    for s in (float("nan"), 0.0, -1.0):
        refused("clip_sigma", clip_sigma=s)
    refused("d_out_f3 overlaps d_color_f3", out=c)
    refused("d_out_f3 overlaps d_history_f3", out=hist)
    refused("d_out_len overlaps d_history_len", out_len=ln)
    buf = torch.zeros(w * h * 3, device=dev)
    refused("d_out_f3 overlaps d_out_len", out=buf, out_len=buf[: w * h])
    bad = copy_cam(r.cam); bad.vertical.y = float("inf")
    with pytest.raises(V.VptError, match="previous.vertical"):
        r.temporal(bad, color=c, vectors=m)
    ctx_args = (None, None, C.byref(r.cam), C.byref(r.cam), None, None, None, 1.0, C.c_void_p(ln.data_ptr()), C.c_void_p(c.data_ptr()), None, None)
    assert V.lib.vpt_temporal(r.ctx, 0, h, C.c_void_p(c.data_ptr()), C.c_void_p(m.data_ptr()), *ctx_args[2:]) == -1
    assert V.lib.vpt_temporal(r.ctx, 65536, 1, C.c_void_p(c.data_ptr()), C.c_void_p(m.data_ptr()), *ctx_args[2:]) == -1
    assert V.lib.vpt_temporal(r.ctx, w, h, None, C.c_void_p(m.data_ptr()), *ctx_args[2:]) == -1
    torch.cuda.synchronize()
    assert r.stats()[0] == launches, "a refused call enqueued work"
    r.temporal(r.cam, color=c, vectors=m, history=hist, history_len=ln)
    assert r.stats()[0] == launches + 1
    r.close()
