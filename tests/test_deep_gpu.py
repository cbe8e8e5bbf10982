"""Deep slices on the GPU (vpt_set_deep_buffers): the compositing AOVs binned by the camera sample's depth, kept by k_resolve next to accum
(include/vpt_b200.h, DESIGN.md section 8h).

The cases of test_aov_gpu.py -- the headline frame (compact records), lights + sphere + thin lens (wide records), the volumetric path
integrator on the tabulated sky, the Bruneton sky, 120 instances, brick and cell mode -- plus the NaN / Inf environment stripes, whose
samples the guard replaces.  Every frame is 8 passes in chunks of 5 + 3."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import deep
from vpt_b200.renderer import stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
from deep_ref import slice_of
from test_adaptive_gpu import CASES as ADAPTIVE_CASES, make_case
from test_aov_gpu import make_aov_case, NAMES
from test_parity_gpu import make_kp
from test_projection_gpu import headline_pano

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
AOVS = ("alpha", "volume")
PASSES = 8                     # in chunks of 5 + 3 (passes_per_chunk = 5)
INF = float("inf")
ALL = [0.0, INF]               # one slice: the AOVs
SENTINEL = 0x7FBADBAD
GROUPS_TOO = ("lights_sphere", "vol_sky_table")      # cases that also run the light groups


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


@pytest.fixture(scope="module")
def cases(dragon, perlin):
    cache = {}
    def get(name):
        if name not in cache: cache[name] = make_aov_case(name, dragon, perlin)
        return cache[name]
    return get


def pattern(K, n, k0, device):
    """(K, n, 4) previous content of slices k0 .. k0 + K - 1: from the slice index and the pixel, multiples of 1/1024 (exact in float32)"""
    j = torch.arange(K, device=device).view(K, 1, 1) + k0
    i = torch.arange(n, device=device).view(1, n, 1)
    c = torch.arange(4, device=device).view(1, 1, 4)
    return ((i * 7 + j * 131 + c * 17) % 4093 + 1).float() / 1024


def run(scene, r, passes=PASSES, single=False, fill=None, k0=0):
    """a new frame of `passes` passes (8 single-pass calls with single=True).  The buffers start from non-zero content, which a sample the
    guard replaces at iteration 0 keeps: the case's prefill (nan_prefilled), the AOVs and slice j from pattern(.., k0 + j) -- so the one
    slice of the frame of interval k (k0 = k) starts from what slice k of a frame of every interval does.  fill: the slice buffer's
    words instead."""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    b, dev = r.buffers, r.buffers.accum.device
    before = None
    if hasattr(r, "prefill"):
        r.prefill(); before = b.accum.clone()
    if b.volume is not None:
        first = pattern(1, r.n_local, k0, dev)[0]
        b.volume.copy_(first[:, :3]); b.alpha.copy_(first[:, 3])
    if b.deep is not None:
        if fill is not None: b.deep.view(torch.int32).fill_(fill)
        else: b.deep.copy_(pattern(b.deep.shape[0], r.n_local, k0, dev))
    if single:
        for _ in range(passes): r.render_pass()
    else:
        r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS + AOVS + ("deep",) if getattr(r.buffers, k) is not None}
    if r.buffers.groups: out.update({"group_" + g: t.clone() for g, t in r.buffers.groups.items()})
    out["blue_noise"] = scene.d_blue_noise.clone()
    if before is not None: out["accum_before"] = before
    return out


def bitwise(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def depth_bounds(scene, mk, K=16):
    """K + 1 non-uniform bounds inside the frame's depth range (quantiles 5 % .. 95 % of one pass's hit depths): z_0 > 0, z_K finite"""
    f = run(scene, mk(), 1)
    d = f["depth"].cpu().numpy()
    d = d[d > 0]
    q = 0.05 + 0.9 * (np.arange(K + 1) / K) ** 1.5
    z = np.unique(np.quantile(d, q).astype(np.float32))
    assert len(z) == K + 1, z
    return [float(v) for v in z]


def mk_deep(mk, bounds, groups=False):
    r = mk()
    if groups: r.enable_light_groups()
    r.enable_deep(bounds)
    return r


@pytest.mark.parametrize("name", NAMES + ["nan_prefilled"])
def test_slices_interfere_with_nothing_and_one_slice_is_the_aovs(cases, name):
    """(1) accum, depth, cost, raw, display, the blue noise, the AOVs and the light groups are bit-identical with the slices off and on;
    (2) K = 1 with {0, inf} is (volume, alpha) bit for bit; (5) the fused 5 + 3 chunks give the slices of 8 single-pass calls, and two
    identical frames give identical slices."""
    scene, mk, _ = cases(name)
    groups = name in GROUPS_TOO
    off_r = mk()
    if groups: off_r.enable_light_groups()
    off = run(scene, off_r)
    r = mk_deep(mk, ALL, groups)
    on = run(scene, r)
    assert r.stats()[0] - off_r.stats()[0] == 2, "one more resolve kernel per chunk (5 + 3) with the slices on"
    for k in off:
        assert bitwise(on[k], off[k]), f"{name}: {k} changes when the slices are on"
    assert float(on["accum"].mean()) > 1e-3 and 0.0 < float(on["alpha"].mean()) < 1.0, "the frame must show volume and background"
    s = on["deep"][0]
    assert bitwise(s[:, :3], on["volume"]), f"{name}: the colour of the one slice {{0, inf}} is not the volume AOV"
    assert bitwise(s[:, 3], on["alpha"]), f"{name}: the coverage of the one slice {{0, inf}} is not alpha"
    single = run(scene, mk_deep(mk, ALL, groups), single=True)
    again = run(scene, r)
    assert bitwise(single["deep"], on["deep"]), f"{name}: 8 single passes differ from the fused 5 + 3 chunks"
    assert bitwise(again["deep"], on["deep"]), f"{name}: two identical frames differ"


@pytest.mark.parametrize("name", ["headline", "lights_sphere", "vol_sky_table", "nan_prefilled"])
def test_each_slice_is_the_frame_of_its_own_interval(cases, name):
    """(3) K = 16 non-uniform bounds inside the depth range, z_0 > 0 and z_K finite: slice k is bit for bit the one slice of a K = 1 frame
    with bounds {z_k, z_{k+1}}, each slice starting from its own previous content; (4) after one pass, slice k is exactly
    (in_k(depth) ? accum : 0, in_k(depth)) -- and where the guard replaced the sample (nan_prefilled: accum kept its prefill), (its previous
    content, in_k(depth))."""
    scene, mk, _ = cases(name)
    b = depth_bounds(scene, mk)
    r = mk_deep(mk, b)
    f = run(scene, r)
    d1 = run(scene, mk(), 1)["depth"].cpu().numpy()
    outside = (d1 > 0) & (slice_of(d1, b) < 0)
    assert outside.any(), "some hits must fall outside every slice"
    one = mk_deep(mk, b[:2])
    for k in range(len(b) - 1):
        one.enable_deep(b[k:k + 2])
        g = run(scene, one, k0=k)
        assert bitwise(g["deep"][0], f["deep"][k]), f"{name}: slice {k} differs from the frame of [{b[k]}, {b[k + 1]})"
        assert float(f["deep"][k][:, 3].max()) > 0.0, f"{name}: slice {k} is empty"

    # one pass: the NumPy binning of depth_buffer selects accum; a bound set with an open end and z_0 = 0 as well
    for bb in (b, [0.0] + b[1:-1] + [INF]):
        r1 = mk_deep(mk, bb)
        o = run(scene, r1, 1)
        depth, accum = o["depth"].cpu().numpy(), o["accum"].cpu().numpy()
        sl = slice_of(depth, bb)
        got = o["deep"].cpu().numpy()
        prev = pattern(len(bb) - 1, r1.n_local, 0, r1.buffers.accum.device).cpu().numpy()
        guarded = np.zeros(len(depth), bool)
        if "accum_before" in o:
            guarded = (o["accum_before"].cpu().numpy().view(np.int32) == accum.view(np.int32)).all(1)
            assert guarded.any() and (~guarded).any() and (guarded & (sl >= 0)).any(), "the frame must have guarded samples in slices"
        for k in range(len(bb) - 1):
            ink = sl == k
            assert (got[k][:, 3] == ink.astype(np.float32)).all(), f"{name}: coverage of slice {k} after one pass"
            want = np.where(guarded[:, None], prev[k][:, :3], np.where(ink[:, None], accum, np.float32(0.0)))
            assert np.array_equal(got[k][:, :3].view(np.int32), want.view(np.int32)), f"{name}: colour of slice {k} after one pass"


@pytest.mark.parametrize("name", ["headline", "vol_sky_table"])
def test_slices_sum_to_the_aovs(cases, name):
    """(6) with z_0 = 0 and z_K = +inf the slices sum to (volume, alpha).  Bound: each of the K + 1 running means (K slices, one AOV) is
    within 4 n eps M of the exact mean of its float32 samples after n passes -- every pass rounds the difference, the fast-math quotient
    (2 ulp) and the sum, each at most eps relative to max(|x|, |s|) <= M, the largest sample -- and the samples are non-negative, so
    M <= n * (the pixel's exact mean), which is within rounding of the AOV.  So |sum_k slice_k - aov| <= (K + 2) * 4 n^2 eps * max(aov,
    max_k slice_k), the extra term for the float32 sum.  deep.exr_samples composited with the deep 'over' gives back those sums too."""
    scene, mk, _ = cases(name)
    b = [0.0] + depth_bounds(scene, mk, K=14) + [INF]
    K, n, eps = len(b) - 1, PASSES, 2.0 ** -24
    r = mk_deep(mk, b)
    f = run(scene, r)
    s = f["deep"].double()
    aov = torch.cat([f["volume"], f["alpha"][:, None]], 1).double()
    scale = torch.maximum(aov.abs(), s.abs().amax(0))
    err = (s.sum(0) - aov).abs()
    tol = (K + 2) * 4 * n * n * eps * scale
    assert bool((err <= tol).all()), f"{name}: worst excess {float((err - tol).max())}"

    # the OpenEXR deep samples of the slices, flattened with 'over' (float64, vectorised over pixels)
    H, W = r.height, r.width
    img = f["deep"].view(K, H, W, 4)
    e = deep.exr_samples(img, b)
    count = e.count.reshape(-1)
    first = torch.cumsum(count, 0) - count
    pix = torch.repeat_interleave(torch.arange(H * W, device=count.device), count)
    pos = torch.arange(len(pix), device=count.device) - first[pix]
    A = torch.zeros(H * W, K, dtype=torch.float64, device=count.device); A[pix, pos] = e.a.double()
    RGB = torch.zeros(H * W, K, 3, dtype=torch.float64, device=count.device); RGB[pix, pos] = e.rgb.double()
    col, t = torch.zeros(H * W, 3, dtype=torch.float64, device=count.device), torch.ones(H * W, dtype=torch.float64, device=count.device)
    for k in range(K):
        col += t[:, None] * RGB[:, k]
        t *= 1.0 - A[:, k]
    fc, fa = deep.flatten(img, b)
    assert torch.allclose(col, fc.reshape(-1, 3).double(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(1.0 - t, fa.reshape(-1).double(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(fc.reshape(-1, 3).double(), s.sum(0)[:, :3], rtol=1e-5, atol=1e-6)


def test_equirect_slices_with_and_without_the_miss_cull(dragon):
    """(2) in an equirectangular panorama with the miss cull, K = 1 with {0, inf} is (volume, alpha) bit for bit; every slice of K = 8 is
    the same with and without the cull."""
    scene, mk = headline_pano(dragon, 512, 256, aovs=True)
    r = mk(1); r.enable_deep(ALL)
    f = run(scene, r)
    assert bitwise(f["deep"][0][:, :3], f["volume"]) and bitwise(f["deep"][0][:, 3], f["alpha"])
    d = f["depth"].cpu().numpy(); d = d[d > 0]
    b = [float(v) for v in np.unique(np.quantile(d, np.linspace(0.0, 1.0, 9) ** 0.7).astype(np.float32))]
    b[0] = 0.0; b[-1] = INF
    culled, kept = mk(1), mk(0)
    culled.enable_deep(b); kept.enable_deep(b)
    a, c = run(scene, culled), run(scene, kept)
    assert float(a["alpha"].mean()) < 0.2, "most of the panorama must be culled"
    for k in ("deep", "accum", "alpha", "volume"):
        assert bitwise(a[k], c[k]), k


@pytest.mark.parametrize("name,W,H,mx,mn,iv,thr", [
    ("headline", 320, 200, 48, 8, 8, 0.05),
    ("vol_sky_table",) + ADAPTIVE_CASES["vol_sky_table"],
])
def test_adaptive_frame_slices_equal_the_fixed_count_frames(dragon, perlin, name, W, H, mx, mn, iv, thr):
    """(7) every pixel's slices (and buffers) equal those of a fixed-count frame of its own pass count, class by class."""
    if name == "headline":
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        cam = scene.frame_camera(W, H)
        mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=100), cam=cam)
    else:
        scene, mk, keep = make_case(name, dragon, perlin)
    b = [0.0] + depth_bounds(scene, mk, K=6) + [INF]
    r, f = mk(), mk()
    r.enable_deep(b); f.enable_deep(b)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    run_, counts = r.render_adaptive(mx, threshold=thr, min_passes=mn, check_interval=iv)
    torch.cuda.synchronize()
    got = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    got["deep"] = r.buffers.deep.clone()
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert len(classes) >= 2 and run_ == max(classes)
    for c in classes:
        f.reset(); f.render(c); torch.cuda.synchronize()
        m = flat == c
        for k in BUFFERS:
            assert torch.equal(got[k][m], getattr(f.buffers, k)[m]), f"{k} differs on the {int(m.sum())} pixels of {c} passes"
        assert bitwise(got["deep"][:, m], f.buffers.deep[:, m]), f"the slices differ on the {int(m.sum())} pixels of {c} passes"


def test_region_writes_no_slice_outside_it(cases):
    """(8) with a render region R the slices inside R equal the full frame's; a sentinel outside R survives."""
    scene, mk, _ = cases("headline")
    b = [0.0] + depth_bounds(scene, mk, K=6) + [INF]
    full = run(scene, mk_deep(mk, b))
    r = mk_deep(mk, b)
    x0, y0, x1, y1 = 301, 203, 1100, 707
    r.set_region(x0, y0, x1, y1)
    got = run(scene, r, fill=SENTINEL)
    H, W = r.height, r.width
    K = len(b) - 1
    g, w = got["deep"].view(K, H, W, 4), full["deep"].view(K, H, W, 4)
    assert bitwise(g[:, y0:y1, x0:x1], w[:, y0:y1, x0:x1])
    inside = torch.zeros(H, W, dtype=torch.bool, device=g.device); inside[y0:y1, x0:x1] = True
    assert bool((g.view(torch.int32)[:, ~inside] == SENTINEL).all()), "a slice was written outside the region"


def test_partitioned_contexts_keep_rank_local_slices(dragon):
    """(9) four shards on one GPU: each shard's rank-local slice rows equal the single-context rows."""
    W, H, R, SR = 320, 200, 4, 8
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    b = [0.0, 20.0, 30.0, 35.0, 40.0, 50.0, INF]
    K = len(b) - 1
    one = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4))
    one.enable_deep(b)
    full = run(scene, one, 3)["deep"].view(K, H, W, 4)
    assert float(full[..., 3].sum()) > 0.0
    for rank in range(R):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=one.cam, rank=rank, n_ranks=R, stripe_rows=SR)
        r.enable_deep(b)
        run(scene, r, 3)
        rows = stripe_rows_of_rank(H, rank, R, SR)
        assert r.deep_image().shape == (K, len(rows), W, 4)
        own = torch.as_tensor(np.nonzero(rows < H)[0], device=full.device)
        glob = torch.as_tensor(rows[rows < H], device=full.device)
        assert bitwise(r.deep_image()[:, own], full[:, glob]), f"rank {rank}"
        r.close()


def test_activation_switch_off_and_refusals(dragon):
    """(10) slices enabled mid-frame stay untouched until the next iteration-0 call; a NULL buffer stops at once; passes beyond
    max_interactions change nothing; every bad slice count or bound is refused when set; every overlap is refused at render time,
    naming the buffer."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda **kw: V.Renderer(scene, W, H, kp=make_kp(ray_depth=4, **kw), cam=cam)
    b = [0.0, 25.0, 35.0, INF]
    ref = mk(); ref.enable_deep(b)
    want = run(scene, ref, 3)

    r = mk()
    with pytest.raises(V.VptError, match="not enabled"):
        r.deep_image()
    scene.reset_blue_noise(); r.render(2)
    r.enable_deep(b)
    r.buffers.deep.fill_(7.0)
    r.render(2); torch.cuda.synchronize()                                      # iteration 2: not active yet
    assert bool((r.buffers.deep == 7.0).all())
    got = run(scene, r, 3)                                                     # iteration 0: active from here on
    assert bitwise(got["deep"], want["deep"]) and bitwise(got["accum"], want["accum"])
    assert r.deep_image().shape == (3, H, W, 4)

    r.disable_deep()
    r.buffers.deep.fill_(7.0)
    r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.deep == 7.0).all())
    r.kp.iteration = 0
    r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.deep == 7.0).all()), "a NULL buffer must stay off at iteration 0 too"

    # passes beyond max_interactions change nothing
    capped = mk(max_interactions=2); capped.enable_deep(b)
    two = run(scene, capped, 2)
    capped.render(3); torch.cuda.synchronize()
    assert bitwise(capped.buffers.deep, two["deep"])

    # refused when set; a refused call leaves the registered slices as they were
    n = W * H
    buf = torch.zeros(32 * n * 4 + 4, dtype=torch.float32, device=r.buffers.accum.device)
    bad = [(0, [0.0]), (33, [float(i) for i in range(34)]), (2, None), (2, [0.0, float("nan"), 2.0]), (2, [-1.0, 1.0, 2.0]),
           (2, [0.0, 2.0, 2.0]), (2, [0.0, 3.0, 2.0]), (2, [0.0, INF, INF]), (2, [INF, 1.0, 2.0])]
    z = mk(); z.enable_deep(b)
    for k, bounds in bad:
        arr = (C.c_float * len(bounds))(*bounds) if bounds is not None else None
        assert V.lib.vpt_set_deep_buffers(z.ctx, C.c_void_p(buf.data_ptr()), k, arr) == -1, (k, bounds)
        assert V.lib.vpt_last_error(z.ctx).startswith(b"vpt_set_deep_buffers")
    one_b = (C.c_float * 2)(0.0, INF)
    assert V.lib.vpt_set_deep_buffers(z.ctx, C.c_void_p(buf.data_ptr() + 4), 1, one_b) == -1
    assert b"16-byte aligned" in V.lib.vpt_last_error(z.ctx)
    with pytest.raises(V.VptError):
        z.enable_deep([1.0, 1.0])
    assert bitwise(run(scene, z, 3)["deep"], want["deep"])
    assert V.lib.vpt_set_deep_buffers(z.ctx, None, 99, None) == 0                 # NULL: K and bounds ignored

    # overlaps: the Kernel_params buffers of `o` sit 64 bytes per pixel apart in one arena, and the AOV and group buffers in another, so a
    # one-slice buffer (16 bytes per pixel) that starts on the last 16 bytes of one of them overlaps that buffer and nothing else (every
    # size is a multiple of 16 bytes here, so the start stays 16-byte aligned)
    o = mk()
    dev = o.buffers.accum.device
    arena = torch.zeros(5 * 16 * n, dtype=torch.float32, device=dev)
    size = {"accum_buffer": 12 * n, "depth_buffer": 4 * n, "cost_buffer": 12 * n, "raw_buffer": 16 * n, "display_buffer": 4 * n}
    for i, name in enumerate(size):
        setattr(o.kp, name, arena.data_ptr() + i * 64 * n)
    layers = torch.zeros(7 * 16 * n, dtype=torch.float32, device=dev)
    lp = [layers.data_ptr() + i * 64 * n for i in range(6)]
    V._native.check(V.lib.vpt_set_aov_buffers(o.ctx, C.c_void_p(lp[0]), C.c_void_p(lp[1])), o.ctx, "vpt_set_aov_buffers")
    V._native.check(V.lib.vpt_set_light_group_buffers(o.ctx, *[C.c_void_p(p) for p in lp[2:]]), o.ctx, "vpt_set_light_group_buffers")
    one = (C.c_float * 2)(0.0, INF)
    assert n % 4 == 0
    refusals = [(getattr(o.kp, name) + size[name] - 16, f"slice buffer overlaps Kernel_params.{name}") for name in size]
    refusals += [(lp[0] + 4 * n - 16, "slice buffer overlaps the alpha AOV buffer"), (lp[1] + 12 * n - 16, "slice buffer overlaps the volume AOV buffer")]
    refusals += [(lp[2 + i] + 12 * n - 16, f"slice buffer overlaps the {g} light-group buffer") for i, g in enumerate(V.LIGHT_GROUPS)]
    for p, msg in refusals:
        V._native.check(V.lib.vpt_set_deep_buffers(o.ctx, C.c_void_p(p), 1, one), o.ctx, "vpt_set_deep_buffers")
        o.kp.iteration = 0
        with pytest.raises(V.VptError, match=msg):
            o.render(1)
    free = torch.zeros(n, 4, dtype=torch.float32, device=dev)
    V._native.check(V.lib.vpt_set_deep_buffers(o.ctx, C.c_void_p(free.data_ptr()), 1, one), o.ctx, "vpt_set_deep_buffers")
    o.kp.iteration = 0
    o.render(1); torch.cuda.synchronize()                                     # a disjoint buffer renders
    assert float(free[:, 3].max()) == 1.0
