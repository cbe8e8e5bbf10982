"""Compositing AOVs on the GPU (vpt_set_aov_buffers): alpha = running mean of [depth > 0], volume = running mean of the sample where
depth > 0 and +0 elsewhere, kept by k_resolve next to accum (include/vpt_b200.h, DESIGN.md section 8c).

Every record layout and resolve variant: the headline frame (compact records), lights + sphere + thin lens (wide records, generic
kernel), the volumetric path integrator (k_resolve<2>), the Bruneton sky with the direct integrator (k_resolve<1>), 120 instances
(2 rays per lane), brick mode and cell mode."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.renderer import stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
from test_adaptive_gpu import CASES as ADAPTIVE_CASES, make_case
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
AOVS = ("alpha", "volume")
PASSES = 8                     # in chunks of 5 + 3 (passes_per_chunk = 5)


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


def make_aov_case(name, dragon, perlin):
    """-> (scene, make_renderer(), keep-alive objects); every renderer fuses at most 5 passes per chunk"""
    if name in ADAPTIVE_CASES:
        scene, mk0, keep = make_case(name, dragon, perlin)
    elif name == "sky":                                          # direct integrator on the precomputed Bruneton sky: k_resolve<1>
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        atm = V.Atmosphere(); atm.apply(scene.atmos)
        cam = scene.frame_camera(200, 120)
        scene, mk0, keep = scene, (lambda: V.Renderer(scene, 200, 120, kp=make_kp(environment_type=0, elevation=25.0, ray_depth=2), cam=cam)), [atm]
    elif name == "cells":                                        # cell mode, as test_hdri_records_gpu.py's `cells` case
        scene = V.Scene([perlin.instance()], env=synthetic_env(512, 256), keep=[perlin])
        cam = scene.frame_camera(64, 36)
        def mk0():
            r = V.Renderer(scene, 64, 36, kp=make_kp(ray_depth=100), cam=cam)
            r.set_cell_volume(perlin)
            return r
        keep = []
    else:
        raise KeyError(name)

    def mk(aovs=True):
        r = mk0()
        r.set_option("passes_per_chunk", 5)
        if aovs: r.enable_aovs()
        return r
    return scene, mk, keep


NAMES = ["headline", "lights_sphere", "vol_sky_table", "sky", "instanced", "brick", "cells"]


@pytest.fixture(scope="module")
def cases(dragon, perlin):
    cache = {}
    def get(name):
        if name not in cache: cache[name] = make_aov_case(name, dragon, perlin)
        return cache[name]
    return get


def frame(scene, r, passes, pass_by_pass=False):
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if pass_by_pass:
        for _ in range(passes): r.render_pass()
    else:
        r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS + AOVS if getattr(r.buffers, k) is not None}
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def bitwise(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("name", NAMES)
def test_aovs_interfere_with_nothing_and_fuse_like_single_passes(cases, name):
    """(1) accum, depth, cost, raw, display and the blue noise are bit-identical with AOVs off and on; (6) the fused 5 + 3 chunks give
    the AOVs of 8 single-pass calls, bit for bit; (10) two identical frames give identical AOVs."""
    scene, mk, _ = cases(name)
    off = frame(scene, mk(aovs=False), PASSES)
    r = mk()
    on = frame(scene, r, PASSES)
    for k in BUFFERS + ("blue_noise",):
        assert bitwise(on[k], off[k]), f"{name}: {k} changes when the AOVs are on"
    assert float(on["accum"].mean()) > 1e-3 and 0.0 < float(on["alpha"].mean()) < 1.0, "the frame must show volume and background"
    single = frame(scene, mk(), PASSES, pass_by_pass=True)
    again = frame(scene, r, PASSES)
    for k in AOVS:
        assert bitwise(single[k], on[k]), f"{name}: {k} of 8 single passes differs from the fused 5 + 3 chunks"
        assert bitwise(again[k], on[k]), f"{name}: {k} differs between two identical frames"
    assert bitwise(single["accum"], on["accum"])


@pytest.mark.parametrize("name", NAMES)
def test_one_pass_frame(cases, name):
    """(2) after one pass, alpha == (depth > 0) and volume == (depth > 0 ? accum : 0), exactly."""
    scene, mk, _ = cases(name)
    out = frame(scene, mk(), 1)
    hit = out["depth"] > 0
    assert bitwise(out["alpha"], hit.float())
    assert torch.equal(out["volume"], torch.where(hit[:, None], out["accum"], torch.zeros_like(out["accum"])))
    assert bool(hit.any()) and not bool(hit.all())


def constant_env_renderer(dragon, value, W=320, H=200, **kw):
    env = np.full((64, 128, 4), value, np.float32)
    scene = V.Scene([dragon.instance()], env=env)
    sp = scene.h_sphere; sp.center = V.f3(0.0, 1e6, 0.0); sp.radius = 1.0        # far out of view
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=100, **kw))
    r.enable_aovs()
    return scene, r


def test_black_environment_volume_is_the_beauty(dragon):
    """(3) with nothing behind the volume, volume == accum bit for bit after 16 passes."""
    scene, r = constant_env_renderer(dragon, 0.0)
    assert r.cam.viz_dof == 0
    out = frame(scene, r, 16)
    assert float(out["accum"].max()) > 1e-3
    assert bitwise(out["volume"], out["accum"])


def test_constant_environment_composites_back_to_the_beauty(dragon):
    """(4) under a constant environment of miss radiance k: accum = volume + (1 - alpha) k up to float rounding."""
    E = 2.0
    scene, r = constant_env_renderer(dragon, E)
    out = frame(scene, r, 16)
    k = (np.float32(E) * np.array([r.kp.sky_color.x, r.kp.sky_color.y, r.kp.sky_color.z], np.float32) *
         np.float32(1.0 / (4.0 * np.pi))).astype(np.float64)
    accum, vol, alpha = (out[n].cpu().numpy().astype(np.float64) for n in ("accum", "volume", "alpha"))
    miss = alpha == 0
    assert miss.any() and (alpha > 0).any()
    assert np.allclose(accum[miss], k, rtol=1e-5, atol=0)                          # the background alone is k
    comp = vol + (1.0 - alpha)[:, None] * k
    err = np.abs(comp - accum)
    assert (err <= 1e-5 * (np.abs(accum) + k.max())).all(), float(err.max())


def test_alpha_against_the_numpy_restatement(dragon):
    """(5) pass by pass with depth_buffer zeroed before each pass, depth_buffer > 0 is the pass's indicator; alpha is their running mean
    restated in float32 (1e-6: fast-math division), exactly 0 / 1 where every indicator is 0 / 1.  The medium is made dense enough
    that rays into the dragon's body collide in every pass."""
    W, H, P = 320, 200, 16
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=100, density_mult=50.0))
    r.enable_aovs()
    scene.reset_blue_noise()
    ind = np.empty((P, W * H), np.float32)
    for p in range(P):
        r.buffers.depth.zero_()
        r.render_pass(); torch.cuda.synchronize()
        ind[p] = (r.buffers.depth.cpu().numpy() > 0).astype(np.float32)
    got = r.buffers.alpha.cpu().numpy()
    want = ind[0].copy()
    for p in range(1, P):
        want = want + (ind[p] - want) / np.float32(p + 1)
    assert want.dtype == np.float32
    assert np.abs(got - want).max() <= 1e-6
    none, every = ind.max(axis=0) == 0, ind.min(axis=0) == 1
    assert none.any() and every.any() and ((~none) & (~every)).any()
    assert (got[none] == 0).all() and (got[every] == 1).all()


@pytest.mark.parametrize("name,W,H,mx,mn,iv,thr", [
    ("headline", 320, 200, 48, 8, 8, 0.05),
    ("vol_sky_table",) + ADAPTIVE_CASES["vol_sky_table"],
])
def test_adaptive_frame_aovs_equal_the_fixed_count_frames(dragon, perlin, name, W, H, mx, mn, iv, thr):
    """(7) every pixel's AOVs (and buffers) equal those of a fixed-count frame of its own pass count, class by class."""
    if name == "headline":
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        cam = scene.frame_camera(W, H)
        mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=100), cam=cam)
    else:
        scene, mk, keep = make_case(name, dragon, perlin)
    r, f = mk(), mk()
    r.enable_aovs(); f.enable_aovs()
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    run, counts = r.render_adaptive(mx, threshold=thr, min_passes=mn, check_interval=iv)
    torch.cuda.synchronize()
    got = {k: getattr(r.buffers, k).clone() for k in BUFFERS + AOVS}
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert len(classes) >= 2 and run == max(classes)
    for c in classes:
        f.reset(); f.render(c); torch.cuda.synchronize()
        m = flat == c
        for k in BUFFERS + AOVS:
            assert torch.equal(got[k][m], getattr(f.buffers, k)[m]), f"{k} differs on the {int(m.sum())} pixels of {c} passes"


def test_partitioned_contexts_keep_rank_local_aovs(dragon):
    """(8) four shards on one GPU: each shard's rank-local AOV rows equal the single-context rows."""
    W, H, R, SR = 320, 200, 4, 8
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    one = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4))
    one.enable_aovs()
    full = frame(scene, one, 3)
    for rank in range(R):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=one.cam, rank=rank, n_ranks=R, stripe_rows=SR)
        r.enable_aovs()
        part = frame(scene, r, 3)
        rows = stripe_rows_of_rank(H, rank, R, SR)
        assert r.alpha_image().shape == (len(rows), W) and r.volume_image().shape == (len(rows), W, 3)
        own = torch.as_tensor(np.nonzero(rows < H)[0], device=one.buffers.accum.device)       # local rows inside the frame
        glob = torch.as_tensor(rows[rows < H], device=own.device)
        assert torch.equal(r.alpha_image()[own], full["alpha"].view(H, W)[glob]), f"rank {rank}: alpha"
        assert torch.equal(r.volume_image()[own], full["volume"].view(H, W, 3)[glob]), f"rank {rank}: volume"
        r.close()


def test_activation_switch_off_and_refusals(dragon):
    """(9) AOVs enabled mid-frame stay untouched until the next iteration-0 call; NULL / NULL turns them off at once; every overlap is
    refused, naming the buffer."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda **kw: V.Renderer(scene, W, H, kp=make_kp(ray_depth=4, **kw), cam=cam)
    ref = mk(); ref.enable_aovs()
    want = frame(scene, ref, 3)

    r = mk()
    scene.reset_blue_noise(); r.render(2)
    r.enable_aovs()
    r.buffers.alpha.fill_(7.0); r.buffers.volume.fill_(-3.0)
    r.render(2); torch.cuda.synchronize()                                      # iteration 2: not active yet
    assert bool((r.buffers.alpha == 7.0).all()) and bool((r.buffers.volume == -3.0).all())
    got = frame(scene, r, 3)                                                  # iteration 0: active from here on
    for k in AOVS + ("accum",):
        assert bitwise(got[k], want[k]), k

    r.disable_aovs()
    r.buffers.alpha.fill_(7.0); r.buffers.volume.fill_(-3.0)
    r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.alpha == 7.0).all()) and bool((r.buffers.volume == -3.0).all())
    r.kp.iteration = 0
    r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.alpha == 7.0).all()) and bool((r.buffers.volume == -3.0).all()), "NULL / NULL must stay off at iteration 0 too"

    check = V._native.check
    # one AOV alone
    a_only = mk()
    alone = torch.zeros_like(want["alpha"])
    check(V.lib.vpt_set_aov_buffers(a_only.ctx, C.c_void_p(alone.data_ptr()), None), a_only.ctx, "vpt_set_aov_buffers")
    frame(scene, a_only, 3)
    assert bitwise(alone, want["alpha"])

    # passes beyond max_interactions change nothing
    capped = mk(max_interactions=2); capped.enable_aovs()
    two = frame(scene, capped, 2)
    capped.render(3); torch.cuda.synchronize()
    assert bitwise(capped.buffers.alpha, two["alpha"]) and bitwise(capped.buffers.volume, two["volume"])

    # overlaps: the Kernel_params buffers of `z` sit 64 bytes per pixel apart in one arena, so an AOV buffer that starts on the last
    # word of one of them overlaps that buffer and nothing else
    n = W * H
    z = mk()
    dev = z.buffers.accum.device
    arena = torch.zeros(5 * 16 * n, dtype=torch.float32, device=dev)
    size = {"accum_buffer": 12 * n, "depth_buffer": 4 * n, "cost_buffer": 12 * n, "raw_buffer": 16 * n, "display_buffer": 4 * n}
    for i, name in enumerate(size):
        setattr(z.kp, name, arena.data_ptr() + i * 64 * n)
    spare = torch.zeros(4 * n, dtype=torch.float32, device=dev)
    other_a = torch.zeros(n, dtype=torch.float32, device=dev)
    other_v = torch.zeros(n, 3, dtype=torch.float32, device=dev)
    refusals = []
    for name in size:
        last = getattr(z.kp, name) + size[name] - 4
        refusals.append((last, other_v.data_ptr(), f"alpha buffer overlaps Kernel_params.{name}"))
        refusals.append((other_a.data_ptr(), last, f"volume buffer overlaps Kernel_params.{name}"))
    refusals.append((spare.data_ptr(), spare.data_ptr() + 4 * (n - 1), "alpha buffer and the volume buffer overlap"))
    for pa, pv, msg in refusals:
        check(V.lib.vpt_set_aov_buffers(z.ctx, C.c_void_p(pa), C.c_void_p(pv)), z.ctx, "vpt_set_aov_buffers")
        z.kp.iteration = 0
        with pytest.raises(V.VptError, match=msg):
            z.render(1)
    check(V.lib.vpt_set_aov_buffers(z.ctx, C.c_void_p(other_a.data_ptr()), C.c_void_p(other_v.data_ptr())), z.ctx, "vpt_set_aov_buffers")
    z.kp.iteration = 0
    z.render(1); torch.cuda.synchronize()                                     # disjoint buffers render
    assert float(other_a.max()) == 1.0
