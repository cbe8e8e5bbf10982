"""The Cryptomatte on the GPU (vpt_set_cryptomatte, vpt_cryptomatte_rank): per-pixel instance coverage counted by the id of each camera
ray's first collision and ranked by count (include/vpt_b200.h, DESIGN.md section 8s).

Cases: the headline frame (lean kernel), lights + sphere + thin lens (generic kernel), the volumetric path integrator on the tabulated
sky, the mixed scene S1 of tests/mixed_scenes.py and bench.py's 1000-instance scene on a small frame.  Frames fuse at most 5 passes per
chunk unless said otherwise."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import vpt_b200 as V
import mixed_scenes as M
import cryptomatte_ref as R
from vpt_b200.renderer import cryptomatte_id, stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
from test_aov_gpu import make_aov_case
from test_deep_gpu import bitwise
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float("inf")
PASSES = 8
OUTPUTS = ("accum", "depth", "cost", "raw", "display", "alpha", "volume", "deep", "mattes", "motion", "position", "normal", "albedo")


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def vols():
    return M.Volumes()


def mixed_case(vols):
    scene = M.build_s1(vols)
    cam = scene.frame_camera(256, 160)
    def mk():
        r = V.Renderer(scene, 256, 160, kp=make_kp(ray_depth=3), cam=cam, options={"passes_per_chunk": 5})
        r.enable_aovs()
        return r
    return scene, mk


def run(scene, r, passes=PASSES, single=False, split=None):
    """a new frame of `passes` passes: fused, pass by pass, or as calls of the sizes in `split`; returns clones of every output"""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if r.buffers.crypto is not None:
        r.buffers.crypto.fill_(0x5A5A5A5A)                          # the iteration-0 clear must not depend on a zeroed state
    if single:
        for _ in range(passes): r.render_pass()
    elif split:
        for n in split: r.render(n)
    else:
        r.render(passes)
    torch.cuda.synchronize()
    b = r.buffers
    out = {k: getattr(b, k).clone() for k in OUTPUTS + ("crypto",) if getattr(b, k) is not None}
    if b.groups: out.update({"group_" + g: t.clone() for g, t in b.groups.items()})
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def state_np(r, words=None):
    """(n, overflow, ids, counts) as uint32 numpy arrays, (H', W) and (S, H', W)"""
    S = r.crypto_capacity
    w = (r.buffers.crypto if words is None else words).cpu().numpy().view(np.uint32).reshape(2 + 2 * S, -1, r.width)
    return w[0], w[1], w[2::2], w[3::2]


def shifted_cam(cam, dx):
    c = V._native.camera.from_buffer_copy(bytes(cam))
    c.origin.x += dx; c.lower_left_corner.x += dx
    return c


@pytest.mark.parametrize("name,cap", [("headline", 32), ("lights_sphere", 4), ("vol_sky_table", 8)])
def test_cryptomatte_changes_no_other_output(dragon, name, cap):
    """Every other output -- accum, depth, cost, raw, display, the blue noise, the AOVs, the light groups (generic and volumetric
    kernels), deep slices, mattes, motion vectors and collision AOVs -- is bit-identical with the Cryptomatte off and on; it adds one
    launch per chunk (5 + 3); fused chunks, single passes and split calls give the same state."""
    scene, mk, _ = make_aov_case(name, dragon, None)
    groups = name != "headline"

    def make(on, mattes=True):
        r = mk()
        if groups: r.enable_light_groups()
        r.enable_deep([0.0, 30.0, INF])
        if mattes: r.enable_mattes([list(range(len(scene.instances)))], sphere=0)
        r.enable_motion_vectors(shifted_cam(r.cam, 0.5))
        r.enable_collision_aovs()
        if on: r.enable_cryptomatte(cap)
        return r

    for mattes in (True, False):                                     # with the mattes the trace kernel is the same; without, it changes
        off_r, r = make(False, mattes), make(True, mattes)
        off, on = run(scene, off_r), run(scene, r)
        assert r.stats()[0] - off_r.stats()[0] == 2, "one more kernel per chunk with the Cryptomatte on"
        for k in off:
            assert bitwise(on[k], off[k]), f"{name}: {k} changes when the Cryptomatte is on (mattes {mattes})"
    n, ovf, ids, counts = state_np(r)
    assert (n == PASSES).all()
    assert counts.sum() > 0, "the frame must show the volume"
    for kw in (dict(single=True), dict(split=[3, 1, 4])):
        again = run(scene, make(True, False), **kw)
        assert bitwise(again["crypto"], on["crypto"]), f"{name}: {kw} changes the state"


def test_exact_identities_against_single_instance_mattes(vols):
    """A scene of at most 31 instances with the sphere in view, one matte per instance and one for the sphere, in the same call as the
    Cryptomatte (capacity 32, so nothing overflows): per pixel round(n * matte_i.w) == count_i, sum(counts) + overflow == round(n * alpha),
    n == passes; cryptomatte_matte agrees with the matte coverage; the ranks equal the NumPy restatement bit for bit."""
    scene, mk = mixed_case(vols)
    n_inst = len(scene.instances)
    assert n_inst <= 31
    P = 24
    r = mk()
    r.enable_mattes([[i] for i in range(n_inst)] + [[]], sphere=n_inst)
    r.enable_cryptomatte(32)
    f = run(scene, r, P)
    n, ovf, ids, counts = state_np(r)
    assert (n == P).all() and (ovf == 0).all()
    H, W = r.height, r.width
    cov = f["mattes"][:, :, 3].double().cpu().numpy().reshape(n_inst + 1, H, W)
    want = np.rint(cov * P).astype(np.int64)                           # (K, H, W) collision counts per matte
    got = np.zeros_like(want)
    for j in range(32):
        c = counts[j].astype(np.int64)
        i = ids[j].astype(np.int64)
        k = np.where(i == R.SPHERE, n_inst, np.minimum(i, n_inst + 1))
        assert ((c == 0) | (k <= n_inst)).all(), "an id outside the scene"
        for kk in range(n_inst + 1):
            got[kk] += np.where((k == kk) & (c > 0), c, 0)
    assert (got == want).all(), f"{int((got != want).sum())} (matte, pixel) counts differ"
    alpha = f["alpha"].double().cpu().numpy().reshape(H, W)
    assert (counts.astype(np.int64).sum(0) + ovf == np.rint(alpha * P)).all()
    assert (got[n_inst] > 0).any(), "the sphere must be seen"
    assert sum(int((got[i] > 0).any()) for i in range(n_inst)) >= 2, "at least two instances must be seen"

    # the keyer: every single instance, the sphere, and a set of several
    for sel, mk_sel in [([i], [i]) for i in range(n_inst)] + [(["sphere"], [n_inst]), (list(range(0, n_inst, 2)), list(range(0, n_inst, 2)))]:
        m = r.cryptomatte_matte(sel).double().cpu().numpy()
        ref = cov[mk_sel].sum(0)
        assert np.all(np.abs(m - ref) <= 1e-5 + 1e-4 * np.abs(ref)), sel

    # the ranks and the id floats
    table = np.array([cryptomatte_id(x)[0] for x in r.crypto_names], np.float32)
    sphere_id = np.float32(cryptomatte_id("sphere")[0])
    assert table.tobytes() == np.array([R.id_float(x) for x in r.crypto_names], np.float32).tobytes()
    img, over = r.cryptomatte_image(ranks=8, overflow=True)
    img = img.cpu().numpy()
    words = r.buffers.crypto.cpu().numpy().view(np.uint32).reshape(2 + 64, H * W)
    ref = np.stack([R.ranks(words[:, p], 32, table, sphere_id, 8) for p in range(H * W)], 1).reshape(4, H, W, 4)
    assert img.tobytes() == ref.tobytes(), "the ranks differ from the restatement"
    assert (over.cpu().numpy() == 0).all()
    ids_seen = set(np.unique(img[..., 0::2]).tolist()) - {0.0}
    assert ids_seen <= set(table.tolist()) | {float(sphere_id)} and len(ids_seen) >= 3


def test_small_table_is_a_prefix_of_the_large_one(dragon):
    """bench.py's 1000-instance scene on a small frame: the S = 2 table is the first two entries of the S = 32 table and its overflow is
    the S = 32 overflow plus the counts of the other entries; the S = 32 ranks of the register-free path match the restatement."""
    sys.path.insert(0, ROOT)
    import bench as B
    wl = B.build_workload(V, 5, "cuda:0")
    scene, kp = wl["scene"], wl["kp"]
    W, H = 320, 180
    r = V.Renderer(scene, W, H, kp=kp, cam=scene.frame_camera(W, H))
    got = {}
    for S in (32, 2):
        r.enable_cryptomatte(S)
        run(scene, r, 16)
        got[S] = state_np(r)
    n32, o32, i32, c32 = got[32]
    n2, o2, i2, c2 = got[2]
    assert (n32 == 16).all() and (n2 == 16).all()
    assert (i2 == i32[:2]).all() and (c2 == c32[:2]).all()
    assert (o2.astype(np.int64) == o32.astype(np.int64) + c32[2:].astype(np.int64).sum(0)).all()
    assert (o2 > 0).any(), "some pixel must overflow two entries"
    assert (c32 > 0).sum(0).max() >= 3, "some pixel must see three instances"


def test_chunks_continued_calls_adaptive_region_and_cull(dragon):
    """A chunk boundary, fused against single passes and a continued call give identical states (above); adaptive frames match the
    fixed-count frame of each pixel's pass count; a render region matches the full frame inside and leaves the state untouched outside;
    on the headline frame (miss cull on) every pixel counts every pass and pixels without coverage hold no entry."""
    scene, mk, _ = make_aov_case("instanced", dragon, None)
    r, f = mk(), mk()
    r.enable_cryptomatte(4); f.enable_cryptomatte(4)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    _, counts = r.render_adaptive(32, threshold=0.12, min_passes=8, check_interval=8)
    torch.cuda.synchronize()
    got = r.buffers.crypto.view(10, -1).clone()
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert len(classes) >= 2
    for c in classes:
        f.reset(); f.render(c); torch.cuda.synchronize()
        m = flat == c
        assert bitwise(got[:, m], f.buffers.crypto.view(10, -1)[:, m]), f"the state differs on the {int(m.sum())} pixels of {c} passes"
    assert bitwise(got[0], flat.to(torch.int32))

    # render region
    full = run(scene, f)["crypto"].view(10, f.height, f.width)
    g = mk(); g.enable_cryptomatte(4)
    x0, y0, x1, y1 = 17, 9, 101, 63
    g.set_region(x0, y0, x1, y1)
    scene.reset_blue_noise(); g.kp.iteration = 0; g.buffers.zero_()
    g.buffers.crypto.fill_(0x7FBADBAD)
    g.render(PASSES); torch.cuda.synchronize()
    st = g.buffers.crypto.view(10, g.height, g.width)
    assert bitwise(st[:, y0:y1, x0:x1], full[:, y0:y1, x0:x1])
    inside = torch.zeros(g.height, g.width, dtype=torch.bool, device=st.device); inside[y0:y1, x0:x1] = True
    assert bool((st[:, ~inside] == 0x7FBADBAD).all()), "the state was written outside the region"

    # the miss cull (headline frame): culled pixels count the passes and hold no entry
    hs, hmk, _ = make_aov_case("headline", dragon, None)
    h = hmk(); h.enable_cryptomatte(2)
    out = run(hs, h)
    n, ovf, ids, cnt = state_np(h)
    alpha = out["alpha"].cpu().numpy().reshape(n.shape)
    assert (n == PASSES).all()
    assert ((cnt.sum(0) + ovf == 0) == (alpha == 0)).all()
    assert (alpha == 0).mean() > 0.3, "most of the headline frame misses the volume"


def test_unsampled_passes_count_and_the_gate_stops(dragon):
    """Passes that sample nothing (Kernel_params.render == 0) count in n and add no id; passes at or past max_interactions change
    nothing; a continued call goes on from the state."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    r.enable_cryptomatte(2)
    three = run(scene, r, 3)["crypto"]
    r.kp.render = 0
    r.render(2); torch.cuda.synchronize()
    n, ovf, ids, counts = state_np(r)
    n3, o3, i3, c3 = state_np(r, three)
    assert (n == 5).all() and (counts == c3).all() and (ids == i3).all() and (ovf == o3).all()
    assert counts.sum() > 0
    r.kp.render = 1
    r.kp.max_interactions = 7
    r.render(4); torch.cuda.synchronize()                          # iterations 5, 6 count; 7 and 8 are gated
    n = state_np(r)[0]
    assert (n == 7).all()
    before = r.buffers.crypto.clone()
    r.render(2); torch.cuda.synchronize()
    assert bitwise(r.buffers.crypto, before)


def test_partitioned_contexts_keep_rank_local_state(dragon):
    """Three shards on one GPU: the rank-local rows of each shard's state, concatenated in global rows, equal the single-context state."""
    W, H, NR, SR = 320, 200, 3, 8
    scene = V.Scene([dragon.instance(pos=(-20.0, 0.0, 0.0)), dragon.instance(pos=(20.0, 0.0, 0.0))], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    one = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    one.enable_cryptomatte(3)
    full = run(scene, one, 3)["crypto"].view(8, H, W)
    assert int(full[3].sum()) > 0
    merged = torch.full_like(full, -7)
    for rank in range(NR):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam, rank=rank, n_ranks=NR, stripe_rows=SR)
        r.enable_cryptomatte(3)
        st = run(scene, r, 3)["crypto"].view(8, -1, W)
        rows = stripe_rows_of_rank(H, rank, NR, SR)
        own = torch.as_tensor(np.nonzero(rows < H)[0], device=full.device)
        merged[:, torch.as_tensor(rows[rows < H], device=full.device)] = st[:, own]
        r.close()
    assert bitwise(merged, full)


def test_distributed_renderer_delegates(dragon, tmp_path):
    """DistributedRenderer's Cryptomatte calls act on the rank's renderer"""
    import torch.distributed as dist
    W, H = 192, 96
    scene = V.Scene([dragon.instance(pos=(-20.0, 0.0, 0.0)), dragon.instance(pos=(20.0, 0.0, 0.0))], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    ref = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    ref.enable_cryptomatte(4, names=["left", "right"])
    want = run(scene, ref, 3)["crypto"]
    own = not dist.is_initialized()
    if own: dist.init_process_group("gloo", init_method=f"file://{tmp_path}/pg", rank=0, world_size=1)
    try:
        d = V.DistributedRenderer(scene, W, H, cam=cam, kp=make_kp(ray_depth=4))
        d.enable_cryptomatte(4, names=["left", "right"])
        scene.reset_blue_noise(); d.render(3); torch.cuda.synchronize()
        assert bitwise(d.r.buffers.crypto, want)
        assert bitwise(d.cryptomatte_image(4), ref.cryptomatte_image(4))
        assert bitwise(d.cryptomatte_matte(["left"]), ref.cryptomatte_matte([0]))
        assert d.cryptomatte_manifest() == ref.cryptomatte_manifest() and d.cryptomatte_metadata() == ref.cryptomatte_metadata()
        assert d.cryptomatte_state()["n"].shape == (H, W)
        d.disable_cryptomatte()
        d.r.buffers.crypto.fill_(7)
        d.r.kp.iteration = 0; d.render(1); torch.cuda.synchronize()
        assert bool((d.r.buffers.crypto == 7).all())
        d.close()
    finally:
        if own: dist.destroy_process_group()


def test_activation_and_refusals(dragon):
    """The state set mid-frame stays untouched until the next iteration-0 call; NULL stops at once; bad arguments are refused when set
    and leave the registration as it was; overlaps and brick mode are refused at render time; the rank call refuses its bad arguments."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    ref = mk(); ref.enable_cryptomatte(2)
    want = run(scene, ref, 3)["crypto"]

    r = mk()
    with pytest.raises(V.VptError, match="not enabled"):
        r.cryptomatte_state()
    scene.reset_blue_noise(); r.render(2)
    r.enable_cryptomatte(2)
    r.buffers.crypto.fill_(7)
    r.render(2); torch.cuda.synchronize()                                      # iteration 2: not active yet
    assert bool((r.buffers.crypto == 7).all())
    assert bitwise(run(scene, r, 3)["crypto"], want)                           # iteration 0: active from here on
    r.disable_cryptomatte()
    r.buffers.crypto.fill_(7)
    r.kp.iteration = 0; r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.crypto == 7).all()), "a NULL state turns the Cryptomatte off"

    z = mk(); z.enable_cryptomatte(2)
    buf = torch.zeros(70 * W * H + 4, dtype=torch.int32, device=z.buffers.accum.device)
    for args in [(C.c_void_p(buf.data_ptr()), 0), (C.c_void_p(buf.data_ptr()), 33), (C.c_void_p(buf.data_ptr() + 2), 4)]:
        assert V.lib.vpt_set_cryptomatte(z.ctx, *args) == -1, args
        assert V.lib.vpt_last_error(z.ctx).startswith(b"vpt_set_cryptomatte")
    with pytest.raises(V.VptError, match="duplicate names"):
        z.enable_cryptomatte(2, names=["sphere"])
    with pytest.raises(V.VptError, match="capacity"):
        z.enable_cryptomatte(0)
    assert bitwise(run(scene, z, 3)["crypto"], want)

    o = mk()
    o.enable_deep([0.0, INF]); o.enable_collision_aovs(); o.enable_aovs()
    # the error names the first buffer of its list that the state overlaps: accum heads the list; the others may have a neighbour
    # allocated right after them inside the state's span
    for target, what in ((o.buffers.accum, "Kernel_params.accum_buffer"), (o.buffers.deep, ""), (o.buffers.normal, ""), (o.buffers.alpha, "")):
        V._native.check(V.lib.vpt_set_cryptomatte(o.ctx, C.c_void_p(target.data_ptr()), 1), o.ctx, "vpt_set_cryptomatte")
        o.kp.iteration = 0
        with pytest.raises(V.VptError, match="state buffer overlaps " + what):
            o.render(1)
    V._native.check(V.lib.vpt_set_cryptomatte(o.ctx, None, 0), o.ctx, "vpt_set_cryptomatte")

    perlin = V.Volume.procedural((48, 40, 36), scale=0.1, seed=3)
    perlin.build_bricks()
    ps = V.Scene([perlin.instance()], env=synthetic_env(512, 256), keep=[perlin])
    b = V.Renderer(ps, 64, 36, kp=make_kp(ray_depth=2), cam=ps.frame_camera(64, 36))
    b.set_brick_volume(perlin)
    b.enable_cryptomatte(2)
    with pytest.raises(V.VptError, match="brick or cell mode"):
        b.render(1)

    # vpt_cryptomatte_rank's refusals
    st, tab = ref.buffers.crypto, ref.crypto_table
    out = torch.zeros(16, W * H, 4, dtype=torch.float32, device=st.device)
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    good = [ref.ctx, W, H, p(st), 2, p(tab), 1, 0.5, 6, p(out), None, None]
    assert V.lib.vpt_cryptomatte_rank(*good) == 0
    bad = {0: None, 3: None, 4: 0, 8: 5, 9: None, 1: 0}
    bad_more = [dict(zip((4,), (33,))), {8: 0}, {8: 34}, {9: p(out, 4)}, {9: p(st)}, {10: p(st)}, {5: None}]
    for change in [{k: v} for k, v in bad.items()] + bad_more:
        args = list(good)
        for k, v in change.items(): args[k] = v
        assert V.lib.vpt_cryptomatte_rank(*args) == -1, change
