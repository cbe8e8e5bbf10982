"""Light groups on the GPU (vpt_set_light_group_buffers): per-pixel running means of the radiance the sun, the point lights, the
volume's emission and the environment added to each sample (include/vpt_b200.h, DESIGN.md section 8d).

Every trace kernel and resolve variant: the headline frame (lean kernel, wide records forced), lights + sphere + thin lens (generic
kernel), the Bruneton sky with and without point lights (k_resolve<1>), 120 instances (2 rays per lane without groups), brick and cell
mode, a synthetic emissive volume under both integrators, and the volumetric path integrator on the tabulated sky (k_resolve<2>)."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.renderer import stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
from test_adaptive_gpu import CASES as ADAPTIVE_CASES, make_case
from test_aov_gpu import make_aov_case
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
AOVS = ("alpha", "volume")
GROUPS = V.LIGHT_GROUPS
PASSES = 8                     # in chunks of 5 + 3 (passes_per_chunk = 5)
LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]


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
    """A synthetic fireball: a soft ball of density with a hot core, so the emission walk has something to add."""
    n = 48
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    c = (n - 1) / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) / c
    density = (np.clip(1.1 - r, 0.0, None) ** 1.5).astype(np.float32)
    heat = (3.0 * np.clip(0.8 - r, 0.0, None)).astype(np.float32)
    return V.Volume.from_dense(density, bbox_min=(-c, -c, -c), emission=heat)


def set_light_power(scene, powers):
    """Rewrites the power of every point light of `scene` in place (positions and count unchanged)."""
    n = scene.lights.num_lights
    pl = (V.point_light * n).from_buffer_copy(scene.d_lights.cpu().numpy().tobytes()[:C.sizeof(V.point_light) * n])
    for i in range(n): pl[i].power = powers[i]
    scene.d_lights[:C.sizeof(pl)].copy_(torch.frombuffer(bytearray(bytes(pl)), dtype=torch.uint8))


def place_sphere(scene):
    sp = scene.h_sphere; sp.center = V.f3(4.0, 6.5, 3.0); sp.radius = 1.2; sp.roughness = 0.7; sp.color = V.f3(0.8, 0.6, 0.3)
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))


def make_group_case(name, dragon, perlin, emissive):
    """-> dict(scene, mk0 (a fresh renderer, nothing registered), integrator, sky ('hdri' | 'bruneton'), lights, emission, keep)"""
    info = dict(integrator=0, sky="hdri", lights=False, emission=False, keep=[])
    if name in ("headline", "lights_sphere", "vol_sky_table", "sky", "instanced", "brick", "cells"):
        scene, mk, keep = make_aov_case(name, dragon, perlin)
        info.update(scene=scene, mk0=lambda: mk(aovs=False), keep=keep, lights=name == "lights_sphere")
        if name == "sky": info["sky"] = "bruneton"
        if name == "vol_sky_table": info.update(integrator=1, sky="bruneton")
        return info
    if name == "sky_lights":                                     # Bruneton sky, point lights, the sphere: the generic kernel into k_resolve<1>
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256), lights=LIGHTS)
        place_sphere(scene)
        atm = V.Atmosphere(); atm.apply(scene.atmos)
        cam = scene.frame_camera(200, 120)
        mk0 = lambda: V.Renderer(scene, 200, 120, kp=make_kp(environment_type=0, elevation=25.0, ray_depth=3), cam=cam)
        info.update(scene=scene, sky="bruneton", lights=True, keep=[atm])
    elif name in ("emissive", "vol_emissive"):                   # emission walk + point lights, direct / volumetric path integrator
        scene = V.Scene([emissive.instance()], env=synthetic_env(512, 256), lights=LIGHTS)
        atm = V.Atmosphere(); atm.apply(scene.atmos)
        cam = scene.frame_camera(160, 120)
        integ = 1 if name == "vol_emissive" else 0
        kw = dict(ray_depth=4, volume_depth=3, emission_scale=1.0, emission_pivot=1.0, integrator=integ)
        mk0 = lambda: V.Renderer(scene, 160, 120, kp=make_kp(**kw), cam=cam)
        info.update(scene=scene, integrator=integ, lights=True, emission=True, keep=[atm])
    else:
        raise KeyError(name)
    info["mk0"] = mk0
    return info


NAMES = ["headline", "lights_sphere", "sky", "sky_lights", "instanced", "brick", "cells", "emissive", "vol_sky_table", "vol_emissive"]
DIRECT = [n for n in NAMES if not n.startswith("vol_")]


@pytest.fixture(scope="module")
def cases(dragon, perlin, emissive):
    cache = {}
    def get(name):
        if name not in cache: cache[name] = make_group_case(name, dragon, perlin, emissive)
        return cache[name]
    return get


def renderer(case, groups=True, aovs=False, **kp):
    r = case["mk0"]()
    r.set_option("passes_per_chunk", 5)
    for k, v in kp.items(): setattr(r.kp, k, v)
    if aovs: r.enable_aovs()
    if groups: r.enable_light_groups()
    return r


def frame(scene, r, passes, pass_by_pass=False):
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if pass_by_pass:
        for _ in range(passes): r.render_pass()
    else:
        r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS + AOVS if getattr(r.buffers, k) is not None}
    if r.buffers.groups is not None:
        out.update({g: t.clone() for g, t in r.buffers.groups.items()})
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def bitwise(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def assert_sum_is_the_beauty(out, what):
    """sum of the groups vs accum: |d| <= 1e-5 + 1e-4 |accum| on >= 99.9 % of the pixels, per channel"""
    accum = out["accum"].double()
    total = sum(out[g].double() for g in GROUPS)
    bad = (total - accum).abs() > 1e-5 + 1e-4 * accum.abs()
    frac = bad.double().mean(dim=0)
    assert bool((frac <= 1e-3).all()), f"{what}: sum of the groups off the beauty on {frac.tolist()} of the pixels"


@pytest.mark.parametrize("name", NAMES)
def test_groups_move_nothing_fuse_like_single_passes_and_sum_to_the_beauty(cases, name):
    """(1) accum, depth, cost, raw, display, the blue noise and the AOVs are bit-identical with groups off and on; (5) the fused 5 + 3
    chunks give the groups of 8 single-pass calls, bit for bit; (8) two identical frames give identical groups; (4) the groups sum to
    the beauty; a class the scene does not have is exactly 0."""
    case = cases(name)
    scene = case["scene"]
    off = frame(scene, renderer(case, groups=False, aovs=True), PASSES)
    r = renderer(case, aovs=True)
    on = frame(scene, r, PASSES)
    for k in BUFFERS + AOVS + ("blue_noise",):
        assert bitwise(on[k], off[k]), f"{name}: {k} changes when the light groups are on"
    single = frame(scene, renderer(case), PASSES, pass_by_pass=True)
    again = frame(scene, r, PASSES)
    for g in GROUPS:
        assert bitwise(single[g], on[g]), f"{name}: group {g} of 8 single passes differs from the fused 5 + 3 chunks"
        assert bitwise(again[g], on[g]), f"{name}: group {g} differs between two identical frames"
    assert_sum_is_the_beauty(on, name)
    assert float(on["sun"].max()) > 1e-3 and float(on["environment"].max()) > 1e-3, f"{name}: sun and environment must show"
    if case["lights"]: assert float(on["point"].max()) > 1e-4, f"{name}: the point lights must show"
    else: assert bool((on["point"] == 0).all()), f"{name}: no point lights, yet the point group is not 0"
    if case["emission"]: assert float(on["emission"].max()) > 1e-4, f"{name}: the emission must show"
    else: assert bool((on["emission"] == 0).all()), f"{name}: no emission, yet the emission group is not 0"
    assert r.light_group_image("sun").shape == (r.n_local // r.width, r.width, 3)


def solo_params(case, lit):
    """Kernel_params overrides and light powers of a render in which only class `lit` is lit (direct integrator)."""
    no_sky = {"bruneton": dict(sky_mult=0.0), "hdri": dict(sky_color=V.f3(0.0, 0.0, 0.0))}[case["sky"]]
    kp, powers_on = {}, False
    if lit != "sun": kp["sun_mult"] = 0.0
    if lit != "environment": kp.update(no_sky)
    if lit == "point": powers_on = True
    return kp, powers_on


@pytest.mark.parametrize("name", DIRECT)
def test_each_group_is_the_render_lit_by_its_class_alone(cases, name):
    """(2) direct integrator: the path's draws do not depend on light intensities, so every group is bit for bit the accum of a render
    in which only that class is lit.  Emission cannot be switched off without dropping the emission walk's draws, so in a scene with
    emission only the emission group is checked this way."""
    case = cases(name)
    scene = case["scene"]
    on = frame(scene, renderer(case), PASSES)
    powers = [l[2] for l in LIGHTS]
    for lit in GROUPS:
        if case["emission"] and lit != "emission": continue
        kp, powers_on = solo_params(case, lit)
        if case["lights"] and not powers_on: set_light_power(scene, [0.0] * len(powers))
        try:
            solo = frame(scene, renderer(case, groups=False, **kp), PASSES)
        finally:
            if case["lights"]: set_light_power(scene, powers)
        assert bitwise(on[lit], solo["accum"]), f"{name}: group {lit} is not the render lit by {lit} alone " \
                                                f"(max |d| {float((on[lit] - solo['accum']).abs().max())})"


def test_volumetric_path_integrator_environment_is_the_render_without_sun(cases):
    """(3) volumetric path integrator, no point lights, no emission: the environment group is bit for bit the accum of the render with
    sun_color = 0 (sun_mult still gates the sun's transmittance walks, so the draws are the same); point and emission are exactly 0."""
    case = cases("vol_sky_table")
    scene = case["scene"]
    on = frame(scene, renderer(case), PASSES)
    solo = frame(scene, renderer(case, groups=False, sun_color=V.f3(0.0, 0.0, 0.0)), PASSES)
    assert bitwise(on["environment"], solo["accum"]), float((on["environment"] - solo["accum"]).abs().max())
    assert bool((on["point"] == 0).all()) and bool((on["emission"] == 0).all())


@pytest.mark.parametrize("name,W,H,mx,mn,iv,thr", [
    ("headline", 320, 200, 48, 8, 8, 0.05),
    ("lights_sphere",) + ADAPTIVE_CASES["lights_sphere"],
    ("vol_sky_table",) + ADAPTIVE_CASES["vol_sky_table"],
])
def test_adaptive_frame_groups_equal_the_fixed_count_frames(dragon, perlin, name, W, H, mx, mn, iv, thr):
    """(6) every pixel's groups (and buffers) equal those of a fixed-count frame of its own pass count, class by class."""
    if name == "headline":
        scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        cam = scene.frame_camera(W, H)
        mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=100), cam=cam)
    else:
        scene, mk, keep = make_case(name, dragon, perlin)
    r, f = mk(), mk()
    r.enable_light_groups(); f.enable_light_groups()
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    run, counts = r.render_adaptive(mx, threshold=thr, min_passes=mn, check_interval=iv)
    torch.cuda.synchronize()
    got = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    got.update({g: t.clone() for g, t in r.buffers.groups.items()})
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert len(classes) >= 2 and run == max(classes)
    for c in classes:
        f.reset(); f.render(c); torch.cuda.synchronize()
        m = flat == c
        for k in BUFFERS:
            assert torch.equal(got[k][m], getattr(f.buffers, k)[m]), f"{k} differs on the {int(m.sum())} pixels of {c} passes"
        for g in GROUPS:
            assert torch.equal(got[g][m], f.buffers.groups[g][m]), f"group {g} differs on the {int(m.sum())} pixels of {c} passes"


def test_partitioned_contexts_keep_rank_local_groups(dragon):
    """(7) four shards on one GPU (generic kernel: point lights): each shard's rank-local group rows equal the single-context rows."""
    W, H, R, SR = 320, 200, 4, 8
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256), lights=LIGHTS)
    one = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4))
    one.enable_light_groups()
    full = frame(scene, one, 3)
    for rank in range(R):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=one.cam, rank=rank, n_ranks=R, stripe_rows=SR)
        r.enable_light_groups()
        frame(scene, r, 3)
        rows = stripe_rows_of_rank(H, rank, R, SR)
        own = torch.as_tensor(np.nonzero(rows < H)[0], device=one.buffers.accum.device)       # local rows inside the frame
        glob = torch.as_tensor(rows[rows < H], device=own.device)
        for g in GROUPS:
            img = r.light_group_image(g)
            assert img.shape == (len(rows), W, 3)
            assert torch.equal(img[own], full[g].view(H, W, 3)[glob]), f"rank {rank}: group {g}"
        r.close()


def test_activation_switch_off_and_refusals(dragon):
    """(8) groups enabled mid-frame stay untouched until the next iteration-0 call; four NULLs turn them off at once; every overlap is
    refused, naming the buffer."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256), lights=LIGHTS)
    cam = scene.frame_camera(W, H)
    mk = lambda **kw: V.Renderer(scene, W, H, kp=make_kp(ray_depth=4, **kw), cam=cam)
    ref = mk(); ref.enable_light_groups()
    want = frame(scene, ref, 3)

    r = mk()
    scene.reset_blue_noise(); r.render(2)
    r.enable_light_groups()
    for t in r.buffers.groups.values(): t.fill_(7.0)
    r.render(2); torch.cuda.synchronize()                                      # iteration 2: not active yet
    assert all(bool((t == 7.0).all()) for t in r.buffers.groups.values())
    got = frame(scene, r, 3)                                                  # iteration 0: active from here on
    for k in GROUPS + ("accum",):
        assert bitwise(got[k], want[k]), k

    r.disable_light_groups()
    for t in r.buffers.groups.values(): t.fill_(7.0)
    r.render(1); torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in r.buffers.groups.values())
    r.kp.iteration = 0
    r.render(1); torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in r.buffers.groups.values()), "four NULLs must stay off at iteration 0 too"
    with pytest.raises(V.VptError, match="not enabled"):
        mk().light_group_image("sun")
    with pytest.raises(V.VptError, match="unknown light group"):
        r.light_group_image("moon")

    check = V._native.check
    # one group alone
    solo = mk()
    alone = torch.zeros_like(want["point"])
    check(V.lib.vpt_set_light_group_buffers(solo.ctx, None, C.c_void_p(alone.data_ptr()), None, None), solo.ctx, "vpt_set_light_group_buffers")
    frame(scene, solo, 3)
    assert bitwise(alone, want["point"])

    # passes beyond max_interactions change nothing
    capped = mk(max_interactions=2); capped.enable_light_groups()
    two = frame(scene, capped, 2)
    capped.render(3); torch.cuda.synchronize()
    for g in GROUPS:
        assert bitwise(capped.buffers.groups[g], two[g]), g

    # overlaps: the Kernel_params buffers of `z` sit 64 bytes per pixel apart in one arena, so a group buffer that starts on the last word
    # of one of them overlaps that buffer and nothing else; likewise the two AOV buffers
    n = W * H
    z = mk()
    dev = z.buffers.accum.device
    arena = torch.zeros(5 * 16 * n, dtype=torch.float32, device=dev)
    size = {"accum_buffer": 12 * n, "depth_buffer": 4 * n, "cost_buffer": 12 * n, "raw_buffer": 16 * n, "display_buffer": 4 * n}
    for i, name in enumerate(size):
        setattr(z.kp, name, arena.data_ptr() + i * 64 * n)
    aov_arena = torch.zeros(2 * 16 * n, dtype=torch.float32, device=dev)
    aov_a, aov_v = aov_arena.data_ptr(), aov_arena.data_ptr() + 64 * n
    check(V.lib.vpt_set_aov_buffers(z.ctx, C.c_void_p(aov_a), C.c_void_p(aov_v)), z.ctx, "vpt_set_aov_buffers")
    spare = [torch.zeros(n, 3, dtype=torch.float32, device=dev) for _ in GROUPS]
    targets = {f"Kernel_params.{k}": getattr(z.kp, k) + size[k] - 4 for k in size}
    targets.update({"the alpha AOV buffer": aov_a + 4 * n - 4, "the volume AOV buffer": aov_v + 12 * n - 4})
    for slot, g in enumerate(GROUPS):
        for what, last in targets.items():
            ptrs = [C.c_void_p(t.data_ptr()) for t in spare]
            ptrs[slot] = C.c_void_p(last)
            check(V.lib.vpt_set_light_group_buffers(z.ctx, *ptrs), z.ctx, "vpt_set_light_group_buffers")
            z.kp.iteration = 0
            with pytest.raises(V.VptError, match=f"the {g} buffer overlaps {what}"):
                z.render(1)
    for j in range(1, len(GROUPS)):                                             # group j starts on the last word of group 0
        ptrs = [C.c_void_p(t.data_ptr()) for t in spare]
        ptrs[j] = C.c_void_p(spare[0].data_ptr() + 12 * n - 4)
        check(V.lib.vpt_set_light_group_buffers(z.ctx, *ptrs), z.ctx, "vpt_set_light_group_buffers")
        z.kp.iteration = 0
        with pytest.raises(V.VptError, match=f"the sun buffer and the {GROUPS[j]} buffer overlap"):
            z.render(1)
    check(V.lib.vpt_set_light_group_buffers(z.ctx, *[C.c_void_p(t.data_ptr()) for t in spare]), z.ctx, "vpt_set_light_group_buffers")
    z.kp.iteration = 0
    z.render(1); torch.cuda.synchronize()                                     # disjoint buffers render
    assert float(spare[0].max()) > 0.0


def test_guarded_samples_leave_every_group_at_its_mean(dragon):
    """(9) an environment map with a NaN region: the guard replaces those samples by accum's mean, and every group by its own mean, so the
    groups stay finite, still sum to the beauty, and pixels that only ever see the NaN region keep 0 everywhere."""
    env = synthetic_env(512, 256)
    env[:, (np.arange(512) % 32) < 16, :3] = np.nan                            # NaN stripes, 16 texels wide, around the whole horizon
    scene = V.Scene([dragon.instance()], env=env)
    cam = scene.frame_camera(240, 160)
    mk = lambda: V.Renderer(scene, 240, 160, kp=make_kp(ray_depth=4), cam=cam)
    off = frame(scene, mk(), PASSES)
    r = mk(); r.enable_light_groups()
    on = frame(scene, r, PASSES)
    assert bitwise(on["accum"], off["accum"])
    for g in GROUPS:
        assert bool(torch.isfinite(on[g]).all()), g
    assert_sum_is_the_beauty(on, "NaN environment")
    dark = (on["accum"] == 0).all(dim=1)
    assert int(dark.sum()) > 0, "no pixel sees only the NaN region"
    for g in GROUPS:
        assert bool((on[g][dark] == 0).all()), g


def test_guarded_samples_leave_every_group_at_its_mean_from_prefilled_buffers(dragon):
    """(9) as above, from prefilled buffers whose groups sum to accum exactly: a sample the guard replaces at iteration 0 takes every
    buffer's previous content (accum, each group, the volume AOV), so pixels that only ever see the NaN / +Inf region keep the prefill of
    all of them bit for bit, and the groups still sum to the beauty."""
    from test_resolve_tail_gpu import prefill, striped_env
    scene = V.Scene([dragon.instance()], env=striped_env())
    cam = scene.frame_camera(240, 160)
    mk = lambda: V.Renderer(scene, 240, 160, kp=make_kp(ray_depth=4), cam=cam)
    rng = np.random.RandomState(37)
    n = 240 * 160
    parts = {g: torch.from_numpy(rng.randint(0, 1024, (n, 3)).astype(np.float32) / 1024).cuda() for g in GROUPS}
    volume0 = torch.from_numpy(rng.randint(0, 1024, (n, 3)).astype(np.float32) / 1024).cuda()

    def fill(r):
        prefill(r.buffers, 37)
        r.buffers.accum.copy_(sum(parts[g] for g in GROUPS))            # sums of multiples of 1/1024 below 4: exact
        if r.buffers.groups is not None:
            for g in GROUPS: r.buffers.groups[g].copy_(parts[g])
        if r.buffers.volume is not None: r.buffers.volume.copy_(volume0)

    def run(r):
        scene.reset_blue_noise(); r.kp.iteration = 0; fill(r)
        r.render(PASSES); torch.cuda.synchronize()
        return r
    off = run(mk())
    r = mk(); r.enable_aovs(); r.enable_light_groups()
    on = run(r)
    assert bitwise(on.buffers.accum, off.buffers.accum)
    out = {"accum": on.buffers.accum, **on.buffers.groups}
    for g in GROUPS:
        assert bool(torch.isfinite(out[g]).all()), g
    assert_sum_is_the_beauty(out, "NaN / +Inf environment from prefilled buffers")
    kept = (on.buffers.accum == sum(parts[g] for g in GROUPS)).all(dim=1)
    assert int(kept.sum()) > 0, "no pixel sees only the non-finite region"
    for g in GROUPS:
        assert bitwise(out[g][kept], parts[g][kept]), g
    assert bitwise(on.buffers.volume[kept], volume0[kept])
