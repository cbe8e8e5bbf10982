"""Collision AOVs (vpt_set_collision_aovs; DESIGN.md section 8q) on the GPU.

1. Layers on and off leave accum, depth, cost, raw, display, the blue noise, the AOVs, light groups, deep slices, mattes and motion vectors
   bit for bit as they are: the lean HDRI kernel, the generic kernel with point lights and the sphere, the volumetric path integrator on
   the precomputed sky and brick mode, across a chunk boundary and a continued call.
2. position.w is the alpha AOV bit for bit (also in adaptive and region frames); n fused passes equal n single-pass calls bit for bit.
3. One pass at iteration 0: P against the float64 ray rebuild (pinhole, thin lens, camera motion); normal and albedo against the
   restatement (tests/collision_aovs_ref.py) at the GPU's own P, in texture, brick and cell mode, on an instanced scene, a coloured volume
   and the sphere.
4. The running mean from prefilled buffers at a continued iteration.
5. Adaptive frames, regions and four partitioned contexts.
6. Refusals, activation at iteration 0 and the launch count."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp
from test_aov_gpu import make_aov_case
from test_motion_vectors_gpu import copy_cam, moved, scale_of, same, bits, SENTINEL
from test_exchange_layers_gpu import FLT_MAX
import adaptive_ref as A
import collision_aovs_ref as R
import motion_ref as MR
import motion_vectors_ref as M
from mixed_scenes import read_tree

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
U24 = 2.0 ** -24
F32 = np.float32


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


def outputs(scene, r):
    b = r.buffers
    out = {k: getattr(b, k).clone() for k in BUFFERS}
    for k in ("alpha", "volume", "deep", "mattes", "motion"):
        if getattr(b, k) is not None: out[k] = getattr(b, k).clone()
    for g, t in (b.groups or {}).items(): out["group_" + g] = t.clone()
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def layers(r):
    return {k: getattr(r.buffers, k).clone() for k in ("position", "normal", "albedo")}


def sequence(scene, r, pass_by_pass=False):
    """8 passes in chunks of 5 + 3 from iteration 0, then a continued call of 3 passes."""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if pass_by_pass:
        for _ in range(11): r.render_pass()
    else:
        r.render(8); r.render(3)
    torch.cuda.synchronize()
    return outputs(scene, r)


# ---- 1, 2: nothing else moves; identities --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["headline", "lights_sphere", "vol_sky_table", "brick"])
def test_nothing_else_moves_and_the_identities_hold(dragon, perlin, name):
    scene, mk, keep = make_aov_case(name, dragon, perlin)

    def renderer(on):
        r = mk()
        r.enable_deep([0.0, float("inf")])
        if name != "brick":
            r.enable_mattes([range(len(scene.instances))], sphere=0)
        if name in ("lights_sphere", "vol_sky_table"):
            r.enable_light_groups()
        r.enable_motion_vectors(moved(r.cam, scale_of(scene)))
        if on:
            r.enable_collision_aovs()
        return r

    off = sequence(scene, renderer(False))
    r = renderer(True)
    on = sequence(scene, r)
    for k in off:
        assert same(on[k], off[k]), f"{name}: {k} changes when the collision AOVs are on"
    got = layers(r)
    assert same(got["position"][:, 3], on["alpha"]), f"{name}: position.w is not the alpha AOV"
    assert float(on["alpha"].max()) > 0
    assert float(got["normal"].abs().max()) > 0.1 and float(got["albedo"].abs().max()) > 0
    sequence(scene, r, pass_by_pass=True)
    for k, t in layers(r).items():
        assert same(t, got[k]), f"{name}: 11 single passes differ from the fused 5 + 3 + 3 in {k}"


# ---- 3: one pass against the rebuild and the restatement -----------------------------------------------------------------------------------
W1, H1 = 192, 96


def one_pass(scene, r):
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(1); torch.cuda.synchronize()
    pos = r.buffers.position.cpu().numpy()
    hit = r.buffers.depth.cpu().numpy() > 0
    assert np.array_equal(pos[:, 3].view(np.int32), hit.astype(F32).view(np.int32)), "coverage must be [depth > 0] bit for bit"
    assert np.array_equal(pos[~hit], np.zeros((int((~hit).sum()), 4), F32)), "a sample without coverage must add exact zeros"
    return pos, hit


@pytest.mark.parametrize("lens", ["pinhole", "thin", "motion"])
def test_position_against_the_ray_rebuild(dragon, lens):
    """P = org + depth dir in float32 against the float64 rebuild of test_motion_vectors_gpu.py.  The kernel's org is exact (pinhole,
    motion: the camera's fields; thin lens: a few float32 roundings of |origin| + |offset|), its dir comes from a normalize whose fast
    rsqrt is good to about 2^-22 relative, and the fma rounds once: 64 ulps of |org| + depth bounds that with a wide margin."""
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W1, H1)
    if lens == "thin":
        cam.lens_radius = np.float32(0.02 * scale_of(scene))
    r = V.Renderer(scene, W1, H1, kp=make_kp(ray_depth=2), cam=cam)
    r.enable_collision_aovs()
    if lens == "motion":
        r.set_camera_motion(moved(cam, 0.5 * scale_of(scene)))
    W, H = W1, H1
    scene.reset_blue_noise()
    bn = scene.d_blue_noise.clone().cpu().numpy().reshape(-1, 3)
    cams = r.motion_cameras().cpu().numpy().reshape(-1, 20) if lens == "motion" else None
    b0 = r.camera_rays().cpu().numpy()[:, :3].astype(np.float64) if lens != "motion" else None
    pos, hit = one_pass(scene, r)
    depth = r.buffers.depth.cpu().numpy().astype(np.float64)
    assert hit.sum() > 200
    idx = np.nonzero(hit)[0]
    ys, xs = idx // W, idx % W
    f = M.fields(r.cam)
    if lens == "pinhole":
        org = np.broadcast_to(f["origin"], (len(idx), 3)); d = b0[idx]
    elif lens == "thin":
        lib, acc, t2, t3 = MR.oracle_lib(), MR.accept_table(), MR.vdc_table(2), MR.vdc_table(3)
        lr = float(np.float32(r.cam.lens_radius))
        uu = np.array([getattr(r.cam.u, a) for a in "xyz"], np.float64); vv = np.array([getattr(r.cam.v, a) for a in "xyz"], np.float64)
        pts = np.array([M.lens_point(MR.Stream(lib, int(y) * W + int(x), 0), acc, t2, t3) for y, x in zip(ys, xs)])
        off = lr * pts[:, :1] * uu + lr * pts[:, 1:] * vv
        org = f["origin"] + off; d = b0[idx] - off
    else:
        c = cams[idx].astype(np.float64)
        o, llc, h, v = c[:, 1:4], c[:, 4:7], c[:, 7:10], c[:, 10:13]
        j = bn[(ys % 256) * 256 + xs % 256].astype(np.float64)
        s = ((xs + j[:, 0]) / W)[:, None]; t = ((ys + j[:, 1]) / H)[:, None]
        org, d = o, llc + s * h + t * v - o
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    P = org + depth[idx, None] * d
    err = np.abs(pos[idx, :3].astype(np.float64) - P).max(axis=1)
    tol = 64 * U24 * (np.linalg.norm(org, axis=1) + depth[idx]) * 2
    assert (err <= tol).all(), f"{lens}: worst {err.max():.3g} against {tol[np.argmax(err - tol)]:.3g}"
    r.close()


def put_sphere(scene, centre, radius, color):
    sp = scene.h_sphere; sp.center = V.f3(*centre); sp.radius = float(radius); sp.color = V.f3(*color); sp.roughness = 1.0
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))


def grid_of(vol):
    dx, dy, dz = vol.dims
    return vol.dense.cpu().numpy().reshape(dz, dy, dx)


def ramp_volume(n=32, seed=0):
    """A smooth 32^3 density (a blob plus a ramp, values 0.05 .. 1.5) and a colour grid that varies across it."""
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float64) + 0.5
    c = n / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) / c
    dens = (np.clip(1.2 - r, 0.0, None) * (1.0 + 0.3 * x / n) + 0.05 * (r < 1.1)).astype(F32)
    rgb = np.stack([0.3 + 0.6 * x / n, 0.9 - 0.5 * y / n, 0.2 + 0.7 * z / n], -1).astype(F32)
    return dens, rgb


def restated_scene(scene, vols):
    """collision_aovs_ref.Scene of `scene`: (instance xform, volume) per instance; the octree for more than one."""
    recs, grids, colors = [], [], []
    for g, vol in zip(scene.instances, vols):
        X = np.array([[g.xform[a][b] for b in range(4)] for a in range(4)], np.float64)
        info = g.vdb_info
        recs.append(R.volume_rec(X, (info.bmin.x, info.bmin.y, info.bmin.z), (info.dim.x, info.dim.y, info.dim.z)))
        grids.append(vol["grid"]); colors.append(vol.get("rgb"))
    tree = read_tree(scene.d_oct_root)
    octree = R.Octree(tree, scene.leaf_lists()) if len(recs) > 1 else None
    return R.Scene(recs, grids, colors=colors if any(c is not None for c in colors) else None, octree=octree), tree[0].max_extinction


CASES = ["texture", "brick", "cells", "coloured", "instanced", "sphere"]


def surface_case(perlin64, name):
    """(scene, renderer, restated scene, max_extinction, exact look-ups)"""
    if name in ("texture", "brick", "cells", "sphere"):
        scene = V.Scene([perlin64.instance()], env=synthetic_env(512, 256), keep=[perlin64])
        vols = [dict(grid=grid_of(perlin64))]
    elif name == "coloured":
        dens, rgb = ramp_volume()
        vol = V.Volume.from_dense(dens, bbox_min=(0, 0, 0), color=rgb)
        scene = V.Scene([vol.instance(pos=(-16.0, -16.0, -16.0))], env=synthetic_env(512, 256), keep=[vol])
        vols = [dict(grid=dens, rgb=rgb)]
    else:                                                       # two overlapping instances of one grid: leaf lists of one and two entries
        dens, _ = ramp_volume()
        vol = V.Volume.from_dense(dens, bbox_min=(0, 0, 0))
        scene = V.Scene([vol.instance(pos=(-24.0, -16.0, -16.0)), vol.instance(pos=(-8.0, -12.0, -16.0), scale=2.0)],
                        env=synthetic_env(512, 256), keep=[vol])
        vols = [dict(grid=dens), dict(grid=dens)]
    if name == "sphere":
        lo, hi = scene.world_bounds()                           # frame_camera looks from centre + dist (1, 1, 1) at the centre
        dist = float(np.linalg.norm(hi - lo))
        u = np.ones(3) / np.sqrt(3.0); side = np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)
        put_sphere(scene, ((lo + hi) / 2 + 0.7 * dist * u + 0.12 * dist * side).tolist(), 0.08 * dist, (0.25, 0.5, 0.75))
    cam = scene.frame_camera(W1, H1)
    r = V.Renderer(scene, W1, H1, kp=make_kp(ray_depth=2), cam=cam)
    if name == "brick": r.set_brick_volume(perlin64)
    if name == "cells": r.set_cell_volume(perlin64)
    r.enable_collision_aovs()
    sc, mx = restated_scene(scene, vols)
    return scene, r, sc, mx, name in ("brick", "cells")


@pytest.fixture(scope="module")
def perlin64():
    """Power-of-two dimensions and an identity transform: volume_coord's every step is exact, so the restatement gets the GPU's uvw."""
    vol = V.Volume.procedural((64, 32, 32), res=1.0, scale=0.12, seed=7)
    vol.build_bricks(); vol.build_cells()
    return vol


@pytest.mark.parametrize("name", CASES)
def test_normal_and_albedo_against_the_restatement(perlin64, name):
    """At the GPU's own P (a one-pass frame holds P exactly):
    normal.  g_i comes from two densities, one float32 subtraction and a product by 1/(2h) (exact for h a power of two), then g . g by two
      fmas, a fast rsqrt (2^-22.9 relative) and three products: a few ulps of a unit vector, 2^-19 covers it.  In texture mode each density
      may differ from the restatement by one ulp of its largest corner texel (DESIGN.md section 3a; R.Scene.density's bound e), which moves
      n by at most 2 |e| / |g| (the change of a unit vector g / |g| under a perturbation e); that is added.
    albedo.  Four float32 products and a fast division (2^-22 relative): 2^-19 relative.  In texture mode Cd differs per channel by one ulp
      of its largest corner texel, which the albedo carries times albedo * lut / extinction * energy_inject.  A sample whose LUT argument
      lies within its own error of an integer may take the neighbouring entry: such ties are counted, capped at 0.1 %, and skipped.
    sphere.  Samples whose first collision is the sphere get normalize(P - c) (the same 2^-19) and the sphere's colour exactly."""
    scene, r, sc, mx, exact = surface_case(perlin64, name)
    pos, hit = one_pass(scene, r)
    nrm = r.buffers.normal.cpu().numpy().astype(np.float64)
    alb = r.buffers.albedo.cpu().numpy().astype(np.float64)
    assert hit.sum() > 300
    idx = np.nonzero(hit)[0]
    P = pos[idx, :3]
    sp = scene.h_sphere
    centre, radius = np.array([sp.center.x, sp.center.y, sp.center.z]), float(sp.radius)
    on_sphere = np.abs(np.linalg.norm(P - centre, axis=1) - radius) < 1e-3 * radius
    if name == "sphere":
        assert on_sphere.sum() > 50 and (~on_sphere).sum() > 50
        s = idx[on_sphere]
        assert np.abs(nrm[s] - R.sphere_normal(P[on_sphere], centre)).max() <= 2.0 ** -19 + 1e-3 * 2, "sphere normals"
        assert np.array_equal(alb[s].astype(F32), np.broadcast_to(np.array([0.25, 0.5, 0.75], F32), (len(s), 3))), "sphere colour"
    else:
        assert not on_sphere.any()
    vol = ~on_sphere
    Pv, iv = P[vol], idx[vol]
    h = float(F32(r.voxel_edge()))
    g, e = R.gradient(sc, Pv, h)
    want_n = R.normal_of_gradient(g)
    gn = np.linalg.norm(g, axis=1)
    bound = np.full(len(Pv), 2.0 ** -19)
    if not exact:
        bound = bound + np.minimum(2.0, 2 * np.linalg.norm(e, axis=1) / np.where(gn > 0, gn, 1e-300))
    err_n = np.abs(nrm[iv] - want_n).max(axis=1)
    assert (err_n <= bound).all(), f"{name}: normal off by {err_n.max():.3g}, bound {bound[np.argmax(err_n - bound)]:.3g}"
    assert (gn > 0).mean() > 0.5, "most collisions should see a density gradient"

    kp = r.kp
    rho, rho_err = sc.density(Pv)
    arg = R.lut_argument(rho, mx, kp.emission_pivot)
    arg_err = (0 if exact else rho_err * 255.0 / float(mx) / float(kp.emission_pivot)) + 8 * U24 * np.abs(arg) + 1e-7
    frac = arg - np.floor(arg)
    tie = (np.minimum(frac, 1 - frac) <= arg_err) & (arg > 0) & (arg < 255)
    assert tie.mean() <= 1e-3, f"{name}: {tie.sum()} LUT-index ties of {len(arg)}"
    lut = scene.d_density_color.cpu().numpy().reshape(256, 3)
    Cd = sc.color(Pv)
    alb_k = np.array([kp.albedo.x, kp.albedo.y, kp.albedo.z]); ext = np.array([kp.extinction.x, kp.extinction.y, kp.extinction.z])
    want_a = R.volume_albedo(alb_k, Cd, lut, R.lut_index(arg), ext, kp.energy_inject)
    tol_a = 2.0 ** -19 * np.abs(want_a) + 1e-30
    if name == "coloured":                                      # Cd through the texture unit: one ulp of each channel's largest corner
        uvw, _ = R.volume_coord(sc.recs[0], Pv)
        cmax = np.stack([np.abs(R.T.sample(sc.colors[0][..., k], uvw)["texels"]).max(1) for k in range(3)], 1)
        tol_a = tol_a + np.spacing(cmax.astype(F32)) * np.abs(R.volume_albedo(alb_k, np.ones_like(Cd), lut, R.lut_index(arg), ext,
                                                                                 kp.energy_inject))
        assert np.ptp(want_a[:, 0]) > 0.1, "the coloured volume must vary the albedo"
    err_a = np.abs(alb[iv] - want_a)
    ok = (err_a <= tol_a).all(axis=1) | tie
    assert ok.all(), f"{name}: albedo off by {err_a[~ok].max():.3g}"
    r.close()


# ---- 4: the running mean -------------------------------------------------------------------------------------------------------------------
def test_running_mean_from_prefilled_buffers(perlin64):
    scene, r, sc, mx, _ = surface_case(perlin64, "cells")
    r.enable_aovs()
    it = 5
    # the samples of pass `it`: a one-pass frame at sample offset `it` draws stream it, as the continued call at iteration it does
    r.set_sample_offset(it)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_(); r.render(1)         # activates the layers, the AOVs and the offset
    pos1 = r.buffers.position.clone(); n1 = r.buffers.normal.clone(); a1 = r.buffers.albedo.clone()
    r.set_sample_offset(0)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(1)                             # offset 0 takes over
    rng = np.random.default_rng(3)
    dev = r.buffers.accum.device
    X4 = torch.tensor(rng.uniform(-4, 4, (r.n_local, 4)).astype(F32), device=dev)
    X4[:, 3] = torch.tensor(rng.uniform(0, 1, r.n_local).astype(F32))
    X3 = torch.tensor(rng.uniform(-1, 1, (r.n_local, 3)).astype(F32), device=dev)
    r.buffers.position.copy_(X4); r.buffers.normal.copy_(X3); r.buffers.albedo.copy_(X3); r.buffers.alpha.copy_(X4[:, 3])
    scene.reset_blue_noise(); r.kp.iteration = it; r.render(1); torch.cuda.synchronize()
    assert same(r.buffers.position[:, 3], r.buffers.alpha), "position.w must be the alpha AOV at a continued iteration"
    for got, x, s in ((r.buffers.position, X4, pos1), (r.buffers.normal, X3, n1), (r.buffers.albedo, X3, a1)):
        want = R.running_mean(x.cpu().numpy(), s.cpu().numpy(), it, r.kp.max_interactions)
        assert np.allclose(got.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    r.close()


# ---- 5: composition ------------------------------------------------------------------------------------------------------------------------
def small_case(dragon, **kw):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(160, 96)
    def mk(**k2):
        r = V.Renderer(scene, 160, 96, kp=make_kp(ray_depth=2), cam=copy_cam(cam), **{**kw, **k2})
        r.set_option("passes_per_chunk", 5)
        return r
    return scene, mk


def test_adaptive_pixels_equal_the_fixed_count_frame_of_their_count(dragon):
    scene, mk = small_case(dragon)
    r = mk(); r.enable_aovs(); r.enable_collision_aovs()
    P, mn, iv = 16, 4, 4
    scene.reset_blue_noise(); r.kp.iteration = 0
    _, _, first = r.render_adaptive(P, threshold=FLT_MAX, min_passes=mn, check_interval=iv, error_map=True)
    thr = float(np.quantile(A.max3x3(first.cpu().numpy()), 0.5))
    scene.reset_blue_noise(); r.kp.iteration = 0
    _, counts = r.render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv)
    torch.cuda.synchronize()
    got = layers(r)
    assert same(got["position"][:, 3], r.buffers.alpha), "position.w must be the alpha AOV in an adaptive frame"
    counts = counts.reshape(-1)
    assert len(torch.unique(counts)) >= 2
    f = mk(); f.enable_collision_aovs()
    for n in torch.unique(counts).tolist():
        scene.reset_blue_noise(); f.kp.iteration = 0; f.render(int(n)); torch.cuda.synchronize()
        sel = counts == n
        for k, t in layers(f).items():
            assert same(got[k][sel], t[sel]), f"{k}: pixels that took {n} passes"


def test_region_equals_the_full_frame_inside_and_writes_nothing_outside(dragon):
    scene, mk = small_case(dragon)
    full = mk(); full.enable_collision_aovs()
    scene.reset_blue_noise(); full.kp.iteration = 0; full.render(8); torch.cuda.synchronize()
    r = mk(); r.enable_aovs(); r.enable_collision_aovs()
    x0, y0, x1, y1 = 37, 11, 121, 70
    r.set_region(x0, y0, x1, y1)
    for k in ("position", "normal", "albedo"): getattr(r.buffers, k).fill_(SENTINEL)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    inside = torch.zeros(96, 160, dtype=torch.bool, device=r.buffers.accum.device); inside[y0:y1, x0:x1] = True
    for k in ("position", "normal", "albedo"):
        c = getattr(r.buffers, k).shape[1]
        got, want = getattr(r.buffers, k).view(96, 160, c), getattr(full.buffers, k).view(96, 160, c)
        assert same(got[inside], want[inside]), k
        assert bool((got[~inside] == SENTINEL).all()), k
    assert same(r.buffers.position.view(96, 160, 4)[inside][:, 3], r.buffers.alpha.view(96, 160)[inside])


def test_four_partitioned_contexts_equal_the_single_context(dragon):
    scene, mk = small_case(dragon)
    one = mk(); one.enable_collision_aovs()
    scene.reset_blue_noise(); one.kp.iteration = 0; one.render(6); torch.cuda.synchronize()
    for k in range(4):
        sc = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        r = V.Renderer(sc, 160, 96, kp=make_kp(ray_depth=2), cam=copy_cam(one.cam), rank=k, n_ranks=4, stripe_rows=8)
        r.set_option("passes_per_chunk", 5)
        r.enable_collision_aovs(step=one.voxel_edge())
        r.kp.iteration = 0; r.render(6); torch.cuda.synchronize()
        rows = V.stripe_rows_of_rank(96, k, 4, 8)
        ok = rows < 96
        for name in ("position", "normal", "albedo"):
            c = getattr(one.buffers, name).shape[1]
            loc = getattr(r.buffers, name).view(-1, 160, c); want = getattr(one.buffers, name).view(96, 160, c)
            assert same(loc[torch.as_tensor(np.nonzero(ok)[0], device=loc.device)], want[torch.as_tensor(rows[ok], device=loc.device)]), f"rank {k} {name}"
        r.close()


# ---- 6: contract ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_activation_and_launch_count(dragon):
    scene, mk = small_case(dragon)
    r = mk()
    dev = r.buffers.accum.device
    buf = torch.zeros(r.n_local, 4, dtype=torch.float32, device=dev)
    for step in (0.0, -1.0, float("nan"), float("inf")):
        assert V.lib.vpt_set_collision_aovs(r.ctx, None, C.c_void_p(buf.data_ptr()), None, step) == -1
        assert b"gradient_step" in V.lib.vpt_last_error(r.ctx)

    # buffers registered mid-frame are not touched before the next iteration-0 call
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(3)
    r.enable_collision_aovs()
    for k in ("position", "normal", "albedo"): getattr(r.buffers, k).fill_(SENTINEL)
    r.render(2); torch.cuda.synchronize()
    for k in ("position", "normal", "albedo"): assert bool((getattr(r.buffers, k) == SENTINEL).all()), k
    before = r.stats()[0]
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    assert float(r.buffers.position[:, 3].max()) > 0.0
    with_layers = r.stats()[0] - before
    r.disable_collision_aovs()
    before = r.stats()[0]
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    assert with_layers - (r.stats()[0] - before) == 2, "one collision-AOV launch per chunk (5 + 3)"

    # a layer left out is not written; one buffer alone works
    r.enable_collision_aovs(position=False, normal=False, albedo=True)
    assert r.buffers.position is None and r.buffers.normal is None
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(2); torch.cuda.synchronize()
    assert float(r.buffers.albedo.abs().max()) > 0
    r.disable_collision_aovs()

    # overlapping buffers, named
    n = r.n_local
    acc = r.buffers.accum
    N.check(V.lib.vpt_set_collision_aovs(r.ctx, C.c_void_p(acc.data_ptr()), None, None, 1.0), r.ctx, "vpt_set_collision_aovs")
    r.kp.iteration = 0
    with pytest.raises(V.VptError, match="position buffer overlaps Kernel_params.accum_buffer"):
        r.render(1)
    r.enable_motion_vectors(copy_cam(r.cam))
    N.check(V.lib.vpt_set_collision_aovs(r.ctx, None, None, C.c_void_p(r.buffers.motion.data_ptr()), 1.0), r.ctx, "vpt_set_collision_aovs")
    r.kp.iteration = 0
    with pytest.raises(V.VptError, match="albedo buffer overlaps the motion-vector buffer"):
        r.render(1)
    r.disable_motion_vectors()
    both = torch.zeros(n * 4, dtype=torch.float32, device=dev)
    N.check(V.lib.vpt_set_collision_aovs(r.ctx, C.c_void_p(both.data_ptr()), C.c_void_p(both.data_ptr() + 4 * n), None, 1.0), r.ctx,
            "vpt_set_collision_aovs")
    r.kp.iteration = 0
    with pytest.raises(V.VptError, match="the position buffer and the normal buffer overlap"):
        r.render(1)
    r.disable_collision_aovs()

    # panoramas
    for kind in ("equirect", "ods"):
        p = mk(); p.set_projection(kind); p.enable_collision_aovs()
        p.kp.iteration = 0
        with pytest.raises(V.VptError, match=r"\(-3\).*collision AOVs"):
            p.render(1)
        p.close()
    r.close()
