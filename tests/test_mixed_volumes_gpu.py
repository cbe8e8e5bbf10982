"""Scenes of DIFFERENT volumes against the reference kernel (tests/mixed_scenes.py: the dragon plus three synthetic volumes with their
own grid sizes, bounds, majorants, a heat grid at its own resolution and a colour grid).

Every multi-instance test elsewhere instances one VDB, so there a kernel that read volume 0's record for every leaf entry, dropped
a leaf entry from the colour or emission loops, or gave every octree node the root's majorant would still pass.  Here:
  * the octree node for node (volume lists, boxes, majorants) and the flat leaf lists against the reference builder;
  * frames against the live reference kernel under both integrators, HDRI, Bruneton sky and tabulated-sky MIS, with emission
    (scale 1 and -0.5), colour, point lights and the sphere; single coloured / emissive volumes; 40 mixed instances; staged assets;
  * this library on the reference's pointer-linked octree, level (A) through the reference loader, lean against generic kernels on
    a coloured volume, four-stripe partitions and light groups;
  * the committed fixture tests/golden/mixed_direct.npz (the reference kernel's own output), which needs no oracle build.
Tolerances as in test_parity_gpu.py.  Each case also checks that its feature is really in the frame: a lit frame, colour grids whose
removal changes more pixels than the tolerance lets flip, an emission that changes it."""
import contextlib
import json
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
import oracle_ref
import mixed_scenes as M
import test_light_groups_gpu as LG
from test_parity_gpu import MAX_FLIPPED, ATOL, RTOL, flipped_fraction, make_kp, needs_ref, _sky_power_table
from test_scale_gpu import LEVEL_A, _launch_candidate, assert_trees_equal

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_live = pytest.mark.skipif(not oracle_ref.available(), reason="oracle/_ref not built")


@pytest.fixture(scope="module")
def vols():
    return M.Volumes()


@pytest.fixture(scope="module")
def atmosphere():
    return V.Atmosphere()


@pytest.fixture(scope="module")
def tables():
    t = V.EnvTables(_sky_power_table())
    yield t
    t.destroy()


SINGLE = {"ember": [("ember", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0)],
          "tint": [("tint", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0)]}


@pytest.fixture(scope="module")
def scenes(vols, atmosphere):
    """name -> Scene (made once; every scene carries this library's Bruneton tables, which HDRI frames never read)."""
    cache = {}
    build = {"S1": M.build_s1, "S2": M.build_s2, "S3": M.build_s3, "S4": M.build_s4}

    def get(name):
        if name not in cache:
            s = build[name](vols) if name in build else M.build(vols, SINGLE[name], lights=False, sphere=False)
            if s is None:
                pytest.skip("fireball.vdb / colored_smoke.vdb not staged (oracle/_ref/assets)")
            atmosphere.apply(s.atmos)
            cache[name] = s
        return cache[name]
    return get


def bad_pixels(got, want):
    got = np.asarray(got, np.float64).reshape(len(want), -1); want = np.asarray(want, np.float64).reshape(len(want), -1)
    return int((np.abs(got - want) > ATOL + RTOL * np.abs(want)).any(axis=1).sum())


def kernel_params(cfg, **over):
    kw = dict(integrator=cfg.get("integrator", 0), environment_type=cfg.get("env", 1), emission_scale=cfg.get("emission", 1.0),
              emission_pivot=1.0, **cfg["kp"])
    if kw["environment_type"] == 0: kw["elevation"] = 35.0
    kw.update(over)
    return make_kp(**kw)


def reference_frame(scene, cfg, orc, tables, cam, root, colour=True, **over):
    """(renderer holding the reference kernel's frame, blue noise after it) from iteration 0 on the reference-built octree;
    colour=False: with every colour grid switched off (mixed_scenes.colour_grids_off)."""
    ref = V.Renderer(scene, cfg["W"], cfg["H"], kp=kernel_params(cfg, **over), cam=cam)
    if ref.kp.integrator == 1 and ref.kp.environment_type == 0: tables.apply(ref.kp)
    ref.params.p_oct.value = root
    with (contextlib.nullcontext() if colour else M.colour_grids_off(scene)):
        scene.reset_blue_noise(); orc.render(ref, cfg["passes"])
    return ref, scene.d_blue_noise.clone()


def colour_moves(with_colour, without, what):
    """The colour grids change more pixels than the parity tolerance lets flip, so a frame that lost them cannot pass."""
    frac = flipped_fraction(with_colour, without)
    print(f"{what}: the colour grids change {100 * frac:.2f} % of the pixels")
    assert frac > 2 * MAX_FLIPPED, f"{what}: the colour grids change only {100 * frac:.3f} % of the pixels"


CASES = {
    "s1_direct_hdri":      dict(scene="S1", W=248, H=152, passes=2, kp=dict(ray_depth=3, volume_depth=2)),
    "s2_direct_hdri":      dict(scene="S2", W=248, H=152, passes=2, kp=dict(ray_depth=3, volume_depth=2)),
    "s1_direct_sky":       dict(scene="S1", W=232, H=136, passes=2, env=0, kp=dict(ray_depth=3, volume_depth=2)),
    "s1_vol_hdri":         dict(scene="S1", W=216, H=136, passes=2, integrator=1, kp=dict(ray_depth=6)),
    "s1_vol_table":        dict(scene="S1", W=200, H=120, passes=2, integrator=1, env=0, kp=dict(ray_depth=6)),
    "s1_direct_emit_neg":  dict(scene="S1", W=200, H=120, passes=2, emission=-0.5, kp=dict(ray_depth=3, volume_depth=2)),
    "s1_vol_emit_neg":     dict(scene="S1", W=200, H=120, passes=2, integrator=1, emission=-0.5, kp=dict(ray_depth=6)),
    "ember_vol":           dict(scene="ember", W=176, H=112, passes=3, integrator=1, kp=dict(ray_depth=6, volume_depth=3)),
    "tint_direct":         dict(scene="tint", W=200, H=128, passes=2, emission=0.0, kp=dict(ray_depth=3, volume_depth=3)),
    "tint_vol":            dict(scene="tint", W=200, H=128, passes=2, integrator=1, emission=0.0, kp=dict(ray_depth=6)),
    "s3_direct":           dict(scene="S3", W=256, H=144, passes=2, kp=dict(ray_depth=2, volume_depth=2)),
    "s4_direct":           dict(scene="S4", W=256, H=144, passes=2, kp=dict(ray_depth=2, volume_depth=2)),
}
TINTED = ("S1", "S2", "S3", "S4", "tint")
EMISSIVE = ("S1", "S2", "S3", "S4", "ember")


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_mixed_volumes_against_reference_kernel(scenes, tables, name):
    cfg = CASES[name]
    scene = scenes(cfg["scene"])
    W, H, P = cfg["W"], cfg["H"], cfg["passes"]
    integ, env, emission = cfg.get("integrator", 0), cfg.get("env", 1), cfg.get("emission", 1.0)
    orc = oracle_ref.RefOracle()
    cam = scene.frame_camera(W, H)
    root = orc.build_octree(scene.h_volumes, len(scene.instances))
    ref, bn_ref = reference_frame(scene, cfg, orc, tables, cam, root)
    mine = V.Renderer(scene, W, H, kp=kernel_params(cfg), cam=cam)
    if integ == 1 and env == 0: tables.apply(mine.kp)
    scene.reset_blue_noise(); mine.render(P); torch.cuda.synchronize()
    bn_mine = scene.d_blue_noise.clone()

    want = ref.buffers.accum.cpu().numpy(); got = mine.buffers.accum.cpu().numpy()
    dist = M.max_distinct_per_leaf(scene)
    print(f"{name}: {bad_pixels(got, want)} of {W * H} pixels outside tolerance, max |d| {np.abs(got - want).max():.3g}, "
          f"reference mean {want.mean():.6g}, max distinct volumes in one leaf {dist}")
    # the feature is in the frame
    assert np.isfinite(want).all() and float(want.mean()) > 1e-3, "the frame must be lit"
    if cfg["scene"] in TINTED:
        grey, _ = reference_frame(scene, cfg, orc, tables, cam, root, colour=False)
        colour_moves(want, grey.buffers.accum.cpu().numpy(), name)
    if cfg["scene"] in EMISSIVE and emission != 0.0:
        dark, _ = reference_frame(scene, cfg, orc, tables, cam, root, emission_scale=0.0)
        same = torch.equal(dark.buffers.accum, ref.buffers.accum)
        # the reference gates the direct integrator's emission walk on > 0 and the volumetric one on != 0
        assert same == (integ == 0 and emission < 0), f"emission_scale {emission} vs 0: frames equal = {same}"

    # integrator 1: the limits measured for the volumetric path integrator (test_parity_gpu); integrator 0: MAX_FLIPPED
    limit = (1e-4 if env == 0 else 0.0) if integ == 1 else MAX_FLIPPED
    assert flipped_fraction(got, want) <= limit
    dfrac = flipped_fraction(mine.buffers.depth.cpu().numpy()[:, None], ref.buffers.depth.cpu().numpy()[:, None])
    assert dfrac <= (0.0 if integ == 1 else MAX_FLIPPED)
    raw_m = mine.buffers.raw.cpu().numpy().reshape(-1, 4); raw_r = ref.buffers.raw.cpu().numpy().reshape(-1, 4)
    if oracle_ref.available():                       # a replayed oracle stores only the transmittance channel of raw
        assert flipped_fraction(raw_m[:, :3], raw_r[:, :3]) <= MAX_FLIPPED
    assert np.mean(np.abs(raw_m[:, 3] - raw_r[:, 3]) > 1e-5) <= MAX_FLIPPED      # tr: replayed depth-walk sum, see DESIGN.md
    dm = mine.buffers.display.cpu().numpy().view(np.uint8).reshape(-1, 4).astype(int)
    dr = ref.buffers.display.cpu().numpy().view(np.uint8).reshape(-1, 4).astype(int)
    assert np.abs(dm - dr).max() <= 1 and np.mean(np.abs(dm - dr).max(axis=1) > 0) <= MAX_FLIPPED
    assert torch.equal(bn_mine, bn_ref), "blue-noise state must be bit-exact"
    assert float(mine.buffers.cost.abs().max()) == 0.0
    assert mine.kp.iteration == ref.kp.iteration == P


@needs_ref
@pytest.mark.parametrize("name", ["S1", "S3"])
def test_octree_and_leaf_lists_node_for_node(scenes, name):
    """bbox, volume lists and both majorants bit for bit against the reference builder; the flat leaf lists the kernels read equal
    the reference's leaf nodes.  The majorants really vary: the root's is ember's, not instance 0's, and (S3) inner nodes differ."""
    scene = scenes(name)
    n = len(scene.instances)
    ref_t = oracle_ref.RefOracle().octree_nodes(scene.h_volumes, n)
    mine_t = M.read_tree(scene.d_oct_root)
    assert_trees_equal(mine_t, ref_t)
    lists = scene.leaf_lists()
    for l in range(512):
        j = 73 + l
        assert lists[l] == (list(ref_t[j].vol_indices[:ref_t[j].num_volumes]) if j in ref_t else []), l
    majorants = sorted({nd.max_extinction for j, nd in ref_t.items() if nd.num_volumes})
    print(f"{name}: {len(ref_t)} nodes, max distinct volumes in one leaf {M.max_distinct_per_leaf(scene)}, node majorants {majorants}")
    assert ref_t[0].max_extinction != scene.h_volumes[0].vdb_info.max_density
    assert len(majorants) >= (3 if name == "S3" else 2)


@needs_live
@pytest.mark.parametrize("name", ["S1", "S3"])
def test_reference_built_octree_renders_like_the_own_octree(scenes, name):
    """k_prepare_scene's flattening of the reference's pointer-linked octree gives the frame of the library's own octree, bit for bit."""
    scene = scenes(name)
    W, H = 200, 120
    kp = dict(ray_depth=3, volume_depth=2, emission_scale=1.0, emission_pivot=1.0)
    mine = V.Renderer(scene, W, H, kp=make_kp(**kp)); foreign = V.Renderer(scene, W, H, kp=make_kp(**kp), cam=mine.cam)
    foreign.params.p_oct.value = oracle_ref.RefOracle().build_octree(scene.h_volumes, len(scene.instances))
    scene.reset_blue_noise(); mine.render(2)
    scene.reset_blue_noise(); foreign.render(2); torch.cuda.synchronize()
    assert float(mine.buffers.accum.mean()) > 1e-3
    for k in ("accum", "depth", "raw", "display"):
        assert torch.equal(getattr(mine.buffers, k), getattr(foreign.buffers, k)), k


@needs_ref
@pytest.mark.skipif(not os.path.exists(LEVEL_A), reason="volume_rt_kernel_b200.cubin not built")
@pytest.mark.parametrize("integrator", [0, 1])
def test_level_a_on_mixed_volumes_through_the_reference_loader(scenes, integrator):
    """Level (A) reads the leaf lists from the caller's OCTNodes and takes single_volume from the root's num_volumes (4 here)."""
    scene = scenes("S1")
    orc = oracle_ref.RefOracle(); orc.load_kernels(); orc.load_candidate(LEVEL_A)
    W, H, P = 200, 120, 2
    kw = dict(integrator=integrator, ray_depth=3 if integrator == 0 else 6, volume_depth=2, emission_scale=1.0, emission_pivot=1.0)
    cam = scene.frame_camera(W, H)
    a = V.Renderer(scene, W, H, kp=make_kp(**kw), cam=cam); ref = V.Renderer(scene, W, H, kp=make_kp(**kw), cam=cam)
    root = orc.build_octree(scene.h_volumes, len(scene.instances))
    a.params.p_oct.value = root; ref.params.p_oct.value = root
    scene.reset_blue_noise(); orc.render(ref, P); bn_ref = scene.d_blue_noise.clone()
    scene.reset_blue_noise(); _launch_candidate(orc, a, P)
    want = ref.buffers.accum.cpu().numpy(); got = a.buffers.accum.cpu().numpy()
    print(f"level A S1 integrator {integrator}: {bad_pixels(got, want)} of {W * H} pixels outside tolerance, max |d| "
          f"{np.abs(got - want).max():.3g}, reference mean {want.mean():.6g}, max distinct volumes in one leaf {M.max_distinct_per_leaf(scene)}")
    assert float(want.mean()) > 1e-3 and flipped_fraction(got, want) <= MAX_FLIPPED
    assert flipped_fraction(a.buffers.depth.cpu().numpy()[:, None], ref.buffers.depth.cpu().numpy()[:, None]) <= MAX_FLIPPED
    assert torch.equal(scene.d_blue_noise, bn_ref)
    assert float(a.buffers.cost.abs().max()) == 0.0
    dm = a.buffers.display.cpu().numpy().view(np.uint8).reshape(-1, 4).astype(int)
    dr = ref.buffers.display.cpu().numpy().view(np.uint8).reshape(-1, 4).astype(int)
    assert np.abs(dm - dr).max() <= 1


def test_lean_and_generic_kernels_agree_bitwise_on_a_coloured_volume(scenes):
    """One volume with a colour grid, no lights, no emission: the lean kernel (colour inline in the tracking step) and the generic
    kernel (colour in scatter_event) give the same frame bit for bit, and in each the colour grid really reaches the frame."""
    scene = scenes("tint")
    frames = {}
    for kernel, opts in (("lean", {}), ("generic", {"generic_kernel": 1})):
        for colour in (True, False):
            r = V.Renderer(scene, 256, 160, kp=make_kp(ray_depth=100, emission_scale=0.0), options=opts)
            with (contextlib.nullcontext() if colour else M.colour_grids_off(scene)):
                scene.reset_blue_noise(); r.render(4); torch.cuda.synchronize()
            frames[kernel, colour] = r
    a, b = frames["lean", True], frames["generic", True]
    for k in ("accum", "depth", "raw", "display"):
        assert torch.equal(getattr(a.buffers, k), getattr(b.buffers, k)), k
    for kernel in ("lean", "generic"):
        colour_moves(frames[kernel, True].buffers.accum.cpu().numpy(), frames[kernel, False].buffers.accum.cpu().numpy(), kernel)


def test_partition_invariance_on_mixed_volumes(scenes):
    W, H = 256, 160
    scene = scenes("S1")
    kp = dict(ray_depth=3, volume_depth=2, emission_scale=1.0, emission_pivot=1.0)
    one = V.Renderer(scene, W, H, kp=make_kp(**kp))
    scene.reset_blue_noise(); one.render(3); torch.cuda.synchronize()
    parts = []
    for rank in range(4):
        r = V.Renderer(scene, W, H, kp=make_kp(**kp), cam=one.cam, rank=rank, n_ranks=4, stripe_rows=8,
                       options=dict(passes_per_chunk=rank + 1))
        scene.reset_blue_noise(); r.render(3); parts.append(r)
    torch.cuda.synchronize()
    full = parts[0].unpermute(torch.cat([p.buffers.accum for p in parts], dim=0), 3)
    assert torch.equal(full, one.buffers.accum)
    for r in parts: r.close()


def test_light_groups_on_mixed_volumes(scenes):
    """Direct integrator on S1: each group is the render lit by its class alone (sun, point and environment without emission; the
    emission group with it) and the groups sum to the beauty."""
    scene = scenes("S1")
    W, H = 200, 120
    cam = scene.frame_camera(W, H)
    powers = [l[2] for l in M.LIGHTS]
    for emission in (0.0, 1.0):
        kw = dict(ray_depth=3, volume_depth=2, emission_scale=emission, emission_pivot=1.0)
        case = dict(scene=scene, mk0=lambda kw=kw: V.Renderer(scene, W, H, kp=make_kp(**kw), cam=cam), integrator=0, sky="hdri",
                    lights=True, emission=emission > 0)
        on = LG.frame(scene, LG.renderer(case), LG.PASSES)
        LG.assert_sum_is_the_beauty(on, f"S1, emission_scale {emission}")
        assert float(on["point"].max()) > 1e-4 and float(on["sun"].max()) > 1e-3 and float(on["environment"].max()) > 1e-3
        if emission: assert float(on["emission"].max()) > 1e-4
        else: assert bool((on["emission"] == 0).all())
        for lit in LG.GROUPS:
            if case["emission"] != (lit == "emission"):
                continue
            kp, powers_on = LG.solo_params(case, lit)
            if not powers_on: LG.set_light_power(scene, [0.0] * len(powers))
            try:
                solo = LG.frame(scene, LG.renderer(case, groups=False, **kp), LG.PASSES)
            finally:
                LG.set_light_power(scene, powers)
            assert LG.bitwise(on[lit], solo["accum"]), f"group {lit} is not the render lit by {lit} alone " \
                                                      f"(max |d| {float((on[lit] - solo['accum']).abs().max())})"


def test_mixed_direct_against_reference_golden(scenes):
    """tests/golden/mixed_direct.npz: the UNMODIFIED reference kernel on S1 (HDRI, point lights, sphere, emission, colour)."""
    g = np.load(os.path.join(GOLD, "mixed_direct.npz"))
    meta = json.loads(str(g["meta"]))
    scene = scenes(meta["scene"])
    H, W = meta["H"], meta["W"]
    r = V.Renderer(scene, W, H, kp=make_kp(**meta["kp"]))
    assert bytes(r.cam) == g["camera"].tobytes(), "camera set-up drifted from the fixture"
    scene.reset_blue_noise(); r.render(meta["passes"]); torch.cuda.synchronize()
    got = r.buffers.accum.cpu().numpy()
    print(f"mixed_direct golden: {bad_pixels(got, g['accum'].reshape(-1, 3))} of {W * H} pixels outside tolerance, max |d| "
          f"{np.abs(got - g['accum'].reshape(-1, 3)).max():.3g}, reference mean {g['accum'].mean():.6g}, "
          f"max distinct volumes in one leaf {M.max_distinct_per_leaf(scene)}")
    assert flipped_fraction(got.reshape(H, W, 3), g["accum"]) <= MAX_FLIPPED
    assert flipped_fraction(r.buffers.depth.cpu().numpy().reshape(H, W, 1), g["depth"][..., None]) <= MAX_FLIPPED
    raw = r.buffers.raw.cpu().numpy().reshape(H, W, 4)
    assert flipped_fraction(raw[..., :3], g["raw"][..., :3]) <= MAX_FLIPPED
    assert np.mean(np.abs(raw[..., 3] - g["raw"][..., 3]) > 1e-5) <= MAX_FLIPPED
    dm = r.buffers.display.cpu().numpy().view(np.uint8).reshape(-1, 4).astype(int)
    dg = g["display"].astype(np.int32).view(np.uint8).reshape(-1, 4).astype(int)
    assert np.abs(dm - dg).max() <= 1 and np.mean(np.abs(dm - dg).max(axis=1) > 0) <= MAX_FLIPPED
    assert np.array_equal(scene.d_blue_noise.cpu().numpy(), g["blue_noise"]), "blue-noise state must be bit-exact"
    assert float(r.buffers.cost.abs().max()) == 0.0
    grey = V.Renderer(scene, W, H, kp=make_kp(**meta["kp"]))
    with M.colour_grids_off(scene):
        scene.reset_blue_noise(); grey.render(meta["passes"]); torch.cuda.synchronize()
    colour_moves(g["accum"].reshape(-1, 3), grey.buffers.accum.cpu().numpy(), "mixed_direct golden")
