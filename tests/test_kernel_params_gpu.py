"""The scene-wide volume, light and phase parameters of Kernel_params against the reference kernel, away from their defaults.

The defaults are multiplicative identities (albedo = extinction = sun_color = sky_color = (1, 1, 1), energy_inject = 1), so a frame
rendered at them cannot show a dropped factor, a swapped channel, albedo and extinction exchanged, a missing sky_color in one of the
places the environment term is finished, or the operation order of the emission walk's fma(-x, rcp(extinction.x), t).  Here:

  P1  collision throughput albedo * Cd * density_colour / extinction * energy_inject: lean kernel at 2 and 3 rays per lane, generic
      kernel, level (A), a colour grid (lean and generic), mixed scene S1 under both integrators and both skies; brick and cell mode
      against the texture path;
  P2  the emission walk's step (1 / extinction.x, tr_depth) on S1 under both integrators and both emission gates (> 0 / != 0);
  P3  sun_color, sun_mult, sky_color, sky_mult through the compact and wide HDRI records, k_resolve<1>, k_resolve<2> with the in-path
      sky, and level (A) on HDRI and the Bruneton sky;
  P4  the sun direction: azimuth and elevation inside and outside their clamps;
  P5  the Henyey-Greenstein phase at |g| around EPS = 0.001 and near +-1, under both integrators;
  P6  the colour and emission LUT index through emission_pivot;
  P7  the NaN / Inf guard fed by the parameters (extinction.y = 0, albedo 0, energy_inject 0) from prefilled buffers;
  P8  the fields the reference never reads (phase_g2, phase_f, min_extinction, transmittance, debug): the frame does not move;
  and the committed fixture tests/golden/mixed_params.npz (the unmodified reference kernel on S1 at non-default parameters).

Rule against the reference (as in the projection, ODS and motion tests): accum, depth and raw.xyz within 1e-5 + 1e-4 |ref| on all but
MAX_FLIPPED of the pixels, raw.w within 1e-5 on as many, display words within 1 LSB, cost and blue noise bit-equal.  Each case prints the
flipped share, the share of bit-equal accum values and the largest |difference|.  Each case also shows that its parameter is in the
frame: the reference frame with the parameter (or the group's parameters) back at the default differs from it on at least 1 % of the
pixels beyond the tolerance -- ten times what the rule lets flip.

Stored reference outputs under tests/golden/oracle/ replay the comparisons where oracle/_ref is not built."""
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
import oracle_ref
import mixed_scenes as M
from vpt_b200.scene import synthetic_env
from test_parity_gpu import GOLD, MAX_FLIPPED, flipped_fraction, make_kp, make_scene, needs_ref, _big_asset
from test_scale_gpu import LEVEL_A, _launch_candidate
from test_resolve_tail_gpu import prefill

pytestmark = pytest.mark.gpu
needs_level_a = pytest.mark.skipif(not os.path.exists(LEVEL_A), reason="volume_rt_kernel_b200.cubin not built")

P1 = dict(albedo=(0.9, 0.55, 0.3), extinction=(0.8, 1.25, 2.0), energy_inject=1.01234)
P3 = dict(sun_color=(1.0, 0.55, 0.2), sun_mult=2.5, sky_color=(0.3, 0.6, 1.2), sky_mult=0.7)
GUARD = 0.01                                   # the parameter moves at least 1 % of the pixels beyond the tolerance
FOV = 20.0                                     # narrower than frame_camera's 30 degrees: the volumes cover more of the small frames
_i = np.arange(256, dtype=np.float32) / np.float32(255)
LUT_RAMP = np.stack([1 - 0.55 * _i, 0.35 + 0.65 * _i, 0.8 + 0.2 * np.cos(3 * _i)], axis=-1).astype(np.float32)


def kp_of(**kw):
    return make_kp(**{k: V.f3(*v) if isinstance(v, (tuple, list)) else v for k, v in kw.items()})


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def vols():
    return M.Volumes()


@pytest.fixture(scope="module")
def atmosphere():
    return V.Atmosphere()


@pytest.fixture(scope="module")
def scenes(dragon, vols, atmosphere):
    """name -> Scene, made once: the dragon over the procedural HDRI (with and without the point lights and the sphere), the tint
    volume alone (a colour grid), S1, and the staged fireball / coloured smoke.  Every scene carries this library's Bruneton tables.
    The density-colour LUT of the assets is white at every index, so a frame cannot show where the kernels index it; every scene here
    carries LUT_RAMP, a coloured ramp, instead (both kernels read the LUT through Kernel_params.density_color_texture)."""
    cache = {}

    def get(name):
        if name not in cache:
            if name == "dragon":
                s = make_scene(dragon)
            elif name == "dragon_lit":
                s = make_scene(dragon, lights=M.LIGHTS); M.place_sphere(s)
            elif name == "tint":
                s = M.build(vols, [("tint", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0)], lights=False, sphere=False)
            elif name == "S1":
                s = M.build_s1(vols)
            else:
                path = _big_asset({"fireball": "fireball.vdb", "smoke": "colored_smoke.vdb"}[name])
                if path is None:
                    pytest.skip(f"{name} asset not staged (oracle/_ref/assets)")
                vol = V.Volume.load_vdb(path)
                s = V.Scene([vol.instance()], env=synthetic_env(512, 256), keep=[vol])
            atmosphere.apply(s.atmos)
            s.d_density_color.copy_(torch.from_numpy(LUT_RAMP).reshape(s.d_density_color.shape))
            cache[name] = s
        return cache[name]
    return get


# ---- running both kernels --------------------------------------------------------------------------------------------------------------
class Frame:
    """One scene, camera and size; renders the reference kernel and this library's variants from the same iteration and blue noise."""

    def __init__(self, scene, W, H, passes, aperture=0.0, fill=None):
        self.scene, self.W, self.H, self.P, self.fill = scene, W, H, passes, fill
        self.cam = scene.frame_camera(W, H, fov=FOV, aperture=aperture)
        self.orc = oracle_ref.RefOracle()
        self.root = self.orc.build_octree(scene.h_volumes, len(scene.instances))
        self.tables = []

    def _renderer(self, kw, options=None):
        kw = dict(kw)
        r = V.Renderer(self.scene, self.W, self.H, kp=kp_of(**kw), cam=self.cam, options=options)
        if r.kp.integrator == 1 and r.kp.environment_type == 0:
            # the reference's create_cdf tabulates the sky of the frame's own azimuth, elevation and sky_color
            t = V.EnvTables(V.sky_power_table(r.kp.azimuth, r.kp.elevation, (r.kp.sky_color.x, r.kp.sky_color.y, r.kp.sky_color.z)))
            t.apply(r.kp); self.tables.append(t)
        if self.fill: self.fill(r.buffers)
        return r

    def _out(self, r):
        torch.cuda.synchronize()
        b = r.buffers
        return dict(accum=b.accum.cpu().numpy(), depth=b.depth.cpu().numpy(), cost=b.cost.cpu().numpy(), raw=b.raw.cpu().numpy(),
                    display=b.display.cpu().numpy().view(np.uint32), bn=self.scene.d_blue_noise.cpu().numpy(), iteration=int(r.kp.iteration))

    def reference(self, full=True, **kw):
        """full=False for a frame that only the non-vacuity check reads: its stored output then carries no cost and no raw.xyz."""
        r = self._renderer(kw)
        r.params.p_oct.value = self.root
        self.scene.reset_blue_noise(); self.orc.render(r, self.P, full=full)
        return self._out(r)

    def library(self, options=None, **kw):
        r = self._renderer(kw, options)
        self.scene.reset_blue_noise(); r.render(self.P)
        return self._out(r)

    def level_a(self, **kw):
        self.orc.load_kernels(); self.orc.load_candidate(LEVEL_A)
        r = self._renderer(kw)
        r.params.p_oct.value = self.root
        self.scene.reset_blue_noise(); _launch_candidate(self.orc, r, self.P)
        return self._out(r)

    def close(self):
        for t in self.tables: t.destroy()
        self.tables.clear()


def stats(got, want):
    a, b = got["accum"], want["accum"]
    return flipped_fraction(a, b), float((a.view(np.int32) == b.view(np.int32)).mean()), float(np.nanmax(np.abs(a.astype(np.float64) - b)))


def assert_matches(got, want, what):
    """The per-pixel rule against the reference kernel's outputs."""
    frac, exact, dmax = stats(got, want)
    print(f"{what}: flipped {frac:.3g}, bit-equal {100 * exact:.2f} %, max |d| {dmax:.3g}")
    assert np.isfinite(want["accum"]).all(), f"{what}: the reference frame is not finite"
    assert frac <= MAX_FLIPPED, f"{what}: accum"
    assert flipped_fraction(got["depth"][:, None], want["depth"][:, None]) <= MAX_FLIPPED, f"{what}: depth"
    assert flipped_fraction(got["raw"][:, :3], want["raw"][:, :3]) <= MAX_FLIPPED, f"{what}: raw.xyz"
    assert np.mean(np.abs(got["raw"][:, 3] - want["raw"][:, 3]) > 1e-5) <= MAX_FLIPPED, f"{what}: raw.w"
    dm = got["display"].view(np.uint8).reshape(-1, 4).astype(int); dr = want["display"].view(np.uint8).reshape(-1, 4).astype(int)
    assert np.abs(dm - dr).max() <= 1 and np.mean(np.abs(dm - dr).max(axis=1) > 0) <= MAX_FLIPPED, f"{what}: display"
    assert np.array_equal(got["cost"].view(np.int32), want["cost"].view(np.int32)), f"{what}: cost must be bit-equal"
    assert np.array_equal(got["bn"], want["bn"]), f"{what}: blue-noise state must be bit-equal"
    assert got["iteration"] == want["iteration"], f"{what}: iteration"


def assert_moves(want, default, what):
    """Non-vacuity: the parameter changes the reference frame on at least GUARD of the pixels beyond the tolerance."""
    frac = flipped_fraction(want["accum"], default["accum"])
    print(f"{what}: the parameter moves {100 * frac:.2f} % of the pixels")
    assert frac >= GUARD, f"{what}: the parameter moves only {100 * frac:.3f} % of the pixels"


# ---- P1: collision throughput ----------------------------------------------------------------------------------------------------------
@needs_ref
@needs_level_a
@pytest.mark.parametrize("name", ["dragon", "tint"])
def test_collision_throughput_single_volume(scenes, name):
    """One volume (the dragon; the tint volume's colour grid, so Cd != 1): the lean kernel inline at 2 and 3 rays per lane (both beta
    layouts), the generic kernel's scatter_event and level (A), all against one reference frame."""
    f = Frame(scenes(name), 200, 120, 2)
    kw = dict(ray_depth=3, volume_depth=2)
    want = f.reference(**kw, **P1)
    assert_moves(want, f.reference(full=False, **kw), f"P1 {name}")
    for label, opts in (("lean", {}), ("lean, 3 rays per lane", {"trace_slots": 3}), ("generic", {"generic_kernel": 1})):
        assert_matches(f.library(opts, **kw, **P1), want, f"P1 {name} {label}")
    assert_matches(f.level_a(**kw, **P1), want, f"P1 {name} level A")


@needs_ref
@pytest.mark.parametrize("name", ["smoke"])
def test_collision_throughput_coloured_smoke(scenes, name):
    """colored_smoke.vdb: a colour grid and the density-colour LUT at density_mult 4."""
    f = Frame(scenes(name), 200, 120, 2)
    kw = dict(ray_depth=2, volume_depth=4, density_mult=4.0)
    want = f.reference(**kw, **P1)
    assert_moves(want, f.reference(full=False, **kw), f"P1 {name}")
    assert_matches(f.library(**kw, **P1), want, f"P1 {name}")


@needs_ref
@needs_level_a
@pytest.mark.parametrize("integrator,env", [(0, 1), (1, 1), (1, 0)])
def test_collision_throughput_mixed_volumes(scenes, integrator, env):
    """S1 (four volumes, emission, colour, point lights, sphere) under both integrators, on the HDRI and (integrator 1) on the
    tabulated sky; this library's wavefront path and level (A)."""
    f = Frame(scenes("S1"), 200, 120, 2)
    kw = dict(integrator=integrator, environment_type=env, ray_depth=3 if integrator == 0 else 6, volume_depth=2,
              emission_scale=1.0, emission_pivot=1.0)
    try:
        want = f.reference(**kw, **P1)
        assert_moves(want, f.reference(full=False, **kw), f"P1 S1 integrator {integrator} env {env}")
        assert_matches(f.library(**kw, **P1), want, f"P1 S1 integrator {integrator} env {env}")
        if env == 1:
            assert_matches(f.level_a(**kw, **P1), want, f"P1 S1 integrator {integrator} env {env} level A")
    finally:
        f.close()


@needs_ref
@pytest.mark.parametrize("env", [1, 0])
def test_collision_throughput_volumetric_integrator_on_the_dragon(scenes, env):
    f = Frame(scenes("dragon"), 200, 120, 2)
    kw = dict(integrator=1, environment_type=env, ray_depth=6)
    try:
        want = f.reference(**kw, **P1)
        assert_moves(want, f.reference(full=False, **kw), f"P1 dragon integrator 1 env {env}")
        assert_matches(f.library(**kw, **P1), want, f"P1 dragon integrator 1 env {env}")
    finally:
        f.close()


@pytest.mark.parametrize("mode", ["brick", "cell"])
def test_collision_throughput_brick_and_cell_modes(mode):
    """The brick (TMA) and cell samplers against the texture path at the P1 parameters, with the tolerance of test_bricks_gpu."""
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks() if mode == "brick" else vol.build_cells()
    scene = V.Scene([vol.instance()], env=synthetic_env(512, 256), keep=[vol])
    scene.d_density_color.copy_(torch.from_numpy(LUT_RAMP).reshape(scene.d_density_color.shape))
    W, H = 320, 200
    cam = scene.frame_camera(W, H, fov=FOV)
    kw = dict(ray_depth=2, volume_depth=2)

    def run(fast, **over):
        r = V.Renderer(scene, W, H, kp=kp_of(**kw, **over), cam=cam)
        if fast: r.set_brick_volume(vol) if mode == "brick" else r.set_cell_volume(vol)
        scene.reset_blue_noise(); r.render(2); torch.cuda.synchronize()
        return r.buffers.accum.cpu().numpy(), r.buffers.depth.cpu().numpy()
    (a, da), (b, db), (d, _) = run(False, **P1), run(True, **P1), run(False)
    frac = flipped_fraction(b, a)
    print(f"P1 {mode} mode vs texture path: flipped {frac:.3g}, max |d| {np.abs(a - b).max():.3g}; P1 moves {100 * flipped_fraction(a, d):.2f} %")
    assert flipped_fraction(a, d) >= GUARD
    assert float(a.mean()) > 1e-3 and np.isfinite(b).all() and frac <= MAX_FLIPPED
    assert flipped_fraction(db[:, None], da[:, None]) <= MAX_FLIPPED


# ---- P2: the emission walk's step -------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("integrator,emission,tr_depth", [(0, 1.0, 0.5), (0, 1.0, 2.0), (1, 1.0, 0.5), (1, 1.0, 2.0),
                                                           (0, -0.5, 2.0), (1, -0.5, 0.5)])
def test_emission_walk_step(scenes, integrator, emission, tr_depth):
    """extinction.x in {0.37, 3} divides the emission walk's step (the direct integrator runs the walk for emission_scale > 0, the
    volumetric one for != 0); tr_depth multiplies it.  extinction.y and .z stay 1, so only the x channel can move the step."""
    f = Frame(scenes("S1"), 200, 120, 1)
    kw = dict(integrator=integrator, ray_depth=3 if integrator == 0 else 6, volume_depth=2, emission_scale=emission, emission_pivot=1.0,
              tr_depth=tr_depth)
    default = f.reference(full=False, **kw)
    for x in (0.37, 3.0):
        what = f"P2 S1 integrator {integrator} emission {emission} tr_depth {tr_depth} extinction.x {x}"
        want = f.reference(**kw, extinction=(x, 1.0, 1.0))
        assert_moves(want, default, what)
        assert_matches(f.library(**kw, extinction=(x, 1.0, 1.0)), want, what)


@needs_ref
@pytest.mark.parametrize("integrator", [0, 1])
def test_emission_walk_step_fireball(scenes, integrator):
    f = Frame(scenes("fireball"), 200, 120, 1)
    kw = dict(integrator=integrator, ray_depth=2 if integrator == 0 else 6, volume_depth=3, emission_scale=1.0, emission_pivot=1.0,
              tr_depth=2.0)
    want = f.reference(**kw, extinction=(0.37, 1.0, 1.0))
    assert_moves(want, f.reference(full=False, **kw), f"P2 fireball integrator {integrator}")
    assert_matches(f.library(**kw, extinction=(0.37, 1.0, 1.0)), want, f"P2 fireball integrator {integrator}")


# ---- P3: light colours ------------------------------------------------------------------------------------------------------------------
P3_CASES = {
    "hdri_compact": dict(scene="dragon", kp=dict(ray_depth=3, volume_depth=2), level_a=True),              # lean kernel, 16-byte records
    "hdri_wide":    dict(scene="dragon_lit", aperture=0.2, kp=dict(ray_depth=3, volume_depth=2), level_a=True),   # generic, sphere branch
    "bruneton":     dict(scene="dragon", kp=dict(environment_type=0, ray_depth=3, volume_depth=2), level_a=True),  # k_resolve<1>
    "vol_table":    dict(scene="dragon", kp=dict(integrator=1, environment_type=0, ray_depth=6)),                # k_resolve<2>, in-path sky
    "vol_hdri":     dict(scene="dragon_lit", kp=dict(integrator=1, ray_depth=6)),
}


@needs_ref
@needs_level_a
@pytest.mark.parametrize("name", list(P3_CASES))
def test_light_colours(scenes, name):
    cfg = P3_CASES[name]
    f = Frame(scenes(cfg["scene"]), 200, 120, 2, aperture=cfg.get("aperture", 0.0))
    try:
        want = f.reference(**cfg["kp"], **P3)
        assert_moves(want, f.reference(full=False, **cfg["kp"]), f"P3 {name}")
        assert_matches(f.library(**cfg["kp"], **P3), want, f"P3 {name}")
        if cfg.get("level_a"):
            assert_matches(f.level_a(**cfg["kp"], **P3), want, f"P3 {name} level A")
    finally:
        f.close()


# ---- P4: sun direction ------------------------------------------------------------------------------------------------------------------
SUN = [dict(azimuth=0.0), dict(azimuth=37.5), dict(azimuth=359.5), dict(elevation=0.0), dict(elevation=90.0), dict(elevation=-10.0)]
P4_PATHS = {"hdri": dict(ray_depth=3, volume_depth=2, phase_g1=0.6),     # forward scattering: the sun estimate follows the direction
            "bruneton": dict(environment_type=0, ray_depth=3, volume_depth=2),
            "vol_hdri": dict(integrator=1, ray_depth=6)}


@needs_ref
@pytest.mark.parametrize("path", list(P4_PATHS))
def test_sun_direction(scenes, path):
    """The sun's azimuth and elevation through the HDRI sun estimate (lean kernel), the Bruneton sky (this library's tables in both
    kernels) and the volumetric path integrator; each value against the default direction (azimuth 120, elevation 30)."""
    f = Frame(scenes("dragon"), 200, 120, 1)
    kw = P4_PATHS[path]
    default = f.reference(full=False, **kw)
    for sun in SUN:
        what = f"P4 {path} {sun}"
        want = f.reference(**kw, **sun)
        assert_moves(want, default, what)
        assert_matches(f.library(**kw, **sun), want, what)


@needs_ref
def test_sun_direction_clamps(scenes):
    """Azimuth is clamped to [0, 360] and elevation to [-90, 90] in both kernels: outside, each kernel's frame is bit for bit its frame
    at the bound, and the library's frame at the bound matches the reference's."""
    f = Frame(scenes("dragon"), 200, 120, 1)
    kw = dict(ray_depth=3, volume_depth=2)
    for out, bound in ((dict(azimuth=-30.0), dict(azimuth=0.0)), (dict(azimuth=400.0), dict(azimuth=360.0)),
                       (dict(elevation=95.0), dict(elevation=90.0)), (dict(elevation=-95.0), dict(elevation=-90.0))):
        ref_out, ref_bound = f.reference(full=False, **kw, **out), f.reference(**kw, **bound)
        mine_out, mine_bound = f.library(**kw, **out), f.library(**kw, **bound)
        for k in ("accum", "depth", "raw", "display", "cost", "bn"):
            assert np.array_equal(mine_out[k].view(np.uint32), mine_bound[k].view(np.uint32)), f"library {out} against {bound}: {k}"
        for k in ("accum", "depth", "display", "bn"):                # what a frame stored without cost and raw.xyz carries
            assert np.array_equal(ref_out[k].view(np.uint32), ref_bound[k].view(np.uint32)), f"reference {out} against {bound}: {k}"
        assert np.array_equal(ref_out["raw"][:, 3].view(np.uint32), ref_bound["raw"][:, 3].view(np.uint32)), f"reference {out}: raw.w"
        assert_matches(mine_bound, ref_bound, f"P4 clamp {bound}")


# ---- P5: phase --------------------------------------------------------------------------------------------------------------------------
G_VALUES = [0.00099, 0.001, -0.001, 0.95, 0.999, -0.999, 1.0, -1.0]


@needs_ref
@pytest.mark.parametrize("integrator", [0, 1])
def test_phase_g(scenes, integrator):
    """phase_g1 around the |g| < EPS branch of the sampler (0.00099 takes the isotropic branch, +-0.001 the HG inversion with its
    cancellation) and near +-1; the direct integrator through the lean and the generic kernel, the volumetric one (HG pdf in its MIS
    weights).  Guard: g = 0.00099 against g = 0.001 (across the branch), every other value against g = 0."""
    f = Frame(scenes("dragon"), 200, 120, 1)
    kw = dict(ray_depth=3, volume_depth=4) if integrator == 0 else dict(integrator=1, ray_depth=8)
    default = f.reference(full=False, **kw)
    want = {}
    for g in G_VALUES:
        want[g] = f.reference(**kw, phase_g1=g)
        variants = (("lean", {}), ("generic", {"generic_kernel": 1})) if integrator == 0 else (("wavefront", {}),)
        for label, opts in variants:
            assert_matches(f.library(opts, **kw, phase_g1=g), want[g], f"P5 integrator {integrator} g {g} {label}")
    for g in G_VALUES:
        if g == 0.00099:
            assert_moves(want[g], want[0.001], f"P5 integrator {integrator} g 0.00099 against 0.001")
        else:
            assert_moves(want[g], default, f"P5 integrator {integrator} g {g}")


# ---- P6: LUT index ----------------------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("name", ["S1", "fireball", "smoke"])
def test_emission_pivot(scenes, name):
    """emission_pivot scales the index of the density-colour LUT (every collision) and of the emission LUT (emissive volumes); 0 sends
    every index to the clamp."""
    f = Frame(scenes(name), 200, 120, 1)
    kw = dict(ray_depth=3, volume_depth=2, emission_scale=1.0)
    if name == "smoke": kw["density_mult"] = 4.0
    default = f.reference(full=False, **kw)
    for pivot in (0.25, 10.0, 0.0):
        want = f.reference(**kw, emission_pivot=pivot)
        assert_moves(want, default, f"P6 {name} emission_pivot {pivot}")
        assert_matches(f.library(**kw, emission_pivot=pivot), want, f"P6 {name} emission_pivot {pivot}")


# ---- P7: the guard fed by the parameters ------------------------------------------------------------------------------------------------
@needs_ref
@needs_level_a
def test_guard_through_parameters(scenes):
    """Iteration 0 from prefilled buffers.  extinction.y = 0 makes beta.y +Inf at a collision, and the guard replaces the sample with the
    previous accum; albedo 0 and energy_inject 0 make beta black at the first collision, where the path ends."""
    f = Frame(scenes("dragon"), 96, 64, 2, fill=lambda b: prefill(b, 31))
    kw = dict(ray_depth=3, volume_depth=2)
    default = f.reference(full=False, **kw)
    start = f._out(f._renderer(kw))
    frames = {}
    for name, over in (("extinction_y_0", dict(extinction=(1.0, 0.0, 1.0))), ("albedo_0", dict(albedo=(0.0, 0.0, 0.0))),
                       ("energy_0", dict(energy_inject=0.0))):
        want = frames[name] = f.reference(**kw, **over)
        assert_moves(want, default, f"P7 {name}")
        for label, opts in (("lean", {}), ("generic", {"generic_kernel": 1})):
            assert_matches(f.library(opts, **kw, **over), want, f"P7 {name} {label}")
        assert_matches(f.level_a(**kw, **over), want, f"P7 {name} level A")
    # the first pass at iteration 0 replaces the prefill unless the guard keeps it; with extinction.y = 0 every collision is non-finite
    kept = (frames["extinction_y_0"]["accum"] == start["accum"]).all(axis=1).mean()
    print(f"P7 extinction_y_0: {100 * kept:.1f} % of the pixels keep their prefill")
    assert kept > 1e-3
    assert np.array_equal(frames["albedo_0"]["accum"].view(np.int32), frames["energy_0"]["accum"].view(np.int32))


# ---- P8: fields the reference never reads -----------------------------------------------------------------------------------------------
UNREAD = dict(phase_g2=0.7, phase_f=0.25, min_extinction=3.5, transmittance=(0.2, 7.0, -1.0), debug=1)


@pytest.mark.parametrize("variant", ["lean", "generic", "vol", "level_a"])
def test_unread_fields_leave_the_frame_unchanged(scenes, variant):
    f = Frame(scenes("dragon_lit" if variant == "generic" else "dragon"), 200, 120, 2)
    kw = dict(integrator=1, ray_depth=6) if variant == "vol" else dict(ray_depth=3, volume_depth=2)
    if variant == "level_a":
        if not os.path.exists(LEVEL_A) or not oracle_ref.usable(): pytest.skip("level (A) needs its cubin and the reference loader")
        a, b = f.level_a(**kw), f.level_a(**kw, **UNREAD)
    else:
        a, b = f.library(**kw), f.library(**kw, **UNREAD)
    assert float(a["accum"].mean()) > 1e-3
    for k in ("accum", "depth", "raw", "display", "cost", "bn"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k


# ---- the committed fixture at non-default parameters --------------------------------------------------------------------------------------
def test_mixed_params_against_reference_golden(vols):
    """tests/golden/mixed_params.npz: the UNMODIFIED reference kernel on S1 at the P1 volume and P3 light parameters, azimuth 200,
    elevation 15, g = 0.9 (with the assets' white density-colour LUT, as the fixture was made)."""
    import json
    g = np.load(os.path.join(GOLD, "mixed_params.npz"))
    meta = json.loads(str(g["meta"]))
    assert meta["scene"] == "S1"
    scene = M.build_s1(vols)
    H, W = meta["H"], meta["W"]
    r = V.Renderer(scene, W, H, kp=kp_of(**meta["kp"]))
    assert bytes(r.cam) == g["camera"].tobytes(), "camera set-up drifted from the fixture"
    scene.reset_blue_noise(); r.render(meta["passes"]); torch.cuda.synchronize()
    got = dict(accum=r.buffers.accum.cpu().numpy(), depth=r.buffers.depth.cpu().numpy(), cost=np.zeros((H * W, 3), np.float32),
               raw=r.buffers.raw.cpu().numpy(), display=r.buffers.display.cpu().numpy().view(np.uint32),
               bn=scene.d_blue_noise.cpu().numpy(), iteration=int(r.kp.iteration))
    want = dict(accum=g["accum"].reshape(-1, 3), depth=g["depth"].reshape(-1), cost=np.zeros((H * W, 3), np.float32),
                raw=g["raw"].reshape(-1, 4), display=g["display"].reshape(-1).view(np.uint32), bn=g["blue_noise"], iteration=meta["passes"])
    assert_matches(got, want, "mixed_params golden")
    assert float(r.buffers.cost.abs().max()) == 0.0
