"""Option "empty_ahead" (on by default): a walk that reaches an empty octree node from which no populated leaf lies in its direction of
travel ends there instead of hopping to the root box's exit (build_empty_ahead, vpt_walk.cuh; DESIGN.md section 8j).  The frame must be
bit for bit the one the hops give: accum, depth, cost, raw, display and the blue noise, with the option on and off, over every trace
kernel and k_generate form -- the headline frame (lean kernel, k_generate's pre-step), the Bruneton sky (lean), camera motion (lean, no
pre-step), and frames whose trace kernel hops as before while the pre-step takes the shortcut: the sphere in view under a thin lens
(generic kernel, no pre-step), 120 instances, the fireball's emission walk under both integrators, the volumetric path integrator and
brick mode.  The hop counters must fall with the option on wherever the shortcut applies."""
import numpy as np
import pytest
import torch

import vpt_b200 as V
from test_light_groups_gpu import make_group_case
from test_motion_gpu import translated

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
PASSES = 8                     # passes_per_chunk 5: chunks of 5 + 3


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
    density = (np.clip(1.1 - r, 0.0, None) ** 1.5).astype(np.float32)
    heat = (3.0 * np.clip(0.8 - r, 0.0, None)).astype(np.float32)
    return V.Volume.from_dense(density, bbox_min=(-c, -c, -c), emission=heat)


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def render(case, on, motion=False):
    scene = case["scene"]
    r = case["mk0"]()
    r.set_option("passes_per_chunk", 5)
    r.set_option("empty_ahead", on)
    r.set_option("count_stats", 1)
    if motion: r.set_camera_motion(translated(r.cam, (0.6, -0.3, 0.4)))
    r.counters(reset=True)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(PASSES)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    out["blue_noise"] = scene.d_blue_noise.clone()
    hops = r.hop_counters()
    r.close()
    return out, hops


LEAN = ("headline", "sky", "motion")       # cases traced by a lean k_trace, which ends walks at "empty ahead"
NAMES = ["headline", "sky", "lights_sphere", "instanced", "brick", "emissive", "vol_emissive", "vol_sky_table", "motion"]


@pytest.mark.parametrize("name", NAMES)
def test_same_frame_and_fewer_hops(dragon, perlin, emissive, name):
    case = make_group_case("headline" if name == "motion" else name, dragon, perlin, emissive)
    on, h_on = render(case, 1, motion=name == "motion")
    off, h_off = render(case, 0, motion=name == "motion")
    for k in on:
        assert torch.equal(bits(on[k]), bits(off[k])), f"{k} differs with empty_ahead on"
    assert float(on["accum"].mean()) > 1e-4
    print(f"\n{name}: off {h_off}\n{name}: on  {h_on}")
    assert h_off["walks_ended_ahead"] == 0 and h_off["prestep_ended_ahead"] == 0
    walk_hops = lambda h: h["hops_delta"] + h["hops_ratio"] + h["hops_emission"]
    total = lambda h: walk_hops(h) + h["prestep_hops"]
    assert h_on["prestep_rays"] == h_off["prestep_rays"]
    if name in ("brick", "emissive", "vol_emissive"):
        # these grids fill their root box: no walk reaches an empty node (k_trace_brick would keep hopping anyway)
        assert total(h_off) == 0 and total(h_on) == 0
        return
    if name in LEAN:
        assert h_on["walks_ended_ahead"] > 0 and walk_hops(h_on) < walk_hops(h_off)
    else:                                                        # the generic kernels keep hopping; only k_generate's pre-step shortens
        assert h_on["walks_ended_ahead"] == 0 and walk_hops(h_on) == walk_hops(h_off)
    if name in LEAN or h_off["prestep_rays"]:
        assert total(h_on) < total(h_off)
