"""Rays per lane of the lean k_trace (DESIGN.md section 4): a lean frame runs the kernel at 2 rays per lane (5 CTAs per SM: more warps to
hide the latency of its look-ups) by default, and the one at 3 rays per lane (16-byte parked records, 4 CTAs per SM) with option
"trace_slots" 3.  Each ray runs the same arithmetic and draws either way, so every output buffer must be bit for bit the same, and so must
the work counters other than the warp iterations and service rounds: the headline frame (BASELINE config 2 at full size) and a frame with
the sphere in view under a thin lens."""
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
SAME_COUNTS = ("lookups", "lane_steps", "rays", "lane_services")


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def headline(dragon):
    scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
    cam = scene.frame_camera(1920, 1080)
    return scene, lambda: V.Renderer(scene, 1920, 1080, kp=make_kp(ray_depth=100), cam=cam), 64


def sphere_lens(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    sp = scene.h_sphere; sp.center = V.f3(4.0, 6.5, 3.0); sp.radius = 1.2; sp.roughness = 0.7; sp.color = V.f3(0.8, 0.6, 0.3)
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    cam = scene.frame_camera(320, 200, aperture=0.15)
    return scene, lambda: V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=3, volume_depth=2), cam=cam), 16


def render(scene, mk, passes, slots):
    r = mk()
    r.set_option("trace_slots", slots)
    r.set_option("count_stats", 1)
    r.counters(reset=True)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    out["blue_noise"] = scene.d_blue_noise.clone()
    hops = r.hop_counters(reset=False)
    counts = r.counters()
    r.close()
    return out, counts, hops


@pytest.mark.parametrize("case", [headline, sphere_lens], ids=["headline", "sphere_lens"])
def test_two_and_three_rays_per_lane_give_the_same_frame(dragon, case):
    scene, mk, passes = case(dragon)
    two, c2, h2 = render(scene, mk, passes, 0)
    three, c3, h3 = render(scene, mk, passes, 3)
    for k in three:
        assert torch.equal(bits(two[k]), bits(three[k])), f"{k} differs between 2 and 3 rays per lane"
    assert float(three["accum"].mean()) > 1e-4
    print(f"\n3 rays per lane {c3} {h3}\n2 rays per lane (default) {c2} {h2}")
    for k in SAME_COUNTS:
        assert c2[k] == c3[k], k
    assert h2 == h3
    assert c2["warp_step_iters"] != c3["warp_step_iters"]           # a different kernel ran
    assert (c2["rays_per_lane"], c3["rays_per_lane"]) == (2, 3)
