"""The 29-word parked record of the lean k_trace at 2 rays per lane (DESIGN.md section 4).  The record drops wdir, the point-light word
and T_c, shares a word between trv and the cached closest-object distance, and keeps the Philox key, without changing a bit of any path: every ray runs the
same arithmetic and draws as in the 3-ray lean kernel (option "trace_slots" 3), which keeps the full 34-word record in 16-byte groups.
So every output buffer must be bit for bit the same, and so must the look-up, step, ray and service totals of `count_stats`.

Frames: the headline scene; the sphere in view under a thin lens (the sphere normal, `sphere_bounced` and the queue slot of a lens ray);
a low sun (long transmittance walks); ray_depth and volume_depth at the ends of the 16 bits the record keeps for them; each rank of a
2-rank partition (the pixel word); a render region; and the instance mattes and compositing AOVs (the matte kernel)."""
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
LAYERS = ("alpha", "volume", "mattes")
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


def sphere_scene(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    sp = scene.h_sphere; sp.center = V.f3(4.0, 6.5, 3.0); sp.radius = 1.2; sp.roughness = 0.7; sp.color = V.f3(0.8, 0.6, 0.3)
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    return scene


def sphere_lens(dragon):
    scene = sphere_scene(dragon)
    cam = scene.frame_camera(320, 200, aperture=0.15)
    return scene, lambda: V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=3, volume_depth=2), cam=cam), 16


def sphere_pinhole(dragon):
    scene = sphere_scene(dragon)
    cam = scene.frame_camera(320, 200)
    return scene, lambda: V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=6, volume_depth=3), cam=cam), 16


def low_sun(dragon):
    scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
    cam = scene.frame_camera(480, 270)
    return scene, lambda: V.Renderer(scene, 480, 270, kp=make_kp(ray_depth=8, volume_depth=2, elevation=2.0, azimuth=75.0), cam=cam), 16


def deep_max(dragon):
    scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
    cam = scene.frame_camera(160, 90)
    return scene, lambda: V.Renderer(scene, 160, 90, kp=make_kp(ray_depth=65535, volume_depth=65535), cam=cam), 4


def deep_over(dragon):
    scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
    cam = scene.frame_camera(160, 90)
    return scene, lambda: V.Renderer(scene, 160, 90, kp=make_kp(ray_depth=65536, volume_depth=65536), cam=cam), 4


def sharded(rank):
    def case(dragon):
        scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
        cam = scene.frame_camera(480, 270)
        return scene, lambda: V.Renderer(scene, 480, 270, kp=make_kp(ray_depth=20), cam=cam, rank=rank, n_ranks=2, stripe_rows=8), 16
    case.__name__ = f"rank{rank}_of_2"
    return case


def region(dragon):
    scene = V.Scene([dragon.instance()], env="Barce_Rooftop_C_3k.hdr")
    cam = scene.frame_camera(480, 270)

    def mk():
        r = V.Renderer(scene, 480, 270, kp=make_kp(ray_depth=20), cam=cam)
        r.set_region(100, 40, 390, 211)
        return r
    return scene, mk, 16


def mattes_aovs(dragon):
    scene = sphere_scene(dragon)
    cam = scene.frame_camera(320, 200)

    def mk():
        r = V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=6, volume_depth=2), cam=cam)
        r.enable_aovs()
        r.enable_mattes([[0]], sphere=0)
        return r
    return scene, mk, 16


CASES = [headline, sphere_lens, sphere_pinhole, low_sun, deep_max, deep_over, sharded(0), sharded(1), region, mattes_aovs]


def render(scene, mk, passes, slots):
    r = mk()
    r.set_option("trace_slots", slots)
    r.set_option("count_stats", 1)
    r.counters(reset=True)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    out.update({k: getattr(r.buffers, k).clone() for k in LAYERS if getattr(r.buffers, k, None) is not None})
    hops = r.hop_counters(reset=False)
    counts = r.counters()
    r.close()
    return out, counts, hops


@pytest.mark.parametrize("case", CASES, ids=[c.__name__ for c in CASES])
def test_lean_record_gives_the_frame_of_the_full_record(dragon, case):
    scene, mk, passes = case(dragon)
    lean2, c2, h2 = render(scene, mk, passes, 2)
    full3, c3, h3 = render(scene, mk, passes, 3)
    assert lean2.keys() == full3.keys()
    for k in full3:
        assert torch.equal(bits(lean2[k]), bits(full3[k])), f"{k} differs between the 29-word and the 34-word record"
    assert float(full3["accum"].float().abs().sum()) > 0.0
    print(f"\n{case.__name__}: 34 words {c3} {h3}\n29 words {c2} {h2}")
    for k in SAME_COUNTS:
        assert c2[k] == c3[k], k
    assert h2 == h3
    # the kernel at 2 rays per lane, then the one at 3 (the warp totals cannot tell: they vary with the scheduling from run to run)
    assert (c2["rays_per_lane"], c3["rays_per_lane"]) == (2, 3)
