"""Pixels culled by k_miss_cull (option "miss_cull", on by default) give the very same frame as with the cull off: k_generate writes no
record for them and k_resolve rebuilds their pinhole miss samples, so accum, depth, cost, raw, display, the blue noise, the AOVs and the
light groups must match bit for bit.  Cases: the headline frame at full size with compact and with wide records (AOVs and light groups
on), an adaptive frame, and a frame of three shards over the peer-memory exchange on one GPU; frames that cull nothing are unchanged by
the option: the Bruneton sky (k_resolve<1>) and the volumetric path integrator (k_resolve<2>), which keep every record, and a thin lens.
Every fixed-count frame has a chunk boundary inside the call."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from test_adaptive_gpu import make_case
from test_aov_gpu import make_aov_case
from test_adaptive_sharded_gpu import Case, Shards
from miss_cull_ref import camera_dict, cull_mask

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


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def outputs(scene, r):
    out = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    for k in ("alpha", "volume"):
        if getattr(r.buffers, k, None) is not None: out[k] = getattr(r.buffers, k).clone()
    if getattr(r.buffers, "groups", None) is not None:
        out.update({"group_" + g: t.clone() for g, t in r.buffers.groups.items()})
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def fixed_frame(scene, mk, cull, aovs=False, groups=False, passes=PASSES):
    r = mk()
    r.set_option("passes_per_chunk", 5)
    r.set_option("miss_cull", cull)
    if aovs: r.enable_aovs()
    if groups: r.enable_light_groups()
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    r.render(passes)
    torch.cuda.synchronize()
    out = outputs(scene, r)
    r.close()
    return out


def assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(bits(a[k]), bits(b[k])), f"{k} differs with the miss cull on"


@pytest.mark.parametrize("records", ["compact", "wide_aov_groups"])
def test_headline_full_size(dragon, perlin, records):
    scene, mk0, keep = make_case("headline", dragon, perlin)
    wide = records != "compact"
    on = fixed_frame(scene, mk0, 1, aovs=wide, groups=wide)
    off = fixed_frame(scene, mk0, 0, aovs=wide, groups=wide)
    assert_same(on, off)
    assert float(on["accum"].mean()) > 1e-4


@pytest.mark.parametrize("name", ["sky", "vol_sky_table", "lights_sphere"])
def test_sky_integrator_and_thin_lens(dragon, perlin, name):
    scene, mk, keep = make_aov_case(name, dragon, perlin)
    mk0 = lambda: mk(aovs=False)
    for aovs in (False, True):                                 # every k_resolve instantiation of the case
        for groups in (False, True):
            assert_same(fixed_frame(scene, mk0, 1, aovs=aovs, groups=groups), fixed_frame(scene, mk0, 0, aovs=aovs, groups=groups))


def test_shard_frame_culls_pixels(dragon):
    """The sharded frame below exercises the cull: the restatement culls a good share of its pixels."""
    case = Case(dragon)
    b6 = (C.c_float * 6)()
    V.lib.vpt_volume_bounds(C.byref(case.inst[0]), b6)
    b6 = np.array(list(b6), dtype=np.float32)
    m = cull_mask(camera_dict(case.cam), case.w, case.h, b6[:3] - np.float32(1), b6[3:] + np.float32(1), (0, 1000, 0), 1.0)   # vpt_octree_build's +-1
    assert 0.2 < m.mean() < 0.95


def test_adaptive_frame(dragon, perlin):
    scene, mk0, keep = make_case("headline", dragon, perlin)
    res = {}
    for cull in (1, 0):
        r = mk0()
        r.set_option("miss_cull", cull)
        r.enable_aovs(); r.enable_light_groups()
        scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
        run, counts, err = r.render_adaptive(32, threshold=0.3, min_passes=8, check_interval=8, error_map=True)
        torch.cuda.synchronize()
        res[cull] = (run, counts.clone(), err.clone(), outputs(scene, r))
        r.close()
    assert res[1][0] == res[0][0]
    assert torch.equal(bits(res[1][1]), bits(res[0][1])) and torch.equal(bits(res[1][2]), bits(res[0][2]))
    assert_same(res[1][3], res[0][3])


def test_three_shards_peer_exchange(dragon):
    case = Case(dragon)
    got = {}
    for cull in (1, 0):
        sh = Shards(case, 3, 8)
        try:
            for r in sh.rs:
                r.set_option("miss_cull", cull); r.set_option("passes_per_chunk", 5)
            sh.reset_blue_noise()
            for r in sh.rs: r.buffers.zero_()
            sh.fixed(PASSES)
            got[cull] = ([{k: getattr(r.buffers, k).clone() for k in BUFFERS} for r in sh.rs],
                         [{k: v.clone() for k, v in f.items()} for f in sh.frames], [s.d_blue_noise.clone() for s in sh.scenes])
            assert sh.abandoned_waits() == [0, 0, 0]
        finally:
            sh.close()
    for k in range(3):
        for name in BUFFERS:
            assert torch.equal(bits(got[1][0][k][name]), bits(got[0][0][k][name])), f"{name} of shard {k}"
        for name in ("accum", "display"):
            assert torch.equal(bits(got[1][1][k][name]), bits(got[0][1][k][name])), f"full-frame {name} held by shard {k}"
        assert torch.equal(got[1][2][k], got[0][2][k])
