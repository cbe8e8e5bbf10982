"""HDRI frames with compact sample records: a lean trace kernel finishes a hit sample's environment term itself and k_resolve<0>
reads one 16-byte record per sample; the generic kernel keeps wide records.  The frames must be the very bits the wide-record layout
produced, so they are compared with tests/golden/hdri_records.npz (written by tests/golden/make_hdri_records.py with a build that used
wide records everywhere) on every trace path: the lean kernel, the brick pool and the cell table (compact), and the generic kernel (wide).
"""
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hdri_records.npz")
OUTPUTS = ("accum", "depth", "raw", "display")

# name -> (volume, width, height, renderer options, trace mode, fixture).  8 passes in chunks of 5 + 3: tr of the last pass of a chunk
# shorter than the fused maximum reaches raw.w.  The generic kernel renders the lean kernel's frame (test_parity_gpu.py).
CASES = {
    "lean": ("dragon", 128, 72, {"passes_per_chunk": 5}, None, "lean"),
    "generic": ("dragon", 128, 72, {"passes_per_chunk": 5, "generic_kernel": 1}, None, "lean"),
    "brick": ("perlin", 64, 36, {"passes_per_chunk": 5}, "brick", "brick"),
    "cells": ("perlin", 64, 36, {"passes_per_chunk": 5}, "cells", "cells"),
}
PASSES = 8


def load_volume(kind):
    if kind == "dragon":
        return V.Volume.load_vdb(V.find_asset("dragon.vdb"))
    return V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)


def render_case(name, volumes):
    """The frame of case `name` after PASSES passes: {output: array}.  volumes caches one Volume per kind."""
    kind, W, H, options, mode, _ = CASES[name]
    if kind not in volumes: volumes[kind] = load_volume(kind)
    vol = volumes[kind]
    scene = V.Scene([vol.instance()], env=synthetic_env(512, 256), keep=[vol])
    kp = V.default_kernel_params(); kp.environment_type = 1; kp.max_interactions = 1000; kp.ray_depth = 100
    r = V.Renderer(scene, W, H, kp=kp, options=options)
    if mode == "brick": r.set_brick_volume(vol)
    elif mode == "cells": r.set_cell_volume(vol)
    scene.reset_blue_noise()
    r.render(PASSES); torch.cuda.synchronize()
    return {k: getattr(r.buffers, k).cpu().numpy() for k in OUTPUTS}


@pytest.fixture(scope="module")
def volumes():
    return {}


@pytest.mark.parametrize("name", list(CASES))
def test_hdri_frame_is_bitwise_the_wide_record_frame(name, volumes):
    g = np.load(GOLDEN)
    got = render_case(name, volumes)
    for out in OUTPUTS:
        want = g[CASES[name][5] + "_" + out]
        assert got[out].shape == want.shape, out
        diff = int((got[out].view(np.uint32) != want.view(np.uint32)).sum())
        assert diff == 0, f"{name}: {out} differs from the fixture in {diff} words"
    assert float(got["accum"].mean()) > 1e-3 and (got["raw"].reshape(-1, 4)[:, 3] > 0).any(), "the frame must hold light and some tr"


def test_switching_between_sky_and_hdri_records(volumes):
    """One context renders a precomputed-sky frame (wide records), an HDRI frame (compact records) and the sky again: each frame
    equals the one a fresh context renders."""
    if "dragon" not in volumes: volumes["dragon"] = load_volume("dragon")
    vol = volumes["dragon"]
    scene = V.Scene([vol.instance()], env=synthetic_env(512, 256), keep=[vol])
    V.Atmosphere().apply(scene.atmos)
    W, H = 256, 144

    def kp_of(env):
        kp = V.default_kernel_params(); kp.environment_type = env; kp.max_interactions = 1000; kp.ray_depth = 20
        return kp

    def frame(r):
        scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
        r.render(4); torch.cuda.synchronize()
        return {k: getattr(r.buffers, k).clone() for k in OUTPUTS}

    sky = frame(V.Renderer(scene, W, H, kp=kp_of(0)))
    hdri = frame(V.Renderer(scene, W, H, kp=kp_of(1)))
    r = V.Renderer(scene, W, H, kp=kp_of(0))
    for env, want in ((0, sky), (1, hdri), (0, sky)):
        r.kp.environment_type = env
        got = frame(r)
        for k in OUTPUTS:
            assert torch.equal(got[k], want[k]), f"environment_type {env}: {k}"
