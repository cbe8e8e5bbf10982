#!/usr/bin/env python3
"""Generates the frame fixtures tests/golden/dragon_*.npz by running THE REFERENCE'S OWN KERNEL (oracle/_ref, compiled from
the reference's source/render_kernel.cu for sm_90a) on an H100:  `python tests/golden/make_golden.py OUT_DIR` writes
OUT_DIR/*.npz, which are then committed under tests/golden/.

Protocol: the UNMODIFIED reference kernel, launched exactly as main.cpp:1823-1829 does.  The frames are 256 pixels wide and at
most 256 high, the one shape at which the kernel's blue-noise read / update is race-free (every thread touches only its own
entry, SURVEY 8(c)(i)); octree built by the reference builder; environment = the deterministic procedural map
`synthetic_env(512, 256)` so that the fixtures need no 13 MB HDRI.

mixed_direct renders scene S1 of tests/mixed_scenes.py (the dragon and three synthetic volumes: a heat grid at its own resolution,
a colour grid, different majorants) with emission, point lights and the sphere.  mixed_params renders the same scene at volume, light and
phase parameters away from their identity defaults (albedo, extinction, energy_inject, sun and sky colours, sun direction, g), so the
CPU suite covers them too.  `make_golden.py OUT_DIR NAME ...` writes only the named fixtures.
"""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import vpt_b200 as V
from vpt_b200.scene import synthetic_env
from oracle_ref import RefOracle

CASES = {
    "dragon_single": dict(W=256, H=128, passes=2, kp=dict(ray_depth=2, volume_depth=1), lights=None),
    "dragon_multi":  dict(W=256, H=128, passes=2, kp=dict(ray_depth=3, volume_depth=3, phase_g1=0.6, density_mult=2.0, tr_depth=1.5),
                          lights=[((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]),
    "mixed_direct":  dict(W=256, H=128, passes=2, kp=dict(ray_depth=3, volume_depth=2, emission_scale=1.0, emission_pivot=1.0),
                          lights=[((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)], scene="S1"),   # = mixed_scenes.LIGHTS
    "mixed_params":  dict(W=256, H=128, passes=2, kp=dict(ray_depth=3, volume_depth=2, emission_scale=1.0, emission_pivot=1.0,
                                                          albedo=[0.9, 0.55, 0.3], extinction=[0.8, 1.25, 2.0], energy_inject=1.01234,
                                                          sun_color=[1.0, 0.55, 0.2], sun_mult=2.5, sky_color=[0.3, 0.6, 1.2], sky_mult=0.7,
                                                          azimuth=200.0, elevation=15.0, phase_g1=0.9),
                          lights=[((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)], scene="S1"),
}


def set_params(kp, over):
    """Kernel_params fields from a fixture's meta; a list is a float3."""
    for k, v in over.items(): setattr(kp, k, V.f3(*v) if isinstance(v, (list, tuple)) else v)
    return kp


def build(case):
    if case.get("scene") == "S1":
        import mixed_scenes
        scene = mixed_scenes.build_s1(mixed_scenes.Volumes())              # its own point lights and sphere
        kp = V.default_kernel_params(); kp.environment_type = 1; kp.max_interactions = 1000
        return scene, set_params(kp, case["kp"])
    vol = V.Volume.load_vdb(V.find_asset("dragon.vdb"))
    scene = V.Scene([vol.instance()], env=synthetic_env(512, 256), lights=case["lights"])
    kp = V.default_kernel_params(); kp.environment_type = 1; kp.max_interactions = 1000
    return scene, set_params(kp, case["kp"])

def main():
    if len(sys.argv) < 2: raise SystemExit("usage: make_golden.py OUT_DIR [NAME ...]")
    out = sys.argv[1]; os.makedirs(out, exist_ok=True)
    orc = RefOracle()
    for name in sys.argv[2:] or CASES:
        case = CASES[name]
        scene, kp = build(case)
        r = V.Renderer(scene, case["W"], case["H"], kp=kp)
        r.params.p_oct.value = orc.build_octree(scene.h_volumes, len(scene.instances))      # reference-built octree
        scene.reset_blue_noise()
        assert case["W"] == 256 and case["H"] <= 256, "the unmodified kernel is race-free only at this shape"
        orc.render(r, case["passes"], race_free=False)
        np.savez_compressed(os.path.join(out, name + ".npz"),
                            accum=r.buffers.accum.cpu().numpy().reshape(case["H"], case["W"], 3),
                            depth=r.buffers.depth.cpu().numpy().reshape(case["H"], case["W"]),
                            raw=r.buffers.raw.cpu().numpy().reshape(case["H"], case["W"], 4),
                            display=r.buffers.display.cpu().numpy().reshape(case["H"], case["W"]),
                            blue_noise=scene.d_blue_noise.cpu().numpy(),
                            camera=np.frombuffer(bytes(r.cam), dtype=np.uint8),
                            meta=json.dumps(dict(case=name, W=case["W"], H=case["H"], passes=case["passes"], kp=case["kp"], lights=case["lights"], scene=case.get("scene"),
                                                 generator="UNMODIFIED reference volume_rt_kernel (sm_90a rebuild, H100), its own launch protocol, race-free frame shape")))
        print("wrote", name, "mean", float(r.buffers.accum.mean()))

if __name__ == "__main__":
    main()
