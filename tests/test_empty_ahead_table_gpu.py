"""The "empty ahead" table a render call builds once (k_empty_ahead) and k_generate / the lean k_trace stage with the octree, read back
with vpt_debug_empty_ahead and checked byte for byte against the CPU construction of test_empty_ahead_cpu.py over the scene's own node
tables: the dragon, eight dragons scattered and rotated (split planes that are not one even grid), and option "empty_ahead" 0 (all zero)."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from test_empty_ahead_cpu import planes_consistent, table_sweeps

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


def node_tables(root):
    """The internal nodes 0..72 of a reference-layout octree in test_empty_ahead_cpu's form, as k_prepare_scene flattens them: child c
    of node j is node 8 j + 1 + c; a non-empty node splits at its child 0's (pmax.x, pmin.y, pmax.z)."""
    nodes = (V.OCTNode * 585)(); ex = (C.c_int * 585)()
    V._native.check(V.lib.vpt_octree_read(root, nodes, ex), None, "vpt_octree_read")
    pmin = np.zeros((73, 3), np.float32); half = np.zeros((73, 3), np.float32); pmax = np.zeros((73, 3), np.float32)
    ce = np.full(73, 0xff, np.uint32)
    for j in range(73):
        if not ex[j] or nodes[j].num_volumes == 0: continue
        b, c0 = nodes[j].bbox, nodes[8 * j + 1].bbox
        pmin[j] = (b.pmin.x, b.pmin.y, b.pmin.z); pmax[j] = (b.pmax.x, b.pmax.y, b.pmax.z)
        half[j] = (c0.pmax.x, c0.pmin.y, c0.pmax.z)
        ce[j] = sum(1 << c for c in range(8) if nodes[8 * j + 1 + c].num_volumes == 0)
    return dict(pmin=pmin, half=half, pmax=pmax, ce=ce, root_min=pmin[0], root_max=pmax[0])


def expected_bytes(t, on):
    tab = table_sweeps(t) if on else np.zeros((584, 8), bool)
    return bytes((tab.astype(np.uint32) << np.arange(8, dtype=np.uint32)).sum(axis=1).astype(np.uint8)) + bytes(8)


def scattered(dragon):
    rng = np.random.RandomState(7)
    inst = []
    for _ in range(8):
        q = rng.randn(4); q /= np.linalg.norm(q)
        inst.append(dragon.instance(pos=tuple(rng.uniform(-6, 6, 3)), quat=tuple(q), scale=float(rng.uniform(0.6, 1.4))))
    return inst


@pytest.mark.parametrize("name, on", [("dragon", 1), ("scattered", 1), ("dragon", 0)])
def test_table_matches_cpu_construction(dragon, name, on):
    scene = V.Scene([dragon.instance()] if name == "dragon" else scattered(dragon), env="Barce_Rooftop_C_3k.hdr")
    t = node_tables(scene.d_oct_root)
    r = V.Renderer(scene, 64, 32)
    r.set_option("empty_ahead", on)
    r.render(1)
    torch.cuda.synchronize()
    got = r.empty_ahead_table()
    want = expected_bytes(t, on)
    print(f"\n{name} empty_ahead={on}: planes consistent {planes_consistent(t)}, {sum(bin(b).count('1') for b in want)} bits set")
    assert len(got) == 592 and got == want
    if on and name == "dragon": assert any(want), "the dragon's table has entries with nothing ahead"
    r.close()
