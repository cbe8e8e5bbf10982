"""Deterministic scenes of DIFFERENT volumes, for the tests that compare multi-volume rendering with the reference.

Three synthetic volumes are made from fixed NumPy formulas (no random state), each with its own grid size, index bounds and voxel
size, none equal to the dragon's:
  * haze  -- wide, smooth, low density (max 0.26; the dragon's is 1.0); no extra grids; a sheared base transform;
  * ember -- the densest volume (max 2.35), so the root majorant never comes from instance 0; a heat grid at its own, coarser
             resolution, which the kernels read with the DENSITY grid's coordinates (quirk Q8);
  * tint  -- a strongly red colour grid at its own resolution; negative densities at its corners, so min_density takes the
             FLT_EPSILON rule (quirk Q10).

A volume without a colour grid reads as WHITE in the leaf's colour maximum, so a colour only shows in leaves that list nothing but
coloured volumes.  S1 therefore has two tint instances that reach out of the other volumes' boxes: some leaves list both (the
maximum of two colours, each 0 outside its own box), some one.

Scenes:
  S1 overlap  -- the dragon, haze, ember and two tint instances, overlapping: some octree leaves list three or more distinct
                 volumes, others only the tints;
  S2 order    -- S1's instances in another order (the leaf sums follow leaf order);
  S3 instanced mix -- 40 instances drawn from the four volumes: node majorants differ across the octree;
  S4 staged assets -- the dragon, fireball.vdb and colored_smoke.vdb, when those assets are staged.

`volume_specs()` and `instance_specs()` need no GPU: tests/test_oracle_cpu.py builds the CPU port's scene from them.  Everything that
creates textures or an octree runs only when called."""
import contextlib
import ctypes as C

import numpy as np
import torch

import vpt_b200 as V
from vpt_b200.scene import instance_xform, load_vdb_grid, synthetic_env

LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]
SPHERE = dict(center=(4.0, 6.5, 3.0), radius=1.2, color=(0.8, 0.6, 0.3), roughness=0.7)      # above the volumes, in view
FLT_EPS = np.float32(np.finfo(np.float32).eps)


def _unit_coords(dx, dy, dz):
    """(z, y, x)-shaped voxel-centre coordinates in [0, 1] along each axis."""
    z, y, x = np.meshgrid(np.linspace(0, 1, dz, dtype=np.float32), np.linspace(0, 1, dy, dtype=np.float32),
                          np.linspace(0, 1, dx, dtype=np.float32), indexing="ij")
    return x, y, z


def _scale_xform(s, shear_xy=0.0):
    X = np.eye(4, dtype=np.float32)
    X[0][0] = X[1][1] = X[2][2] = np.float32(s)
    X[0][1] = np.float32(shear_xy)
    return X


def volume_specs():
    """name -> dict(density (z,y,x), emission (z,y,x) | None, color (z,y,x,3) | None, bbox_min, voxelsize, xform (base, 4x4))"""
    x, y, z = _unit_coords(48, 24, 20)
    haze = 0.3 * np.exp(-((x - 0.5) ** 2 / 0.08 + (y - 0.4) ** 2 / 0.12 + (z - 0.5) ** 2 / 0.1)) * (0.8 + 0.2 * np.cos(7.0 * x) * np.sin(5.0 * z + 1.0))
    x, y, z = _unit_coords(24, 24, 24)
    r = np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2) / 0.5
    ember = 2.5 * np.clip(1.0 - r, 0.0, None) ** 0.8
    hx, hy, hz = _unit_coords(12, 10, 14)                                             # heat grid: 12 x 10 x 14 against 24^3
    hr = np.sqrt((hx - 0.45) ** 2 + (hy - 0.55) ** 2 + (hz - 0.5) ** 2) / 0.5
    heat = 2.0 * np.clip(0.9 - hr, 0.0, None) + 0.1 * hx
    x, y, z = _unit_coords(30, 18, 22)
    tint = 1.7 * np.exp(-((x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2) / 0.15) - 0.2   # < 0 towards the corners
    cx, cy, cz = _unit_coords(10, 6, 8)                                               # colour grid: 10 x 6 x 8 against 30 x 18 x 22
    color = np.stack([0.9 + 0.1 * cx, 0.25 + 0.35 * cy, 0.04 + 0.12 * cz], axis=-1)
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {
        "haze": dict(density=f(haze), emission=None, color=None, bbox_min=(-4, 2, 3), voxelsize=0.2, xform=_scale_xform(0.2, shear_xy=0.03)),
        "ember": dict(density=f(ember), emission=f(heat), color=None, bbox_min=(2, -3, 5), voxelsize=0.15, xform=_scale_xform(0.15)),
        "tint": dict(density=f(tint), emission=None, color=f(color), bbox_min=(5, 7, -2), voxelsize=0.18, xform=_scale_xform(0.18)),
    }


def dragon_spec():
    dens, meta = load_vdb_grid(V.find_asset("dragon.vdb"), "density")
    return dict(density=dens, emission=None, color=None, bbox_min=meta["bbox_min"], bbox_max=meta["bbox_max"], voxelsize=meta["voxel_size"],
                xform=meta["xform"])


# (volume name, position, quaternion, scale): S1 overlaps all four around the dragon (world box ~ (1.6..8.5, 0.1..4.9, 3.5..6.5));
# the tints reach beyond x = 9.7 and below y = 0.1, where no uncoloured volume is
S1 = [("dragon", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0),
      ("haze", (1.3, -0.2, 2.5), (0.0, 0.0871557, 0.0, 0.9961947), 1.0),
      ("ember", (3.2, 1.4, 2.6), (0.0, 0.0, 0.0, 1.0), 1.1),
      ("tint", (7.0, -1.5, 4.0), (0.0, 0.0, 0.1305262, 0.9914449), 1.2),
      ("tint", (8.5, -2.5, 5.0), (0.0, 0.258819, 0.0, 0.9659258), 1.1)]
S2 = [S1[3], S1[2], S1[0], S1[4], S1[1]]


def s3_instances(n=40, seed=5):
    rng = np.random.RandomState(seed)
    names = ("dragon", "haze", "ember", "tint")
    out = []
    for i in range(n):
        q = rng.randn(4); q /= np.linalg.norm(q)
        out.append((names[i % 4], tuple(rng.uniform(-9.0, 9.0, 3)), tuple(q), float(rng.uniform(0.7, 1.3))))
    return out


def instance_specs(layout):
    """Host-side description of a layout's instances for the CPU port: the volume specs with the instance transform applied and the
    max / min density rule of Volume.from_dense."""
    specs = volume_specs(); specs["dragon"] = dragon_spec()
    out = []
    for name, pos, quat, scale in layout:
        s = dict(specs[name])
        d = s["density"]; dz, dy, dx = d.shape
        if "bbox_max" not in s:
            s["bbox_max"] = (s["bbox_min"][0] + dx - 1, s["bbox_min"][1] + dy - 1, s["bbox_min"][2] + dz - 1)
        s["max_density"] = float(max(np.float32(0.0), d.max()))
        s["min_density"] = float(np.maximum(FLT_EPS, d).min())
        s["xform"] = instance_xform(s["xform"], pos, quat, scale)
        out.append(s)
    return out


class Volumes:
    """The four volumes as GPU textures, made once per test module."""

    def __init__(self):
        self.vols = {"dragon": V.Volume.load_vdb(V.find_asset("dragon.vdb"))}
        for name, s in volume_specs().items():
            self.vols[name] = V.Volume.from_dense(s["density"], bbox_min=s["bbox_min"], xform=s["xform"], voxelsize=s["voxelsize"],
                                                  emission=s["emission"], color=s["color"])
        assert self.vols["ember"].rec.vdb_info.max_density > max(v.rec.vdb_info.max_density for k, v in self.vols.items() if k != "ember")
        t = self.vols["tint"].rec.vdb_info
        assert float(volume_specs()["tint"]["density"].min()) < 0 and t.min_density == float(FLT_EPS)

    def __getitem__(self, name):
        return self.vols[name]


def place_sphere(scene):
    sp = scene.h_sphere; sp.center = V.f3(*SPHERE["center"]); sp.radius = SPHERE["radius"]
    sp.color = V.f3(*SPHERE["color"]); sp.roughness = SPHERE["roughness"]
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))


@contextlib.contextmanager
def colour_grids_off(scene):
    """While the block runs, the device instance records of `scene` have has_color cleared: every volume then reads as WHITE, as
    one without a colour grid does.  The textures, the octree and the host records stay as they are.  Frames rendered inside the
    block must start at iteration 0, where the library re-reads the instance records."""
    n = len(scene.instances)
    grey = (V.GPU_VDB * n)()
    C.memmove(grey, scene.h_volumes, C.sizeof(grey))
    for g in grey: g.vdb_info.has_color = 0
    scene.d_volumes[:C.sizeof(grey)].copy_(torch.frombuffer(bytearray(bytes(grey)), dtype=torch.uint8))
    try:
        yield
    finally:
        scene.d_volumes[:C.sizeof(grey)].copy_(torch.frombuffer(bytearray(bytes(scene.h_volumes)), dtype=torch.uint8))
        torch.cuda.synchronize()


def read_tree(root):
    """{node number: OCTNode} of a reference-layout octree (this library's or the reference builder's)."""
    nodes = (V.OCTNode * 585)(); ex = (C.c_int * 585)()
    V._native.check(V.lib.vpt_octree_read(root, nodes, ex), None, "vpt_octree_read")
    return {j: nodes[j] for j in range(585) if ex[j]}


def max_distinct_per_leaf(scene):
    """The largest number of distinct VOLUMES (not instances) that one octree leaf lists."""
    return max(len({scene.volume_names[i] for i in lst}) for lst in scene.leaf_lists())


def build(vols, layout, lights=True, sphere=True):
    """A Scene of `layout` [(volume name, pos, quat, scale), ...] over the procedural HDRI of the golden fixtures."""
    inst = [vols[name].instance(pos=pos, quat=quat, scale=scale) for name, pos, quat, scale in layout]
    scene = V.Scene(inst, env=synthetic_env(512, 256), lights=LIGHTS if lights else None, keep=[vols])
    scene.volume_names = [name for name, *_ in layout]
    if sphere: place_sphere(scene)
    return scene


def build_s1(vols, order=S1, **kw):
    scene = build(vols, order, **kw)
    root = read_tree(scene.d_oct_root)[0]
    assert max_distinct_per_leaf(scene) >= 3, "S1 must have leaves that list three or more distinct volumes"
    assert root.max_extinction != scene.h_volumes[0].vdb_info.max_density, "the root majorant must not come from instance 0"
    assert root.max_extinction == vols["ember"].rec.vdb_info.max_density
    tinted_only = [lst for lst in scene.leaf_lists() if lst and all(scene.volume_names[i] == "tint" for i in lst)]
    assert any(len(lst) == 2 for lst in tinted_only) and any(len(lst) == 1 for lst in tinted_only), \
        "S1 must have leaves that list only the two tints, and only one of them"
    return scene


def build_s2(vols, **kw):
    return build_s1(vols, order=S2, **kw)


def build_s3(vols, **kw):
    scene = build(vols, s3_instances(), **kw)
    tree = read_tree(scene.d_oct_root)
    below = [j for j, nd in tree.items() if j and nd.num_volumes and nd.max_extinction < tree[0].max_extinction]
    assert len(below) >= 8, f"only {len(below)} octree nodes have a majorant below the root's"
    assert len(set(scene.volume_names)) == 4
    return scene


def build_s4(vols, **kw):
    """The dragon with the staged fireball.vdb (emission, sigma_max 12.47, heat grid at its own resolution) and colored_smoke.vdb
    (colour grid) overlapping it.  The fireball is instanced at half size and the smoke reaches beyond both other boxes, so some
    leaves list the smoke alone and its colour shows.
    None when those assets are not staged."""
    paths = [V.find_asset(n) for n in ("fireball.vdb", "colored_smoke.vdb")]
    if not all(paths):
        return None
    staged = {"dragon": vols["dragon"], "fireball": V.Volume.load_vdb(paths[0]), "smoke": V.Volume.load_vdb(paths[1])}
    assert staged["fireball"].rec.vdb_info.has_emission and staged["smoke"].rec.vdb_info.has_color
    layout = [("dragon", (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0),
              ("fireball", (0.0, -0.5, 1.5), (0.0, 0.0, 0.0, 1.0), 0.5),
              ("smoke", (6.0, 0.0, 3.0), (0.0, 0.0, 0.0, 1.0), 1.0)]
    scene = build(staged, layout, **kw)
    assert max_distinct_per_leaf(scene) == 3 and [2] in scene.leaf_lists()
    return scene
