"""Frames for testing the run-time Bruneton sky look-up (vpt_atmosphere.cuh: sample_atmosphere and the Sky<kInPath> methods) by itself.

Each GEOMETRY is a pinhole camera (vpt_camera_look_at: position, view direction, up, vertical fov, size) with two or three suns, and
names the branches of the look-up its frame is meant to reach.  Every frame here is miss-only: the single volume instance and the
reference sphere sit behind the camera plane, so every pixel is sample_atmosphere(camera origin, jittered direction) through the
resolve tail and nothing else.  tests/test_sky_lookup_cpu.py shows in float64 that each frame reaches what it claims and that no ray
of it can reach the volume's root box or the sphere; tests/test_sky_lookup_gpu.py renders the frames with this library and with the
reference kernel.

World units are metres; the planet centre is at (0, -Rg, 0), so world y is the altitude above x = z = 0.  A view direction is given
by yaw (degrees from +x towards +z, the convention of the sun's azimuth) and pitch (degrees above the world xz plane).

Claims (every one is checked on pixels whose centre and four corner rays agree, so any jitter of such a pixel lands on that side):
  split  "ground"       the ray meets the ground (sample_atmosphere's to_ground > 0) / it does not
         "hits_ground"  hits_ground(r, mu) of sky_radiance (at the camera, or where the ray enters the atmosphere from space)
         "space"        to_top > 0: the viewer is above the atmosphere and the ray enters it
         "past"         r > Rt and to_top <= 0: the ray passes the atmosphere (zero radiance, transmittance 1)
         "disc"         dot(ray, sun) > cos(sun_angular_radius): inside the sun disc
  all    "all_past"     every pixel passes the atmosphere
  state  "below_ground" the camera is below the ground sphere (r < Rg)
         "mu_s+", "mu_s0", "mu_s-"   some look-up (sky at the camera or the entry point, or the ground point) has mu_s > 0,
                        mu_s_min < mu_s < 0, or mu_s < mu_s_min (the clamp of u_mu_s)
"""
import ctypes as C
import functools
import math
from dataclasses import dataclass

import numpy as np

f32 = np.float32

# the parameters of V.Atmosphere() the geometry depends on (vpt_atmosphere_host.cpp; test_sky_lookup_gpu checks them against the block)
RG, RT = 6360000.0, 6420000.0
SUN_ANGULAR_RADIUS = float(f32(0.00935 / 2.0))
MU_S_MIN = float(f32(math.cos(120.0 / 180.0 * float(f32(math.pi)))))
W, H = 64, 48                       # frame size of every miss-only case
FOCUS = 1.0e5                       # look-at distance: keeps lower_left_corner's rounding far below a pixel at every altitude used
BEHIND = 20000.0                    # the instance's box centre this far behind the camera plane
SPHERE_RADIUS = 1.0                 # the reference sphere, moved to the same place
BAND_MARGIN = 1e-3                  # a mu_s value counts for a band only this far inside it


@dataclass(frozen=True)
class Sun:
    azimuth: float
    elevation: float
    claims: tuple = ()              # claims that depend on the sun: "disc" and the mu_s bands


@dataclass(frozen=True)
class Geometry:
    name: str
    pos: tuple
    yaw: float
    pitch: float
    fov: float
    suns: tuple
    claims: tuple = ()
    up: tuple = (0.0, 1.0, 0.0)
    size: tuple = (W, H)


def dip(h):
    """Geometric horizon dip (degrees below the horizontal) seen from altitude h."""
    return math.degrees(math.acos(RG / (RG + h)))


_Z = (0.0, 0.0, 1.0)                # up for views near the zenith or the nadir ((0, 1, 0) makes the look-at basis degenerate)

GEOMETRIES = [
    # ground level: the horizon and the sky above it, wide
    Geometry("ground_horizon", (0.0, 1.5, 0.0), 30.0, 0.0, 120.0, (Sun(120.0, 30.0, ("mu_s+",)), Sun(300.0, -15.0, ("mu_s0",)), Sun(220.0, -40.0, ("mu_s-",))),
             ("ground", "hits_ground")),
    Geometry("ground_up", (0.0, 1.5, 0.0), 200.0, 60.0, 150.0, (Sun(200.0, 45.0, ("mu_s+",)), Sun(0.0, 90.0, ("mu_s+",)), Sun(90.0, 3.0, ("mu_s+",))),
             ("ground", "hits_ground")),
    # horizon bands: 0.4 degrees across the geometric horizon, rows on both sides
    *[Geometry(f"horizon_{h:g}m", (0.0, float(h), 0.0), 75.0, -dip(h), 0.4,
               (Sun(75.0, 3.0, ("mu_s+",)), Sun(250.0 if h < 10000 else 75.0, -0.5, ("mu_s0",))), ("ground", "hits_ground"))
      for h in (10.0, 2000.0, 12000.0, 45000.0)],
    # altitude sweep: wide frames looking 20 degrees down
    *[Geometry(f"altitude_{h:g}m", (0.0, float(h), 0.0), 160.0, -20.0, 100.0,
               (Sun(120.0, 30.0, ("mu_s+",)), Sun(300.0, -15.0, ("mu_s0",))), ("ground", "hits_ground")) for h in (500.0, 5000.0, 20000.0, 40000.0, 59900.0)],
    # the top boundary, 1 m inside and 1 m outside the atmosphere
    Geometry("top_inside", (0.0, RT - RG - 1.0, 0.0), 10.0, -10.0, 120.0, (Sun(10.0, 45.0, ("mu_s+",)), Sun(190.0, -15.0, ("mu_s0",))),
             ("ground", "hits_ground")),
    Geometry("top_outside", (0.0, RT - RG + 1.0, 0.0), 10.0, -10.0, 120.0, (Sun(10.0, 45.0, ("mu_s+",)), Sun(190.0, -15.0, ("mu_s0",))),
             ("ground", "hits_ground", "space", "past")),
    # space: 150 km looking down across the limb, 150 km looking up, 1500 km across the limb
    Geometry("space_down_150km", (0.0, 150000.0, 0.0), 0.0, -45.0, 90.0, (Sun(120.0, 30.0, ("mu_s+",)), Sun(180.0, 3.0, ("mu_s+", "mu_s0")), Sun(200.0, -15.0, ("mu_s0",))),
             ("ground", "hits_ground", "space", "past")),
    Geometry("space_up_150km", (0.0, 150000.0, 0.0), 0.0, 90.0, 100.0, (Sun(0.0, 90.0), Sun(120.0, 45.0)), ("all_past",), up=_Z),
    Geometry("limb_1500km", (0.0, 1500000.0, 0.0), 45.0, -(dip(1500000.0) + math.degrees(math.acos(RT / (RG + 1500000.0)))) / 2.0, 2.0,
             (Sun(45.0, 30.0, ("mu_s+",)), Sun(45.0, -40.0, ("mu_s0",))), ("ground", "hits_ground", "space", "past")),
    # the sun disc, a 1.5-degree frame centred on the sun
    Geometry("disc_2m_sun30", (0.0, 2.0, 0.0), 120.0, 30.0, 1.5, (Sun(120.0, 30.0, ("disc", "mu_s+")),)),
    Geometry("disc_2m_sun3", (0.0, 2.0, 0.0), 200.0, 3.0, 1.5, (Sun(200.0, 3.0, ("disc", "mu_s+")),)),
    Geometry("disc_150km_sun30", (0.0, 150000.0, 0.0), 120.0, 30.0, 1.5, (Sun(120.0, 30.0, ("disc",)),), ("all_past",)),
    Geometry("disc_150km_sun3", (0.0, 150000.0, 0.0), 200.0, 3.0, 1.5, (Sun(200.0, 3.0, ("disc",)),), ("all_past",)),
    # all three components of the camera position large
    Geometry("offset_40km", (40000.0, 1000.0, 0.0), 200.0, -5.0, 90.0, (Sun(120.0, 30.0, ("mu_s+",)), Sun(300.0, -15.0, ("mu_s0",))),
             ("ground", "hits_ground")),
    # below the ground sphere
    Geometry("below_ground", (0.0, -2.0, 0.0), 30.0, 0.0, 120.0, (Sun(120.0, 30.0), Sun(300.0, -15.0)), ("hits_ground", "below_ground")),
]
GEOMETRY = {g.name: g for g in GEOMETRIES}
CASES = [(g.name, i) for g in GEOMETRIES for i in range(len(g.suns))]


def case_id(case):
    g, i = GEOMETRY[case[0]], case[1]
    s = g.suns[i]
    return f"{g.name}-az{s.azimuth:g}-el{s.elevation:g}"


def view_direction(yaw, pitch):
    y, p = math.radians(yaw), math.radians(pitch)
    return np.array([math.cos(p) * math.cos(y), math.sin(p), math.cos(p) * math.sin(y)])


def sun_vector(azimuth, elevation):
    """The direction sun_direction(azimuth, elevation) normalises, in float64."""
    return view_direction(azimuth, elevation)


def camera(g):
    """The library's camera of a geometry (vpt_camera_look_at), made on the host."""
    import vpt_b200 as V
    from vpt_b200 import _native as N
    pos = np.asarray(g.pos, dtype=np.float32)
    target = (np.asarray(g.pos, np.float64) + FOCUS * view_direction(g.yaw, g.pitch)).astype(np.float32)
    cam = N.camera()
    N.lib.vpt_camera_look_at(C.byref(cam), N.fvec(pos), N.fvec(target), N.fvec(g.up), float(g.fov), float(g.size[0]) / float(g.size[1]), 0.0)
    return cam


def cam_arrays(cam):
    v = lambda f: np.array([f.x, f.y, f.z], dtype=np.float64)
    return dict(origin=v(cam.origin), llc=v(cam.lower_left_corner), horizontal=v(cam.horizontal), vertical=v(cam.vertical), w=v(cam.w))


@functools.lru_cache(maxsize=1)
def dragon_meta():
    import vpt_b200 as V
    from vpt_b200.scene import load_vdb_grid
    return load_vdb_grid(V.find_asset("dragon.vdb"), "density")[1]


def instance_bounds(pos):
    """vpt_volume_bounds of the dragon instanced at `pos` (float32 [pmin, pmax])."""
    from vpt_b200 import _native as N
    from vpt_b200.scene import instance_xform
    meta = dragon_meta()
    g = N.GPU_VDB()
    g.vdb_info.bmin = N.f3(*[float(b) for b in meta["bbox_min"]]); g.vdb_info.bmax = N.f3(*[float(b) for b in meta["bbox_max"]])
    X = instance_xform(np.array(meta["xform"], dtype=np.float32), pos, (0, 0, 0, 1), 1.0)
    for a in range(4):
        for b in range(4):
            g.xform[a][b] = float(X[a][b])
    b6 = (C.c_float * 6)()
    N.lib.vpt_volume_bounds(C.byref(g), b6)
    return np.array(list(b6), dtype=np.float32)


def placement(g):
    """(instance position, sphere centre): the instance's box centred BEHIND metres behind the camera plane, the sphere at that centre."""
    c0 = instance_bounds((0.0, 0.0, 0.0)).astype(np.float64)
    centre0 = (c0[:3] + c0[3:]) / 2
    w = cam_arrays(camera(g))["w"]                              # backwards: from the look-at point to the camera
    at = np.asarray(g.pos, np.float64) + BEHIND * w
    return tuple(float(v) for v in (at - centre0).astype(np.float32)), tuple(float(v) for v in at.astype(np.float32))


def root_box(pos):
    """The octree's root box of the one-instance scene: the instance's bounds grown by 1 m (vpt_octree_build)."""
    b = instance_bounds(pos)
    return b[:3] - f32(1), b[3:] + f32(1)


JITTERS = ((0.5, 0.5), (0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (1.0, 1.0))   # the pixel centre, then its corners


def rays(cam, size, jitter):
    """float64 unit directions [H, W, 3] of the pinhole rays at jitter (jx, jy): normalize(llc + u horizontal + v vertical - origin),
    u = (x + jx) / W, v = (y + jy) / H (row 0 at the bottom)."""
    Wd, Hd = size
    a = cam_arrays(cam)
    u = (np.arange(Wd)[None, :] + jitter[0]) / Wd
    v = (np.arange(Hd)[:, None] + jitter[1]) / Hd
    b0 = a["llc"][None, None] + u[..., None] * a["horizontal"][None, None] + v[..., None] * a["vertical"][None, None] - a["origin"][None, None]
    return b0 / np.linalg.norm(b0, axis=-1, keepdims=True)


def lookup(origin, d, sun):
    """The branch quantities of sample_atmosphere / sky_radiance for rays `d` from world point `origin`, in float64."""
    p = np.asarray(origin, np.float64) - np.array([0.0, -RG, 0.0])
    pv = d @ p
    pp = p @ p
    with np.errstate(invalid="ignore"):
        to_ground = -pv - np.sqrt(pv * pv - pp + RG * RG)
        ground = to_ground > 0
        r = math.sqrt(pp)
        to_top = -pv - np.sqrt(pv * pv - r * r + RT * RT)
    space = to_top > 0
    past = ~space & (r > RT)
    pe = p[None, None] + d * np.where(space, to_top, 0.0)[..., None]      # the look-up point: the camera, or the entry point
    re = np.where(space, RT, r)
    rmu = np.where(space, pv + to_top, pv)
    mu = rmu / re
    hits_ground = (mu < 0) & (re * re * (mu * mu - 1) + RG * RG >= 0) & ~past
    mu_s = np.where(past, np.nan, (pe @ sun) / re)
    pg = p[None, None] + d * np.where(ground, to_ground, 0.0)[..., None]
    mu_s_ground = np.where(ground, (pg @ sun) / np.linalg.norm(pg, axis=-1), np.nan)
    disc = d @ sun > math.cos(SUN_ANGULAR_RADIUS)
    return dict(ground=ground, hits_ground=hits_ground, space=space, past=past, disc=disc, mu_s=mu_s, mu_s_ground=mu_s_ground, r=r)


SPLITS = ("ground", "hits_ground", "space", "past", "disc")


def classify(g, sun_index):
    """Per pixel and split predicate: +1 where the centre and all four corner rays are on its true side, -1 where all are on its false
    side, 0 where the jitter decides.  Also the mu_s values of the pixel centres and the camera's radius."""
    s = g.suns[sun_index]
    cam = camera(g)
    sun = sun_vector(s.azimuth, s.elevation)
    origin = cam_arrays(cam)["origin"]
    per = [lookup(origin, rays(cam, g.size, j), sun) for j in JITTERS]
    out = {}
    for k in SPLITS:
        a = np.stack([q[k] for q in per])
        out[k] = np.where(a.all(axis=0), 1, np.where(~a.any(axis=0), -1, 0))
    out["mu_s"] = np.concatenate([per[0]["mu_s"].ravel(), per[0]["mu_s_ground"].ravel()])
    out["r"] = per[0]["r"]
    return out


def band_present(mu_s, band):
    v = mu_s[np.isfinite(mu_s)]
    if band == "mu_s+":
        return bool((v > BAND_MARGIN).any())
    if band == "mu_s0":
        return bool(((v > MU_S_MIN + BAND_MARGIN) & (v < -BAND_MARGIN)).any())
    if band == "mu_s-":
        return bool((v < MU_S_MIN - BAND_MARGIN).any())
    raise KeyError(band)


def claims_of(g, sun_index):
    return tuple(g.claims) + tuple(g.suns[sun_index].claims)


def disc_masks(g, sun_index, ring=4.0):
    """(inside, ring) [H, W] bool: pixels inside the sun disc for every jitter, and pixels outside it for every jitter whose centre lies
    within `ring` disc radii of the sun."""
    s = g.suns[sun_index]
    cam = camera(g)
    sun = sun_vector(s.azimuth, s.elevation)
    cosines = np.stack([rays(cam, g.size, j) @ sun for j in JITTERS])
    c = math.cos(SUN_ANGULAR_RADIUS)
    inside = (cosines > c).all(axis=0)
    outside = (cosines <= c).all(axis=0)
    return inside, outside & (cosines[0] > math.cos(ring * SUN_ANGULAR_RADIUS))


def off_disc(g, sun_index):
    s = g.suns[sun_index]
    cam = camera(g)
    sun = sun_vector(s.azimuth, s.elevation)
    return (np.stack([rays(cam, g.size, j) @ sun for j in JITTERS]) <= math.cos(SUN_ANGULAR_RADIUS)).all(axis=0)
