"""Headless scene set-up: the host work `source/main.cpp` does before its frame loop.

Builds, with the library's own loaders and builders (no reference code involved):
  * GPU_VDB instances from .vdb files or dense numpy grids   (gpu_vdb.cpp:105-472 -> vpt_vdb_load + vpt_texture_create_3d)
  * `.ins` style instancing transforms                        (main.cpp:1059-1099)
  * the depth-3 instance octree in the reference node layout  (bvh_builder.cpp:61-96 -> vpt_octree_build)
  * environment map, blue-noise buffer, blackbody / density-colour LUTs, reference sphere
  * the nine launch parameters of `volume_rt_kernel`          (main.cpp:1826)
Device memory is held in torch tensors (plumbing only); textures are CUDA arrays made by the library.
"""
import ctypes as C
import math
import os

import numpy as np
import torch

from . import _native as N
from ._native import lib, check

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ASSET_DIRS = [os.path.join(_REPO, "tests", "golden", "assets"), os.path.join(_REPO, "oracle", "_ref", "assets")]


def find_asset(name):
    for d in ASSET_DIRS:
        p = os.path.join(d, name)
        if os.path.exists(p):
            return p
    return None


def _dev_bytes(buf: bytes, device):
    t = torch.empty(max(len(buf), 1), dtype=torch.uint8, device=device)
    if len(buf):
        t.copy_(torch.frombuffer(bytearray(buf), dtype=torch.uint8))
    return t


class Texture:
    def __init__(self, tex, array):
        self.tex, self.array = int(tex), array

    def destroy(self):
        if self.tex:
            lib.vpt_texture_destroy(self.tex, self.array)
            self.tex, self.array = 0, None


def texture_3d(data: np.ndarray) -> Texture:
    """data: (z, y, x) float32 or (z, y, x, 4) float32."""
    data = np.ascontiguousarray(data, dtype=np.float32)
    ch = 1 if data.ndim == 3 else data.shape[3]
    dz, dy, dx = data.shape[:3]
    tex, arr = C.c_uint64(0), C.c_void_p(0)
    check(lib.vpt_texture_create_3d(data.ctypes.data_as(C.POINTER(C.c_float)), ch, dx, dy, dz, C.byref(tex), C.byref(arr)),
          None, "vpt_texture_create_3d")
    return Texture(tex.value, arr)


def texture_env(rgba: np.ndarray) -> Texture:
    rgba = np.ascontiguousarray(rgba, dtype=np.float32)
    h, w = rgba.shape[:2]
    tex, arr = C.c_uint64(0), C.c_void_p(0)
    check(lib.vpt_texture_create_env(rgba.ctypes.data_as(C.POINTER(C.c_float)), w, h, C.byref(tex), C.byref(arr)), None, "vpt_texture_create_env")
    return Texture(tex.value, arr)


def sky_power_table(azimuth=120.0, elevation=30.0, sky_color=(1.0, 1.0, 1.0), res=180) -> np.ndarray:
    """The res x res table create_cdf builds from the reference's host-side analytic sky (vpt_env_sky_tabulate)."""
    out = np.empty((res, res), dtype=np.float32)
    col = (C.c_float * 3)(*[float(c) for c in sky_color])
    check(lib.vpt_env_sky_tabulate(float(azimuth), float(elevation), col, int(res), out.ctypes.data_as(C.POINTER(C.c_float))), None, "vpt_env_sky_tabulate")
    return out


class EnvTables:
    """Sky-sampling tables of the volumetric path integrator (Kernel_params.env_*_tex), built by vpt_env_tables_create."""
    def __init__(self, func: np.ndarray):
        func = np.ascontiguousarray(func, dtype=np.float32)
        assert func.ndim == 2 and func.shape[0] == func.shape[1]
        self.res = int(func.shape[0])
        tex = (C.c_uint64 * 4)(); arr = (C.c_void_p * 4)(); mint = C.c_float(0)
        check(lib.vpt_env_tables_create(func.ctypes.data_as(C.POINTER(C.c_float)), self.res, tex, arr, C.byref(mint)), None, "vpt_env_tables_create")
        self.textures = [Texture(tex[i], arr[i]) for i in range(4)]
        self.marginal_int = float(mint.value)

    def apply(self, kp):
        kp.env_func_tex, kp.env_cdf_tex, kp.env_marginal_func_tex, kp.env_marginal_cdf_tex = (t.tex for t in self.textures)
        kp.env_marginal_int = self.marginal_int; kp.env_sample_tex_res = self.res

    def destroy(self):
        for t in self.textures: t.destroy()


def load_vdb_grid(path, grid):
    """-> (values (z,y,x[,3]) float32, info dict) or None when the grid is absent."""
    vals = C.POINTER(C.c_float)()
    info = (C.c_int * 13)(); xf = (C.c_float * 16)(); st = (C.c_float * 4)()
    rc = lib.vpt_vdb_load(path.encode(), grid.encode(), C.byref(vals), info, xf, st)
    if rc == 1:
        return None
    check(rc, None, f"vpt_vdb_load({path}, {grid})")
    dx, dy, dz = info[0], info[1], info[2]
    ch = info[9]
    n = dx * dy * dz * ch
    arr = np.ctypeslib.as_array(vals, shape=(n,)).copy()
    lib.vpt_free(vals)
    arr = arr.reshape((dz, dy, dx) if ch == 1 else (dz, dy, dx, ch))
    meta = dict(dim=(dx, dy, dz), bbox_min=(info[3], info[4], info[5]), bbox_max=(info[6], info[7], info[8]), channels=ch,
                leaf_count=info[10], active_voxels=(info[11] & 0xffffffff) | (info[12] << 32),
                xform=np.array(list(xf), dtype=np.float32).reshape(4, 4), max_value=st[0], min_density=st[1],
                voxel_size=st[2], background=st[3])
    return arr, meta


def load_hdr(path):
    px = C.POINTER(C.c_float)(); w = C.c_uint(0); h = C.c_uint(0)
    check(lib.vpt_hdr_load(path.encode(), C.byref(px), C.byref(w), C.byref(h)), None, "vpt_hdr_load")
    a = np.ctypeslib.as_array(px, shape=(h.value, w.value, 4)).copy()
    lib.vpt_free(px)
    return a


def load_bmp_rbg(path):
    px = C.POINTER(C.c_float)(); w = C.c_int(0); h = C.c_int(0)
    check(lib.vpt_bmp_load_rbg(path.encode(), C.byref(px), C.byref(w), C.byref(h)), None, "vpt_bmp_load_rbg")
    a = np.ctypeslib.as_array(px, shape=(h.value, w.value, 3)).copy()
    lib.vpt_free(px)
    return a


def load_exr_rgb(path):
    px = C.POINTER(C.c_float)(); w = C.c_int(0); h = C.c_int(0)
    check(lib.vpt_exr_load_rgb(path.encode(), C.byref(px), C.byref(w), C.byref(h)), None, "vpt_exr_load_rgb")
    a = np.ctypeslib.as_array(px, shape=(h.value, w.value, 3)).copy()
    lib.vpt_free(px)
    return a


# ---- reference mat4 algebra (m[col][row] memory image), float32, no FMA ------------------------------
def mat4_identity():
    return np.eye(4, dtype=np.float32)


def mat4_mul_ref(A, B):
    """The reference's `mat4::operator*(mat4)` (matrix_math.h:130-162): with a_rc = A.m[c][r] it stores
    ret.m[r][c] = sum_k a_rk * b_kc -- i.e. the memory image of the result is (A^T_mem ... ) as coded, not a
    textbook product; reproduced literally so instance transforms match."""
    a = A.T.astype(np.float32)   # a[r][c] = A.m[c][r]
    b = B.T.astype(np.float32)
    R = np.zeros((4, 4), dtype=np.float32)
    for r in range(4):
        for c in range(4):
            acc = np.float32(a[r][0] * b[0][c])
            for k in range(1, 4):
                acc = np.float32(acc + np.float32(a[r][k] * b[k][c]))
            R[r][c] = acc            # ret[r][c] = ret.m[r][c]
    return R


def quaternion_to_mat4(x, y, z, w):
    """matrix_math.h:378-412 (double overload; normalisation uses sqrtf)."""
    n = 1.0 / float(np.sqrt(np.float32(x * x + y * y + z * z + w * w)))
    x, y, z, w = x * n, y * n, z * n, w * n
    f = np.float32
    m11, m12, m13 = f(1.0 - 2.0 * y * y - 2.0 * z * z), f(2.0 * x * y + 2.0 * z * w), f(2.0 * x * z - 2.0 * y * w)
    m21, m22, m23 = f(2.0 * x * y - 2.0 * z * w), f(1.0 - 2.0 * x * x - 2.0 * z * z), f(2.0 * y * z + 2.0 * x * w)
    m31, m32, m33 = f(2.0 * x * z + 2.0 * y * w), f(2.0 * y * z - 2.0 * x * w), f(1.0 - 2.0 * x * x - 2.0 * y * y)
    M = np.zeros((4, 4), dtype=np.float32)
    # mat4(m11..m44) stores m[0][0]=m11, m[1][0]=m12, m[2][0]=m13, m[3][0]=m14, m[0][1]=m21, ...
    rows = [[m11, m12, m13, 0.0], [m21, m22, m23, 0.0], [m31, m32, m33, 0.0], [0.0, 0.0, 0.0, 1.0]]
    for r in range(4):
        for c in range(4):
            M[c][r] = rows[r][c]
    return M


def instance_xform(base_xform, pos, quat, scale):
    """main.cpp:1066-1097: zero the translation, scale the diagonal, rotate, translate."""
    X = np.array(base_xform, dtype=np.float32).copy()
    X[0][3] = X[1][3] = X[2][3] = np.float32(0.0)
    s = np.float32(scale)
    X[0][0] *= s; X[1][1] *= s; X[2][2] *= s
    R = quaternion_to_mat4(*[float(q) for q in quat])
    X = mat4_mul_ref(R, X)
    X[0][3] += np.float32(pos[0]); X[1][3] += np.float32(pos[1]); X[2][3] += np.float32(pos[2])
    return X


class Volume:
    """One unique VDB: textures + the GPU_VDB record the kernels read (GPU_VDB::loadVDB, gpu_vdb.cpp:105-472)."""

    def __init__(self):
        self.textures = []
        self.rec = N.GPU_VDB()

    @staticmethod
    def from_dense(density: np.ndarray, bbox_min=(0, 0, 0), xform=None, voxelsize=1.0, emission=None, color=None):
        v = Volume()
        dz, dy, dx = density.shape
        info = v.rec.vdb_info
        info.voxelsize = float(voxelsize)
        info.dim = N.i3(dx, dy, dz)
        info.bmin = N.f3(*[float(b) for b in bbox_min])
        info.bmax = N.f3(float(bbox_min[0] + dx - 1), float(bbox_min[1] + dy - 1), float(bbox_min[2] + dz - 1))
        d32 = np.ascontiguousarray(density, dtype=np.float32)
        # max/min rule of gpu_vdb.cpp:206-207 (VDB_INFO defaults 0 / FLT_MAX): min over max(FLT_EPSILON, v) -- quirk Q10
        info.max_density = float(max(np.float32(0.0), d32.max()))
        info.min_density = float(np.minimum(np.maximum(np.float32(np.finfo(np.float32).eps), d32), np.float32(3.4028235e38)).min())
        t = texture_3d(d32); v.textures.append(t); info.density_texture = t.tex
        if emission is not None:
            t = texture_3d(np.ascontiguousarray(emission, dtype=np.float32)); v.textures.append(t)
            info.emission_texture = t.tex; info.has_emission = 1
        if color is not None:
            c4 = np.zeros(color.shape[:3] + (4,), dtype=np.float32); c4[..., :3] = color[..., :3]; c4[..., 3] = 1.0
            t = texture_3d(c4); v.textures.append(t)
            info.color_texture = t.tex; info.has_color = 1
        X = mat4_identity() if xform is None else np.array(xform, dtype=np.float32)
        for a in range(4):
            for b in range(4):
                v.rec.xform[a][b] = float(X[a][b])
        return v

    @staticmethod
    def procedural(dims, box_min=None, res=1.0, scale=0.1, seed=123, device="cuda:0", keep_dense=True):
        """GPU_PROC_VOL::create_volume (gpu_vdb.cpp:508-609) headless: Perlin density grid filled on the device by the library
        (vpt_procedural_fill: the reference's fill_volume_buffer, noise type 0, zero jitter), turned into the same clamp /
        linear / normalised 3-D texture, with the VDB_INFO the reference hard-codes for procedural volumes (max 1, min 0,
        bmax = bmin + dim, xform = scale(res); quirk Q10).  dims = (dx, dy, dz) voxels."""
        dx, dy, dz = [int(d) for d in dims]
        v = Volume()
        torch.cuda.set_device(torch.device(device))
        dense = torch.empty(dz * dy * dx, dtype=torch.float32, device=device)
        check(lib.vpt_procedural_fill(C.c_void_p(dense.data_ptr()), dx, dy, dz, 0, float(scale), int(seed), None), None, "vpt_procedural_fill")
        torch.cuda.synchronize()
        tex, arr = C.c_uint64(0), C.c_void_p(0)
        check(lib.vpt_texture_create_3d_from_device(C.c_void_p(dense.data_ptr()), 1, dx, dy, dz, C.byref(tex), C.byref(arr)), None, "vpt_texture_create_3d_from_device")
        t = Texture(tex.value, arr); v.textures.append(t)
        if box_min is None: box_min = (-dx * res / 2.0, -dy * res / 2.0, -dz * res / 2.0)
        info = v.rec.vdb_info
        info.voxelsize = float(res); info.dim = N.i3(dx, dy, dz)
        info.bmin = N.f3(*[float(b) for b in box_min]); info.bmax = N.f3(float(box_min[0] + dx), float(box_min[1] + dy), float(box_min[2] + dz))
        info.max_density = 1.0; info.min_density = 0.0; info.density_texture = t.tex
        X = mat4_identity()
        X[0][0] = X[1][1] = X[2][2] = np.float32(res)                     # mat4::scale(res) on the identity
        for a in range(4):
            for b in range(4):
                v.rec.xform[a][b] = float(X[a][b])
        v.dims = (dx, dy, dz)
        v.dense = dense if keep_dense else None
        v.brick_pool = 0
        return v

    def build_bricks(self):
        """Brick pool of the density grid for fast mode (vpt_bricks_create); needs the dense device grid kept by procedural()."""
        assert getattr(self, "dense", None) is not None, "no dense device grid kept for this volume"
        pool = C.c_uint64(0); nbytes = C.c_ulonglong(0)
        dx, dy, dz = self.dims
        check(lib.vpt_bricks_create(C.c_void_p(self.dense.data_ptr()), dx, dy, dz, C.byref(pool), C.byref(nbytes)), None, "vpt_bricks_create")
        self.brick_pool = pool.value; self.brick_bytes = int(nbytes.value)
        return self.brick_pool

    def build_cells(self):
        """Cell table of the density grid for cell mode (vpt_cells_create: 32 bytes per texel cell, one sector per look-up)."""
        assert getattr(self, "dense", None) is not None, "no dense device grid kept for this volume"
        tab = C.c_uint64(0); nbytes = C.c_ulonglong(0)
        dx, dy, dz = self.dims
        check(lib.vpt_cells_create(C.c_void_p(self.dense.data_ptr()), dx, dy, dz, C.byref(tab), C.byref(nbytes)), None, "vpt_cells_create")
        self.cell_table = tab.value; self.cell_bytes = int(nbytes.value)
        return self.cell_table

    @staticmethod
    def load_vdb(path, density="density", emission="heat", color="Cd"):
        got = load_vdb_grid(path, density)
        if got is None:
            raise N.VptError(f"{path}: no grid named {density!r}")
        dens, meta = got
        em = load_vdb_grid(path, emission) if emission else None
        cd = load_vdb_grid(path, color) if color else None
        v = Volume.from_dense(dens, bbox_min=meta["bbox_min"], xform=meta["xform"], voxelsize=meta["voxel_size"],
                              emission=None if em is None else em[0], color=None if cd is None else cd[0])
        # bmax is the inclusive index bbox max (gpu_vdb.cpp:453-455)
        v.rec.vdb_info.bmax = N.f3(*[float(b) for b in meta["bbox_max"]])
        v.meta = meta
        return v

    def instance(self, pos=(0, 0, 0), quat=(0, 0, 0, 1), scale=1.0) -> N.GPU_VDB:
        g = N.GPU_VDB()
        C.memmove(C.byref(g), C.byref(self.rec), C.sizeof(N.GPU_VDB))
        base = np.array([[self.rec.xform[a][b] for b in range(4)] for a in range(4)], dtype=np.float32)
        X = instance_xform(base, pos, quat, scale)
        for a in range(4):
            for b in range(4):
                g.xform[a][b] = float(X[a][b])
        return g


def load_ins(path):
    """Parse a reference `.ins` scene / light file (read_instance_file, main.cpp:980-1040) with the library's reader.
    -> {"kind": "volumes", "files": [{"path": str, "instances": [(pos3, quat4, scale), ...]}, ...]}
     | {"kind": "lights",  "lights": [(pos3, rgb3, power), ...]}"""
    hp = C.POINTER(N.ins_header)()
    check(lib.vpt_ins_load(os.fsencode(path), C.byref(hp)), None, "vpt_ins_load")
    try:
        h = hp.contents
        base = C.addressof(h) + C.sizeof(N.ins_header)
        entries = (N.ins_file_entry * h.n_files).from_address(base)
        recs = np.ctypeslib.as_array((C.c_double * (8 * h.n_records)).from_address(base + h.n_files * C.sizeof(N.ins_file_entry))).reshape(-1, 8).copy()
        if h.kind == 1:
            return {"kind": "lights", "lights": [(tuple(r[0:3]), tuple(r[3:6]), float(r[6])) for r in recs]}
        files = []
        for e in entries:
            rr = recs[e.first_record:e.first_record + e.n_instances]
            files.append({"path": e.path.decode(), "instances": [(tuple(r[0:3]), tuple(r[3:7]), float(r[7])) for r in rr]})
        return {"kind": "volumes", "files": files}
    finally:
        lib.vpt_free(hp)


def scene_from_ins(path, env=None, resolve=None, device="cuda:0"):
    """Build a Scene the way the reference does for an `.ins` argument (main.cpp:1040-1102): every listed .vdb is loaded once
    and instanced with its (position, quaternion, scale) records; a "light" file yields the point-light list instead.
    `resolve(path) -> path` maps the verbatim paths of the file (the reference uses them relative to its CWD).  The scene's
    instance_names are "<vdb stem>.<k>", the k-th instance of that file (the names Renderer.enable_cryptomatte hashes)."""
    d = load_ins(path)
    if d["kind"] == "lights":
        return d["lights"]
    instances, names = [], []
    for f in d["files"]:
        vol = Volume.load_vdb(resolve(f["path"]) if resolve else f["path"])
        instances += [vol.instance(pos, quat, scale) for pos, quat, scale in f["instances"]]
        stem = os.path.splitext(os.path.basename(f["path"].replace("\\", "/")))[0]
        names += [f"{stem}.{k}" for k in range(len(f["instances"]))]
    return Scene(instances, env=env, device=device, instance_names=names)


def synthetic_env(width=3000, height=1500):
    """Procedural HDR sky of the reference HDRI's shape, used only when the asset is not on the box."""
    v = np.linspace(0.0, 1.0, height, dtype=np.float32)[:, None]
    u = np.linspace(0.0, 1.0, width, dtype=np.float32)[None, :]
    sky = 0.25 + 0.75 * (1.0 - v) ** 2
    sun = 40.0 * np.exp(-((u - 0.3) ** 2 + (v - 0.25) ** 2) / 0.0005)
    rgba = np.zeros((height, width, 4), dtype=np.float32)
    rgba[..., 0] = 0.6 * sky + sun; rgba[..., 1] = 0.75 * sky + 0.9 * sun; rgba[..., 2] = 1.0 * sky + 0.8 * sun
    return rgba


def synthetic_blue_noise():
    rng = np.random.RandomState(1234)
    return rng.rand(256, 256, 3).astype(np.float32)


class Scene:
    """Everything the nine launch parameters point at (main.cpp:1299-1313, 1378-1403, 1480-1502)."""

    def __init__(self, instances, device="cuda:0", env="Barce_Rooftop_C_3k.hdr", lights=None, keep=None, instance_names=None):
        self.device = torch.device(device)
        # one name per instance (Renderer.enable_cryptomatte's default names), or None
        self.instance_names = [str(x) for x in instance_names] if instance_names is not None else None
        torch.cuda.set_device(self.device)
        self.keep = keep or []
        self.instances = list(instances)
        n = len(self.instances)
        arr = (N.GPU_VDB * n)(*self.instances)
        self.h_volumes = arr
        self.d_volumes = _dev_bytes(bytes(arr), self.device)
        root = C.c_uint64(0)
        check(lib.vpt_octree_build(arr, n, C.byref(root)), None, "vpt_octree_build")
        self.d_oct_root = root.value
        self.own_octree = True
        # reference sphere (main.cpp:1480-1488)
        sp = N.sphere(); sp.center = N.f3(0, 1000, 0); sp.radius = 1.0; sp.color = N.f3(10.0, 0, 0); sp.roughness = 1.0
        self.h_sphere = sp
        self.d_sphere = _dev_bytes(bytes(sp), self.device)
        self.d_geo_list = _dev_bytes(bytes(N.geometry_list()), self.device)
        self.d_bvh = _dev_bytes(bytes(N.BVHNode()), self.device)
        # lights (managed memory in the reference; plain device memory is equivalent for the kernels)
        self.lights = N.light_list()
        if lights:
            pl = (N.point_light * len(lights))()
            for i, (pos, col, power) in enumerate(lights):
                pl[i].pos = N.f3(*pos); pl[i].color = N.f3(*col); pl[i].power = float(power)
            self.d_lights = _dev_bytes(bytes(pl), self.device)
            self.lights.num_lights = len(lights); self.lights.light_ptr = self.d_lights.data_ptr()
        # blue noise (fileIO.cpp:460-495), LUTs (main.cpp:1389-1402)
        p = find_asset("BN0.bmp")
        bn = load_bmp_rbg(p) if p else synthetic_blue_noise()
        self.data_notes = [] if p else ["blue noise: synthetic (BN0.bmp not found)"]
        self.bn_host = np.ascontiguousarray(bn.reshape(-1, 3), dtype=np.float32)
        self.d_blue_noise = torch.from_numpy(self.bn_host.copy()).to(self.device)
        p = find_asset("blackbody_texture.exr")
        bb = load_exr_rgb(p).reshape(-1, 3) if p else np.linspace(0, 1, 256, dtype=np.float32)[:, None].repeat(3, 1)
        self.d_emission_lut = torch.from_numpy(np.ascontiguousarray(bb, dtype=np.float32)).to(self.device)
        p = find_asset("density_color_texture2.exr")
        dc = load_exr_rgb(p).reshape(-1, 3) if p else np.ones((256, 3), dtype=np.float32)
        self.d_density_color = torch.from_numpy(np.ascontiguousarray(dc, dtype=np.float32)).to(self.device)
        # environment (main.cpp:945-978)
        self.env_tex = None
        if env is not None:
            if isinstance(env, np.ndarray):
                rgba = env
            else:
                p = find_asset(env)
                if p:
                    rgba = load_hdr(p)
                else:
                    rgba = synthetic_env(); self.data_notes.append(f"environment: synthetic 3000x1500 ({env} not found)")
            self.env_tex = texture_env(rgba)
        # atmosphere block: the render path with an HDRI never reads the LUTs, but the reference kernel still
        # issues two (dead) fetches from them in estimate_sun, so give it valid 1-texel textures
        self.atmos = N.AtmosphereParameters()
        self._dummy2d = texture_env(np.zeros((1, 1, 4), dtype=np.float32))
        self._dummy3d = texture_3d(np.zeros((1, 1, 1, 4), dtype=np.float32))
        self.atmos.transmittance_texture = self._dummy2d.tex; self.atmos.irradiance_texture = self._dummy2d.tex
        self.atmos.scattering_texture = self._dummy3d.tex; self.atmos.single_mie_scattering_texture = self._dummy3d.tex
        self.atmos.bottom_radius = 6360.0; self.atmos.top_radius = 6420.0

    def octree_info(self):
        n = C.c_int(0); ref = C.c_int(0); tot = C.c_longlong(0); mx = C.c_int(0)
        check(lib.vpt_octree_info(self.d_oct_root, C.byref(n), C.byref(ref), C.byref(tot), C.byref(mx)), None, "vpt_octree_info")
        return dict(n=n.value, reference_layout=bool(ref.value), total_leaf_entries=tot.value, max_leaf_entries=mx.value)

    def leaf_lists(self):
        """The flat (CSR) leaf lists the render kernels read: list of 512 ascending instance-id lists."""
        tab = (C.c_uint * 1024)()
        check(lib.vpt_octree_read_flat(self.d_oct_root, tab, None, 0), None, "vpt_octree_read_flat")
        total = sum(tab[2 * l + 1] for l in range(512))
        idx = (C.c_int * max(total, 1))()
        check(lib.vpt_octree_read_flat(self.d_oct_root, tab, idx, total), None, "vpt_octree_read_flat")
        return [list(idx[tab[2 * l]:tab[2 * l] + tab[2 * l + 1]]) for l in range(512)]

    def build_bvh(self):
        """LBVH over the instances in the reference's BVHNode layout (vpt_bvh_build); keeps the device arrays alive in
        self.bvh and points params[5] (`root_node`) at them.  Returns the host view (pointers as indices)."""
        n = len(self.instances)
        nodes = C.c_uint64(0); leaves = C.c_uint64(0); sb = (C.c_float * 6)()
        codes = (C.c_ulonglong * n)(); ids = (C.c_int * n)()
        check(lib.vpt_bvh_build(self.h_volumes, n, C.byref(nodes), C.byref(leaves), sb, codes, ids), None, "vpt_bvh_build")
        self.bvh = (nodes.value, leaves.value)
        return read_bvh(nodes.value, leaves.value, n) | dict(scene_bounds=list(sb), codes=list(codes), ids=list(ids), d_nodes=nodes.value, d_leaves=leaves.value)

    def reset_blue_noise(self):
        self.d_blue_noise.copy_(torch.from_numpy(self.bn_host))

    def world_bounds(self):
        """bbox used by the F-key framing (main.cpp:525-543): min/max with the origin included."""
        lo = np.zeros(3, dtype=np.float32); hi = np.zeros(3, dtype=np.float32)
        for g in self.instances:
            X = np.array([[g.xform[a][b] for b in range(4)] for a in range(4)], dtype=np.float32)
            for corner, agg in ((g.vdb_info.bmin, "lo"), (g.vdb_info.bmax, "hi")):
                p = np.array([corner.x, corner.y, corner.z, 1.0], dtype=np.float32)
                w = np.array([np.dot(X[r], p) for r in range(3)], dtype=np.float32)   # xform.transpose().transform_point
                if agg == "lo": lo = np.minimum(lo, w)
                else: hi = np.maximum(hi, w)
        return lo, hi

    def frame_camera(self, width, height, fov=30.0, aperture=0.0) -> N.camera:
        lo, hi = self.world_bounds()
        center = (hi + lo) / np.float32(2)
        dist = float(np.linalg.norm(hi - lo))
        lookfrom = center + np.float32(dist)
        cam = N.camera()
        lib.vpt_camera_look_at(C.byref(cam), N.fvec(lookfrom), N.fvec(center), N.fvec((0, 1, 0)), float(fov), float(width) / float(height), float(aperture))
        return cam

    def destroy(self):
        if self.own_octree and self.d_oct_root:
            lib.vpt_octree_destroy(self.d_oct_root); self.d_oct_root = 0
        if getattr(self, "bvh", None):
            lib.vpt_bvh_destroy(*self.bvh); self.bvh = None
        for t in (self.env_tex, self._dummy2d, self._dummy3d):
            if t: t.destroy()


class Atmosphere:
    """The Bruneton sky model + its four precomputed look-up textures, built by the library (vpt_atmosphere_precompute:
    replaces atmosphere::init, source/atmosphere/atmosphere.cpp:1177-1291).  `apply(scene.atmos)` fills a Scene's
    AtmosphereParameters block in place."""

    SHAPES = dict(transmittance=(256, 64, 0), scattering=(256, 128, 32), irradiance=(256, 64, 0), single_mie=(256, 128, 32))

    def __init__(self, use_constant_solar_spectrum=True, use_ozone=True, luminance=0, white_balance=True, exposure=1.0, orders=4):
        o = N.atmosphere_options()
        lib.vpt_atmosphere_options_defaults(C.byref(o))
        o.use_constant_solar_spectrum = int(use_constant_solar_spectrum); o.use_ozone = int(use_ozone); o.luminance_mode = int(luminance)
        o.do_white_balance = int(white_balance); o.exposure = float(exposure); o.num_scattering_orders = int(orders)
        self.params = N.AtmosphereParameters(); self.handle = C.c_void_p(0)
        check(lib.vpt_atmosphere_precompute(C.byref(o), C.byref(self.params), C.byref(self.handle)), None, "vpt_atmosphere_precompute")

    def apply(self, atmos):
        C.memmove(C.byref(atmos), C.byref(self.params), C.sizeof(N.AtmosphereParameters))

    def destroy(self):
        if self.handle: lib.vpt_atmosphere_destroy(self.handle); self.handle = C.c_void_p(0)


def read_atmosphere_tables(atmos):
    """The four look-up textures of an AtmosphereParameters block (this library's or the reference's) as numpy arrays [..., 4]."""
    out = {}
    for name, tex in (("transmittance", atmos.transmittance_texture), ("scattering", atmos.scattering_texture),
                      ("irradiance", atmos.irradiance_texture), ("single_mie", atmos.single_mie_scattering_texture)):
        w, h, d = Atmosphere.SHAPES[name]
        a = np.empty((max(d, 1), h, w, 4), dtype=np.float32)
        check(lib.vpt_texture_read_f4(tex, w, h, d, a.ctypes.data_as(C.POINTER(C.c_float))), None, "vpt_texture_read_f4")
        out[name] = a if d else a[0]
    return out


def read_bvh(d_nodes, d_leaves, n):
    """Host view of a BVH in the reference layout (either builder's): child / parent fields as indices (-1 = none)."""
    hn = (N.BVHNode * max(n - 1, 1))(); hl = (N.BVHNode * n)()
    check(lib.vpt_bvh_read(d_nodes, d_leaves, n, hn, hl), None, "vpt_bvh_read")
    def view(b, leaf):
        sx = lambda v: -1 if v == 0xffffffffffffffff else int(v)
        return dict(minId=b.minId, maxId=b.maxId, volIndex=b.volIndex, left=sx(b.leftChild), right=sx(b.rightChild), parent=sx(b.parent),
                    box=bytes(b.boundingBox), leaf=leaf)
    return dict(nodes=[view(hn[i], False) for i in range(n - 1)], leaves=[view(hl[i], True) for i in range(n)])


def default_kernel_params() -> N.Kernel_params:
    kp = N.Kernel_params()
    lib.vpt_kernel_params_defaults(C.byref(kp))
    return kp
