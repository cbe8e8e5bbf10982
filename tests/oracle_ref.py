"""Test-side wrapper of the ORACLE: the reference's own `volume_rt_kernel`, octree builder and
blue-noise update, compiled from the reference tree by oracle/Makefile into oracle/_ref/.

Where oracle/_ref is not built, the oracle REPLAYS the outputs stored under tests/golden/oracle/ for the same test and call,
after checking that a hash of the inputs matches.  To store them: run the tests with the oracle built and VPT_ORACLE_RECORD=<dir>,
then `python tests/oracle_ref.py <dir> [first pack number]`.  What has no stored output (or did not fit in 1 MB) skips without the oracle.

Only tests/, __graft_entry__.smoke() and bench.py's reference arm may import this module.
"""
import ctypes as C
import hashlib
import json
import os
import re

import numpy as np
import torch

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(_REPO, "oracle", "_ref")
LIB = os.path.join(REF_DIR, "libvpt_ref.so")


_ATMO_CACHE = {}
_ATMO_TABLES = ("transmittance_texture", "scattering_texture", "irradiance_texture", "single_mie_scattering_texture")


GOLDEN_DIR = os.path.join(_REPO, "tests", "golden", "oracle")
RECORD_DIR = os.environ.get("VPT_ORACLE_RECORD")
MAX_FILE_BYTES = 1_000_000


def available():
    return all(os.path.exists(os.path.join(REF_DIR, f)) for f in
               ("libvpt_ref.so", "render_kernel_ref.cubin", "render_kernel_ref_nobn.cubin", "bn_advance_ref.cubin"))


def replaying():
    """No oracle build here, but stored oracle outputs are."""
    return not available() and os.path.isdir(GOLDEN_DIR)


def usable():
    return available() or replaying()


_call = {"test": None, "n": 0}


def _key(kind):
    """<test id>.<call number within the test>.<kind>: the same test makes the same calls in the same order."""
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    if test != _call["test"]:
        _call.update(test=test, n=0)
    _call["n"] += 1
    return re.sub(r"[^A-Za-z0-9_.-]+", "_", os.path.basename(test)) + f".{_call['n']}.{kind}"


def _digest(*parts):
    h = hashlib.sha256()
    for p in parts:
        h.update(p if isinstance(p, (bytes, bytearray)) else repr(p).encode())
    return h.hexdigest()


def _kp_scalars(kp):
    """Kernel_params without its device pointers (those differ from run to run)."""
    b = bytearray(bytes(kp))
    for name, t in type(kp)._fields_:
        if t is C.c_uint64:
            off = getattr(type(kp), name).offset
            b[off:off + 8] = bytes(8)
    return bytes(b)


def _volumes_digest(h_volumes, n):
    """The instance list without its texture handles."""
    out = []
    for i in range(n):
        v = h_volumes[i]
        b = bytearray(bytes(v))
        info = type(v.vdb_info)
        for name in ("density_texture", "emission_texture", "color_texture"):
            off = getattr(info, name).offset
            b[off:off + 8] = bytes(8)
        out.append(bytes(b))
    return _digest(*out)


def _store(key, arrays):
    """One compressed file per array (<key>.<name>.npz); a case with any file above MAX_FILE_BYTES is not stored at all."""
    if not RECORD_DIR:
        return
    os.makedirs(RECORD_DIR, exist_ok=True)
    paths = []
    for name, arr in arrays.items():
        paths.append(os.path.join(RECORD_DIR, f"{key}.{name}.npz"))
        np.savez_compressed(paths[-1], a=arr)
    if any(os.path.getsize(q) > MAX_FILE_BYTES for q in paths):
        for q in paths: os.remove(q)


_packs = {}


def _stored_names():
    """array name -> pack file, over tests/golden/oracle/pack*.npz"""
    if not _packs and os.path.isdir(GOLDEN_DIR):
        for f in sorted(os.listdir(GOLDEN_DIR)):
            if f.startswith("pack") and f.endswith(".npz"):
                with np.load(os.path.join(GOLDEN_DIR, f)) as z:
                    _packs.update({n: f for n in z.files})
    return _packs


class _Stored(str):
    def __getitem__(self, name):
        full = f"{self}.{name}"
        if full not in _stored_names():                  # stored once under another key (pack: SAME_AS)
            with np.load(os.path.join(GOLDEN_DIR, _stored_names()[full + SAME_AS])) as z:
                full = str(z[full + SAME_AS])
        with np.load(os.path.join(GOLDEN_DIR, _stored_names()[full])) as z:
            return z[full]


def _load(key, digest):
    import pytest
    if f"{key}.digest" not in _stored_names():
        pytest.skip(f"oracle/_ref not built and no stored oracle output {key}")
    z = _Stored(key)
    assert str(z["digest"]) == digest, f"{key}: the inputs differ from those the stored oracle output was made with"
    return z


class _NoLibrary:
    """Replaying: any direct use of the reference build skips the test."""
    def __getattr__(self, name):
        import pytest
        pytest.skip(f"oracle/_ref not built: {name} has no stored output")


SAME_AS = "@"


def pack(record_dir, out_dir=GOLDEN_DIR, limit=990_000, first=0):
    """Pack the per-array files of a recording run (<key>.<name>.npz) into as few files below 1 MB as the array sizes allow, numbered
    from pack<first>: a run that recorded only some tests packs them after the existing packs.  An array equal to one packed before it
    (the blue-noise state after the same number of passes over the same frame size, say) is stored once: the later key holds only the
    earlier key's name, under <key>.<name>@."""
    entries, seen = [], {}                               # (array name, array, compressed size)
    for f in sorted(os.listdir(record_dir)):
        name, a = f[:-len(".npz")], np.load(os.path.join(record_dir, f))["a"]
        h = (a.dtype.str, a.shape, hashlib.sha256(a.tobytes()).hexdigest())
        if h in seen and a.nbytes > 1024:
            entries.append((name + SAME_AS, np.array(seen[h]), 256))
        else:
            seen.setdefault(h, name)
            entries.append((name, a, os.path.getsize(os.path.join(record_dir, f))))
    os.makedirs(out_dir, exist_ok=True)
    groups, cur, size = [], [], 0
    for e in entries:
        if cur and size + e[2] > limit:
            groups.append(cur); cur, size = [], 0
        cur.append(e); size += e[2]
    if cur: groups.append(cur)
    for i, g in enumerate(groups):
        path = os.path.join(out_dir, f"pack{first + i:02d}.npz")
        np.savez_compressed(path, **{name: a for name, a, _ in g})
        assert os.path.getsize(path) <= MAX_FILE_BYTES, path


def create_cdf(func):
    """The reference's own create_cdf arithmetic (oracle/_ref/libcreate_cdf_ref.so, host only) on a res x res table:
    (func as read back, conditional cdf, marginal func, marginal cdf, marginal integral as a c_float)."""
    res = func.shape[0]
    key, digest = _key("cdf"), _digest(np.ascontiguousarray(func, dtype=np.float32).tobytes())
    path = os.path.join(REF_DIR, "libcreate_cdf_ref.so")
    if not os.path.exists(path):
        z = _load(key, digest)
        return z["func"], z["cdf"], z["mf"], z["mc"], C.c_float(float(z["integral"]))
    lib = C.CDLL(path)
    lib.vptref_create_cdf.argtypes = [C.POINTER(C.c_float)] * 5 + [C.POINTER(C.c_float), C.c_float]
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    r_func = np.empty((res, res), np.float32); r_cdf = np.empty((res, res), np.float32)
    r_mf = np.empty(res, np.float32); r_mc = np.empty(res, np.float32); r_int = C.c_float(0)
    assert lib.vptref_create_cdf(fp(func), fp(r_func), fp(r_cdf), fp(r_mf), fp(r_mc), C.byref(r_int), 0.0) == 0
    _store(key, dict(digest=np.array(digest), func=r_func, cdf=r_cdf, mf=r_mf, mc=r_mc, integral=np.array(r_int.value, np.float32)))
    return r_func, r_cdf, r_mf, r_mc, r_int


class RefOracle:
    """Drives the reference kernel with a byte-identical parameter block (LaunchParams.array)."""
    UNMODIFIED, NOBN, CANDIDATE = 0, 1, 2

    def __init__(self):
        self.replay = replaying()
        if self.replay:
            self.lib = _NoLibrary()
            self._loaded = False
            return
        if not available():
            raise RuntimeError("oracle/_ref is not built (run `make -C oracle ref REF=<reference tree>`)")
        self.lib = C.CDLL(LIB)
        L = self.lib
        L.vptref_load_kernel.argtypes = [C.c_char_p, C.c_int]; L.vptref_load_kernel.restype = C.c_int
        L.vptref_load_bn_kernel.argtypes = [C.c_char_p]; L.vptref_load_bn_kernel.restype = C.c_int
        L.vptref_launch.argtypes = [C.POINTER(C.c_void_p), C.c_uint, C.c_uint, C.c_int, C.c_int]; L.vptref_launch.restype = C.c_int
        L.vptref_bn_advance.argtypes = [C.c_void_p, C.c_int, C.c_uint]; L.vptref_bn_advance.restype = C.c_int
        L.vptref_build_octree.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]; L.vptref_build_octree.restype = C.c_int
        L.vptref_build_bvh.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_float)]
        L.vptref_build_bvh.restype = C.c_int
        L.vptref_fill_volume.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int]; L.vptref_fill_volume.restype = C.c_int
        L.vptref_sizes.argtypes = [C.POINTER(C.c_size_t), C.c_int]; L.vptref_sizes.restype = C.c_int
        L.vptref_update_camera.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, C.c_float]
        L.vptref_bounds.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        L.vptref_instance_xform.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.POINTER(C.c_float)]
        L.vptref_atmosphere_init.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]
        L.vptref_atmosphere_init.restype = C.c_int
        L.vptref_atmosphere_stage.argtypes = [C.c_char_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_float), C.c_int]
        L.vptref_atmosphere_stage.restype = C.c_int
        self._loaded = False

    def atmosphere_init(self, atmos, use_constant_solar_spectrum=True, use_ozone=True, luminance=0, white_balance=True, exposure=1.0):
        """Run the reference's own Bruneton precompute (atmosphere::init, defaults of main.cpp:1433-1436) and
        write the resulting AtmosphereParameters (scalars + the four look-up textures) into `atmos` in place.
        Replaying: the stored scalars, with the look-up textures of this library's precompute of the same model (the tables
        themselves are not stored: a test that compares tables needs the reference build)."""
        assert C.sizeof(atmos) == 464
        key = (bool(use_constant_solar_spectrum), bool(use_ozone), int(luminance), bool(white_balance), float(exposure))
        skey, digest = _key("atmosphere"), _digest(key)
        if self.replay:
            import vpt_b200 as V
            if key not in _ATMO_CACHE:
                _ATMO_CACHE[key] = V.Atmosphere(use_constant_solar_spectrum=key[0], use_ozone=key[1], luminance=key[2],
                                                white_balance=key[3], exposure=key[4])
            own = _ATMO_CACHE[key].params
            C.memmove(C.byref(atmos), _load(skey, digest)["params"].tobytes(), 464)
            for name in _ATMO_TABLES:
                setattr(atmos, name, getattr(own, name))
            return
        if not os.path.exists(os.path.join(REF_DIR, "atmo", "atmosphere_kernels.ptx")):
            raise RuntimeError("oracle/_ref/atmo is not built")
        if key not in _ATMO_CACHE:                       # one precompute per model per process (the textures stay alive)
            buf = (C.c_ubyte * 464)()
            rc = self.lib.vptref_atmosphere_init(os.path.join(REF_DIR, "atmo").encode(), int(key[0]), int(key[1]),
                                                 key[2], int(key[3]), key[4], C.cast(buf, C.c_void_p))
            if rc: raise RuntimeError(f"vptref_atmosphere_init -> {rc}")
            _ATMO_CACHE[key] = bytes(buf)
        C.memmove(C.byref(atmos), _ATMO_CACHE[key], 464)
        params = type(atmos).from_buffer_copy(_ATMO_CACHE[key])
        for name in _ATMO_TABLES + ("scratch_buffers",):
            f = getattr(type(atmos), name); C.memset(C.addressof(params) + f.offset, 0, f.size)
        _store(skey, dict(digest=np.array(digest), params=np.frombuffer(bytes(params), dtype=np.uint8)))

    def atmosphere_stage(self, stage, atmos, blend=0, lfr=(1, 0, 0, 0, 1, 0, 0, 0, 1), order=0):
        """One launch of the reference's own precompute kernel for `stage` (VPT_BRUNETON_* numbering) on the buffers that
        `atmos.scratch_buffers` points to, with atmosphere::precompute's launch shape and argument bytes.  `lfr`: the
        luminance-from-radiance matrix, row-major.  Needs the reference build (no stored outputs: the inputs are device tables)."""
        assert C.sizeof(atmos) == 464
        m = (C.c_float * 9)(*[float(v) for v in lfr])
        rc = self.lib.vptref_atmosphere_stage(os.path.join(REF_DIR, "atmo").encode(), int(stage), C.cast(C.byref(atmos), C.c_void_p),
                                              int(blend), m, int(order))
        if rc: raise RuntimeError(f"vptref_atmosphere_stage({stage}) -> {rc}")

    def fill_volume(self, d_buffer_ptr, dims, scale=0.1, noise_type=0):
        """The reference's fill_volume_buffer into a device buffer of dims[0]*dims[1]*dims[2] floats."""
        from cuda.bindings import runtime as rt
        key, digest = _key("fill"), _digest(tuple(int(d) for d in dims), float(scale), int(noise_type))
        n = int(dims[0]) * int(dims[1]) * int(dims[2])
        if self.replay:
            src = torch.from_numpy(_load(key, digest)["dense"]).cuda()
            rt.cudaMemcpy(d_buffer_ptr, src.data_ptr(), 4 * n, rt.cudaMemcpyKind.cudaMemcpyDeviceToDevice)
            torch.cuda.synchronize()
            return
        p = os.path.join(REF_DIR, "texture_kernels_ref.cubin")
        rc = self.lib.vptref_fill_volume(p.encode(), C.c_void_p(d_buffer_ptr), int(dims[0]), int(dims[1]), int(dims[2]), float(scale), int(noise_type))
        if rc: raise RuntimeError(f"vptref_fill_volume -> {rc}")
        if RECORD_DIR:
            out = torch.empty(n, dtype=torch.float32, device="cuda")
            rt.cudaMemcpy(out.data_ptr(), d_buffer_ptr, 4 * n, rt.cudaMemcpyKind.cudaMemcpyDeviceToDevice)
            torch.cuda.synchronize()
            _store(key, dict(digest=np.array(digest), dense=out.cpu().numpy()))

    def instance_xform(self, base, pos, quat, scale):
        """The reference's instance transform (mat4 algebra of its .ins loader) as a 4x4 float32 array."""
        import vpt_b200 as V
        base, pos, quat = (np.asarray(a, dtype=np.float32) for a in (base, pos, quat))
        key, digest = _key("xform"), _digest(base.tobytes(), pos.tobytes(), quat.tobytes(), float(scale))
        if self.replay:
            return _load(key, digest)["m"]
        out = (C.c_float * 16)()
        self.lib.vptref_instance_xform(V._native.fvec(base.reshape(-1)), V._native.fvec(pos), V._native.fvec(quat), float(scale), out)
        m = np.array(list(out), dtype=np.float32).reshape(4, 4)
        _store(key, dict(digest=np.array(digest), m=m))
        return m

    def load_kernels(self):
        if self._loaded or self.replay:
            return
        for which, name in ((0, "render_kernel_ref.cubin"), (1, "render_kernel_ref_nobn.cubin")):
            rc = self.lib.vptref_load_kernel(os.path.join(REF_DIR, name).encode(), which)
            if rc: raise RuntimeError(f"vptref_load_kernel({name}) -> {rc}")
        rc = self.lib.vptref_load_bn_kernel(os.path.join(REF_DIR, "bn_advance_ref.cubin").encode())
        if rc: raise RuntimeError(f"vptref_load_bn_kernel -> {rc}")
        self._loaded = True

    def load_candidate(self, cubin_path):
        """Load another module through the reference loader sequence (cuModuleLoad + cuModuleGetFunction("volume_rt_kernel")).
        Replaying: the same two Driver-API calls through vpt_b200.LevelAModule."""
        if self.replay:
            import vpt_b200 as V
            self._candidate = V.LevelAModule(os.fspath(cubin_path))
            return
        rc = self.lib.vptref_load_kernel(os.fspath(cubin_path).encode(), self.CANDIDATE)
        if rc: raise RuntimeError(f"vptref_load_kernel({cubin_path}) -> {rc}")

    def sizes(self):
        out = (C.c_size_t * 12)(); n = self.lib.vptref_sizes(out, 12)
        return list(out)[:n]

    def build_octree(self, h_volumes, n):
        """Reference octree (device heap).  Returns the device root pointer.  Replaying: the same pointer-linked layout
        built by this library (node for node equal to the reference's: octree_nodes / test_scale_gpu check it)."""
        if self.replay:
            import vpt_b200 as V
            root = C.c_uint64(0)
            V._native.check(V.lib.vpt_octree_build(C.cast(h_volumes, C.POINTER(V.GPU_VDB)), n, C.byref(root)), None, "vpt_octree_build")
            return root.value
        root = C.c_void_p(0)
        rc = self.lib.vptref_build_octree(C.cast(h_volumes, C.c_void_p), n, C.byref(root))
        if rc: raise RuntimeError(f"vptref_build_octree -> {rc}")
        return root.value

    def octree_nodes(self, h_volumes, n):
        """{node number: OCTNode} of the reference builder's octree for these instances."""
        import vpt_b200 as V
        key, digest = _key("octree"), _digest(_volumes_digest(h_volumes, n), n)
        if self.replay:
            z = _load(key, digest)
            return {int(j): V.OCTNode.from_buffer_copy(z["nodes"][i].tobytes()) for i, j in enumerate(z["index"])}
        nodes = (V.OCTNode * 585)(); ex = (C.c_int * 585)()
        V._native.check(V.lib.vpt_octree_read(self.build_octree(h_volumes, n), nodes, ex), None, "vpt_octree_read")
        out = {j: nodes[j] for j in range(585) if ex[j]}
        idx = np.array(sorted(out), dtype=np.int32)
        _store(key, dict(digest=np.array(digest), index=idx,
                         nodes=np.stack([np.frombuffer(bytes(out[j]), dtype=np.uint8) for j in idx]) if len(idx) else np.zeros((0, C.sizeof(V.OCTNode)), np.uint8)))
        return out

    def bvh(self, h_volumes, n):
        """The reference BuildBVH for these instances: (scene bounds, vpt_b200.read_bvh view of nodes and leaves)."""
        import vpt_b200 as V
        key, digest = _key("bvh"), _digest(_volumes_digest(h_volumes, n), n)
        if self.replay:
            z = _load(key, digest)
            out = json.loads(str(z["bvh"]))
            for part in ("nodes", "leaves"):
                for e in out[part]: e["box"] = bytes.fromhex(e["box"])
            return [float(x) for x in z["bounds"]], out
        dn, dl = C.c_void_p(0), C.c_void_p(0); sb = (C.c_float * 6)()
        rc = self.lib.vptref_build_bvh(C.cast(h_volumes, C.c_void_p), n, C.byref(dn), C.byref(dl), sb)
        if rc: raise RuntimeError(f"vptref_build_bvh -> {rc}")
        out = V.read_bvh(dn.value, dl.value, n)
        enc = {part: [dict(e, box=e["box"].hex()) for e in out[part]] for part in ("nodes", "leaves")}
        _store(key, dict(digest=np.array(digest), bounds=np.array(list(sb), dtype=np.float32), bvh=np.array(json.dumps(enc))))
        return list(sb), out

    def launch(self, params_array, width, height, which=NOBN, sync=True):
        """One progressive pass exactly as main.cpp:1823-1829 issues it (caller bumps kp.iteration)."""
        if self.replay and which == self.CANDIDATE:
            c = self._candidate
            err, = c.drv.cuLaunchKernel(c.fn, int(width) // 16 + 1, int(height) // 16 + 1, 1, 16, 16, 1, 0, 0, C.addressof(params_array), 0)
            if int(err): raise RuntimeError(f"cuLaunchKernel(volume_rt_kernel) -> {err}")
            if sync: torch.cuda.synchronize()
            return
        self.load_kernels()
        rc = self.lib.vptref_launch(params_array, width, height, which, 1 if sync else 0)
        if rc: raise RuntimeError(f"vptref_launch -> {rc}")

    def bn_advance(self, kp, sync=True):
        """The reference's own update statements for the entries a pass really advances: min(W*H, 65536)."""
        self.load_kernels()
        rc = self.lib.vptref_bn_advance(C.cast(C.byref(kp), C.c_void_p), 1 if sync else 0, min(int(kp.resolution.x) * int(kp.resolution.y), 65536))
        if rc: raise RuntimeError(f"vptref_bn_advance -> {rc}")

    def render(self, renderer, n_passes, race_free=True, full=False):
        """Run n reference passes on `renderer`'s parameter block and buffers (race-free protocol: the
        'nobn' build + the reference's own blue-noise statements as a separate launch, SURVEY 8(c)).
        Replaying: accum, depth, display, the transmittance channel of raw and the blue-noise entries the passes changed
        come from the stored output; the colour channels of raw, which no test compares with the oracle's, are left at zero.
        full=True (for calls that start from non-zero buffers): the starting contents of accum, depth and cost are part of the
        inputs' hash, and cost and all four channels of raw are stored and replayed too."""
        key = _key("render")
        b = renderer.buffers
        start = (b.accum.cpu().numpy().tobytes(), b.depth.cpu().numpy().tobytes(), b.cost.cpu().numpy().tobytes()) if full else ()
        digest = _digest(bytes(renderer.cam), _kp_scalars(renderer.kp), renderer.width, renderer.height, int(n_passes), bool(race_free),
                         _volumes_digest(renderer.scene.h_volumes, len(renderer.scene.instances)), *start)
        bn = renderer.scene.d_blue_noise
        if self.replay:
            z = _load(key, digest)
            b.accum.copy_(torch.from_numpy(z["accum"])); b.depth.copy_(torch.from_numpy(z["depth"]))
            b.display.copy_(torch.from_numpy(z["display"]))
            if full:
                b.cost.copy_(torch.from_numpy(z["cost"])); b.raw.copy_(torch.from_numpy(z["raw"]))
            else:
                b.raw.zero_(); b.raw[:, 3].copy_(torch.from_numpy(z["raw_w"]))
            flat = bn.view(bn.shape[0], -1)
            flat[torch.from_numpy(z["bn_index"]).long().to(bn.device)] = torch.from_numpy(z["bn_value"]).to(bn.device)
            renderer.kp.iteration += int(n_passes)
            torch.cuda.synchronize()
            return
        bn0 = bn.clone() if RECORD_DIR else None
        for _ in range(n_passes):
            if race_free:
                self.launch(renderer.params.array, renderer.width, renderer.height, self.NOBN)
                self.bn_advance(renderer.kp)
            else:
                self.launch(renderer.params.array, renderer.width, renderer.height, self.UNMODIFIED)
            renderer.kp.iteration += 1
        torch.cuda.synchronize()
        if RECORD_DIR:
            flat, flat0 = bn.view(bn.shape[0], -1), bn0.view(bn0.shape[0], -1)
            changed = torch.nonzero((flat != flat0).any(dim=1)).flatten()
            out = dict(digest=np.array(digest), accum=b.accum.cpu().numpy(), depth=b.depth.cpu().numpy(), display=b.display.cpu().numpy(),
                       bn_index=changed.cpu().numpy().astype(np.int32), bn_value=flat[changed].cpu().numpy())
            if full: out.update(cost=b.cost.cpu().numpy(), raw=b.raw.cpu().numpy())
            else: out.update(raw_w=b.raw[:, 3].contiguous().cpu().numpy())
            _store(key, out)


if __name__ == "__main__":
    import sys
    pack(sys.argv[1], first=int(sys.argv[2]) if len(sys.argv) > 2 else 0)
