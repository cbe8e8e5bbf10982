"""Render loop on top of the C ABI: the headless counterpart of the reference frame loop
(source/main.cpp:1527-1860) -- fill Kernel_params, issue passes, keep `iteration`.

`Renderer.render_pass()` is one reference launch (`vpt_render_pass`); `Renderer.render(n)` is n of them
fused (`vpt_render_passes`).  `DistributedRenderer` shards the frame by interleaved row stripes over the
ranks of a torch.distributed job, replicates the scene, and all-gathers the rank-local accumulators
(one NCCL all-gather per call) before un-permuting them into a full frame.
"""
import ctypes as C
import json

import numpy as np
import torch

from . import _native as N
from ._native import lib, check
from .scene import Scene, default_kernel_params


# the light groups of vpt_set_light_group_buffers, in its argument order
LIGHT_GROUPS = ("sun", "point", "emission", "environment")


class FrameBuffers:
    """accum/cost (float3), depth (float), raw (float4), display (uint32) for `n_pixels` pixels; alpha (float) and volume (float3),
    the compositing AOVs, once Renderer.enable_aovs() has allocated them (None until then); `groups`, the light groups (name -> float3
    tensor, LIGHT_GROUPS order), once Renderer.enable_light_groups() has allocated them (None until then); `deep`, the deep slices
    ((K, n, 4) float32), once Renderer.enable_deep() has allocated them (None until then); `mattes`, the instance mattes ((K, n, 4) float32),
    once Renderer.enable_mattes() has allocated them (None until then); `motion`, the motion vectors ((n, 3) float32: the means of c vx,
    c vy and c), once Renderer.enable_motion_vectors() has allocated them (None until then); `position` ((n, 4): the means of c P and c),
    `normal` and `albedo` ((n, 3): the means of c n and c a), the collision AOVs, once Renderer.enable_collision_aovs() has allocated them
    (None until then); `crypto`, the Cryptomatte state ((2 + 2 S) * n int32 words, plane-major), once Renderer.enable_cryptomatte() has
    allocated it (None until then)."""

    def __init__(self, n_pixels, device):
        self.n = int(n_pixels)
        self.accum = torch.zeros(self.n, 3, dtype=torch.float32, device=device)
        self.cost = torch.zeros(self.n, 3, dtype=torch.float32, device=device)
        self.depth = torch.zeros(self.n, dtype=torch.float32, device=device)
        self.raw = torch.zeros(self.n, 4, dtype=torch.float32, device=device)
        self.display = torch.zeros(self.n, dtype=torch.int32, device=device)
        self.alpha = None
        self.volume = None
        self.groups = None
        self.deep = None
        self.mattes = None
        self.motion = None
        self.position = None
        self.normal = None
        self.albedo = None
        self.crypto = None

    def zero_(self):
        for t in (self.accum, self.cost, self.depth, self.raw, self.display, self.alpha, self.volume, self.deep, self.mattes, self.motion,
                  self.position, self.normal, self.albedo, self.crypto,
                  *(self.groups.values() if self.groups else ())):
            if t is not None:
                t.zero_()

    def bind(self, kp: N.Kernel_params):
        kp.accum_buffer = self.accum.data_ptr(); kp.cost_buffer = self.cost.data_ptr(); kp.depth_buffer = self.depth.data_ptr()
        kp.raw_buffer = self.raw.data_ptr(); kp.display_buffer = self.display.data_ptr()


class LaunchParams:
    """The `void* params[9]` array of main.cpp:1826, kept alive together with the values it points at."""

    def __init__(self, scene: Scene, cam: N.camera, kp: N.Kernel_params):
        self.cam, self.kp, self.scene = cam, kp, scene
        self.lights = scene.lights
        self.p_vol = C.c_uint64(scene.d_volumes.data_ptr())
        self.p_sphere = C.c_uint64(scene.d_sphere.data_ptr())
        self.p_geo = C.c_uint64(scene.d_geo_list.data_ptr())
        self.p_bvh = C.c_uint64(scene.bvh[0] if getattr(scene, "bvh", None) else scene.d_bvh.data_ptr())
        self.p_oct = C.c_uint64(scene.d_oct_root)
        self.atmos = scene.atmos
        self.array = (C.c_void_p * 9)(
            C.cast(C.byref(self.cam), C.c_void_p), C.cast(C.byref(self.lights), C.c_void_p),
            C.cast(C.byref(self.p_vol), C.c_void_p), C.cast(C.byref(self.p_sphere), C.c_void_p),
            C.cast(C.byref(self.p_geo), C.c_void_p), C.cast(C.byref(self.p_bvh), C.c_void_p),
            C.cast(C.byref(self.p_oct), C.c_void_p), C.cast(C.byref(self.atmos), C.c_void_p),
            C.cast(C.byref(self.kp), C.c_void_p))


class Renderer:
    def __init__(self, scene: Scene, width, height, cam: N.camera = None, kp: N.Kernel_params = None,
                 rank=0, n_ranks=1, stripe_rows=16, options=None):
        self.scene, self.width, self.height = scene, int(width), int(height)
        self.ctx = C.c_void_p(0)
        check(lib.vpt_create(C.byref(self.ctx)), None, "vpt_create")
        check(lib.vpt_set_partition(self.ctx, rank, n_ranks, stripe_rows), self.ctx, "vpt_set_partition")
        for k, v in (options or {}).items():
            check(lib.vpt_set_option(self.ctx, k.encode(), int(v)), self.ctx, f"vpt_set_option({k})")
        self.rank, self.n_ranks = rank, n_ranks
        self.n_local = int(lib.vpt_local_pixels(self.ctx, self.width, self.height))
        self.kp = kp if kp is not None else default_kernel_params()
        self.kp.resolution = N.u2(self.width, self.height)
        self.cam = cam if cam is not None else scene.frame_camera(self.width, self.height)
        self.buffers = FrameBuffers(self.n_local, scene.device)
        self.buffers.bind(self.kp)
        self.kp.blue_noise_buffer = scene.d_blue_noise.data_ptr()
        self.kp.emission_texture = scene.d_emission_lut.data_ptr()
        self.kp.density_color_texture = scene.d_density_color.data_ptr()
        if scene.env_tex is not None:
            self.kp.env_tex = scene.env_tex.tex
        self.params = LaunchParams(scene, self.cam, self.kp)

    # -- the reference frame loop body: launch, ++iteration --
    def render_pass(self, stream=None):
        check(lib.vpt_render_pass(self.ctx, self.params.array, C.c_void_p(stream or 0)), self.ctx, "vpt_render_pass")
        self.kp.iteration += 1

    def render(self, n_passes, stream=None):
        check(lib.vpt_render_passes(self.ctx, self.params.array, int(n_passes), C.c_void_p(stream or 0)), self.ctx, "vpt_render_passes")
        self.kp.iteration += int(n_passes)

    def render_adaptive(self, max_passes, threshold=0.01, min_passes=16, check_interval=16, error_map=False, stream=None):
        """One new frame (kp.iteration must be 0) of at most `max_passes` passes in which converged pixels stop early
        (vpt_render_adaptive).  Returns (passes_run, counts) or, with error_map=True, (passes_run, counts, rel_error): counts is the
        (H, W) int32 number of passes each pixel took, rel_error the (H, W) float32 relative error each pixel stopped with.  Every pixel
        holds what render(counts[pixel]) would have left in it.  The frame is final: render() cannot continue it.
        Partitioned (n_ranks > 1, peer-memory exchange active): this rank's share of the frame, counts and rel_error shaped
        (local_rows, W) in rank-local order (padding rows 0); every rank must make the same call, each from its own thread or process."""
        opt = N.adaptive_options(int(min_passes), int(check_interval), float(threshold))
        dev = self.buffers.accum.device
        counts = torch.empty(self.n_local, dtype=torch.int32, device=dev)
        err = torch.empty(self.n_local, dtype=torch.float32, device=dev) if error_map else None
        run = C.c_uint(0)
        check(lib.vpt_render_adaptive(self.ctx, self.params.array, int(max_passes), C.byref(opt), C.c_void_p(counts.data_ptr()),
                                      C.c_void_p(err.data_ptr()) if err is not None else None, C.byref(run), C.c_void_p(stream or 0)),
              self.ctx, "vpt_render_adaptive")
        self.kp.iteration += int(run.value)
        rows = self.n_local // self.width
        counts = counts.view(rows, self.width)
        return (int(run.value), counts, err.view(rows, self.width)) if error_map else (int(run.value), counts)

    def denoise(self, color=None, depth=True, rel_error=None, out=None, display=False, iterations=5, sigma_luminance=4.0,
                sigma_depth=0.2, stream=None):
        """Edge-avoiding a-trous filter of a full frame (vpt_denoise), enqueued on `stream`.  Returns the (H, W, 3) float32 result, or
        (result, display words (H, W) int32) with display=True, packed with kp.exposure_scale as k_resolve packs them.
        color: (H, W, 3) float32 HDR frame; None = this renderer's accumulator.  depth: True = this renderer's depth buffer, None / False =
        no depth term, or an (H, W) float32 tensor.  rel_error: the (H, W) error map of render_adaptive(..., error_map=True); None = the
        spatial noise estimate.  out: None = a new tensor, or any (H, W, 3) float32 tensor -- `color` itself denoises in place.
        On a partitioned renderer `color` must be given (a full frame, e.g. DistributedRenderer.full_accum()) and depth=True means none."""
        H, W = self.height, self.width
        if color is None:
            if self.n_ranks > 1:
                raise N.VptError("Renderer.denoise: a partitioned renderer holds no full frame; pass `color` (e.g. DistributedRenderer.full_accum())")
            color = self.buffers.accum
        if depth is True:
            depth = self.buffers.depth if self.n_ranks == 1 else None
        elif depth is False:
            depth = None
        dev = color.device
        color = _frame_tensor(color, H * W * 3, "color", dev)
        depth = _frame_tensor(depth, H * W, "depth", dev)
        rel_error = _frame_tensor(rel_error, H * W, "rel_error", dev)
        out = torch.empty(H, W, 3, dtype=torch.float32, device=dev) if out is None else _frame_tensor(out, H * W * 3, "out", dev)
        words = torch.empty(H, W, dtype=torch.int32, device=dev) if display else None
        opt = N.denoise_options(int(iterations), float(sigma_luminance), float(sigma_depth))
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(lib.vpt_denoise(self.ctx, W, H, ptr(color), ptr(depth), ptr(rel_error), C.byref(opt), float(self.kp.exposure_scale),
                              ptr(out), ptr(words), C.c_void_p(stream or 0)), self.ctx, "vpt_denoise")
        out = out.view(H, W, 3)
        return (out, words) if display else out

    def set_sample_offset(self, offset):
        """Draw pass p of a render call at kp.iteration = i from the Philox stream of iteration offset + i + p (vpt_set_sample_offset),
        from the next call with kp.iteration == 0 on.  Every other use of the iteration keeps kp.iteration.  0 is the reference stream."""
        check(lib.vpt_set_sample_offset(self.ctx, int(offset) & 0xFFFFFFFF), self.ctx, "vpt_set_sample_offset")

    def temporal(self, previous_cam: N.camera, color=None, vectors=None, history=None, history_len=None, max_history=None, clip_sigma=None,
                 display=False, out=None, out_len=None, stream=None):
        """Temporal accumulation of a full frame (vpt_temporal), enqueued on `stream`: blends `color` into the history carried along each
        pixel's motion from this renderer's camera to `previous_cam`.  Returns (out (H, W, 3), out_len (H, W)) float32, plus the display
        words (H, W) int32 with display=True (packed with kp.exposure_scale).  color: None = this renderer's accumulator; vectors: None =
        buffers.motion (rendered with target = previous_cam); history / history_len: the previous call's out / out_len, both None = no
        history.  max_history / clip_sigma: None = the library's defaults (clip_sigma = inf: no clip).  out / out_len: None = new
        tensors, or tensors to write (they may not overlap any input).  On a partitioned renderer pass full frames."""
        H, W = self.height, self.width
        if color is None:
            if self.n_ranks > 1:
                raise N.VptError("Renderer.temporal: a partitioned renderer holds no full frame; pass `color` and `vectors`")
            color = self.buffers.accum
        if vectors is None:
            if self.buffers.motion is None or self.n_ranks > 1:
                raise N.VptError("Renderer.temporal: no motion vectors (Renderer.enable_motion_vectors(previous_cam)) and none passed")
            vectors = self.buffers.motion
        dev = color.device
        color = _frame_tensor(color, H * W * 3, "color", dev)
        vectors = _frame_tensor(vectors, H * W * 3, "vectors", dev)
        history = _frame_tensor(history, H * W * 3, "history", dev)
        history_len = _frame_tensor(history_len, H * W, "history_len", dev)
        out = torch.empty(H, W, 3, dtype=torch.float32, device=dev) if out is None else _frame_tensor(out, H * W * 3, "out", dev)
        out_len = torch.empty(H, W, dtype=torch.float32, device=dev) if out_len is None else _frame_tensor(out_len, H * W, "out_len", dev)
        words = torch.empty(H, W, dtype=torch.int32, device=dev) if display else None
        opt = N.temporal_options()
        lib.vpt_temporal_options_defaults(C.byref(opt))
        if max_history is not None: opt.max_history = int(max_history)
        if clip_sigma is not None: opt.clip_sigma = float(clip_sigma)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(lib.vpt_temporal(self.ctx, W, H, ptr(color), ptr(vectors), C.byref(self.cam), C.byref(previous_cam), ptr(history), ptr(history_len),
                               C.byref(opt), float(self.kp.exposure_scale), ptr(out), ptr(out_len), ptr(words), C.c_void_p(stream or 0)),
              self.ctx, "vpt_temporal")
        out, out_len = out.view(H, W, 3), out_len.view(H, W)
        return (out, out_len, words) if display else (out, out_len)

    def enable_temporal(self, max_history=None, clip_sigma=None, layers=()):
        """Start temporal accumulation for render_temporal(): a viewer loop that restarts every frame at kp.iteration = 0 keeps converging
        while the camera moves.  Allocates the motion vectors and two history buffers; the next render_temporal() has no history.
        max_history / clip_sigma: vpt_temporal's options (None = the library's defaults).  layers: names of Renderer.temporal_layers
        (e.g. ("alpha", "volume", *LIGHT_GROUPS)), each of which must be enabled; every frame then blends them with the beauty's taps
        (vpt_temporal_layers) into two history buffers of their own, read by temporal_layer_images().  One context only (n_ranks == 1)."""
        if self.n_ranks > 1:
            raise N.VptError("Renderer.enable_temporal: one context only; a partitioned frame calls Renderer.temporal on full frames")
        names = tuple(layers)
        for name in names:
            if name not in _TEMPORAL_LAYERS:
                raise N.VptError(f"Renderer.enable_temporal: unknown layer {name!r} (one of {', '.join(_TEMPORAL_LAYERS)})")
            self._layer_buffer(name, "Renderer.enable_temporal")
        dev = self.buffers.accum.device
        self.buffers.motion = torch.zeros(self.n_local, 3, dtype=torch.float32, device=dev)
        n = self.width * self.height
        self._temporal = {"max_history": max_history, "clip_sigma": clip_sigma, "passes": 0, "prev_cam": None, "size": None, "k": 0,
                          "out": [torch.empty(n * 3, dtype=torch.float32, device=dev) for _ in range(2)],
                          "len": [torch.empty(n, dtype=torch.float32, device=dev) for _ in range(2)],
                          "layers": {name: [torch.empty(self._temporal_layer_shape(name), dtype=torch.float32, device=dev) for _ in range(2)]
                                     for name in names}}

    def render_temporal(self, cam: N.camera, n_passes, display=False):
        """One frame of a moving camera: n_passes passes from kp.iteration = 0 with camera `cam`, filtered against the previous frame's
        output (Renderer.temporal).  In order: the motion vectors target the previous frame's camera, the sample offset is the number of
        passes rendered since enable_temporal() (so every frame draws new samples), the frame renders, the filter blends it into the
        history, and the output becomes the next frame's history.  The first frame after enable_temporal() has no history, and neither
        has one after a change of resolution.  Returns Renderer.temporal's result; buffers.accum holds the unfiltered frame."""
        st = getattr(self, "_temporal", None)
        if st is None:
            raise N.VptError("Renderer.render_temporal: temporal accumulation is not enabled (Renderer.enable_temporal())")
        size = (self.width, self.height)
        have = st["prev_cam"] is not None and st["size"] == size
        prev = st["prev_cam"] if have else cam
        check(lib.vpt_set_motion_vectors(self.ctx, C.c_void_p(self.buffers.motion.data_ptr()), C.byref(prev)), self.ctx, "vpt_set_motion_vectors")
        self.set_sample_offset(st["passes"])
        C.memmove(C.byref(self.cam), C.byref(cam), C.sizeof(self.cam))
        self.kp.iteration = 0
        self.render(n_passes)
        k = st["k"]
        kw = dict(history=st["out"][k ^ 1] if have else None, history_len=st["len"][k ^ 1] if have else None, max_history=st["max_history"],
                  clip_sigma=st["clip_sigma"], display=display)
        if st["layers"]:
            lay = self.temporal_layers(prev, tuple(st["layers"]), layer_history={n: b[k ^ 1] for n, b in st["layers"].items()} if have else None,
                                       out={"beauty": st["out"][k], "len": st["len"][k], **{n: b[k] for n, b in st["layers"].items()}}, **kw)
            res = (lay["beauty"], lay["len"], lay["display"]) if display else (lay["beauty"], lay["len"])
        else:
            res = self.temporal(prev, out=st["out"][k], out_len=st["len"][k], **kw)
        st["passes"] += int(n_passes)
        st["prev_cam"] = type(cam).from_buffer_copy(cam)
        st["size"] = size
        st["k"] = k ^ 1
        return res

    def temporal_layer_images(self):
        """The layers enable_temporal(layers=...) named, as the last render_temporal() filtered them: a dict of views of the history
        buffers in Renderer.temporal_layers' shapes (the next render_temporal() overwrites the other buffer, not these)."""
        st = getattr(self, "_temporal", None)
        if st is None:
            raise N.VptError("Renderer.temporal_layer_images: temporal accumulation is not enabled (Renderer.enable_temporal())")
        if st["prev_cam"] is None:
            raise N.VptError("Renderer.temporal_layer_images: no frame rendered since enable_temporal()")
        return {name: b[st["k"] ^ 1] for name, b in st["layers"].items()}

    def disable_temporal(self):
        """Stop temporal accumulation: drops the history, turns the motion vectors off and sets the sample offset back to 0 (from the next
        call with kp.iteration == 0 on)."""
        self._temporal = None
        self.disable_motion_vectors()
        self.set_sample_offset(0)

    def temporal_layers(self, previous_cam: N.camera, layers, layer_history=None, color=None, vectors=None, history=None, history_len=None,
                        max_history=None, clip_sigma=None, display=False, stream=None, out=None):
        """Renderer.temporal of `color` together with layers blended with the beauty's own taps and history length (vpt_temporal_layers),
        so the filtered layers still add up to the filtered frame (DESIGN.md section 8r).  Returns a dict: "beauty" (H, W, 3) and "len"
        (H, W), equal bit for bit to Renderer.temporal with the same arguments, "display" with display=True, and one entry per layer:
        "alpha" (H, W); "volume", each name of LIGHT_GROUPS, "normal" and "albedo" (H, W, 3); "position" (H, W, 4); "deep" and "mattes"
        (K, H, W, 4).
        layers: an iterable of those names, taken from this renderer's buffers (they must be enabled), or a dict mapping names to full-frame
        tensors of those shapes (a partitioned renderer must pass a dict).  layer_history: a dict of the previous call's layer outputs by
        name, given exactly when `history` is.  The other arguments are Renderer.temporal's.  out: None = new tensors, or a dict of tensors
        to write for "beauty", "len" and every layer (none may overlap an input or another output)."""
        H, W = self.height, self.width
        if color is None:
            if self.n_ranks > 1:
                raise N.VptError("Renderer.temporal_layers: a partitioned renderer holds no full frame; pass `color` and `vectors`")
            color = self.buffers.accum
        if vectors is None:
            if self.buffers.motion is None or self.n_ranks > 1:
                raise N.VptError("Renderer.temporal_layers: no motion vectors (Renderer.enable_motion_vectors(previous_cam)) and none passed")
            vectors = self.buffers.motion
        if (layer_history is None) != (history is None):
            raise N.VptError("Renderer.temporal_layers: layer_history must be given exactly when history is")
        dev = color.device
        color = _frame_tensor(color, H * W * 3, "color", dev)
        vectors = _frame_tensor(vectors, H * W * 3, "vectors", dev)
        history = _frame_tensor(history, H * W * 3, "history", dev)
        history_len = _frame_tensor(history_len, H * W, "history_len", dev)
        named = dict(layers) if isinstance(layers, dict) else {name: None for name in layers}
        if len(named) > N.VPT_TEMPORAL_MAX_LAYERS:
            raise N.VptError(f"Renderer.temporal_layers: {len(named)} layers (at most {N.VPT_TEMPORAL_MAX_LAYERS})")
        out = dict(out or {})
        res = {"beauty": out.get("beauty"), "len": out.get("len")}
        res["beauty"] = torch.empty(H, W, 3, dtype=torch.float32, device=dev) if res["beauty"] is None else \
            _frame_tensor(res["beauty"], H * W * 3, "out beauty", dev)
        res["len"] = torch.empty(H, W, dtype=torch.float32, device=dev) if res["len"] is None else _frame_tensor(res["len"], H * W, "out len", dev)
        if display:
            res["display"] = torch.empty(H, W, dtype=torch.int32, device=dev)
        descs = (N.temporal_layer * max(1, len(named)))()
        for i, (name, t) in enumerate(named.items()):
            if name not in _TEMPORAL_LAYERS:
                raise N.VptError(f"Renderer.temporal_layers: unknown layer {name!r} (one of {', '.join(_TEMPORAL_LAYERS)})")
            if t is None:
                if self.n_ranks > 1:
                    raise N.VptError(f"Renderer.temporal_layers: a partitioned renderer holds no full frame of {name!r}; pass a dict of "
                                     "full-frame tensors")
                t = self._layer_buffer(name, "Renderer.temporal_layers")
            k = t.shape[0] if name in ("deep", "mattes") else 1
            ch = _TEMPORAL_LAYERS[name]
            t = _frame_tensor(t, k * H * W * ch, name, dev)
            hist = None
            if layer_history is not None:
                if name not in layer_history:
                    raise N.VptError(f"Renderer.temporal_layers: layer_history has no {name!r}")
                hist = _frame_tensor(layer_history[name], k * H * W * ch, f"{name} history", dev)
            shape = self._temporal_layer_shape(name, k)
            dst = torch.empty(shape, dtype=torch.float32, device=dev) if out.get(name) is None else \
                _frame_tensor(out[name], k * H * W * ch, f"out {name}", dev).view(shape)
            res[name] = dst
            descs[i] = N.temporal_layer(t.data_ptr(), hist.data_ptr() if hist is not None else None, dst.data_ptr(), ch, k)
        opt = N.temporal_options()
        lib.vpt_temporal_options_defaults(C.byref(opt))
        if max_history is not None: opt.max_history = int(max_history)
        if clip_sigma is not None: opt.clip_sigma = float(clip_sigma)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(lib.vpt_temporal_layers(self.ctx, W, H, ptr(color), ptr(vectors), C.byref(self.cam), C.byref(previous_cam), ptr(history),
                                      ptr(history_len), C.byref(opt), float(self.kp.exposure_scale), ptr(res["beauty"]), ptr(res["len"]),
                                      ptr(res.get("display")), descs, len(named), C.c_void_p(stream or 0)), self.ctx, "vpt_temporal_layers")
        res["beauty"], res["len"] = res["beauty"].view(H, W, 3), res["len"].view(H, W)
        return res

    def _temporal_layer_shape(self, name, k=None):
        """The full-frame shape of layer `name` as Renderer.temporal_layers returns it (k: the planes of deep / mattes; None = this
        renderer's own)."""
        H, W, ch = self.height, self.width, _TEMPORAL_LAYERS[name]
        if name in ("deep", "mattes"):
            return (self._layer_buffer(name).shape[0] if k is None else k, H, W, ch)
        return (H, W) if ch == 1 else (H, W, ch)

    def denoise_layers(self, layers, color=None, depth=True, rel_error=None, iterations=5, sigma_luminance=4.0, sigma_depth=0.2,
                       stream=None, display=False):
        """Renderer.denoise of `color` together with layers filtered by the beauty's own weights (vpt_denoise_layers), so the denoised
        layers still add up to the denoised frame (DESIGN.md section 8n).  Returns a dict of new tensors: "beauty" (H, W, 3), equal bit
        for bit to Renderer.denoise with the same arguments, and one entry per layer: "alpha" (H, W); "volume" and each name of
        LIGHT_GROUPS (H, W, 3); "deep" and "mattes" (K, H, W, 4).
        layers: an iterable of those names, taken from this renderer's buffers (they must be enabled), or a dict mapping names to
        full-frame tensors of those shapes (a partitioned renderer must pass a dict, e.g. DistributedRenderer.denoise_layers does).
        color, depth, rel_error and the options are Renderer.denoise's; display=True adds "display", the (H, W) int32 display words
        Renderer.denoise(..., display=True) returns."""
        H, W = self.height, self.width
        if color is None:
            if self.n_ranks > 1:
                raise N.VptError("Renderer.denoise_layers: a partitioned renderer holds no full frame; pass `color` "
                                 "(e.g. DistributedRenderer.full_accum())")
            color = self.buffers.accum
        if depth is True:
            depth = self.buffers.depth if self.n_ranks == 1 else None
        elif depth is False:
            depth = None
        dev = color.device
        color = _frame_tensor(color, H * W * 3, "color", dev)
        depth = _frame_tensor(depth, H * W, "depth", dev)
        rel_error = _frame_tensor(rel_error, H * W, "rel_error", dev)
        if isinstance(layers, dict):
            named = dict(layers)
        else:
            named = {name: None for name in layers}
        srcs = {}
        for name, t in named.items():
            if name not in _DENOISE_LAYERS:
                raise N.VptError(f"Renderer.denoise_layers: unknown layer {name!r} (one of {', '.join(_DENOISE_LAYERS)})")
            if t is None:
                if self.n_ranks > 1:
                    raise N.VptError(f"Renderer.denoise_layers: a partitioned renderer holds no full frame of {name!r}; pass a dict of "
                                     "full-frame tensors (e.g. DistributedRenderer.denoise_layers)")
                t = self._layer_buffer(name)
            k = t.shape[0] if name in ("deep", "mattes") else 1
            ch = _DENOISE_LAYERS[name]
            srcs[name] = (_frame_tensor(t, k * H * W * ch, name, dev), ch, k)
        out = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
        words = torch.empty(H, W, dtype=torch.int32, device=dev) if display else None
        res = {"beauty": out, **({"display": words} if display else {})}
        descs = (N.denoise_layer * max(1, len(srcs)))()
        for i, (name, (t, ch, k)) in enumerate(srcs.items()):
            shape = (k, H, W, ch) if name in ("deep", "mattes") else (H, W) if ch == 1 else (H, W, ch)
            res[name] = torch.empty(shape, dtype=torch.float32, device=dev)
            descs[i] = N.denoise_layer(t.data_ptr(), res[name].data_ptr(), ch, k)
        opt = N.denoise_options(int(iterations), float(sigma_luminance), float(sigma_depth))
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(lib.vpt_denoise_layers(self.ctx, W, H, ptr(color), ptr(depth), ptr(rel_error), C.byref(opt), float(self.kp.exposure_scale),
                                     ptr(out), ptr(words), descs, len(srcs), C.c_void_p(stream or 0)), self.ctx, "vpt_denoise_layers")
        return res

    def _layer_buffer(self, name, caller="Renderer.denoise_layers"):
        """This renderer's own buffer of layer `name`, or VptError (naming `caller`) when it is not enabled."""
        b = self.buffers
        if name in ("alpha", "volume"):
            if getattr(b, name) is None:
                raise N.VptError(f"{caller}: layer {name!r} needs the AOVs (Renderer.enable_aovs())")
            return getattr(b, name)
        if name in LIGHT_GROUPS:
            if b.groups is None:
                raise N.VptError(f"{caller}: layer {name!r} needs the light groups (Renderer.enable_light_groups())")
            return b.groups[name]
        if name in ("position", "normal", "albedo"):
            if getattr(b, name) is None:
                raise N.VptError(f"{caller}: layer {name!r} needs the collision AOVs (Renderer.enable_collision_aovs())")
            return getattr(b, name)
        if name == "deep":
            if b.deep is None:
                raise N.VptError(f"{caller}: layer 'deep' needs the deep slices (Renderer.enable_deep(bounds))")
            return b.deep
        if b.mattes is None:
            raise N.VptError(f"{caller}: layer 'mattes' needs the instance mattes (Renderer.enable_mattes(sets))")
        return b.mattes

    def enable_aovs(self):
        """Allocate and register the compositing AOVs (vpt_set_aov_buffers): buffers.alpha (n,) float32, the running mean of the
        coverage [depth > 0], and buffers.volume (n, 3) float32, the volume's share of accum.  They take over at the next render call with
        kp.iteration == 0.  Under a constant environment of radiance k, accum = volume + (1 - alpha) * k up to rounding; a new plate P
        composites as volume + (1 - alpha) * P (DESIGN.md section 8c).  n is the renderer's local pixel count (rank-local rows on a partitioned renderer)."""
        dev = self.buffers.accum.device
        self.buffers.alpha = torch.zeros(self.n_local, dtype=torch.float32, device=dev)
        self.buffers.volume = torch.zeros(self.n_local, 3, dtype=torch.float32, device=dev)
        check(lib.vpt_set_aov_buffers(self.ctx, C.c_void_p(self.buffers.alpha.data_ptr()), C.c_void_p(self.buffers.volume.data_ptr())),
              self.ctx, "vpt_set_aov_buffers")

    def disable_aovs(self):
        """Turn the AOVs off at once; buffers.alpha / buffers.volume keep what they hold."""
        check(lib.vpt_set_aov_buffers(self.ctx, None, None), self.ctx, "vpt_set_aov_buffers")

    def alpha_image(self):
        """(H, W) float32 view of buffers.alpha ((local rows, W) on a partitioned renderer)."""
        if self.buffers.alpha is None:
            raise N.VptError("Renderer.alpha_image: AOVs are not enabled (Renderer.enable_aovs())")
        return self.buffers.alpha.view(self.n_local // self.width, self.width)

    def volume_image(self):
        """(H, W, 3) float32 view of buffers.volume ((local rows, W, 3) on a partitioned renderer)."""
        if self.buffers.volume is None:
            raise N.VptError("Renderer.volume_image: AOVs are not enabled (Renderer.enable_aovs())")
        return self.buffers.volume.view(self.n_local // self.width, self.width, 3)

    def enable_light_groups(self):
        """Allocate and register the light groups (vpt_set_light_group_buffers): buffers.groups[name] (n, 3) float32 for every name of
        LIGHT_GROUPS -- the running means of the radiance the sun, the point lights, the volume's emission and the environment added to
        each sample.  They take over at the next render call with kp.iteration == 0, and sum to accum up to the rounding of the separate
        sums (DESIGN.md section 8d).  n is the renderer's local pixel count (rank-local rows on a partitioned renderer)."""
        dev = self.buffers.accum.device
        self.buffers.groups = {name: torch.zeros(self.n_local, 3, dtype=torch.float32, device=dev) for name in LIGHT_GROUPS}
        ptrs = [C.c_void_p(self.buffers.groups[name].data_ptr()) for name in LIGHT_GROUPS]
        check(lib.vpt_set_light_group_buffers(self.ctx, *ptrs), self.ctx, "vpt_set_light_group_buffers")

    def disable_light_groups(self):
        """Turn the light groups off at once; buffers.groups keeps what it holds."""
        check(lib.vpt_set_light_group_buffers(self.ctx, None, None, None, None), self.ctx, "vpt_set_light_group_buffers")

    def light_group_image(self, name):
        """(H, W, 3) float32 view of light group `name` (one of LIGHT_GROUPS; (local rows, W, 3) on a partitioned renderer)."""
        if self.buffers.groups is None:
            raise N.VptError("Renderer.light_group_image: light groups are not enabled (Renderer.enable_light_groups())")
        if name not in self.buffers.groups:
            raise N.VptError(f"Renderer.light_group_image: unknown light group {name!r} (one of {', '.join(LIGHT_GROUPS)})")
        return self.buffers.groups[name].view(self.n_local // self.width, self.width, 3)

    def enable_deep(self, bounds):
        """Allocate and register the deep slices (vpt_set_deep_buffers): `bounds` z_0 < z_1 < ... < z_K (K = 1..VPT_DEEP_MAX_SLICES;
        z_K may be inf) are K depth intervals in the units of the depth buffer.  buffers.deep (K, n, 4) float32 holds per slice and pixel
        the running means (premultiplied colour, coverage) of the samples whose depth d has z_k <= d < z_{k+1}: the compositing AOVs binned
        by depth, so an element can be inserted at a depth inside the volume (deep.flatten).  They take over at the next render call with
        kp.iteration == 0 (DESIGN.md section 8h).  Bad bounds raise VptError and leave the slices as they were.  n is the renderer's
        local pixel count (rank-local rows on a partitioned renderer)."""
        z = np.asarray(bounds, dtype=np.float32).reshape(-1)
        k = len(z) - 1
        if not 1 <= k <= N.VPT_DEEP_MAX_SLICES:
            raise N.VptError(f"Renderer.enable_deep: {len(z)} bounds give {k} slices (1..{N.VPT_DEEP_MAX_SLICES})")
        deep = torch.zeros(k, self.n_local, 4, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_set_deep_buffers(self.ctx, C.c_void_p(deep.data_ptr()), k, z.ctypes.data_as(C.POINTER(C.c_float))),
              self.ctx, "vpt_set_deep_buffers")
        self.buffers.deep, self.deep_bounds = deep, tuple(float(v) for v in z)

    def disable_deep(self):
        """Turn the deep slices off at once; buffers.deep keeps what it holds."""
        check(lib.vpt_set_deep_buffers(self.ctx, None, 0, None), self.ctx, "vpt_set_deep_buffers")

    def deep_image(self):
        """(K, H, W, 4) float32 view of buffers.deep ((K, local rows, W, 4) on a partitioned renderer); the bounds are deep_bounds."""
        if self.buffers.deep is None:
            raise N.VptError("Renderer.deep_image: deep slices are not enabled (Renderer.enable_deep(bounds))")
        return self.buffers.deep.view(self.buffers.deep.shape[0], self.n_local // self.width, self.width, 4)

    def enable_mattes(self, sets, sphere=None):
        """Allocate and register the instance mattes (vpt_set_instance_mattes): `sets` is a list of K iterables of instance indices
        (K = 1..VPT_MATTE_MAX), matte k selecting the instances of sets[k]; `sphere` is the matte of the reference sphere (None: none).
        buffers.mattes (K, n, 4) float32 holds per matte and pixel the running means (premultiplied colour, coverage) of the samples whose
        camera ray collided first with an instance of the set: the compositing AOVs split by instance.  They take over at the next render
        call with kp.iteration == 0 (DESIGN.md section 8l).  An index in two sets, or outside the scene's instances, raises VptError and
        leaves the mattes as they were.  n is the renderer's local pixel count (rank-local rows on a partitioned renderer)."""
        sets = [sorted({int(i) for i in s}) for s in sets]
        k = len(sets)
        if not 1 <= k <= N.VPT_MATTE_MAX:
            raise N.VptError(f"Renderer.enable_mattes: {k} sets (1..{N.VPT_MATTE_MAX})")
        n_inst = len(self.scene.instances)
        matte_of = np.full(n_inst, -1, dtype=np.int32)
        for m, s in enumerate(sets):
            for i in s:
                if not 0 <= i < n_inst:
                    raise N.VptError(f"Renderer.enable_mattes: instance {i} of set {m} is outside the scene's {n_inst} instances")
                if matte_of[i] >= 0:
                    raise N.VptError(f"Renderer.enable_mattes: instance {i} is in set {int(matte_of[i])} and set {m}")
                matte_of[i] = m
        if sphere is not None and not 0 <= int(sphere) < k:
            raise N.VptError(f"Renderer.enable_mattes: sphere matte {sphere} is outside 0..{k - 1}")
        mattes = torch.zeros(k, self.n_local, 4, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_set_instance_mattes(self.ctx, C.c_void_p(mattes.data_ptr()), k, matte_of.ctypes.data_as(C.POINTER(C.c_int)), n_inst,
                                          -1 if sphere is None else int(sphere)), self.ctx, "vpt_set_instance_mattes")
        self.buffers.mattes, self.matte_sets = mattes, tuple(tuple(s) for s in sets)

    def disable_mattes(self):
        """Turn the instance mattes off at once; buffers.mattes keeps what it holds."""
        check(lib.vpt_set_instance_mattes(self.ctx, None, 0, None, 0, -1), self.ctx, "vpt_set_instance_mattes")

    def matte_image(self):
        """(K, H, W, 4) float32 view of buffers.mattes ((K, local rows, W, 4) on a partitioned renderer); the sets are matte_sets."""
        if self.buffers.mattes is None:
            raise N.VptError("Renderer.matte_image: instance mattes are not enabled (Renderer.enable_mattes(sets))")
        return self.buffers.mattes.view(self.buffers.mattes.shape[0], self.n_local // self.width, self.width, 4)

    def enable_motion_vectors(self, target_cam: N.camera):
        """Allocate and register the motion vectors (vpt_set_motion_vectors): buffers.motion (n, 3) float32 holds per pixel the running
        means of (c vx, c vy, c), c the coverage [depth > 0] and (vx, vy) the film motion in pixels of each sample's first collision from
        this renderer's camera to `target_cam` (e.g. the next frame's look_at camera; copied).  They take over at the next render call with
        kp.iteration == 0 (DESIGN.md section 8o).  A non-finite field of the target raises VptError and leaves the vectors as they were.
        n is the renderer's local pixel count (rank-local rows on a partitioned renderer)."""
        motion = torch.zeros(self.n_local, 3, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_set_motion_vectors(self.ctx, C.c_void_p(motion.data_ptr()), C.byref(target_cam)), self.ctx, "vpt_set_motion_vectors")
        self.buffers.motion = motion

    def disable_motion_vectors(self):
        """Turn the motion vectors off at once; buffers.motion keeps what it holds."""
        check(lib.vpt_set_motion_vectors(self.ctx, None, None), self.ctx, "vpt_set_motion_vectors")

    def motion_vector_image(self):
        """(vectors, coverage): (H, W, 2) float32 unpremultiplied vectors xy / z in pixels (0 where the coverage z is 0) and the (H, W)
        coverage z, which is the alpha AOV ((local rows, ...) on a partitioned renderer)."""
        if self.buffers.motion is None:
            raise N.VptError("Renderer.motion_vector_image: motion vectors are not enabled (Renderer.enable_motion_vectors(target_cam))")
        return unpremultiply_vectors(self.buffers.motion.view(self.n_local // self.width, self.width, 3))

    def voxel_edge(self):
        """The shortest world-space edge of one voxel of volume 0 (the length of the shortest of its xform's three index-axis columns)."""
        g = self.scene.instances[0]
        X = np.array([[g.xform[a][b] for b in range(4)] for a in range(4)], dtype=np.float64)
        return float(np.linalg.norm(X[:3, :3], axis=0).min())

    def enable_collision_aovs(self, position=True, normal=True, albedo=True, step=None):
        """Allocate and register the collision AOVs (vpt_set_collision_aovs): buffers.position (n, 4) float32 holds per pixel the running
        means of (c Px, c Py, c Pz, c), buffers.normal and buffers.albedo (n, 3) those of c n and c a, c the coverage [depth > 0] and P, n,
        a the world position, normal and albedo at each sample's first collision (DESIGN.md section 8q).  A layer passed as False stays None
        and is not kept.  step: the world step h of the density gradient's central differences; None = one voxel edge of volume 0 in world
        units (voxel_edge()).  They take over at the next render call with kp.iteration == 0.  A step that is not finite or <= 0 with the
        normal raises VptError and leaves the layers as they were.  n is the renderer's local pixel count."""
        dev = self.buffers.accum.device
        h = self.voxel_edge() if step is None else float(step)
        pos = torch.zeros(self.n_local, 4, dtype=torch.float32, device=dev) if position else None
        nrm = torch.zeros(self.n_local, 3, dtype=torch.float32, device=dev) if normal else None
        alb = torch.zeros(self.n_local, 3, dtype=torch.float32, device=dev) if albedo else None
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(lib.vpt_set_collision_aovs(self.ctx, ptr(pos), ptr(nrm), ptr(alb), h), self.ctx, "vpt_set_collision_aovs")
        self.buffers.position, self.buffers.normal, self.buffers.albedo = pos, nrm, alb

    def disable_collision_aovs(self):
        """Turn the collision AOVs off at once; the buffers keep what they hold."""
        check(lib.vpt_set_collision_aovs(self.ctx, None, None, None, 0.0), self.ctx, "vpt_set_collision_aovs")

    def collision_images(self):
        """(P, n, albedo, coverage): the (H, W, 3) float32 unpremultiplied world position, normal and albedo (each divided by the coverage,
        0 where it is 0; None for a layer not enabled) and the (H, W) coverage, which is the alpha AOV ((local rows, ...) on a partitioned
        renderer).  The normal is the mean of unit normals: normalise it for a unit vector."""
        b = self.buffers
        if b.position is None:
            raise N.VptError("Renderer.collision_images: no position layer, which holds the coverage (Renderer.enable_collision_aovs())")
        rows = self.n_local // self.width
        z = b.position[:, 3]
        cov = z > 0
        den = torch.where(cov, z, torch.ones_like(z)).unsqueeze(-1)
        def unpre(t, k):
            if t is None: return None
            return torch.where(cov.unsqueeze(-1), t[:, :k] / den, torch.zeros_like(t[:, :k])).view(rows, self.width, k)
        return unpre(b.position, 3), unpre(b.normal, 3), unpre(b.albedo, 3), z.view(rows, self.width)

    def enable_cryptomatte(self, capacity=16, names=None, sphere="sphere"):
        """Allocate and register the Cryptomatte (vpt_set_cryptomatte): buffers.crypto ((2 + 2 capacity) * n int32 words, read as uint32)
        keeps per pixel the passes counted, the overflow and up to `capacity` (id, count) entries of the instances its camera rays collided
        with first (DESIGN.md section 8s).  names: one per instance, the names the ids are hashed from (default: the scene's
        instance_names, else "instance<i>"); sphere: the sphere's name.  Duplicate names raise VptError.  The state takes over at the next
        render call with kp.iteration == 0.  n is the renderer's local pixel count (rank-local rows on a partitioned renderer)."""
        cap = int(capacity)
        if not 1 <= cap <= N.VPT_CRYPTO_MAX_ENTRIES:
            raise N.VptError(f"Renderer.enable_cryptomatte: capacity {cap} (1..{N.VPT_CRYPTO_MAX_ENTRIES})")
        n_inst = len(self.scene.instances)
        if names is None:
            names = getattr(self.scene, "instance_names", None) or [f"instance{i}" for i in range(n_inst)]
        names = [str(x) for x in names]
        if len(names) != n_inst:
            raise N.VptError(f"Renderer.enable_cryptomatte: {len(names)} names for {n_inst} instances")
        everything = names + [str(sphere)]
        if len(set(everything)) != len(everything):
            dup = sorted({x for x in everything if everything.count(x) > 1})
            raise N.VptError(f"Renderer.enable_cryptomatte: duplicate names {dup}")
        dev = self.buffers.accum.device
        state = torch.zeros((2 + 2 * cap) * self.n_local, dtype=torch.int32, device=dev)
        table = torch.tensor([cryptomatte_id(x)[0] for x in names], dtype=torch.float32, device=dev)
        check(lib.vpt_set_cryptomatte(self.ctx, C.c_void_p(state.data_ptr()), cap), self.ctx, "vpt_set_cryptomatte")
        self.buffers.crypto = state
        self.crypto_capacity, self.crypto_names, self.crypto_sphere, self.crypto_table = cap, names, str(sphere), table

    def disable_cryptomatte(self):
        """Turn the Cryptomatte off at once; buffers.crypto keeps what it holds."""
        check(lib.vpt_set_cryptomatte(self.ctx, None, 0), self.ctx, "vpt_set_cryptomatte")

    def _crypto_state(self, caller):
        if self.buffers.crypto is None:
            raise N.VptError(f"{caller}: the Cryptomatte is not enabled (Renderer.enable_cryptomatte())")
        return self.buffers.crypto

    def cryptomatte_state(self):
        """Views of buffers.crypto: {"n": (H, W), "overflow": (H, W), "ids": (S, H, W), "counts": (S, H, W)}, int32 holding the uint32 words
        (the sphere's id 0xffffffff reads as -1); (local rows, W) on a partitioned renderer."""
        s = self._crypto_state("Renderer.cryptomatte_state")
        rows, S = self.n_local // self.width, self.crypto_capacity
        planes = s.view(2 + 2 * S, rows, self.width)
        return {"n": planes[0], "overflow": planes[1], "ids": planes[2::2], "counts": planes[3::2]}

    def cryptomatte_image(self, ranks=6, overflow=False, stream=None):
        """(ranks / 2, H, W, 4) float32: the Cryptomatte ranks (vpt_cryptomatte_rank), rank r in plane r // 2 as (id float, coverage) at
        components 2 (r % 2), 2 (r % 2) + 1 -- the channels CryptoObject00.RGBA, CryptoObject01.RGBA, ... of the EXR layer.  overflow=True
        also returns the (H, W) overflow / n."""
        s = self._crypto_state("Renderer.cryptomatte_image")
        ranks = int(ranks)
        rows = self.n_local // self.width
        out = torch.empty(max(ranks // 2, 1), self.n_local, 4, dtype=torch.float32, device=s.device)
        ovf = torch.empty(self.n_local, dtype=torch.float32, device=s.device) if overflow else None
        sphere_id = cryptomatte_id(self.crypto_sphere)[0]
        check(lib.vpt_cryptomatte_rank(self.ctx, self.width, rows, C.c_void_p(s.data_ptr()), self.crypto_capacity,
                                       C.c_void_p(self.crypto_table.data_ptr()) if len(self.crypto_names) else None, len(self.crypto_names),
                                       sphere_id, ranks, C.c_void_p(out.data_ptr()), C.c_void_p(ovf.data_ptr()) if overflow else None,
                                       C.c_void_p(stream or 0)), self.ctx, "vpt_cryptomatte_rank")
        img = out.view(-1, rows, self.width, 4)
        return (img, ovf.view(rows, self.width)) if overflow else img

    def cryptomatte_manifest(self):
        """{name: "%08x" of its Cryptomatte float's bits} for every instance and the sphere"""
        if not hasattr(self, "crypto_names"):
            raise N.VptError("Renderer.cryptomatte_manifest: the Cryptomatte is not enabled (Renderer.enable_cryptomatte())")
        return {x: cryptomatte_id(x)[1] for x in self.crypto_names + [self.crypto_sphere]}

    def cryptomatte_metadata(self, layer="CryptoObject"):
        """The four EXR header attributes of the Cryptomatte layer `layer` (channels <layer>00.RGBA, <layer>01.RGBA, ... from
        cryptomatte_image()): cryptomatte/<key>/name, hash, conversion and manifest, <key> the first 7 hex digits of the layer name's hash."""
        key = "%08x" % int(lib.vpt_cryptomatte_hash(layer.encode("utf-8"), len(layer.encode("utf-8")), None))
        pre = f"cryptomatte/{key[:7]}/"
        return {pre + "name": layer, pre + "hash": "MurmurHash3_32", pre + "conversion": "uint32_to_float32",
                pre + "manifest": json.dumps(self.cryptomatte_manifest(), sort_keys=True)}

    def cryptomatte_matte(self, selection):
        """(H, W) float32 coverage of the instances in `selection` (names or indices; the sphere by its name or by VPT_CRYPTO_SPHERE): the
        sum of their counts over n, read from the full state (every entry, not the ranks); 0 where n == 0.  Entries lost to the overflow are
        not in it."""
        st = self.cryptomatte_state()
        index = {x: i for i, x in enumerate(self.crypto_names)}
        want = set()
        for x in selection:
            if isinstance(x, str):
                if x == self.crypto_sphere: want.add(N.VPT_CRYPTO_SPHERE)
                elif x in index: want.add(index[x])
                else: raise N.VptError(f"Renderer.cryptomatte_matte: no instance named {x!r}")
            else:
                want.add(int(x) & 0xFFFFFFFF)
        ids = st["ids"].long() & 0xFFFFFFFF
        counts = st["counts"].long() & 0xFFFFFFFF
        sel = torch.zeros_like(ids, dtype=torch.bool)
        for i in want:
            sel |= ids == i
        total = torch.where(sel & (counts > 0), counts, torch.zeros_like(counts)).sum(0).double()
        n = (st["n"].long() & 0xFFFFFFFF).double()
        return torch.where(n > 0, total / torch.where(n > 0, n, torch.ones_like(n)), torch.zeros_like(n)).float()

    def set_region(self, x0, y0, x1, y1):
        """Render only the full-frame pixels [x0, x1) x [y0, y1) (vpt_set_render_region) from the next call with kp.iteration == 0 on:
        inside it every buffer gets what a full-frame render gives there, bit for bit; outside it nothing is written, so the display keeps
        the last full frame there.  Set kp.iteration = 0 when the region moves (reset() also zeroes the buffers).  A bad rectangle is
        refused by that next render call."""
        check(lib.vpt_set_render_region(self.ctx, int(x0), int(y0), int(x1), int(y1)), self.ctx, "vpt_set_render_region")

    def clear_region(self):
        """Render the whole frame again from the next call with kp.iteration == 0 on."""
        check(lib.vpt_set_render_region(self.ctx, 0, 0, 0, 0), self.ctx, "vpt_set_render_region")

    def set_projection(self, kind, hfov=360.0, vfov=180.0, ipd=None, layout=None, pole_merge=None):
        """Camera projection (vpt_set_projection) from the next call with kp.iteration == 0 on: "perspective", the reference camera (the
        default), or "equirect", a latitude-longitude panorama of hfov x vfov degrees (hfov in (0, 360], vfov in (0, 180]) around the
        camera's origin, oriented by its u, v, w (forward -w).  "ods" (vpt_set_projection_ods) is the omni-directional stereo panorama of
        hfov x vfov per eye: interocular distance `ipd` in scene units (None: 0.064), layout "over_under" (left eye on top; the default),
        "left" or "right", and the eye separation merged to 0 between the |elevation| angles pole_merge = (from, to) in degrees (None:
        (60, 75); DESIGN.md section 8k).  A bad kind, field of view or ODS option, or an ODS option given with another kind, raises
        VptError here; a panorama with a lens (cam.lens_radius != 0) is refused by the render call, and so is an over-under frame of odd
        height."""
        kinds = {"perspective": N.VPT_PROJECTION_PERSPECTIVE, "equirect": N.VPT_PROJECTION_EQUIRECT, "ods": N.VPT_PROJECTION_ODS}
        if kind not in kinds:
            raise N.VptError(f"Renderer.set_projection: unknown projection {kind!r} (one of {', '.join(kinds)})")
        if kind != "ods":
            if ipd is not None or layout is not None or pole_merge is not None:
                raise N.VptError(f"Renderer.set_projection: ipd, layout and pole_merge are options of the 'ods' projection, not of {kind!r}")
            check(lib.vpt_set_projection(self.ctx, kinds[kind], float(hfov), float(vfov)), self.ctx, "vpt_set_projection")
            return
        layouts = {"left": N.VPT_ODS_LEFT, "right": N.VPT_ODS_RIGHT, "over_under": N.VPT_ODS_OVER_UNDER}
        layout = "over_under" if layout is None else layout
        if layout not in layouts:
            raise N.VptError(f"Renderer.set_projection: unknown ODS layout {layout!r} (one of {', '.join(layouts)})")
        opt = N.ods_options()
        lib.vpt_ods_options_defaults(C.byref(opt))
        if ipd is not None: opt.ipd = float(ipd)
        opt.layout = layouts[layout]
        if pole_merge is not None: opt.pole_merge_from_deg, opt.pole_merge_to_deg = (float(a) for a in pole_merge)
        check(lib.vpt_set_projection_ods(self.ctx, float(hfov), float(vfov), C.byref(opt)), self.ctx, "vpt_set_projection_ods")

    def ods_cameras(self):
        """(local_rows, W, 8) float32: per local pixel the camera of its sample in the next render call's first pass under the ODS
        projection -- origin' (3), lower_left_corner' (3), the eye e (-1 left, +1 right) and the pole merge k (vpt_debug_ods_cameras).
        Writes nothing else and leaves the blue noise as it is.  Raises VptError when the next call has no ODS projection."""
        out = torch.empty(self.n_local, 8, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_debug_ods_cameras(self.ctx, self.params.array, C.c_void_p(out.data_ptr())), self.ctx, "vpt_debug_ods_cameras")
        return out.view(self.n_local // self.width, self.width, 8)

    def camera_rays(self):
        """(n_local, 4) float32: per local pixel (b0, 0), the ray direction before normalize that the next render call's first pass takes
        (vpt_debug_camera_rays).  Writes nothing else and leaves the blue noise as it is."""
        out = torch.empty(self.n_local, 4, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_debug_camera_rays(self.ctx, self.params.array, C.c_void_p(out.data_ptr())), self.ctx, "vpt_debug_camera_rays")
        return out

    def set_camera_motion(self, cam_close: N.camera):
        """Camera motion blur (vpt_set_camera_motion) from the next call with kp.iteration == 0 on: self.cam is the pose at shutter open,
        `cam_close` (e.g. a second look_at camera) the pose at shutter close; each sample's shutter draw xi places its camera between them
        (DESIGN.md section 8i).  The pose is copied.  A non-finite field raises VptError and leaves the motion as it was."""
        check(lib.vpt_set_camera_motion(self.ctx, C.byref(cam_close)), self.ctx, "vpt_set_camera_motion")

    def clear_camera_motion(self):
        """Back to the static camera from the next call with kp.iteration == 0 on."""
        check(lib.vpt_set_camera_motion(self.ctx, None), self.ctx, "vpt_set_camera_motion")

    def motion_cameras(self):
        """(local_rows, W, 20) float32: per local pixel the shutter draw xi of the next render call's first pass, then the origin,
        lower_left_corner, horizontal, vertical, u and v of that sample's camera, padded with 0 (vpt_debug_motion_cameras).  Writes nothing
        else and leaves the blue noise as it is.  Raises VptError when the next call has no camera motion."""
        out = torch.empty(self.n_local, 20, dtype=torch.float32, device=self.buffers.accum.device)
        check(lib.vpt_debug_motion_cameras(self.ctx, self.params.array, C.c_void_p(out.data_ptr())), self.ctx, "vpt_debug_motion_cameras")
        return out.view(self.n_local // self.width, self.width, 20)

    def reset(self):
        self.kp.iteration = 0
        self.buffers.zero_()
        self.scene.reset_blue_noise()

    def stats(self, with_queue=False):
        n = C.c_ulonglong(0); q = C.c_uint(0)
        check(lib.vpt_get_stats(self.ctx, C.byref(n), C.byref(q) if with_queue else None), self.ctx, "vpt_get_stats")
        return int(n.value), int(q.value)

    def set_option(self, key, value):
        check(lib.vpt_set_option(self.ctx, key.encode(), int(value)), self.ctx, f"vpt_set_option({key})")

    def set_brick_volume(self, volume):
        """Fast mode: trace volume 0 from `volume`'s brick pool (None: back to the tex3D parity path)."""
        if volume is None:
            check(lib.vpt_set_brick_volume(self.ctx, 0, 0, 0, 0), self.ctx, "vpt_set_brick_volume")
        else:
            if not getattr(volume, "brick_pool", 0): volume.build_bricks()
            check(lib.vpt_set_brick_volume(self.ctx, volume.brick_pool, *volume.dims), self.ctx, "vpt_set_brick_volume")

    def set_cell_volume(self, volume):
        """Cell mode: trace volume 0 from `volume`'s cell table (None: back to the texture path)."""
        if volume is None:
            check(lib.vpt_set_cell_volume(self.ctx, 0, 0, 0, 0), self.ctx, "vpt_set_cell_volume")
        else:
            if not getattr(volume, "cell_table", 0): volume.build_cells()
            check(lib.vpt_set_cell_volume(self.ctx, volume.cell_table, *volume.dims), self.ctx, "vpt_set_cell_volume")

    def counters(self, reset=True):
        out = (C.c_ulonglong * 8)()
        check(lib.vpt_get_counters(self.ctx, out, 1 if reset else 0), self.ctx, "vpt_get_counters")
        v = list(out)
        return dict(lookups=v[0], lane_steps=v[1], warp_step_iters=v[2], lane_services=v[3], warp_service_rounds=v[4], rays=v[5], brick_fetches=v[6],
                    rays_per_lane=v[7])

    def hop_counters(self, reset=True):
        """Hop statistics (option "count_stats"); read them before counters(reset=True), which clears them too."""
        out = (C.c_ulonglong * 8)()
        check(lib.vpt_get_hop_counters(self.ctx, out, 1 if reset else 0), self.ctx, "vpt_get_hop_counters")
        v = list(out)
        return dict(hops_delta=v[0], hops_ratio=v[1], hops_emission=v[2], walks_ended_ahead=v[3],
                    prestep_rays=v[4], prestep_hops=v[5], prestep_ended_ahead=v[6])

    def empty_ahead_table(self):
        """The last render call's "empty ahead" table: 592 bytes, entry 8 * node + child of the 73 internal nodes, then 8 zero bytes."""
        out = (C.c_uint8 * 592)()
        check(lib.vpt_debug_empty_ahead(self.ctx, out), self.ctx, "vpt_debug_empty_ahead")
        return bytes(out)

    def kernel_times(self):
        ms = (C.c_float * 4)(); n = (C.c_int * 4)()
        check(lib.vpt_get_kernel_times(self.ctx, ms, n), self.ctx, "vpt_get_kernel_times")
        names = ("generate", "trace", "resolve", "bn_advance")
        return {k: dict(ms=float(ms[i]), launches=int(n[i])) for i, k in enumerate(names)}

    def accum_image(self):
        """(H, W, 3) float32 linear radiance (single rank only)."""
        assert self.n_ranks == 1
        return self.buffers.accum.view(self.height, self.width, 3)

    def unpermute(self, gathered: torch.Tensor, elem_floats: int):
        full = torch.empty(self.height * self.width, elem_floats, dtype=gathered.dtype, device=gathered.device)
        check(lib.vpt_unpermute(self.ctx, C.c_void_p(gathered.data_ptr()), C.c_void_p(full.data_ptr()), self.width, self.height,
                                4 * elem_floats, C.c_void_p(0)), self.ctx, "vpt_unpermute")
        return full

    def close(self):
        if self.ctx:
            lib.vpt_destroy(self.ctx); self.ctx = C.c_void_p(0)


def _frame_tensor(t, numel, name, device):
    """A full-frame float32 operand of vpt_denoise: contiguous, on `device`, `numel` elements (None passes through)."""
    if t is None:
        return None
    if t.dtype != torch.float32 or not t.is_contiguous() or t.device != device or t.numel() != numel:
        raise N.VptError(f"Renderer.denoise: `{name}` must be a contiguous float32 tensor of {numel} elements on {device} "
                         f"(got {t.dtype}, {tuple(t.shape)}, contiguous={t.is_contiguous()}, {t.device})")
    return t


def cryptomatte_id(name):
    """(id float, manifest hex) of a Cryptomatte name: the library's MurmurHash3_x86_32 of its UTF-8 bytes (vpt_cryptomatte_hash), bit 23
    flipped where the exponent is 0 or 255, as float bits and as "%08x" of those bits"""
    b = str(name).encode("utf-8")
    f = C.c_float(0.0)
    lib.vpt_cryptomatte_hash(b, len(b), C.byref(f))
    return f.value, "%08x" % int.from_bytes(bytes(f), "little")


def unpremultiply_vectors(m):
    """(vectors, coverage) of a (..., 3) motion-vector buffer (c vx, c vy, c): xy / z where z > 0, else 0, and z."""
    z = m[..., 2]
    v = torch.where((z > 0).unsqueeze(-1), m[..., :2] / torch.where(z > 0, z, torch.ones_like(z)).unsqueeze(-1), torch.zeros_like(m[..., :2]))
    return v, z


# the layers DistributedRenderer(..., layers=...) takes: the exchange layers of vpt_comm_p2p_export_layers in block order
_EXCHANGE_LAYERS = {**N.LAYER_BITS, "motion": N.VPT_LAYER_MOTION}

# the layers Renderer.denoise_layers takes by name, and their channels per pixel
_DENOISE_LAYERS = {"alpha": 1, "volume": 3, **{g: 3 for g in LIGHT_GROUPS}, "deep": 4, "mattes": 4}
# the layers Renderer.temporal_layers takes by name: the denoise layers and the collision AOVs (the motion vectors and depth are the
# filter's inputs, not its layers)
_TEMPORAL_LAYERS = {**_DENOISE_LAYERS, "position": 4, "normal": 3, "albedo": 3}


def _layer_names(layers):
    """The exchange layers asked for, checked against _EXCHANGE_LAYERS, in bit order without repeats."""
    unknown = [n for n in layers if n not in _EXCHANGE_LAYERS]
    if unknown:
        raise N.VptError(f"DistributedRenderer: unknown layer(s) {', '.join(map(repr, unknown))} (one of {', '.join(_EXCHANGE_LAYERS)})")
    return tuple(n for n in _EXCHANGE_LAYERS if n in layers)


def _layer_mask(names):
    m = 0
    for n in names:
        m |= _EXCHANGE_LAYERS[n]
    return m


def _binned_counts(deep_slices, n_mattes):
    """The binned layers asked for: 0 (not carried) or 1..VPT_DEEP_MAX_SLICES / 1..VPT_MATTE_MAX."""
    d, m = int(deep_slices), int(n_mattes)
    if not 0 <= d <= N.VPT_DEEP_MAX_SLICES:
        raise N.VptError(f"DistributedRenderer: deep_slices={d} (0 or 1..{N.VPT_DEEP_MAX_SLICES})")
    if not 0 <= m <= N.VPT_MATTE_MAX:
        raise N.VptError(f"DistributedRenderer: n_mattes={m} (0 or 1..{N.VPT_MATTE_MAX})")
    return d, m


class _DeviceView:
    """Zero-copy torch view of library-owned device memory (__cuda_array_interface__)."""
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


class DistributedRenderer:
    """Frame sharded over the ranks of a torch.distributed job (one process per GPU); scene replicated on each.

    torch.distributed is only the BOOTSTRAP here: it carries the 64-byte IPC handles (exchange="p2p") or the 128-byte NCCL id
    (exchange="nccl") between the ranks.  The exchange itself is the C++ library's:
      * "p2p" (default, up to 8 GPUs of one NVSwitch domain): the last resolve kernel of a render call stores every finished pixel
        straight into every rank's full frame over peer mappings -- gather and stripe un-permutation fused into the producer;
      * "nccl": one ncclAllGather of the rank-local accumulators + an un-permutation kernel behind the last kernel of the call.
    Pixels are independent and every Philox stream is keyed by the GLOBAL pixel index, so the gathered frame is bit-identical to a
    single-GPU render whatever the partition (SURVEY 8(e)).

    layers: names of N.LAYER_BITS -- "depth", "alpha", "volume" and the LIGHT_GROUPS -- and "motion" that the peer-memory exchange also
    carries full-frame to every rank (vpt_comm_p2p_export_layers): full_depth(), full_alpha(), full_volume(), full_light_group(name),
    full_motion_vectors().  The AOVs, groups and vectors must be enabled on every rank (enable_aovs(), enable_light_groups(),
    enable_motion_vectors(target)) and take over at the next call with kp.iteration == 0.

    deep_slices, n_mattes: the binned layers the peer-memory exchange also carries full-frame (vpt_comm_p2p_export_binned): K deep slices
    (full_deep()) and K mattes (full_mattes()), 0 = not carried.  Every rank enables exactly that many (enable_deep(bounds) with K + 1
    bounds, enable_mattes(sets) with K sets), with the same bounds and sets; changing K needs a new DistributedRenderer."""

    def __init__(self, scene: Scene, width, height, cam=None, kp=None, stripe_rows=16, options=None, gather_display=False, exchange="p2p",
                 layers=(), deep_slices=0, n_mattes=0):
        import torch.distributed as dist
        self.dist = dist
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        if self.world > 8 and exchange == "p2p": exchange = "nccl"
        self.exchange = exchange if self.world > 1 else "none"
        self.layers = _layer_names(layers)
        self.deep_slices, self.n_mattes = _binned_counts(deep_slices, n_mattes)
        self.r = Renderer(scene, width, height, cam=cam, kp=kp, rank=self.rank, n_ranks=self.world,
                          stripe_rows=stripe_rows, options=options)
        self.last_adaptive = False; self._err1 = None
        n_px = self.r.height * self.r.width
        self.full = None; self.full_display = None
        self.collective_note = "none (1 rank)"
        if self.world > 1 and self.exchange == "p2p":
            # set-up can fail on one rank only (no peer access between two devices, IPC disabled in a container): every rank reports, and
            # all of them fall back to NCCL together
            ok, err = 1, ""
            raw = (C.c_ubyte * 64)()
            try:
                check(lib.vpt_comm_p2p_export_binned(self.r.ctx, self.rank, self.world, stripe_rows, self.r.width, self.r.height,
                                                     1 if gather_display else 0, _layer_mask(self.layers), self.deep_slices, self.n_mattes, raw),
                      self.r.ctx, "vpt_comm_p2p_export_binned")
            except N.VptError as e:
                ok, err = 0, str(e)
            mine = torch.tensor(list(raw), dtype=torch.uint8, device=scene.device)
            allh = [torch.zeros(64, dtype=torch.uint8, device=scene.device) for _ in range(self.world)]
            dist.all_gather(allh, mine)                                        # bootstrap only
            if ok:
                blob = (C.c_ubyte * (64 * self.world))(*torch.cat(allh).cpu().tolist())
                try:
                    check(lib.vpt_comm_p2p_import(self.r.ctx, blob), self.r.ctx, "vpt_comm_p2p_import")
                except N.VptError as e:
                    ok, err = 0, str(e)
            flag = torch.tensor([ok], dtype=torch.int32, device=scene.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)                        # also: every rank has mapped every block before the first exchange
            if int(flag.item()) == 0:
                if ok: lib.vpt_comm_p2p_enable(self.r.ctx, 0)
                self.exchange = "nccl"; self.p2p_error = err or "another rank could not set up the peer mappings"
        if self.world > 1 and self.exchange == "p2p":
            self._map_frame(gather_display)
            self.collective_note = ("peer-memory exchange: the last resolve kernel stores each pixel into every rank's frame over NVLink peer mappings "
                                    "(all-gather + un-permutation fused into the producer), two flag exchanges per call; no NCCL on the data path")
        else:
            self.full = torch.zeros(n_px, 3, dtype=torch.float32, device=scene.device)
            self.full_display = torch.zeros(n_px, dtype=torch.int32, device=scene.device) if gather_display else None
        if self.world > 1 and self.exchange == "nccl":
            idb = torch.zeros(128, dtype=torch.uint8)
            if self.rank == 0:
                raw = (C.c_ubyte * 128)()
                check(lib.vpt_comm_get_unique_id(raw), None, "vpt_comm_get_unique_id")
                idb = torch.tensor(list(raw), dtype=torch.uint8)
            idb = idb.to(scene.device); dist.broadcast(idb, src=0)          # bootstrap only
            raw = (C.c_ubyte * 128)(*idb.cpu().tolist())
            check(lib.vpt_comm_init(self.r.ctx, raw, self.rank, self.world, stripe_rows), self.r.ctx, "vpt_comm_init")
            self.set_gather(True)
            v = C.c_int(0); lib.vpt_comm_info(self.r.ctx, C.byref(v), None, None)
            self.collective_note = (f"1 ncclAllGather (NCCL {v.value}) of the float3 accumulators per step, issued by libvpt_b200.so behind the last "
                                    "resolve kernel, + stripe un-permutation kernel")

    @classmethod
    def over_exchange(cls, renderer: Renderer, layers=(), gather_display=False, deep_slices=0, n_mattes=0):
        """A DistributedRenderer over a partitioned `renderer` whose peer-memory exchange is already active (vpt_comm_p2p_export_layers with
        the mask of `layers`, or vpt_comm_p2p_export_binned with that mask, deep_slices and n_mattes, then vpt_comm_p2p_import or
        _import_local): what __init__ leaves after its torch.distributed bootstrap.  For one process that drives several shards (one Renderer
        per GPU, or several on one GPU), each shard's calls on its own thread."""
        self = cls.__new__(cls)
        self.dist = None
        self.rank, self.world, self.r = renderer.rank, renderer.n_ranks, renderer
        self.exchange = "p2p" if self.world > 1 else "none"
        self.layers = _layer_names(layers)
        self.deep_slices, self.n_mattes = _binned_counts(deep_slices, n_mattes)
        self.last_adaptive = False; self._err1 = None
        self.full = None; self.full_display = None
        self.collective_note = "peer-memory exchange set up by the caller"
        if self.world > 1:
            for which, want, name in ((N.VPT_BINNED_DEEP, self.deep_slices, "deep_slices"), (N.VPT_BINNED_MATTES, self.n_mattes, "n_mattes")):
                p, k = C.c_uint64(0), C.c_uint(0)
                have = int(k.value) if lib.vpt_comm_p2p_binned(renderer.ctx, which, C.byref(p), C.byref(k)) == 0 else 0
                if have != want:
                    raise N.VptError(f"DistributedRenderer.over_exchange: {name}={want}, but the exchange block was exported with {have}")
        self._map_frame(gather_display)
        return self

    def _map_frame(self, gather_display):
        """Zero-copy views of this rank's exchange block: the full-frame accumulators (and display words)."""
        n_px, dev = self.r.height * self.r.width, self.r.buffers.accum.device
        pa, pd = C.c_uint64(0), C.c_uint64(0)
        check(lib.vpt_comm_p2p_frame(self.r.ctx, C.byref(pa), C.byref(pd)), self.r.ctx, "vpt_comm_p2p_frame")
        self.full = torch.as_tensor(_DeviceView(pa.value, (n_px, 3), "<f4"), device=dev)
        if gather_display: self.full_display = torch.as_tensor(_DeviceView(pd.value, (n_px,), "<i4"), device=dev)

    def render(self, n_passes, stream=None):
        self.r.render(n_passes, stream=stream)                               # the exchange is part of the call
        self.last_adaptive = False
        if self.world == 1:
            self.full.copy_(self.r.buffers.accum)
            if self.full_display is not None: self.full_display.copy_(self.r.buffers.display)

    def render_adaptive(self, max_passes, threshold=0.01, min_passes=16, check_interval=16, error_map=False, stream=None):
        """One adaptive frame of the whole image (Renderer.render_adaptive), sharded over the ranks; every rank makes the same call.
        Returns (passes_run, counts) or, with error_map=True, (passes_run, counts, rel_error), full-frame (H, W) tensors -- with more
        than one rank, views of this rank's exchange block that the next render call overwrites.  full_accum() then holds the frame.
        Needs the peer-memory exchange: with exchange="nccl" it raises VptError."""
        if self.world > 1 and self.exchange != "p2p":
            raise N.VptError("DistributedRenderer.render_adaptive: adaptive frames need the peer-memory exchange (exchange='p2p'); "
                             "the NCCL exchange does not support them")
        out = self.r.render_adaptive(max_passes, threshold=threshold, min_passes=min_passes, check_interval=check_interval,
                                     error_map=error_map or self.world == 1, stream=stream)      # one rank: denoise() keeps the error map
        self.last_adaptive = True
        H, W = self.r.height, self.r.width
        if self.world == 1:
            self.full.copy_(self.r.buffers.accum)
            if self.full_display is not None: self.full_display.copy_(self.r.buffers.display)
            self._err1 = out[2]
            return out if error_map else out[:2]
        pc, pe = C.c_uint64(0), C.c_uint64(0)
        check(lib.vpt_comm_p2p_adaptive_frame(self.r.ctx, C.byref(pc), C.byref(pe)), self.r.ctx, "vpt_comm_p2p_adaptive_frame")
        dev = self.full.device
        counts = torch.as_tensor(_DeviceView(pc.value, (H, W), "<i4"), device=dev)
        if not error_map:
            return out[0], counts
        return out[0], counts, torch.as_tensor(_DeviceView(pe.value, (H, W), "<f4"), device=dev)

    def enable_aovs(self):
        """Renderer.enable_aovs on this rank; every rank enables them.  With layers "alpha" / "volume" the exchange carries them."""
        self.r.enable_aovs()

    def enable_light_groups(self):
        """Renderer.enable_light_groups on this rank; every rank enables them.  With LIGHT_GROUPS names in `layers` the exchange carries them."""
        self.r.enable_light_groups()

    def _layer(self, name, caller):
        """(H*W, k) full frame of layer `name`: a view of this rank's exchange block, or on one rank a copy of the renderer's buffer."""
        if name not in self.layers:
            raise N.VptError(f"DistributedRenderer.{caller}: layer {name!r} was not requested (DistributedRenderer(..., layers=...) has "
                             f"{', '.join(self.layers) or 'none'})")
        n_px = self.r.height * self.r.width
        k = 1 if name in ("depth", "alpha") else 3
        if self.world == 1:
            b = self.r.buffers
            src = b.depth if name == "depth" else getattr(b, name) if name in ("alpha", "volume", "motion") else (b.groups or {}).get(name)
            if src is None:
                what = "AOVs are" if name in ("alpha", "volume") else "motion vectors are" if name == "motion" else "light groups are"
                raise N.VptError(f"DistributedRenderer.{caller}: {what} not enabled (enable_aovs() / enable_light_groups() / "
                                 "enable_motion_vectors(target))")
            return src.reshape(n_px, k).clone()
        if self.exchange != "p2p":
            raise N.VptError(f"DistributedRenderer.{caller}: the {self.exchange} exchange does not carry layers, they stay rank-local; the "
                             f"peer-memory exchange could not be set up ({getattr(self, 'p2p_error', 'exchange=' + repr(self.exchange))})")
        p = C.c_uint64(0)
        check(lib.vpt_comm_p2p_layer(self.r.ctx, _EXCHANGE_LAYERS[name], C.byref(p)), self.r.ctx, "vpt_comm_p2p_layer")
        return torch.as_tensor(_DeviceView(p.value, (n_px, k), "<f4"), device=self.full.device)

    def full_depth(self):
        """(H, W) float32 depth of the whole frame: a view of this rank's exchange block that the next call overwrites (a copy on one rank)."""
        return self._layer("depth", "full_depth").view(self.r.height, self.r.width)

    def full_alpha(self):
        """(H, W) float32 alpha AOV of the whole frame (see full_depth)."""
        return self._layer("alpha", "full_alpha").view(self.r.height, self.r.width)

    def full_volume(self):
        """(H, W, 3) float32 volume AOV of the whole frame (see full_depth)."""
        return self._layer("volume", "full_volume").view(self.r.height, self.r.width, 3)

    def full_light_group(self, name):
        """(H, W, 3) float32 light group `name` (one of LIGHT_GROUPS) of the whole frame (see full_depth)."""
        if name not in LIGHT_GROUPS:
            raise N.VptError(f"DistributedRenderer.full_light_group: unknown light group {name!r} (one of {', '.join(LIGHT_GROUPS)})")
        return self._layer(name, "full_light_group").view(self.r.height, self.r.width, 3)

    def enable_motion_vectors(self, target_cam):
        """Renderer.enable_motion_vectors on this rank; every rank sets the same target.  With layer "motion" the exchange carries them."""
        self.r.enable_motion_vectors(target_cam)

    def disable_motion_vectors(self):
        self.r.disable_motion_vectors()

    def enable_collision_aovs(self, position=True, normal=True, albedo=True, step=None):
        """Renderer.enable_collision_aovs on this rank: the buffers stay rank-local (no exchange carries them); every rank passes the same
        step (None: one voxel edge of volume 0, the same on every rank)."""
        self.r.enable_collision_aovs(position, normal, albedo, step)

    def disable_collision_aovs(self):
        self.r.disable_collision_aovs()

    def enable_cryptomatte(self, capacity=16, names=None, sphere="sphere"):
        """Renderer.enable_cryptomatte on this rank: the state stays rank-local (no exchange carries it)."""
        self.r.enable_cryptomatte(capacity, names, sphere)

    def disable_cryptomatte(self):
        self.r.disable_cryptomatte()

    def cryptomatte_state(self):
        return self.r.cryptomatte_state()

    def cryptomatte_image(self, ranks=6, overflow=False, stream=None):
        return self.r.cryptomatte_image(ranks, overflow, stream)

    def cryptomatte_manifest(self):
        return self.r.cryptomatte_manifest()

    def cryptomatte_metadata(self, layer="CryptoObject"):
        return self.r.cryptomatte_metadata(layer)

    def cryptomatte_matte(self, selection):
        return self.r.cryptomatte_matte(selection)

    def set_sample_offset(self, offset):
        """Renderer.set_sample_offset on this rank; every rank sets the same offset, so the sharded frame draws the streams a single
        context draws."""
        self.r.set_sample_offset(offset)

    def full_motion_vectors(self):
        """(H, W, 3) float32 motion-vector buffer (c vx, c vy, c) of the whole frame (see full_depth); unpremultiply_vectors() of it gives
        what Renderer.motion_vector_image() gives on one context."""
        return self._layer("motion", "full_motion_vectors").view(self.r.height, self.r.width, 3)

    def denoise(self, depth=True, out=None, display=False, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, stream=None):
        """Renderer.denoise of this rank's full frame: full_accum() guided by full_depth() (depth=False: no depth term) and, after an
        adaptive frame, by its error map.  Returns what Renderer.denoise returns; equal bit for bit to Renderer.denoise of the same frame
        rendered on one context."""
        depth = self.full_depth() if depth else None
        return self.r.denoise(color=self.full_accum(), depth=depth if depth is not None else False, rel_error=self._rel_error(), out=out,
                              display=display, iterations=iterations, sigma_luminance=sigma_luminance, sigma_depth=sigma_depth, stream=stream)

    def denoise_layers(self, layers, depth=True, iterations=5, sigma_luminance=4.0, sigma_depth=0.2, stream=None, display=False):
        """Renderer.denoise_layers of this rank's full frame: full_accum() guided by full_depth() (depth=False: no depth term) and, after
        an adaptive frame, by its error map, with the layers named in `layers` taken from full_alpha(), full_volume(),
        full_light_group(name), full_deep() and full_mattes().  A layer the exchange does not carry raises VptError.  Returns what
        Renderer.denoise_layers returns; equal bit for bit to Renderer.denoise_layers of the same frame rendered on one context."""
        full = {"alpha": self.full_alpha, "volume": self.full_volume, "deep": self.full_deep, "mattes": self.full_mattes}
        frames = {}
        for name in layers:
            if name in LIGHT_GROUPS:
                frames[name] = self.full_light_group(name)
            elif name in full:
                frames[name] = full[name]()
            else:
                raise N.VptError(f"DistributedRenderer.denoise_layers: unknown layer {name!r} (one of {', '.join(_DENOISE_LAYERS)})")
        depth = self.full_depth() if depth else None
        return self.r.denoise_layers(frames, color=self.full_accum(), depth=depth if depth is not None else False,
                                     rel_error=self._rel_error(), iterations=iterations, sigma_luminance=sigma_luminance,
                                     sigma_depth=sigma_depth, stream=stream, display=display)

    def _rel_error(self):
        """The error map of the last frame when it was adaptive (full frame), else None."""
        if not self.last_adaptive:
            return None
        if self.world == 1:
            return self._err1
        pe = C.c_uint64(0)
        check(lib.vpt_comm_p2p_adaptive_frame(self.r.ctx, None, C.byref(pe)), self.r.ctx, "vpt_comm_p2p_adaptive_frame")
        return torch.as_tensor(_DeviceView(pe.value, (self.r.height, self.r.width), "<f4"), device=self.full.device)

    def _check_binned_count(self, k, exported, what, caller):
        """An exchange that carries a binned layer refuses a render call with another count: refuse it here already."""
        if self.world > 1 and self.exchange == "p2p" and exported and k != exported:
            raise N.VptError(f"DistributedRenderer.{caller}: {k} {what}, but the peer-memory exchange carries {exported} (set K = {exported}, "
                             f"or make a new DistributedRenderer with another count)")

    def enable_deep(self, bounds):
        """Renderer.enable_deep on this rank; every rank enables the same bounds.  With deep_slices = K the peer-memory exchange carries
        them (full_deep()), and len(bounds) - 1 must be K: another count raises VptError."""
        self._check_binned_count(len(np.asarray(bounds).reshape(-1)) - 1, self.deep_slices, "deep slices", "enable_deep")
        self.r.enable_deep(bounds)

    def disable_deep(self):
        """Renderer.disable_deep on this rank."""
        self.r.disable_deep()

    def deep_image(self):
        """Renderer.deep_image of this rank: (K, local rows, W, 4), the rows of stripe_rows_of_rank(H, rank, world, stripe_rows)."""
        return self.r.deep_image()

    def enable_mattes(self, sets, sphere=None):
        """Renderer.enable_mattes on this rank; every rank enables the same sets.  With n_mattes = K the peer-memory exchange carries
        them (full_mattes()), and len(sets) must be K: another count raises VptError."""
        self._check_binned_count(len(sets), self.n_mattes, "mattes", "enable_mattes")
        self.r.enable_mattes(sets, sphere)

    def disable_mattes(self):
        """Renderer.disable_mattes on this rank."""
        self.r.disable_mattes()

    def matte_image(self):
        """Renderer.matte_image of this rank: (K, local rows, W, 4), the rows of stripe_rows_of_rank(H, rank, world, stripe_rows).
        full_mattes() is the whole frame."""
        return self.r.matte_image()

    def _binned(self, which, caller):
        """(K, H, W, 4) full frame of a binned layer: a view of this rank's exchange block, or on one rank a copy of the renderer's buffer."""
        deep = which == N.VPT_BINNED_DEEP
        what, count, arg = ("deep slices", self.deep_slices, "deep_slices") if deep else ("mattes", self.n_mattes, "n_mattes")
        if not count:
            raise N.VptError(f"DistributedRenderer.{caller}: {what} were not requested (DistributedRenderer(..., {arg}=K))")
        if self.world == 1:
            return (self.r.deep_image() if deep else self.r.matte_image()).clone()
        if self.exchange != "p2p":
            raise N.VptError(f"DistributedRenderer.{caller}: the {self.exchange} exchange does not carry {what}, they stay rank-local; the "
                             f"peer-memory exchange could not be set up ({getattr(self, 'p2p_error', 'exchange=' + repr(self.exchange))})")
        p, k = C.c_uint64(0), C.c_uint(0)
        check(lib.vpt_comm_p2p_binned(self.r.ctx, which, C.byref(p), C.byref(k)), self.r.ctx, "vpt_comm_p2p_binned")
        return torch.as_tensor(_DeviceView(p.value, (int(k.value), self.r.height, self.r.width, 4), "<f4"), device=self.full.device)

    def full_deep(self):
        """(K, H, W, 4) float32 deep slices of the whole frame, slice-major like Renderer.deep_image(): a view of this rank's exchange block
        that the next call overwrites (a copy on one rank).  The bounds are those given to enable_deep (self.r.deep_bounds), so
        deep.flatten / insert / exr_samples take it as they take a single context's deep_image()."""
        return self._binned(N.VPT_BINNED_DEEP, "full_deep")

    def full_mattes(self):
        """(K, H, W, 4) float32 instance mattes of the whole frame, matte-major like Renderer.matte_image() (see full_deep)."""
        return self._binned(N.VPT_BINNED_MATTES, "full_mattes")

    def set_region(self, x0, y0, x1, y1):
        """Renderer.set_region on this rank; every rank sets the same region.  The peer-memory exchange then stores only the region's
        pixels into full_accum(); the NCCL exchange gathers each rank's buffers whole, so outside the region they hold what they held."""
        self.r.set_region(x0, y0, x1, y1)

    def clear_region(self):
        self.r.clear_region()

    def set_projection(self, kind, hfov=360.0, vfov=180.0, ipd=None, layout=None, pole_merge=None):
        """Renderer.set_projection on this rank; every rank sets the same projection."""
        self.r.set_projection(kind, hfov=hfov, vfov=vfov, ipd=ipd, layout=layout, pole_merge=pole_merge)

    def set_camera_motion(self, cam_close):
        """Renderer.set_camera_motion on this rank; every rank sets the same poses."""
        self.r.set_camera_motion(cam_close)

    def clear_camera_motion(self):
        self.r.clear_camera_motion()

    def set_gather(self, enabled: bool):
        """Switch the per-call exchange off (rank-local work only: profiling runs that not every rank takes part in) or back on."""
        if self.world == 1: return
        if self.exchange == "p2p":
            check(lib.vpt_comm_p2p_enable(self.r.ctx, 1 if enabled else 0), self.r.ctx, "vpt_comm_p2p_enable")
        elif enabled:
            check(lib.vpt_comm_set_gather(self.r.ctx, C.c_void_p(self.full.data_ptr()),
                                          C.c_void_p(self.full_display.data_ptr()) if self.full_display is not None else None), self.r.ctx, "vpt_comm_set_gather")
        else:
            check(lib.vpt_comm_set_gather(self.r.ctx, None, None), self.r.ctx, "vpt_comm_set_gather")

    def abandoned_waits(self):
        if self.exchange != "p2p": return 0
        n = C.c_uint64(0); check(lib.vpt_comm_p2p_status(self.r.ctx, C.byref(n)), self.r.ctx, "vpt_comm_p2p_status"); return int(n.value)

    def full_accum(self):
        return self.full.view(self.r.height, self.r.width, 3)

    def close(self):
        self.full = None; self.full_display = None
        self.r.close()


class LevelAModule:
    """Level (A) of the drop-in boundary driven the way the reference application drives its kernel (main.cpp:1221-1236, 1823-1829):
    cuModuleLoad -> cuModuleGetFunction("volume_rt_kernel") -> cuLaunchKernel(grid (w/16+1, h/16+1), block (16,16), params[9]),
    through the CUDA Driver API (cuda-python).  `Renderer` only supplies the parameter block."""

    def __init__(self, cubin_path=None):
        import os
        from cuda.bindings import driver as drv
        self.drv = drv
        torch.cuda.current_stream()                                   # make sure the primary context exists and is current
        path = cubin_path or os.path.join(os.path.dirname(N.LIB_PATH), "volume_rt_kernel_b200.cubin")
        err, self.module = drv.cuModuleLoad(path.encode())
        if int(err): raise N.VptError(f"cuModuleLoad({path}) -> {err}")
        err, self.fn = drv.cuModuleGetFunction(self.module, b"volume_rt_kernel")
        if int(err): raise N.VptError(f"cuModuleGetFunction(volume_rt_kernel) -> {err}")

    def launch(self, r: "Renderer", sync=True):
        """One progressive pass; the caller keeps doing ++iteration like the reference loop."""
        gx, gy = int(r.width // 16) + 1, int(r.height // 16) + 1
        err, = self.drv.cuLaunchKernel(self.fn, gx, gy, 1, 16, 16, 1, 0, 0, C.addressof(r.params.array), 0)
        if int(err): raise N.VptError(f"cuLaunchKernel(volume_rt_kernel) -> {err}")
        r.kp.iteration += 1
        if sync: torch.cuda.synchronize()

    def close(self):
        if getattr(self, "module", None) is not None:
            self.drv.cuModuleUnload(self.module); self.module = None


def stripe_rows_of_rank(height, rank, n_ranks, stripe_rows):
    """Host-side mirror of the kernel's local-row -> global-row map (used by the CPU/gloo tests)."""
    if n_ranks == 1:
        return np.arange(height)
    stripes = (height + stripe_rows - 1) // stripe_rows
    per_rank = (stripes + n_ranks - 1) // n_ranks
    rows = []
    for lr in range(per_rank * stripe_rows):
        s = lr // stripe_rows
        rows.append((s * n_ranks + rank) * stripe_rows + lr % stripe_rows)
    return np.array(rows)
