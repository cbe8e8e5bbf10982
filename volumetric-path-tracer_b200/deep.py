"""Deep slices on the host side: the holdout composite and the OpenEXR deep-sample view of Renderer.deep_image().

The renderer's deep slices (vpt_set_deep_buffers, DESIGN.md section 8h) hold, per depth interval [z_k, z_{k+1}) and pixel, the running
means c_k (premultiplied colour) and p_k (coverage) of the camera samples whose first collision lies in that interval.  The intervals are
disjoint, so the means add: the slices in front of a depth z together are the volume that an element at z is behind.

Plain torch on whatever device the slices live on (no kernel of this library runs here).
  flatten(slices, bounds, z=None)              -> (colour (H, W, 3), coverage (H, W)) of the slices whose back bound is <= z
  insert(slices, bounds, z, element, plate)    -> (colour, alpha): a premultiplied element put into the volume at depth z
  exr_samples(slices, bounds)                  -> ExrSamples, the OpenEXR deep convention of the same data
"""
from collections import namedtuple

import torch

__all__ = ["flatten", "insert", "exr_samples", "ExrSamples"]

# OpenEXR deep samples: `count` (H, W) int64 samples per pixel; then every sample of every pixel, pixel by pixel in row-major order and
# front to back within a pixel (the layout of a deep scanline image): z, zback (N,), a (N,) and rgb (N, 3)
ExrSamples = namedtuple("ExrSamples", "count z zback a rgb")


def _check(slices, bounds):
    if slices.dim() != 4 or slices.shape[-1] != 4:
        raise ValueError(f"deep slices must be (K, H, W, 4), got {tuple(slices.shape)}")
    z = torch.as_tensor(bounds, dtype=torch.float32, device=slices.device).reshape(-1)
    if z.numel() != slices.shape[0] + 1:
        raise ValueError(f"{slices.shape[0]} slices need {slices.shape[0] + 1} bounds, got {z.numel()}")
    return z


def flatten(slices, bounds, z=None):
    """The slices in front of depth z, summed: (colour (H, W, 3), coverage (H, W)).  A slice counts when its back bound z_{k+1} <= z (an
    open last slice only for z = inf); z is a number or an (H, W) tensor of holdout depths, None takes every slice.  These are means over
    ALL the pixel's samples, not over those that reach z: an element at z is seen through 1 - coverage, and what lies behind it (every
    slice minus these) is already weighted by the samples that get there -- insert() puts the two together.  A holdout inside a slice
    is not split: choose bounds at the depths where elements go."""
    zb = _check(slices, bounds)
    if z is None:
        keep = torch.ones(slices.shape[:3], dtype=torch.bool, device=slices.device)
    else:
        zt = torch.as_tensor(z, dtype=torch.float32, device=slices.device)
        keep = zb[1:].view(-1, 1, 1) <= zt                        # (K, H, W), a scalar z broadcast
        keep = keep.expand(slices.shape[:3])
    picked = torch.where(keep[..., None], slices, torch.zeros((), dtype=slices.dtype, device=slices.device))
    total = picked.sum(0)
    return total[..., :3], total[..., 3]


def insert(slices, bounds, z, element, plate=None):
    """The volume with an element inside it: a premultiplied element (H, W, 4) (rgb already times its alpha a) at depth z (a number or
    an (H, W) tensor), over a plate (H, W, 3) or black.  -> (colour (H, W, 3), alpha (H, W)).
    With F, f = flatten(slices, bounds, z) (the volume in front of z) and V, A = flatten(slices, bounds) (all of it):
        colour = F + (1 - f) * rgb + (1 - a) * ((V - F) + (1 - A) * plate)
        alpha  = f + (1 - f) * a + (1 - a) * (A - f)
    A sample that collides in front of z is the volume's; of the rest a fraction a is the element's, and the others go on to collide
    behind z (V - F: already weighted by the samples that get there, so not scaled by 1 - f again) or to the plate.  An empty element
    gives V + (1 - A) * plate, the flat composite of the AOVs; an opaque one F + (1 - f) * rgb."""
    front_c, front_a = flatten(slices, bounds, z)
    all_c, all_a = flatten(slices, bounds)
    e = torch.as_tensor(element, dtype=slices.dtype, device=slices.device)
    if e.shape != (*slices.shape[1:3], 4):
        raise ValueError(f"element must be (H, W, 4), got {tuple(e.shape)}")
    rgb, a = e[..., :3], e[..., 3]
    behind = all_c - front_c
    if plate is not None:
        behind = behind + (1 - all_a)[..., None] * torch.as_tensor(plate, dtype=slices.dtype, device=slices.device)
    colour = front_c + (1 - front_a)[..., None] * rgb + (1 - a)[..., None] * behind
    alpha = front_a + (1 - front_a) * a + (1 - a) * (all_a - front_a)
    return colour, alpha


def exr_samples(slices, bounds):
    """The slices as OpenEXR deep samples, keeping per pixel the non-empty slices (coverage or colour not 0): Z = z_k, ZBack = z_{k+1},
    A_k = p_k / T_k and RGB_k = c_k / T_k with T_k = 1 - sum_{j<k} p_j, the transmittance in front of the slice.  Compositing a
    pixel's samples front to back with the deep "over" operator, C += T * RGB_k, T *= 1 - A_k, gives back sum c_k and 1 - T = sum p_k.
    A sample behind full coverage (T_k <= 0, which the means reach only through rounding) is opaque black: nothing behind it shows."""
    zb = _check(slices, bounds)
    p, c = slices[..., 3], slices[..., :3]
    t = 1.0 - (torch.cumsum(p, 0) - p)                            # T_k, (K, H, W)
    seen = t > 0
    one = torch.ones((), dtype=slices.dtype, device=slices.device)
    a = torch.where(seen, p / torch.where(seen, t, one), one)
    rgb = torch.where(seen[..., None], c / torch.where(seen, t, one)[..., None], torch.zeros((), dtype=slices.dtype, device=slices.device))
    keep = (p != 0) | (c != 0).any(-1)                           # (K, H, W)
    order = (1, 2, 0)                                            # pixel-major, slices front to back within a pixel
    kp = keep.permute(*order)
    zs = zb[:-1].view(-1, 1, 1).expand_as(p).permute(*order)[kp]
    zbs = zb[1:].view(-1, 1, 1).expand_as(p).permute(*order)[kp]
    return ExrSamples(kp.sum(-1), zs, zbs, a.permute(*order)[kp], rgb.permute(1, 2, 0, 3)[kp])
