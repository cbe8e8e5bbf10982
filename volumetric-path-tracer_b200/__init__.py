"""volumetric-path-tracer_b200: H100-native (sm_90a) replacement for the render pass of
sergeneren/Volumetric-Path-Tracer, behind the reference's own launch-parameter ABI.

The directory name carries a hyphen (it mirrors the reference's repository name); import it through the
top-level shim `vpt_b200` (repo root), which loads this package under that name.
"""
from ._native import (lib, VptError, camera, light_list, point_light, GPU_VDB, VDB_INFO, AABB, OCTNode, BVHNode, sphere,
                      geometry_list, AtmosphereParameters, Kernel_params, f3, i3, u2, LIB_PATH)
from .scene import Scene, Volume, EnvTables, sky_power_table, default_kernel_params, find_asset, load_ins, scene_from_ins, read_bvh, Atmosphere, read_atmosphere_tables
from .renderer import Renderer, DistributedRenderer, LevelAModule, FrameBuffers, LaunchParams, stripe_rows_of_rank, LIGHT_GROUPS
from . import deep

__all__ = ["lib", "VptError", "camera", "light_list", "point_light", "GPU_VDB", "VDB_INFO", "AABB", "OCTNode", "BVHNode",
           "sphere", "geometry_list", "AtmosphereParameters", "Kernel_params", "f3", "i3", "u2", "Scene", "Volume",
           "EnvTables", "sky_power_table", "load_ins", "scene_from_ins", "read_bvh", "Atmosphere", "read_atmosphere_tables", "default_kernel_params", "find_asset", "Renderer", "DistributedRenderer", "LevelAModule", "FrameBuffers", "LaunchParams",
           "stripe_rows_of_rank", "LIGHT_GROUPS", "LIB_PATH", "deep"]
