"""ctypes binding of libvpt_b200.so (include/vpt_b200.h) and mirrors of the boundary structs.

The structures below are the host-side mirror of the reference's launch-parameter types
(`camera`, `light_list`, `GPU_VDB`, `sphere`, `OCTNode`, `AtmosphereParameters`,
`Kernel_params`; layouts in include/vpt_abi.h, reference declarations cited there).  They keep
the reference's field names so that code and tests read like code written against the reference.

There is no fallback: if the CUDA extension is missing, importing this module raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", os.environ.get("VPT_LIB_NAME", "libvpt_b200.so"))   # VPT_LIB_NAME: tuning builds only


class NativeLibraryMissing(ImportError):
    pass


if not os.path.exists(LIB_PATH):
    raise NativeLibraryMissing(
        f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(volumetric-path-tracer_b200/csrc/build.sh). There is no Python/CPU fallback for the render path.")

lib = C.CDLL(LIB_PATH)


# ---- plain vector types --------------------------------------------------------------------------
class f3(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("z", C.c_float)]

    def __init__(self, x=0.0, y=0.0, z=0.0):
        super().__init__(float(x), float(y), float(z))

    def tup(self):
        return (self.x, self.y, self.z)


class i3(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("z", C.c_int32)]


class u2(C.Structure):
    _fields_ = [("x", C.c_uint32), ("y", C.c_uint32)]


# ---- camera (source/gpu_vdb/camera.h:94-148) ------------------------------------------------------
class camera(C.Structure):
    _fields_ = [("time1", C.c_float), ("time0", C.c_float), ("origin", f3), ("focus_dist", C.c_float),
                ("lower_left_corner", f3), ("horizontal", f3), ("vertical", f3),
                ("u", f3), ("v", f3), ("w", f3), ("lens_radius", C.c_float),
                ("viz_dof", C.c_uint8), ("_pad", C.c_uint8 * 3)]


class point_light(C.Structure):
    _fields_ = [("_vptr", C.c_uint64), ("pos", f3), ("dir", f3), ("power", C.c_float), ("color", f3)]


class light_list(C.Structure):
    _fields_ = [("num_lights", C.c_uint32), ("_pad", C.c_uint32), ("light_ptr", C.c_uint64)]


# ---- VDB_INFO / GPU_VDB (source/gpu_vdb/gpu_vdb.h:59-154) ------------------------------------------
class VDB_INFO(C.Structure):
    _fields_ = [("voxelsize", C.c_float), ("dim", i3), ("bmin", f3), ("bmax", f3),
                ("max_density", C.c_float), ("min_density", C.c_float),
                ("has_color", C.c_uint8), ("has_emission", C.c_uint8), ("matte", C.c_uint8), ("_pad", C.c_uint8 * 5),
                ("density_texture", C.c_uint64), ("emission_texture", C.c_uint64), ("color_texture", C.c_uint64)]


class GPU_VDB(C.Structure):
    _fields_ = [("vdb_info", VDB_INFO), ("xform", (C.c_float * 4) * 4)]


class AABB(C.Structure):
    _fields_ = [("pmin", f3), ("pmax", f3)]


class OCTNode(C.Structure):
    _fields_ = [("num_volumes", C.c_int32), ("vol_indices", C.c_int32 * 600),
                ("max_extinction", C.c_float), ("min_extinction", C.c_float), ("voxel_size", C.c_float),
                ("depth", C.c_int32), ("has_children", C.c_uint8), ("_pad", C.c_uint8 * 3),
                ("children", C.c_uint64 * 8), ("parent", C.c_uint64), ("bbox", AABB)]


class BVHNode(C.Structure):
    _fields_ = [("minId", C.c_int32), ("maxId", C.c_int32), ("volIndex", C.c_int32), ("_pad", C.c_int32),
                ("leftChild", C.c_uint64), ("rightChild", C.c_uint64), ("parent", C.c_uint64), ("boundingBox", AABB)]


class sphere(C.Structure):
    _fields_ = [("_vptr", C.c_uint64), ("center", f3), ("radius", C.c_float), ("color", f3), ("roughness", C.c_float)]


class geometry_list(C.Structure):
    _fields_ = [("list", C.c_uint64), ("list_size", C.c_int32), ("_pad", C.c_int32)]


class DensityProfileLayer(C.Structure):
    _fields_ = [("width", C.c_float), ("exp_term", C.c_float), ("exp_scale", C.c_float),
                ("linear_term", C.c_float), ("const_term", C.c_float), ("_pad", C.c_float * 3)]


class DensityProfile(C.Structure):
    _fields_ = [("layers", DensityProfileLayer * 2)]


class AtmosphereParameters(C.Structure):
    _fields_ = [("sky_spectral_radiance_to_luminance", f3), ("sun_spectral_radiance_to_luminance", f3),
                ("solar_irradiance", f3), ("angle", C.c_float), ("bottom_radius", C.c_float), ("top_radius", C.c_float),
                ("use_luminance", C.c_int32), ("_pad0", C.c_uint8 * 12),
                ("rayleigh_density", DensityProfile), ("rayleigh_scattering", f3), ("_pad1", C.c_uint8 * 4),
                ("mie_density", DensityProfile), ("mie_scattering", f3), ("mie_extinction", f3),
                ("mie_phase_function_g", C.c_float), ("_pad2", C.c_uint8 * 4),
                ("absorption_density", DensityProfile), ("absorption_extinction", f3), ("ground_albedo", f3),
                ("sun_angular_radius", C.c_float), ("mu_s_min", C.c_float), ("exposure", C.c_float), ("white_point", f3),
                ("scratch_buffers", C.c_uint64 * 9),
                ("transmittance_texture", C.c_uint64), ("scattering_texture", C.c_uint64),
                ("irradiance_texture", C.c_uint64), ("single_mie_scattering_texture", C.c_uint64), ("_pad3", C.c_uint8 * 8)]


# ---- Kernel_params (source/kernel_params.h:39-109) -------------------------------------------------
class Kernel_params(C.Structure):
    _fields_ = [("render", C.c_uint8), ("debug", C.c_uint8), ("_pad0", C.c_uint8 * 6),
                ("resolution", u2), ("exposure_scale", C.c_float), ("_pad1", C.c_uint8 * 4),
                ("display_buffer", C.c_uint64), ("raw_buffer", C.c_uint64), ("blue_noise_buffer", C.c_uint64),
                ("emission_texture", C.c_uint64), ("emission_scale", C.c_float), ("emission_pivot", C.c_float),
                ("density_color_texture", C.c_uint64), ("iteration", C.c_uint32), ("_pad2", C.c_uint8 * 4),
                ("accum_buffer", C.c_uint64), ("depth_buffer", C.c_uint64),
                ("max_interactions", C.c_uint32), ("ray_depth", C.c_int32), ("volume_depth", C.c_int32),
                ("min_extinction", C.c_float), ("phase_g1", C.c_float), ("phase_g2", C.c_float), ("phase_f", C.c_float),
                ("albedo", f3), ("extinction", f3), ("transmittance", f3), ("tr_depth", C.c_float), ("density_mult", C.c_float),
                ("environment_type", C.c_uint32), ("azimuth", C.c_float), ("elevation", C.c_float),
                ("sun_color", f3), ("sky_color", f3), ("sun_mult", C.c_float), ("sky_mult", C.c_float), ("_pad3", C.c_uint8 * 4),
                ("energy_inject", C.c_double), ("env_tex", C.c_uint64), ("env_sample_tex_res", C.c_int32), ("_pad4", C.c_uint8 * 4),
                ("sky_tex", C.c_uint64), ("env_func_tex", C.c_uint64), ("env_cdf_tex", C.c_uint64),
                ("env_marginal_func_tex", C.c_uint64), ("env_marginal_cdf_tex", C.c_uint64),
                ("env_marginal_int", C.c_float), ("_pad5", C.c_uint8 * 4),
                ("debug_buffer", C.c_uint64), ("cost_buffer", C.c_uint64), ("integrator", C.c_int32), ("_pad6", C.c_uint8 * 4)]


ABI_STRUCTS = [camera, light_list, GPU_VDB, sphere, geometry_list, BVHNode, OCTNode, AtmosphereParameters,
               Kernel_params, point_light, VDB_INFO, AABB]
ABI_SIZES = [104, 16, 144, 40, 16, 64, 2520, 464, 312, 48, 80, 24]

# every symbol include/vpt_b200.h declares (tests check that the library exports them all)
EXPORTED_SYMBOLS = [
    "vpt_create", "vpt_destroy", "vpt_last_error", "vpt_version", "vpt_abi_sizes", "vpt_set_option", "vpt_set_partition",
    "vpt_local_pixels", "vpt_unpermute", "vpt_render_pass", "vpt_render_passes", "vpt_invalidate_scene", "vpt_get_stats",
    "vpt_texture_create_3d", "vpt_texture_create_env", "vpt_texture_destroy", "vpt_vdb_load", "vpt_hdr_load",
    "vpt_bmp_load_rbg", "vpt_exr_load_rgb", "vpt_free", "vpt_octree_build", "vpt_octree_destroy", "vpt_volume_bounds",
    "vpt_camera_look_at", "vpt_kernel_params_defaults", "vpt_get_counters", "vpt_get_hop_counters", "vpt_debug_empty_ahead", "vpt_get_kernel_times", "vpt_octree_read",
    "vpt_env_tables_create", "vpt_ins_load", "vpt_env_sky_tabulate",
    "vpt_octree_info", "vpt_octree_read_flat", "vpt_bvh_build", "vpt_bvh_read", "vpt_bvh_destroy", "vpt_env_tables_compute",
    "vpt_comm_get_unique_id", "vpt_comm_init", "vpt_comm_set_gather", "vpt_comm_wait", "vpt_comm_info", "vpt_comm_destroy",
    "vpt_texture_create_3d_from_device", "vpt_procedural_fill", "vpt_bricks_create", "vpt_bricks_destroy", "vpt_set_brick_volume", "vpt_bricks_read", "vpt_debug_sampler_compare", "vpt_debug_software_sample", "vpt_atmosphere_options_defaults", "vpt_atmosphere_precompute", "vpt_atmosphere_destroy",
    "vpt_texture_read_f4", "vpt_debug_texture_sample", "vpt_debug_bruneton_stage",
    "vpt_cells_create", "vpt_cells_read", "vpt_cells_destroy", "vpt_set_cell_volume",
    "vpt_comm_p2p_export", "vpt_comm_p2p_import", "vpt_comm_p2p_import_local", "vpt_comm_p2p_block", "vpt_comm_p2p_frame", "vpt_comm_p2p_enable", "vpt_comm_p2p_status",
    "vpt_adaptive_options_defaults", "vpt_render_adaptive", "vpt_comm_p2p_adaptive_frame", "vpt_debug_adapt_rule",
    "vpt_denoise_options_defaults", "vpt_denoise", "vpt_denoise_layers",
    "vpt_set_aov_buffers", "vpt_set_light_group_buffers", "vpt_set_render_region", "vpt_set_projection", "vpt_debug_camera_rays",
    "vpt_comm_p2p_export_layers", "vpt_comm_p2p_layer", "vpt_comm_p2p_block_bytes",
    "vpt_set_deep_buffers", "vpt_set_camera_motion", "vpt_debug_motion_cameras",
    "vpt_ods_options_defaults", "vpt_set_projection_ods", "vpt_debug_ods_cameras",
    "vpt_set_instance_mattes",
    "vpt_comm_p2p_export_binned", "vpt_comm_p2p_binned", "vpt_comm_p2p_block_bytes_binned",
    "vpt_set_motion_vectors", "vpt_set_sample_offset", "vpt_temporal_options_defaults", "vpt_temporal", "vpt_temporal_layers",
    "vpt_set_collision_aovs", "vpt_set_cryptomatte", "vpt_cryptomatte_rank", "vpt_cryptomatte_hash",
]

# exchange layers of vpt_comm_p2p_export_layers: name -> VPT_LAYER_* bit (bit order = plane order in the block)
LAYER_BITS = {"depth": 0x01, "alpha": 0x02, "volume": 0x04, "sun": 0x08, "point": 0x10, "emission": 0x20, "environment": 0x40}
VPT_LAYER_MOTION = 0x100                                            # the motion vectors' exchange plane (after the seven above)

# ---- prototypes ------------------------------------------------------------------------------------
_vp = C.c_void_p
lib.vpt_create.argtypes = [C.POINTER(_vp)]; lib.vpt_create.restype = C.c_int
lib.vpt_destroy.argtypes = [_vp]; lib.vpt_destroy.restype = None
lib.vpt_last_error.argtypes = [_vp]; lib.vpt_last_error.restype = C.c_char_p
lib.vpt_version.argtypes = []; lib.vpt_version.restype = C.c_char_p
lib.vpt_abi_sizes.argtypes = [C.POINTER(C.c_size_t), C.c_int]; lib.vpt_abi_sizes.restype = C.c_int
lib.vpt_set_option.argtypes = [_vp, C.c_char_p, C.c_int]; lib.vpt_set_option.restype = C.c_int
lib.vpt_set_partition.argtypes = [_vp, C.c_int, C.c_int, C.c_int]; lib.vpt_set_partition.restype = C.c_int
lib.vpt_local_pixels.argtypes = [_vp, C.c_uint, C.c_uint]; lib.vpt_local_pixels.restype = C.c_longlong
lib.vpt_unpermute.argtypes = [_vp, _vp, _vp, C.c_uint, C.c_uint, C.c_int, _vp]; lib.vpt_unpermute.restype = C.c_int
lib.vpt_render_pass.argtypes = [_vp, C.POINTER(_vp), _vp]; lib.vpt_render_pass.restype = C.c_int
lib.vpt_render_passes.argtypes = [_vp, C.POINTER(_vp), C.c_uint, _vp]; lib.vpt_render_passes.restype = C.c_int
lib.vpt_invalidate_scene.argtypes = [_vp]; lib.vpt_invalidate_scene.restype = C.c_int


class adaptive_options(C.Structure):
    _fields_ = [("min_passes", C.c_uint), ("check_interval", C.c_uint), ("threshold", C.c_float)]


lib.vpt_adaptive_options_defaults.argtypes = [C.POINTER(adaptive_options)]; lib.vpt_adaptive_options_defaults.restype = None
lib.vpt_render_adaptive.argtypes = [_vp, C.POINTER(_vp), C.c_uint, C.POINTER(adaptive_options), _vp, _vp, C.POINTER(C.c_uint), _vp]
lib.vpt_render_adaptive.restype = C.c_int
# vpt_debug_adapt_rule(samples, width, height, n_passes, opt, region[4] or NULL, pass_count, rel_error, test_err, max_tests, passes_run, n_tests)
lib.vpt_debug_adapt_rule.argtypes = [_vp, C.c_uint, C.c_uint, C.c_uint, C.POINTER(adaptive_options), C.POINTER(C.c_uint), _vp, _vp, _vp,
                                     C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_uint)]
lib.vpt_debug_adapt_rule.restype = C.c_int
lib.vpt_set_aov_buffers.argtypes = [_vp, _vp, _vp]; lib.vpt_set_aov_buffers.restype = C.c_int
lib.vpt_set_light_group_buffers.argtypes = [_vp, _vp, _vp, _vp, _vp]; lib.vpt_set_light_group_buffers.restype = C.c_int
VPT_DEEP_MAX_SLICES = 32                                            # vpt_set_deep_buffers: most slices
lib.vpt_set_deep_buffers.argtypes = [_vp, _vp, C.c_uint, C.POINTER(C.c_float)]; lib.vpt_set_deep_buffers.restype = C.c_int
VPT_MATTE_MAX = 32                                                  # vpt_set_instance_mattes: most mattes
lib.vpt_set_instance_mattes.argtypes = [_vp, _vp, C.c_uint, C.POINTER(C.c_int), C.c_uint, C.c_int]
lib.vpt_set_instance_mattes.restype = C.c_int
lib.vpt_set_render_region.argtypes = [_vp, C.c_uint, C.c_uint, C.c_uint, C.c_uint]; lib.vpt_set_render_region.restype = C.c_int
VPT_PROJECTION_PERSPECTIVE, VPT_PROJECTION_EQUIRECT, VPT_PROJECTION_ODS = 0, 1, 2   # vpt_set_projection kinds
lib.vpt_set_projection.argtypes = [_vp, C.c_int, C.c_double, C.c_double]; lib.vpt_set_projection.restype = C.c_int
lib.vpt_debug_camera_rays.argtypes = [_vp, C.POINTER(_vp), _vp]; lib.vpt_debug_camera_rays.restype = C.c_int
VPT_ODS_LEFT, VPT_ODS_RIGHT, VPT_ODS_OVER_UNDER = 0, 1, 2          # vpt_ods_options.layout


class ods_options(C.Structure):
    _fields_ = [("ipd", C.c_float), ("layout", C.c_int), ("pole_merge_from_deg", C.c_float), ("pole_merge_to_deg", C.c_float)]


lib.vpt_ods_options_defaults.argtypes = [C.POINTER(ods_options)]; lib.vpt_ods_options_defaults.restype = None
lib.vpt_set_projection_ods.argtypes = [_vp, C.c_double, C.c_double, C.POINTER(ods_options)]; lib.vpt_set_projection_ods.restype = C.c_int
lib.vpt_debug_ods_cameras.argtypes = [_vp, C.POINTER(_vp), _vp]; lib.vpt_debug_ods_cameras.restype = C.c_int


class denoise_options(C.Structure):
    _fields_ = [("iterations", C.c_uint), ("sigma_luminance", C.c_float), ("sigma_depth", C.c_float)]


lib.vpt_denoise_options_defaults.argtypes = [C.POINTER(denoise_options)]; lib.vpt_denoise_options_defaults.restype = None
lib.vpt_denoise.argtypes = [_vp, C.c_uint, C.c_uint, _vp, _vp, _vp, C.POINTER(denoise_options), C.c_float, _vp, _vp, _vp]
lib.vpt_denoise.restype = C.c_int


class denoise_layer(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("channels", C.c_uint), ("count", C.c_uint)]


lib.vpt_denoise_layers.argtypes = [_vp, C.c_uint, C.c_uint, _vp, _vp, _vp, C.POINTER(denoise_options), C.c_float, _vp, _vp,
                                   C.POINTER(denoise_layer), C.c_uint, _vp]
lib.vpt_denoise_layers.restype = C.c_int
lib.vpt_get_stats.argtypes = [_vp, C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint)]; lib.vpt_get_stats.restype = C.c_int
lib.vpt_get_counters.argtypes = [_vp, C.POINTER(C.c_ulonglong), C.c_int]; lib.vpt_get_counters.restype = C.c_int
lib.vpt_get_hop_counters.argtypes = [_vp, C.POINTER(C.c_ulonglong), C.c_int]; lib.vpt_get_hop_counters.restype = C.c_int
lib.vpt_debug_empty_ahead.argtypes = [_vp, C.POINTER(C.c_uint8)]; lib.vpt_debug_empty_ahead.restype = C.c_int
lib.vpt_get_kernel_times.argtypes = [_vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]; lib.vpt_get_kernel_times.restype = C.c_int
lib.vpt_texture_create_3d.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(_vp)]
lib.vpt_texture_create_3d.restype = C.c_int
lib.vpt_texture_create_env.argtypes = [C.POINTER(C.c_float), C.c_uint, C.c_uint, C.POINTER(C.c_uint64), C.POINTER(_vp)]
lib.vpt_texture_create_env.restype = C.c_int
lib.vpt_texture_destroy.argtypes = [C.c_uint64, _vp]; lib.vpt_texture_destroy.restype = C.c_int
lib.vpt_env_tables_create.argtypes = [C.POINTER(C.c_float), C.c_uint, C.POINTER(C.c_uint64), C.POINTER(_vp), C.POINTER(C.c_float)]
lib.vpt_env_tables_create.restype = C.c_int


lib.vpt_env_tables_compute.argtypes = [C.POINTER(C.c_float), C.c_uint, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]
lib.vpt_env_tables_compute.restype = C.c_int


lib.vpt_comm_get_unique_id.argtypes = [C.POINTER(C.c_ubyte)]; lib.vpt_comm_get_unique_id.restype = C.c_int
lib.vpt_comm_init.argtypes = [_vp, C.POINTER(C.c_ubyte), C.c_int, C.c_int, C.c_int]; lib.vpt_comm_init.restype = C.c_int
lib.vpt_comm_set_gather.argtypes = [_vp, _vp, _vp]; lib.vpt_comm_set_gather.restype = C.c_int
lib.vpt_comm_wait.argtypes = [_vp, _vp]; lib.vpt_comm_wait.restype = C.c_int
lib.vpt_comm_info.argtypes = [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]; lib.vpt_comm_info.restype = C.c_int
lib.vpt_comm_destroy.argtypes = [_vp]; lib.vpt_comm_destroy.restype = C.c_int
lib.vpt_comm_p2p_export.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_int, C.POINTER(C.c_ubyte)]; lib.vpt_comm_p2p_export.restype = C.c_int
lib.vpt_comm_p2p_import.argtypes = [_vp, C.POINTER(C.c_ubyte)]; lib.vpt_comm_p2p_import.restype = C.c_int
lib.vpt_comm_p2p_import_local.argtypes = [_vp, C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_import_local.restype = C.c_int
lib.vpt_comm_p2p_block.argtypes = [_vp, C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_block.restype = C.c_int
lib.vpt_comm_p2p_frame.argtypes = [_vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_frame.restype = C.c_int
lib.vpt_comm_p2p_adaptive_frame.argtypes = [_vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_adaptive_frame.restype = C.c_int
lib.vpt_comm_p2p_enable.argtypes = [_vp, C.c_int]; lib.vpt_comm_p2p_enable.restype = C.c_int
lib.vpt_comm_p2p_status.argtypes = [_vp, C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_status.restype = C.c_int
lib.vpt_comm_p2p_export_layers.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_uint, C.POINTER(C.c_ubyte)]
lib.vpt_comm_p2p_export_layers.restype = C.c_int
lib.vpt_comm_p2p_layer.argtypes = [_vp, C.c_uint, C.POINTER(C.c_uint64)]; lib.vpt_comm_p2p_layer.restype = C.c_int
lib.vpt_comm_p2p_block_bytes.argtypes = [C.c_uint, C.c_uint, C.c_int, C.c_uint, C.POINTER(C.c_size_t)]; lib.vpt_comm_p2p_block_bytes.restype = C.c_int
VPT_BINNED_DEEP, VPT_BINNED_MATTES = 1, 2                          # vpt_comm_p2p_binned: which binned layer
lib.vpt_comm_p2p_export_binned.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_uint, C.c_uint, C.c_uint,
                                           C.POINTER(C.c_ubyte)]
lib.vpt_comm_p2p_export_binned.restype = C.c_int
lib.vpt_comm_p2p_binned.argtypes = [_vp, C.c_uint, C.POINTER(C.c_uint64), C.POINTER(C.c_uint)]; lib.vpt_comm_p2p_binned.restype = C.c_int
lib.vpt_comm_p2p_block_bytes_binned.argtypes = [C.c_uint, C.c_uint, C.c_int, C.c_uint, C.c_uint, C.c_uint, C.POINTER(C.c_size_t)]
lib.vpt_comm_p2p_block_bytes_binned.restype = C.c_int


lib.vpt_texture_create_3d_from_device.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(_vp)]
lib.vpt_texture_create_3d_from_device.restype = C.c_int
lib.vpt_procedural_fill.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, _vp]; lib.vpt_procedural_fill.restype = C.c_int
lib.vpt_bricks_create.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_ulonglong)]; lib.vpt_bricks_create.restype = C.c_int
lib.vpt_bricks_read.argtypes = [C.c_uint64, C.c_ulonglong, C.c_ulonglong, C.POINTER(C.c_float)]; lib.vpt_bricks_read.restype = C.c_int
lib.vpt_debug_sampler_compare.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint, C.POINTER(C.c_double)]
lib.vpt_debug_sampler_compare.restype = C.c_int
lib.vpt_debug_software_sample.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float)]
lib.vpt_debug_software_sample.restype = C.c_int
lib.vpt_bricks_destroy.argtypes = [C.c_uint64]; lib.vpt_bricks_destroy.restype = C.c_int
lib.vpt_cells_create.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_ulonglong)]; lib.vpt_cells_create.restype = C.c_int
lib.vpt_cells_read.argtypes = [C.c_uint64, C.c_ulonglong, C.c_ulonglong, C.POINTER(C.c_float)]; lib.vpt_cells_read.restype = C.c_int
lib.vpt_cells_destroy.argtypes = [C.c_uint64]; lib.vpt_cells_destroy.restype = C.c_int
lib.vpt_set_cell_volume.argtypes = [_vp, C.c_uint64, C.c_int, C.c_int, C.c_int]; lib.vpt_set_cell_volume.restype = C.c_int
lib.vpt_set_brick_volume.argtypes = [_vp, C.c_uint64, C.c_int, C.c_int, C.c_int]; lib.vpt_set_brick_volume.restype = C.c_int


class atmosphere_options(C.Structure):
    _fields_ = [("use_constant_solar_spectrum", C.c_int), ("use_ozone", C.c_int), ("luminance_mode", C.c_int), ("do_white_balance", C.c_int),
                ("exposure", C.c_float), ("num_scattering_orders", C.c_int)]


lib.vpt_atmosphere_options_defaults.argtypes = [C.POINTER(atmosphere_options)]; lib.vpt_atmosphere_options_defaults.restype = None
lib.vpt_atmosphere_precompute.argtypes = [C.POINTER(atmosphere_options), C.POINTER(AtmosphereParameters), C.POINTER(_vp)]; lib.vpt_atmosphere_precompute.restype = C.c_int
lib.vpt_atmosphere_destroy.argtypes = [_vp]; lib.vpt_atmosphere_destroy.restype = C.c_int
lib.vpt_texture_read_f4.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float)]; lib.vpt_texture_read_f4.restype = C.c_int
lib.vpt_debug_texture_sample.argtypes = [C.c_uint64, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float)]; lib.vpt_debug_texture_sample.restype = C.c_int
# vpt_debug_bruneton_stage: stage numbers (VPT_BRUNETON_*)
BRUNETON_TRANSMITTANCE, BRUNETON_DIRECT_IRRADIANCE, BRUNETON_SINGLE_SCATTERING = 0, 1, 2
BRUNETON_SCATTERING_DENSITY, BRUNETON_INDIRECT_IRRADIANCE, BRUNETON_MULTIPLE_SCATTERING = 3, 4, 5
lib.vpt_debug_bruneton_stage.argtypes = [C.c_int, C.POINTER(AtmosphereParameters), C.POINTER(C.c_uint64), C.POINTER(C.c_float), C.c_int, C.c_int]
lib.vpt_debug_bruneton_stage.restype = C.c_int


class ins_header(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_files", C.c_int32), ("n_records", C.c_int32), ("reserved", C.c_int32)]


class ins_file_entry(C.Structure):
    _fields_ = [("path", C.c_char * 1024), ("first_record", C.c_int32), ("n_instances", C.c_int32)]


lib.vpt_env_sky_tabulate.argtypes = [C.c_float, C.c_float, C.POINTER(C.c_float), C.c_uint, C.POINTER(C.c_float)]; lib.vpt_env_sky_tabulate.restype = C.c_int
lib.vpt_ins_load.argtypes = [C.c_char_p, C.POINTER(C.POINTER(ins_header))]; lib.vpt_ins_load.restype = C.c_int
lib.vpt_vdb_load.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_float)]
lib.vpt_vdb_load.restype = C.c_int
lib.vpt_hdr_load.argtypes = [C.c_char_p, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_uint), C.POINTER(C.c_uint)]; lib.vpt_hdr_load.restype = C.c_int
lib.vpt_bmp_load_rbg.argtypes = [C.c_char_p, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_int), C.POINTER(C.c_int)]; lib.vpt_bmp_load_rbg.restype = C.c_int
lib.vpt_exr_load_rgb.argtypes = [C.c_char_p, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_int), C.POINTER(C.c_int)]; lib.vpt_exr_load_rgb.restype = C.c_int
lib.vpt_free.argtypes = [_vp]; lib.vpt_free.restype = None
lib.vpt_octree_build.argtypes = [C.POINTER(GPU_VDB), C.c_int, C.POINTER(C.c_uint64)]; lib.vpt_octree_build.restype = C.c_int
lib.vpt_octree_destroy.argtypes = [C.c_uint64]; lib.vpt_octree_destroy.restype = C.c_int
lib.vpt_octree_read.argtypes = [C.c_uint64, C.POINTER(OCTNode), C.POINTER(C.c_int)]; lib.vpt_octree_read.restype = C.c_int
lib.vpt_octree_info.argtypes = [C.c_uint64, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_int)]; lib.vpt_octree_info.restype = C.c_int
lib.vpt_octree_read_flat.argtypes = [C.c_uint64, C.POINTER(C.c_uint), C.POINTER(C.c_int), C.c_longlong]; lib.vpt_octree_read_flat.restype = C.c_int
lib.vpt_bvh_build.argtypes = [C.POINTER(GPU_VDB), C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_float), C.POINTER(C.c_ulonglong), C.POINTER(C.c_int)]
lib.vpt_bvh_build.restype = C.c_int
lib.vpt_bvh_read.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.POINTER(BVHNode), C.POINTER(BVHNode)]; lib.vpt_bvh_read.restype = C.c_int
lib.vpt_bvh_destroy.argtypes = [C.c_uint64, C.c_uint64]; lib.vpt_bvh_destroy.restype = C.c_int
lib.vpt_volume_bounds.argtypes = [C.POINTER(GPU_VDB), C.POINTER(C.c_float)]; lib.vpt_volume_bounds.restype = None
lib.vpt_camera_look_at.argtypes = [C.POINTER(camera), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, C.c_float]
lib.vpt_camera_look_at.restype = None
lib.vpt_set_camera_motion.argtypes = [_vp, C.POINTER(camera)]; lib.vpt_set_camera_motion.restype = C.c_int
lib.vpt_debug_motion_cameras.argtypes = [_vp, C.POINTER(_vp), _vp]; lib.vpt_debug_motion_cameras.restype = C.c_int
lib.vpt_set_motion_vectors.argtypes = [_vp, _vp, C.POINTER(camera)]; lib.vpt_set_motion_vectors.restype = C.c_int
lib.vpt_set_sample_offset.argtypes = [_vp, C.c_uint32]; lib.vpt_set_sample_offset.restype = C.c_int
lib.vpt_set_collision_aovs.argtypes = [_vp, _vp, _vp, _vp, C.c_float]; lib.vpt_set_collision_aovs.restype = C.c_int
VPT_CRYPTO_MAX_ENTRIES = 32                                         # vpt_set_cryptomatte: most entries per pixel
VPT_CRYPTO_SPHERE = 0xFFFFFFFF                                      # the sphere's id in the Cryptomatte state (and the mattes' id plane)
lib.vpt_set_cryptomatte.argtypes = [_vp, _vp, C.c_uint]; lib.vpt_set_cryptomatte.restype = C.c_int
lib.vpt_cryptomatte_rank.argtypes = [_vp, C.c_uint, C.c_uint, _vp, C.c_uint, _vp, C.c_uint, C.c_float, C.c_uint, _vp, _vp, _vp]
lib.vpt_cryptomatte_rank.restype = C.c_int
lib.vpt_cryptomatte_hash.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_float)]; lib.vpt_cryptomatte_hash.restype = C.c_uint32


class temporal_options(C.Structure):
    _fields_ = [("max_history", C.c_uint), ("clip_sigma", C.c_float)]


lib.vpt_temporal_options_defaults.argtypes = [C.POINTER(temporal_options)]; lib.vpt_temporal_options_defaults.restype = None
lib.vpt_temporal.argtypes = [_vp, C.c_uint, C.c_uint, _vp, _vp, C.POINTER(camera), C.POINTER(camera), _vp, _vp, C.POINTER(temporal_options),
                             C.c_float, _vp, _vp, _vp, _vp]
lib.vpt_temporal.restype = C.c_int
VPT_TEMPORAL_MAX_LAYERS = 16


class temporal_layer(C.Structure):
    _fields_ = [("src", _vp), ("history", _vp), ("dst", _vp), ("channels", C.c_uint), ("count", C.c_uint)]


lib.vpt_temporal_layers.argtypes = [_vp, C.c_uint, C.c_uint, _vp, _vp, C.POINTER(camera), C.POINTER(camera), _vp, _vp,
                                    C.POINTER(temporal_options), C.c_float, _vp, _vp, _vp, C.POINTER(temporal_layer), C.c_uint, _vp]
lib.vpt_temporal_layers.restype = C.c_int


def temporal_defaults():
    """(max_history, clip_sigma) of vpt_temporal_options_defaults"""
    o = temporal_options()
    lib.vpt_temporal_options_defaults(C.byref(o))
    return int(o.max_history), float(o.clip_sigma)
lib.vpt_kernel_params_defaults.argtypes = [C.POINTER(Kernel_params)]; lib.vpt_kernel_params_defaults.restype = None


class VptError(RuntimeError):
    pass


def check(rc, ctx=None, what=""):
    if rc < 0:
        msg = lib.vpt_last_error(ctx).decode(errors="replace") if True else ""
        raise VptError(f"{what} failed ({rc}): {msg}")
    return rc


def fvec(vals):
    return (C.c_float * len(vals))(*[float(v) for v in vals])
