"""ctypes binding of the C-ABI (include/nvblox_b200.h -> libnvblox_b200.so).

The product path has no CPU fallback: if the CUDA library is missing this module
raises at load() time, and nvb_mapper_create fails with NVB_ERR_NO_DEVICE when no
GPU is visible.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnvblox_b200.so")

NVB_OK = 0
NVB_ERR_INDEX_RANGE, NVB_ERR_IO = -4, -6
NVB_MEM_HOST, NVB_MEM_DEVICE = 0, 1
NVB_LAYER_TSDF, NVB_LAYER_ESDF, NVB_LAYER_OCCUPANCY, NVB_LAYER_FREESPACE, NVB_LAYER_COLOR, NVB_LAYER_MESH = 0, 1, 2, 3, 4, 5
NVB_PROJECTIVE_TSDF, NVB_PROJECTIVE_OCCUPANCY, NVB_PROJECTIVE_TSDF_WITH_FREESPACE = 0, 1, 2
NVB_SPLIT_BACKGROUND, NVB_SPLIT_FOREGROUND, NVB_SPLIT_OVERLAY = 0, 1, 2

# Every symbol include/nvblox_b200.h declares (checked by tests/test_cabi_symbols.py).
EXPORTED_SYMBOLS = [
    "nvb_last_error", "nvb_version", "nvb_device_count",
    "nvb_default_mapper_options", "nvb_default_tsdf_params", "nvb_default_esdf_params",
    "nvb_default_occupancy_params", "nvb_mapper_set_occupancy_params", "nvb_mapper_get_occupancy_params",
    "nvb_default_tsdf_decay_params", "nvb_mapper_set_tsdf_decay_params", "nvb_mapper_get_tsdf_decay_params",
    "nvb_default_occupancy_decay_params", "nvb_mapper_set_occupancy_decay_params",
    "nvb_mapper_get_occupancy_decay_params", "nvb_mapper_decay", "nvb_mapper_decay_exclude_last_view",
    "nvb_default_freespace_params", "nvb_mapper_set_freespace_params", "nvb_mapper_get_freespace_params",
    "nvb_mapper_update_freespace", "nvb_freespace_update_blocks",
    "nvb_mapper_mark_unobserved_free_inside_radius",
    "nvb_default_color_params", "nvb_mapper_set_color_params", "nvb_mapper_get_color_params",
    "nvb_mapper_integrate_color", "nvb_mapper_last_color_blocks", "nvb_sphere_tracer_render_depth",
    "nvb_default_esdf_slice_params", "nvb_mapper_set_esdf_slice_params", "nvb_mapper_get_esdf_slice_params",
    "nvb_mapper_update_esdf_slice", "nvb_esdf_integrate_slice_blocks", "nvb_esdf_slice_distance_image",
    "nvb_mapper_update_esdf_slice_planar", "nvb_esdf_integrate_slice_planar_blocks",
    "nvb_mapper_create", "nvb_mapper_destroy", "nvb_mapper_clear",
    "nvb_mapper_set_tsdf_params", "nvb_mapper_get_tsdf_params",
    "nvb_mapper_set_esdf_params", "nvb_mapper_get_esdf_params",
    "nvb_mapper_voxel_size", "nvb_mapper_block_size",
    "nvb_view_raycast", "nvb_mapper_integrate_depth", "nvb_mapper_integrate_depth_async",
    "nvb_mapper_update_esdf", "nvb_mapper_update_esdf_async", "nvb_esdf_integrate_blocks",
    "nvb_mapper_synchronize", "nvb_mapper_last_frame_block_count", "nvb_mapper_last_frame_blocks",
    "nvb_mapper_stream", "nvb_mapper_join_streams", "nvb_blocks_union",
    "nvb_layer_num_blocks", "nvb_layer_block_indices", "nvb_layer_slab_stats", "nvb_layer_get_blocks",
    "nvb_layer_set_blocks", "nvb_layer_block_device_ptr", "nvb_layer_block_bytes",
    "nvb_mapper_last_esdf_stats", "nvb_mapper_set_cache_last_viewpoint", "nvb_mapper_get_cache_last_viewpoint", "nvb_mapper_set_depth_preprocessing", "nvb_mapper_get_depth_preprocessing", "nvb_depth_dilate_invalid", "nvb_esdf_slice_aabb", "nvb_esdf_dense_grid_in_aabb", "nvb_esdf_slice_distance_image_in_aabb", "nvb_mapper_set_esdf_reserved_sms", "nvb_mapper_get_esdf_reserved_sms", "nvb_default_mesh_params", "nvb_mapper_set_mesh_params", "nvb_mapper_get_mesh_params", "nvb_mapper_update_mesh", "nvb_mesh_integrate_blocks", "nvb_mesh_update_color", "nvb_mesh_block_sizes", "nvb_mesh_get_blocks", "nvb_mesh_arena_stats", "nvb_mapper_append_frame_blocks", "nvb_blocks_union_segments", "nvb_blocks_union_status", "nvb_mapper_esdf_time_split", "nvb_mapper_esdf_clear_blocks_read", "nvb_mapper_debug_phase_max", "nvb_mapper_enable_profiling", "nvb_mapper_stage_times",
    "nvb_mapper_kernel_launches", "nvb_mapper_esdf_split_stats",
    "nvb_mapper_clear_outside_radius", "nvb_mapper_clear_tsdf_inside_shapes", "nvb_layer_clear_shapes",
    "nvb_mapper_get_cleared_blocks",
    "nvb_default_ground_plane_params", "nvb_mapper_set_ground_plane_params", "nvb_mapper_get_ground_plane_params",
    "nvb_mapper_compute_ground_plane", "nvb_mapper_ground_plane", "nvb_mapper_ground_plane_points", "nvb_ransac_fit_plane",
    "nvb_mapper_compute_dynamics", "nvb_mapper_remove_small_components", "nvb_mapper_dynamic_mask", "nvb_mapper_dynamic_overlay",
    "nvb_mapper_dynamic_points", "nvb_mapper_dynamics_device_buffers", "nvb_mapper_wait_for",
    "nvb_default_image_masker_params", "nvb_mapper_split_depth_image", "nvb_mapper_split_output",
    "nvb_mapper_split_device_buffers", "nvb_mapper_split_color_image",
    "nvb_layer_query_voxels", "nvb_layer_interpolate", "nvb_query_esdf", "nvb_query_tsdf", "nvb_query_occupancy",
    "nvb_mapper_save_map", "nvb_mapper_load_map", "nvb_layer_export_points",
    "nvb_default_sphere_tracer_params", "nvb_render_depth", "nvb_render_rgbd",
    "nvb_scene_render_depth", "nvb_scene_signed_distance", "nvb_scene_generate_layer", "nvb_scene_to_mapper",
]


class NvbCamera(C.Structure):
    _fields_ = [("fu", C.c_float), ("fv", C.c_float), ("cu", C.c_float), ("cv", C.c_float),
                ("width", C.c_int32), ("height", C.c_int32), ("has_distortion", C.c_int32),
                ("k1", C.c_float), ("k2", C.c_float), ("k3", C.c_float), ("k4", C.c_float),
                ("k5", C.c_float), ("k6", C.c_float), ("p1", C.c_float), ("p2", C.c_float)]


class NvbTsdfParams(C.Structure):
    _fields_ = [("truncation_distance_vox", C.c_float),
                ("max_integration_distance_m", C.c_float),
                ("max_weight", C.c_float),
                ("invalid_depth_decay_factor", C.c_float),
                ("weighting_type", C.c_int32),
                ("raycast_subsampling", C.c_int32),
                ("workspace_bounds_type", C.c_int32),
                ("workspace_min", C.c_float * 3),
                ("workspace_max", C.c_float * 3)]


class NvbEsdfParams(C.Structure):
    _fields_ = [("max_esdf_distance_m", C.c_float),
                ("max_site_distance_vox", C.c_float),
                ("min_weight", C.c_float),
                ("occupied_threshold", C.c_float)]


class NvbOccupancyParams(C.Structure):
    _fields_ = [("free_region_occupancy_probability", C.c_float),
                ("occupied_region_occupancy_probability", C.c_float),
                ("unobserved_region_occupancy_probability", C.c_float),
                ("occupied_region_half_width_m", C.c_float)]


class NvbMeshParams(C.Structure):
    _fields_ = [("min_weight", C.c_float), ("weld_vertices", C.c_int32), ("cutoff_distance_vox", C.c_float)]


class NvbEsdfSliceParams(C.Structure):
    _fields_ = [("slice_min_height_m", C.c_float), ("slice_max_height_m", C.c_float), ("slice_height_m", C.c_float),
                ("slice_height_above_plane_m", C.c_float), ("slice_height_thickness_m", C.c_float)]


class NvbColorParams(C.Structure):
    _fields_ = [("max_integration_distance_m", C.c_float), ("truncation_distance_vox", C.c_float),
                ("max_weight", C.c_float), ("measurement_weight", C.c_float),
                ("sphere_tracing_ray_subsampling_factor", C.c_int32), ("sphere_tracer_maximum_steps", C.c_int32),
                ("sphere_tracer_maximum_ray_length_m", C.c_float), ("sphere_tracer_surface_distance_epsilon_vox", C.c_float),
                ("workspace_bounds_type", C.c_int32), ("workspace_min", C.c_float * 3), ("workspace_max", C.c_float * 3)]


class NvbSphereTracerParams(C.Structure):
    _fields_ = [("maximum_steps", C.c_int32), ("maximum_ray_length_m", C.c_float),
                ("surface_distance_epsilon_vox", C.c_float)]


NVB_PRIM_PLANE, NVB_PRIM_CUBE, NVB_PRIM_SPHERE, NVB_PRIM_CYLINDER = 0, 1, 2, 3


class NvbPrimitive(C.Structure):
    _fields_ = [("type", C.c_int32), ("center", C.c_float * 3), ("params", C.c_float * 4)]


class NvbScene(C.Structure):
    _fields_ = [("primitives", C.POINTER(NvbPrimitive)), ("num_primitives", C.c_int32), ("aabb_min", C.c_float * 3),
                ("aabb_max", C.c_float * 3)]


class NvbFreespaceParams(C.Structure):
    _fields_ = [("max_tsdf_distance_for_occupancy_m", C.c_float),
                ("max_unobserved_to_keep_consecutive_occupancy_ms", C.c_int64),
                ("min_duration_since_occupied_for_freespace_ms", C.c_int64),
                ("min_consecutive_occupancy_duration_for_reset_ms", C.c_int64),
                ("check_neighborhood", C.c_int32), ("initialize_to_high_confidence_freespace", C.c_int32)]


class NvbTsdfDecayParams(C.Structure):
    _fields_ = [("decay_factor", C.c_float), ("decayed_weight_threshold", C.c_float),
                ("set_free_distance_on_decayed", C.c_int32), ("free_distance_vox", C.c_float),
                ("deallocate_decayed_blocks", C.c_int32)]


class NvbOccupancyDecayParams(C.Structure):
    _fields_ = [("free_region_decay_probability", C.c_float), ("occupied_region_decay_probability", C.c_float),
                ("decay_to_probability", C.c_float), ("deallocate_decayed_blocks", C.c_int32)]


class NvbDecayExclusion(C.Structure):
    _fields_ = [("excluded_blocks_xyz_host", C.POINTER(C.c_int32)), ("num_excluded_blocks", C.c_int32),
                ("has_exclusion_sphere", C.c_int32), ("exclusion_center", C.c_float * 3),
                ("exclusion_radius_m", C.c_float)]


NVB_SHAPE_SPHERE, NVB_SHAPE_AABB = 0, 1


class NvbBoundingShape(C.Structure):
    _fields_ = [("type", C.c_int32), ("a", C.c_float * 3), ("b", C.c_float * 3)]


NVB_GROUND_POINTS_CROSSINGS, NVB_GROUND_POINTS_CANDIDATES = 0, 1


class NvbGroundPlaneParams(C.Structure):
    _fields_ = [("ground_points_candidates_min_z_m", C.c_float), ("ground_points_candidates_max_z_m", C.c_float),
                ("ransac_distance_threshold_m", C.c_float), ("num_ransac_iterations", C.c_int32),
                ("min_tsdf_weight", C.c_float), ("max_crossings", C.c_int32)]


class NvbDynamicsBuffers(C.Structure):
    _fields_ = [("depth", C.c_void_p), ("mask", C.c_void_p), ("cleaned_mask", C.c_void_p), ("overlay", C.c_void_p),
                ("points", C.c_void_p), ("num_points", C.c_void_p), ("rows", C.c_int32), ("cols", C.c_int32)]


class NvbImageMaskerParams(C.Structure):
    _fields_ = [("occlusion_threshold_m", C.c_float), ("depth_masked_image_invalid_pixel", C.c_float),
                ("depth_unmasked_image_invalid_pixel", C.c_float)]


class NvbSplitBuffers(C.Structure):
    _fields_ = [("background", C.c_void_p), ("foreground", C.c_void_p), ("overlay", C.c_void_p), ("rows", C.c_int32),
                ("cols", C.c_int32)]


class NvbMapperOptions(C.Structure):
    _fields_ = [("voxel_size_m", C.c_float), ("device", C.c_int32),
                ("tsdf_capacity_blocks", C.c_int32), ("esdf_capacity_blocks", C.c_int32),
                ("esdf_persistent", C.c_int32), ("projective_layer_type", C.c_int32),
                ("keep_last_view", C.c_int32)]


class NvbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("nvblox_b200 error %d: %s" % (code, msg))
        self.code = code


_lib = None


def load(path=None):
    """Load libnvblox_b200.so (build it first with build_ext.build()). `path` overrides LIB_PATH (a variant build, e.g. the
    profiling library of tools/wavex_profile.py); it has to be given before the first load of the process."""
    global _lib, LIB_PATH
    if path is not None and _lib is None:
        LIB_PATH = path
    elif path is not None and os.path.abspath(path) != os.path.abspath(LIB_PATH):
        raise RuntimeError("%s is already loaded; cannot switch to %s" % (LIB_PATH, path))
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback for the depth-integration path." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
    fp, ip, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
    L.nvb_last_error.restype = C.c_char_p
    L.nvb_version.restype = C.c_char_p
    L.nvb_device_count.restype = i32
    L.nvb_default_mapper_options.argtypes = [C.POINTER(NvbMapperOptions)]
    L.nvb_default_tsdf_params.argtypes = [C.POINTER(NvbTsdfParams)]
    L.nvb_default_esdf_params.argtypes = [C.POINTER(NvbEsdfParams)]
    L.nvb_default_occupancy_params.argtypes = [C.POINTER(NvbOccupancyParams)]
    L.nvb_default_occupancy_params.restype = None
    L.nvb_mapper_set_occupancy_params.argtypes = [vp, C.POINTER(NvbOccupancyParams)]
    L.nvb_mapper_get_occupancy_params.argtypes = [vp, C.POINTER(NvbOccupancyParams)]
    L.nvb_default_tsdf_decay_params.argtypes = [C.POINTER(NvbTsdfDecayParams)]
    L.nvb_default_tsdf_decay_params.restype = None
    L.nvb_mapper_set_tsdf_decay_params.argtypes = [vp, C.POINTER(NvbTsdfDecayParams)]
    L.nvb_mapper_get_tsdf_decay_params.argtypes = [vp, C.POINTER(NvbTsdfDecayParams)]
    L.nvb_default_occupancy_decay_params.argtypes = [C.POINTER(NvbOccupancyDecayParams)]
    L.nvb_default_occupancy_decay_params.restype = None
    L.nvb_mapper_set_occupancy_decay_params.argtypes = [vp, C.POINTER(NvbOccupancyDecayParams)]
    L.nvb_mapper_get_occupancy_decay_params.argtypes = [vp, C.POINTER(NvbOccupancyDecayParams)]
    L.nvb_mapper_decay.argtypes = [vp, C.POINTER(NvbDecayExclusion), vp, i32, i32, i32, fp, C.POINTER(NvbCamera), ip, i32, ip]
    L.nvb_default_esdf_slice_params.argtypes = [C.POINTER(NvbEsdfSliceParams)]
    L.nvb_default_esdf_slice_params.restype = None
    L.nvb_mapper_set_esdf_slice_params.argtypes = [vp, C.POINTER(NvbEsdfSliceParams)]
    L.nvb_mapper_get_esdf_slice_params.argtypes = [vp, C.POINTER(NvbEsdfSliceParams)]
    L.nvb_mapper_update_esdf_slice.argtypes = [vp, i32]
    L.nvb_esdf_integrate_slice_blocks.argtypes = [vp, ip, i32]
    L.nvb_mapper_update_esdf_slice_planar.argtypes = [vp, fp, i32]
    L.nvb_esdf_integrate_slice_planar_blocks.argtypes = [vp, fp, ip, i32]
    L.nvb_esdf_slice_distance_image.argtypes = [vp, f32, f32, fp, fp, C.POINTER(C.c_int8), i32, ip, ip]
    L.nvb_mapper_mark_unobserved_free_inside_radius.argtypes = [vp, fp, f32, ip, i32, ip]
    L.nvb_default_color_params.argtypes = [C.POINTER(NvbColorParams)]
    L.nvb_default_color_params.restype = None
    L.nvb_mapper_set_color_params.argtypes = [vp, C.POINTER(NvbColorParams)]
    L.nvb_mapper_get_color_params.argtypes = [vp, C.POINTER(NvbColorParams)]
    L.nvb_mapper_integrate_color.argtypes = [vp, vp, vp, i32, i32, i32, i32, fp, C.POINTER(NvbCamera), ip, i32, ip]
    L.nvb_mapper_last_color_blocks.argtypes = [vp, ip, i32, ip]
    L.nvb_sphere_tracer_render_depth.argtypes = [vp, fp, C.POINTER(NvbCamera), f32, i32, fp]
    L.nvb_default_freespace_params.argtypes = [C.POINTER(NvbFreespaceParams)]
    L.nvb_default_freespace_params.restype = None
    L.nvb_mapper_set_freespace_params.argtypes = [vp, C.POINTER(NvbFreespaceParams)]
    L.nvb_mapper_get_freespace_params.argtypes = [vp, C.POINTER(NvbFreespaceParams)]
    L.nvb_mapper_update_freespace.argtypes = [vp, C.c_int64, vp, i32, i32, i32, fp, C.POINTER(NvbCamera), i32]
    L.nvb_freespace_update_blocks.argtypes = [vp, ip, i32, C.c_int64, vp, i32, i32, i32, fp, C.POINTER(NvbCamera), f32, f32]
    L.nvb_mapper_decay_exclude_last_view.argtypes = [vp, C.POINTER(NvbDecayExclusion), ip, i32, ip]
    L.nvb_mapper_create.argtypes = [C.POINTER(NvbMapperOptions), C.POINTER(vp)]
    L.nvb_mapper_create.restype = i32
    L.nvb_mapper_destroy.argtypes = [vp]
    L.nvb_mapper_destroy.restype = None
    L.nvb_mapper_clear.argtypes = [vp]
    L.nvb_mapper_set_tsdf_params.argtypes = [vp, C.POINTER(NvbTsdfParams)]
    L.nvb_mapper_get_tsdf_params.argtypes = [vp, C.POINTER(NvbTsdfParams)]
    L.nvb_mapper_set_esdf_params.argtypes = [vp, C.POINTER(NvbEsdfParams)]
    L.nvb_mapper_get_esdf_params.argtypes = [vp, C.POINTER(NvbEsdfParams)]
    L.nvb_mapper_voxel_size.argtypes = [vp]
    L.nvb_mapper_voxel_size.restype = f32
    L.nvb_mapper_block_size.argtypes = [vp]
    L.nvb_mapper_block_size.restype = f32
    L.nvb_view_raycast.argtypes = [vp, vp, i32, i32, i32, fp, C.POINTER(NvbCamera), f32, f32, f32, ip, i32, ip]
    L.nvb_mapper_integrate_depth.argtypes = [vp, vp, vp, i32, i32, i32, i32, fp, C.POINTER(NvbCamera), ip, i32, ip]
    L.nvb_mapper_integrate_depth_async.argtypes = [vp, vp, vp, i32, i32, i32, i32, fp, C.POINTER(NvbCamera)]
    L.nvb_mapper_update_esdf.argtypes = [vp, i32]
    L.nvb_mapper_update_esdf_async.argtypes = [vp, i32]
    L.nvb_esdf_integrate_blocks.argtypes = [vp, ip, i32]
    L.nvb_mapper_synchronize.argtypes = [vp]
    L.nvb_mapper_last_frame_block_count.argtypes = [vp, ip]
    L.nvb_mapper_last_frame_blocks.argtypes = [vp, ip, i32, ip]
    L.nvb_mapper_join_streams.argtypes = [vp]
    L.nvb_blocks_union.argtypes = [vp, vp, i32, ip, ip, vp, i32, ip]
    L.nvb_mapper_stream.argtypes = [vp]
    L.nvb_mapper_stream.restype = vp
    L.nvb_layer_num_blocks.argtypes = [vp, i32, ip]
    L.nvb_layer_block_indices.argtypes = [vp, i32, ip, i32, ip]
    L.nvb_layer_slab_stats.argtypes = [vp, i32, C.POINTER(C.c_int64)]
    L.nvb_layer_get_blocks.argtypes = [vp, i32, ip, i32, vp, u8p]
    L.nvb_layer_set_blocks.argtypes = [vp, i32, ip, i32, vp]
    L.nvb_layer_block_device_ptr.argtypes = [vp, i32, ip, C.POINTER(vp)]
    L.nvb_layer_block_bytes.argtypes = [i32]
    L.nvb_mapper_save_map.argtypes = [vp, C.c_char_p]
    L.nvb_mapper_load_map.argtypes = [vp, C.c_char_p, ip]
    L.nvb_layer_export_points.argtypes = [vp, i32, i32, vp, C.c_int64, C.POINTER(C.c_int64)]
    L.nvb_mapper_last_esdf_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    L.nvb_mapper_set_cache_last_viewpoint.argtypes = [vp, C.c_int32]
    L.nvb_mapper_get_cache_last_viewpoint.argtypes = [vp]
    L.nvb_mapper_set_depth_preprocessing.argtypes = [vp, C.c_int32, C.c_int32]
    L.nvb_mapper_get_depth_preprocessing.argtypes = [vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.nvb_depth_dilate_invalid.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float]
    L.nvb_esdf_slice_aabb.argtypes = [vp, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    L.nvb_esdf_dense_grid_in_aabb.argtypes = [vp, C.POINTER(C.c_float), C.c_float, i32, vp, C.c_int64, ip, ip]
    L.nvb_esdf_slice_distance_image_in_aabb.argtypes = [vp, C.c_float, C.c_float, C.POINTER(C.c_float), vp, vp, C.c_int32,
                                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.nvb_mapper_set_esdf_reserved_sms.argtypes = [vp, C.c_int32]
    L.nvb_mapper_get_esdf_reserved_sms.argtypes = [vp]
    L.nvb_default_mesh_params.argtypes = [C.POINTER(NvbMeshParams)]
    L.nvb_default_mesh_params.restype = None
    L.nvb_mapper_set_mesh_params.argtypes = [vp, C.POINTER(NvbMeshParams)]
    L.nvb_mapper_get_mesh_params.argtypes = [vp, C.POINTER(NvbMeshParams)]
    L.nvb_mapper_update_mesh.argtypes = [vp, C.c_int32]
    L.nvb_mesh_integrate_blocks.argtypes = [vp, C.POINTER(C.c_int32), C.c_int32, C.c_int32]
    L.nvb_mesh_update_color.argtypes = [vp, C.POINTER(C.c_int32), C.c_int32]
    L.nvb_mesh_block_sizes.argtypes = [vp, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32)]
    L.nvb_mesh_get_blocks.argtypes = [vp, C.POINTER(C.c_int32), C.c_int32, vp, vp, vp, vp, C.POINTER(C.c_int64)]
    L.nvb_mesh_arena_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    L.nvb_mapper_append_frame_blocks.argtypes = [vp, vp, C.c_int32]
    L.nvb_blocks_union_segments.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp]
    L.nvb_blocks_union_status.argtypes = [vp, C.POINTER(C.c_int32)]
    L.nvb_mapper_esdf_time_split.argtypes = [vp, C.POINTER(C.c_int64)]
    L.nvb_mapper_esdf_clear_blocks_read.argtypes = [vp, C.POINTER(C.c_int64)]
    L.nvb_mapper_esdf_split_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    L.nvb_mapper_debug_phase_max.argtypes = [vp, C.POINTER(C.c_int64), i32]
    L.nvb_mapper_enable_profiling.argtypes = [vp, i32]
    L.nvb_mapper_stage_times.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_int64), i32]
    L.nvb_mapper_kernel_launches.argtypes = [vp]
    L.nvb_mapper_clear_outside_radius.argtypes = [vp, fp, f32, ip, i32, ip]
    L.nvb_mapper_clear_tsdf_inside_shapes.argtypes = [vp, C.POINTER(NvbBoundingShape), i32, ip, i32, ip]
    L.nvb_layer_clear_shapes.argtypes = [vp, i32, C.POINTER(NvbBoundingShape), i32, ip, i32, ip]
    L.nvb_mapper_get_cleared_blocks.argtypes = [vp, ip, i32, ip, i32, ip]
    L.nvb_default_ground_plane_params.argtypes = [C.POINTER(NvbGroundPlaneParams)]
    L.nvb_default_ground_plane_params.restype = None
    L.nvb_mapper_set_ground_plane_params.argtypes = [vp, C.POINTER(NvbGroundPlaneParams)]
    L.nvb_mapper_get_ground_plane_params.argtypes = [vp, C.POINTER(NvbGroundPlaneParams)]
    L.nvb_mapper_compute_ground_plane.argtypes = [vp, fp, ip]
    L.nvb_mapper_ground_plane.argtypes = [vp, fp, ip]
    L.nvb_mapper_ground_plane_points.argtypes = [vp, i32, fp, i32, ip, ip]
    L.nvb_ransac_fit_plane.argtypes = [vp, vp, i32, i32, i32, f32, fp, ip]
    L.nvb_mapper_compute_dynamics.argtypes = [vp, vp, i32, i32, i32, fp, C.POINTER(NvbCamera)]
    L.nvb_mapper_remove_small_components.argtypes = [vp, vp, vp, i32, i32, i32, i32]
    L.nvb_mapper_dynamic_mask.argtypes = [vp, vp, i32, ip, ip]
    L.nvb_mapper_dynamic_overlay.argtypes = [vp, vp, i32, ip, ip]
    L.nvb_mapper_dynamic_points.argtypes = [vp, vp, i32, i32, ip]
    L.nvb_mapper_dynamics_device_buffers.argtypes = [vp, C.POINTER(NvbDynamicsBuffers)]
    L.nvb_mapper_wait_for.argtypes = [vp, vp]
    L.nvb_default_image_masker_params.argtypes = [C.POINTER(NvbImageMaskerParams)]
    L.nvb_default_image_masker_params.restype = None
    L.nvb_mapper_split_depth_image.argtypes = [vp, vp, i32, i32, vp, i32, i32, i32, fp, C.POINTER(NvbCamera),
                                               C.POINTER(NvbCamera), C.POINTER(NvbImageMaskerParams), i32]
    L.nvb_mapper_split_output.argtypes = [vp, i32, vp, i32, ip, ip]
    L.nvb_mapper_split_device_buffers.argtypes = [vp, C.POINTER(NvbSplitBuffers)]
    L.nvb_mapper_split_color_image.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp]
    i64 = C.c_int64
    L.nvb_layer_query_voxels.argtypes = [vp, i32, vp, i32, i64, vp, vp]
    L.nvb_layer_interpolate.argtypes = [vp, i32, vp, i32, i64, vp, vp]
    L.nvb_query_esdf.argtypes = [C.POINTER(vp), i32, vp, i64, i32, vp, vp]
    L.nvb_query_tsdf.argtypes = [C.POINTER(vp), i32, vp, i64, vp, vp]
    L.nvb_query_occupancy.argtypes = [C.POINTER(vp), i32, vp, i64, vp, vp]
    L.nvb_default_sphere_tracer_params.argtypes = [C.POINTER(NvbSphereTracerParams)]
    L.nvb_default_sphere_tracer_params.restype = None
    L.nvb_render_depth.argtypes = [vp, C.POINTER(NvbSphereTracerParams), fp, C.POINTER(NvbCamera), f32, i32, i32, vp, vp]
    L.nvb_render_rgbd.argtypes = [vp, C.POINTER(NvbSphereTracerParams), fp, C.POINTER(NvbCamera), f32, i32, i32, vp, vp, vp]
    L.nvb_scene_render_depth.argtypes = [C.POINTER(NvbScene), C.POINTER(NvbCamera), fp, f32, f32, i32, vp, vp]
    L.nvb_scene_signed_distance.argtypes = [C.POINTER(NvbScene), vp, i32, i64, f32, vp, vp]
    L.nvb_scene_generate_layer.argtypes = [vp, i32, C.POINTER(NvbScene), f32]
    L.nvb_scene_to_mapper.argtypes = [vp, C.POINTER(NvbScene)]
    L.nvb_mapper_kernel_launches.restype = C.c_int64
    for name in EXPORTED_SYMBOLS:
        f = getattr(L, name)
        if f.restype is C.c_int and name not in ("nvb_device_count", "nvb_layer_block_bytes"):
            f.restype = i32
    _lib = L
    return L


def check(rc):
    if rc != NVB_OK:
        raise NvbError(rc, load().nvb_last_error().decode("utf-8", "replace"))
