"""Every C-ABI call that takes an NvbMemory rejects a kind other than NVB_MEM_HOST and NVB_MEM_DEVICE with
NVB_ERR_INVALID_ARGUMENT, before anything is enqueued. The buffers are valid device buffers, so a call that took the kind
for device memory would run and succeed. The masker, render and scene calls are checked with their other arguments."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
BAD_KIND = 2
ROWS, COLS = 24, 32


def _call(name):
    import torch
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import _lib
    from isaac_ros_nvblox_b200.mapper import _fp, colmajor
    fs = name in ("update_freespace", "freespace_update_blocks", "compute_dynamics", "dynamic_mask", "dynamic_overlay",
                  "dynamic_points")
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64,
                   projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace if fs else nvb.ProjectiveLayerType.kTsdf)
    L, h, K = m._L, m._h, BAD_KIND
    cam = nvb.Camera(20.0, 20.0, COLS / 2, ROWS / 2, COLS, ROWS).c
    Tm = colmajor(np.eye(4, dtype=np.float32))
    T = _fp(Tm)
    dev = torch.ones(ROWS * COLS * 4, dtype=torch.float32, device="cuda")  # room for every buffer below
    b = torch.zeros(ROWS * COLS * 4, dtype=torch.uint8, device="cuda")
    d, u8 = dev.data_ptr(), b.data_ptr()
    blocks = np.zeros(3, np.int32)
    i32 = C.c_int32(0)
    i32b = C.c_int32(0)
    i64 = C.c_int64(0)
    plane = (C.c_float * 4)()
    torch.cuda.synchronize()
    calls = {
        "view_raycast": lambda: L.nvb_view_raycast(h, d, K, ROWS, COLS, T, C.byref(cam), 0.4, 0.2, 5.0, None, 0, None),
        "integrate_depth": lambda: L.nvb_mapper_integrate_depth(h, d, None, 0, K, ROWS, COLS, T, C.byref(cam), None, 0, None),
        "integrate_depth_async": lambda: L.nvb_mapper_integrate_depth_async(h, d, None, 0, K, ROWS, COLS, T, C.byref(cam)),
        "integrate_color": lambda: L.nvb_mapper_integrate_color(h, u8, None, 0, K, ROWS, COLS, T, C.byref(cam), None, 0, None),
        "decay": lambda: L.nvb_mapper_decay(h, None, d, K, ROWS, COLS, T, C.byref(cam), None, 0, None),
        "update_freespace": lambda: L.nvb_mapper_update_freespace(h, 0, d, K, ROWS, COLS, T, C.byref(cam), 0),
        "freespace_update_blocks": lambda: L.nvb_freespace_update_blocks(h, blocks.ctypes.data_as(C.POINTER(C.c_int32)), 1, 0, d,
                                                                         K, ROWS, COLS, T, C.byref(cam), 5.0, 0.2),
        "ransac_fit_plane": lambda: L.nvb_ransac_fit_plane(h, d, K, 3, 10, 0.1, plane, C.byref(i32)),
        "compute_dynamics": lambda: L.nvb_mapper_compute_dynamics(h, d, K, ROWS, COLS, T, C.byref(cam)),
        "remove_small_components": lambda: L.nvb_mapper_remove_small_components(h, u8, u8, K, ROWS, COLS, 4),
        "dynamic_mask": lambda: L.nvb_mapper_dynamic_mask(h, u8, K, C.byref(i32), C.byref(i32b)),
        "dynamic_overlay": lambda: L.nvb_mapper_dynamic_overlay(h, u8, K, C.byref(i32), C.byref(i32b)),
        "dynamic_points": lambda: L.nvb_mapper_dynamic_points(h, d, K, 8, C.byref(i32)),
        "export_points": lambda: L.nvb_layer_export_points(h, _lib.NVB_LAYER_TSDF, K, d, 8, C.byref(i64)),
        "query_voxels": lambda: L.nvb_layer_query_voxels(h, _lib.NVB_LAYER_TSDF, d, K, 8, d + 4 * 4 * 8, u8),
        "interpolate": lambda: L.nvb_layer_interpolate(h, _lib.NVB_LAYER_TSDF, d, K, 8, d + 4 * 4 * 8, u8),
    }
    try:
        return calls[name]()
    finally:
        m.close()


@pytest.mark.parametrize("name", ["view_raycast", "integrate_depth", "integrate_depth_async", "integrate_color", "decay",
                                  "update_freespace", "freespace_update_blocks", "ransac_fit_plane", "compute_dynamics",
                                  "remove_small_components", "dynamic_mask", "dynamic_overlay", "dynamic_points",
                                  "export_points", "query_voxels", "interpolate"])
def test_bad_memory_kind_is_rejected(gpu, name):
    assert _call(name) == -1  # NVB_ERR_INVALID_ARGUMENT
