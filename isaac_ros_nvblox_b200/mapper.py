"""Host-side mirror of nvblox::Mapper for the depth-integration path.

Same names and argument meaning as the reference's C++ classes, restricted to this
path (nvblox/include/nvblox/mapper/mapper.h:107-836):
    Mapper(voxel_size_m)                       mapper.h:119-124
    Mapper.integrate_depth(depth, T_L_C, cam)  mapper.h:167-172  (integrateDepth)
    Mapper.update_esdf()                       mapper.h:326      (updateEsdf)
    Mapper.tsdf_layer() / esdf_layer()         mapper.h:372,393
    Mapper.tsdf_integrator() / esdf_integrator()  parameter setters
    Mapper(voxel_size_m, projective_layer_type=ProjectiveLayerType.kOccupancy)  mapper.h:52-53,119-124
    Mapper.occupancy_layer() / occupancy_integrator()  mapper.h:374,456
    ViewCalculator.get_blocks_in_image_view_raycast  view_calculator.h:75-80
Everything forwards to the C-ABI in libnvblox_b200.so through ctypes; numpy arrays
are host buffers, integers are raw device pointers.
"""
import ctypes as C
import os

import numpy as np

from . import _lib
from . import io as _io
from ._lib import (NvbBoundingShape, NvbCamera, NvbDecayExclusion, NvbEsdfParams, NvbEsdfSliceParams, NvbFreespaceParams, NvbGroundPlaneParams, NvbMapperOptions, NvbOccupancyDecayParams,
                   NvbOccupancyParams, NvbTsdfDecayParams, NvbTsdfParams, check)

TSDF_VOXEL_DTYPE = np.dtype([("distance", "<f4"), ("weight", "<f4")])
ESDF_VOXEL_DTYPE = np.dtype(
    [("squared_distance_vox", "<f4"), ("parent_direction", "<i4", (3,)),
     ("is_inside", "u1"), ("observed", "u1"), ("is_site", "u1"), ("pad", "u1")])

OCCUPANCY_VOXEL_DTYPE = np.dtype([("log_odds", "<f4")])  # map/voxels.h:51-53
COLOR_VOXEL_DTYPE = np.dtype([("color", "u1", (3,)), ("pad", "u1"), ("weight", "<f4")])  # ColorVoxel (map/voxels.h:77-83)
FREESPACE_VOXEL_DTYPE = np.dtype([("last_occupied_timestamp_ms", "<i8"), ("consecutive_occupancy_duration_ms", "<i8"),
                                  ("is_high_confidence_freespace", "u1"), ("pad", "u1", (7,))])  # map/voxels.h:38-52


class ProjectiveLayerType:
    """mapper/mapper.h:52-53."""
    kTsdf = _lib.NVB_PROJECTIVE_TSDF
    kOccupancy = _lib.NVB_PROJECTIVE_OCCUPANCY
    kTsdfWithFreespace = _lib.NVB_PROJECTIVE_TSDF_WITH_FREESPACE


STAGE_NAMES = ("view_calculator/raycast", "tsdf/integrate/allocate_blocks", "tsdf/integrate/update_blocks",
               "esdf/integrate/mark_sites", "esdf/integrate/clear", "esdf/integrate/compute")


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def colmajor(T):
    """4x4 transform -> 16 float32 in Eigen::Isometry3f::data() (column-major) order."""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float32).T).reshape(16)


class Camera:
    """nvblox::Camera(fu, fv, cu, cv, width, height, distortion_params) (sensors/camera.h:33-203).
    radial = (k1..k6), tangential = (p1, p2) = RadialTangentialDistortionParams; None = std::nullopt."""

    def __init__(self, fu, fv, cu, cv, width, height, radial=None, tangential=None):
        has = radial is not None or tangential is not None
        k = [float(v) for v in (radial or (0, 0, 0, 0, 0, 0))]
        p = [float(v) for v in (tangential or (0, 0))]
        self.c = NvbCamera(float(fu), float(fv), float(cu), float(cv), int(width), int(height), 1 if has else 0,
                           *k, *p)

    fu = property(lambda s: s.c.fu)
    fv = property(lambda s: s.c.fv)
    cu = property(lambda s: s.c.cu)
    cv = property(lambda s: s.c.cv)
    width = property(lambda s: s.c.width)
    height = property(lambda s: s.c.height)


class BoundingSphere:
    """nvblox::BoundingSphere(center, radius) (geometry/bounding_spheres.h): contains p when |center - p| <= radius."""

    def __init__(self, center, radius):
        self.center = np.asarray(center, dtype=np.float32).reshape(3)
        self.radius = np.float32(radius)

    def _c(self):
        return NvbBoundingShape(_lib.NVB_SHAPE_SPHERE, (C.c_float * 3)(*self.center.tolist()),
                                (C.c_float * 3)(float(self.radius), 0.0, 0.0))


class AxisAlignedBoundingBox:
    """nvblox::AxisAlignedBoundingBox(min, max) (Eigen::AlignedBox3f, geometry/bounding_boxes.h): inclusive on both sides."""

    def __init__(self, min, max):  # noqa: A002 (the reference's argument names)
        self.min = np.asarray(min, dtype=np.float32).reshape(3)
        self.max = np.asarray(max, dtype=np.float32).reshape(3)

    def _c(self):
        return NvbBoundingShape(_lib.NVB_SHAPE_AABB, (C.c_float * 3)(*self.min.tolist()), (C.c_float * 3)(*self.max.tolist()))


def _shape_array(shapes):
    shapes = list(shapes)
    arr = (NvbBoundingShape * max(len(shapes), 1))()
    for i, s in enumerate(shapes):
        arr[i] = s._c()
    return arr, len(shapes)


def _block_list(fn, cap, *args, reread=None):
    """Call fn(*args, out, cap, &n), which returns a list of n block indices with at most `cap` of them in `out`, and return
    the (n, 3) int32 indices it wrote. A list longer than `cap` is read again in full through `reread`, (fn, *args) of an
    entry point that returns the same list without changing the map; without one, the first `cap` indices are returned."""
    cap = max(int(cap), 1)
    out = np.empty((cap, 3), dtype=np.int32)
    n = C.c_int32(0)
    check(fn(*args, _ip(out), cap, C.byref(n)))
    if n.value > cap and reread is not None:
        return _block_list(reread[0], n.value, *reread[1:])
    return out[:n.value].copy()


class _Layer:
    """BlockLayer queries (map/layer.h:76-311) answered from the device-resident map."""

    def __init__(self, mapper, layer_id, dtype):
        self._m, self._id, self._dtype = mapper, layer_id, dtype

    def num_blocks(self):
        n = C.c_int32(0)
        check(self._m._L.nvb_layer_num_blocks(self._m._h, self._id, C.byref(n)))
        return n.value

    def get_all_block_indices(self):
        return _block_list(self._m._L.nvb_layer_block_indices, self.num_blocks(), self._m._h, self._id)

    def slab_stats(self):
        """Storage of the layer: slab capacity, high-water mark and free-stack size in blocks, and the hash-table size."""
        out = (C.c_int64 * 4)()
        check(self._m._L.nvb_layer_slab_stats(self._m._h, self._id, out))
        return {"capacity": out[0], "high_water": out[1], "free": out[2], "hash_size": out[3]}

    def get_blocks(self, indices):
        """(n,3) int32 -> ((n,8,8,8) voxel array, (n,) found mask)."""
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        n = idx.shape[0]
        out = np.zeros((max(n, 1), 8, 8, 8), dtype=self._dtype)
        found = np.zeros(max(n, 1), dtype=np.uint8)
        check(self._m._L.nvb_layer_get_blocks(self._m._h, self._id, _ip(idx), n, out.ctypes.data,
                                              found.ctypes.data_as(C.POINTER(C.c_uint8))))
        return out[:n], found[:n].astype(bool)

    def get_block_at_index(self, index):
        v, f = self.get_blocks(np.asarray(index, dtype=np.int32).reshape(1, 3))
        return v[0] if f[0] else None

    def is_block_allocated(self, index):
        return self.get_block_at_index(index) is not None

    def set_blocks(self, indices, voxels):
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        v = np.ascontiguousarray(voxels, dtype=self._dtype).reshape(idx.shape[0], 8, 8, 8)
        check(self._m._L.nvb_layer_set_blocks(self._m._h, self._id, _ip(idx), idx.shape[0], v.ctypes.data))

    def clear_shapes(self, shapes):
        """ShapeClearer<LayerType>::clear(shapes, layer) (integrators/shape_clearer.h) on a TSDF, occupancy or colour layer:
        voxels whose centre lies in a BoundingSphere / AxisAlignedBoundingBox are reset. The tracker is not told. Returns the
        touched (n, 3) block indices in (x, y, z) order."""
        arr, n = _shape_array(shapes)
        return _block_list(self._m._L.nvb_layer_clear_shapes, self.num_blocks(), self._m._h, self._id, arr, n)

    def block_device_ptr(self, index):
        k = np.asarray(index, dtype=np.int32)
        p = C.c_void_p(0)
        check(self._m._L.nvb_layer_block_device_ptr(self._m._h, self._id, _ip(k), C.byref(p)))
        return p.value or 0

    def as_dict(self):
        idx = self.get_all_block_indices()
        if len(idx) == 0:
            return {}
        v, _ = self.get_blocks(idx)
        return {tuple(int(c) for c in k): v[i] for i, k in enumerate(idx)}

    def export_points(self):
        """io::outputVoxelLayerToPly's points (io/pointcloud_io.cpp:23-73) of a TSDF, occupancy, freespace or ESDF layer:
        (n, 4) float32 {x, y, z, intensity} at the kept voxels' centres, blocks in (x, y, z) order, then voxels in x, y, z
        order."""
        n = C.c_int64(0)
        check(self._m._L.nvb_layer_export_points(self._m._h, self._id, _lib.NVB_MEM_HOST, None, 0, C.byref(n)))
        out = np.zeros((max(n.value, 1), 4), dtype=np.float32)
        check(self._m._L.nvb_layer_export_points(self._m._h, self._id, _lib.NVB_MEM_HOST, out.ctypes.data, n.value, C.byref(n)))
        return out[:n.value]

    def get_voxels(self, points):
        """VoxelBlockLayer::getVoxels / getVoxelsGPU (map/layer.h:265-295): the voxel holding each point, as stored, and
        whether its block exists. `points` is an (n, 3) float32 host array -> (structured voxel array, bool array), or a CUDA
        tensor -> ((n, voxel bytes) uint8 tensor, bool tensor) on its device, ordered after torch's current stream without a
        host synchronisation; `.cpu().numpy().view(dtype)` of the first gives the structured voxels. Missed voxels are zero."""
        vb = self._dtype.itemsize
        if _is_tensor(points):
            return self._device_query(self._m._L.nvb_layer_query_voxels, points, (vb,), "uint8")
        pts = _host_points(points)
        out = np.zeros(pts.shape[0], dtype=self._dtype)
        ok = np.zeros(pts.shape[0], dtype=np.uint8)
        check(self._m._L.nvb_layer_query_voxels(self._m._h, self._id, pts.ctypes.data, _lib.NVB_MEM_HOST, pts.shape[0],
                                                out.ctypes.data, ok.ctypes.data))
        return out, ok.astype(bool)

    def interpolate(self, points):
        """interpolation::interpolateOnCPU (interpolation/interpolation_3d.h) on the GPU, for a TSDF (distance), ESDF
        (unsigned distance in voxels) or occupancy (probability) layer: (values, successes); a failed point has value 0.
        Host array -> numpy arrays; CUDA tensor -> tensors on its device, as get_voxels."""
        if _is_tensor(points):
            return self._device_query(self._m._L.nvb_layer_interpolate, points, (), "float32")
        pts = _host_points(points)
        out = np.zeros(pts.shape[0], dtype=np.float32)
        ok = np.zeros(pts.shape[0], dtype=np.uint8)
        check(self._m._L.nvb_layer_interpolate(self._m._h, self._id, pts.ctypes.data, _lib.NVB_MEM_HOST, pts.shape[0],
                                               out.ctypes.data, ok.ctypes.data))
        return out, ok.astype(bool)

    def _device_query(self, fn, points, shape, dtype):
        import torch
        pts = _device_points(points, 3, self._m._device)
        n = pts.shape[0]
        out = torch.zeros((n,) + shape, dtype=getattr(torch, dtype), device=pts.device)
        ok = torch.zeros(n, dtype=torch.uint8, device=pts.device)
        # No record_stream on the mapper's stream: torch's stream waits for the call, so a later reuse of these tensors' memory
        # on it is ordered after the call, and nothing is recorded on a stream that closing the mapper destroys.
        with _on_mapper_stream(self._m, pts.device):
            check(fn(self._m._h, self._id, pts.data_ptr(), _lib.NVB_MEM_DEVICE, n, out.data_ptr(), ok.data_ptr()))
        return out, ok.bool()


def _is_tensor(a):
    return hasattr(a, "data_ptr") and hasattr(a, "is_cuda")


def _host_points(points):
    pts = np.ascontiguousarray(points, dtype=np.float32)
    if pts.ndim != 2 or pts.shape[1] != 3:
        raise ValueError("points must be an (n, 3) array")
    return pts


def _device_points(t, cols, device, name="points"):
    """Check a query tensor before anything is enqueued: a float32 (n, cols) CUDA tensor on the mappers' device."""
    import torch
    if not _is_tensor(t) or not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor" % name)
    if t.dtype != torch.float32:
        raise ValueError("%s must be float32, not %s" % (name, t.dtype))
    cols = (cols,) if isinstance(cols, int) else tuple(cols)
    if t.ndim != 2 or t.shape[1] not in cols:
        raise ValueError("%s must have shape (n, %s), not %s" % (name, " or ".join(map(str, cols)), tuple(t.shape)))
    if t.device.index != device:
        raise ValueError("%s are on cuda:%d, the mapper on cuda:%d" % (name, t.device.index, device))
    return t.detach().contiguous()


class _on_mapper_stream:
    """Runs a call enqueued on a mapper's stream between torch's current stream and its next work: the mapper's stream waits
    for what torch enqueued so far, torch's stream waits for the call. Event hops only, no host synchronisation."""

    def __init__(self, mapper, device):
        import torch
        self._torch = torch.cuda.current_stream(device)
        self._ms = torch.cuda.ExternalStream(mapper._L.nvb_mapper_stream(mapper._h), device=device)

    def __enter__(self):
        self._ms.wait_stream(self._torch)

    def __exit__(self, *exc):
        self._torch.wait_stream(self._ms)
        return False


class _TsdfIntegrator:
    """ProjectiveTsdfIntegrator parameter surface (projective_tsdf_integrator.h:59-121,
    projective_integrator.h:56-85, view_calculator.h:88-145)."""

    def __init__(self, mapper):
        self._m = mapper

    def _get(self):
        p = NvbTsdfParams()
        check(self._m._L.nvb_mapper_get_tsdf_params(self._m._h, C.byref(p)))
        return p

    def _set(self, **kw):
        p = self._get()
        for k, v in kw.items():
            if k in ("workspace_min", "workspace_max"):
                setattr(p, k, (C.c_float * 3)(*v))
            else:
                setattr(p, k, v)
        check(self._m._L.nvb_mapper_set_tsdf_params(self._m._h, C.byref(p)))

    def params(self, **kw):
        if kw:
            self._set(**kw)
        return self._get()

    def truncation_distance_vox(self, v=None):
        if v is not None:
            self._set(truncation_distance_vox=float(v))
        return self._get().truncation_distance_vox

    def max_integration_distance_m(self, v=None):
        if v is not None:
            self._set(max_integration_distance_m=float(v))
        return self._get().max_integration_distance_m

    def max_weight(self, v=None):
        if v is not None:
            self._set(max_weight=float(v))
        return self._get().max_weight

    def invalid_depth_decay_factor(self, v=None):
        if v is not None:
            self._set(invalid_depth_decay_factor=float(v))
        return self._get().invalid_depth_decay_factor

    def weighting_function_type(self, v=None):
        if v is not None:
            self._set(weighting_type=int(v))
        return self._get().weighting_type

    def cache_last_viewpoint(self, v=None):
        """ViewCalculator::cache_last_viewpoint (view_calculator.h:196): on by default, like the reference."""
        if v is not None:
            check(self._m._L.nvb_mapper_set_cache_last_viewpoint(self._m._h, 1 if v else 0))
        return bool(self._m._L.nvb_mapper_get_cache_last_viewpoint(self._m._h))

    def raycast_subsampling_factor(self, v=None):
        if v is not None:
            self._set(raycast_subsampling=int(v))
        return self._get().raycast_subsampling


class _OccupancyIntegrator(_TsdfIntegrator):
    """ProjectiveOccupancyIntegrator parameter surface (projective_occupancy_integrator.h:57-109) on top of
    the shared ProjectiveIntegrator / ViewCalculator one."""

    def _get_occ(self):
        p = NvbOccupancyParams()
        check(self._m._L.nvb_mapper_get_occupancy_params(self._m._h, C.byref(p)))
        return p

    def occupancy_params(self, **kw):
        p = self._get_occ()
        for k, v in kw.items():
            setattr(p, k, float(v))
        if kw:
            check(self._m._L.nvb_mapper_set_occupancy_params(self._m._h, C.byref(p)))
        return p

    def free_region_occupancy_probability(self, v=None):
        return self.occupancy_params(**({} if v is None else {"free_region_occupancy_probability": v})) \
            .free_region_occupancy_probability

    def occupied_region_occupancy_probability(self, v=None):
        return self.occupancy_params(**({} if v is None else {"occupied_region_occupancy_probability": v})) \
            .occupied_region_occupancy_probability

    def unobserved_region_occupancy_probability(self, v=None):
        return self.occupancy_params(**({} if v is None else {"unobserved_region_occupancy_probability": v})) \
            .unobserved_region_occupancy_probability

    def occupied_region_half_width_m(self, v=None):
        return self.occupancy_params(**({} if v is None else {"occupied_region_half_width_m": v})) \
            .occupied_region_half_width_m


class _ColorIntegrator:
    """ProjectiveColorIntegrator parameter surface (projective_appearance_integrator.h:96-148) and its SphereTracer."""

    def __init__(self, mapper):
        self._m = mapper

    def params(self, **kw):
        p = _lib.NvbColorParams()
        check(self._m._L.nvb_mapper_get_color_params(self._m._h, C.byref(p)))
        for k, v in kw.items():
            setattr(p, k, v)
        if kw:
            check(self._m._L.nvb_mapper_set_color_params(self._m._h, C.byref(p)))
        return p

    def render_depth(self, T_L_C, camera, truncation_distance_m, ray_subsampling_factor=1):
        """SphereTracer::renderImageOnGPU(camera, T_L_C, tsdf_layer, truncation_distance_m, ..., ray_subsampling_factor)
        -> (height / f, width / f) float32, -1 where a ray found no surface."""
        f = int(ray_subsampling_factor)
        out = np.zeros((max(camera.c.height // max(f, 1), 1), max(camera.c.width // max(f, 1), 1)), np.float32)
        T = colmajor(T_L_C)
        check(self._m._L.nvb_sphere_tracer_render_depth(self._m._h, _fp(T), C.byref(camera.c), float(truncation_distance_m), f,
                                                        _fp(out)))
        return out


class _FreespaceIntegrator:
    """FreespaceIntegrator parameter surface (freespace_integrator.h:75-128) + updateFreespaceLayer on a block list."""

    def __init__(self, mapper):
        self._m = mapper

    def params(self, **kw):
        p = NvbFreespaceParams()
        check(self._m._L.nvb_mapper_get_freespace_params(self._m._h, C.byref(p)))
        for k, v in kw.items():
            setattr(p, k, v)
        if kw:
            check(self._m._L.nvb_mapper_set_freespace_params(self._m._h, C.byref(p)))
        return p

    def update_freespace_layer(self, block_indices, update_time_ms, depth=None, T_L_C=None, camera=None,
                               max_view_distance_m=0.0, truncation_distance_m=0.0):
        idx = np.ascontiguousarray(block_indices, dtype=np.int32).reshape(-1, 3)
        if depth is not None:
            depth = np.ascontiguousarray(depth, dtype=np.float32)
            T = colmajor(T_L_C)
            check(self._m._L.nvb_freespace_update_blocks(self._m._h, _ip(idx), idx.shape[0], int(update_time_ms),
                                                         depth.ctypes.data, _lib.NVB_MEM_HOST, depth.shape[0], depth.shape[1],
                                                         _fp(T), C.byref(camera.c), float(max_view_distance_m),
                                                         float(truncation_distance_m)))
        else:
            check(self._m._L.nvb_freespace_update_blocks(self._m._h, _ip(idx), idx.shape[0], int(update_time_ms), None, 0, 0, 0,
                                                         None, None, 0.0, 0.0))


class _DecayIntegrator:
    """TsdfDecayIntegrator / OccupancyDecayIntegrator parameter surface (tsdf_decay_integrator.h:73-101,
    occupancy_decay_integrator.h:72-101, internal/decay_integrator_base.h:50-58)."""

    def __init__(self, mapper, occupancy):
        self._m, self._occ = mapper, occupancy

    def params(self, **kw):
        L, h = self._m._L, self._m._h
        p = NvbOccupancyDecayParams() if self._occ else NvbTsdfDecayParams()
        get = L.nvb_mapper_get_occupancy_decay_params if self._occ else L.nvb_mapper_get_tsdf_decay_params
        put = L.nvb_mapper_set_occupancy_decay_params if self._occ else L.nvb_mapper_set_tsdf_decay_params
        check(get(h, C.byref(p)))
        for k, v in kw.items():
            setattr(p, k, v)
        if kw:
            check(put(h, C.byref(p)))
        return p

    def deallocate_decayed_blocks(self, v=None):
        return bool(self.params(**({} if v is None else {"deallocate_decayed_blocks": 1 if v else 0})).deallocate_decayed_blocks)

    def decay_factor(self, v=None):
        return self.params(**({} if v is None else {"decay_factor": float(v)})).decay_factor

    def decay_to_free(self, v):
        """OccupancyDecayIntegrator::decay_to_free (src/integrators/occupancy_decay_integrator.cu:59-72)."""
        return self.params(decay_to_probability=0.49 if v else 0.5).decay_to_probability


class _EsdfIntegrator:
    """EsdfIntegrator parameter surface (esdf_integrator.h:178-283) + integrateBlocks."""

    def __init__(self, mapper):
        self._m = mapper

    def _get(self):
        p = NvbEsdfParams()
        check(self._m._L.nvb_mapper_get_esdf_params(self._m._h, C.byref(p)))
        return p

    def params(self, **kw):
        p = self._get()
        for k, v in kw.items():
            setattr(p, k, v)
        if kw:
            check(self._m._L.nvb_mapper_set_esdf_params(self._m._h, C.byref(p)))
        return p

    def max_esdf_distance_m(self, v=None):
        return self.params(**({} if v is None else {"max_esdf_distance_m": float(v)})).max_esdf_distance_m

    def max_site_distance_vox(self, v=None):
        return self.params(**({} if v is None else {"max_site_distance_vox": float(v)})).max_site_distance_vox

    def min_weight(self, v=None):
        return self.params(**({} if v is None else {"min_weight": float(v)})).min_weight

    def occupied_threshold(self, v=None):
        return self.params(**({} if v is None else {"occupied_threshold": float(v)})).occupied_threshold

    def slice_params(self, **kw):
        """esdf_slice_min_height / esdf_slice_max_height / esdf_slice_height (esdf_integrator.h:216-256)."""
        p = NvbEsdfSliceParams()
        check(self._m._L.nvb_mapper_get_esdf_slice_params(self._m._h, C.byref(p)))
        for k, v in kw.items():
            setattr(p, k, float(v))
        if kw:
            check(self._m._L.nvb_mapper_set_esdf_slice_params(self._m._h, C.byref(p)))
        return p

    def integrate_slice(self, block_indices, ground_plane=None):
        """EsdfIntegrator::integrateSlice(layer, block_indices[, ground_plane], esdf_layer): constant-z slice, or the planar
        one when ground_plane = (nx, ny, nz, d) (unit normal, n . p + d = 0) is given."""
        idx = np.ascontiguousarray(block_indices, dtype=np.int32).reshape(-1, 3)
        if ground_plane is None:
            check(self._m._L.nvb_esdf_integrate_slice_blocks(self._m._h, _ip(idx), idx.shape[0]))
        else:
            pl = np.ascontiguousarray(ground_plane, dtype=np.float32).reshape(4)
            check(self._m._L.nvb_esdf_integrate_slice_planar_blocks(self._m._h, _fp(pl), _ip(idx), idx.shape[0]))

    def integrate_blocks(self, block_indices):
        """EsdfIntegrator::integrateBlocks(tsdf_layer | occupancy_layer, block_indices, esdf_layer)."""
        idx = np.ascontiguousarray(block_indices, dtype=np.int32).reshape(-1, 3)
        check(self._m._L.nvb_esdf_integrate_blocks(self._m._h, _ip(idx), idx.shape[0]))

    def last_stats(self):
        out = (C.c_int64 * 8)()
        check(self._m._L.nvb_mapper_last_esdf_stats(self._m._h, out))
        keys = ("marked", "with_sites", "to_clear", "clear_candidates", "cleared", "swept", "face_passes", "rings")
        s = dict(zip(keys, list(out)))
        # exchange-slab wavefront: candidates whose own block was fetched split, and those that then fetched the rest
        split = (C.c_int64 * 2)()
        check(self._m._L.nvb_mapper_esdf_split_stats(self._m._h, split))
        s.update(split_candidates=split[0], rest_fetches=split[1])
        return s

    def clear_blocks_read(self):
        """Blocks the last clear pass read (<= clear_candidates: candidates whose parents cannot lie in a to-clear block are skipped)."""
        out = C.c_int64(0)
        check(self._m._L.nvb_mapper_esdf_clear_blocks_read(self._m._h, C.byref(out)))
        return int(out.value)


class _MeshIntegrator:
    """MeshIntegrator parameters (mesh/mesh_integrator.h:83-87,126-133)."""

    def __init__(self, mapper):
        self._m = mapper

    def params(self, **kw):
        p = _lib.NvbMeshParams()
        check(self._m._L.nvb_mapper_get_mesh_params(self._m._h, C.byref(p)))
        if kw:
            for k, v in kw.items():
                setattr(p, k, v)
            check(self._m._L.nvb_mapper_set_mesh_params(self._m._h, C.byref(p)))
        return p

    def min_weight(self, v=None):
        return self.params(**({} if v is None else {"min_weight": float(v)})).min_weight

    def weld_vertices(self, v=None):
        return bool(self.params(**({} if v is None else {"weld_vertices": 1 if v else 0})).weld_vertices)

    def integrate_blocks(self, blocks, update_color=False):
        """MeshIntegrator::integrateBlocksGPU(tsdf_layer, block_indices, mesh_layer) [+ updateAppearance]."""
        b = np.ascontiguousarray(blocks, dtype=np.int32).reshape(-1, 3)
        check(self._m._L.nvb_mesh_integrate_blocks(self._m._h, _ip(b), b.shape[0], 1 if update_color else 0))

    def integrate_mesh_from_distance_field(self, update_color=False):
        """MeshIntegrator::integrateMeshFromDistanceField: every block of the TSDF layer."""
        self.integrate_blocks(self._m.tsdf_layer().get_all_block_indices(), update_color)

    def update_color(self, blocks=None):
        """MeshIntegrator::updateAppearance (blocks=None: every mesh block)."""
        if blocks is None:
            blocks = self._m.mesh_layer().get_all_block_indices()
        b = np.ascontiguousarray(blocks, dtype=np.int32).reshape(-1, 3)
        check(self._m._L.nvb_mesh_update_color(self._m._h, _ip(b), b.shape[0]))


class _MeshLayer:
    """MeshBlockLayer queries (mesh/mesh_block.h:32-83; map/layer.h) answered from the device arena."""

    def __init__(self, mapper):
        self._m = mapper

    def num_blocks(self):
        n = C.c_int32(0)
        rc = self._m._L.nvb_layer_num_blocks(self._m._h, _lib.NVB_LAYER_MESH, C.byref(n))
        return n.value if rc == 0 else 0  # no mesh update yet: an empty layer

    def get_all_block_indices(self):
        n = self.num_blocks()
        if not n:  # no mesh update yet: the layer does not exist
            return np.zeros((0, 3), dtype=np.int32)
        return _block_list(self._m._L.nvb_layer_block_indices, n, self._m._h, _lib.NVB_LAYER_MESH)

    def block_sizes(self, indices):
        """(n,3) -> (n,3) int32 {vertices, triangle indices, colours}; -1 where there is no mesh block."""
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        out = np.full((max(idx.shape[0], 1), 3), -1, dtype=np.int32)
        check(self._m._L.nvb_mesh_block_sizes(self._m._h, _ip(idx), idx.shape[0], _ip(out)))
        return out[:idx.shape[0]]

    def get_blocks(self, indices):
        """(n,3) -> list of {"vertices" (v,3) f32, "normals" (v,3) f32, "triangles" (t,) i32, "colors" (c,4) u8} or None."""
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        sz = self.block_sizes(idx)
        live = np.maximum(sz, 0).astype(np.int64)
        tv, tt, tc = (int(x) for x in live.sum(axis=0)) if idx.shape[0] else (0, 0, 0)
        V, N = np.zeros((max(tv, 1), 3), np.float32), np.zeros((max(tv, 1), 3), np.float32)
        T, Cc = np.zeros(max(tt, 1), np.int32), np.zeros((max(tc, 1), 4), np.uint8)
        caps = (C.c_int64 * 3)(tv, tt, tc)
        check(self._m._L.nvb_mesh_get_blocks(self._m._h, _ip(idx), idx.shape[0], V.ctypes.data, N.ctypes.data, T.ctypes.data,
                                             Cc.ctypes.data, caps))
        out, ov, ot, oc = [], 0, 0, 0
        for i in range(idx.shape[0]):
            if sz[i, 0] < 0:
                out.append(None)
                continue
            nv, nt, nc = (int(x) for x in sz[i])
            out.append({"vertices": V[ov:ov + nv].copy(), "normals": N[ov:ov + nv].copy(), "triangles": T[ot:ot + nt].copy(),
                        "colors": Cc[oc:oc + nc].copy()})
            ov, ot, oc = ov + nv, ot + nt, oc + nc
        return out

    def get_block_at_index(self, index):
        return self.get_blocks(np.asarray(index, dtype=np.int32).reshape(1, 3))[0]

    def is_block_allocated(self, index):
        return bool(self.block_sizes(np.asarray(index, dtype=np.int32).reshape(1, 3))[0, 0] >= 0)

    def as_dict(self):
        idx = self.get_all_block_indices()
        return {tuple(int(c) for c in k): b for k, b in zip(idx, self.get_blocks(idx))}

    def arena_stats(self):
        out = (C.c_int64 * 4)()
        check(self._m._L.nvb_mesh_arena_stats(self._m._h, out))
        return {"capacity": out[0], "used": out[1], "last_update_vertices": out[2]}


class EsdfSlicer:
    """EsdfSlicer (integrators/esdf_slicer.h:36-138): distance-map image and occupancy grid of an ESDF slice."""

    def __init__(self, mapper):
        self._m = mapper

    def slice_layer_to_distance_image(self, slice_height, unobserved_value=1000.0, with_occupancy_grid=False):
        """-> (aabb [min xyz, max xyz], (rows, cols) float32 image[, int8 grid]); rows follow y, columns x."""
        L, h = self._m._L, self._m._h
        aabb = np.zeros(6, np.float32)
        r, c = C.c_int32(0), C.c_int32(0)
        check(L.nvb_esdf_slice_distance_image(h, float(slice_height), float(unobserved_value), _fp(aabb), None, None, 0,
                                              C.byref(r), C.byref(c)))
        img = np.zeros((max(r.value, 1), max(c.value, 1)), np.float32)
        grid = np.zeros((max(r.value, 1), max(c.value, 1)), np.int8)
        if r.value * c.value > 0:
            check(L.nvb_esdf_slice_distance_image(h, float(slice_height), float(unobserved_value), _fp(aabb), _fp(img),
                                                  grid.ctypes.data_as(C.POINTER(C.c_int8)) if with_occupancy_grid else None,
                                                  r.value * c.value, C.byref(r), C.byref(c)))
        img = img[:r.value, :c.value]
        return (aabb, img, grid[:r.value, :c.value]) if with_occupancy_grid else (aabb, img)

    def get_aabb_of_layer_at_height(self, slice_height):
        """EsdfSlicer::getAabbOfLayerAtHeight (esdf_slicer.h:29-35) -> (6,) float32, or None for an empty box."""
        aabb = np.zeros(6, np.float32)
        empty = C.c_int32(1)
        check(self._m._L.nvb_esdf_slice_aabb(self._m._h, float(slice_height), _fp(aabb), C.byref(empty)))
        return None if empty.value else aabb

    def slice_layer_to_distance_image_in_aabb(self, slice_height, aabb, unobserved_value=1000.0):
        """EsdfSlicer::sliceLayerToDistanceImage(layer, slice_height, unobserved_value, aabb, image): a given box."""
        L, h = self._m._L, self._m._h
        box = np.ascontiguousarray(aabb, np.float32).reshape(6)
        r, c = C.c_int32(0), C.c_int32(0)
        check(L.nvb_esdf_slice_distance_image_in_aabb(h, float(slice_height), float(unobserved_value), _fp(box), None, None, 0,
                                                      C.byref(r), C.byref(c)))
        img = np.zeros((max(r.value, 1), max(c.value, 1)), np.float32)
        if r.value * c.value > 0:
            check(L.nvb_esdf_slice_distance_image_in_aabb(h, float(slice_height), float(unobserved_value), _fp(box), _fp(img), None,
                                                          r.value * c.value, C.byref(r), C.byref(c)))
        return img[:r.value, :c.value]

    def slice_layers_to_combined_distance_image(self, other_mapper, slice_height_1, slice_height_2, unobserved_value=1000.0,
                                                with_occupancy_grid=False):
        """EsdfSlicer::sliceLayersToCombinedDistanceImage (esdf_slicer.h:78-118, src/integrators/esdf_slicer.cu:201-240): this
        mapper's ESDF layer and another mapper's (e.g. MultiMapper's static and dynamic maps) sliced on the merged box of their
        slices, element-wise minimum. -> (aabb, image[, grid]); (None, None[, None]) if neither layer has a block there."""
        other = EsdfSlicer(other_mapper)
        boxes = [b for b in (self.get_aabb_of_layer_at_height(slice_height_1), other.get_aabb_of_layer_at_height(slice_height_2))
                 if b is not None]
        if not boxes:
            return (None, None, None) if with_occupancy_grid else (None, None)
        aabb = np.concatenate([np.min([b[:3] for b in boxes], axis=0), np.max([b[3:] for b in boxes], axis=0)]).astype(np.float32)
        img = np.minimum(self.slice_layer_to_distance_image_in_aabb(slice_height_1, aabb, unobserved_value),
                         other.slice_layer_to_distance_image_in_aabb(slice_height_2, aabb, unobserved_value))
        if not with_occupancy_grid:
            return aabb, img
        # occupancyGridFromSliceImageKernel (src/integrators/esdf_slicer.cu:78-110)
        grid = np.where(img < np.float32(1e-2), 100, 0).astype(np.int8)
        grid[np.abs(img - np.float32(unobserved_value)) < np.float32(1e-2)] = -1
        return aabb, img, grid


def _plane_or_none(fn, *args):
    pl = (C.c_float * 4)()
    found = C.c_int32(0)
    check(fn(*args, pl, C.byref(found)))
    return tuple(float(v) for v in pl) if found.value else None


class GroundPlaneEstimator:
    """GroundPlaneEstimator (experimental/ground_plane/ground_plane_estimator.h) of one mapper: the TSDF zero crossings from
    above, the ground candidates among them (min_z <= z <= max_z) and their MSAC plane. Planes are (nx, ny, nz, d) with
    n . p + d = 0; point lists are (n, 3) float32 in block-index (x, y, z) order, then voxel (x, y, z) order."""

    def __init__(self, mapper):
        self._m = mapper

    def params(self, **kw):
        """Sets the given fields of NvbGroundPlaneParams (ground_points_candidates_min_z_m / max_z_m,
        ransac_distance_threshold_m, num_ransac_iterations, min_tsdf_weight, max_crossings); returns them all as a dict."""
        p = NvbGroundPlaneParams()
        check(self._m._L.nvb_mapper_get_ground_plane_params(self._m._h, C.byref(p)))
        for k, v in kw.items():
            if k not in dict(p._fields_):
                raise TypeError("unknown ground-plane parameter %r" % k)
            setattr(p, k, v)
        if kw:
            check(self._m._L.nvb_mapper_set_ground_plane_params(self._m._h, C.byref(p)))
        return {k: getattr(p, k) for k, _ in p._fields_}

    def compute_ground_plane(self):
        """computeGroundPlane(tsdf_layer): the plane, or None (the last crossings, candidates and plane are then cleared)."""
        return _plane_or_none(self._m._L.nvb_mapper_compute_ground_plane, self._m._h)

    def ground_plane(self):
        return _plane_or_none(self._m._L.nvb_mapper_ground_plane, self._m._h)

    def _points(self, which):
        L, h = self._m._L, self._m._h
        n, valid = C.c_int32(0), C.c_int32(0)
        check(L.nvb_mapper_ground_plane_points(h, which, None, 0, C.byref(n), C.byref(valid)))
        if not valid.value:
            return None
        out = np.zeros((n.value, 3), dtype=np.float32)
        if n.value:
            check(L.nvb_mapper_ground_plane_points(h, which, _fp(out), n.value, C.byref(n), C.byref(valid)))
        return out

    def tsdf_zero_crossings(self):
        return self._points(_lib.NVB_GROUND_POINTS_CROSSINGS)

    def tsdf_zero_crossings_ground_candidates(self):
        return self._points(_lib.NVB_GROUND_POINTS_CANDIDATES)


_fit_mappers = {}


def ransac_fit_plane(points, num_ransac_iterations=1000, ransac_distance_threshold_m=0.2, mapper=None, device=0):
    """RansacPlaneFitter::fit (experimental/ground_plane/ransac_plane_fitter.h), MSAC on the GPU: (nx, ny, nz, d) or None.
    `points` is an (n, 3) float32 array (host) or a CUDA tensor (device). Runs on `mapper`'s device and stream; without one,
    on a small mapper kept per device."""
    if mapper is None:
        mapper = _fit_mappers.get(device)
        if mapper is None:
            mapper = _fit_mappers[device] = Mapper(0.05, device=device, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    if hasattr(points, "data_ptr"):  # a CUDA tensor
        import torch
        if not points.is_cuda:
            raise ValueError("a tensor of points must be on the GPU")
        if points.device.index != mapper._device:
            raise ValueError("the points are on cuda:%d, the mapper on cuda:%d" % (points.device.index, mapper._device))
        t = points.detach().float().contiguous().reshape(-1, 3)
        # The mapper's stream does not wait for torch's: order this call after the producer of the points and after the
        # conversion / copy above, both enqueued on torch's current stream.
        torch.cuda.current_stream(t.device).synchronize()
        ptr, n, mem, keep = t.data_ptr(), t.shape[0], _lib.NVB_MEM_DEVICE, t
    else:
        a = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
        ptr, n, mem, keep = a.ctypes.data, a.shape[0], _lib.NVB_MEM_HOST, a
    pl = (C.c_float * 4)()
    found = C.c_int32(0)
    check(mapper._L.nvb_ransac_fit_plane(mapper._h, C.c_void_p(ptr), mem, int(n), int(num_ransac_iterations),
                                          float(ransac_distance_threshold_m), pl, C.byref(found)))
    del keep
    return tuple(float(v) for v in pl) if found.value else None


class DynamicsDetection:
    """DynamicsDetection (dynamics/dynamics_detection.h) on the freespace layer of one kTsdfWithFreespace mapper: a depth pixel
    is dynamic when its surface point falls into a high-confidence freespace voxel. Outputs stay on the device until a getter
    reads them; points come in row-major pixel order. The *_device variants take and fill raw device pointers, enqueued on
    the mapper's stream (cuda_stream()) without synchronising."""

    def __init__(self, mapper):
        self._m = mapper

    def compute_dynamics(self, depth, T_L_C, camera):
        """computeDynamics(depth_frame, freespace_layer, camera, T_L_C); depth: (rows, cols) float32 host array."""
        d = np.ascontiguousarray(depth, dtype=np.float32)
        check(self._m._L.nvb_mapper_compute_dynamics(self._m._h, d.ctypes.data, _lib.NVB_MEM_HOST, d.shape[0], d.shape[1],
                                                     _fp(colmajor(T_L_C)), C.byref(camera.c)))

    def compute_dynamics_device(self, depth_ptr, rows, cols, T_L_C, camera):
        check(self._m._L.nvb_mapper_compute_dynamics(self._m._h, depth_ptr, _lib.NVB_MEM_DEVICE, int(rows), int(cols),
                                                     _fp(colmajor(T_L_C)), C.byref(camera.c)))

    def _image(self, fn, channels):
        rows, cols = C.c_int32(0), C.c_int32(0)
        check(fn(self._m._h, None, _lib.NVB_MEM_HOST, C.byref(rows), C.byref(cols)))
        out = np.zeros((rows.value, cols.value, channels) if channels > 1 else (rows.value, cols.value), dtype=np.uint8)
        if out.size:
            check(fn(self._m._h, out.ctypes.data, _lib.NVB_MEM_HOST, C.byref(rows), C.byref(cols)))
        return out

    def dynamic_mask(self):
        """getDynamicMaskImage(): (rows, cols) uint8, 255 on dynamic pixels."""
        return self._image(self._m._L.nvb_mapper_dynamic_mask, 1)

    def dynamic_overlay(self):
        """getDynamicOverlayImage(): (rows, cols, 3) uint8 RGB."""
        return self._image(self._m._L.nvb_mapper_dynamic_overlay, 3)

    def dynamic_mask_device(self, out_ptr):
        """Copies the mask into rows x cols device bytes at out_ptr (enqueued); returns (rows, cols)."""
        rows, cols = C.c_int32(0), C.c_int32(0)
        check(self._m._L.nvb_mapper_dynamic_mask(self._m._h, out_ptr, _lib.NVB_MEM_DEVICE, C.byref(rows), C.byref(cols)))
        return rows.value, cols.value

    def dynamic_overlay_device(self, out_ptr):
        rows, cols = C.c_int32(0), C.c_int32(0)
        check(self._m._L.nvb_mapper_dynamic_overlay(self._m._h, out_ptr, _lib.NVB_MEM_DEVICE, C.byref(rows), C.byref(cols)))
        return rows.value, cols.value

    def dynamic_points(self):
        """getDynamicPointsHost(): (n, 3) float32, in row-major pixel order."""
        n = C.c_int32(0)
        check(self._m._L.nvb_mapper_dynamic_points(self._m._h, None, _lib.NVB_MEM_HOST, 0, C.byref(n)))
        out = np.zeros((n.value, 3), dtype=np.float32)
        if n.value:
            check(self._m._L.nvb_mapper_dynamic_points(self._m._h, out.ctypes.data, _lib.NVB_MEM_HOST, n.value, C.byref(n)))
        return out

    def dynamic_points_device(self, out_ptr, cap):
        """Copies up to cap points (3 floats each) to device memory at out_ptr; returns the number of dynamic points."""
        n = C.c_int32(0)
        check(self._m._L.nvb_mapper_dynamic_points(self._m._h, out_ptr, _lib.NVB_MEM_DEVICE, int(cap), C.byref(n)))
        return n.value

    def device_buffers(self):
        """The detector's own device buffers (raw pointers), valid until the next compute_dynamics on this mapper."""
        b = _lib.NvbDynamicsBuffers()
        check(self._m._L.nvb_mapper_dynamics_device_buffers(self._m._h, C.byref(b)))
        return {k: getattr(b, k) for k, _ in b._fields_}


class ImageMasker:
    """ImageMasker (semantics/image_masker.h) on one mapper's device and stream: split_depth sends each depth pixel that
    lands, unoccluded, on a set pixel of a mask seen from another camera to the foreground, the rest to the background.
    The depth split's outputs live in the mapper until its next split; the colour split writes the caller's buffers."""

    def __init__(self, mapper):
        self._m = mapper
        self._p = _lib.NvbImageMaskerParams()
        mapper._L.nvb_default_image_masker_params(C.byref(self._p))

    def params(self, occlusion_threshold_m=None, depth_masked_image_invalid_pixel=None,
               depth_unmasked_image_invalid_pixel=None):
        """Sets the given parameters; returns all three as a dict."""
        for k, v in (("occlusion_threshold_m", occlusion_threshold_m),
                     ("depth_masked_image_invalid_pixel", depth_masked_image_invalid_pixel),
                     ("depth_unmasked_image_invalid_pixel", depth_unmasked_image_invalid_pixel)):
            if v is not None:
                setattr(self._p, k, float(v))
        return {k: getattr(self._p, k) for k, _ in self._p._fields_}

    def _split(self, depth, depth_rows, depth_cols, mask, mask_rows, mask_cols, memory, T_CM_CD, depth_camera, mask_camera,
               overlay):
        check(self._m._L.nvb_mapper_split_depth_image(self._m._h, depth, int(depth_rows), int(depth_cols), mask,
                                                      int(mask_rows), int(mask_cols), memory, _fp(colmajor(T_CM_CD)),
                                                      C.byref(depth_camera.c), C.byref(mask_camera.c), C.byref(self._p),
                                                      1 if overlay else 0))

    def split_depth(self, depth, mask, T_CM_CD, depth_camera, mask_camera, overlay=False):
        """splitImageOnGPU(depth, mask, T_CM_CD, depth_camera, mask_camera, ...): host arrays in, host arrays out ->
        (background, foreground) float32, plus the (rows, cols, 3) uint8 overlay when `overlay`."""
        d = np.ascontiguousarray(depth, dtype=np.float32)
        mk = np.ascontiguousarray(mask, dtype=np.uint8)
        if d.ndim != 2 or mk.ndim != 2:
            raise ValueError("depth and mask must be (rows, cols) images")
        self._split(d.ctypes.data, d.shape[0], d.shape[1], mk.ctypes.data, mk.shape[0], mk.shape[1], _lib.NVB_MEM_HOST,
                    T_CM_CD, depth_camera, mask_camera, overlay)
        out = (self.output(_lib.NVB_SPLIT_BACKGROUND), self.output(_lib.NVB_SPLIT_FOREGROUND))
        return out + (self.output(_lib.NVB_SPLIT_OVERLAY),) if overlay else out

    def split_depth_device(self, depth_ptr, depth_rows, depth_cols, mask_ptr, mask_rows, mask_cols, T_CM_CD, depth_camera,
                           mask_camera, overlay=False):
        """The same on raw device pointers, enqueued on mapper.cuda_stream() without synchronising -> device_buffers()."""
        self._split(depth_ptr, depth_rows, depth_cols, mask_ptr, mask_rows, mask_cols, _lib.NVB_MEM_DEVICE, T_CM_CD,
                    depth_camera, mask_camera, overlay)
        return self.device_buffers()

    def output(self, which):
        """One output of the last split (NVB_SPLIT_BACKGROUND / _FOREGROUND / _OVERLAY) as a host array."""
        rows, cols = C.c_int32(0), C.c_int32(0)
        fn = self._m._L.nvb_mapper_split_output
        check(fn(self._m._h, int(which), None, _lib.NVB_MEM_HOST, C.byref(rows), C.byref(cols)))
        if which == _lib.NVB_SPLIT_OVERLAY:
            out = np.zeros((rows.value, cols.value, 3), np.uint8)
        else:
            out = np.zeros((rows.value, cols.value), np.float32)
        if out.size:
            check(fn(self._m._h, int(which), out.ctypes.data, _lib.NVB_MEM_HOST, C.byref(rows), C.byref(cols)))
        return out

    def device_buffers(self):
        """The last split's device buffers (raw pointers; overlay None when it made none), valid until the next split."""
        b = _lib.NvbSplitBuffers()
        check(self._m._L.nvb_mapper_split_device_buffers(self._m._h, C.byref(b)))
        return {k: getattr(b, k) for k, _ in b._fields_}

    def split_color(self, rgb, mask, overlay=False):
        """splitImageOnGPU(color, mask, ...): (rows, cols, 3) uint8 and a (rows, cols) mask on top of it -> (unmasked,
        masked), plus the overlay when `overlay`."""
        c = np.ascontiguousarray(rgb, dtype=np.uint8)
        mk = np.ascontiguousarray(mask, dtype=np.uint8)
        if c.ndim != 3 or c.shape[2] != 3 or mk.shape != c.shape[:2]:
            raise ValueError("rgb must be (rows, cols, 3) and mask (rows, cols)")
        outs = [np.empty_like(c) for _ in range(3 if overlay else 2)]
        check(self._m._L.nvb_mapper_split_color_image(self._m._h, c.ctypes.data, mk.ctypes.data, _lib.NVB_MEM_HOST,
                                                      c.shape[0], c.shape[1], outs[0].ctypes.data, outs[1].ctypes.data,
                                                      outs[2].ctypes.data if overlay else None))
        return tuple(outs)

    def split_color_device(self, rgb_ptr, mask_ptr, rows, cols, unmasked_ptr, masked_ptr, overlay_ptr=None):
        """The same on raw device pointers, enqueued on mapper.cuda_stream() without synchronising."""
        check(self._m._L.nvb_mapper_split_color_image(self._m._h, rgb_ptr, mask_ptr, _lib.NVB_MEM_DEVICE, int(rows),
                                                      int(cols), unmasked_ptr, masked_ptr, overlay_ptr))


_filter_mappers = {}


def remove_small_connected_components(mask, threshold, mapper=None, device=0):
    """MaskPreprocessor::removeSmallConnectedComponents(mask, threshold): (rows, cols) uint8 host mask -> the filtered mask of
    the same size (survivors 254, the rest 0; a trailing odd row / column is 0). Runs on `mapper`'s device, stream and
    scratch; without one, on a small mapper kept per device."""
    if mapper is None:
        mapper = _filter_mappers.get(device)
        if mapper is None:
            mapper = _filter_mappers[device] = Mapper(0.05, device=device, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    a = np.ascontiguousarray(mask, dtype=np.uint8)
    if a.ndim != 2:
        raise ValueError("the mask must be a (rows, cols) image")
    out = np.empty_like(a)
    check(mapper._L.nvb_mapper_remove_small_components(mapper._h, a.ctypes.data, out.ctypes.data, _lib.NVB_MEM_HOST,
                                                        a.shape[0], a.shape[1], int(threshold)))
    return out


def remove_small_connected_components_device(mask_in_ptr, mask_out_ptr, rows, cols, threshold, mapper):
    """The same on rows x cols device bytes, enqueued on mapper.cuda_stream() without synchronising."""
    check(mapper._L.nvb_mapper_remove_small_components(mapper._h, mask_in_ptr, mask_out_ptr, _lib.NVB_MEM_DEVICE, int(rows),
                                                        int(cols), int(threshold)))


class Mapper:
    """nvblox::Mapper(voxel_size_m, projective_layer_type) with a projective (TSDF or occupancy) and an ESDF layer."""

    def esdf_time_split(self):
        out = (C.c_int64 * 4)()
        check(self._L.nvb_mapper_esdf_time_split(self._h, out))
        return {"barrier_wait_ns_cta0": out[0], "axis_ns_cta0": out[1], "slowest_cta_work_ns": out[2], "barriers": out[3]}

    def debug_phase_max(self, n=4000):
        """The wavefront's per-phase debug words of the last update (filled only by a -DNVB_WAVEX_PROF=1 build; see
        tools/wavex_profile.py for the layout) as an int64 array of `n` <= 4000 entries."""
        out = (C.c_int64 * n)()
        check(self._L.nvb_mapper_debug_phase_max(self._h, out, n))
        return np.frombuffer(out, dtype=np.int64).copy()

    def __init__(self, voxel_size_m, device=0, tsdf_capacity_blocks=0, esdf_capacity_blocks=0,
                 esdf_persistent=3, projective_layer_type=ProjectiveLayerType.kTsdf, keep_last_view=False):
        self._L = _lib.load()
        o = NvbMapperOptions()
        self._L.nvb_default_mapper_options(C.byref(o))
        o.voxel_size_m = float(voxel_size_m)
        o.device = int(device)
        self._device = int(device)
        if tsdf_capacity_blocks:
            o.tsdf_capacity_blocks = int(tsdf_capacity_blocks)
        if esdf_capacity_blocks:
            o.esdf_capacity_blocks = int(esdf_capacity_blocks)
        o.esdf_persistent = 1 if esdf_persistent is True else int(esdf_persistent)  # (True: the four-phase wavefront, as in round 1) 0 host loop, 1 four-phase wavefront, 2 gather-replay wavefront, 3 exchange-slab wavefront
        o.projective_layer_type = int(projective_layer_type)
        o.keep_last_view = 1 if keep_last_view else 0
        self._projective_layer_type = int(projective_layer_type)
        h = C.c_void_p(0)
        check(self._L.nvb_mapper_create(C.byref(o), C.byref(h)))
        self._h = h
        self._tsdf = _Layer(self, _lib.NVB_LAYER_TSDF, TSDF_VOXEL_DTYPE)
        self._occupancy = _Layer(self, _lib.NVB_LAYER_OCCUPANCY, OCCUPANCY_VOXEL_DTYPE)
        self._freespace = _Layer(self, _lib.NVB_LAYER_FREESPACE, FREESPACE_VOXEL_DTYPE)
        self._esdf = _Layer(self, _lib.NVB_LAYER_ESDF, ESDF_VOXEL_DTYPE)
        self._color = _Layer(self, _lib.NVB_LAYER_COLOR, COLOR_VOXEL_DTYPE)
        self._keep = []  # host buffers of in-flight async frames

    def close(self):
        if getattr(self, "_h", None):
            self._L.nvb_mapper_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- accessors -------------------------------------------------------
    def voxel_size(self):
        return self._L.nvb_mapper_voxel_size(self._h)

    def block_size(self):
        return self._L.nvb_mapper_block_size(self._h)

    def tsdf_layer(self):
        return self._tsdf

    def ground_plane_estimator(self):
        """MultiMapper::ground_plane_estimator() of this mapper (its state lives in the mapper)."""
        return GroundPlaneEstimator(self)

    def dynamics_detection(self):
        """The DynamicsDetection of this mapper's freespace layer (its state lives in the mapper)."""
        return DynamicsDetection(self)

    def wait_for(self, producer):
        """Later work on this mapper's stream runs after everything enqueued so far on producer's (device-side)."""
        check(self._L.nvb_mapper_wait_for(self._h, producer._h))

    def occupancy_layer(self):
        return self._occupancy

    def freespace_layer(self):
        return self._freespace

    def mark_unobserved_tsdf_free_inside_radius(self, center, radius):
        """Mapper::markUnobservedTsdfFreeInsideRadius(center, radius) (mapper.h:352-356) -> the blocks inside the radius."""
        c = np.ascontiguousarray(center, dtype=np.float32).reshape(3)
        # room for every block of the sphere's block box, computed in float32 as the library bounds its own list; the call
        # fails for a box of more than 2^26 blocks or a radius that is not positive
        r, bs = np.float32(radius), np.float32(self.block_size())
        cells = np.prod(np.floor((c + r) / bs) - np.floor((c - r) / bs) + 1, dtype=np.float64)
        cap = int(cells) if 1 <= cells <= (1 << 26) else 1
        return _block_list(self._L.nvb_mapper_mark_unobserved_free_inside_radius, cap, self._h, _fp(c), float(radius))

    def color_layer(self):
        return self._color

    def mesh_layer(self):
        """Mapper::color_mesh_layer()."""
        return _MeshLayer(self)

    def mesh_integrator(self):
        """Mapper::color_mesh_integrator()."""
        return _MeshIntegrator(self)

    def save_color_mesh_as_ply(self, filename):
        """Mapper::saveColorMeshAsPly (src/mapper/mapper.cpp:694-696)."""
        from . import io as _io
        return _io.output_color_mesh_layer_to_ply(self.mesh_layer(), filename)

    def update_mesh(self, update_full_layer=False):
        """Mapper::updateColorMesh(UpdateFullLayer) (mapper.h; src/mapper/mapper.cpp:371-406)."""
        check(self._L.nvb_mapper_update_mesh(self._h, 1 if update_full_layer else 0))

    def color_integrator(self):
        return _ColorIntegrator(self)

    def integrate_color(self, color, T_L_C, camera, mask=None, mask_mode=0, return_blocks=True):
        """Mapper::integrateColor(color_frame[, mask], T_L_C, camera) (mapper.h:202-207). color: (rows, cols, 3) uint8 RGB.
        Returns updated_blocks (n, 3) (unordered)."""
        c = np.ascontiguousarray(color, dtype=np.uint8)
        if c.ndim != 3 or c.shape[2] != 3:
            raise ValueError("color must be (rows, cols, 3) uint8")
        mk = None
        if mask is not None:
            mk = np.ascontiguousarray(mask, dtype=np.uint8)
            if mk.shape != c.shape[:2]:
                raise ValueError("mask must have the colour image's size")
        T = colmajor(T_L_C)
        args = (self._h, c.ctypes.data, None if mk is None else mk.ctypes.data, mask_mode, _lib.NVB_MEM_HOST, c.shape[0],
                c.shape[1], _fp(T), C.byref(camera.c))
        if not return_blocks:
            check(self._L.nvb_mapper_integrate_color(*args, None, 0, None))
            return None
        return _block_list(self._L.nvb_mapper_integrate_color, 1 << 14, *args,
                           reread=(self._L.nvb_mapper_last_color_blocks, self._h))

    def integrate_color_device(self, color_ptr, rows, cols, T_L_C, camera, mask_ptr=0, mask_mode=0):
        """Same, for an RGB frame already resident in HBM (raw device pointers); enqueued without synchronising."""
        T = colmajor(T_L_C)
        check(self._L.nvb_mapper_integrate_color(self._h, color_ptr, mask_ptr or None, mask_mode, _lib.NVB_MEM_DEVICE, rows, cols,
                                                 _fp(T), C.byref(camera.c), None, 0, None))

    def last_color_blocks(self):
        """updated_blocks of the last colour frame (after synchronize())."""
        n = C.c_int32(0)
        check(self._L.nvb_mapper_last_color_blocks(self._h, None, 0, C.byref(n)))
        return _block_list(self._L.nvb_mapper_last_color_blocks, n.value, self._h)

    def freespace_integrator(self):
        return _FreespaceIntegrator(self)

    def update_freespace(self, update_time_ms, depth=None, T_L_C=None, camera=None, update_full_layer=False):
        """Mapper::updateFreespace(update_time_ms, T_L_C, sensor, depth_frame, update_full_layer) (mapper.h:196-214)."""
        if depth is not None:
            depth = np.ascontiguousarray(depth, dtype=np.float32)
            T = colmajor(T_L_C)
            check(self._L.nvb_mapper_update_freespace(self._h, int(update_time_ms), depth.ctypes.data, _lib.NVB_MEM_HOST,
                                                      depth.shape[0], depth.shape[1], _fp(T), C.byref(camera.c),
                                                      1 if update_full_layer else 0))
        else:
            check(self._L.nvb_mapper_update_freespace(self._h, int(update_time_ms), None, 0, 0, 0, None, None,
                                                      1 if update_full_layer else 0))

    def esdf_layer(self):
        return self._esdf

    def esdf_dense_grid_in_aabb(self, aabb, default_value):
        """voxelLayerToDenseVoxelGridInAABBAsync on the ESDF layer with the EsdfAndGradients service's conversion: aabb =
        (6,) {min xyz, max xyz} in metres -> (min_index (3,) int32, (X, Y, Z) float32 grid of distances in metres, negative
        inside, `default_value` where unknown). An empty box gives an empty grid."""
        box = np.ascontiguousarray(aabb, dtype=np.float32).reshape(6)
        mn, dims = np.zeros(3, np.int32), np.zeros(3, np.int32)
        check(self._L.nvb_esdf_dense_grid_in_aabb(self._h, _fp(box), float(default_value), _lib.NVB_MEM_HOST, None, 0, _ip(mn),
                                                  _ip(dims)))
        out = np.zeros(max(int(np.prod(dims.astype(np.int64))), 1), np.float32)
        if dims.all():
            check(self._L.nvb_esdf_dense_grid_in_aabb(self._h, _fp(box), float(default_value), _lib.NVB_MEM_HOST,
                                                      out.ctypes.data, out.size, _ip(mn), _ip(dims)))
        return mn, out[:int(np.prod(dims.astype(np.int64)))].reshape(tuple(int(d) for d in dims))

    def projective_layer_type(self):
        return self._projective_layer_type

    def tsdf_integrator(self):
        return _TsdfIntegrator(self)

    def occupancy_integrator(self):
        return _OccupancyIntegrator(self)

    def esdf_integrator(self):
        return _EsdfIntegrator(self)

    def tsdf_decay_integrator(self):
        return _DecayIntegrator(self, False)

    def occupancy_decay_integrator(self):
        return _DecayIntegrator(self, True)

    def decay(self, depth=None, T_L_C=None, camera=None, excluded_blocks=None, exclusion_center=None,
              exclusion_radius_m=None):
        """Mapper::decayTsdf / decayOccupancy on the mapper's projective layer (mapper.h:268-292). depth=None: every
        voxel decays (decay*AllVoxels); with a view, voxels that have a depth measurement in it are spared
        (decay*ExcludeLastView -- pass the last integrated frame). Returns the (n,3) indices of the deallocated
        blocks (gone from the projective and the ESDF layer)."""
        x = NvbDecayExclusion()
        keep = None
        if excluded_blocks is not None and len(excluded_blocks):
            keep = np.ascontiguousarray(excluded_blocks, dtype=np.int32).reshape(-1, 3)
            x.excluded_blocks_xyz_host, x.num_excluded_blocks = _ip(keep), keep.shape[0]
        if exclusion_center is not None and exclusion_radius_m is not None:
            x.has_exclusion_sphere = 1
            x.exclusion_center = (C.c_float * 3)(*[float(v) for v in exclusion_center])
            x.exclusion_radius_m = float(exclusion_radius_m)
        if depth is not None:
            depth = np.ascontiguousarray(depth, dtype=np.float32)
            T = colmajor(T_L_C)
            view = (depth.ctypes.data, _lib.NVB_MEM_HOST, depth.shape[0], depth.shape[1], _fp(T), C.byref(camera.c))
        else:
            view = (None, 0, 0, 0, None, None)
        return _block_list(self._L.nvb_mapper_decay, self._projective_num_blocks(), self._h, C.byref(x), *view)

    def clear_outside_radius(self, center, radius):
        """Mapper::clearOutsideRadius(center, radius) (mapper.h; src/mapper/mapper.cpp:473-492): deallocates every projective
        block farther than `radius` from `center`, with its ESDF, freespace, colour and mesh twins. Returns the removed (n, 3)
        block indices in (x, y, z) order."""
        c = np.ascontiguousarray(center, dtype=np.float32).reshape(3)
        return _block_list(self._L.nvb_mapper_clear_outside_radius, self._projective_num_blocks(), self._h, _fp(c),
                           float(radius))

    def clear_tsdf_inside_shapes(self, shapes):
        """Mapper::clearTsdfInsideShapes(shapes) (src/mapper/mapper.cpp:364-368): TSDF voxels inside the shapes are reset and
        their blocks join the tracker. Returns the touched (n, 3) block indices in (x, y, z) order (none on an occupancy
        mapper)."""
        arr, n = _shape_array(shapes)
        cap = self._tsdf.num_blocks() if self._projective_layer_type != ProjectiveLayerType.kOccupancy else 0
        return _block_list(self._L.nvb_mapper_clear_tsdf_inside_shapes, cap, self._h, arr, n)

    def get_cleared_blocks(self, blocks_to_ignore=()):
        """Mapper::getClearedBlocks(blocks_to_ignore) (src/mapper/mapper.cpp:509-521): the blocks deallocated by
        clear_outside_radius or a decay since the last call, minus `blocks_to_ignore`, in (x, y, z) order; empties the set."""
        ign = np.ascontiguousarray(np.asarray(blocks_to_ignore, dtype=np.int32).reshape(-1, 3))
        n = C.c_int32(0)
        check(self._L.nvb_mapper_get_cleared_blocks(self._h, None, 0, None, 0, C.byref(n)))
        return _block_list(self._L.nvb_mapper_get_cleared_blocks, n.value, self._h, _ip(ign) if len(ign) else None, len(ign))

    def decay_exclude_last_view(self):
        """Mapper::decayTsdfExcludeLastView / decayOccupancyExcludeLastView with the view kept by the mapper
        (Mapper(..., keep_last_view=True))."""
        return _block_list(self._L.nvb_mapper_decay_exclude_last_view, self._projective_num_blocks(), self._h, None)

    def _projective_num_blocks(self):
        """Blocks of the projective layer: a bound on what a decay or a clear removes."""
        return (self._occupancy if self._projective_layer_type == ProjectiveLayerType.kOccupancy else self._tsdf).num_blocks()

    def decay_tsdf(self, **kw):
        assert self._projective_layer_type != ProjectiveLayerType.kOccupancy
        return self.decay(**kw)

    def decay_occupancy(self, **kw):
        assert self._projective_layer_type == ProjectiveLayerType.kOccupancy
        return self.decay(**kw)

    def cuda_stream(self):
        return self._L.nvb_mapper_stream(self._h)

    def esdf_reserved_sms(self, v=None):
        """SMs the ESDF wavefront leaves to concurrently running kernels (default 2; 4 on a multi-GPU rank that merges)."""
        if v is not None:
            check(self._L.nvb_mapper_set_esdf_reserved_sms(self._h, int(v)))
        return int(self._L.nvb_mapper_get_esdf_reserved_sms(self._h))

    def do_depth_preprocessing(self, v=None):
        """Mapper::do_depth_preprocessing (mapper.h; mapper_params.h:33-37, default off)."""
        en, n = C.c_int32(0), C.c_int32(0)
        check(self._L.nvb_mapper_get_depth_preprocessing(self._h, C.byref(en), C.byref(n)))
        if v is not None:
            check(self._L.nvb_mapper_set_depth_preprocessing(self._h, 1 if v else 0, n.value))
            return bool(v)
        return bool(en.value)

    def depth_preprocessing_num_dilations(self, v=None):
        """Mapper::depth_preprocessing_num_dilations (mapper_params.h:39-42, default 4)."""
        en, n = C.c_int32(0), C.c_int32(0)
        check(self._L.nvb_mapper_get_depth_preprocessing(self._h, C.byref(en), C.byref(n)))
        if v is not None:
            check(self._L.nvb_mapper_set_depth_preprocessing(self._h, en.value, int(v)))
            return int(v)
        return int(n.value)

    def dilate_invalid_regions_device(self, depth_ptr, out_ptr, rows, cols, num_dilations, invalid_depth_threshold=1e-2,
                                      invalid_depth_value=0.0):
        """DepthPreprocessor::dilateInvalidRegionsAsync (sensors/depth_preprocessing.h:33-38) on device images, enqueued on
        cuda_stream(); the output must not alias the input."""
        check(self._L.nvb_depth_dilate_invalid(self._h, depth_ptr, out_ptr, rows, cols, int(num_dilations),
                                               float(invalid_depth_threshold), float(invalid_depth_value)))

    def clear(self):
        check(self._L.nvb_mapper_clear(self._h))

    # --- map files (Mapper::saveLayerCake / loadMap, src/mapper/mapper.cpp:636-687) and voxel PLY export ------------
    MAP_FILE_LAYERS = ("tsdf", "esdf", "occupancy", "freespace", "color", "feature")

    def save_layer_cake(self, path):
        """Writes the map to `path` (truncated) in the reference's .nvblx format: all six layers' tables, rows in (x, y, z)
        block-index order."""
        check(self._L.nvb_mapper_save_map(self._h, os.fsencode(path)))
        return True

    def load_map(self, path):
        """Replaces the map with the one in `path`; the voxel size follows the file. Returns the blocks loaded per layer,
        {"tsdf", "esdf", "occupancy", "freespace", "color", "feature"}: 0 for a table this mapper cannot hold (skipped)."""
        out = (C.c_int32 * 6)()
        check(self._L.nvb_mapper_load_map(self._h, os.fsencode(path), out))
        return dict(zip(self.MAP_FILE_LAYERS, list(out)))

    def _save_layer_as_ply(self, layer, filename):
        pts = layer.export_points()
        return _io.output_points_to_ply(pts[:, :3], pts[:, 3], filename)

    def save_tsdf_as_ply(self, filename):
        """Mapper::saveTsdfAsPly: io::outputVoxelLayerToPly(tsdf_layer()). False (no file) without points."""
        return self._save_layer_as_ply(self._tsdf, filename)

    def save_esdf_as_ply(self, filename):
        return self._save_layer_as_ply(self._esdf, filename)

    def save_occupancy_as_ply(self, filename):
        return self._save_layer_as_ply(self._occupancy, filename)

    def save_freespace_as_ply(self, filename):
        return self._save_layer_as_ply(self._freespace, filename)

    # --- the hot path ----------------------------------------------------
    @staticmethod
    def _frame_args(depth, mask):
        if isinstance(depth, (int, np.integer)):
            raise TypeError("pass device frames through integrate_depth_device")
        d = np.ascontiguousarray(depth, dtype=np.float32)
        mk = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        return d, mk

    def integrate_depth(self, depth, T_L_C, camera, mask=None, mask_mode=0, return_blocks=True):
        """Mapper::integrateDepth. depth: (rows, cols) float32 host array. Returns updated_blocks (n,3)."""
        d, mk = self._frame_args(depth, mask)
        T = colmajor(T_L_C)
        args = (self._h, d.ctypes.data, None if mk is None else mk.ctypes.data, mask_mode, _lib.NVB_MEM_HOST, d.shape[0],
                d.shape[1], _fp(T), C.byref(camera.c))
        if not return_blocks:
            check(self._L.nvb_mapper_integrate_depth(*args, None, 0, None))
            return None
        return _block_list(self._L.nvb_mapper_integrate_depth, 1 << 14, *args,
                           reread=(self._L.nvb_mapper_last_frame_blocks, self._h))

    def integrate_depth_device(self, depth_ptr, rows, cols, T_L_C, camera, mask_ptr=0, mask_mode=0, sync=False):
        """Same, for a frame already resident in HBM (raw device pointers). Asynchronous unless sync."""
        T = colmajor(T_L_C)
        check(self._L.nvb_mapper_integrate_depth_async(self._h, depth_ptr, mask_ptr or None, mask_mode,
                                                       _lib.NVB_MEM_DEVICE, rows, cols, _fp(T), C.byref(camera.c)))
        if sync:
            self.synchronize()

    def integrate_depth_async(self, depth, T_L_C, camera, mask=None, mask_mode=0):
        """Host frame, enqueued without synchronising (buffers are kept alive until synchronize())."""
        d, mk = self._frame_args(depth, mask)
        T = colmajor(T_L_C)
        self._keep.append((d, mk))
        check(self._L.nvb_mapper_integrate_depth_async(self._h, d.ctypes.data, None if mk is None else mk.ctypes.data,
                                                       mask_mode, _lib.NVB_MEM_HOST, d.shape[0], d.shape[1], _fp(T),
                                                       C.byref(camera.c)))

    def integrate_depth_host_ptr_async(self, depth_host_ptr, rows, cols, T_L_C, camera):
        """Host frame given as a raw (ideally pinned) pointer the caller keeps alive."""
        T = colmajor(T_L_C)
        check(self._L.nvb_mapper_integrate_depth_async(self._h, depth_host_ptr, None, 0, _lib.NVB_MEM_HOST, rows, cols,
                                                       _fp(T), C.byref(camera.c)))

    def update_esdf(self, update_full_layer=False, sync=True):
        """Mapper::updateEsdf."""
        if sync:
            check(self._L.nvb_mapper_update_esdf(self._h, 1 if update_full_layer else 0))
            self._keep.clear()
        else:
            check(self._L.nvb_mapper_update_esdf_async(self._h, 1 if update_full_layer else 0))

    def update_esdf_slice(self, update_full_layer=False, ground_plane=None):
        """Mapper::updateEsdfSlice(update_full_layer, ground_plane) (mapper.h:331-343): the 2-D ESDF on the slice layer."""
        if ground_plane is None:
            check(self._L.nvb_mapper_update_esdf_slice(self._h, 1 if update_full_layer else 0))
        else:
            pl = np.ascontiguousarray(ground_plane, dtype=np.float32).reshape(4)
            check(self._L.nvb_mapper_update_esdf_slice_planar(self._h, _fp(pl), 1 if update_full_layer else 0))

    def synchronize(self):
        check(self._L.nvb_mapper_synchronize(self._h))
        self._keep.clear()

    def join_streams(self):
        """Make later work on cuda_stream() wait for the ESDF side stream (device-side, no host sync)."""
        check(self._L.nvb_mapper_join_streams(self._h))

    def last_frame_block_count(self):
        n = C.c_int32(0)
        check(self._L.nvb_mapper_last_frame_block_count(self._h, C.byref(n)))
        return n.value

    # --- instrumentation -------------------------------------------------
    def enable_profiling(self, on=True):
        check(self._L.nvb_mapper_enable_profiling(self._h, 1 if on else 0))

    def stage_times(self, reset=False):
        ms = (C.c_double * 6)()
        calls = (C.c_int64 * 6)()
        check(self._L.nvb_mapper_stage_times(self._h, ms, calls, 1 if reset else 0))
        return {STAGE_NAMES[i]: (ms[i], calls[i]) for i in range(6)}

    def kernel_launches(self):
        return int(self._L.nvb_mapper_kernel_launches(self._h))


class ViewCalculator:
    """ViewCalculator::getBlocksInImageViewRaycast (view_calculator.h:75-80)."""

    def __init__(self, mapper):
        self._m = mapper

    def get_blocks_in_image_view_raycast(self, depth, T_L_C, camera, block_size,
                                         max_integration_distance_behind_surface_m, max_integration_distance_m):
        d = np.ascontiguousarray(depth, dtype=np.float32)
        T = colmajor(T_L_C)
        L, h = self._m._L, self._m._h
        return _block_list(L.nvb_view_raycast, 1 << 16, h, d.ctypes.data, _lib.NVB_MEM_HOST, d.shape[0], d.shape[1], _fp(T),
                           C.byref(camera.c), float(block_size), float(max_integration_distance_behind_surface_m),
                           float(max_integration_distance_m), reread=(L.nvb_mapper_last_frame_blocks, h))
