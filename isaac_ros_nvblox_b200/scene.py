"""Scenes of primitives (planes, cubes, spheres, cylinders) and the exact maps and depth images they give, computed on the GPU:
nvblox::primitives::Scene (primitives/scene.h) and nvblox_torch's Scene (nvblox_torch/scene.py, cpp/src/py_scene.cu), with
their names.

nvblox_torch's methods are all here. `add_primitive('plane', params)` takes the centre, then the unit normal, which is what
py_scene.cu does whatever its docstring says; a 'cylinder' takes the centre, the radius and the height (axis along z).
`to_mapper` returns one Mapper for one voxel size and a list of Mappers for several, the forms `query_layer` accepts.

The direct methods `render_depth`, `signed_distance` and `generate_layer` are Scene::generateDepthImageFromScene,
getSignedDistanceToPoint and generateLayerFromScene. They take float32 CUDA tensors, enqueued on torch's current stream
without synchronising, or numpy arrays, computed before the call returns.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import NvbPrimitive, NvbScene, check
from .mapper import Mapper, ProjectiveLayerType, _device_points, _fp, _is_tensor, colmajor

# Primitive::toString (src/primitives/primitives.cpp), by NVB_PRIM_* type
TYPE_NAMES = ("kPlane", "kCube", "kSphere", "kCylinder")
_PARAMS = {"cube": (_lib.NVB_PRIM_CUBE, 6), "sphere": (_lib.NVB_PRIM_SPHERE, 4), "plane": (_lib.NVB_PRIM_PLANE, 6),
           "cylinder": (_lib.NVB_PRIM_CYLINDER, 5)}
# Scene::Scene() (src/primitives/scene.cpp)
DEFAULT_AABB = ((-5.0, -5.0, -1.0), (5.0, 5.0, 9.0))


class Scene:
    """A set of primitives and the AABB a generated layer covers."""

    def __init__(self):
        self._L = _lib.load()
        self._prims = []  # NvbPrimitive, in insertion order
        self._aabb = [list(DEFAULT_AABB[0]), list(DEFAULT_AABB[1])]

    # --- nvblox_torch's Scene ------------------------------------------------------------------------------------------
    def set_aabb(self, low, high):
        assert len(low) == 3
        assert len(high) == 3
        self._aabb = [[float(np.float32(v)) for v in low], [float(np.float32(v)) for v in high]]

    def get_aabb(self):
        return list(self._aabb[0]), list(self._aabb[1])

    def _add(self, type_, center, params):
        p = list(params) + [0.0] * (4 - len(params))
        self._prims.append(NvbPrimitive(type_, (C.c_float * 3)(*map(float, center)), (C.c_float * 4)(*map(float, p))))

    def add_plane_boundaries(self, x_min, x_max, y_min, y_max):
        """Scene::addPlaneBoundaries: four planes facing inwards, x_min, x_max, y_min, y_max in that order."""
        self._add(_lib.NVB_PRIM_PLANE, (x_min, 0, 0), (1, 0, 0))
        self._add(_lib.NVB_PRIM_PLANE, (x_max, 0, 0), (-1, 0, 0))
        self._add(_lib.NVB_PRIM_PLANE, (0, y_min, 0), (0, 1, 0))
        self._add(_lib.NVB_PRIM_PLANE, (0, y_max, 0), (0, -1, 0))

    def add_ground_level(self, level):
        self._add(_lib.NVB_PRIM_PLANE, (0, 0, level), (0, 0, 1))

    def add_ceiling(self, ceiling):
        self._add(_lib.NVB_PRIM_PLANE, (0, 0, ceiling), (0, 0, -1))

    def add_primitive(self, primitive_type, params):
        """'cube': centre + size (6), 'sphere': centre + radius (4), 'plane': centre + unit normal (6), 'cylinder': centre +
        radius + height (5). A plane's normal must have norm 1 +- 1e-3 (the reference's CHECK_NEAR)."""
        if primitive_type not in _PARAMS:
            raise ValueError("unknown primitive type %r" % (primitive_type,))
        type_, n = _PARAMS[primitive_type]
        params = [float(v) for v in params]
        if len(params) != n:
            raise ValueError("a %s takes %d parameters, not %d" % (primitive_type, n, len(params)))
        if type_ == _lib.NVB_PRIM_PLANE:
            nx, ny, nz = np.float32(params[3]), np.float32(params[4]), np.float32(params[5])
            norm = float(np.sqrt(nx * nx + (ny * ny + nz * nz)))
            if not (1.0 - 1e-3 <= norm <= 1.0 + 1e-3):
                raise ValueError("a plane's normal must be unit length, not %g" % norm)
        self._add(type_, params[:3], params[3:])

    def create_dummy_map(self):
        """py_scene.cu's createDummyMap: a box of four walls, floor and ceiling around a cube and a sphere."""
        self.set_aabb([-5.5, -5.5, -0.5], [5.5, 5.5, 5.5])
        self.add_plane_boundaries(-5.0, 5.0, -5.0, 5.0)
        self.add_ground_level(0.0)
        self.add_ceiling(5.0)
        self.add_primitive("cube", [0.0, 0.0, 2.0, 2.0, 2.0, 2.0])
        self.add_primitive("sphere", [0.0, 0.0, 2.0, 2.0])

    def get_primitives_type_list(self):
        return [TYPE_NAMES[p.type] for p in self._prims]

    def clear(self):
        self._prims = []

    def append_to_mapper(self, mapper, mapper_id=-1):
        """Scene::toMapper: each mapper (or mappers[mapper_id]) gets the scene's projective layer with max_dist = 4 voxels,
        every block marked for update, then its ESDF updated."""
        mappers = list(mapper) if isinstance(mapper, (list, tuple)) else [mapper]
        if mapper_id >= 0:
            mappers = [mappers[mapper_id]]
        s = self._c()
        for m in mappers:
            check(self._L.nvb_scene_to_mapper(m._h, C.byref(s)))

    def to_mapper(self, voxel_sizes_m, integrator_types=None, mapper_parameters=None, mapper_id=-1, device=0):
        """New mappers, one per voxel size (ProjectiveLayerType per mapper, TSDF by default), with the scene appended.
        mapper_parameters takes the place of nvblox_torch's MapperParams: None, or a dict of keyword arguments for each new
        Mapper. -> a Mapper for one voxel size, else a list of them."""
        sizes = list(voxel_sizes_m)
        types = list(integrator_types) if integrator_types is not None else [ProjectiveLayerType.kTsdf] * len(sizes)
        if len(types) != len(sizes):
            raise ValueError("one integrator type per voxel size")
        if mapper_parameters is not None and not isinstance(mapper_parameters, dict):
            raise TypeError("mapper_parameters must be None or a dict of Mapper keyword arguments")
        kw = dict(mapper_parameters or {})
        mappers = [Mapper(v, device=device, projective_layer_type=t, **kw) for v, t in zip(sizes, types)]
        self.append_to_mapper(mappers, mapper_id)
        return mappers[0] if len(mappers) == 1 else mappers

    # --- Scene on the GPU --------------------------------------------------------------------------------------------
    def _c(self):
        arr = (NvbPrimitive * max(len(self._prims), 1))(*self._prims)
        s = NvbScene(C.cast(arr, C.POINTER(NvbPrimitive)), len(self._prims), (C.c_float * 3)(*self._aabb[0]),
                     (C.c_float * 3)(*self._aabb[1]))
        s._keep = arr
        return s

    def render_depth(self, camera, T_S_C, max_dist, invalid_depth=0.0, device=None):
        """generateDepthImageFromScene(camera, T_S_C, max_dist, &depth, invalid_depth) -> (height, width) float32: the camera-
        frame z of each pixel's nearest hit, invalid_depth where there is none. A CUDA tensor on `device` (an int; torch's
        current stream) or, with device=None, a numpy array."""
        s, T = self._c(), colmajor(T_S_C)
        if device is None:
            out = np.empty((camera.height, camera.width), np.float32)
            check(self._L.nvb_scene_render_depth(C.byref(s), C.byref(camera.c), _fp(T), float(max_dist), float(invalid_depth),
                                                 _lib.NVB_MEM_HOST, out.ctypes.data, None))
            return out
        import torch
        dev = torch.device("cuda", int(device))
        out = torch.empty((camera.height, camera.width), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            check(self._L.nvb_scene_render_depth(C.byref(s), C.byref(camera.c), _fp(T), float(max_dist), float(invalid_depth),
                                                 _lib.NVB_MEM_DEVICE, out.data_ptr(), stream))
        return out

    def signed_distance(self, points, max_dist):
        """getSignedDistanceToPoint of each of the (n, 3) points -> (n,) float32, on the device of a CUDA tensor (torch's
        current stream) or as numpy."""
        s = self._c()
        if _is_tensor(points):
            import torch
            pts = _device_points(points, 3, points.device.index)
            out = torch.empty((pts.shape[0],), dtype=torch.float32, device=pts.device)
            with torch.cuda.device(pts.device):
                stream = C.c_void_p(torch.cuda.current_stream(pts.device).cuda_stream)
                check(self._L.nvb_scene_signed_distance(C.byref(s), pts.data_ptr(), _lib.NVB_MEM_DEVICE, pts.shape[0],
                                                        float(max_dist), out.data_ptr(), stream))
            return out
        pts = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
        out = np.empty((pts.shape[0],), np.float32)
        check(self._L.nvb_scene_signed_distance(C.byref(s), pts.ctypes.data, _lib.NVB_MEM_HOST, pts.shape[0], float(max_dist),
                                                out.ctypes.data, None))
        return out

    def generate_layer(self, mapper, layer_id, max_dist):
        """generateLayerFromScene(max_dist, layer) on the mapper's TSDF, occupancy or freespace layer (an NVB_LAYER_* id):
        allocates the blocks the AABB touches and writes every voxel inside it. The block-update tracker is not told."""
        check(self._L.nvb_scene_generate_layer(mapper._h, int(layer_id), C.byref(self._c()), float(max_dist)))


def getSphereInBox():
    """The reference tests' sphere in a box (tests/lib/integrator_utils.cpp): AABB (-5, -5, 0) to (5, 5, 5), floor at 0,
    ceiling at 5, a sphere of radius 2 at (0, 0, 2), and walls at +-5 in x and y."""
    s = Scene()
    s.set_aabb([-5.0, -5.0, 0.0], [5.0, 5.0, 5.0])
    s.add_ground_level(0.0)
    s.add_ceiling(5.0)
    s.add_primitive("sphere", [0.0, 0.0, 2.0, 2.0])
    s.add_plane_boundaries(-5.0, 5.0, -5.0, 5.0)
    return s
