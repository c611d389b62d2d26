"""Depth and colour images of a mapper's map, rendered on the GPU by sphere tracing its TSDF layer: nvblox::SphereTracer
(rays/sphere_tracer.h) and nvblox_torch's rendering functions (nvblox_torch/rendering.py), with their names and argument
order. nvblox_torch's functions take layer views; these take the Mapper whose TSDF (and colour) layer is rendered.

Outputs are CUDA tensors on the mapper's device: an (H, W) float32 depth image, -1 where a ray found no surface, and an
(H, W, 3) uint8 RGB image, black where no surface or no colour block was found. A render is enqueued on torch's current
stream after the work already on it and on the mapper, and the mapper's later work follows it; nothing synchronises.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import NvbSphereTracerParams, check
from .mapper import Camera, _fp, colmajor

# nvblox_torch/cpp/src/py_rendering.cpp: the truncation distance is 4 voxels (projective_integrator_base.h's default)
TRUNCATION_DISTANCE_VOX = 4.0


class SphereTracer:
    """nvblox::SphereTracer: maximum_steps 100, maximum_ray_length_m 15, surface_distance_epsilon_vox 0.1 by default. Each
    parameter method is the reference's getter without an argument and its setter with one; a setter rejects values that are
    not positive, as the reference's CHECK_GTs do."""

    def __init__(self):
        self._L = _lib.load()
        self._p = NvbSphereTracerParams()
        self._L.nvb_default_sphere_tracer_params(C.byref(self._p))

    def _param(self, name, v, cast):
        if v is not None:
            if not cast(v) > 0:
                raise ValueError("%s must be positive" % name)
            setattr(self._p, name, cast(v))
        return getattr(self._p, name)

    def maximum_steps(self, v=None):
        return self._param("maximum_steps", v, int)

    def maximum_ray_length_m(self, v=None):
        return self._param("maximum_ray_length_m", v, float)

    def surface_distance_epsilon_vox(self, v=None):
        return self._param("surface_distance_epsilon_vox", v, float)

    @staticmethod
    def get_subsampled_image_size(camera, subsampling_factor):
        """getSubsampledImageSize -> (rows, cols) = (height / f, width / f)."""
        f = int(subsampling_factor)
        return camera.height // f, camera.width // f

    def _render(self, mapper, T_L_C, camera, truncation_distance_m, ray_subsampling_factor, rgb):
        f = int(ray_subsampling_factor)
        rows, cols = self.get_subsampled_image_size(camera, f) if f > 0 else (0, 0)
        dev = torch.device("cuda", mapper._device)
        depth = torch.empty((rows, cols), dtype=torch.float32, device=dev)
        color = torch.empty((rows, cols, 3), dtype=torch.uint8, device=dev) if rgb else None
        T = colmajor(T_L_C)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        args = (mapper._h, C.byref(self._p), _fp(T), C.byref(camera.c), float(truncation_distance_m), f, _lib.NVB_MEM_DEVICE,
                depth.data_ptr())
        if rgb:
            check(self._L.nvb_render_rgbd(*args, color.data_ptr(), stream))
            return depth, color
        check(self._L.nvb_render_depth(*args, stream))
        return depth

    def render_depth(self, mapper, T_L_C, camera, truncation_distance_m, ray_subsampling_factor=1):
        """renderImageOnGPU(camera, T_L_C, tsdf_layer, truncation_distance_m, &depth, kDevice, ray_subsampling_factor) of the
        mapper's TSDF layer -> (height / f, width / f) float32 CUDA tensor."""
        return self._render(mapper, T_L_C, camera, truncation_distance_m, ray_subsampling_factor, False)

    def render_rgbd(self, mapper, T_L_C, camera, truncation_distance_m, ray_subsampling_factor=1):
        """renderRgbdImageOnGPU(camera, T_L_C, tsdf_layer, color_layer, ...) of the mapper's layers -> (depth, colour): the
        colour of the voxel holding each hit point whatever its weight (grey 127 in a block that was never coloured). A
        mapper that never integrated colour renders black."""
        return self._render(mapper, T_L_C, camera, truncation_distance_m, ray_subsampling_factor, True)


def _args(mapper, camera_pose, intrinsics, height, width, max_ray_length, max_steps):
    """py_rendering.cpp: T_L_C from the 4x4 pose, the camera from K's fu, fv, cu, cv, a tracer with the given ray length and
    steps, truncation = 4 voxels."""
    T = torch.as_tensor(camera_pose).detach().to("cpu", torch.float32).numpy()
    K = torch.as_tensor(intrinsics).detach().to("cpu", torch.float32).numpy()
    if T.shape != (4, 4) or K.shape != (3, 3):
        raise ValueError("camera_pose must be 4x4 and intrinsics 3x3")
    cam = Camera(K[0, 0], K[1, 1], K[0, 2], K[1, 2], int(width), int(height))
    tracer = SphereTracer()
    tracer.maximum_ray_length_m(max_ray_length)
    tracer.maximum_steps(max_steps)
    trunc = np.float32(mapper.voxel_size()) * np.float32(TRUNCATION_DISTANCE_VOX)
    return tracer, T, cam, trunc


def render_depth_image(mapper, camera_pose, intrinsics, height, width, max_ray_length, max_steps):
    """nvblox_torch.rendering.render_depth_image on the mapper's TSDF layer. camera_pose is T_L_C (camera to layer, which is
    what nvblox_torch's binding uses); intrinsics is the 3x3 K matrix. -> (height, width) float32 CUDA tensor."""
    tracer, T, cam, trunc = _args(mapper, camera_pose, intrinsics, height, width, max_ray_length, max_steps)
    return tracer.render_depth(mapper, T, cam, trunc)


def render_depth_and_color_image(mapper, camera_pose, intrinsics, height, width, max_ray_length, max_steps):
    """nvblox_torch.rendering.render_depth_and_color_image on the mapper's TSDF and colour layers -> ((height, width) float32,
    (height, width, 3) uint8) CUDA tensors."""
    tracer, T, cam, trunc = _args(mapper, camera_pose, intrinsics, height, width, max_ray_length, max_steps)
    return tracer.render_rgbd(mapper, T, cam, trunc)
