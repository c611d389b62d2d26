"""H100-native drop-in for nvblox_core's depth-integration hot path.

ViewCalculator raycast -> ProjectiveTsdfIntegrator::integrateFrame ->
EsdfIntegrator::integrateBlocks, behind nvblox::Mapper's interface, as hand-written
sm_90a kernels in libnvblox_b200.so (C-ABI: include/nvblox_b200.h).
"""
from .mapper import (AxisAlignedBoundingBox, BoundingSphere, Camera, DynamicsDetection, EsdfSlicer, GroundPlaneEstimator, ImageMasker, Mapper, ProjectiveLayerType, ViewCalculator, ESDF_VOXEL_DTYPE,  # noqa: F401
                     OCCUPANCY_VOXEL_DTYPE, FREESPACE_VOXEL_DTYPE, COLOR_VOXEL_DTYPE, TSDF_VOXEL_DTYPE, STAGE_NAMES,
                     ransac_fit_plane, remove_small_connected_components)  # noqa: F401
from . import synthetic  # noqa: F401

__all__ = ["AxisAlignedBoundingBox", "BoundingSphere", "Camera", "DynamicsDetection", "EsdfSlicer", "GroundPlaneEstimator", "ImageMasker", "Mapper", "ProjectiveLayerType", "ViewCalculator", "ESDF_VOXEL_DTYPE", "OCCUPANCY_VOXEL_DTYPE", "FREESPACE_VOXEL_DTYPE", "COLOR_VOXEL_DTYPE",
           "TSDF_VOXEL_DTYPE", "STAGE_NAMES", "ransac_fit_plane", "remove_small_connected_components", "synthetic"]
