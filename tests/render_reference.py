"""A restatement of SphereTracer's depth and RGBD renders (src/rays/sphere_tracer.cu: sphereTracingKernel :134-173,
sphereTracingKernelWithColor :239-300) for the tests, in binary32.

Each ray's direction is computed in numpy float32 with the kernel's operation order (pixel coordinate f * (c, r) + f / 2,
Camera::vectorFromImagePlaneCoordinates, Eigen's normalized(), then T_L_C's rotation, sums as a0 + (a1 + a2)); a distorted
camera takes its undistorted ray from the oracle (or_camera_vector_from_image_plane). The cast itself is the oracle's
single-ray SphereTracer::castOnGPU (or_sphere_trace_ray), on an OracleMap holding the TSDF blocks. From the converged t the
depth is t * d_C.z, and the colour is that of the voxel holding origin + t * d_L (getBlockAndVoxelIndexFromPositionInLayer)
in a {block index: (8, 8, 8) COLOR_VOXEL_DTYPE} layer, whatever its weight; a miss, or a hit without a colour block, is -1
and black. No operation is contracted into an FMA (numpy rounds each one, the oracle is built with -ffp-contract=off).
"""
import ctypes as C

import numpy as np

F = np.float32


def pixel_rays(cam, T_L_C, f):
    """-> (dz (rows, cols), dir_L (rows, cols, 3)) float32 of the f-subsampled image's rays. cam is an oracle Camera."""
    from oracle import oracle as orc
    T = np.asarray(T_L_C, F)
    rows, cols = cam.height // f, cam.width // f
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    half = F(0.5) * F(f)
    px = (c * f).astype(F) + half * F(1.0)
    py = (r * f).astype(F) + half * F(1.0)
    if cam.has_distortion:
        v = np.array([[orc.camera_vector_from_image_plane(cam, u, w) for u, w in zip(pu, pw)] for pu, pw in zip(px, py)], F)
        nx, ny = v[..., 0], v[..., 1]
    else:
        nx = (px - F(cam.cu)) / F(cam.fu)
        ny = (py - F(cam.cv)) / F(cam.fv)
    one = F(1.0)
    norm = np.sqrt(nx * nx + (ny * ny + one * one))
    dx, dy, dz = nx / norm, ny / norm, one / norm
    R = T[:3, :3]
    d = np.stack([R[i, 0] * dx + (R[i, 1] * dy + R[i, 2] * dz) for i in range(3)], axis=-1).astype(F)
    return dz.astype(F), d


def voxel_index(p, block_size):
    """getBlockAndVoxelIndexFromPositionInLayer in binary32 for (..., 3) points -> (block (..., 3), voxel (..., 3)) int64."""
    bs = F(block_size)
    inv = F(1.0 / float(bs * F(0.125)))
    b = np.floor(p / bs).astype(np.int64)
    v = np.minimum(((p - bs * b.astype(F)) * inv).astype(np.int64), 7)
    return b, v


def _pack(idx):
    """(n, 3) block indices -> sortable int64 keys (each component biased into 22 bits)."""
    k = idx.astype(np.int64) + (1 << 21)
    return (k[:, 0] << 44) | (k[:, 1] << 22) | k[:, 2]


def render(o, T_L_C, cam, truncation_distance_m, color_layer=None, maximum_steps=100, maximum_ray_length_m=15.0,
           surface_distance_epsilon_m=None, ray_subsampling_factor=1):
    """-> (depth (rows / f, cols / f) float32, rgb (rows / f, cols / f, 3) uint8) of the OracleMap o's TSDF layer and the
    colour layer dict (None: no colour layer, every hit black)."""
    from oracle import oracle as orc
    f = int(ray_subsampling_factor)
    if surface_distance_epsilon_m is None:
        surface_distance_epsilon_m = F(0.1) * F(o.voxel_size)
    dz, dirs = pixel_rays(cam, T_L_C, f)
    T = np.asarray(T_L_C, F)
    origin = np.ascontiguousarray(T[:3, 3])
    fp = C.POINTER(C.c_float)
    o_buf = (C.c_float * 3)(*origin.tolist())
    d_buf, t_buf = (C.c_float * 3)(), (C.c_float * 1)()
    cast = orc.lib().or_sphere_trace_ray
    args = (float(truncation_distance_m), int(maximum_steps), float(maximum_ray_length_m), float(surface_distance_epsilon_m))
    flat = dirs.reshape(-1, 3)
    t = np.zeros(flat.shape[0], F)
    ok = np.zeros(flat.shape[0], bool)
    for i, d in enumerate(flat.tolist()):
        d_buf[0], d_buf[1], d_buf[2] = d
        if cast(o._h, C.cast(o_buf, fp), C.cast(d_buf, fp), *args, C.cast(t_buf, fp)):
            ok[i], t[i] = True, t_buf[0]
    ok, t = ok.reshape(dz.shape), t.reshape(dz.shape)
    depth = np.where(ok, t * dz, F(-1.0)).astype(F)
    rgb = np.zeros(dz.shape + (3,), np.uint8)
    if color_layer:
        p = (origin + t[..., None] * dirs).astype(F)  # Ray::pointAt, per component origin + t * d
        b, v = voxel_index(p, F(o.voxel_size) * F(8.0))
        keys = sorted(color_layer)
        colors = np.stack([color_layer[k]["color"] for k in keys])  # (n, 8, 8, 8, 3)
        packed = _pack(np.array(keys, np.int64))
        q = _pack(b[ok])
        j = np.minimum(np.searchsorted(packed, q), len(keys) - 1)
        found = packed[j] == q
        vv = v[ok]
        hit_rgb = np.zeros((q.shape[0], 3), np.uint8)
        hit_rgb[found] = colors[j[found], vv[found, 0], vv[found, 1], vv[found, 2]]
        rgb[ok] = hit_rgb
    return depth, rgb
