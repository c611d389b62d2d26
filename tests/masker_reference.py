"""Restatement of the image masker (csrc/nvb_masker.cu) in numpy, binary32 with one rounding per operation in the
library's evaluation order; the reference's algorithm (ImageMasker::splitImageOnGPU, src/semantics/image_masker.cu), not its
code:
  * the min-depth scatter (getMinimumDepthKernel<5>): unproject, T_CM_CD, Camera::project into the mask camera, and the
    minimum of z over the 5 x 5 patch at (int)((u + k) - 2.0f), (int)((v + k) - 2.0f), truncated toward zero;
  * the split (splitDepthImageKernel): masked when the pixel projects, the mask is set at (int)(u, v) and
    min_depth + occlusion_threshold_m >= z; +-inf always unmasked; the overlay grey fmin(12.75 * depth, 255);
  * the colour split (splitColorImageKernel).
The library's two deviations are restated too: a projection exactly on u == width or v == height is a miss (the
reference reads past the mask's row there), and a negative depth has grey 0 (undefined in the reference).
Cameras are dicts: width, height, fu, fv, cu, cv, and optionally radial / tangential (None: no distortion).
"""
import numpy as np

import dynamics_reference as dref

f32 = np.float32
FLT_MAX = np.finfo(np.float32).max
PATCH = 5


def _distorted(c):
    return c.get("radial") is not None or c.get("tangential") is not None


def apply_distortion(x, y, c):
    """applyDistortion (nvb_internal.cuh, sensors/internal/impl/distortion_impl.h:37-60), vectorised: the float / double
    promotions of the reference's literals spelled out."""
    k = [float(f32(v)) for v in (c.get("radial") or (0,) * 6)]
    p1, p2 = (float(f32(v)) for v in (c.get("tangential") or (0, 0)))
    x, y = x.astype(f32), y.astype(f32)
    r2 = x * x + y * y
    r4 = r2 * r2
    r6 = r2 * r4
    d = np.float64
    num = (1.0 + (f32(k[0]) * r2).astype(d) + (f32(k[1]) * r4).astype(d) + (f32(k[2]) * r6).astype(d)).astype(f32)
    den = (1.0 + (f32(k[3]) * r2).astype(d) + (f32(k[4]) * r4).astype(d) + (f32(k[5]) * r6).astype(d)).astype(f32)
    scale = num / den
    xy = x * y
    tx = (2.0 * p1 * xy.astype(d) + p2 * (r2.astype(d) + 2.0 * x.astype(d) * x.astype(d))).astype(f32)
    ty = (2.0 * p2 * xy.astype(d) + p1 * (r2.astype(d) + 2.0 * y.astype(d) * y.astype(d))).astype(f32)
    return x * scale + tx, y * scale + ty


def project_into_mask(depth, T_CM_CD, depth_cam, mask_cam):
    """-> (ok, z, u, v) per depth pixel: Camera::project of T_CM_CD * unprojectFromPixelIndices(pixel, depth)."""
    depth = np.asarray(depth, f32)
    rows, cols = depth.shape
    rr, cc = np.mgrid[0:rows, 0:cols]
    with np.errstate(all="ignore"):
        p = dref.unproject_transform(depth, T_CM_CD, depth_cam, rr, cc)
        x, y, z = p[..., 0], p[..., 1], p[..., 2]
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (z >= f32(1e-6))
        un, vn = x / z, y / z
        if _distorted(mask_cam):
            un, vn = apply_distortion(un, vn, mask_cam)
        u = un * f32(mask_cam["fu"]) + f32(mask_cam["cu"])
        v = vn * f32(mask_cam["fv"]) + f32(mask_cam["cv"])
        ok &= ~((u > f32(mask_cam["width"])) | (v > f32(mask_cam["height"])) | (u < f32(0)) | (v < f32(0)))
    return ok, z, u, v


def min_depth_image(depth, T_CM_CD, depth_cam, mask_cam):
    """The mask-sized min-depth image after the scatter (FLT_MAX where nothing was written)."""
    ok, z, u, v = project_into_mask(depth, T_CM_CD, depth_cam, mask_cam)
    mrows, mcols = mask_cam["height"], mask_cam["width"]
    md = np.full((mrows, mcols), FLT_MAX, f32)
    zs, us, vs = z[ok], u[ok], v[ok]
    for pr in range(PATCH):
        row = dref.float_to_int_rz((vs + f32(pr)) - f32(PATCH // 2))
        for pc in range(PATCH):
            col = dref.float_to_int_rz((us + f32(pc)) - f32(PATCH // 2))
            inb = (row >= 0) & (row < mrows) & (col >= 0) & (col < mcols)
            np.minimum.at(md, (row[inb], col[inb]), zs[inb])
    return md


def overlay_grey(depth):
    """fmin(12.75f * depth, 255) as uint8: 255 for NaN and +inf, 0 for a negative value."""
    with np.errstate(all="ignore"):
        x = f32(255.0 / 20.0) * np.asarray(depth, f32)
        return np.where(~(x <= f32(255)), 255, np.where(x > f32(0), np.trunc(np.where(x > 0, x, 0)), 0)).astype(np.uint8)


def split_depth(depth, mask, T_CM_CD, depth_cam, mask_cam, occlusion_threshold_m=0.25, masked_invalid=-1.0,
                unmasked_invalid=-1.0):
    """-> (background, foreground, overlay, is_masked)."""
    depth = np.asarray(depth, f32)
    mask = np.asarray(mask, np.uint8)
    assert depth.shape == (depth_cam["height"], depth_cam["width"]) and mask.shape == (mask_cam["height"], mask_cam["width"])
    md = min_depth_image(depth, T_CM_CD, depth_cam, mask_cam)
    ok, z, u, v = project_into_mask(depth, T_CM_CD, depth_cam, mask_cam)
    ok &= ~np.isinf(depth)
    ui = np.where(ok, dref.float_to_int_rz(u), 0)
    vi = np.where(ok, dref.float_to_int_rz(v), 0)
    ok &= (ui < mask.shape[1]) & (vi < mask.shape[0])
    ui, vi = np.where(ok, ui, 0), np.where(ok, vi, 0)
    with np.errstate(all="ignore"):
        occluded = md[vi, ui] + f32(occlusion_threshold_m) < z
    masked = ok & (mask[vi, ui] != 0) & ~occluded
    bg = np.where(masked, f32(unmasked_invalid), depth).astype(f32)
    fg = np.where(masked, depth, f32(masked_invalid)).astype(f32)
    g = overlay_grey(depth)
    overlay = np.stack([np.where(masked, np.uint8(255), g), g, g], -1).astype(np.uint8)
    return bg, fg, overlay, masked


def split_color(rgb, mask):
    """-> (unmasked, masked, overlay) for a mask lying on top of the image; the invalid colour is black."""
    rgb = np.asarray(rgb, np.uint8)
    m = (np.asarray(mask, np.uint8) != 0)[..., None]
    overlay = rgb.copy()
    overlay[..., 0] = np.where(m[..., 0], np.uint8(255), rgb[..., 0])
    return np.where(m, np.uint8(0), rgb), np.where(m, rgb, np.uint8(0)), overlay


# ---------------------------------------------------------------------------------------------------------------------
# Inputs shared by the known-answer tests and the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
def cam(width, height, fu, fv, cu, cv, radial=None, tangential=None):
    return dict(width=int(width), height=int(height), fu=float(fu), fv=float(fv), cu=float(cu), cv=float(cv), radial=radial,
                tangential=tangential)


def masker_test_camera(cols, rows):
    """getTestCamera (tests/test_image_masker.cpp:27-33)."""
    return cam(cols, rows, 300.0, 300.0, cols / 2.0, rows / 2.0)


def rotation_y_f32(angle):
    """Eigen::AngleAxisf(angle, UnitY).toRotationMatrix() in binary32."""
    a = f32(angle)
    c, s = f32(np.cos(a)), f32(np.sin(a))
    one_minus_c = f32(f32(1) - c)
    R = np.zeros((3, 3), f32)
    R[0, 0], R[1, 1], R[2, 2] = c, f32(one_minus_c + c), c
    R[0, 2], R[2, 0] = s, -s
    return R


def perpendicular_transform():
    """PerpendicularTransformMask's T_CM_CD: a 90 degree rotation about y, then a translation of (1, 0, 5)."""
    T = np.eye(4, dtype=f32)
    T[:3, :3] = rotation_y_f32(-0.5 * np.pi)
    T[:3, 3] = (1.0, 0.0, 5.0)
    return T


def random_mask(rows, cols, seed=0, p=0.5):
    return (np.random.default_rng(seed).random((rows, cols)) < p).astype(np.uint8)


def special_depths(rows, cols, seed, lo=0.3, hi=6.0):
    """Uniform depths with 0, -1, NaN, +inf and -inf pixels sprinkled in."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(lo, hi, (rows, cols)).astype(f32)
    k = rng.integers(0, 30, (rows, cols))
    d[k == 0], d[k == 1], d[k == 2], d[k == 3], d[k == 4] = 0.0, -1.0, np.nan, np.inf, -np.inf
    return d


def inverse(T):
    """A rigid transform's inverse in float64, stored as float32."""
    T = np.asarray(T, np.float64)
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out.astype(f32)


def colour_camera_case(seed=3):
    """The 640 x 480 depth / 1280 x 720 colour pair of camera_pose_cases (5 cm baseline, 1 degree rotation): a depth frame
    of a slanted wall with a box in front of it, and a blocky mask of the colour camera."""
    rng = np.random.default_rng(seed)
    import camera_pose_cases as cpc
    dc, mc = cpc.COLOR_DEPTH_CAM, cpc.COLOR_CAM
    r, c = np.mgrid[0:dc["height"], 0:dc["width"]]
    depth = (3.0 + 0.002 * c + 0.001 * r).astype(np.float32)
    depth[150:330, 200:420] = 1.6
    depth += rng.normal(0, 0.01, depth.shape).astype(np.float32)
    blocks = rng.random((mc["height"] // 40 + 1, mc["width"] // 40 + 1)) < 0.5
    mask = np.repeat(np.repeat(blocks, 40, 0), 40, 1)[:mc["height"], :mc["width"]].astype(np.uint8) * 255
    T_CM_CD = inverse(cpc.T_D_C)
    return depth, mask, T_CM_CD, dc, mc
