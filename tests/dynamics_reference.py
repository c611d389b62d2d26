"""Restatement of the dynamics detection and of the connected-component mask filter (csrc/nvb_dynamics.cu) in numpy,
binary32 with one rounding per operation in the library's evaluation order; the reference's algorithms, not its code:
  * DynamicsDetection::computeDynamics (dynamics/internal/cuda/impl/dynamics_detection_impl.cuh:26-87) over a freespace
    layer given as {block index: (8, 8, 8) FreespaceVoxel block} (read back from the GPU, from the oracle, or built by hand);
  * MaskPreprocessor::removeSmallConnectedComponents (src/sensors/mask_preprocessor.cpp:24-183, image.cu:323-404), with the
    components labelled by scipy.ndimage (4-connected) instead of the reference's host BFS; the output keeps the input's
    size (a trailing odd row / column is 0) where the reference's shrinks to an even size.
"""
import numpy as np
from scipy import ndimage

f32 = np.float32
MASKED = 255     # image::kMaskedValue
SURVIVOR = 254   # the reference's 255 with its visited bit 0x01 cleared
FOUR_CONNECTED = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]])


def _radial_scale_d(r2, k):
    r4 = r2 * r2
    r6 = r2 * r4
    return (1.0 + k[0] * r2 + k[1] * r4 + k[2] * r6) / (1.0 + k[3] * r2 + k[4] * r4 + k[5] * r6)


def remove_distortion(ux, uy, radial, tangential):
    """removeDistortion (nvb_internal.cuh, sensors/internal/impl/distortion_impl.h:93-176), term for term in double."""
    k = [float(f32(v)) for v in radial]
    p1, p2 = (float(f32(v)) for v in tangential)
    k1, k2, k3, k4, k5, k6 = k
    u_in_x, u_in_y = float(ux), float(uy)
    x, y = u_in_x, u_in_y
    for _ in range(6):
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        R = _radial_scale_d(r2, k)
        xy = x * y
        tan_x = 2.0 * p1 * xy + p2 * (r2 + 2.0 * x * x)
        tan_y = 2.0 * p2 * xy + p1 * (r2 + 2.0 * y * y)
        error_x, error_y = (x * R + tan_x) - u_in_x, (y * R + tan_y) - u_in_y
        q = r2
        q2 = q * q
        q3 = q2 * q
        ja = k1 + 2. * k2 * q + 3. * k3 * q2
        jc = k4 + 2. * k5 * q + 3. * k6 * q2
        jb = k4 * q + k5 * q2 + k6 * q3 + 1.
        jd = k1 * q + k2 * q2 + k3 * q3 + 1.
        dR_dr2 = (ja * jb - jc * jd) / (jb * jb)
        dR_dx, dR_dy = 2.0 * x * dR_dr2, 2.0 * y * dR_dr2
        a = R + x * dR_dx + 2 * p1 * y + 6 * p2 * x
        b = x * dR_dy + 2 * p1 * x + 2 * p2 * y
        cc = y * dR_dx + 2 * p2 * y + 2 * p1 * x
        d = R + y * dR_dy + 2 * p2 * x + 6 * p1 * y
        det = a * d - b * cc
        with np.errstate(all="ignore"):
            delta_x = (d * error_x - b * error_y) / det if det != 0.0 else float("nan")
            delta_y = (-cc * error_x + a * error_y) / det if det != 0.0 else float("nan")
        if np.isfinite(delta_x) and np.isfinite(delta_y):
            x, y = x - delta_x, y - delta_y
        if delta_x * delta_x + delta_y * delta_y < 1e-20:
            break
    return f32(x), f32(y)


def float_to_int_rz(x):
    """__float2int_rz: NaN -> 0, saturating, towards zero."""
    x = np.asarray(x, np.float64)
    x = np.where(np.isnan(x), 0.0, x)
    return np.trunc(np.clip(x, -2147483648.0, 2147483647.0)).astype(np.int64)


def unproject_transform(depth, T_L_C, cam, rows_idx, cols_idx):
    """T_L_C * unprojectFromPixelIndices((c, r), depth) for the given pixels, in binary32. cam: fu, fv, cu, cv, and
    optionally radial / tangential (None: no distortion)."""
    fu, fv, cu, cv = (f32(cam[k]) for k in ("fu", "fv", "cu", "cv"))
    u = ((cols_idx.astype(f32) + f32(0.5)) - cu) / fu
    v = ((rows_idx.astype(f32) + f32(0.5)) - cv) / fv
    if cam.get("radial") is not None or cam.get("tangential") is not None:
        radial, tangential = cam.get("radial") or (0,) * 6, cam.get("tangential") or (0, 0)
        for i in range(u.size):
            u.flat[i], v.flat[i] = remove_distortion(u.flat[i], v.flat[i], radial, tangential)
    d = depth.astype(f32)
    p = np.stack([d * u, d * v, d * f32(1.0)], -1).astype(f32)
    T = np.asarray(T_L_C, f32)
    R, t = T[:3, :3], T[:3, 3]
    out = np.empty_like(p)
    for i in range(3):
        out[..., i] = t[i] + (R[i, 0] * p[..., 0] + (R[i, 1] * p[..., 1] + R[i, 2] * p[..., 2]))
    return out


def compute_dynamics(depth, T_L_C, cam, freespace_layer, block_size):
    """-> (mask (rows, cols) uint8, overlay (rows, cols, 3) uint8, points (n, 3) float32 in row-major pixel order).
    freespace_layer: {(x, y, z): (8, 8, 8) array with an is_high_confidence_freespace field, or a bool array}."""
    depth = np.asarray(depth, f32)
    rows, cols = depth.shape
    mask = np.zeros((rows, cols), np.uint8)
    overlay = np.full((rows, cols, 3), 255, np.uint8)
    with np.errstate(invalid="ignore"):
        go = ~(depth <= f32(0.0))  # NaN goes on
    rr, cc = np.nonzero(go)
    if rr.size == 0:
        return mask, overlay, np.zeros((0, 3), f32)
    with np.errstate(all="ignore"):
        p = unproject_transform(depth[rr, cc], T_L_C, cam, rr, cc)
        bs = f32(block_size)
        blk = float_to_int_rz(np.floor(p / bs))
        inv = f32(1.0 / float(bs * f32(0.125)))
        vox = np.minimum(float_to_int_rz((p - bs * blk.astype(f32)) * inv), 7)
    found = np.zeros(rr.size, bool)
    dyn = np.zeros(rr.size, bool)
    for i in range(rr.size):
        b = freespace_layer.get((int(blk[i, 0]), int(blk[i, 1]), int(blk[i, 2])))
        if b is None:
            continue
        found[i] = True
        hc = b["is_high_confidence_freespace"] if b.dtype.names else b
        dyn[i] = bool(hc[vox[i, 0], vox[i, 1], vox[i, 2]])
    with np.errstate(invalid="ignore"):
        s = np.fmin(f32(255.0 / 10.0) * depth[rr, cc], f32(255.0)).astype(np.uint8)  # getOverlayColor
    fr, fc = rr[found], cc[found]
    mask[fr, fc] = np.where(dyn[found], MASKED, 0)
    overlay[fr, fc, 0] = np.where(dyn[found], 255, 0)
    overlay[fr, fc, 1] = s[found]
    overlay[fr, fc, 2] = s[found]
    return mask, overlay, p[dyn].astype(f32)


def remove_small_connected_components(mask, threshold):
    """The filtered mask, same size as `mask`: survivors 254, the rest 0."""
    mask = np.asarray(mask, np.uint8)
    if threshold <= 0:
        return mask.copy()
    rows, cols = mask.shape
    dr, dc = rows // 2, cols // 2
    out = np.zeros((rows, cols), np.uint8)
    if dr == 0 or dc == 0:
        return out
    down = mask[0:2 * dr:2, 0:2 * dc:2] > 0
    labels, _ = ndimage.label(down, structure=FOUR_CONNECTED)
    sizes = np.bincount(labels.ravel())
    keep = down & (sizes[labels] >= threshold // 4)  # size_threshold / (kDownScaleFactor * kDownScaleFactor)
    out[:2 * dr, :2 * dc] = np.where(np.repeat(np.repeat(keep, 2, 0), 2, 1), SURVIVOR, 0)
    return out


def component_sizes(mask):
    """Sizes of the 4-connected components of the 2x-downscaled mask (for building thresholds)."""
    rows, cols = mask.shape
    down = mask[0:2 * (rows // 2):2, 0:2 * (cols // 2):2] > 0
    labels, n = ndimage.label(down, structure=FOUR_CONNECTED)
    return np.bincount(labels.ravel())[1:]


# ---------------------------------------------------------------------------------------------------------------------
# Inputs shared by the known-answer tests and the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
GOLDEN = __import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "golden")


def load_human_fixture():
    """(K float32 3x3, depth frames (2, 480, 640) float32 in metres, mask_21 uint8) of tests/golden/dynamics_human.npz."""
    z = np.load(__import__("os").path.join(GOLDEN, "dynamics_human.npz"))
    depth = z["depth_u16"].astype(f32) * f32(1.0 / 1000.0)  # io::readFromPng: float(u16) * kDefaultUintDepthScaleFactor
    return z["intrinsics"], depth.astype(f32), z["mask_21"]


def _square(mask, r0, c0, nr, nc):  # drawSquare (tests/lib/utils.cpp:74-83)
    mask[max(r0, 0):r0 + nr, max(c0, 0):c0 + nc] = 255


def reference_masks(mask_21):
    """test_mask_preprocessor.cpp's cases: name -> (mask, threshold, expected number of pixels > 0)."""
    z = np.zeros((480, 640), np.uint8)
    full = np.full((480, 640), 255, np.uint8)
    grid = z.copy()
    grid[::4, ::4] = 255
    two = z.copy()
    _square(two, 50, 50, 20, 20)
    _square(two, 50, 100, 30, 30)
    return {
        "RealMask": (mask_21, 10000, 11480),
        "EmptyMask": (z, 10000, 0),
        "FullMask": (full, 10000, 640 * 480),
        "TwoSquares_keepBoth": (two, 400, 400 + 900),
        "TwoSquares_keepOne": (two, 400 + 4, 900),
        "TwoSquares_keepNone": (two, 900 + 4, 0),
        "GridPattern": (grid, 1, 640 * 480 // 4),
    }


def corner_blobs():
    """ConnectedComponents.BlobIn*Corner: 10 x 10 masks at threshold 3 whose pixels all survive."""
    out = {}
    for name, px in (("TopLeft", [(0, 0), (0, 1), (1, 0), (1, 1)]), ("TopRight", [(0, 9), (1, 9), (0, 8), (1, 8)]),
                     ("BottomLeft", [(9, 0), (9, 1), (8, 0)]), ("BottomRight", [(9, 9), (9, 8), (8, 9), (8, 8)])):
        m = np.zeros((10, 10), np.uint8)
        for r, c in px:
            m[r, c] = 255
        out[name] = (m, px)
    return out


def spiral_mask(rows, cols):
    """A one-pixel-wide rectangular spiral with one-pixel gaps between its arms, drawn in the downscaled image and upscaled:
    a single component that winds across the whole image."""
    dr, dc = rows // 2, cols // 2
    d = np.zeros((dr, dc), bool)
    r = c = 0
    d[0, 0] = True
    hl, vl = dc - 1, dr - 1
    moves = [((0, 1), hl), ((1, 0), vl), ((0, -1), hl)]
    k = 0
    while True:
        if k % 2 == 0:
            vl -= 2
            step = ((-1, 0), vl) if k % 4 == 0 else ((1, 0), vl)
        else:
            hl -= 2
            step = ((0, 1), hl) if k % 4 == 1 else ((0, -1), hl)
        if step[1] <= 0:
            break
        moves.append(step)
        k += 1
    for (drr, dcc), n in moves:
        for _ in range(n):
            r, c = r + drr, c + dcc
            d[r, c] = True
    out = np.zeros((rows, cols), np.uint8)
    out[:2 * dr, :2 * dc] = np.repeat(np.repeat(d, 2, 0), 2, 1) * 255
    return out
