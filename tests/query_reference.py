"""The reference's point queries restated in float32 numpy, one point at a time, on {block index: (8, 8, 8) voxel array}
layers (the form Layer.as_dict() and the oracle return).

- getVoxelAtPosition / queryVoxelsKernel (gpu_hash/internal/cuda/gpu_indexing.cuh:56-64, map/internal/cuda/impl/
  layer_impl.cuh:29-47): helpers.voxel_at_position.
- interpolateOnCPU (src/interpolation/interpolation_3d.cpp, interpolation/internal/impl/interpolation_3d_impl.h): the 8
  voxels around p - voxel_size / 2 (up to 8 blocks), the member of each layer and its validity rule, and q . (T . m) with
  the sums running left to right over the table's non-zero entries -- the order the kernel follows.
- nvblox_torch's queries (nvblox_torch/cpp/src/sdf_query.cu:63-354, sdf_query.cuh:30-31): the ESDF sphere query with its
  multi-mapper early exit, the TSDF minimum and the occupancy maximum; outputs a query never writes keep their contents.
- The library's deviations: a non-finite point, or one whose block index lies outside +-2^20, is a miss.
"""
import math

import numpy as np

from helpers import voxel_at_position

F = np.float32
KEY_LIMIT = 1 << 20
MAX_DISTANCE = F(100.0)          # kMaxDistance = kESDFUnknownDistance
TSDF_MIN_WEIGHT = F(1e-4)        # interpolation_3d.cpp:31
GRADIENT_EPSILON = F(1e-6)       # sdf_query.cu:106

# interpolation_3d_impl.h:150-161
TABLE = np.array([[1, 0, 0, 0, 0, 0, 0, 0],
                  [-1, 0, 0, 0, 1, 0, 0, 0],
                  [-1, 0, 1, 0, 0, 0, 0, 0],
                  [-1, 1, 0, 0, 0, 0, 0, 0],
                  [1, 0, -1, 0, -1, 0, 1, 0],
                  [1, -1, -1, 1, 0, 0, 0, 0],
                  [1, -1, 0, 0, -1, 1, 0, 0],
                  [-1, 1, 1, -1, 1, -1, -1, 1]], dtype=np.int32)


def log_odds_from_probability(p):
    """logOddsFromProbability (core/log_odds.h:23-30) with a correctly rounded log."""
    p = min(max(F(p), F(1e-3)), F(1.0) - F(1e-3))
    return F(math.log(float(F(p / (F(1.0) - p)))))


def sizes(voxel_size):
    vs = F(voxel_size)
    bs = F(8) * vs
    return vs, bs, F(1.0 / (float(bs) / 8))


def block_and_voxel(p, voxel_size):
    """getBlockAndVoxelIndexFromPositionInLayer -> (block, voxel) int arrays, or None for a point the library rejects."""
    p = np.asarray(p, F)
    if not np.all(np.isfinite(p)):
        return None
    _, bs, inv = sizes(voxel_size)
    b = np.floor(p / bs)
    if np.any(b < -KEY_LIMIT) or np.any(b >= KEY_LIMIT):
        return None
    b = b.astype(np.int64)
    v = np.minimum(((p - bs * b.astype(F)) * inv).astype(np.int64), 7)
    return b, v


def lookup(layer, p, voxel_size):
    """The voxel record at p, or None (missing block or rejected point)."""
    if block_and_voxel(p, voxel_size) is None:
        return None
    return voxel_at_position(layer, p, voxel_size)


def _member(kind, vox):
    """(value, valid) of one voxel (interpolation_3d.cpp:21-69)."""
    if kind == "tsdf":
        return F(vox["distance"]), bool(F(vox["weight"]) > TSDF_MIN_WEIGHT)
    if kind == "esdf":
        return np.sqrt(F(vox["squared_distance_vox"])), bool(vox["observed"])
    lo = F(vox["log_odds"] if vox.dtype.names else vox)
    e = np.exp(lo)
    return F(e / (F(1.0) + e)), True


def surrounding(layer, p, voxel_size):
    """getSurroundingVoxels3D: (the 8 voxel records in x, y, z nested order or None, offset in voxels)."""
    vs, bs, _ = sizes(voxel_size)
    p = np.asarray(p, F)
    half = vs * F(0.5)
    bv = block_and_voxel(p - half, voxel_size)
    if bv is None:
        return None, None
    b, v = bv
    corner = (bs * b.astype(F) + vs * v.astype(F)) + half
    offset = (p - corner) / vs
    out = []
    for i in range(8):
        d = np.array([i >> 2, (i >> 1) & 1, i & 1])
        vi, bi = v + d, b.copy()
        c = vi == 8
        bi[c] += 1
        vi[c] = 0
        blk = layer.get(tuple(int(x) for x in bi))
        if blk is None:
            return None, offset
        out.append(blk[vi[0], vi[1], vi[2]])
    return out, offset


def interpolate(layer, p, voxel_size, kind):
    """interpolateOnCPU(p, layer) for kind 'tsdf', 'esdf' or 'occupancy' -> (success, value); a failure gives value 0."""
    voxels, o = surrounding(layer, p, voxel_size)
    if voxels is None:
        return False, F(0.0)
    m = []
    for vox in voxels:
        val, ok = _member(kind, vox)
        if not ok:
            return False, F(0.0)
        m.append(val)
    t = []
    for row in TABLE:
        acc = None
        for c in range(8):
            if row[c] == 0:
                continue
            term = m[c] if row[c] > 0 else -m[c]
            acc = term if acc is None else F(acc + term)
        t.append(acc)
    ox, oy, oz = F(o[0]), F(o[1]), F(o[2])
    q = [F(1.0), ox, oy, oz, F(ox * oy), F(oy * oz), F(oz * ox), F(F(ox * oy) * oz)]
    r = F(q[0] * t[0])
    for k in range(1, 8):
        r = F(r + F(q[k] * t[k]))
    return True, r


def query_esdf(layers, spheres, with_gradient, out):
    """queryESDFKernel (one layer) / queryESDFMultiMapperKernel (several): layers = [(esdf dict, voxel_size)], spheres
    (n, 4); out (n, 4) or (n, 1), pre-filled, updated in place and returned."""
    multi = len(layers) > 1
    for i, s in enumerate(np.asarray(spheres, F)):
        p, radius = s[:3], F(s[3])
        min_distance = MAX_DISTANCE
        for layer, voxel_size in layers:
            vs = F(voxel_size)
            vox = lookup(layer, p, voxel_size)
            if vox is None:
                continue
            di = 3 if with_gradient else 0
            if not vox["observed"]:
                out[i, di] = MAX_DISTANCE
                continue
            distance = F(vs * np.sqrt(F(vox["squared_distance_vox"])))
            if vox["is_inside"]:
                distance = -distance
            sphere_distance = F(distance - radius)
            if multi:
                if sphere_distance > min_distance:
                    out[i, di] = min_distance
                    continue
                min_distance = sphere_distance
            out[i, di] = sphere_distance
            if with_gradient:
                if distance > GRADIENT_EPSILON:
                    f = F(-vs / distance)
                    out[i, :3] = [F(f * F(c)) for c in vox["parent_direction"]]
                else:
                    out[i, :3] = 0.0
    return out


def query_tsdf(layers, points, out):
    """queryTSDFKernel / queryTSDFMultiMapperKernel: layers = [(tsdf dict, voxel_size)], out (n, 2) pre-filled."""
    for i, p in enumerate(np.asarray(points, F)):
        if len(layers) == 1:
            vox = lookup(layers[0][0], p, layers[0][1])
            if vox is not None:
                out[i] = [vox["distance"], vox["weight"]]
            continue
        min_distance, weight_at_min = MAX_DISTANCE, F(0.0)
        for layer, voxel_size in layers:
            vox = lookup(layer, p, voxel_size)
            if vox is not None and F(vox["distance"]) < min_distance:
                min_distance, weight_at_min = F(vox["distance"]), F(vox["weight"])
        out[i] = [min_distance, weight_at_min]
    return out


def query_occupancy(layers, points):
    """queryOccupancyMultiMapperKernel: the largest log-odds from logOddsFromProbability(0) -> (n, 1)."""
    pts = np.asarray(points, F)
    out = np.empty((len(pts), 1), F)
    for i, p in enumerate(pts):
        best = log_odds_from_probability(0.0)
        for layer, voxel_size in layers:
            vox = lookup(layer, p, voxel_size)
            if vox is not None:
                lo = F(vox["log_odds"] if vox.dtype.names else vox)
                if lo > best:
                    best = lo
        out[i, 0] = best
    return out


def query_voxels(layer, points, voxel_size, dtype):
    """getVoxels: (voxels, found) -- missed voxels stay zero."""
    pts = np.asarray(points, F)
    out = np.zeros(len(pts), dtype)
    found = np.zeros(len(pts), bool)
    for i, p in enumerate(pts):
        vox = lookup(layer, p, voxel_size)
        if vox is not None:
            out[i] = vox
            found[i] = True
    return out, found
