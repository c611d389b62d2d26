"""A restatement of primitives::Scene (src/primitives/primitives.cpp, scene.cpp, primitives/internal/impl/scene_impl.h) for
the tests, in numpy: binary32 where the reference computes in float, float64 where its literals promote to double.

It follows nvb_scene.cu's reading of what the source leaves open: an unqualified `sqrt` of a float is the float square root;
Eigen sums three terms as a0 + (a1 + a2) and two as a0 + a1; std::max(a, b) is (a < b) ? b : a; maxCoeff of three is
max(a0, max(a1, a2)). numpy rounds every operation once, like the library built with -fmad=false, so the kernels' outputs
must equal these bit for bit.

A primitive is (type, center (3,) float32, params (4,) float32) with the NVB_PRIM_* types; `primitives_of(scene)` reads them
from an isaac_ros_nvblox_b200.scene.Scene.
"""
import numpy as np

F = np.float32
D = np.float64
EPS = F(1e-4)  # Primitive::kEpsilon
PLANE, CUBE, SPHERE, CYLINDER = 0, 1, 2, 3


def primitives_of(scene):
    return [(p.type, np.array(p.center[:], F), np.array(p.params[:], F)) for p in scene._prims]


def aabb_of(scene):
    lo, hi = scene.get_aabb()
    return np.array(lo, F), np.array(hi, F)


def _sum3(a0, a1, a2):
    return a0 + (a1 + a2)


def _dot(a, b):
    """(..., 3) . (..., 3) in float32, a0 + (a1 + a2)."""
    return _sum3(a[..., 0] * b[..., 0], a[..., 1] * b[..., 1], a[..., 2] * b[..., 2])


def _max(a, b):
    """std::max: (a < b) ? b : a."""
    return np.where(a < b, b, a)


def distance(prim, p):
    """Primitive::getDistanceToPoint of (n, 3) float32 points -> (n,) float32."""
    t, c, q = prim
    p = np.asarray(p, F).reshape(-1, 3)
    if t == PLANE:
        n = q[:3]
        d = -_dot(n, c)
        off = F(d / np.sqrt(_dot(n, n)))
        return _dot(np.broadcast_to(n, p.shape), p) + off
    if t == CUBE:
        s = q[:3]
        lo = (c.astype(D) - s.astype(D) / 2.0) - p.astype(D)
        hi = (p - c).astype(D) - s.astype(D) / 2.0
        v = _max(_max(lo, 0.0), hi).astype(F)
        dist = np.sqrt(_dot(v, v))
        w = _max(lo, hi).astype(F)
        inside = _max(w[:, 0], _max(w[:, 1], w[:, 2]))
        return np.where(dist < EPS, inside, dist).astype(F)
    if t == SPHERE:
        d = c - p
        return np.sqrt(_dot(d, d)) - q[0]
    r, h = q[0], q[1]
    zmin = F(D(c[2]) - D(h) / 2.0)
    zmax = F(D(c[2]) + D(h) / 2.0)
    dx, dy = p[:, 0] - c[0], p[:, 1] - c[1]
    sq = dx * dx + dy * dy
    side = np.sqrt(sq) - r
    dz = np.where(p[:, 2] > zmax, p[:, 2] - zmax, p[:, 2] - zmin)
    cap = np.sqrt(_max(sq - r * r, F(0.0)) + dz * dz)
    return np.where((p[:, 2] >= zmin) & (p[:, 2] <= zmax), side, cap).astype(F)


def ray(prim, o, u, max_dist):
    """Primitive::getRayIntersection of the rays o + t * u ((3,) origin, (n, 3) unit directions) -> (hit (n,), t (n,))."""
    t_, c, q = prim
    o = np.asarray(o, F)
    u = np.asarray(u, F).reshape(-1, 3)
    md = F(max_dist)
    with np.errstate(all="ignore"):
        if t_ == PLANE:
            n = np.broadcast_to(q[:3], u.shape)
            den = _dot(u, n)
            d = _dot(np.broadcast_to(c - o, u.shape), n) / den
            hit = ~(np.abs(den) < EPS) & ~(d < 0) & ~(d > md)
            return hit, d.astype(F)
        if t_ == CUBE:
            s = q[:3]
            inv = (1.0 / u.astype(D)).astype(F)
            b0, b1 = c - s / F(2.0), c + s / F(2.0)
            neg = inv < 0
            tlo = (np.where(neg, b1, b0) - o) * inv
            thi = (np.where(neg, b0, b1) - o) * inv
            tmin, tmax = tlo[:, 0].copy(), thi[:, 0].copy()
            miss = (tmin > thi[:, 1]) | (tlo[:, 1] > tmax)
            tmin = np.where(tlo[:, 1] > tmin, tlo[:, 1], tmin)
            tmax = np.where(thi[:, 1] < tmax, thi[:, 1], tmax)
            miss |= (tmin > thi[:, 2]) | (tlo[:, 2] > tmax)
            tmin = np.where(tlo[:, 2] > tmin, tlo[:, 2], tmin)
            tmax = np.where(thi[:, 2] < tmax, thi[:, 2], tmax)
            t = np.where(tmin < 0, tmax, tmin)
            hit = ~miss & ~(t < 0) & ~(t > md)
            return hit, t.astype(F)
        if t_ == SPHERE:
            oc = np.broadcast_to(o - c, u.shape)
            b = _dot(u, oc)
            r = D(q[0])
            disc = ((b.astype(D) * b.astype(D) - D(_dot(oc, oc)[0])) + r * r).astype(F)
            d = -b - np.sqrt(disc)
            hit = ~(disc < 0) & ~(d < 0) & ~(d > md)
            return hit, d.astype(F)
        r, h = q[0], q[1]
        E = o - c
        a = u[:, 0] * u[:, 0] + u[:, 1] * u[:, 1]
        b = F(2.0) * E[0] * u[:, 0] + F(2.0) * E[1] * u[:, 1]
        cc = (E[0] * E[0] + E[1] * E[1]) - r * r
        disc = b * b - F(4.0) * a * cc
        single = disc <= EPS
        sq = np.sqrt(disc)
        t1 = np.where(single, -b / (F(2.0) * a), (-b + sq) / (F(2.0) * a)).astype(F)
        t2 = np.where(single, F(-1.0), (-b - sq) / (F(2.0) * a)).astype(F)
        hh = D(h) / 2.0
        z1, z2 = E[2] + t1 * u[:, 2], E[2] + t2 * u[:, 2]
        v1 = (t1 >= 0) & (z1.astype(D) >= -hh) & (z1.astype(D) <= hh)
        v2 = (t2 >= 0) & (z2.astype(D) >= -hh) & (z2.astype(D) <= hh)
        caps = np.abs(u[:, 2]) > EPS
        t3 = ((-D(h) / 2.0 - D(E[2])) / u[:, 2].astype(D)).astype(F)
        t4 = ((D(h) / 2.0 - D(E[2])) / u[:, 2].astype(D)).astype(F)

        def in_cap(tc):
            qx, qy = E[0] + tc * u[:, 0], E[1] + tc * u[:, 1]
            return np.sqrt(qx * qx + qy * qy) < r
        v3 = caps & (t3 >= 0) & in_cap(t3)
        v4 = caps & (t4 >= 0) & in_cap(t4)
        t = np.full(u.shape[0], md, F)
        for v, tc in ((v1, t1), (v2, t2), (v3, t3), (v4, t4)):
            t = np.where(v & (tc < t), tc, t)
        hit = ~(np.abs(a) < EPS) & ~(disc < 0) & (v1 | v2 | v3 | v4) & ~(t >= md)
        return hit, t.astype(F)


def signed_distance(prims, p, max_dist):
    """Scene::getSignedDistanceToPoint: max_dist, lowered by every primitive closer than the running minimum."""
    p = np.asarray(p, F).reshape(-1, 3)
    d = np.full(p.shape[0], F(max_dist), F)
    for prim in prims:
        ds = distance(prim, p)
        d = np.where(ds < d, ds, d)
    return d


def scene_ray(prims, o, u, max_dist):
    """Scene::getRayIntersection -> (hit, t): the first primitive with the smallest t."""
    u = np.asarray(u, F).reshape(-1, 3)
    hit = np.zeros(u.shape[0], bool)
    best = np.full(u.shape[0], F(max_dist), F)
    for prim in prims:
        h, t = ray(prim, o, u, max_dist)
        take = h & (~hit | (t < best))
        best = np.where(take, t, best)
        hit |= take
    return hit, best


def depth_image(prims, cam, T_S_C, max_dist, invalid_depth=0.0):
    """Scene::generateDepthImageFromScene with an oracle Camera -> (height, width) float32."""
    from render_reference import pixel_rays
    T = np.asarray(T_S_C, F)
    _, u = pixel_rays(cam, T, 1)
    shape = u.shape[:2]
    u = u.reshape(-1, 3)
    o = np.ascontiguousarray(T[:3, 3])
    hit, t = scene_ray(prims, o, u, max_dist)
    p = o + t[:, None] * u  # o + t * u per component
    R = T[:3, :3]
    Rt = np.ascontiguousarray(R.T)
    t_cs = -_sum3(Rt[2, 0] * o[0], Rt[2, 1] * o[1], Rt[2, 2] * o[2])  # T_C_S = T_S_C.inverse(): z row only
    z = t_cs + _sum3(Rt[2, 0] * p[:, 0], Rt[2, 1] * p[:, 1], Rt[2, 2] * p[:, 2])
    return np.where(hit, z, F(invalid_depth)).astype(F).reshape(shape)


# ---------------------------------------------------------------------------------------------------------------------
# Layers
# ---------------------------------------------------------------------------------------------------------------------
def block_box(block_size, aabb):
    """getBlockIndicesTouchedByBoundingBox -> (lo (3,), hi (3,)) int64 block indices: floor(p / block_size) in binary32."""
    bs = F(block_size)
    lo = np.floor(np.asarray(aabb[0], F) / bs).astype(np.int64)
    hi = np.floor(np.asarray(aabb[1], F) / bs).astype(np.int64)
    return lo, hi


def blocks_touched(block_size, aabb):
    """The enumeration itself, x slowest and z fastest -> (n, 3) int64."""
    lo, hi = block_box(block_size, aabb)
    if np.any(hi < lo):
        return np.zeros((0, 3), np.int64)
    g = np.meshgrid(*[np.arange(lo[k], hi[k] + 1) for k in range(3)], indexing="ij")
    return np.stack([x.reshape(-1) for x in g], axis=1)


def voxel_centers(block_size, idx):
    """getCenterPositionFromBlockIndexAndVoxelIndex of a block -> (8, 8, 8, 3) float32."""
    bs = F(block_size)
    vs, half = bs * F(1.0 / 8), bs * F(0.5 / 8)
    v = np.arange(8, dtype=F)
    c = [(bs * F(idx[k]) + vs * v) + half for k in range(3)]
    X, Y, Z = np.meshgrid(c[0], c[1], c[2], indexing="ij")
    return np.stack([X, Y, Z], axis=-1)


def occupied_threshold(voxel_size):
    """sqrt(3.0) * voxel_size rounded to float, then halved (exactly, in double)."""
    return F(F(np.sqrt(3.0) * D(F(voxel_size))) / F(2.0))


def log_odds(p):
    """logOddsFromProbability with the clamp to [1e-3, 1 - 1e-3] in binary32, through glibc's logf like the library."""
    import ctypes as C
    logf = C.CDLL("libm.so.6").logf
    logf.restype, logf.argtypes = C.c_float, [C.c_float]
    p = min(max(F(p), F(1e-3)), F(1.0) - F(1e-3))
    return F(logf(float(F(p / (F(1.0) - p)))))


def generate_block(prims, aabb, block_size, idx, max_dist, kind, old=None):
    """generateLayerFromScene's values for one block: kind 'tsdf' -> (8, 8, 8, 2) [distance, weight], 'occupancy' ->
    (8, 8, 8) log odds, 'freespace' -> (8, 8, 8) bool is_high_confidence_freespace. `old` (same shape) holds the values of
    voxels outside the AABB (zero / False by default)."""
    p = voxel_centers(block_size, idx)
    lo, hi = np.asarray(aabb[0], F), np.asarray(aabb[1], F)
    inside = np.all((lo <= p) & (p <= hi), axis=-1)
    sdf = signed_distance(prims, p.reshape(-1, 3), max_dist).reshape(8, 8, 8)
    voxel_size = F(block_size) * F(1.0 / 8)
    if kind == "tsdf":
        new = np.stack([_max(sdf, -F(max_dist)), np.ones_like(sdf)], axis=-1).astype(F)
        old = np.zeros((8, 8, 8, 2), F) if old is None else old
        return np.where(inside[..., None], new, old)
    obj = sdf <= occupied_threshold(voxel_size)
    if kind == "occupancy":
        new = np.where(obj, log_odds(1.0), log_odds(0.0)).astype(F)
        old = np.zeros((8, 8, 8), F) if old is None else old
        return np.where(inside, new, old)
    old = np.zeros((8, 8, 8), bool) if old is None else old
    return np.where(inside, ~obj, old)
