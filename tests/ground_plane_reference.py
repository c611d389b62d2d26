"""Restatement of the ground-plane estimator (experimental/ground_plane/) in numpy binary32, one rounding per operation in
the library's evaluation order, so that the GPU results can be compared with it bit for bit:

* zero_crossings(): TsdfZeroCrossingsExtractor::computeZeroCrossingsFromAboveOnGPU (tsdf_zero_crossings_extractor.cu:24-146)
  in the canonical order (block index (x, y, z) lexicographically, then voxel (x, y, z)), and the ground-candidate filter
  getPointsWithinMinMaxZCPU (ground_plane_estimator.cpp:109-125);
* Xorwow: curand's XORWOW generator, curand_init(seed, subsequence, 0) with the subsequence skip-ahead (2^67 draws per
  subsequence) done with a GF(2) jump matrix;
* ransac_fit(): RansacPlaneFitter::fit (ransac_plane_fitter.cu:29-144), MSAC, Plane::planeFromPoints (plane_impl.h:34-52);
* estimate(): GroundPlaneEstimator::computeGroundPlane (ground_plane_estimator.cpp:27-62).
"""
import numpy as np

F = np.float32
FLT_MAX = np.finfo(np.float32).max
M32 = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------------------------ XORWOW
def _step(v):
    """One xorshift step of the five state words (curand(), without the Weyl counter d)."""
    t = (v[0] ^ (v[0] >> 2)) & M32
    return [v[1], v[2], v[3], v[4], ((v[4] ^ ((v[4] << 4) & M32)) ^ (t ^ ((t << 1) & M32))) & M32]


def _bits(v):
    return np.array([(v[w] >> k) & 1 for w in range(5) for k in range(32)], dtype=np.uint8)


def _words(b):
    b = np.asarray(b, dtype=np.uint64).reshape(5, 32)
    return [int((b[w] << np.arange(32, dtype=np.uint64)).sum()) for w in range(5)]


def _gf2_mul(a, b):
    return ((a.astype(np.int64) @ b.astype(np.int64)) & 1).astype(np.uint8)


_JUMP = None


def _jump_matrix():
    """M^(2^67): the state transition of one subsequence, M being the 160 x 160 matrix of one step."""
    global _JUMP
    if _JUMP is None:
        cols = []
        for j in range(160):
            e = [0] * 5
            e[j // 32] = 1 << (j % 32)
            cols.append(_bits(_step(e)))
        m = np.stack(cols, axis=1)
        for _ in range(67):
            m = _gf2_mul(m, m)
        _JUMP = m
    return _JUMP


class Xorwow:
    """curandStateXORWOW after curand_init(seed, subsequence, 0) (curand_kernel.h: _curand_init_scratch)."""

    def __init__(self, seed, subsequence=0, _v=None):
        s0 = (seed & M32) ^ 0xaad26b49
        s1 = ((seed >> 32) & M32) ^ 0xf7dcefdd
        t0 = (1099087573 * s0) & M32
        t1 = (2591861531 * s1) & M32
        self.d = (6615241 + t1 + t0) & M32
        if _v is not None:
            self.v = list(_v)
            return
        self.v = [(123456789 + t0) & M32, 362436069 ^ t0, (521288629 + t1) & M32, 88675123 ^ t1, (5783321 + t0) & M32]
        if subsequence:
            b = _bits(self.v)
            j = _jump_matrix()
            p = subsequence
            while p:  # J^subsequence by binary powers
                if p & 1:
                    b = (j.astype(np.int64) @ b.astype(np.int64) & 1).astype(np.uint8)
                p >>= 1
                if p:
                    j = _gf2_mul(j, j)
            self.v = _words(b)

    def next(self):
        self.v = _step(self.v)
        self.d = (self.d + 362437) & M32
        return (self.v[4] + self.d) & M32


def xorwow_states(seed, n):
    """The n states curand_init(seed, i, 0), i < n, by repeated jumps (cheaper than n independent skip-aheads)."""
    j = _jump_matrix().astype(np.int64)
    first = Xorwow(seed)
    b = _bits(first.v).astype(np.int64)
    out = []
    for _ in range(n):
        out.append(Xorwow(seed, _v=_words(b)))
        b = (j @ b) & 1
    return out


# ------------------------------------------------------------------------------------------------------------------- plane
def _sum3(a0, a1, a2):
    return F(a0 + F(a1 + a2))


def _normalized(v):
    z = _sum3(F(v[0] * v[0]), F(v[1] * v[1]), F(v[2] * v[2]))
    if z > F(0):
        s = F(np.sqrt(z))
        return [F(v[0] / s), F(v[1] / s), F(v[2] / s)]
    return list(v)


def plane_from_points(a, b, c):
    """Plane::planeFromPoints: (nx, ny, nz, d) as float32, or None (two points equal, or collinear: cross product isZero(1e-6)).
    Plane(normal, point) delegates to Plane(normal.normalized(), -point.dot(normal.normalized())), which normalises again."""
    a, b, c = (np.asarray(p, F) for p in (a, b, c))
    if np.all(a == b) or np.all(a == c) or np.all(b == c):
        return None
    ab, ac = b - a, c - a
    v = [F(ab[1] * ac[2]) - F(ab[2] * ac[1]), F(ab[2] * ac[0]) - F(ab[0] * ac[2]), F(ab[0] * ac[1]) - F(ab[1] * ac[0])]
    v = [F(x) for x in v]
    if all(abs(x) <= F(1e-6) for x in v):
        return None
    n1 = _normalized(v)
    n2 = _normalized(n1)
    d = F(-_sum3(F(a[0] * n2[0]), F(a[1] * n2[1]), F(a[2] * n2[2])))
    n3 = _normalized(n2)
    return np.array([n3[0], n3[1], n3[2], d], F)


def msac_cost(plane, pts, threshold):
    """sum over the points, in order and in float, of d^2 if |d| < t else t^2 (d = n . p + d0, Plane::signedDistance)."""
    t = F(threshold)
    t2 = F(t * t)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    dist = np.abs((plane[0] * x + (plane[1] * y + plane[2] * z)) + plane[3]).astype(F)
    terms = np.where(dist < t, dist * dist, t2).astype(F)
    if len(terms) == 0:
        return F(0)
    return F(np.add.accumulate(terms, dtype=F)[-1])  # strictly sequential, unlike np.sum's pairwise reduction


def ransac_fit(points, num_ransac_iterations=1000, ransac_distance_threshold_m=0.2, return_costs=False):
    """RansacPlaneFitter::fit: (nx, ny, nz, d) float32 array or None."""
    pts = np.ascontiguousarray(points, F).reshape(-1, 3)
    n = len(pts)
    if n < 3:
        return (None, None) if return_costs else None
    costs = np.full(num_ransac_iterations, FLT_MAX, F)
    planes = np.zeros((num_ransac_iterations, 4), F)
    for i, st in enumerate(xorwow_states(1234, num_ransac_iterations)):
        i1, i2, i3 = st.next() % n, st.next() % n, st.next() % n
        pl = plane_from_points(pts[i1], pts[i2], pts[i3])
        if pl is None:
            continue
        costs[i] = msac_cost(pl, pts, ransac_distance_threshold_m)
        planes[i] = pl
    best = int(np.argmin(costs))  # first minimum, like std::min_element
    res = None if costs[best] == FLT_MAX else planes[best]
    return (res, costs) if return_costs else res


# ------------------------------------------------------------------------------------------------------ zero crossings
def zero_crossings(layer, voxel_size, min_tsdf_weight=0.1):
    """The crossings of a {block index: (8, 8, 8) TSDF voxels} layer as (n, 3) float32 in canonical order."""
    vs = F(voxel_size)
    bs = F(8) * vs
    vsz, hvs = bs * F(0.125), bs * F(0.0625)
    w_min = F(min_tsdf_weight)
    out = []
    for key in sorted(layer):
        blk = layer[key]
        d, w = blk["distance"].astype(F), blk["weight"].astype(F)
        up_d = np.zeros_like(d)
        up_w = np.zeros_like(w)
        valid = np.ones(d.shape, bool)
        up_d[:, :, :7], up_w[:, :, :7] = d[:, :, 1:], w[:, :, 1:]
        above = layer.get((key[0], key[1], key[2] + 1))
        if above is None:
            valid[:, :, 7] = False
        else:
            up_d[:, :, 7], up_w[:, :, 7] = above["distance"][:, :, 0], above["weight"][:, :, 0]
        hit = valid & (up_w >= w_min) & (w >= w_min) & (up_d > F(0)) & (d <= F(0))
        vx, vy, vz = np.nonzero(hit)  # C order: voxel (x, y, z) lexicographically
        if len(vx) == 0:
            continue
        px = (bs * F(key[0]) + vsz * vx.astype(F)) + hvs
        py = (bs * F(key[1]) + vsz * vy.astype(F)) + hvs
        pz = (bs * F(key[2]) + vsz * vz.astype(F)) + hvs
        db, da = d[vx, vy, vz], up_d[vx, vy, vz]
        with np.errstate(all="ignore"):
            dz = ((-db) * vs) / (da - db)
        out.append(np.stack([px, py, (pz + dz).astype(F)], axis=1).astype(F))
    return np.concatenate(out).astype(F) if out else np.zeros((0, 3), F)


def ground_candidates(crossings, min_z=-0.1, max_z=0.15):
    c = np.asarray(crossings, F).reshape(-1, 3)
    keep = np.all(np.isfinite(c), axis=1) & (c[:, 2] >= F(min_z)) & (c[:, 2] <= F(max_z))
    return c[keep]


def estimate(layer, voxel_size, min_z=-0.1, max_z=0.15, ransac_distance_threshold_m=0.2, num_ransac_iterations=1000,
             min_tsdf_weight=0.1, max_crossings=360000):
    """GroundPlaneEstimator::computeGroundPlane -> (plane or None, crossings or None, candidates or None)."""
    if not layer:
        return None, None, None
    cr = zero_crossings(layer, voxel_size, min_tsdf_weight)
    if len(cr) >= max_crossings:
        return None, None, None
    cand = ground_candidates(cr, min_z, max_z)
    plane = ransac_fit(cand, num_ransac_iterations, ransac_distance_threshold_m)
    if plane is None:
        return None, None, None
    return plane, cr, cand
