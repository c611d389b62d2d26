"""Shared helpers for the parity tests (CUDA path vs the CPU oracle)."""
import numpy as np

from isaac_ros_nvblox_b200 import synthetic as syn


def cameras(width=640, height=480, f=300.0, radial=None, tangential=None):
    """(synthetic, product, oracle) camera objects with the reference's test intrinsics
    (nvblox/tests/test_esdf_integrator.cpp:121), scaled to the image size; optional lens distortion
    for the product and oracle cameras (the synthetic renderer stays pinhole: it only makes inputs)."""
    import isaac_ros_nvblox_b200 as nvb
    from oracle import oracle as orc
    s = f * width / 640.0
    cs = syn.PinholeCamera(s, s, width / 2.0, height / 2.0, width, height)
    ocam = orc.Camera(cs.fu, cs.fv, cs.cu, cs.cv, width, height)
    if radial is not None or tangential is not None:
        ocam = ocam.with_distortion(k=radial or (0,) * 6, p=tangential or (0, 0))
    return cs, nvb.Camera(cs.fu, cs.fv, cs.cu, cs.cv, width, height, radial, tangential), ocam


def sort_rows(a):
    a = np.asarray(a).reshape(-1, 3)
    return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]


def assert_tsdf_equal(gpu_layer, cpu_layer, atol=1e-4, exact=True):
    assert set(gpu_layer) == set(cpu_layer), "allocated TSDF block sets differ"
    worst = 0.0
    for k, c in cpu_layer.items():
        g = gpu_layer[k]
        if exact:
            # same operation order, no FMA on either side -> bit-identical
            assert np.array_equal(g["distance"].view(np.uint32), c["distance"].view(np.uint32)), ("tsdf distance bits", k)
            assert np.array_equal(g["weight"].view(np.uint32), c["weight"].view(np.uint32)), ("tsdf weight bits", k)
        d = float(np.max(np.abs(g["distance"] - c["distance"]))) if g.size else 0.0
        w = float(np.max(np.abs(g["weight"] - c["weight"]))) if g.size else 0.0
        worst = max(worst, d, w)
    assert worst <= atol, "TSDF differs by %g (tolerance %g, BASELINE.json north_star)" % (worst, atol)
    return worst


ESDF_FIELDS = ("squared_distance_vox", "parent_direction", "is_inside", "observed", "is_site")


def assert_esdf_equal(gpu_layer, cpu_layer):
    assert set(gpu_layer) == set(cpu_layer), "allocated ESDF block sets differ"
    for k, c in cpu_layer.items():
        g = gpu_layer[k]
        for f in ESDF_FIELDS:
            if not np.array_equal(g[f], c[f]):
                bad = np.argwhere(g[f] != c[f])
                raise AssertionError("ESDF field %s differs in block %s at %d voxels (first %s: gpu %s cpu %s)" %
                                     (f, k, len(bad), tuple(bad[0]), g[f][tuple(bad[0])], c[f][tuple(bad[0])]))


def layer_checksum(layer, fields):
    """Order-independent checksum of a {index: voxels} layer (sum of per-block CRCs)."""
    import zlib
    total = 0
    for k in sorted(layer):
        h = zlib.crc32(np.asarray(k, dtype=np.int32).tobytes())
        for f in fields:
            h = zlib.crc32(np.ascontiguousarray(layer[k][f]).tobytes(), h)
        total = (total + h) & 0xFFFFFFFFFFFF
    return total


# ---------------------------------------------------------------------------
# The reference's slicing known-answer cases (tests/test_esdf_integrator_slicing.cu), shared by the oracle KATs
# (test_oracle_kat.py) and the GPU parity tests (test_gpu_esdf_slice.py).
# ---------------------------------------------------------------------------
SLICING_VOXEL = np.float32(0.05)
_FREE, _OCC = 1.0, -0.025  # kFreeDistance, kOccupiedDistance (:53-54)
TSDF_DT = np.dtype([("distance", "<f4"), ("weight", "<f4")])


def _tsdf_block(distance):
    b = np.zeros((8, 8, 8), TSDF_DT)
    b["distance"], b["weight"] = distance, 1.0
    return b


def unit_plane(normal, point):
    """Plane(normal, point) (geometry/internal/impl/plane_impl.h:25-32) -> (nx, ny, nz, d), float32."""
    n = np.asarray(normal, np.float32)
    n = (n / np.float32(np.sqrt(np.float32(np.dot(n, n))))).astype(np.float32)
    d = -np.float32(np.dot(np.asarray(point, np.float32), n))
    return np.array([n[0], n[1], n[2], d], np.float32)


def slicing_case(name, planar):
    """-> (blocks {idx: tsdf block}, slice kwargs, expected) for SingleBlock (:109-208), AcrossBlock (:210-287) and
    45DegreeSlice (:353-483). expected = {'num_esdf_blocks': n, 'sites': {block idx: set of (x, y) site columns or 'all'}}.
    The output slice is z = 0 (voxel layer 0 of block layer 0)."""
    vs = float(SLICING_VOXEL)
    if name == "single_block":
        blocks = {(0, 0, 0): _tsdf_block(_OCC), (1, 0, 0): _tsdf_block(_FREE), (2, 0, 0): _tsdf_block(_FREE),
                  (3, 0, 0): _tsdf_block(_FREE)}
        blocks[(2, 0, 0)]["distance"][3, 3, 3] = _OCC
        blocks[(3, 0, 0)]["distance"][5, 5, 5] = _OCC  # just above the band
        zmin, zmax = 0.0, np.float32(3.5 * SLICING_VOXEL)
        plane = unit_plane((0, 0, 1), (0, 0, zmin))
        exp = {"num_esdf_blocks": 4, "sites": {(0, 0, 0): "all", (1, 0, 0): set(), (2, 0, 0): {(3, 3)}, (3, 0, 0): set()}}
    elif name == "across_block":
        blocks = {(0, 0, 0): _tsdf_block(_FREE), (0, 0, 1): _tsdf_block(_FREE)}
        blocks[(0, 0, 1)]["distance"][0, 0, 1] = _OCC
        zmin, zmax = 0.0, np.float32(9.5 * SLICING_VOXEL)  # 2nd voxel of the top block
        plane = unit_plane((0, 0, 1), (0, 0, zmin))
        exp = {"num_esdf_blocks": 1, "sites": {(0, 0, 0): {(0, 0)}}}
    elif name == "45_degree":
        blocks = {(0, 0, 0): _tsdf_block(_FREE)}
        for v in ((1, 1, 1), (2, 2, 3), (3, 3, 6)):
            blocks[(0, 0, 0)]["distance"][v] = _OCC
        zmin, zmax = 0.0, np.float32(2.0 * SLICING_VOXEL)
        plane = unit_plane((-1, 0, 1), (0, 0, zmin))
        exp = {"num_esdf_blocks": 1, "sites": {(0, 0, 0): {(1, 1), (2, 2)} if planar else {(1, 1)}}}
    else:
        raise KeyError(name)
    if planar:
        kw = dict(plane=plane, above_plane_m=0.0, thickness_m=float(np.float32(zmax) - np.float32(zmin)), z_output_m=0.0)
    else:
        kw = dict(z_min_m=float(zmin), z_max_m=float(zmax), z_output_m=0.0)
    return blocks, kw, exp


def check_slicing_sites(esdf_layer, exp):
    assert len(esdf_layer) == exp["num_esdf_blocks"]
    for idx, sites in exp["sites"].items():
        got = esdf_layer[idx]["is_site"][:, :, 0].astype(bool)
        want = np.ones((8, 8), bool) if sites == "all" else np.zeros((8, 8), bool)
        if sites != "all":
            for x, y in sites:
                want[x, y] = True
        assert np.array_equal(got, want), (idx, np.argwhere(got != want))


def tsdf_layer_from_distance(distance_fn, aabb_min, aabb_max, voxel_size, truncation_m):
    """Scene::generateLayerFromScene (primitives/internal/impl/scene_impl.h:105-140): the blocks touched by the AABB are
    allocated; every voxel whose centre lies in the AABB gets the ground-truth distance clipped to +-truncation and
    weight 1, the others stay unset. distance_fn maps (..., 3) float32 points to signed distances.
    -> (block indices (n, 3) int32, voxels (n, 8, 8, 8) TSDF_DT)."""
    bs = np.float32(8) * np.float32(voxel_size)
    lo = [int(np.floor(np.float32(a) / bs)) for a in aabb_min]  # getBlockIndicesTouchedByBoundingBox
    hi = [int(np.floor(np.float32(a) / bs)) for a in aabb_max]
    # getCenterPositionFromBlockIndexAndVoxelIndex in binary32, like the reference (indexing_impl.h:51-81)
    vs32, half32 = bs * np.float32(1.0 / 8), bs * np.float32(0.5 / 8)
    ax = []
    for l, h in zip(lo, hi):
        b = np.repeat(np.arange(l, h + 1), 8).astype(np.float32)
        v = np.tile(np.arange(8), h - l + 1).astype(np.float32)
        ax.append((bs * b + vs32 * v) + half32)
    P = np.stack(np.meshgrid(*ax, indexing="ij"), axis=-1)  # float32
    D = np.clip(distance_fn(P), -truncation_m, truncation_m).astype(np.float32)
    inside = np.all((P >= np.asarray(aabb_min, np.float32)) & (P <= np.asarray(aabb_max, np.float32)), axis=-1)
    D = np.where(inside, D, np.float32(0.0)).astype(np.float32)
    W = inside.astype(np.float32)
    n = [h - l + 1 for l, h in zip(lo, hi)]
    vox = np.zeros((n[0], n[1], n[2], 8, 8, 8), TSDF_DT)
    vox["distance"] = D.reshape(n[0], 8, n[1], 8, n[2], 8).transpose(0, 2, 4, 1, 3, 5)
    vox["weight"] = W.reshape(n[0], 8, n[1], 8, n[2], 8).transpose(0, 2, 4, 1, 3, 5)
    gx, gy, gz = np.meshgrid(np.arange(lo[0], hi[0] + 1), np.arange(lo[1], hi[1] + 1), np.arange(lo[2], hi[2] + 1), indexing="ij")
    idx = np.stack([gx, gy, gz], axis=-1).reshape(-1, 3).astype(np.int32)
    return idx, vox.reshape(-1, 8, 8, 8)


def sphere_in_box_signed_distance(P):
    """Scene::getSignedDistanceToPoint for the sphere-in-a-box scene of the reference's tests (ground 0, ceiling 5, walls at
    +-5 with inward normals, sphere r = 2 at (0, 0, 2)): the minimum of the primitives' signed distances, negative behind
    a wall and inside the sphere."""
    P = np.asarray(P, np.float64)
    x, y, z = P[..., 0], P[..., 1], P[..., 2]
    d = np.minimum.reduce([z, 5.0 - z, x + 5.0, 5.0 - x, y + 5.0, 5.0 - y])
    return np.minimum(d, np.linalg.norm(P - (0.0, 0.0, 2.0), axis=-1) - 2.0)


def sphere_scene_tsdf_layer(voxel_size=0.05, truncation_m=0.2):
    return tsdf_layer_from_distance(sphere_in_box_signed_distance, (-5.0, -5.0, 0.0), (5.0, 5.0, 5.0), voxel_size, truncation_m)


def spheres_distance(centers, radius):
    def fn(P):
        return np.min([np.linalg.norm(P - np.asarray(c, float), axis=-1) - radius for c in centers], axis=0)
    return fn


def points_on_a_sphere(radius, center, points_per_rad=10):
    """getPointsOnASphere (tests/test_color_integrator.cpp:88-107)."""
    pts = []
    for a in range(2 * points_per_rad):
        for e in range(points_per_rad):
            az = a * np.pi / points_per_rad - np.pi
            el = e * np.pi / points_per_rad - np.pi / 2.0
            pts.append(radius * np.array([np.cos(az) * np.sin(el), np.sin(az) * np.sin(el), np.cos(el)]) + np.asarray(center, float))
    return np.asarray(pts, np.float32)


def voxel_at_position(layer, p, voxel_size):
    """getVoxelAtPosition on a {block index: (8, 8, 8) array} layer -> the voxel record or None."""
    bs = np.float32(8) * np.float32(voxel_size)
    p = np.asarray(p, np.float32)
    b = np.floor(p / bs).astype(int)
    v = np.minimum(((p - bs * b.astype(np.float32)) * np.float32(1.0 / (float(bs) / 8))).astype(int), 7)
    blk = layer.get(tuple(int(c) for c in b))
    return None if blk is None else blk[v[0], v[1], v[2]]


def rotation_y(angle):
    c, s = np.cos(angle), np.sin(angle)
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], np.float32)
    return T


def check_sphere_scene_slice(esdf_layer, planar, voxel_size=0.05):
    """TestScene (:536-555): the inside voxels of the slice lie within the sphere's outline."""
    n_inside = 0
    for (bx, by, bz), blk in esdf_layer.items():
        ins = np.argwhere(blk["is_inside"].astype(bool))
        for vx, vy, vz in ins:
            x = (8 * bx + vx + 0.5) * voxel_size
            y = (8 * by + vy + 0.5) * voxel_size
            assert np.hypot(x, y) < 2.0
            assert x < (2.0 if planar else 2.0 * np.sqrt(2.0))
            n_inside += 1
    return n_inside


def assert_color_equal(gpu_layer, cpu_layer):
    """ColorLayer parity: same block set, identical colour bytes, bit-identical weights."""
    assert set(gpu_layer) == set(cpu_layer), (len(gpu_layer), len(cpu_layer), sorted(set(gpu_layer) ^ set(cpu_layer))[:5])
    for k, g in gpu_layer.items():
        c = cpu_layer[k]
        if not np.array_equal(g["color"], c["color"]):
            bad = np.argwhere(np.any(g["color"] != c["color"], axis=-1))
            raise AssertionError(("color", k, len(bad), bad[:3], g["color"][tuple(bad[0])], c["color"][tuple(bad[0])]))
        if not np.array_equal(g["weight"].view(np.uint32), c["weight"].view(np.uint32)):
            bad = np.argwhere(g["weight"] != c["weight"])
            raise AssertionError(("weight", k, len(bad), bad[:3], g["weight"][tuple(bad[0])], c["weight"][tuple(bad[0])]))


def _remove_distortion(x_in, y_in, radial, tangential):
    """removeDistortion (nvb_internal.cuh): Newton-Raphson in double, at most 6 iterations."""
    k1, k2, k3, k4, k5, k6 = (float(np.float32(k)) for k in radial)
    p1, p2 = (float(np.float32(p)) for p in tangential)
    x, y = float(x_in), float(y_in)
    for _ in range(6):
        r2 = x * x + y * y
        q, q2, q3 = r2, r2 * r2, r2 * r2 * r2
        R = (1.0 + k1 * r2 + k2 * q2 + k3 * q3) / (1.0 + k4 * r2 + k5 * q2 + k6 * q3)
        ex = x * R + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x) - x_in
        ey = y * R + 2.0 * p2 * x * y + p1 * (r2 + 2.0 * y * y) - y_in
        ja, jc = k1 + 2. * k2 * q + 3. * k3 * q2, k4 + 2. * k5 * q + 3. * k6 * q2
        jb, jd = k4 * q + k5 * q2 + k6 * q3 + 1., k1 * q + k2 * q2 + k3 * q3 + 1.
        dR = (ja * jb - jc * jd) / (jb * jb)
        a = R + x * 2.0 * x * dR + 2 * p1 * y + 6 * p2 * x
        b = x * 2.0 * y * dR + 2 * p1 * x + 2 * p2 * y
        c = y * 2.0 * x * dR + 2 * p2 * y + 2 * p1 * x
        d = R + y * 2.0 * y * dR + 2 * p2 * x + 6 * p1 * y
        det = a * d - b * c
        dx, dy = (d * ex - b * ey) / det, (-c * ex + a * ey) / det
        if np.isfinite(dx) and np.isfinite(dy):
            x, y = x - dx, y - dy
        if dx * dx + dy * dy < 1e-20:
            break
    return np.float32(x), np.float32(y)


def view_grid(fu, fv, cu, cv, width, height, T_L_C, block_size, max_dist, radial=None, tangential=None, workspace=None):
    """computeViewGrid (nvb_api.cu) in binary32: Camera::getViewAABB (the four corner rays of the image plane at depth 0
    and max_dist, transformed into the layer frame, min / max), the workspace clip (None, ("height", zmin, zmax) or
    ("box", lo3, hi3)) and the floor(p / block_size) block-index AABB.
    -> (min block index (3,) int64, size (3,) int64, cells) or None when the clipped AABB is empty."""
    f32 = np.float32
    T = np.asarray(T_L_C, f32)
    R, t = T[:3, :3], T[:3, 3]
    corners = []
    for u, v in ((0.0, 0.0), (width, 0.0), (width, height), (0.0, height)):
        nx, ny = (f32(u) - f32(cu)) / f32(fu), (f32(v) - f32(cv)) / f32(fv)
        if radial is not None or tangential is not None:
            nx, ny = _remove_distortion(nx, ny, radial or (0,) * 6, tangential or (0, 0))
        for d in (f32(0.0), f32(max_dist)):
            p = np.array([d * nx, d * ny, d * f32(1.0)], f32)
            # translation + linear * p, the row sums in Eigen's a0 + (a1 + a2) order
            corners.append([t[i] + (R[i, 0] * p[0] + (R[i, 1] * p[1] + R[i, 2] * p[2])) for i in range(3)])
    P = np.array(corners, f32)
    lo, hi = P.min(axis=0), P.max(axis=0)
    if workspace is not None:
        if workspace[0] == "height":
            lo[2], hi[2] = max(lo[2], f32(workspace[1])), min(hi[2], f32(workspace[2]))
        else:
            lo = np.maximum(np.asarray(workspace[1], f32), lo)
            hi = np.minimum(np.asarray(workspace[2], f32), hi)
    if np.any(lo > hi):
        return None
    bs = f32(block_size)
    mn = np.floor(lo / bs).astype(np.int64)
    mx = np.floor(hi / bs).astype(np.int64)
    size = mx - mn + 1
    return mn, size, int(np.prod(size))


def validate_esdf(layer, max_sq):
    """validateEsdf (tests/test_esdf_integrator.cpp:340-460) on a {block index: ESDF block} layer: sites have distance 0 and
    no parent; a parent direction's squared length is the distance and it points at a site; voxels without a parent sit at
    the maximum distance. -> (observed voxels, sites)."""
    keys = np.array(list(layer))
    lo, hi = keys.min(0), keys.max(0)
    shape = tuple((hi - lo + 1) * 8)
    fields = ("squared_distance_vox", "parent_direction", "is_site", "observed")
    d = {f: np.zeros(shape + ((3,) if f == "parent_direction" else ()), layer[tuple(keys[0])][f].dtype) for f in fields}
    have = np.zeros(shape, bool)
    for k, blk in layer.items():
        o = (np.asarray(k) - lo) * 8
        sl = (slice(o[0], o[0] + 8), slice(o[1], o[1] + 8), slice(o[2], o[2] + 8))
        have[sl] = True
        for f in fields:
            d[f][sl] = blk[f]
    obs, site = d["observed"].astype(bool), d["is_site"].astype(bool)
    sq, p = d["squared_distance_vox"], d["parent_direction"].astype(np.int64)
    has_parent = p.any(axis=-1)
    assert np.all(sq[site & obs] == 0.0) and not has_parent[site & obs].any()
    w = obs & ~site & has_parent
    assert np.all(sq[w] == (p[w] ** 2).sum(-1).astype(np.float32))
    pos = np.argwhere(w) + p[w]
    assert (pos >= 0).all() and (pos < np.array(have.shape)).all()
    assert site[pos[:, 0], pos[:, 1], pos[:, 2]].all(), "parent must be a site"
    n = obs & ~site & ~has_parent
    assert np.all(sq[n] >= max_sq - 1e-3)
    return int(obs.sum()), int(site.sum())


def textured_image(rows, cols, seed=0):
    """A smooth-plus-noise RGB test image."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:rows, 0:cols]
    img = np.stack([(x * 255 // max(cols - 1, 1)), (y * 255 // max(rows - 1, 1)), ((x // 16 + y // 16) % 2) * 200 + 20], axis=-1)
    img = img + rng.integers(-20, 21, size=img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)
