"""Hand-set TSDF layers that drive the marching-cubes mesh (isaac_ros_nvblox_b200/csrc/nvb_mesh.cu) through the branches
inside a block's cubes, and float64 restatements of what the mesh must be for them. Nothing here uses oracle/: the case
table comes from the reference's own table (tests/golden/marching_cubes_reference.npz), the corner and edge numbering from
nvblox/mesh/internal/impl/marching_cubes_table.h:326-333, the rules from marching_cubes_impl.h and mesh_integrator.cu.

A case is a `Case`: TSDF blocks {(bx, by, bz): (8, 8, 8) TSDF_VOXEL_DTYPE}, optional colour blocks, the mesh parameters,
and what it was built to contain (`info`). The generators:
  * config_sweep_case    -- every one of the 256 corner-sign configurations in each of the 8 position classes of a cube
                            (voxel index 7 or not on x, y, z: whether the cube reaches into the next block);
  * neighbour_sweep_case -- all 128 subsets of a block's 7 upper neighbours, the surface crossing every face, edge and
                            corner the neighbours supply;
  * degenerate_case      -- corners at 0.0 / -0.0, |sa - sb| at 1e-4f and one ulp either side, equal magnitudes,
                            coincident edge vertices (zero-area triangles), weights at min_weight / one ulp below / 0 /
                            +inf, smallest |d| exactly at the meshability cutoff and one ulp above;
  * weld_size_case       -- blocks whose vertex counts sit on both sides of every bitonic sort size and of 2560;
  * weld_origin_case, weld_collision_case, weld_saturation_case -- weld keys: truncation towards zero around 0, two
                            vertices 17.191 m apart with one key (the 17191 multiplier), x * 1000 past the int32 range;
  * plane_cases          -- seeded planes through block interiors, faces, edges, corners and voxel centres, near and far
                            from the origin;
  * colour_case          -- a colour per voxel, vertices on the upper faces (index 8 clamps to 7), blocks without colour;
  * noise_case           -- enough vertices for one call to outgrow the mesh arena.

The float64 checks (check_unwelded, check_welded, expected_colors) restate the operation: classification `d < 0`, cubes
with a missing or low-weight corner skipped, the table's triangles in (c, b, a) order, the vertex at
p0 + sa / (sa - sb) (p1 - p0) or the edge midpoint when the float32 |sa - sb| < 1e-4f, the weld's 1 mm keys, and the
closest colour voxel. Values that the reference defines in float32 (the stored TSDF, the 1e-4f switch, the cutoff, the
weld key's v * 1000.0f) are taken in float32; geometry is float64."""
import os
from dataclasses import dataclass, field

import numpy as np

from isaac_ros_nvblox_b200 import COLOR_VOXEL_DTYPE, TSDF_VOXEL_DTYPE

VOXEL = 0.1
WELD_MAX = 128 * 20  # weldVerticesCubKernel<128, 20>: blocks with this many vertices or more are not welded
# every switch of the weld's sort size (a power of two from 32 to 4096) and the weld limit, as unwelded vertex counts;
# counts are multiples of 3, so each switch 2^k is bracketed by the nearest multiples of 3 at or below it and above it
WELD_SIZES = (30, 33, 126, 129, 255, 258, 510, 513, 1023, 1026, 2046, 2049, 2559, 2562)

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "marching_cubes_reference.npz")
_T = np.load(_GOLDEN)
TRI_TABLE = _T["triangle_table"].astype(np.int64)   # (256, 16) edge numbers, -1 terminated
TRI_COUNT = _T["num_triangles"].astype(np.int64)     # (256,)
EDGE_CORNERS = np.array([(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)])
CORNER_OFFSETS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)])
# emission order of a configuration's vertices: triangle (a, b, c) of the table is stored as (c, b, a)
EMIT_EDGES = np.full((256, 15), -1, np.int64)
for _c in range(256):
    for _t in range(TRI_COUNT[_c]):
        EMIT_EDGES[_c, 3 * _t:3 * _t + 3] = TRI_TABLE[_c, 3 * _t:3 * _t + 3][::-1]
NB_DIRS = [((j >> 2) & 1, (j >> 1) & 1, j & 1) for j in range(8)]  # neighborIndexFromDirection order


@dataclass
class Case:
    name: str
    layer: dict
    voxel: float = VOXEL
    color: dict = None
    min_weight: float = 1e-4
    cutoff_vox: float = 5.0
    planes: dict = field(default_factory=dict)  # block -> (point, unit normal) of the plane its TSDF samples
    info: dict = field(default_factory=dict)


def _blk(d, w=1.0):
    v = np.zeros((8, 8, 8), TSDF_VOXEL_DTYPE)
    v["distance"] = np.asarray(d, np.float32)
    v["weight"] = np.asarray(w, np.float32)
    return v


def _mags(rng, shape, lo=0.02, hi=0.3):
    """Distinct magnitudes (a random float32 in [lo, hi) per voxel)."""
    return rng.uniform(lo, hi, shape).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- float64
def voxel32(case):
    return float(np.float32(case.voxel))


def grid(case, key):
    """(distance, weight) of block `key` plus the first layer of its 7 upper neighbours, (9, 9, 9) float32; a missing
    neighbour's cells read weight -inf."""
    d = np.zeros((9, 9, 9), np.float32)
    w = np.full((9, 9, 9), -np.inf, np.float32)
    for ox, oy, oz in NB_DIRS:
        b = case.layer.get((key[0] + ox, key[1] + oy, key[2] + oz))
        if b is None:
            continue
        src = b[:8 - 7 * ox, :8 - 7 * oy, :8 - 7 * oz]
        dst = (slice(8 * ox, 9 if ox else 8), slice(8 * oy, 9 if oy else 8), slice(8 * oz, 9 if oz else 8))
        d[dst], w[dst] = src["distance"], src["weight"]
    return d, w


def cube_configs(case, key):
    """(8, 8, 8) configuration of every cube of the block (bit i <=> corner i has d < 0), -1 where a corner is missing or
    below min_weight."""
    d, w = grid(case, key)
    mw = np.float32(case.min_weight)
    cfg = np.zeros((8, 8, 8), np.int64)
    ok = np.ones((8, 8, 8), bool)
    for i, (ox, oy, oz) in enumerate(CORNER_OFFSETS):
        s = (slice(ox, ox + 8), slice(oy, oy + 8), slice(oz, oz + 8))
        ok &= w[s] >= mw
        cfg |= (d[s] < 0).astype(np.int64) << i
    return np.where(ok, cfg, -1)


def meshable(case, key):
    """isBlockMeshableKernel: some voxel of the block with |d| <= cutoff_distance_vox * voxel_size and weight >= min_weight."""
    b = case.layer[key]
    cutoff = np.float32(case.cutoff_vox) * np.float32(case.voxel)
    return bool(np.any((np.abs(b["distance"]) <= cutoff) & (b["weight"] >= np.float32(case.min_weight))))


def expected_vertices(case, key):
    """The block's unwelded vertices in emission order (cubes x-major, table triangles as (c, b, a)), float64, with the
    edge each came from: dict(v, pa, pb, mid, cube) or None if the block gets no mesh block."""
    if key not in case.layer or not meshable(case, key):
        return None
    cfg = cube_configs(case, key).ravel()
    nv = np.where(cfg >= 0, 3 * TRI_COUNT[np.maximum(cfg, 0)], 0)
    if nv.sum() == 0:
        return None
    d, _ = grid(case, key)
    cube = np.repeat(np.arange(512), nv)
    local = np.arange(len(cube)) - np.repeat(np.cumsum(nv) - nv, nv)
    e = EMIT_EDGES[cfg[cube], local]
    assert np.all(e >= 0)
    cv = np.stack([cube >> 6, (cube >> 3) & 7, cube & 7], axis=1)
    ga, gb = cv + CORNER_OFFSETS[EDGE_CORNERS[e, 0]], cv + CORNER_OFFSETS[EDGE_CORNERS[e, 1]]
    sa, sb = d[tuple(ga.T)], d[tuple(gb.T)]
    vox = voxel32(case)
    bp = np.asarray(key, np.float64) * (8 * vox)
    pa, pb = bp + vox * (ga + 0.5), bp + vox * (gb + 0.5)
    mid = np.abs(sa - sb) < np.float32(1e-4)  # float32 difference, as kMinSdfDifference is applied
    sa64, sb64 = sa.astype(np.float64), sb.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(mid, 0.5, sa64 / (sa64 - sb64))
    v = np.where(mid[:, None], 0.5 * (pa + pb), pa + t[:, None] * (pb - pa))
    return {"v": v, "pa": pa, "pb": pb, "mid": mid, "cube": cube, "cfg": cfg}


def coord_tol(case, *arrays):
    """A few float32 ulp of the coordinates involved and of the voxel size."""
    m = np.max(np.abs(np.stack(arrays)), axis=0)
    return 4 * np.spacing(m.astype(np.float32)).astype(np.float64) + 4 * float(np.spacing(np.float32(case.voxel)))


def check_unwelded(case, mesh):
    """An unwelded mesh layer {key: {"vertices", "normals", "triangles"}} against the float64 restatement."""
    want_keys = {k for k in case.layer if expected_vertices(case, k) is not None}
    assert set(mesh) == want_keys, (case.name, sorted(set(mesh) ^ want_keys)[:8])
    for k, b in mesh.items():
        ex = expected_vertices(case, k)
        V, N, T = b["vertices"], b["normals"], b["triangles"]
        cfg = ex["cfg"]
        ntri = int(TRI_COUNT[cfg[cfg >= 0]].sum())
        assert len(T) == 3 * ntri == len(V) == len(N), (case.name, k, len(T), 3 * ntri)  # table count over the cubes
        assert np.array_equal(T, np.arange(len(T))), (case.name, k)
        v64 = V.astype(np.float64)
        err = np.abs(v64 - ex["v"])
        tol = coord_tol(case, ex["v"], ex["pa"], ex["pb"])
        bad = np.any(err > tol, axis=1)
        assert not bad.any(), (case.name, k, int(np.argmax(bad)), v64[bad][:2], ex["v"][bad][:2], ex["mid"][bad][:2])
        check_normals(case, k, V, N)
        if k in case.planes:
            check_plane(case, k, V, N, ex)


def check_normals(case, k, V, N):
    """Flat normals: every triangle's three normals are equal, unit length within 1e-6 or exactly zero when two of its
    vertices coincide, and along the float64 cross product (v1 - v0) x (v2 - v0) of its float32 vertices."""
    tri = V.astype(np.float64).reshape(-1, 3, 3)
    n3 = N.reshape(-1, 3, 3)
    assert np.array_equal(n3[:, 0], n3[:, 1]) and np.array_equal(n3[:, 0], n3[:, 2]), (case.name, k)
    n = n3[:, 0].astype(np.float64)
    assert np.all(np.isfinite(n)), (case.name, k)
    px, py = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    cr = np.cross(px, py)
    lc = np.linalg.norm(cr, axis=1)
    ln = np.linalg.norm(n, axis=1)
    v32 = V.reshape(-1, 3, 3)
    coincide = (np.all(v32[:, 0] == v32[:, 1], axis=1) | np.all(v32[:, 1] == v32[:, 2], axis=1) |
                np.all(v32[:, 0] == v32[:, 2], axis=1))
    assert np.all(ln[coincide] == 0.0), (case.name, k)
    tiny = lc * lc < np.finfo(np.float32).tiny  # the float32 squared length is subnormal: normalisation loses its precision
    ok = (ln == 0.0) | (np.abs(ln - 1.0) <= 1e-6) | tiny
    assert ok.all(), (case.name, k, ln[~ok][:4])
    assert np.all(lc[ln == 0.0] <= 1e-6 * np.linalg.norm(px, axis=1)[ln == 0.0] * np.linalg.norm(py, axis=1)[ln == 0.0] + 1e-30)
    live = (ln > 0) & ~tiny
    with np.errstate(divide="ignore", invalid="ignore"):
        u = cr / lc[:, None]
        bound = 1e-6 + 8 * 2.0 ** -24 * np.linalg.norm(px, axis=1) * np.linalg.norm(py, axis=1) / lc
    chk = live & (bound < 0.5)
    dev = np.linalg.norm(n - u, axis=1)
    assert np.all(dev[chk] <= bound[chk]), (case.name, k, np.max(dev[chk] - bound[chk]))


def check_plane(case, k, V, N, ex):
    """On a plane case every vertex lies on the plane and every well-conditioned triangle's normal is the plane normal
    (pointing to positive distance, as PlaneMesh's (-1, 0, 0) for the plane of normal (-1, 0, 0))."""
    c, n = case.planes[k]
    v = V.astype(np.float64)
    tol = coord_tol(case, ex["v"], ex["pa"], ex["pb"]).max(axis=1) * np.sqrt(3) + np.where(ex["mid"], 0.5e-4, 1e-7)
    off = np.abs((v - c) @ n)
    assert np.all(off <= tol), (case.name, k, off.max())
    tri = v.reshape(-1, 3, 3)
    px, py = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    lc = np.linalg.norm(np.cross(px, py), axis=1)
    per = np.linalg.norm(px, axis=1) + np.linalg.norm(py, axis=1) + np.linalg.norm(tri[:, 2] - tri[:, 1], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        bound = 1e-6 + 4 * tol.reshape(-1, 3).max(axis=1) * per / lc
    chk = (lc > 0) & (bound < 0.25)
    assert chk.sum() > 0, (case.name, k)
    dev = np.linalg.norm(N.reshape(-1, 3, 3)[:, 0].astype(np.float64) - n, axis=1)
    assert np.all(dev[chk] <= bound[chk]), (case.name, k, np.max(dev[chk] - bound[chk]))


def weld_key_coord(v):
    """Index3D(v * 1000) of weldVerticesCubKernel (mesh_integrator.cu:755-757): the float32 product, truncated towards zero
    by the device's float-to-int conversion (saturating at the int32 limits, NaN -> 0)."""
    s = np.asarray(v, np.float32) * np.float32(1000.0)
    out = np.trunc(s.astype(np.float64))
    out = np.where(np.isnan(out), 0.0, np.clip(out, -2.0 ** 31, 2.0 ** 31 - 1))
    return out.astype(np.int64)


def weld_keys(vertices):
    """Index3DHash (core/hash.h:32-40): x + y * 17191 + z * 17191^2 in size_t arithmetic."""
    q = weld_key_coord(vertices).astype(np.uint64)  # int64 -> uint64 wraps like the size_t conversion
    sl = np.uint64(17191)
    with np.errstate(over="ignore"):
        return q[:, 0] + q[:, 1] * sl + q[:, 2] * (sl * sl)


def expected_weld(block):
    """The weld of one unwelded block: vertices / normals of the first vertex, in (key, index) order, of every key group;
    triangles[i] = the group of vertex i; nothing changes at WELD_MAX vertices or more."""
    V, N, T = block["vertices"], block["normals"], block["triangles"]
    nv = len(V)
    if nv >= WELD_MAX:
        return V, N, T
    keys = weld_keys(V)
    order = np.lexsort((np.arange(nv), keys))
    sk = keys[order]
    head = np.ones(nv, bool)
    head[1:] = sk[1:] != sk[:-1]
    group = np.cumsum(head) - 1
    tri = np.empty(nv, np.int32)
    tri[order] = group
    heads = order[head]
    return V[heads], N[heads], tri


def check_welded(unwelded, welded, name=""):
    assert set(unwelded) == set(welded), name
    for k, u in unwelded.items():
        w = welded[k]
        ev, en, et = expected_weld(u)
        assert len(w["triangles"]) == len(u["triangles"]), (name, k)
        assert len(w["vertices"]) == len(ev) == len(w["normals"]), (name, k, len(w["vertices"]), len(ev))
        assert np.array_equal(w["vertices"], ev) and np.array_equal(w["normals"], en), (name, k)
        assert np.array_equal(w["triangles"], et), (name, k)


def expected_colors(case, mesh):
    """updateAppearanceBlockByClosestVoxel (mesh_integrator_appearance.cu:98-147): the colour voxel the vertex lies in,
    floor((v - block_origin) / voxel) clamped to 0..7, of the co-located colour block; Gray (127) without one. Returns
    {key: (n, 3) uint8} and the number of vertices whose index was clamped from 8."""
    out, clamped = {}, 0
    vox = voxel32(case)
    for k, b in mesh.items():
        v = b["vertices"].astype(np.float64)
        cb = (case.color or {}).get(k)
        if cb is None:
            out[k] = np.full((len(v), 3), 127, np.uint8)
            continue
        q = (v - np.asarray(k, np.float64) * 8 * vox) / vox
        frac = np.abs(q - np.round(q))
        assert np.all((frac > 1e-4) | (np.round(q) <= 0) | (np.round(q) >= 8)), (case.name, k)  # no vertex on a voxel boundary
        vi = np.floor(q).astype(np.int64)
        clamped += int(np.sum(vi >= 8))
        vi = np.clip(vi, 0, 7)
        out[k] = cb["color"][vi[:, 0], vi[:, 1], vi[:, 2]]
    return out, clamped


# -------------------------------------------------------------------------------------------------------------- generators
def position_class(vx, vy, vz):
    return (int(vx == 7) << 2) | (int(vy == 7) << 1) | int(vz == 7)


def config_sweep_case(seed=0):
    """256 blocks (8 x 4 x 8) plus their upper neighbours. Per block and axis the chosen cubes sit at voxel 1, 3, 5 (inside)
    and 7 (reaching into the next block), so no two chosen cubes share a corner: 27 + 3 * 9 + 3 * 3 + 1 cubes per block,
    and every class gets each of the 256 configurations at least once. Every other voxel is positive."""
    rng = np.random.default_rng(seed)
    lat = [(x, y, z) for x in range(8) for y in range(4) for z in range(8)]
    pad = {(x + dx, y + dy, z + dz) for (x, y, z) in lat for dx, dy, dz in NB_DIRS}
    dist = {k: _mags(rng, (8, 8, 8), 0.05, 0.3) for k in pad}
    slots = {c: [] for c in range(8)}
    for key in lat:
        for vx in (1, 3, 5, 7):
            for vy in (1, 3, 5, 7):
                for vz in (1, 3, 5, 7):
                    slots[position_class(vx, vy, vz)].append((key, vx, vy, vz))
    placed = {c: [] for c in range(8)}
    for c, sl in slots.items():
        cfgs = np.concatenate([rng.permutation(256) for _ in range(-(-len(sl) // 256))])[:len(sl)]
        for (key, vx, vy, vz), cfg in zip(sl, cfgs):
            for i, (ox, oy, oz) in enumerate(CORNER_OFFSETS):
                gx, gy, gz = vx + ox, vy + oy, vz + oz
                bk = (key[0] + gx // 8, key[1] + gy // 8, key[2] + gz // 8)
                m = dist[bk][gx % 8, gy % 8, gz % 8]
                dist[bk][gx % 8, gy % 8, gz % 8] = -abs(m) if (cfg >> i) & 1 else abs(m)
            placed[c].append(int(cfg))
    layer = {k: _blk(v) for k, v in dist.items()}
    return Case("config_sweep", layer, info={"lattice": lat, "placed": placed})


def neighbour_pattern(case, key):
    return sum(1 << j for j, (ox, oy, oz) in enumerate(NB_DIRS) if j and (key[0] + ox, key[1] + oy, key[2] + oz) in case.layer)


def neighbour_sweep_case(seed=1):
    """128 centre blocks two blocks apart, centre i has the upper neighbours of the bits of i. The centre's last voxel layers
    and each neighbour's facing voxels alternate in sign (checkerboard), so every cube that reaches into a neighbour
    crosses the surface; the rest of every block is positive."""
    rng = np.random.default_rng(seed)
    layer, centres = {}, []
    for i in range(128):
        c = (2 * (i & 7), 2 * ((i >> 3) & 3), 2 * (i >> 5))
        centres.append(c)
        for j, (ox, oy, oz) in enumerate(NB_DIRS):
            if j and not (i >> (j - 1)) & 1:
                continue
            k = (c[0] + ox, c[1] + oy, c[2] + oz)
            d = _mags(rng, (8, 8, 8), 0.05, 0.3)
            x, y, z = np.meshgrid(np.arange(8), np.arange(8), np.arange(8), indexing="ij")
            near = (x == (0 if ox else 7)) | (y == (0 if oy else 7)) | (z == (0 if oz else 7)) if j else \
                (x >= 6) | (y >= 6) | (z >= 6)
            d = np.where(near & ((x + y + z) % 2 == 1), -d, d)  # one checkerboard across the blocks (8 is even)
            layer[k] = _blk(d)
    return Case("neighbour_sweep", layer, info={"centres": centres})


def _threshold_pair(target):
    """(sa > 0, sb < 0) float32 with float32(sa - sb) == target exactly and sa ~ 0.7 target."""
    sb = -np.float32(target * 0.3)
    sa = np.float32(target * 0.7)
    for _ in range(200):
        diff = np.float32(sa - sb)
        if diff == target:
            return sa, sb
        sa = np.nextafter(sa, np.float32(np.inf) if diff < target else np.float32(0))
    raise AssertionError("no float32 pair for %r" % target)


def degenerate_case(seed=2):
    """Isolated blocks (three apart, no neighbours: the cubes at index 7 have no corners) holding one degenerate value kind
    each, on a positive background."""
    rng = np.random.default_rng(seed)
    v = VOXEL
    blocks, info = {}, {}

    def base():
        return _mags(rng, (8, 8, 8), 0.1, 0.3)

    # zeros: +0.0 and -0.0 (not inside: the classification is d < 0) next to positive and negative voxels; a +0.0 voxel
    # whose 26 neighbours are all negative: its 8 cubes each get one triangle whose three vertices sit on that voxel
    d = base()
    d[2, 2, 2], d[2, 2, 3] = 0.0, -0.2
    d[5, 2, 5], d[5, 3, 5] = -0.0, -0.15
    d[5, 5, 5] = -0.0
    d[1, 5, 1] = np.float32(0.0)
    d[1, 6, 1] = -0.0
    d[3:6, 4:7, 0:3] = -_mags(rng, (3, 3, 3), 0.1, 0.3)
    d[4, 5, 1] = 0.0
    blocks[(0, 0, 0)] = _blk(d)
    # |sa - sb| == 1e-4f and one ulp either side, equal magnitudes (t = 0.5 exactly)
    d = base()
    t = np.float32(1e-4)
    pairs = [_threshold_pair(t), _threshold_pair(np.nextafter(t, np.float32(0))), _threshold_pair(np.nextafter(t, np.float32(1)))]
    for (sa, sb), y in zip(pairs, (1, 3, 5)):
        d[2, y, 2], d[3, y, 2] = sa, sb
    d[5:7, 1:3, 5:7] = np.float32(0.05) * np.where((np.indices((2, 2, 2)).sum(0) % 2) == 0, 1, -1)
    d[2, 5, 5], d[2, 6, 5] = np.float32(0.07), np.float32(-0.07)
    blocks[(3, 0, 0)] = _blk(d)
    info["threshold_pairs"] = [(float(a), float(b)) for a, b in pairs]
    # weights: exactly min_weight (used), one ulp below (cube skipped), 0, +inf (used)
    mw = np.float32(1e-4)
    d = np.where(rng.random((8, 8, 8)) < 0.4, -1, 1) * _mags(rng, (8, 8, 8), 0.05, 0.3)
    w = np.ones((8, 8, 8), np.float32)
    w[1, 1, 1], w[3, 3, 3], w[5, 5, 5], w[1, 5, 3] = mw, np.nextafter(mw, np.float32(0)), 0.0, np.inf
    w[6, 2, 5] = mw
    blocks[(0, 3, 0)] = _blk(d, w)
    # meshability: smallest |d| exactly cutoff_distance_vox * voxel (meshable) and one ulp above (not meshable)
    cut = np.float32(5.0) * np.float32(v)
    sign = np.where((np.indices((8, 8, 8)).sum(0) % 3) == 0, -1, 1).astype(np.float32)
    for key, lo in (((3, 3, 0), cut), ((0, 0, 3), np.nextafter(cut, np.float32(1)))):
        d = sign * np.maximum(_mags(rng, (8, 8, 8), float(cut) * 1.1, float(cut) * 1.5), lo)
        d[4, 4, 4] = -lo
        blocks[key] = _blk(d)
    # weight at min_weight on the only voxel within the cutoff (meshable) and one ulp below (not meshable)
    for key, wlo in (((3, 0, 3), mw), ((0, 3, 3), np.nextafter(mw, np.float32(0)))):
        d = sign * _mags(rng, (8, 8, 8), float(cut) * 1.1, float(cut) * 1.5)
        w = np.ones((8, 8, 8), np.float32)
        d[2, 2, 2], w[2, 2, 2] = np.float32(0.01), wlo
        blocks[key] = _blk(d, w)
    info["cutoff"] = float(cut)
    info["meshable"] = {(3, 3, 0): True, (0, 0, 3): False, (3, 0, 3): True, (0, 3, 3): False}
    return Case("degenerate", blocks, info=info)


def _configs(neg):
    """Configurations of the 7 x 7 x 7 cubes of an isolated block with the given inside mask."""
    cfg = np.zeros((7, 7, 7), np.int64)
    for i, (ox, oy, oz) in enumerate(CORNER_OFFSETS):
        cfg |= neg[ox:ox + 7, oy:oy + 7, oz:oz + 7].astype(np.int64) << i
    return cfg


def _flip_deltas(cfg):
    """Change of the block's triangle count when voxel p flips sign, for every p."""
    delta = np.zeros((8, 8, 8), np.int64)
    for i, (ox, oy, oz) in enumerate(CORNER_OFFSETS):
        delta[ox:ox + 7, oy:oy + 7, oz:oz + 7] += TRI_COUNT[cfg ^ (1 << i)] - TRI_COUNT[cfg]
    return delta


def _block_with_triangles(m, rng):
    """An inside mask whose 7 x 7 x 7 cubes hold exactly m triangles: the longest prefix of a random voxel order that stays
    at or below m, then single flips (the one that lands on m, else the closest)."""
    order = rng.permutation(512)
    neg = np.zeros(512, bool)
    for p in order:
        neg[p] = True
        if TRI_COUNT[_configs(neg.reshape(8, 8, 8))].sum() > m:
            neg[p] = False
            break
    neg = neg.reshape(8, 8, 8)
    for _ in range(2000):
        cfg = _configs(neg)
        need = m - int(TRI_COUNT[cfg].sum())
        if need == 0:
            return neg
        miss = np.abs(_flip_deltas(cfg) - need).ravel()
        best = np.flatnonzero(miss == miss.min())
        neg.ravel()[rng.choice(best) if miss.min() < abs(need) else rng.integers(512)] ^= True
    raise AssertionError("no block with %d triangles" % m)


def weld_size_case(seed=3, sizes=WELD_SIZES):
    """One isolated block per vertex count in `sizes`."""
    rng = np.random.default_rng(seed)
    layer, want = {}, {}
    for i, n in enumerate(sizes):
        neg = _block_with_triangles(n // 3, rng)
        key = (3 * i, 0, 0)
        layer[key] = _blk(np.where(neg, -1, 1) * _mags(rng, (8, 8, 8), 0.05, 0.3))
        want[key] = n
    return Case("weld_sizes", layer, info={"vertices": want})


def weld_origin_case(seed=4):
    """0.8 mm voxels around the origin: voxel centres at +-0.4 mm, so vertices on both sides of 0 share the key 0 (the
    conversion truncates towards zero), many distinct vertices lie within one 1 mm cell, and a vertex at x in (-2, -1] mm,
    y, z in (-1, 1) mm has the key 2^64 - 1 that the sort pads with."""
    rng = np.random.default_rng(seed)
    layer = {}
    for k in [(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)]:
        d = np.where(rng.random((8, 8, 8)) < 0.12, -1, 1) * _mags(rng, (8, 8, 8), 2e-4, 8e-4)  # sparse: < 2560 vertices
        layer[k] = d
    # x = -1.2 mm (block -1, voxel 6), y = -0.4 / +0.4 mm, z = +0.4 mm: a y-edge crossing at x key -1, y key 0, z key 0
    layer[(-1, -1, 0)][6, 7, 0], layer[(-1, 0, 0)][6, 0, 0] = np.float32(3e-4), np.float32(-5e-4)
    return Case("weld_origin", {k: _blk(v) for k, v in layer.items()}, voxel=0.0008)


def _f32_vertex_x(p0, p1, sa, sb):
    """The kernel's float32 vertex coordinate on an edge (no FMA)."""
    p0, p1, sa, sb = np.float32(p0), np.float32(p1), np.float32(sa), np.float32(sb)
    t = np.float32(sa / np.float32(sa - sb))
    return np.float32(p0 + np.float32(t * np.float32(p1 - p0)))


def weld_collision_case():
    """2.4 m voxels, one block: a vertex v1 on a y-edge at x = voxel 0's centre and a vertex v2 on an x-edge 17.191 m further
    in x and one 1 mm cell lower in y, so x2 = x1 + 17191 and y2 = y1 - 1 in key units: the same Index3DHash. The weld merges
    the two distinct vertices (as the reference does)."""
    vox = np.float32(2.4)
    d = np.full((8, 8, 8), np.float32(1.0))
    nxt = np.full((8, 8, 8), np.float32(1.0))
    jy, jz = 2, 3
    cx = lambda i: np.float32(np.float32(0.0) + np.float32(vox * np.float32(np.float32(i) + np.float32(0.5))))  # noqa: E731
    x1, yc = cx(0), cx(jy)
    ky = int(weld_key_coord(yc))
    kx1 = int(weld_key_coord(x1))
    # v1: y-edge from (0, jy, jz) to (0, jy + 1, jz), landing in y key ky + 1
    # (the table walks this edge from the upper corner down; the value picked is the middle of the key cell's range)
    hit = [s for s in np.linspace(1e-4, 3e-3, 4000)
           if int(weld_key_coord(_f32_vertex_x(cx(jy + 1), yc, np.float32(s - 1.0), np.float32(s)))) == ky + 1]
    s1 = hit[len(hit) // 2]
    d[0, jy, jz], d[0, jy + 1, jz] = np.float32(s1), np.float32(s1 - 1.0)
    # v2: x-edge from (7, jy, jz) to the +x neighbour's (0, jy, jz), landing in x key kx1 + 17191
    hit = [s for s in np.linspace(0.1, 0.3, 20000)
           if int(weld_key_coord(_f32_vertex_x(cx(7), cx(8), np.float32(s), np.float32(s - 1.0)))) == kx1 + 17191]
    s2 = hit[len(hit) // 2]
    d[7, jy, jz], nxt[0, jy, jz] = np.float32(s2), np.float32(s2 - 1.0)
    return Case("weld_collision", {(0, 0, 0): _blk(d), (1, 0, 0): _blk(nxt)}, voxel=2.4,
                info={"v1": (float(x1), float(yc)), "keys": (kx1, ky)})


def weld_saturation_case(seed=5):
    """0.5 m voxels at the block-key limits (+-2^20, |x| ~ 4.2e6 m) and around x = 2147483.648 m, where x * 1000 leaves the
    int32 range: the key's x saturates to INT32_MAX / INT32_MIN, so vertices with equal y, z keys weld across x."""
    rng = np.random.default_rng(seed)
    layer = {}
    lim = 1 << 20
    sat = int(2147483.648 / 4.0)  # block 536870 spans x = 2147480 .. 2147484 m
    keys = [(lim - 1, 0, 0), (lim - 2, 0, 0), (-lim, 0, 0), (-lim, 1, 0), (sat, 0, 0), (sat + 1, 0, 0), (-sat - 1, 0, 0),
            (-sat, 0, 0), (3, lim - 1, -lim)]
    for k in keys:
        d = np.where(rng.random((8, 8, 8)) < 0.12, -1, 1) * _mags(rng, (8, 8, 8), 0.05, 1.0)  # sparse: < 2560 vertices
        layer[k] = _blk(d)
    return Case("weld_saturation", layer, voxel=0.5)


def _plane_layer(point, normal, vox, blocks):
    layer = {}
    g = (np.arange(8) + 0.5)
    for k in blocks:
        bp = np.asarray(k, np.float64) * 8 * vox
        p = np.stack(np.meshgrid(bp[0] + vox * g, bp[1] + vox * g, bp[2] + vox * g, indexing="ij"), axis=-1)
        d = np.clip((p - point) @ normal, -4 * vox, 4 * vox)
        layer[k] = _blk(d.astype(np.float32))
    return layer


def plane_cases(seed=6):
    """Planes at random normals through a block interior, a face, an edge, a corner and a voxel centre (exact zeros), near
    the origin and ~2 km from it, each sampled on the 3 x 3 x 3 blocks around its point (regions far apart)."""
    rng = np.random.default_rng(seed)
    vox = float(np.float32(VOXEL))
    B = 8 * vox
    layer, planes, kinds = {}, {}, []
    for r, origin in enumerate([(0, 0, 0), (2500, -1250, 625)]):  # block offsets
        o = np.asarray(origin, np.float64)
        for j, kind in enumerate(["origin", "interior", "face", "edge", "corner", "voxel", "axis_face", "axis"]):
            base = o + np.array([10 * j, 0, 0])
            u = rng.random(3)
            if kind == "origin":
                if r:
                    continue
                pt = np.zeros(3)
            elif kind == "interior":
                pt = (base + 0.1 + 0.8 * u) * B
            elif kind == "face":
                pt = (base + np.array([0.0, u[1], u[2]])) * B
            elif kind == "edge":
                pt = (base + np.array([0.0, 0.0, u[2]])) * B
            elif kind in ("corner", "axis_face"):
                pt = base * B
            else:  # a voxel centre: the voxels on the plane hold exactly 0
                pt = base * B + vox * (np.array([3, 4, 5]) + 0.5)
            n = rng.normal(size=3) if not kind.startswith("axis") else np.eye(3)[j % 3] * (-1) ** j
            n = n / np.linalg.norm(n)
            c = np.floor(pt / B).astype(int)
            ks = [(c[0] + a, c[1] + b, c[2] + e) for a in (-1, 0, 1) for b in (-1, 0, 1) for e in (-1, 0, 1)]
            for k, v in _plane_layer(pt, n, vox, ks).items():
                assert k not in layer
                layer[k] = v
                planes[k] = (pt, n)
            kinds.append((kind, r))
    return Case("planes", layer, planes=planes, info={"kinds": kinds})


def colour_case(seed=7):
    """A 3 x 3 x 2 lattice with a colour per voxel ((32 x + 5, 32 y + 9, 32 z + 13) plus a per-block shift) on all but two
    blocks. Positive magnitudes 0.1..0.3, negative 0.02..0.09: every vertex sits > 2.6 % of a voxel from a voxel boundary,
    so the closest-voxel rule has one answer; the cubes at index 7 put vertices past the upper faces (index 8 -> 7)."""
    rng = np.random.default_rng(seed)
    keys = [(x, y, z) for x in range(3) for y in range(3) for z in range(2)]
    layer, color = {}, {}
    x, y, z = np.indices((8, 8, 8))
    for i, k in enumerate(keys):
        neg = rng.random((8, 8, 8)) < 0.45
        layer[k] = _blk(np.where(neg, -_mags(rng, (8, 8, 8), 0.02, 0.09), _mags(rng, (8, 8, 8), 0.1, 0.3)))
        if k in ((1, 1, 0), (2, 0, 1)):
            continue
        c = np.zeros((8, 8, 8), COLOR_VOXEL_DTYPE)
        c["color"] = np.stack([32 * x + 5 + i, 32 * y + 9 + 2 * i, 32 * z + 13 + 3 * i], axis=-1) % 256
        c["weight"] = 1.0
        color[k] = c
    return Case("colour", layer, color=color)


def noise_case(n_blocks=300, seed=8):
    """Blocks of uniform noise in +-0.4 (about 4900 vertices each): ~1.5 M vertices in one call, past the arena's first
    2^20-entry capacity."""
    rng = np.random.default_rng(seed)
    side = int(np.ceil(n_blocks ** (1 / 3)))
    keys = [(x, y, z) for x in range(side) for y in range(side) for z in range(side)][:n_blocks]
    return Case("noise", {k: _blk(rng.uniform(-0.4, 0.4, (8, 8, 8))) for k in keys})


def all_cases():
    return [config_sweep_case(), neighbour_sweep_case(), degenerate_case(), weld_size_case(), weld_origin_case(),
            weld_collision_case(), weld_saturation_case(), plane_cases(), colour_case()]
