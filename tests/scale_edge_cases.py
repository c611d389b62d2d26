"""Configurations that cross the size and coordinate thresholds where the CUDA path switches code paths, shared by the
non-GPU precondition checks (test_scale_edges_guard.py) and the GPU parity tests (test_gpu_scale_edges.py).

Thresholds (nvb_view.cu):
  * SMEM_CELLS: a view AABB with more cells than the raycast's shared-memory bitset (kMaxSmemWords = 12 288 words) marks
    straight into the global bitset (viewRaycastKernel<false>);
  * CHAINED_CELLS: a bitset of more than kChainedThresholdWords = 65 536 words is compacted with the ticketed chained scan.
A case is meant to sit at least MARGIN (20 %) beyond the threshold it tests, on the intended side.
"""
import numpy as np

from helpers import cameras, view_grid
from isaac_ros_nvblox_b200 import synthetic as syn

SMEM_CELLS = 12288 * 32        # 393 216
CHAINED_CELLS = 65536 * 32     # 2 097 152
MARGIN = 1.2
TSDF_SLAB_LIMIT_CELLS = 1 << 22  # a frame of more cells would grow the TSDF slab to 2^23 blocks (32 GiB)
KEY_LIMIT = 1 << 20              # block indices must lie in [-2^20, 2^20) (21-bit hash key)

FIXTURE_RADIAL = (0.1, 0.1, 0.01, 0.001, 0.001, 0.001)  # tests/include/nvblox/tests/sensor_fixture.h:97-104
FIXTURE_TANGENTIAL = (0.01, 0.02)


def case_cells(case):
    """-> (min block index, size, cells) of a case's view AABB."""
    cs, _, _ = cameras(case["width"], case["height"])
    return view_grid(cs.fu, cs.fv, cs.cu, cs.cv, cs.width, cs.height, case["pose"], 8 * case["voxel"], case["max_dist"],
                     radial=case.get("radial"), tangential=case.get("tangential"))


def random_depth(case, seed):
    """Uniform depth in [0.5, 0.95 max] m, so the touched cells spread over the whole view AABB."""
    rng = np.random.default_rng(seed)
    return rng.uniform(0.5, 0.95 * case["max_dist"], size=(case["height"], case["width"])).astype(np.float32)


def _case(name, width, height, voxel, max_dist, theta, path, **kw):
    return dict(name=name, width=width, height=height, voxel=voxel, max_dist=max_dist, pose=syn.circle_pose(theta),
                path=path, **kw)


# path: "smem" (shared-memory bitset, tiles independent), "global" (global bitset, tiles independent), "chained" (global
# bitset, chained scan).
VIEW_CASES = [
    _case("640x480_5cm_25m", 640, 480, 0.05, 25.0, 1.1, "global"),
    _case("1280x720_5cm_25m", 1280, 720, 0.05, 25.0, 0.3, "global"),
    _case("640x480_2cm_10m", 640, 480, 0.02, 10.0, 0.3, "global"),
    _case("640x480_5cm_25m_distorted", 640, 480, 0.05, 25.0, 0.6, "global", radial=FIXTURE_RADIAL,
          tangential=FIXTURE_TANGENTIAL),
    _case("640x480_5cm_15m", 640, 480, 0.05, 15.0, 0.0, "smem"),
    _case("640x480_5cm_40m", 640, 480, 0.05, 40.0, 0.0, "chained"),
    _case("640x480_5cm_40m_b", 640, 480, 0.05, 40.0, 1.1, "chained"),
]
VIEW = {c["name"]: c for c in VIEW_CASES}
SMALL_VIEW = _case("640x480_5cm_7m", 640, 480, 0.05, 7.0, 0.7, "smem")

# Integration over the shared-memory threshold: 2 cm voxels, 10 m (the frames themselves only see the 10 m room).
INTEGRATE_2CM = [_case("320x240_2cm_10m_%d" % i, 320, 240, 0.02, 10.0, th, "global") for i, th in enumerate((0.0, 0.35, 0.7))]
# One frame on the chained path: 5 cm, 40 m. Its cells decide how far the TSDF slab grows (2^22 blocks = 16 GiB).
INTEGRATE_CHAINED = _case("320x240_5cm_40m", 320, 240, 0.05, 40.0, 0.0, "chained")

# The union of block lists over an AABB of more than CHAINED_CELLS cells.
UNION_BOX = ((-150, -150, -15), (150, 150, 15))


def union_cells():
    lo, hi = np.array(UNION_BOX[0]), np.array(UNION_BOX[1])
    return int(np.prod(hi - lo + 1))


def union_lists(seed=2):
    """Two block lists whose union spans UNION_BOX (its corners are in the lists), with overlap between them."""
    rng = np.random.default_rng(seed)
    lo, hi = np.array(UNION_BOX[0]), np.array(UNION_BOX[1])
    a = rng.integers(lo, hi + 1, size=(60000, 3)).astype(np.int32)
    b = rng.integers(lo, hi + 1, size=(40000, 3)).astype(np.int32)
    b[:5000] = a[:5000]
    a[0], a[1] = lo, hi
    return a, b


# Far from the origin: the pose's translation is shifted by these offsets (m).
FAR_OFFSETS = [(12345.6, -23456.7, 345.6), (-4096.3, 2500.7, -300.2)]


def shifted(T, offset):
    T = np.array(T, np.float32)
    T[:3, 3] = (T[:3, 3].astype(np.float64) + np.asarray(offset, np.float64)).astype(np.float32)
    return T


KEY_LIMIT_SHIFTS = {
    "x_high": (KEY_LIMIT - 1, 0, 0),            # x in {2^20 - 2, 2^20 - 1}
    "x_low": (-KEY_LIMIT + 1, 0, 0),            # x in {-2^20, -2^20 + 1}
    "corner_high": (KEY_LIMIT - 1,) * 3,        # at the limit on all three axes
    "corner_low": (-KEY_LIMIT + 1,) * 3,
}


def key_limit_blocks(name):
    """A sphere (r = 0.25 m, 5 cm voxels, truncation 0.2 m) in the 2 x 2 x 2 blocks -1..0, moved to the hash-key limit.
    -> (block indices (8, 3) int32, TSDF voxels (8, 8, 8, 8))."""
    from helpers import spheres_distance, tsdf_layer_from_distance
    idx, vox = tsdf_layer_from_distance(spheres_distance([(0.0, 0.0, 0.0)], 0.25), (-0.4, -0.4, -0.4), (0.39, 0.39, 0.39),
                                        0.05, 0.2)
    return (idx + np.asarray(KEY_LIMIT_SHIFTS[name], np.int32)).astype(np.int32), vox


def key_limit_block_sets():
    return [key_limit_blocks(n)[0] for n in KEY_LIMIT_SHIFTS]


# ---------------------------------------------------------------------------------------------------------------------
# Long-range ESDF scene: 2 cm voxels, a slab of observed free space with small site clusters, max distance 4 m (200 voxels,
# 25 blocks), so that parents lie more than 15 blocks away (the "unknown box" branch of the exchange-slab wavefront).
# ---------------------------------------------------------------------------------------------------------------------
LR_VOXEL = 0.02
LR_MAX_DIST = 4.0
LR_TRUNC = 4 * LR_VOXEL
LR_SLAB = (40, 40, 6)
LR_CLUSTERS = {"a": (20, 20, 2), "b": (33, 9, 3), "c": (8, 34, 2)}  # block of each cluster's 3x3x3 voxel cube


def lr_free_block():
    from helpers import TSDF_DT
    b = np.zeros((8, 8, 8), TSDF_DT)
    b["distance"], b["weight"] = np.float32(LR_TRUNC), np.float32(1.0)
    return b


def lr_cluster_block(name):
    b = lr_free_block()
    b["distance"][3:6, 2:5, 4:7] = np.float32(-0.01)
    b["distance"][2, 2, 2] = np.float32(0.0)
    return np.asarray(LR_CLUSTERS[name], np.int32), b


def lr_steps():
    """-> list of (blocks to set: (idx (n, 3), voxels (n, 8, 8, 8)), blocks to integrate (m, 3)): the full slab with clusters
    a and b, then cluster a removed, then cluster c added."""
    nx, ny, nz = LR_SLAB
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    vox = np.repeat(lr_free_block()[None], len(g), axis=0)
    for name in ("a", "b"):
        k, b = lr_cluster_block(name)
        vox[np.all(g == k, axis=1)] = b
    steps = [((g, vox), g)]
    ka, _ = lr_cluster_block("a")
    steps.append(((ka[None], lr_free_block()[None]), ka[None]))
    kc, bc = lr_cluster_block("c")
    steps.append(((kc[None], bc[None]), kc[None]))
    return steps


def far_parent_voxels(esdf_layer):
    """Voxels whose parent lies in a block more than 15 blocks away on some axis (block offset floor((voxel + parent) / 8)
    outside [-16, 15]): the parent box of such a block does not fit the wavefront's 5-bit fields.
    -> (voxels with an offset below -16, voxels with an offset above 15)."""
    v = np.stack(np.meshgrid(np.arange(8), np.arange(8), np.arange(8), indexing="ij"), -1)
    low = high = 0
    for blk in esdf_layer.values():
        p = blk["parent_direction"].astype(np.int64)
        has = p.any(axis=-1)
        off = np.floor_divide(v + p, 8)
        low += int((has & np.any(off < -16, axis=-1)).sum())
        high += int((has & np.any(off > 15, axis=-1)).sum())
    return low, high


# ---------------------------------------------------------------------------------------------------------------------
# Deallocation, slot reuse and slab growth (nvb_api.cu nvb_mapper_decay / ensureTsdfCapacity / LayerSlab::grow, nvb_util.cu
# removeBlocksKernel, nvb_esdf.cu esdfRemoveBlocksKernel, nvb_internal.cuh hashFindOrInsert):
#   * REMOVE_GRID: the remove kernels launch at most 1184 CTAs, one dead block per CTA and round; more dead blocks than
#     that take several rounds;
#   * a frame that allocates more new blocks than the free stack holds empties the stack inside one allocation launch
#     (atomicSub below zero, atomicAdd back) and continues with fresh slots;
#   * a frame whose view AABB does not fit behind the slab's high-water mark doubles the slab (LayerSlab::grow copies the
#     free stack and rehashes up to the high-water mark), here while the stack is not empty.
# The churn sequence: 2 cm voxels, three frames at a 4 m range, a decay that removes everything outside a sphere, then one
# frame at a 7 m range (its view AABB is ~5x larger than the 4 m frames').
# ---------------------------------------------------------------------------------------------------------------------
REMOVE_GRID = 1184
CHURN = dict(voxel=0.02, width=320, height=240, near_m=4.0, far_m=7.0, capacity=4096, radius_m=2.5, frames=3)


def churn_frames():
    """-> (frames [(depth, T)] * 4, product camera, oracle camera): three frames to build the map, one after the decay."""
    cs, cam, ocam = cameras(CHURN["width"], CHURN["height"])
    return syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:CHURN["frames"] + 1]), cam, ocam


def churn_exclusion_center(frames):
    """2.5 m in front of the first camera: the decay keeps the blocks within CHURN['radius_m'] of it."""
    T = frames[0][1]
    return tuple(float(c) for c in T[:3, 3] + np.float32(2.5) * T[:3, 2])


def churn_cells(T, max_dist):
    cs, _, _ = cameras(CHURN["width"], CHURN["height"])
    return view_grid(cs.fu, cs.fv, cs.cu, cs.cv, cs.width, cs.height, T, 8 * CHURN["voxel"], max_dist)[2]


def grown_capacity(capacity, high_water, cells):
    """ensureTsdfCapacity: the slab doubles until the frame's view cells fit behind the high-water mark."""
    while capacity < high_water + cells:
        capacity *= 2
    return capacity


# Occupancy decay parameters that take every observed voxel to 0.5 in one step (free +4.6, occupied -4.6 log odds).
OCC_WIPE = dict(free_region_decay_probability=0.99, occupied_region_decay_probability=0.01)
TSDF_WIPE = dict(decay_factor=1e-6, decayed_weight_threshold=1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# Mesh arena (nvb_api.cu MeshArena::repack): at least 2^20 entries, and after a repack at least twice the live data plus the
# update. MESH_ARENA_TARGET: a 2 cm full-layer update grows it past 2^22 entries.
# Freespace (nvb_api.cu updateFreespaceImpl): freespaceUpdateKernel runs on 4 CTAs per SM; H100 SXM has 132 SMs.
# ---------------------------------------------------------------------------------------------------------------------
MESH_ARENA_MIN = 1 << 20
MESH_ARENA_TARGET = 1 << 22
FREESPACE_GRID_H100 = 4 * 132


# ---------------------------------------------------------------------------------------------------------------------
# The long-range scene restated as an occupancy layer: a voxel is occupied (log odds +6.9) where its TSDF distance is at or
# below zero, free (-6.9) elsewhere; the occupancy ESDF marks the same sites as the TSDF one.
# ---------------------------------------------------------------------------------------------------------------------
def occupancy_from_tsdf(vox):
    """(n, 8, 8, 8) TSDF voxels -> (n, 8, 8, 8) float32 log odds."""
    return np.where(vox["distance"] <= 0.0, np.float32(6.9), np.float32(-6.9)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# 2-D slices. SLICER_AABB: an EsdfSlicer image box of SLICER_PIXELS at 2 cm voxels (one thread per pixel, a 2-D grid of
# 16 x 16 tiles). The far-origin slice heights follow the z offsets of FAR_OFFSETS (+345.6 m and -300.2 m).
# ---------------------------------------------------------------------------------------------------------------------
SLICER_AABB = (-30.0, -25.0, 0.0, 30.0, 25.0, 0.0)  # min x, min y, min z, max x, max y, max z (m)
SLICE_Z = dict(slice_min_height_m=0.25, slice_max_height_m=1.45, slice_height_m=0.9)


def slicer_pixels(voxel=0.02):
    """Image size of EsdfSlicer::sliceLayerToDistanceImage over SLICER_AABB: ceil(extent / voxel) per axis."""
    x0, y0, _, x1, y1, _ = SLICER_AABB
    return int(np.ceil((x1 - x0) / voxel)) * int(np.ceil((y1 - y0) / voxel))


def gyroid_layer(lo=(-2.4, -2.4, 0.0), hi=(2.39, 2.39, 1.91), voxel=0.02, period=0.24, trunc=0.08):
    """A gyroid-like periodic surface (sin x cos y + sin y cos z + sin z cos x = 0, scaled to a distance) filling a box:
    every block of the box crosses the surface, so a full-layer mesh update emits ~250 vertices per block.
    -> (block indices (n, 3), TSDF voxels (n, 8, 8, 8))."""
    from helpers import tsdf_layer_from_distance
    k = 2.0 * np.pi / period

    def fn(P):
        x, y, z = (k * P[..., i].astype(np.float64) for i in range(3))
        return (np.sin(x) * np.cos(y) + np.sin(y) * np.cos(z) + np.sin(z) * np.cos(x)) / k

    return tsdf_layer_from_distance(fn, lo, hi, voxel, trunc)


def smooth_image(rows, cols):
    """RGB ramps without texture: a colour sample moved by a fraction of a pixel changes by at most a few levels."""
    y, x = np.mgrid[0:rows, 0:cols]
    return np.stack([x * 255 // (cols - 1), y * 255 // (rows - 1), (x + y) * 255 // (rows + cols - 2)], -1).astype(np.uint8)


def far_colour_differences(far_layer, near_layer, offset, voxel):
    """Largest colour-channel difference of each voxel coloured (weight > 0) in both maps, matched by the voxel-index shift
    offset / voxel, and the fraction of the origin map's coloured voxels that were matched."""
    shift = np.round(np.asarray(offset, np.float64) / voxel).astype(np.int64)

    def coloured(layer):
        out = {}
        for k, b in layer.items():
            for v in np.argwhere(b["weight"] > 0):
                out[tuple(np.asarray(k, np.int64) * 8 + v)] = b["color"][tuple(v)].astype(np.int64)
        return out

    f, n = coloured(far_layer), coloured(near_layer)
    diff = [int(np.max(np.abs(f[tuple(np.asarray(k) + shift)] - c))) for k, c in n.items() if tuple(np.asarray(k) + shift) in f]
    return np.asarray(diff), len(diff) / max(len(n), 1)


def far_vertex_distances(far_mesh, near_mesh, offset):
    """Distance of every origin-map mesh vertex to the nearest far-map vertex shifted back by offset (float64)."""
    from scipy.spatial import cKDTree
    fv = np.concatenate([b["vertices"] for b in far_mesh.values()]).astype(np.float64) - np.asarray(offset, np.float64)
    nv = np.concatenate([b["vertices"] for b in near_mesh.values()]).astype(np.float64)
    return cKDTree(fv).query(nv)[0]


def far_colour_bounds(offset):
    """Bounds on far_colour_differences, calibrated on the oracle with smooth_image: matched fraction, median and 99th
    percentile (colour levels; the 99th percentile scales with the float32 spacing at the offset)."""
    spacing = float(np.spacing(np.float32(np.max(np.abs(offset)))))
    return 0.97, 0, 4096.0 * spacing


def far_vertex_bounds(offset, voxel):
    """Bounds on far_vertex_distances: median within one float32 spacing at the offset, 99th percentile within half a
    voxel (a voxel distance that rounds differently moves a surface crossing along its edge)."""
    return float(np.spacing(np.float32(np.max(np.abs(offset))))), 0.5 * voxel
