"""The reference's map clearing restated on the oracle, for the clearing tests.

- Mapper::clearOutsideRadius (src/mapper/mapper.cpp:473-492): the blocks outside the radius (getBlocksOutsideRadius,
  src/geometry/bounding_spheres.cpp:23-31,47-50,69-74) go through Mapper::clearBlocksInLayers, which the oracle
  restates for the decay. A decay that spares every other block and fully decays every voxel it touches removes exactly
  the chosen blocks through that same code, so the deallocation is not restated twice.
- ShapeClearer::clear (integrators/internal/cuda/impl/shape_clearer_impl.cuh:22-127) with BoundingShape::touchesBlock
  / contains (src/geometry/bounding_shape.cpp:48-66, bounding_spheres.h:29-32, Eigen AlignedBox): float32 numpy in the
  reference's evaluation order, written back through the oracle's block setters.
- Mapper::getClearedBlocks (mapper.cpp:509-521): a set fed by every clearBlocksInLayers (ClearedSet below).
"""
import numpy as np

from oracle import oracle as orc

F = np.float32
VOXEL_CENTRES = np.indices((8, 8, 8)).reshape(3, -1).T.astype(np.float32)  # voxel (x, y, z) of linear offset (x*8+y)*8+z


class Sphere:
    def __init__(self, center, radius):
        self.center, self.radius = np.asarray(center, F).reshape(3), F(radius)


class Box:
    def __init__(self, mn, mx):
        self.min, self.max = np.asarray(mn, F).reshape(3), np.asarray(mx, F).reshape(3)


def block_exterior_distance(blocks, block_size, center):
    """AlignedBox::exteriorDistance(center) of getAABBOfBlock for each (n, 3) block: the axes accumulate from 0 in order."""
    b = np.asarray(blocks, np.int32).reshape(-1, 3).astype(F)
    bs, c = F(block_size), np.asarray(center, F).reshape(3)
    dist2 = np.zeros(len(b), F)
    for k in range(3):
        bmin, bmax = b[:, k] * bs, (b[:, k] + F(1.0)) * bs
        aux = np.where(bmin > c[k], bmin - c[k], np.where(c[k] > bmax, c[k] - bmax, F(0)))
        dist2 = (dist2 + aux * aux).astype(F)
    return np.sqrt(dist2).astype(F)


def blocks_outside_radius(blocks, block_size, center, radius):
    blocks = np.asarray(blocks, np.int32).reshape(-1, 3)
    return blocks[block_exterior_distance(blocks, block_size, center) > F(radius)]


def touches_block(shape, blocks, block_size):
    blocks = np.asarray(blocks, np.int32).reshape(-1, 3)
    if isinstance(shape, Sphere):
        return block_exterior_distance(blocks, block_size, shape.center) < shape.radius
    b, bs = blocks.astype(F), F(block_size)
    bmin, bmax = b * bs, (b + F(1.0)) * bs
    return np.all((shape.min <= bmax) & (bmin <= shape.max), axis=1)


def voxel_centres(block, block_size):
    """getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81) for the 512 voxels."""
    bs = F(block_size)
    vs, hv = bs * F(1.0 / 8), bs * F(0.5 / 8)
    return ((bs * np.asarray(block, F).reshape(1, 3) + vs * VOXEL_CENTRES) + hv).astype(F)


def contains(shape, p):
    if isinstance(shape, Sphere):
        d = (shape.center - p).astype(F)
        d2 = (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(F)  # Eigen a0 + (a1 + a2)
        return np.sqrt(d2) <= shape.radius
    return np.all((shape.min <= p) & (p <= shape.max), axis=1)


def shape_clear_plan(blocks, block_size, shapes):
    """ShapeClearer::clear's selection -> {block: (512,) bool voxels to reset} for the touched blocks."""
    blocks = np.asarray(blocks, np.int32).reshape(-1, 3)
    touched = np.zeros(len(blocks), bool)
    for s in shapes:
        touched |= touches_block(s, blocks, block_size)
    plan = {}
    for k in blocks[touched]:
        p = voxel_centres(k, block_size)
        inside = np.zeros(512, bool)
        for s in shapes:
            inside |= contains(s, p)
        plan[tuple(int(c) for c in k)] = inside
    return plan


def clear_shapes(m, shapes, kind):
    """ShapeClearer<kind layer>::clear on the oracle map (kind: 'tsdf' or 'occupancy'); returns the touched blocks sorted."""
    bs = F(8) * F(m.voxel_size)
    blocks = m.tsdf_block_indices() if kind == "tsdf" else m.occupancy_block_indices()
    plan = shape_clear_plan(blocks, bs, shapes)
    for k, inside in plan.items():
        if kind == "tsdf":
            v = m.tsdf_block(k).reshape(512).copy()
            v["distance"][inside], v["weight"][inside] = 0.0, 0.0
            m.set_tsdf_block(k, v.reshape(8, 8, 8))
        else:
            v = _occ_block(m, k)
            v[inside] = 0.0
            m.set_occupancy_block(k, v.reshape(8, 8, 8))
    return sorted(plan)


def _occ_block(m, k):
    blk = np.zeros(512, np.float32)
    orc.lib().or_occupancy_get_block(m._h, orc._ip(np.ascontiguousarray(k, dtype=np.int32)), blk.ctypes.data)
    return blk


def clear_color_shapes(color_layer, block_size, shapes):
    """ShapeClearer<ColorLayer>::clear on a {block: (8,8,8) COLOR_VOXEL_DTYPE} dict: Color::Gray() (127, 127, 127), weight 0."""
    out = {k: v.copy() for k, v in color_layer.items()}
    plan = shape_clear_plan(np.asarray(sorted(out), np.int32).reshape(-1, 3), block_size, shapes)
    for k, inside in plan.items():
        v = out[k].reshape(512)
        v["color"][inside] = 127
        v["weight"][inside] = 0.0
    return out, sorted(plan)


class ClearedSet:
    """Mapper::cleared_blocks_ and getClearedBlocks (mapper.cpp:509-521)."""

    def __init__(self):
        self.s = set()

    def add(self, blocks):
        self.s.update(tuple(int(c) for c in k) for k in np.asarray(blocks).reshape(-1, 3))

    def get(self, ignore=()):
        self.s.difference_update(tuple(int(c) for c in k) for k in np.asarray(ignore, np.int32).reshape(-1, 3))
        out = np.asarray(sorted(self.s), np.int32).reshape(-1, 3)
        self.s.clear()
        return out


def remove_blocks(m, blocks, occupancy=False, esdf_2d=False):
    """Mapper::clearBlocksInLayers(blocks) on the oracle map, through its decay: every other projective block is spared,
    and the chosen ones decay to fully decayed in one step (TSDF: weight -> threshold; occupancy: log odds -> 0)."""
    blocks = np.asarray(blocks, np.int32).reshape(-1, 3)
    if len(blocks) == 0:
        return blocks
    proj = m.occupancy_block_indices() if occupancy else m.tsdf_block_indices()
    drop = {tuple(int(c) for c in k) for k in blocks}
    keep = np.asarray([k for k in proj if tuple(int(c) for c in k) not in drop], np.int32).reshape(-1, 3)
    clear_esdf = 2 if esdf_2d else 1
    if occupancy:
        p = orc.default_occupancy_decay_params(free_region_decay_probability=1.0, occupied_region_decay_probability=0.0,
                                               decay_to_probability=0.5, deallocate_decayed_blocks=1)
        removed = m.decay_occupancy(p, excluded_blocks=keep if len(keep) else None, clear_esdf=clear_esdf)
    else:
        p = orc.default_tsdf_decay_params(decay_factor=1e-6, deallocate_decayed_blocks=1, set_free_distance_on_decayed=0)
        removed = m.decay_tsdf(p, excluded_blocks=keep if len(keep) else None, clear_esdf=clear_esdf)
    assert {tuple(int(c) for c in k) for k in removed} == drop & {tuple(int(c) for c in k) for k in proj}
    return removed


def clear_outside_radius(m, center, radius, occupancy=False, esdf_2d=False):
    """Mapper::clearOutsideRadius on the oracle map -> the removed blocks, sorted."""
    proj = m.occupancy_block_indices() if occupancy else m.tsdf_block_indices()
    out = blocks_outside_radius(proj, F(8) * F(m.voxel_size), center, radius)
    remove_blocks(m, out, occupancy, esdf_2d)
    return np.asarray(sorted(tuple(int(c) for c in k) for k in out), np.int32).reshape(-1, 3)
