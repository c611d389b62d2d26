"""Known answers of map clearing on the oracle (tests/clearing_reference.py), pinned to the reference's own tests:
test_shape_clearer.cpp:62-258 (TSDF and occupancy layers), test_mapper.cpp:74-125 (ClearOutsideSphere) and
test_mapper_block_allocation.cpp:319-332 (ClearOutsideRadius); plus the strict edges of the two sphere predicates and the
cleared-blocks set. No GPU."""
import numpy as np
import pytest

import clearing_reference as cr
from helpers import cameras
from isaac_ros_nvblox_b200 import synthetic as syn
from oracle import oracle as orc

VOXEL = 0.2  # ShapeClearerTest: kVoxelSizeM 0.2, kTruncationDistanceVox 2


def _log_odds(p):
    return np.float32(np.log(p / (1.0 - p))) if 0.0 < p < 1.0 else np.float32(np.inf if p >= 1.0 else -np.inf)


def _gt_map(kind):
    """Scene::generateLayerFromScene of getSphereInBox over the scene AABB (scene_impl.h:105-145), TSDF or occupancy."""
    scene = syn.sphere_in_box()
    m = orc.OracleMap(VOXEL)
    ii = np.indices((8, 8, 8)).reshape(3, -1).T + 0.5
    bs = 8 * VOXEL
    lo_b = np.floor(np.array([-5.5, -5.5, -0.5]) / bs).astype(int)
    hi_b = np.floor(np.array([5.5, 5.5, 5.5]) / bs).astype(int)
    for x in range(lo_b[0], hi_b[0] + 1):
        for y in range(lo_b[1], hi_b[1] + 1):
            for z in range(lo_b[2], hi_b[2] + 1):
                pos = (np.array([x, y, z]) * 8 + ii) * VOXEL
                inside = np.all((pos >= [-5.5, -5.5, -0.5]) & (pos <= [5.5, 5.5, 5.5]), axis=1)
                dist = scene.distance(pos)
                if kind == "tsdf":
                    blk = np.zeros(512, dtype=orc.TSDF_VOXEL_DTYPE)
                    blk["distance"] = np.where(inside, np.clip(dist, -2 * VOXEL, 2 * VOXEL), 0).astype(np.float32)
                    blk["weight"] = inside.astype(np.float32)
                    m.set_tsdf_block((x, y, z), blk.reshape(8, 8, 8))
                else:
                    occ = dist <= np.sqrt(3.0) * VOXEL / 2.0
                    blk = np.where(inside, np.where(occ, np.float32(2.0), np.float32(-2.0)), np.float32(0)).astype(np.float32)
                    m.set_occupancy_block((x, y, z), blk.reshape(8, 8, 8))
    return m


def _values(m, kind):
    """{block: (512,) value the reference's test compares} -- TSDF weight, occupancy log odds."""
    if kind == "tsdf":
        return {k: v["weight"].reshape(512).copy() for k, v in m.tsdf_layer().items()}
    return {k: v.reshape(512).copy() for k, v in m.occupancy_layer().items()}


def _value_at(m, kind, p):
    b = tuple(int(c) for c in np.floor(np.asarray(p, np.float32) / np.float32(8 * VOXEL)).astype(int))
    v = np.floor((np.asarray(p, np.float32) - np.asarray(b) * np.float32(8 * VOXEL)) / np.float32(VOXEL)).astype(int)
    return _values(m, kind)[b][(v[0] * 8 + v[1]) * 8 + v[2]]


def _check_clearing(kind, shapes):
    """testClearingLayer (test_shape_clearer.cpp:81-139)."""
    m = _gt_map(kind)
    before = _values(m, kind)
    touched = cr.clear_shapes(m, shapes, kind)
    after = _values(m, kind)
    assert set(after) == set(before)  # no deallocation
    assert len(touched) > 0
    bs = np.float32(8 * VOXEL)
    n_before = n_after = 0
    for k, v in after.items():
        inside = np.zeros(512, bool)
        p = cr.voxel_centres(k, bs)
        for s in shapes:
            inside |= cr.contains(s, p)
        assert np.all(v[inside] == 0.0)  # cleared
        assert np.array_equal(v[~inside], before[k][~inside])  # untouched
        n_before += int(np.sum(before[k] == 0.0))
        n_after += int(np.sum(v == 0.0))
    assert n_after > n_before > 0
    return m


@pytest.mark.parametrize("kind", ["tsdf", "occupancy"])
def test_shape_clearer_empty_layer(kind):
    m = orc.OracleMap(0.05)
    assert cr.clear_shapes(m, [], kind) == []
    assert len(m.tsdf_block_indices()) == 0 and len(m.occupancy_block_indices()) == 0


@pytest.mark.parametrize("kind", ["tsdf", "occupancy"])
def test_shape_clearer_bounding_box(kind):
    h = np.float32(VOXEL / 2.0)
    c3 = np.array([2.5, 3.5, 2.1], np.float32)
    shapes = [cr.Box((-2.0, -1.0, -1.0), (0.0, 3.0, 2.5)), cr.Box((-1.0, -2.0, 2.0), (6.0, 1.0, 6.0)), cr.Box(c3 - h, c3 + h)]
    m = _check_clearing(kind, shapes)
    assert _value_at(m, kind, c3) == 0.0  # the single voxel of aabb_3
    assert _value_at(m, kind, c3 + np.float32(VOXEL)) != 0.0  # its +1 voxel neighbour


@pytest.mark.parametrize("kind", ["tsdf", "occupancy"])
def test_shape_clearer_sphere(kind):
    c3 = np.array([-4.1, -4.1, 2.1], np.float32)
    shapes = [cr.Sphere((-2.0, 1.0, 1.0), 2.0), cr.Sphere((0.0, 1.0, 2.0), 3.0), cr.Sphere(c3, VOXEL / 2.0)]
    m = _check_clearing(kind, shapes)
    assert _value_at(m, kind, c3) == 0.0
    assert _value_at(m, kind, c3 + np.float32(VOXEL)) != 0.0


@pytest.mark.parametrize("kind", ["tsdf", "occupancy"])
def test_shape_clearer_mixed_shapes(kind):
    _check_clearing(kind, [cr.Sphere((-2.0, 1.0, 1.0), 2.0), cr.Box((-1.0, -2.0, 2.0), (6.0, 1.0, 6.0))])


def _mapped(occupancy=False, frames=3):
    cs, _, ocam = cameras(320, 240)
    seq = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:frames])
    m = orc.OracleMap(0.05)
    tp = orc.default_tsdf_params()
    for d, T in seq:
        (m.integrate_occupancy(d, T, ocam, tp) if occupancy else m.integrate_depth(d, T, ocam))
    blocks = m.occupancy_block_indices() if occupancy else m.tsdf_block_indices()
    (m.integrate_esdf_occupancy if occupancy else m.integrate_esdf)(blocks)
    return m, seq, ocam


def _sphere_in_a_box_tsdf(voxel, center, radius, max_dist):
    """getSphereInABoxScene (test_mapper.cpp:34-45) through Scene::generateLayerFromScene(max_dist): ground 0, ceiling 10,
    walls at +-10, the sphere; every block of the scene AABB (-11, -11, -1)..(11, 11, 11), distances clipped to +-max_dist,
    weight 1."""
    def distance(p):  # Scene::getSignedDistanceToPoint: the planes' normals face into the room, negative beyond them
        planes = np.minimum.reduce([p[:, 2], 10.0 - p[:, 2], p[:, 0] + 10.0, 10.0 - p[:, 0], p[:, 1] + 10.0, 10.0 - p[:, 1]])
        return np.minimum(planes, np.linalg.norm(p - np.asarray(center, np.float64), axis=1) - radius)

    m = orc.OracleMap(voxel)
    ii = np.indices((8, 8, 8)).reshape(3, -1).T + 0.5
    bs = 8 * voxel
    lo = np.array([-11.0, -11.0, -1.0])
    hi = np.array([11.0, 11.0, 11.0])
    lo_b, hi_b = np.floor(lo / bs).astype(int), np.floor(hi / bs).astype(int)
    for x in range(lo_b[0], hi_b[0] + 1):
        for y in range(lo_b[1], hi_b[1] + 1):
            for z in range(lo_b[2], hi_b[2] + 1):
                pos = (np.array([x, y, z]) * 8 + ii) * voxel
                inside = np.all((pos >= lo) & (pos <= hi), axis=1)
                if not inside.any():
                    continue
                blk = np.zeros(512, dtype=orc.TSDF_VOXEL_DTYPE)
                blk["distance"] = np.where(inside, np.clip(distance(pos), -max_dist, max_dist), 0).astype(np.float32)
                blk["weight"] = inside.astype(np.float32)
                m.set_tsdf_block((x, y, z), blk.reshape(8, 8, 8))
    return m


def _all_mesh_points_on_sphere(m, center, radius):
    """allMeshPointsOnSphere (test_mapper.cpp:47-60): | |p - c| - r | <= 0.01 for every vertex."""
    v = [b["vertices"] for b in m.mesh_layer().values() if len(b["vertices"])]
    v = np.concatenate(v)
    return bool(np.all(np.abs(np.linalg.norm(v - center, axis=1) - radius) <= 0.01))


def test_clear_outside_sphere_mesh_on_sphere():
    """ClearOutsideSphere (test_mapper.cpp:74-125) on its scene: before the clear not every mesh point is on the sphere (the
    walls are meshed too); after clearOutsideRadius(sphere centre, sphere radius) the TSDF block count dropped, the ESDF has
    exactly the TSDF's blocks and every remaining mesh point lies on the sphere. (The reference also allocates a colour block
    at every TSDF block to count them; the oracle allocates colour blocks only by integrating colour frames.)"""
    center, radius = np.array([0.0, 0.0, 5.0], np.float32), 2.0
    m = _sphere_in_a_box_tsdf(0.1, center, radius, 1.0)
    blocks = m.tsdf_block_indices()
    m.integrate_mesh(blocks)
    m.integrate_esdf(blocks)
    n0 = len(blocks)
    assert not _all_mesh_points_on_sphere(m, center, radius)
    cr.clear_outside_radius(m, center, radius)
    tsdf = set(map(tuple, m.tsdf_block_indices().tolist()))
    assert 0 < len(tsdf) < n0
    assert set(map(tuple, m.esdf_block_indices().tolist())) == tsdf
    assert set(map(tuple, m.mesh_block_indices().tolist())) <= tsdf
    assert _all_mesh_points_on_sphere(m, center, radius)


@pytest.mark.parametrize("occupancy", [False, True])
def test_clear_outside_radius_every_layer_same_blocks(occupancy):
    """ClearOutsideRadius (test_mapper_block_allocation.cpp:319-332, testBlocksInLayers :109-160): after clearing around the
    origin, the ESDF and the freespace layer have exactly the projective layer's blocks, and the colour and mesh layers none
    that it lacks; fewer projective blocks than before."""
    m, seq, ocam = _mapped(occupancy)
    proj0 = m.occupancy_block_indices() if occupancy else m.tsdf_block_indices()
    if not occupancy:
        for i, (d, T) in enumerate(seq):
            m.integrate_color(np.full((240, 320, 3), 30 * i, np.uint8), T, ocam)
        m.integrate_mesh(proj0)
        m.update_freespace(proj0, 1000)
        assert len(m.freespace_block_indices()) == len(proj0) and len(m.color_block_indices()) > 0
    cr.clear_outside_radius(m, (0.0, 0.0, 1.0), 2.5, occupancy=occupancy)
    proj = set(map(tuple, (m.occupancy_block_indices() if occupancy else m.tsdf_block_indices()).tolist()))
    assert 0 < len(proj) < len(proj0)
    assert set(map(tuple, m.esdf_block_indices().tolist())) == proj
    if not occupancy:
        assert set(map(tuple, m.freespace_block_indices().tolist())) == proj
        assert 0 < len(m.color_block_indices()) and set(map(tuple, m.color_block_indices().tolist())) <= proj
        assert set(map(tuple, m.mesh_block_indices().tolist())) <= proj


def test_strict_edges():
    """A block face exactly at `radius`: kept by clearOutsideRadius (>), not touched by a sphere shape (<)."""
    bs = np.float32(0.4)
    blocks = np.array([[1, 0, 0], [-1, 0, 0], [0, 2, 0]], np.int32)
    center = np.array([0.0, 0.2, 0.2], np.float32)  # block (1, 0, 0) starts at x = 0.4; (-1, 0, 0) ends at x = 0
    d = cr.block_exterior_distance(blocks, bs, center)
    assert d[0] == bs and d[1] == 0.0 and d[2] > bs
    assert len(cr.blocks_outside_radius(blocks[:1], bs, center, bs)) == 0  # kept
    assert not cr.touches_block(cr.Sphere(center, bs), blocks[:1], bs)[0]  # not touched
    assert cr.touches_block(cr.Box((-1.0, 0.0, 0.0), (0.4, 0.4, 0.4)), blocks[:1], bs)[0]  # inclusive intersects
    assert len(cr.blocks_outside_radius(blocks, bs, center, 0.0)) == 2  # radius 0: all but the block holding the centre


def test_cleared_set_semantics():
    """getClearedBlocks (mapper.cpp:509-521): a set; ignored blocks leave it; a read empties it; decay deallocations feed
    it (clearBlocksInLayers, mapper_impl.h:226,263)."""
    s = cr.ClearedSet()
    s.add([[1, 2, 3], [0, 0, 0]])
    s.add([[1, 2, 3]])  # cleared, reallocated, cleared again
    m, _, _ = _mapped(frames=1)
    s.add(m.decay_tsdf(orc.default_tsdf_decay_params(decay_factor=0.01)))
    got = s.get(ignore=[[0, 0, 0]])
    assert [1, 2, 3] in got.tolist() and [0, 0, 0] not in got.tolist() and len(got) > 1
    assert got.tolist() == sorted(got.tolist()) and len({tuple(r) for r in got.tolist()}) == len(got)
    assert len(s.get()) == 0


def test_remove_blocks_removes_exactly_the_chosen_blocks():
    m, _, _ = _mapped(occupancy=True, frames=1)
    blocks = m.occupancy_block_indices()
    before = m.occupancy_layer()
    chosen = blocks[::4]
    cr.remove_blocks(m, chosen, occupancy=True)
    after = m.occupancy_layer()
    assert set(after) == set(before) - set(map(tuple, chosen.tolist()))
    assert all(np.array_equal(after[k], before[k]) for k in after)


def test_clearing_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_clearing_dropin.cpp (nvblox_ros' clearing calls through nvblox/nvblox.h) builds with plain g++ against the
    C-ABI library; without a GPU it reports that and exits 77."""
    import subprocess
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_clearing_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
