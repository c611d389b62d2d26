"""Map clearing on the GPU (isaac_ros_nvblox_b200/csrc/nvb_clear.cu and the shared deallocation path) vs the oracle:
Mapper::clearOutsideRadius, clearTsdfInsideShapes, getClearedBlocks and ShapeClearer on the TSDF, occupancy and colour
layers. Bars: removed / touched block sets equal, voxels bit-identical, and the following ESDF, freespace and mesh updates
exact with the oracle given the tracked blocks minus the cleared ones (the incrementally updated mesh by block set, a
full-layer remesh array for array)."""
import numpy as np
import pytest

import clearing_reference as cr
from helpers import assert_color_equal, assert_esdf_equal, assert_tsdf_equal, cameras, textured_image
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

SLICE = dict(slice_min_height_m=0.25, slice_max_height_m=1.45, slice_height_m=0.9)
FS_TIME = 1000


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _set(a):
    return set(map(tuple, np.asarray(a).reshape(-1, 3).tolist()))


def _arr(s):
    return np.asarray(sorted(s), np.int32).reshape(-1, 3)


def _assert_occ_equal(g, c):
    assert set(g) == set(c), "allocated occupancy block sets differ"
    for k in c:
        assert np.array_equal(g[k]["log_odds"].view(np.uint32), c[k].view(np.uint32)), k


def _assert_mesh_blocks_equal(g, c):
    assert set(g) == set(c), "mesh block sets differ"


def _assert_mesh_full_layer_equal(p):
    """updateColorMesh(UpdateFullLayer::kYes) against the oracle's mesh of every TSDF block: vertices, normals and triangles
    of the blocks next to the removed or cleared ones included."""
    p.m.update_mesh(update_full_layer=True)
    p.o.integrate_mesh(p.o.tsdf_block_indices())
    g, c = p.m.mesh_layer().as_dict(), p.o.mesh_layer()
    assert set(g) == set(c), "mesh block sets differ"
    for k, cb in c.items():
        for f in ("vertices", "normals", "triangles"):
            assert np.array_equal(g[k][f], cb[f]), (k, f)
    assert sum(len(b["triangles"]) for b in c.values()) > 0


def _assert_marked_equal(p):
    """The ESDF update covered exactly the tracked blocks: a removed slot left in the todo list, or a reused slot listed
    twice, would change the GPU's count of marked blocks."""
    assert p.m.esdf_integrator().last_stats()["marked"] == p.o.esdf_stats()["marked"]


class Pair:
    """A mapper and the oracle map fed the same frames, with the oracle side of the tracker kept by hand."""

    def __init__(self, kind, esdf_2d, voxel=0.05):
        nvb, orc = _nvb(), _orc()
        self.kind, self.esdf_2d, self.occ = kind, esdf_2d, kind == "occupancy"
        plt = {"tsdf": nvb.ProjectiveLayerType.kTsdf, "freespace": nvb.ProjectiveLayerType.kTsdfWithFreespace,
               "occupancy": nvb.ProjectiveLayerType.kOccupancy}[kind]
        self.m, self.o = nvb.Mapper(voxel, projective_layer_type=plt), orc.OracleMap(voxel)
        self.tp = orc.default_tsdf_params()
        if esdf_2d:
            self.m.esdf_integrator().slice_params(**SLICE)
        self.cs, self.cam, self.ocam = cameras(320, 240)
        self.tracked = None  # None: the next update covers every block (update-all)
        self.tracked_mesh = None  # the colour mesh's consumer also hears of colour-integrated blocks
        self.color = not self.occ

    def proj_blocks(self):
        return self.o.occupancy_block_indices() if self.occ else self.o.tsdf_block_indices()

    def frame(self, d, T, i=0):
        b = self.m.integrate_depth(d, T, self.cam)
        if self.occ:
            self.o.integrate_occupancy(d, T, self.ocam, self.tp)
        else:
            self.o.integrate_depth(d, T, self.ocam)
        if self.tracked is not None:
            self.tracked |= _set(b)
            self.tracked_mesh |= _set(b)
        if self.color:
            img = textured_image(240, 320, seed=i)
            bc = self.m.integrate_color(img, T, self.cam)
            assert _set(bc) == _set(self.o.integrate_color(img, T, self.ocam))
            if self.tracked_mesh is not None:
                self.tracked_mesh |= _set(bc)
        return b

    def touch(self, blocks):
        """BlocksToUpdateTracker::addBlocksToUpdate for every consumer."""
        if self.tracked is not None:
            self.tracked |= _set(blocks)
            self.tracked_mesh |= _set(blocks)

    def _todo(self, mesh=False):
        t = self.tracked_mesh if mesh else self.tracked
        return self.proj_blocks() if t is None else _arr(t)

    def update(self):
        """updateEsdf / updateEsdfSlice, then updateFreespace and updateColorMesh where the mapper has them."""
        todo = self._todo()
        if self.esdf_2d:
            self.m.update_esdf_slice()
            self.o.integrate_esdf_slice(todo, z_min_m=SLICE["slice_min_height_m"], z_max_m=SLICE["slice_max_height_m"],
                                        z_output_m=SLICE["slice_height_m"], from_occupancy=self.occ,
                                        use_freespace=self.kind == "freespace")
        else:
            self.m.update_esdf()
            if self.occ:
                self.o.integrate_esdf_occupancy(todo)
            elif self.kind == "freespace":
                self.o.integrate_esdf_with_freespace(todo)
            else:
                self.o.integrate_esdf(todo)
        if self.kind == "freespace":
            self.m.update_freespace(FS_TIME)
            self.o.update_freespace(todo, FS_TIME)
        if not self.occ:
            self.m.update_mesh()
            self.o.integrate_mesh(self._todo(mesh=True))
        self.tracked, self.tracked_mesh = set(), set()

    def check(self):
        if self.occ:
            _assert_occ_equal(self.m.occupancy_layer().as_dict(), self.o.occupancy_layer())
        else:
            assert_tsdf_equal(self.m.tsdf_layer().as_dict(), self.o.tsdf_layer())
            assert_color_equal(self.m.color_layer().as_dict(), self.o.color_layer())
            _assert_mesh_blocks_equal(self.m.mesh_layer().as_dict(), self.o.mesh_layer())
        if self.kind == "freespace":
            g, c = self.m.freespace_layer().as_dict(), self.o.freespace_layer()
            assert set(g) == set(c)
            for k in c:
                assert g[k].tobytes() == c[k].tobytes(), k
        assert_esdf_equal(self.m.esdf_layer().as_dict(), self.o.esdf_layer())

    def clear_outside_radius(self, center, radius):
        r_gpu = self.m.clear_outside_radius(center, radius)
        r_cpu = cr.clear_outside_radius(self.o, center, radius, occupancy=self.occ, esdf_2d=self.esdf_2d)
        assert np.array_equal(r_gpu, r_cpu)
        if self.tracked is not None:  # removeClearedBlocksFromTracking
            self.tracked -= _set(r_cpu)
            self.tracked_mesh -= _set(r_cpu)
        return r_gpu

    def close(self):
        self.m.close()


def _frames(n=4):
    cs, _, _ = cameras(320, 240)
    return syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:n])


@pytest.mark.parametrize("esdf_2d", [False, True], ids=["esdf3d", "slice2d"])
@pytest.mark.parametrize("kind", ["tsdf", "freespace", "occupancy"])
def test_clear_outside_radius_parity(gpu, kind, esdf_2d):
    """clearOutsideRadius between frames, before the ESDF update: every layer equal after the clear and after the following
    updates, which cover the tracked blocks minus the cleared ones. getClearedBlocks lists exactly the removed blocks."""
    frames = _frames(5)
    p = Pair(kind, esdf_2d)
    for i, (d, T) in enumerate(frames[:3]):
        p.frame(d, T, i)
        p.update()
    p.check()
    p.frame(*frames[3], 3)
    center = frames[3][1][:3, 3]
    removed = p.clear_outside_radius(center, 3.0)
    assert len(removed) > 50 and (p.m.occupancy_layer() if p.occ else p.m.tsdf_layer()).num_blocks() > 50
    assert np.array_equal(p.m.get_cleared_blocks(), removed)
    assert len(p.m.get_cleared_blocks()) == 0
    p.check()
    p.update()
    p.check()
    _assert_marked_equal(p)
    # the freed slots are reused by the next frame, and those blocks are tracked once
    st = (p.m.occupancy_layer() if p.occ else p.m.tsdf_layer()).slab_stats()
    assert st["free"] == len(removed)
    p.frame(*frames[4], 4)
    assert (p.m.occupancy_layer() if p.occ else p.m.tsdf_layer()).slab_stats()["free"] < st["free"]
    p.update()
    p.check()
    _assert_marked_equal(p)
    if not p.occ:
        _assert_mesh_full_layer_equal(p)
    p.close()


def test_clear_that_removes_nothing_changes_nothing(gpu):
    frames = _frames(3)
    p = Pair("tsdf", False)
    for i, (d, T) in enumerate(frames[:2]):
        p.frame(d, T, i)
        p.update()
    p.frame(*frames[2], 2)
    before = {name: getattr(p.m, name)().as_dict() for name in ("tsdf_layer", "esdf_layer", "color_layer")}
    launches = p.m.kernel_launches()
    assert len(p.clear_outside_radius((0.0, 0.0, 1.0), 1000.0)) == 0
    assert p.m.kernel_launches() - launches == 1  # the selection kernel only
    for name, layer in before.items():
        after = getattr(p.m, name)().as_dict()
        assert set(after) == set(layer)
        assert all(after[k].tobytes() == layer[k].tobytes() for k in layer), name
    assert len(p.m.get_cleared_blocks()) == 0
    p.update()  # the pending tracker lists are what they were: the update still equals the oracle's over the frame
    p.check()
    p.close()


def test_clear_after_async_esdf_update_equals_sequential(gpu):
    nvb = _nvb()
    frames = _frames(3)
    cs, cam, _ = cameras(320, 240)
    a, b = nvb.Mapper(0.05), nvb.Mapper(0.05)
    for d, T in frames:
        a.integrate_depth(d, T, cam), b.integrate_depth(d, T, cam)
    a.update_esdf(sync=False)  # still running when the clear arrives
    ra = a.clear_outside_radius((0.5, 0.0, 1.0), 2.5)
    b.update_esdf()
    rb = b.clear_outside_radius((0.5, 0.0, 1.0), 2.5)
    assert np.array_equal(ra, rb) and len(ra) > 0
    assert_tsdf_equal(a.tsdf_layer().as_dict(), b.tsdf_layer().as_dict())
    assert_esdf_equal(a.esdf_layer().as_dict(), b.esdf_layer().as_dict())
    a.close(), b.close()


def test_cleared_set_collects_clears_and_decay(gpu):
    """getClearedBlocks: a block cleared, allocated again and cleared again is listed once; ignored blocks are dropped; the
    set is empty after a read; blocks the decay deallocates are in it too."""
    orc = _orc()
    frames = _frames(3)
    p = Pair("tsdf", False)
    ref = cr.ClearedSet()
    p.frame(*frames[0], 0)
    ref.add(p.clear_outside_radius(frames[0][1][:3, 3], 2.0))
    p.frame(*frames[0], 0)  # the same view allocates the cleared blocks again
    ref.add(p.clear_outside_radius(frames[0][1][:3, 3], 2.0))
    p.frame(*frames[1], 1)
    p.m.tsdf_decay_integrator().params(decay_factor=0.05)
    dp = orc.default_tsdf_decay_params(decay_factor=0.05)
    for _ in range(3):
        r = p.m.decay()
        assert _set(r) == _set(p.o.decay_tsdf(dp))
        ref.add(r)
    ignore = _arr(ref.s)[::3]
    got = p.m.get_cleared_blocks(ignore)
    assert np.array_equal(got, ref.get(ignore)) and len(got) > 0
    assert len(p.m.get_cleared_blocks()) == 0
    p.check()
    p.close()


def _shapes(n):
    rng = np.random.default_rng(n)
    out = []
    for i in range(n):
        c = rng.uniform([-3, -3, 0], [3, 3, 3]).astype(np.float32)
        if i % 2:
            out.append(cr.Sphere(c, rng.uniform(0.05, 0.6)))
        else:
            h = rng.uniform(0.02, 0.5, 3).astype(np.float32)
            out.append(cr.Box(c - h, c + h))
    return out


def _gpu_shapes(shapes):
    nvb = _nvb()
    return [nvb.BoundingSphere(s.center, s.radius) if isinstance(s, cr.Sphere) else nvb.AxisAlignedBoundingBox(s.min, s.max)
            for s in shapes]


@pytest.mark.parametrize("n_shapes", [1, 3, 300])
def test_clear_tsdf_inside_shapes_then_update(gpu, n_shapes):
    """clearTsdfInsideShapes: TSDF equal; the following updateEsdf covers tracked + touched blocks and the mesh loses the
    cleared surface. 300 shapes take two passes over the shared-memory shape tiles."""
    frames = _frames(3)
    p = Pair("tsdf", False)
    for i, (d, T) in enumerate(frames[:2]):
        p.frame(d, T, i)
        p.update()
    p.frame(*frames[2], 2)
    shapes = _shapes(n_shapes) if n_shapes != 1 else [cr.Sphere((2.0, 0.0, 2.0), 0.6)]  # on the scene's sphere
    touched = p.m.clear_tsdf_inside_shapes(_gpu_shapes(shapes))
    assert np.array_equal(touched, _arr(cr.clear_shapes(p.o, shapes, "tsdf"))) and len(touched) > 0
    p.touch(touched)
    assert_tsdf_equal(p.m.tsdf_layer().as_dict(), p.o.tsdf_layer())
    def near_centre():  # mesh vertices well inside the cleared sphere
        v = [b["vertices"] for b in p.m.mesh_layer().as_dict().values() if len(b["vertices"])]
        return int(np.sum(np.linalg.norm(np.concatenate(v) - shapes[0].center, axis=1) < shapes[0].radius - 0.15))
    n_near = near_centre() if n_shapes == 1 else 0
    p.update()
    p.check()
    _assert_marked_equal(p)
    _assert_mesh_full_layer_equal(p)
    if n_shapes == 1:
        assert n_near > 0 and near_centre() == 0
    assert len(p.m.get_cleared_blocks()) == 0  # nothing was deallocated
    p.close()


def test_layer_clear_shapes_occupancy_and_color(gpu):
    frames = _frames(2)
    shapes = _shapes(3) + [cr.Sphere((0.0, 0.0, 1.0), 1.0)]
    occ = Pair("occupancy", False)
    for i, (d, T) in enumerate(frames):
        occ.frame(d, T, i)
    assert len(occ.m.clear_tsdf_inside_shapes(_gpu_shapes(shapes))) == 0  # no TSDF layer: a no-op
    touched = occ.m.occupancy_layer().clear_shapes(_gpu_shapes(shapes))
    assert np.array_equal(touched, _arr(cr.clear_shapes(occ.o, shapes, "occupancy"))) and len(touched) > 0
    _assert_occ_equal(occ.m.occupancy_layer().as_dict(), occ.o.occupancy_layer())
    more = _shapes(40) + [cr.Sphere((0.0, 0.0, 1.0), 1.0)]  # a longer list on the same mapper: the shape buffer grows
    touched = occ.m.occupancy_layer().clear_shapes(_gpu_shapes(more))
    assert np.array_equal(touched, _arr(cr.clear_shapes(occ.o, more, "occupancy"))) and len(touched) > 0
    _assert_occ_equal(occ.m.occupancy_layer().as_dict(), occ.o.occupancy_layer())
    occ.close()
    p = Pair("tsdf", False)
    for i, (d, T) in enumerate(frames):
        p.frame(d, T, i)
    expect, touched_ref = cr.clear_color_shapes(p.o.color_layer(), np.float32(0.4), shapes)
    touched = p.m.color_layer().clear_shapes(_gpu_shapes(shapes))
    assert np.array_equal(touched, _arr(touched_ref)) and len(touched) > 0
    assert_color_equal(p.m.color_layer().as_dict(), expect)
    assert_tsdf_equal(p.m.tsdf_layer().as_dict(), p.o.tsdf_layer())  # the TSDF is not touched
    p.close()


def _blocks_pair(keys, voxel, seed=0):
    """A TSDF map of the given blocks (random observed voxels), on the GPU and in the oracle."""
    nvb, orc = _nvb(), _orc()
    rng = np.random.default_rng(seed)
    keys = np.asarray(keys, np.int32).reshape(-1, 3)
    vox = np.zeros((len(keys), 8, 8, 8), dtype=nvb.TSDF_VOXEL_DTYPE)
    vox["distance"] = rng.uniform(-0.1, 0.1, vox.shape).astype(np.float32)
    vox["weight"] = rng.uniform(0.5, 2.0, vox.shape).astype(np.float32)
    m, o = nvb.Mapper(voxel), orc.OracleMap(voxel)
    m.tsdf_layer().set_blocks(keys, vox)
    for k, v in zip(keys, vox):
        o.set_tsdf_block(k, v)
    return m, o


def _shell(lo, hi):
    g = np.stack(np.meshgrid(*[np.arange(a, b) for a, b in zip(lo, hi)], indexing="ij"), -1).reshape(-1, 3)
    return g.astype(np.int32)


def test_scale_two_cm_clear_past_the_remove_grid_then_esdf(gpu):
    """2 cm blocks: one clear removes more than the 1184-CTA remove grid handles in one pass; the ESDF update over the
    remaining map follows."""
    keys = _shell((-30, -30, -4), (30, 30, 4))  # 28 800 blocks of 16 cm
    m, o = _blocks_pair(keys, 0.02)
    m.update_esdf()
    o.integrate_esdf(o.tsdf_block_indices())
    r = m.clear_outside_radius((0.0, 0.0, 0.0), 2.0)
    assert len(r) > 2 * 1184
    assert np.array_equal(r, cr.clear_outside_radius(o, (0.0, 0.0, 0.0), 2.0))
    assert m.tsdf_layer().slab_stats()["free"] == len(r)
    m.update_esdf(update_full_layer=True)
    o.integrate_esdf(o.tsdf_block_indices())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()


@pytest.mark.parametrize("where", ["km", "key_limit_pos", "key_limit_neg"])
def test_scale_clear_far_from_origin(gpu, where):
    """Kilometres from the origin, and at the +-2^20 hash-key limit, where the block boxes' float bounds are coarse and the
    hash keys sit at the ends of their 21-bit fields. Outside-radius and sphere/box shape predicates both equal the oracle."""
    voxel = 0.05
    bs = np.float32(8 * voxel)
    if where == "km":
        base = np.array([7500, -5000, 10], np.int32)  # 3 km, -2 km
    elif where == "key_limit_pos":
        base = np.array([(1 << 20) - 12, (1 << 20) - 12, (1 << 20) - 12], np.int32)
    else:
        base = np.array([-(1 << 20), -(1 << 20), -(1 << 20)], np.int32)
    keys = base + _shell((0, 0, 0), (12, 12, 12))
    m, o = _blocks_pair(keys, voxel, seed=1)
    center = ((base + 6).astype(np.float32) * bs).astype(np.float32)
    shapes = [cr.Sphere(center + np.float32(0.3), 1.1), cr.Box(center - np.float32(1.7), center - np.float32(0.9))]
    touched = m.clear_tsdf_inside_shapes(_gpu_shapes(shapes))
    assert np.array_equal(touched, _arr(cr.clear_shapes(o, shapes, "tsdf"))) and len(touched) > 0
    r = m.clear_outside_radius(center, 1.5)
    assert np.array_equal(r, cr.clear_outside_radius(o, center, 1.5))
    assert 0 < len(r) < len(keys)
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert np.array_equal(m.get_cleared_blocks(), r)
    m.close()


def test_strict_edges_on_the_gpu(gpu):
    """A block face exactly at `radius` from the centre: kept by clearOutsideRadius (> is strict), not touched by a sphere
    of that radius (< is strict); an AABB that only shares the face touches it (intersects is inclusive)."""
    keys = np.array([[0, 0, 0], [1, 0, 0], [3, 0, 0]], np.int32)
    m, o = _blocks_pair(keys, 0.05)
    bs = np.float32(0.4)
    center = np.array([0.0, 0.2, 0.2], np.float32)  # inside block (0, 0, 0); block (1, 0, 0) starts at x = 0.4
    assert len(m.clear_tsdf_inside_shapes(_gpu_shapes([cr.Sphere((-0.4, 0.2, 0.2), bs)]))) == 0
    touched = m.clear_tsdf_inside_shapes(_gpu_shapes([cr.Box((-1.0, 0.0, 0.0), (0.0, 0.4, 0.4))]))
    assert _set(touched) == {(0, 0, 0)}
    cr.clear_shapes(o, [cr.Box((-1.0, 0.0, 0.0), (0.0, 0.4, 0.4))], "tsdf")
    r = m.clear_outside_radius(center, bs)
    assert _set(r) == {(3, 0, 0)}
    assert np.array_equal(r, cr.clear_outside_radius(o, center, bs))
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()


def test_clearing_dropin_program(gpu, tmp_path):
    """tests/cpp/test_clearing_dropin.cpp: clearOutsideRadius, clearTsdfInsideShapes with getShapesToClear's shapes,
    updateEsdf, getClearedBlocks and ShapeClearer<ColorLayer> through the C++ mirror."""
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_clearing_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "clearing drop-in ok" in out.stdout
