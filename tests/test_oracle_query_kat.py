"""The point-query restatement (tests/query_reference.py) pinned to the reference's own tests: test_3d_interpolation.cpp
(NeighboursTest, OffsetTest, InterpolationTest), test_layer.cpp (CopyVoxelsToHost, GetTsdfVoxelsOnDevice) and nvblox_torch's
test_query.py / test_query_esdf.py / test_esdf_gradients.py (bounds and gradient directions on a sphere map the oracle builds).
No GPU needed."""
import numpy as np
import pytest

import query_reference as qr
from helpers import spheres_distance, tsdf_layer_from_distance

F = np.float32
K_FLOAT_EPSILON = 1e-6  # test_3d_interpolation.cpp
TSDF_DT = np.dtype([("distance", "<f4"), ("weight", "<f4")])
ESDF_DT = np.dtype([("squared_distance_vox", "<f4"), ("parent_direction", "<i4", (3,)), ("is_inside", "u1"), ("observed", "u1"),
                    ("is_site", "u1"), ("pad", "u1")])


def _indices_block(axis, offset=0, esdf=False):
    """fillVoxelsWithIndices (test_3d_interpolation.cpp:33-77): every voxel holds its index along `axis` (+ offset)."""
    idx = np.indices((8, 8, 8))[axis].astype(F) + F(offset)
    if esdf:
        b = np.zeros((8, 8, 8), ESDF_DT)
        b["squared_distance_vox"] = idx * idx
        b["observed"] = 1
        return b
    b = np.zeros((8, 8, 8), TSDF_DT)
    b["distance"], b["weight"] = idx, 1.0
    return b


def test_neighbours():
    """NeighboursTest: no neighbours below the first voxel centre; the x-ordered 8 voxels; crossing into block (1, 0, 0)."""
    layer = {(0, 0, 0): _indices_block(0)}
    assert qr.surrounding(layer, np.zeros(3, F), 1.0)[0] is None
    assert qr.surrounding(layer, np.full(3, 0.1, F), 1.0)[0] is None
    vox, _ = qr.surrounding(layer, np.full(3, 0.6, F), 1.0)
    assert [float(v["distance"]) for v in vox] == [0, 0, 0, 0, 1, 1, 1, 1]
    p = np.array([8.0, 0.6, 0.6], F)
    assert qr.surrounding(layer, p, 1.0)[0] is None
    layer[(1, 0, 0)] = _indices_block(0)
    vox, _ = qr.surrounding(layer, p, 1.0)
    assert [float(v["distance"]) for v in vox] == [7, 7, 7, 7, 0, 0, 0, 0]


def test_offset():
    """OffsetTest: the offset of p from the low corner voxel's centre, in voxels."""
    layer = {(0, 0, 0): _indices_block(0)}
    _, o = qr.surrounding(layer, np.full(3, 0.5, F), 1.0)
    assert np.all(np.abs(o) < K_FLOAT_EPSILON)
    _, o = qr.surrounding(layer, np.ones(3, F), 1.0)
    assert np.all(np.abs(o - 0.5) < K_FLOAT_EPSILON)


@pytest.mark.parametrize("esdf", [False, True])
def test_interpolation_of_linear_fields(esdf):
    """InterpolationTest: on layers whose voxels hold their x, y or z index, the interpolated value at a random point inside
    the block's interior is the point's coordinate minus half a voxel (the ESDF member is sqrt(index^2))."""
    rng = np.random.default_rng(0)
    kind = "esdf" if esdf else "tsdf"
    for axis in range(3):
        layer = {(0, 0, 0): _indices_block(axis, esdf=esdf)}
        for p in rng.uniform(0.5, 7.5, (1000, 3)).astype(F):
            ok, v = qr.interpolate(layer, p, 1.0, kind)
            assert ok and abs(float(v) - (float(p[axis]) - 0.5)) < 1e-5


def test_interpolation_validity_rules():
    """A voxel of weight <= 1e-4 (TSDF) or not observed (ESDF) makes the point fail; every occupancy voxel is valid and the
    member is the probability."""
    t = _indices_block(0)
    t["weight"][3, 3, 3] = F(1e-4)
    assert not qr.interpolate({(0, 0, 0): t}, np.full(3, 3.6, F), 1.0, "tsdf")[0]
    assert qr.interpolate({(0, 0, 0): t}, np.full(3, 2.4, F), 1.0, "tsdf")[0]
    e = _indices_block(0, esdf=True)
    e["observed"][4, 4, 4] = 0
    assert not qr.interpolate({(0, 0, 0): e}, np.full(3, 4.2, F), 1.0, "esdf")[0]
    occ = np.zeros((8, 8, 8), F)
    ok, v = qr.interpolate({(0, 0, 0): occ}, np.full(3, 4.2, F), 1.0, "occupancy")
    assert ok and v == F(0.5)


def test_get_voxels_copy_to_host():
    """CopyVoxelsToHost / GetTsdfVoxelsOnDevice (test_layer.cpp): the voxel at each voxel centre of an allocated block is that
    voxel; points in unallocated blocks fail; rejected points fail."""
    blk = _indices_block(1, offset=3)
    layer = {(0, 0, 0): blk, (-1, 2, 0): _indices_block(2)}
    centres = (np.indices((8, 8, 8)).reshape(3, -1).T.astype(F) + F(0.5)) * F(0.05)
    vox, found = qr.query_voxels(layer, centres, 0.05, TSDF_DT)
    assert found.all() and np.array_equal(vox, blk.reshape(-1))
    pts = np.array([[1.0, 1.0, 1.0], [np.nan, 0, 0], [0.4 * (1 << 20) + 1, 0, 0], [-0.01, 0.81, 0.01]], F)
    vox, found = qr.query_voxels(layer, pts, 0.05, TSDF_DT)
    assert found.tolist() == [False, False, False, True]


@pytest.fixture(scope="module")
def sphere_map():
    """The oracle's ESDF of two spheres of radius 0.5 (the scene of nvblox_torch's query tests, made smaller)."""
    from oracle import oracle as orc
    voxel = 0.05
    fn = spheres_distance([(0.0, 0.0, 0.0), (1.5, 0.0, 0.0)], 0.5)
    idx, tsdf = tsdf_layer_from_distance(fn, (-1.0, -1.0, -1.0), (2.5, 1.0, 1.0), voxel, 4 * voxel)
    m = orc.OracleMap(voxel)
    for k, v in zip(idx, tsdf):
        m.set_tsdf_block(k, v)
    m.integrate_esdf(idx, orc.default_esdf_params(max_esdf_distance_m=2.0, min_weight=1e-4))
    return m.esdf_layer(), voxel, fn


def test_esdf_query_bounds_and_gradients(sphere_map):
    """test_query_esdf.py / test_esdf_gradients.py: inside a sphere the distance is negative, outside positive and close to
    the true distance; the gradient points away from the surface outside, towards it inside; unobserved / missing voxels
    give the unknown distance 100 with the gradient left as pre-filled."""
    layer, voxel, fn = sphere_map
    rng = np.random.default_rng(1)
    dirs = rng.normal(size=(300, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    r = rng.uniform(0.65, 0.9, (300, 1))
    outside = (dirs * r).astype(F)
    spheres = np.concatenate([outside, np.zeros((300, 1), F)], 1)
    out = qr.query_esdf([(layer, voxel)], spheres, True, np.full((300, 4), 100.0, F))
    assert np.all(out[:, 3] > 0) and np.all(np.abs(out[:, 3] - fn(outside)) < 3 * voxel)
    cos = np.sum(out[:, :3] * dirs, 1) / np.maximum(np.linalg.norm(out[:, :3], axis=1), 1e-9)
    assert np.mean(cos > 0.7) > 0.9  # away from the sphere
    inside = (dirs * rng.uniform(0.1, 0.35, (300, 1))).astype(F)
    spheres_in = np.concatenate([inside, np.zeros((300, 1), F)], 1)
    out_in = qr.query_esdf([(layer, voxel)], spheres_in, True, np.full((300, 4), 100.0, F))
    assert np.all(out_in[:, 3] < 0)
    # the radius is subtracted
    spheres_r = spheres.copy()
    spheres_r[:, 3] = 0.1
    out_r = qr.query_esdf([(layer, voxel)], spheres_r, False, np.full((300, 1), 100.0, F))
    assert np.array_equal(out_r[:, 0], (out[:, 3] - F(0.1)).astype(F))
    far = qr.query_esdf([(layer, voxel)], np.array([[40.0, 0, 0, 0]], F), True, np.full((1, 4), 7.0, F))
    assert far.tolist() == [[7.0, 7.0, 7.0, 7.0]]


def test_multi_mapper_rules():
    """queryESDFMultiMapperKernel's early exit, the TSDF minimum and the occupancy maximum on hand-set voxels."""
    def esdf_layer(sq, inside=0, observed=1, parent=(1, 0, 0)):
        b = np.zeros((8, 8, 8), ESDF_DT)
        b["squared_distance_vox"], b["is_inside"], b["observed"], b["parent_direction"] = sq, inside, observed, parent
        return {(0, 0, 0): b}
    s = np.array([[0.1, 0.1, 0.1, 0.0]], F)
    a, b = esdf_layer(4.0, parent=(2, 0, 0)), esdf_layer(1.0, parent=(0, 1, 0))
    out = qr.query_esdf([(a, 0.1), (b, 0.1)], s, True, np.full((1, 4), 100.0, F))
    assert np.allclose(out, [[0.0, -1.0, 0.0, 0.1]])           # the second mapper is the minimum: its gradient
    out = qr.query_esdf([(b, 0.1), (a, 0.1)], s, True, np.full((1, 4), 100.0, F))
    assert np.allclose(out, [[0.0, -1.0, 0.0, 0.1]])           # the larger second one writes the minimum, keeps the gradient
    out = qr.query_esdf([(b, 0.1), (esdf_layer(0.0, observed=0), 0.1)], s, True, np.full((1, 4), 100.0, F))
    assert out[0, 3] == 100.0 and np.allclose(out[0, :3], [0.0, -1.0, 0.0])  # unobserved overwrites the distance
    t1 = {(0, 0, 0): np.full((8, 8, 8), np.array((0.3, 2.0), TSDF_DT))}
    t2 = {(0, 0, 0): np.full((8, 8, 8), np.array((-0.1, 5.0), TSDF_DT))}
    p = np.array([[0.1, 0.1, 0.1], [-1.0, 0.1, 0.1]], F)
    assert qr.query_tsdf([(t1, 0.1), (t2, 0.1)], p, np.zeros((2, 2), F)).tolist() == [[F(-0.1), 5.0], [100.0, 0.0]]
    assert qr.query_tsdf([(t1, 0.1)], p, np.zeros((2, 2), F)).tolist() == [[F(0.3), 2.0], [0.0, 0.0]]
    o1 = {(0, 0, 0): np.full((8, 8, 8), -2.0, F)}
    o2 = {(0, 0, 0): np.full((8, 8, 8), 1.5, F)}
    occ = qr.query_occupancy([(o1, 0.1), (o2, 0.1)], p)
    assert occ[0, 0] == F(1.5) and occ[1, 0] == qr.log_odds_from_probability(0.0)
    assert abs(float(occ[1, 0]) - np.log(1e-3 / (1 - 1e-3))) < 1e-5


def test_query_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_query_dropin.cpp (getVoxels and interpolateOnCPU through nvblox/nvblox.h) builds with plain g++ against
    the C-ABI library; without a GPU it reports that and exits 77."""
    import subprocess
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_query_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
