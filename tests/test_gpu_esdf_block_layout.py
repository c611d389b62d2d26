"""The ESDF layer's block format on the device (a plane of 16-byte cells, then a plane of flag words) against the reference's
20-byte EsdfVoxel records that every host-facing path keeps: random blocks through set_blocks / get_blocks, the device bytes
behind block_device_ptr, every reader of the layer (voxel lookups, interpolation, distance-and-gradient queries, the slice
image, the point export) on such a map, and a save / load round trip."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import map_io_reference as mref  # noqa: E402
import query_reference as qr  # noqa: E402

pytestmark = pytest.mark.gpu
VOXEL = 0.05
F = np.float32


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _split(records):
    """(8, 8, 8) EsdfVoxel records -> the 10 240 device bytes: cells {sq, parent} in voxel order, then the flag words."""
    words = np.frombuffer(records.tobytes(), np.uint32).reshape(512, 5)
    return np.concatenate([words[:, :4].reshape(-1), words[:, 4]]).tobytes()


def _device_bytes(ptr, n):
    import torch

    class _Dev:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}

    return torch.as_tensor(_Dev(), device="cuda").cpu().numpy().tobytes()


def _random_blocks(rng, n, dtype, every_bit):
    vox = np.zeros((n, 8, 8, 8), dtype)
    if every_bit:  # any 20 bytes, padding and negative parents included
        vox = np.frombuffer(rng.integers(0, 256, size=n * 512 * 20, dtype=np.uint8).tobytes(), dtype).reshape(n, 8, 8, 8).copy()
    else:  # values the readers take: finite squared distances, parents of either sign, flags with a random padding byte;
        # most voxels observed, so that most interpolations find their eight neighbours observed
        vox["squared_distance_vox"] = rng.integers(0, 400, size=vox.shape).astype(F)
        vox["parent_direction"] = rng.integers(-12, 13, size=vox.shape + (3,))
        for f in ("is_inside", "is_site"):
            vox[f] = rng.integers(0, 2, size=vox.shape)
        vox["observed"] = rng.uniform(size=vox.shape) < 0.97
        vox["pad"] = rng.integers(0, 256, size=vox.shape)
    return vox


def _indices(n):
    g = np.stack(np.meshgrid(np.arange(-2, 2), np.arange(-1, 2), np.arange(-1, 1), indexing="ij"), -1).reshape(-1, 3)
    return g[:n].astype(np.int32)


def test_random_blocks_round_trip_and_device_bytes(gpu):
    nvb = _nvb()
    m = nvb.Mapper(VOXEL)
    rng = np.random.default_rng(11)
    idx = _indices(12)
    vox = _random_blocks(rng, len(idx), nvb.mapper.ESDF_VOXEL_DTYPE, every_bit=True)
    layer = m.esdf_layer()
    layer.set_blocks(idx, vox)
    got, found = layer.get_blocks(np.vstack([idx, [[40, 40, 40]]]))
    assert found.tolist() == [True] * len(idx) + [False]
    assert got[:-1].tobytes() == vox.tobytes() and not got[-1].tobytes().strip(b"\0")
    for i, k in enumerate(idx):
        p = layer.block_device_ptr(k)
        assert p
        assert _device_bytes(p, 10240) == _split(vox[i]), tuple(k)
    assert layer.block_device_ptr([40, 40, 40]) == 0
    m.close()


@pytest.fixture(scope="module")
def random_map(built):
    nvb = _nvb()
    m = nvb.Mapper(VOXEL)
    rng = np.random.default_rng(5)
    idx = _indices(24)
    vox = _random_blocks(rng, len(idx), nvb.mapper.ESDF_VOXEL_DTYPE, every_bit=False)
    m.esdf_layer().set_blocks(idx, vox)
    yield dict(m=m, layer={tuple(int(c) for c in k): vox[i] for i, k in enumerate(idx)}, idx=idx, rng=rng)
    m.close()


def _points(rng, n):
    bs = 8 * VOXEL
    return np.concatenate([rng.uniform([-2 * bs, -bs, -bs], [2 * bs, 2 * bs, bs], size=(n, 3)),
                           rng.uniform(-3 * bs, 3 * bs, size=(64, 3))]).astype(F)


def test_voxel_lookups_and_interpolation(random_map):
    m, d, rng = random_map["m"], random_map["layer"], random_map["rng"]
    nvb = _nvb()
    pts = _points(rng, 3000)
    got, ok = m.esdf_layer().get_voxels(pts)
    exp, eok = qr.query_voxels(d, pts, VOXEL, nvb.mapper.ESDF_VOXEL_DTYPE)
    assert np.array_equal(ok, eok) and 0 < ok.sum() < len(pts)
    assert got.tobytes() == exp.tobytes()
    vals, vok = m.esdf_layer().interpolate(pts)
    ref = [qr.interpolate(d, p, VOXEL, "esdf") for p in pts]
    assert np.array_equal(vok, np.array([r[0] for r in ref])) and vok.sum() > 100
    ev = np.array([r[1] for r in ref], F)
    assert np.all(np.abs(vals[vok] - ev[vok]) <= 1e-6 * np.maximum(1.0, np.abs(ev[vok])))


@pytest.mark.parametrize("grad", [False, True])
def test_distance_and_gradient_queries(random_map, grad):
    import torch
    from isaac_ros_nvblox_b200 import query as q
    m, d, rng = random_map["m"], random_map["layer"], random_map["rng"]
    pts = _points(rng, 2000)
    spheres = np.concatenate([pts, rng.uniform(0, 0.1, size=(len(pts), 1)).astype(F)], 1)
    got = q.query_layer(m, q.QueryType.ESDF_GRAD if grad else q.QueryType.ESDF, torch.from_numpy(spheres).cuda()).cpu().numpy()
    out = np.full((len(spheres), 4 if grad else 1), q.ESDF_UNKNOWN_DISTANCE, F)
    assert got.tobytes() == qr.query_esdf([(d, VOXEL)], spheres, grad, out).tobytes()


def test_slice_image(random_map):
    nvb = _nvb()
    m, d = random_map["m"], random_map["layer"]
    for z in (-0.3, -0.12, 0.01, 0.37):
        aabb, img, grid = nvb.EsdfSlicer(m).slice_layer_to_distance_image(z, 1000.0, with_occupancy_grid=True)
        rows, cols = img.shape
        assert rows * cols > 0
        ys = aabb[1] + VOXEL / 2 + VOXEL * np.arange(rows, dtype=F)
        xs = aabb[0] + VOXEL / 2 + VOXEL * np.arange(cols, dtype=F)
        exp = np.full((rows, cols), 1000.0, F)
        for r in range(rows):
            for c in range(cols):
                v = qr.lookup(d, np.array([xs[c], ys[r], z], F), VOXEL)
                if v is not None and v["observed"]:
                    dist = F(VOXEL) * np.sqrt(v["squared_distance_vox"])
                    exp[r, c] = -dist if v["is_inside"] else dist
        assert img.tobytes() == exp.tobytes(), z
        eg = np.where(np.abs(exp - 1000.0) < 1e-2, -1, (exp < 1e-2) * 100).astype(np.int8)
        assert np.array_equal(grid, eg), z


def test_point_export(random_map):
    m, d = random_map["m"], random_map["layer"]
    got = m.esdf_layer().export_points()
    exp = mref.export_points("esdf", d, 8 * VOXEL, VOXEL)
    assert len(got) > 0 and got.tobytes() == np.asarray(exp, F).tobytes()


def test_save_load_keeps_the_records(random_map, tmp_path):
    nvb = _nvb()
    m, d = random_map["m"], random_map["layer"]
    path = str(tmp_path / "random.nvblx")
    m.save_layer_cake(path)
    rows = mref.read_map(path)["esdf_layer"]
    assert sorted(map(tuple, rows["xyz"])) == sorted(d)
    for k, blob in zip(map(tuple, rows["xyz"]), rows["blobs"]):
        assert blob == d[k].tobytes(), k
    m2 = nvb.Mapper(VOXEL)
    assert m2.load_map(path)["esdf"] == len(d)
    got = m2.esdf_layer().as_dict()
    assert set(got) == set(d) and all(got[k].tobytes() == d[k].tobytes() for k in d)
    for k in d:
        assert _device_bytes(m2.esdf_layer().block_device_ptr(k), 10240) == _split(d[k]), k
    m2.close()


def _robust_floor(x):
    """robustFloor of nvblox's layer_to_3d_grid_impl.cuh, in float32."""
    x = F(x)
    nearest = int(np.copysign(np.floor(abs(float(x)) + 0.5), float(x)))
    return nearest if abs(F(x - F(nearest))) < F(1e-4) else int(np.floor(x))


def _dense_grid_expected(d, aabb, default_value):
    inv = F(1.0) / F(VOXEL)
    mn = np.array([_robust_floor(F(aabb[a]) * inv) for a in range(3)])
    dims = np.array([_robust_floor(F(aabb[3 + a]) * inv) for a in range(3)]) - mn + 1
    out = np.full(tuple(dims), default_value, F)
    for ix in range(dims[0]):
        for iy in range(dims[1]):
            for iz in range(dims[2]):
                g = mn + (ix, iy, iz)
                blk = d.get(tuple(int(c) for c in g // 8))
                if blk is None:
                    continue
                v = blk[tuple(g % 8)]
                if v["observed"]:
                    dist = np.sqrt(v["squared_distance_vox"]) * F(VOXEL)
                    out[ix, iy, iz] = -dist if v["is_inside"] else dist
    return mn, out


def test_dense_grid_in_aabb(random_map):
    """The EsdfAndGradients service's dense grid: the allocated blocks' box (getAABBOfAllocatedBlocks), a box that is not
    block-aligned and reaches past the allocated blocks, and a device-memory output."""
    import ctypes as C
    import torch
    from isaac_ros_nvblox_b200 import _lib
    m, d, idx = random_map["m"], random_map["layer"], random_map["idx"]
    bs = F(8 * VOXEL)
    allocated = np.concatenate([idx.min(0) * bs, (idx.max(0) + 1) * bs]).astype(F)
    for aabb, default in ((allocated, 1000.0), (np.array([-0.93, -0.27, -0.51, 0.61, 0.33, 0.12], F), -7.5)):
        mn, grid = m.esdf_dense_grid_in_aabb(aabb, default)
        emn, exp = _dense_grid_expected(d, aabb, default)
        assert mn.tolist() == emn.tolist() and grid.shape == exp.shape
        assert grid.tobytes() == exp.tobytes()
        assert (grid != F(default)).any() and (grid == F(default)).any()
    out = torch.zeros(exp.size, dtype=torch.float32, device="cuda")
    dmn, dims = np.zeros(3, np.int32), np.zeros(3, np.int32)
    assert m._L.nvb_esdf_dense_grid_in_aabb(m._h, aabb.ctypes.data_as(C.POINTER(C.c_float)), -7.5, _lib.NVB_MEM_DEVICE,
                                            out.data_ptr(), out.numel(), dmn.ctypes.data_as(C.POINTER(C.c_int32)),
                                            dims.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    assert dims.tolist() == list(exp.shape) and out.cpu().numpy().tobytes() == exp.tobytes()
    mn, grid = m.esdf_dense_grid_in_aabb(np.array([0.1, 0.1, 0.1, 0.0, 0.2, 0.2], F), 0.0)
    assert grid.size == 0
