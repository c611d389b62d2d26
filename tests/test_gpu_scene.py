"""primitives::Scene on the GPU (nvb_scene_*, isaac_ros_nvblox_b200.scene) against its numpy restatement
(tests/scene_reference.py): depth images and generated layers bit for bit, nvblox_torch's toMapper against the oracle's ESDF
and mesh of the same blocks, and the reference's accuracy criteria against the scene's ground truth. The library is built
with -fmad=false, so the kernels and the restatement do the same binary32 and binary64 operations."""
import ctypes as C

import numpy as np
import pytest

import camera_pose_cases as cpc
import scene_reference as sr
from helpers import assert_esdf_equal

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(autouse=True)
def _release_mappers():
    """A Mapper and its layer views reference each other: collect them after each test, so that the many mappers made
    here do not pile up device memory."""
    yield
    import gc
    gc.collect()


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _sc():
    from isaac_ros_nvblox_b200 import scene
    return scene


def _orc():
    from oracle import oracle as orc
    return orc


def _cams(w=640, h=480, f=300.0):
    from oracle import oracle as orc
    return _nvb().Camera(f, f, w / 2.0, h / 2.0, w, h), orc.Camera(f, f, w / 2.0, h / 2.0, w, h)


def _look_at(pos, target):
    pos, target = np.asarray(pos, np.float64), np.asarray(target, np.float64)
    z = target - pos
    z /= np.linalg.norm(z)
    x = np.cross(z, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, np.cross(z, x), z, pos
    return T.astype(F)


def circle_poses(n=80, radius=3.5, height=2.0):
    """n cameras on a horizontal circle around the z axis, each looking at (0, 0, height)."""
    return [_look_at([radius * np.cos(a), radius * np.sin(a), height], [0, 0, height])
            for a in np.linspace(0, 2 * np.pi, n, endpoint=False)]


def dummy():
    s = _sc().Scene()
    s.create_dummy_map()
    return s


def _depth_eq(s, cam, ocam, T, max_dist, invalid=0.0):
    got = s.render_depth(cam, T, max_dist, invalid, device=0).cpu().numpy()
    want = sr.depth_image(sr.primitives_of(s), ocam, T, max_dist, invalid)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.argwhere(got != want)[:5]
    return got


# ---------------------------------------------------------------------------------------------------------------------
# Depth images
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["dummy", "sphere_in_box"])
def test_depth_along_the_circle(gpu, which):
    s = dummy() if which == "dummy" else _sc().getSphereInBox()
    cam, ocam = _cams()
    hits = 0
    for T in circle_poses():
        d = _depth_eq(s, cam, ocam, T, 20.0)
        hits += int(np.count_nonzero(d > 0))
    assert hits > 0.9 * 80 * 640 * 480


@pytest.mark.parametrize("name", ["aniso_0.9", "half_integer_317x239", "distorted"])
def test_depth_general_and_distorted_cameras(gpu, name):
    _, cam, ocam = cpc.cameras(cpc.CAMS[name])
    s = dummy()
    for T in circle_poses(4, 3.0, 1.5):
        _depth_eq(s, cam, ocam, T, 20.0)


def test_depth_cut_off_and_invalid_value(gpu):
    cam, ocam = _cams(320, 240, 150.0)
    s = dummy()
    T = circle_poses(1)[0]
    d = _depth_eq(s, cam, ocam, T, 2.0, invalid=-7.5)
    assert np.any(d == F(-7.5)) and np.any(d != F(-7.5))


def test_depth_parallel_rays_and_cameras_inside_primitives(gpu):
    cam, ocam = _cams(320, 240, 150.0)
    s = _sc().Scene()
    s.add_ground_level(0.0)  # the camera's horizontal rays run parallel to it
    s.add_primitive("cube", [0, 0, 1, 2, 2, 2])
    s.add_primitive("sphere", [4, 0, 1, 1.5])
    s.add_primitive("cylinder", [-4, 0, 1, 1.5, 2])
    for pos in ([0, 0, 1], [4, 0, 1], [-4, 0, 1], [0, -6, 1]):
        for target in ([1, 0, 1], [0, 1, 1], [3, 3, 0.2]):
            _depth_eq(s, cam, ocam, _look_at(pos, target), 20.0)


def test_depth_far_from_the_origin(gpu):
    off = np.array(cpc.FAR_OFFSET, F)
    s = _sc().Scene()
    s.add_primitive("plane", list(off + [0, 0, 0]) + [0, 0, 1])
    s.add_primitive("cube", list(off + [1, 0, 1]) + [1, 1, 1])
    s.add_primitive("sphere", list(off + [0, 2, 1]) + [0.7])
    s.add_primitive("cylinder", list(off + [-1, -1, 1]) + [0.5, 2])
    cam, ocam = _cams(320, 240, 150.0)
    for a in np.linspace(0, 2 * np.pi, 4, endpoint=False):
        _depth_eq(s, cam, ocam, _look_at(off + [4 * np.cos(a), 4 * np.sin(a), 1.5], off + [0, 0, 1]), 20.0)


def test_depth_1080p_and_host_equals_device_and_other_streams(gpu):
    import torch
    cam, ocam = _cams(1920, 1080, 900.0)
    s = dummy()
    T = circle_poses(3)[1]
    dev = _depth_eq(s, cam, ocam, T, 20.0)
    host = s.render_depth(cam, T, 20.0)
    assert np.array_equal(host.view(np.uint32), dev.view(np.uint32))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = s.render_depth(cam, T, 20.0, device=0)
        again = out.clone()
    st.synchronize()
    assert np.array_equal(again.cpu().numpy().view(np.uint32), dev.view(np.uint32))


def test_signed_distance_host_and_device(gpu):
    import torch
    s = dummy()
    p = np.random.default_rng(3).uniform(-6, 6, (100000, 3)).astype(F)
    want = sr.signed_distance(sr.primitives_of(s), p, 1.5)
    assert np.array_equal(s.signed_distance(p, 1.5).view(np.uint32), want.view(np.uint32))
    got = s.signed_distance(torch.from_numpy(p).cuda(), 1.5).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# Layers
# ---------------------------------------------------------------------------------------------------------------------
_KINDS = {"tsdf": (0, "TSDF"), "occupancy": (1, "OCCUPANCY"), "freespace": (2, "FREESPACE")}


def _mapper(kind, voxel=0.1):
    nvb = _nvb()
    t = {"tsdf": nvb.ProjectiveLayerType.kTsdf, "occupancy": nvb.ProjectiveLayerType.kOccupancy,
         "freespace": nvb.ProjectiveLayerType.kTsdfWithFreespace}[kind]
    return nvb.Mapper(voxel, projective_layer_type=t)


def _layer(m, kind):
    return {"tsdf": m.tsdf_layer, "occupancy": m.occupancy_layer, "freespace": m.freespace_layer}[kind]()


def _values(kind, v):
    if kind == "tsdf":
        return np.stack([v["distance"], v["weight"]], axis=-1)
    if kind == "occupancy":
        return v["log_odds"]
    return v["is_high_confidence_freespace"] != 0


def _layer_id(kind):
    return getattr(_nvb()._lib, "NVB_LAYER_" + _KINDS[kind][1])


def _check_layer(s, m, kind, max_dist, sample=None, old=None):
    got = _layer(m, kind).as_dict()
    bs = m.block_size()
    want_blocks = {tuple(b) for b in sr.blocks_touched(bs, sr.aabb_of(s)).tolist()} | set(old or {})
    assert set(got) == want_blocks
    keys = sorted(got)
    if sample is not None and len(keys) > sample:
        keys = [keys[i] for i in np.random.default_rng(0).choice(len(keys), sample, replace=False)]
    prims, aabb = sr.primitives_of(s), sr.aabb_of(s)
    for k in keys:
        want = sr.generate_block(prims, aabb, bs, k, max_dist, kind, None if old is None or k not in old else old[k])
        g = _values(kind, got[k])
        assert np.array_equal(g.view(np.uint32) if kind != "freespace" else g,
                              want.view(np.uint32) if kind != "freespace" else want), k


@pytest.mark.parametrize("kind", sorted(_KINDS))
def test_layer_equals_the_restatement(gpu, kind):
    s = dummy()
    m = _mapper(kind, 0.2)
    s.generate_layer(m, _layer_id(kind), 0.4)
    _check_layer(s, m, kind, 0.4, sample=200)


@pytest.mark.parametrize("kind", sorted(_KINDS))
def test_layer_aabb_faces_on_voxel_centres_and_pre_existing_blocks(gpu, kind):
    m = _mapper(kind, 0.1)
    lid = _layer_id(kind)
    # an earlier scene fills a wider box
    first = _sc().Scene()
    first.set_aabb([-1.6, -1.6, -0.8], [1.6, 1.6, 1.6])
    first.add_primitive("sphere", [0.3, -0.2, 0.4, 0.6])
    first.generate_layer(m, lid, 0.3)
    old = {k: _values(kind, v).copy() for k, v in _layer(m, kind).as_dict().items()}
    # the second AABB's six faces are voxel centres (binary32, as the kernel computes them), so the closed box's faces count
    bs = m.block_size()
    lo = sr.voxel_centers(bs, (-1, -1, 0))[2, 4, 0]
    hi = sr.voxel_centers(bs, (0, 0, 1))[7, 4, 1]
    s = _sc().Scene()
    s.set_aabb(lo.tolist(), hi.tolist())
    alo, ahi = sr.aabb_of(s)
    for k in range(3):
        along = np.concatenate([sr.voxel_centers(bs, tuple(b))[..., k].reshape(-1) for b in sr.blocks_touched(bs, (alo, ahi))])
        assert alo[k] in along and ahi[k] in along, k
    s.add_primitive("cube", [0.1, 0.0, 0.5, 0.6, 0.4, 0.3])
    s.add_primitive("cylinder", [-0.2, 0.1, 0.4, 0.25, 0.5])
    s.add_ground_level(0.15)
    s.generate_layer(m, lid, 0.3)
    _check_layer(s, m, kind, 0.3, old=old)


def test_default_box_at_2cm_grows_the_slab(gpu):
    s = dummy()
    s.set_aabb(*_sc().DEFAULT_AABB)
    m = _nvb().Mapper(0.02, tsdf_capacity_blocks=1 << 16)  # 64^3 blocks need two doublings
    cap0 = m.tsdf_layer().slab_stats()["capacity"]
    s.generate_layer(m, _nvb()._lib.NVB_LAYER_TSDF, 0.08)
    assert m.tsdf_layer().slab_stats()["capacity"] > cap0
    assert m.tsdf_layer().num_blocks() == len(sr.blocks_touched(m.block_size(), sr.aabb_of(s)))
    _check_layer(s, m, "tsdf", 0.08, sample=40)


def test_more_primitives_than_one_shared_memory_tile(gpu):
    rng = np.random.default_rng(1)
    s = _sc().Scene()
    s.set_aabb([-2, -2, -2], [2, 2, 2])
    for c in rng.uniform(-2, 2, (5000, 3)):
        s.add_primitive("cube", list(c) + list(rng.uniform(0.02, 0.1, 3)))
    for kind in ("tsdf", "occupancy"):
        m = _mapper(kind, 0.1)
        s.generate_layer(m, _layer_id(kind), 0.4)
        _check_layer(s, m, kind, 0.4, sample=12)
    p = rng.uniform(-2, 2, (3000, 3)).astype(F)
    assert np.array_equal(s.signed_distance(p, 1.0), sr.signed_distance(sr.primitives_of(s), p, 1.0))
    cam, ocam = _cams(64, 48, 30.0)
    _depth_eq(s, cam, ocam, _look_at([3, 3, 3], [0, 0, 0]), 20.0)


def test_capacity_error_leaves_the_map_unchanged(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.1)
    small = _sc().Scene()
    small.set_aabb([-0.5, -0.5, -0.5], [0.5, 0.5, 0.5])
    small.add_primitive("sphere", [0, 0, 0, 0.3])
    small.append_to_mapper(m)
    before_t, before_e = m.tsdf_layer().as_dict(), m.esdf_layer().as_dict()
    huge = _sc().Scene()
    huge.set_aabb([-400, -400, -200], [400, 400, 200])  # 1000 x 1000 x 500 blocks of 0.8 m > 2^28
    huge.add_primitive("sphere", [0, 0, 0, 1])
    for call in (lambda: huge.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 0.4), lambda: huge.append_to_mapper(m)):
        with pytest.raises(nvb._lib.NvbError) as e:
            call()
        assert e.value.code == -3
    after_t = m.tsdf_layer().as_dict()
    assert set(after_t) == set(before_t) and all(np.array_equal(after_t[k], before_t[k]) for k in before_t)
    assert set(m.esdf_layer().as_dict()) == set(before_e)


# ---------------------------------------------------------------------------------------------------------------------
# toMapper / append_to_mapper
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_esdf_of(m, occupancy=False):
    o = _orc().OracleMap(m.voxel_size())
    if occupancy:
        layer = m.occupancy_layer().as_dict()
        for k, v in layer.items():
            o.set_occupancy_block(k, v["log_odds"])
        o.integrate_esdf_occupancy(np.array(sorted(layer), np.int32))
    else:
        layer = m.tsdf_layer().as_dict()
        for k, v in layer.items():
            o.set_tsdf_block(k, v)
        o.integrate_esdf(np.array(sorted(layer), np.int32))
    return o


@pytest.mark.parametrize("kind", ["tsdf", "occupancy"])
def test_to_mapper_layer_esdf_and_mesh(gpu, kind):
    nvb = _nvb()
    s = dummy()
    types = [nvb.ProjectiveLayerType.kTsdf if kind == "tsdf" else nvb.ProjectiveLayerType.kOccupancy]
    m = s.to_mapper([0.2], types)
    assert isinstance(m, nvb.Mapper)
    _check_layer(s, m, kind, F(4.0) * F(m.voxel_size()), sample=150)
    o = _oracle_esdf_of(m, occupancy=kind == "occupancy")
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    if kind == "tsdf":
        from test_gpu_mesh import assert_mesh_equal
        m.update_mesh()
        o.integrate_mesh(blocks=o.tsdf_block_indices())
        assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer())


def test_append_to_a_mapper_that_integrated_frames(gpu):
    """Frames first (ESDF and mesh consumers started), then the scene: the projective layer is replaced, every block is
    marked, and the ESDF and a mesh update equal the oracle's on the same history."""
    from test_gpu_mesh import assert_mesh_equal
    nvb = _nvb()
    s = _sc().getSphereInBox()
    s.set_aabb([-5.5, -5.5, -0.5], [5.5, 5.5, 5.5])
    cam, ocam = _cams(160, 120, 75.0)
    m, o = nvb.Mapper(0.2), _orc().OracleMap(0.2)
    for T in circle_poses(3):
        depth = s.render_depth(cam, T, 20.0)
        b = m.integrate_depth(depth, T, cam)
        m.update_esdf()
        m.update_mesh()
        o.integrate_esdf(o.integrate_depth(depth, T, ocam))
    assert all(k in {tuple(x) for x in sr.blocks_touched(m.block_size(), sr.aabb_of(s)).tolist()} for k in m.tsdf_layer().as_dict())
    s.append_to_mapper([m], 0)
    _check_layer(s, m, "tsdf", F(4.0) * F(0.2), sample=100)
    layer = m.tsdf_layer().as_dict()
    for k, v in layer.items():
        o.set_tsdf_block(k, v)
    o.integrate_esdf(np.array(sorted(layer), np.int32))
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.update_mesh()
    o.integrate_mesh(blocks=o.tsdf_block_indices())
    assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer())


def test_nvblox_torch_to_mapper_and_map_sdf_flow(gpu):
    """nvblox_torch's test_scene.py::test_to_mapper and test_map_sdf.py's flow: a dummy map at 2 cm, update_esdf, then
    query_differentiable_layer gives finite distances and gradients."""
    import torch
    from isaac_ros_nvblox_b200.query import QueryType, query_layer
    s = dummy()
    m = s.to_mapper(voxel_sizes_m=[0.1])
    assert m.tsdf_layer().num_blocks() > 0
    m2 = s.to_mapper(voxel_sizes_m=[0.02])
    m2.update_esdf()
    q = torch.tensor([[1.5, 1.5, 1.0], [-3.0, 2.0, 2.5], [0.0, 3.5, 4.0]], dtype=torch.float32, device="cuda")
    out = query_layer(m2, QueryType.ESDF_GRAD, q)
    torch.cuda.synchronize()
    assert torch.all(torch.isfinite(out)) and torch.all(out[:, 3] > 0) and torch.all(out[:, 3] < 2.5)
    many = s.to_mapper([0.2, 0.1])
    assert isinstance(many, list) and len(many) == 2


# ---------------------------------------------------------------------------------------------------------------------
# Ground truth
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["dummy", "sphere_in_box"])
def test_esdf_of_the_ground_truth_tsdf_against_the_scene(gpu, which):
    """test_esdf_integrator.cpp's criterion: at most 0.2 % of the observed ESDF voxels within the ESDF's range are more
    than one voxel from the scene's signed distance at their centres. The AABB reaches past the walls, so that the voxels
    behind them hold the negative distances the ESDF's sites need."""
    s = dummy() if which == "dummy" else _sc().getSphereInBox()
    s.set_aabb([-5.5, -5.5, -0.5], [5.5, 5.5, 5.5])
    m = s.to_mapper([0.1])
    vs, bs = m.voxel_size(), m.block_size()
    esdf = m.esdf_layer().as_dict()
    pts, dist = [], []
    for k, v in esdf.items():
        obs = v["observed"] != 0
        d = vs * np.sqrt(v["squared_distance_vox"]) * np.where(v["is_inside"] != 0, -1.0, 1.0)
        pts.append(sr.voxel_centers(bs, k)[obs])
        dist.append(d[obs])
    pts, dist = np.concatenate(pts).astype(F), np.concatenate(dist)
    gt = s.signed_distance(pts, 100.0)
    lo, hi = sr.aabb_of(s)
    keep = (np.abs(gt) < 1.5) & np.all((pts >= lo) & (pts <= hi), axis=1)
    bad = np.abs(dist[keep] - gt[keep]) > vs
    assert keep.sum() > 10000 and bad.mean() <= 0.002, (bad.mean(), keep.sum())


def test_tsdf_integrated_from_scene_depth_against_the_ground_truth(gpu):
    """SphereSceneTest's criterion: the TSDF integrated from the scene's depth images along the circle differs from the
    ground-truth TSDF by more than the truncation distance at under 0.4 % of the voxels both observe."""
    s = _sc().getSphereInBox()
    cam, _ = _cams()
    m = _nvb().Mapper(0.05)
    for T in circle_poses(40, 3.5, 2.0):
        m.integrate_depth_async(s.render_depth(cam, T, 20.0), T, cam)
    m.synchronize()
    trunc = F(4.0) * F(0.05)
    got = m.tsdf_layer().as_dict()
    gt_m = _nvb().Mapper(0.05)
    s.generate_layer(gt_m, _nvb()._lib.NVB_LAYER_TSDF, trunc)
    gt = gt_m.tsdf_layer().as_dict()
    n = bad = 0
    for k, v in got.items():
        if k not in gt:
            continue
        both = (v["weight"] > 0) & (gt[k]["weight"] > 0) & (np.abs(gt[k]["distance"]) < trunc)
        n += int(both.sum())
        bad += int((np.abs(v["distance"][both] - gt[k]["distance"][both]) > trunc).sum())
    assert n > 50000 and bad / n < 0.004, (bad, n)


# ---------------------------------------------------------------------------------------------------------------------
# Errors
# ---------------------------------------------------------------------------------------------------------------------
def test_invalid_arguments(gpu):
    nvb = _nvb()
    L = nvb._lib.load()
    lib = nvb._lib
    cam, _ = _cams(32, 24, 20.0)
    from isaac_ros_nvblox_b200.mapper import colmajor
    T = colmajor(np.eye(4))
    out = np.zeros((24, 32), F)
    fp = T.ctypes.data_as(C.POINTER(C.c_float))

    def scene_of(*prims):
        arr = (lib.NvbPrimitive * max(len(prims), 1))(*prims)
        s = lib.NvbScene(C.cast(arr, C.POINTER(lib.NvbPrimitive)), len(prims), (C.c_float * 3)(-1, -1, -1),
                         (C.c_float * 3)(1, 1, 1))
        return s, arr

    good, _a = scene_of(lib.NvbPrimitive(lib.NVB_PRIM_SPHERE, (C.c_float * 3)(0, 0, 2), (C.c_float * 4)(1, 0, 0, 0)))
    bad_type, _b = scene_of(lib.NvbPrimitive(7, (C.c_float * 3)(0, 0, 2), (C.c_float * 4)(1, 0, 0, 0)))
    bad_normal, _c = scene_of(lib.NvbPrimitive(lib.NVB_PRIM_PLANE, (C.c_float * 3)(0, 0, 2), (C.c_float * 4)(0, 0, 1.002, 0)))
    null_list = lib.NvbScene(None, 2, (C.c_float * 3)(), (C.c_float * 3)())
    H = lib.NVB_MEM_HOST
    assert L.nvb_scene_render_depth(C.byref(good), C.byref(cam.c), fp, 5.0, 0.0, H, out.ctypes.data, None) == 0
    bad = -1
    for s in (bad_type, bad_normal, null_list):
        assert L.nvb_scene_render_depth(C.byref(s), C.byref(cam.c), fp, 5.0, 0.0, H, out.ctypes.data, None) == bad
    assert L.nvb_scene_render_depth(None, C.byref(cam.c), fp, 5.0, 0.0, H, out.ctypes.data, None) == bad
    assert L.nvb_scene_render_depth(C.byref(good), None, fp, 5.0, 0.0, H, out.ctypes.data, None) == bad
    assert L.nvb_scene_render_depth(C.byref(good), C.byref(cam.c), fp, 5.0, 0.0, H, None, None) == bad
    assert L.nvb_scene_render_depth(C.byref(good), C.byref(cam.c), fp, 5.0, 0.0, 5, out.ctypes.data, None) == bad
    xyz = np.zeros((4, 3), F)
    d = np.zeros(4, F)
    assert L.nvb_scene_signed_distance(C.byref(good), xyz.ctypes.data, H, 4, 1.0, d.ctypes.data, None) == 0
    assert L.nvb_scene_signed_distance(C.byref(good), None, H, 4, 1.0, d.ctypes.data, None) == bad
    assert L.nvb_scene_signed_distance(C.byref(good), xyz.ctypes.data, 9, 4, 1.0, d.ctypes.data, None) == bad
    assert L.nvb_scene_signed_distance(C.byref(bad_normal), xyz.ctypes.data, H, 4, 1.0, d.ctypes.data, None) == bad
    import torch
    tx, td = torch.zeros((24, 32), dtype=torch.float32, device="cuda"), torch.zeros((24, 32), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert L.nvb_scene_render_depth(C.byref(good), C.byref(cam.c), fp, 5.0, 0.0, 2, td.data_ptr(), None) == bad
    assert L.nvb_scene_signed_distance(C.byref(good), tx.data_ptr(), 2, 4, 1.0, td.data_ptr(), None) == bad
    m = nvb.Mapper(0.1)
    for lid in (lib.NVB_LAYER_ESDF, lib.NVB_LAYER_COLOR, lib.NVB_LAYER_FREESPACE, lib.NVB_LAYER_OCCUPANCY, 42):
        assert L.nvb_scene_generate_layer(m._h, lid, C.byref(good), 0.4) == bad, lid
    assert L.nvb_scene_generate_layer(None, lib.NVB_LAYER_TSDF, C.byref(good), 0.4) == bad
    assert L.nvb_scene_generate_layer(m._h, lib.NVB_LAYER_TSDF, None, 0.4) == bad
    assert L.nvb_scene_generate_layer(m._h, lib.NVB_LAYER_TSDF, C.byref(bad_type), 0.4) == bad
    assert L.nvb_scene_to_mapper(None, C.byref(good)) == bad
    assert L.nvb_scene_to_mapper(m._h, C.byref(bad_normal)) == bad
    assert m.tsdf_layer().num_blocks() == 0
    assert L.nvb_scene_generate_layer(m._h, lib.NVB_LAYER_TSDF, C.byref(good), 0.4) == 0
    assert L.nvb_scene_to_mapper(m._h, C.byref(good)) == 0


def test_append_a_disjoint_scene_to_a_mapper_with_small_slabs(gpu):
    """Frames over one region, then a scene whose blocks lie elsewhere: the ESDF, colour, mesh and freespace layers keep the
    frames' blocks while the projective layer holds only the scene's, so their slabs must hold both. The ESDF of the scene's
    blocks equals the oracle's, and later updates, colour and mesh keep working."""
    nvb = _nvb()
    room = _sc().getSphereInBox()
    cam, ocam = _cams(160, 120, 75.0)
    m = nvb.Mapper(0.2, tsdf_capacity_blocks=512, esdf_capacity_blocks=512,
                   projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)
    for T in circle_poses(4):
        m.integrate_depth(room.render_depth(cam, T, 20.0), T, cam)
        m.integrate_color(np.full((120, 160, 3), 200, np.uint8), T, cam)
        m.update_esdf()
        m.update_mesh()
        m.update_freespace(1000)
    old_esdf = set(m.esdf_layer().as_dict())
    assert len(old_esdf) > 200
    far = _sc().Scene()  # 8 x 8 x 7 = 448 blocks of 1.6 m, 100 m away from the room
    far.set_aabb([100.1, 0.1, 0.1], [111.9, 12.7, 11.1])
    far.add_primitive("sphere", [106.4, 6.4, 5.6, 3.0])
    far.add_ground_level(2.0)
    far.append_to_mapper(m)
    scene_blocks = {tuple(b) for b in sr.blocks_touched(m.block_size(), sr.aabb_of(far)).tolist()}
    assert len(scene_blocks) == 448 and not scene_blocks & old_esdf
    assert set(m.tsdf_layer().as_dict()) == scene_blocks
    esdf = m.esdf_layer().as_dict()
    assert set(esdf) == old_esdf | scene_blocks
    o = _orc().OracleMap(0.2)
    layer = m.tsdf_layer().as_dict()
    for k, v in layer.items():
        o.set_tsdf_block(k, v)
    o.integrate_esdf(np.array(sorted(layer), np.int32))
    assert_esdf_equal({k: esdf[k] for k in scene_blocks}, o.esdf_layer())
    # the frames' region again, then every consumer
    for T in circle_poses(2, 3.0, 1.5):
        m.integrate_depth(room.render_depth(cam, T, 20.0), T, cam)
        m.integrate_color(np.full((120, 160, 3), 100, np.uint8), T, cam)
    m.update_esdf()
    m.update_mesh()
    m.update_freespace(2000)
    assert scene_blocks <= set(m.esdf_layer().as_dict())


def test_device_outputs_do_not_wait_for_the_stream(gpu):
    """With device outputs, the depth and distance calls return while earlier work on the caller's stream still runs: the
    primitives' copy and the launch are only enqueued."""
    import time
    import torch
    s = dummy()
    cam, _ = _cams(320, 240, 150.0)
    T = circle_poses(1)[0]
    pts = torch.zeros((1000, 3), dtype=torch.float32, device="cuda")
    s.render_depth(cam, T, 20.0, device=0)  # module loads and the memory pool, outside the timed calls
    torch.cuda.synchronize()
    for call in (lambda: s.render_depth(cam, T, 20.0, device=0), lambda: s.signed_distance(pts, 1.0)):
        torch.cuda._sleep(2_000_000_000)  # about a second of GPU time on the current stream
        t0 = time.perf_counter()
        call()
        returned = time.perf_counter() - t0
        pending = not torch.cuda.current_stream().query()
        torch.cuda.synchronize()
        assert pending and returned < 0.2, returned


def test_scene_dropin_runs(gpu, tmp_path):
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_scene_dropin")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
