"""The ground-plane estimator on the GPU (GroundPlaneEstimator, experimental/ground_plane/) against its numpy restatement
(tests/ground_plane_reference.py): zero crossings and ground candidates equal bit for bit and in order, planes and found
flags bit for bit, the estimator's state after each failure mode, and the 2-D ESDF on the estimated plane against the oracle."""
import numpy as np
import pytest

import ground_plane_reference as gpr
from helpers import assert_esdf_equal, cameras, tsdf_layer_from_distance
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

WIDE_Z = dict(ground_points_candidates_min_z_m=-1e9, ground_points_candidates_max_z_m=1e9)


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _mapper_with_layer(voxel_size, idx, vox, **kw):
    m = _nvb().Mapper(voxel_size, **kw)
    if len(idx):
        m.tsdf_layer().set_blocks(idx, vox)
    return m


def _layer_dict(idx, vox):
    return {tuple(int(v) for v in k): b for k, b in zip(idx, vox)}


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check_estimator(m, layer, voxel_size, **params):
    """compute_ground_plane on the GPU vs gpr.estimate on the same layer: plane, crossings and candidates bit for bit."""
    est = m.ground_plane_estimator()
    p = est.params(**params)
    plane = est.compute_ground_plane()
    r_plane, r_cross, r_cand = gpr.estimate(layer, voxel_size, min_z=p["ground_points_candidates_min_z_m"],
                                            max_z=p["ground_points_candidates_max_z_m"],
                                            ransac_distance_threshold_m=p["ransac_distance_threshold_m"],
                                            num_ransac_iterations=p["num_ransac_iterations"],
                                            min_tsdf_weight=p["min_tsdf_weight"], max_crossings=p["max_crossings"])
    assert (plane is None) == (r_plane is None)
    if r_plane is None:
        assert est.ground_plane() is None and est.tsdf_zero_crossings() is None
        assert est.tsdf_zero_crossings_ground_candidates() is None
        return None, None
    assert np.array_equal(_bits(plane), _bits(r_plane)), (plane, r_plane)
    assert np.array_equal(_bits(est.ground_plane()), _bits(r_plane))
    cr, cand = est.tsdf_zero_crossings(), est.tsdf_zero_crossings_ground_candidates()
    assert cr.shape == r_cross.shape and np.array_equal(_bits(cr), _bits(r_cross))
    assert cand.shape == r_cand.shape and np.array_equal(_bits(cand), _bits(r_cand))
    return plane, cr


def _plane_layer(z, voxel_size=0.1, aabb=((0.0, 0.0, -2.0), (0.2, 0.2, 2.0))):
    return tsdf_layer_from_distance(lambda P: P[..., 2] - z, aabb[0], aabb[1], voxel_size, 1.0)


@pytest.mark.parametrize("z", [-1.0, 0.04])
def test_reference_plane_scenes(gpu, z):
    """ZeroCrossingsFromAboveSimplePlane / ...AtBoundary (test_zero_crossings_extractor.cu): four crossings at the voxel
    centres' x, y and the plane's z."""
    idx, vox = _plane_layer(z)
    m = _mapper_with_layer(0.1, idx, vox)
    _, cr = _check_estimator(m, _layer_dict(idx, vox), 0.1, **WIDE_Z)
    assert len(cr) == 4
    assert np.allclose(cr, [[0.05, 0.05, z], [0.05, 0.15, z], [0.15, 0.05, z], [0.15, 0.15, z]], atol=1e-6)
    m.close()


def test_reference_sphere_scene(gpu):
    """ZeroCrossingsFromAboveSimpleSphere: r = 0.1 at the origin; the four crossings near z = 0.0707 (tolerance 0.004)."""
    idx, vox = tsdf_layer_from_distance(lambda P: np.linalg.norm(P, axis=-1) - 0.1, (-0.5, -0.5, -0.5), (0.5, 0.5, 0.5), 0.1, 1.0)
    m = _mapper_with_layer(0.1, idx, vox)
    _, cr = _check_estimator(m, _layer_dict(idx, vox), 0.1, **WIDE_Z)
    assert len(cr) == 4
    assert np.allclose(np.abs(cr[:, :2]), 0.05, atol=1e-6) and np.allclose(cr[:, 2], 0.07071, atol=0.004)
    m.close()


def test_state_cleared_after_success(gpu):
    """After a plane was found: a map cleared to no blocks, then a map whose candidates are collinear (every RANSAC sample
    degenerate) give no plane, and the crossings, candidates and plane are all cleared."""
    idx, vox = _plane_layer(0.0, aabb=((-1.0, -1.0, -0.5), (1.0, 1.0, 0.5)))
    m = _mapper_with_layer(0.1, idx, vox)
    est = m.ground_plane_estimator()
    assert _check_estimator(m, _layer_dict(idx, vox), 0.1)[0] is not None
    m.clear()
    assert est.compute_ground_plane() is None
    assert est.ground_plane() is None and est.tsdf_zero_crossings() is None and est.tsdf_zero_crossings_ground_candidates() is None
    assert _check_estimator(m, {}, 0.1) == (None, None)
    m.tsdf_layer().set_blocks(idx, vox)
    assert _check_estimator(m, _layer_dict(idx, vox), 0.1)[0] is not None
    m.clear()
    line_idx, line_vox = _plane_layer(0.0, aabb=((0.0, 0.0, -0.5), (0.08, 0.8, 0.5)))  # one voxel column wide: a line
    line = _layer_dict(line_idx, line_vox)
    assert len(gpr.zero_crossings(line, 0.1)) >= 3 and gpr.estimate(line, 0.1)[0] is None
    m.tsdf_layer().set_blocks(line_idx, line_vox)
    assert _check_estimator(m, line, 0.1) == (None, None)
    m.close()


def test_max_crossings_edges_and_empty(gpu):
    """count >= max_crossings gives no plane and clears the state; count == max_crossings - 1 gives one; an empty layer
    and an occupancy mapper give none."""
    idx, vox = _plane_layer(0.0, aabb=((-1.0, -1.0, -0.5), (1.0, 1.0, 0.5)))
    layer = _layer_dict(idx, vox)
    n = len(gpr.zero_crossings(layer, 0.1))
    assert n > 100
    m = _mapper_with_layer(0.1, idx, vox)
    est = m.ground_plane_estimator()
    assert est.compute_ground_plane() is not None and est.tsdf_zero_crossings() is not None
    _check_estimator(m, layer, 0.1, max_crossings=n)  # not found
    assert est.ground_plane() is None and est.tsdf_zero_crossings_ground_candidates() is None
    plane, cr = _check_estimator(m, layer, 0.1, max_crossings=n + 1)
    assert plane is not None and len(cr) == n
    # fewer than three candidates: not found, state cleared
    _check_estimator(m, layer, 0.1, ground_points_candidates_min_z_m=5.0, ground_points_candidates_max_z_m=6.0)
    m.close()
    empty = _nvb().Mapper(0.1)
    assert empty.ground_plane_estimator().compute_ground_plane() is None
    assert empty.ground_plane_estimator().tsdf_zero_crossings() is None
    empty.close()
    occ = _nvb().Mapper(0.1, projective_layer_type=_nvb().ProjectiveLayerType.kOccupancy)
    assert occ.ground_plane_estimator().compute_ground_plane() is None
    occ.close()


def _tilted_sequence(n_frames=12, deg=4.0):
    """sphere_in_box seen through poses premultiplied by a fixed rotation about x and an offset: in the map frame the
    ground is tilted by `deg` and passes near z = 0 under the trajectory."""
    a = np.deg2rad(deg)
    G = np.eye(4)
    G[:3, :3] = [[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]]
    G[:3, 3] = [0.3, -0.2, 0.05]
    cs, cam, ocam = cameras(320, 240)
    poses = syn.circle_trajectory(40)[:n_frames]
    frames = syn.make_sequence(syn.sphere_in_box(), cs, poses)
    return [(d, (G @ T).astype(np.float32)) for d, T in frames], cam, ocam, G


def test_integrated_tilted_ground(gpu):
    frames, cam, _, G = _tilted_sequence()
    m = _nvb().Mapper(0.05)
    for d, T in frames:
        m.integrate_depth(d, T, cam)
    plane, cr = _check_estimator(m, m.tsdf_layer().as_dict(), 0.05)
    assert plane is not None and len(cr) > 1000
    n = np.asarray(plane[:3], np.float64) * np.sign(plane[2])
    assert np.abs(n - G[:3, 2]).max() < 1e-3, (n, G[:3, 2])  # sanity: the tilt, not a parity check
    m.close()


def test_two_cm_map_many_blocks(gpu):
    idx, vox = tsdf_layer_from_distance(lambda P: P[..., 2] - 0.013 * P[..., 0] - 0.004, (-3.6, -3.6, -0.4), (3.6, 3.6, 0.4), 0.02,
                                        0.08)
    assert len(idx) > 10000
    m = _mapper_with_layer(0.02, idx, vox)
    plane, cr = _check_estimator(m, _layer_dict(idx, vox), 0.02)
    assert plane is not None and len(cr) > 50000
    m.close()


def test_far_from_origin(gpu):
    idx, vox = tsdf_layer_from_distance(lambda P: P[..., 2] - 0.02, (300.0, 300.0, -0.5), (302.0, 302.5, 0.5), 0.05, 0.2)
    m = _mapper_with_layer(0.05, idx, vox)
    plane, _ = _check_estimator(m, _layer_dict(idx, vox), 0.05)
    assert plane is not None
    m.close()


def _fit_both(points, iterations, threshold=0.2, mapper=None):
    g = _nvb().ransac_fit_plane(points, iterations, threshold, mapper=mapper)
    r = gpr.ransac_fit(points, iterations, threshold)
    assert (g is None) == (r is None)
    if r is not None:
        assert np.array_equal(_bits(g), _bits(r)), (g, r)
    return g


def test_fit_small_sets(gpu):
    """RansacPlaneFitter cases: no points, two points, duplicates only, collinear points, three points."""
    assert _fit_both(np.zeros((0, 3), np.float32), 1000) is None
    assert _fit_both(np.array([[0, 0, 0], [1, 0, 0]], np.float32), 1000) is None
    assert _fit_both(np.ones((50, 3), np.float32), 1000) is None
    t = np.linspace(0, 1, 40, dtype=np.float32)
    assert _fit_both(np.stack([t, 2 * t, 3 * t], 1).astype(np.float32), 1000) is None
    assert _fit_both(np.array([[0, 0, 1], [1, 0, 1], [0, 1, 1]], np.float32), 1000) is not None


def _plane_with_outliers(n_plane, n_out, seed=0):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-5, 5, (n_plane, 2))
    plane_pts = np.column_stack([xy, 0.02 * xy[:, 0] - 0.01 * xy[:, 1] + 0.1])
    return np.vstack([plane_pts, rng.normal(0.0, 2.0, (n_out, 3))]).astype(np.float32)[rng.permutation(n_plane + n_out)]


@pytest.mark.parametrize("iterations,n", [(1, 6000), (1000, 6000), (5003, 20000)])
def test_fit_iterations(gpu, iterations, n):
    _fit_both(_plane_with_outliers(n * 5 // 6, n // 6), iterations)


def test_fit_large_and_growing_iterations(gpu):
    """~300 k points; then a second mapper whose iteration count grows between fits (cached states extended)."""
    pts = _plane_with_outliers(250000, 50000, seed=1)
    assert _fit_both(pts, 1000) is not None
    m = _nvb().Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    small = pts[:5000]
    for it in (10, 1000, 37, 2000):
        _fit_both(small, it, mapper=m)
    m.close()


def test_fit_device_points(gpu):
    """CUDA tensors: float32 contiguous; float64, strided and just computed on torch's stream (the conversion and the
    producing kernels must be complete before the mapper's stream reads the points); a CPU tensor is refused."""
    import torch
    pts = _plane_with_outliers(250000, 50000, seed=2)
    want = gpr.ransac_fit(pts, 1000)
    assert np.array_equal(_bits(_nvb().ransac_fit_plane(torch.from_numpy(pts).cuda(), 1000)), _bits(want))
    base = torch.from_numpy(pts.astype(np.float64)).cuda()
    for _ in range(3):
        fresh = (torch.cat([base * 4.0, torch.ones_like(base)], dim=1) / 4.0)[:, :3]  # exact, float64, a strided view
        assert fresh.dtype == torch.float64 and not fresh.is_contiguous()
        assert np.array_equal(_bits(_nvb().ransac_fit_plane(fresh, 1000)), _bits(want))
    with pytest.raises(ValueError):
        _nvb().ransac_fit_plane(torch.from_numpy(pts), 1000)


@pytest.mark.parametrize("ltype", ["tsdf", "occupancy"])
def test_planar_slice_on_estimated_plane(gpu, ltype):
    """The 2-D ESDF on the estimated plane equals the oracle's planar slice on the reference's estimated plane; an
    occupancy mapper has no plane and keeps the constant-z slice."""
    from oracle import oracle as orc
    nvb = _nvb()
    frames, cam, ocam, _ = _tilted_sequence(6)
    kind = nvb.ProjectiveLayerType.kTsdf if ltype == "tsdf" else nvb.ProjectiveLayerType.kOccupancy
    m, o = nvb.Mapper(0.05, projective_layer_type=kind), orc.OracleMap(0.05)
    m.esdf_integrator().slice_params(slice_height_above_plane_m=0.3, slice_height_thickness_m=0.85, slice_height_m=1.0)
    for i, (d, T) in enumerate(frames):
        b = m.integrate_depth(d, T, cam)
        if ltype == "tsdf":
            o.integrate_depth(d, T, ocam)
        else:
            o.integrate_occupancy(d, T, ocam, orc.default_tsdf_params())
        plane = m.ground_plane_estimator().compute_ground_plane()
        blocks = b if i else (o.tsdf_block_indices() if ltype == "tsdf" else o.occupancy_block_indices())
        if ltype == "occupancy":
            assert plane is None
            m.update_esdf_slice()
            o.integrate_esdf_slice(blocks, from_occupancy=True)
        else:
            r_plane = gpr.estimate(o.tsdf_layer(), 0.05)[0]
            assert r_plane is not None and np.array_equal(_bits(plane), _bits(r_plane))
            m.update_esdf_slice(ground_plane=np.asarray(plane, np.float32))
            o.integrate_esdf_slice_planar(blocks, r_plane, above_plane_m=0.3, thickness_m=0.85, z_output_m=1.0)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


def test_ground_plane_dropin_program(gpu, tmp_path):
    """tests/cpp/test_ground_plane_dropin.cpp: MultiMapper with experimental_use_ground_plane_estimation in 2-D, the node's
    two estimator getters, and RansacPlaneFitter::fit on a Pointcloud through the C++ mirror."""
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_ground_plane_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "ground plane drop-in ok" in out.stdout
