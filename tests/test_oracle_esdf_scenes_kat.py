"""The oracle's ESDF (3-D and 2-D slice, with and without the freespace layer) on the reference's parameterised obstacle
scenes: tests/test_esdf_integrator.cpp SingleEsdfTestGPU (:511-552), AllFreespaceTest (:595-652), ActualFreespaceTest (:654-713),
with its compareEsdfToGt / compareEsdfToEsdf / validateEsdf checks (:238-460) vectorised."""
import numpy as np
import pytest

from helpers import tsdf_layer_from_distance, validate_esdf
from oracle import oracle as orc

VOXEL, MAX_DIST = 0.1, 4.0
VERY_SMALL_CUTOFF = 2e-3
SLICE = dict(z_min_m=1.0, z_max_m=3.0, z_output_m=2.0)


def _room(P):
    x, y, z = P[..., 0], P[..., 1], P[..., 2]
    return np.minimum.reduce([z, 5.0 - z, x + 5.0, 5.0 - x, y + 5.0, 5.0 - y])


def _cube(P, center, size):
    q = np.abs(P - np.asarray(center, float)) - np.asarray(size, float) / 2.0
    return np.linalg.norm(np.maximum(q, 0.0), axis=-1) + np.minimum(np.max(q, axis=-1), 0.0)


_N45 = np.float32(1.0) / np.sqrt(np.float32(2.0))

# addParameterizedObstacleToScene (:105-147): (signed distance, AABB)
BIG, SMALL = ((-5.5, -5.5, -0.5), (5.5, 5.5, 5.5)), ((-3.0, -3.0, 0.0), (3.0, 3.0, 3.0))
OBSTACLES = {
    "axis_aligned_plane": (lambda P: -(P[..., 0] - 0.05), SMALL),
    # Plane::getDistanceToPoint = (p - center) . normal with normal = Vector3f(1, 1, 0).normalized(), in binary32 and Eigen's
    # a0 + (a1 + a2) order: which on-plane voxels come out <= 0 (inside, hence sites) depends on exactly this rounding
    "angled_plane": (lambda P: P[..., 0] * _N45 + (P[..., 1] * _N45 + P[..., 2] * np.float32(0.0)), SMALL),
    "sphere_origin": (lambda P: np.linalg.norm(P, axis=-1) - 2.0, SMALL),
    "box": (_room, BIG),
    "box_with_sphere": (lambda P: np.minimum(_room(P), np.linalg.norm(P - (0.0, 0.0, 2.0), axis=-1) - 2.0), BIG),
    "box_with_cube": (lambda P: np.minimum(_room(P), _cube(P, (0.0, 0.0, 2.0), (2.0, 2.0, 2.0))), BIG),
}


def _freespace_blocks(distance_fn, aabb):
    """generateLayerFromScene<FreespaceVoxel> (scene_impl.h:56-103): high-confidence freespace where no object reaches into the
    voxel (distance > half the body diagonal); voxels outside the AABB stay default (not freespace)."""
    idx, vox = tsdf_layer_from_distance(distance_fn, aabb[0], aabb[1], VOXEL, 1e9)
    fs = np.zeros(vox.shape, orc.FREESPACE_VOXEL_DTYPE)
    fs["is_high_confidence_freespace"] = ((vox["distance"] > np.sqrt(3.0) * VOXEL / 2.0) & (vox["weight"] > 0)).astype(np.uint8)
    return idx, fs


def _map(idx, tsdf, fs=None):
    m = orc.OracleMap(VOXEL)
    for k, v in zip(idx, tsdf):
        m.set_tsdf_block(k, v)
    if fs is not None:
        for k, v in zip(idx, fs):
            m.set_freespace_block(k, v)
    return m


def _dense(layer, fields):
    keys = np.array(list(layer))
    lo, hi = keys.min(0), keys.max(0)
    shape = tuple((hi - lo + 1) * 8)
    out = {f: np.zeros(shape + (() if f != "parent_direction" else (3,)), layer[tuple(keys[0])][f].dtype) for f in fields}
    have = np.zeros(shape, bool)
    for k, blk in layer.items():
        o = (np.asarray(k) - lo) * 8
        sl = (slice(o[0], o[0] + 8), slice(o[1], o[1] + 8), slice(o[2], o[2] + 8))
        have[sl] = True
        for f in fields:
            out[f][sl] = blk[f]
    return lo, have, out


def _signed(d):
    dist = VOXEL * np.sqrt(d["squared_distance_vox"].astype(np.float32))
    return np.where(d["is_inside"].astype(bool), -dist, dist)


@pytest.mark.parametrize("name", list(OBSTACLES))
def test_single_esdf_against_ground_truth(name):
    """SingleEsdfTestGPU (:511-552): ESDF of the ground-truth TSDF vs the ground-truth SDF up to the maximum distance: at most
    0.2 % of the observed voxels are off by more than one voxel."""
    fn, aabb = OBSTACLES[name]
    idx, tsdf = tsdf_layer_from_distance(fn, aabb[0], aabb[1], VOXEL, 4 * VOXEL)
    _, gt = tsdf_layer_from_distance(fn, aabb[0], aabb[1], VOXEL, MAX_DIST)
    m = _map(idx, tsdf)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    m.integrate_esdf(idx, ep)
    layer = m.esdf_layer()
    n_obs, n_site = validate_esdf(layer, (MAX_DIST / VOXEL) ** 2)
    assert n_obs > 100000 and n_site > 1000
    gt_layer = {tuple(int(c) for c in k): v for k, v in zip(idx, gt)}
    over = total = 0
    for k, blk in layer.items():
        obs = blk["observed"].astype(bool)
        diff = np.abs(_signed(blk) - gt_layer[k]["distance"])
        over += int((obs & (diff > VOXEL)).sum())
        total += int(obs.sum())
    assert over / total <= VERY_SMALL_CUTOFF, (over, total)


@pytest.mark.parametrize("name", list(OBSTACLES))
def test_all_freespace(name):
    """AllFreespaceTest (:595-652): with every voxel high-confidence freespace nothing is a site: the ESDF (3-D and slice)
    equals the empty scene's ground truth, the maximum distance everywhere."""
    fn, aabb = OBSTACLES[name]
    idx, tsdf = tsdf_layer_from_distance(fn, aabb[0], aabb[1], VOXEL, 4 * VOXEL)
    _, fs = _freespace_blocks(lambda P: np.full(P.shape[:-1], 1e3), BIG)
    idx_fs, _ = tsdf_layer_from_distance(lambda P: np.full(P.shape[:-1], 1e3), BIG[0], BIG[1], VOXEL, 1.0)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    for sliced in (False, True):
        m = _map(idx, tsdf)
        for k, v in zip(idx_fs, fs):
            m.set_freespace_block(k, v)
        if sliced:
            m.integrate_esdf_slice(idx, ep, use_freespace=True, **SLICE)
        else:
            m.integrate_esdf_with_freespace(idx, ep)
        layer = m.esdf_layer()
        n_obs, n_site = validate_esdf(layer, (MAX_DIST / VOXEL) ** 2)
        assert n_obs > 1000 and n_site == 0
        for blk in layer.values():
            obs = blk["observed"].astype(bool)
            assert np.all(np.abs(_signed(blk)[obs] - MAX_DIST) <= VOXEL)  # compareEsdfToGt against the empty scene


@pytest.mark.parametrize("name", list(OBSTACLES))
def test_actual_freespace(name):
    """ActualFreespaceTest (:654-713): with the scene's own freespace layer the ESDF (3-D and slice) stays within 1.5 voxels of
    the one computed without it for all but 0.2 % of the observed voxels."""
    fn, aabb = OBSTACLES[name]
    idx, tsdf = tsdf_layer_from_distance(fn, aabb[0], aabb[1], VOXEL, 4 * VOXEL)
    _, fs = _freespace_blocks(fn, aabb)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    for sliced in (False, True):
        plain, withfs = _map(idx, tsdf), _map(idx, tsdf, fs)
        if sliced:
            plain.integrate_esdf_slice(idx, ep, **SLICE)
            withfs.integrate_esdf_slice(idx, ep, use_freespace=True, **SLICE)
        else:
            plain.integrate_esdf(idx, ep)
            withfs.integrate_esdf_with_freespace(idx, ep)
        a, b = withfs.esdf_layer(), plain.esdf_layer()
        validate_esdf(a, (MAX_DIST / VOXEL) ** 2)
        over = total = 0
        for k, blk in a.items():
            if k not in b:
                continue
            obs = blk["observed"].astype(bool)
            over += int((obs & (np.abs(_signed(blk) - _signed(b[k])) > 1.5 * VOXEL)).sum())
            total += int(obs.sum())
        assert total > 1000 and over / total <= VERY_SMALL_CUTOFF, (sliced, over, total)


SMALL_CUTOFF = 2e-2  # small_cutoff_ (:79)


def _compare_esdf(a, b, threshold, negative=True):
    """compareEsdfToEsdf (:287-338): fraction of a's observed voxels that differ from b's by more than threshold."""
    over = total = 0
    for k, blk in a.items():
        if k not in b:
            continue
        obs = blk["observed"].astype(bool)
        ref = _signed(b[k])
        if not negative:
            obs = obs & (ref >= 0.0)
        over += int((obs & (np.abs(_signed(blk) - ref) > threshold)).sum())
        total += int(obs.sum())
    return over / max(total, 1), total


def _set_tsdf(m, idx, vox):
    for k, v in zip(idx, vox):
        m.set_tsdf_block(k, v)


@pytest.mark.parametrize("name", ["box", "box_with_sphere", "box_with_cube"])
@pytest.mark.parametrize("thin", [False, True])
def test_incremental_esdf_with_object_removal(name, thin):
    """IncrementalEsdfWithObjectRemoval (:1060-1117) and IncrementalEsdf2DWithObjectRemoval (:901-962, a one-voxel-thick layer at
    z = 1 m): the obstacle disappears from the ground-truth TSDF between two ESDF updates over all blocks; the incremental
    result matches a batch ESDF of the final TSDF within one voxel for all but 2 % of the observed voxels."""
    fn, aabb = OBSTACLES[name]
    if thin:
        aabb = ((-5.5, -5.5, float(np.float32(1.0) - np.float32(VOXEL) / np.float32(2.0))),
                (5.5, 5.5, float(np.float32(1.0) + np.float32(VOXEL) / np.float32(2.0))))
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    m = orc.OracleMap(VOXEL)
    for scene_fn in (fn, _room):
        idx, tsdf = tsdf_layer_from_distance(scene_fn, aabb[0], aabb[1], VOXEL, MAX_DIST)
        _set_tsdf(m, idx, tsdf)
        m.integrate_esdf(idx, ep)
    batch = _map(idx, tsdf)
    batch.integrate_esdf(idx, ep)
    inc = m.esdf_layer()
    frac, total = _compare_esdf(inc, batch.esdf_layer(), VOXEL)
    assert total > 5000 and frac <= SMALL_CUTOFF, (frac, total)
    validate_esdf(inc, (MAX_DIST / VOXEL) ** 2)
    if name != "box":  # the obstacle's sites are really gone
        obstacle_only = fn(np.array([[0.0, 0.0, 2.0]], np.float32))[0] < 0
        assert obstacle_only


@pytest.mark.parametrize("name", ["box", "box_with_sphere", "box_with_cube"])
def test_incremental_esdf_slice_with_object_removal(name):
    """IncrementalEsdfSliceWithObjectRemovalGPU (:964-1058): a thin ground-truth layer at 1.5 m, sliced (band 1..2 m, output
    1.5 m) from the TSDF and from the occupancy layer, before and after the obstacle is removed; against the batch 3-D ESDF of the
    final TSDF: within one voxel (TSDF) / 1.5 voxels on non-negative distances (occupancy) for all but 2 %."""
    fn, _ = OBSTACLES[name]
    h = 1.5
    aabb = ((-5.5, -5.5, float(np.float32(h) - np.float32(VOXEL) / np.float32(2.0))),
            (5.5, 5.5, float(np.float32(h) + np.float32(VOXEL) / np.float32(2.0))))
    sl = dict(z_min_m=1.0, z_max_m=2.0, z_output_m=h)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    mt, mo = orc.OracleMap(VOXEL), orc.OracleMap(VOXEL)
    hi, lo = np.float32(np.inf), np.float32(-np.inf)  # logOddsFromProbability(1), (0) (scene_impl.h:48-50)
    for scene_fn in (fn, _room):
        idx, tsdf = tsdf_layer_from_distance(scene_fn, aabb[0], aabb[1], VOXEL, 4 * VOXEL)
        _, full = tsdf_layer_from_distance(scene_fn, aabb[0], aabb[1], VOXEL, 1e9)
        _set_tsdf(mt, idx, tsdf)
        for k, v in zip(idx, full):
            occ = np.where(v["weight"] > 0, np.where(v["distance"] <= np.sqrt(3.0) * VOXEL / 2.0, hi, lo), np.float32(0.0))
            mo.set_occupancy_block(k, occ.astype(np.float32))
        mt.integrate_esdf_slice(idx, ep, **sl)
        mo.integrate_esdf_slice(idx, ep, from_occupancy=True, **sl)
    batch = _map(idx, tsdf)
    batch.integrate_esdf(idx, ep)
    b = batch.esdf_layer()
    frac, total = _compare_esdf(mt.esdf_layer(), b, VOXEL)
    assert total > 5000 and frac <= SMALL_CUTOFF, (frac, total)
    frac, total = _compare_esdf(mo.esdf_layer(), b, 1.5 * VOXEL, negative=False)
    assert total > 5000 and frac <= SMALL_CUTOFF, (frac, total)
    validate_esdf(mt.esdf_layer(), (MAX_DIST / VOXEL) ** 2)
    validate_esdf(mo.esdf_layer(), (MAX_DIST / VOXEL) ** 2)


def test_slice_image_of_an_empty_layer():
    """sliceLayerToDistanceImage_emptyLayer (:794-806): no blocks at the height -> empty AABB, 0 x 0 image."""
    m = orc.OracleMap(VOXEL)
    aabb, img, grid = m.esdf_slice_image(1.0)
    assert img.size == 0 and grid.size == 0


def _syn_scene(name):
    from isaac_ros_nvblox_b200 import synthetic as syn
    s = syn.Scene()
    s.add_plane(2, 0.0).add_plane(2, 5.0).add_plane(0, -5.0).add_plane(0, 5.0).add_plane(1, -5.0).add_plane(1, 5.0)
    if name == "box_with_sphere":
        s.add_sphere((0.0, 0.0, 2.0), 2.0)
    elif name == "box_with_cube":
        s.add_box((-1.0, -1.0, 1.0), (1.0, 1.0, 3.0))
    return s


@pytest.mark.parametrize("name", ["box_with_sphere", "box_with_cube"])
def test_complex_scene_with_tsdf(name):
    """ComplexSceneWithTsdf (:715-792): 80 rendered views on the circle integrated into the TSDF (max distance 15 m), one
    ESDF over all blocks: at most 30 % of the observed voxels are further than 4 voxels from the ground truth; validateEsdf."""
    from isaac_ros_nvblox_b200 import synthetic as syn
    fn, aabb = OBSTACLES[name]
    cs = syn.PinholeCamera(300.0, 300.0, 320.0, 240.0, 640, 480)
    cam = orc.Camera(300.0, 300.0, 320.0, 240.0, 640, 480)
    scene = _syn_scene(name)
    m = orc.OracleMap(VOXEL)
    tp = orc.default_tsdf_params(max_integration_distance_m=15.0)
    for T in syn.circle_trajectory(80)[::2]:  # every other pose of the reference's 80: same coverage, half the time
        m.integrate_depth(syn.render_depth(scene, cs, T, max_dist=15.0), T, cam, tp)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    m.integrate_esdf(m.tsdf_block_indices(), ep)
    layer = m.esdf_layer()
    validate_esdf(layer, (MAX_DIST / VOXEL) ** 2)
    idx, gt = tsdf_layer_from_distance(fn, aabb[0], aabb[1], VOXEL, MAX_DIST)
    gt_layer = {tuple(int(c) for c in k): v for k, v in zip(idx, gt)}
    over = total = 0
    for k, blk in layer.items():
        if k not in gt_layer:
            continue
        obs = blk["observed"].astype(bool)
        over += int((obs & (np.abs(_signed(blk) - gt_layer[k]["distance"]) > 4 * VOXEL)).sum())
        total += int(obs.sum())
    assert total > 100000 and over / total <= 0.30, (over, total)


@pytest.mark.parametrize("name", ["box_with_sphere", "box_with_cube"])
def test_incremental_tsdf_and_esdf_with_object_removal(name):
    """IncrementalTsdfAndEsdfWithObjectRemovalGPU (:808-899): one view with the obstacle, the same view without it, an ESDF update
    on each frame's updated blocks; vs a batch ESDF of the final TSDF: within one voxel for all but 2 %."""
    from isaac_ros_nvblox_b200 import synthetic as syn
    cs = syn.PinholeCamera(300.0, 300.0, 320.0, 240.0, 640, 480)
    cam = orc.Camera(300.0, 300.0, 320.0, 240.0, 640, 480)
    tp = orc.default_tsdf_params(max_integration_distance_m=15.0)
    ep = orc.default_esdf_params(max_esdf_distance_m=MAX_DIST, min_weight=1.0)
    m = orc.OracleMap(VOXEL)
    poses = syn.circle_trajectory(1)  # kNumTrajectoryPoints = 1: theta = 0 for both frames
    for i, scene in enumerate((_syn_scene(name), _syn_scene("box"))):
        T = poses[0]
        b = m.integrate_depth(syn.render_depth(scene, cs, T, max_dist=15.0), T, cam, tp)
        m.integrate_esdf(b, ep)
    batch = orc.OracleMap(VOXEL)
    for k, v in m.tsdf_layer().items():
        batch.set_tsdf_block(k, v)
    batch.integrate_esdf(m.tsdf_block_indices(), ep)
    frac, total = _compare_esdf(m.esdf_layer(), batch.esdf_layer(), VOXEL)
    assert total > 1000 and frac <= SMALL_CUTOFF, (frac, total)  # (min_weight = 1 leaves only the voxels near the camera)
    validate_esdf(m.esdf_layer(), (MAX_DIST / VOXEL) ** 2)
