"""Parity of the CUDA path (through the C-ABI) with the CPU oracle on identical inputs.

Bars (BASELINE.json north_star): block-index sets/lists bit-exact; float SDF values within
1e-4 (they are in fact bit-identical: same operation order, no FMA on either side);
all five EsdfVoxel fields exact.
"""
import os

import numpy as np
import pytest

from helpers import ESDF_FIELDS, assert_esdf_equal, assert_tsdf_equal, cameras, layer_checksum, sort_rows
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _set_params(m, o_params, **kw):
    m.tsdf_integrator().params(**kw)
    for k, v in kw.items():
        if k in ("workspace_min", "workspace_max"):
            import ctypes as C
            setattr(o_params, k, (C.c_float * 3)(*v))
        else:
            setattr(o_params, k, v)


# ----------------------------------------------------------------------------------------
# View calculation
# ----------------------------------------------------------------------------------------
def test_view_raycast_matches_oracle_in_content_and_order(gpu):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras()
    scene = syn.sphere_in_box()
    m = nvb.Mapper(0.05)
    vc = nvb.ViewCalculator(m)
    for T in syn.circle_trajectory(80)[::9]:
        depth = syn.render_depth(scene, cs, T)
        got = vc.get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
        want = orc.view_raycast(depth, T, ocam, 0.4, 0.2)
        assert len(want) > 1000
        assert np.array_equal(got, want)
    assert m.tsdf_layer().num_blocks() == 0  # the view calculator does not touch the map
    m.close()


@pytest.mark.parametrize("subsample", [1, 2, 3, 4, 7])
def test_view_raycast_subsampling_and_frustum_kat(gpu, subsample):
    """FrustumRayTracingSubsamplingTest.RayTracePixels (tests/test_frustum.cpp:352-416) on the GPU."""
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(0.125)
    if subsample <= 2:
        cam, ocam = nvb.Camera(5.0, 5.0, 1.0, 1.0, 3, 3), orc.Camera(5.0, 5.0, 1.0, 1.0, 3, 3)
        depth = np.full((3, 3), 2.5, np.float32)
        T = np.eye(4, dtype=np.float32)
        T[:3, 3] = [1, 1, 0]
        m.tsdf_integrator().raycast_subsampling_factor(subsample)
        got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 1.0, 0.0, 3.5)
        assert len(got) == 12
        assert set(map(tuple, got)) == {(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1, 2)}
    cs, cam, ocam = cameras(320, 240)
    depth = syn.render_depth(syn.box_with_cube(), cs, syn.circle_pose(0.7))
    m.tsdf_integrator().raycast_subsampling_factor(subsample)
    got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, syn.circle_pose(0.7), cam, 0.4, 0.2, 7.0)
    want = orc.view_raycast(depth, syn.circle_pose(0.7), ocam, 0.4, 0.2, orc.default_tsdf_params(raycast_subsampling=subsample))
    assert np.array_equal(got, want)
    m.close()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 0.0, -1.0])
def test_view_raycast_invalid_depth(gpu, bad):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(160, 120)
    depth = np.full((120, 160), bad, np.float32)
    T = syn.circle_pose(0.3)
    m = nvb.Mapper(0.05)
    got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
    want = orc.view_raycast(depth, T, ocam, 0.4, 0.2)
    assert np.array_equal(got, want)
    m.close()


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (7, 2), (33, 17), (121, 161)])
def test_view_raycast_ragged_images(gpu, shape):
    nvb, orc = _nvb(), _orc()
    h, w = shape
    cam, ocam = nvb.Camera(40.0, 40.0, w / 2.0, h / 2.0, w, h), orc.Camera(40.0, 40.0, w / 2.0, h / 2.0, w, h)
    rng = np.random.default_rng(h * 100 + w)
    depth = rng.uniform(0.5, 6.0, size=shape).astype(np.float32)
    T = syn.circle_pose(1.1)
    m = nvb.Mapper(0.05)
    got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
    want = orc.view_raycast(depth, T, ocam, 0.4, 0.2)
    assert np.array_equal(got, want)
    m.close()


def test_view_raycast_workspace_bounds(gpu):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    T = syn.circle_pose(2.0)
    depth = syn.render_depth(syn.sphere_in_box(), cs, T)
    for kw in (dict(workspace_bounds_type=1, workspace_min=(0, 0, 0.5), workspace_max=(0, 0, 2.5)),
               dict(workspace_bounds_type=2, workspace_min=(-2, -2, 0), workspace_max=(3, 3, 3)),
               dict(workspace_bounds_type=2, workspace_min=(50, 50, 50), workspace_max=(60, 60, 60))):
        m = nvb.Mapper(0.05)
        p = orc.default_tsdf_params()
        _set_params(m, p, **kw)
        got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
        want = orc.view_raycast(depth, T, ocam, 0.4, 0.2, p)
        assert np.array_equal(got.reshape(-1, 3), want.reshape(-1, 3))
        m.close()


# ----------------------------------------------------------------------------------------
# TSDF
# ----------------------------------------------------------------------------------------
def _run_pair(voxel, frames, cam, ocam, esdf=False, tsdf_kw=None, mapper_kw=None, masks=None, mask_mode=0,
              check_every_frame=True):
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(voxel, **(mapper_kw or {}))
    o = orc.OracleMap(voxel)
    p = orc.default_tsdf_params()
    if tsdf_kw:
        _set_params(m, p, **tsdf_kw)
    for i, (depth, T) in enumerate(frames):
        mask = None if masks is None else masks[i]
        b_gpu = m.integrate_depth(depth, T, cam, mask=mask, mask_mode=mask_mode)
        b_cpu = o.integrate_depth(depth, T, ocam, p, mask=mask, mask_mode=mask_mode)
        assert np.array_equal(b_gpu, b_cpu), "updated_blocks of frame %d differ" % i
        if esdf:
            m.update_esdf()
            o.integrate_esdf(b_cpu if i > 0 else o.tsdf_block_indices())
            if check_every_frame:
                assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    if esdf:
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    return m, o


def test_tsdf_sequence_640x480_5cm(gpu):
    cs, cam, ocam = cameras()
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80)[:6])
    m, o = _run_pair(0.05, frames, cam, ocam)
    assert m.tsdf_layer().num_blocks() > 3000
    m.close()


@pytest.mark.parametrize("wtype", [0, 1, 2, 3, 4, 5])
def test_tsdf_all_weighting_functions(gpu, wtype):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(40)[:3], noise_sigma_rel=0.01, seed=3)
    m, _ = _run_pair(0.05, frames, cam, ocam, tsdf_kw=dict(weighting_type=wtype))
    m.close()


def test_tsdf_noise_dropout_and_decay(gpu):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:4], noise_sigma_rel=0.01,
                               dropout=0.13, seed=1)
    m, _ = _run_pair(0.05, frames, cam, ocam, tsdf_kw=dict(invalid_depth_decay_factor=0.8))
    m.close()


@pytest.mark.parametrize("mask_mode", [0, 1])
def test_tsdf_masked_frames(gpu, mask_mode):
    cs, cam, ocam = cameras(320, 240)
    seq = syn.moving_sphere_sequence(cs, syn.circle_trajectory(40)[:3])
    frames = [(d, T) for d, T, _ in seq]
    masks = [mk for _, _, mk in seq]
    m, _ = _run_pair(0.05, frames, cam, ocam, masks=masks, mask_mode=mask_mode)
    m.close()


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 0.0, -10.0])
def test_tsdf_invalid_frames_integrate_nothing(gpu, bad):
    """InvalidDepthHandling (tests/test_tsdf_integrator.cpp:588-722)."""
    cs, cam, ocam = cameras(160, 120)
    T = syn.circle_pose(0.0)
    good = syn.render_depth(syn.sphere_in_box(), cs, T)
    frames = [(good, T), (np.full_like(good, bad), T)]
    m, o = _run_pair(0.05, frames, cam, ocam)
    m.close()


def test_tsdf_max_integration_distance_and_truncation(gpu):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:2])
    m, _ = _run_pair(0.05, frames, cam, ocam, tsdf_kw=dict(max_integration_distance_m=4.0, truncation_distance_vox=2.0,
                                                             max_weight=100.0))
    m.close()


def test_tsdf_2cm_voxels(gpu):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(80)[:2])
    m, _ = _run_pair(0.02, frames, cam, ocam, tsdf_kw=dict(max_integration_distance_m=4.0))
    assert m.tsdf_layer().num_blocks() > 10000
    m.close()


def test_layer_grows_past_initial_capacity(gpu):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:4])
    m, _ = _run_pair(0.05, frames, cam, ocam, esdf=True, mapper_kw=dict(tsdf_capacity_blocks=512, esdf_capacity_blocks=512),
                     check_every_frame=False)
    assert m.tsdf_layer().num_blocks() > 512
    m.close()


def test_async_frames_equal_sync_frames(gpu):
    nvb = _nvb()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:5])
    a, b = nvb.Mapper(0.05), nvb.Mapper(0.05)
    for depth, T in frames:
        a.integrate_depth(depth, T, cam)
        a.update_esdf()
        b.integrate_depth_async(depth, T, cam)
        b.update_esdf(sync=False)
    b.synchronize()
    assert_tsdf_equal(b.tsdf_layer().as_dict(), a.tsdf_layer().as_dict())
    assert_esdf_equal(b.esdf_layer().as_dict(), a.esdf_layer().as_dict())
    a.close(), b.close()


def test_clear_and_reuse(gpu):
    nvb = _nvb()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(40)[:3])
    m = nvb.Mapper(0.05)
    sums = []
    for rep in range(2):
        for depth, T in frames:
            m.integrate_depth(depth, T, cam)
            m.update_esdf()
        sums.append((layer_checksum(m.tsdf_layer().as_dict(), ("distance", "weight")),
                     layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS)))
        m.clear()
        assert m.tsdf_layer().num_blocks() == 0 and m.esdf_layer().num_blocks() == 0
    assert sums[0] == sums[1]
    m.close()


def test_block_round_trip_and_device_pointers(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.05)
    rng = np.random.default_rng(0)
    idx = np.array([[0, 0, 0], [-3, 7, 2], [100000, -100000, 5], [-1, -1, -1]], np.int32)
    vox = np.zeros((4, 8, 8, 8), nvb.TSDF_VOXEL_DTYPE)
    vox["distance"] = rng.normal(size=(4, 8, 8, 8)).astype(np.float32)
    vox["weight"] = rng.uniform(size=(4, 8, 8, 8)).astype(np.float32)
    m.tsdf_layer().set_blocks(idx, vox)
    got, found = m.tsdf_layer().get_blocks(np.vstack([idx, [[9, 9, 9]]]))
    assert found.tolist() == [True, True, True, True, False]
    assert np.array_equal(got[:4], vox) and not got[4]["weight"].any()
    assert sorted(map(tuple, m.tsdf_layer().get_all_block_indices())) == sorted(map(tuple, idx))
    p0, p1 = m.tsdf_layer().block_device_ptr(idx[0]), m.tsdf_layer().block_device_ptr(idx[1])
    assert p0 and p1 and abs(p1 - p0) % 4096 == 0
    assert m.tsdf_layer().block_device_ptr([9, 9, 9]) == 0
    with pytest.raises(Exception):
        m.tsdf_layer().set_blocks(np.array([[1 << 21, 0, 0]], np.int32), vox[:1])
    m.close()


# ----------------------------------------------------------------------------------------
# ESDF
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("persistent", [1, 0, 3])
def test_esdf_incremental_sequence(gpu, persistent):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:5])
    m, o = _run_pair(0.05, frames, cam, ocam, esdf=True, mapper_kw=dict(esdf_persistent=persistent))
    s_gpu, s_cpu = m.esdf_integrator().last_stats(), o.esdf_stats()
    for k in ("marked", "with_sites", "to_clear", "clear_candidates", "cleared", "swept", "face_passes", "rings"):
        assert s_gpu[k] == s_cpu[k], (k, s_gpu, s_cpu)
    m.close()


@pytest.mark.parametrize("switch", [0, 40, 160, 100000])
def test_esdf_gather_replay_wavefront(gpu, monkeypatch, switch):
    """esdf_persistent=2: rings with more than `switch` members run as four-phase rings, the others as gather-replay
    rings (every candidate block replays the six face passes on its one-voxel halo). Same results, bit for bit."""
    monkeypatch.setenv("NVB_GES_SWITCH", str(switch))
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:6], noise_sigma_rel=0.005, seed=11)
    m, o = _run_pair(0.05, frames, cam, ocam, esdf=True, mapper_kw=dict(esdf_persistent=2))
    s_gpu, s_cpu = m.esdf_integrator().last_stats(), o.esdf_stats()
    for k in ("marked", "with_sites", "to_clear", "cleared", "swept", "face_passes", "rings"):
        assert s_gpu[k] == s_cpu[k], (k, s_gpu, s_cpu)
    m.close()


@pytest.mark.parametrize("mode", [2, 3])
def test_esdf_gather_replay_640x480_with_growth(gpu, mode):
    cs, cam, ocam = cameras()
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(80)[:5])
    m, _ = _run_pair(0.05, frames, cam, ocam, esdf=True, check_every_frame=False,
                     mapper_kw=dict(esdf_persistent=mode, tsdf_capacity_blocks=1024, esdf_capacity_blocks=1024))
    m.close()


def test_esdf_exchange_slab_wavefront_noisy_scene_every_frame(gpu):
    """esdf_persistent=3 (one barrier per ring: exchange slabs by ring parity, candidate records, single-CTA tail rings):
    same results and the same per-update statistics as the oracle after every frame of a noisy sequence."""
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:8], noise_sigma_rel=0.005, seed=11)
    m, o = _run_pair(0.05, frames, cam, ocam, esdf=True, mapper_kw=dict(esdf_persistent=3))
    s_gpu, s_cpu = m.esdf_integrator().last_stats(), o.esdf_stats()
    for k in ("marked", "with_sites", "to_clear", "cleared", "swept", "face_passes", "rings"):
        assert s_gpu[k] == s_cpu[k], (k, s_gpu, s_cpu)
    m.close()


@pytest.mark.parametrize("mode", [3, 1, 2, 0])
def test_esdf_hand_derived_order_kats(gpu, mode):
    """tests/esdf_order_cases.py: known answers written down from the reference's source (the scan's "last taker" rule; the
    propagation across a block face with its ring statistics), for every wavefront formulation."""
    from esdf_order_cases import ACROSS_FACE_STATS, across_face_case, check_across_face, check_last_taker, last_taker_case
    nvb = _nvb()
    tsdf, esdf, expected = last_taker_case(nvb.TSDF_VOXEL_DTYPE, nvb.ESDF_VOXEL_DTYPE)
    m = nvb.Mapper(0.05, esdf_persistent=mode)
    idx = np.array(list(tsdf), np.int32)
    m.tsdf_layer().set_blocks(idx, np.stack([tsdf[tuple(k)] for k in idx]))
    m.esdf_layer().set_blocks(idx, np.stack([esdf[tuple(k)] for k in idx]))
    m.esdf_integrator().integrate_blocks(idx)
    s = m.esdf_integrator().last_stats()
    assert s["with_sites"] == 1 and s["to_clear"] == 0 and s["swept"] == 1 and s["rings"] == 1, s
    check_last_taker(m.esdf_layer().as_dict()[(0, 0, 0)], expected)
    m.close()
    tsdf, parents = across_face_case(nvb.TSDF_VOXEL_DTYPE)
    m = nvb.Mapper(0.05, esdf_persistent=mode)
    idx = np.array(list(tsdf), np.int32)
    m.tsdf_layer().set_blocks(idx, np.stack([tsdf[tuple(k)] for k in idx]))
    m.esdf_integrator().integrate_blocks(idx)
    s = m.esdf_integrator().last_stats()
    for k, v in ACROSS_FACE_STATS.items():
        assert s[k] == v, (k, s)
    check_across_face(m.esdf_layer().as_dict(), parents)
    m.close()


@pytest.mark.parametrize("prune", ["1", "0"])
def test_esdf_clear_pass_pruning_is_exact(gpu, monkeypatch, prune):
    """The clear pass only READS candidates whose parent box (per-block bound of where the voxels' parents live, kept by the
    exchange-slab wavefront) contains a to-clear block. Same layers and statistics as the oracle after every frame with the
    pruning on and off (NVB_CLEAR_PRUNE=0); `clear_candidates` keeps counting the reference's candidates."""
    monkeypatch.setenv("NVB_CLEAR_PRUNE", prune)
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:10], noise_sigma_rel=0.005, seed=7)
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    read, cands, cleared = 0, 0, 0
    for i, (depth, T) in enumerate(frames):
        b = m.integrate_depth(depth, T, cam)
        o.integrate_depth(depth, T, ocam)
        m.update_esdf()
        o.integrate_esdf(b if i > 0 else o.tsdf_block_indices())
        s_gpu, s_cpu = m.esdf_integrator().last_stats(), o.esdf_stats()
        for k in ("to_clear", "clear_candidates", "cleared", "swept", "face_passes", "rings"):
            assert s_gpu[k] == s_cpu[k], (i, k, s_gpu, s_cpu)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        read += m.esdf_integrator().clear_blocks_read()
        cands += s_gpu["clear_candidates"]
        cleared += s_gpu["cleared"]
    assert cleared > 0 and cands > 0
    if prune == "1":
        assert cleared <= read < cands / 2, (cleared, read, cands)
    else:
        assert read == cands
    m.close()


def test_esdf_small_grids_exercise_multi_round_paths(gpu):
    """Runs in a subprocess with NVB_ESDF_GRID_CAP=3 (the cap is read once per process): three CTAs of esdfMarkTmaKernel
    mark ~1000 blocks each (per-CTA lists flush when full) and esdfClearKernel needs several selection rounds of 256
    slots per CTA. (The plain-staged esdfMarkKernel on a capped grid: test_gpu_scale_edges_f.py, with freespace.)"""
    import subprocess, sys, textwrap
    code = textwrap.dedent("""
        import sys
        sys.path.insert(0, %r); sys.path.insert(0, %r)
        import numpy as np
        from helpers import assert_esdf_equal, assert_tsdf_equal, cameras
        from isaac_ros_nvblox_b200 import synthetic as syn
        import isaac_ros_nvblox_b200 as nvb
        from oracle import oracle as orc
        cs, cam, ocam = cameras(320, 240)
        frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:4])
        m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
        for i, (d, T) in enumerate(frames):
            b = m.integrate_depth(d, T, cam)
            o.integrate_depth(d, T, ocam)
            m.update_esdf()
            o.integrate_esdf(b if i > 0 else o.tsdf_block_indices())
        assert m.esdf_layer().num_blocks() > 3 * 256 * 2
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        m.close()
        print("ok")
    """) % (os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    env = dict(os.environ, NVB_ESDF_GRID_CAP="3")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("mode", [2, 3])
def test_esdf_gather_replay_2cm_many_candidates(gpu, mode):
    """2 cm voxels: rings with thousands of candidates (several chunks of 32 per CTA in the gather-replay kernel, several
    candidates per 64-thread group in the exchange-slab kernel)."""
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(80)[:2])
    import os as _os
    _os.environ["NVB_GES_SWITCH"] = "100000"
    try:
        m, o = _run_pair(0.02, frames, cam, ocam, esdf=True, tsdf_kw=dict(max_integration_distance_m=4.0),
                         mapper_kw=dict(esdf_persistent=mode), check_every_frame=False)
    finally:
        _os.environ.pop("NVB_GES_SWITCH", None)
    assert m.esdf_layer().num_blocks() > 10000
    m.close()


def test_esdf_640x480_5cm_sequence(gpu):
    cs, cam, ocam = cameras()
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80)[:4])
    m, o = _run_pair(0.05, frames, cam, ocam, esdf=True, check_every_frame=False)
    m.close()


def test_esdf_cube_scene_with_noise(gpu):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(40)[:4], noise_sigma_rel=0.01,
                               dropout=0.05, seed=5)
    m, _ = _run_pair(0.05, frames, cam, ocam, esdf=True)
    m.close()


def test_esdf_explicit_block_lists_and_params(gpu):
    """EsdfIntegrator::integrateBlocks on caller lists, non-default parameters, duplicate and
    unallocated indices, empty list."""
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:3])
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    ep = orc.default_esdf_params(max_esdf_distance_m=1.0, max_site_distance_vox=1.5, min_weight=0.01)
    m.esdf_integrator().params(max_esdf_distance_m=1.0, max_site_distance_vox=1.5, min_weight=0.01)
    m.esdf_integrator().integrate_blocks(np.zeros((0, 3), np.int32))  # no-op
    for depth, T in frames:
        b = m.integrate_depth(depth, T, cam)
        o.integrate_depth(depth, T, ocam)
        lst = np.vstack([b, b[:10], [[500, 500, 500]]]).astype(np.int32)  # duplicates + a block without TSDF
        m.esdf_integrator().integrate_blocks(lst)
        o.integrate_esdf(lst, ep)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    # a list several times longer than any before, on the same mapper: the upload buffer grows
    far = np.stack([500 + np.arange(4 * len(lst)), np.full(4 * len(lst), 500), np.full(4 * len(lst), 500)], axis=1)
    lst = np.vstack([m.tsdf_layer().get_all_block_indices(), far]).astype(np.int32)
    m.esdf_integrator().integrate_blocks(lst)
    o.integrate_esdf(lst, ep)
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


def test_esdf_update_without_new_frames_changes_nothing(gpu):
    nvb = _nvb()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:2])
    m = nvb.Mapper(0.05)
    for depth, T in frames:
        m.integrate_depth(depth, T, cam)
        m.update_esdf()
    before = layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS)
    m.update_esdf()  # tracker is empty: Mapper::updateEsdf hands an empty list -> early return
    assert layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS) == before
    m.close()


def test_esdf_full_layer_update(gpu):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(40)[:3])
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    for depth, T in frames:
        m.integrate_depth(depth, T, cam)
        o.integrate_depth(depth, T, ocam)
    m.update_esdf()  # first query of the tracker = all blocks
    o.integrate_esdf(o.tsdf_block_indices())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.update_esdf(update_full_layer=True)
    o.integrate_esdf(o.tsdf_block_indices())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


# ----------------------------------------------------------------------------------------
# Golden fixtures + size-independent properties at full size
# ----------------------------------------------------------------------------------------
def test_golden_fixture(gpu):
    """tests/golden/c2_small.npz was produced by the oracle (tests/golden/make_golden.py)."""
    nvb = _nvb()
    g = np.load(os.path.join(GOLDEN, "c2_small.npz"))
    cam = nvb.Camera(*[float(v) for v in g["cam"][:4]], int(g["cam"][4]), int(g["cam"][5]))
    m = nvb.Mapper(float(g["voxel_size"]))
    for i in range(len(g["depth"])):
        b = m.integrate_depth(g["depth"][i], g["poses"][i], cam)
        assert np.array_equal(b, g["blocks_%d" % i])
        m.update_esdf()
    assert layer_checksum(m.tsdf_layer().as_dict(), ("distance", "weight")) == int(g["tsdf_checksum"])
    assert layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS) == int(g["esdf_checksum"])
    m.close()


def test_full_sequence_properties(gpu):
    """Every 4th frame of the C2 sequence at full size: size-independent properties of the result (the bit-for-bit
    comparison of the whole 80-frame sequence with the oracle is tests/test_gpu_bench_pipeline.py)."""
    nvb = _nvb()
    cs, cam, ocam = cameras()
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80)[::4])
    m = nvb.Mapper(0.05)
    seen = set()
    for depth, T in frames:
        b = m.integrate_depth(depth, T, cam)
        assert len({tuple(r) for r in b}) == len(b)  # unique
        seen |= {tuple(r) for r in b}
        m.update_esdf()
    tsdf = m.tsdf_layer().as_dict()
    esdf = m.esdf_layer().as_dict()
    assert set(tsdf) == seen == set(esdf)  # allocated blocks = union of updated_blocks
    max_sq = (2.0 / 0.05) ** 2
    for k, blk in esdf.items():
        obs = blk["observed"].astype(bool)
        site = blk["is_site"].astype(bool)
        assert not (site & ~obs).any()
        assert np.all(blk["squared_distance_vox"][site] == 0)
        p = blk["parent_direction"].astype(np.int64)
        has_parent = obs & ~site & (p != 0).any(axis=-1)
        sq = (p * p).sum(-1).astype(np.float32)
        assert np.array_equal(blk["squared_distance_vox"][has_parent], sq[has_parent])  # sq == |parent|^2
        t = tsdf[k]
        assert np.all(np.abs(t["distance"]) <= 0.2 + 1e-6) and np.all(t["weight"] <= 5.0)
        # observed <=> tsdf weight >= min_weight, inside <=> distance <= 0 (TsdfSiteFunctor)
        assert np.array_equal(obs, t["weight"] >= np.float32(1e-4))
        assert np.array_equal(blk["is_inside"].astype(bool) & obs, (t["distance"] <= 0) & obs)
        assert np.all(blk["squared_distance_vox"][obs] <= np.float32(max_sq))
    m.close()


@pytest.mark.parametrize("name,ok", [("test_mapper_dropin", "drop-in C++ API ok"), ("test_multi_mapper_dropin", "MultiMapper drop-in ok"), ("test_mesh_dropin", "mesh drop-in ok"), ("test_streamer_dropin", "streamer drop-in ok")])
def test_cpp_dropin_program(gpu, tmp_path, name, ok):
    """tests/cpp/*.cpp: the reference-style C++ tests through include/nvblox/ (Mapper with the reference's constructor
    signature, occupancy and freespace mappers, MultiMapper as nvblox_ros drives it)."""
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, name)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert ok in out.stdout


def test_viewpoint_cache_matches_oracle(gpu):
    """ViewpointCache (view_calculator.h:196,211-244), on by default: (1) the reference's InvalidDepthHandling sequence
    (test_tsdf_integrator.cpp:588-722) -- six all-invalid frames at one pose, a valid one, three invalid ones -- gives the
    same lists and the same voxels as the oracle's (the valid frame integrates the NaN frame's cached single block, the
    later invalid frames decay it); (2) hits and misses by pose / sensor tolerance and the two-entry capacity; (3) the cache
    can be switched off."""
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras()
    T = np.eye(4, dtype=np.float32)
    m, o = nvb.Mapper(0.2), orc.OracleMap(0.2)
    p = orc.default_tsdf_params(invalid_depth_decay_factor=0.8, weighting_type=orc.WEIGHT_CONSTANT)
    m.tsdf_integrator().params(invalid_depth_decay_factor=0.8, weighting_type=orc.WEIGHT_CONSTANT)
    for v in (np.nan, np.inf, -np.inf, -1.0, 0.0, -10.0, 2.0, np.inf, -1.0, 0.0):
        d = np.full((480, 640), v, np.float32)
        assert np.array_equal(m.integrate_depth(d, T, cam), o.integrate_depth(d, T, ocam, p)), v
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    w = sum(float(b["weight"].sum(dtype=np.float64)) for b in m.tsdf_layer().as_dict().values())
    n = sum(int((b["weight"] > 0).sum()) for b in m.tsdf_layer().as_dict().values())
    assert n > 0 and abs(w - n * 0.8 ** 3) < 1e-3
    m.close()
    # keys and capacity, side by side with the oracle
    m, o = nvb.Mapper(0.2), orc.OracleMap(0.2)
    p = orc.default_tsdf_params()
    near, far = np.full((480, 640), 1.0, np.float32), np.full((480, 640), 4.0, np.float32)
    poses = []
    for dx in (0.0, 0.0005, 0.002):
        Tx = np.eye(4, dtype=np.float32)
        Tx[0, 3] = dx
        poses.append(Tx)
    c, s_ = np.float32(np.cos(np.deg2rad(0.05))), np.float32(np.sin(np.deg2rad(0.05)))
    R = np.eye(4, dtype=np.float32)
    R[0, 0], R[0, 2], R[2, 0], R[2, 2] = c, s_, -s_, c
    cs2, cam2, ocam2 = cameras(f=300.2)
    seq = [(near, poses[0], cam, ocam), (far, poses[1], cam, ocam), (far, poses[2], cam, ocam), (far, R, cam, ocam),
           (far, poses[0], cam2, ocam2), (far, poses[0], cam, ocam)]
    counts = []
    for d, Tq, cg, co in seq:
        bg, bo = m.integrate_depth(d, Tq, cg), o.integrate_depth(d, Tq, co, p)
        assert np.array_equal(bg, bo)
        counts.append(len(bg))
    assert counts[1] == counts[0] and counts[3] == counts[0] and counts[2] > 2 * counts[0] and counts[5] == counts[2]
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    # off: every frame raycasts
    m.tsdf_integrator().cache_last_viewpoint(False)
    o.cache_last_viewpoint(False)
    assert not m.tsdf_integrator().cache_last_viewpoint()
    bg, bo = m.integrate_depth(far, poses[0], cam), o.integrate_depth(far, poses[0], ocam, p)
    bg, bo = m.integrate_depth(near, poses[0], cam), o.integrate_depth(near, poses[0], ocam, p)
    assert np.array_equal(bg, bo) and len(bg) == counts[0]
    m.close()


def test_device_resident_block_list_merge(gpu):
    """nvb_mapper_append_frame_blocks + nvb_blocks_union_segments: frame lists appended on the device, gathered segments
    merged into the sorted unique union (x fastest) with AABB / bitset / compaction sized on the device; BatchMerger's
    double-buffered batches on one rank."""
    import ctypes as C
    import torch
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import multi_gpu
    from isaac_ros_nvblox_b200._lib import check
    m = nvb.Mapper(0.05)
    rng = np.random.default_rng(11)
    cap, world = 2000, 5
    lists = [rng.integers(-60, 60, size=(n, 3)).astype(np.int32) for n in (700, 0, 2000, 1, 1500)]
    lists[4][:300] = lists[0][:300]  # overlap between ranks
    segs = np.stack([multi_gpu.make_segment(l, cap) for l in lists])
    segs[3, 4:] = 12345  # garbage beyond a segment's count must be ignored
    want = multi_gpu.union_segments_reference(segs, cap)
    gathered = torch.from_numpy(segs.reshape(-1)).cuda()
    out = torch.zeros((world * cap, 3), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(2):  # twice: the bitset is left clean
        check(m._L.nvb_blocks_union_segments(m._h, gathered.data_ptr(), world, 1 + 3 * cap, cap, out.data_ptr(), out.shape[0],
                                             cnt.data_ptr(), None))
        m.synchronize()
        got = out[:int(cnt.item())].cpu().numpy()
        assert np.array_equal(got, want)
    err = C.c_int32(0)
    check(m._L.nvb_blocks_union_status(m._h, C.byref(err)))
    assert err.value == 0
    # all segments empty
    empty = torch.zeros(world * (1 + 3 * cap), dtype=torch.int32, device="cuda")
    check(m._L.nvb_blocks_union_segments(m._h, empty.data_ptr(), world, 1 + 3 * cap, cap, out.data_ptr(), out.shape[0], cnt.data_ptr(), None))
    m.synchronize()
    assert int(cnt.item()) == 0
    # frames appended on the device, batch by batch
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:6])
    bm = multi_gpu.BatchMerger(m, cap_entries=3 * 4096)
    per_frame = []
    for i, (depth, T) in enumerate(frames):
        per_frame.append(m.integrate_depth(depth, T, cam))
        bm.append_last_frame()
        if i % 3 == 2:
            bm.merge(timed=True)
            u = np.unique(np.concatenate(per_frame[i - 2:i + 1]), axis=0)
            assert np.array_equal(bm.result().cpu().numpy(), u[np.lexsort((u[:, 0], u[:, 1], u[:, 2]))])
    assert len(bm.merge_ms()) == 2 and all(t > 0 for t in bm.merge_ms())
    # a segment that is too small is reported, not silently truncated
    small = multi_gpu.BatchMerger(m, cap_entries=100)
    m.integrate_depth(frames[0][0], frames[0][1], cam)
    small.append_last_frame()
    with pytest.raises(Exception):
        m.synchronize()
    m.close()


def test_block_list_union_kernel(gpu):
    """nvb_blocks_union == sort(unique(concat)) as a set, in x-fastest order, with padding and duplicates."""
    import torch
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import multi_gpu
    m = nvb.Mapper(0.05)
    rng = np.random.default_rng(4)
    lists = [rng.integers(-30, 30, size=(n, 3)).astype(np.int32) for n in (700, 0, 1500)]
    cap = 1500
    padded = np.full((3, cap, 3), multi_gpu.PAD, np.int32)
    for r, l in enumerate(lists):
        padded[r, :len(l)] = l
    got = multi_gpu.union_on_device(m, torch.from_numpy(padded.reshape(-1, 3)).cuda()).cpu().numpy()
    want = np.unique(np.concatenate(lists), axis=0)
    assert len(got) == len(want)
    assert np.array_equal(sort_rows(got), want)
    lin = got[:, 0].astype(np.int64) + 1000 * got[:, 1] + 1000000 * got[:, 2]
    assert np.all(np.diff(lin) > 0)  # x fastest, then y, then z
    assert len(multi_gpu.union_on_device(m, torch.from_numpy(padded[1]).cuda())) == 0
    # world size 1 path used by bench.py
    u = multi_gpu.merge_block_lists_device(m, torch.from_numpy(lists[0]).cuda()).cpu().numpy()
    assert np.array_equal(sort_rows(u), np.unique(lists[0], axis=0))
    m.close()


FIXTURE_RADIAL = (0.1, 0.1, 0.01, 0.001, 0.001, 0.001)  # tests/include/nvblox/tests/sensor_fixture.h:97-104
FIXTURE_TANGENTIAL = (0.01, 0.02)


@pytest.mark.parametrize("dist", [(FIXTURE_RADIAL, FIXTURE_TANGENTIAL), ((-0.05, 0.01, 0, 0.02, 0, 0), (0.001, -0.0005)),
                                  ((0,) * 6, (0, 0))])
def test_distorted_camera_full_path(gpu, dist):
    """Camera with RadialTangentialDistortionParams through raycast (removeDistortion), TSDF (applyDistortion)
    and ESDF: block lists, TSDF bits and ESDF fields equal the oracle's."""
    cs, cam, ocam = cameras(320, 240, radial=dist[0], tangential=dist[1])
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:3], noise_sigma_rel=0.005, seed=11)
    m, _ = _run_pair(0.05, frames, cam, ocam, esdf=True)
    m.close()


def test_distorted_view_raycast_640x480(gpu):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(radial=FIXTURE_RADIAL, tangential=FIXTURE_TANGENTIAL)
    m = nvb.Mapper(0.05)
    for T in syn.circle_trajectory(80)[::20]:
        depth = syn.render_depth(syn.box_with_cube(), cs, T)
        got = nvb.ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
        want = orc.view_raycast(depth, T, ocam, 0.4, 0.2)
        assert np.array_equal(got, want)
    m.close()


@pytest.mark.parametrize("mode", ["tsdf", "occupancy", "tsdf_freespace"])
def test_mark_unobserved_free_inside_radius(gpu, mode):
    """Mapper::markUnobservedTsdfFreeInsideRadius (tests/test_mapper.cpp GenerateEsdfInFakeObservedAreas): same block set,
    identical projective voxels, and the ESDF of the following updates (tracker-driven here, explicit lists on the oracle)
    exact -- before the tracker's first query, after it, and with later frames on top."""
    import isaac_ros_nvblox_b200 as nvb
    from oracle import oracle as orc
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:4])
    ltype = {"tsdf": nvb.ProjectiveLayerType.kTsdf, "occupancy": nvb.ProjectiveLayerType.kOccupancy,
             "tsdf_freespace": nvb.ProjectiveLayerType.kTsdfWithFreespace}[mode]
    occ = mode == "occupancy"
    m, o = nvb.Mapper(0.1, projective_layer_type=ltype), orc.OracleMap(0.1)
    tp = orc.default_tsdf_params()

    def integrate(d, T):
        b = m.integrate_depth(d, T, cam)
        if occ:
            o.integrate_occupancy(d, T, ocam, tp)
        else:
            o.integrate_depth(d, T, ocam)
        return b

    def esdf(blocks):
        m.update_esdf()
        (o.integrate_esdf_occupancy if occ else o.integrate_esdf)(blocks)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())

    def proj_equal():
        if occ:
            g, c = m.occupancy_layer().as_dict(), o.occupancy_layer()
            assert set(g) == set(c)
            for k in g:
                assert np.array_equal(g[k]["log_odds"].view(np.uint32), np.asarray(c[k]).view(np.uint32)), k
        else:
            assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())

    # 1. before the tracker was ever queried
    d, T = frames[0]
    integrate(d, T)
    center = T[:3, 3] + np.float32(0.123)
    bg = m.mark_unobserved_tsdf_free_inside_radius(center, 1.7)
    bc = o.mark_unobserved_free_inside_radius(center, 1.7, occupancy=occ)
    assert set(map(tuple, bg.tolist())) == set(map(tuple, bc.tolist())) and len(bg) == len(bc) > 50
    proj_equal()
    esdf(o.occupancy_block_indices() if occ else o.tsdf_block_indices())
    # 2. with the tracker running: new frame + a second sphere elsewhere, then an update driven by the tracker
    d, T = frames[1]
    b = integrate(d, T)
    if mode == "tsdf_freespace":
        m.update_freespace(1000)
    c2 = np.array([-2.0, 1.0, 0.9], np.float32)
    bg = m.mark_unobserved_tsdf_free_inside_radius(c2, 2.3)
    bc = o.mark_unobserved_free_inside_radius(c2, 2.3, occupancy=occ)
    assert set(map(tuple, bg.tolist())) == set(map(tuple, bc.tolist()))
    proj_equal()
    if mode != "tsdf_freespace":  # (the oracle's plain ESDF has no freespace input; the freespace case checks the layers only)
        esdf(np.vstack([b, bc]))
        # 3. later frames integrate on top of the slightly observed voxels
        for d, T in frames[2:]:
            esdf(integrate(d, T))
        proj_equal()
    with pytest.raises(Exception):
        m.mark_unobserved_tsdf_free_inside_radius(c2, 0.0)
    m.close()


def test_golden_fixture_f_rows(gpu):
    """The CUDA path reproduces tests/golden/f_rows_small.npz (the oracle's checksums of the SURVEY.md 8(f) rows)."""
    from golden_f_rows import run_gpu
    g = np.load(os.path.join(GOLDEN, "c2_small.npz"))
    want = np.load(os.path.join(GOLDEN, "f_rows_small.npz"))
    got = run_gpu(g)
    assert set(got) == set(want.files)
    for k, v in got.items():
        assert int(want[k]) == v, k


def test_depth_preprocessing_matches_oracle(gpu):
    """Mapper::do_depth_preprocessing (mapper.cpp:335-352; mapper_impl.h:38-76) and DepthPreprocessor::dilateInvalidRegionsAsync
    (sensors/depth_preprocessing.cpp:36-58): (1) the dilation kernel on the reference-held 3DMatch frame and on random images
    with ragged sizes, every n, bit for bit; (2) a mapper with preprocessing on against the oracle with preprocessing on --
    lists, TSDF, ESDF -- through the synchronous host API and the asynchronous device API; (3) the last view kept for the
    decay exclusion is the dilated image; (4) argument checks."""
    import os
    import torch
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(0.05)
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "threedmatch_seq01.npz"))
    real = (fx["depth_u16"][0].astype(np.float32) / np.float32(1000.0)).astype(np.float32)
    rng = np.random.default_rng(5)
    images = [(real, n) for n in (0, 1, 4, 9)]
    for (r, c) in ((3, 3), (9, 9), (37, 61), (8, 32), (65, 33)):
        img = rng.uniform(0.5, 5.0, (r, c)).astype(np.float32)
        img[rng.random((r, c)) < 0.03] = 0.0
        img[rng.random((r, c)) < 0.01] = np.nan
        img[rng.random((r, c)) < 0.01] = -np.inf
        images += [(img, n) for n in (0, 1, 2, 5, 64)]
    for img, n in images:
        d = torch.from_numpy(img).cuda()
        out = torch.empty_like(d)
        m.dilate_invalid_regions_device(d.data_ptr(), out.data_ptr(), img.shape[0], img.shape[1], n)
        m.synchronize()
        assert np.array_equal(out.cpu().numpy(), orc.dilate_invalid(img, n), equal_nan=True), (img.shape, n)
    d = torch.from_numpy(real).cuda()
    out = torch.empty_like(d)
    m.dilate_invalid_regions_device(d.data_ptr(), out.data_ptr(), 480, 640, 2, invalid_depth_threshold=1.5, invalid_depth_value=-3.0)
    m.synchronize()
    assert np.array_equal(out.cpu().numpy(), orc.dilate_invalid(real, 2, threshold=1.5, value=-3.0))
    with pytest.raises(RuntimeError):
        m.dilate_invalid_regions_device(d.data_ptr(), d.data_ptr(), 480, 640, 1)
    with pytest.raises(RuntimeError):
        m.dilate_invalid_regions_device(d.data_ptr(), out.data_ptr(), 2, 640, 1)
    with pytest.raises(RuntimeError):
        m.depth_preprocessing_num_dilations(-1)
    assert m.do_depth_preprocessing() is False and m.depth_preprocessing_num_dilations() == 4
    m.close()

    K = fx["intrinsics"]
    cam = nvb.Camera(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 640, 480)
    ocam = orc.Camera(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 640, 480)
    frames = [(fx["depth_u16"][i].astype(np.float32) / np.float32(1000.0)).astype(np.float32) for i in range(3)]
    o = orc.OracleMap(0.05)
    o.depth_preprocessing(True, 4)
    lists = []
    for i, f in enumerate(frames):
        lists.append(o.integrate_depth(f, fx["poses"][i], ocam))
        o.integrate_esdf(lists[-1])
    plain = orc.OracleMap(0.05)
    plain.integrate_depth(frames[0], fx["poses"][0], ocam)
    for api in ("host", "device"):
        m = nvb.Mapper(0.05)
        m.do_depth_preprocessing(True)
        assert m.do_depth_preprocessing() is True and m.depth_preprocessing_num_dilations() == 4
        dev = torch.from_numpy(np.stack(frames)).cuda()
        for i, f in enumerate(frames):
            if api == "host":
                assert np.array_equal(m.integrate_depth(f, fx["poses"][i], cam), lists[i])
                m.update_esdf()
            else:
                m.integrate_depth_device(dev[i].data_ptr(), 480, 640, fx["poses"][i], cam)
                m.update_esdf(sync=False)
        m.synchronize()
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        assert np.array_equal(dev[2].cpu().numpy(), frames[2])  # the caller's image is not modified
        m.close()
    assert layer_checksum(o.tsdf_layer(), ("distance", "weight")) != layer_checksum(plain.tsdf_layer(), ("distance", "weight"))
    # the view saved for decayTsdfExcludeLastView is the preprocessed one (mapper_impl.h:60-76)
    m, o2 = nvb.Mapper(0.05, keep_last_view=True), orc.OracleMap(0.05)
    m.do_depth_preprocessing(True)
    m.depth_preprocessing_num_dilations(6)
    o2.depth_preprocessing(True, 6)
    m.integrate_depth(frames[0], fx["poses"][0], cam)
    o2.integrate_depth(frames[0], fx["poses"][0], ocam)
    m.decay_exclude_last_view()
    o2.decay_tsdf(depth=orc.dilate_invalid(frames[0], 6), T_L_C=fx["poses"][0], cam=ocam)
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o2.tsdf_layer())
    m.close()


@pytest.mark.parametrize("variant", ["registers"])
def test_tsdf_kernel_variants_equal_oracle(gpu, variant):
    """The register-prefetch TSDF update kernel: TSDF bits equal to the oracle's over frames with masks, invalid depth, a
    lens distortion, and a slab that grows past its initial 1 024 blocks."""
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:6])
    rng = np.random.default_rng(3)
    m, o = nvb.Mapper(0.05, tsdf_capacity_blocks=1024, esdf_capacity_blocks=1024), orc.OracleMap(0.05)
    for i, (d, T) in enumerate(frames):
        d = d.copy()
        d[rng.random(d.shape) < 0.05] = 0.0
        mask = (rng.random(d.shape) < 0.2).astype(np.uint8) if i % 2 else None
        b = m.integrate_depth(d, T, cam, mask=mask)
        assert np.array_equal(b, o.integrate_depth(d, T, ocam, mask=mask))
    assert m.tsdf_layer().num_blocks() > 1024
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()
    # a distorted camera (separate instantiation of the kernel) at 2 cm (many blocks per CTA)
    _, dc, odc = cameras(320, 240, radial=(0.05, -0.02, 0.001, 0.0, 0.0, 0.0), tangential=(0.001, -0.001))
    m, o = nvb.Mapper(0.02), orc.OracleMap(0.02)
    for d, T in frames[:2]:
        assert np.array_equal(m.integrate_depth(d, T, dc), o.integrate_depth(d, T, odc))
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()
