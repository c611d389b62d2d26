"""Dynamics detection, the connected-component mask filter and the kDynamic pipeline on the GPU, bit for bit against the
restatement (tests/dynamics_reference.py) and the CPU oracle."""
import subprocess

import numpy as np
import pytest

import dynamics_reference as dref
from helpers import assert_tsdf_equal, cameras
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
FS_FIELDS = ("last_occupied_timestamp_ms", "consecutive_occupancy_duration_ms", "is_high_confidence_freespace")


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _fs_mapper(voxel=0.05):
    nvb = _nvb()
    return nvb.Mapper(voxel, projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)


def _cam_dict(cam, radial=None, tangential=None):
    return {"fu": cam.fu, "fv": cam.fv, "cu": cam.cu, "cv": cam.cv, "radial": radial, "tangential": tangential}


def _detect_and_compare(m, depth, T, cam, cam_d):
    """Runs the detection on the GPU and asserts mask, overlay and point bytes equal the restatement's on the GPU's own
    freespace layer. -> points."""
    fs = m.freespace_layer().as_dict()
    det = m.dynamics_detection()
    det.compute_dynamics(depth, T, cam)
    mask, overlay, pts = dref.compute_dynamics(depth, T, cam_d, fs, m.block_size())
    g_mask, g_ov, g_pts = det.dynamic_mask(), det.dynamic_overlay(), det.dynamic_points()
    assert np.array_equal(g_mask, mask)
    assert np.array_equal(g_ov, overlay)
    # row-major order, bit for bit; a NaN depth makes a NaN point, whose payload is the hardware's
    assert g_pts.shape == pts.shape and np.array_equal(np.isnan(g_pts), np.isnan(pts))
    ok = ~np.isnan(pts)
    assert np.array_equal(g_pts[ok].view(np.uint32), pts[ok].view(np.uint32))
    return g_pts


def _static_map(m, depth, T, frames=12, step_ms=100, **fs_kw):
    m.freespace_integrator().params(**fs_kw)
    for i in range(frames):
        m.integrate_depth(depth, T, m._cam)
        m.update_freespace(step_ms * i, depth=depth, T_L_C=T, camera=m._cam)


def test_detection_primitive_scene_with_added_box(gpu):
    """PrimitiveScene's shape: a static wall integrated into TSDF + freespace, then frames with a box in front of it: no
    points without the box, points with it, every one on the box (+-1e-4)."""
    cs, cam, _ = cameras(320, 240)
    T = np.eye(4, dtype=np.float32)
    wall = syn.render_depth(syn.plane_scene(4.0), cs, np.eye(4), max_dist=8.0)
    m = _fs_mapper()
    m._cam = cam
    _static_map(m, wall, T, min_duration_since_occupied_for_freespace_ms=300)
    assert len(_detect_and_compare(m, wall, T, cam, _cam_dict(cam))) == 0
    for k in range(3):
        d = wall.copy()
        r0, c0 = 80, 60 + 40 * k
        d[r0:r0 + 60, c0:c0 + 80] = 2.0
        pts = _detect_and_compare(m, d, T, cam, _cam_dict(cam))
        assert len(pts) > 0
        assert np.all(np.abs(pts[:, 2] - 2.0) <= 1e-4)
        c = pts[:, 0] / pts[:, 2] * cam.fu + cam.cu
        r = pts[:, 1] / pts[:, 2] * cam.fv + cam.cv
        assert np.all((c >= c0 - 1e-3) & (c <= c0 + 80 + 1e-3) & (r >= r0 - 1e-3) & (r <= r0 + 60 + 1e-3))
    # the same view at twice the resolution on the same mapper: the detector's per-pixel buffers grow
    cs2, cam2, _ = cameras(640, 480)
    d = syn.render_depth(syn.plane_scene(4.0), cs2, np.eye(4), max_dist=8.0)
    d[160:280, 120:280] = 2.0
    assert len(_detect_and_compare(m, d, T, cam2, _cam_dict(cam2))) > 0
    m.close()


def test_detection_human_dataset(gpu):
    """test_dynamics.cpp HumanDataset (Camera) on the GPU: the freespace of frame 1 after two updates 1 000 ms apart, then
    the detection on frame 2."""
    nvb = _nvb()
    K, depth, _ = dref.load_human_fixture()
    rows, cols = depth.shape[1:]
    cam = nvb.Camera(K[0, 0], K[1, 1], K[0, 2], K[1, 2], cols, rows)
    m = _fs_mapper()
    m.tsdf_integrator().params(truncation_distance_vox=4.0, max_integration_distance_m=20.0)
    T = np.eye(4, dtype=np.float32)
    m.integrate_depth(depth[0], T, cam)
    m.freespace_integrator().params(max_tsdf_distance_for_occupancy_m=float(np.float32(0.2) * np.float32(0.75)),
                                    min_duration_since_occupied_for_freespace_ms=1000, check_neighborhood=0)
    blocks = m.tsdf_layer().get_all_block_indices()
    for t in (100, 1100):
        m.freespace_integrator().update_freespace_layer(blocks, t)
    pts = _detect_and_compare(m, depth[1], T, cam, _cam_dict(cam))
    assert rows * cols / 20.0 < len(pts) < rows * cols / 5.0
    m.close()


def _handmade_freespace(m, T, cam_s, rows, cols, seed, depth_range=(0.5, 4.0)):
    """Freespace blocks over the view with random high-confidence voxels, set directly; a depth image with 0, negative,
    NaN and +-inf pixels."""
    nvb = _nvb()
    rng = np.random.default_rng(seed)
    depth = rng.uniform(*depth_range, size=(rows, cols)).astype(np.float32)
    special = rng.integers(0, 40, size=(rows, cols))
    depth[special == 0] = 0.0
    depth[special == 1] = -1.0
    depth[special == 2] = np.nan
    depth[special == 3] = np.inf
    depth[special == 4] = -np.inf
    cam_d = {"fu": cam_s.fu, "fv": cam_s.fv, "cu": cam_s.cu, "cv": cam_s.cv}
    rr, cc = np.nonzero(np.isfinite(depth) & (depth > 0))
    p = dref.unproject_transform(depth[rr, cc], T, cam_d, rr, cc)
    keys = np.unique(np.floor(p / np.float32(m.block_size())).astype(np.int32), axis=0)
    keep = rng.random(len(keys)) < 0.8  # some blocks missing
    keys = np.unique(np.concatenate([keys[keep], np.zeros((1, 3), np.int32)]), axis=0)  # (0, 0, 0): where NaN depths land
    vox = np.zeros((len(keys), 8, 8, 8), nvb.FREESPACE_VOXEL_DTYPE)
    vox["is_high_confidence_freespace"] = rng.random((len(keys), 8, 8, 8)) < 0.5
    m.freespace_layer().set_blocks(keys, vox)
    return depth


@pytest.mark.parametrize("case", ["pinhole", "distorted", "far_300m", "hd_1080p", "empty_layer"])
def test_detection_handmade_layers(gpu, case):
    """Hand-built freespace layers: a distorted camera, a map at +300 m, 1920 x 1080 frames, no blocks at all; depth images
    with 0, negative, NaN and +-inf pixels."""
    nvb = _nvb()
    rows, cols = (1080, 1920) if case == "hd_1080p" else ((60, 80) if case == "distorted" else (240, 320))
    radial, tangential = ((0.1, -0.05, 0.01, 0.0, 0.0, 0.0), (0.001, -0.002)) if case == "distorted" else (None, None)
    cs, cam, _ = cameras(cols, rows, radial=radial, tangential=tangential)
    T = np.eye(4, dtype=np.float32)
    if case == "far_300m":
        T[:3, 3] = (300.0, -300.0, 300.0)
    m = _fs_mapper()
    if case == "empty_layer":
        depth = np.full((rows, cols), 2.0, np.float32)
        depth[0, 0] = np.nan
    else:
        depth = _handmade_freespace(m, T, cs, rows, cols, seed=len(case))
    pts = _detect_and_compare(m, depth, T, cam, _cam_dict(cam, radial, tangential))
    if case == "empty_layer":
        assert len(pts) == 0 and np.all(m.dynamics_detection().dynamic_overlay() == 255)
    else:
        assert len(pts) > 0
    m.close()


def test_detection_initialize_to_high_confidence_freespace(gpu):
    """initialize_to_high_confidence_freespace: new freespace voxels start high-confidence, so a box in front of a wall seen
    once is dynamic at once."""
    cs, cam, _ = cameras(160, 120)
    T = np.eye(4, dtype=np.float32)
    wall = syn.render_depth(syn.plane_scene(3.0), cs, np.eye(4), max_dist=8.0)
    m = _fs_mapper()
    m._cam = cam
    _static_map(m, wall, T, frames=1, initialize_to_high_confidence_freespace=1)
    d = wall.copy()
    d[40:80, 50:110] = 1.5
    assert len(_detect_and_compare(m, d, T, cam, _cam_dict(cam))) > 0
    m.close()


def test_detection_needs_a_freespace_layer(gpu):
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import _lib
    _, cam, _ = cameras(64, 48)
    for lt in (nvb.ProjectiveLayerType.kTsdf, nvb.ProjectiveLayerType.kOccupancy):
        m = nvb.Mapper(0.05, projective_layer_type=lt)
        with pytest.raises(_lib.NvbError) as ei:
            m.dynamics_detection().compute_dynamics(np.ones((48, 64), np.float32), np.eye(4), cam)
        assert ei.value.code == -1  # NVB_ERR_INVALID_ARGUMENT
        m.close()


# ---------------------------------------------------------------------------------------------------------------------
# The connected-component filter
# ---------------------------------------------------------------------------------------------------------------------
def _filter_cases():
    _, _, mask_21 = dref.load_human_fixture()
    cases = [(name, m, t) for name, (m, t, _) in dref.reference_masks(mask_21).items()]
    cases += [("corner_" + n, m, 3) for n, (m, _) in dref.corner_blobs().items()]
    rng = np.random.default_rng(7)
    for dens in (0.3, 0.5, 0.593, 0.7):
        m = ((rng.random((480, 640)) < dens) * rng.integers(1, 256, (480, 640))).astype(np.uint8)
        sizes = dref.component_sizes(m)
        for t in (0, 1, 3, 4, 5, int(4 * np.median(sizes)), int(4 * sizes.max()) - 4, int(4 * sizes.max()),
                  int(4 * sizes.max()) + 4, 10 ** 7):
            cases.append(("random_%g_t%d" % (dens, t), m, t))
    spiral = dref.spiral_mask(480, 640)
    n = int(dref.component_sizes(spiral)[0])
    cases += [("spiral_t%d" % t, spiral, t) for t in (4 * n - 4, 4 * n, 4 * n + 4)]
    # combs whose teeth cross every 64-pixel tile border (32 x 32 labelling tiles in the downscaled image)
    comb = np.zeros((480, 640), np.uint8)
    comb[0:4, :] = 255
    comb[:, ::4] = 255
    comb2 = np.zeros((1080, 1920), np.uint8)
    comb2[:, 0:2] = 255
    comb2[::4, :] = 255
    yy, xx = np.mgrid[0:480, 0:640]
    checker = (((yy // 2) + (xx // 2)) % 2 * 255).astype(np.uint8)  # downscaled: a checkerboard of single pixels
    checker64 = (((yy // 62) + (xx // 66)) % 2 * 255).astype(np.uint8)  # large squares, off the tile grid
    cases += [("comb", comb, 4 * 10000), ("comb_1080p", comb2, 8), ("checker", checker, 4), ("checker_1px_t1", checker, 1),
              ("checker64", checker64, 4 * 990)]
    for shape in ((1, 1), (2, 2), (1, 17), (17, 1), (2, 17), (37, 53), (641, 479), (1080, 1920)):
        m = ((rng.random(shape) < 0.55) * 255).astype(np.uint8)
        for t in (0, 1, 4, 8, 40):
            cases.append(("size_%dx%d_t%d" % (shape + (t,)), m, t))
    cases += [("full_1080p", np.full((1080, 1920), 9, np.uint8), 4 * 518400), ("empty_1080p", np.zeros((1080, 1920), np.uint8), 8)]
    return cases


_CASES = None


def _cases():
    global _CASES
    if _CASES is None:
        _CASES = _filter_cases()
    return _CASES


def test_filter_bit_for_bit(gpu):
    """removeSmallConnectedComponents on the GPU against the restatement, byte for byte: the reference's KAT masks, random
    masks around the percolation density, a one-pixel-wide spiral, combs and checkerboards across every tile border,
    degenerate and odd sizes, thresholds at and around a component's size x 4."""
    nvb = _nvb()
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    bad = []
    for name, mask, t in _cases():
        got = nvb.remove_small_connected_components(mask, t, mapper=m)
        want = dref.remove_small_connected_components(mask, t)
        if not np.array_equal(got, want):
            bad.append((name, int((got != want).sum())))
    assert not bad, bad
    _, _, mask_21 = dref.load_human_fixture()
    assert int((nvb.remove_small_connected_components(mask_21, 10000, mapper=m) > 0).sum()) == 11480
    m.close()


def test_filter_device_buffers_in_place(gpu):
    """The device entry point, in place (mask_in == mask_out), on the mapper's stream."""
    import torch
    from isaac_ros_nvblox_b200.mapper import remove_small_connected_components_device
    nvb = _nvb()
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    mask = dref.spiral_mask(480, 640)
    mask[300:340, 10:30] = 255  # a second, small component
    t = torch.from_numpy(mask).cuda()
    torch.cuda.synchronize()
    remove_small_connected_components_device(t.data_ptr(), t.data_ptr(), 480, 640, 1000, m)
    m.synchronize()
    assert np.array_equal(t.cpu().numpy(), dref.remove_small_connected_components(mask, 1000))
    m.close()


# ---------------------------------------------------------------------------------------------------------------------
# The kDynamic pipeline
# ---------------------------------------------------------------------------------------------------------------------
def test_kdynamic_pipeline_against_restatement_and_oracle(gpu):
    """MultiMapper kDynamic's order with two mappers through the Python API, over a sequence with a moving sphere:
    background TSDF + freespace, the detection on the background's freespace, the filter, the foreground's occupancy under
    the cleaned mask (ordered on the device), then updateFreespace. Per frame: the masks equal the restatement's; at the end
    the background TSDF and freespace fields and the foreground occupancy log odds are bit-identical with the oracle's run
    under the restatement's masks."""
    nvb = _nvb()
    from oracle import oracle as orc
    cs, cam, ocam = cameras(320, 240)
    T = np.eye(4, dtype=np.float32)
    wall = syn.render_depth(syn.plane_scene(4.0), cs, np.eye(4), max_dist=8.0)
    rng = np.random.default_rng(11)
    seq = []
    for i in range(12):  # the static wall, then a box moving across it and a few isolated specks (removed by the filter)
        d = wall.copy()
        if i >= 6:
            d[80:140, 40 + 30 * (i - 6):120 + 30 * (i - 6)] = 2.0
            d[rng.integers(0, 240, 20), rng.integers(0, 320, 20)] = 2.5
        seq.append((d, T, None))
    kw = dict(max_unobserved_to_keep_consecutive_occupancy_ms=250, min_duration_since_occupied_for_freespace_ms=300,
              min_consecutive_occupancy_duration_for_reset_ms=400)
    bg = _fs_mapper()
    fg = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    bg.freespace_integrator().params(**kw)
    o_bg, o_fg = orc.OracleMap(0.05), orc.OracleMap(0.05)
    fp_ = orc.default_freespace_params(**kw)
    threshold = 200
    n_dyn = 0
    for i, (d, T, _) in enumerate(seq):
        t_ms = 100 * i
        fs_before = bg.freespace_layer().as_dict()
        b = bg.integrate_depth(d, T, cam)
        o_bg.integrate_depth(d, T, ocam)
        det = bg.dynamics_detection()
        det.compute_dynamics(d, T, cam)
        buf = det.device_buffers()
        nvb.mapper.remove_small_connected_components_device(buf["mask"], buf["cleaned_mask"], 240, 320, threshold, bg)
        fg.wait_for(bg)
        fg.integrate_depth_device(buf["depth"], 240, 320, T, cam, mask_ptr=buf["cleaned_mask"], sync=True)
        bg.update_freespace(t_ms, depth=d, T_L_C=T, camera=cam)
        # restatement + oracle
        raw, _, _ = dref.compute_dynamics(d, T, _cam_dict(cam), fs_before, bg.block_size())
        clean = dref.remove_small_connected_components(raw, threshold)
        assert np.array_equal(det.dynamic_mask(), raw), i
        o_fg.integrate_occupancy(d, T, ocam, mask=clean, mask_mode=0)
        o_bg.update_freespace(o_bg.tsdf_block_indices() if i == 0 else b, t_ms, fp_, depth=d, T_L_C=T, cam=ocam,
                              max_view_distance_m=7.0, truncation_distance_m=2 * 4 * 0.05)
        n_dyn += int((clean > 0).sum())
    assert n_dyn > 0
    assert_tsdf_equal(bg.tsdf_layer().as_dict(), o_bg.tsdf_layer())
    g_fs, c_fs = bg.freespace_layer().as_dict(), o_bg.freespace_layer()
    assert set(g_fs) == set(c_fs)
    for k in c_fs:
        for f in FS_FIELDS:
            assert np.array_equal(g_fs[k][f], c_fs[k][f]), (f, k)
    g_occ, c_occ = fg.occupancy_layer().as_dict(), o_fg.occupancy_layer()
    assert set(g_occ) == set(c_occ)
    for k in c_occ:
        assert np.array_equal(g_occ[k]["log_odds"].view(np.uint32), c_occ[k].view(np.uint32)), k
    bg.close()
    fg.close()


def test_dynamics_dropin_program(gpu, tmp_path):
    """tests/cpp/test_dynamics_dropin.cpp: nvblox_ros' kDynamic calls without setDynamicMask through the C++ mirror."""
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_dynamics_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "dynamics drop-in ok" in out.stdout
