"""The image masker on the GPU, bit for bit against the restatement (tests/masker_reference.py), and the human-mapping
pipeline composed from it (filter, split, TSDF background, occupancy foreground) against the CPU oracle."""
import subprocess

import numpy as np
import pytest

import camera_pose_cases as cpc
import dynamics_reference as dref
import masker_reference as mr
from helpers import assert_esdf_equal, assert_tsdf_equal

pytestmark = pytest.mark.gpu
FLT_MAX = float(mr.FLT_MAX)
I4 = np.eye(4, dtype=np.float32)


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _camera(c):
    return _nvb().Camera(c["fu"], c["fv"], c["cu"], c["cv"], c["width"], c["height"], c.get("radial"), c.get("tangential"))


def _mapper():
    return _nvb().Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _check(masker, depth, mask, T, dc, mc, threshold=0.25, overlay=True):
    """Host split on the GPU against the restatement: depth outputs as uint32 views (NaN payloads included), overlay bytes."""
    masker.params(occlusion_threshold_m=threshold)
    got = masker.split_depth(depth, mask, T, _camera(dc), _camera(mc), overlay=overlay)
    bg, fg, ov, _ = mr.split_depth(depth, mask, T, dc, mc, occlusion_threshold_m=threshold)
    assert _same_bits(got[0], bg), "background"
    assert _same_bits(got[1], fg), "foreground"
    if overlay:
        assert np.array_equal(got[2], ov), "overlay"
    else:
        assert masker.output(_nvb()._lib.NVB_SPLIT_OVERLAY).size == 0
    return got


def _kat_cases():
    """(name, depth, mask, T_CM_CD, depth_cam, mask_cam, thresholds) of the known-answer tests."""
    out = []
    rows, cols = 480, 640
    for a in (0, 256, -256):
        dc, mc = mr.masker_test_camera(cols, rows), mr.masker_test_camera(cols + a, rows + a)
        out.append(("random_mask_%d" % a, np.ones((rows, cols), np.float32), mr.random_mask(rows + a, cols + a, seed=a + 1000), I4, dc,
                    mc, (0.25,)))
    c = mr.masker_test_camera(641, 481)
    centre = np.zeros((481, 641), np.uint8)
    centre[240, 320] = 1
    out.append(("perpendicular", np.ones((481, 641), np.float32), centre, mr.perpendicular_transform(), c, c, (0.0, FLT_MAX)))
    for cu in (0.6, 1.5, 9.6, 4.0, 10.0, 9.99):
        out.append(("edge_%g" % cu, np.full((1, 1), 2.0, np.float32), np.ones((10, 10), np.uint8), I4, mr.cam(1, 1, 1.0, 1.0, 0.5, 0.5),
                    mr.cam(10, 10, 100.0, 100.0, cu, 5.0 if cu >= 9.9 else cu), (0.25,)))
    c8 = mr.cam(8, 1, 4.0, 4.0, 4.0, 0.5)
    out.append(("special", np.array([[0.0, -1.0, np.inf, -np.inf, np.nan, 1.0, 30.0, 0.1]], np.float32), np.ones((1, 8), np.uint8), I4,
                c8, c8, (0.25, FLT_MAX)))
    d = np.zeros((3, 3), np.float32)
    d[1, 1] = 3.0
    T = I4.copy()
    T[2, 3] = 2.0
    out.append(("zero_depth_translated", d, np.ones((9, 9), np.uint8), T, mr.cam(3, 3, 1.0, 1.0, 1.5, 1.5),
                mr.cam(9, 9, 10.0, 10.0, 4.5, 4.5), (0.25, FLT_MAX)))
    mask = np.zeros((10, 80), np.uint8)
    mask[5, 52] = 1
    out.append(("distorted_mask_camera", np.full((1, 1), 2.0, np.float32), mask, I4, mr.cam(1, 1, 1.0, 1.0, 0.0, 0.5),
                mr.cam(80, 10, 100.0, 100.0, 0.0, 5.0, radial=(0.2, 0, 0, 0, 0, 0), tangential=(0.0, 0.02)), (0.25,)))
    depth, mask, T, dc, mc = mr.colour_camera_case()
    out.append(("colour_camera_pair", depth, mask, T, dc, mc, (0.0, 0.25, FLT_MAX)))
    return out


def test_split_bit_for_bit_on_the_known_answers(gpu):
    """Every known-answer case of test_oracle_masker_kat.py, the 640 x 480 depth / 1280 x 720 colour-camera pair of
    camera_pose_cases.py, with the overlay on and off, on one mapper (its buffers grow and shrink with the frames)."""
    nvb = _nvb()
    m = _mapper()
    masker = nvb.ImageMasker(m)
    for name, depth, mask, T, dc, mc, thresholds in _kat_cases():
        for t in thresholds:
            for overlay in (True, False):
                try:
                    _check(masker, depth, mask, T, dc, mc, t, overlay)
                except AssertionError as e:
                    raise AssertionError("%s threshold %g overlay %s: %s" % (name, t, overlay, e))
    m.close()


def _random_pose(rng):
    a = rng.normal(size=3)
    R = cpc._axis_angle(a, rng.uniform(0.0, 25.0))
    T = cpc.pose64(R, rng.uniform(-0.3, 0.3, 3))
    return T.astype(np.float32)


@pytest.mark.parametrize("seed", range(6))
def test_split_random_poses_and_masks(gpu, seed):
    """Random poses, cameras (a distorted depth camera on two small frames: the restatement undistorts per pixel), sizes down to 1 x 1 and odd, masks, depths with special
    values; thresholds 0, 0.25 and FLT_MAX."""
    nvb = _nvb()
    rng = np.random.default_rng(seed)
    m = _mapper()
    masker = nvb.ImageMasker(m)
    sizes = [(1, 1), (7, 13), (241, 317), (480, 640), (33, 1), (1, 45)]
    rows, cols = sizes[seed]
    mrows, mcols = [(1, 1), (9, 11), (360, 641), (720, 1280), (17, 29), (5, 3)][seed]
    dist = dict(radial=(0.05, -0.01, 0.002, 0.0, 0.0, 0.0), tangential=(0.001, -0.0005)) if seed in (1, 5) else {}
    dc = mr.cam(cols, rows, rng.uniform(0.8, 1.2) * max(cols, 2), rng.uniform(0.8, 1.2) * max(cols, 2), cols * rng.uniform(0.4, 0.6),
                rows * rng.uniform(0.4, 0.6), **dist)
    mc = mr.cam(mcols, mrows, rng.uniform(0.8, 1.2) * max(mcols, 2), rng.uniform(0.8, 1.2) * max(mcols, 2),
                mcols * rng.uniform(0.4, 0.6), mrows * rng.uniform(0.4, 0.6))
    depth = mr.special_depths(rows, cols, seed)
    mask = (mr.random_mask(mrows, mcols, seed, p=0.6) * rng.integers(1, 256, (mrows, mcols))).astype(np.uint8)
    T = _random_pose(rng)
    for t in (0.0, 0.25, FLT_MAX):
        _check(masker, depth, mask, T, dc, mc, t, overlay=bool(seed % 2))
    m.close()


def test_split_device_inputs_and_growth(gpu):
    """Device inputs enqueued without a synchronisation, read through the device buffers; then a larger frame on the
    same mapper (its buffers grow), then a smaller one; the invalid values set through params()."""
    import ctypes as C
    import torch
    from isaac_ros_nvblox_b200 import _lib
    nvb = _nvb()
    m = _mapper()
    masker = nvb.ImageMasker(m)
    masker.params(depth_masked_image_invalid_pixel=0.0, depth_unmasked_image_invalid_pixel=-7.5)
    depth, mask, T, dc, mc = mr.colour_camera_case(seed=9)
    small = (depth[::4, ::4].copy(), mr.cam(160, 120, dc["fu"] / 4, dc["fv"] / 4, dc["cu"] / 4, dc["cv"] / 4))
    for d, c in (small, (depth, dc), small):
        td, tm = torch.from_numpy(d).cuda(), torch.from_numpy(mask).cuda()
        torch.cuda.synchronize()
        b = masker.split_depth_device(td.data_ptr(), d.shape[0], d.shape[1], tm.data_ptr(), mask.shape[0], mask.shape[1], T,
                                      _camera(c), _camera(mc), overlay=True)
        assert (b["rows"], b["cols"]) == d.shape
        bg, fg, ov, masked = mr.split_depth(d, mask, T, c, mc, masked_invalid=0.0, unmasked_invalid=-7.5)
        assert b["background"] and b["foreground"] and b["overlay"]
        outs = [torch.empty(d.shape, dtype=torch.float32, device="cuda") for _ in range(2)]
        outs.append(torch.empty(d.shape + (3,), dtype=torch.uint8, device="cuda"))
        rows, cols = C.c_int32(0), C.c_int32(0)
        for which, o in enumerate(outs):  # device copies, enqueued on the mapper's stream
            _lib.check(m._L.nvb_mapper_split_output(m._h, which, o.data_ptr(), _lib.NVB_MEM_DEVICE, C.byref(rows), C.byref(cols)))
        m.synchronize()
        assert _same_bits(outs[0].cpu().numpy(), bg)
        assert _same_bits(outs[1].cpu().numpy(), fg)
        assert np.array_equal(outs[2].cpu().numpy(), ov)
        assert 0 < masked.sum() < masked.size
    m.close()


def test_split_color(gpu):
    """splitColorImageKernel: host and device buffers, with and without the overlay, odd sizes."""
    import torch
    nvb = _nvb()
    m = _mapper()
    masker = nvb.ImageMasker(m)
    rng = np.random.default_rng(4)
    for rows, cols in ((1, 1), (37, 53), (720, 1280)):
        rgb = rng.integers(0, 256, (rows, cols, 3), dtype=np.uint8)
        mask = (rng.random((rows, cols)) < 0.4).astype(np.uint8) * rng.integers(1, 256, (rows, cols)).astype(np.uint8)
        want = mr.split_color(rgb, mask)
        got = masker.split_color(rgb, mask, overlay=True)
        assert all(np.array_equal(g, w) for g, w in zip(got, want))
        got = masker.split_color(rgb, mask)
        assert len(got) == 2 and all(np.array_equal(g, w) for g, w in zip(got, want[:2]))
        t_rgb, t_mask = torch.from_numpy(rgb).cuda(), torch.from_numpy(mask).cuda()
        outs = [torch.empty_like(t_rgb) for _ in range(3)]
        torch.cuda.synchronize()
        masker.split_color_device(t_rgb.data_ptr(), t_mask.data_ptr(), rows, cols, *(o.data_ptr() for o in outs))
        m.synchronize()
        assert all(np.array_equal(o.cpu().numpy(), w) for o, w in zip(outs, want))
    m.close()


def test_argument_checks(gpu):
    """The reference's CHECKs (sizes against the cameras, empty images) and null pointers, bad memory kinds and images
    above the per-image pixel limit are NVB_ERR_INVALID_ARGUMENT."""
    import ctypes as C
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import _lib
    m = _mapper()
    masker = nvb.ImageMasker(m)
    import torch
    d, mk = np.ones((4, 6), np.float32), np.ones((4, 6), np.uint8)
    cam = nvb.Camera(5.0, 5.0, 3.0, 2.0, 6, 4)
    # device buffers for the kind 2 cases: a call that took the kind for device memory would succeed on them
    td, tb = torch.ones((4, 6), dtype=torch.float32, device="cuda"), torch.ones((4, 6, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r, c = C.c_int32(0), C.c_int32(0)
    bad = [
        lambda: masker.split_depth(np.ones((4, 5), np.float32), mk, I4, cam, cam),       # depth size != depth camera
        lambda: masker.split_depth(d, np.ones((5, 6), np.uint8), I4, cam, cam),            # mask size != mask camera
        lambda: masker.split_depth(np.ones((0, 6), np.float32), mk, I4, nvb.Camera(5, 5, 3, 2, 6, 0), cam),  # empty
        lambda: masker.split_depth(d, np.ones((0, 6), np.uint8), I4, cam, nvb.Camera(5, 5, 3, 2, 6, 0)),
        lambda: masker._split(d.ctypes.data, 4, 6, mk.ctypes.data, 4, 6, 7, I4, cam, cam, False),  # memory kind
        lambda: masker._split(td.data_ptr(), 4, 6, tb.data_ptr(), 4, 6, 2, I4, cam, cam, False),
        lambda: _lib.check(m._L.nvb_mapper_split_output(m._h, _lib.NVB_SPLIT_BACKGROUND, td.data_ptr(), 2, C.byref(r), C.byref(c))),
        lambda: _lib.check(m._L.nvb_mapper_split_color_image(m._h, tb.data_ptr(), tb.data_ptr(), 2, 4, 6, tb.data_ptr(), tb.data_ptr(),
                                                             None)),
        lambda: masker._split(None, 4, 6, mk.ctypes.data, 4, 6, _lib.NVB_MEM_HOST, I4, cam, cam, False),
        lambda: masker._split(d.ctypes.data, 4, 6, None, 4, 6, _lib.NVB_MEM_HOST, I4, cam, cam, False),
        lambda: masker._split(d.ctypes.data, 1 << 15, 1 << 14, mk.ctypes.data, 4, 6, _lib.NVB_MEM_HOST, I4,
                              nvb.Camera(5, 5, 3, 2, 1 << 14, 1 << 15), cam, False),   # 2^29 pixels
        lambda: masker.output(3),
        lambda: masker.split_color_device(None, 0, 4, 6, 0, 0),
        lambda: check_color(m, 0, 6),
    ]

    def check_color(mp, rows, cols):
        z = np.zeros(max(rows * cols * 3, 3), np.uint8)
        _lib.check(mp._L.nvb_mapper_split_color_image(mp._h, z.ctypes.data, z.ctypes.data, _lib.NVB_MEM_HOST, rows, cols,
                                                      z.ctypes.data, z.ctypes.data, None))

    for i, f in enumerate(bad):
        with pytest.raises(_lib.NvbError) as ei:
            f()
        assert ei.value.code == -1, i
    b = _lib.NvbSplitBuffers()
    assert m._L.nvb_mapper_split_device_buffers(None, C.byref(b)) == -1
    # before any split the outputs are empty; a failed call leaves the last split's outputs in place
    assert masker.output(_lib.NVB_SPLIT_BACKGROUND).shape == (0, 0)
    masker.split_depth(d, mk, I4, cam, cam)
    with pytest.raises(_lib.NvbError):
        masker.split_depth(d, np.ones((5, 6), np.uint8), I4, cam, cam)
    assert masker.output(_lib.NVB_SPLIT_FOREGROUND).shape == (4, 6)
    m.close()


def test_human_pipeline_against_restatement_and_oracle(gpu):
    """MultiMapper's human frame composed through the Python API over a sequence of the 640 x 480 depth / 1280 x 720 colour
    pair: the filter and the split on the background mapper's stream (device inputs, no synchronisation), the TSDF
    background integrating the split's background frame, the occupancy foreground its foreground frame behind an event.
    The TSDF, the occupancy and both ESDFs equal the oracle's after it integrates the restatement's split frames."""
    import torch
    nvb = _nvb()
    from oracle import oracle as orc
    dc, mc = cpc.COLOR_DEPTH_CAM, cpc.COLOR_CAM
    _, cam, ocam = cpc.cameras(dc)
    mcam = _camera(mc)
    T_CM_CD = mr.inverse(cpc.T_D_C)
    bg = nvb.Mapper(0.05)
    fg = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    masker = nvb.ImageMasker(bg)
    o_bg, o_fg = orc.OracleMap(0.05), orc.OracleMap(0.05)
    threshold = 2000
    n_fg = 0
    for i, (T_L_D, _) in enumerate(cpc.color_poses(4)):
        depth, mask, _, _, _ = mr.colour_camera_case(seed=20 + i)
        mask[:6, :] = 0
        mask[::97, ::89] = 255  # isolated specks: the filter removes them
        td, tm = torch.from_numpy(depth).cuda(), torch.from_numpy(mask).cuda()
        tclean = torch.empty_like(tm)
        torch.cuda.synchronize()
        nvb.mapper.remove_small_connected_components_device(tm.data_ptr(), tclean.data_ptr(), mc["height"], mc["width"], threshold, bg)
        b = masker.split_depth_device(td.data_ptr(), dc["height"], dc["width"], tclean.data_ptr(), mc["height"], mc["width"],
                                      T_CM_CD, cam, mcam)
        bg.integrate_depth_device(b["background"], dc["height"], dc["width"], T_L_D, cam)
        fg.wait_for(bg)
        fg.integrate_depth_device(b["foreground"], dc["height"], dc["width"], T_L_D, cam, sync=True)
        bg.synchronize()
        bg.update_esdf()
        fg.update_esdf()
        clean = dref.remove_small_connected_components(mask, threshold)
        r_bg, r_fg, _, masked = mr.split_depth(depth, clean, T_CM_CD, dc, mc)
        assert _same_bits(masker.output(nvb._lib.NVB_SPLIT_BACKGROUND), r_bg), i
        ob = o_bg.integrate_depth(r_bg, T_L_D, ocam)
        of = o_fg.integrate_occupancy(r_fg, T_L_D, ocam)
        o_bg.integrate_esdf(ob if i > 0 else o_bg.tsdf_block_indices())
        o_fg.integrate_esdf_occupancy(of if i > 0 else o_fg.occupancy_block_indices())
        n_fg += int(masked.sum())
    assert n_fg > 10000
    assert_tsdf_equal(bg.tsdf_layer().as_dict(), o_bg.tsdf_layer())
    g_occ, c_occ = fg.occupancy_layer().as_dict(), o_fg.occupancy_layer()
    assert set(g_occ) == set(c_occ)
    for k in c_occ:
        assert np.array_equal(g_occ[k]["log_odds"].view(np.uint32), c_occ[k].view(np.uint32)), k
    assert_esdf_equal(bg.esdf_layer().as_dict(), o_bg.esdf_layer())
    assert_esdf_equal(fg.esdf_layer().as_dict(), o_fg.esdf_layer())
    bg.close()
    fg.close()


def test_human_mapping_dropin_program(gpu, tmp_path):
    """tests/cpp/test_human_mapping_dropin.cpp: MultiMapper's human overload with a separate 1280 x 720 mask camera, its
    getters, the kept identity path, and identity with other intrinsics going through the re-projection."""
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_human_mapping_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "human mapping drop-in ok" in out.stdout
