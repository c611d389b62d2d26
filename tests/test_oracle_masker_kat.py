"""The image masker's restatement (tests/masker_reference.py) pinned to the reference's tests/test_image_masker.cpp and to
hand-derived cases: the asymmetric patch at the image edges, a projection exactly on u == width, special depth values,
zero-depth pixels under a translated T_CM_CD, and a distorted mask camera. No GPU."""
import numpy as np
import pytest

import camera_pose_cases as cpc
import masker_reference as mr

FLT_MAX = float(mr.FLT_MAX)
I4 = np.eye(4, dtype=np.float32)


@pytest.mark.parametrize("size_addon", [0, 256, -256])
def test_random_mask(size_addon):
    """ParameterizedImageMaskerTest.RandomMask: depth 1.0 everywhere; a depth camera of 640 x 480 with a mask camera of
    the mask's size (centred principal points, so depth pixel (r, c) lands on mask pixel (r + a / 2, c + a / 2)); the
    same camera for both; and the colour split. Any mask: a seeded one stands in for std::rand."""
    rows, cols = 480, 640
    mrows, mcols = rows + size_addon, cols + size_addon
    mask = mr.random_mask(mrows, mcols, seed=size_addon + 1000)
    depth_cam, mask_cam = mr.masker_test_camera(cols, rows), mr.masker_test_camera(mcols, mrows)
    depth = np.ones((rows, cols), np.float32)
    bg, fg, _, _ = mr.split_depth(depth, mask, I4, depth_cam, mask_cam)
    r, c = np.mgrid[0:rows, 0:cols]
    mrow, mcol = r + size_addon // 2, c + size_addon // 2
    inside = (mrow >= 0) & (mcol >= 0) & (mrow < mrows) & (mcol < mcols)
    want = inside & (mask[np.clip(mrow, 0, mrows - 1), np.clip(mcol, 0, mcols - 1)] != 0)
    assert np.array_equal(fg, np.where(want, 1.0, -1.0).astype(np.float32))
    assert np.array_equal(bg, np.where(want, -1.0, 1.0).astype(np.float32))
    # the same camera: pixel for pixel
    same = np.ones((mrows, mcols), np.float32)
    bg, fg, _, _ = mr.split_depth(same, mask, I4, mask_cam, mask_cam)
    assert np.array_equal(fg, np.where(mask != 0, 1.0, -1.0).astype(np.float32))
    assert np.array_equal(bg, np.where(mask != 0, -1.0, 1.0).astype(np.float32))
    # colour: white in, black where the pixel went to the other output
    white = np.full((mrows, mcols, 3), 255, np.uint8)
    unmasked, masked, _ = mr.split_color(white, mask)
    m3 = np.repeat((mask != 0)[..., None], 3, -1)
    assert np.array_equal(masked, np.where(m3, 255, 0).astype(np.uint8))
    assert np.array_equal(unmasked, np.where(m3, 0, 255).astype(np.uint8))


def test_perpendicular_transform_mask():
    """ImageMaskerTest.PerpendicularTransformMask: 641 x 481, the mask's centre pixel set, the mask camera turned 90 degrees
    about y and 5 m away. Threshold 0: only the leftmost centre-row pixel is masked (the others are occluded by it);
    threshold FLT_MAX: the whole centre row."""
    rows, cols = 481, 641
    c = mr.masker_test_camera(cols, rows)
    mask = np.zeros((rows, cols), np.uint8)
    mask[rows // 2, cols // 2] = 1
    depth = np.ones((rows, cols), np.float32)
    T = mr.perpendicular_transform()
    r, col = np.mgrid[0:rows, 0:cols]
    bg, fg, _, _ = mr.split_depth(depth, mask, T, c, c, occlusion_threshold_m=0.0)
    centre = (col == 0) & (r == rows // 2)
    far = (col != 0) | (np.abs(r - rows // 2) > 1)
    assert fg[centre].tolist() == [1.0] and bg[centre].tolist() == [-1.0]
    assert np.all(fg[far & ~centre] == -1.0) and np.all(bg[far & ~centre] == 1.0)
    bg, fg, _, _ = mr.split_depth(depth, mask, T, c, c, occlusion_threshold_m=FLT_MAX)
    row = r == rows // 2
    assert np.all(fg[row] == 1.0) and np.all(bg[row] == -1.0)
    far = np.abs(r - rows // 2) > 3
    assert np.all(fg[far] == -1.0) and np.all(bg[far] == 1.0)


def _one_pixel(cu, cv, width=10, height=10):
    """A 1 x 1 depth camera whose pixel's ray is the optical axis, and a mask camera with principal point (cu, cv): the
    pixel projects exactly onto (cu, cv) under the identity."""
    return mr.cam(1, 1, 1.0, 1.0, 0.5, 0.5), mr.cam(width, height, 100.0, 100.0, cu, cv)


@pytest.mark.parametrize("cu, cols", [(0.6, [0, 1, 2]), (1.5, [0, 1, 2, 3]), (9.6, [7, 8, 9]), (4.0, [2, 3, 4, 5, 6])])
def test_patch_truncates_toward_zero(cu, cols):
    """The patch column is (int)((u + k) - 2.0f): at u = 0.6 the columns are -1.4 -> -1 (dropped), -0.4 -> 0, 0, 1, 2, so
    the patch holds columns 0-2 (rounding would give 0-3); at the right edge columns past the image are dropped. Rows
    follow the same rule."""
    dc, mc = _one_pixel(cu, cu)
    md = mr.min_depth_image(np.full((1, 1), 2.0, np.float32), I4, dc, mc)
    written = md != mr.FLT_MAX
    assert sorted(set(np.nonzero(written)[1].tolist())) == cols
    assert sorted(set(np.nonzero(written)[0].tolist())) == cols
    assert np.all(md[written] == 2.0)


def test_projection_on_the_far_edge_is_a_miss():
    """u == width passes Camera::project's viewport test (u > width fails); the reference then reads column `width`. Here the
    pixel goes to the unmasked output. Just inside the edge it is masked; exactly on v == height likewise a miss."""
    full = np.ones((10, 10), np.uint8)
    d = np.full((1, 1), 2.0, np.float32)
    for cu, cv, want in ((10.0, 5.0, False), (9.99, 5.0, True), (5.0, 10.0, False), (5.0, 9.99, True), (0.0, 0.0, True)):
        dc, mc = _one_pixel(cu, cv)
        ok, _, u, v = mr.project_into_mask(d, I4, dc, mc)
        assert ok[0, 0] and (u[0, 0], v[0, 0]) == (np.float32(cu), np.float32(cv))
        bg, fg, _, masked = mr.split_depth(d, full, I4, dc, mc)
        assert bool(masked[0, 0]) == want, (cu, cv)
        assert (fg[0, 0], bg[0, 0]) == ((2.0, -1.0) if want else (-1.0, 2.0))


def test_special_depth_values():
    """0, -1, +-inf and NaN never reach the masked output under the identity; the overlay's grey: 12.75 * depth truncated,
    255 for NaN, +inf and depths of 20 m and more, 0 for negative depths (the library's choice where the reference is
    undefined)."""
    c = mr.cam(8, 1, 4.0, 4.0, 4.0, 0.5)
    d = np.array([[0.0, -1.0, np.inf, -np.inf, np.nan, 1.0, 30.0, 0.1]], np.float32)
    mask = np.ones((1, 8), np.uint8)
    bg, fg, ov, masked = mr.split_depth(d, mask, I4, c, c, occlusion_threshold_m=FLT_MAX)  # 0.1 m occludes its neighbours
    assert masked[0].tolist() == [False] * 5 + [True] * 3
    assert np.array_equal(bg[0, :5].view(np.uint32), d[0, :5].view(np.uint32))
    assert np.all(fg[0, :5] == -1.0) and np.all(bg[0, 5:] == -1.0) and np.array_equal(fg[0, 5:], d[0, 5:])
    assert ov[0, :, 1].tolist() == [0, 0, 255, 0, 255, 12, 255, 1]
    assert ov[0, :, 0].tolist() == [0, 0, 255, 0, 255, 255, 255, 255]


def test_zero_depth_pixels_write_the_translation():
    """Depth 0 unprojects to the depth camera's origin, which T_CM_CD = translation (0, 0, 2) puts 2 m in front of the mask
    camera: those pixels write z = 2 into the patch at its principal point. The centre pixel at 3 m (5 m from the mask
    camera) projects there too, and is occluded by them at threshold 0.25; at FLT_MAX it is masked. The zero-depth pixels
    themselves land on the set mask unoccluded: the foreground gets their depth 0."""
    dc = mr.cam(3, 3, 1.0, 1.0, 1.5, 1.5)
    mc = mr.cam(9, 9, 10.0, 10.0, 4.5, 4.5)
    d = np.zeros((3, 3), np.float32)
    d[1, 1] = 3.0
    T = I4.copy()
    T[2, 3] = 2.0
    md = mr.min_depth_image(d, T, dc, mc)
    assert md[4, 4] == 2.0 and md[2, 2] == 2.0 and md[6, 6] == 2.0 and md[1, 1] == mr.FLT_MAX
    mask = np.ones((9, 9), np.uint8)
    _, fg, _, masked = mr.split_depth(d, mask, T, dc, mc)
    centre = np.zeros((3, 3), bool)
    centre[1, 1] = True
    assert np.array_equal(masked, ~centre) and fg[1, 1] == -1.0 and np.all(fg[~centre] == 0.0)
    _, fg, _, masked = mr.split_depth(d, mask, T, dc, mc, occlusion_threshold_m=FLT_MAX)
    assert masked.all() and fg[1, 1] == 3.0
    # without the translation nothing projects from a zero depth
    assert mr.min_depth_image(d, I4, dc, mc)[4, 4] == 3.0


def test_distorted_mask_camera():
    """A point at normalised (0.5, 0) with k1 = 0.2 lands at 0.5 * (1 + 0.2 * 0.25) = 0.525, pixel column 52 with fu = 100
    and cu = 0; without distortion at column 50."""
    dc = mr.cam(1, 1, 1.0, 1.0, 0.0, 0.5)  # pixel (0, 0): x = 0.5, y = 0
    radial = (0.2, 0.0, 0.0, 0.0, 0.0, 0.0)
    mc = mr.cam(80, 10, 100.0, 100.0, 0.0, 5.0, radial=radial, tangential=(0.0, 0.0))
    plain = mr.cam(80, 10, 100.0, 100.0, 0.0, 5.0)
    d = np.full((1, 1), 2.0, np.float32)
    mask = np.zeros((10, 80), np.uint8)
    mask[5, 52] = 1
    ok, _, u, v = mr.project_into_mask(d, I4, dc, mc)
    assert ok[0, 0] and int(u[0, 0]) == 52 and abs(float(u[0, 0]) - 52.5) < 1e-4 and int(v[0, 0]) == 5
    assert mr.split_depth(d, mask, I4, dc, mc)[3][0, 0]
    assert not mr.split_depth(d, mask, I4, dc, plain)[3][0, 0]
    # tangential terms move it as well
    tang = mr.cam(80, 10, 100.0, 100.0, 0.0, 5.0, radial=(0.0,) * 6, tangential=(0.0, 0.02))
    _, _, u, _ = mr.project_into_mask(d, I4, dc, tang)  # x + p2 * (r2 + 2 x^2) = 0.5 + 0.02 * 0.75
    assert abs(float(u[0, 0]) - 51.5) < 1e-4


@pytest.mark.parametrize("what", ["f", "c"])
def test_exchanged_mask_intrinsics_change_the_split(what):
    """Guard: with the mask camera's fu / fv, or cu / cv, exchanged the general colour-camera case splits differently."""
    depth, mask, T, dc, mc = mr.colour_camera_case()
    _, fg, _, masked = mr.split_depth(depth, mask, T, dc, mc)
    _, fg_s, _, masked_s = mr.split_depth(depth, mask, T, dc, cpc.swapped(mc, what))
    assert 0.2 < masked.mean() < 0.8
    assert (masked != masked_s).sum() > 1000


def test_human_mapping_dropin_compiles(built, tmp_path):
    """tests/cpp/test_human_mapping_dropin.cpp builds with plain g++ against the mirror headers and the C ABI; without a
    GPU it reports that and exits 77."""
    import subprocess
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_human_mapping_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
