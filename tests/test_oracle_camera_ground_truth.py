"""The oracle against float64 geometry with general cameras (tests/camera_ground_truth.py), independent of any parity
claim: if the oracle and the kernels shared a camera slip, these checks would still see it. The same checks run on the GPU
mapper in tests/test_gpu_camera_pose.py.

Bounds (TSDF on the plane, errors gt - distance in metres):
  * reference setup: error < voxel / 10 (the reference's one-sided bound), and |error| <= 0.006 two-sided (measured on the
    oracle: -0.00450 .. 0.00493);
  * general setup (fu != fv, mirrored off-centre principal points, both cameras pitched 12 degrees): |error| <= 0.011
    (measured on the oracle: -0.00894 .. 0.00833; the more oblique rays make the closest-pixel lookup's error larger than the
    reference's voxel / 10);
  * both: more than 70 000 checked voxels, the two layers' means within 0.1 (reference) and within 1e-3 (measured: equal
    to 1e-8 by symmetry).
"""
import numpy as np
import pytest

import camera_ground_truth as gt
import camera_pose_cases as cpc
import dynamics_reference as dref
from isaac_ros_nvblox_b200 import synthetic as syn

PLANE_BOUNDS = {False: dict(one_sided=cpc.VOXEL / 10.0, two_sided=0.006), True: dict(one_sided=0.011, two_sided=0.011)}
RAYCAST_CASES = ["pitch_down_20", "pitch_down_50", "roll_plus_30", "roll_minus_30", "straight_up", "far_tilted"]


def _orc():
    from oracle import oracle as orc
    return orc


def check_plane(layer_1, layer_2, setup, general):
    r = gt.plane_tsdf_errors(layer_1, layer_2, setup)
    e, b = r["errors"], PLANE_BOUNDS[general]
    assert r["n"] > 70000, r["n"]
    assert e.max() < b["one_sided"], e.max()
    assert np.abs(e).max() <= b["two_sided"], (e.min(), e.max())
    assert abs(r["mean_1"] - r["mean_2"]) < 0.1 and abs(r["mean_1"] - r["mean_2"]) < 1e-3, (r["mean_1"], r["mean_2"])
    return r


def plane_frames(general):
    out = []
    for c, T in cpc.plane_setup(general):
        cs = cpc.cameras(c)[0]
        out.append((c, syn.render_depth(cpc.plane_scene(), cs, T, max_dist=cpc.PLANE_MAX_DIST), T))
    return out


@pytest.mark.parametrize("general", [False, True])
def test_tsdf_symmetric_view_on_plane(general):
    """TsdfErrorTest.SymmetricViewOnPlane (nvblox/tests/test_tsdf_error.cpp:56-224), and its general-camera variant."""
    orc = _orc()
    layers = []
    for c, d, T in plane_frames(general):
        o = orc.OracleMap(cpc.VOXEL)
        o.integrate_depth(d, T, cpc.cameras(c)[2])
        layers.append(o.tsdf_layer())
    check_plane(layers[0], layers[1], cpc.plane_setup(general), general)


@pytest.mark.parametrize("what", ["f", "c"])
def test_plane_check_sees_exchanged_intrinsics(what):
    orc = _orc()
    layers = []
    for c, d, T in plane_frames(True):
        o = orc.OracleMap(cpc.VOXEL)
        o.integrate_depth(d, T, cpc.cameras(cpc.swapped(c, what))[2])
        layers.append(o.tsdf_layer())
    with pytest.raises(AssertionError):
        check_plane(layers[0], layers[1], cpc.plane_setup(True), True)


def check_raycast_covers_surface(block_list, depth, case):
    miss, n = gt.missing_blocks(block_list, depth, case["cam"], case["pose"])
    assert n > 40, n
    assert len(miss) == 0, miss[:5]


def clean_frame(case):
    """The case's first frame without noise: depth and pose."""
    cs = cpc.cameras(case["cam"])[0]
    return syn.render_depth(cpc.scene_of(case), cs, cpc.local_pose(case)), case["pose"]


@pytest.mark.parametrize("name", RAYCAST_CASES)
def test_view_raycast_covers_the_back_projected_surface(name):
    orc = _orc()
    case = cpc.CASE[name]
    d, T = clean_frame(case)
    check_raycast_covers_surface(orc.view_raycast(d, T, cpc.cameras(case["cam"])[2], cpc.BLOCK, 4 * cpc.VOXEL), d, case)
    bad = orc.view_raycast(d, T, cpc.cameras(cpc.swapped(case["cam"], "c"))[2], cpc.BLOCK, 4 * cpc.VOXEL)
    with pytest.raises(AssertionError):
        check_raycast_covers_surface(bad, d, case)


def check_colour_stripes(color_layer, scene, inputs):
    bad, n = gt.stripe_colour_mismatches(color_layer, scene, [(cpc.COLOR_CAM, T_C, img) for _, _, img, T_C in inputs])
    assert n > 5000, n
    assert bad == 0, (bad, n)


def colour_inputs():
    """[(depth image, T_L_D, stripe image, T_L_C)] of the separate colour camera over the box-with-cube room."""
    scene = syn.box_with_cube()
    dcs = cpc.cameras(cpc.COLOR_DEPTH_CAM)[0]
    return [(syn.render_depth(scene, dcs, T_D), T_D, cpc.stripe_image(scene, cpc.COLOR_CAM, T_C), T_C)
            for T_D, T_C in cpc.color_poses(3)]


@pytest.mark.parametrize("variant", ["colour", "f", "c"])
def test_colour_from_a_separate_camera_matches_the_world_stripes(variant):
    """Painted with the colour camera the stripes match; painted with its fu / fv or cu / cv exchanged they do not."""
    orc = _orc()
    o = orc.OracleMap(cpc.VOXEL)
    c = cpc.COLOR_CAM if variant == "colour" else cpc.swapped(cpc.COLOR_CAM, variant)
    docam, cocam = cpc.cameras(cpc.COLOR_DEPTH_CAM)[2], cpc.cameras(c)[2]
    inputs = colour_inputs()
    for d, T_D, img, T_C in inputs:
        o.integrate_depth(d, T_D, docam)
        o.integrate_color(img, T_C, cocam)
    if variant == "colour":
        check_colour_stripes(o.color_layer(), syn.box_with_cube(), inputs)
    else:
        with pytest.raises(AssertionError):
            check_colour_stripes(o.color_layer(), syn.box_with_cube(), inputs)


def _oracle_freespace_map():
    orc = _orc()
    c = gt.DYN_CAM
    ocam = cpc.cameras(c)[2]
    wall = gt.dynamics_wall()
    T = np.eye(4, dtype=np.float32)
    o = orc.OracleMap(cpc.VOXEL)
    fp = orc.default_freespace_params(min_duration_since_occupied_for_freespace_ms=300)
    for i in range(12):
        b = o.integrate_depth(wall, T, ocam)
        o.update_freespace(b, 100 * i, fp, depth=wall, T_L_C=T, cam=ocam)
    return o, wall


def check_dynamics_points(points, k):
    assert len(points) > 100
    assert np.all(np.abs(points[:, 2] - gt.DYN_BOX_DEPTH) <= 1e-4)
    assert gt.dynamics_points_outside_box(points, k) == 0


def test_dynamics_points_reproject_into_the_box():
    """A box in front of a static wall, seen by a camera with fu != fv and an off-centre principal point: every detected
    point re-projects with the float64 intrinsics into the box's pixel rectangle (restatement on the oracle's freespace)."""
    o, wall = _oracle_freespace_map()
    c = gt.DYN_CAM
    T = np.eye(4, dtype=np.float32)
    cam = {k: c[k] for k in ("fu", "fv", "cu", "cv")}
    _, _, pts = dref.compute_dynamics(wall, T, cam, o.freespace_layer(), cpc.BLOCK)
    assert len(pts) == 0
    for k in range(len(gt.DYN_BOXES)):
        _, _, pts = dref.compute_dynamics(gt.dynamics_box_frame(wall, k), T, cam, o.freespace_layer(), cpc.BLOCK)
        check_dynamics_points(pts, k)
    _, _, pts = dref.compute_dynamics(gt.dynamics_box_frame(wall, 0), T, cpc.swapped(cam, "f"), o.freespace_layer(), cpc.BLOCK)
    with pytest.raises(AssertionError):
        check_dynamics_points(pts, 0)
