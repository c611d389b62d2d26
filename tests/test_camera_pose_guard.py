"""The general-camera cases (tests/camera_pose_cases.py) test what they claim, checked on the oracle without a GPU: each has
the property its name states, integrates enough blocks, and integrating it with fu / fv or cu / cv exchanged changes the
result, so a kernel that made either slip would fail the GPU parity tests (tests/test_gpu_camera_pose.py)."""
import math

import numpy as np
import pytest

import camera_pose_cases as cpc
from isaac_ros_nvblox_b200 import synthetic as syn


def _orc():
    from oracle import oracle as orc
    return orc


ALL_CAMS = list(cpc.CAMS.values()) + [cpc.COLOR_DEPTH_CAM, cpc.COLOR_CAM, cpc.PLANE_CAM_GENERAL] + list(cpc.RIG_CAMS.values())


@pytest.mark.parametrize("i", range(len(ALL_CAMS)))
def test_intrinsics_are_general(i):
    """fu and fv differ by at least 5 %, the principal point lies off the image centre on both axes."""
    c = ALL_CAMS[i]
    assert abs(c["fu"] / c["fv"] - 1.0) >= 0.05, c
    assert abs(c["cu"] - c["width"] / 2.0) >= 0.05 * c["width"] or c["cu"] % 1.0 == 0.5, c
    assert abs(c["cv"] - c["height"] / 2.0) >= 0.05 * c["height"] or c["cv"] % 1.0 == 0.5, c
    assert c["cu"] != c["width"] / 2.0 and c["cv"] != c["height"] / 2.0


def test_intrinsics_cover_the_named_shapes():
    c = cpc.CAMS
    assert abs(c["aniso_0.9"]["fu"] / c["aniso_0.9"]["fv"] - 0.9) < 1e-9 and abs(c["aniso_1.1"]["fu"] / c["aniso_1.1"]["fv"] - 1.1) < 1e-9
    for name in ("aniso_0.9", "aniso_1.1", "odd_641x481"):
        for k, n in (("cu", "width"), ("cv", "height")):
            assert 0.10 <= abs(c[name][k] / c[name][n] - 0.5) <= 0.15, (name, k)
    h = c["half_integer_317x239"]
    _, v = cpc.pixel_rays(h)
    assert np.sum(v[0, :, 0] == 0.0) == 1 and np.sum(v[:, 0, 1] == 0.0) == 1  # one column and one row on the axis
    assert (h["width"], h["height"]) == (317, 239) and (c["odd_641x481"]["width"], c["odd_641x481"]["height"]) == (641, 481)
    assert c["distorted"]["radial"] is not None and c["distorted"]["fu"] != c["distorted"]["fv"]
    assert {(r["width"], r["height"]) for r in cpc.RIG_CAMS.values()} == {(640, 480), (1280, 720), (424, 240)}
    assert (cpc.COLOR_CAM["width"], cpc.COLOR_CAM["height"]) != (cpc.COLOR_DEPTH_CAM["width"], cpc.COLOR_DEPTH_CAM["height"])


@pytest.mark.parametrize("name", list(cpc.CASE))
def test_case_has_its_stated_pose(name):
    """The stated pitch, roll or optical axis within 1e-6 (radians / unit-vector components) on the float32 pose."""
    case = cpc.CASE[name]
    T, cl = case["pose"], case["claims"]
    R = np.asarray(T, np.float64)[:3, :3]
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-6)
    if "pitch_deg" in cl:
        assert abs(math.radians(cpc.pitch_deg(T) - cl["pitch_deg"])) < 1e-6
        assert abs(math.radians(cpc.roll_deg(T) - cl["roll_deg"])) < 1e-6
    if "axis" in cl:
        assert np.all(np.abs(cpc.optical_axis(T) - cl["axis"]) < 1e-6)
    if cl.get("block_corner"):
        t = np.asarray(T, np.float32)[:3, 3]
        k = np.round(t / np.float32(cpc.BLOCK))
        assert np.array_equal(np.float32(cpc.BLOCK) * k.astype(np.float32), t)
    if cl.get("far"):
        assert np.allclose(np.asarray(T, np.float64)[:3, 3] - cpc.local_pose(case)[:3, 3], cpc.FAR_OFFSET)
    names = {c["name"] for c in cpc.CASES}
    assert {"pitch_down_20", "pitch_down_50", "roll_plus_30", "roll_minus_30", "straight_down", "straight_up",
            "identity_on_block_corner", "far_tilted"} <= names


def _integrate(frames, c):
    orc = _orc()
    _, _, ocam = cpc.cameras(c)
    o = orc.OracleMap(cpc.VOXEL)
    lists = [o.integrate_depth(d, T, ocam) for d, T in frames]
    return lists, o.tsdf_layer()


def _same(a, b):
    la, ta = a
    lb, tb = b
    if len(la) != len(lb) or any(not np.array_equal(x, y) for x, y in zip(la, lb)) or set(ta) != set(tb):
        return False
    return all(np.array_equal(ta[k].view(np.uint32), tb[k].view(np.uint32)) for k in ta)


@pytest.mark.parametrize("name", list(cpc.CASE))
def test_case_integrates_and_is_sensitive_to_exchanged_intrinsics(name):
    case = cpc.CASE[name]
    fr = cpc.frames(case, 1)
    base = _integrate(fr, case["cam"])
    assert len(base[0][0]) > case["min_blocks"]
    for what in ("f", "c"):
        assert not _same(base, _integrate(fr, cpc.swapped(case["cam"], what))), what


def test_colour_case_differs_from_its_depth_camera_and_is_sensitive():
    """The colour camera has its own intrinsics, resolution and pose (5 cm baseline, 1 degree); painting with the depth
    camera and pose instead, or with fu / fv or cu / cv exchanged, changes the colour layer."""
    orc = _orc()
    R = cpc.T_D_C[:3, :3]
    assert abs(np.linalg.norm(cpc.T_D_C[:3, 3]) - 0.05) < 1e-12
    assert abs(math.degrees(math.acos((np.trace(R) - 1.0) / 2.0)) - 1.0) < 1e-9
    scene = syn.box_with_cube()
    dcs, _, docam = cpc.cameras(cpc.COLOR_DEPTH_CAM)
    (T_D, T_C), = cpc.color_poses(1)
    img = cpc.stripe_image(scene, cpc.COLOR_CAM, T_C)
    base = None
    for variant in ("colour", "depth_camera", "f", "c"):
        oc = orc.OracleMap(cpc.VOXEL)
        oc.integrate_depth(syn.render_depth(scene, dcs, T_D), T_D, docam)
        if variant == "colour":
            cam, T, im = cpc.cameras(cpc.COLOR_CAM)[2], T_C, img
        elif variant == "depth_camera":
            cam, T, im = docam, T_D, cpc.stripe_image(scene, cpc.COLOR_DEPTH_CAM, T_C)
        else:
            cam, T, im = cpc.cameras(cpc.swapped(cpc.COLOR_CAM, variant))[2], T_C, img
        oc.integrate_color(im, T, cam)
        layer = oc.color_layer()
        sig = {k: (b["color"].tobytes(), b["weight"].tobytes()) for k, b in layer.items()}
        if base is None:
            base = sig
            assert len(base) > 300
        else:
            assert sig != base, variant


def test_rig_frames_repeat_poses_and_differ_in_resolution():
    fr = cpc.rig_frames()
    assert {d.shape for _, d, _ in fr} == {(480, 640), (720, 1280), (240, 424)}
    seen = {}
    repeats = 0
    for name, d, T in fr:
        key = (name, T.tobytes())
        repeats += key in seen
        seen[key] = True
    assert repeats >= 3
    for a, b in zip(fr, fr[1:]):
        assert a[0] != b[0] or not np.array_equal(a[1], b[1])  # a repeated pose comes with a new noise draw
