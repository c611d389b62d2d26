"""The SphereTracer renders' restatement (tests/render_reference.py: depth, and RGBD with the colour lookup) against the
oracle's depth render and the reference's own tests: tests/test_sphere_tracing.cpp's cases that
tests/test_oracle_color_kat.py does not already restate, nvblox_torch's tests/test_rendering.py, and a float64 restatement of
which colour voxel holds each hit point. Also the parameter surface of isaac_ros_nvblox_b200.rendering.SphereTracer and the
C++ drop-in program of nvblox_torch's rendering calls."""
import numpy as np
import pytest

import render_reference as rr
from helpers import cameras, sphere_scene_tsdf_layer, tsdf_layer_from_distance
from isaac_ros_nvblox_b200 import synthetic as syn
from oracle import oracle as orc

F = np.float32


def _map(voxel, idx, vox):
    m = orc.OracleMap(voxel)
    for k, v in zip(idx, vox):
        m.set_tsdf_block(k, v)
    return m


def _rotation(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    x, y, z = axis
    K = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]], float)
    return np.eye(3) + s * K + (1 - c) * K @ K


def test_casting_from_positive_and_negative():
    """CastingFromPositiveAndNegative (test_sphere_tracing.cpp:570-676): a plane tilted by 10 degrees about x and y through
    the origin; rays from the voxel centres of the z = 0 grid go down where the start distance is positive and up where it is
    negative. More than 98 % hit, and the hits lie on average within a voxel of the true intersection."""
    voxel, trunc = 0.05, 0.2
    n = _rotation((1, 0, 0), 10) @ _rotation((0, 1, 0), 10) @ np.array([0.0, 0.0, 1.0])
    idx, vox = tsdf_layer_from_distance(lambda P: (P @ n.astype(F)).astype(F), (-5.0, -5.0, -2.5), (5.0, 5.0, 2.5), voxel, trunc)
    m = _map(voxel, idx, vox)
    # generatePlanarGrid: voxel centres inside the box, half a voxel in from its corners, at height 0
    c = (np.arange(-5.0 + voxel / 2, 5.0, voxel)).astype(F)
    gx, gy = np.meshgrid(c, c, indexing="ij")
    pts = np.stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)], axis=1).astype(F)
    hits, errs = 0, []
    for p in pts[::7]:
        start = float(p.astype(float) @ n)  # the ground-truth distance the voxel holds (|d| < trunc at z = 0 near the plane)
        d = np.array([0.0, 0.0, -1.0 if start >= 0.0 else 1.0], F)
        ok, t = m.sphere_trace_ray(p, d, trunc)
        if not ok:
            continue
        hits += 1
        gt_t = -float(p.astype(float) @ n) / float(d.astype(float) @ n)  # Ray::intersection(plane)
        errs.append(abs(t - gt_t))
    assert hits * 100.0 / len(pts[::7]) > 98.0
    assert np.mean(errs) < voxel


def test_sphere_tracer_parameters():
    """GettersAndSetters (test_sphere_tracing.cpp:520-529), and the setters' CHECK_GTs (sphere_tracer.cu:319-333) as errors."""
    from isaac_ros_nvblox_b200.rendering import SphereTracer
    st = SphereTracer()
    assert (st.maximum_steps(), st.maximum_ray_length_m(), st.surface_distance_epsilon_vox()) == (100, 15.0, F(0.1))
    st.maximum_steps(1)
    st.maximum_ray_length_m(2.0)
    st.surface_distance_epsilon_vox(3.0)
    assert (st.maximum_steps(), st.maximum_ray_length_m(), st.surface_distance_epsilon_vox()) == (1, 2.0, 3.0)
    for setter in (st.maximum_steps, st.maximum_ray_length_m, st.surface_distance_epsilon_vox):
        for bad in (0, -1):
            with pytest.raises(ValueError):
                setter(bad)
    assert (st.maximum_steps(), st.maximum_ray_length_m(), st.surface_distance_epsilon_vox()) == (1, 2.0, 3.0)
    cam = syn.PinholeCamera(300.0, 300.0, 320.0, 240.0, 640, 480)
    assert SphereTracer.get_subsampled_image_size(cam, 4) == (120, 160)


def _layer(idx, fill):
    """A colour layer {block: (8, 8, 8) COLOR_VOXEL_DTYPE} over the blocks idx, fill(block index, voxel grid) -> colours."""
    g = np.indices((8, 8, 8)).transpose(1, 2, 3, 0)
    out = {}
    for k in idx:
        blk = np.zeros((8, 8, 8), orc.COLOR_VOXEL_DTYPE)
        blk["color"] = fill(np.asarray(k), g)
        blk["weight"] = 1.0
        out[tuple(int(c) for c in k)] = blk
    return out


@pytest.mark.parametrize("f", [1, 4])
@pytest.mark.parametrize("distorted", [False, True])
def test_restated_depth_is_the_oracles(f, distorted):
    """The restatement's rays and depth are the oracle's depth render (or_sphere_trace_image) bit for bit, so the colour
    lookup sits on the same t; with the tracer's defaults and with 7 steps."""
    voxel = 0.1
    idx, vox = sphere_scene_tsdf_layer(voxel_size=voxel, truncation_m=0.4)
    m = _map(voxel, idx, vox)
    _, _, cam = cameras(320, 240, radial=(0.05, -0.02, 0.003, 0, 0, 0) if distorted else None,
                        tangential=(0.001, -0.0005) if distorted else None)
    for i, steps, min_hits in ((5, 100, 0.05), (40, 7, 0.0)):
        T = syn.circle_trajectory(80)[i]
        exp = m.sphere_trace_image(T, cam, 0.4, maximum_steps=steps, ray_subsampling_factor=f)
        got, rgb = rr.render(m, T, cam, 0.4, maximum_steps=steps, ray_subsampling_factor=f)
        assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)) and (got > 0).mean() > min_hits
        assert np.all(rgb == 0)  # no colour layer


def test_nvblox_torch_rendering():
    """nvblox_torch tests/test_rendering.py: a 1 m sphere at (0, 0, 3) in a 10 m scene (5 cm voxels, truncation 4 voxels),
    K with a 570 px focal length, the identity pose, ray length 20 m and 100 steps; every colour block red. The depth image
    hits the sphere, and the colour image is (255, 0, 0) exactly where the depth is valid and black elsewhere."""
    voxel = 0.05
    idx, vox = tsdf_layer_from_distance(lambda P: np.linalg.norm(P - np.array([0.0, 0.0, 3.0], F), axis=-1) - F(1.0),
                                        (-5.0,) * 3, (5.0,) * 3, voxel, 4 * voxel)
    m = _map(voxel, idx, vox)
    cam = orc.Camera(570.0, 570.0, 320.0, 240.0, 640, 480)
    T = np.eye(4, dtype=np.float32)
    depth_only = m.sphere_trace_image(T, cam, 4 * voxel, maximum_steps=100, maximum_ray_length_m=20.0)
    assert (depth_only > 0).sum() > 0
    red = _layer(idx, lambda k, g: (255, 0, 0))
    depth, rgb = rr.render(m, T, cam, 4 * voxel, red, maximum_steps=100, maximum_ray_length_m=20.0)
    assert np.array_equal(depth.view(np.uint32), depth_only.view(np.uint32))
    valid = depth > 0
    assert 0.1 < valid.mean() < 0.9
    assert np.all(rgb[valid] == (255, 0, 0)) and np.all(rgb[~valid] == 0)
    assert np.all(depth[~valid] == -1.0)
    # on the sphere: the depth of the nearest point is 2 m, within a voxel
    assert abs(float(depth[240, 320]) - 2.0) < voxel


def _pixel_rays(cam, T, f):
    """The rays of the f-subsampled image in float64: (dir_C z, layer-frame direction), shape (rows, cols) and (rows, cols, 3)."""
    r, c = np.meshgrid(np.arange(cam.height // f), np.arange(cam.width // f), indexing="ij")
    px, py = c * f + f / 2.0, r * f + f / 2.0
    d = np.stack([(px - cam.cu) / cam.fu, (py - cam.cv) / cam.fv, np.ones(px.shape)], axis=-1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d[..., 2], d @ np.asarray(T, float)[:3, :3].T


@pytest.mark.parametrize("f", [1, 3])
def test_hit_colour_is_the_voxel_holding_the_hit_point(f):
    """sphereTracingKernelWithColor (sphere_tracer.cu:239-300): each colour voxel carries its global voxel index (mod 256) as
    its colour; the colour of every hit is the voxel that holds origin + t * dir, restated in float64 from the rendered depth.
    Hit points within 1e-4 m of a voxel face are skipped (binary32 rounding may put them on either side)."""
    voxel = 0.1
    idx, vox = sphere_scene_tsdf_layer(voxel_size=voxel, truncation_m=0.4)
    m = _map(voxel, idx, vox)
    layer = _layer(idx, lambda k, g: (k * 8 + g) % 256)
    cam = orc.Camera(300.0, 300.0, 320.0, 240.0, 640, 480)
    checked = 0
    for i in (3, 29, 61):
        T = syn.circle_trajectory(80)[i]
        depth, rgb = rr.render(m, T, cam, 0.4, layer, ray_subsampling_factor=f)
        dz, dirs = _pixel_rays(cam, T, f)
        hit = depth > 0
        t = depth.astype(float) / dz
        p = np.asarray(T, float)[:3, 3] + t[..., None] * dirs
        q = p / voxel
        far_from_faces = np.all(np.abs(q - np.round(q)) > 1e-4 / voxel, axis=-1)
        sel = hit & far_from_faces
        exp = np.floor(q).astype(np.int64) % 256
        assert np.array_equal(rgb[sel], exp[sel].astype(np.uint8))
        assert np.all(rgb[~hit] == 0)
        checked += int(sel.sum())
    assert checked > 0.2 * 3 * (480 // f) * (640 // f)


def test_rendering_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_rendering_dropin.cpp (nvblox_torch's py_rendering.cpp calls through nvblox/nvblox.h) builds with plain
    g++ against the C-ABI library; without a GPU it reports that and exits 77."""
    import subprocess
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_rendering_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
