"""The SphereTracer renders on the GPU (nvb_render_depth / nvb_render_rgbd, isaac_ros_nvblox_b200.rendering) against their
restatement (tests/render_reference.py, the oracle's cast with the colour lookup): depth and colour bit for bit, on the same
map, and the depth also against the oracle's own depth render. The oracle's copy of a map is made from the GPU mapper's own
TSDF and colour blocks, so what is compared is the render alone (the integrators' parity is tested elsewhere). The library is
built with -fmad=false, so the kernel and the restatement do the same binary32 operations."""
import ctypes as C

import numpy as np
import pytest

import camera_pose_cases as cpc
import render_reference as rr
import scale_edge_cases as sec
from helpers import cameras, sphere_scene_tsdf_layer, textured_image
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _rendering():
    from isaac_ros_nvblox_b200 import rendering
    return rendering


def _oracle_copy(m, color=False):
    """(OracleMap holding the mapper's TSDF blocks, its colour layer as a dict with `color`, else None)."""
    o = _orc().OracleMap(m.voxel_size())
    for k, v in m.tsdf_layer().as_dict().items():
        o.set_tsdf_block(k, v)
    return o, (m.color_layer().as_dict() if color else None)


def _check(m, ref, T, cam, ocam, trunc, f=1, tracer=None):
    """GPU depth and RGBD renders (device tensors) == the restatement's, bit for bit, and the depth == the oracle's depth
    render. Returns (depth, rgb) as numpy arrays."""
    o, layer = ref
    st = tracer or _rendering().SphereTracer()
    kw = dict(maximum_steps=st.maximum_steps(), maximum_ray_length_m=st.maximum_ray_length_m(),
              surface_distance_epsilon_m=np.float32(st.surface_distance_epsilon_vox()) * np.float32(m.voxel_size()),
              ray_subsampling_factor=f)
    d_exp, c_exp = rr.render(o, T, ocam, trunc, layer, **kw)
    assert np.array_equal(d_exp.view(np.uint32), o.sphere_trace_image(T, ocam, trunc, **kw).view(np.uint32))
    d_only = st.render_depth(m, T, cam, trunc, f).cpu().numpy()
    d, c = st.render_rgbd(m, T, cam, trunc, f)
    d, c = d.cpu().numpy(), c.cpu().numpy()
    assert d.shape == d_exp.shape == (cam.height // f, cam.width // f) and c.shape == d.shape + (3,)
    bad = np.argwhere(d.view(np.uint32) != d_exp.view(np.uint32))
    assert bad.size == 0, (bad[:5], d[tuple(bad[0])], d_exp[tuple(bad[0])])
    assert np.array_equal(d_only.view(np.uint32), d.view(np.uint32))
    bad = np.argwhere(np.any(c != c_exp, axis=-1))
    assert bad.size == 0, (bad[:5], c[tuple(bad[0])], c_exp[tuple(bad[0])])
    return d, c


def _host_rgbd(m, T, cam, trunc, f=1, params=None):
    """nvb_render_rgbd with host outputs -> (rc, depth, rgb)."""
    from isaac_ros_nvblox_b200 import _lib
    from isaac_ros_nvblox_b200.mapper import _fp, colmajor
    p = params or _default_params()
    rows, cols = cam.height // f, cam.width // f
    d = np.zeros((rows, cols), np.float32)
    c = np.zeros((rows, cols, 3), np.uint8)
    rc = m._L.nvb_render_rgbd(m._h, C.byref(p), _fp(colmajor(T)), C.byref(cam.c), float(trunc), int(f), _lib.NVB_MEM_HOST,
                              d.ctypes.data, c.ctypes.data, None)
    return rc, d, c


def _default_params():
    from isaac_ros_nvblox_b200 import _lib
    p = _lib.NvbSphereTracerParams()
    _lib.load().nvb_default_sphere_tracer_params(C.byref(p))
    return p


@pytest.fixture(scope="module")
def c2(gpu):
    """bench.py's map: 80 frames of the sphere-in-box circle, 640x480, 5 cm voxels, TSDF plus colour from textured images."""
    import bench
    nvb = _nvb()
    cam_s, frames = bench.make_frames(80, 0, 1)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ocam = _orc().Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    m = nvb.Mapper(0.05)
    for i, (d, T) in enumerate(frames):
        m.integrate_depth(d, T, cam, return_blocks=False)
        if i % 4 == 0:
            m.integrate_color(textured_image(cam_s.height, cam_s.width, seed=i), T, cam, return_blocks=False)
    o = _oracle_copy(m, color=True)
    yield dict(m=m, o=o, frames=frames, cam=cam, ocam=ocam)
    m.close()


@pytest.mark.parametrize("f", [1, 2, 4])
def test_c2_renders_bit_identical(c2, f):
    m, o, cam, ocam = c2["m"], c2["o"], c2["cam"], c2["ocam"]
    for i in (0, 21, 57):
        T = c2["frames"][i][1]
        d, c = _check(m, o, T, cam, ocam, np.float32(0.2), f)
        hit = d > 0
        assert hit.mean() > 0.5
        assert np.any(c[hit] != 0, axis=-1).mean() > 0.5 and np.all(c[~hit] == 0)


def test_c2_host_outputs_equal_device_outputs(c2):
    m, cam = c2["m"], c2["cam"]
    T = c2["frames"][33][1]
    for f in (1, 4):
        rc, dh, ch = _host_rgbd(m, T, cam, 0.2, f)
        assert rc == 0
        d, c = _rendering().SphereTracer().render_rgbd(m, T, cam, 0.2, f)
        assert np.array_equal(dh.view(np.uint32), d.cpu().numpy().view(np.uint32)) and np.array_equal(ch, c.cpu().numpy())


def test_c2_1920x1080(c2):
    nvb = _nvb()
    cam = nvb.Camera(1050.0, 1050.0, 960.0, 540.0, 1920, 1080)
    ocam = _orc().Camera(1050.0, 1050.0, 960.0, 540.0, 1920, 1080)
    for f in (1, 4):
        d, _ = _check(c2["m"], c2["o"], c2["frames"][11][1], cam, ocam, 0.2, f)
        assert (d > 0).mean() > 0.5


def test_short_rays_and_one_step(c2):
    m, o, cam, ocam = c2["m"], c2["o"], c2["cam"], c2["ocam"]
    T = c2["frames"][5][1]
    st = _rendering().SphereTracer()
    st.maximum_steps(1)
    d, c = _check(m, o, T, cam, ocam, 0.2, 2, tracer=st)
    st = _rendering().SphereTracer()
    st.maximum_ray_length_m(1e-3)
    d2, _ = _check(m, o, T, cam, ocam, 0.2, 2, tracer=st)
    assert np.all(d2 == -1.0)  # no ray gets past its first sample
    st = _rendering().SphereTracer()
    st.maximum_steps(7)
    st.surface_distance_epsilon_vox(2.5)
    _check(m, o, T, cam, ocam, 0.2, 1, tracer=st)


def test_nvblox_torch_functions(c2):
    """render_depth_image / render_depth_and_color_image (nvblox_torch's names and argument order) == the oracle with
    truncation 4 voxels, f = 1, the given ray length and steps."""
    import torch
    r = _rendering()
    m, o = c2["m"], c2["o"]
    T = c2["frames"][44][1]
    K = torch.tensor([[300.0, 0, 320.0], [0, 310.0, 250.0], [0, 0, 1]], dtype=torch.float32)
    pose = torch.from_numpy(np.array(T, np.float32))
    ocam = _orc().Camera(300.0, 310.0, 320.0, 250.0, 640, 480)
    d_exp, c_exp = rr.render(o[0], T, ocam, np.float32(0.05) * np.float32(4.0), o[1], maximum_steps=80,
                             maximum_ray_length_m=9.0)
    d = r.render_depth_image(m, pose, K, 480, 640, 9.0, 80)
    d2, c = r.render_depth_and_color_image(m, pose.cuda(), K, 480, 640, 9.0, 80)
    assert d.is_cuda and d.dtype == torch.float32 and d.shape == (480, 640)
    assert c.is_cuda and c.dtype == torch.uint8 and c.shape == (480, 640, 3)
    assert np.array_equal(d.cpu().numpy().view(np.uint32), d_exp.view(np.uint32))
    assert np.array_equal(d2.cpu().numpy().view(np.uint32), d_exp.view(np.uint32))
    assert np.array_equal(c.cpu().numpy(), c_exp)


def _integrated(cs, cam, frames, offset=None):
    """A TSDF + colour mapper (5 cm voxels) from (depth, T) frames; with `offset`, integrated at the shifted poses."""
    m = _nvb().Mapper(0.05)
    if cs.width % 4 or cs.height % 4:  # the colour integrator's own tracer subsamples by 4 unless told otherwise
        m.color_integrator().params(sphere_tracing_ray_subsampling_factor=1)
    for i, (d, T) in enumerate(frames):
        Tm = sec.shifted(T, offset) if offset is not None else T
        m.integrate_depth(d, Tm, cam, return_blocks=False)
        m.integrate_color(textured_image(cs.height, cs.width, seed=i), Tm, cam, return_blocks=False)
    return m


@pytest.mark.parametrize("cam_name", ["aniso_0.9", "aniso_1.1", "half_integer_317x239", "odd_641x481", "distorted"])
def test_general_cameras(gpu, cam_name):
    c = cpc.CAMS[cam_name]
    cs, cam, ocam = cpc.cameras(c)
    scene = syn.sphere_in_box()
    poses = [cpc.f32(cpc.pose64(cpc.looking_at_centre(p, pitch=pitch, roll=roll), p))
             for p, pitch, roll in (((3.0, -1.5, 1.2), -8.0, 4.0), ((-2.5, 2.0, 2.6), 12.0, 0.0))]
    frames = syn.make_sequence(scene, cs, poses + syn.circle_trajectory(24)[::3])
    m = _integrated(cs, cam, frames)
    o = _oracle_copy(m, color=True)
    for T in poses:
        fs = [f for f in (1, 2, 4) if c["width"] % f == 0 and c["height"] % f == 0]
        for f in fs:
            d, _ = _check(m, o, T, cam, ocam, 0.2, f)
            assert (d > 0).mean() > 0.3
    m.close()


@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_from_origin(gpu, offset):
    cs, cam, ocam = cameras(320, 240, f=150.0)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(24)[::4])
    m = _integrated(cs, cam, frames, offset=offset)
    o = _oracle_copy(m, color=True)
    for i in (0, 3):
        d, c = _check(m, o, sec.shifted(frames[i][1], offset), cam, ocam, 0.2, 1)
        assert (d > 0).mean() > 0.3 and np.any(c != 0)
    m.close()


def _hand_mapper(voxel=0.1, color_layer=False, grey_blocks=False):
    """The sphere-in-box ground-truth TSDF (10 cm voxels) on the GPU; optionally colour blocks that were never coloured."""
    nvb = _nvb()
    idx, vox = sphere_scene_tsdf_layer(voxel_size=voxel, truncation_m=0.4)
    m = nvb.Mapper(voxel)
    m.tsdf_layer().set_blocks(idx, vox)
    if grey_blocks:
        blk = np.zeros((len(idx), 8, 8, 8), nvb.mapper.COLOR_VOXEL_DTYPE)
        blk["color"] = 127  # ColorVoxel(): Gray, weight 0
        m.color_layer().set_blocks(idx, blk)
    return m


def test_camera_inside_the_surface(gpu):
    """A camera inside the sphere starts at a negative distance and finds the negative -> positive crossing."""
    m = _hand_mapper()
    o = _oracle_copy(m)
    _, cam, ocam = cameras(320, 240, f=150.0)
    T = np.eye(4, dtype=np.float32)
    T[:3, 3] = (0.1, -0.2, 2.1)  # inside the 2 m sphere centred at (0, 0, 2)
    d, c = _check(m, o, T, cam, ocam, 0.4, 1)
    assert (d > 0).mean() > 0.9 and np.all(c == 0)  # no colour layer: black
    m.close()


def test_mapper_without_colour_layer_renders_black(gpu):
    m = _hand_mapper()
    o = _oracle_copy(m)
    _, cam, ocam = cameras(640, 480)
    for T in syn.circle_trajectory(80)[::20]:
        d, c = _check(m, o, T, cam, ocam, 0.4, 2)
        assert (d > 0).mean() > 0.3 and np.all(c == 0)
    m.close()


def test_uncoloured_blocks_render_grey(gpu):
    m = _hand_mapper(grey_blocks=True)
    o = _oracle_copy(m, color=True)
    _, cam, ocam = cameras(640, 480)
    d, c = _check(m, o, syn.circle_trajectory(80)[9], cam, ocam, 0.4, 1)
    hit = d > 0
    assert hit.mean() > 0.3 and np.all(c[hit] == 127) and np.all(c[~hit] == 0)
    m.close()


def test_empty_map(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.05)
    o = (_orc().OracleMap(0.05), None)
    _, cam, ocam = cameras(320, 240)
    d, c = _check(m, o, syn.circle_trajectory(8)[1], cam, ocam, 0.2, 1)
    assert np.all(d == -1.0) and np.all(c == 0)
    m.close()


def test_render_after_async_integration_sees_the_map(gpu):
    """A device render enqueued right after integrate_depth_async, with no synchronisation, renders the integrated frames."""
    nvb = _nvb()
    cs, cam, ocam = cameras(640, 480)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80)[:3])
    m = nvb.Mapper(0.05)
    st = _rendering().SphereTracer()
    for d, T in frames:
        m.integrate_depth_async(d, T, cam)
    dev, _ = st.render_rgbd(m, frames[-1][1], cam, 0.2)
    got = dev.cpu().numpy()
    m.synchronize()
    o = _oracle_copy(m)
    exp = o[0].sphere_trace_image(frames[-1][1], ocam, 0.2)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)) and (got > 0).mean() > 0.5
    m.close()


def test_argument_errors(gpu):
    from isaac_ros_nvblox_b200 import _lib
    from isaac_ros_nvblox_b200.mapper import _fp, colmajor
    nvb = _nvb()
    m = _hand_mapper()
    _, cam, _ = cameras(320, 240)
    T = _fp(colmajor(np.eye(4, dtype=np.float32)))
    d = np.zeros((240, 320), np.float32)
    c = np.zeros((240, 320, 3), np.uint8)
    p = _default_params()
    L, H = m._L, _lib.NVB_MEM_HOST
    assert L.nvb_render_depth(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, None) == 0
    assert L.nvb_render_rgbd(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, c.ctypes.data, None) == 0
    bad = -1  # NVB_ERR_INVALID_ARGUMENT
    for f in (0, -2, 7):  # the factor must divide 320 x 240
        assert L.nvb_render_depth(m._h, C.byref(p), T, C.byref(cam.c), 0.4, f, H, d.ctypes.data, None) == bad
    for name, v in (("maximum_steps", 0), ("maximum_steps", -3), ("maximum_ray_length_m", 0.0),
                    ("maximum_ray_length_m", -1.0), ("maximum_ray_length_m", float("nan")),
                    ("surface_distance_epsilon_vox", 0.0), ("surface_distance_epsilon_vox", -0.1)):
        q = _default_params()
        setattr(q, name, v)
        assert L.nvb_render_rgbd(m._h, C.byref(q), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, c.ctypes.data, None) == bad
    assert L.nvb_render_depth(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, None, None) == bad
    assert L.nvb_render_rgbd(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, None, None) == bad
    assert L.nvb_render_rgbd(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, None, c.ctypes.data, None) == bad
    assert L.nvb_render_depth(m._h, None, T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, None) == bad
    assert L.nvb_render_depth(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, 7, d.ctypes.data, None) == bad  # memory kind
    import torch
    td, tc = torch.zeros((240, 320), dtype=torch.float32, device="cuda"), torch.zeros((240, 320, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert L.nvb_render_depth(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, 2, td.data_ptr(), None) == bad
    assert L.nvb_render_rgbd(m._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, 2, td.data_ptr(), tc.data_ptr(), None) == bad
    occ = nvb.Mapper(0.1, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    assert L.nvb_render_depth(occ._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, None) == bad
    assert L.nvb_render_rgbd(occ._h, C.byref(p), T, C.byref(cam.c), 0.4, 1, H, d.ctypes.data, c.ctypes.data, None) == bad
    with pytest.raises(Exception):
        _rendering().SphereTracer().render_depth(m, np.eye(4), cam, 0.4, 3)
    occ.close()
    m.close()


def test_rendering_dropin_program(gpu, tmp_path):
    """tests/cpp/test_rendering_dropin.cpp: nvblox_torch's rendering calls through the C++ mirror."""
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_rendering_dropin")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "rendering drop-in ok" in r.stdout
