"""Parity of the pipeline bench.py TIMES with the CPU oracle, at the bench's full size.

bench.py's `value` comes from device-resident frames pushed through `integrate_depth_device` +
`update_esdf(sync=False)`: no host synchronisation between frames, the ESDF chain of frame k on the mapper's side
stream while the raycast / compaction / TSDF update of frame k+1 runs on the main stream. These tests run exactly
that on the whole 80-frame 640x480 C2 sequence (and its colour leg, the 2 cm shape, a layer growth in the middle
of the asynchronous sequence) and compare block lists, TSDF bits and all five EsdfVoxel fields with the oracle.
"""
import numpy as np
import pytest

from helpers import ESDF_FIELDS, assert_color_equal, assert_esdf_equal, assert_tsdf_equal, cameras, layer_checksum
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

ROWS, COLS = 480, 640


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _bench_frames(n=80):
    import bench
    cam_s, frames = bench.make_frames(n, 0, 1)
    assert (cam_s.width, cam_s.height) == (COLS, ROWS)
    return cam_s, frames


def _device_frames(frames):
    import torch
    depth = torch.from_numpy(np.stack([d for d, _ in frames])).cuda()
    return depth


def _oracle_sequence(frames, ocam, voxel, colors=None):
    orc = _orc()
    o = orc.OracleMap(voxel)
    lists = []
    for i, (depth, T) in enumerate(frames):
        b = o.integrate_depth(depth, T, ocam)
        if colors is not None:
            o.integrate_color(colors[i], T, ocam)
        o.integrate_esdf(b)
        lists.append(b)
    return o, lists


@pytest.fixture(scope="module")
def c2(gpu):
    """The bench's workload and the oracle's map of it (built once, ~4 s)."""
    nvb, orc = _nvb(), _orc()
    cam_s, frames = _bench_frames(80)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ocam = orc.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    o, lists = _oracle_sequence(frames, ocam, 0.05)
    return dict(frames=frames, cam=cam, ocam=ocam, oracle=o, lists=lists)


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_bench_pipeline_async_80_frames_equals_oracle(c2, mode):
    """The timed pipeline, verbatim (bench.py step_device), twice in a row on the same mapper like the bench's
    warm-up + timed steps; every wavefront formulation the library ships."""
    nvb = _nvb()
    frames, cam = c2["frames"], c2["cam"]
    depth_dev = _device_frames(frames)
    m = nvb.Mapper(0.05, esdf_persistent=mode)
    for rep in range(2):
        m.clear()
        for i, (_, T) in enumerate(frames):
            m.integrate_depth_device(depth_dev[i].data_ptr(), ROWS, COLS, T, cam)
            m.update_esdf(sync=False)
        m.synchronize()
        assert_tsdf_equal(m.tsdf_layer().as_dict(), c2["oracle"].tsdf_layer())
        assert_esdf_equal(m.esdf_layer().as_dict(), c2["oracle"].esdf_layer())
    m.close()


def test_bench_e2e_sync_80_frames_lists_equal_oracle(c2):
    """The `e2e` leg (synchronous calls, host depth, updated_blocks read back per frame): every frame's block list
    equal to the oracle's in content and order, final layers equal."""
    nvb = _nvb()
    m = nvb.Mapper(0.05)
    for (depth, T), want in zip(c2["frames"], c2["lists"]):
        got = m.integrate_depth(depth, T, c2["cam"])
        assert np.array_equal(got, want)
        m.update_esdf()
    assert_tsdf_equal(m.tsdf_layer().as_dict(), c2["oracle"].tsdf_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), c2["oracle"].esdf_layer())
    m.close()


def test_bench_pipeline_async_host_frames_equals_oracle(c2):
    """The `e2e.async_api` leg: host frames through the staging ring, no synchronisation until the end."""
    import torch
    nvb = _nvb()
    frames = c2["frames"]
    host = torch.from_numpy(np.stack([d for d, _ in frames])).pin_memory()
    m = nvb.Mapper(0.05)
    for i, (_, T) in enumerate(frames):
        m.integrate_depth_host_ptr_async(host[i].data_ptr(), ROWS, COLS, T, c2["cam"])
        m.update_esdf(sync=False)
    m.synchronize()
    assert layer_checksum(m.tsdf_layer().as_dict(), ("distance", "weight")) == layer_checksum(c2["oracle"].tsdf_layer(), ("distance", "weight"))
    assert layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS) == layer_checksum(c2["oracle"].esdf_layer(), ESDF_FIELDS)
    m.close()


def test_bench_with_color_leg_equals_oracle(gpu):
    """bench.py's `with_color` leg (BASELINE configs[1]: TSDF + colour + ESDF) on 640x480 over the whole 80-frame sequence:
    depth frame, colour frame, ESDF update per frame, all asynchronous and device-resident."""
    import torch
    nvb, orc = _nvb(), _orc()
    cam_s, frames = _bench_frames(80)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ocam = orc.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    yy, xx = np.mgrid[0:ROWS, 0:COLS]
    base = np.stack([xx * 255 // (COLS - 1), yy * 255 // (ROWS - 1), ((xx // 16 + yy // 16) % 2) * 200 + 20], axis=-1)
    colors = np.stack([np.roll(base, 7 * i, axis=1) for i in range(len(frames))]).astype(np.uint8)
    o, _ = _oracle_sequence(frames, ocam, 0.05, colors)
    depth_dev, color_dev = _device_frames(frames), torch.from_numpy(colors).cuda()
    m = nvb.Mapper(0.05)
    for i, (_, T) in enumerate(frames):
        m.integrate_depth_device(depth_dev[i].data_ptr(), ROWS, COLS, T, cam)
        m.integrate_color_device(color_dev[i].data_ptr(), ROWS, COLS, T, cam)
        m.update_esdf(sync=False)
    m.synchronize()
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


def test_redwood_shape_2cm_full_size_equals_oracle(gpu):
    """BASELINE configs[2] shape: 640x480 at 2 cm voxels (the block count per frame is ~10x the 5 cm one), 4 frames,
    asynchronous device-resident pipeline."""
    nvb, orc = _nvb(), _orc()
    cam_s, frames = _bench_frames(80)
    frames = frames[:4]
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ocam = orc.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    o, lists = _oracle_sequence(frames, ocam, 0.02)
    depth_dev = _device_frames(frames)
    m = nvb.Mapper(0.02)
    for i, (_, T) in enumerate(frames):
        m.integrate_depth_device(depth_dev[i].data_ptr(), ROWS, COLS, T, cam)
        m.update_esdf(sync=False)
    m.synchronize()
    assert m.last_frame_block_count() == len(lists[-1])
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


@pytest.mark.parametrize("mode", [1, 3])
def test_async_pipeline_with_layer_growth_mid_sequence(c2, mode):
    """A slab that is too small forces LayerSlab::grow (a synchronising reallocation of both layers and of the ESDF scratch)
    while wavefronts of earlier frames are in flight on the side stream."""
    nvb = _nvb()
    frames = c2["frames"][:24]
    orc = _orc()
    o, _ = _oracle_sequence(frames, c2["ocam"], 0.05)
    depth_dev = _device_frames(frames)
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=2048, esdf_capacity_blocks=2048, esdf_persistent=mode)
    for i, (_, T) in enumerate(frames):
        m.integrate_depth_device(depth_dev[i].data_ptr(), ROWS, COLS, T, c2["cam"])
        m.update_esdf(sync=False)
    m.synchronize()
    assert m.tsdf_layer().num_blocks() > 2048
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


def test_threedmatch_reference_data_equals_oracle(gpu):
    """The reference's own real-data fixture (nvblox/tests/data/3dmatch/seq-01; tests/golden/threedmatch_seq01.npz): five real
    640x480 depth frames (13 % invalid pixels), the colour image of the first, an ESDF update per frame. Per-frame block lists,
    TSDF bits, colour bytes and all five EsdfVoxel fields equal to the oracle's, and to the committed checksums."""
    import os
    import sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    import make_threedmatch_fixture as mk
    nvb = _nvb()
    fx = np.load(os.path.join(golden, "threedmatch_seq01.npz"))
    K = fx["intrinsics"]
    o, lists = mk.run_oracle(K, fx["depth_u16"], fx["poses"], fx["color0"], float(fx["voxel_size"]))
    cam = nvb.Camera(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 640, 480)
    m = nvb.Mapper(float(fx["voxel_size"]))
    for i in range(len(fx["depth_u16"])):
        b = m.integrate_depth(mk.depth_to_float(fx["depth_u16"][i]), fx["poses"][i], cam)
        assert np.array_equal(b, lists[i]) and np.array_equal(b, fx["blocks_%d" % i]), i
        if i == 0:
            m.integrate_color(fx["color0"], fx["poses"][0], cam)
        m.update_esdf()
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert layer_checksum(m.tsdf_layer().as_dict(), ("distance", "weight")) == int(fx["tsdf_checksum"])
    assert layer_checksum(m.esdf_layer().as_dict(), ESDF_FIELDS) == int(fx["esdf_checksum"])
    assert layer_checksum(m.color_layer().as_dict(), ("color", "weight")) == int(fx["color_checksum"])
    m.close()
