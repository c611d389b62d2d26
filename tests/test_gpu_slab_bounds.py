"""Block writes through nvb_layer_set_blocks reserve room in the slab they write, whichever layer holds it: the projective
slab of an occupancy mapper grows and counts the blocks in its fill-level bound like a TSDF slab does, the ESDF consumer
sees them, and a slab that follows the projective slab (colour) grows with it."""
import numpy as np
import pytest

from helpers import assert_esdf_equal, cameras
from isaac_ros_nvblox_b200 import synthetic as syn
from test_gpu_occupancy import assert_occupancy_equal

pytestmark = pytest.mark.gpu


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _occupancy_mapper(voxel, **kw):
    nvb = _nvb()
    return nvb.Mapper(voxel, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy, **kw)


def _distinct_blocks(n, origin=(0, 0, 0), side=16):
    """n distinct block indices filling a side x side x ... box from `origin`."""
    i = np.arange(n)
    return (np.stack([i % side, (i // side) % side, i // (side * side)], axis=1) + np.asarray(origin)).astype(np.int32)


def test_occupancy_set_blocks_grows_the_projective_slab(gpu):
    nvb = _nvb()
    m = _occupancy_mapper(0.05, tsdf_capacity_blocks=1024)
    idx = _distinct_blocks(1500)
    vox = np.zeros((len(idx), 8, 8, 8), nvb.OCCUPANCY_VOXEL_DTYPE)
    vox["log_odds"] = np.random.default_rng(3).normal(size=(len(idx), 8, 8, 8)).astype(np.float32)
    m.occupancy_layer().set_blocks(idx, vox)
    assert m.occupancy_layer().num_blocks() == 1500
    got, found = m.occupancy_layer().get_blocks(idx)
    assert found.all() and np.array_equal(got, vox)
    m.close()


def test_occupancy_set_blocks_counts_in_the_projective_bound(gpu):
    """Blocks written close to the slab's capacity, away from the camera, then a frame whose view AABB (648 blocks) fits the
    capacity on its own but not beside the written blocks: the frame grows the slab instead of overflowing it."""
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(160, 120)
    T = np.eye(4, dtype=np.float32)
    depth = syn.render_depth(syn.plane_scene(1.5), cs, T)
    m = _occupancy_mapper(0.05, tsdf_capacity_blocks=1024)
    o = orc.OracleMap(0.05)
    m.occupancy_integrator().params(max_integration_distance_m=2.0)
    idx = _distinct_blocks(1000, origin=(100, 0, 0))
    vox = np.zeros((len(idx), 8, 8, 8), nvb.OCCUPANCY_VOXEL_DTYPE)
    vox["log_odds"] = np.random.default_rng(4).normal(size=(len(idx), 8, 8, 8)).astype(np.float32)
    m.occupancy_layer().set_blocks(idx, vox)
    for k, v in zip(idx, vox["log_odds"]):
        o.set_occupancy_block(k, v)
    b_gpu = m.integrate_depth(depth, T, cam)
    b_cpu = o.integrate_occupancy(depth, T, ocam, orc.default_tsdf_params(max_integration_distance_m=2.0))
    assert len(b_cpu) > 1024 - len(idx)  # the frame's blocks do not fit beside the written ones
    assert np.array_equal(b_gpu, b_cpu)
    assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
    m.close()


def test_occupancy_set_blocks_reach_a_started_esdf(gpu):
    """update_esdf on the empty map starts the ESDF consumer; blocks written afterwards are in the next update."""
    nvb, orc = _nvb(), _orc()
    voxel = 0.2
    scene = syn.sphere_in_box()
    m = _occupancy_mapper(voxel)
    o = orc.OracleMap(voxel)
    m.esdf_integrator().params(max_esdf_distance_m=4.0)
    m.update_esdf()
    ii = np.indices((8, 8, 8)).reshape(3, -1).T + 0.5
    keys, blocks = [], []
    for x in range(-4, 4):
        for y in range(-4, 4):
            for z in range(-1, 4):
                pos = (np.array([x, y, z]) * 8 + ii) * voxel
                occ = scene.distance(pos) <= np.sqrt(3.0) * voxel / 2.0
                blk = np.where(occ, np.float32(6.9), np.float32(-6.9)).astype(np.float32).reshape(8, 8, 8)
                keys.append((x, y, z)), blocks.append(blk)
                o.set_occupancy_block((x, y, z), blk)
    keys = np.asarray(keys, np.int32)
    vox = np.zeros((len(keys), 8, 8, 8), nvb.OCCUPANCY_VOXEL_DTYPE)
    vox["log_odds"] = np.stack(blocks)
    m.occupancy_layer().set_blocks(keys, vox)
    m.update_esdf()
    o.integrate_esdf_occupancy(keys, orc.default_esdf_params(max_esdf_distance_m=4.0))
    e_gpu, e_cpu = m.esdf_layer().as_dict(), o.esdf_layer()
    assert len(e_cpu) == len(keys)
    assert_esdf_equal(e_gpu, e_cpu)
    m.close()


def test_color_set_blocks_grow_the_color_slab(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=1024)
    idx = _distinct_blocks(1500, origin=(-8, -8, 0))
    rng = np.random.default_rng(5)
    vox = np.zeros((len(idx), 8, 8, 8), nvb.COLOR_VOXEL_DTYPE)
    vox["color"] = rng.integers(0, 256, size=(len(idx), 8, 8, 8, 3), dtype=np.uint8)
    vox["weight"] = rng.random(size=(len(idx), 8, 8, 8)).astype(np.float32)
    m.color_layer().set_blocks(idx, vox)
    assert m.color_layer().num_blocks() == 1500
    got, found = m.color_layer().get_blocks(idx)
    assert found.all() and np.array_equal(got, vox)
    m.close()
