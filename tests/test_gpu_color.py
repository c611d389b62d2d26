"""Parity of the colour path (Mapper::integrateColor = ProjectiveColorIntegrator::integrateFrame with its sphere tracer)
with the CPU oracle, through the C-ABI: same updated-block sets, identical colour bytes, bit-identical weights and
synthetic depth images. The reference's own colour-test scenes are replayed on the GPU as well."""
import numpy as np
import pytest

from helpers import (assert_color_equal, assert_tsdf_equal, cameras, points_on_a_sphere, rotation_y, sphere_scene_tsdf_layer,
                     spheres_distance, textured_image, tsdf_layer_from_distance, voxel_at_position)
from isaac_ros_nvblox_b200 import synthetic as syn
from test_gpu_mesh import assert_mesh_equal

pytestmark = pytest.mark.gpu

RED, GREEN, BLUE = (255, 0, 0), (0, 255, 0), (0, 0, 255)


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _solid(color, rows=480, cols=640):
    img = np.zeros((rows, cols, 3), np.uint8)
    img[:] = color
    return img


def _pair_with_layer(voxel, idx, vox):
    nvb, orc = _nvb(), _orc()
    m, o = nvb.Mapper(voxel), orc.OracleMap(voxel)
    m.tsdf_layer().set_blocks(idx, vox)
    for k, v in zip(idx, vox):
        o.set_tsdf_block(k, v)
    return m, o


def _blockset(a):
    return set(map(tuple, np.asarray(a).reshape(-1, 3).tolist()))


def test_sphere_tracer_matches_oracle(gpu):
    nvb, orc = _nvb(), _orc()
    idx, vox = sphere_scene_tsdf_layer(voxel_size=0.1, truncation_m=0.4)
    m, o = _pair_with_layer(0.1, idx, vox)
    cs, cam, ocam = cameras(640, 480)
    m.color_integrator().params(sphere_tracer_maximum_ray_length_m=15.0)
    for i, f in ((0, 1), (7, 4), (23, 2), (41, 8)):
        T = syn.circle_trajectory(80)[i]
        g = m.color_integrator().render_depth(T, cam, 0.4, ray_subsampling_factor=f)
        c = o.sphere_trace_image(T, ocam, 0.4, maximum_ray_length_m=15.0, ray_subsampling_factor=f)
        assert g.shape == c.shape == (480 // f, 640 // f)
        assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), np.argwhere(g != c)[:5]
        assert (g > 0).mean() > 0.3  # the sphere; the walls end at the layer's edge and do not converge
    with pytest.raises(Exception):
        m.color_integrator().render_depth(T, cam, 0.4, ray_subsampling_factor=7)  # must divide the image size
    m.close()


def test_color_ground_truth_field_red_image(gpu):
    """IntegrateColorToGroundTruthDistanceField (tests/test_color_integrator.cpp:225-331) on the GPU, every 4th pose."""
    idx, vox = sphere_scene_tsdf_layer(voxel_size=0.1, truncation_m=0.4)
    m, o = _pair_with_layer(0.1, idx, vox)
    cs, cam, ocam = cameras(640, 480)
    img = _solid(RED)
    for T in syn.circle_trajectory(80)[::4]:
        bg = m.integrate_color(img, T, cam)
        bc = o.integrate_color(img, T, ocam)
        assert _blockset(bg) == _blockset(bc) and len(bg) == len(bc)
    layer = m.color_layer().as_dict()
    assert_color_equal(layer, o.color_layer())
    for blk in layer.values():
        seen = blk["weight"] > 0.0
        assert np.all(blk["color"][seen] == RED) and np.all(blk["color"][~seen] == 127)
    vs = [voxel_at_position(layer, p, 0.1) for p in points_on_a_sphere(2.0, (0.0, 0.0, 2.0))]
    assert all(v is not None for v in vs) and np.mean([v["weight"] >= 1.0 for v in vs]) > 0.5
    assert set(layer) <= _blockset(idx)
    m.close()


def test_colored_spheres_and_occlusion(gpu):
    """ColoredSpheres (:333-440) and OcclusionTesting (:442-508)."""
    centers = [(5.0, 0.0, 0.0), (5.0, 5.0, 0.0), (5.0, 10.0, 0.0)]
    idx, vox = tsdf_layer_from_distance(spheres_distance(centers, 2.0), (-5.0, -5.0, -5.0), (10.0, 15.0, 5.0), 0.1, 0.2)
    m, o = _pair_with_layer(0.1, idx, vox)
    cs, cam, ocam = cameras(640, 480, f=450.0)
    for y, color in zip((0.0, 5.0, 10.0), (RED, GREEN, BLUE)):
        T = rotation_y(np.pi / 2)
        T[:3, 3] = (0.0, y, 0.0)
        assert _blockset(m.integrate_color(_solid(color), T, cam)) == _blockset(o.integrate_color(_solid(color), T, ocam))
    layer = m.color_layer().as_dict()
    assert_color_equal(layer, o.color_layer())
    for c, color in zip(centers, (RED, GREEN, BLUE)):
        obs = [v for v in (voxel_at_position(layer, p, 0.1) for p in points_on_a_sphere(2.0, c)) if v["weight"] >= 1e-3]
        assert len(obs) > 0.2 * 200 and all(tuple(v["color"]) == color for v in obs)
    m.close()
    c1, c2 = (5.0, 0.0, 0.0), (10.0, 0.0, 0.0)
    idx, vox = tsdf_layer_from_distance(spheres_distance([c1, c2], 2.0), (-5.0, -5.0, -5.0), (15.0, 15.0, 5.0), 0.1, 0.4)
    m, o = _pair_with_layer(0.1, idx, vox)
    cs, cam, ocam = cameras(640, 480)
    m.integrate_color(_solid(RED), rotation_y(np.pi / 2), cam)
    o.integrate_color(_solid(RED), rotation_y(np.pi / 2), ocam)
    layer = m.color_layer().as_dict()
    assert_color_equal(layer, o.color_layer())
    for p in points_on_a_sphere(2.0, c2):
        v = voxel_at_position(layer, p, 0.1)
        assert v is None or v["weight"] == 0.0
    m.close()


@pytest.mark.parametrize("distorted", [False, True])
def test_color_on_reconstruction_textured_masked(gpu, distorted):
    """The whole mapper path: depth frames build the TSDF, textured colour frames (with a mask on every other frame, both mask
    modes) paint it; parameters away from the defaults; with and without lens distortion."""
    nvb, orc = _nvb(), _orc()
    kw = dict(radial=(0.05, -0.02, 0.003, 0.0, 0.0, 0.0), tangential=(0.001, -0.0005)) if distorted else {}
    cs, cam, ocam = cameras(320, 240, f=160.0, **kw)
    frames = syn.make_sequence(syn.box_with_cube(), cs, syn.circle_trajectory(40)[:6], noise_sigma_rel=0.002)
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    pk = dict(measurement_weight=0.35, max_weight=1.5, truncation_distance_vox=3.0, max_integration_distance_m=5.0,
              sphere_tracing_ray_subsampling_factor=2, sphere_tracer_maximum_ray_length_m=6.0)
    m.color_integrator().params(**pk)
    op = orc.default_color_params(**pk)
    rng = np.random.default_rng(1)
    for i, (d, T) in enumerate(frames):
        m.integrate_depth(d, T, cam)
        o.integrate_depth(d, T, ocam)
        img = textured_image(240, 320, seed=i)
        mask = (rng.random((240, 320)) < 0.7).astype(np.uint8) if i % 2 else None
        mode = (i // 2) % 2
        bg = m.integrate_color(img, T, cam, mask=mask, mask_mode=mode)
        bc = o.integrate_color(img, T, ocam, op, mask=mask, mask_mode=mode)
        assert _blockset(bg) == _blockset(bc) and len(bg) == len(bc) and len(bg) > 50
        assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    layer = m.color_layer().as_dict()
    w = np.concatenate([b["weight"].ravel() for b in layer.values()])
    assert (w > 0).sum() > 20000 and w.max() == np.float32(1.5)
    assert len({tuple(c) for b in layer.values() for c in b["color"][b["weight"] > 0][::50]}) > 100  # many distinct colours
    m.close()


def test_color_layer_follows_decay_and_occupancy_mapper_ignores_color(gpu):
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240, f=160.0)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:3])
    m, o = nvb.Mapper(0.1), orc.OracleMap(0.1)
    assert m.color_layer().num_blocks() == 0 and m.color_layer().as_dict() == {}
    for d, T in frames:
        m.integrate_depth(d, T, cam), o.integrate_depth(d, T, ocam)
        m.integrate_color(_solid(GREEN, 240, 320), T, cam), o.integrate_color(_solid(GREEN, 240, 320), T, ocam)
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    n0 = m.color_layer().num_blocks()
    # Mapper::decayTsdf deallocates fully decayed blocks from every layer (clearBlocksInLayers, src/mapper/mapper.cpp:546-557)
    m.tsdf_decay_integrator().params(decay_factor=0.1)
    dp = orc.default_tsdf_decay_params(decay_factor=0.1)
    for _ in range(6):
        m.decay()
        o.decay_tsdf(dp)
        assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    assert m.color_layer().num_blocks() < n0
    # painting again after the deallocation reuses freed colour slots, which must come back Gray / weight 0
    for d, T in frames[:2]:
        m.integrate_depth(d, T, cam), o.integrate_depth(d, T, ocam)
        m.integrate_color(_solid(BLUE, 240, 320), T, cam), o.integrate_color(_solid(BLUE, 240, 320), T, ocam)
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    m.update_mesh()
    assert m.mesh_layer().num_blocks() > 0
    m.clear()
    assert m.color_layer().num_blocks() == 0 and m.mesh_layer().num_blocks() == 0
    # the cleared colour and mesh layers take a new map as a fresh mapper would
    o = orc.OracleMap(0.1)
    for d, T in frames:
        m.integrate_depth(d, T, cam), o.integrate_depth(d, T, ocam)
        m.integrate_color(_solid(RED, 240, 320), T, cam), o.integrate_color(_solid(RED, 240, 320), T, ocam)
    m.update_mesh()
    o.integrate_mesh()
    o.update_mesh_color()
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer(), colors=True)
    m.close()
    mo = nvb.Mapper(0.1, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    d, T = frames[0]
    mo.integrate_depth(d, T, cam)
    assert len(mo.integrate_color(_solid(RED, 240, 320), T, cam)) == 0  # "Color is only integrated for Tsdf layers"
    mo.close()


def test_color_parameter_checks(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.05)
    p = m.color_integrator().params()
    assert (p.max_integration_distance_m, p.truncation_distance_vox, p.max_weight, p.sphere_tracing_ray_subsampling_factor) == \
        (7.0, 4.0, 5.0, 4) and abs(p.measurement_weight - 0.8) < 1e-7
    for bad in (dict(measurement_weight=0.0), dict(measurement_weight=1.5), dict(max_weight=0.0),
                dict(sphere_tracing_ray_subsampling_factor=0)):
        with pytest.raises(Exception):
            m.color_integrator().params(**bad)
    cs, cam, _ = cameras(320, 240)
    with pytest.raises(Exception):
        m.integrate_color(np.zeros((240, 320), np.uint8), np.eye(4, dtype=np.float32), cam)
    m.close()


def test_device_resident_frames_stay_asynchronous_and_match(gpu):
    """Depth and colour frames already in HBM (raw device pointers): enqueued without a host synchronisation, same result."""
    import torch
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240, f=160.0)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:5])
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    depth_dev = torch.from_numpy(np.stack([d for d, _ in frames])).cuda()
    imgs = np.stack([textured_image(240, 320, seed=10 + i) for i in range(len(frames))])
    color_dev = torch.from_numpy(imgs).cuda()
    mask = (np.random.default_rng(4).random((240, 320)) < 0.8).astype(np.uint8)
    mask_dev = torch.from_numpy(mask).cuda()
    torch.cuda.synchronize()
    for i, (d, T) in enumerate(frames):
        m.integrate_depth_device(depth_dev[i].data_ptr(), 240, 320, T, cam)
        m.integrate_color_device(color_dev[i].data_ptr(), 240, 320, T, cam, mask_ptr=mask_dev.data_ptr() if i == 3 else 0)
        m.update_esdf(sync=False)
        o.integrate_depth(d, T, ocam)
        bc = o.integrate_color(imgs[i], T, ocam, mask=mask if i == 3 else None)
    m.synchronize()
    assert _blockset(m.last_color_blocks()) == _blockset(bc)
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    m.close()
