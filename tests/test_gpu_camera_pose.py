"""Every projective consumer with general cameras and poses (tests/camera_pose_cases.py), bit for bit against the oracle:
fu != fv, principal points off the image centre, odd image sizes, lens distortion, pitched, rolled, straight-down and
straight-up views, a pose on a block corner and one kilometres away, a separate colour camera, and a rig of three depth
cameras of different resolutions feeding one mapper through the synchronous, asynchronous and device APIs. The float64
geometry checks of tests/test_oracle_camera_ground_truth.py run on the mapper's layers as well."""
import numpy as np
import pytest

import camera_ground_truth as gt
import camera_pose_cases as cpc
import test_oracle_camera_ground_truth as ogt
from helpers import assert_color_equal, assert_esdf_equal, assert_tsdf_equal
from isaac_ros_nvblox_b200 import synthetic as syn
from test_gpu_dynamics import _detect_and_compare, _static_map
from test_gpu_freespace import assert_freespace_equal
from test_gpu_mesh import assert_mesh_equal
from test_gpu_occupancy import assert_occupancy_equal

pytestmark = pytest.mark.gpu

TRUNC = 4 * cpc.VOXEL


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _blockset(a):
    return set(map(tuple, np.asarray(a).reshape(-1, 3).tolist()))


# ----------------------------------------------------------------------------------------
# View raycast and TSDF / ESDF per case
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(cpc.CASE))
def test_view_raycast_lists(gpu, name):
    """ViewCalculator lists equal the oracle's in content and order; for the tilted, undistorted cases they contain every
    block that holds a float64 back-projected surface point."""
    nvb, orc = _nvb(), _orc()
    case = cpc.CASE[name]
    _, cam, ocam = cpc.cameras(case["cam"])
    m = nvb.Mapper(cpc.VOXEL)
    vc = nvb.ViewCalculator(m)
    d0, T0 = ogt.clean_frame(case)
    for d, T in [(d0, T0)] + cpc.frames(case, 2, seed=1):
        got = vc.get_blocks_in_image_view_raycast(d, T, cam, cpc.BLOCK, TRUNC, 7.0)
        assert np.array_equal(got, orc.view_raycast(d, T, ocam, cpc.BLOCK, TRUNC))
    if name in ogt.RAYCAST_CASES:
        ogt.check_raycast_covers_surface(vc.get_blocks_in_image_view_raycast(d0, T0, cam, cpc.BLOCK, TRUNC, 7.0), d0, case)
    m.close()


@pytest.mark.parametrize("i", range(len(cpc.CASES)))
def test_tsdf_and_esdf_sequence(gpu, i):
    """Three frames per case through integrate_depth and the tracker-driven ESDF, the weighting function cycling over the
    six types with the cases: lists, TSDF bits and ESDF every frame."""
    nvb, orc = _nvb(), _orc()
    case = cpc.CASES[i]
    _, cam, ocam = cpc.cameras(case["cam"])
    wtype = i % 6
    m, o = nvb.Mapper(cpc.VOXEL), orc.OracleMap(cpc.VOXEL)
    m.tsdf_integrator().params(weighting_type=wtype)
    p = orc.default_tsdf_params(weighting_type=wtype)
    for k, (d, T) in enumerate(cpc.frames(case, 3, seed=i)):
        b = m.integrate_depth(d, T, cam)
        bo = o.integrate_depth(d, T, ocam, p)
        assert np.array_equal(b, bo), k
        m.update_esdf()
        o.integrate_esdf(bo if k > 0 else o.tsdf_block_indices())
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert m.tsdf_layer().num_blocks() > case["min_blocks"]
    m.close()


MIXED = ["pitch_down_50", "roll_plus_30", "straight_down", "identity_on_block_corner", "roll_minus_30"]


def _mixed_frames(names=MIXED, n=2):
    """Frames of several cases (different cameras and sizes) interleaved: [(case, depth, T)]."""
    per = [[(cpc.CASE[nm], d, T) for d, T in cpc.frames(cpc.CASE[nm], n, seed=7)] for nm in names]
    return [f for group in zip(*per) for f in group]


def test_occupancy_mapper_mixed_cameras(gpu):
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(cpc.VOXEL, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    o = orc.OracleMap(cpc.VOXEL)
    p, op = orc.default_tsdf_params(), orc.default_occupancy_params()
    for k, (case, d, T) in enumerate(_mixed_frames()):
        _, cam, ocam = cpc.cameras(case["cam"])
        b = m.integrate_depth(d, T, cam)
        bo = o.integrate_occupancy(d, T, ocam, p, op)
        assert np.array_equal(b, bo), k
        m.update_esdf()
        o.integrate_esdf_occupancy(bo if k > 0 else o.occupancy_block_indices())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
    m.close()


def test_freespace_mapper_mixed_cameras(gpu):
    """TSDF with freespace: update_freespace(depth, T, camera) with the frame's own camera (view exclusion at twice the
    truncation), then the freespace ESDF."""
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(cpc.VOXEL, projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)
    o = orc.OracleMap(cpc.VOXEL)
    kw = dict(min_duration_since_occupied_for_freespace_ms=300)
    m.freespace_integrator().params(**kw)
    fp = orc.default_freespace_params(**kw)
    for k, (case, d, T) in enumerate(_mixed_frames(MIXED[:3], 3)):
        _, cam, ocam = cpc.cameras(case["cam"])
        t_ms = 1000 + 150 * k
        b = m.integrate_depth(d, T, cam)
        bo = o.integrate_depth(d, T, ocam)
        assert np.array_equal(b, bo), k
        m.update_freespace(t_ms, depth=d, T_L_C=T, camera=cam)
        o.update_freespace(o.tsdf_block_indices() if k == 0 else bo, t_ms, fp, depth=d, T_L_C=T, cam=ocam,
                           max_view_distance_m=7.0, truncation_distance_m=2 * TRUNC)
        assert_freespace_equal(m.freespace_layer().as_dict(), o.freespace_layer())
        m.update_esdf()
        o.integrate_esdf_with_freespace(o.tsdf_block_indices() if k == 0 else bo)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()


def test_decay_with_views_of_different_cameras(gpu):
    """decay(depth, T, camera) with an earlier frame's camera, then decay_exclude_last_view after a frame of another camera
    and size (the saved last view carries its own camera)."""
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(cpc.VOXEL, keep_last_view=True)
    o = orc.OracleMap(cpc.VOXEL)
    kw = dict(decay_factor=0.5)
    m.tsdf_decay_integrator().params(**kw)
    dp = orc.default_tsdf_decay_params(**kw)
    frames = _mixed_frames(["roll_minus_30", "pitch_down_20", "straight_up"], 2)
    for case, d, T in frames:
        _, cam, ocam = cpc.cameras(case["cam"])
        assert np.array_equal(m.integrate_depth(d, T, cam), o.integrate_depth(d, T, ocam))
    removed = 0
    for it in range(6):
        if it % 2 == 0:
            case, d, T = frames[0]  # the 641 x 481 camera, not the last frame's
            _, cam, ocam = cpc.cameras(case["cam"])
            r = m.decay(depth=d, T_L_C=T, camera=cam)
        else:
            case, d, T = frames[-1]
            _, _, ocam = cpc.cameras(case["cam"])
            r = m.decay_exclude_last_view()
        ro = o.decay_tsdf(dp, depth=d, T_L_C=T, cam=ocam, max_view_distance_m=7.0, truncation_distance_m=TRUNC)
        assert _blockset(r) == _blockset(ro), it
        removed += len(r)
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert removed > 100
    m.close()


# ----------------------------------------------------------------------------------------
# Colour from a separate camera, the sphere tracer, the coloured mesh
# ----------------------------------------------------------------------------------------
def test_colour_from_a_separate_camera(gpu):
    """Depth 640x480, colour 1280x720 with its own intrinsics and a 5 cm / 1 degree offset: colour block lists and layer
    equal the oracle's, the sphere tracer's depth from the colour camera is bit-identical, and the mesh's vertex colours
    equal the oracle's."""
    nvb, orc = _nvb(), _orc()
    _, dcam, docam = cpc.cameras(cpc.COLOR_DEPTH_CAM)
    _, ccam, cocam = cpc.cameras(cpc.COLOR_CAM)
    m, o = nvb.Mapper(cpc.VOXEL), orc.OracleMap(cpc.VOXEL)
    m.color_integrator().params(sphere_tracer_maximum_ray_length_m=15.0)
    cp = orc.default_color_params(sphere_tracer_maximum_ray_length_m=15.0)
    inputs = ogt.colour_inputs()
    for k, (d, T_D, img, T_C) in enumerate(inputs):
        assert np.array_equal(m.integrate_depth(d, T_D, dcam), o.integrate_depth(d, T_D, docam))
        bg, bc = m.integrate_color(img, T_C, ccam), o.integrate_color(img, T_C, cocam, cp)
        assert _blockset(bg) == _blockset(bc) and len(bg) == len(bc) and len(bg) > 100, k
        assert_color_equal(m.color_layer().as_dict(), o.color_layer())
        g = m.color_integrator().render_depth(T_C, ccam, TRUNC, ray_subsampling_factor=4)
        c = o.sphere_trace_image(T_C, cocam, TRUNC, maximum_ray_length_m=15.0, ray_subsampling_factor=4)
        assert g.shape == c.shape == (720 // 4, 1280 // 4)
        assert np.array_equal(g.view(np.uint32), c.view(np.uint32)), np.argwhere(g != c)[:5]
        assert (g > 0).mean() > 0.3  # the walls beyond the layer's edge do not converge
    m.update_mesh()
    o.integrate_mesh()
    o.update_mesh_color()
    mesh = m.mesh_layer().as_dict()
    assert len(mesh) > 100
    assert_mesh_equal(mesh, o.mesh_layer(), colors=True)
    m.close()


# ----------------------------------------------------------------------------------------
# Ground truth on the mapper: colour stripes, the plane, dynamics
# ----------------------------------------------------------------------------------------
def test_colour_from_a_separate_camera_matches_the_world_stripes(gpu):
    nvb = _nvb()
    dcam, ccam = cpc.cameras(cpc.COLOR_DEPTH_CAM)[1], cpc.cameras(cpc.COLOR_CAM)[1]
    m = nvb.Mapper(cpc.VOXEL)
    inputs = ogt.colour_inputs()
    for d, T_D, img, T_C in inputs:
        m.integrate_depth(d, T_D, dcam)
        m.integrate_color(img, T_C, ccam)
    ogt.check_colour_stripes(m.color_layer().as_dict(), syn.box_with_cube(), inputs)
    m.close()


@pytest.mark.parametrize("general", [False, True])
def test_tsdf_symmetric_view_on_plane(gpu, general):
    nvb = _nvb()
    layers = []
    for c, d, T in ogt.plane_frames(general):
        m = nvb.Mapper(cpc.VOXEL)
        m.integrate_depth(d, T, cpc.cameras(c)[1])
        layers.append(m.tsdf_layer().as_dict())
        m.close()
    ogt.check_plane(layers[0], layers[1], cpc.plane_setup(general), general)


def test_dynamics_points_reproject_into_the_box(gpu):
    """Dynamics detection with fu != fv and an off-centre principal point: bit for bit against the restatement on the GPU's
    freespace layer, and every point re-projects (float64) into the box's pixel rectangle."""
    nvb = _nvb()
    c = gt.DYN_CAM
    _, cam, _ = cpc.cameras(c)
    cd = {"fu": cam.fu, "fv": cam.fv, "cu": cam.cu, "cv": cam.cv, "radial": None, "tangential": None}
    T = np.eye(4, dtype=np.float32)
    wall = gt.dynamics_wall()
    m = nvb.Mapper(cpc.VOXEL, projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)
    m._cam = cam
    _static_map(m, wall, T, min_duration_since_occupied_for_freespace_ms=300)
    assert len(_detect_and_compare(m, wall, T, cam, cd)) == 0
    for k in range(len(gt.DYN_BOXES)):
        ogt.check_dynamics_points(_detect_and_compare(m, gt.dynamics_box_frame(wall, k), T, cam, cd), k)
    m.close()


# ----------------------------------------------------------------------------------------
# A rig of three depth cameras feeding one mapper
# ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rig_oracle():
    """The rig frames and, per frame, the oracle's block list, TSDF and ESDF layers."""
    orc = _orc()
    frames = cpc.rig_frames()
    o = orc.OracleMap(cpc.VOXEL)
    out = []
    for k, (name, d, T) in enumerate(frames):
        bo = o.integrate_depth(d, T, cpc.cameras(cpc.RIG_CAMS[name])[2])
        o.integrate_esdf(bo if k > 0 else o.tsdf_block_indices())
        out.append((bo, o.tsdf_layer(), o.esdf_layer()))
    return frames, out


CHECKPOINTS = (2, 5, 8, 10)  # frames after which the asynchronous and device runs synchronise and compare


@pytest.mark.parametrize("api", ["sync", "async", "device"])
def test_rig_of_three_cameras_into_one_mapper(gpu, rig_oracle, api):
    """640x480, 1280x720 and 424x240 depth cameras with their own intrinsics and extrinsics, interleaved into one mapper;
    repeated poses make the two-entry view-point cache hit, miss and evict. Synchronous API: every frame's list, TSDF and
    ESDF. Asynchronous host API (the staging ring regrows while earlier frames are in flight) and device API: several
    frames enqueued between synchronisations, then the last frame's list length, TSDF and ESDF."""
    import torch
    nvb = _nvb()
    frames, want = rig_oracle
    m = nvb.Mapper(cpc.VOXEL)
    dev = [torch.from_numpy(d).cuda() for _, d, _ in frames] if api == "device" else None
    if dev is not None:
        torch.cuda.synchronize()
    lens = []
    for k, (name, d, T) in enumerate(frames):
        cam = cpc.cameras(cpc.RIG_CAMS[name])[1]
        bo, tsdf, esdf = want[k]
        if api == "sync":
            b = m.integrate_depth(d, T, cam)
            assert np.array_equal(b, bo), k
            m.update_esdf()
        elif api == "async":
            m.integrate_depth_async(d, T, cam)
            m.update_esdf(sync=False)
        else:
            m.integrate_depth_device(dev[k].data_ptr(), d.shape[0], d.shape[1], T, cam)
            m.update_esdf(sync=False)
        lens.append(len(bo))
        if api == "sync" or k in CHECKPOINTS:
            m.synchronize()
            assert m.last_frame_block_count() == len(bo), k
            assert_tsdf_equal(m.tsdf_layer().as_dict(), tsdf)
            assert_esdf_equal(m.esdf_layer().as_dict(), esdf)
    # the cache did reuse lists: a repeated pose's list equals its first list although the depth differs
    assert any(lens[i] == lens[j] and frames[i][0] == frames[j][0] and not np.array_equal(frames[i][1], frames[j][1])
               for i in range(len(frames)) for j in range(i))
    m.close()
