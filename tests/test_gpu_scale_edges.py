"""The CUDA path where its kernels switch code paths, against the oracle: view AABBs beyond the raycast's shared-memory
bitset and beyond the compaction's independent-tile limit (the ticketed chained scan, shared with the block-list union),
maps kilometres from the origin and at the 21-bit hash-key limit, ESDF parents more than 15 blocks away, and the
exchange-slab wavefront with reserved SMs. Each case also asserts that it runs the branch it is meant to test
(tests/scale_edge_cases.py; the same preconditions are checked without a GPU in tests/test_scale_edges_guard.py).

Device memory: a default mapper holds ~9 GiB (2^18-block TSDF and ESDF slabs plus the wavefront's two exchange slabs). The
2 cm integrate case grows the TSDF slab to 2^21 blocks (~16 GiB in all); the last case (one 40 m frame on the chained path)
grows it to 2^22 blocks (~17 GiB) and runs alone at the end of the module.
"""
import numpy as np
import pytest

import scale_edge_cases as sec
from helpers import assert_esdf_equal, assert_tsdf_equal, cameras, validate_esdf
from isaac_ros_nvblox_b200 import synthetic as syn
from test_scale_edges_guard import far_frames, far_origin_bounds, far_origin_differences, FAR_SEQ

pytestmark = pytest.mark.gpu

STATS = ("marked", "with_sites", "to_clear", "clear_candidates", "cleared", "swept", "face_passes", "rings")


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _view_pair(m, case, depth, subsample=1):
    """(GPU list, oracle list) of ViewCalculator::getBlocksInImageViewRaycast for a case."""
    orc = _orc()
    _, cam, ocam = cameras(case["width"], case["height"], radial=case.get("radial"), tangential=case.get("tangential"))
    bs, trunc = 8 * case["voxel"], 4 * case["voxel"]
    m.tsdf_integrator().raycast_subsampling_factor(subsample)
    got = _nvb().ViewCalculator(m).get_blocks_in_image_view_raycast(depth, case["pose"], cam, bs, trunc, case["max_dist"])
    p = orc.default_tsdf_params(max_integration_distance_m=case["max_dist"], raycast_subsampling=subsample)
    want = orc.view_raycast(depth, case["pose"], ocam, bs, trunc, p, cap=sec.case_cells(case)[2])
    return got, want


def _assert_path(case, path):
    cells = sec.case_cells(case)[2]
    if path == "smem":
        assert cells * sec.MARGIN <= sec.SMEM_CELLS, cells
    elif path == "global":
        assert sec.MARGIN * sec.SMEM_CELLS <= cells and cells * sec.MARGIN <= sec.CHAINED_CELLS, cells
    else:
        assert cells >= sec.MARGIN * sec.CHAINED_CELLS, cells
    assert case["path"] == path


# ----------------------------------------------------------------------------------------
# 1. View-volume sizes
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("subsample", [1, 3])
@pytest.mark.parametrize("name", [c["name"] for c in sec.VIEW_CASES if c["path"] != "chained"])
def test_view_raycast_global_and_shared_bitset(gpu, name, subsample):
    """viewRaycastKernel<false> (marks straight into the global bitset) for AABBs of 0.6 - 1.1 M cells, and the
    shared-memory kernel just below its limit: content and order equal the oracle's."""
    case = sec.VIEW[name]
    _assert_path(case, case["path"])
    m = _nvb().Mapper(case["voxel"])
    got, want = _view_pair(m, case, sec.random_depth(case, 0), subsample)
    assert len(want) > 1000
    assert np.array_equal(got, want)
    m.close()


def test_view_raycast_chained_compaction_and_union_share_the_ticket_counter(gpu):
    """Bitsets beyond 2^16 words are compacted with the ticketed chained scan. View lists on one mapper that alternate
    chained / small sizes, with a block-list union over a chained-size AABB in between (the union and the view path share
    the mapper's ticket counter and tile states): every list equals the oracle's, the union equals np.unique."""
    import torch
    from isaac_ros_nvblox_b200 import multi_gpu
    big_a, big_b, small = sec.VIEW["640x480_5cm_40m"], sec.VIEW["640x480_5cm_40m_b"], sec.SMALL_VIEW
    for c in (big_a, big_b):
        _assert_path(c, "chained")
    _assert_path(small, "smem")
    assert sec.union_cells() >= sec.MARGIN * sec.CHAINED_CELLS
    a, b = sec.union_lists()
    union_want = np.unique(np.concatenate([a, b]), axis=0)
    padded = np.full((2, len(a), 3), multi_gpu.PAD, np.int32)
    padded[0], padded[1, :len(b)] = a, b
    m = _nvb().Mapper(0.05)
    for step, what in enumerate(("chained_a", "small", "chained_b", "union", "small", "chained_a")):
        if what == "union":
            got = multi_gpu.union_on_device(m, torch.from_numpy(padded.reshape(-1, 3)).cuda()).cpu().numpy()
            assert len(got) == len(union_want) and np.array_equal(np.unique(got, axis=0), union_want), step
            lin = got[:, 0].astype(np.int64) + 1000 * got[:, 1] + 1000000 * got[:, 2].astype(np.int64)
            assert np.all(np.diff(lin) > 0)  # x fastest, then y, then z
            continue
        case = {"chained_a": big_a, "chained_b": big_b, "small": small}[what]
        got, want = _view_pair(m, case, sec.random_depth(case, step))
        assert len(want) > 1000 and np.array_equal(got, want), (step, what)
    m.close()


def _integrate_pair(voxel, frames, cam, ocam, max_dist, esdf=True, mapper_kw=None):
    nvb, orc = _nvb(), _orc()
    m, o = nvb.Mapper(voxel, **(mapper_kw or {})), orc.OracleMap(voxel)
    m.tsdf_integrator().params(max_integration_distance_m=max_dist)
    p = orc.default_tsdf_params(max_integration_distance_m=max_dist)
    for i, (depth, T) in enumerate(frames):
        b = m.integrate_depth(depth, T, cam)
        bo = o.integrate_depth(depth, T, ocam, p)
        assert np.array_equal(b, bo), i
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
        if esdf:
            m.update_esdf()
            o.integrate_esdf(bo if i > 0 else o.tsdf_block_indices())
            assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    return m, o


def test_integrate_2cm_10m_over_the_shared_memory_bitset(gpu):
    """Three noisy frames at 2 cm voxels and a 10 m range (view AABBs of ~0.9 - 1.1 M cells): lists, TSDF and ESDF every
    frame."""
    for c in sec.INTEGRATE_2CM:
        _assert_path(c, "global")
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, [c["pose"] for c in sec.INTEGRATE_2CM], noise_sigma_rel=0.01, seed=4)
    m, _ = _integrate_pair(0.02, frames, cam, ocam, 10.0)
    m.close()


@pytest.mark.parametrize("subsample", [1, 3])
@pytest.mark.parametrize("size", [(1280, 720), (848, 480)])
def test_large_frames_at_the_default_range(gpu, size, subsample):
    """1280x720 and 848x480 (a width that is not a multiple of the 16-ray tile) through raycast, TSDF and ESDF."""
    w, h = size
    cs, cam, ocam = cameras(w, h)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:3], noise_sigma_rel=0.005, seed=9)
    nvb, orc = _nvb(), _orc()
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    m.tsdf_integrator().raycast_subsampling_factor(subsample)
    p = orc.default_tsdf_params(raycast_subsampling=subsample)
    for i, (depth, T) in enumerate(frames):
        b = m.integrate_depth(depth, T, cam)
        assert np.array_equal(b, o.integrate_depth(depth, T, ocam, p)), i
        m.update_esdf()
        o.integrate_esdf(b if i > 0 else o.tsdf_block_indices())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    m.close()


# ----------------------------------------------------------------------------------------
# 2. Far from the origin and at the hash-key limit
# ----------------------------------------------------------------------------------------
def _assert_mesh_equal(m, o):
    g, c = m.mesh_layer().as_dict(), o.mesh_layer()
    assert set(g) == set(c) and len(c) > 0
    for k in c:
        for f in ("vertices", "normals", "triangles"):
            assert np.array_equal(g[k][f], c[k][f]), (k, f)


@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_origin_sequence(gpu, offset):
    """Poses kilometres from the origin (large block indices of both signs, coarse float32 positions): lists, TSDF, ESDF and
    mesh equal the oracle's every frame, and the TSDF equals the same sequence integrated at the origin up to float32
    rounding at the offset (bounds calibrated on the oracle in tests/test_scale_edges_guard.py)."""
    nvb, orc = _nvb(), _orc()
    frames, cam, ocam = far_frames()
    m, o = nvb.Mapper(FAR_SEQ["voxel"]), orc.OracleMap(FAR_SEQ["voxel"])
    near = nvb.Mapper(FAR_SEQ["voxel"])
    for i, (depth, T) in enumerate(frames):
        Tf = sec.shifted(T, offset)
        b = m.integrate_depth(depth, Tf, cam)
        bo = o.integrate_depth(depth, Tf, ocam)
        assert np.array_equal(b, bo), i
        near.integrate_depth(depth, T, cam)
        m.update_esdf()
        o.integrate_esdf(bo if i > 0 else o.tsdf_block_indices())
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        _assert_mesh_equal(m, o)
    far_layer = m.tsdf_layer().as_dict()
    assert max(abs(int(c)) for k in far_layer for c in k) > 5000
    diff, matched = far_origin_differences(far_layer, near.tsdf_layer().as_dict(), offset, FAR_SEQ["voxel"])
    med, p99 = far_origin_bounds(offset)
    assert matched > 0.995
    assert np.median(diff) <= med and np.percentile(diff, 99) <= p99, (np.median(diff), np.percentile(diff, 99), med, p99)
    m.close(), near.close()


@pytest.mark.parametrize("mode", [3, 2, 1, 0])
@pytest.mark.parametrize("where", list(sec.KEY_LIMIT_SHIFTS))
def test_blocks_at_the_hash_key_limit(gpu, where, mode):
    """TSDF blocks of a sphere at block indices next to +-2^20 (the 21-bit key's bias limit; their neighbours beyond the limit
    cannot exist): ESDF under every wavefront mode and the mesh equal the oracle's."""
    nvb, orc = _nvb(), _orc()
    idx, vox = sec.key_limit_blocks(where)
    assert np.any(idx == sec.KEY_LIMIT - 1) or np.any(idx == -sec.KEY_LIMIT)
    m, o = nvb.Mapper(0.05, esdf_persistent=mode), orc.OracleMap(0.05)
    m.tsdf_layer().set_blocks(idx, vox)
    for k, v in zip(idx, vox):
        o.set_tsdf_block(k, v)
    m.esdf_integrator().integrate_blocks(idx)
    o.integrate_esdf(idx)
    e = o.esdf_layer()
    assert sum(int(b["is_site"].sum()) for b in e.values()) > 100
    assert_esdf_equal(m.esdf_layer().as_dict(), e)
    validate_esdf(m.esdf_layer().as_dict(), (2.0 / 0.05) ** 2)
    if mode == 3:
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        _assert_mesh_equal(m, o)
    m.close()


def test_view_raycast_beyond_the_key_limit(gpu):
    """The view calculator does not touch the hash: a pose ~430 km out (beyond 2^20 blocks of 0.4 m) gives the oracle's list."""
    cs, cam, ocam = cameras(320, 240)
    T = sec.shifted(syn.circle_pose(0.4), (430000.0, -1000.0, 10.0))
    depth = syn.render_depth(syn.sphere_in_box(), cs, syn.circle_pose(0.4))
    m = _nvb().Mapper(0.05)
    got = _nvb().ViewCalculator(m).get_blocks_in_image_view_raycast(depth, T, cam, 0.4, 0.2, 7.0)
    want = _orc().view_raycast(depth, T, ocam, 0.4, 0.2)
    assert len(want) > 1000 and got[:, 0].min() >= sec.KEY_LIMIT
    assert np.array_equal(got, want)
    m.close()


def test_frame_crossing_the_key_limit_raises_then_clear_recovers(gpu):
    """A frame whose view straddles x = 2^20 blocks reports NVB_ERR_INDEX_RANGE. Its in-range blocks are allocated and
    integrated before the error is read back (DESIGN.md section 5); clear() then gives a map that equals the oracle's
    again."""
    from isaac_ros_nvblox_b200._lib import NvbError
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras(320, 240)
    T0 = syn.circle_pose(0.0)  # looks towards -x from x = 4
    depth = syn.render_depth(syn.sphere_in_box(), cs, T0)
    limit_m = sec.KEY_LIMIT * 0.4
    T = sec.shifted(T0, (limit_m + 2.0, 0.0, 0.0))  # the far wall lies below the limit, the camera above it
    m = nvb.Mapper(0.05)
    with pytest.raises(NvbError) as e:
        m.integrate_depth(depth, T, cam)
    assert e.value.code == -4
    left = m.tsdf_layer().get_all_block_indices()
    assert len(left) > 0 and np.all(left[:, 0] < sec.KEY_LIMIT)  # the in-range part of the frame was integrated
    m.clear()
    assert m.tsdf_layer().num_blocks() == 0
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:2])
    o = orc.OracleMap(0.05)
    for i, (d, Ti) in enumerate(frames):
        b = m.integrate_depth(d, Ti, cam)
        bo = o.integrate_depth(d, Ti, ocam)
        assert np.array_equal(b, bo)
        m.update_esdf()
        o.integrate_esdf(bo if i > 0 else o.tsdf_block_indices())
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


# ----------------------------------------------------------------------------------------
# 3. ESDF at long range, 4. reserved SMs
# ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def long_range_oracle():
    """The oracle's ESDF layer and statistics after each step of the long-range scene."""
    orc = _orc()
    o = orc.OracleMap(sec.LR_VOXEL)
    ep = orc.default_esdf_params(max_esdf_distance_m=sec.LR_MAX_DIST)
    out = []
    for (idx, vox), upd in sec.lr_steps():
        for k, v in zip(idx, vox):
            o.set_tsdf_block(k, v)
        o.integrate_esdf(upd, ep)
        out.append((o.esdf_layer(), o.esdf_stats()))
    return out


def _run_long_range(want, mode, reserved=None):
    m = _nvb().Mapper(sec.LR_VOXEL, esdf_persistent=mode)
    m.esdf_integrator().params(max_esdf_distance_m=sec.LR_MAX_DIST)
    if reserved is not None:
        m.esdf_reserved_sms(reserved)
        assert m.esdf_reserved_sms() == reserved
    for i, ((idx, vox), upd) in enumerate(sec.lr_steps()):
        m.tsdf_layer().set_blocks(idx, vox)
        m.esdf_integrator().integrate_blocks(upd)
        layer = m.esdf_layer().as_dict()
        assert_esdf_equal(layer, want[i][0])
        s = m.esdf_integrator().last_stats()
        for k in STATS:
            if mode == 2 and k == "clear_candidates":  # (the gather-replay wavefront does not count them)
                continue
            assert s[k] == want[i][1][k], (i, k, s, want[i][1])
        assert min(sec.far_parent_voxels(layer)) > 10000, i  # parents more than 15 blocks away: the "unknown box" branch
        validate_esdf(layer, (sec.LR_MAX_DIST / sec.LR_VOXEL) ** 2)
    m.close()


@pytest.mark.parametrize("mode,prune", [(3, "1"), (3, "0"), (2, "1"), (1, "1"), (0, "1")])
def test_esdf_long_range_parents_beyond_15_blocks(gpu, monkeypatch, long_range_oracle, mode, prune):
    """2 cm voxels, 4 m ESDF range over a 40 x 40 x 6 block slab of observed free space with site clusters: a full update,
    a cluster removed (the clear pass on blocks whose parent box is "unknown"), a cluster added. Layers and statistics equal
    the oracle's for every wavefront, with the clear-pass pruning on and off."""
    monkeypatch.setenv("NVB_CLEAR_PRUNE", prune)
    assert long_range_oracle[1][1]["cleared"] > 1000
    _run_long_range(long_range_oracle, mode)


@pytest.mark.parametrize("reserved", [0, 2, 36, 64])
def test_esdf_wavefront_with_reserved_sms(gpu, long_range_oracle, reserved):
    """The exchange-slab wavefront launched on fewer CTAs (SMs left to other kernels): its candidate-record segments follow
    the launched grid. Long-range scene, and a full-layer update of a 640x480 map."""
    _run_long_range(long_range_oracle, 3, reserved)
    nvb, orc = _nvb(), _orc()
    cs, cam, ocam = cameras()
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80)[:4])
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    m.esdf_reserved_sms(reserved)
    assert m.esdf_reserved_sms() == reserved
    for depth, T in frames:
        m.integrate_depth(depth, T, cam)
        o.integrate_depth(depth, T, ocam)
    m.update_esdf(update_full_layer=True)
    o.integrate_esdf(o.tsdf_block_indices())
    s, so = m.esdf_integrator().last_stats(), o.esdf_stats()
    for k in STATS:
        assert s[k] == so[k], (k, s, so)
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


# ----------------------------------------------------------------------------------------
# Last: the largest allocation of the module
# ----------------------------------------------------------------------------------------
def test_integrate_one_frame_on_the_chained_path(gpu):
    """One frame with a 40 m range at 5 cm (~3.5 M view cells: the chained compaction with allocation). Needs ~17 GiB of
    device memory: the frame grows the TSDF slab to 2^22 blocks (16 GiB). One frame, and the mapper is closed."""
    case = sec.INTEGRATE_CHAINED
    _assert_path(case, "chained")
    assert sec.case_cells(case)[2] < sec.TSDF_SLAB_LIMIT_CELLS
    cs, cam, ocam = cameras(case["width"], case["height"])
    depth = syn.render_depth(syn.box_with_cube(), cs, case["pose"], max_dist=case["max_dist"])
    # (small initial slabs and no exchange-slab scratch: the TSDF slab is the only large allocation)
    m, _ = _integrate_pair(case["voxel"], [(depth, case["pose"])], cam, ocam, case["max_dist"], esdf=False,
                           mapper_kw=dict(tsdf_capacity_blocks=1024, esdf_capacity_blocks=1024, esdf_persistent=1))
    m.close()
