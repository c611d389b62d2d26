"""The colour, mesh, occupancy, decay, freespace and slice paths past the sizes and coordinates where their kernels switch
code paths, against the oracle: deallocations of more blocks than the remove kernels' grid, a free stack that runs dry
inside one allocation launch, slabs that grow while their free stacks are not empty, mesh-arena repacks past 2^22
entries and right after a large removal, occupancy behind the global-bitset and chained view paths and with parents
more than 15 blocks away, capped ESDF mark grids with occupancy and freespace, slicer images of millions of pixels, and
colour, mesh and slices kilometres from the origin and at the hash-key limit. Each case asserts the branch it runs from
what the library reports (slab and arena statistics, removed-block counts); the configurations are in
tests/scale_edge_cases.py and their preconditions are checked without a GPU in tests/test_scale_edges_guard.py.

Device memory: the churn cases grow the TSDF slab to 2^19 blocks (2 GiB; the colour and freespace slabs follow it); the
last case (one 40 m occupancy frame on the chained path) grows the occupancy slab to 2^22 blocks (8 GiB). Mappers are
closed between cases.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import scale_edge_cases as sec
from helpers import (assert_color_equal, assert_esdf_equal, assert_tsdf_equal, cameras, sort_rows, textured_image,
                     unit_plane, validate_esdf)
from isaac_ros_nvblox_b200 import synthetic as syn
from test_gpu_freespace import assert_freespace_equal
from test_gpu_mesh import assert_mesh_equal
from test_gpu_occupancy import assert_occupancy_equal
from test_scale_edges_guard import FAR_SEQ, far_frames

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _orc():
    from oracle import oracle as orc
    return orc


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------
# 1. Deallocation, slot reuse and slab growth
# ----------------------------------------------------------------------------------------
def test_decay_churn_tsdf_with_freespace_colour_and_mesh(gpu):
    """2 cm map with freespace, colour, ESDF and a coloured mesh from a 4096-block slab: three frames, a decay that removes
    everything outside a sphere (more blocks than the remove kernels' 1184 CTAs, in every layer), an ESDF update over the
    remaining map, then a 7 m frame that needs more new blocks than the free stacks hold and grows the slabs while the
    stacks are full. Every layer, block list and removed set equals the oracle's after every step."""
    nvb, orc = _nvb(), _orc()
    C = sec.CHURN
    frames, cam, ocam = sec.churn_frames()
    m = nvb.Mapper(C["voxel"], projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace,
                   tsdf_capacity_blocks=C["capacity"])
    o = orc.OracleMap(C["voxel"])
    fp = orc.default_freespace_params()

    def check_all():
        assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
        assert_color_equal(m.color_layer().as_dict(), o.color_layer())
        assert_freespace_equal(m.freespace_layer().as_dict(), o.freespace_layer())
        assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer(), colors=True)

    def frame(i, max_dist, all_for_freespace, all_for_esdf):
        d, T = frames[i]
        m.tsdf_integrator().params(max_integration_distance_m=max_dist)
        b = m.integrate_depth(d, T, cam)
        assert np.array_equal(b, o.integrate_depth(d, T, ocam, orc.default_tsdf_params(max_integration_distance_m=max_dist)))
        img = textured_image(C["height"], C["width"], seed=i)
        assert np.array_equal(sort_rows(m.integrate_color(img, T, cam)), sort_rows(o.integrate_color(img, T, ocam)))
        updated = o.tsdf_block_indices() if all_for_freespace else b
        m.update_freespace(1000 + 100 * i)
        o.update_freespace(updated, 1000 + 100 * i, fp)
        assert len(updated) >= sec.MARGIN * 4 * _num_sms()  # freespaceUpdateKernel: several blocks per CTA
        m.update_esdf()
        o.integrate_esdf_with_freespace(o.tsdf_block_indices() if all_for_esdf else b)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        o.update_mesh_color()
        check_all()
        t, c = m.tsdf_layer().slab_stats(), m.color_layer().slab_stats()
        assert c["capacity"] == t["capacity"] and m.freespace_layer().slab_stats()["capacity"] == t["capacity"]
        return b

    for i in range(C["frames"]):
        frame(i, C["near_m"], i == 0, i == 0)
    built = m.tsdf_layer().num_blocks()
    colour_built = m.color_layer().num_blocks()
    cap0 = m.tsdf_layer().slab_stats()["capacity"]
    assert cap0 > C["capacity"]  # the colour layer was created on a smaller slab and followed it (checked each frame)

    m.tsdf_decay_integrator().params(**sec.TSDF_WIPE)
    center = sec.churn_exclusion_center(frames)
    gone = m.decay(exclusion_center=center, exclusion_radius_m=C["radius_m"])
    gone_o = o.decay_tsdf(orc.default_tsdf_decay_params(**sec.TSDF_WIPE), exclusion_center=center,
                          exclusion_radius_m=C["radius_m"])
    assert np.array_equal(sort_rows(gone), sort_rows(gone_o))
    removed = len(gone)
    assert removed >= sec.MARGIN * sec.REMOVE_GRID and m.tsdf_layer().num_blocks() >= 0.2 * built, (removed, built)
    check_all()
    assert set(m.esdf_layer().as_dict()) == set(o.esdf_layer())
    st = {n: L.slab_stats() for n, L in (("tsdf", m.tsdf_layer()), ("color", m.color_layer()), ("fs", m.freespace_layer()))}
    assert st["tsdf"]["free"] == removed and st["fs"]["free"] == removed
    colour_removed = colour_built - m.color_layer().num_blocks()
    assert st["color"]["free"] == colour_removed >= sec.MARGIN * sec.REMOVE_GRID
    # the ESDF over the remaining map: voxels whose parents were removed are cleared
    m.update_esdf()
    o.integrate_esdf_with_freespace(o.tsdf_block_indices())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    assert m.esdf_integrator().last_stats()["cleared"] == o.esdf_stats()["cleared"]

    left = m.tsdf_layer().num_blocks()
    frame(C["frames"], C["far_m"], True, False)
    new = m.tsdf_layer().num_blocks() - left
    after = {n: L.slab_stats() for n, L in (("tsdf", m.tsdf_layer()), ("color", m.color_layer()), ("fs", m.freespace_layer()))}
    assert new >= sec.MARGIN * removed, (new, removed)  # the stack ran dry inside the allocation launch ...
    assert after["tsdf"]["free"] == 0 and after["tsdf"]["high_water"] == st["tsdf"]["high_water"] + new - removed
    assert after["tsdf"]["capacity"] > st["tsdf"]["capacity"]  # ... of a frame that grew the slab with a full stack
    assert after["color"]["capacity"] == after["fs"]["capacity"] == after["tsdf"]["capacity"]
    assert after["color"]["free"] == 0 and after["fs"]["free"] == 0
    m.close()


def test_decay_churn_occupancy(gpu):
    """The churn sequence on an occupancy mapper with its ESDF: a one-step decay to 0.5 outside a sphere, then a 7 m frame
    that empties the free stack and grows the slab."""
    nvb, orc = _nvb(), _orc()
    C = sec.CHURN
    frames, cam, ocam = sec.churn_frames()
    m = nvb.Mapper(C["voxel"], projective_layer_type=nvb.ProjectiveLayerType.kOccupancy, tsdf_capacity_blocks=C["capacity"])
    o = orc.OracleMap(C["voxel"])

    def frame(i, max_dist, all_for_esdf):
        d, T = frames[i]
        m.occupancy_integrator().params(max_integration_distance_m=max_dist)
        b = m.integrate_depth(d, T, cam)
        bo = o.integrate_occupancy(d, T, ocam, orc.default_tsdf_params(max_integration_distance_m=max_dist))
        assert np.array_equal(b, bo), i
        assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
        m.update_esdf()
        o.integrate_esdf_occupancy(o.occupancy_block_indices() if all_for_esdf else b)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())

    for i in range(C["frames"]):
        frame(i, C["near_m"], i == 0)
    built = m.occupancy_layer().num_blocks()
    m.occupancy_decay_integrator().params(**sec.OCC_WIPE)
    center = sec.churn_exclusion_center(frames)
    gone = m.decay(exclusion_center=center, exclusion_radius_m=C["radius_m"])
    gone_o = o.decay_occupancy(orc.default_occupancy_decay_params(**sec.OCC_WIPE), exclusion_center=center,
                               exclusion_radius_m=C["radius_m"])
    assert np.array_equal(sort_rows(gone), sort_rows(gone_o))
    removed = len(gone)
    assert removed >= sec.MARGIN * sec.REMOVE_GRID and m.occupancy_layer().num_blocks() >= 0.2 * built, (removed, built)
    assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
    assert set(m.esdf_layer().as_dict()) == set(o.esdf_layer())
    st = m.occupancy_layer().slab_stats()
    assert st["free"] == removed
    left = m.occupancy_layer().num_blocks()
    frame(C["frames"], C["far_m"], True)
    new = m.occupancy_layer().num_blocks() - left
    after = m.occupancy_layer().slab_stats()
    assert new >= sec.MARGIN * removed and after["free"] == 0, (new, removed)
    assert after["high_water"] == st["high_water"] + new - removed and after["capacity"] > st["capacity"]
    m.close()


# ----------------------------------------------------------------------------------------
# 2. Mesh arena
# ----------------------------------------------------------------------------------------
def test_mesh_arena_repacks_past_2_22_entries_and_after_a_large_decay(gpu):
    """2 cm gyroid layer (11 532 blocks, 2.7 M vertices), set in halves with full-layer updates: the arena is repacked
    past 2^22 entries at least twice. Then a decay removes every block outside a sphere (several thousand mesh headers) and
    further full-layer updates repack the arena around the removed segments. Mesh equals the oracle's after every step."""
    nvb, orc = _nvb(), _orc()
    idx, vox = sec.gyroid_layer()
    half = len(idx) // 2
    m, o = nvb.Mapper(0.02), orc.OracleMap(0.02)
    caps = []
    for part in (slice(0, half), slice(half, None), None):
        if part is not None:
            m.tsdf_layer().set_blocks(idx[part], vox[part])
            for k, v in zip(idx[part], vox[part]):
                o.set_tsdf_block(k, v)
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer())
        caps.append(m.mesh_layer().arena_stats()["capacity"])
    grows = [b for a, b in zip([0] + caps, caps) if b > a]
    assert len(grows) >= 2 and caps[-1] >= sec.MARGIN * sec.MESH_ARENA_TARGET, caps
    kw = dict(decay_factor=1e-6, decayed_weight_threshold=1e-3)
    m.tsdf_decay_integrator().params(**kw)
    gone = m.decay(exclusion_center=(0.0, 0.0, 1.0), exclusion_radius_m=1.6)
    gone_o = o.decay_tsdf(orc.default_tsdf_decay_params(**kw), exclusion_center=(0.0, 0.0, 1.0), exclusion_radius_m=1.6)
    assert np.array_equal(sort_rows(gone), sort_rows(gone_o)) and len(gone) >= sec.MARGIN * sec.REMOVE_GRID
    assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer())
    used = [m.mesh_layer().arena_stats()["used"]]
    for _ in range(4):
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer())
        used.append(m.mesh_layer().arena_stats()["used"])
    assert any(b < a for a, b in zip(used, used[1:])), used  # a repack dropped the removed blocks' segments
    m.close()


# ----------------------------------------------------------------------------------------
# 3. Colour and mesh far from the origin and at the key limit
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_origin_colour_tracer_and_colour_mesh(gpu, offset):
    """Depth + colour frames kilometres from the origin: colour lists and layers, the sphere tracer's image and the
    coloured mesh (Mapper::updateColorMesh) equal the oracle's; colours and mesh vertices equal the same sequence at the
    origin within the bounds calibrated on the oracle (tests/test_scale_edges_guard.py)."""
    nvb, orc = _nvb(), _orc()
    frames, cam, ocam = far_frames()
    img = sec.smooth_image(FAR_SEQ["height"], FAR_SEQ["width"])
    m, o, near = nvb.Mapper(FAR_SEQ["voxel"]), orc.OracleMap(FAR_SEQ["voxel"]), nvb.Mapper(FAR_SEQ["voxel"])
    for i, (d, T) in enumerate(frames):
        Tf = sec.shifted(T, offset)
        assert np.array_equal(m.integrate_depth(d, Tf, cam), o.integrate_depth(d, Tf, ocam))
        assert np.array_equal(sort_rows(m.integrate_color(img, Tf, cam)), sort_rows(o.integrate_color(img, Tf, ocam)))
        near.integrate_depth(d, T, cam), near.integrate_color(img, T, cam)
        g = m.color_integrator().render_depth(Tf, cam, 0.2, ray_subsampling_factor=4)
        c = o.sphere_trace_image(Tf, ocam, 0.2, maximum_ray_length_m=7.0, ray_subsampling_factor=4)  # the mapper's default
        assert np.array_equal(g.view(np.uint32), c.view(np.uint32)) and (g > 0).mean() > 0.5, i
        m.update_mesh(update_full_layer=True)
        o.integrate_mesh()
        o.update_mesh_color()
        assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer(), colors=True)
    assert_color_equal(m.color_layer().as_dict(), o.color_layer())
    diff, matched = sec.far_colour_differences(m.color_layer().as_dict(), near.color_layer().as_dict(), offset,
                                               FAR_SEQ["voxel"])
    frac, med, p99 = sec.far_colour_bounds(offset)
    assert matched >= frac and np.median(diff) <= med and np.percentile(diff, 99) <= p99, (matched, np.percentile(diff, 99))
    near.update_mesh(update_full_layer=True)
    dist = sec.far_vertex_distances(m.mesh_layer().as_dict(), near.mesh_layer().as_dict(), offset)
    med, p99 = sec.far_vertex_bounds(offset, FAR_SEQ["voxel"])
    assert np.median(dist) <= med and np.percentile(dist, 99) <= p99, (np.median(dist), np.percentile(dist, 99))
    m.close(), near.close()


@pytest.mark.parametrize("where", ["x_high", "corner_low"])
def test_colour_and_colour_mesh_at_the_key_limit(gpu, where):
    """A sphere's TSDF blocks next to +-2^20, painted from a camera 1 m away: the tracer's rays leave the key range (hashFind
    is -1 there), the colour blocks and the coloured mesh (whose +x / -x neighbours do not exist) equal the oracle's."""
    nvb, orc = _nvb(), _orc()
    idx, vox = sec.key_limit_blocks(where)
    centre = (np.asarray(sec.KEY_LIMIT_SHIFTS[where], np.float64)) * 0.4  # the sphere's centre (block corner 0 moved)
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    m.tsdf_layer().set_blocks(idx, vox)
    for k, v in zip(idx, vox):
        o.set_tsdf_block(k, v)
    cs, cam, ocam = cameras(320, 240)
    T = np.eye(4, dtype=np.float32)  # looks along +z from 1 m below the sphere's centre
    T[:3, 3] = (centre + (0.0, 0.0, -1.0)).astype(np.float32)
    img = textured_image(240, 320, seed=3)
    for _ in range(2):
        assert np.array_equal(sort_rows(m.integrate_color(img, T, cam)), sort_rows(o.integrate_color(img, T, ocam)))
    g = m.color_integrator().render_depth(T, cam, 0.2, ray_subsampling_factor=4)
    c = o.sphere_trace_image(T, ocam, 0.2, maximum_ray_length_m=7.0, ray_subsampling_factor=4)
    assert np.array_equal(g.view(np.uint32), c.view(np.uint32)) and (g > 0).any()
    layer = m.color_layer().as_dict()
    assert_color_equal(layer, o.color_layer())
    assert any(np.any(np.asarray(k) == sec.KEY_LIMIT - 1) or np.any(np.asarray(k) == -sec.KEY_LIMIT) for k in layer)
    assert sum(int((b["weight"] > 0).sum()) for b in layer.values()) > 100
    m.update_mesh(update_full_layer=True)
    o.integrate_mesh()
    o.update_mesh_color()
    assert_mesh_equal(m.mesh_layer().as_dict(), o.mesh_layer(), colors=True)
    m.close()


# ----------------------------------------------------------------------------------------
# 4. Occupancy
# ----------------------------------------------------------------------------------------
def test_occupancy_on_the_global_bitset_view_path(gpu):
    """Occupancy integration behind the global-bitset raycast (2 cm, 10 m: view AABBs of ~1 M cells) with its ESDF."""
    nvb, orc = _nvb(), _orc()
    for c in sec.INTEGRATE_2CM:
        assert sec.MARGIN * sec.SMEM_CELLS <= sec.case_cells(c)[2] and sec.case_cells(c)[2] * sec.MARGIN <= sec.CHAINED_CELLS
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.box_with_cube(), cs, [c["pose"] for c in sec.INTEGRATE_2CM], noise_sigma_rel=0.01, seed=4)
    m = nvb.Mapper(0.02, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    o = orc.OracleMap(0.02)
    m.occupancy_integrator().params(max_integration_distance_m=10.0)
    p = orc.default_tsdf_params(max_integration_distance_m=10.0)
    for i, (d, T) in enumerate(frames):
        b = m.integrate_depth(d, T, cam)
        assert np.array_equal(b, o.integrate_occupancy(d, T, ocam, p)), i
        assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
        m.update_esdf()
        o.integrate_esdf_occupancy(b if i else o.occupancy_block_indices())
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()


def _grid_cap_run(kind):
    code = textwrap.dedent("""
        import sys
        sys.path.insert(0, %r); sys.path.insert(0, %r)
        import numpy as np
        from helpers import assert_esdf_equal, cameras
        from isaac_ros_nvblox_b200 import synthetic as syn
        import isaac_ros_nvblox_b200 as nvb
        from oracle import oracle as orc
        kind = %r
        cs, cam, ocam = cameras(320, 240)
        frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:4])
        t = {"occupancy": nvb.ProjectiveLayerType.kOccupancy, "freespace": nvb.ProjectiveLayerType.kTsdfWithFreespace}[kind]
        m, o = nvb.Mapper(0.05, projective_layer_type=t), orc.OracleMap(0.05)
        for i, (d, T) in enumerate(frames):
            b = m.integrate_depth(d, T, cam)
            if kind == "occupancy":
                o.integrate_occupancy(d, T, ocam)
                all_blocks = o.occupancy_block_indices()
            else:
                o.integrate_depth(d, T, ocam)
                all_blocks = o.tsdf_block_indices()
                m.update_freespace(1000 + 100 * i)
                o.update_freespace(b if i else all_blocks, 1000 + 100 * i)
            m.update_esdf()
            (o.integrate_esdf_occupancy if kind == "occupancy" else o.integrate_esdf_with_freespace)(b if i else all_blocks)
            assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        assert m.esdf_layer().num_blocks() > 3 * 256 * 2
        m.close()
        print("ok")
    """) % (HERE, os.path.dirname(HERE), kind)
    env = dict(os.environ, NVB_ESDF_GRID_CAP="3")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("kind", ["occupancy", "freespace"])
def test_esdf_mark_with_a_capped_grid_from_occupancy_and_with_freespace(gpu, kind):
    """Runs in a subprocess with NVB_ESDF_GRID_CAP=3 (read once per process): esdfMarkOccupancyKernel, and the non-TMA
    esdfMarkKernel that a freespace layer selects, on three CTAs over thousands of blocks (per-CTA lists flush when full)."""
    _grid_cap_run(kind)


@pytest.mark.parametrize("mode", [3, 1])
def test_occupancy_esdf_long_range_parents_beyond_15_blocks(gpu, mode):
    """The long-range ESDF scene restated as an occupancy layer (2 cm, 4 m range, 40 x 40 x 6 blocks): each step's ESDF
    and statistics equal the oracle's, with parents more than 15 blocks away."""
    nvb, orc = _nvb(), _orc()
    m = nvb.Mapper(sec.LR_VOXEL, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy, esdf_persistent=mode)
    m.esdf_integrator().params(max_esdf_distance_m=sec.LR_MAX_DIST)
    o = orc.OracleMap(sec.LR_VOXEL)
    ep = orc.default_esdf_params(max_esdf_distance_m=sec.LR_MAX_DIST)
    for i, ((idx, vox), upd) in enumerate(sec.lr_steps()):
        lo = sec.occupancy_from_tsdf(vox)
        v = np.zeros((len(idx), 8, 8, 8), nvb.OCCUPANCY_VOXEL_DTYPE)
        v["log_odds"] = lo
        m.occupancy_layer().set_blocks(idx, v)
        for k, b in zip(idx, lo):
            o.set_occupancy_block(k, b)
        m.esdf_integrator().integrate_blocks(upd)
        o.integrate_esdf_occupancy(upd, ep)
        layer = m.esdf_layer().as_dict()
        assert_esdf_equal(layer, o.esdf_layer())
        s, so = m.esdf_integrator().last_stats(), o.esdf_stats()
        for k in ("marked", "with_sites", "to_clear", "cleared", "swept"):
            assert s[k] == so[k], (i, k, s, so)
        assert min(sec.far_parent_voxels(layer)) > 10000, i
        validate_esdf(layer, (sec.LR_MAX_DIST / sec.LR_VOXEL) ** 2)
    m.close()


# ----------------------------------------------------------------------------------------
# 5. Slices
# ----------------------------------------------------------------------------------------
def test_slice_on_a_growing_2cm_slab_and_a_slicer_image_of_millions_of_pixels(gpu):
    """2 cm slices from a small slab: the first update sizes the column set from the slab, a 7 m frame then grows the slab,
    so the next update reallocates the set. Then EsdfSlicer images over the map's own box and over a 60 m x 50 m box
    (7.5 M pixels) equal the oracle's bit for bit."""
    nvb, orc = _nvb(), _orc()
    C = sec.CHURN
    frames, cam, ocam = sec.churn_frames()
    m, o = nvb.Mapper(C["voxel"], tsdf_capacity_blocks=C["capacity"]), orc.OracleMap(C["voxel"])
    m.esdf_integrator().slice_params(**sec.SLICE_Z)
    z = dict(z_min_m=sec.SLICE_Z["slice_min_height_m"], z_max_m=sec.SLICE_Z["slice_max_height_m"],
             z_output_m=sec.SLICE_Z["slice_height_m"])
    caps = []
    for i, max_dist in ((0, C["near_m"]), (3, C["far_m"])):
        d, T = frames[i]
        m.tsdf_integrator().params(max_integration_distance_m=max_dist)
        b = m.integrate_depth(d, T, cam)
        assert np.array_equal(b, o.integrate_depth(d, T, ocam, orc.default_tsdf_params(max_integration_distance_m=max_dist)))
        m.update_esdf_slice()
        o.integrate_esdf_slice(b if i else o.tsdf_block_indices(), **z)
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        caps.append(m.tsdf_layer().slab_stats()["capacity"])
    assert caps[1] > caps[0] > C["capacity"], caps
    layer = m.esdf_layer().as_dict()
    assert len(layer) > 1500 and sum(int(v["is_site"].sum()) for v in layer.values()) > 400
    h = sec.SLICE_Z["slice_height_m"]
    aabb_g, img_g, grid_g = nvb.EsdfSlicer(m).slice_layer_to_distance_image(h, 1000.0, with_occupancy_grid=True)
    aabb_c, img_c, grid_c = o.esdf_slice_image(h, 1000.0)
    assert np.array_equal(aabb_g, aabb_c) and np.array_equal(img_g.view(np.uint32), img_c.view(np.uint32))
    assert np.array_equal(grid_g, grid_c)
    box = np.asarray(sec.SLICER_AABB, np.float32)
    img_g = nvb.EsdfSlicer(m).slice_layer_to_distance_image_in_aabb(h, box)
    img_c = o.esdf_slice_image_in_aabb(h, box)
    assert img_g.size == img_c.size == sec.slicer_pixels() >= 5_000_000
    assert np.array_equal(img_g.view(np.uint32), img_c.view(np.uint32))
    assert (img_g != 1000.0).sum() > 10000
    m.close()


@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_origin_slices(gpu, offset):
    """Constant-z slices whose band lies 345 m above or 300 m below the origin (floor(h / block_size) of negative heights):
    the slice ESDF equals the oracle's every frame, and its slicer image equals the same sequence at the origin."""
    nvb, orc = _nvb(), _orc()
    frames, cam, ocam = far_frames()
    dz = float(offset[2])
    zf = {k: float(np.float32(v + dz)) for k, v in sec.SLICE_Z.items()}
    m, o, near = nvb.Mapper(FAR_SEQ["voxel"]), orc.OracleMap(FAR_SEQ["voxel"]), nvb.Mapper(FAR_SEQ["voxel"])
    m.esdf_integrator().slice_params(**zf)
    near.esdf_integrator().slice_params(**sec.SLICE_Z)
    for i, (d, T) in enumerate(frames):
        Tf = sec.shifted(T, offset)
        b = m.integrate_depth(d, Tf, cam)
        assert np.array_equal(b, o.integrate_depth(d, Tf, ocam))
        m.update_esdf_slice()
        o.integrate_esdf_slice(b if i else o.tsdf_block_indices(), z_min_m=zf["slice_min_height_m"],
                               z_max_m=zf["slice_max_height_m"], z_output_m=zf["slice_height_m"])
        assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
        near.integrate_depth(d, T, cam)
        near.update_esdf_slice()
    layer = m.esdf_layer().as_dict()
    assert len({k[2] for k in layer}) == 1 and sum(int(v["is_site"].sum()) for v in layer.values()) > 100
    assert next(iter(layer))[2] == int(np.floor(np.float32(zf["slice_height_m"]) / np.float32(0.4)))
    _, img_far = nvb.EsdfSlicer(m).slice_layer_to_distance_image(zf["slice_height_m"])
    _, img_near = nvb.EsdfSlicer(near).slice_layer_to_distance_image(sec.SLICE_Z["slice_height_m"])
    assert abs(img_far.shape[0] - img_near.shape[0]) <= 8 and abs(img_far.shape[1] - img_near.shape[1]) <= 8
    assert abs(int((img_far < 0.01).sum()) - int((img_near < 0.01).sum())) <= 0.02 * int((img_near < 0.01).sum())
    m.close(), near.close()


@pytest.mark.parametrize("planar", [False, True])
@pytest.mark.parametrize("where", ["corner_high", "corner_low"])
def test_slices_at_the_key_limit(gpu, where, planar):
    """Constant-z and planar slices of a sphere's TSDF blocks at the hash-key limit on all three axes: the slice columns'
    neighbours beyond the limit do not exist; the slice ESDF equals the oracle's."""
    nvb, orc = _nvb(), _orc()
    idx, vox = sec.key_limit_blocks(where)
    cx, cy, zc = (float(np.float32(s) * np.float32(0.4)) for s in sec.KEY_LIMIT_SHIFTS[where])  # the sphere's centre
    m, o = nvb.Mapper(0.05), orc.OracleMap(0.05)
    m.tsdf_layer().set_blocks(idx, vox)
    for k, v in zip(idx, vox):
        o.set_tsdf_block(k, v)
    zmin, zmax, zout = zc - 0.1, zc + 0.1, zc
    if planar:
        pl = unit_plane((0.05, -0.03, 1.0), (cx, cy, zmin))
        m.esdf_integrator().slice_params(slice_height_above_plane_m=0.0, slice_height_thickness_m=0.2, slice_height_m=zout)
        m.esdf_integrator().integrate_slice(idx, ground_plane=pl)
        o.integrate_esdf_slice_planar(idx, pl, above_plane_m=0.0, thickness_m=0.2, z_output_m=zout)
    else:
        m.esdf_integrator().slice_params(slice_min_height_m=zmin, slice_max_height_m=zmax, slice_height_m=zout)
        m.esdf_integrator().integrate_slice(idx)
        o.integrate_esdf_slice(idx, z_min_m=zmin, z_max_m=zmax, z_output_m=zout)
    layer = m.esdf_layer().as_dict()
    assert_esdf_equal(layer, o.esdf_layer())
    assert any(np.any(np.asarray(k[:2]) == sec.KEY_LIMIT - 1) or np.any(np.asarray(k[:2]) == -sec.KEY_LIMIT) for k in layer)
    assert sum(int(v["is_site"].sum()) for v in layer.values()) > 20
    m.close()


# ----------------------------------------------------------------------------------------
# Last: the largest allocation of the module
# ----------------------------------------------------------------------------------------
def test_occupancy_one_frame_on_the_chained_path(gpu):
    """One occupancy frame with a 40 m range at 5 cm (~3.5 M view cells: the chained compaction with allocation). The frame
    grows the occupancy slab to 2^22 blocks (8 GiB). One frame, and the mapper is closed."""
    nvb, orc = _nvb(), _orc()
    case = sec.INTEGRATE_CHAINED
    assert sec.case_cells(case)[2] >= sec.MARGIN * sec.CHAINED_CELLS
    cs, cam, ocam = cameras(case["width"], case["height"])
    depth = syn.render_depth(syn.box_with_cube(), cs, case["pose"], max_dist=case["max_dist"])
    m = nvb.Mapper(case["voxel"], projective_layer_type=nvb.ProjectiveLayerType.kOccupancy, tsdf_capacity_blocks=1024,
                   esdf_capacity_blocks=1024, esdf_persistent=1)
    o = orc.OracleMap(case["voxel"])
    m.occupancy_integrator().params(max_integration_distance_m=case["max_dist"])
    b = m.integrate_depth(depth, case["pose"], cam)
    assert np.array_equal(b, o.integrate_occupancy(depth, case["pose"], ocam,
                                                   orc.default_tsdf_params(max_integration_distance_m=case["max_dist"])))
    assert_occupancy_equal(m.occupancy_layer().as_dict(), o.occupancy_layer())
    assert m.occupancy_layer().slab_stats()["capacity"] <= 1 << 22
    m.close()
