"""Preconditions of tests/test_gpu_scale_edges.py, checkable without a GPU: every configuration there sits at least 20 %
beyond the threshold whose branch it is meant to run (tests/scale_edge_cases.py), the numpy restatement of the view AABB
contains every block the oracle's raycast returns, and the far-from-origin tolerances hold on the oracle."""
import numpy as np
import pytest

import scale_edge_cases as sec
from helpers import cameras, textured_image, validate_esdf
from isaac_ros_nvblox_b200 import synthetic as syn


def _on_side(cells, path):
    if path == "smem":
        assert cells * sec.MARGIN <= sec.SMEM_CELLS, (cells, sec.SMEM_CELLS)
    elif path == "global":
        assert cells >= sec.MARGIN * sec.SMEM_CELLS, (cells, sec.SMEM_CELLS)
        assert cells * sec.MARGIN <= sec.CHAINED_CELLS, (cells, sec.CHAINED_CELLS)
    else:
        assert cells >= sec.MARGIN * sec.CHAINED_CELLS, (cells, sec.CHAINED_CELLS)


@pytest.mark.parametrize("name", [c["name"] for c in sec.VIEW_CASES])
def test_view_case_crosses_its_threshold_and_contains_the_oracle_blocks(name):
    from oracle import oracle as orc
    case = sec.VIEW[name]
    mn, size, cells = sec.case_cells(case)
    _on_side(cells, case["path"])
    _, _, ocam = cameras(case["width"], case["height"], radial=case.get("radial"), tangential=case.get("tangential"))
    p = orc.default_tsdf_params(max_integration_distance_m=case["max_dist"])
    got = orc.view_raycast(sec.random_depth(case, 0), case["pose"], ocam, 8 * case["voxel"], 4 * case["voxel"], p, cap=cells)
    assert len(got) > cells // 20  # the marks spread over the AABB
    assert np.all(got >= mn) and np.all(got < mn + size)


def test_small_view_and_integrate_cases_cross_their_thresholds():
    _on_side(sec.case_cells(sec.SMALL_VIEW)[2], "smem")
    for case in sec.INTEGRATE_2CM:
        _on_side(sec.case_cells(case)[2], "global")
    cells = sec.case_cells(sec.INTEGRATE_CHAINED)[2]
    _on_side(cells, "chained")
    # one frame of this many cells grows the TSDF slab to 2^22 blocks (16 GiB), not 2^23
    assert cells < sec.TSDF_SLAB_LIMIT_CELLS
    assert sec.union_cells() >= sec.MARGIN * sec.CHAINED_CELLS
    a, b = sec.union_lists()
    u = np.unique(np.concatenate([a, b]), axis=0)
    assert np.array_equal(u.min(0), sec.UNION_BOX[0]) and np.array_equal(u.max(0), sec.UNION_BOX[1])


def _observed_voxels(layer):
    """-> (global voxel indices (n, 3) int64, distances (n,)) of the voxels with weight > 0."""
    keys, dist = [], []
    for k, b in layer.items():
        v = np.argwhere(b["weight"] > 0)
        keys.append(np.asarray(k, np.int64) * 8 + v)
        dist.append(b["distance"][v[:, 0], v[:, 1], v[:, 2]])
    return np.concatenate(keys), np.concatenate(dist)


def far_origin_differences(far_layer, origin_layer, offset, voxel):
    """|TSDF distance differences| of the voxels observed in both maps, matched by the voxel-index shift offset / voxel,
    and the fraction of the origin map's observed voxels that were matched."""
    shift = np.round(np.asarray(offset, np.float64) / voxel).astype(np.int64)
    kf, df = _observed_voxels(far_layer)
    ko, do = _observed_voxels(origin_layer)
    kf = kf - shift
    base = np.minimum(kf.min(0), ko.min(0))
    ext = np.maximum(kf.max(0), ko.max(0)) - base + 1

    def lin(k):
        k = k - base
        return (k[:, 2] * ext[1] + k[:, 1]) * ext[0] + k[:, 0]

    lf, lo = lin(kf), lin(ko)
    common, i_f, i_o = np.intersect1d(lf, lo, assume_unique=True, return_indices=True)
    return np.abs(df[i_f].astype(np.float64) - do[i_o].astype(np.float64)), len(common) / len(lo)


def far_origin_bounds(offset):
    """Median and 99th-percentile bounds on those differences: the float32 spacing at the offset is the rounding step of a
    voxel centre and of the camera's position there."""
    spacing = float(np.spacing(np.float32(np.max(np.abs(offset)))))
    return 0.5 * spacing, 2.0 * spacing


FAR_SEQ = dict(width=320, height=240, voxel=0.05, frames=3)


def far_frames():
    cs, cam, ocam = cameras(FAR_SEQ["width"], FAR_SEQ["height"])
    return syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:FAR_SEQ["frames"]]), cam, ocam


@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_origin_map_matches_the_origin_map_on_the_oracle(offset):
    """The oracle's map integrated kilometres from the origin equals its map at the origin up to float32 rounding at the
    offset (same depth images, poses shifted by a whole number of voxels)."""
    from oracle import oracle as orc
    frames, _, ocam = far_frames()
    near, far = orc.OracleMap(FAR_SEQ["voxel"]), orc.OracleMap(FAR_SEQ["voxel"])
    for d, T in frames:
        near.integrate_depth(d, T, ocam)
        far.integrate_depth(d, sec.shifted(T, offset), ocam)
    diff, matched = far_origin_differences(far.tsdf_layer(), near.tsdf_layer(), offset, FAR_SEQ["voxel"])
    med, p99 = far_origin_bounds(offset)
    assert matched > 0.995
    assert np.median(diff) <= med and np.percentile(diff, 99) <= p99, (np.median(diff), np.percentile(diff, 99), med, p99)
    assert np.any(np.abs(far.tsdf_block_indices()) > 5000)  # large block indices


def test_key_limit_blocks_are_at_the_limit():
    for idx in sec.key_limit_block_sets():
        assert np.all(idx >= -sec.KEY_LIMIT) and np.all(idx < sec.KEY_LIMIT)
        assert np.any(idx == sec.KEY_LIMIT - 1) or np.any(idx == -sec.KEY_LIMIT)


def test_long_range_scene_has_parents_beyond_15_blocks_on_the_oracle():
    from oracle import oracle as orc
    o = orc.OracleMap(sec.LR_VOXEL)
    ep = orc.default_esdf_params(max_esdf_distance_m=sec.LR_MAX_DIST)
    for i, ((idx, vox), upd) in enumerate(sec.lr_steps()):
        for k, v in zip(idx, vox):
            o.set_tsdf_block(k, v)
        o.integrate_esdf(upd, ep)
        layer = o.esdf_layer()
        assert min(sec.far_parent_voxels(layer)) > 10000, i
        validate_esdf(layer, (sec.LR_MAX_DIST / sec.LR_VOXEL) ** 2)
        if i == 1:  # removing a cluster clears voxels (the clear pass runs on blocks with "unknown" parent boxes)
            assert o.esdf_stats()["cleared"] > 1000


# ---------------------------------------------------------------------------------------------------------------------
# Preconditions of tests/test_gpu_scale_edges_f.py
# ---------------------------------------------------------------------------------------------------------------------
def churn_on_the_oracle(occupancy=False):
    """The churn sequence (scale_edge_cases.CHURN) on the oracle, with the TSDF slab's capacity restated from
    ensureTsdfCapacity. -> dict of block counts and capacities."""
    from oracle import oracle as orc
    C = sec.CHURN
    frames, _, ocam = sec.churn_frames()
    o = orc.OracleMap(C["voxel"])
    blocks = o.occupancy_block_indices if occupancy else o.tsdf_block_indices
    cap, hw = C["capacity"], 0
    for i, (d, T) in enumerate(frames[:C["frames"]]):
        cap = sec.grown_capacity(cap, hw, sec.churn_cells(T, C["near_m"]))
        p = orc.default_tsdf_params(max_integration_distance_m=C["near_m"])
        o.integrate_occupancy(d, T, ocam, p) if occupancy else o.integrate_depth(d, T, ocam, p)
        if not occupancy:
            o.integrate_color(textured_image(C["height"], C["width"], seed=i), T, ocam)
        hw = len(blocks())
    colour_built = len(o.color_block_indices())
    center = sec.churn_exclusion_center(frames)
    if occupancy:
        removed = o.decay_occupancy(orc.default_occupancy_decay_params(**sec.OCC_WIPE), exclusion_center=center,
                                    exclusion_radius_m=C["radius_m"])
    else:
        removed = o.decay_tsdf(orc.default_tsdf_decay_params(**sec.TSDF_WIPE), exclusion_center=center,
                               exclusion_radius_m=C["radius_m"])
    left = len(blocks())
    colour_removed = colour_built - len(o.color_block_indices())
    d, T = frames[C["frames"]]
    far_cells = sec.churn_cells(T, C["far_m"])
    p = orc.default_tsdf_params(max_integration_distance_m=C["far_m"])
    o.integrate_occupancy(d, T, ocam, p) if occupancy else o.integrate_depth(d, T, ocam, p)
    return dict(built=hw, capacity=cap, removed=len(removed), colour_removed=colour_removed, left=left, new=len(blocks()) - left, far_cells=far_cells,
                grown=sec.grown_capacity(cap, hw, far_cells))


@pytest.mark.parametrize("occupancy", [False, True])
def test_churn_crosses_the_remove_grid_the_free_stack_and_the_capacity(occupancy):
    r = churn_on_the_oracle(occupancy)
    assert r["removed"] >= sec.MARGIN * sec.REMOVE_GRID, r  # several rounds of the remove kernels
    assert occupancy or r["colour_removed"] >= sec.MARGIN * sec.REMOVE_GRID, r
    assert r["left"] >= 0.2 * r["built"], r                  # a partial removal
    assert r["new"] >= sec.MARGIN * r["removed"], r          # the free stack runs dry in the frame after the decay
    assert r["built"] + r["far_cells"] >= sec.MARGIN * r["capacity"] and r["grown"] > r["capacity"], r  # ... which grows it
    assert 20000 <= r["built"] + r["new"] and r["grown"] <= 1 << 22, r


def test_gyroid_mesh_needs_an_arena_past_2_22_entries():
    from oracle import oracle as orc
    idx, vox = sec.gyroid_layer()
    o = orc.OracleMap(0.02)
    for k, v in zip(idx, vox):
        o.set_tsdf_block(k, v)
    o.integrate_mesh()
    verts = sum(len(b["vertices"]) for b in o.mesh_layer().values())
    # a repack makes room for twice the live data plus the update: one full-layer update on top of half the layer
    assert 2 * (verts // 2 + verts) >= sec.MARGIN * sec.MESH_ARENA_TARGET, verts
    assert len(idx) >= 10000


@pytest.mark.parametrize("offset", sec.FAR_OFFSETS)
def test_far_origin_colour_and_mesh_match_the_origin_on_the_oracle(offset):
    from oracle import oracle as orc
    frames, _, ocam = far_frames()
    img = sec.smooth_image(FAR_SEQ["height"], FAR_SEQ["width"])
    near, far = orc.OracleMap(FAR_SEQ["voxel"]), orc.OracleMap(FAR_SEQ["voxel"])
    for d, T in frames:
        near.integrate_depth(d, T, ocam), near.integrate_color(img, T, ocam)
        far.integrate_depth(d, sec.shifted(T, offset), ocam), far.integrate_color(img, sec.shifted(T, offset), ocam)
    diff, matched = sec.far_colour_differences(far.color_layer(), near.color_layer(), offset, FAR_SEQ["voxel"])
    frac, med, p99 = sec.far_colour_bounds(offset)
    assert matched >= frac and np.median(diff) <= med and np.percentile(diff, 99) <= p99, (matched, np.percentile(diff, 99))
    near.integrate_mesh(), far.integrate_mesh()
    dist = sec.far_vertex_distances(far.mesh_layer(), near.mesh_layer(), offset)
    med, p99 = sec.far_vertex_bounds(offset, FAR_SEQ["voxel"])
    assert np.median(dist) <= med and np.percentile(dist, 99) <= p99, (np.median(dist), np.percentile(dist, 99))


def test_slicer_image_and_slice_heights_cross_their_thresholds():
    assert sec.slicer_pixels() >= 5_000_000
    assert min(o[2] for o in sec.FAR_OFFSETS) <= -300.0 and max(o[2] for o in sec.FAR_OFFSETS) >= 300.0
    # below the origin floor(h / block_size) and a truncating cast differ, so a slice split that truncated moves the band
    for o in sec.FAR_OFFSETS:
        for h in sec.SLICE_Z.values():
            if o[2] < 0:
                assert np.floor((h + o[2]) / 0.4) != np.trunc((h + o[2]) / 0.4)
