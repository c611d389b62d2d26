"""Known-answer tests of the dynamics restatement (tests/dynamics_reference.py), no GPU: the reference's
MaskPreprocessor tests (T/test_mask_preprocessor.cpp, every case), its DynamicsDetection HumanDataset test
(T/test_dynamics.cpp, Camera) on the oracle's TSDF and freespace layers, and the drop-in program's build."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import dynamics_reference as dref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_fixture_matches_the_reference_files():
    """tests/golden/dynamics_human.npz holds the arrays read from the reference's PNGs (digests recorded when it was made)."""
    z = np.load(os.path.join(GOLDEN, "dynamics_human.npz"))
    want = json.load(open(os.path.join(GOLDEN, "dynamics_human_sources.json")))
    for name, d in want.items():
        a = np.ascontiguousarray(z[name])
        assert a.dtype.str == d["dtype"] and list(a.shape) == d["shape"]
        assert hashlib.sha256(a.tobytes()).hexdigest() == d["sha256"], name
    assert int((z["mask_21"] > 0).sum()) == 14073


@pytest.mark.parametrize("case", ["RealMask", "EmptyMask", "FullMask", "TwoSquares_keepBoth", "TwoSquares_keepOne",
                                  "TwoSquares_keepNone", "GridPattern"])
def test_mask_preprocessor_fixture_cases(case):
    _, _, mask_21 = dref.load_human_fixture()
    mask, threshold, expected = dref.reference_masks(mask_21)[case]
    out = dref.remove_small_connected_components(mask, threshold)
    assert int((out > 0).sum()) == expected
    assert set(np.unique(out)) <= {0, 254}


@pytest.mark.parametrize("corner", ["TopLeft", "TopRight", "BottomLeft", "BottomRight"])
def test_mask_preprocessor_blob_in_corner(corner):
    mask, pixels = dref.corner_blobs()[corner]
    out = dref.remove_small_connected_components(mask, 3)
    assert all(out[r, c] > 0 for r, c in pixels)


def test_mask_preprocessor_conventions():
    """threshold <= 0 copies; thresholds 1-3 remove nothing (3 / 4 == 0); odd sizes keep their size with a zero trailing
    row / column; a 1 x N mask has no downscaled pixel and comes out empty."""
    rng = np.random.default_rng(3)
    m = (rng.random((37, 53)) < 0.3).astype(np.uint8) * 7
    assert np.array_equal(dref.remove_small_connected_components(m, 0), m)
    assert np.array_equal(dref.remove_small_connected_components(m, -5), m)
    down = m[0:36:2, 0:52:2] > 0
    for t in (1, 2, 3):
        out = dref.remove_small_connected_components(m, t)
        assert out.shape == m.shape and not out[36].any() and not out[:, 52].any()
        assert np.array_equal(out[:36, :52] > 0, np.repeat(np.repeat(down, 2, 0), 2, 1))
    assert not dref.remove_small_connected_components(np.full((1, 9), 255, np.uint8), 4).any()


def test_dynamics_human_dataset_on_the_oracle():
    """HumanDataset (Camera): frame 1 through the oracle's TSDF, two freespace updates 1 000 ms apart (check_neighborhood off,
    max_tsdf_distance_for_occupancy_m = 0.75 x truncation), detection on frame 2: a plausible share of dynamic pixels."""
    from oracle import oracle as orc
    K, depth, _ = dref.load_human_fixture()
    rows, cols = depth.shape[1:]
    ocam = orc.Camera(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), cols, rows)
    voxel = np.float32(0.05)
    trunc_m = np.float32(4) * voxel
    o = orc.OracleMap(float(voxel))
    tp = orc.default_tsdf_params(truncation_distance_vox=4.0, max_integration_distance_m=20.0)
    o.integrate_depth(depth[0], np.eye(4, dtype=np.float32), ocam, tp)
    fp_ = orc.default_freespace_params(max_tsdf_distance_for_occupancy_m=float(trunc_m * np.float32(0.75)),
                                       min_duration_since_occupied_for_freespace_ms=1000, check_neighborhood=0)
    for t in (100, 1100):
        o.update_freespace(o.tsdf_block_indices(), t, fp_)
    cam = {"fu": K[0, 0], "fv": K[1, 1], "cu": K[0, 2], "cv": K[1, 2]}
    mask, overlay, pts = dref.compute_dynamics(depth[1], np.eye(4, dtype=np.float32), cam, o.freespace_layer(), voxel * 8)
    n = rows * cols
    assert n / 20.0 < len(pts) < n / 5.0
    assert int((mask == 255).sum()) == len(pts)
    assert np.array_equal(overlay[..., 0] == 255, (mask == 255) | np.all(overlay == 255, axis=-1))


def test_dynamics_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_dynamics_dropin.cpp (nvblox_ros' kDynamic calls without setDynamicMask, DynamicsDetection and
    MaskPreprocessor through nvblox/nvblox.h) builds with plain g++; without a GPU it exits 77."""
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_dynamics_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
