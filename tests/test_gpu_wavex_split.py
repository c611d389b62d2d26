"""The exchange-slab wavefront's split own-block fetch against the oracle, bit for bit.

Grid rings with at least kSplitMinK candidates fetch a candidate's own block in two parts: the boundary planes along the
live passes' axes with the halo, and the rest of the block only if the block changed. NVB_WAVEX_SPLIT_MIN_K replaces the
threshold and is read once per process, so each case runs in a subprocess twice: with 0 (every grid ring fetches split)
and with 1000000000 (none does). The launch statistics `split_candidates` and `rest_fetches` show which path ran.

    python tests/test_gpu_wavex_split.py CASE   (run by the tests below, with NVB_WAVEX_SPLIT_MIN_K set)
"""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

ALWAYS, NEVER = "0", "1000000000"
CASES = ("c2_pipeline", "long_range", "reserved_36", "c2_2cm")
STATS = ("marked", "with_sites", "to_clear", "clear_candidates", "cleared", "swept", "face_passes", "rings")


def _add(acc, s):
    acc["split_candidates"] += int(s["split_candidates"])
    acc["rest_fetches"] += int(s["rest_fetches"])


def _c2(voxel, n):
    """bench.py's c2 frames (the first n) through its timed pipeline: device depth, asynchronous ESDF updates."""
    import numpy as np
    import torch
    import bench
    import isaac_ros_nvblox_b200 as nvb
    from helpers import assert_esdf_equal, assert_tsdf_equal
    from oracle import oracle as orc
    cam_s, frames = bench.make_frames(80, 0, 1)
    frames = frames[:n]
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ocam = orc.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    o = orc.OracleMap(voxel)
    for depth, T in frames:
        o.integrate_esdf(o.integrate_depth(depth, T, ocam))
    depth_dev = torch.from_numpy(np.stack([d for d, _ in frames])).cuda()
    m = nvb.Mapper(voxel)
    acc = {"split_candidates": 0, "rest_fetches": 0}
    for i, (_, T) in enumerate(frames):
        m.integrate_depth_device(depth_dev[i].data_ptr(), cam_s.height, cam_s.width, T, cam)
        m.update_esdf(sync=False)
        _add(acc, m.esdf_integrator().last_stats())  # (synchronises: the statistics of this update)
    m.synchronize()
    assert_tsdf_equal(m.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_esdf_equal(m.esdf_layer().as_dict(), o.esdf_layer())
    m.close()
    return acc


def _long_range(reserved):
    """2 cm voxels, 4 m ESDF range, parents more than 15 blocks away (test_gpu_scale_edges.py's long-range scene)."""
    import isaac_ros_nvblox_b200 as nvb
    import scale_edge_cases as sec
    from helpers import assert_esdf_equal
    from oracle import oracle as orc
    o = orc.OracleMap(sec.LR_VOXEL)
    ep = orc.default_esdf_params(max_esdf_distance_m=sec.LR_MAX_DIST)
    m = nvb.Mapper(sec.LR_VOXEL, esdf_persistent=3)
    m.esdf_integrator().params(max_esdf_distance_m=sec.LR_MAX_DIST)
    if reserved is not None:
        m.esdf_reserved_sms(reserved)
        assert m.esdf_reserved_sms() == reserved
    acc = {"split_candidates": 0, "rest_fetches": 0}
    for i, ((idx, vox), upd) in enumerate(sec.lr_steps()):
        for k, v in zip(idx, vox):
            o.set_tsdf_block(k, v)
        o.integrate_esdf(upd, ep)
        m.tsdf_layer().set_blocks(idx, vox)
        m.esdf_integrator().integrate_blocks(upd)
        layer = m.esdf_layer().as_dict()
        assert_esdf_equal(layer, o.esdf_layer())
        s, so = m.esdf_integrator().last_stats(), o.esdf_stats()
        for k in STATS:
            assert s[k] == so[k], (i, k, s, so)
        assert min(sec.far_parent_voxels(layer)) > 10000, i
        _add(acc, s)
    m.close()
    return acc


def run_case(case):
    if case == "c2_pipeline":
        return _c2(0.05, 80)
    if case == "c2_2cm":
        return _c2(0.02, 4)
    if case == "long_range":
        return _long_range(None)
    if case == "reserved_36":
        return _long_range(36)
    raise ValueError(case)


@pytest.mark.gpu
@pytest.mark.parametrize("split_min_k", [ALWAYS, NEVER])
@pytest.mark.parametrize("case", CASES)
def test_split_fetch_equals_oracle(gpu, case, split_min_k):
    env = dict(os.environ, NVB_WAVEX_SPLIT_MIN_K=split_min_k)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), case], env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    acc = json.loads(r.stdout.strip().splitlines()[-1])
    if split_min_k == ALWAYS:
        # every grid ring fetched split, and some of its candidates changed and fetched the rest of their block
        assert acc["split_candidates"] > 0 and 0 < acc["rest_fetches"] < acc["split_candidates"], acc
    else:
        assert acc == {"split_candidates": 0, "rest_fetches": 0}, acc


if __name__ == "__main__":
    sys.path[:0] = [HERE, ROOT]
    print(json.dumps(run_case(sys.argv[1])))
