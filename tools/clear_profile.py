"""Cost of map clearing on the GPU: Mapper::clear_outside_radius and clear_tsdf_inside_shapes on two maps.

  bench : bench.py's c2 map (80 frames of the sphere-in-box circle, 640x480, 5 cm voxels, TSDF + ESDF + mesh)
  2cm   : the first 20 of those frames at 2 cm voxels (more blocks per frame, a slab of several 10^4 blocks)

For each map: clear_outside_radius that removes nothing (median over repeats; the map is unchanged by it), about 10 % and
about 50 % of the blocks removed (each on a fresh copy of the map, the radius picked from the blocks' distances), and
clear_tsdf_inside_shapes with 4 shapes (2 spheres, 2 boxes) around the circle's centre. Every call is synchronous, so a
host clock around it is the call's full cost, read-backs included. Prints one JSON object with the card's name and power
limit.

    python tools/clear_profile.py [--repeats 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - the numbers are still worth printing without it
        return {"error": str(e)}


def build_map(nvb, frames, cam, voxel):
    m = nvb.Mapper(voxel)
    for d, T in frames:
        m.integrate_depth(d, T, cam, return_blocks=False)
        m.update_esdf()
    m.update_mesh()
    return m


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e6, out


def radius_removing(m, center, share):
    """The radius for which about `share` of the blocks lie farther than it (block-centre distances)."""
    bs = m.block_size()
    c = (m.tsdf_layer().get_all_block_indices().astype(np.float64) + 0.5) * bs
    return float(np.quantile(np.linalg.norm(c - center, axis=1), 1.0 - share))


def profile(nvb, frames, cam, voxel, repeats):
    center = np.array([0.0, 0.0, 2.0], np.float32)  # the trajectory circles (0, 0) at 2 m height
    m = build_map(nvb, frames, cam, voxel)
    n_blocks = m.tsdf_layer().num_blocks()
    far = 1e6
    m.clear_outside_radius(center, far)  # warm-up
    t_none = [timed(lambda: m.clear_outside_radius(center, far))[0] for _ in range(repeats)]
    out = {"voxel_m": voxel, "tsdf_blocks": n_blocks, "tsdf_capacity": m.tsdf_layer().slab_stats()["capacity"],
           "nothing_removed_us": {"median": float(np.median(t_none)), "min": float(np.min(t_none))}}
    for share in (0.1, 0.5):
        ts, removed = [], 0
        for _ in range(3):
            mm = build_map(nvb, frames, cam, voxel)
            r = radius_removing(mm, center, share)
            t, rem = timed(lambda: mm.clear_outside_radius(center, r))
            ts.append(t), mm.close()
            removed = len(rem)
        out["removed_%d_pct" % int(share * 100)] = {"median_us": float(np.median(ts)), "blocks_removed": removed}
    shapes = [nvb.BoundingSphere(center, 1.0), nvb.BoundingSphere(center + np.float32(2.0), 0.5),
              nvb.AxisAlignedBoundingBox(center - np.float32(3.0), center - np.float32(2.0)),
              nvb.AxisAlignedBoundingBox((-0.5, -4.0, 0.0), (0.5, 4.0, 1.0))]
    t_sh, touched = [], 0
    for _ in range(repeats):
        t, tb = timed(lambda: m.clear_tsdf_inside_shapes(shapes))
        t_sh.append(t)
        touched = len(tb)
    out["shapes_4"] = {"median_us": float(np.median(t_sh)), "blocks_touched": touched}
    m.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=50)
    args = ap.parse_args()
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import synthetic as syn
    scam = syn.PinholeCamera()
    cam = nvb.Camera(scam.fu, scam.fv, scam.cu, scam.cv, scam.width, scam.height)
    frames = syn.make_sequence(syn.sphere_in_box(), scam, syn.circle_trajectory(80))
    res = {"gpu": gpu_info(), "bench": profile(nvb, frames, cam, 0.05, args.repeats),
           "2cm": profile(nvb, frames[:20], cam, 0.02, args.repeats)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
