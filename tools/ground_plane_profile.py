"""Cost of the ground-plane estimator on the GPU (GroundPlaneEstimator::computeGroundPlane) on three maps:

  bench : bench.py's c2 map (80 frames of the sphere-in-box circle, 640x480, 5 cm voxels)
  2cm   : a flat, slightly tilted ground at 2 cm voxels uploaded with Layer.set_blocks, about 100 k ground candidates
  300k  : the same at about 300 k candidates

For each map: the host time of the synchronous compute_ground_plane call (median over repeats, read-backs included), the
host time of the fit alone (ransac_fit_plane on the candidates, 1 000 iterations), and the device time per kernel from
torch.profiler. Prints one JSON object with the card's name and power limit.

    python tools/ground_plane_profile.py [--repeats 20]
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 - the numbers are still worth printing without it
        return {"error": str(e)}


def ground_layer(voxel, half_extent, tilt=0.01):
    """TSDF blocks of the ground z = tilt * x around the origin (distance clipped to +-4 voxels, weight 1)."""
    from isaac_ros_nvblox_b200.mapper import TSDF_VOXEL_DTYPE
    bs = np.float32(8 * voxel)
    nb = int(np.ceil(half_extent / bs))
    bx = np.arange(-nb, nb)
    idx, vox = [], []
    v = (np.arange(8, dtype=np.float32) + np.float32(0.5)) * np.float32(voxel)
    for bz in (-1, 0):
        for x in bx:
            for y in bx:
                px = np.float32(x) * bs + v
                pz = np.float32(bz) * bs + v
                d = pz[None, None, :] - np.float32(tilt) * px[:, None, None]
                blk = np.zeros((8, 8, 8), TSDF_VOXEL_DTYPE)
                blk["distance"] = np.clip(np.broadcast_to(d, (8, 8, 8)), -4 * voxel, 4 * voxel)
                blk["weight"] = 1.0
                idx.append((x, y, bz))
                vox.append(blk)
    return np.asarray(idx, np.int32), np.stack(vox)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e6, out


KERNELS = ("groundCountKernel", "exclusiveScanInt2Kernel", "groundEmitKernel", "ransacFitKernel", "ransacArgminKernel")


def kernel_times(m, repeats):
    import torch
    from torch.profiler import ProfilerActivity, profile
    est = m.ground_plane_estimator()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            est.compute_ground_plane()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in KERNELS:
            if name in e.key:
                out[name] = {"us": round(e.device_time_total / max(e.count, 1), 2), "calls": e.count}
    return out


def profile_map(nvb, m, repeats):
    est = m.ground_plane_estimator()
    est.compute_ground_plane()  # warm-up: scratch allocation, generator states
    ts = [timed(est.compute_ground_plane)[0] for _ in range(repeats)]
    plane = est.ground_plane()
    cand = est.tsdf_zero_crossings_ground_candidates()
    out = {"tsdf_blocks": m.tsdf_layer().num_blocks(), "crossings": len(est.tsdf_zero_crossings()),
           "candidates": len(cand), "plane": plane,
           "compute_ground_plane_us": {"median": float(np.median(ts)), "min": float(np.min(ts))}}
    p0 = nvb.ransac_fit_plane(cand, 1000, mapper=m)
    tf = [timed(lambda: nvb.ransac_fit_plane(cand, 1000, mapper=m))[0] for _ in range(repeats)]
    out["fit_us"] = {"median": float(np.median(tf)), "min": float(np.min(tf)), "same_plane": p0 == plane}
    out["kernel_us"] = kernel_times(m, repeats)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import synthetic as syn
    scam = syn.PinholeCamera()
    cam = nvb.Camera(scam.fu, scam.fv, scam.cu, scam.cv, scam.width, scam.height)
    res = {"gpu": gpu_info()}
    m = nvb.Mapper(0.05)
    for d, T in syn.make_sequence(syn.sphere_in_box(), scam, syn.circle_trajectory(80)):
        m.integrate_depth(d, T, cam, return_blocks=False)
        m.update_esdf()
    res["bench"] = profile_map(nvb, m, args.repeats)
    m.close()
    for name, half in (("2cm_100k", 3.2), ("2cm_300k", 5.5)):
        idx, vox = ground_layer(0.02, half)
        m = nvb.Mapper(0.02)
        m.tsdf_layer().set_blocks(idx, vox)
        res[name] = profile_map(nvb, m, args.repeats)
        m.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
