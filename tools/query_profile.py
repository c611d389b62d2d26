"""Throughput of the point queries on the GPU (nvb_query.cu), timed with CUDA events over many launches after warm-up.

Map: bench.py's c2 map (80 frames of the sphere-in-box circle, 640x480, 5 cm voxels, TSDF + ESDF); the two-mapper rows add a
second mapper of 8 cm voxels over the same frames. Point workloads, N = 2^16, 2^20 and 2^24:
  uniform : uniform in the map's AABB;
  planner : clusters of 64 spheres along random trajectories (a robot's collision spheres along candidate paths), so that
            neighbouring threads read the same blocks.
Query kinds: ESDF distance, ESDF + gradient, TSDF, occupancy (a hand-filled occupancy mapper over the same blocks),
interpolation (TSDF) and voxel lookup (ESDF). For each: queries/s and algorithmic bytes/s -- point in, result out, per mapper
one hash probe (8-byte key + 4-byte slot) and the voxel words the query reads -- against the 3.35 TB/s HBM3 bound of the
H100 SXM data sheet. Prints one JSON object with the card's name and power limit. Fails without a GPU.

    python tools/query_profile.py [--launches 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def build_maps(nvb, frames, cam):
    ms = []
    for voxel in (0.05, 0.08):
        m = nvb.Mapper(voxel)
        for d, T in frames:
            m.integrate_depth(d, T, cam, return_blocks=False)
            m.update_esdf()
        ms.append(m)
    occ = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    idx = ms[0].tsdf_layer().get_all_block_indices()
    v = np.zeros((len(idx), 8, 8, 8), nvb.mapper.OCCUPANCY_VOXEL_DTYPE)
    v["log_odds"] = np.random.default_rng(0).uniform(-4, 4, v.shape).astype(np.float32)
    occ.occupancy_layer().set_blocks(idx, v)
    return ms, occ, idx


def workloads(torch, idx, bs, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo = torch.tensor(idx.min(0) * bs, dtype=torch.float32, device="cuda")
    hi = torch.tensor((idx.max(0) + 1) * bs, dtype=torch.float32, device="cuda")
    uniform = lo + torch.rand((n, 3), device="cuda", generator=g) * (hi - lo)
    k = n // 64  # trajectories x waypoints: each waypoint is a cluster of 64 spheres within 0.3 m
    starts = lo + torch.rand((max(k // 32, 1), 3), device="cuda", generator=g) * (hi - lo)
    steps = torch.randn((max(k // 32, 1), 32, 3), device="cuda", generator=g) * 0.05
    way = (starts[:, None, :] + torch.cumsum(steps, 1)).reshape(-1, 3)[:k]
    planner = (way[:, None, :] + (torch.rand((k, 64, 3), device="cuda", generator=g) - 0.5) * 0.6).reshape(-1, 3)
    return {"uniform": uniform.contiguous(), "planner": planner.contiguous()}


def time_launches(torch, fn, launches, stream):
    """Seconds per launch, from CUDA events recorded on the stream the query runs on."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(launches):
        fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / launches


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("query_profile: no CUDA device; the numbers are only meaningful on the GPU")
    info = gpu_info()
    import bench
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import _lib
    cam_s, frames = bench.make_frames(80, 0, 1)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    ms, occ, idx = build_maps(nvb, frames, cam)
    L = _lib.load()
    # the nvb_query_* calls run on the caller's stream (torch's current one); the per-layer calls on the mapper's stream
    mapper_stream = torch.cuda.ExternalStream(L.nvb_mapper_stream(ms[0]._h))
    rows = []
    for n in (1 << 16, 1 << 20, 1 << 24):
        for wname, pts in workloads(torch, idx, 0.4, n, 1).items():
            spheres = torch.cat([pts, torch.full((n, 1), 0.05, device="cuda")], 1)
            out4 = torch.full((n, 4), 100.0, device="cuda")
            out2 = torch.zeros((n, 2), device="cuda")
            out1 = torch.zeros((n, 1), device="cuda")
            vox = torch.zeros((n, 20), dtype=torch.uint8, device="cuda")
            ok = torch.zeros(n, dtype=torch.uint8, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream
            for k in (1, 2):
                hs = (C_void_p_array(k))(*[m._h.value for m in ms[:k]])
                # (name, call, bytes per query excluding the probes, voxel bytes read per mapper)
                kinds = [
                    ("esdf", lambda: L.nvb_query_esdf(hs, k, spheres.data_ptr(), n, 0, out1.data_ptr(), stream), 16 + 4, 8),
                    ("esdf_grad", lambda: L.nvb_query_esdf(hs, k, spheres.data_ptr(), n, 1, out4.data_ptr(), stream), 16 + 16, 20),
                    ("tsdf", lambda: L.nvb_query_tsdf(hs, k, pts.data_ptr(), n, out2.data_ptr(), stream), 12 + 8, 8),
                ]
                if k == 1:
                    ho = (C_void_p_array(1))(occ._h.value)
                    kinds += [
                        ("occupancy", lambda: L.nvb_query_occupancy(ho, 1, pts.data_ptr(), n, out1.data_ptr(), stream), 12 + 4, 4),
                        ("interpolate_tsdf", lambda: L.nvb_layer_interpolate(ms[0]._h, _lib.NVB_LAYER_TSDF, pts.data_ptr(),
                                                                             _lib.NVB_MEM_DEVICE, n, out1.data_ptr(), ok.data_ptr()),
                         12 + 5, 8 * 8),
                        ("voxels_esdf", lambda: L.nvb_layer_query_voxels(ms[0]._h, _lib.NVB_LAYER_ESDF, pts.data_ptr(),
                                                                         _lib.NVB_MEM_DEVICE, n, vox.data_ptr(), ok.data_ptr()),
                         12 + 21, 20),
                    ]
                for name, fn, io_bytes, voxel_bytes in kinds:
                    _lib.check(fn())
                    on_mapper = name in ("interpolate_tsdf", "voxels_esdf")
                    t = time_launches(torch, lambda: _lib.check(fn()), args.launches,
                                      mapper_stream if on_mapper else torch.cuda.current_stream())
                    probes = 1 if name == "interpolate_tsdf" else k  # interpolation: most points' 8 voxels share one block
                    bytes_q = io_bytes + probes * 12 + k * voxel_bytes
                    rows.append({"n": n, "workload": wname, "mappers": k, "kind": name, "time_us": t * 1e6,
                                 "queries_per_s": n / t, "alg_bytes_per_s": n * bytes_q / t,
                                 "share_of_hbm_bound": n * bytes_q / t / HBM_BYTES_PER_S})
    for m in ms + [occ]:
        m.close()
    print(json.dumps({"gpu": info, "hbm_bound_bytes_per_s": HBM_BYTES_PER_S, "rows": rows}))


def C_void_p_array(k):
    import ctypes
    return ctypes.c_void_p * k


if __name__ == "__main__":
    main()
