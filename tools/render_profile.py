"""Throughput of the SphereTracer renders on the GPU (nvb_render_depth / nvb_render_rgbd in nvb_color.cu), timed with CUDA
events over many launches after warm-up.

Map: bench.py's c2 map (80 frames of the sphere-in-box circle, 640x480, 5 cm voxels) with colour integrated from every 4th
frame. Renders from three of its poses, depth and RGBD, at 640x480 and 1920x1080 (the same field of view), with ray
subsampling 1 and 4, truncation 4 voxels and the tracer's defaults (100 steps, 15 m). For each: time per render, rays/s and
the share of rays that hit. Prints one JSON object with the card's name and power limit. Fails without a GPU.

    python tools/render_profile.py [--launches 50]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def time_launches(torch, fn, launches):
    """Seconds per launch, from CUDA events recorded on torch's current stream (the one the renders run on)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / launches


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("render_profile: no CUDA device; the numbers are only meaningful on the GPU")
    info = gpu_info()
    import bench
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import _lib
    from isaac_ros_nvblox_b200.mapper import _fp, colmajor
    cam_s, frames = bench.make_frames(80, 0, 1)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    m = nvb.Mapper(0.05)
    rng = np.random.default_rng(0)
    for i, (d, T) in enumerate(frames):
        m.integrate_depth(d, T, cam, return_blocks=False)
        if i % 4 == 0:
            m.integrate_color(rng.integers(0, 256, (cam_s.height, cam_s.width, 3), dtype=np.uint8), T, cam, return_blocks=False)
    m.synchronize()
    L = _lib.load()
    p = _lib.NvbSphereTracerParams()
    L.nvb_default_sphere_tracer_params(C.byref(p))
    trunc = 4.0 * m.voxel_size()
    scale = 1920.0 / cam_s.width
    cams = {"640x480": cam, "1920x1080": nvb.Camera(cam_s.fu * scale, cam_s.fv * scale, 960.0, 540.0, 1920, 1080)}
    rows = []
    for size, c in cams.items():
        for f in (1, 4):
            h, w = c.height // f, c.width // f
            depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
            rgb = torch.empty((h, w, 3), dtype=torch.uint8, device="cuda")
            for i in (0, 27, 53):
                T = _fp(colmajor(frames[i][1]))
                stream = torch.cuda.current_stream().cuda_stream
                kinds = {
                    "depth": lambda: L.nvb_render_depth(m._h, C.byref(p), T, C.byref(c.c), trunc, f, _lib.NVB_MEM_DEVICE,
                                                        depth.data_ptr(), stream),
                    "rgbd": lambda: L.nvb_render_rgbd(m._h, C.byref(p), T, C.byref(c.c), trunc, f, _lib.NVB_MEM_DEVICE,
                                                      depth.data_ptr(), rgb.data_ptr(), stream),
                }
                for kind, fn in kinds.items():
                    _lib.check(fn())
                    t = time_launches(torch, lambda: _lib.check(fn()), args.launches)
                    hits = float((depth > 0).float().mean())
                    rows.append({"image": size, "f": f, "pose": i, "kind": kind, "rays": h * w, "time_us": t * 1e6,
                                 "rays_per_s": h * w / t, "hit_fraction": hits})
    m.close()
    print(json.dumps({"gpu": info, "rows": rows}))


if __name__ == "__main__":
    main()
