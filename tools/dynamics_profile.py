"""Cost of the dynamics detection, of the connected-component mask filter and of a whole kDynamic frame on the GPU.

  detection : DynamicsDetection::computeDynamics at 640x480 and 1920x1080, every looked-up voxel high-confidence freespace
              (the most points to emit), device time per kernel from torch.profiler
  filter    : removeSmallConnectedComponents at 640x480 on a random mask at the 4-connected percolation density (0.593)
              and on a one-pixel-wide spiral, device time per kernel
  frame     : one kDynamic frame (background integrateDepth, detection, filter, the foreground's masked occupancy
              integration behind an event, updateFreespace) next to one kStaticTsdf frame (integrateDepth), host time
              with the synchronisations the calls make themselves
  syncs     : the host synchronisations and synchronous copies in the runtime trace of one kDynamic frame, and of the part
              between the detection and the foreground integration

Prints one JSON object with the card's name and power limit.

    python tools/dynamics_profile.py [--repeats 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from ground_plane_profile import gpu_info  # noqa: E402

DETECT_KERNELS = ("dynamicsDetectKernel", "exclusiveScanInt2Kernel", "dynamicsEmitKernel")
FILTER_KERNELS = ("ccLocalKernel", "ccMergeKernel", "ccCountKernel", "ccOutputKernel")
SYNC_CALLS = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy", "cuStreamSynchronize",
              "cuMemcpyDtoH_v2", "cuMemcpyHtoD_v2")


def kernel_times(fn, names, repeats):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in names:
            if name in e.key:
                out[name] = {"us": round(e.device_time_total / max(e.count, 1), 2), "calls": e.count}
    return out


def sync_calls(fn):
    """Synchronising runtime / driver calls traced while fn runs (exact names; cudaMemcpyAsync is not one of them)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
    torch.cuda.synchronize()
    counts = {}
    for e in prof.events():
        if e.name in SYNC_CALLS:
            counts[e.name] = counts.get(e.name, 0) + 1
    return counts


def host_us(fn, repeats):
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e6)
    return {"median": float(np.median(ts)), "min": float(np.min(ts))}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import torch
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import synthetic as syn
    from isaac_ros_nvblox_b200.mapper import remove_small_connected_components_device
    import dynamics_reference as dref
    res = {"gpu": gpu_info()}

    # detection on a freespace layer that is high-confidence everywhere in view
    res["detection"] = {}
    for rows, cols in ((480, 640), (1080, 1920)):
        f = 300.0 * cols / 640.0
        cam = nvb.Camera(f, f, cols / 2.0, rows / 2.0, cols, rows)
        m = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)
        rng = np.random.default_rng(0)
        depth = rng.uniform(0.5, 4.0, (rows, cols)).astype(np.float32)
        rr, cc = np.nonzero(depth > 0)
        p = dref.unproject_transform(depth[rr, cc], np.eye(4), {"fu": f, "fv": f, "cu": cols / 2.0, "cv": rows / 2.0}, rr, cc)
        keys = np.unique(np.floor(p / np.float32(0.4)).astype(np.int32), axis=0)
        vox = np.zeros((len(keys), 8, 8, 8), nvb.FREESPACE_VOXEL_DTYPE)
        vox["is_high_confidence_freespace"] = 1
        m.freespace_layer().set_blocks(keys, vox)
        d_dev = torch.from_numpy(depth).cuda()
        torch.cuda.synchronize()
        det = m.dynamics_detection()
        T = np.eye(4, dtype=np.float32)
        run = lambda: det.compute_dynamics_device(d_dev.data_ptr(), rows, cols, T, cam)  # noqa: E731
        run()
        m.synchronize()
        res["detection"]["%dx%d" % (cols, rows)] = {"points": len(det.dynamic_points()),
                                                    "kernel_us": kernel_times(run, DETECT_KERNELS, args.repeats)}
        m.close()

    # the filter at 640x480
    m = nvb.Mapper(0.05, tsdf_capacity_blocks=64, esdf_capacity_blocks=64)
    rng = np.random.default_rng(1)
    masks = {"random_0.593": ((rng.random((480, 640)) < 0.593) * 255).astype(np.uint8), "spiral": dref.spiral_mask(480, 640)}
    res["filter_640x480"] = {}
    for name, mk in masks.items():
        src = torch.from_numpy(mk).cuda()
        dst = torch.empty_like(src)
        torch.cuda.synchronize()
        run = lambda: remove_small_connected_components_device(src.data_ptr(), dst.data_ptr(), 480, 640, 2000, m)  # noqa: E731
        run()
        m.synchronize()
        assert np.array_equal(dst.cpu().numpy(), dref.remove_small_connected_components(mk, 2000))
        kt = kernel_times(run, FILTER_KERNELS, args.repeats)
        res["filter_640x480"][name] = {"components": int(len(dref.component_sizes(mk))), "kernel_us": kt,
                                       "total_us": round(sum(v["us"] for v in kt.values()), 2)}
    m.close()
    r = res["filter_640x480"]
    res["filter_640x480"]["spiral_over_random"] = round(r["spiral"]["total_us"] / max(r["random_0.593"]["total_us"], 1e-9), 3)

    # one kDynamic frame next to one kStaticTsdf frame (640x480, a wall with a box moving across it)
    scam = syn.PinholeCamera()
    cam = nvb.Camera(scam.fu, scam.fv, scam.cu, scam.cv, scam.width, scam.height)
    T = np.eye(4, dtype=np.float32)
    wall = syn.render_depth(syn.plane_scene(4.0), scam, np.eye(4), max_dist=8.0)
    bg = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kTsdfWithFreespace)
    fg = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    st = nvb.Mapper(0.05)
    state = {"i": 0}

    def frame_depth():
        i = state["i"]
        d = wall.copy()
        c0 = 100 + (i * 7) % 400
        d[150:330, c0:c0 + 120] = 2.0
        return d

    def detect_and_filter(d):
        det = bg.dynamics_detection()
        det.compute_dynamics(d, T, cam)
        b = det.device_buffers()
        remove_small_connected_components_device(b["mask"], b["cleaned_mask"], 480, 640, 2000, bg)
        fg.wait_for(bg)
        return b

    def dynamic_frame():
        d = frame_depth()
        bg.integrate_depth(d, T, cam, return_blocks=False)
        b = detect_and_filter(d)
        fg.integrate_depth_device(b["depth"], 480, 640, T, cam, mask_ptr=b["cleaned_mask"], sync=True)
        bg.update_freespace(100 * state["i"], depth=d, T_L_C=T, camera=cam)
        state["i"] += 1

    def static_frame():
        st.integrate_depth(frame_depth(), T, cam, return_blocks=False)
        state["i"] += 1

    for _ in range(15):  # warm-up; the wall's freespace turns high-confidence
        dynamic_frame()
        static_frame()
    res["frame_640x480_us"] = {"kDynamic": host_us(dynamic_frame, args.repeats), "kStaticTsdf": host_us(static_frame, args.repeats)}
    res["dynamic_points_last_frame"] = len(bg.dynamics_detection().dynamic_points())
    d = frame_depth()
    # "empty": what tracing nothing records (the profiler's own calls), to subtract from the two others
    res["sync_calls"] = {"empty": sync_calls(lambda: None), "kDynamic_frame": sync_calls(dynamic_frame),
                         "detection_to_foreground": sync_calls(lambda: detect_and_filter(d))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
