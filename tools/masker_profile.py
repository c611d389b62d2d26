"""Cost of the image masker and of a whole human-mapping frame on the GPU, for a 640 x 480 depth frame with a 1280 x 720
mask camera (the depth / colour pair of tests/camera_pose_cases.py: 5 cm baseline, 1 degree rotation).

  split   : the three-launch depth split (fill, min depth, split) with device inputs, timed with CUDA events on the
            mapper's stream over many splits; and the device time of each kernel from torch.profiler
  frame   : one human frame as MultiMapper runs it: the connected-component filter and the split on the background
            mapper's stream, the TSDF background integrating the background frame, the occupancy foreground integrating
            the foreground frame behind an event; CUDA events from the first launch to the foreground's last kernel
            (integrateDepth waits for its kernels, so the events bracket the whole frame)

Prints one JSON object with the card's name and power limit.

    python tools/masker_profile.py [--repeats 200]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from dynamics_profile import kernel_times  # noqa: E402
from ground_plane_profile import gpu_info  # noqa: E402

SPLIT_KERNELS = ("maskerFillKernel", "maskerMinDepthKernel", "maskerSplitDepthKernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=200)
    args = ap.parse_args()
    import torch
    import camera_pose_cases as cpc
    import isaac_ros_nvblox_b200 as nvb
    import masker_reference as mr
    dc, mc = cpc.COLOR_DEPTH_CAM, cpc.COLOR_CAM
    cam = nvb.Camera(dc["fu"], dc["fv"], dc["cu"], dc["cv"], dc["width"], dc["height"])
    mcam = nvb.Camera(mc["fu"], mc["fv"], mc["cu"], mc["cv"], mc["width"], mc["height"])
    depth, mask, T_CM_CD, _, _ = mr.colour_camera_case()
    T_L_D = cpc.color_poses(1)[0][0]
    td, tm = torch.from_numpy(depth).cuda(), torch.from_numpy(mask).cuda()
    tclean = torch.empty_like(tm)
    rows, cols, mrows, mcols = dc["height"], dc["width"], mc["height"], mc["width"]
    out = {"gpu": gpu_info(), "depth": [rows, cols], "mask": [mrows, mcols], "repeats": args.repeats,
           "masked_fraction": float(mr.split_depth(depth, mask, T_CM_CD, dc, mc)[3].mean())}

    bg = nvb.Mapper(0.05)
    fg = nvb.Mapper(0.05, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy)
    masker = nvb.ImageMasker(bg)
    stream = torch.cuda.ExternalStream(bg.cuda_stream())
    torch.cuda.synchronize()

    def split():
        masker.split_depth_device(td.data_ptr(), rows, cols, tm.data_ptr(), mrows, mcols, T_CM_CD, cam, mcam, overlay=True)

    for _ in range(20):
        split()
    bg.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(args.repeats):
        split()
    e1.record(stream)
    e1.synchronize()
    out["split_us_per_call"] = round(e0.elapsed_time(e1) * 1000.0 / args.repeats, 2)
    out["split_kernels"] = kernel_times(lambda: (split(), bg.synchronize()), SPLIT_KERNELS, 50)

    def frame():
        nvb.mapper.remove_small_connected_components_device(tm.data_ptr(), tclean.data_ptr(), mrows, mcols, 2000, bg)
        b = masker.split_depth_device(td.data_ptr(), rows, cols, tclean.data_ptr(), mrows, mcols, T_CM_CD, cam, mcam, overlay=True)
        bg.integrate_depth_device(b["background"], rows, cols, T_L_D, cam)
        fg.wait_for(bg)
        fg.integrate_depth_device(b["foreground"], rows, cols, T_L_D, cam, sync=True)

    for _ in range(10):
        frame()
    bg.synchronize()
    times = []
    fstream = torch.cuda.ExternalStream(fg.cuda_stream())
    for _ in range(max(args.repeats // 4, 10)):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(stream)
        frame()
        e.record(fstream)
        e.synchronize()
        times.append(s.elapsed_time(e) * 1000.0)
    bg.synchronize()
    out["human_frame_us_median"] = round(float(np.median(times)), 1)
    out["human_frame_us_p10_p90"] = [round(float(np.percentile(times, 10)), 1), round(float(np.percentile(times, 90)), 1)]
    bg.close()
    fg.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
