"""Time primitives::Scene on the GPU with CUDA events: depth images (640x480, 1920x1080) of the dummy scene and of 1000
primitives, layer generation of the default 10 x 10 x 10 m box at 5 cm and 2 cm, and nvblox_torch's toMapper with its ESDF
update. The card's name and power limit are read in the same run. Writes one JSON object to stdout (and to --out)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps, warmup=5):
    """Mean milliseconds per call between CUDA events, after `warmup` calls (module loads, the stream-ordered memory pool)."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import scene as sc
    dummy = sc.Scene()
    dummy.create_dummy_map()
    many = sc.Scene()
    rng = np.random.default_rng(0)
    for c in rng.uniform(-4, 4, (1000, 3)):
        kind = rng.integers(0, 3)
        if kind == 0:
            many.add_primitive("cube", list(c) + list(rng.uniform(0.1, 0.5, 3)))
        elif kind == 1:
            many.add_primitive("sphere", list(c) + [float(rng.uniform(0.1, 0.4))])
        else:
            many.add_primitive("cylinder", list(c) + [float(rng.uniform(0.1, 0.3)), float(rng.uniform(0.2, 1.0))])
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = [[0, 0, 1], [-1, 0, 0], [0, -1, 0]]  # looking along +x
    T[:3, 3] = [-4.5, 0.0, 2.0]
    res = {"card": card()}
    for name, s in (("dummy", dummy), ("1000_primitives", many)):
        for w, h, f in ((640, 480, 320.0), (1920, 1080, 960.0)):
            cam = nvb.Camera(f, f, w / 2, h / 2, w, h)
            res["depth_%s_%dx%d_ms" % (name, w, h)] = timed(lambda: s.render_depth(cam, T, 20.0, device=0), 50)
    box = sc.Scene()
    box.create_dummy_map()
    box.set_aabb(*sc.DEFAULT_AABB)
    for vs in (0.05, 0.02):
        m = nvb.Mapper(vs)
        box.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 4 * vs)  # slab growth out of the timed window
        res["generate_tsdf_default_box_%gcm_ms" % (vs * 100)] = timed(
            lambda: box.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 4 * vs), 5)
        res["blocks_%gcm" % (vs * 100)] = m.tsdf_layer().num_blocks()
        res["to_mapper_with_esdf_%gcm_ms" % (vs * 100)] = timed(lambda: box.append_to_mapper(m), 3)
    # the same fill with one plane instead of the dummy scene's 8 primitives: what is left is allocation and stores
    plane = sc.Scene()
    plane.add_ground_level(0.0)
    m = nvb.Mapper(0.02)
    plane.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 0.08)
    res["generate_tsdf_default_box_2cm_one_plane_ms"] = timed(lambda: plane.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 0.08), 5)
    cube = sc.Scene()
    cube.add_primitive("cube", [0, 0, 2, 2, 2, 2])
    cube.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 0.08)
    res["generate_tsdf_default_box_2cm_one_cube_ms"] = timed(lambda: cube.generate_layer(m, nvb._lib.NVB_LAYER_TSDF, 0.08), 5)
    torch.cuda.synchronize()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
