"""Times the map file and point export paths on one GPU: save_layer_cake, load_map, a full colour-mesh update alone (the last
step of a load) and export_points per layer, on an 80-frame map of the synthetic sphere-in-box scene at 640x480 and 5 cm voxels.
Prints one JSON line with the card's name and power limit. Writes only under the given directory (default: a temporary one).
    python tools/map_io_profile.py [--out DIR] [--repeats N]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, repeats):
    best = float("inf")
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()  # every call below ends in a device synchronisation
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import isaac_ros_nvblox_b200 as nvb
    from isaac_ros_nvblox_b200 import synthetic as syn
    cs = syn.PinholeCamera(300.0, 300.0, 320.0, 240.0, 640, 480)
    cam = nvb.Camera(cs.fu, cs.fv, cs.cu, cs.cv, cs.width, cs.height)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(80), noise_sigma_rel=0.005, seed=7)
    m = nvb.Mapper(0.05)
    for d, T in frames:
        m.integrate_depth(d, T, cam)
        m.update_esdf()
    m.update_mesh()
    out = args.out or tempfile.mkdtemp()
    path = os.path.join(out, "map.nvblx")
    m2 = nvb.Mapper(0.05)
    res = {"tsdf_blocks": m.tsdf_layer().num_blocks(), "esdf_blocks": m.esdf_layer().num_blocks(),
           "save_ms": timed(lambda: m.save_layer_cake(path), args.repeats), "file_bytes": os.path.getsize(path),
           "load_ms": timed(lambda: m2.load_map(path), args.repeats),
           "full_mesh_update_ms": timed(lambda: m2.update_mesh(update_full_layer=True), args.repeats)}
    for name in ("tsdf", "esdf"):
        layer = getattr(m, name + "_layer")()
        res["export_%s_ms" % name] = timed(layer.export_points, args.repeats)
        res["export_%s_points" % name] = len(layer.export_points())
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = smi.stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
