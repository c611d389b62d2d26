"""Generates tests/golden/map_small.nvblx: the CPU oracle's TSDF and ESDF of the c2_small inputs (tests/golden/c2_small.npz,
4 frames, 160x120, 10 cm voxels), the first NUM_BLOCKS blocks in (x, y, z) order of each (the file stays small), in the
reference's map file layout, written with the reference's statements
(tests/map_io_reference.py) in one fixed table order. Run from the repo root:
    python tests/golden/make_map_fixture.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import map_io_reference as ref  # noqa: E402
from oracle import oracle as orc  # noqa: E402

# a fixed order that is not the loader's own table order
NUM_BLOCKS = 24
ORDER = ("esdf_layer", "color_layer", "occupancy_layer", "freespace_layer", "feature_layer", "tsdf_layer")


def oracle_map():
    g = np.load(os.path.join(HERE, "c2_small.npz"))
    c = g["cam"]
    cam = orc.Camera(float(c[0]), float(c[1]), float(c[2]), float(c[3]), int(c[4]), int(c[5]))
    o = orc.OracleMap(float(g["voxel_size"]))
    for d, T in zip(g["depth"], g["poses"]):
        o.integrate_esdf(o.integrate_depth(d, T, cam))
    return o, float(g["voxel_size"])


def first_blocks(layer):
    return {k: layer[k] for k in sorted(layer)[:NUM_BLOCKS]}


def main():
    o, voxel = oracle_map()
    layers = {"tsdf_layer": ref.layer_rows(first_blocks(o.tsdf_layer()), orc.TSDF_VOXEL_DTYPE),
              "esdf_layer": ref.layer_rows(first_blocks(o.esdf_layer()), orc.ESDF_VOXEL_DTYPE)}
    path = os.path.join(HERE, "map_small.nvblx")
    if os.path.exists(path):
        os.remove(path)
    ref.write_map(path, layers, np.float32(voxel) * np.float32(8), ORDER)
    print(path, {k: len(v[1]) for k, v in layers.items()})


if __name__ == "__main__":
    main()
