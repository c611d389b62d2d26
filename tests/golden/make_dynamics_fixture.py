"""Builds tests/golden/dynamics_human.npz from the reference's own test data, given a checkout of
NVIDIA-ISAAC-ROS/isaac_ros_nvblox:

    python tests/golden/make_dynamics_fixture.py <isaac_ros_nvblox checkout>

  * nvblox/tests/data/human_dataset/depth_image_{1,2}.png: two 16-bit depth frames of a static camera with a person walking
    (test_dynamics.cpp HumanDataset), stored raw (uint16 millimetres); the tests convert them like io::readFromPng,
    float(u16) * kDefaultUintDepthScaleFactor with kDefaultUintDepthScaleFactor = 1.0f / 1000.0f (a multiply);
  * its camera-intrinsics.txt, parsed like parseCameraFromFile (float32 3x3);
  * nvblox/tests/data/dynamic_mask/mask_21.png: the 8-bit mask of test_mask_preprocessor.cpp RealMask.
SHA-256 digests of the arrays as read from the reference's files go to dynamics_human_sources.json, which
tests/test_oracle_dynamics_kat.py checks the fixture against.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
DATA_IN_CHECKOUT = os.path.join("nvblox_ros", "nvblox_core", "nvblox", "tests", "data")
OUT = os.path.join(ROOT, "tests", "golden", "dynamics_human.npz")
SOURCES = os.path.join(ROOT, "tests", "golden", "dynamics_human_sources.json")
INPUT_NAMES = ("intrinsics", "depth_u16", "mask_21")


def array_digest(a):
    a = np.ascontiguousarray(a)
    return {"dtype": a.dtype.str, "shape": list(a.shape), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def load_reference_data(checkout):
    from PIL import Image
    data = os.path.join(checkout, DATA_IN_CHECKOUT)
    human = os.path.join(data, "human_dataset")
    K = np.array([[np.float32(t) for t in line.split()] for line in open(os.path.join(human, "camera-intrinsics.txt")) if line.strip()],
                 np.float32)
    depth = []
    for i in (1, 2):
        d = np.array(Image.open(os.path.join(human, "depth_image_%d.png" % i)))
        assert d.dtype == np.uint16 and d.ndim == 2
        depth.append(d)
    mask = np.array(Image.open(os.path.join(data, "dynamic_mask", "mask_21.png")))
    assert mask.dtype == np.uint8 and mask.shape == (480, 640)
    assert int((mask > 0).sum()) == 14073
    return K, np.stack(depth), mask


def main(checkout):
    arrays = load_reference_data(checkout)
    np.savez_compressed(OUT, **dict(zip(INPUT_NAMES, arrays)))
    with open(SOURCES, "w") as f:
        json.dump({n: array_digest(a) for n, a in zip(INPUT_NAMES, arrays)}, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, SOURCES)


if __name__ == "__main__":
    main(sys.argv[1])
