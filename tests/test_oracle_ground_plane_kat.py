"""Known-answer tests of the ground-plane restatement (tests/ground_plane_reference.py), no GPU: its XORWOW against the
toolkit's own curand_kernel.h generator run on the host, the reference's RansacPlaneFitter tests
(T/test_ransac_plane_fitter.cpp) and its zero-crossing tests (T/test_zero_crossings_extractor.cu)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import ground_plane_reference as gpr
from helpers import tsdf_layer_from_distance

NVCC = os.environ.get("NVCC") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc"))

_CURAND_HOST = r"""
#define QUALIFIERS static inline __host__ __device__
#include <curand_kernel.h>
#include <cstdio>
#include <cstdlib>
int main(int argc, char** argv) {
  const int n = atoi(argv[1]), draws = atoi(argv[2]);
  for (int i = 0; i < n; i++) {
    curandStateXORWOW_t s;
    curand_init(1234ull, (unsigned long long)i, 0ull, &s);
    for (int k = 0; k < draws; k++) printf("%u%c", curand(&s), k + 1 < draws ? ' ' : '\n');
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def curand_host(tmp_path_factory):
    if not NVCC:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("curand")
    src, exe = d / "xorwow.cu", d / "xorwow"
    src.write_text(_CURAND_HOST)
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(exe), str(src)])
    return str(exe)


def test_xorwow_first_draws_pinned():
    s = gpr.Xorwow(1234, 0)
    assert [s.next() for _ in range(3)] == [624778773, 1867875844, 3739671282]


def test_xorwow_matches_toolkit(curand_host):
    """curand_init(1234, i, 0) and the first draws for every subsequence 0..4096, as RansacPlaneFitter's iterations use them."""
    n, draws = 4097, 4
    out = subprocess.check_output([curand_host, str(n), str(draws)], text=True).split("\n")
    want = [list(map(int, line.split())) for line in out if line]
    got = [[st.next() for _ in range(draws)] for st in gpr.xorwow_states(1234, n)]
    assert got == want
    # the direct skip-ahead agrees with the chained one
    for i in (1, 77, 4096):
        s = gpr.Xorwow(1234, i)
        assert [s.next() for _ in range(draws)] == want[i]


def test_msac_sum_is_sequential():
    """np.add.accumulate keeps the float running sum of the kernel (np.sum would reduce pairwise)."""
    rng = np.random.default_rng(3)
    pts = rng.normal(0, 3, (3000, 3)).astype(np.float32)
    pl = gpr.plane_from_points(pts[0], pts[1], pts[2])
    cost = np.float32(0)
    t = np.float32(0.2)
    for p in pts:
        dist = np.float32(abs(np.float32(pl[0] * p[0] + np.float32(pl[1] * p[1] + pl[2] * p[2])) + pl[3]))
        cost = np.float32(cost + (np.float32(dist * dist) if dist < t else np.float32(t * t)))
    assert gpr.msac_cost(pl, pts, 0.2).view(np.uint32) == cost.view(np.uint32)


def _verify_plane_fit(plane, expected_normal, expected_offset, eps=1e-4):
    """verifyPlaneFit (T/lib/ransac_plane_fitter_utils.cpp:59-75), with its sign-flip rule."""
    assert plane is not None
    n, d = np.asarray(plane[:3], np.float64), float(plane[3])
    if np.float32(d) == -np.float32(expected_offset):
        assert abs(-expected_offset - d) <= eps and np.linalg.norm(np.asarray(expected_normal) - n) <= eps
    else:
        assert abs(expected_offset - d) <= eps and np.linalg.norm(-np.asarray(expected_normal) - n) <= eps


def test_fitter_degenerate_point_sets():
    """NoPointsPointCloud, TwoPointsPointCloud, ColliniearPointsPointCloud; duplicates only; a plane from three points."""
    assert gpr.ransac_fit(np.zeros((0, 3), np.float32)) is None
    assert gpr.ransac_fit(np.array([[0, 0, 0.1], [1, 0, 0.1]], np.float32)) is None
    assert gpr.ransac_fit(np.array([[0, 0, 0.1], [9, 0, 0.1], [1, 0, 0.1]], np.float32)) is None
    assert gpr.ransac_fit(np.tile(np.float32([1, 2, 3]), (10, 1))) is None
    assert gpr.plane_from_points([0, 0, 0], [1, 0, 0], [2, 0, 1e-7]) is None  # |cross| <= 1e-6: collinear
    assert gpr.plane_from_points([0, 0, 0], [1, 0, 0], [0, 0, 1e-5]) is not None


def test_fitter_known_planar_points():
    """FitToKnownPlanarPoints: seven points on z = 0.1."""
    pts = np.array([[0, 0, .1], [1, 0, .1], [2, 0, .1], [0, 1, .1], [1, 1, .1], [2, 1, .1], [.5, .5, .1]], np.float32)
    _verify_plane_fit(gpr.ransac_fit(pts), (0.0, 0.0, 1.0), 0.1)


def test_fitter_planar_points_with_corruption():
    """FitToPlanarPointsWithCorruption: 5 000 points on z = 10 over +-1000 m and 1 000 Gaussian outliers (sigma 2000, 2000,
    1 m about the origin)."""
    rng = np.random.default_rng(0)
    plane = np.column_stack([rng.uniform(-1000, 1000, (5000, 2)), np.full(5000, 10.0)])
    noise = rng.normal(0.0, (2000.0, 2000.0, 1.0), (1000, 3))
    _verify_plane_fit(gpr.ransac_fit(np.vstack([plane, noise]).astype(np.float32)), (0.0, 0.0, 1.0), 10.0)


def _layer(distance_fn, aabb_min, aabb_max, voxel_size=0.1, truncation_m=1.0):
    idx, vox = tsdf_layer_from_distance(distance_fn, aabb_min, aabb_max, voxel_size, truncation_m)
    return {tuple(int(v) for v in k): b for k, b in zip(idx, vox)}


@pytest.mark.parametrize("z", [-1.0, 0.04])
def test_zero_crossings_plane(z):
    """ZeroCrossingsFromAboveSimplePlane (z = -1) and ...AtBoundary (z = 0.04, in the lower half of the lowest voxels)."""
    cr = gpr.zero_crossings(_layer(lambda P: P[..., 2] - z, (0, 0, -2), (0.2, 0.2, 2)), 0.1)
    assert np.allclose(cr, [[0.05, 0.05, z], [0.05, 0.15, z], [0.15, 0.05, z], [0.15, 0.15, z]], atol=1e-6)


def test_zero_crossings_sphere():
    """ZeroCrossingsFromAboveSimpleSphere: r = 0.1 at the origin, four crossings at (+-0.05, +-0.05, 0.07071), tolerance 0.004."""
    cr = gpr.zero_crossings(_layer(lambda P: np.linalg.norm(P, axis=-1) - 0.1, (-0.5, -0.5, -0.5), (0.5, 0.5, 0.5)), 0.1)
    assert len(cr) == 4
    want = [[-0.05, -0.05, 0.07071], [-0.05, 0.05, 0.07071], [0.05, -0.05, 0.07071], [0.05, 0.05, 0.07071]]
    assert np.abs(cr - np.asarray(want)).max() <= 0.004


def test_max_crossings_and_empty_scene():
    """ZeroCrossingsFromAboveMaxCrossings: count >= max_crossings is 'not found'; an empty layer too."""
    layer = _layer(lambda P: P[..., 2], (-1, -1, -0.5), (1, 1, 0.5))
    n = len(gpr.zero_crossings(layer, 0.1))
    assert n == 400
    assert gpr.estimate(layer, 0.1, max_crossings=n) == (None, None, None)
    plane, cr, cand = gpr.estimate(layer, 0.1, max_crossings=n + 1)
    assert plane is not None and len(cr) == n and len(cand) == n
    assert gpr.estimate({}, 0.1) == (None, None, None)


def test_canonical_order():
    """Crossings come block by block in (x, y, z) order, then voxel (x, y, z) within a block."""
    layer = _layer(lambda P: P[..., 2] - 0.013 * P[..., 0], (-1.7, -1.7, -0.9), (1.7, 1.7, 0.9))
    cr = gpr.zero_crossings(layer, 0.1)
    bs = np.float32(0.8)
    blk = np.floor(cr[:, :2] / bs).astype(int)
    keys = list(zip(blk[:, 0], blk[:, 1]))
    assert keys == sorted(keys)


def test_ground_plane_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_ground_plane_dropin.cpp (nvblox_ros' ground-plane calls, MultiMapper with the estimator, the fitter on a
    Pointcloud, through nvblox/nvblox.h) builds with plain g++ against the mirror headers and the library."""
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_ground_plane_dropin")
    assert os.path.exists(exe)
