"""primitives::Scene without a GPU: the numpy restatement (tests/scene_reference.py) against float64 geometry, each of the
reference's quirks at +-1 ulp around kEpsilon where it switches, the reference's camera cases of tests/test_scene.cpp,
nvblox_torch's tests/test_scene.py on isaac_ros_nvblox_b200.scene.Scene, and the AABB's block enumeration."""
import math

import numpy as np
import pytest

import scene_reference as sr

F = np.float32
EPS = sr.EPS


def _unit(v):
    v = np.asarray(v, np.float64)
    return (v / np.linalg.norm(v)).astype(F)


def _prim(t, c, params):
    return (t, np.asarray(c, F), np.asarray(list(params) + [0.0] * (4 - len(params)), F))


PRIMS = {
    "plane": _prim(sr.PLANE, [0.3, 0.1, -0.2], _unit([0.0, 0.6, 0.8])),
    "cube": _prim(sr.CUBE, [0.2, -0.1, 0.3], [1.0, 0.5, 2.0]),
    "sphere": _prim(sr.SPHERE, [0.1, 0.2, 0.3], [1.2]),
    "cylinder": _prim(sr.CYLINDER, [-0.4, 0.3, 0.1], [0.7, 1.5]),
}


def _distance64(prim, p):
    t, c, q = prim
    p, c = p.astype(np.float64), c.astype(np.float64)
    if t == sr.PLANE:
        return (p - c) @ q[:3].astype(np.float64)
    if t == sr.SPHERE:
        return np.linalg.norm(p - c, axis=1) - q[0]
    if t == sr.CUBE:
        h = q[:3].astype(np.float64) / 2
        d = np.abs(p - c) - h
        out = np.linalg.norm(np.maximum(d, 0), axis=1)
        return np.where(out > 0, out, d.max(axis=1))
    r, h = float(q[0]), float(q[1]) / 2
    rho = np.linalg.norm(p[:, :2] - c[:2], axis=1)
    dz = np.abs(p[:, 2] - c[2]) - h
    side = rho - r
    cap = np.sqrt(np.maximum(rho ** 2 - r ** 2, 0) + dz ** 2)
    return np.where(dz <= 0, side, cap)


def _ray64(prim, o, u):
    """Nearest t >= 0 (inf if none) in float64; a sphere counts only from outside, a cylinder only its side and caps."""
    t, c, q = prim
    o, u, c = o.astype(np.float64), u.astype(np.float64), c.astype(np.float64)
    if t == sr.PLANE:
        n = q[:3].astype(np.float64)
        d = ((c - o) @ n) / (u @ n)
        return np.where(d >= 0, d, np.inf)
    if t == sr.SPHERE:
        oc = o - c
        b = u @ oc
        disc = b * b - oc @ oc + float(q[0]) ** 2
        d = -b - np.sqrt(np.maximum(disc, 0))
        return np.where((disc >= 0) & (d >= 0), d, np.inf)
    if t == sr.CUBE:
        h = q[:3].astype(np.float64) / 2
        with np.errstate(divide="ignore", invalid="ignore"):
            t1, t2 = (c - h - o) / u, (c + h - o) / u
        lo, hi = np.minimum(t1, t2).max(axis=1), np.maximum(t1, t2).min(axis=1)
        tt = np.where(lo >= 0, lo, hi)
        return np.where((lo <= hi) & (tt >= 0), tt, np.inf)
    raise NotImplementedError


@pytest.mark.parametrize("name", sorted(PRIMS))
def test_distances_match_float64_geometry(name):
    rng = np.random.default_rng(7)
    p = rng.uniform(-3, 3, (20000, 3)).astype(F)
    d = sr.distance(PRIMS[name], p)
    assert d.dtype == F
    np.testing.assert_allclose(d, _distance64(PRIMS[name], p), rtol=0, atol=4e-6)


@pytest.mark.parametrize("name", ["plane", "sphere", "cube"])
def test_ray_hits_match_float64_geometry(name):
    rng = np.random.default_rng(11)
    u = rng.normal(size=(20000, 3))
    u = (u / np.linalg.norm(u, axis=1)[:, None]).astype(F)
    o = np.array([2.5, 0.1, 0.2], F)
    hit, t = sr.ray(PRIMS[name], o, u, 100.0)
    t64 = _ray64(PRIMS[name], o, u)
    # away from grazing rays the two agree on hit / miss, and on t
    sure = np.isinf(t64) | (t64 < 50)
    if name == "plane":
        sure &= np.abs(u.astype(np.float64) @ PRIMS[name][2][:3]) > 1e-3
    assert np.mean(hit[sure] == np.isfinite(t64[sure])) > 0.999
    both = hit & np.isfinite(t64)
    np.testing.assert_allclose(t[both], t64[both], rtol=2e-5, atol=2e-5)


def _cylinder_ray64(prim, o, u):
    """Nearest t >= 0 (inf if none) of the rays with the cylinder's side (|z| <= h / 2) and caps (rho <= r), in float64."""
    c, r, h = prim[1].astype(np.float64), float(prim[2][0]), float(prim[2][1]) / 2
    E, u = o.astype(np.float64) - c, u.astype(np.float64)
    a = u[:, 0] ** 2 + u[:, 1] ** 2
    b = 2 * (E[0] * u[:, 0] + E[1] * u[:, 1])
    cc = E[0] ** 2 + E[1] ** 2 - r * r
    disc = b * b - 4 * a * cc
    best = np.full(u.shape[0], np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        for sgn in (-1, 1):
            t = (-b + sgn * np.sqrt(np.maximum(disc, 0))) / (2 * a)
            ok = (disc >= 0) & (t >= 0) & (np.abs(E[2] + t * u[:, 2]) <= h)
            best = np.where(ok & (t < best), t, best)
        for zc in (-h, h):
            t = (zc - E[2]) / u[:, 2]
            rho = np.hypot(E[0] + t * u[:, 0], E[1] + t * u[:, 1])
            ok = (t >= 0) & (rho <= r)
            best = np.where(ok & (t < best), t, best)
    return best


def test_cylinder_rays_match_float64_geometry():
    prim = PRIMS["cylinder"]
    rng = np.random.default_rng(5)
    u = rng.normal(size=(20000, 3))
    u = (u / np.linalg.norm(u, axis=1)[:, None]).astype(F)
    for o in (np.array([2.5, 0.1, 0.2], F), np.array([-0.3, 0.2, 2.0], F)):  # beside it, and above its top cap
        hit, t = sr.ray(prim, o, u, 100.0)
        t64 = _cylinder_ray64(prim, o, u)
        # away from near-vertical rays (which the reference ignores) the two agree on hit / miss, and on t
        sure = (u[:, 0].astype(np.float64) ** 2 + u[:, 1].astype(np.float64) ** 2) > 1e-3
        assert np.mean(hit[sure] == np.isfinite(t64[sure])) > 0.999
        assert np.isfinite(t64[sure]).sum() > 300
        both = hit & np.isfinite(t64)
        np.testing.assert_allclose(t[both], t64[both], rtol=2e-5, atol=2e-5)


# ---------------------------------------------------------------------------------------------------------------------
# Quirks, at +-1 ulp where they switch
# ---------------------------------------------------------------------------------------------------------------------
def _ulps_around(x, n=3):
    x = F(x)
    out = [x]
    lo = hi = x
    for _ in range(n):
        lo, hi = np.nextafter(lo, F(-np.inf)), np.nextafter(hi, F(np.inf))
        out = [lo] + out + [hi]
    return np.array(out, F)


def test_plane_distance_is_signed_and_ignores_parallel_rays():
    plane = _prim(sr.PLANE, [0, 0, 1], [0, 0, 1])
    assert sr.distance(plane, np.array([[0, 0, 0.25], [0, 0, 1.75]], F)).tolist() == [-0.75, 0.75]
    o = np.zeros(3, F)
    for z in _ulps_around(EPS):
        u = np.array([[np.sqrt(1 - np.float64(z) ** 2), 0, z]], F)
        den = sr._dot(u, np.array([0, 0, 1], F))[0]
        hit, t = sr.ray(plane, o, u, 1e6)
        assert bool(hit[0]) == (not abs(den) < EPS), z


def test_cube_distance_switches_to_the_largest_axis_term_below_kepsilon():
    cube = _prim(sr.CUBE, [0, 0, 0], [2, 2, 2])
    # outside near the x = y = 1 edge: the clamped norm a * sqrt(2) against the largest term a
    seen = set()
    for a in np.linspace(6e-5, 8e-5, 200).astype(F):
        p = np.array([[F(1) + a, F(1) + a, 0]], F)
        v = (p.astype(np.float64) - 1.0).astype(F)[0, :2]
        norm = np.sqrt(v[0] * v[0] + (v[1] * v[1] + F(0)))
        d = sr.distance(cube, p)[0]
        if norm < EPS:
            assert d == max(v[0], v[1]), a
            seen.add("max")
        else:
            assert d == norm, a
            seen.add("norm")
    assert seen == {"max", "norm"}
    # inside: the largest (negative) per-axis term
    assert sr.distance(cube, np.array([[0.5, 0.25, -0.1]], F))[0] == F(-0.5)


def test_sphere_ray_from_inside_misses_and_cube_ray_from_inside_exits():
    u = np.array([[1, 0, 0]], F)
    sphere, cube = _prim(sr.SPHERE, [0, 0, 0], [1]), _prim(sr.CUBE, [0, 0, 0], [2, 2, 2])
    assert not sr.ray(sphere, np.zeros(3, F), u, 10)[0][0]
    hit, t = sr.ray(cube, np.zeros(3, F), u, 10)
    assert hit[0] and t[0] == 1.0
    hit, t = sr.ray(sphere, np.array([-3, 0, 0], F), u, 10)
    assert hit[0] and t[0] == 2.0


def test_cylinder_ignores_near_vertical_rays_even_through_its_caps():
    cyl = _prim(sr.CYLINDER, [0, 0, 0], [1, 2])
    o = np.array([0, 0, 5], F)
    # a = ux^2 around kEpsilon: below it the ray misses although it crosses the top cap at t ~ 4
    results = {}
    for ux in _ulps_around(F(np.sqrt(np.float64(EPS))), 4):
        u = np.array([[ux, 0, -np.sqrt(1 - np.float64(ux) ** 2)]], F)
        a = u[0, 0] * u[0, 0] + u[0, 1] * u[0, 1]
        hit, t = sr.ray(cyl, o, u, 100)
        assert bool(hit[0]) == (not abs(a) < EPS), ux
        if hit[0]:
            assert abs(t[0] - 4.0) < 1e-3
        results[bool(hit[0])] = True
    assert results == {True: True, False: True}


def test_cylinder_treats_a_small_discriminant_as_one_root():
    cyl = _prim(sr.CYLINDER, [0, 0, 0], [1, 2])
    u = np.array([[0, 1, 0]], F)
    # disc = 4 (r^2 - x0^2): step x0 in ulps across disc = kEpsilon
    x0 = F(np.sqrt(1 - 2.5e-5))
    seen = set()
    for k in range(-40, 41):
        x = x0
        for _ in range(abs(k)):
            x = np.nextafter(x, F(np.inf) if k > 0 else F(-np.inf))
        o = np.array([x, -5, 0], F)
        E = o
        b = F(2) * E[0] * u[0, 0] + F(2) * E[1] * u[0, 1]
        cc = (E[0] * E[0] + E[1] * E[1]) - F(1)
        disc = b * b - F(4) * (u[0, 1] * u[0, 1]) * cc
        hit, t = sr.ray(cyl, o, u, 100)
        if disc < 0:
            assert not hit[0]
        elif disc <= EPS:
            assert hit[0] and t[0] == -b / (F(2) * F(1)), (k, disc)
            seen.add("one")
        else:
            assert hit[0] and t[0] == (-b - np.sqrt(disc)) / F(2), (k, disc)
            seen.add("two")
    assert seen == {"one", "two"}


def test_cylinder_caps_count_only_strictly_inside_the_radius():
    cyl = _prim(sr.CYLINDER, [0, 0, 0], [1, 2])
    # steep rays onto the top cap from above, landing at rho just inside / outside r (the side is not reached above z = 1)
    u = _unit([0.2, 0.0, -1.0])[None]
    for x_land, expect in ((0.999, True), (1.001, False)):
        o = np.array([x_land - 0.2 * 4, 0, 5], F)
        hit, t = sr.ray(cyl, o, u, 100)
        assert bool(hit[0]) == expect


# ---------------------------------------------------------------------------------------------------------------------
# The reference's tests/test_scene.cpp (camera) and nvblox_torch's tests/test_scene.py
# ---------------------------------------------------------------------------------------------------------------------
def _ocam():
    from oracle import oracle as orc
    return orc.Camera(300.0, 300.0, 320.0, 240.0, 640, 480)


def _quat_z_to_x():
    """Eigen::Quaternionf::FromTwoVectors((0, 0, 1), (1, 0, 0)) as a rotation matrix: +90 degrees about y."""
    return np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]], np.float64)


def test_blank_map(built):
    assert sr.signed_distance([], np.zeros((1, 3), F), 1.0)[0] == 1.0
    d = sr.depth_image([], _ocam(), np.eye(4, dtype=F), 1.0)
    assert np.all(d == 0.0)


@pytest.mark.parametrize("case", ["PlaneScene", "PlaneSceneVertical", "PlaneSceneVerticalOffset"])
def test_plane_scenes(built, case):
    T = np.eye(4)
    target = 1.0
    if case == "PlaneScene":
        plane = _prim(sr.PLANE, [0, 0, 1], [0, 0, -1])
    else:
        T[:3, :3] = _quat_z_to_x()
        plane = _prim(sr.PLANE, [1, 0, 0], [-1, 0, 0])
        if case == "PlaneSceneVerticalOffset":
            T[:3, 3] = [-1, 0, 0]
            target = 2.0
    d = sr.depth_image([plane], _ocam(), T.astype(F), 4.0, invalid_depth=-1.0)
    np.testing.assert_allclose(d, target, rtol=0, atol=1.1920929e-07 * 4)


def test_types_list(built):
    from isaac_ros_nvblox_b200.scene import Scene
    s = Scene()
    s.add_primitive("plane", [1, 0, 0, -1, 0, 0])
    s.add_primitive("sphere", [0, 0, 0, 1])
    s.add_primitive("cube", [0, 0, 0, 1, 1, 1])
    s.add_primitive("cylinder", [0, 0, 0, 1, 1])
    assert s.get_primitives_type_list() == ["kPlane", "kSphere", "kCube", "kCylinder"]


def test_nvblox_torch_scene_construction(built):
    """nvblox_torch's test_scene.py, less test_to_mapper (a GPU test in test_gpu_scene.py)."""
    from isaac_ros_nvblox_b200.scene import Scene
    s = Scene()
    assert s.get_aabb() == ([-5.0, -5.0, -1.0], [5.0, 5.0, 9.0])
    s.set_aabb([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])
    assert s.get_aabb() == ([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])
    s = Scene()
    s.add_plane_boundaries(x_min=0, x_max=1, y_min=2, y_max=3)
    assert s.get_primitives_type_list() == ["kPlane"] * 4
    s = Scene()
    s.add_ground_level(0.0)
    s.add_ceiling(1.0)
    assert s.get_primitives_type_list() == ["kPlane"] * 2
    s = Scene()
    s.add_primitive("cube", [0.0, 0.0, 0.0] + [1.0, 2.0, 3.0])
    s.add_primitive("sphere", [0.0, 0.0, 0.0] + [1.0])
    assert s.get_primitives_type_list() == ["kCube", "kSphere"]
    s = Scene()
    s.create_dummy_map()
    assert s.get_primitives_type_list() == ["kPlane"] * 6 + ["kCube", "kSphere"]
    s = Scene()
    s.add_primitive("plane", [0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    assert s.get_primitives_type_list() == ["kPlane"]
    # the plane's centre comes first, then its normal (py_scene.cu)
    p = sr.primitives_of(s)[0]
    assert p[1].tolist() == [0, 0, 0] and p[2][:3].tolist() == [0, 0, 1]


def test_scene_rejects_bad_primitives(built):
    from isaac_ros_nvblox_b200.scene import Scene
    s = Scene()
    with pytest.raises(ValueError):
        s.add_primitive("plane", [0, 0, 0, 0, 0, 1.01])
    with pytest.raises(ValueError):
        s.add_primitive("torus", [0, 0, 0, 1])
    with pytest.raises(ValueError):
        s.add_primitive("sphere", [0, 0, 0])
    s.add_primitive("plane", [0, 0, 0, 0, 0, 1.0009])  # within CHECK_NEAR's 1e-3


def test_plane_boundaries_order(built):
    from isaac_ros_nvblox_b200.scene import Scene
    s = Scene()
    s.add_plane_boundaries(-1, 2, -3, 4)
    got = [(p[1].tolist(), p[2][:3].tolist()) for p in sr.primitives_of(s)]
    assert got == [([-1, 0, 0], [1, 0, 0]), ([2, 0, 0], [-1, 0, 0]), ([0, -3, 0], [0, 1, 0]), ([0, 4, 0], [0, -1, 0])]


# ---------------------------------------------------------------------------------------------------------------------
# getBlockIndicesTouchedByBoundingBox
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aabb", [((-0.5, -0.1, 0.0), (0.3, 0.1, 0.4)), ((-5.3, -0.41, -2.0), (-4.01, -0.39, -1.99)),
                                  ((0.4, 0.4, 0.4), (0.8, 0.8, 0.8)), ((1.0, 1.0, 1.0), (1.0, 1.0, 1.0))])
def test_block_enumeration(aabb):
    bs = F(0.4)
    got = sr.blocks_touched(bs, aabb)
    lo, hi = np.asarray(aabb[0], F), np.asarray(aabb[1], F)
    # every block whose box [i * bs, (i + 1) * bs] contains the floor-indexed corners, and nothing else
    exp = [(x, y, z) for x in range(-20, 20) for y in range(-20, 20) for z in range(-20, 20)
           if all(math.floor(lo[k] / bs) <= (x, y, z)[k] <= math.floor(hi[k] / bs) for k in range(3))]
    assert [tuple(b) for b in got.tolist()] == exp
    assert len(got) == np.prod(np.floor(hi / bs) - np.floor(lo / bs) + 1)


def test_scene_dropin_compiles_against_the_mirror_headers(built, tmp_path):
    """tests/cpp/test_scene_dropin.cpp (the reference test's and py_scene.cu's calls through nvblox/nvblox.h) builds with
    plain g++ against the C-ABI library; its host-only part runs, and without a GPU it then exits 77."""
    import subprocess
    from isaac_ros_nvblox_b200 import _lib
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_scene_dropin")
    if _lib.load().nvb_device_count() == 0:
        assert subprocess.call([exe]) == 77
