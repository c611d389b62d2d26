"""The cube-by-cube mesh cases (tests/mesh_cube_cases.py): what they cover, and the oracle's mesh of every one of them
(oracle/nvblox_oracle.c, MeshIntegrator::integrateBlocksGPU) against the float64 restatement -- unwelded: the table's
triangle count per block, every vertex on its cube edge, unit or zero normals, planes on their plane; welded: the first
vertex of every 1 mm key group. This pins the oracle's mesh to geometry as well as to the reference's test_mesh.cpp."""
import numpy as np
import pytest

import mesh_cube_cases as mcc
from oracle import oracle as orc

CASES = {f.__name__: f for f in (mcc.config_sweep_case, mcc.neighbour_sweep_case, mcc.degenerate_case, mcc.weld_size_case,
                                 mcc.weld_origin_case, mcc.weld_collision_case, mcc.weld_saturation_case, mcc.plane_cases,
                                 mcc.colour_case)}
_cache = {}


def case(name):
    if name not in _cache:
        _cache[name] = CASES[name]()
    return _cache[name]


def oracle_mesh(c, weld):
    o = orc.OracleMap(c.voxel)
    for k, v in c.layer.items():
        o.set_tsdf_block(k, v)
    o.integrate_mesh(min_weight=c.min_weight, weld_vertices=weld, cutoff_distance_vox=c.cutoff_vox)
    return o.mesh_layer()


# ---- coverage of the generators
def test_config_sweep_has_all_256_configurations_in_each_of_the_8_position_classes():
    c = case("config_sweep_case")
    seen = {cls: set() for cls in range(8)}
    for key in c.info["lattice"]:
        cfg = mcc.cube_configs(c, key)
        for vx, vy, vz in np.argwhere(cfg >= 0):
            seen[mcc.position_class(vx, vy, vz)].add(int(cfg[vx, vy, vz]))
    assert all(len(seen[cls]) == 256 for cls in range(8)), {cls: len(s) for cls, s in seen.items()}
    assert all(set(p) == set(range(256)) for p in c.info["placed"].values())  # the isolated, chosen cubes alone cover them


def test_neighbour_sweep_has_all_128_upper_neighbour_patterns_and_crosses_every_supplied_face_edge_and_corner():
    c = case("neighbour_sweep_case")
    patterns = set()
    for key in c.info["centres"]:
        pat = mcc.neighbour_pattern(c, key)
        patterns.add(pat)
        cfg = mcc.cube_configs(c, key)
        for j, (ox, oy, oz) in enumerate(mcc.NB_DIRS[1:], start=1):
            # the cubes that reach into exactly the neighbours of direction j (and those between it and the block)
            sel = cfg[7 if ox else slice(0, 7), 7 if oy else slice(0, 7), 7 if oz else slice(0, 7)]
            needs = [jj for jj, d in enumerate(mcc.NB_DIRS) if jj and all(d[a] <= (ox, oy, oz)[a] for a in range(3))]
            if all((pat >> jj) & 1 for jj in needs):
                assert np.all((sel > 0) & (sel < 255)), (key, j)  # every such cube crosses the surface
            else:
                assert np.all(sel == -1), (key, j)
    assert len(patterns) == 128


def test_weld_sizes_straddle_every_sort_size_and_the_weld_limit():
    c = case("weld_size_case")
    got = sorted(len(mcc.expected_vertices(c, k)["v"]) for k in c.layer)
    assert got == sorted(mcc.WELD_SIZES)
    sort_size = [max(32, 1 << int(np.ceil(np.log2(n)))) for n in got if n < mcc.WELD_MAX]
    assert sorted(set(sort_size)) == [32, 64, 128, 256, 512, 1024, 2048, 4096]
    for p in (32, 128, 256, 512, 1024, 2048):  # each switch from both sides
        assert any(p // 2 < n <= p for n in got) and any(p < n <= 2 * p for n in got), p
    assert mcc.WELD_MAX - 1 in got and any(n >= mcc.WELD_MAX for n in got)


def test_degenerate_case_holds_the_values_it_names():
    c = case("degenerate_case")
    d = {k: v["distance"] for k, v in c.layer.items()}
    assert np.any((d[(0, 0, 0)] == 0) & ~np.signbit(d[(0, 0, 0)])) and np.any((d[(0, 0, 0)] == 0) & np.signbit(d[(0, 0, 0)]))
    t = np.float32(1e-4)
    diffs = sorted(np.float32(np.float32(a) - np.float32(b)) for a, b in c.info["threshold_pairs"])
    assert diffs == [np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))]
    ex = mcc.expected_vertices(c, (0, 0, 0))["v"].reshape(-1, 3, 3)
    assert np.any(np.all(ex[:, 0] == ex[:, 1], axis=1) & np.all(ex[:, 1] == ex[:, 2], axis=1))  # zero-area triangles
    w = c.layer[(0, 3, 0)]["weight"]
    mw = np.float32(c.min_weight)
    assert {float(x) for x in np.unique(w)} == {0.0, float(np.nextafter(mw, np.float32(0))), float(mw), 1.0, float("inf")}
    for k, want in c.info["meshable"].items():
        assert mcc.meshable(c, k) is want, k
        assert np.any((mcc.cube_configs(c, k) > 0) & (mcc.cube_configs(c, k) < 255)), k  # its cubes do cross
    cut = np.float32(c.info["cutoff"])
    assert np.abs(d[(3, 3, 0)]).min() == cut and np.abs(d[(0, 0, 3)]).min() == np.nextafter(cut, np.float32(1))


def test_weld_key_cases_reach_the_key_edges():
    u = oracle_mesh(case("weld_origin_case"), False)
    V = np.concatenate([b["vertices"] for b in u.values()])
    keys = mcc.weld_keys(V)
    assert np.any(keys == np.uint64(2 ** 64 - 1))
    kx = mcc.weld_key_coord(V[:, 0])
    assert np.any((kx == 0) & (V[:, 0] < 0)) and np.any((kx == 0) & (V[:, 0] > 0))
    # one block: two vertices more than 17 m apart with one key
    u = oracle_mesh(case("weld_collision_case"), False)
    V = u[(0, 0, 0)]["vertices"]
    keys = mcc.weld_keys(V)
    far = [(i, j) for i in range(len(V)) for j in range(len(V)) if keys[i] == keys[j] and V[j, 0] - V[i, 0] > 17.0]
    assert far
    # x * 1000 past both int32 limits, and one block with vertices on both sides of +2147483.647 m
    u = oracle_mesh(case("weld_saturation_case"), False)
    V = np.concatenate([b["vertices"] for b in u.values()])
    s = V[:, 0].astype(np.float32) * np.float32(1000)
    assert np.any(s >= 2.0 ** 31) and np.any(s < -2.0 ** 31)
    assert any(np.any(b["vertices"][:, 0] * np.float32(1000) >= 2.0 ** 31) and np.any(b["vertices"][:, 0] * np.float32(1000) < 2.0 ** 31)
               for b in u.values())


def test_plane_cases_cover_interiors_faces_edges_corners_and_voxel_centres_near_and_far():
    c = case("plane_cases")
    kinds = set(c.info["kinds"])
    assert {k for k, _ in kinds} == {"origin", "interior", "face", "edge", "corner", "voxel", "axis_face", "axis"}
    assert {r for _, r in kinds} == {0, 1}
    assert any(np.any(v["distance"] == 0) for v in c.layer.values())


# ---- the oracle against the float64 restatement
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_mesh_matches_float64_geometry(name):
    c = case(name)
    plain = oracle_mesh(c, False)
    mcc.check_unwelded(c, plain)
    mcc.check_welded(plain, oracle_mesh(c, True), name)
