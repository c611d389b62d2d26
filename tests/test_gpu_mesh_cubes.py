"""The mesh kernels (isaac_ros_nvblox_b200/csrc/nvb_mesh.cu) cube by cube, on the cases of tests/mesh_cube_cases.py: all
256 configurations in every position class, all 128 upper-neighbour patterns, degenerate values, every weld sort size,
weld-key edges, planes and per-voxel colours. Every case goes through the explicit block list
(MeshIntegrator::integrateBlocksGPU) and the full-layer tracker update (Mapper::updateColorMesh(kFull)), welded and
unwelded, and must equal the oracle array for array; the unwelded mesh must also equal the float64 restatement, and the
welded mesh the 1 mm key grouping of the unwelded one. The TSDF is placed with set_blocks, which the mesh tracker does not
hear about, so the tracker path runs as a full-layer update."""
import numpy as np
import pytest

import mesh_cube_cases as mcc
from test_gpu_mesh import assert_mesh_equal

pytestmark = pytest.mark.gpu

CASES = {f.__name__: f for f in (mcc.config_sweep_case, mcc.neighbour_sweep_case, mcc.degenerate_case, mcc.weld_size_case,
                                 mcc.weld_origin_case, mcc.weld_collision_case, mcc.weld_saturation_case, mcc.plane_cases,
                                 mcc.colour_case)}
PATHS = ("list", "tracker")


def _mapper(c, weld):
    import isaac_ros_nvblox_b200 as nvb
    m = nvb.Mapper(c.voxel)
    keys = np.array(sorted(c.layer), np.int32)
    m.tsdf_layer().set_blocks(keys, np.stack([c.layer[tuple(k)] for k in keys]))
    if c.color:
        ck = np.array(sorted(c.color), np.int32)
        m.color_layer().set_blocks(ck, np.stack([c.color[tuple(k)] for k in ck]))
    m.mesh_integrator().params(min_weight=c.min_weight, weld_vertices=1 if weld else 0, cutoff_distance_vox=c.cutoff_vox)
    return m


def gpu_mesh(c, weld, path):
    m = _mapper(c, weld)
    if path == "list":
        m.mesh_integrator().integrate_blocks(np.array(sorted(c.layer), np.int32), update_color=c.color is not None)
    else:
        m.update_mesh(update_full_layer=True)
    out = m.mesh_layer().as_dict()
    m.close()
    return out


def oracle_mesh(c, weld):
    from oracle import oracle as orc
    o = orc.OracleMap(c.voxel)
    for k, v in c.layer.items():
        o.set_tsdf_block(k, v)
    o.integrate_mesh(min_weight=c.min_weight, weld_vertices=weld, cutoff_distance_vox=c.cutoff_vox)
    return o.mesh_layer()


@pytest.fixture(scope="module")
def runs(gpu):
    """{name: case}, {(name, path or "oracle", weld): mesh layer}."""
    cases, meshes = {}, {}
    for name, f in CASES.items():
        c = cases[name] = f()
        for weld in (False, True):
            meshes[(name, "oracle", weld)] = oracle_mesh(c, weld)
            for path in PATHS:
                meshes[(name, path, weld)] = gpu_mesh(c, weld, path)
    return cases, meshes


@pytest.mark.parametrize("weld", [False, True])
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_mesh_equals_oracle(runs, name, path, weld):
    _, meshes = runs
    assert_mesh_equal(meshes[(name, path, weld)], meshes[(name, "oracle", weld)])


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_unwelded_mesh_matches_float64_geometry(runs, name, path):
    """Per block the table's triangle count over its valid cubes; every vertex on its cube edge (interpolated, or the
    midpoint below the 1e-4f switch) within a few float32 ulp; unit or zero normals; plane vertices on their plane."""
    cases, meshes = runs
    mcc.check_unwelded(cases[name], meshes[(name, path, False)])


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_welded_mesh_is_the_key_grouping_of_the_unwelded_mesh(runs, name, path):
    """Welded corners are the first vertex, in (key, index) order, of their 1 mm key group; nv is the number of keys below
    2560 vertices and unchanged from 2560; `triangles` keeps its length."""
    _, meshes = runs
    mcc.check_welded(meshes[(name, path, False)], meshes[(name, path, True)], name)


@pytest.mark.parametrize("weld", [False, True])
@pytest.mark.parametrize("path", PATHS)
def test_vertex_colours_are_the_closest_colour_voxel(runs, path, weld):
    cases, meshes = runs
    c = cases["colour_case"]
    mesh = meshes[("colour_case", path, weld)]
    want, clamped = mcc.expected_colors(c, mesh)
    assert clamped > 0  # vertices past the upper faces, whose index 8 clamps to 7
    assert any(k not in c.color for k in mesh)  # blocks without a colour block: Gray
    for k, b in mesh.items():
        assert len(b["colors"]) == len(b["vertices"]), k
        assert np.array_equal(b["colors"][:, :3], want[k]), k
        assert np.all(b["colors"][:, 3] == 255), k


def test_one_call_outgrows_the_mesh_arena(gpu):
    """A single call needs more arena than is left after a first, small one: the arena is repacked inside the call and the
    mesh equals the oracle's and the float64 restatement."""
    c = mcc.noise_case()
    first = {k: v for k, v in list(c.layer.items())[:2]}
    m = _mapper(c, False)
    mi = m.mesh_integrator()
    mi.integrate_blocks(np.array(sorted(first), np.int32))
    before = m.mesh_layer().arena_stats()
    mi.integrate_blocks(np.array(sorted(c.layer), np.int32))
    after = m.mesh_layer().arena_stats()
    assert after["last_update_vertices"] > before["capacity"] - before["used"]
    assert after["capacity"] > before["capacity"] and after["used"] <= after["capacity"]
    got = m.mesh_layer().as_dict()
    m.close()
    mcc.check_unwelded(c, got)
    assert_mesh_equal(got, oracle_mesh(c, False))
