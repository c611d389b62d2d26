"""Map files and voxel-layer point export on the GPU: save / load round trips against the restatement of the reference's file
(tests/map_io_reference.py), the reference-layout fixture, continuing a loaded map against the oracle, the failure cases,
and the PLY points of every voxel layer."""
import os
import shutil
import sqlite3
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import map_io_reference as ref  # noqa: E402
from helpers import assert_esdf_equal, assert_tsdf_equal, cameras  # noqa: E402
from isaac_ros_nvblox_b200 import synthetic as syn  # noqa: E402

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(HERE, "golden", "map_small.nvblx")
LAYERS = ("tsdf", "esdf", "occupancy", "freespace", "color")


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _frames(n, cs, start=0):
    return syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(24)[start:start + n], noise_sigma_rel=0.005, seed=7)


def _layer(m, name):
    return {"tsdf": m.tsdf_layer, "esdf": m.esdf_layer, "occupancy": m.occupancy_layer, "freespace": m.freespace_layer,
            "color": m.color_layer}[name]()


def _dump(m, names):
    return {n: _layer(m, n).as_dict() for n in names}


def _assert_same_layers(a, b):
    for n in a:
        assert set(a[n]) == set(b[n]), n
        for k in a[n]:
            assert a[n][k].tobytes() == b[n][k].tobytes(), (n, k)


def _mesh(m):
    return m.mesh_layer().as_dict()


def _assert_same_mesh(a, b):
    assert set(a) == set(b)
    for k in a:
        for f in ("vertices", "normals", "triangles", "colors"):
            assert np.array_equal(np.asarray(a[k][f]), np.asarray(b[k][f])), (k, f)


def _assert_file_matches_restatement(path, m, names, block_size, tmp_path):
    """Schema and rows of a saved file equal what the restatement writes for the same blocks."""
    layers = {}
    for n in names:
        d = _layer(m, n).as_dict()
        layers[n + "_layer"] = ref.layer_rows(d, next(iter(d.values())).dtype if d else np.uint8)
    expect = str(tmp_path / "expect.nvblx")
    ref.write_map(expect, layers, block_size)
    assert ref.schema(path) == ref.schema(expect)
    got, want = ref.read_map(path), ref.read_map(expect)
    assert set(got) == set(ref.LAYER_NAMES)
    for n in ref.LAYER_NAMES:
        assert got[n]["block_size"] == want[n]["block_size"] and got[n]["type"] == n
        assert np.array_equal(got[n]["xyz"], want[n]["xyz"]) and got[n]["blobs"] == want[n]["blobs"], n
    db = sqlite3.connect(path)
    assert db.execute("SELECT typeof(value_float) FROM tsdf_layer_metadata WHERE param_name='block_size'").fetchone()[0] == "real"
    db.close()


def _tsdf_map(nvb, cam, frames, layer_type=0, voxel=0.05):
    m = nvb.Mapper(voxel, projective_layer_type=layer_type)
    rgb = np.full((cam.height, cam.width, 3), 120, np.uint8)
    rgb[:, : cam.width // 2] = (200, 40, 10)
    for d, T in frames:
        m.integrate_depth(d, T, cam)
        m.integrate_color(rgb, T, cam)
        m.update_esdf()
    m.update_mesh()
    return m


@pytest.mark.parametrize("layer_type", [0, 2])
def test_round_trip_tsdf_color_esdf_mesh(gpu, tmp_path, layer_type):
    nvb = _nvb()
    cs, cam, _ = cameras(160, 120)
    m = _tsdf_map(nvb, cam, _frames(4, cs), layer_type)
    names = ["tsdf", "esdf", "color"]
    if layer_type == 2:
        m.update_freespace(1000, update_full_layer=True)
        names.append("freespace")
    p = str(tmp_path / "a.nvblx")
    assert m.save_layer_cake(p)
    _assert_file_matches_restatement(p, m, names, np.float32(m.block_size()), tmp_path)
    before = _dump(m, names)
    m.update_mesh(update_full_layer=True)
    mesh = _mesh(m)
    m2 = nvb.Mapper(0.08, projective_layer_type=layer_type)
    counts = m2.load_map(p)
    assert counts["tsdf"] == len(before["tsdf"]) and counts["esdf"] == len(before["esdf"])
    assert counts["color"] == len(before["color"]) and counts["occupancy"] == 0 and counts["feature"] == 0
    assert m2.voxel_size() == m.voxel_size() and m2.block_size() == m.block_size()
    _assert_same_layers(before, _dump(m2, names))
    _assert_same_mesh(mesh, _mesh(m2))
    # a second save of the loaded map holds the same rows
    p2 = str(tmp_path / "b.nvblx")
    m2.save_layer_cake(p2)
    a, b = ref.read_map(p), ref.read_map(p2)
    for n in ref.LAYER_NAMES:
        assert np.array_equal(a[n]["xyz"], b[n]["xyz"]) and a[n]["blobs"] == b[n]["blobs"]
    m.close(), m2.close()


def test_round_trip_occupancy(gpu, tmp_path):
    nvb = _nvb()
    cs, cam, _ = cameras(160, 120)
    m = nvb.Mapper(0.05, projective_layer_type=1)
    for d, T in _frames(4, cs):
        m.integrate_depth(d, T, cam)
        m.update_esdf()
    p = str(tmp_path / "o.nvblx")
    m.save_layer_cake(p)
    _assert_file_matches_restatement(p, m, ["occupancy", "esdf"], np.float32(m.block_size()), tmp_path)
    assert len(ref.read_map(p)["tsdf_layer"]["blobs"]) == 0
    before = _dump(m, ["occupancy", "esdf"])
    m2 = nvb.Mapper(0.1, projective_layer_type=1)
    counts = m2.load_map(p)
    assert counts["occupancy"] == len(before["occupancy"]) and counts["tsdf"] == 0
    _assert_same_layers(before, _dump(m2, ["occupancy", "esdf"]))
    m.close(), m2.close()


def test_fixture_loads_the_oracles_blocks(gpu):
    nvb = _nvb()
    m = nvb.Mapper(0.05)
    counts = m.load_map(FIXTURE)
    want = ref.read_map(FIXTURE)
    assert counts["tsdf"] == 24 and counts["esdf"] == 24
    assert m.voxel_size() == np.float32(0.1)
    for n in ("tsdf", "esdf"):
        got = _layer(m, n).as_dict()
        w = want[n + "_layer"]
        assert sorted(got) == [tuple(k) for k in w["xyz"]]
        for k, blob in zip(w["xyz"], w["blobs"]):
            assert got[tuple(k)].tobytes() == blob
    m.close()


@pytest.mark.parametrize("persistent", [3, 1])
def test_continuation_after_load_matches_the_oracle(gpu, tmp_path, persistent):
    nvb = _nvb()
    from oracle import oracle as orc
    cs, cam, ocam = cameras(320, 240)
    first, rest = _frames(4, cs), _frames(4, cs, start=4)
    m = nvb.Mapper(0.05, esdf_persistent=persistent)
    for d, T in first:
        m.integrate_depth(d, T, cam)
        m.update_esdf()
    p = str(tmp_path / "c.nvblx")
    m.save_layer_cake(p)
    m2 = nvb.Mapper(0.05, esdf_persistent=persistent)
    m2.load_map(p)
    o = orc.OracleMap(0.05)
    for k, v in m.tsdf_layer().as_dict().items():
        o.set_tsdf_block(k, v)
    for k, v in m.esdf_layer().as_dict().items():
        o.set_esdf_block(k, v)
    o.integrate_mesh(blocks=o.tsdf_block_indices())  # the load's full mesh update
    read, cands, pending = 0, 0, []
    for i, (d, T) in enumerate(rest):
        b = m2.integrate_depth(d, T, cam)
        pending.append(b)
        o.integrate_depth(d, T, ocam)
        m2.update_esdf()
        o.integrate_esdf(b if i > 0 else o.tsdf_block_indices())  # the first update after a load covers every block
        s_gpu, s_cpu = m2.esdf_integrator().last_stats(), o.esdf_stats()
        for key in ("to_clear", "clear_candidates", "cleared"):
            assert s_gpu[key] == s_cpu[key], (i, key)
        read += m2.esdf_integrator().clear_blocks_read()
        cands += s_gpu["clear_candidates"]
    assert_tsdf_equal(m2.tsdf_layer().as_dict(), o.tsdf_layer())
    assert_esdf_equal(m2.esdf_layer().as_dict(), o.esdf_layer())
    m2.update_mesh()
    o.integrate_mesh(blocks=np.unique(np.concatenate(pending), axis=0))
    g_mesh, c_mesh = _mesh(m2), o.mesh_layer()
    assert set(g_mesh) == set(c_mesh)
    for k in c_mesh:
        for f in ("vertices", "normals", "triangles"):
            assert np.array_equal(g_mesh[k][f], c_mesh[k][f]), (k, f)
    if persistent == 3 and cands > 0:
        assert read < cands, (read, cands)  # pruning is still on after the load
    m.close(), m2.close()


def _bad_file(tmp_path, name, edit):
    p = str(tmp_path / name)
    shutil.copyfile(FIXTURE, p)  # contents only: from a read-only checkout, shutil.copy would make the copy read-only too
    db = sqlite3.connect(p)
    edit(db)
    db.commit()
    db.close()
    return p


def test_failed_loads_leave_the_map_as_it_was(gpu, tmp_path):
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import _lib
    cs, cam, _ = cameras(160, 120)
    m = nvb.Mapper(0.05)
    for d, T in _frames(2, cs):
        m.integrate_depth(d, T, cam)
        m.update_esdf()
    before = _dump(m, ["tsdf", "esdf"])
    cases = [
        (str(tmp_path / "missing.nvblx"), _lib.NVB_ERR_IO),
        (_bad_file(tmp_path, "no_tsdf.nvblx", lambda db: (db.execute("DROP TABLE tsdf_layer_metadata"),
                                                           db.execute("DROP TABLE tsdf_layer_data"))), _lib.NVB_ERR_IO),
        (_bad_file(tmp_path, "blob.nvblx", lambda db: db.execute(
            "UPDATE esdf_layer_data SET data = zeroblob(100) WHERE rowid = (SELECT min(rowid) FROM esdf_layer_data)")), _lib.NVB_ERR_IO),
        (_bad_file(tmp_path, "range.nvblx", lambda db: db.execute(
            "UPDATE tsdf_layer_data SET index_x = 1048576 WHERE rowid = (SELECT min(rowid) FROM tsdf_layer_data)")),
         _lib.NVB_ERR_INDEX_RANGE),
        (_bad_file(tmp_path, "sizes.nvblx", lambda db: db.execute(
            "UPDATE esdf_layer_metadata SET value_float = 0.4 WHERE param_name = 'block_size'")), _lib.NVB_ERR_IO),
    ]
    for path, status in cases:
        with pytest.raises(_lib.NvbError) as ei:
            m.load_map(path)
        assert ei.value.code == status, (path, str(ei.value))
        _assert_same_layers(before, _dump(m, ["tsdf", "esdf"]))
        assert m.voxel_size() == np.float32(0.05)
    m.close()


def test_occupancy_table_is_skipped_by_a_tsdf_mapper(gpu, tmp_path):
    nvb = _nvb()
    cs, cam, _ = cameras(160, 120)
    mo = nvb.Mapper(0.05, projective_layer_type=1)
    for d, T in _frames(2, cs):
        mo.integrate_depth(d, T, cam)
    p = str(tmp_path / "occ.nvblx")
    mo.save_layer_cake(p)
    assert len(ref.read_map(p)["occupancy_layer"]["blobs"]) > 0
    m = nvb.Mapper(0.05)
    counts = m.load_map(p)
    assert counts["occupancy"] == 0 and counts["tsdf"] == 0
    assert m.tsdf_layer().num_blocks() == 0
    mo.close(), m.close()


def test_overwrite_keeps_only_the_second_map(gpu, tmp_path):
    """The reference's OverwriteTest (tests/test_serialization.cpp): saving over a file replaces it."""
    nvb = _nvb()
    cs, cam, _ = cameras(160, 120)
    a, b = nvb.Mapper(0.05), nvb.Mapper(0.05)
    frames = _frames(8, cs)
    a.integrate_depth(*frames[0], cam)
    b.integrate_depth(*frames[7], cam)
    p = str(tmp_path / "o.nvblx")
    a.save_layer_cake(p)
    b.save_layer_cake(p)
    got = ref.read_map(p)["tsdf_layer"]
    want = sorted(b.tsdf_layer().as_dict())
    assert [tuple(k) for k in got["xyz"]] == want
    a.close(), b.close()


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("kind", ["tsdf", "esdf", "freespace", "occupancy"])
def test_export_points_equal_the_restatement(gpu, tmp_path, kind):
    nvb = _nvb()
    from isaac_ros_nvblox_b200 import io
    cs, cam, _ = cameras(160, 120)
    layer_type = {"tsdf": 0, "esdf": 0, "freespace": 2, "occupancy": 1}[kind]
    m = nvb.Mapper(0.05, projective_layer_type=layer_type)
    for i, (d, T) in enumerate(_frames(3, cs)):
        m.integrate_depth(d, T, cam)
        m.update_esdf()
        if kind == "freespace":
            m.update_freespace(1000 * (i + 1))
    layer = _layer(m, kind)
    got = layer.export_points()
    want = ref.export_points(kind, layer.as_dict(), np.float32(m.block_size()), np.float32(m.voxel_size()))
    assert got.shape == want.shape and len(got) > 0
    assert _bits_equal(got[:, :3], want[:, :3])
    if kind == "occupancy":  # the device's expf may differ from the host's by one ulp
        gi, wi = got[:, 3].view(np.int32), want[:, 3].view(np.int32)
        assert np.max(np.abs(gi.astype(np.int64) - wi)) <= 1
    else:
        assert _bits_equal(got[:, 3], want[:, 3])
    ply = str(tmp_path / ("%s.ply" % kind))
    assert getattr(m, "save_%s_as_ply" % kind)(ply)
    props, verts, _ = io.read_ply(ply)
    assert props == ["x", "y", "z", "intensity"] and verts.shape == (len(got), 4)
    assert np.allclose(verts, got, rtol=1e-5, atol=1e-6)
    m.close()


def test_cpp_dropin_save_load_and_ply(gpu, tmp_path):
    """tests/cpp/test_map_io_dropin.cpp: nvblox_ros' save_map / load_map / save_ply handlers through include/nvblox only."""
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_map_io_dropin")
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "map io drop-in ok" in out.stdout
