"""The map file fixture (tests/golden/map_small.nvblx) against the restatement of the reference's format
(tests/map_io_reference.py): schema, metadata rows, blob sizes, and a read-back of what the generator put in. No GPU."""
import os
import sqlite3
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import map_io_reference as ref  # noqa: E402

FIXTURE = os.path.join(HERE, "golden", "map_small.nvblx")


def test_fixture_schema_is_the_references():
    expected = sorted([(n + "_data", ref.data_ddl(n)) for n in ref.LAYER_NAMES] +
                      [(n + "_metadata", ref.metadata_ddl(n)) for n in ref.LAYER_NAMES])
    assert ref.schema(FIXTURE) == expected


def test_fixture_metadata_rows():
    db = sqlite3.connect(FIXTURE)
    for n in ref.LAYER_NAMES:
        rows = db.execute("SELECT param_name, value_string, value_int, value_float, typeof(value_float) FROM " + n +
                          "_metadata ORDER BY param_name").fetchall()
        assert rows == [("block_size", None, None, 0.8, "real"), ("type", n, None, None, "null")], (n, rows)
    db.close()


def test_fixture_blob_sizes_and_order():
    m = ref.read_map(FIXTURE)
    assert set(m) == set(ref.LAYER_NAMES)
    for n in ("tsdf_layer", "esdf_layer"):
        assert len(m[n]["blobs"]) == 24 and all(len(b) == ref.BLOCK_BYTES[n] for b in m[n]["blobs"])
        xyz = m[n]["xyz"]
        assert np.array_equal(xyz, xyz[np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0]))])
    for n in ("color_layer", "occupancy_layer", "freespace_layer", "feature_layer"):
        assert len(m[n]["blobs"]) == 0


def test_restatement_reads_back_what_it_wrote(tmp_path):
    rng = np.random.default_rng(3)
    xyz = np.array([[1, -2, 3], [-1048576, 0, 1048575], [0, 0, 0]], np.int32)
    blobs = [rng.integers(0, 256, 4096, dtype=np.uint8).tobytes() for _ in range(3)]
    p = str(tmp_path / "m.nvblx")
    ref.write_map(p, {"tsdf_layer": (xyz, blobs)}, np.float32(0.05) * np.float32(8))
    m = ref.read_map(p)
    order = np.lexsort((xyz[:, 2], xyz[:, 1], xyz[:, 0]))
    assert np.array_equal(m["tsdf_layer"]["xyz"], xyz[order])
    assert m["tsdf_layer"]["blobs"] == [blobs[i] for i in order]
    assert m["tsdf_layer"]["block_size"] == 0.4 and ref.to_string(np.float32(0.4)) == "0.400000"
    assert all(len(m[n]["blobs"]) == 0 and m[n]["type"] == n for n in ref.LAYER_NAMES[1:])


def test_point_rules_on_a_hand_made_block():
    """The restatement's per-layer rules and centre arithmetic on one block with known voxels."""
    dt = np.dtype([("distance", "<f4"), ("weight", "<f4")])
    b = np.zeros((8, 8, 8), dt)
    b["weight"][1, 2, 3] = 1.0
    b["distance"][1, 2, 3] = -0.25
    b["weight"][0, 0, 0] = 1e-4  # not above the minimum weight
    p = ref.export_points("tsdf", {(2, -1, 0): b}, np.float32(0.4), np.float32(0.05))
    assert p.shape == (1, 4)
    bs, vs, h = np.float32(0.4), np.float32(0.05), np.float32(0.025)
    assert np.array_equal(p[0], np.array([(bs * 2 + vs * 1) + h, (bs * -1 + vs * 2) + h, (bs * 0 + vs * 3) + h, -0.25],
                                         np.float32))
