"""A restatement of the reference's map file (.nvblx) and of its voxel-layer PLY rules, for the tests.

The file (nvblox/src/map_saving/serializer.cpp, sqlite_database.cpp, block_serialization_impl.h) is an SQLite database with,
per layer name L, a table L_metadata of ('type', value_string = L) and ('block_size', value_float) rows and a table L_data of
(index_x, index_y, index_z, data) rows, data being the block's voxels[8][8][8] byte for byte. The statements below are the
reference's string-built ones. Points (io/pointcloud_io.cpp:23-73, pointcloud_io_impl.h) are the kept voxels' centres
(getCenterPositionFromBlockIndexAndVoxelIndex) with an intensity per layer rule, here in canonical order: blocks in
(x, y, z) order, voxels in x, y, z order."""
import sqlite3

import numpy as np

LAYER_NAMES = ("tsdf_layer", "esdf_layer", "occupancy_layer", "freespace_layer", "color_layer", "feature_layer")
BLOCK_BYTES = {"tsdf_layer": 4096, "esdf_layer": 10240, "occupancy_layer": 2048, "freespace_layer": 12288, "color_layer": 4096}


def metadata_ddl(name):
    return ("CREATE TABLE " + name + "_metadata(param_name TEXT PRIMARY KEY UNIQUE NOT NULL,value_string TEXT,value_int INT,"
            "value_float FLOAT)")


def data_ddl(name):
    return ("CREATE TABLE " + name + "_data(index_x INT NOT NULL,index_y INT NOT NULL,index_z INT NOT NULL,data BLOB,"
            "PRIMARY KEY(index_x, index_y, index_z))")


def to_string(f):
    """std::to_string(float): "%f" of the value promoted to double."""
    return "%f" % float(np.float32(f))


def write_map(path, layers, block_size, order=LAYER_NAMES):
    """layers: {name: (xyz (n, 3) int, list of n blobs)}; every name of `order` gets its tables (empty when absent), in that
    order, each with the reference's statements: the DDL and metadata in autocommit, the rows in one transaction."""
    db = sqlite3.connect(path, isolation_level=None)
    for name in order:
        db.execute(metadata_ddl(name) + ";")
        db.execute(data_ddl(name) + ";")
        db.execute("INSERT INTO " + name + "_metadata (param_name, value_string) VALUES('type','" + name + "');")
        db.execute("INSERT INTO " + name + "_metadata (param_name, value_float) VALUES ('block_size','" + to_string(block_size) +
                   "');")
        xyz, blobs = layers.get(name, (np.zeros((0, 3), np.int32), []))
        db.execute("BEGIN TRANSACTION;")
        for (x, y, z), b in zip(np.asarray(xyz).reshape(-1, 3), blobs):
            db.execute("INSERT INTO " + name + "_data (index_x, index_y, index_z, data) VALUES (%d,%d,%d,?)" % (x, y, z),
                       (bytes(b),))
        db.execute("END TRANSACTION;")
    db.close()


def read_map(path):
    """{name: {"block_size": float, "type": str, "xyz": (n, 3) int32 sorted, "blobs": [bytes]}} of every layer in the file."""
    db = sqlite3.connect(path)
    names = [r[0][:-len("_metadata")] for r in
             db.execute("SELECT name FROM sqlite_master WHERE type='table' AND name LIKE '%_metadata'")]
    out = {}
    for name in names:
        meta = dict((r[0], r[1] if r[1] is not None else r[2]) for r in
                    db.execute("SELECT param_name, value_string, value_float FROM " + name + "_metadata"))
        rows = db.execute("SELECT index_x, index_y, index_z, data FROM " + name + "_data ORDER BY index_x, index_y, index_z").fetchall()
        out[name] = {"block_size": meta.get("block_size"), "type": meta.get("type"),
                     "xyz": np.array([r[:3] for r in rows], np.int32).reshape(-1, 3), "blobs": [bytes(r[3]) for r in rows]}
    db.close()
    return out


def schema(path):
    """[(name, sql)] of the file's tables, by name."""
    db = sqlite3.connect(path)
    s = sorted(db.execute("SELECT name, sql FROM sqlite_master WHERE type='table'").fetchall())
    db.close()
    return s


def layer_rows(layer_dict, dtype):
    """{(x, y, z): (8, 8, 8) voxels} -> (sorted xyz, blobs)."""
    keys = sorted(layer_dict)
    return (np.array(keys, np.int32).reshape(-1, 3),
            [np.ascontiguousarray(layer_dict[k], dtype=dtype).tobytes() for k in keys])


def export_points(kind, layer_dict, block_size, voxel_size):
    """(n, 4) float32 {x, y, z, intensity}: io::outputVoxelLayerToPly's points of a {(x, y, z): voxels} layer, kind in
    "tsdf", "occupancy", "freespace", "esdf"."""
    f32 = np.float32
    bs = f32(block_size)
    vs, half = bs * f32(1.0 / 8), bs * f32(0.5 / 8)
    v = np.arange(512)
    vi = np.stack([v >> 6, (v >> 3) & 7, v & 7], 1).astype(f32)
    out = []
    for k in sorted(layer_dict):
        blk = layer_dict[k].reshape(512)
        if kind == "tsdf":
            keep, inten = blk["weight"] > f32(1e-4), blk["distance"]
        elif kind == "occupancy":
            lo = blk["log_odds"].astype(f32)
            p = (np.exp(lo) / (f32(1.0) + np.exp(lo))).astype(f32)
            keep, inten = p > f32(0.5), p
        elif kind == "freespace":
            keep, inten = np.ones(512, bool), (blk["is_high_confidence_freespace"] != 0).astype(f32)
        else:
            d = f32(voxel_size) * np.sqrt(blk["squared_distance_vox"].astype(f32))
            inten = np.where(blk["is_inside"] != 0, -d, d).astype(f32)
            keep = blk["observed"] != 0
        b = np.array(k, f32)
        c = (bs * b[None, :] + vs * vi) + half
        out.append(np.concatenate([c, inten[:, None].astype(f32)], 1)[keep])
    return np.concatenate(out).astype(f32) if out else np.zeros((0, 4), f32)
