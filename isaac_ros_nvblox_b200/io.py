"""Mesh export: MeshBlockLayer::getMesh (nvblox/include/nvblox/map/internal/cuda/impl/layer_impl.cuh:97-190) and
io::outputColorMeshLayerToPly (nvblox/src/io/mesh_io.cpp:26-56, nvblox/src/io/ply_writer.cpp:22-150). Host-side conveniences on
top of the mesh layer's read-back; nothing here is on the integration path."""
import numpy as np


def _blocks_of(mesh_layer):
    """{(x, y, z): block dict} from a mapper's mesh layer (isaac_ros_nvblox_b200.mapper._MeshLayer) or from such a dict."""
    return mesh_layer if isinstance(mesh_layer, dict) else mesh_layer.as_dict()


def get_mesh(mesh_layer):
    """MeshBlockLayer::getMesh: the blocks appended to one monolithic mesh in the layer's block order; triangle indices are
    offset by the number of vertices before their block. -> {"vertices" (v, 3) f32, "vertex_normals" (v, 3) f32,
    "vertex_appearances" (c, 4) u8 (empty if the blocks carry no colours), "triangles" (t,) i32}."""
    blocks = _blocks_of(mesh_layer)
    V, N, A, T = [], [], [], []
    next_vertex = 0
    for b in blocks.values():
        if b is None:
            continue
        nv = len(b["vertices"])
        # (layer_impl.cuh:134-139: a block has one normal / appearance per vertex, or none at all)
        assert len(b["normals"]) in (0, nv) and len(b["colors"]) in (0, nv)
        V.append(np.asarray(b["vertices"], np.float32).reshape(-1, 3))
        N.append(np.asarray(b["normals"], np.float32).reshape(-1, 3))
        A.append(np.asarray(b["colors"], np.uint8).reshape(-1, 4))
        T.append(np.asarray(b["triangles"], np.int32) + np.int32(next_vertex))
        next_vertex += nv
    cat = lambda parts, shape, dt: np.concatenate(parts) if parts else np.zeros(shape, dt)
    return {"vertices": cat(V, (0, 3), np.float32), "vertex_normals": cat(N, (0, 3), np.float32),
            "vertex_appearances": cat(A, (0, 4), np.uint8), "triangles": cat(T, (0,), np.int32)}


def _fmt(x):
    """operator<< of a float with the default precision (6 significant digits, %g)."""
    return "%g" % float(x)


def output_mesh_to_ply(mesh, filename):
    """PlyWriter::write (ply_writer.cpp:22-150): ASCII PLY, `x y z [nx ny nz] [red green blue]` per vertex and
    `3 i j k` per face under `property list uchar int vertex_indices`. Returns False (and writes nothing) without vertices,
    like the reference."""
    v, n, a, t = mesh["vertices"], mesh["vertex_normals"], mesh["vertex_appearances"], mesh["triangles"]
    if len(v) == 0:
        return False
    has_n, has_c = len(n) > 0, len(a) > 0
    if (has_n and len(n) != len(v)) or (has_c and len(a) != len(v)):
        return False
    with open(filename, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n" % len(v))
        if has_n:
            f.write("property float nx\nproperty float ny\nproperty float nz\n")
        if has_c:
            f.write("property uchar red\nproperty uchar green\nproperty uchar blue\n")
        f.write("element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(t) // 3))
        for i in range(len(v)):
            row = [_fmt(c) for c in v[i]]
            if has_n:
                row += [_fmt(c) for c in n[i]]
            if has_c:
                row += [str(int(c)) for c in a[i][:3]]
            f.write(" ".join(row) + "\n")
        for i in range(0, len(t) - len(t) % 3, 3):
            f.write("3 %d %d %d\n" % (t[i], t[i + 1], t[i + 2]))
    return True


def output_color_mesh_layer_to_ply(mesh_layer, filename):
    """io::outputColorMeshLayerToPly(layer, filename) (mesh_io.cpp:26-56); Mapper::saveColorMeshAsPly (src/mapper/mapper.cpp:694-696)."""
    return output_mesh_to_ply(get_mesh(mesh_layer), filename)


def output_points_to_ply(points, intensities, filename):
    """io::outputPointsToPly (pointcloud_io.cpp) through PlyWriter: `x y z intensity` per point under `property float
    intensity`, no faces. False (and no file) without points, like the reference."""
    p = np.asarray(points, np.float32).reshape(-1, 3)
    t = np.asarray(intensities, np.float32).reshape(-1)
    if len(p) == 0 or len(t) != len(p):
        return False
    with open(filename, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "property float intensity\nend_header\n" % len(p))
        f.write("".join("%s %s %s %s\n" % (_fmt(a), _fmt(b), _fmt(c), _fmt(i)) for (a, b, c), i in zip(p, t)))
    return True


def read_ply(filename):
    """Minimal reader of the files written above (for the tests): -> (header property names, (v, k) float array, (f, 3) int array)."""
    with open(filename) as f:
        lines = f.read().split("\n")
    assert lines[0] == "ply" and lines[1] == "format ascii 1.0"
    end = lines.index("end_header")
    nv = int([l for l in lines[:end] if l.startswith("element vertex")][0].split()[-1])
    faces = [l for l in lines[:end] if l.startswith("element face")]
    nf = int(faces[0].split()[-1]) if faces else 0
    props = [l.split()[-1] for l in lines[:end] if l.startswith("property") and "list" not in l]
    body = lines[end + 1:]
    verts = np.array([[float(x) for x in l.split()] for l in body[:nv]], np.float64).reshape(nv, len(props))
    faces = np.array([[int(x) for x in l.split()[1:]] for l in body[nv:nv + nf]], np.int64).reshape(nf, 3)
    return props, verts, faces
