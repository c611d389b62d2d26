"""Block-index lists across the C ABI: every call that takes a caller's list applies one rule set to it, and every call that
returns a list writes its count and up to `cap` indices the same way.

- A negative count is NVB_ERR_INVALID_ARGUMENT for every list-taking call.
- A list that would insert an index outside +-2^20 is NVB_ERR_INDEX_RANGE, and nothing of the map changes.
- nvb_layer_set_blocks rejects a repeated index, since each index carries its own payload.
- An output shorter than the list still reports the whole count, and holds the list's first `cap` indices.
- The Python calls that change the map return the whole list however long it is."""
import ctypes as C

import numpy as np
import pytest

from helpers import cameras, textured_image
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

INVALID_ARGUMENT = -1
LAYERS = ("TSDF", "ESDF", "FREESPACE", "COLOR", "MESH")


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _set(a):
    return set(map(tuple, np.asarray(a).reshape(-1, 3).tolist()))


def _map(freespace=False):
    """A small deterministic map: two depth frames, two colour frames, the ESDF and the mesh."""
    nvb = _nvb()
    plt = nvb.ProjectiveLayerType.kTsdfWithFreespace if freespace else nvb.ProjectiveLayerType.kTsdf
    m = nvb.Mapper(0.05, projective_layer_type=plt)
    cs, cam, _ = cameras(320, 240)
    for i, (d, T) in enumerate(syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(8)[:2])):
        m.integrate_depth(d, T, cam)
        m.integrate_color(textured_image(240, 320, seed=i), T, cam)
    m.update_esdf()
    m.update_mesh()
    return m


def _layer_stats(m, layer):
    out = (C.c_int64 * 4)()
    rc = m._L.nvb_layer_slab_stats(m._h, layer, out)
    return tuple(out) if rc == 0 else rc


def _list_calls(m, xyz, n):
    """Every call that takes a host list of n block indices, on mapper m (one with a freespace layer)."""
    from isaac_ros_nvblox_b200 import _lib
    L, h, p = m._L, m._h, _ip(xyz)
    payload = np.zeros(max(n, 1) * 8 * 8 * 8 * 8, np.uint8)
    found = np.zeros(max(n, 1), np.uint8)
    sizes = np.zeros(max(n, 1) * 3, np.int32)
    plane = (C.c_float * 4)(0.0, 0.0, 1.0, 0.0)
    caps = (C.c_int64 * 3)(0, 0, 0)
    count = C.c_int32(0)
    x = _lib.NvbDecayExclusion()
    x.excluded_blocks_xyz_host, x.num_excluded_blocks = p, n
    return {
        "esdf_integrate_blocks": lambda: L.nvb_esdf_integrate_blocks(h, p, n),
        "esdf_integrate_slice_blocks": lambda: L.nvb_esdf_integrate_slice_blocks(h, p, n),
        "esdf_integrate_slice_planar_blocks": lambda: L.nvb_esdf_integrate_slice_planar_blocks(h, plane, p, n),
        "freespace_update_blocks": lambda: L.nvb_freespace_update_blocks(h, p, n, 0, None, 0, 0, 0, None, None, 5.0, 0.2),
        "mesh_integrate_blocks": lambda: L.nvb_mesh_integrate_blocks(h, p, n, 0),
        "mesh_update_color": lambda: L.nvb_mesh_update_color(h, p, n),
        "layer_set_blocks": lambda: L.nvb_layer_set_blocks(h, _lib.NVB_LAYER_TSDF, p, n, payload.ctypes.data),
        "layer_get_blocks": lambda: L.nvb_layer_get_blocks(h, _lib.NVB_LAYER_TSDF, p, n, payload.ctypes.data,
                                                           found.ctypes.data_as(C.POINTER(C.c_uint8))),
        "mesh_block_sizes": lambda: L.nvb_mesh_block_sizes(h, p, n, _ip(sizes)),
        "mesh_get_blocks": lambda: L.nvb_mesh_get_blocks(h, p, n, None, None, None, None, caps),
        "decay_exclusion": lambda: L.nvb_mapper_decay(h, C.byref(x), None, 0, 0, 0, None, None, None, 0, None),
        "get_cleared_blocks": lambda: L.nvb_mapper_get_cleared_blocks(h, p, n, None, 0, C.byref(count)),
    }


INSERTS = ["esdf_integrate_blocks", "esdf_integrate_slice_blocks", "esdf_integrate_slice_planar_blocks",
           "freespace_update_blocks", "mesh_integrate_blocks", "mesh_update_color", "layer_set_blocks"]


def test_negative_count_is_rejected(gpu):
    m = _map(freespace=True)
    xyz = np.zeros((1, 3), np.int32)
    for name, call in _list_calls(m, xyz, -1).items():
        assert call() == INVALID_ARGUMENT, name
    m.close()


def test_index_out_of_range_changes_nothing(gpu):
    from isaac_ros_nvblox_b200 import _lib
    m = _map(freespace=True)
    xyz = np.asarray([[0, 0, 0], [1, 2, 3], [1 << 20, 0, 0], [-2, 1, 0]], np.int32)
    stats = lambda: {k: _layer_stats(m, getattr(_lib, "NVB_LAYER_" + k)) for k in LAYERS}  # noqa: E731
    before = stats()
    esdf, mesh = m.esdf_layer().as_dict(), m.mesh_layer().as_dict()
    calls = _list_calls(m, xyz, len(xyz))
    for name in INSERTS:
        assert calls[name]() == _lib.NVB_ERR_INDEX_RANGE, name
        assert stats() == before, name
    esdf_after, mesh_after = m.esdf_layer().as_dict(), m.mesh_layer().as_dict()
    assert set(esdf_after) == set(esdf) and set(mesh_after) == set(mesh)
    for k in esdf:
        assert esdf_after[k].tobytes() == esdf[k].tobytes(), k
    for k in mesh:
        for f in ("vertices", "normals", "triangles", "colors"):
            assert np.array_equal(mesh_after[k][f], mesh[k][f]), (k, f)
    m.close()


def test_set_blocks_rejects_a_repeated_index(gpu):
    from isaac_ros_nvblox_b200 import _lib
    nvb = _nvb()
    m = _map()
    layer = m.tsdf_layer()
    before = layer.slab_stats(), layer.as_dict()
    v = np.zeros((3, 8, 8, 8), nvb.mapper.TSDF_VOXEL_DTYPE)
    v["weight"] = 1.0
    with pytest.raises(_lib.NvbError) as e:
        layer.set_blocks(np.asarray([[40, 40, 40], [41, 40, 40], [40, 40, 40]], np.int32), v)
    assert e.value.code == INVALID_ARGUMENT
    after = layer.slab_stats(), layer.as_dict()
    assert after[0] == before[0] and set(after[1]) == set(before[1])
    for k in before[1]:
        assert after[1][k].tobytes() == before[1][k].tobytes(), k
    m.close()


def _short(fn, *args, n):
    """fn(*args, out, n - 1, &count) -> (count, the n - 1 indices written)."""
    out = np.full((n - 1, 3), -7, np.int32)
    count = C.c_int32(0)
    assert fn(*args, _ip(out), n - 1, C.byref(count)) == 0
    return count.value, out


def test_short_outputs_hold_the_lists_first_indices(gpu):
    from isaac_ros_nvblox_b200 import _lib
    nvb = _nvb()
    # lists read back without changing the map: the same list twice
    m = _map()
    for fn in (m._L.nvb_mapper_last_frame_blocks, m._L.nvb_mapper_last_color_blocks):
        full = nvb.mapper._block_list(fn, 1 << 20, m._h)
        assert len(full) > 1
        count, out = _short(fn, m._h, n=len(full))
        assert count == len(full) and np.array_equal(out, full[:-1])
    m.close()
    # calls that change the map: an identical mapper gives the full list
    center = np.asarray([0.3, -0.2, 1.0], np.float32)
    shapes = (nvb.mapper.NvbBoundingShape * 1)(nvb.BoundingSphere(center, 1.5)._c())
    sorted_calls = {
        "clear_outside_radius": (lambda a: a.clear_outside_radius(center, 1.5),
                                 lambda a, n: _short(a._L.nvb_mapper_clear_outside_radius, a._h,
                                                     center.ctypes.data_as(C.POINTER(C.c_float)), 1.5, n=n)),
        "clear_tsdf_inside_shapes": (lambda a: a.clear_tsdf_inside_shapes([nvb.BoundingSphere(center, 1.5)]),
                                     lambda a, n: _short(a._L.nvb_mapper_clear_tsdf_inside_shapes, a._h, shapes, 1, n=n)),
    }
    for name, (py, raw) in sorted_calls.items():
        a, b = _map(), _map()
        full = py(b)
        assert len(full) > 1, name
        count, out = raw(a, len(full))
        assert count == len(full) and np.array_equal(out, full[:-1]), name
        a.close(), b.close()
    # device-order lists (appended with atomics): the first indices are distinct members of the list
    unsorted_calls = {
        "mark_unobserved_free_inside_radius": (
            lambda a: a.mark_unobserved_tsdf_free_inside_radius(center, 2.0),
            lambda a, n: _short(a._L.nvb_mapper_mark_unobserved_free_inside_radius, a._h,
                                center.ctypes.data_as(C.POINTER(C.c_float)), 2.0, n=n)),
        "decay": (lambda a: a.decay(),
                  lambda a, n: _short(a._L.nvb_mapper_decay, a._h, C.byref(_lib.NvbDecayExclusion()), None, 0, 0, 0, None,
                                      None, n=n)),
    }
    for name, (py, raw) in unsorted_calls.items():
        a, b = _map(), _map()
        for x in (a, b):
            x.tsdf_decay_integrator().params(decay_factor=0.01, decayed_weight_threshold=1.0)
        full = py(b)
        assert len(full) > 1, name
        count, out = raw(a, len(full))
        assert count == len(full), name
        assert len(_set(out)) == len(out) and _set(out) <= _set(full), name
        a.close(), b.close()


def test_mark_unobserved_returns_every_block_of_a_large_sphere(gpu):
    """A radius of 11 m at 5 cm voxels covers far more blocks than a fixed output buffer would hold."""
    m = _nvb().Mapper(0.05)
    blocks = m.mark_unobserved_tsdf_free_inside_radius(np.asarray([0.1, 0.2, 0.3], np.float32), 11.0)
    assert len(blocks) > 65536
    assert len(_set(blocks)) == len(blocks)
    assert _set(blocks) == _set(m.tsdf_layer().get_all_block_indices())
    m.close()


def test_integrate_color_returns_every_block_of_a_wide_view(gpu):
    """A colour frame that touches more blocks than the first output buffer holds returns the whole list. The TSDF blocks
    are written directly, each with voxels in the truncation band, filling the camera's view between 2 m and 4 m."""
    nvb = _nvb()
    voxel = 0.015
    m = nvb.Mapper(voxel)
    m.color_integrator().params(max_integration_distance_m=10.0)
    bs = voxel * 8
    g = np.arange(-40, 41)
    bx, by, bz = np.meshgrid(g, g, np.arange(int(2.0 / bs), int(4.0 / bs)), indexing="ij")
    c = (np.stack([bx, by, bz], -1).reshape(-1, 3) + 0.5) * bs
    keep = (np.abs(c[:, 0]) <= 0.9 * c[:, 2]) & (np.abs(c[:, 1]) <= 0.65 * c[:, 2])
    idx = np.stack([bx, by, bz], -1).reshape(-1, 3)[keep].astype(np.int32)
    v = np.zeros((len(idx), 8, 8, 8), nvb.mapper.TSDF_VOXEL_DTYPE)
    v["weight"] = 1.0
    m.tsdf_layer().set_blocks(idx, v)
    cam = nvb.Camera(320.0, 320.0, 320.0, 240.0, 640, 480)
    blocks = m.integrate_color(textured_image(480, 640), np.eye(4, dtype=np.float32), cam)
    assert len(blocks) > 16384
    assert np.array_equal(blocks, m.last_color_blocks())
    assert _set(blocks) == _set(idx)
    m.close()
