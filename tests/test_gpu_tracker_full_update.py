"""A full-layer update while the block-update tracker still holds pending blocks, for each of its consumers (3-D ESDF, ESDF
slice, freespace, mesh). setUpdateAllBlocks drops the pending set, so the list of that update is every live block once,
and the incremental update after it covers exactly the blocks integrated since. Every layer the update writes is compared
with the oracle after each update: the oracle runs the full update over all blocks, then the incremental one over the
blocks tracked since.

The pending list before the full update is the whole map again, so pending plus live blocks is about twice the live count:
more than the live count rounded up to the 256-thread grid the allocate kernels are sized from when the host's bound of
the block count is tight, and far below the slab capacity (2^18)."""
import numpy as np
import pytest

from helpers import assert_esdf_equal, assert_tsdf_equal, cameras
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

SLICE = dict(slice_min_height_m=0.25, slice_max_height_m=1.45, slice_height_m=0.9)
FS_FIELDS = ("last_occupied_timestamp_ms", "consecutive_occupancy_duration_ms", "is_high_confidence_freespace")


def _set(a):
    return set(map(tuple, np.asarray(a).reshape(-1, 3).tolist()))


def _arr(s):
    return np.asarray(sorted(s), np.int32).reshape(-1, 3)


class Consumer:
    """One tracker consumer on a mapper and the oracle: update(full) runs it on both, check() compares what it wrote."""

    def __init__(self, kind):
        import isaac_ros_nvblox_b200 as nvb
        from oracle import oracle as orc
        self.kind = kind
        plt = nvb.ProjectiveLayerType.kTsdfWithFreespace if kind == "freespace" else nvb.ProjectiveLayerType.kTsdf
        self.m, self.o = nvb.Mapper(0.05, projective_layer_type=plt), orc.OracleMap(0.05)
        if kind == "slice2d":
            self.m.esdf_integrator().slice_params(**SLICE)
        self.fp = orc.default_freespace_params() if kind == "freespace" else None
        self.t_ms = 1000

    def update(self, todo, full):
        if self.kind == "esdf3d":
            self.m.update_esdf(update_full_layer=full)
            self.o.integrate_esdf(todo)
        elif self.kind == "slice2d":
            self.m.update_esdf_slice(update_full_layer=full)
            self.o.integrate_esdf_slice(todo, z_min_m=SLICE["slice_min_height_m"], z_max_m=SLICE["slice_max_height_m"],
                                        z_output_m=SLICE["slice_height_m"])
        elif self.kind == "freespace":
            self.t_ms += 400
            self.m.update_freespace(self.t_ms, update_full_layer=full)
            self.o.update_freespace(todo, self.t_ms, self.fp)
        else:
            self.m.update_mesh(update_full_layer=full)
            self.o.integrate_mesh(blocks=todo)

    def check(self):
        assert_tsdf_equal(self.m.tsdf_layer().as_dict(), self.o.tsdf_layer())
        if self.kind in ("esdf3d", "slice2d"):
            assert_esdf_equal(self.m.esdf_layer().as_dict(), self.o.esdf_layer())
            # a slot listed twice would be marked twice
            assert self.m.esdf_integrator().last_stats()["marked"] == self.o.esdf_stats()["marked"]
        elif self.kind == "freespace":
            g, c = self.m.freespace_layer().as_dict(), self.o.freespace_layer()
            assert set(g) == set(c), "freespace block sets differ"
            for k in c:
                for f in FS_FIELDS:
                    assert np.array_equal(g[k][f], c[k][f]), (f, k)
        else:
            g, c = self.m.mesh_layer().as_dict(), self.o.mesh_layer()
            assert set(g) == set(c), "mesh block sets differ"
            for k, cb in c.items():
                for f in ("vertices", "normals", "triangles"):
                    assert np.array_equal(g[k][f], cb[f]), (k, f)
            assert sum(len(b["triangles"]) for b in c.values()) > 0


@pytest.mark.parametrize("kind", ["esdf3d", "slice2d", "freespace", "mesh"])
def test_full_update_with_pending_blocks(gpu, kind):
    cs, cam, ocam = cameras(320, 240)
    frames = syn.make_sequence(syn.sphere_in_box(), cs, syn.circle_trajectory(40)[:5])
    p = Consumer(kind)

    def integrate(idx):
        seen = set()
        for i in idx:
            b = p.m.integrate_depth(*frames[i], cam)
            assert np.array_equal(b, p.o.integrate_depth(*frames[i], ocam))
            seen |= _set(b)
        return seen

    integrate([0, 1, 2])
    p.update(p.o.tsdf_block_indices(), full=False)  # the first update covers every block
    p.check()
    pending = integrate([0, 1, 2, 3])  # the whole map again, and a new view
    live = len(p.o.tsdf_block_indices())
    assert len(pending) == live and live + len(pending) > 256 * ((live + 255) // 256) and live > 3000
    p.update(p.o.tsdf_block_indices(), full=True)
    p.check()
    tracked = integrate([1, 2, 4])  # revisits earlier blocks
    p.update(_arr(tracked), full=False)
    p.check()
    p.m.close()
