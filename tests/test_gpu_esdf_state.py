"""Mapper.clear() empties the ESDF integrator's state for every wavefront driver: a cleared mapper computes the same ESDF
layer and statistics as a fresh one, and clear() turns the clear pass's parent-box pruning back on after a deallocating
decay switched it off."""
import numpy as np
import pytest

from helpers import ESDF_FIELDS, cameras
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

DRIVERS = [3, 1, 2, 0]  # esdf_persistent: exchange-slab, persistent, gather-replay, host loop


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _sequences():
    cs, cam, _ = cameras(320, 240)
    traj = syn.circle_trajectory(40)
    first = syn.make_sequence(syn.sphere_in_box(), cs, traj[:3])
    second = syn.make_sequence(syn.box_with_cube(), cs, traj[10:13])
    return cam, first, second


def _integrate(m, cam, frames):
    for depth, T in frames:
        m.integrate_depth(depth, T, cam)
        m.update_esdf()


def _outputs(m):
    e = m.esdf_integrator()
    return m.esdf_layer().as_dict(), e.last_stats(), e.clear_blocks_read()


def _fresh(driver, cam, frames):
    m = _nvb().Mapper(0.05, esdf_persistent=driver)
    _integrate(m, cam, frames)
    out = _outputs(m)
    m.close()
    return out


def _assert_same_esdf(got, want):
    assert set(got) == set(want)
    for k in want:
        for f in ESDF_FIELDS:
            assert np.array_equal(got[k][f], want[k][f]), (k, f)


@pytest.mark.parametrize("driver", DRIVERS)
@pytest.mark.parametrize("decay_first", [False, True])
def test_cleared_mapper_equals_fresh_mapper(gpu, driver, decay_first):
    """decay_first: a decay deallocates blocks before clear(), which switches pruning off until the layer is emptied; the
    clear pass of the next sequence then reads as few blocks as a fresh mapper's does."""
    cam, first, second = _sequences()
    m = _nvb().Mapper(0.05, esdf_persistent=driver)
    _integrate(m, cam, first)
    if decay_first:
        m.tsdf_decay_integrator().params(decay_factor=0.3)
        removed = 0
        for _ in range(12):
            removed += len(m.decay())
            if removed:
                break
        assert removed > 0
    m.clear()
    _integrate(m, cam, second)
    layer, stats, blocks_read = _outputs(m)
    m.close()
    want_layer, want_stats, want_blocks_read = _fresh(driver, cam, second)
    _assert_same_esdf(layer, want_layer)
    assert stats == want_stats
    assert blocks_read == want_blocks_read
