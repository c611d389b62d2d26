"""Point queries on the GPU against their float32 restatement (tests/query_reference.py): voxel lookups, trilinear
interpolation and nvblox_torch's ESDF / TSDF / occupancy queries over one or several mappers.

Voxel lookups, success flags and the ESDF / TSDF / occupancy query outputs are compared bit for bit: the kernels and the
restatement do the same float32 operations in the same order (the library is built with -fmad=false, so nothing is
contracted into an FMA). Interpolated values are compared within 1e-6 * max(1, |v|): the occupancy member goes through
expf, which is not correctly rounded on the GPU, and numpy's float32 exp is not the same function either.
"""
import numpy as np
import pytest

import query_reference as qr
from isaac_ros_nvblox_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

F = np.float32


def _nvb():
    import isaac_ros_nvblox_b200 as nvb
    return nvb


def _q():
    from isaac_ros_nvblox_b200 import query
    return query


@pytest.fixture(scope="module")
def c2(gpu):
    """bench.py's map: 80 frames of the sphere-in-box circle, 640x480, 5 cm voxels, TSDF + ESDF."""
    import bench
    nvb = _nvb()
    cam_s, frames = bench.make_frames(80, 0, 1)
    cam = nvb.Camera(cam_s.fu, cam_s.fv, cam_s.cu, cam_s.cv, cam_s.width, cam_s.height)
    m = nvb.Mapper(0.05)
    for d, T in frames:
        m.integrate_depth(d, T, cam, return_blocks=False)
        m.update_esdf()
    yield dict(m=m, tsdf=m.tsdf_layer().as_dict(), esdf=m.esdf_layer().as_dict(), frames=frames, cam=cam)
    m.close()


def _aabb(layer, voxel):
    idx = np.array(list(layer.keys()))
    bs = 8 * voxel
    return idx.min(0) * bs, (idx.max(0) + 1) * bs


def _points(layer, voxel, n, seed=0):
    """Random points in the map's AABB, plus points exactly on voxel and block faces, negative coordinates, and the rejects."""
    rng = np.random.default_rng(seed)
    lo, hi = _aabb(layer, voxel)
    p = rng.uniform(lo - 0.3, hi + 0.3, (n, 3)).astype(F)
    faces = (np.round(p[: n // 8] / F(voxel)) * F(voxel)).astype(F)        # voxel faces (and block faces among them)
    bfaces = (np.round(p[: n // 16] / F(8 * voxel)) * F(8 * voxel)).astype(F)
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [3e38, 0, 0], [-3e38, 1, 1],
                    [8 * voxel * (1 << 20) + 1.0, 0, 0], [-8 * voxel * (1 << 20) - 1.0, 0, 0], [-1e-7, -1e-7, -1e-7]], F)
    return np.concatenate([p, faces, bfaces, -np.abs(p[:16]), bad]).astype(F)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_get_voxels_bit_identical(c2):
    m = c2["m"]
    nvb = _nvb()
    pts = _points(c2["tsdf"], 0.05, 4000)
    for layer, d, dt in ((m.tsdf_layer(), c2["tsdf"], nvb.mapper.TSDF_VOXEL_DTYPE),
                         (m.esdf_layer(), c2["esdf"], nvb.mapper.ESDF_VOXEL_DTYPE)):
        got, ok = layer.get_voxels(pts)
        exp, eok = qr.query_voxels(d, pts, 0.05, dt)
        assert np.array_equal(ok, eok)
        assert got.tobytes() == exp.tobytes()
        assert 0 < ok.sum() < len(pts) and not ok[-8:-1].any()
        # device path: same bytes
        gd, okd = layer.get_voxels(_cuda(pts))
        assert np.array_equal(okd.cpu().numpy(), eok)
        assert gd.cpu().numpy().tobytes() == exp.tobytes()


def _close(a, b):
    return np.all(np.abs(a - b) <= 1e-6 * np.maximum(1.0, np.abs(b)))


@pytest.mark.parametrize("kind", ["tsdf", "esdf"])
def test_interpolate_matches_restatement(c2, kind):
    m = c2["m"]
    layer = m.tsdf_layer() if kind == "tsdf" else m.esdf_layer()
    pts = _points(c2[kind], 0.05, 3000, seed=1)
    got, ok = layer.interpolate(pts)
    exp = [qr.interpolate(c2[kind], p, 0.05, kind) for p in pts]
    eok = np.array([e[0] for e in exp])
    ev = np.array([e[1] for e in exp], F)
    assert np.array_equal(ok, eok) and ok.sum() > 100
    assert _close(got[ok], ev[ok]) and np.all(got[~ok] == 0)
    gd, okd = layer.interpolate(_cuda(pts))
    assert np.array_equal(okd.cpu().numpy(), ok) and np.array_equal(gd.cpu().numpy(), got)


def _hand_layer(nvb, voxel, keys, occupancy=False, seed=0):
    """A mapper with hand-set blocks: TSDF distance = x + 2y + 3z (linear), weight 1; or occupancy log-odds."""
    rng = np.random.default_rng(seed)
    m = nvb.Mapper(voxel, projective_layer_type=nvb.ProjectiveLayerType.kOccupancy if occupancy else nvb.ProjectiveLayerType.kTsdf)
    keys = np.array(keys, np.int32)
    vc = np.indices((8, 8, 8)).transpose(1, 2, 3, 0).astype(F)
    if occupancy:
        v = np.zeros((len(keys), 8, 8, 8), nvb.mapper.OCCUPANCY_VOXEL_DTYPE)
        v["log_odds"] = rng.uniform(-5, 5, v.shape).astype(F)
        m.occupancy_layer().set_blocks(keys, v)
        return m, m.occupancy_layer()
    v = np.zeros((len(keys), 8, 8, 8), nvb.mapper.TSDF_VOXEL_DTYPE)
    for i, k in enumerate(keys):
        c = (k.astype(F) * 8 + vc + F(0.5)) * F(voxel)
        v[i]["distance"] = c[..., 0] + 2 * c[..., 1] + 3 * c[..., 2]
        v[i]["weight"] = 1.0
    m.tsdf_layer().set_blocks(keys, v)
    return m, m.tsdf_layer()


def test_interpolation_across_eight_blocks_and_missing_neighbour(gpu):
    """The low corner on a block's last voxel on every axis: the 8 neighbours lie in 8 blocks; a linear field is reproduced;
    removing one of the blocks makes exactly the points that need it fail. Far from the origin and at negative indices."""
    nvb = _nvb()
    for origin in ((0, 0, 0), (-3, -5, -2), (1200, -900, 40)):
        o = np.array(origin)
        keys = [tuple(o + np.array([i >> 2, (i >> 1) & 1, i & 1])) for i in range(8)]
        m, layer = _hand_layer(nvb, 0.05, keys)
        corner = (o + 1).astype(F) * F(0.4)  # the shared corner of the 8 blocks
        rng = np.random.default_rng(2)
        pts = (corner + rng.uniform(-0.025, 0.025, (500, 3))).astype(F)
        got, ok = layer.interpolate(pts)
        d = layer.as_dict()
        exp = [qr.interpolate(d, p, 0.05, "tsdf") for p in pts]
        assert np.array_equal(ok, [e[0] for e in exp]) and ok.all()
        assert _close(got, np.array([e[1] for e in exp], F))
        lin = pts[:, 0] + 2 * pts[:, 1] + 3 * pts[:, 2]
        assert np.all(np.abs(got - lin) < 1e-3 * np.maximum(1.0, np.abs(lin)))
        m.close()
        m, layer = _hand_layer(nvb, 0.05, keys[:7])  # block (1, 1, 1) missing: needed only by points near the corner
        pts = (corner + rng.uniform(-0.2, 0.025, (500, 3))).astype(F)
        got, ok = layer.interpolate(pts)
        exp = np.array([qr.interpolate(layer.as_dict(), p, 0.05, "tsdf")[0] for p in pts])
        assert np.array_equal(ok, exp) and not ok.all() and ok.any()
        assert np.all(got[~ok] == 0)
        m.close()


def test_occupancy_interpolate_and_query(gpu):
    nvb, q = _nvb(), _q()
    keys = [(x, y, z) for x in range(-2, 2) for y in range(-1, 2) for z in range(0, 2)]
    m, layer = _hand_layer(nvb, 0.1, keys, occupancy=True)
    d = layer.as_dict()
    pts = _points(d, 0.1, 3000, seed=3)
    got, ok = layer.interpolate(pts)
    exp = [qr.interpolate(d, p, 0.1, "occupancy") for p in pts]
    assert np.array_equal(ok, [e[0] for e in exp]) and ok.sum() > 100
    assert _close(got[ok], np.array([e[1] for e in exp], F)[ok])
    out = q.query_layer(m, q.QueryType.OCCUPANCY, _cuda(pts)).cpu().numpy()
    assert out.tobytes() == qr.query_occupancy([(d, 0.1)], pts).tobytes()
    m.close()


def _esdf_expected(layers, spheres, grad):
    out = np.full((len(spheres), 4 if grad else 1), qr.MAX_DISTANCE, F)
    return qr.query_esdf(layers, spheres, grad, out)


@pytest.mark.parametrize("grad", [False, True])
def test_esdf_query_single_mapper(c2, grad):
    q = _q()
    pts = _points(c2["esdf"], 0.05, 4000, seed=4)
    r = np.random.default_rng(5).uniform(0, 0.3, (len(pts), 1)).astype(F)
    spheres = np.concatenate([pts, r], 1)
    got = q.query_layer(c2["m"], q.QueryType.ESDF_GRAD if grad else q.QueryType.ESDF, _cuda(spheres)).cpu().numpy()
    exp = _esdf_expected([(c2["esdf"], 0.05)], spheres, grad)
    assert got.tobytes() == exp.tobytes()


def test_tsdf_query_single_mapper(c2):
    q = _q()
    pts = _points(c2["tsdf"], 0.05, 4000, seed=6)
    got = q.query_layer(c2["m"], q.QueryType.TSDF, _cuda(pts)).cpu().numpy()
    exp = qr.query_tsdf([(c2["tsdf"], 0.05)], pts, np.zeros((len(pts), 2), F))
    assert got.tobytes() == exp.tobytes()


@pytest.fixture(scope="module")
def three(gpu):
    """Three mappers with different voxel sizes over parts of the sphere-in-box scene."""
    nvb = _nvb()
    scam = syn.PinholeCamera(150.0, 150.0, 80.0, 60.0, 160, 120)
    cam = nvb.Camera(scam.fu, scam.fv, scam.cu, scam.cv, scam.width, scam.height)
    frames = syn.make_sequence(syn.sphere_in_box(), scam, syn.circle_trajectory(12))
    ms = []
    for voxel, part in ((0.05, frames[0:5]), (0.08, frames[4:9]), (0.13, frames[8:12])):
        m = nvb.Mapper(voxel)
        for d, T in part:
            m.integrate_depth(d, T, cam, return_blocks=False)
            m.update_esdf()
        ms.append(m)
    layers = [(m.esdf_layer().as_dict(), m.voxel_size()) for m in ms]
    tsdfs = [(m.tsdf_layer().as_dict(), m.voxel_size()) for m in ms]
    yield dict(ms=ms, esdf=layers, tsdf=tsdfs)
    for m in ms:
        m.close()


@pytest.mark.parametrize("k", [2, 3])
def test_multi_mapper_queries(three, k):
    q = _q()
    ms, esdf, tsdf = three["ms"][:k], three["esdf"][:k], three["tsdf"][:k]
    pts = _points(esdf[0][0], 0.05, 3000, seed=7)
    spheres = np.concatenate([pts, np.random.default_rng(8).uniform(0, 0.2, (len(pts), 1)).astype(F)], 1)
    for grad in (False, True):
        got = q.query_layer(ms, q.QueryType.ESDF_GRAD if grad else q.QueryType.ESDF, _cuda(spheres)).cpu().numpy()
        assert got.tobytes() == _esdf_expected(esdf, spheres, grad).tobytes()
    got = q.query_layer(ms, q.QueryType.TSDF, _cuda(pts)).cpu().numpy()
    assert got.tobytes() == qr.query_tsdf(tsdf, pts, np.zeros((len(pts), 2), F)).tobytes()
    # an (n, 3) ESDF query is a zero radius
    got3 = q.query_layer(ms, q.QueryType.ESDF, _cuda(pts)).cpu().numpy()
    z = np.concatenate([pts, np.zeros((len(pts), 1), F)], 1)
    assert got3.tobytes() == _esdf_expected(esdf, z, False).tobytes()


def test_query_right_after_async_update_equals_synchronous(c2, gpu):
    """Device frames through integrate_depth_device + update_esdf(sync=False) while a torch stream is current, then queries
    on that stream, with no host synchronisation in between: the same as after the synchronous calls."""
    import torch
    nvb, q = _nvb(), _q()
    frames, cam = c2["frames"][:20], c2["cam"]
    pts = _cuda(_points(c2["esdf"], 0.05, 20000, seed=9))
    spheres = torch.cat([pts, torch.zeros((pts.shape[0], 1), device=pts.device)], 1)
    a, b = nvb.Mapper(0.05), nvb.Mapper(0.05)
    for d, T in frames:
        b.integrate_depth(d, T, cam, return_blocks=False)
        b.update_esdf()
    ref = q.query_layer(b, q.QueryType.ESDF_GRAD, spheres).cpu()
    ref_t = q.query_layer(b, q.QueryType.TSDF, pts).cpu()
    depth = torch.from_numpy(np.stack([d for d, _ in frames])).cuda()
    rows, cols = depth.shape[1:]
    torch.cuda.synchronize()  # the frames are resident before the sequence starts
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i, (_, T) in enumerate(frames):
            a.integrate_depth_device(depth[i].data_ptr(), rows, cols, T, cam)
            a.update_esdf(sync=False)
        out = q.query_layer(a, q.QueryType.ESDF_GRAD, spheres)
        out_t = q.query_layer(a, q.QueryType.TSDF, pts)
        vox, ok = a.esdf_layer().get_voxels(pts)
    s.synchronize()
    assert torch.equal(out.cpu(), ref) and torch.equal(out_t.cpu(), ref_t)
    rv, rok = b.esdf_layer().get_voxels(pts)
    assert torch.equal(ok.cpu(), rok.cpu()) and torch.equal(vox.cpu(), rv.cpu())
    a.close(), b.close()


def test_query_after_clear_outside_radius(c2, gpu):
    """regression_test_query_after_clear.cu: blocks removed by clearOutsideRadius are misses afterwards."""
    nvb, q = _nvb(), _q()
    m = nvb.Mapper(0.05)
    for d, T in c2["frames"][:10]:
        m.integrate_depth(d, T, c2["cam"], return_blocks=False)
        m.update_esdf()
    pts = _points(m.esdf_layer().as_dict(), 0.05, 4000, seed=10)
    before = q.query_layer(m, q.QueryType.ESDF, _cuda(pts)).cpu().numpy()
    m.clear_outside_radius(np.array([0.0, 0.0, 2.0], F), 2.5)
    d = m.esdf_layer().as_dict()
    after = q.query_layer(m, q.QueryType.ESDF, _cuda(pts)).cpu().numpy()
    assert after.tobytes() == _esdf_expected([(d, 0.05)], np.concatenate([pts, np.zeros((len(pts), 1), F)], 1), False).tobytes()
    assert (after == qr.MAX_DISTANCE).sum() > (before == qr.MAX_DISTANCE).sum()
    m.close()


def test_empty_and_bad_inputs(c2):
    import torch
    q = _q()
    m = c2["m"]
    e = torch.zeros((0, 3), device="cuda")
    assert q.query_layer(m, q.QueryType.ESDF, e).shape == (0, 1)
    assert q.query_layer(m, q.QueryType.TSDF, e).shape == (0, 2)
    v, ok = m.tsdf_layer().get_voxels(np.zeros((0, 3), F))
    assert len(v) == 0 and len(ok) == 0
    with pytest.raises(ValueError):
        q.query_layer(m, q.QueryType.ESDF, torch.zeros((4, 4)))                     # CPU tensor
    with pytest.raises(ValueError):
        q.query_layer(m, q.QueryType.TSDF, torch.zeros((4, 4), device="cuda"))     # wrong shape
    with pytest.raises(ValueError):
        q.query_layer(m, q.QueryType.ESDF, torch.zeros((4, 4), device="cuda", dtype=torch.float64))
    with pytest.raises(ValueError):
        q.query_layer(m, q.QueryType.ESDF, torch.zeros((4, 4), device="cuda"), output=torch.zeros((3, 1), device="cuda"))
    from isaac_ros_nvblox_b200 import _lib
    with pytest.raises(_lib.NvbError):
        _nvb().mapper._Layer(m, _lib.NVB_LAYER_MESH, np.dtype("u1")).get_voxels(np.zeros((2, 3), F))
    with pytest.raises(_lib.NvbError):
        _nvb().mapper._Layer(m, 77, np.dtype("u1")).interpolate(np.zeros((2, 3), F))


def test_large_query_sampled(c2):
    """N = 2^24 spheres in one launch, checked against the restatement on a sample."""
    import torch
    q = _q()
    n = 1 << 24
    lo, hi = _aabb(c2["esdf"], 0.05)
    g = torch.Generator(device="cuda").manual_seed(11)
    pts = torch.rand((n, 3), device="cuda", generator=g) * torch.tensor(hi - lo + 0.4, dtype=torch.float32, device="cuda") \
        + torch.tensor(lo - 0.2, dtype=torch.float32, device="cuda")
    spheres = torch.cat([pts, torch.full((n, 1), 0.1, device="cuda")], 1)
    out = q.query_layer(c2["m"], q.QueryType.ESDF_GRAD, spheres)
    idx = np.random.default_rng(12).choice(n, 3000, replace=False)
    idx = np.concatenate([idx, [0, n - 1]])
    s = spheres[torch.from_numpy(idx).cuda()].cpu().numpy()
    assert out[torch.from_numpy(idx).cuda()].cpu().numpy().tobytes() == _esdf_expected([(c2["esdf"], 0.05)], s, True).tobytes()


def test_differentiable_esdf_backward(c2):
    import torch
    q = _q()
    pts = _points(c2["esdf"], 0.05, 2000, seed=13)[:-8]
    for cols in (3, 4):
        x = _cuda(np.concatenate([pts, np.full((len(pts), 1), 0.05, F)], 1)[:, :cols]).requires_grad_(True)
        d = q.query_differentiable_layer(c2["m"], q.QueryType.ESDF, x)
        w = torch.linspace(-1, 1, d.shape[0], device="cuda")
        (d * w).sum().backward()
        xyzd = q.query_layer(c2["m"], q.QueryType.ESDF_GRAD, x.detach()).cpu().numpy()
        assert np.array_equal(d.detach().cpu().numpy(), xyzd[:, 3])
        expect = xyzd.copy()
        expect[:, 3] = -1.0
        expect = (w.cpu().numpy()[:, None] * expect)[:, :cols]
        assert np.array_equal(x.grad.cpu().numpy(), expect.astype(F))


def test_query_dropin_program(gpu, tmp_path):
    """tests/cpp/test_query_dropin.cpp: getVoxels and interpolateOnCPU through the C++ mirror."""
    import subprocess
    from test_cabi_symbols import _compile_cpp_dropin
    exe = _compile_cpp_dropin(tmp_path, "test_query_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "query drop-in ok" in out.stdout
