"""Float64 geometry checks of the projective paths that do not go through the oracle. Each takes {block index: voxels}
layers (or lists), so that tests/test_oracle_camera_ground_truth.py runs it on the oracle and tests/test_gpu_camera_pose.py
on the mapper."""
import numpy as np

import camera_pose_cases as cpc


def _voxels(layer, keep):
    """-> (voxel centres (n, 3) float64, global voxel indices (n, 3), records (n,)) of the voxels where keep(block) holds."""
    P, K, R = [], [], []
    for k, b in layer.items():
        v = np.argwhere(keep(b))
        if len(v) == 0:
            continue
        g = np.asarray(k, np.int64) * 8 + v
        K.append(g)
        P.append((g.astype(np.float64) + 0.5) * cpc.VOXEL)
        R.append(b[v[:, 0], v[:, 1], v[:, 2]])
    if not P:
        return np.zeros((0, 3)), np.zeros((0, 3), np.int64), None
    return np.concatenate(P), np.concatenate(K), np.concatenate(R)


def _gt_plane_tsdf(P, T_L_C):
    """Camera-z depth difference between the float64 hit of the ray from the camera centre through each voxel centre on the
    plane z = PLANE_Z and the voxel centre (positive in front of the surface)."""
    T = np.asarray(T_L_C, np.float64)
    t = T[:3, 3]
    s = (cpc.PLANE_Z - t[2]) / (P[:, 2] - t[2])
    hit = t + (P - t) * s[:, None]
    return ((hit - P) @ T[:3, :3])[:, 2]


def plane_tsdf_errors(layer_1, layer_2, setup, truncation_m=4 * cpc.VOXEL):
    """TsdfErrorTest.SymmetricViewOnPlane (nvblox/tests/test_tsdf_error.cpp:117-208): over the voxels observed (weight >
    1e-4) and inside the truncation band (distance < truncation) in both layers, the error gt - distance of layer 1, and
    both layers' mean distances. -> dict(n, errors (n,) float64, mean_1, mean_2)."""
    def keep(b):
        return (b["weight"] > 1e-4) & (b["distance"] < np.float32(truncation_m))

    P1, K1, V1 = _voxels(layer_1, keep)
    P2, K2, V2 = _voxels(layer_2, keep)
    k1 = {tuple(k): i for i, k in enumerate(K1.tolist())}
    both = [(k1[tuple(k)], j) for j, k in enumerate(K2.tolist()) if tuple(k) in k1]
    i1 = np.array([a for a, _ in both], np.int64)
    i2 = np.array([b for _, b in both], np.int64)
    d1 = V1["distance"][i1].astype(np.float64)
    d2 = V2["distance"][i2].astype(np.float64)
    err = _gt_plane_tsdf(P1[i1], setup[0][1]) - d1
    if len(i1) == 0:
        return dict(n=0, errors=err, mean_1=np.nan, mean_2=np.nan)
    return dict(n=len(i1), errors=err, mean_1=float(d1.mean()), mean_2=float(d2.mean()))


def back_projected_blocks(depth, c, T_L_C, max_dist=7.0, face_margin=1e-4):
    """Blocks that contain the float64 back-projection of each valid pixel (depth > 0, ray length below max_dist), skipping
    points within face_margin of a block face. -> (n, 3) int64 unique."""
    _, v = cpc.pixel_rays(c)
    T = np.asarray(T_L_C, np.float64)
    d = np.asarray(depth, np.float64)
    ok = d > 0
    p_C = v[ok] * d[ok][:, None]
    ok_len = np.linalg.norm(p_C, axis=-1) < max_dist
    p_L = p_C[ok_len] @ T[:3, :3].T + T[:3, 3]
    q = p_L / cpc.BLOCK
    b = np.floor(q)
    frac = (q - b) * cpc.BLOCK
    away = np.all((frac > face_margin) & (frac < cpc.BLOCK - face_margin), axis=-1)
    return np.unique(b[away].astype(np.int64), axis=0)


def missing_blocks(block_list, depth, c, T_L_C, max_dist=7.0):
    """Blocks holding a back-projected surface point that the frame's block list lacks. -> (missing (m, 3), checked n)."""
    want = back_projected_blocks(depth, c, T_L_C, max_dist)
    have = set(map(tuple, np.asarray(block_list, np.int64).reshape(-1, 3).tolist()))
    miss = np.array([k for k in want.tolist() if tuple(k) not in have], np.int64).reshape(-1, 3)
    return miss, len(want)


def stripe_colour_mismatches(color_layer, scene, views, window=2):
    """Coloured voxels (weight > 0) within one voxel of the surface and more than two voxels from a stripe edge whose colour
    is not their stripe's. views: [(intrinsics, T_L_C, stripe image)] of the colour frames. A voxel is left out if, in a
    frame whose image it projects into (float64 projection), the pixel's ray hits the scene more than two voxels from the
    voxel centre (another surface covers it there, within the occlusion test's truncation band) or the image is not one
    colour within `window` pixels (the bilinear lookup blends across an occlusion edge). -> (mismatching, checked)."""
    P, _, V = _voxels(color_layer, lambda b: b["weight"] > 0)
    if V is None:
        return 0, 0
    x = P[:, 0] / cpc.STRIPE_PERIOD
    edge = np.abs(x - np.round(x)) * cpc.STRIPE_PERIOD
    sel = (np.abs(scene.distance(P)) <= cpc.VOXEL) & (edge > 2 * cpc.VOXEL)
    for c, T_L_C, img in views:
        T = np.asarray(T_L_C, np.float64)
        hits = cpc.world_hits(scene, c, T)
        p_C = (P - T[:3, 3]) @ T[:3, :3]
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = reproject(p_C, c)
        inside = (p_C[:, 2] > 0) & (u >= 0) & (v >= 0) & (u < c["width"]) & (v < c["height"])
        for i in np.flatnonzero(sel & inside):
            iu, iv = int(u[i]), int(v[i])
            h = hits[iv, iu]
            w = img[max(iv - window, 0):iv + window + 1, max(iu - window, 0):iu + window + 1].reshape(-1, 3)
            if not (np.linalg.norm(h - P[i]) <= 2 * cpc.VOXEL and np.all(w == w[0])):
                sel[i] = False
    want = np.asarray(cpc.STRIPE_COLORS, np.uint8)[cpc.stripe_index(P[sel, 0])]
    bad = np.any(V["color"][sel] != want, axis=-1)
    return int(bad.sum()), int(sel.sum())


def reproject(points_C, c):
    """float64 pixel coordinates (u, v) of camera-frame points."""
    p = np.asarray(points_C, np.float64)
    return p[:, 0] / p[:, 2] * c["fu"] + c["cu"], p[:, 1] / p[:, 2] * c["fv"] + c["cv"]


# Dynamics: a wall 4 m in front of an identity-pose camera, later a box at 2 m covering a pixel rectangle
DYN_CAM = cpc.intrinsics(320, 240, 150.0, 168.0, 160 + 0.12 * 320, 120 - 0.12 * 240)
DYN_BOXES = [(70, 50), (90, 130), (120, 190)]  # (first row, first column) of a 50 x 70 pixel box
DYN_BOX_SIZE = (50, 70)
DYN_BOX_DEPTH = 2.0


def dynamics_wall():
    cs = cpc.cameras(DYN_CAM)[0]
    import isaac_ros_nvblox_b200.synthetic as syn
    return syn.render_depth(syn.plane_scene(4.0), cs, np.eye(4), max_dist=8.0)


def dynamics_box_frame(wall, k):
    d = wall.copy()
    r0, c0 = DYN_BOXES[k]
    d[r0:r0 + DYN_BOX_SIZE[0], c0:c0 + DYN_BOX_SIZE[1]] = DYN_BOX_DEPTH
    return d


def dynamics_points_outside_box(points, k, tol=1e-3):
    """Detected points (camera frame = world frame here) re-projected with the float64 (fu, fv, cu, cv) that fall outside
    box k's pixel rectangle. -> count."""
    r0, c0 = DYN_BOXES[k]
    u, v = reproject(points, DYN_CAM)
    inside = (u >= c0 - tol) & (u <= c0 + DYN_BOX_SIZE[1] + tol) & (v >= r0 - tol) & (v <= r0 + DYN_BOX_SIZE[0] + tol)
    return int((~inside).sum())
