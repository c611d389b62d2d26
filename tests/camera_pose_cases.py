"""General cameras and poses for the projective paths, shared by the non-GPU checks (test_camera_pose_guard.py,
test_oracle_camera_ground_truth.py) and the GPU parity tests (test_gpu_camera_pose.py).

Every camera here has fu != fv and a principal point away from the image centre; the poses pitch, roll, look straight
down or up, sit on a block corner or kilometres from the origin. Rotations are built in float64 and stored as float32,
like poses that arrive over TF. Camera axes: x right, y down, z forward (optical axis).

A case is a dict: name, scene ("sphere_in_box" / "box_with_cube"), cam (intrinsics dict), pose (float32 4x4 T_L_C),
claims (what its name states: pitch_deg, roll_deg, axis, block_corner, far), min_blocks (the oracle integrates more TSDF
blocks than this from the case's first frame).
"""
import math

import numpy as np

from isaac_ros_nvblox_b200 import synthetic as syn

VOXEL = 0.05
BLOCK = float(np.float32(8) * np.float32(VOXEL))
FAR_OFFSET = (12345.6, -23456.7, 345.6)  # scale_edge_cases.FAR_OFFSETS[0]


# ---------------------------------------------------------------------------------------------------------------------
# Intrinsics
# ---------------------------------------------------------------------------------------------------------------------
def intrinsics(width, height, fu, fv, cu, cv, radial=None, tangential=None):
    return dict(width=int(width), height=int(height), fu=float(fu), fv=float(fv), cu=float(cu), cv=float(cv), radial=radial,
                tangential=tangential)


CAMS = {
    # fu / fv = 0.9, principal point 12 % right of and 13 % above the centre
    "aniso_0.9": intrinsics(320, 240, 140.0, 140.0 / 0.9, 160 + 0.12 * 320, 120 - 0.13 * 240),
    # fu / fv = 1.1, principal point 14 % left of and 11 % below the centre
    "aniso_1.1": intrinsics(320, 240, 165.0, 150.0, 160 - 0.14 * 320, 120 + 0.11 * 240),
    # half-integer principal point: pixel column 140 and row 130 have an exactly zero ray component; odd size
    "half_integer_317x239": intrinsics(317, 239, 160.0, 145.0, 140.5, 130.5),
    "odd_641x481": intrinsics(641, 481, 300.0, 330.0, 641 / 2.0 + 0.1 * 641, 481 / 2.0 - 0.12 * 481),
    # radial / tangential distortion with fu != fv
    "distorted": intrinsics(320, 240, 150.0, 165.0, 160 + 0.11 * 320, 120 + 0.12 * 240, radial=(0.05, -0.02, 0.003, 0.0, 0.0, 0.0),
                            tangential=(0.001, -0.0005)),
}


def cameras(c):
    """(synthetic, product, oracle) cameras of an intrinsics dict."""
    import isaac_ros_nvblox_b200 as nvb
    from oracle import oracle as orc
    cs = syn.PinholeCamera(c["fu"], c["fv"], c["cu"], c["cv"], c["width"], c["height"])
    ocam = orc.Camera(c["fu"], c["fv"], c["cu"], c["cv"], c["width"], c["height"])
    if c.get("radial") is not None or c.get("tangential") is not None:
        ocam = ocam.with_distortion(k=c.get("radial") or (0,) * 6, p=c.get("tangential") or (0, 0))
    return cs, nvb.Camera(c["fu"], c["fv"], c["cu"], c["cv"], c["width"], c["height"], c.get("radial"), c.get("tangential")), ocam


def swapped(c, what):
    """The intrinsics with fu / fv ("f") or cu / cv ("c") exchanged: the slip a kernel could make."""
    c = dict(c)
    if what == "f":
        c["fu"], c["fv"] = c["fv"], c["fu"]
    else:
        c["cu"], c["cv"] = c["cv"], c["cu"]
    return c


# ---------------------------------------------------------------------------------------------------------------------
# Poses (float64, stored as float32)
# ---------------------------------------------------------------------------------------------------------------------
def _rx(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def _rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def rotation(yaw_deg, pitch_deg=0.0, roll_deg=0.0):
    """R_L_C of a camera whose optical axis has heading yaw (from +x towards +y), pitched down by pitch and rolled about
    the optical axis by roll (degrees). pitch 90: looking straight down (-z); pitch -90: straight up."""
    y = math.radians(yaw_deg)
    f = np.array([math.cos(y), math.sin(y), 0.0])
    d = np.array([0.0, 0.0, -1.0])
    level = np.stack([np.cross(d, f), d, f], axis=1)  # columns: x right, y down, z forward
    return level @ _rx(-math.radians(pitch_deg)) @ _rz(math.radians(roll_deg))


def pose64(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def f32(T):
    return np.asarray(T, np.float64).astype(np.float32)


def optical_axis(T):
    return np.asarray(T, np.float64)[:3, 2]


def pitch_deg(T):
    """Angle of the optical axis below the horizontal."""
    return math.degrees(math.asin(float(np.clip(-optical_axis(T)[2], -1.0, 1.0))))


def roll_deg(T):
    """Rotation about the optical axis (zero when the camera x axis is horizontal), for a pitch away from +-90 degrees."""
    x = np.asarray(T, np.float64)[:3, 0]
    return math.degrees(math.asin(float(np.clip(-x[2] / math.cos(math.radians(pitch_deg(T))), -1.0, 1.0))))


def looking_at_centre(position, pitch=0.0, roll=0.0):
    """Heading from `position` towards the room's vertical axis."""
    return rotation(math.degrees(math.atan2(-position[1], -position[0])), pitch, roll)


def _case(name, scene, cam, R, t, claims, min_blocks, far=None):
    T = pose64(R, t)
    if far is not None:
        T[:3, 3] += np.asarray(far, np.float64)
    return dict(name=name, scene=scene, cam=CAMS[cam], cam_name=cam, pose=f32(T), claims=claims, min_blocks=min_blocks)


_CORNER = np.float32(BLOCK) * np.array([-5, 3, 2], np.float32)  # a block corner as the kernels compute it (block_size * index)

CASES = [
    _case("pitch_down_20", "sphere_in_box", "aniso_0.9", looking_at_centre((4.0, 1.0, 2.2), 20.0), (4.0, 1.0, 2.2),
          dict(pitch_deg=20.0, roll_deg=0.0), 1500),
    _case("pitch_down_50", "box_with_cube", "aniso_1.1", looking_at_centre((3.5, -2.0, 3.0), 50.0), (3.5, -2.0, 3.0),
          dict(pitch_deg=50.0, roll_deg=0.0), 1000),
    _case("roll_plus_30", "sphere_in_box", "half_integer_317x239", looking_at_centre((-3.8, 1.5, 1.8), 5.0, 30.0),
          (-3.8, 1.5, 1.8), dict(pitch_deg=5.0, roll_deg=30.0), 1500),
    _case("roll_minus_30", "box_with_cube", "odd_641x481", looking_at_centre((1.0, 4.0, 2.0), 10.0, -30.0), (1.0, 4.0, 2.0),
          dict(pitch_deg=10.0, roll_deg=-30.0), 1500),
    _case("straight_down", "box_with_cube", "aniso_0.9", rotation(30.0, 90.0), (2.6, 2.2, 1.5),
          dict(axis=(0.0, 0.0, -1.0)), 180),
    _case("straight_up", "sphere_in_box", "aniso_1.1", rotation(-60.0, -90.0), (2.5, -2.5, 1.0),
          dict(axis=(0.0, 0.0, 1.0)), 500),
    _case("identity_on_block_corner", "sphere_in_box", "distorted", np.eye(3), _CORNER.astype(np.float64),
          dict(axis=(0.0, 0.0, 1.0), block_corner=True), 500),
    _case("far_tilted", "sphere_in_box", "aniso_1.1", looking_at_centre((-1.0, -4.0, 2.5), 25.0, 10.0), (-1.0, -4.0, 2.5),
          dict(pitch_deg=25.0, roll_deg=10.0, far=True), 1500, far=FAR_OFFSET),
]
CASE = {c["name"]: c for c in CASES}


def scene_of(case):
    return {"sphere_in_box": syn.sphere_in_box, "box_with_cube": syn.box_with_cube}[case["scene"]]()


def local_pose(case):
    """The case's pose with the far offset taken off (the scene is rendered at the origin)."""
    T = np.array(case["pose"], np.float64)
    if case["claims"].get("far"):
        T[:3, 3] -= np.asarray(FAR_OFFSET, np.float64)
    return T


def yawed(T, deg):
    """T turned by deg about the world vertical through the camera's position (float64 in, float32 out)."""
    T = np.array(T, np.float64)
    T[:3, :3] = _rz(math.radians(deg)) @ T[:3, :3]
    return f32(T)


def frames(case, n=3, step_deg=4.0, noise=0.005, seed=0):
    """n noisy frames of the case, the camera turning step_deg about the vertical between frames: [(depth, T_L_C)]."""
    cs = syn.PinholeCamera(*(case["cam"][k] for k in ("fu", "fv", "cu", "cv", "width", "height")))
    scene = scene_of(case)
    out = []
    rng = np.random.default_rng(seed)
    for i in range(n):
        T_local = yawed(local_pose(case), step_deg * i)
        d = syn.render_depth(scene, cs, T_local)
        d = (d + rng.normal(0.0, 1.0, d.shape).astype(np.float32) * np.float32(noise) * d).astype(np.float32)
        T = np.array(T_local, np.float64)
        if case["claims"].get("far"):
            T[:3, 3] += np.asarray(FAR_OFFSET, np.float64)
        out.append((d, f32(T)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# A separate colour camera: different intrinsics and resolution, 5 cm baseline and a 1 degree rotation from the depth camera
# ---------------------------------------------------------------------------------------------------------------------
COLOR_DEPTH_CAM = intrinsics(640, 480, 290.0, 320.0, 320 + 0.12 * 640, 240 - 0.11 * 480)
COLOR_CAM = intrinsics(1280, 720, 610.0, 560.0, 640 - 0.13 * 1280, 360 + 0.12 * 720)


def _axis_angle(axis, deg):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    th = math.radians(deg)
    return np.eye(3) + math.sin(th) * K + (1.0 - math.cos(th)) * K @ K


T_D_C = pose64(_axis_angle((0.3, 1.0, 0.2), 1.0), (0.05, 0.0, 0.0))  # colour camera in the depth camera's frame


def color_poses(n=3):
    """[(T_L_D, T_L_C)] float32: the depth camera on a pitched, rolled path round the room and the colour camera on it."""
    out = []
    for i in range(n):
        p = (4.0 * math.cos(0.35 * i), 4.0 * math.sin(0.35 * i), 2.3)
        T_L_D = pose64(looking_at_centre(p, 15.0, 8.0), p)
        out.append((f32(T_L_D), f32(T_L_D @ T_D_C)))
    return out


STRIPE_PERIOD = 0.5
STRIPE_COLORS = ((230, 30, 20), (20, 40, 220))


def stripe_index(x):
    return np.floor(np.asarray(x, np.float64) / STRIPE_PERIOD).astype(np.int64) % 2


def stripe_image(scene, c, T_L_C, max_dist=20.0):
    """Colour image of `scene` seen by intrinsics c from T_L_C, painted by the float64 world hit point: stripes along world x
    with a STRIPE_PERIOD period; grey where no surface is hit."""
    hits = world_hits(scene, c, T_L_C, max_dist)
    img = np.full((c["height"], c["width"], 3), 127, np.uint8)
    ok = np.all(np.isfinite(hits), axis=-1)
    s = stripe_index(np.where(ok, hits[..., 0], 0.0))
    for k, col in enumerate(STRIPE_COLORS):
        img[ok & (s == k)] = col
    return img


def pixel_rays(c):
    """Unit camera-frame rays through the pixel centres (float64, (rows, cols, 3)), and their un-normalised z = 1 form."""
    cols = (np.arange(c["width"], dtype=np.float64) + 0.5 - c["cu"]) / c["fu"]
    rows = (np.arange(c["height"], dtype=np.float64) + 0.5 - c["cv"]) / c["fv"]
    vx, vy = np.meshgrid(cols, rows)
    v = np.stack([vx, vy, np.ones_like(vx)], axis=-1)
    return v / np.linalg.norm(v, axis=-1, keepdims=True), v


def world_hits(scene, c, T_L_C, max_dist=20.0):
    """float64 world points where the pixel-centre rays hit the scene; NaN where nothing is hit."""
    T = np.asarray(T_L_C, np.float64)
    d_C, _ = pixel_rays(c)
    d_L = d_C @ T[:3, :3].T
    t = scene.ray_distance(T[:3, 3], d_L, max_dist)
    return np.where(np.isfinite(t)[..., None], T[:3, 3] + d_L * t[..., None], np.nan)


# ---------------------------------------------------------------------------------------------------------------------
# A rig of three depth cameras on one body
# ---------------------------------------------------------------------------------------------------------------------
RIG_CAMS = {
    "front": intrinsics(640, 480, 300.0, 325.0, 320 + 0.1 * 640, 240 + 0.12 * 480),
    "side": intrinsics(1280, 720, 640.0, 590.0, 640 - 0.11 * 1280, 360 - 0.1 * 720),
    "rear": intrinsics(424, 240, 210.0, 190.0, 212 + 0.13 * 424, 120 - 0.14 * 240),
}
RIG_EXTRINSICS = {  # T_B_C: body frame x forward, y left, z up
    "front": pose64(rotation(0.0, 15.0), (0.25, 0.0, 0.45)),
    "side": pose64(rotation(90.0, 8.0, 4.0), (0.0, 0.15, 0.55)),
    "rear": pose64(rotation(180.0, 25.0, -6.0), (-0.25, 0.0, 0.35)),
}


def body_pose(i):
    th = 0.4 * i
    return pose64(_rz(th + math.pi / 2), (3.0 * math.cos(th), 3.0 * math.sin(th), 0.3))


# Frames of the rig, in order: (camera, body pose index). Each camera's pose comes back, with other cameras in between, so
# that the two-entry view-point cache (keyed on pose and camera) hits, misses and evicts.
RIG_ORDER = [("front", 0), ("side", 0), ("front", 0), ("rear", 0), ("side", 0), ("front", 1), ("rear", 1), ("rear", 1),
             ("side", 1), ("front", 1), ("front", 0)]


def rig_frames(noise=0.004, seed=5):
    """[(camera name, depth, T_L_C float32)] in RIG_ORDER, a fresh noise draw per frame (a cache hit reuses the block list
    of an earlier, different depth image)."""
    rng = np.random.default_rng(seed)
    scene = syn.box_with_cube()
    out = []
    for name, i in RIG_ORDER:
        c = RIG_CAMS[name]
        T = f32(body_pose(i) @ RIG_EXTRINSICS[name])
        cs = syn.PinholeCamera(*(c[k] for k in ("fu", "fv", "cu", "cv", "width", "height")))
        d = syn.render_depth(scene, cs, T)
        d = (d + rng.normal(0.0, 1.0, d.shape).astype(np.float32) * np.float32(noise) * d).astype(np.float32)
        out.append((name, d, T))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# The reference's symmetric view on a plane (tests/test_tsdf_error.cpp:56-224) and its general-camera variant
# ---------------------------------------------------------------------------------------------------------------------
PLANE_Z = 3.0
PLANE_THETA = math.pi / 8.0
PLANE_OFFSET = 2.0
PLANE_MAX_DIST = 100.0
PLANE_CAM = intrinsics(640, 480, 300.0, 300.0, 320.0, 240.0)  # TsdfErrorTest (:46-53)
PLANE_CAM_GENERAL = intrinsics(640, 480, 280.0, 315.0, 320 + 0.12 * 640, 240 - 0.1 * 480)
PLANE_PITCH_DEG = 12.0


def plane_scene():
    return syn.Scene().add_plane(2, PLANE_Z)


def plane_setup(general):
    """-> [(intrinsics, T_L_C float32)] for the two cameras. The reference: identity rotated by +-pi/8 about y, shifted by
    -+2 m in x. The general variant: fu != fv, the principal point mirrored between the cameras (cu' = W - cu), and both
    cameras pitched by the same angle about their x axis."""
    out = []
    for sign in (1.0, -1.0):
        R = _axis_angle((0.0, 1.0, 0.0), math.degrees(sign * PLANE_THETA))
        c = PLANE_CAM
        if general:
            R = R @ _rx(math.radians(PLANE_PITCH_DEG))
            c = dict(PLANE_CAM_GENERAL)
            if sign < 0:
                c["cu"] = c["width"] - c["cu"]
        out.append((c, f32(pose64(R, (-sign * PLANE_OFFSET, 0.0, 0.0)))))
    return out
