"""Deterministic synthetic LiDAR-camera bags for the BASELINE.json configs (SURVEY.md section 8d).

A box-room scene with a procedural albedo texture is seen by a LiDAR (ray-cast sampling pattern) and by a camera
(ray-cast render through the ground-truth camera model).  The outputs have the same statistics the reference's
preprocessing produces: xyz float32-representable (PLY floats, preprocess.cpp:167-169), LiDAR intensities
rank-equalised to k/256 (preprocess.cpp:464-473), image histogram-equalised uint8 (preprocess.cpp:419), so that the
NID objective has a genuine minimum at the ground-truth extrinsics.  numpy only; seeds are explicit.
"""
from __future__ import annotations

import math

import numpy as np

# camera frame: z forward, x right, y down; LiDAR frame: x forward, y left, z up
R_CAMERA_LIDAR = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])


def gt_T_camera_lidar(t=(0.05, -0.08, -0.03)) -> np.ndarray:
    T = np.eye(4)
    T[:3, :3] = R_CAMERA_LIDAR
    T[:3, 3] = t
    return T


def perturb(T: np.ndarray, rot_deg=(0.5, 0.5, 0.5), trans=(0.02, 0.02, 0.02)) -> np.ndarray:
    """T * Exp(rot, trans) with the closed-form SE(3) exponential (numpy; test/bench input only)."""
    w = np.deg2rad(np.asarray(rot_deg, dtype=np.float64))
    v = np.asarray(trans, dtype=np.float64)
    th = np.linalg.norm(w)
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        R, V = np.eye(3) + W, np.eye(3)
    else:
        A, B, Cc = math.sin(th) / th, (1 - math.cos(th)) / th**2, (th - math.sin(th)) / th**3
        R = np.eye(3) + A * W + B * W @ W
        V = np.eye(3) + B * W + Cc * W @ W
    E = np.eye(4)
    E[:3, :3] = R
    E[:3, 3] = V @ v
    return T @ E


# ---------------------------------------------------------------------------------------------
# scene
# ---------------------------------------------------------------------------------------------

ROOM_MIN = np.array([-10.0, -10.0, -2.0])
ROOM_MAX = np.array([10.0, 10.0, 3.0])


def _boxes(seed: int, count: int = 20):
    rng = np.random.default_rng(seed)
    centers = np.stack([rng.uniform(3.0, 9.0, count), rng.uniform(-7.0, 7.0, count), rng.uniform(-1.5, 1.5, count)], axis=1)
    half = rng.uniform(0.25, 1.0, (count, 3))
    return centers - half, centers + half


def _raycast(origin: np.ndarray, dirs: np.ndarray, boxes) -> np.ndarray:
    """First hit distance of rays (origin inside the room) with the room walls and the boxes."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
        # room: exit distance (origin is inside)
        t1 = (ROOM_MIN - origin) * inv
        t2 = (ROOM_MAX - origin) * inv
        t_room = np.nanmin(np.maximum(t1, t2), axis=1)
        t_hit = t_room
        lo, hi = boxes
        for k in range(lo.shape[0]):
            a = (lo[k] - origin) * inv
            b = (hi[k] - origin) * inv
            tn = np.nanmax(np.minimum(a, b), axis=1)
            tf = np.nanmin(np.maximum(a, b), axis=1)
            ok = (tn <= tf) & (tn > 0.05)
            t_hit = np.where(ok & (tn < t_hit), tn, t_hit)
    return t_hit


def albedo(X: np.ndarray) -> np.ndarray:
    """Procedural surface texture in [0,1] as a function of the 3-D position (LiDAR frame)."""
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    a = 0.5 + 0.22 * np.sin(1.7 * x + 0.9 * y) * np.cos(2.3 * z - 0.4 * y) + 0.18 * np.sin(5.1 * y + 1.3 * z + 0.7 * x)
    checker = ((np.floor(x * 0.8) + np.floor(y * 0.8) + np.floor(z * 0.8)) % 2) * 0.25 - 0.125
    stripes = 0.1 * np.sign(np.sin(9.0 * (x + y + z)))
    return np.clip(a + checker + stripes, 0.0, 1.0)


# ---------------------------------------------------------------------------------------------
# camera models: forward = the product/oracle; here only the INVERSE (pixel -> ray) for rendering
# ---------------------------------------------------------------------------------------------

def pixel_rays(model: str, intr, dist, width: int, height: int) -> np.ndarray:
    """Unit ray (camera frame) through every pixel centre, (H*W,3); NaN rows where no ray exists."""
    u, v = np.meshgrid(np.arange(width) + 0.5, np.arange(height) + 0.5)
    u, v = u.reshape(-1), v.reshape(-1)
    intr = np.asarray(intr, dtype=np.float64)
    d = np.zeros(8)
    d[: len(dist)] = dist
    if model == "equirectangular":
        lon = (u / intr[0] - 0.5) * 2.0 * math.pi
        lat = (0.5 - v / intr[1]) * math.pi
        by = -np.sin(lat)
        c = np.cos(lat)
        return np.stack([c * np.sin(lon), by, c * np.cos(lon)], axis=1)
    xd, yd = (u - intr[2]) / intr[0], (v - intr[3]) / intr[1]
    if model == "plumb_bob":
        k1, k2, p1, p2, k3 = d[:5]
        x, y = xd.copy(), yd.copy()
        for _ in range(20):  # fixed-point inverse of the plumb-bob distortion
            r2 = x * x + y * y
            rc = 1 + k1 * r2 + k2 * r2**2 + k3 * r2**3
            dx = 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
            dy = p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
            x, y = (xd - dx) / rc, (yd - dy) / rc
        rays = np.stack([x, y, np.ones_like(x)], axis=1)
    elif model in ("fisheye", "equidistant"):
        k1, k2, k3, k4 = d[:4]
        thd = np.sqrt(xd * xd + yd * yd)
        th = thd.copy()
        for _ in range(20):  # Newton on theta_d(theta)
            t2 = th * th
            f = th * (1 + k1 * t2 + k2 * t2**2 + k3 * t2**3 + k4 * t2**4) - thd
            fp = 1 + 3 * k1 * t2 + 5 * k2 * t2**2 + 7 * k3 * t2**3 + 9 * k4 * t2**4
            th = th - f / fp
        s = np.where(thd > 1e-12, np.sin(th) / np.maximum(thd, 1e-12), 1.0)
        rays = np.stack([xd * s, yd * s, np.cos(th)], axis=1)
        rays[th > 0.5 * math.pi - 1e-3] = np.nan  # abs(z) in the forward model folds the back hemisphere
    else:
        raise ValueError(f"no inverse projection for {model}")
    return rays / np.linalg.norm(rays, axis=1, keepdims=True)


def _equalize_u8(img: np.ndarray) -> np.ndarray:
    """cv::equalizeHist on a uint8 image (numpy restatement; preprocess.cpp:419)."""
    hist = np.bincount(img.reshape(-1), minlength=256)
    nz = np.nonzero(hist)[0]
    if nz.size <= 1:
        return img.copy()
    cdf = np.cumsum(hist)
    cdf_min = cdf[nz[0]]
    total = img.size
    lut = np.clip(np.round((cdf - cdf_min) / float(total - cdf_min) * 255.0), 0, 255).astype(np.uint8)
    return lut[img]


def render_image(model: str, intr, dist, width: int, height: int, T_camera_lidar: np.ndarray, scene_seed: int, noise_seed: int, noise_sigma: float = 4.0) -> np.ndarray:
    rays_c = pixel_rays(model, intr, dist, width, height)
    R, t = T_camera_lidar[:3, :3], T_camera_lidar[:3, 3]
    origin = -R.T @ t  # camera centre in the LiDAR frame
    bad = ~np.isfinite(rays_c).all(axis=1)
    rays_c = np.where(bad[:, None], np.array([0.0, 0.0, 1.0]), rays_c)
    dirs = rays_c @ R  # R^T applied to each row
    boxes = _boxes(scene_seed)
    img = np.empty(width * height)
    chunk = 1 << 19
    for s in range(0, dirs.shape[0], chunk):
        dseg = dirs[s : s + chunk]
        th = _raycast(origin, dseg, boxes)
        img[s : s + chunk] = albedo(origin + dseg * th[:, None])
    rng = np.random.default_rng(noise_seed)
    img = img * 255.0 + rng.normal(0.0, noise_sigma, img.shape)
    img[bad] = 0.0
    img8 = np.clip(np.round(img), 0, 255).astype(np.uint8).reshape(height, width)
    return _equalize_u8(img8)


# ---------------------------------------------------------------------------------------------
# LiDAR sampling patterns
# ---------------------------------------------------------------------------------------------

def lidar_directions(pattern: str, n: int, rng: np.random.Generator, az_half_deg: float = 65.0) -> np.ndarray:
    if pattern == "os1_64":  # 64 rings in +-16.6 deg, azimuth restricted to the camera side, small vertical dither
        ring = rng.integers(0, 64, n)
        el = np.deg2rad(-16.6 + 33.2 * ring / 63.0 + rng.uniform(-0.25, 0.25, n))
        az = np.deg2rad(rng.uniform(-az_half_deg, az_half_deg, n))
    elif pattern == "avia":  # non-repetitive: uniform over a 70.4 x 77.2 deg window
        az = np.deg2rad(rng.uniform(-35.2, 35.2, n))
        el = np.deg2rad(rng.uniform(-38.6, 38.6, n))
    elif pattern == "frustum":  # 100 x 80 deg window (C1: ~20 % outside a 640x480 f=400 pinhole)
        az = np.deg2rad(rng.uniform(-50.0, 50.0, n))
        el = np.deg2rad(rng.uniform(-40.0, 40.0, n))
    elif pattern == "sphere":  # full sphere (equirectangular)
        az = rng.uniform(-math.pi, math.pi, n)
        el = np.arcsin(rng.uniform(-0.95, 0.95, n))
    else:
        raise ValueError(pattern)
    ce = np.cos(el)
    return np.stack([ce * np.cos(az), ce * np.sin(az), np.sin(el)], axis=1)


def make_cloud(pattern: str, n: int, scene_seed: int, seed: int, intensity_sigma: float = 0.05):
    """Returns (points_xyzw float64 (n,4) float32-representable, intensities float64 (n,) in {k/256})."""
    rng = np.random.default_rng(seed)
    boxes = _boxes(scene_seed)
    origin = np.zeros(3)
    pts = np.empty((n, 3))
    chunk = 1 << 19
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        dirs = lidar_directions(pattern, m, rng)
        th = _raycast(origin, dirs, boxes)
        pts[s : s + m] = dirs * th[:, None]
    pts = pts.astype(np.float32).astype(np.float64)  # PLY floats
    a = albedo(pts) + rng.normal(0.0, intensity_sigma, n)
    order = np.argsort(a, kind="stable")  # rank equalisation (preprocess.cpp:464-473)
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n)
    inten = np.floor(256.0 * rank / n) / 256.0
    xyzw = np.concatenate([pts, np.ones((n, 1))], axis=1)
    return np.ascontiguousarray(xyzw), np.ascontiguousarray(inten)


# ---------------------------------------------------------------------------------------------
# BASELINE.json configs
# ---------------------------------------------------------------------------------------------

CAMERAS = {
    "pinhole_640x480": ("plumb_bob", [400.0, 400.0, 320.0, 240.0], [-0.04, 0.08, 1e-4, -3e-4, -0.04], 640, 480),
    "pinhole_1920x1080": ("plumb_bob", [1000.0, 1000.0, 960.0, 540.0], [-0.04, 0.08, 1e-4, -3e-4, -0.04], 1920, 1080),
    "equirect_3840x1920": ("equirectangular", [3840.0, 1920.0], [], 3840, 1920),
    "fisheye_1920x1080": ("fisheye", [600.0, 600.0, 960.0, 540.0], [0.01, -0.02, 0.003, -0.001], 1920, 1080),
    "atan_1920x1080": ("atan", [1000.0, 1000.0, 960.0, 540.0], [0.9], 1920, 1080),
    "omnidir_1920x1080": ("omnidir", [700.0, 700.0, 960.0, 540.0, 1.1], [-0.1, 0.02, 1e-3, -2e-3], 1920, 1080),
    "rational_1920x1080": ("rational_polynomial", [1000.0, 1000.0, 960.0, 540.0], [-0.04, 0.08, 1e-4, -3e-4, -0.04, 0.01, 0.02, -0.005], 1920, 1080),
}

SEED0 = 20260922


def make_bag(camera_key: str, pattern: str, n_points: int, config_index: int = 0, bag_index: int = 0, scale: float = 1.0):
    """One (camera, image, cloud) bag. `scale` < 1 shrinks image size and focal lengths (tests)."""
    model, intr, dist, w, h = CAMERAS[camera_key]
    intr = list(intr)
    if scale != 1.0:
        w, h = int(round(w * scale)), int(round(h * scale))
        if model == "equirectangular":
            intr = [float(w), float(h)]
        else:
            intr = [v * scale for v in intr]
    seed = SEED0 + 1000 * config_index + bag_index
    T_gt = gt_T_camera_lidar()
    pts, inten = make_cloud(pattern, n_points, scene_seed=seed, seed=seed + 1)
    image = render_image(model, intr, dist, w, h, T_gt, scene_seed=seed, noise_seed=seed + 2)
    return {"camera_model": model, "intrinsics": intr, "distortion": list(dist), "width": w, "height": h, "image": image, "points": pts, "intensities": inten, "T_gt": T_gt}


def config_c1():
    return make_bag("pinhole_640x480", "frustum", 100_000, config_index=0)


def config_c2(n_points: int = 1_000_000):
    bag = make_bag("pinhole_1920x1080", "os1_64", n_points, config_index=1)
    bag["T_init"] = perturb(bag["T_gt"], (0.5, 0.5, 0.5), (0.02, 0.02, 0.02))
    return bag


def config_c3(n_points: int = 5_000_000, camera_key: str = "equirect_3840x1920"):
    return make_bag(camera_key, "avia", n_points, config_index=2)


def pose_grid(T_center: np.ndarray, n_rot=(8, 8, 8), n_trans=(2, 4, 4), rot_half_deg=4.0, trans_half=0.10) -> np.ndarray:
    """C5: 8x8x8 rotations (+-4 deg per axis) x 2x4x4 translations (+-10 cm) about T_center -> (P,4,4)."""
    axes_r = [np.linspace(-rot_half_deg, rot_half_deg, k) for k in n_rot]
    axes_t = [np.linspace(-trans_half, trans_half, k) for k in n_trans]
    out = []
    for rx in axes_r[0]:
        for ry in axes_r[1]:
            for rz in axes_r[2]:
                for tx in axes_t[0]:
                    for ty in axes_t[1]:
                        for tz in axes_t[2]:
                            out.append(perturb(T_center, (rx, ry, rz), (tx, ty, tz)))
    return np.stack(out)


# ---------------------------------------------------------------------------------------------
# initial_guess_auto datasets
# ---------------------------------------------------------------------------------------------

def _axis_rotation(axis: int, angle: float) -> np.ndarray:
    c, s = math.cos(angle), math.sin(angle)
    i, j = (axis + 1) % 3, (axis + 2) % 3
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def virtual_lidar_camera(lidar_fov: float):
    """The virtual camera preprocess renders the LiDAR image with (preprocess.cpp:180-197): below a 150 deg LiDAR FoV a
    1024 x 1024 pinhole looking along LiDAR +x, otherwise a 1920 x 960 equirectangular image.
    -> (camera_model, intrinsics, (W, H), T_camera_lidar of the virtual camera)."""
    T_lidar_camera = np.eye(4)
    if lidar_fov < math.radians(150.0):
        W, H = 1024, 1024
        T_lidar_camera[:3, :3] = _axis_rotation(1, math.pi / 2) @ _axis_rotation(2, -math.pi / 2)
        fx = W / (2.0 * math.tan(lidar_fov / 2.0))
        model, intr = "plumb_bob", [fx, fx, W / 2.0, H / 2.0]
    else:
        W, H = 1920, 960
        T_lidar_camera[:3, :3] = _axis_rotation(0, -math.pi / 2)
        model, intr = "equirectangular", [float(W), float(H)]
    T_camera_lidar = np.eye(4)
    T_camera_lidar[:3, :3] = T_lidar_camera[:3, :3].T
    return model, intr, (W, H), T_camera_lidar


def write_initial_guess_dataset(
    data_path: str, n_bags: int = 2, camera_key: str = "pinhole_640x480", pattern: str = "frustum", n_points: int = 30_000, n_matches: int = 300,
    outlier_fraction: float = 0.25, unmatched_fraction: float = 0.1, blank_fraction: float = 0.05, lidar_fov_deg: float = 120.0, seed: int = 0, device: int = -1):
    """A preprocessed dataset as initial_guess_auto finds it: calib.json (camera + meta.bag_names, no results), and per bag
    <bag>.png, <bag>.ply, <bag>_lidar_indices.png (generate_lidar_image through the virtual LiDAR camera, on the GPU) and
    <bag>_matches.json.  Matches pair a LiDAR-image pixel (float keypoint inside it) with the ground-truth projection of its
    point into the camera (float keypoint); `outlier_fraction` of the matches get a random camera keypoint instead, and the
    file also holds unmatched keypoints (match -1) and matches onto blank LiDAR-image pixels.  Returns the bags (make_bag
    dicts) with the ground truth T_gt (T_camera_lidar)."""
    import json
    import os

    import cv2

    from . import io as vio
    from .camera import create_camera
    from .culling import generate_lidar_image

    rng = np.random.default_rng(seed)
    vmodel, vintr, vsize, T_vcam_lidar = virtual_lidar_camera(math.radians(lidar_fov_deg))
    vproj = create_camera(vmodel, vintr, [])
    bags, names = [], []
    for b in range(n_bags):
        bag = make_bag(camera_key, pattern, n_points, config_index=7, bag_index=b)
        name = f"bag{b}"
        cv2.imwrite(os.path.join(data_path, name + ".png"), bag["image"])
        vio.save_ply_binary(os.path.join(data_path, name + ".ply"), bag["points"][:, :3], bag["intensities"])
        _, index_image = generate_lidar_image(vproj, vsize, T_vcam_lidar, bag["points"], bag["intensities"], device=device)
        vio.save_lidar_indices(os.path.join(data_path, name + "_lidar_indices.png"), index_image)

        # LiDAR-image pixels whose point lands in front of the camera, inside the image
        proj = create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
        ys, xs = np.nonzero(index_image >= 0)
        pick = rng.permutation(xs.size)[: 4 * n_matches]
        xs, ys = xs[pick], ys[pick]
        pc = bag["points"][index_image[ys, xs], :3] @ bag["T_gt"][:3, :3].T + bag["T_gt"][:3, 3]
        uv = proj.project(pc)
        ok = (pc[:, 2] > 0.1) & (uv[:, 0] >= 0) & (uv[:, 0] < bag["width"]) & (uv[:, 1] >= 0) & (uv[:, 1] < bag["height"])
        xs, ys, uv = xs[ok][:n_matches], ys[ok][:n_matches], uv[ok][:n_matches]
        n = xs.size
        n_out = int(round(outlier_fraction * n))
        uv[:n_out] = rng.uniform([0.0, 0.0], [bag["width"], bag["height"]], (n_out, 2))  # wrong matches
        kpts1 = np.stack([xs, ys], axis=1) + rng.uniform(0.0, 0.999, (n, 2))
        kpts0 = uv
        matches = np.arange(n)
        # matches onto blank LiDAR-image pixels, and unmatched keypoints
        by, bx = np.nonzero(index_image < 0)
        n_blank = int(round(blank_fraction * n))
        pick = rng.choice(bx.size, n_blank, replace=False)
        kpts1 = np.concatenate([kpts1, np.stack([bx[pick], by[pick]], axis=1) + 0.5])
        kpts0 = np.concatenate([kpts0, rng.uniform([0.0, 0.0], [bag["width"], bag["height"]], (n_blank, 2))])
        matches = np.concatenate([matches, n + np.arange(n_blank)])
        n_unmatched = int(round(unmatched_fraction * n))
        kpts0 = np.concatenate([kpts0, rng.uniform([0.0, 0.0], [bag["width"], bag["height"]], (n_unmatched, 2))])
        matches = np.concatenate([matches, -np.ones(n_unmatched, dtype=np.int64)])
        order = rng.permutation(matches.size)
        result = {
            "kpts0": kpts0[order].reshape(-1).tolist(), "kpts1": kpts1.reshape(-1).tolist(),
            "matches": [int(v) for v in matches[order]], "confidence": rng.uniform(0.2, 1.0, matches.size).tolist(),
        }
        with open(os.path.join(data_path, name + "_matches.json"), "w") as f:
            json.dump(result, f)
        bag["n_outliers"] = n_out
        bags.append(bag)
        names.append(name)
    model, intr, dist = bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"]
    config = {"camera": {"camera_model": model, "intrinsics": list(intr), "distortion_coeffs": list(dist)}, "meta": {"bag_names": names}}
    vio.save_calib_json(data_path, config)
    return bags
