"""`preprocess_map`: a calibration dataset from a point-cloud map and one camera image (src/preprocess_map.cpp).

    map (PCD / PLY) --load_map_cloud--> ApproximateVoxelGrid (GPU) --> rank equalisation (GPU) --> 000000.ply
                                        estimate_lidar_fov: VoxelGrid 0.2 m + norm filter (GPU), qhull hull (host),
                                                            min pairwise bearing cosine (GPU)
                                        virtual LiDAR camera --> generate_lidar_image (GPU, K5)
                                                             --> 000000_lidar_intensities.png, 000000_lidar_indices.png
    image --equalizeHist--> 000000.png;  calib.json (camera + meta)

The files are the ones the reference's preprocess_map writes, so initial_guess_auto and calibrate read them unchanged.
Deviations (DESIGN §4 "preprocess_map"): ties of the rank equalisation go by point index, the 0.2 m voxel sums run in
point-index order, and input the reference is undefined or silently wrong on is refused."""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np

from . import _lib
from . import io as vio


def _i64():
    return C.c_int64()


def approximate_voxel_grid(points_xyzi, leaf_size: float = 0.002, device: int = -1, stats: dict | None = None) -> np.ndarray:
    """pcl::ApproximateVoxelGrid<PointXYZI> with leaf float(leaf_size) on float32 (N, 4) x, y, z, intensity
    (preprocess_map.cpp:140-147) -> float32 (M, 4) centroids in the reference's output order.  `stats` (optional dict)
    receives `out_of_range_points` and `stage_ms` (keys, sort, runs, order)."""
    L = _lib.load_library()
    pts = np.ascontiguousarray(np.asarray(points_xyzi, dtype=np.float32).reshape(-1, 4))
    out = np.empty_like(pts) if pts.shape[0] else np.empty((1, 4), np.float32)
    n_out, oor = _i64(), _i64()
    ms = (C.c_double * 4)()
    _lib.check(L.vlcal_approximate_voxel_grid(device, pts.ctypes.data, pts.shape[0], float(leaf_size), out.ctypes.data, C.byref(n_out), C.byref(oor),
                                              ms if stats is not None else None))
    if stats is not None:
        stats["out_of_range_points"] = int(oor.value)
        stats["stage_ms"] = list(ms)
    elif oor.value:
        print(f"warning: {oor.value} points have a voxel index outside int range at leaf {leaf_size}; like the reference, "
              "their index becomes INT_MIN, which merges voxels along that axis")
    return out[: n_out.value].copy()


def equalize_intensities(intensities, device: int = -1, stats: dict | None = None) -> np.ndarray:
    """The rank equalisation of preprocess_map.cpp:158-167 on float32 intensities -> float64 k/256 per point; ties by
    point index."""
    L = _lib.load_library()
    ins = np.ascontiguousarray(np.asarray(intensities, dtype=np.float32).reshape(-1))
    out = np.empty(ins.shape[0], dtype=np.float64)
    ms = C.c_double()
    _lib.check(L.vlcal_equalize_intensities(device, ins.ctypes.data, ins.shape[0], out.ctypes.data, C.byref(ms)))
    if stats is not None:
        stats["kernel_ms"] = ms.value
    return out


def lidar_fov_candidates(points_xyz, device: int = -1, stats: dict | None = None):
    """estimate_fov.cpp:53-66: VoxelGrid 0.2 m (or the input, where PCL's grid would overflow int32), then the points with
    norm < 1 removed -> (float32 (K, 3), unfiltered: bool)."""
    L = _lib.load_library()
    pts = np.ascontiguousarray(np.asarray(points_xyz, dtype=np.float32)[:, :3])
    out = np.empty((max(pts.shape[0], 1), 3), dtype=np.float32)
    n_out, unfiltered, ms = _i64(), C.c_int(), C.c_double()
    _lib.check(L.vlcal_lidar_fov_candidates(device, pts.ctypes.data, pts.shape[0], out.ctypes.data, C.byref(n_out), C.byref(unfiltered), C.byref(ms)))
    if stats is not None:
        stats["kernel_ms"] = ms.value
    if unfiltered.value:
        print("warning: leaf size is too small for the input dataset; integer indices would overflow (PCL VoxelGrid): the FoV hull uses every point")
    return out[: n_out.value].copy(), bool(unfiltered.value)


def min_bearing_cosine(vertices_xyz, device: int = -1) -> float:
    """min over vertex pairs i < j of dot(normalized(v_i), normalized(v_j)) in double, starting from M_PI
    (estimate_fov.cpp:78-89)."""
    L = _lib.load_library()
    v = np.ascontiguousarray(np.asarray(vertices_xyz, dtype=np.float32).reshape(-1, 3))
    out = C.c_double()
    _lib.check(L.vlcal_min_bearing_cosine(device, v.ctypes.data, v.shape[0], C.byref(out)))
    return out.value


def hull_vertices(points_xyz) -> np.ndarray:
    """The vertices of pcl::ConvexHull<PointXYZ>::reconstruct (qhull, via scipy) -> float32 (V, 3) in input order.

    Refused where the reference's result is not a 3-D hull: fewer than 4 points, a flat cloud (PCL's dimension test: the
    smallest covariance eigenvalue below 1e-3 of the largest, where PCL switches to a 2-D hull), or a qhull failure.  The
    reference would then compute acos(M_PI) = NaN or a 2-D FoV and pick its virtual camera from that."""
    pts = np.asarray(points_xyz, dtype=np.float32).reshape(-1, 3)
    if pts.shape[0] < 4:
        raise ValueError(f"estimate_lidar_fov: {pts.shape[0]} points remain after the 0.2 m voxel grid and the 1 m range cut; a 3-D hull needs at least 4")
    p = pts.astype(np.float64)
    cov = np.cov(p, rowvar=False, bias=True)
    ev = np.linalg.eigvalsh(cov)
    if abs(ev[0]) < np.finfo(np.float64).eps or abs(ev[0] / ev[2]) < 1.0e-3:
        raise ValueError("estimate_lidar_fov: the filtered cloud is flat (smallest covariance eigenvalue < 1e-3 of the largest); "
                         "the reference would take a 2-D hull there")
    from scipy.spatial import ConvexHull, QhullError

    try:
        hull = ConvexHull(p)
    except QhullError as e:
        raise ValueError(f"estimate_lidar_fov: qhull failed: {str(e).splitlines()[0]}") from None
    return pts[np.sort(hull.vertices)]


def estimate_lidar_fov(points_xyz, device: int = -1, stats: dict | None = None) -> float:
    """vlcal::estimate_lidar_fov (estimate_fov.cpp:53-91) -> the LiDAR FoV in radians."""
    cand, _ = lidar_fov_candidates(points_xyz, device=device, stats=stats)
    verts = hull_vertices(cand)
    if stats is not None:
        stats["candidates"] = int(cand.shape[0])
        stats["hull_vertices"] = int(verts.shape[0])
    return math.acos(min_bearing_cosine(verts, device=device))


# ---- the virtual LiDAR camera (preprocess_map.cpp:183-197), with Eigen's arithmetic -----------------------------------

def _angle_axis_quaternion(angle: float, axis):
    """AngleAxisd -> Quaterniond: (cos(a/2), sin(a/2) * axis) -> (w, x, y, z)."""
    ha = 0.5 * angle
    s = math.sin(ha)
    return (math.cos(ha), s * axis[0], s * axis[1], s * axis[2])


def _quaternion_product(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by + ay * bw + az * bx - ax * bz,
        aw * bz + az * bw + ax * by - ay * bx,
    )


def _quaternion_to_matrix(q) -> np.ndarray:
    """Eigen's Quaternion::toRotationMatrix."""
    w, x, y, z = q
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([
        [1.0 - (tyy + tzz), txy - twz, txz + twy],
        [txy + twz, 1.0 - (txx + tzz), tyz - twx],
        [txz - twy, tyz + twx, 1.0 - (txx + tyy)],
    ])


def _angle_axis_to_matrix(angle: float, axis) -> np.ndarray:
    """Eigen's AngleAxis::toRotationMatrix."""
    sin_axis = [math.sin(angle) * a for a in axis]
    c = math.cos(angle)
    cos1_axis = [(1.0 - c) * a for a in axis]
    R = np.empty((3, 3))
    tmp = cos1_axis[0] * axis[1]
    R[0, 1], R[1, 0] = tmp - sin_axis[2], tmp + sin_axis[2]
    tmp = cos1_axis[0] * axis[2]
    R[0, 2], R[2, 0] = tmp + sin_axis[1], tmp - sin_axis[1]
    tmp = cos1_axis[1] * axis[2]
    R[1, 2], R[2, 1] = tmp - sin_axis[0], tmp + sin_axis[0]
    for i in range(3):
        R[i, i] = cos1_axis[i] * axis[i] + c
    return R


def virtual_lidar_rotation(lidar_fov: float) -> np.ndarray:
    """T_lidar_camera.linear() of the virtual LiDAR camera: below 150 deg
    (AngleAxis(pi/2, Y) * AngleAxis(-pi/2, Z)).toRotationMatrix(), a quaternion product and Quaternion::toRotationMatrix;
    otherwise AngleAxis(-pi/2, X).toRotationMatrix()."""
    if lidar_fov < 150.0 * math.pi / 180.0:
        q = _quaternion_product(_angle_axis_quaternion(math.pi / 2, (0.0, 1.0, 0.0)), _angle_axis_quaternion(-math.pi / 2, (0.0, 0.0, 1.0)))
        return _quaternion_to_matrix(q)
    return _angle_axis_to_matrix(-math.pi / 2, (1.0, 0.0, 0.0))


def virtual_lidar_camera(lidar_fov: float):
    """preprocess_map.cpp:183-197 -> (camera_model, intrinsics, (W, H), T_camera_lidar = T_lidar_camera.inverse())."""
    if lidar_fov < 150.0 * math.pi / 180.0:
        W, H = 1024, 1024
        fx = W / (2.0 * math.tan(lidar_fov / 2.0))
        model, intr = "plumb_bob", [fx, fx, W / 2.0, H / 2.0]
    else:
        W, H = 1920, 960
        model, intr = "equirectangular", [float(W), float(H)]
    R = virtual_lidar_rotation(lidar_fov)
    T = np.eye(4)
    T[:3, :3] = R.T
    for i in range(3):  # Isometry3d::inverse(): -(R^T t), t = 0
        T[i, 3] = -((R[0, i] * 0.0 + R[1, i] * 0.0) + R[2, i] * 0.0)
    return model, intr, (W, H), T


def lidar_intensity_png(intensity_image) -> np.ndarray:
    """intensities.convertTo(CV_8UC1, 255.0): v * 255 rounded half to even, saturated."""
    return np.clip(np.rint(np.asarray(intensity_image, dtype=np.float64) * 255.0), 0, 255).astype(np.uint8)


def parse_values(text: str, name: str) -> list:
    """boost::split(text, ",") then std::stod on each token (preprocess_map.cpp:87-92)."""
    try:
        return [float(tok) for tok in text.split(",")]
    except ValueError:
        raise ValueError(f"--{name}: expected comma-separated numbers without spaces, got {text!r}") from None


def calib_config(map_path: str, camera_model: str, intrinsics, distortion) -> dict:
    """calib.json of preprocess_map (preprocess_map.cpp:100-109)."""
    return {
        "camera": {"camera_model": camera_model, "distortion_coeffs": list(distortion), "intrinsics": list(intrinsics)},
        "meta": {
            "bag_names": ["000000"], "camera_info_topic": "N/A", "data_path": map_path, "image_topic": "N/A", "intensity_channel": "N/A",
            "points_topic": "N/A",
        },
    }


def preprocess_map(map_path: str, image_path: str, dst_path: str, camera_model: str, intrinsics, distortion, voxel_resolution: float = 0.002,
                   device: int = -1, stats: dict | None = None) -> dict:
    """PreprocessMap::run without the viewer (preprocess_map.cpp:34-127): writes 000000.png, 000000.ply,
    000000_lidar_intensities.png, 000000_lidar_indices.png and calib.json into dst_path.  Returns the calib.json content.
    `stats` (optional dict) receives the counts, the FoV and the per-stage GPU times."""
    import cv2

    from .camera import create_camera
    from .culling import generate_lidar_image

    stats = {} if stats is None else stats
    os.makedirs(dst_path, exist_ok=True)
    image = vio.load_image_gray(image_path)
    cv2.imwrite(os.path.join(dst_path, "000000.png"), cv2.equalizeHist(image))

    cloud = vio.load_map_cloud(map_path)
    if cloud.shape[0] == 0:
        raise ValueError(f"no map points in {map_path}")
    avg_stats, eq_stats, fov_stats = {}, {}, {}
    filtered = approximate_voxel_grid(cloud, voxel_resolution, device=device, stats=avg_stats)
    if avg_stats["out_of_range_points"]:
        print(f"warning: {avg_stats['out_of_range_points']} points have a voxel index outside int range at leaf {voxel_resolution}; like the "
              "reference, their index becomes INT_MIN, which merges voxels along that axis")
    print(f"map_points={cloud.shape[0]} filtered={filtered.shape[0]}")
    intensities = equalize_intensities(filtered[:, 3], device=device, stats=eq_stats)
    vio.save_ply_binary(os.path.join(dst_path, "000000.ply"), filtered[:, :3], intensities)

    lidar_fov = estimate_lidar_fov(filtered[:, :3], device=device, stats=fov_stats)
    print(f"LiDAR FoV: {lidar_fov * 180.0 / math.pi}[deg]")
    model, intr, size, T_camera_lidar = virtual_lidar_camera(lidar_fov)
    points = np.concatenate([filtered[:, :3].astype(np.float64), np.ones((filtered.shape[0], 1))], axis=1)
    inten_img, index_img = generate_lidar_image(create_camera(model, intr, []), size, T_camera_lidar, points, intensities, device=device)
    cv2.imwrite(os.path.join(dst_path, "000000_lidar_intensities.png"), lidar_intensity_png(inten_img))
    vio.save_lidar_indices(os.path.join(dst_path, "000000_lidar_indices.png"), index_img)

    config = calib_config(map_path, camera_model, intrinsics, distortion)
    with open(os.path.join(dst_path, "calib.json"), "w") as f:
        f.write(json.dumps(config, indent=2, sort_keys=True) + "\n")  # nlohmann's std::map keeps keys sorted
    stats.update(map_points=int(cloud.shape[0]), filtered=int(filtered.shape[0]), lidar_fov=lidar_fov, virtual_camera=model,
                 voxel_grid=avg_stats, equalize=eq_stats, fov=fov_stats)
    return config


# ---- `preprocess` on the command line of the reference (src/vlcal/preprocess/preprocess.cpp:37-82) ----------------------

def build_parser():
    import argparse

    ap = argparse.ArgumentParser(prog="preprocess", description="calibration dataset from a directory of ROS 1 / ROS 2 (sqlite3) bags")
    ap.add_argument("data_path", nargs="?", help="directory that contains rosbags for calibration")
    ap.add_argument("dst_path", nargs="?", help="directory to save preprocessed data")
    ap.add_argument("--bag_id", type=int, help="specify the bag to use (just for evaluation)")
    ap.add_argument("--first_n_bags", type=int, help="use only the first N bags (just for evaluation)")
    ap.add_argument("-a", "--auto_topic", action="store_true", help="automatically select topics")
    ap.add_argument("-d", "--dynamic_lidar_integration", action="store_true", help="not supported: only the static integrator is implemented")
    ap.add_argument("-i", "--intensity_channel", default="auto", help="auto or channel name")
    ap.add_argument("--camera_info_topic")
    ap.add_argument("--image_topic")
    ap.add_argument("--points_topic")
    ap.add_argument("--camera_model", default="auto", help="auto, plumb_bob, fisheye(=equidistant), omnidir, or equirectangular")
    ap.add_argument("--camera_intrinsics", help="camera intrinsic parameters [fx,fy,cx,cy(,xi)] (don't put spaces between values!!)")
    ap.add_argument("--camera_distortion_coeffs", help="camera distortion parameters [k1,k2,p1,p2,k3] (don't put spaces between values!!)")
    ap.add_argument("--k_neighbors", type=int, default=20, help="used by the dynamic integrator only")
    ap.add_argument("--voxel_resolution", type=float, default=0.002, help="voxel grid resolution")
    ap.add_argument("--min_distance", type=float, default=1.0, help="minimum point distance. Points closer than this value will be discarded")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("-v", "--visualize", action="store_true", help="no viewer here: prints a note and continues")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: the current one)")
    return ap


def main(argv=None) -> int:
    """python -m direct_visual_lidar_calibration_b200.preprocess <data_path> <dst_path> [flags].  As in the reference, a
    missing path prints the usage and exits 0."""
    import sys

    from . import bag_io
    from . import preprocess_bag as PB

    ap = build_parser()
    args = ap.parse_args(argv)
    if args.data_path is None or args.dst_path is None:
        ap.print_help()
        return 0
    if args.dynamic_lidar_integration:
        bags = PB.list_bags(args.data_path) if os.path.isdir(args.data_path) else []
        names = ", ".join(os.path.basename(b) for b in bags) or args.data_path
        print(f"error: {names}: dynamic LiDAR integration (-d, CT-GICP odometry) is not supported; only the static integrator is",
              file=sys.stderr)
        return 1
    if args.visualize:
        print("note: there is no viewer (-v); continuing without it")
    print(f"data_path: {args.data_path}\ndst_path : {args.dst_path}")
    try:
        PB.preprocess_bags(args.data_path, args.dst_path, auto_topic=args.auto_topic, camera_info_topic=args.camera_info_topic,
                           image_topic=args.image_topic, points_topic=args.points_topic, intensity_channel=args.intensity_channel,
                           camera_model=args.camera_model, camera_intrinsics=args.camera_intrinsics,
                           camera_distortion_coeffs=args.camera_distortion_coeffs, voxel_resolution=args.voxel_resolution,
                           min_distance=args.min_distance, bag_id=args.bag_id, first_n_bags=args.first_n_bags, device=args.device)
    except (ValueError, FileNotFoundError, bag_io.BagError) as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    import sys

    sys.exit(main())
