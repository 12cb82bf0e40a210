"""`preprocess_map` on the command line of the reference (src/preprocess_map.cpp).

    python -m direct_visual_lidar_calibration_b200.preprocess_map --map_path MAP --image_path IMAGE --dst_path DST
        --camera_model MODEL --camera_intrinsics fx,fy,cx,cy --camera_distortion_coeffs k1,k2,p1,p2,k3
        [--voxel_resolution 0.002] [--min_distance 1.0] [--device D]

Builds a calibration dataset (000000.png / .ply / _lidar_intensities.png / _lidar_indices.png, calib.json) from a dense
map (PCD or PLY) and one camera image; initial_guess_auto and calibrate then run on it.  As in the reference, a missing
required flag prints the usage and exits 0, and --min_distance is accepted but has no effect.  No viewer (-v).
A list that starts with a minus sign is passed as --camera_distortion_coeffs=-0.04,0.08,... ."""
from __future__ import annotations

import argparse
import sys

REQUIRED = ("map_path", "image_path", "dst_path", "camera_model", "camera_intrinsics", "camera_distortion_coeffs")


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="preprocess_map")
    ap.add_argument("--map_path", help="path to input point cloud map (PCD or PLY)")
    ap.add_argument("--image_path", help="path to input image (PNG or JPG)")
    ap.add_argument("--dst_path", help="directory to save preprocessed data")
    ap.add_argument("--camera_model", help="atan, plumb_bob, fisheye, omnidir, or equirectangular")
    ap.add_argument("--camera_intrinsics", help="camera intrinsic parameters [fx,fy,cx,cy(,xi)] (don't put spaces between values!!)")
    ap.add_argument("--camera_distortion_coeffs", help="camera distortion parameters [k1,k2,p1,p2,k3] (don't put spaces between values!!)")
    ap.add_argument("--voxel_resolution", type=float, default=0.002, help="voxel grid resolution")
    ap.add_argument("--min_distance", type=float, default=None, help="accepted for compatibility; has no effect (default 1.0)")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: the current one)")
    return ap


def main(argv=None) -> int:
    ap = build_parser()
    args = ap.parse_args(argv)
    if any(getattr(args, k) is None for k in REQUIRED):
        ap.print_help()
        return 0
    if args.min_distance is not None:
        print("warning: --min_distance has no effect: preprocess_map keeps every point of the map, as the reference does")
    from .preprocess import parse_values, preprocess_map

    try:
        intrinsics = parse_values(args.camera_intrinsics, "camera_intrinsics")
        distortion = parse_values(args.camera_distortion_coeffs, "camera_distortion_coeffs")
        preprocess_map(args.map_path, args.image_path, args.dst_path, args.camera_model, intrinsics, distortion, args.voxel_resolution, device=args.device)
    except (ValueError, FileNotFoundError) as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
