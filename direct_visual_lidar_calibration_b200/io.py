"""On-disk formats either side of the hot path (SURVEY.md section 8f-3): what the reference's `preprocess` writes and what
`calibrate` reads / writes.

  <data_path>/<bag>.png   first camera image, grayscale uint8                       (preprocess.cpp:160-161, visual_lidar_data.cpp:13)
  <data_path>/<bag>.ply   binary PLY, float x y z + float intensity per vertex      (preprocess.cpp:163-169, visual_lidar_data.cpp:19-26)
  <data_path>/calib.json  camera.{camera_model,intrinsics,distortion_coeffs}, meta.bag_names,
                          results.{init_T_lidar_camera[_auto], T_lidar_camera} = [x y z qx qy qz qw] of T_lidar_camera
                          (preprocess.cpp:220-232, calibrate.cpp:38-45,57-76,128-140)
  <data_path>/<bag>_lidar_indices.png  int32 point-index map of the LiDAR image as 8UC4  (preprocess.cpp:205-211)
  <data_path>/<bag>_matches.json       kpts0 / kpts1 / matches / confidence  (find_matches_superglue.py:115-117)
The PLY writer/reader of the reference is Iridescence's glk::save_ply_binary / glk::load_ply (not vendored); the reader here
parses the header generically (binary little endian or ascii, any property order, float/double/int types)."""
from __future__ import annotations

import json
import os

import numpy as np

_PLY_TYPES = {
    "char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
    "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8",
}


def save_ply_binary(path: str, points_xyz, intensities=None, colors=None) -> None:
    """Binary little-endian PLY with float x, y, z (+ float intensity), the layout of preprocess.cpp:163-169.  colors:
    (N, 4) RGBA in [0, 1] (the viewer's coloured cloud), appended as uchar red green blue alpha = round(c * 255)."""
    pts = np.asarray(points_xyz, dtype=np.float32).reshape(-1, 3)
    cols = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if intensities is not None:
        cols.append(("intensity", "<f4"))
    if colors is not None:
        cols += [(name, "u1") for name in ("red", "green", "blue", "alpha")]
    rec = np.empty(pts.shape[0], dtype=cols)
    rec["x"], rec["y"], rec["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    if intensities is not None:
        rec["intensity"] = np.asarray(intensities, dtype=np.float32).reshape(-1)
    if colors is not None:
        rgba = np.rint(np.clip(np.asarray(colors, dtype=np.float64).reshape(-1, 4) * 255.0, 0.0, 255.0)).astype(np.uint8)
        rec["red"], rec["green"], rec["blue"], rec["alpha"] = rgba.T
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {pts.shape[0]}"]
    header += [f"property {'uchar' if t == 'u1' else 'float'} {name}" for name, t in cols]
    header.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(rec.tobytes())


def load_ply(path: str):
    """Returns (points float64 (N,3), intensities float64 (N,) or None).  Values are the file's floats widened to double,
    exactly what FrameCPU(ply->vertices) + add_intensities do (frame_cpu.cpp:79-86,127-132)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n_vertex, props, in_vertex = None, 0, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii", errors="replace").split()
            if not tok or tok[0] == "comment":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n_vertex = int(tok[2])
                elif props and n_vertex:
                    pass  # elements after the vertices are ignored
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties on vertices are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        names = [p[0] for p in props]
        if fmt == "ascii":
            data = np.loadtxt(f, max_rows=n_vertex, ndmin=2) if n_vertex else np.zeros((0, len(props)))
            col = {n: data[:, i] for i, n in enumerate(names)}
        elif fmt in ("binary_little_endian", "binary_big_endian"):
            order = "<" if fmt == "binary_little_endian" else ">"
            dt = np.dtype([(n, order + t) for n, t in props])
            rec = np.frombuffer(f.read(dt.itemsize * n_vertex), dtype=dt, count=n_vertex)
            col = {n: rec[n] for n in names}
        else:
            raise ValueError(f"{path}: unknown PLY format {fmt}")
    pts = np.stack([np.asarray(col[k], dtype=np.float64) for k in ("x", "y", "z")], axis=1)
    inten = np.asarray(col["intensity"], dtype=np.float64) if "intensity" in col else None
    return np.ascontiguousarray(pts), inten


# PCD TYPE/SIZE -> numpy type
_PCD_TYPES = {
    ("I", "1"): "i1", ("I", "2"): "i2", ("I", "4"): "i4", ("I", "8"): "i8",
    ("U", "1"): "u1", ("U", "2"): "u2", ("U", "4"): "u4", ("U", "8"): "u8",
    ("F", "4"): "f4", ("F", "8"): "f8",
}


def _read_pcd_fields(path: str):
    """PCD v0.7 (ascii or binary) -> [(name, numpy type, count, values (N, count))]."""
    with open(path, "rb") as f:
        head = {}
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PCD header")
            tok = line.decode("ascii", errors="replace").split()
            if not tok or tok[0].startswith("#"):
                continue
            head[tok[0].upper()] = tok[1:]
            if tok[0].upper() == "DATA":
                break
        for key in ("FIELDS", "SIZE", "TYPE"):
            if key not in head:
                raise ValueError(f"{path}: PCD header has no {key} line")
        names, sizes, types = head["FIELDS"], head["SIZE"], head["TYPE"]
        counts = [int(c) for c in head.get("COUNT", ["1"] * len(names))]
        if not (len(names) == len(sizes) == len(types) == len(counts)):
            raise ValueError(f"{path}: PCD FIELDS / SIZE / TYPE / COUNT lengths differ")
        if "POINTS" in head:
            n = int(head["POINTS"][0])
        else:
            n = int(head.get("WIDTH", ["0"])[0]) * int(head.get("HEIGHT", ["1"])[0])
        try:
            dtypes = [_PCD_TYPES[(t.upper(), s)] for t, s in zip(types, sizes)]
        except KeyError as e:
            raise ValueError(f"{path}: unknown PCD field type {e.args[0]}") from None
        data = head["DATA"][0].lower() if head["DATA"] else ""
        if data == "binary_compressed":
            raise ValueError(f"{path}: binary_compressed (LZF) PCD is not supported; save the map as binary or ascii PCD")
        widths = [max(c, 1) for c in counts]
        if data == "binary":
            dt = np.dtype([(f"f{i}", "<" + t, (w,)) for i, (t, w) in enumerate(zip(dtypes, widths))])
            raw = f.read(dt.itemsize * n)
            if len(raw) < dt.itemsize * n:
                raise ValueError(f"{path}: PCD data holds fewer than the {n} points its header declares")
            rec = np.frombuffer(raw, dtype=dt, count=n)
            cols = [rec[f"f{i}"].reshape(n, widths[i]) for i in range(len(names))]
        elif data == "ascii":
            total = sum(widths)
            vals = np.loadtxt(f, dtype=np.float64, max_rows=n, ndmin=2) if n else np.zeros((0, total))
            if vals.shape != (n, total):
                raise ValueError(f"{path}: ascii PCD data is {vals.shape[0]} x {vals.shape[1]}, the header declares {n} x {total}")
            cols, c0 = [], 0
            for t, w in zip(dtypes, widths):
                cols.append(vals[:, c0 : c0 + w].astype(t))
                c0 += w
        else:
            raise ValueError(f"{path}: unknown PCD DATA kind {data!r}")
    return [(nm, t, c, col) for nm, t, c, col in zip(names, dtypes, counts, cols)]


def _read_ply_fields(path: str):
    """PLY vertex properties (ascii or binary) -> [(name, numpy type, 1, values (N, 1))]."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n_vertex, props, elements, in_vertex = None, 0, [], [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii", errors="replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append(tok[1])
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n_vertex = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties on vertices are not supported")
                if tok[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY property type {tok[1]}")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if elements and elements[0] != "vertex":
            raise ValueError(f"{path}: the vertex element must come first")
        if fmt == "ascii":
            vals = np.loadtxt(f, dtype=np.float64, max_rows=n_vertex, ndmin=2) if n_vertex else np.zeros((0, len(props)))
            if vals.shape != (n_vertex, len(props)):
                raise ValueError(f"{path}: ascii PLY vertex data does not match its header")
            cols = [vals[:, i : i + 1].astype(t) for i, (_, t) in enumerate(props)]
        elif fmt in ("binary_little_endian", "binary_big_endian"):
            order = "<" if fmt == "binary_little_endian" else ">"
            dt = np.dtype([(f"p{i}", order + t) for i, (_, t) in enumerate(props)])
            raw = f.read(dt.itemsize * n_vertex)
            if len(raw) < dt.itemsize * n_vertex:
                raise ValueError(f"{path}: PLY data holds fewer than the {n_vertex} vertices its header declares")
            rec = np.frombuffer(raw, dtype=dt, count=n_vertex)
            cols = [rec[f"p{i}"].astype(t).reshape(n_vertex, 1) for i, (_, t) in enumerate(props)]
        else:
            raise ValueError(f"{path}: unknown PLY format {fmt}")
    return [(nm, t, 1, col) for (nm, t), col in zip(props, cols)]


def load_map_cloud(path: str, warn=print) -> np.ndarray:
    """pcl::io::load(path, PointCloud<PointXYZI>) for a map (preprocess_map.cpp:134), chosen by extension: .pcd (ascii or
    binary) or .ply (ascii or binary) -> float32 (N, 4) of x, y, z, intensity in file order.

    PCL copies a field into the point only when its name matches, its type is float32 and its count is 1; any other
    field keeps PointXYZI's default 0 and PCL warns.  Here an x, y or z that does not match (double coordinates, say) is
    refused, since PCL would silently give zeros; a missing or non-float32 intensity becomes 0 with a warning, as in
    PCL.  Non-finite coordinates or intensities are refused (the voxel filter and the sort are undefined on them), and
    so is binary_compressed PCD."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".pcd":
        fields = _read_pcd_fields(path)
    elif ext == ".ply":
        fields = _read_ply_fields(path)
    else:
        raise ValueError(f"{path}: unsupported map format {ext or '(no extension)'}; expected .pcd or .ply")
    n = fields[0][3].shape[0] if fields else 0
    out = np.zeros((n, 4), dtype=np.float32)
    for c, name in enumerate(("x", "y", "z", "intensity")):
        named = [fd for fd in fields if fd[0] == name]
        match = [fd for fd in named if fd[1] == "f4" and fd[2] in (0, 1)]  # pcl::FieldMatches
        if match:
            out[:, c] = match[0][3][:, 0]
        elif c < 3:
            got = f"{named[0][1]} x {named[0][2]}" if named else "missing"
            raise ValueError(f"{path}: field {name} must be float32 with count 1 (got {got}); PCL would silently load zeros for it")
        else:
            warn(f"warning: {path}: no float32 intensity field (got {'%s x %d' % named[0][1:3] if named else 'none'}); intensities are 0, as PCL loads them")
    if not np.all(np.isfinite(out)):
        bad = int((~np.isfinite(out).all(axis=1)).sum())
        raise ValueError(f"{path}: {bad} points have a non-finite coordinate or intensity")
    return out


def load_image_gray(path: str) -> np.ndarray:
    """cv::imread(path, 0)."""
    import cv2

    img = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
    if img is None:
        raise FileNotFoundError(f"failed to load {path}")
    return img


def load_visual_lidar_data(data_path: str, bag_name: str):
    """vlcal::VisualLiDARData(data_path, bag_name) (visual_lidar_data.cpp:10-27)."""
    from .cost import VisualLiDARData

    image = load_image_gray(os.path.join(data_path, bag_name + ".png"))
    pts, inten = load_ply(os.path.join(data_path, bag_name + ".ply"))
    if inten is None:
        raise ValueError(f"{bag_name}.ply has no intensity property")
    return VisualLiDARData(image, pts, inten)


def save_lidar_indices(path: str, index_image) -> None:
    """<bag>_lidar_indices.png: the int32 point-index map (-1 = no point) written as an 8UC4 PNG, the way preprocess does
    (preprocess.cpp:207-211).  cv2 swaps B and R on write and back on read, so the bytes round-trip exactly."""
    import cv2

    idx = np.ascontiguousarray(np.asarray(index_image, dtype="<i4"))
    if idx.ndim != 2:
        raise ValueError("index image must be H x W")
    if not cv2.imwrite(path, idx.view(np.uint8).reshape(idx.shape[0], idx.shape[1], 4)):
        raise OSError(f"failed to write {path}")


def load_lidar_indices(path: str) -> np.ndarray:
    """cv::imread(path, -1) reinterpreted as CV_32SC1 (initial_guess_auto.cpp:82-83) -> int32 (H, W)."""
    import cv2

    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(f"failed to load {path}")
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 4:
        raise ValueError(f"{path}: expected an 8-bit 4-channel PNG (the int32 point-index map), got {img.dtype} {img.shape}")
    return np.ascontiguousarray(img).view("<i4").reshape(img.shape[0], img.shape[1]).astype(np.int32)


def _json_ints(values, name: str) -> np.ndarray:
    """std::vector<int> from a JSON number array: nlohmann converts each number with static_cast<int> (truncation)."""
    a = np.trunc(np.asarray(values, dtype=np.float64).reshape(-1))
    if not np.all(np.isfinite(a)) or np.any(np.abs(a) > 2**31 - 1):
        raise ValueError(f"{name}: values must be finite and fit in int32")
    return a.astype(np.int64)


def load_matches(path: str) -> dict:
    """<bag>_matches.json of find_matches_superglue.py (:115-117): flat kpts0 / kpts1 lists of x, y pairs, matches (index into
    kpts1 or -1 per kpts0 entry), confidence.  Keypoints and matches come back as the reference reads them: truncated ints."""
    with open(path) as f:
        m = json.load(f)
    kpts0, kpts1, matches = (_json_ints(m[k], k) for k in ("kpts0", "kpts1", "matches"))
    if kpts0.size % 2 or kpts1.size % 2 or matches.size != kpts0.size // 2:
        raise ValueError(f"{path}: kpts0 / kpts1 must hold x, y pairs and matches one entry per kpts0 keypoint")
    return {"kpts0": kpts0.reshape(-1, 2), "kpts1": kpts1.reshape(-1, 2), "matches": matches, "confidence": np.asarray(m.get("confidence", []), dtype=np.float64)}


# the 8 neighbours of a keypoint, nearest first (initial_guess_auto.cpp:35-43)
_PICK_OFFSETS = [(dx, dy) for dx in (-1, 0, 1) for dy in (-1, 0, 1) if (dx, dy) != (0, 0)]
_PICK_OFFSETS.sort(key=lambda o: o[0] * o[0] + o[1] * o[1])


def read_correspondences(data_path: str, bag_name: str, points):
    """InitialGuessAuto::read_correspondences (initial_guess_auto.cpp:81-125) -> (kp0 float64 (K,2), points float64 (K,3)).

    A match is used when matches[i] >= 0 and the LiDAR-image keypoint kpts1[matches[i]] lies on a pixel with a point; the 3-D
    point is points[index] of the bag's full cloud, the 2-D point the truncated camera keypoint.  Where the pixel is blank the
    reference searches the 8 neighbours but then skips the match whatever it found (the found index is never used); that
    behaviour is kept on purpose, so results match the reference's, with its warning when no neighbour has a point either.
    Unlike the reference, a kpts1 keypoint outside the index image, a match index past kpts1 or a point index past the cloud
    is an error instead of an out-of-bounds read."""
    pts = np.asarray(points, dtype=np.float64)
    index_image = load_lidar_indices(os.path.join(data_path, bag_name + "_lidar_indices.png"))
    m = load_matches(os.path.join(data_path, bag_name + "_matches.json"))
    H, W = index_image.shape
    kp0_out, pt_out = [], []
    for i, match in enumerate(m["matches"]):
        if match < 0:
            continue
        if match >= m["kpts1"].shape[0]:
            raise ValueError(f"{bag_name}_matches.json: matches[{i}] = {match} is past the {m['kpts1'].shape[0]} kpts1 keypoints")
        x, y = (int(v) for v in m["kpts1"][match])
        if not (0 <= x < W and 0 <= y < H):
            raise ValueError(f"{bag_name}_matches.json: kpts1[{match}] = ({x}, {y}) is outside the {W}x{H} LiDAR index image")
        index = int(index_image[y, x])
        if index < 0:
            found = any(0 <= x + dx < W and 0 <= y + dy < H and index_image[y + dy, x + dx] >= 0 for dx, dy in _PICK_OFFSETS)
            if not found:
                print("warning: ignore keypoint in a blank region!!")
            continue
        if index >= pts.shape[0]:
            raise ValueError(f"{bag_name}_lidar_indices.png: point index {index} at ({x}, {y}) is past the {pts.shape[0]} points of {bag_name}.ply")
        kp0_out.append(m["kpts0"][i].astype(np.float64))
        pt_out.append(pts[index, :3])
    return np.array(kp0_out, dtype=np.float64).reshape(-1, 2), np.array(pt_out, dtype=np.float64).reshape(-1, 3)


def load_calib_json(data_path: str) -> dict:
    with open(os.path.join(data_path, "calib.json")) as f:
        return json.load(f)


def save_calib_json(data_path: str, config: dict) -> None:
    with open(os.path.join(data_path, "calib.json"), "w") as f:
        f.write(json.dumps(config, indent=2) + "\n")  # config.dump(2) << std::endl  (calibrate.cpp:140)


# ---- pose <-> [x y z qx qy qz qw] (TUM order) of T_lidar_camera -------------------------------------------------------

def quat_to_matrix(qx, qy, qz, qw) -> np.ndarray:
    """Eigen::Quaterniond(w,x,y,z).normalized().toRotationMatrix() (calibrate.cpp:72)."""
    q = np.array([qx, qy, qz, qw], dtype=np.float64)
    q = q / np.linalg.norm(q)
    x, y, z, w = q
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)],
    ])


def matrix_to_quat(R) -> np.ndarray:
    """Eigen::Quaterniond(Matrix3d) -> (x, y, z, w)."""
    R = np.asarray(R, dtype=np.float64)
    t = np.trace(R)
    q = np.empty(4)
    if t > 0:
        s = np.sqrt(t + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[0], q[1], q[2] = (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (R[k, j] - R[j, k]) * s
        q[j] = (R[j, i] + R[i, j]) * s
        q[k] = (R[k, i] + R[i, k]) * s
    return q


def tum_to_T(values) -> np.ndarray:
    T = np.eye(4)
    T[:3, 3] = values[0:3]
    T[:3, :3] = quat_to_matrix(values[3], values[4], values[5], values[6])
    return T


def T_to_tum(T) -> list:
    q = matrix_to_quat(np.asarray(T)[:3, :3])
    t = np.asarray(T)[:3, 3]
    return [float(t[0]), float(t[1]), float(t[2]), float(q[0]), float(q[1]), float(q[2]), float(q[3])]


def invert_isometry(T) -> np.ndarray:
    T = np.asarray(T, dtype=np.float64)
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out
