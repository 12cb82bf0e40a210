"""Coarse pose-grid initial guess (BASELINE.json config 5; SURVEY.md section 8f-4).

The reference's `initial_guess_auto` needs SuperGlue 2D-3D matches (src/initial_guess_auto.cpp:113-139); with the batched
NID kernel a brute-force alternative becomes cheap: score an SE(3) grid around a rough pose (8 poses per pass over the
cloud), keep the best few, optionally refine each with the Nelder-Mead inner solve.  There is no reference behaviour to
match here beyond the per-pose NID values, which are the ones of CostCalculatorNID::calculate.

Pose sharding over GPUs (axis ii of SURVEY 8e): rank r scores poses r, r+G, ... on its replica of the cloud; the scores
are gathered on the host side -- no collective on the data path."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .cost import CostCalculatorNID


def pose_grid(T_center: np.ndarray, n_rot=(8, 8, 8), n_trans=(2, 4, 4), rot_half_deg: float = 4.0, trans_half: float = 0.10) -> np.ndarray:
    """T_center * Exp(rot, trans) over a regular grid: prod(n_rot) * prod(n_trans) poses, (P, 4, 4)."""
    from .synthetic import perturb

    axes_r = [np.linspace(-rot_half_deg, rot_half_deg, k) if k > 1 else np.zeros(1) for k in n_rot]
    axes_t = [np.linspace(-trans_half, trans_half, k) if k > 1 else np.zeros(1) for k in n_trans]
    out = []
    for rx in axes_r[0]:
        for ry in axes_r[1]:
            for rz in axes_r[2]:
                for tx in axes_t[0]:
                    for ty in axes_t[1]:
                        for tz in axes_t[2]:
                            out.append(perturb(T_center, (rx, ry, rz), (tx, ty, tz)))
    return np.stack(out)


def score_poses(cost: CostCalculatorNID, poses: np.ndarray, rank: int = 0, world: int = 1) -> np.ndarray:
    """NID of every pose.  One persistent launch scores this rank's whole share of the list (vlcal_nid_score_poses);
    with world > 1 rank r scores poses[r::world] and the full vector is assembled with one all_gather of the device
    tensors (NCCL) -- the only exchange of the whole search."""
    from .cost import score_poses as _score

    mine = poses[rank::world]
    vals = _score([cost], mine) if len(mine) else np.zeros(0)
    if world == 1:
        return vals
    import torch
    import torch.distributed as dist

    per = (len(poses) + world - 1) // world  # ranks at the tail may hold one pose less: pad to a common length
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    local = torch.full((per,), float("nan"), dtype=torch.float64, device=dev)
    local[: len(vals)] = torch.from_numpy(vals).to(dev)
    parts = torch.empty((world, per), dtype=torch.float64, device=dev)
    dist.all_gather_into_tensor(parts, local)
    parts = parts.cpu().numpy()
    full = np.empty(len(poses))
    for r in range(world):
        k = len(poses[r::world])
        full[r::world] = parts[r, :k]
    return full


def sweep_poses(costs, poses: np.ndarray, return_hist: bool = False, kernel_only: bool = False):
    """score_poses for very long lists on small clouds: the pose-parallel sweep kernel (vlcal_nid_sweep_poses), same
    scores bit for bit.  return_hist: also the joint histograms of costs[0], [P, image_bin, lidar_bin].  kernel_only: the
    sweep kernel even beyond the cloud size where the entry point hands over to the persistent kernel (measurements)."""
    from . import _lib
    from .camera import _dp
    from .cost import T_to_colmajor

    Tc = T_to_colmajor(poses)
    P = Tc.shape[0]
    out = np.empty(P)
    bins = costs[0].params.bins
    hist = np.empty((P, bins * bins), dtype=np.int32) if return_hist else None
    handles = (C.c_void_p * len(costs))(*[c.handle for c in costs])
    L = _lib.load_library()
    fn = L.vlcal_nid_debug_sweep_kernel if kernel_only else L.vlcal_nid_sweep_poses
    _lib.check(fn(handles, len(costs), _dp(Tc), P, _dp(out), hist.ctypes.data if return_hist else None))
    if return_hist:
        return out, np.swapaxes(hist.reshape(P, bins, bins), 1, 2).copy()
    return out


# ---- search sets: pose lists described by small tables (vlcal_search_set) ----------------------------------------------------

class SearchSet:
    """Pose i = (ib * n_left + il) * n_offset + io of the set is T_camera_lidar = [R | R (center[ib] + offset[io])] with
    R = left[il] @ base[ib]; `indices` selects a subset.  With center = -(camera position in the LiDAR frame) the offsets
    move the camera position and leave the rotation alone.  poses() evaluates this on the host with the operations, and
    in the order, the device generator uses -- one IEEE rounding per product and per sum -- so both give the same bits."""

    def __init__(self, left, base, center, offset, indices=None):
        self.left = np.ascontiguousarray(np.asarray(left, dtype=np.float64).reshape(-1, 3, 3))
        self.base = np.ascontiguousarray(np.asarray(base, dtype=np.float64).reshape(-1, 3, 3))
        self.center = np.ascontiguousarray(np.asarray(center, dtype=np.float64).reshape(-1, 3))
        self.offset = np.ascontiguousarray(np.asarray(offset, dtype=np.float64).reshape(-1, 3))
        if self.center.shape[0] != self.base.shape[0]:
            raise ValueError("one center per base rotation")
        full = self.left.shape[0] * self.base.shape[0] * self.offset.shape[0]
        if full >= 2**31:
            raise ValueError("a search set holds fewer than 2^31 combinations")
        self.indices = None if indices is None else np.ascontiguousarray(np.asarray(indices, dtype=np.int32).reshape(-1))
        if self.indices is not None and self.indices.size and (self.indices.min() < 0 or self.indices.max() >= full):
            raise ValueError("index out of range")
        self.n_poses = full if self.indices is None else int(self.indices.size)

    def split(self, flat=None):
        """(ib, il, io) of the given flat indices (default: of every pose of the set)."""
        i = (np.arange(self.n_poses, dtype=np.int64) if self.indices is None else self.indices.astype(np.int64)) if flat is None else np.asarray(flat, dtype=np.int64)
        n_l, n_o = self.left.shape[0], self.offset.shape[0]
        return i // (n_o * n_l), (i // n_o) % n_l, i % n_o

    def rotations(self, ib, il) -> np.ndarray:
        L, B = self.left[il], self.base[ib]
        R = np.empty((L.shape[0], 3, 3))
        for r in range(3):
            for c in range(3):
                R[:, r, c] = (L[:, r, 0] * B[:, 0, c] + L[:, r, 1] * B[:, 1, c]) + L[:, r, 2] * B[:, 2, c]
        return R

    def poses(self, which=None) -> np.ndarray:
        """(P, 4, 4) T_camera_lidar of the set's poses, or of the poses at positions `which` of the set."""
        flat = None
        if which is not None:
            which = np.asarray(which, dtype=np.int64)
            flat = which if self.indices is None else self.indices[which].astype(np.int64)
        ib, il, io = self.split(flat)
        R = self.rotations(ib, il)
        v = self.center[ib] + self.offset[io]
        T = np.zeros((R.shape[0], 4, 4))
        T[:, :3, :3] = R
        for r in range(3):
            T[:, r, 3] = (R[:, r, 0] * v[:, 0] + R[:, r, 1] * v[:, 1]) + R[:, r, 2] * v[:, 2]
        T[:, 3, 3] = 1.0
        return T

    def as_struct(self):
        """The vlcal_search_set view of the tables (which stay owned by this object)."""
        from . import _lib

        dp = C.POINTER(C.c_double)
        s = _lib.SearchSet()
        s.left, s.base = self.left.ctypes.data_as(dp), self.base.ctypes.data_as(dp)
        s.center, s.offset = self.center.ctypes.data_as(dp), self.offset.ctypes.data_as(dp)
        s.indices = self.indices.ctypes.data_as(C.POINTER(C.c_int32)) if self.indices is not None else None
        s.n_left, s.n_base, s.n_offset = self.left.shape[0], self.base.shape[0], self.offset.shape[0]
        s.n_poses = self.n_poses
        return s

    def device_poses(self, device: int = -1) -> np.ndarray:
        """(P, 4, 4): the poses as the device generates them (test hook for the agreement with poses())."""
        from . import _lib
        from .camera import _dp
        from .cost import colmajor_to_T

        out = np.empty((self.n_poses, 16))
        s = self.as_struct()
        _lib.check(_lib.load_library().vlcal_search_set_poses(device, C.byref(s), _dp(out)))
        return colmajor_to_T(out)


def sweep_search_set(costs, sset: SearchSet):
    """(scores, inliers, kernel_ms): sum over the cost objects of calculate(T), and of the points it counted, for every pose
    of the set, generated on the device."""
    from . import _lib
    from .camera import _dp

    out = np.empty(sset.n_poses)
    handles = (C.c_void_p * len(costs))(*[c.handle for c in costs])
    s = sset.as_struct()
    L = _lib.load_library()
    inliers = np.empty(sset.n_poses, dtype=np.int64)
    _lib.check(L.vlcal_nid_sweep_search_set_inliers(handles, len(costs), C.byref(s), _dp(out), inliers.ctypes.data_as(C.POINTER(C.c_int64))))
    return out, inliers, float(L.vlcal_nid_sweep_last_kernel_ms())


def rotation_angle_deg(Ra, Rb) -> np.ndarray:
    """Angle of Ra Rb^T in degrees; broadcasts over leading dimensions."""
    tr = np.einsum("...ij,...ij->...", np.asarray(Ra), np.asarray(Rb))
    return np.degrees(np.arccos(np.clip((tr - 1.0) / 2.0, -1.0, 1.0)))


def _rodrigues(w: np.ndarray) -> np.ndarray:
    th = float(np.linalg.norm(w))
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + W
    return np.eye(3) + (np.sin(th) / th) * W + ((1 - np.cos(th)) / th**2) * (W @ W)


def rotation_set_counts(step_deg: float):
    """(optical-axis directions, roll angles) of the level-0 rotation set: ceil(4 pi / d^2) x ceil(2 pi / d)."""
    d = np.radians(step_deg)
    return int(np.ceil(4.0 * np.pi / d**2)), int(np.ceil(2.0 * np.pi / d))


def rotation_set(step_deg: float, prior_T_lidar_camera=None, rot_range_deg: float = 180.0) -> SearchSet:
    """Near-uniform cover of SO(3) as S^2 x S^1: a Fibonacci lattice of LiDAR-frame directions for the camera's optical
    axis x equally spaced rolls about it.  base[k] turns direction k into the camera's +z (rows: e_phi, -e_theta, e_r of
    the direction's spherical frame), left[j] is the roll Rz(2 pi j / n_roll).  With a prior only the rotations within
    rot_range_deg of the prior's are kept; the camera position is the prior's (default: the LiDAR origin)."""
    n_dir, n_roll = rotation_set_counts(step_deg)
    k = np.arange(n_dir, dtype=np.float64)
    z = 1.0 - (2.0 * k + 1.0) / n_dir
    phi = k * (np.pi * (3.0 - np.sqrt(5.0)))  # golden angle
    st = np.sqrt((1.0 - z) * (1.0 + z))
    cp, sp = np.cos(phi), np.sin(phi)
    base = np.zeros((n_dir, 3, 3))
    base[:, 0, 0], base[:, 0, 1] = -sp, cp
    base[:, 1, 0], base[:, 1, 1], base[:, 1, 2] = -z * cp, -z * sp, st
    base[:, 2, 0], base[:, 2, 1], base[:, 2, 2] = st * cp, st * sp, z
    roll = 2.0 * np.pi * np.arange(n_roll, dtype=np.float64) / n_roll
    left = np.zeros((n_roll, 3, 3))
    left[:, 0, 0], left[:, 0, 1], left[:, 1, 0], left[:, 1, 1], left[:, 2, 2] = np.cos(roll), -np.sin(roll), np.sin(roll), np.cos(roll), 1.0
    position = np.zeros(3) if prior_T_lidar_camera is None else np.asarray(prior_T_lidar_camera, dtype=np.float64)[:3, 3]
    center = np.tile(-position, (n_dir, 1))
    full = SearchSet(left, base, center, np.zeros((1, 3)))
    if prior_T_lidar_camera is None or rot_range_deg >= 180.0:
        return full
    R_prior = np.asarray(prior_T_lidar_camera, dtype=np.float64)[:3, :3].T  # R_camera_lidar
    keep = []
    per = max(1, (1 << 18) // n_roll)
    for b0 in range(0, n_dir, per):  # in slabs of base rotations: the whole list of matrices is never held at once
        ib = np.repeat(np.arange(b0, min(n_dir, b0 + per)), n_roll)
        il = np.tile(np.arange(n_roll), ib.size // n_roll)
        inside = rotation_angle_deg(full.rotations(ib, il), R_prior) <= rot_range_deg
        keep.append((ib * n_roll + il)[inside])
    return SearchSet(left, base, center, np.zeros((1, 3)), indices=np.concatenate(keep))


def local_set(candidates: np.ndarray, step_deg: float, trans_spacing: float, trans_half_steps: int) -> SearchSet:
    """Around every candidate T_camera_lidar: a 3x3x3 grid of rotations Exp((i, j, k) step) applied on the camera side x
    a (2 h + 1)^3 grid of camera positions (LiDAR frame) at trans_spacing."""
    candidates = np.asarray(candidates, dtype=np.float64).reshape(-1, 4, 4)
    d = np.radians(step_deg)
    g = (-1.0, 0.0, 1.0)
    left = np.stack([_rodrigues(np.array([i, j, k]) * d) for i in g for j in g for k in g])
    h = np.arange(-trans_half_steps, trans_half_steps + 1, dtype=np.float64) * trans_spacing
    offset = np.stack([np.array([x, y, z]) for x in h for y in h for z in h])
    base = candidates[:, :3, :3]
    center = np.einsum("nji,nj->ni", base, candidates[:, :3, 3])  # R^T t = -(camera position in the LiDAR frame)
    return SearchSet(left, base, center, offset)


def nms_top_k(poses_of, scores: np.ndarray, keep: int, min_sep_deg: float):
    """Positions of the best `keep` poses such that no two lie within min_sep_deg (rotation angle) of each other: greedy
    in ascending score, ties in list order, NaN (no inliers) last.  poses_of(positions) -> (n, 4, 4)."""
    scores = np.asarray(scores, dtype=np.float64)
    order = np.argsort(np.where(np.isnan(scores), np.inf, scores), kind="stable")
    kept, kept_R = [], np.empty((0, 3, 3))
    block = 256
    for s in range(0, order.size, block):
        if len(kept) >= keep:
            break
        cand = order[s : s + block]
        R = poses_of(cand)[:, :3, :3]
        for j, pos in enumerate(cand):
            if kept_R.shape[0] and rotation_angle_deg(kept_R, R[j]).min() <= min_sep_deg:
                continue
            kept.append(int(pos))
            kept_R = np.concatenate([kept_R, R[j : j + 1]])
            if len(kept) >= keep:
                break
    return np.asarray(kept, dtype=np.int64)


# ---- level data: image and cloud pyramids ------------------------------------------------------------------------------------

def box_halve(image: np.ndarray) -> np.ndarray:
    """2x2 box means of a uint8 image, rounded half up; an odd last row / column is cropped."""
    h, w = image.shape[0] // 2 * 2, image.shape[1] // 2 * 2
    a = image[:h, :w].astype(np.uint16)
    return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)


def pyramid_image(image: np.ndarray, scale: int) -> np.ndarray:
    """The image at 1 / scale (a power of two): box_halve log2(scale) times, then cv::equalizeHist as preprocess applies
    it to the full-resolution image."""
    import cv2

    if scale < 1 or scale & (scale - 1):
        raise ValueError("scale must be a power of two")
    out = np.ascontiguousarray(image, dtype=np.uint8)
    if scale == 1:
        return out
    while scale > 1:
        out = box_halve(out)
        scale //= 2
    return cv2.equalizeHist(out)


def pyramid_intrinsics(camera_model: str, intrinsics, scale: int) -> list:
    """fx, fy, cx, cy (equirectangular: W, H) divided by scale; any further parameter unchanged."""
    intr = [float(v) for v in intrinsics]
    n = 2 if camera_model == "equirectangular" else 4
    return [v / scale for v in intr[:n]] + intr[n:]


def cloud_subset(n_cloud: int, n_keep: int, seed: int) -> np.ndarray:
    """Indices of a seeded subset of n_keep points (capped at the cloud): the head of one seeded permutation, so the
    subsets of a bag are nested."""
    return np.random.default_rng(seed).permutation(n_cloud)[: min(n_cloud, n_keep)]


def grid_search(cost: CostCalculatorNID, T_center: np.ndarray, top_k: int = 5, rank: int = 0, world: int = 1, **grid_kwargs):
    """Returns (poses[top_k], nid[top_k]) of the best grid poses (NaN scores -- no inliers -- rank last)."""
    poses = pose_grid(T_center, **grid_kwargs)
    nid = score_poses(cost, poses, rank, world)
    order = np.argsort(np.where(np.isnan(nid), np.inf, nid), kind="stable")[:top_k]
    return poses[order], nid[order]
