"""ctypes wrapper of tests/cpp/pose_oracle.c, the CPU checker of PoseEstimation (built on first use into a temporary
directory, linked against the CPU oracle)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        O.build()
        oracle_so = O._LIB_PATH
        out = os.path.join(tempfile.mkdtemp(prefix="pose_oracle_"), "libpose_oracle.so")
        subprocess.run(
            ["/usr/bin/gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", f"-I{os.path.join(_ROOT, 'oracle')}",
             "-o", out, os.path.join(_HERE, "cpp", "pose_oracle.c"), oracle_so, f"-Wl,-rpath,{os.path.dirname(oracle_so)}", "-lm"],
            check=True,
        )
        O.lib()  # the oracle's symbols first, so that the two share one copy
        L = C.CDLL(out)
        cam, dp, vp = C.POINTER(O.Camera), C.POINTER(C.c_double), C.c_void_p
        L.pose_oracle_direction.argtypes = [cam, dp, dp]
        L.pose_oracle_bearings.argtypes = [cam, dp, dp, C.c_int, dp, dp]
        L.pose_oracle_score.argtypes = [cam, dp, dp, dp, C.c_int, vp, C.c_int, C.c_double, vp, vp, vp]
        L.pose_oracle_rotation.argtypes = [dp, dp, dp, dp, dp]
        L.pose_oracle_rotation.restype = C.c_int
        L.pose_oracle_errors.argtypes = [cam, dp, dp, dp, C.c_int, dp]
        L.pose_oracle_correspondences.argtypes = [vp, C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, dp, C.c_int64, vp, vp, C.POINTER(C.c_int)]
        _lib = L
    return _lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def bearings(cam, kp0, points):
    """-> (camera bearings (M,3), LiDAR bearings (M,3))"""
    kp = np.ascontiguousarray(kp0, dtype=np.float64)
    pts = np.ascontiguousarray(np.asarray(points, dtype=np.float64)[:, :3])
    dc, dl = np.empty((kp.shape[0], 3)), np.empty((kp.shape[0], 3))
    lib().pose_oracle_bearings(C.byref(cam), _dp(kp), _dp(pts), kp.shape[0], _dp(dc), _dp(dl))
    return dc, dl


def score(cam, kp0, points, pairs, thresh):
    """-> (counts, degenerate, near-threshold counts) per hypothesis"""
    kp = np.ascontiguousarray(kp0, dtype=np.float64)
    dc, dl = bearings(cam, kp, points)
    return score_bearings(cam, kp, dc, dl, pairs, thresh)


def score_bearings(cam, kp0, dc, dl, pairs, thresh):
    """score() on bearings computed once with bearings()"""
    kp = np.ascontiguousarray(kp0, dtype=np.float64)
    dc, dl = np.ascontiguousarray(dc, dtype=np.float64), np.ascontiguousarray(dl, dtype=np.float64)
    pr = np.ascontiguousarray(pairs, dtype=np.int32)
    h = pr.shape[0]
    counts, degenerate, near = np.empty(h, np.int32), np.empty(h, np.uint8), np.empty(h, np.int32)
    lib().pose_oracle_score(C.byref(cam), _dp(kp), _dp(dc), _dp(dl), kp.shape[0], pr.ctypes.data, h, float(thresh), counts.ctypes.data, degenerate.ctypes.data, near.ctypes.data)
    return counts, degenerate.astype(bool), near


def rotation(c1, c2, l1, l2):
    """The kernel's rotation R (3x3, c_k = R l_k) of one hypothesis from its two bearing pairs, or None where the pair is
    degenerate."""
    v = [np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(3)) for x in (c1, c2, l1, l2)]
    R = np.empty(9)
    ok = lib().pose_oracle_rotation(*[_dp(x) for x in v], _dp(R))
    return R.reshape(3, 3) if ok else None


def pair_rotation(dc, dl, pair):
    """rotation() of the index pair (i, j) of bearings (M,3); None where the RANSAC rule calls it degenerate (i == j too)."""
    i, j = int(pair[0]), int(pair[1])
    return None if i == j else rotation(dc[i], dc[j], dl[i], dl[j])


def errors(cam, R, kp0, dl):
    """-> e (M,): |kp0_j - project(R dl_j)|^2 in the kernel's order; correspondence j is an inlier iff e[j] < pow(thresh, 2)."""
    kp = np.ascontiguousarray(kp0, dtype=np.float64)
    d = np.ascontiguousarray(dl, dtype=np.float64)
    Rf = np.ascontiguousarray(np.asarray(R, dtype=np.float64).reshape(9))
    e = np.empty(kp.shape[0])
    lib().pose_oracle_errors(C.byref(cam), _dp(Rf), _dp(kp), _dp(d), kp.shape[0], _dp(e))
    return e


def correspondences(index_image, kpts0, kpts1, matches, n_points):
    """-> (used kpts0 indices, point indices, blank warnings); raises ValueError where the loader must reject the input"""
    idx = np.ascontiguousarray(index_image, dtype=np.int32)
    k0 = np.ascontiguousarray(np.asarray(kpts0, dtype=np.float64).reshape(-1))
    k1 = np.ascontiguousarray(np.asarray(kpts1, dtype=np.float64).reshape(-1))
    mt = np.ascontiguousarray(np.asarray(matches, dtype=np.float64).reshape(-1))
    kp_out, pt_out = np.empty(max(mt.size, 1), np.int32), np.empty(max(mt.size, 1), np.int32)
    warn = C.c_int()
    n = lib().pose_oracle_correspondences(idx.ctypes.data, idx.shape[1], idx.shape[0], _dp(k0), mt.size, _dp(k1), k1.size // 2, _dp(mt), int(n_points),
                                          kp_out.ctypes.data, pt_out.ctypes.data, C.byref(warn))
    if n < 0:
        raise ValueError({-1: "match index past kpts1", -2: "kpts1 keypoint outside the image", -3: "point index past the cloud"}[n])
    return kp_out[:n], pt_out[:n], warn.value
