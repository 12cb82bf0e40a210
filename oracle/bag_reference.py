"""ctypes binding of oracle/_ref/libvlcal_bag_ref.so -- the REFERENCE's own extract_raw_points, TimeKeeper and static
integrator, compiled from a reference checkout against oracle/ref_standin_bag/ (oracle/bag_ref_shim.cpp,
`make -C oracle -f bag_ref.mk ref REF=<checkout>`, or build() with VLCAL_REFERENCE=<checkout> in the environment).

TEST INFRASTRUCTURE ONLY: tests/golden/make_reference_bag_outputs.py records what it returns on the test scans
(tests/golden/reference_bag_outputs.json), which tests/test_bag_reference_pin.py holds the bag checker to."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libvlcal_bag_ref.so")
REFERENCE_ROOT = os.environ.get("VLCAL_REFERENCE", "")
_lib = None


def build() -> str | None:
    if REFERENCE_ROOT and os.path.isdir(os.path.join(REFERENCE_ROOT, "src")):
        subprocess.run(["make", "-C", _HERE, "-s", "-f", "bag_ref.mk", "ref", f"REF={REFERENCE_ROOT}"], check=True)
    return LIB_PATH if os.path.exists(LIB_PATH) else None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        vp, i64p = C.c_void_p, C.POINTER(C.c_int64)
        L.bagref_extract.restype = C.c_int
        L.bagref_extract.argtypes = [vp, C.c_int64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_char_p), vp, vp, C.c_char_p, C.c_uint32,
                                     C.c_uint32, vp, vp, i64p, vp, i64p, C.POINTER(C.c_double)]
        L.bagref_time_keeper.restype = None
        L.bagref_time_keeper.argtypes = [C.c_int, vp, vp, vp, vp, vp]
        L.bagref_integrate.restype = C.c_int64
        L.bagref_integrate.argtypes = [C.c_int, vp, vp, vp, C.c_double, C.c_double, vp]
        _lib = L
    return _lib


def extract(data: bytes, width, height, point_step, fields, intensity_channel, sec=0, nsec=0):
    """fields: [(name, offset, datatype)] -> None (nullptr) or dict(points (n, 4), intensities, times, stamp)."""
    n = max(width * height, 0)
    buf = np.frombuffer(bytes(data) + b"\0", np.uint8)
    names = (C.c_char_p * max(len(fields), 1))(*[f[0].encode() for f in fields])
    offs = np.array([f[1] for f in fields] or [0], np.uint32)
    types = np.array([f[2] for f in fields] or [0], np.uint8)
    pts, inten, times = np.zeros((max(n, 1), 4)), np.zeros(max(n, 1)), np.zeros(max(n, 1))
    ni, nt, stamp = C.c_int64(), C.c_int64(), C.c_double()
    ok = lib().bagref_extract(buf.ctypes.data, len(data), width, height, point_step, len(fields), names, offs.ctypes.data, types.ctypes.data,
                              intensity_channel.encode(), sec, nsec, pts.ctypes.data, inten.ctypes.data, C.byref(ni), times.ctypes.data, C.byref(nt),
                              C.byref(stamp))
    if not ok:
        return None
    return {"points": pts[:n], "intensities": inten[: ni.value], "times": times[: nt.value], "stamp": stamp.value}


def time_keeper(frames):
    """frames: [(stamp, n_points, times array)] -> [accepted]"""
    stamps = np.array([f[0] for f in frames], np.float64)
    npts = np.array([f[1] for f in frames], np.int64)
    first = np.concatenate([[0], np.cumsum([len(f[2]) for f in frames])]).astype(np.int64)
    times = np.concatenate([np.asarray(f[2], np.float64) for f in frames] + [np.zeros(1)])
    acc = np.zeros(len(frames), np.int32)
    lib().bagref_time_keeper(len(frames), stamps.ctypes.data, npts.ctypes.data, first.ctypes.data, times.ctypes.data, acc.ctypes.data)
    return [bool(a) for a in acc]


def integrate(frames, voxel_resolution, min_distance):
    """frames: [(xyz (n, 3) float64, intensities (n,))] -> (M, 4) float64 in the hash table's order."""
    xyzw = np.concatenate([np.concatenate([np.asarray(p, np.float64), np.ones((len(p), 1))], axis=1) for p, _ in frames])
    inten = np.concatenate([np.asarray(w, np.float64) for _, w in frames])
    first = np.concatenate([[0], np.cumsum([len(p) for p, _ in frames])]).astype(np.int64)
    out = np.zeros((max(len(xyzw), 1), 4))
    m = lib().bagref_integrate(len(frames), first.ctypes.data, np.ascontiguousarray(xyzw).ctypes.data, inten.ctypes.data, float(voxel_resolution),
                               float(min_distance), out.ctypes.data)
    return out[:m]
