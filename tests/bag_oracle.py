"""ctypes wrapper of tests/cpp/bag_oracle.c, the sequential CPU checker of the bag decoder and static integrator (built on
first use into a temporary directory)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from direct_visual_lidar_calibration_b200 import _lib as VL

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="bag_oracle_"), "libbag_oracle.so")
        subprocess.run(["/usr/bin/gcc", "-O2", "-std=c11", "-D_DEFAULT_SOURCE", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", out,
                        os.path.join(_HERE, "cpp", "bag_oracle.c"), "-lm"], check=True)
        L = C.CDLL(out)
        vp = C.c_void_p
        L.orc_bag_integrate.argtypes = [vp, C.POINTER(VL.ScanDesc), C.c_int64, C.c_double, C.c_double, vp, C.POINTER(C.c_int64)]
        L.orc_bag_integrate.restype = C.c_int64
        L.orc_extract_scan.argtypes = [vp, C.POINTER(VL.ScanDesc), vp]
        L.orc_extract_scan.restype = None
        _lib = L
    return _lib


def bag_integrate(blob, descs, voxel_resolution=0.002, min_distance=1.0):
    """-> (float32 (M, 4) in first-write order, out-of-range count)"""
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    arr = (VL.ScanDesc * max(len(descs), 1))(*descs)
    total = sum(d.n_points for d in descs)
    out = np.empty((max(total, 1), 4), np.float32)
    oor = C.c_int64()
    m = lib().orc_bag_integrate(blob.ctypes.data, arr, len(descs), float(voxel_resolution), float(min_distance), out.ctypes.data, C.byref(oor))
    assert m >= 0
    return out[:m].copy(), int(oor.value)


def extract_scan(blob, desc):
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    out = np.empty((max(desc.n_points, 1), 4))
    lib().orc_extract_scan(blob.ctypes.data, C.byref(desc), out.ctypes.data)
    return out[: desc.n_points]
