"""The reference-side C++ bindings compile against stand-in reference headers and link to the C-ABI library:
include/vlcal_b200/cost_calculator_nid_cuda.hpp behaves like a vlcal::CostCalculator, and
include/vlcal_b200/nid_cost_cuda.hpp (the NID_BFGS branch) like the ceres::FirstOrderFunction it replaces."""
import os
import struct
import subprocess

import numpy as np
import pytest

import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _build(vlcal, tmp_path):
    exe = str(tmp_path / "cpp_shim")
    libdir = os.path.dirname(vlcal.library_path())
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(HERE, "cpp_stubs"), "-I", os.path.join(ROOT, "include"),
           os.path.join(HERE, "cpp_shim_main.cpp"), "-o", exe, "-L", libdir, "-lvlcal_nid", f"-Wl,-rpath,{libdir}"]
    subprocess.run(cmd, check=True)
    return exe


def _write_problem(path, pr):
    with open(path, "wb") as f:
        f.write(struct.pack("iii", pr["W"], pr["H"], pr["points"].shape[0]))
        f.write(pr["image"].tobytes())
        f.write(np.ascontiguousarray(pr["points"]).tobytes())
        f.write(np.ascontiguousarray(pr["intensities"]).tobytes())
        f.write(np.ascontiguousarray(pr["T"].T).tobytes())  # column-major


def test_shim_compiles_and_fails_loudly_without_gpu(vlcal, tmp_path):
    exe = _build(vlcal, tmp_path)
    if vlcal.device_count() > 0:
        pytest.skip("a GPU is present; covered by the gpu test")
    pr = util.random_problem("plumb_bob", n=100, seed=1)
    _write_problem(tmp_path / "p.bin", pr)
    out = subprocess.run([exe, str(tmp_path / "p.bin")], capture_output=True, text=True)
    assert out.returncode == 3 and "no CUDA device" in out.stdout


@pytest.mark.gpu
def test_shim_matches_python_surface_and_oracle(gpu, oracle, tmp_path):
    exe = _build(gpu, tmp_path)
    pr = util.random_problem("plumb_bob", n=20000, seed=2)
    _write_problem(tmp_path / "p.bin", pr)
    out = subprocess.run([exe, str(tmp_path / "p.bin")], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    vals = [float(v) for v in out.stdout.split()[1:]]
    cam = gpu.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    ref = gpu.CostCalculatorNID(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])).calculate(pr["T"])
    assert vals[0] == ref and vals[1] == ref and vals[2] == ref
    assert vals[3] == ref  # CostCalculatorNIDCuda(proj, data, params): the reference's constructor shape, through CameraParamsView
    assert vals[4] == 1.0 and vals[5] == 1.0  # a camera without the view throws; unknown model -> nullptr like the reference
    ocam = oracle.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    onid = oracle.nid_calculate(ocam, pr["image"], pr["points"], pr["intensities"], 16, oracle.estimate_camera_fov(ocam, pr["W"], pr["H"]), pr["T"])[0]
    assert abs(vals[0] - onid) < 1e-12


def _build_bfgs(vlcal, tmp_path):
    """tests/cpp_bfgs_main.cpp: the BFGS binding against the Ceres / Sophus / Eigen / cv::Mat stand-ins of oracle/ref_standin
    (listed first, so they win over tests/cpp_stubs, which only adds vlcal/common/frame.hpp here)."""
    exe = str(tmp_path / "cpp_bfgs")
    libdir = os.path.dirname(vlcal.library_path())
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "oracle", "ref_standin"), "-I", os.path.join(HERE, "cpp_stubs"),
           "-I", os.path.join(ROOT, "include"), os.path.join(HERE, "cpp_bfgs_main.cpp"), "-o", exe, "-L", libdir, "-lvlcal_nid", f"-Wl,-rpath,{libdir}"]
    subprocess.run(cmd, check=True)
    return exe


def test_bfgs_binding_compiles_and_fails_loudly_without_gpu(vlcal, tmp_path):
    exe = _build_bfgs(vlcal, tmp_path)
    if vlcal.device_count() > 0:
        pytest.skip("a GPU is present; covered by the gpu test")
    out = subprocess.run([exe], capture_output=True, text=True)
    # no CPU fallback: the NIDCostCuda constructor throws with the library's message
    assert out.returncode == 3 and out.stdout.startswith("EXCEPTION") and "no CUDA device" in out.stdout, out.stdout + out.stderr


def _bfgs_main_problem():
    """The inputs tests/cpp_bfgs_main.cpp builds: a 64x48 image, 500 points on a plane 2 m in front of the camera."""
    W, H, N = 64, 48, 500
    image = ((np.arange(W * H) * 37) % 251).astype(np.uint8).reshape(H, W)
    i = np.arange(N)
    pts = np.stack([-0.8 + 1.6 * (i % 25) / 24.0, -0.6 + 1.2 * (i // 25) / 19.0, np.full(N, 2.0), np.ones(N)], axis=1)
    return image, pts, (i % 16) / 16.0


@pytest.mark.gpu
def test_bfgs_binding_matches_python_surface(gpu, tmp_path):
    exe = _build_bfgs(gpu, tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("EVAL ok=1 n=7 "), out.stdout + out.stderr
    fields = dict(kv.split("=") for kv in out.stdout.split()[1:])
    image, pts, ins = _bfgs_main_problem()
    cam = gpu.create_camera("plumb_bob", [60.0, 60.0, 32.0, 24.0], [])
    ok, nid, grad = gpu.NIDCost(cam, gpu.VisualLiDARData(image, pts, ins), 16).evaluate_with_gradient(np.array([[0, 0, 0, 1, 0, 0, 0.0]]))
    assert bool(ok[0]) and np.isfinite(nid[0])
    assert abs(float(fields["cost"]) - nid[0]) < 1e-12 and abs(float(fields["g0"]) - grad[0][0]) < 1e-12 * max(1.0, abs(grad[0][0]))
