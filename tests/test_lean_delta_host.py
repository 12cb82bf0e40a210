"""CPU check of the equirectangular delta step of the persistent kernel (csrc/lean_filter.cuh: classify_lean_anchor,
classify_lean_delta) against the exact double path: tests/cpp/lean_delta_check.cu is the SAME source the kernel's packed
twin follows, built host-only.  Poses 1..7 of a batch lie on a line through pose 0 at 1e-6 .. 5e-3 rad / m; points are
nudged to within 1e-3 .. 1e-8 px of a pixel edge at those poses, some near the poles and the seam.  Every verdict the
delta step keeps must be the exact path's.  The GPU suite repeats the check with the device intrinsics
(tests/test_gpu_delta_poses.py)."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")


@pytest.fixture(scope="module")
def lean_delta_check(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("lean_delta") / "lean_delta_check")
    subprocess.run(
        [nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off", f"-I{CSRC}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
         os.path.join(ROOT, "tests", "cpp", "lean_delta_check.cu")],
        check=True,
    )
    return exe


def test_delta_step_never_contradicts_the_exact_path(lean_delta_check):
    out = subprocess.run([lean_delta_check, "40000"], check=True, capture_output=True, text=True).stdout
    cases = json.loads(out)
    assert len(cases) == 3
    for c in cases:
        assert c["enabled"] == 1, c
        assert c["point_poses"] == 40000 * 7
        assert c["mismatches"] == 0, c
        assert c["max_error_over_bound_ppm"] < 1_000_000, c
        assert c["accepted"] > 0.35 * c["point_poses"], c
        # the adversarial points (nudged to an edge, near the poles and the seam) defer often with either classifier; the
        # remainder term and the guards of the delta step may add a few per cent on top of the plain classifier's share
        print(f"case {c['case']}: {c['uncertain'] / c['point_poses']:.3%} of the delta point-poses deferred, plain classifier {c['plain_uncertain'] / c['point_poses']:.3%}")
        assert (c["uncertain"] - c["plain_uncertain"]) / c["point_poses"] < 0.1, c
