"""CPU check of the lean fp32 classifier of the persistent kernel (csrc/lean_filter.cuh) against the exact double path
(csrc/exact_classify.cuh; reference decisions: src/vlcal/calib/cost_calculator_nid.cpp:31-38): tests/cpp/lean_check.cu
is the SAME source the kernel compiles, built host-only.  Every verdict the filter keeps must be the exact path's --
including the reference's truncation toward zero for u, v in (-1, 0) -- on random and on edge-adversarial points
(pixel coordinates nudged to within 1e-3 .. 1e-8 px of an integer) and on the FoV cone (points at max_fov (1 +- 10^[-12,
-3]) from the optical axis).  The GPU suite repeats the checks with the device intrinsics
(tests/test_gpu_parity.py::test_filter_error_bound_is_sound, tests/test_gpu_filter_decision_edges.py)."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")


@pytest.fixture(scope="module")
def lean_check(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("lean") / "lean_check")
    subprocess.run(
        [nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off", f"-I{CSRC}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
         os.path.join(ROOT, "tests", "cpp", "lean_check.cu")],
        check=True,
    )
    return exe


@pytest.mark.parametrize("adversarial", [1, 0])
def test_lean_classifier_never_contradicts_the_exact_path(lean_check, adversarial):
    out = subprocess.run([lean_check, "60000", str(adversarial)], check=True, capture_output=True, text=True).stdout
    cases = json.loads(out)
    assert len(cases) == 9
    for c in cases:
        assert c["enabled"] == 1, c
        assert c["point_poses"] == 240000
        assert c["mismatches"] == 0, c
        assert c["accepted"] > 50000, c
        # the filter must actually decide most point-poses (natural deferral rate of the C2 camera: ~3 %)
        assert c["uncertain"] / c["point_poses"] < (0.15 if adversarial else 0.08), c
    # the reference truncates toward zero: u in (-1, 0) is column 0 (cost_calculator_nid.cpp:37) -- the strip must be hit
    assert sum(c["accepted_in_minus_one_strip"] for c in cases if c["model"] == 0) > 100


def _check_cone(lean_check, *translation):
    out = subprocess.run([lean_check, "100000", "2", *translation], check=True, capture_output=True, text=True).stdout
    cases = json.loads(out)
    assert len(cases) == 16 and {c["model"] for c in cases} == set(range(6))
    for c in cases:
        assert c["enabled"] == 1 and c["points"] == 100000, c
        assert c["mismatches"] == 0, c
        assert c["uncertain"] / c["points"] > 0.5, c  # offsets 10^-12 .. 10^-6 of the angle sit inside the band
        assert c["in_image_without_fov"] / c["points"] > 0.3, c  # the cone crosses the image interior


def test_lean_classifier_on_the_fov_cone(lean_check):
    """Every model at explicit max_fov values where the cone crosses the image, beyond 90 degrees for fisheye, omnidir
    and equirectangular (cos_fov < 0): no verdict may contradict the exact path, and most of the points must fall inside
    the uncertain band (otherwise the mode would not reach the decision it is meant to test)."""
    _check_cone(lean_check)


@pytest.mark.parametrize("translation", ["30", "300"])
def test_lean_classifier_on_the_fov_cone_far_from_the_lidar_origin(lean_check, translation):
    """The cone cases with pose translations up to 30 and 300 m: the camera stands far from the LiDAR origin, as in a
    map frame, and the max|t| term is a large part of the bound."""
    _check_cone(lean_check, translation)
