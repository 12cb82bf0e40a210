"""CPU check of the anchor rule of the equirectangular delta step (csrc/lean_filter.cuh: lean_delta_anchor, the function
the persistent kernel's warp-parallel pick, the host's instance pick and the verify kernel follow): the most central pose
of a batch, lowest index on ties."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")


@pytest.fixture(scope="module")
def anchors(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("delta_anchor") / "delta_anchor_check")
    subprocess.run(
        [nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off", f"-I{CSRC}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
         os.path.join(ROOT, "tests", "cpp", "delta_anchor_check.cu")],
        check=True,
    )
    return json.loads(subprocess.run([exe], check=True, capture_output=True, text=True).stdout)


def test_iteration_batch_is_anchored_at_the_reflection(anchors):
    assert anchors["iteration"] == 1  # {xo, xr, xe, xc}: xr is |diff| from every other pose


def test_initial_simplex_is_anchored_at_its_start(anchors):
    assert anchors["simplex"] == 0


def test_ties_and_single_poses_go_to_the_lowest_index(anchors):
    assert anchors["equal"] == 0
    assert anchors["single"] == 0


def test_eight_pose_line_is_anchored_at_its_centre(anchors):
    assert anchors["central"] == 3
