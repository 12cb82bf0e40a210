"""CPU check of the centroid elision of the Nelder-Mead state machine (csrc/nm_machine.cuh): stepping a solve without
scoring the centroid of its iterations must give the same result, simplex and counters as scoring it, with exactly one
pose fewer per iteration batch, and must report the same evaluations minus the centroids.  tests/cpp/nm_centroid_check.cu
is built host-only from the header the host loop and the persistent kernel share; the GPU suite compares the two solver
paths with the elision on (tests/test_gpu_centroid_elision.py)."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("nm_centroid") / "nm_centroid_check")
    subprocess.run(
        [nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off", f"-I{CSRC}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
         os.path.join(ROOT, "tests", "cpp", "nm_centroid_check.cu")],
        check=True,
    )
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    return json.loads(out)


def test_every_objective_and_dimension_is_covered(cases):
    assert len(cases) == 5 * 2 * 3 * 4
    assert {c["objective"] for c in cases} == {"quadratic", "rosenbrock", "plateau", "nan_region", "constant"}
    assert {c["n"] for c in cases} == {2, 6}
    # the cases reach every branch that matters: shrinks, convergence, the iteration limit, and solves without iterations
    assert any(c["converged"][0] for c in cases) and any(not c["converged"][0] for c in cases)
    assert any(c["num_batches"][0] > c["iteration_batches"][0] + 1 for c in cases)  # a shrink batch happened
    assert any(c["iteration_batches"][0] == 0 for c in cases)


def test_elision_keeps_the_trajectory(cases):
    for c in cases:
        assert c["same_x"] and c["same_y"] and c["same_simplex"], c
        for k in ("converged", "num_iterations", "num_evaluations", "num_batches", "iteration_batches"):
            assert c[k][0] == c[k][1], (k, c)


def test_elision_scores_one_pose_fewer_per_iteration_batch(cases):
    for c in cases:
        scored, elided = c["computed"]
        assert scored - elided == c["iteration_batches"][0], c


def test_elision_reports_the_reference_evaluations_but_the_centroids(cases):
    for c in cases:
        assert c["obs_match"], c
        assert c["reported"][0] == c["num_evaluations"][0], c
        assert c["reported"][0] - c["reported"][1] == c["iteration_batches"][0], c
