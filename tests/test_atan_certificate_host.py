"""Exhaustive certificate of the lean classifier's arctangent (csrc/lean_filter.cuh, lean_atan2_turns): tests/cpp/
atan_certificate.cu evaluates the polynomial for every float t in [0, 1 + 2^-20] exactly as the kernel compiles it and
compares with a long double atan; the whole routine is then checked against atan2l on random pairs.  The error the
equirectangular bounds charge (LEAN_ATAN_ERR_TURNS) must cover the measured polynomial error plus the analytic quotient
and octant-fold terms stated in the header."""
import json
import math
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")


@pytest.fixture(scope="module")
def certificate(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("atan") / "atan_certificate")
    subprocess.run(
        [nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-fopenmp,-ffp-contract=off", f"-I{CSRC}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
         os.path.join(ROOT, "tests", "cpp", "atan_certificate.cu"), "-lgomp"],
        check=True,
    )
    out = subprocess.run([exe, "20000000"], check=True, capture_output=True, text=True).stdout
    return json.loads(out)


def test_polynomial_error_is_certified_for_every_float(certificate):
    c = certificate
    assert c["values"] == 0x3F800000 + 9  # every float from +0 to 1 + 8 ulp
    assert c["t_hi"] > 1.0 + 2.0**-23  # the largest quotient mn * rcp(mx) can produce
    assert c["non_finite"] == 0
    assert c["max_err_rounded"] <= c["poly_bound"], c
    assert c["max_err_unrounded"] <= c["poly_bound"], c
    # the fit is not slack either: the bound stays within 2 % of what the sweep measures
    assert c["poly_bound"] < 1.02 * max(c["max_err_rounded"], c["max_err_unrounded"]), c
    # the first octant fold 0.25 - p needs p in [0, 0.126]
    assert c["p_min"] >= 0.0 and c["p_max"] <= 0.126, c


def test_analytic_terms_and_charge(certificate):
    c = certificate
    u = 2.0**-24
    assert c["quot_bound"] >= (3 * u + 2 * u * u) / (4 * math.pi) * (1 + 1e-6)
    assert c["fold_bound"] >= 2.0**-27 + 2.0**-26
    assert c["cert"] >= c["poly_bound"] + c["quot_bound"] + c["fold_bound"] - 1e-22
    assert c["charged"] >= 1.05 * c["cert"], c


def test_whole_routine_stays_within_the_certificate(certificate):
    c = certificate
    assert c["pairs"] == 20000000
    assert 0.0 < c["pairs_max_err"] <= c["cert"], c
