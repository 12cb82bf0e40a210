"""CPU suite, part 2: the C-ABI library loads, exports every symbol include/vlcal_nid.h declares, and its HOST logic
(camera factory rules, projection, GTSAM expmap, estimate_camera_fov, batched Nelder-Mead) agrees with the oracle.
No compute kernels run here (no GPU)."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(vlcal):
    hdr = open(os.path.join(ROOT, "include", "vlcal_nid.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = sorted(set(re.findall(r"\b(vlcal_[a-z0-9_]+)\s*\(", hdr)))
    # typedef'd function-pointer types are not symbols
    names = [n for n in names if not n.endswith("_fn") and n not in ("vlcal_pose_callback",)]
    assert len(names) >= 30
    lib = C.CDLL(vlcal.library_path())
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_library_has_sm90a_code(vlcal):
    out = subprocess.run(["cuobjdump", "-lelf", vlcal.library_path()], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout


def test_product_does_not_link_or_import_the_oracle(vlcal):
    ldd = subprocess.run(["ldd", vlcal.library_path()], capture_output=True, text=True).stdout
    assert "oracle" not in ldd
    pkg = os.path.join(ROOT, "direct_visual_lidar_calibration_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert "vlcal_oracle" not in src and "from oracle" not in src and "import oracle" not in src, f


def test_no_device_is_a_loud_error(vlcal):
    if vlcal.device_count() > 0:
        pytest.skip("a GPU is present")
    cam = vlcal.create_camera("plumb_bob", [400, 410, 320, 240], [])
    data = vlcal.VisualLiDARData(np.zeros((48, 64), np.uint8), np.ones((10, 4)), np.zeros(10))
    with pytest.raises(vlcal.VlcalError) as e:
        vlcal.CostCalculatorNID(cam, data)
    assert e.value.code == -5 and "no CPU fallback" in str(e.value)
    with pytest.raises(vlcal.VlcalError):
        vlcal.ViewCulling(cam, (64, 48)).cull_indices(np.ones((10, 4)), np.eye(4))
    with pytest.raises(vlcal.VlcalError):
        vlcal.VisualCameraCalibration(cam, [data]).calibrate(np.eye(4))


def test_create_camera_mirrors_reference_rules(vlcal, capsys):
    assert vlcal.create_camera("nope", [1, 2, 3, 4], []) is None
    assert "unknown camera model nope" in capsys.readouterr().err
    assert vlcal.create_camera("plumb_bob", [1, 2, 3], []) is None
    assert "num of intrinsic parameters mismatch" in capsys.readouterr().err
    cam = vlcal.create_camera("plumb_bob", [1, 2, 3, 4], [0.1, 0.2])
    assert list(cam.distortion) == [0.1, 0.2, 0.0, 0.0, 0.0]
    assert list(vlcal.create_camera("fisheye", [1, 2, 3, 4], [1, 2, 3, 4, 5, 6]).distortion) == [1, 2, 3, 4]
    assert vlcal.create_camera("equidistant", [1, 2, 3, 4], []).model_id == vlcal.create_camera("fisheye", [1, 2, 3, 4], []).model_id


@pytest.mark.parametrize("model", util.MODELS)
def test_host_projection_is_bit_identical_to_oracle(vlcal, oracle, model):
    intr, dist, _ = util.CAMERAS[model]
    cam = vlcal.create_camera(model, intr, dist)
    ocam = oracle.create_camera(model, intr, dist)
    rng = np.random.default_rng(11)
    pts = rng.normal(size=(300, 3)) * [2, 2, 3]
    pts[:5] = [[0, 0, 1], [0, 0, -1], [1e-3, 1e-3, 1e-3], [0, 0, 0], [1, 1, 0]]
    a, b = cam.project(pts), oracle.project(ocam, pts)
    assert np.array_equal(a, b, equal_nan=True)


def test_expmap_and_fov_are_bit_identical_to_oracle(vlcal, oracle):
    rng = np.random.default_rng(2)
    for scale in (0.0, 1e-9, 1e-3, 0.5):
        xi = rng.normal(size=6) * scale
        assert np.array_equal(vlcal.se3_expmap(xi), oracle.se3_expmap(xi))
    for model in util.MODELS:
        intr, dist, (W, H) = util.CAMERAS[model]
        a = vlcal.estimate_camera_fov(vlcal.create_camera(model, intr, dist), (W, H))
        b = oracle.estimate_camera_fov(oracle.create_camera(model, intr, dist), W, H)
        assert a == b, model


OBJECTIVES = {
    "quadratic": lambda x: float(np.sum((x - np.arange(1, x.size + 1) * 0.01) ** 2 * np.arange(1, x.size + 1))),
    "rosenbrock": lambda x: float(sum(100 * (x[i + 1] - x[i] ** 2) ** 2 + (1 - x[i]) ** 2 for i in range(x.size - 1))),
    "plateaus": lambda x: float(np.floor(np.sum(np.abs(x)) * 50) / 50),  # many exact ties, like an integer histogram
    "nan_region": lambda x: float("nan") if x[0] > 0.05 else float(np.sum(x * x)),
}


@pytest.mark.parametrize("name", list(OBJECTIVES))
@pytest.mark.parametrize("n", [2, 6])
def test_batched_nelder_mead_follows_the_serial_trajectory(vlcal, oracle, name, n):
    f = OBJECTIVES[name]
    x0 = np.full(n, 0.02)
    kw = dict(init_step=1e-2, max_iterations=80, convergence_var_thresh=1e-12)
    ref = oracle.nelder_mead(f, x0, **kw)
    nm = vlcal.NelderMead(vlcal.NelderMeadParams(**kw))
    res = nm.optimize(f, x0)
    assert res["converged"] == ref["converged"] and res["num_iterations"] == ref["num_iterations"]
    assert np.array_equal(res["x"], ref["x"]) and (res["y"] == ref["y"] or (math.isnan(res["y"]) and math.isnan(ref["y"])))
    # same evaluations, same order (these are the ones whose side effects the reference would fire)
    assert res["num_evaluations"] == ref["num_evaluations"] == len(nm.observed)
    for (xa, ya), (xb, yb) in zip(nm.observed, ref["calls"]):
        assert np.array_equal(xa, xb) and (ya == yb or (math.isnan(ya) and math.isnan(yb)))
    # batching: one call per iteration (+ shrink batches), speculative evaluations accounted separately
    assert res["num_batches"] <= ref["num_iterations"] * 2 + 3
    assert res["num_evaluations_computed"] >= res["num_evaluations"]


def test_default_params_match_reference(vlcal):
    p = vlcal.VisualCameraCalibrationParams().to_c()
    assert (p.max_outer_iterations, p.max_inner_iterations, p.nid_bins) == (10, 256, 16)
    assert p.delta_trans_thresh == 0.1 and p.delta_rot_thresh == 0.5 * math.pi / 180.0
    assert p.nelder_mead_init_step == 1e-3 and p.nelder_mead_convergence_criteria == 1e-8
    q = vlcal.NelderMeadParams().to_c()
    assert (q.init_step, q.alpha, q.gamma, q.rho, q.sigma, q.max_iterations, q.convergence_var_thresh) == (0.1, 1.0, 2.0, 0.5, 0.5, 1024, 1e-5)


WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
import direct_visual_lidar_calibration_b200 as V
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
# bag-sharded objective: each rank owns one "bag" term; the per-pose partial sums are all-reduced before Nelder-Mead
# consumes them, so every rank walks the identical trajectory (DESIGN.md, multi-GPU).
centers = [np.array([0.01, -0.02, 0.03, 0.0, 0.01, -0.01]), np.array([-0.02, 0.01, 0.0, 0.02, -0.01, 0.03])]
def local(X): return np.sum((X - centers[rank]) ** 2, axis=1) * (rank + 1)
def batch(X):
    t = torch.from_numpy(local(X).copy())
    dist.all_reduce(t)
    return t.numpy()
nm = V.NelderMead(V.NelderMeadParams(init_step=1e-3, max_iterations=120, convergence_var_thresh=1e-14))
res = nm.optimize_batched(batch, np.zeros(6))
out = torch.from_numpy(np.concatenate([res["x"], [res["y"], res["num_iterations"], res["num_evaluations"]]]))
gathered = [torch.zeros_like(out) for _ in range(world)]
dist.all_gather(gathered, out)
if rank == 0:
    assert all(torch.equal(g, gathered[0]) for g in gathered), "ranks diverged"
    # single-process reference: same objective with the sum done locally in rank order
    nm1 = V.NelderMead(V.NelderMeadParams(init_step=1e-3, max_iterations=120, convergence_var_thresh=1e-14))
    ref = nm1.optimize_batched(lambda X: sum(np.sum((X - centers[r]) ** 2, axis=1) * (r + 1) for r in range(world)), np.zeros(6))
    assert np.allclose(ref["x"], res["x"], atol=1e-12) and ref["num_iterations"] == res["num_iterations"]
    print("GLOO_OK", res["num_iterations"], res["y"])
dist.destroy_process_group()
"""


def test_bag_sharded_objective_over_gloo_world_size_2(vlcal, tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29533", WORLD_SIZE="2", OMP_NUM_THREADS="1")
    procs = [subprocess.Popen([sys.executable, str(script), ROOT], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert "GLOO_OK" in outs[0]
