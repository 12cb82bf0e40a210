"""Concurrent use of the library, as the reference uses it: one cost object per bag, calculate() from the workers of an
OpenMP loop (visual_camera_calibration.cpp:107-110), and the header's promise that different contexts may be used from
different host threads at once (include/vlcal_nid.h).

- tests/cpp/omp_bag_loop.cpp is that loop, literally, through include/vlcal_b200/cost_calculator_nid_cuda.hpp: bags are
  built, scored and destroyed from `#pragma omp parallel for`, over several rounds with the bag sizes moved between
  threads.  Per-bag values must be bit-equal between one thread and B threads, and within 1e-12 of the oracle.
- The threaded cases run Python threads (ctypes releases the GIL during a call) from one barrier.  Each first computes
  its expected values serially in the same process and checks them against the oracle, then runs the threads, and
  asserts that the calls' perf_counter windows really overlapped.  They run in a worker subprocess with a wall-clock
  timeout, so a stuck call fails its test instead of wedging the session.
- The async pair (vlcal_nid_evaluate_async / vlcal_nid_wait) on one thread: several contexts in flight, waited on in
  reverse order, the busy and idle errors, and _wait refusing histograms that the evaluation in flight did not compute."""
import ctypes as C
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import _lib
from direct_visual_lidar_calibration_b200 import calibration as _VC
from direct_visual_lidar_calibration_b200 import synthetic as _S
from direct_visual_lidar_calibration_b200.cost import T_to_colmajor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NID_TOL = 1e-12
PK_THREADS = 768  # threads per block of the persistent kernel: a bag above 2 x SMs x 768 points gives a grid that fills the device
CASE_TIMEOUT_S = 600


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _max_in_flight(spans):
    """The largest number of (start, end) windows that contain one instant."""
    ev = sorted([(t0, 1) for t0, _ in spans] + [(t1, -1) for _, t1 in spans])  # at equal times an end sorts first
    cur = best = 0
    for _, d in ev:
        cur += d
        best = max(best, cur)
    return best


def _assert_nid(got, want, tol=NID_TOL):
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    m = ~np.isnan(want)
    assert np.all(np.abs(got[m] - want[m]) < tol), np.abs(got[m] - want[m]).max()


def _oracle_eval(O, pr, Ts, bins=16):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    big = pr["points"].shape[0] * len(Ts) > 2_000_000
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T, omp=big) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _cost(V, pr, bins=16, variant=0):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    cost = V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins))
    if variant:
        cost.set_kernel_variant(variant)
    return cost


# ---- A. the reference's OpenMP bag loop ---------------------------------------------------------------------------------


def _build_omp_loop(vlcal, tmp_path):
    exe = str(tmp_path / "omp_bag_loop")
    libdir = os.path.dirname(vlcal.library_path())
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-fopenmp", "-I", os.path.join(HERE, "cpp_stubs"), "-I", os.path.join(ROOT, "include"),
           os.path.join(HERE, "cpp", "omp_bag_loop.cpp"), "-o", exe, "-L", libdir, "-lvlcal_nid", f"-Wl,-rpath,{libdir}"]
    subprocess.run(cmd, check=True)
    return exe


def _write_bags(path, prs, Ts, rounds):
    with open(path, "wb") as f:
        f.write(np.array([len(prs), len(Ts), rounds], dtype=np.int32).tobytes())
        for pr in prs:
            f.write(np.array([pr["W"], pr["H"], pr["points"].shape[0]], dtype=np.int32).tobytes())
            f.write(np.ascontiguousarray(pr["image"]).tobytes())
            f.write(np.ascontiguousarray(pr["points"], dtype=np.float64).tobytes())
            f.write(np.ascontiguousarray(pr["intensities"], dtype=np.float64).tobytes())
        for T in Ts:
            f.write(np.ascontiguousarray(np.asarray(T, dtype=np.float64).T).tobytes())  # column-major


def _run_omp_loop(exe, path, threads):
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=CASE_TIMEOUT_S, env=dict(os.environ, OMP_NUM_THREADS=str(threads)))
    return out.returncode, out.stdout, out.stderr


def _parse_omp_loop(stdout):
    """{(bag, pose): printed value} (every round and slot must print the same bits for a bag), in-flight maxima."""
    vals, inflight = {}, {}
    for line in stdout.splitlines():
        f = line.split()
        if f[0] == "VAL":
            key = (int(f[3]), int(f[4]))
            assert vals.setdefault(key, f[5]) == f[5], (key, vals[key], f[5])
        elif f[0] == "INFLIGHT":
            inflight[f[1]] = int(f[2])
    return vals, inflight


def _omp_bags(n_bags, sms):
    """Bag sizes: 0, 1 and 10^3 points, bags whose persistent grid fills the device, one double-layout bag (round-1 path)."""
    big = 2 * sms * PK_THREADS + 4_099
    sizes = {
        2: [(big, True), (1_000, False)],
        8: [(big, True), (0, True), (1, True), (1_000, True), (1_000, False), (big + 1, True), (20_000, True), (1_000, True)],
        16: [(big, True), (big + 7, True), (0, True), (1, True), (1_000, True), (1_000, True), (1_000, False), (5_000, True),
             (20_000, True), (60_000, True), (0, True), (1, True), (1_000, True), (3_000, True), (big + 13, True), (1_000, True)],
    }[n_bags]
    return [util.random_problem("plumb_bob", n=n, seed=100 + k, f32=f32) for k, (n, f32) in enumerate(sizes)]


def test_omp_bag_loop_compiles_and_fails_loudly_without_gpu(vlcal, tmp_path):
    exe = _build_omp_loop(vlcal, tmp_path)
    if vlcal.device_count() > 0:
        pytest.skip("a GPU is present; covered by the gpu test")
    prs = [util.random_problem("plumb_bob", n=n, seed=k) for k, n in enumerate((100, 0))]
    _write_bags(tmp_path / "bags.bin", prs, [prs[0]["T"]], 1)
    rc, out, err = _run_omp_loop(exe, tmp_path / "bags.bin", 2)
    assert rc == 3 and out.startswith("EXCEPTION") and "no CUDA device" in out, out + err


@pytest.mark.gpu
@pytest.mark.parametrize("n_bags", [2, 8, 16])
def test_omp_bag_loop_matches_one_thread_and_the_oracle(gpu, oracle, tmp_path, n_bags):
    import torch

    sms = int(torch.cuda.get_device_properties(0).multi_processor_count)
    exe = _build_omp_loop(gpu, tmp_path)
    prs = _omp_bags(n_bags, sms)
    assert max(pr["points"].shape[0] for pr in prs) > 2 * sms * PK_THREADS
    Ts = util.random_poses(prs[0]["T"], 4, seed=n_bags)
    rounds = 3
    _write_bags(tmp_path / "bags.bin", prs, Ts, rounds)
    runs = {}
    for threads in (1, n_bags):
        rc, out, err = _run_omp_loop(exe, tmp_path / "bags.bin", threads)
        assert rc == 0 and out.rstrip().endswith("OK"), out[-2000:] + err[-2000:]
        runs[threads] = _parse_omp_loop(out)
    (serial, inflight1), (parallel, inflight_b) = runs[1], runs[n_bags]
    assert len(serial) == n_bags * len(Ts) and parallel == serial  # bit for bit: the same printed digits
    assert inflight1["calc"] == 1 and inflight_b["calc"] >= 2, (inflight1, inflight_b)
    for b, pr in enumerate(prs):
        want, _ = _oracle_eval(oracle, pr, Ts)
        _assert_nid([float(serial[(b, p)]) for p in range(len(Ts))], want)
    print(f"omp bag loop B={n_bags}: in flight at once: calculate {inflight_b['calc']}, constructors {inflight_b['create']}")


# ---- B. Python threads, each case in a worker subprocess ---------------------------------------------------------------


class _Windows:
    """perf_counter windows around library calls, from any thread."""

    def __init__(self):
        self.spans = []
        self._lock = threading.Lock()

    def call(self, fn, *args, **kwargs):
        t0 = time.perf_counter()
        try:
            return fn(*args, **kwargs)
        finally:
            t1 = time.perf_counter()
            with self._lock:
                self.spans.append((t0, t1))

    def assert_overlapped(self, name):
        k = _max_in_flight(self.spans)
        print(f"INFLIGHT {name} {k}")
        assert k >= 2, f"{name}: the calls never overlapped"


def _run_threads(bodies):
    """bodies[k]() on thread k, all released by one barrier; re-raises the first failure.  Returns their results."""
    barrier = threading.Barrier(len(bodies))
    results, errors = [None] * len(bodies), [None] * len(bodies)

    def run(k):
        try:
            barrier.wait()
            results[k] = bodies[k]()
        except BaseException as e:  # noqa: BLE001 -- re-raised on the main thread
            errors[k] = e

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(bodies))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errors:
        if e is not None:
            raise e
    return results


def _libs():
    import direct_visual_lidar_calibration_b200 as V
    from oracle import oracle as O

    O.build()
    if V.device_count() < 1:
        raise RuntimeError("no CUDA device visible")
    return V, O


def _case_histograms_k1p_and_round1():
    """calculate_batch(return_hist=True) on persistent-kernel contexts (16 and 32 bins) beside round-1 contexts (64 bins,
    the double layout, the exact kernel of variant 1)."""
    V, O = _libs()
    specs = [  # (points, bins, f32, variant, persistent kernel)
        (260_000, 16, True, 0, True), (120_000, 32, True, 0, True), (60_000, 64, True, 0, False), (40_000, 16, False, 0, False), (60_000, 16, True, 1, False),
    ]
    work = []
    for k, (n, bins, f32, variant, pk) in enumerate(specs):
        pr = util.random_problem("plumb_bob", n=n, seed=200 + k, f32=f32)
        Ts = util.random_poses(pr["T"], 8, seed=k)
        cost = _cost(V, pr, bins, variant)
        nid, hist = cost.calculate_batch(Ts, return_hist=True)
        assert cost.last_points_per_lane() > 0 if pk else cost.last_points_per_lane() == 0, (k, cost.last_points_per_lane())
        onid, ohist = _oracle_eval(O, pr, Ts, bins)
        assert np.array_equal(hist, ohist) and hist.sum() > 1000
        _assert_nid(nid, onid)
        work.append((cost, Ts, nid, hist))
    w = _Windows()

    def body(cost, Ts, nid, hist):
        def run():
            for _ in range(6):
                n2, h2 = w.call(cost.calculate_batch, Ts, return_hist=True)
                assert np.array_equal(n2, nid, equal_nan=True) and np.array_equal(h2, hist)
        return run

    _run_threads([body(*x) for x in work])
    w.assert_overlapped("histograms")


def _case_score_poses_disjoint_lists():
    """score_poses over a multi-bag list per thread, the lists disjoint."""
    V, O = _libs()
    lists = []
    for t in range(4):
        prs = [util.random_problem("plumb_bob", n=n, seed=300 + 10 * t + b) for b, n in enumerate((220_000 if t < 2 else 60_000, 30_000, 1_000))]
        costs = [_cost(V, pr) for pr in prs]
        Ts = util.random_poses(prs[0]["T"], 10, seed=30 + t)
        per_bag = []
        for pr, c in zip(prs, costs):
            nid = c.calculate_batch(Ts)
            _assert_nid(nid, _oracle_eval(O, pr, Ts)[0])
            per_bag.append(nid)
        want = per_bag[0] + per_bag[1] + per_bag[2]  # summed in bag order, as score_poses sums
        got = V.score_poses(costs, Ts)
        assert np.array_equal(got, want, equal_nan=True)
        lists.append((costs, Ts, got))
    w = _Windows()

    def body(costs, Ts, want):
        def run():
            for _ in range(6):
                assert np.array_equal(w.call(V.score_poses, costs, Ts), want, equal_nan=True)
        return run

    _run_threads([body(*x) for x in lists])
    w.assert_overlapped("score_poses")


def _sophus_params(T):
    from scipy.spatial.transform import Rotation

    return np.concatenate([Rotation.from_matrix(T[:3, :3]).as_quat(), T[:3, 3]])  # qx qy qz qw tx ty tz


def _case_mode_b():
    """NIDCost.evaluate(return_hist=True) and evaluate_with_gradient per thread: fixed-point weights make the values and
    histograms bit-stable; the gradients' double atomics may move the last bits."""
    V, O = _libs()
    work = []
    for t in range(4):
        pr = util.random_problem("plumb_bob", n=(150_000 if t == 0 else 40_000), seed=400 + t)
        tps = np.stack([_sophus_params(T) for T in util.random_poses(pr["T"], 3, seed=40 + t)])
        cost = V.NIDCost(V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"]), V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), 16)
        ok, nid, hist = cost.evaluate(tps, return_hist=True)
        gok, gnid, grad = cost.evaluate_with_gradient(tps)
        ocam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
        for p in range(len(tps)):
            rok, rnid, rhist = O.nid_cost_bspline(ocam, pr["image"], pr["points"], pr["intensities"], 16, tps[p])
            assert bool(ok[p]) == rok and abs(nid[p] - rnid) < 1e-9 and np.abs(hist[p] - rhist).max() < 1e-6
            gok_r, gnid_r, grad_r = O.nid_cost_bspline_grad(ocam, pr["image"], pr["points"], pr["intensities"], 16, tps[p])
            assert bool(gok[p]) == gok_r and abs(gnid[p] - gnid_r) < 1e-9
            assert np.abs(grad[p] - grad_r).max() < 1e-8 * max(1.0, np.abs(grad_r).max())
        work.append((cost, tps, ok, nid, hist, gok, gnid, grad))
    w = _Windows()

    def body(cost, tps, ok, nid, hist, gok, gnid, grad):
        def run():
            for _ in range(4):
                ok2, nid2, hist2 = w.call(cost.evaluate, tps, return_hist=True)
                assert np.array_equal(ok2, ok) and np.array_equal(nid2, nid, equal_nan=True) and np.array_equal(hist2, hist)
                gok2, gnid2, grad2 = w.call(cost.evaluate_with_gradient, tps)
                assert np.array_equal(gok2, gok) and np.array_equal(gnid2, gnid, equal_nan=True)
                assert np.abs(grad2 - grad).max() <= 1e-10 * max(1.0, np.abs(grad).max())
        return run

    _run_threads([body(*x) for x in work])
    w.assert_overlapped("mode_b")


def _case_legacy_stream_entry_points():
    """View culling, generate_lidar_image and the RANSAC scoring (legacy default stream) while persistent-kernel contexts
    are busy on their own streams."""
    V, O = _libs()
    import pose_oracle
    from direct_visual_lidar_calibration_b200 import pose_estimation as PE

    pr = util.random_problem("plumb_bob", n=200_000, seed=500)
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    ocam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(ocam, pr["W"], pr["H"])
    W, H, T = pr["W"], pr["H"], pr["T"]
    culling = V.ViewCulling(cam, (W, H))
    idx = culling.cull_indices(pr["points"], T)
    assert np.array_equal(idx, O.view_cull(ocam, W, H, fov, True, pr["points"], T)) and idx.size > 1000
    img = V.generate_lidar_image(cam, (W, H), T, pr["points"], pr["intensities"])
    oimg = O.generate_lidar_image(ocam, W, H, T, pr["points"], pr["intensities"])
    assert np.array_equal(img[0], oimg[0], equal_nan=True) and np.array_equal(img[1], oimg[1]) and (img[1] >= 0).sum() > 1000
    # RANSAC scoring: keypoints are the projections of the cloud's first points, a third replaced by random pixels
    rng = np.random.default_rng(5)
    m = 2_000
    pts = pr["points"][:m, :3].copy()
    pc = pts @ T[:3, :3].T + T[:3, 3]
    kp = np.array([O.project(ocam, p) for p in pc]) + rng.normal(0.0, 1.0, (m, 2))
    out = rng.random(m) < 0.3
    kp[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    pairs = PE.sample_pairs(m, 8192)
    counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
    ref_counts, ref_degenerate, ref_near = pose_oracle.score(ocam, kp, pts, pairs, 5.0)
    assert np.array_equal(degenerate, ref_degenerate) and np.all(np.abs(counts.astype(np.int64) - ref_counts) <= ref_near)
    busy = []
    for k in range(2):
        bpr = util.random_problem("plumb_bob", n=260_000, seed=510 + k)
        Ts = util.random_poses(bpr["T"], 8, seed=51 + k)
        cost = _cost(V, bpr)
        nid = cost.calculate_batch(Ts)
        _assert_nid(nid, _oracle_eval(O, bpr, Ts)[0])
        busy.append((cost, Ts, nid))
    w = _Windows()

    def k1p(cost, Ts, nid):
        def run():
            for _ in range(12):
                assert np.array_equal(w.call(cost.calculate_batch, Ts), nid, equal_nan=True)
        return run

    def cull():
        for _ in range(8):
            assert np.array_equal(w.call(culling.cull_indices, pr["points"], T), idx)

    def lidar_image():
        for _ in range(8):
            a, b = w.call(V.generate_lidar_image, cam, (W, H), T, pr["points"], pr["intensities"])
            assert np.array_equal(a, img[0], equal_nan=True) and np.array_equal(b, img[1])

    def ransac():
        for _ in range(8):
            c2, d2 = w.call(PE.score_pairs, cam, kp, pts, pairs, 5.0)
            assert np.array_equal(c2, counts) and np.array_equal(d2, degenerate)

    _run_threads([k1p(*busy[0]), k1p(*busy[1]), cull, lidar_image, ransac])
    w.assert_overlapped("legacy_stream")


def _synthetic_bag(n, cfg):
    bag = _S.make_bag("pinhole_640x480", "frustum", n, config_index=cfg, scale=0.5)
    bag["T_init"] = _S.perturb(bag["T_gt"], (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))
    return bag


def _case_solves():
    """Whole inner solves per thread with the solve trace armed in each thread, in solver modes 0 and 1 (set
    process-wide before the threads start), then one calibrate on two bags per thread."""
    V, O = _libs()
    bags = [_synthetic_bag(n, cfg=3 + k) for k, n in enumerate((200_000, 12_000, 8_000))]
    cam_args = (bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    cam, ocam = V.create_camera(*cam_args), O.create_camera(*cam_args)
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 20
    op = O.default_calib_params()
    op.max_inner_iterations = 20
    datasets = [[V.VisualLiDARData(b["image"], b["points"], b["intensities"])] for b in bags]
    oracle_traces = [O.estimate_pose_nelder_mead(ocam, [(b["image"], b["points"], b["intensities"])], b["T_init"], op) for b in bags]
    w = _Windows()

    def solve(k):
        _VC.record_solve_trace(True)
        try:
            calib = V.VisualCameraCalibration(cam, datasets[k], params)
            T, r = w.call(calib.estimate_pose_nelder_mead, bags[k]["T_init"])
            return T, r["x"], [c for _, c in calib.trace], _VC.last_solve_trace()
        finally:
            _VC.record_solve_trace(False)

    try:
        for mode in (0, 1):
            V.set_solver_mode(mode)
            serial = [solve(k) for k in range(len(bags))]
            for (T, x, costs, trace), ref in zip(serial, oracle_traces):
                assert np.array_equal(x, ref["x"]) and np.abs(T - ref["T"]).max() == 0.0 and trace.shape == ref["trace"].shape
                assert np.array_equal(trace[:, :6], ref["trace"][:, :6])
                _assert_nid(trace[:, 6], ref["trace"][:, 6])
            got = _run_threads([lambda k=k: solve(k) for k in range(len(bags))])
            for (T, x, costs, trace), (T1, x1, costs1, trace1) in zip(got, serial):
                assert np.array_equal(T, T1) and np.array_equal(x, x1) and np.array_equal(costs, costs1, equal_nan=True) and np.array_equal(trace, trace1, equal_nan=True)
    finally:
        V.set_solver_mode(0)
    # calibrate on two bags per thread
    pairs = [(0, 1), (1, 2), (2, 0)]
    params.max_outer_iterations, params.max_inner_iterations = 2, 15
    op.max_outer_iterations, op.max_inner_iterations = 2, 15

    def calibrate(k):
        a, b = pairs[k]
        calib = V.VisualCameraCalibration(cam, datasets[a] + datasets[b], params)
        T = w.call(calib.calibrate, bags[a]["T_init"])
        return T, calib.stats["total_evaluations"], [c for _, c in calib.trace]

    serial = [calibrate(k) for k in range(len(pairs))]
    for (T, evals, _), (a, b) in zip(serial, pairs):
        ref = O.calibrate(ocam, [(bags[i]["image"], bags[i]["points"], bags[i]["intensities"]) for i in (a, b)], bags[a]["T_init"], op)
        assert evals == ref["total_evaluations"] and np.abs(T - ref["T"]).max() < 1e-15
    got = _run_threads([lambda k=k: calibrate(k) for k in range(len(pairs))])
    for (T, evals, costs), (T1, evals1, costs1) in zip(got, serial):
        assert np.array_equal(T, T1) and evals == evals1 and np.array_equal(costs, costs1, equal_nan=True)
    w.assert_overlapped("solves")


def _case_error_isolation():
    """Failing calls on some threads, succeeding ones on others: every thread reads its own last-error message."""
    V, O = _libs()
    L = V.load_library()
    pr = util.random_problem("plumb_bob", n=40_000, seed=600)
    bcost = V.NIDCost(V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"]), V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), 16)
    hcost = _cost(V, pr)
    Tc = np.ascontiguousarray(pr["T"].T).reshape(16)
    msg_bspline = "context was created in B-spline mode; use vlcal_nid_evaluate_bspline"
    msg_pass = "poses_per_pass must be in [1, 8]"
    good = []
    for k in range(2):
        gpr = util.random_problem("plumb_bob", n=260_000, seed=610 + k)
        Ts = util.random_poses(gpr["T"], 8, seed=61 + k)
        cost = _cost(V, gpr)
        nid = cost.calculate_batch(Ts)
        _assert_nid(nid, _oracle_eval(O, gpr, Ts)[0])
        good.append((cost, Ts, nid))
    w = _Windows()

    def last_error():
        return L.vlcal_nid_last_error().decode()

    def hist_on_bspline():
        out, hist = np.empty(1), np.empty(256, dtype=np.int32)
        for _ in range(300):
            rc = w.call(L.vlcal_nid_evaluate, bcost.handle, _dp(Tc), 1, _dp(out), hist.ctypes.data)
            assert rc == _lib.ERR_INVALID_ARGUMENT and last_error() == msg_bspline, (rc, last_error())
        return last_error()

    def bad_poses_per_pass():
        for _ in range(300):
            with pytest.raises(V.VlcalError) as e:
                w.call(hcost.set_poses_per_pass, 0)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT and e.value.message == msg_pass
        return last_error()

    def succeed(cost, Ts, nid):
        def run():
            for _ in range(10):
                assert np.array_equal(w.call(cost.calculate_batch, Ts), nid, equal_nan=True)
            return last_error()
        return run

    errs = _run_threads([hist_on_bspline, bad_poses_per_pass, succeed(*good[0]), succeed(*good[1])])
    assert errs[0] == msg_bspline and errs[1] == msg_pass
    assert errs[2] not in (msg_bspline, msg_pass) and errs[3] not in (msg_bspline, msg_pass), errs
    w.assert_overlapped("errors")


def _case_churn():
    """Create, evaluate and destroy from every thread over several rounds, each bag on another thread every round, so that
    pooled blocks of every size class change hands; the idle main thread trims the pool between rounds."""
    V, O = _libs()
    L = V.load_library()
    specs = [(260_000, True), (60_000, True), (3_000, True), (40_000, False), (1, True)]
    bags = []
    for k, (n, f32) in enumerate(specs):
        pr = util.random_problem("plumb_bob", n=n, seed=700 + k, f32=f32)
        Ts = util.random_poses(pr["T"], 6, seed=70 + k)
        cost = _cost(V, pr)
        nid, hist = cost.calculate_batch(Ts, return_hist=True)
        cost.close()
        onid, ohist = _oracle_eval(O, pr, Ts)
        assert np.array_equal(hist, ohist)
        _assert_nid(nid, onid)
        bags.append((pr, Ts, nid, hist))
    w = _Windows()

    def body(pr, Ts, nid, hist):
        def run():
            cost = w.call(_cost, V, pr)
            n2, h2 = w.call(cost.calculate_batch, Ts, return_hist=True)
            n3 = w.call(cost.calculate_batch, Ts[::-1])
            w.call(cost.close)
            assert np.array_equal(n2, nid, equal_nan=True) and np.array_equal(h2, hist) and np.array_equal(n3, nid[::-1], equal_nan=True)
        return run

    for r in range(5):
        _run_threads([body(*bags[(k + r) % len(bags)]) for k in range(len(bags))])
        assert L.vlcal_nid_trim_memory() == _lib.OK
    w.assert_overlapped("churn")


_CASES = {
    "histograms": _case_histograms_k1p_and_round1,
    "score_poses": _case_score_poses_disjoint_lists,
    "mode_b": _case_mode_b,
    "legacy_stream": _case_legacy_stream_entry_points,
    "solves_auto_and_host": _case_solves,
    "errors": _case_error_isolation,
    "churn": _case_churn,
}

WORKER = r"""
import sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_gpu_concurrency as M
M._CASES[sys.argv[3]]()
print("CASE_OK", sys.argv[3])
"""


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(_CASES))
def test_threads(gpu, oracle, tmp_path, case):
    script = tmp_path / "concurrency_worker.py"
    script.write_text(WORKER)
    out = subprocess.run([sys.executable, str(script), ROOT, HERE, case], capture_output=True, text=True, timeout=CASE_TIMEOUT_S)
    assert out.returncode == 0 and f"CASE_OK {case}" in out.stdout, out.stdout[-4000:] + out.stderr[-6000:]
    inflight = [int(line.split()[2]) for line in out.stdout.splitlines() if line.startswith("INFLIGHT ")]
    assert inflight and min(inflight) >= 2, out.stdout
    print(out.stdout.strip())


# ---- C. the async pair, one thread ---------------------------------------------------------------------------------------


def _async_contexts(V):
    """A persistent-kernel-capable context, 64 bins, the double layout and the exact kernel of variant 1."""
    specs = [(60_000, 16, True, 0), (30_000, 64, True, 0), (20_000, 16, False, 0), (30_000, 16, True, 1)]
    out = []
    for k, (n, bins, f32, variant) in enumerate(specs):
        pr = util.random_problem("plumb_bob", n=n, seed=800 + k, f32=f32)
        out.append((pr, bins, _cost(V, pr, bins, variant), util.random_poses(pr["T"], 5, seed=80 + k)))
    return out


@pytest.mark.gpu
def test_async_on_four_contexts_waited_in_reverse_order(gpu, oracle):
    L = gpu.load_library()
    ctxs = _async_contexts(gpu)
    want = []
    for pr, bins, cost, Ts in ctxs:
        nid, hist = cost.calculate_batch(Ts, return_hist=True)
        onid, ohist = _oracle_eval(oracle, pr, Ts, bins)
        assert np.array_equal(hist, ohist)
        _assert_nid(nid, onid)
        want.append(nid)
    Tcs = [T_to_colmajor(Ts) for _, _, _, Ts in ctxs]
    for (_, _, cost, Ts), Tc in zip(ctxs, Tcs):
        assert L.vlcal_nid_evaluate_async(cost.handle, _dp(Tc), len(Ts)) == _lib.OK
    for k in reversed(range(len(ctxs))):
        out = np.full(len(Tcs[k]), -1.0)
        assert L.vlcal_nid_wait(ctxs[k][2].handle, _dp(out), None) == _lib.OK
        assert np.array_equal(out, want[k], equal_nan=True), k


@pytest.mark.gpu
def test_async_busy_and_idle_errors(gpu):
    L = gpu.load_library()
    pr, bins, cost, Ts = _async_contexts(gpu)[0]
    other = _cost(gpu, util.random_problem("plumb_bob", n=5_000, seed=899))
    want, want_other = cost.calculate_batch(Ts), other.calculate_batch(Ts)
    Tc = T_to_colmajor(Ts)
    out = np.empty(len(Ts))
    # nothing in flight
    assert L.vlcal_nid_wait(cost.handle, _dp(out), None) == _lib.ERR_INVALID_ARGUMENT
    assert L.vlcal_nid_last_error().decode() == "no evaluation in flight on this context"
    assert L.vlcal_nid_evaluate_async(cost.handle, _dp(Tc), len(Ts)) == _lib.OK
    busy = "an evaluation is already in flight on this context"
    assert L.vlcal_nid_evaluate_async(cost.handle, _dp(Tc), len(Ts)) == _lib.ERR_BUSY and L.vlcal_nid_last_error().decode() == busy
    assert L.vlcal_nid_evaluate(cost.handle, _dp(Tc), len(Ts), _dp(out), None) == _lib.ERR_BUSY and L.vlcal_nid_last_error().decode() == busy
    handles = (C.c_void_p * 1)(cost.handle)
    assert L.vlcal_nid_score_poses(handles, 1, _dp(Tc), len(Ts), _dp(out)) == _lib.ERR_BUSY and L.vlcal_nid_last_error().decode() == busy
    # another context evaluates meanwhile
    assert np.array_equal(other.calculate_batch(Ts), want_other, equal_nan=True)
    res = np.full(len(Ts), -1.0)
    assert L.vlcal_nid_wait(cost.handle, _dp(res), None) == _lib.OK
    assert np.array_equal(res, want, equal_nan=True)
    assert L.vlcal_nid_wait(cost.handle, _dp(res), None) == _lib.ERR_INVALID_ARGUMENT
    assert np.array_equal(cost.calculate_batch(Ts), want, equal_nan=True)


@pytest.mark.gpu
def test_wait_refuses_histograms_the_async_evaluation_did_not_compute(gpu, oracle):
    """A round-1 evaluate with histograms leaves them in the context's device buffer; a later _async computes none, so
    _wait must refuse hist_out rather than hand back the earlier histograms.  Same pose count both times, so the buffer
    is large enough either way."""
    L = gpu.load_library()
    pr = util.random_problem("plumb_bob", n=30_000, seed=850)
    cost = _cost(gpu, pr, 16, variant=1)
    T1 = util.random_poses(pr["T"], 4, seed=1)
    T2 = util.random_poses(pr["T"], 4, seed=2)
    P, nb = len(T1), 16 * 16
    nid1, hist1 = np.empty(P), np.zeros(P * nb, dtype=np.int32)
    assert L.vlcal_nid_evaluate(cost.handle, _dp(T_to_colmajor(T1)), P, _dp(nid1), hist1.ctypes.data) == _lib.OK
    want2, whist2 = cost.calculate_batch(T2, return_hist=True)
    _assert_nid(want2, _oracle_eval(oracle, pr, T2)[0])
    # T1's histograms again in the buffer, then T2 without histograms
    assert L.vlcal_nid_evaluate(cost.handle, _dp(T_to_colmajor(T1)), P, _dp(nid1), hist1.ctypes.data) == _lib.OK
    assert L.vlcal_nid_evaluate_async(cost.handle, _dp(T_to_colmajor(T2)), P) == _lib.OK
    nid2, hist2 = np.full(P, -1.0), np.full(P * nb, -1, dtype=np.int32)
    rc = L.vlcal_nid_wait(cost.handle, _dp(nid2), hist2.ctypes.data)
    stale = np.array_equal(hist2, hist1)
    assert rc == _lib.ERR_INVALID_ARGUMENT, f"wait returned {rc} with {'the previous evaluation' if stale else 'unrequested'} histograms"
    assert L.vlcal_nid_last_error().decode() == "histograms were not requested for the evaluation in flight"
    assert np.all(hist2 == -1)
    assert np.array_equal(nid2, want2, equal_nan=True)  # the scores are still delivered
    assert L.vlcal_nid_wait(cost.handle, _dp(nid2), None) == _lib.ERR_INVALID_ARGUMENT  # and the evaluation is over
    nid3, hist3 = cost.calculate_batch(T2, return_hist=True)
    assert np.array_equal(nid3, want2, equal_nan=True) and np.array_equal(hist3, whist2)
