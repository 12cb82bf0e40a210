"""Small workload that touches every kernel once (for compute-sanitizer memcheck / racecheck / initcheck)."""
import sys

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import direct_visual_lidar_calibration_b200 as V
import util

for model in util.MODELS:
    pr = util.random_problem(model, n=6000, seed=3)
    Ts = util.random_poses(pr["T"], 5, seed=1)
    cam = V.create_camera(model, pr["intrinsics"], pr["distortion"])
    data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
    cost = V.CostCalculatorNID(cam, data)
    a = cost.calculate_batch(Ts, return_hist=True)
    cost.set_kernel_variant(1)
    b = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(a[1], b[1])
    cost.reorder_for_pose(Ts[0])
    cost.set_kernel_variant(0)
    c = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(a[1], c[1])
    cost.debug_filter_check(Ts)
    V.ViewCulling(cam, (pr["W"], pr["H"])).cull_indices(pr["points"], pr["T"])
    from scipy.spatial.transform import Rotation

    tp = np.concatenate([Rotation.from_matrix(pr["T"][:3, :3]).as_quat(), pr["T"][:3, 3]])
    V.NIDCost(cam, data, 16).evaluate(tp[None])
pr = util.random_problem("plumb_bob", n=8000, seed=4)
cam = V.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
params = V.VisualCameraCalibrationParams()
params.max_inner_iterations, params.max_outer_iterations = 12, 2
V.VisualCameraCalibration(cam, [data, data], params).calibrate(pr["T"])  # host loop, two bags on two streams
V.set_solver_mode(1)  # one bag, host loop
V.VisualCameraCalibration(cam, [data], params).calibrate(pr["T"])
V.set_solver_mode(0)
print("SANITIZE_WORKLOAD_OK")
