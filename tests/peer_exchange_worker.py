"""torchrun worker for tests/test_gpu_peer_exchange_edges.py: the cross-rank score exchange (vlcal_nid_p2p_*) at its edges.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node W --master-addr 127.0.0.1 --master-port PORT \
        tests/peer_exchange_worker.py CASE [CASE ...]

Every rank sits on device 0 (handles over gloo; the GPU time-slices the ranks' spinning kernels) unless --spread is given
and the box has at least W GPUs.  Every rank's bag is a pure function of (case, call, rank), so rank 0 rebuilds all of
them in one process without an exchange and checks every rank's result against that reference.  Rank 0 prints one line
per case: `PX_CASE {json}` with the case's name, world and one boolean per property checked."""
import argparse
import datetime
import json
import os
import sys
import time

import numpy as np
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402

import direct_visual_lidar_calibration_b200 as V  # noqa: E402
from direct_visual_lidar_calibration_b200 import _lib  # noqa: E402
from direct_visual_lidar_calibration_b200 import calibration as VC  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402
from direct_visual_lidar_calibration_b200.distributed import PeerExchange  # noqa: E402

NID_TOL = 1e-12  # tests/test_gpu_parity.py: NID against the oracle

ap = argparse.ArgumentParser()
ap.add_argument("cases", nargs="+")
ap.add_argument("--spread", action="store_true", help="one rank per GPU when the box has enough of them")
args = ap.parse_args()

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
device = rank if (args.spread and V.device_count() >= world) else 0
dist.init_process_group("gloo", timeout=datetime.timedelta(minutes=10))
px = PeerExchange(device, rank, world)
px.connect_with_torch()


def gather(obj):
    out = [None] * world
    dist.all_gather_object(out, obj)
    return out


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def same_bits(a, b):
    """Bit-equal arrays; a NaN equals a NaN (its payload is not part of the result)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    m = ~np.isnan(a)
    return bool(np.array_equal(bits(a[m]), bits(b[m])))


def rank_sum(vs):
    """0.0 + v_0 + v_1 + ... in float64, in the given order."""
    total = np.zeros_like(np.asarray(vs[0], dtype=np.float64))
    for v in vs:
        total = total + v
    return total


# ---- bags ----------------------------------------------------------------------------------------------------------
# point counts far apart, so that the ranks' NIDs differ in magnitude and the order of the sum shows in its bits
SIZES = [30000, 400, 6000, 150, 12000, 900, 2500, 300]


def r1_bag(kind, call, r):
    """One round-1 bag: plain (float4, plumb_bob), double (double layout), fisheye or empty (0 points)."""
    model = "fisheye" if kind == "fisheye" else "plumb_bob"
    pr = util.random_problem(model, n=SIZES[(r + call) % len(SIZES)], seed=1000 * call + r, f32=kind != "double")
    if kind == "empty":
        pr["points"], pr["intensities"] = np.zeros((0, 4)), np.zeros(0)
    return pr


def r1_cost(pr, bins):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins), device=device)


def solve_bag(b, n_points, double=False):
    bag = S.make_bag("pinhole_640x480", "frustum", n_points + 700 * b, config_index=11, bag_index=b, scale=0.5)
    if double:  # intensities a float cannot hold: the bag uploads in the double layout
        bag["intensities"] = bag["intensities"] + 2.0**-40
    return bag


def solve_cam():
    b = solve_bag(0, 10)
    return V.create_camera(b["camera_model"], b["intrinsics"], b["distortion"])


def solve_cost(bag):
    return V.CostCalculatorNID(solve_cam(), V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"]), device=device)


T0 = S.perturb(S.gt_T_camera_lidar(), (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))


def solve_params(iters=30):
    p = V.VisualCameraCalibrationParams()
    p.max_inner_iterations = iters
    return p


def solve_summary(T, r, trace):
    return {"T": bits(T).tolist(), "y": bits([r["y"]]).tolist(), "it": r["num_iterations"], "ev": r["num_evaluations"], "trace": bits(trace).tolist()}


# ---- round-1 exchange: calculate_batch on attached contexts ------------------------------------------------------------
def r1_calls(mixed, short=False):
    """(bins, poses) of the calls of one case.  Plain: every bins x every pose count; world 8 a few short calls."""
    if mixed or short:
        return [(16, 9), (16, 17), (33, 8)]
    if world == 8:
        return [(16, 8), (16, 16), (16, 9), (128, 2)]
    return [(b, p) for b in (16, 33, 56, 128) for p in (1, 7, 8, 9, 17)]


def r1_kinds(mixed):
    if not mixed:
        return ["plain"] * world
    kinds = ["plain", "double", "fisheye", "empty"]  # rank 1: double layout, rank 2: another camera model, rank 3: no points
    return [kinds[r] if r < len(kinds) else "plain" for r in range(world)]


def case_r1(name, mixed=False, short=False, sleep_rank=None):
    kinds = r1_kinds(mixed)
    calls = r1_calls(mixed, short)
    mine = []
    for call, (bins, P) in enumerate(calls):
        pr = r1_bag(kinds[rank], call, rank)
        c = r1_cost(pr, bins)
        c.attach_peer_exchange(px)
        Ts = util.random_poses(pr["T"], P, seed=77 + call, rot_deg=1.0, trans=0.05)
        if sleep_rank == rank and call == 0:
            time.sleep(3.0)  # this rank enters its first exchange 3 s after the others
        mine.append(c.calculate_batch(Ts))
        c.close()
    every = gather([bits(v).tolist() for v in mine])
    res = {"case": name, "world": world}
    if rank == 0:
        from oracle import oracle as O

        ranks_identical = all(every[r] == every[0] for r in range(world))
        exact = hist_ok = oracle_ok = True
        order_sensitive = False
        nan_everywhere = None
        for call, (bins, P) in enumerate(calls):
            got = np.asarray(every[0][call], dtype=np.uint64).view(np.float64)
            vs, ovs = [], []
            for r in range(world):
                pr = r1_bag(kinds[r], call, r)
                c = r1_cost(pr, bins)  # no exchange: this process alone
                Ts = util.random_poses(pr["T"], P, seed=77 + call, rot_deg=1.0, trans=0.05)
                v, h = c.calculate_batch(Ts, return_hist=True)
                ocam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
                ov = []
                for p in range(P):
                    onid, ohist = O.nid_calculate(ocam, pr["image"], pr["points"], pr["intensities"], bins, c.max_fov, Ts[p])
                    hist_ok = hist_ok and bool(np.array_equal(h[p], ohist))
                    ov.append(onid)
                c.close()
                vs.append(v)
                ovs.append(np.array(ov))
            ref = rank_sum(vs)
            exact = exact and same_bits(got, ref)
            oref = rank_sum(ovs)
            oracle_ok = oracle_ok and bool(np.array_equal(np.isnan(got), np.isnan(oref)) and np.all(np.abs(got - oref)[~np.isnan(oref)] < world * NID_TOL))
            order_sensitive = order_sensitive or not same_bits(ref, rank_sum(vs[::-1]))
            if "empty" in kinds:
                nan_everywhere = bool(np.all(np.isnan(got))) if nan_everywhere is None else nan_everywhere and bool(np.all(np.isnan(got)))
        res.update(ranks_identical=ranks_identical, equals_rank_order_sum=exact, hist_equals_oracle=hist_ok, sum_close_to_oracle=oracle_ok)
        if world >= 3 and "empty" not in kinds:
            res["order_sensitive"] = order_sensitive  # two addends commute: only three or more can show the order
        if nan_everywhere is not None:
            res["empty_bag_nan_on_every_rank"] = nan_everywhere
    return res


# ---- solves ---------------------------------------------------------------------------------------------------------
def distributed_solve(bags_per_rank, mode, n_points, double_rank=None):
    """This rank's bags [rank*B, (rank+1)*B), attached exchange, one inner solve."""
    mine = [solve_cost(solve_bag(rank * bags_per_rank + k, n_points, double=rank == double_rank)) for k in range(bags_per_rank)]
    for c in mine:
        c.attach_peer_exchange(px)
    V.set_solver_mode(mode)
    trace = []
    try:
        T, r = VC.estimate_pose_on_costs(mine, T0, solve_params(), callback=lambda T, c: trace.append(c))
        out = solve_summary(T, r, trace)
    except _lib.VlcalError as e:
        out = {"error": e.code, "message": e.message}
    finally:
        V.set_solver_mode(0)
        for c in mine:
            c.attach_peer_exchange(None)
            c.close()
    return out


def reference_solves(n_bags, n_points, double_rank=None, bags_per_rank=1):
    """Rank 0 alone: every bag in one process, host loop (mode 1) and, where one launch holds them, persistent (mode 3)."""
    costs = [solve_cost(solve_bag(b, n_points, double=double_rank is not None and b // bags_per_rank == double_rank)) for b in range(n_bags)]
    refs = []
    modes = [1] + ([3] if n_bags <= 8 and double_rank is None else [])
    for mode in modes:
        V.set_solver_mode(mode)
        trace = []
        T, r = VC.estimate_pose_on_costs(costs, T0, solve_params(), callback=lambda T, c: trace.append(c))
        refs.append(solve_summary(T, r, trace))
    V.set_solver_mode(0)
    for c in costs:
        c.close()
    return refs


def case_solve(name, bags_per_rank, mode, n_points, double_rank=None, sleep_rank=None):
    if sleep_rank == rank:
        time.sleep(3.0)
    out = distributed_solve(bags_per_rank, mode, n_points, double_rank)
    every = gather(out)
    res = {"case": name, "world": world, "bags_per_rank": bags_per_rank}
    if rank == 0:
        res["no_error"] = all("error" not in e for e in every)
        if not res["no_error"]:
            res["errors"] = [e.get("message") for e in every]
        res["ranks_identical"] = all(e == every[0] for e in every)
        refs = reference_solves(world * bags_per_rank, n_points, double_rank, bags_per_rank)
        res["equals_single_process_host_loop"] = every[0] == refs[0]
        if len(refs) > 1:
            res["equals_single_process_one_launch"] = every[0] == refs[1]
    dist.barrier()
    return res


def case_refused(name, bags_of_rank, n_points, need):
    """Every rank must refuse the solve with VLCAL_ERR_UNSUPPORTED and a message containing `need`."""
    B = bags_of_rank(rank)
    mine = [solve_cost(solve_bag(rank * 8 + k, n_points)) for k in range(B)]
    for c in mine:
        c.attach_peer_exchange(px)
    try:
        VC.estimate_pose_on_costs(mine, T0, solve_params(5))
        out = {"code": 0, "message": ""}
    except _lib.VlcalError as e:
        out = {"code": e.code, "message": e.message}
    for c in mine:
        c.attach_peer_exchange(None)
        c.close()
    every = gather(out)
    res = {"case": name, "world": world}
    if rank == 0:
        res["refused_on_every_rank"] = all(e["code"] == _lib.ERR_UNSUPPORTED and need in e["message"] for e in every)
        res["messages"] = sorted({e["message"] for e in every})
    return res


def calib_bags(n_points, double_rank, counts):
    """Rank r's bags for calibrate: counts[r] bags; rank double_rank's in the double layout."""
    first = sum(counts[:rank])
    return [solve_bag(first + k, n_points, double=rank == double_rank) for k in range(counts[rank])]


def run_calibrate(bags):
    params = solve_params(25)
    params.max_outer_iterations = 2
    data = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    calib = V.VisualCameraCalibration(solve_cam(), data, params, device=device)
    T = calib.calibrate(T0)
    return {"T": bits(T).tolist(), "trace": bits([c for _, c in calib.trace]).tolist()}


def case_calibrate(name, n_points, double_rank, counts, need=None):
    """calibrate() with the exchange set as default: agrees (one bag each) or refuses on every rank (bag counts differ)."""
    px.set_default(True)
    try:
        out = run_calibrate(calib_bags(n_points, double_rank, counts))
    except _lib.VlcalError as e:
        out = {"code": e.code, "message": e.message}
    finally:
        px.set_default(False)
    every = gather(out)
    res = {"case": name, "world": world}
    if rank == 0:
        if need is not None:
            res["refused_on_every_rank"] = all(e.get("code") == _lib.ERR_UNSUPPORTED and need in e.get("message", "") for e in every)
        else:
            res["no_error"] = all("code" not in e for e in every)
            res["ranks_identical"] = all(e == every[0] for e in every)
            allbags = [solve_bag(b, n_points, double=double_rank is not None and b == double_rank) for b in range(world)]
            V.set_solver_mode(1)
            res["equals_single_process_host_loop"] = every[0] == run_calibrate(allbags)
            V.set_solver_mode(0)
    dist.barrier()
    return res


CASES = {
    "r1": lambda: case_r1("r1"),
    "r1_mixed": lambda: case_r1("r1_mixed", mixed=True),
    "r1_short": lambda: case_r1("r1_short", short=True),
    "r1_skew": lambda: case_r1("r1_skew", short=True, sleep_rank=world - 1),
    "r1_solve": lambda: case_solve("r1_solve", 1, 1, 6000),
    "pk1": lambda: case_solve("pk1", 1, 3, 6000),
    "pk2": lambda: case_solve("pk2", 2, 3, 4000),
    "pk8": lambda: case_solve("pk8", 8, 3, 1500),
    "pk_skew": lambda: case_solve("pk_skew", 1, 0, 6000, sleep_rank=world - 1),
    "pk_refuse_5x7": lambda: case_refused("pk_refuse_5x7", lambda r: 7, 600, "world x local bags must be <= 32"),
    "disagree_layout_costs": lambda: case_solve("disagree_layout_costs", 1, 0, 6000, double_rank=1),
    "disagree_layout_calibrate": lambda: case_calibrate("disagree_layout_calibrate", 6000, 1, [1] * world),
    "disagree_bag_counts": lambda: case_refused("disagree_bag_counts", lambda r: 2 if r == 0 else 1, 3000, "solve plans differ (rank(s) " + ", ".join(str(r) for r in range(1, world)) + " against rank 0"),
    "disagree_bag_counts_calibrate": lambda: case_calibrate("disagree_bag_counts_calibrate", 3000, None, [2] + [1] * (world - 1), need="solve plans differ"),
}

for case in args.cases:
    if case == "interleave":  # round-1 calls and persistent solves alternating on one PeerExchange
        for i, step in enumerate(["r1_short", "pk1", "r1_mixed", "pk2"]):
            res = CASES[step]()
            if rank == 0:
                res["case"] = f"interleave_{i}_{step}"
                print("PX_CASE " + json.dumps(res), flush=True)
        continue
    res = CASES[case]()
    if rank == 0:
        print("PX_CASE " + json.dumps(res), flush=True)
    dist.barrier()

dist.barrier()
px.close()
dist.destroy_process_group()
