"""The cross-rank score exchange (vlcal_nid_p2p_*, cudaIpc-shared mailboxes) at its edges, with several processes on one GPU.

Two implementations share one mailbox allocation and one exchange counter per PeerExchange:
  * round 1: the finalizing block of every round-1 launch on an attached context (nid_peer_allreduce): every
    calculate_batch with an exchange attached, and the host-loop solve with one bag per rank;
  * persistent: the persistent solve's (rank, bag) words (nid_persistent.cuh).
Each case runs tests/peer_exchange_worker.py under torchrun.  Rank 0 rebuilds every rank's bag in one process without an
exchange and checks every rank's result against it:
  * bit-equal: the exchanged value is 0.0 + v_0 + v_1 + ... in float64, v_r the single-process calculate_batch of rank
    r's bag; the bags' NIDs differ in magnitude so that the reversed order gives other bits (asserted for world >= 3);
  * the oracle: every bag's joint histograms equal the C oracle's, and the sum is within the parity tolerance of the
    oracle's sum;
  * solves: T, y, iterations, evaluations and the best-cost trace bit-equal to the single-process solves over all bags;
  * every rank returns identical bits.
Ranks that disagree on the solve path (a double-layout bag beside float4 ones, different bag counts) agree on the host
loop or refuse together (agree_solve_path in csrc/calibration.cu); a rank entering 3 s late stays within the default
timeout."""
import json
import os
import signal
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "peer_exchange_worker.py")

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _launch(world, cases, timeout=900, default_timeout=False):
    """Runs the worker with `world` ranks in its own session; on timeout the whole process group is killed.  Returns the
    parsed PX_CASE lines of rank 0."""
    env = dict(os.environ, OMP_NUM_THREADS="2", VLCAL_SYNC_TIMEOUT_MS="30000")
    if default_timeout:
        env.pop("VLCAL_SYNC_TIMEOUT_MS")
    cmd = [
        sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
        WORKER, *cases,
    ]
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, cwd=ROOT, start_new_session=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        out, err = proc.communicate()
        pytest.fail(f"world {world} {cases}: no result after {timeout} s\n{out[-3000:]}\n{err[-3000:]}")
    finally:
        try:  # nothing of the job may outlive the test
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
    assert proc.returncode == 0, f"world {world} {cases}: exit {proc.returncode}\n{out[-3000:]}\n{err[-3000:]}"
    return [json.loads(ln[len("PX_CASE "):]) for ln in out.splitlines() if ln.startswith("PX_CASE ")]


def _assert_all_true(results, expect_names):
    assert [r["case"] for r in results] == expect_names, results
    for r in results:
        checks = {k: v for k, v in r.items() if isinstance(v, bool)}
        assert checks, r
        assert all(checks.values()), r


@pytest.fixture(scope="module")
def built(gpu, oracle):
    """The library and the C oracle are built before any worker starts (rank 0 loads the oracle)."""
    return gpu


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_round1_exchange_equals_the_rank_order_sum(built, world):
    """calculate_batch on attached contexts: bins 16/33/56/128 x 1/7/8/9/17 poses (several launches, both slots), one call
    after another with new poses; then a double-layout bag, a fisheye bag and an empty bag (its NaN reaches every rank).
    World 8 fills the [8][2][8] mailbox with a few short calls."""
    cases = ["r1", "r1_mixed"]
    res = _launch(world, cases)
    _assert_all_true(res, cases)
    if world >= 3:
        assert res[0]["order_sensitive"]
    if world >= 4:
        assert res[1]["empty_bag_nan_on_every_rank"]


@pytest.mark.parametrize("world", [2, 3])
def test_round1_exchange_inside_a_host_loop_solve(built, world):
    """Solver mode 1, one bag per rank: every rank ends with the bits of the single-process mode-1 solve over all bags."""
    _assert_all_true(_launch(world, ["r1_solve"]), ["r1_solve"])


@pytest.mark.parametrize("world", [3, 4])
def test_persistent_exchange_several_bags_per_rank(built, world):
    """1, 2 and 8 bags per rank (world 4 x 8 bags: all 32 words of the mailbox) equal the single-process solves."""
    res = _launch(world, ["pk1", "pk2", "pk8"])
    _assert_all_true(res, ["pk1", "pk2", "pk8"])
    for r in res[:2]:
        assert "equals_single_process_one_launch" in r


def test_persistent_exchange_refuses_more_than_32_words(built):
    """World 5 x 7 bags is refused on every rank before the solve launches; the exchange stays usable (a round-1 case
    follows on the same PeerExchange, at a world that is not a power of two)."""
    _assert_all_true(_launch(5, ["pk_refuse_5x7", "r1_short"]), ["pk_refuse_5x7", "r1_short"])


def test_round1_and_persistent_exchanges_interleaved(built):
    """Round-1 calls and persistent solves alternate on one PeerExchange: they share its counter, tags and slots."""
    _assert_all_true(_launch(3, ["interleave"]), ["interleave_0_r1_short", "interleave_1_pk1", "interleave_2_r1_mixed", "interleave_3_pk2"])


def test_ranks_that_disagree_on_the_solve_path(built):
    """One rank's bag in the double layout: every rank takes the host loop (estimate_pose_on_costs, and calibrate with
    the exchange as default) and equals the single-process solve.  Different bag counts: every rank refuses, naming
    the ranks whose plan differs.  A round-1 case afterwards shows the ranks still in step."""
    cases = ["disagree_layout_costs", "disagree_layout_calibrate", "disagree_bag_counts", "disagree_bag_counts_calibrate", "r1_short"]
    _assert_all_true(_launch(3, cases), cases)


def test_a_rank_entering_late_stays_within_the_default_timeout(built):
    """One rank enters its first exchange 3 s after the others, round 1 and solve, with VLCAL_SYNC_TIMEOUT_MS unset."""
    _assert_all_true(_launch(3, ["r1_skew", "pk_skew"], default_timeout=True), ["r1_skew", "pk_skew"])
