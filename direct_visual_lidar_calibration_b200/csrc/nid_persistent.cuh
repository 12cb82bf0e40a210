// nid_persistent.cuh -- K1p: the NID hot path as ONE persistent cooperative kernel per inner solve (sm_90a).
//
// Replaces, for a whole dfo::NelderMead<6> inner solve (reference: include/dfo/nelder_mead.hpp:32-101 driving
// CostCalculatorNID::calculate, src/vlcal/calib/cost_calculator_nid.cpp:21-67, through the objective of
// src/vlcal/calib/visual_camera_calibration.cpp:103-119), the round-1 scheme "one launch per Nelder-Mead batch + host
// round trip" (a launch ramp, a serial tail and a host gap for every one of the ~115 batches of a C2 solve).
//
// One launch, grid = one 768-thread block per SM, all co-resident (cooperative launch, so the waits below cannot deadlock);
// tile k (64 consecutive points of the tile-ordered cloud) belongs to warp k mod W of its bag for the whole solve.
// Per Nelder-Mead batch:
//   (A) every block scores the batch's P <= 8 candidate poses on its tiles -- lean fp32 filter, two points per packed
//       two interleaved points per lane (lean_filter.cuh, lean_filter2.cuh), with the exact fp64 recheck for the ~2-3 % of point-poses
//       near a decision edge (exact_classify.cuh), privatised shared-memory histograms -- and merges its non-zero bins,
//       its marginals and its inlier counts into the global accumulators (red.global), then arrives (one fence per block);
//   (B) EVERY block waits for the arrivals and reduces every (bag, pose) accumulator to its NID score itself (:54-64; all
//       entropy terms in parallel, then per item the canonical summation order of nid_finalize, so a score is a function of
//       the histogram alone); the accumulators rotate over three buffers that are zeroed two batches ahead;
//   (C) world > 1: one block per item stores the score, as two tagged 8-byte words, into the mailboxes of the other ranks
//       (NVLink peer stores) and every block polls its own rank's mailbox for the remote words; then all blocks add the
//       world x bags contributions per pose in (rank, bag) order -- the joint objective sum_bags NID (:105-110),
//       bit-identical everywhere -- and warp 0 steps the Nelder-Mead state machine REDUNDANTLY in the block's shared memory
//       (warp-parallel over the simplex coordinates, nm_warp_step below; same operations in the same order as
//       NmMachine::step) and computes the next candidates' poses T = init_T * Expmap(x) (:104), three lanes per candidate,
//       while the other warps clear the histogram copies.  No broadcast of poses, no host, no launch.
// The same kernel in pose-list mode (no step (C): the next 8 poses come from a device array, and an owner block per
// (bag, pose) finalizes behind the scoring blocks, which run up to two chunks ahead) serves batched evaluation
// (vlcal_nid_evaluate) and the pose-grid search (vlcal_nid_score_poses): one launch for any number of poses.
//
// Several bags per GPU: the grid is partitioned over the bags in proportion to their sizes (one tail for all bags).
#pragma once

#include <cfloat>
#include <cstdint>

#include "exact_classify.cuh"
#include "lean_filter.cuh"
#include "lean_filter2.cuh"
#include "nid_kernels.cuh"
#include "nm_machine.cuh"

namespace vlcal {

// Launch shape: ONE block of 768 threads per SM (24 warps, <= 85 registers: 768 threads fill the register file).  Three
// blocks of 256 threads hold the same 24 warps, but the warp scheduler prefers higher warp slots, so the three blocks of
// an SM finish their equal slices at different times and every Nelder-Mead batch waits for the slowest; one block also
// merges once instead of three times and arrives once.
constexpr int PK_THREADS = 768;
constexpr int PK_WARPS = PK_THREADS / 32;
constexpr int PK_MAX_POSES = 8;
constexpr int PK_MAX_BAGS = 8;
constexpr int PK_MAX_WORDS = 256;  // world x bags x 8 score words per batch, one polling thread each
constexpr int PK_QUEUE = 64;
constexpr int PK_MAX_BINS = 32;  // nb <= 1024
constexpr int PK_MARG_STRIDE = 2 * PK_MAX_BINS + 32;  // ints per (bag, pose) record of PkArgs::gmarg
constexpr int PK_STAMP_SLOTS = 8;
constexpr unsigned int PK_TILE_ROWS = 4;
// Tile ring: every warp streams its tiles through PK_RING shared-memory slots filled by per-lane 16-byte cp.async copies.
// PK_RING - 1 tiles are in flight; every slot more takes 24 KB of the SM's L1 for shared memory.
constexpr int PK_RING = 2;
// Equirectangular batches of nearby poses: every pose but the anchor as a first-order update from it (classify_lean2_delta);
// 0: every pose through the plain classifier (A/B build, `make alt`)
#ifndef PK_DELTA_POSES
#define PK_DELTA_POSES 1
#endif
// dynamic shared memory of the block's tile rings: PK_WARPS x PK_RING slots of one 32*k-point tile (float4 rows)
__host__ __device__ constexpr unsigned int pk_ring_bytes(int k) { return static_cast<unsigned int>(PK_WARPS * PK_RING * 32 * k * 16); }

// score exchange: every double travels as two 8-byte words {32 data bits | 32-bit sequence tag} (an aligned 8-byte store
// is never torn, so the data is its own arrival flag).  w[slot][(rank * n_bags + bag) * 8 + pose][lo, hi]
struct PkMailbox {
  unsigned long long w[2][PK_MAX_WORDS][2];
};

struct PkBag {
  const float4* points;
  const uint8_t* bin_image;
  unsigned int n;
  int block_begin, block_count;  // blocks [block_begin, block_begin + block_count) of the grid work on this bag
};

// Nelder-Mead solve: initial state in device memory (every block copies it into its shared memory once) ...
struct PkSolve {
  NmMachine nm;  // after NmMachine::begin on the host: first batch pending
  double init_T[16];
};
// ... and the outcome in MAPPED PINNED HOST memory, written by block 0 (no device-to-host copy, the host polls done_host)
struct PkResult {
  NmMachine nm;                   // final state (result_x, result_y, converged, counters)
  unsigned long long batches;     // Nelder-Mead batches executed
  unsigned long long poses;       // poses scored (speculative ones included)
  int trace_count;                // reference-order evaluations written to the trace (may exceed the capacity: truncated)
  int pad_;
};

// 64-byte aligned: with the kernel's parameter block at 8-byte alignment, ptxas allocates registers differently and the
// plumb_bob K = 4 instance spills 28 bytes instead of 16 (and reloads 148 instead of 20), omnidir K = 2 reloads 120
// bytes instead of 100
struct alignas(64) PkArgs {
  // camera + image geometry (shared by all bags of the launch: one camera, equal image sizes)
  int width, height, bins, nb;
  double cos_fov;
  CameraParams cam;
  FastCam fast;
  LeanCam lean;
  int n_bags;
  PkBag bag[PK_MAX_BAGS];
  int copies;  // shared-memory histogram copies per block
  unsigned int ring_off;  // byte offset of the tile rings in dynamic shared memory (128-byte aligned, behind the histogram copies)
  // work source
  const PkSolve* solve;      // Nelder-Mead mode when non-null
  PkResult* result_host;     // Nelder-Mead mode: outcome (mapped pinned host memory)
  double* trace_host;        // [trace_cap][NM_MAX_N + 1] evaluations (x, y) in the reference's order, for the callback replay
  int trace_cap;
  const double* poses_in;    // pose-list mode: [n_total][12] row-major 3x4 [R|t]
  int n_total;
  int chunk;                 // pose-list mode: poses per pass over the cloud (8; smaller only for roofline measurements)
  double* scores_out;        // pose-list mode: [n_total] (sum over bags of this launch)
  int* hist_out;             // optional [n_total][nb] (bag 0 only)
  // synchronisation scratch (zero on entry)
  int* ghist;                // [3][n_bags][8][nb] joint accumulators (three rotating buffers in Nelder-Mead mode, two in pose-list mode)
  int* gmarg;                // [3][n_bags][8][PK_MARG_STRIDE] Nelder-Mead mode: marginals (image bins, then lidar bins) and [2*PK_MAX_BINS] the inlier count
  unsigned int* arrive;      // [3][PK_MAX_BAGS]
  unsigned int* fin_done;    // [2]
  unsigned int* abort_flag;  // set by any block that timed out: everybody leaves
  PkMailbox* box[P2P_MAX_RANKS];  // box[r]: rank r's mailbox as mapped here (self included; world == 1: local scratch)
  int world, rank;
  unsigned long long* seq_counter;  // persistent exchange counter (device word of the peer exchange; local scratch otherwise)
  unsigned long long timeout_ns;
  int* error_host;                  // mapped host word: 1 = wait timed out
  unsigned long long* done_host;    // mapped host word: receives done_seq when the results are visible
  unsigned long long done_seq;
  unsigned long long* stamps;       // optional [cap][PK_STAMP_SLOTS] globaltimer stamps per batch
  int stamps_cap;
  // [4]: passes (batches / chunks) that took the delta step and their poses (block 0), point-poses deferred to the exact
  // path in the other passes and in those passes (every block)
  unsigned long long* delta_stats;
  unsigned long long* block_times;  // optional [grid][4]: every block's {enter, hist zeroed, main loop done, arrived} stamps of batch block_times_batch
  int block_times_batch;
};

struct PkShared {
  NmMachine nm;
  double init_T[16];
  double pose64[PK_MAX_POSES][12];
  float4 pose32[PK_MAX_POSES][4];  // rows: [R00 R01 R02 t0] [R10 R11 R12 t1] [R20 R21 R22 t2] [max|t| 0 0 0]
  // delta step: [1, P) the poses other than the anchor in candidate order, relative to it, as lean_delta_pose writes them,
  // with .z / .w of row 3 holding the pose's histogram byte offset and its bit of a tile's deferral mask (pk_delta_rows);
  // [0] holds the anchor: its pose32 rows 0-2 and {index, -, offset, bit}
  float4 dpose[PK_MAX_POSES][4];
  int delta_on;                    // the batch takes the delta step (block-uniform)
  double ys[PK_MAX_POSES];
  double parts[PK_MAX_WORDS];
  double fin_out[PK_WARPS];  // NIDs of the items one finalizer round covers (Nelder-Mead mode)
  int bmarg[PK_MAX_POSES][2 * PK_MAX_BINS];  // Nelder-Mead mode: this block's marginals of the batch (zero between batches)
  float tmax;
  int n_poses;
  int wait_failed;
  int trace_count;
  unsigned long long poses_scored;
  unsigned long long seq_base;
  int s_cnt[PK_WARPS];
  unsigned int q_idx[PK_WARPS][PK_QUEUE];
  unsigned char q_pose[PK_WARPS][PK_QUEUE];
  int q_cnt[PK_WARPS];  // fill count of each warp's queue
  uint4 ring_state[PK_WARPS];  // tile ring bookkeeping of each warp: {next tile, tiles left in the pass, tile step, slot}
  unsigned int deferred[PK_WARPS][2];  // point-poses each warp deferred to the exact path: plain passes, delta passes
};

// ---- small PTX helpers ---------------------------------------------------------------------------------------------

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// histogram increment, under `if (counted)`: ptxas emits BSSY / BRA / ATOMS.POPC.INC / BSYNC (lanes of a warp that hit the
// same bin are merged by the hardware; predication is not available for this form, hence the branch).  An unconditional
// red.shared.add of a 0 / 1 register (one ATOMS.ADD, no branch, but same-bin lanes serialise) measured slower.
__device__ __forceinline__ void red_shared_inc(unsigned int smem_addr) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(smem_addr) : "memory");
}

// 1-byte read-only gather under a predicate; -1 when off (the sign doubles as the "counted" flag one pose later)
__device__ __forceinline__ int ldg_u8_or_neg(bool pred, const uint8_t* p) {
  int v;
  asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %1, 0;\n\tmov.u32 %0, -1;\n\t@q ld.global.nc.u8 %0, [%2];\n\t}" : "=r"(v) : "r"(static_cast<int>(pred)), "l"(p));
  return v;
}

// ---- warp-parallel Nelder-Mead step --------------------------------------------------------------------------------
// NmMachine::step / loop_top (nm_machine.cuh) executed by one warp on a machine that lives in shared memory: lane d owns
// column d of the simplex (d = 0 the values, d = 1..n the coordinates).  Every element sees the same operations in the
// same order as in the serial code (the serial loops run over independent columns), so the state is bit-identical; only
// the sort permutation and the scalar decisions are computed redundantly by every lane.

__device__ __forceinline__ void nm_warp_observe(NmMachine& s, int lane, const double* vertex, double y) {
  const int k = s.n_obs;
  if (lane >= 1 && lane <= s.n) s.obs_x[k][lane - 1] = vertex[lane];
  __syncwarp();
  if (lane == 0) {
    s.obs_y[k] = y;
    s.n_obs = k + 1;
    s.num_evaluations++;
  }
  __syncwarp();
}

__device__ __forceinline__ void nm_warp_finish(NmMachine& s, int lane) {
  if (lane >= 1 && lane <= s.n) s.result_x[lane - 1] = s.x[0][lane];  // :99
  if (lane == 0) {
    s.result_y = s.x[0][0];  // :100
    s.n_cand = 0;
    s.phase = 3;
  }
  __syncwarp();
}

// M: compile-time bound of the simplex size m = n + 1 (7 for the 6-D pose solve; the generic instance covers n <= 8)
template <int M>
static __device__ void nm_warp_loop_top(NmMachine& s, int lane) {
  const int n = s.n, m = n + 1;
  if (s.it >= s.params.max_iterations) {
    nm_warp_finish(s, lane);
    return;
  }
  __syncwarp();
  if (lane == 0) s.num_iterations = s.it;  // :50
  // :51 std::sort = libstdc++ insertion sort on the values.  It is a STABLE sort whenever `<` is a strict weak order on the
  // values, i.e. when none of them is NaN: row i then lands at rank_i = #{j : v_j < v_i} + #{j < i : v_j == v_i}, which
  // lane i computes with m compares.  With a NaN among the values the result depends on the insertion order itself and
  // the literal restatement below (every lane walks the insertion sort in registers) takes over.
  const double my_v = lane < m ? s.x[lane][0] : 0.0;
  const bool any_nan = __any_sync(0xffffffffu, lane < m && my_v != my_v);
  int ord[M];  // ord[k] = row of the old simplex that becomes row k
  if (!any_nan) {
    int rank = 0;
#pragma unroll
    for (int j = 0; j < M; j++) {
      const double vj = __shfl_sync(0xffffffffu, my_v, j);
      if (j < m) rank += (vj < my_v || (j < lane && vj == my_v)) ? 1 : 0;
    }
    int inv[M];  // inv[i] = new row of old row i
#pragma unroll
    for (int i = 0; i < M; i++) inv[i] = __shfl_sync(0xffffffffu, rank, i);
#pragma unroll
    for (int k = 0; k < M; k++) {
      int o = 0;
#pragma unroll
      for (int i = 0; i < M; i++)
        if (i < m && inv[i] == k) o = i;
      ord[k] = o;
    }
  } else {
    double val[M];
#pragma unroll
    for (int i = 0; i < M; i++) {
      val[i] = i < m ? s.x[i][0] : 0.0;
      ord[i] = i;
    }
#pragma unroll
    for (int i = 1; i < M; i++) {
      if (i < m) {
        const double v = val[i];
        const int o = ord[i];
        // unguarded linear insert: walk left while v < element; the first branch (v < *first) moves to the front
        bool cont = true;
        int cnt = 0;
#pragma unroll
        for (int k = M - 1; k >= 0; k--) {
          if (k < i) {
            cont = cont && (v < val[k]);
            cnt += cont ? 1 : 0;
          }
        }
        const int pos = (v < val[0]) ? 0 : i - cnt;
#pragma unroll
        for (int k = M - 1; k >= 1; k--) {
          if (k <= i && k > pos) {
            val[k] = val[k - 1];
            ord[k] = ord[k - 1];
          }
        }
#pragma unroll
        for (int k = 0; k < M; k++) {
          if (k <= i && k == pos) {
            val[k] = v;
            ord[k] = o;
          }
        }
      }
    }
  }
  __syncwarp();
  const bool mine = lane < m;
  {
    double tmp[M];
#pragma unroll
    for (int k = 0; k < M; k++) tmp[k] = (mine && k < m) ? s.x[ord[k]][lane] : 0.0;
    __syncwarp();
#pragma unroll
    for (int k = 0; k < M; k++)
      if (mine && k < m) s.x[k][lane] = tmp[k];
  }
  __syncwarp();
  // :52-55, :105-113 convergence: sum over the coordinates of sum_k (x_k - mean)^2
  double var = 0.0;
  if (mine) {
    xd sum(0.0);
    for (int k = 0; k < m; k++) sum = sum + xd(s.x[k][lane]);
    const xd mean = sum / xd(static_cast<double>(m));
    xd acc(0.0);
    for (int k = 0; k < m; k++) {
      const xd e = xd(s.x[k][lane]) - mean;
      acc = acc + e * e;
    }
    var = acc.v;
  }
  xd total(0.0);
  for (int d = 1; d < m; d++) total = total + xd(__shfl_sync(0xffffffffu, var, d));
  if (total.v < s.params.convergence_var_thresh) {
    if (lane == 0) s.converged = 1;
    __syncwarp();
    nm_warp_finish(s, lane);
    return;
  }
  // :57, :60, :66, :75  xo, xr, xe, xc -> cand = {xr, xe, xc, xo} (xo scored only when s.score_centroid)
  if (mine) {
    xd sum(0.0);
    for (int k = 0; k < n; k++) sum = sum + xd(s.x[k][lane]);
    const xd xo = sum / xd(static_cast<double>(n));
    const xd diff = xo - xd(s.x[n][lane]);
    s.cand[0][lane] = (xo + xd(s.params.alpha) * diff).v;
    s.cand[1][lane] = (xo + xd(s.params.gamma) * diff).v;
    s.cand[2][lane] = (xo + xd(s.params.rho) * diff).v;
    s.cand[3][lane] = xo.v;
  }
  if (lane == 0) {
    s.n_cand = s.score_centroid ? 4 : 3;
    s.phase = 1;
  }
  __syncwarp();
}

__device__ __forceinline__ void nm_warp_loop_top_dispatch(NmMachine& s, int lane) {
  if (s.n == 6) nm_warp_loop_top<7>(s, lane);
  else nm_warp_loop_top<NM_MAX_N + 1>(s, lane);
}

// consume the scores ys[0..n_cand) of the pending batch (one warp, all 32 lanes call)
static __device__ __noinline__ void nm_warp_step(NmMachine& s, const double* ys, int lane) {
  const int n = s.n, m = n + 1;
  const int phase = s.phase;
  const bool mine = lane < m;
  __syncwarp();
  if (lane == 0) {
    s.n_obs = 0;
    s.num_batches++;
    s.num_evaluations_computed += s.n_cand;
  }
  __syncwarp();
  if (phase == 0) {
    for (int k = 0; k < m; k++) {
      if (mine) s.x[k][lane] = lane == 0 ? ys[k] : s.cand[k][lane];
      __syncwarp();
      nm_warp_observe(s, lane, s.x[k], ys[k]);
    }
    nm_warp_loop_top_dispatch(s, lane);
  } else if (phase == 1) {
    const double f0 = s.x[0][0], fn1 = s.x[n - 1][0], fn = s.x[n][0];
    // scores of cand = {xr, xe, xc, xo}
    const double yr = ys[0], ye = ys[1], yc = ys[2];
    const bool score_centroid = s.score_centroid != 0;
    __syncwarp();
    if (lane == 0) {
      s.cand[0][0] = yr;
      if (score_centroid) s.cand[3][0] = ys[3];
    }
    __syncwarp();
    if (score_centroid) {
      nm_warp_observe(s, lane, s.cand[3], ys[3]);  // :58 evaluated, never used in a decision
    } else {
      if (lane == 0) s.num_evaluations++;  // :58 requested by the reference; nobody reads its value
      __syncwarp();
    }
    nm_warp_observe(s, lane, s.cand[0], yr);  // :61
    bool shrink = false;
    if (f0 <= yr && yr < fn1) {  // :63-64
      if (mine) s.x[n][lane] = s.cand[0][lane];
    } else if (yr < f0) {  // :65-73 expansion
      if (lane == 0) s.cand[1][0] = ye;
      __syncwarp();
      nm_warp_observe(s, lane, s.cand[1], ye);
      const int pick = (ye < yr) ? 1 : 0;
      if (mine) s.x[n][lane] = s.cand[pick][lane];
    } else {  // :74-86
      if (lane == 0) s.cand[2][0] = yc;
      __syncwarp();
      nm_warp_observe(s, lane, s.cand[2], yc);
      if (yc < fn) {
        if (mine) s.x[n][lane] = s.cand[2][lane];
      } else {
        shrink = true;
        if (mine) {
          const xd x0(s.x[0][lane]);
          for (int j = 1; j < m; j++) {
            const double v = (x0 + xd(s.params.rho) * (xd(s.x[j][lane]) - x0)).v;  // :82 (rho, not sigma)
            s.x[j][lane] = v;
            s.cand[j - 1][lane] = v;
          }
        }
        if (lane == 0) {
          s.n_cand = n;
          s.phase = 2;
        }
      }
    }
    __syncwarp();
    if (!shrink) {
      if (lane == 0) s.it++;
      __syncwarp();
      nm_warp_loop_top_dispatch(s, lane);
    }
  } else if (phase == 2) {
    for (int j = 1; j < m; j++) {
      if (lane == 0) s.x[j][0] = ys[j - 1];
      __syncwarp();
      nm_warp_observe(s, lane, s.x[j], ys[j - 1]);
    }
    if (lane == 0) s.it++;
    __syncwarp();
    nm_warp_loop_top_dispatch(s, lane);
  }
  __syncwarp();
}

// T = init_T * Expmap(x) (visual_camera_calibration.cpp:104) for the n_cand <= 8 pending candidates, by one warp: lane 3c + i
// computes row i of candidate c.  Same operations in the same order as se3_expmap_gtsam_hd + isometry_mul_hd (se3_math.cuh)
// for every matrix entry (the rows of R, t and of the product are independent of each other), so the poses are
// bit-identical to the serial code, which ran on one lane in every Nelder-Mead batch.
static __device__ __noinline__ void pk_poses_of_candidates(PkShared& sh, int n_cand, int lane) {
  const int c = lane / 3, i = lane - 3 * c;
  const bool active = c < n_cand;
  double* Erow = &sh.parts[0];  // scratch [8][3][4]: rows of E = Expmap(x) (sh.parts is free between the score sum and the next batch)
  if (active) {
    const double* xi = &sh.nm.cand[c][1];
    const xd w[3] = {xd(xi[0]), xd(xi[1]), xd(xi[2])};
    const xd v[3] = {xd(xi[3]), xd(xi[4]), xd(xi[5])};
    const xd theta2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2];
    const xd zero(0.0);
    const xd W[3][3] = {{zero, -w[2], w[1]}, {w[2], zero, -w[0]}, {-w[1], w[0], zero}};
    xd Ri[3], ti;
    if (theta2.v <= DBL_EPSILON) {  // nearZero: R = I + W, t = v
#pragma unroll
      for (int j = 0; j < 3; j++) {
        xd e(0.0);
#pragma unroll
        for (int r = 0; r < 3; r++)
          if (r == i) e = W[r][j] + xd(r == j ? 1.0 : 0.0);
        Ri[j] = e;
      }
      ti = i == 0 ? v[0] : (i == 1 ? v[1] : v[2]);
    } else {
      const xd theta = xsqrt(theta2);
      const xd sin_theta(sin(theta.v));
      const xd s2(sin((theta / xd(2.0)).v));
      const xd one_minus_cos = xd(2.0) * s2 * s2;
      // K = W / theta entry by entry: the six non-zero entries are +-w_k / theta -- IEEE division is sign-symmetric, so three
      // divisions give the same bits as the nine of the serial code -- and 0 / theta = +0
      const xd k0 = w[0] / theta, k1 = w[1] / theta, k2 = w[2] / theta;
      const xd K[3][3] = {{zero, -k2, k1}, {k2, zero, -k0}, {-k1, k0, zero}};
      xd Krow[3];
#pragma unroll
      for (int j = 0; j < 3; j++) Krow[j] = i == 0 ? K[0][j] : (i == 1 ? K[1][j] : K[2][j]);
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const xd KKij = Krow[0] * K[0][j] + Krow[1] * K[1][j] + Krow[2] * K[2][j];
        Ri[j] = xd(i == j ? 1.0 : 0.0) + sin_theta * Krow[j] + one_minus_cos * KKij;
      }
      const xd wv = (w[0] * v[0] + w[1] * v[1]) + w[2] * v[2];
      const xd cr[3] = {w[1] * v[2] - w[2] * v[1], w[2] * v[0] - w[0] * v[2], w[0] * v[1] - w[1] * v[0]};
      const xd Rc = Ri[0] * cr[0] + Ri[1] * cr[1] + Ri[2] * cr[2];
      const xd ci = i == 0 ? cr[0] : (i == 1 ? cr[1] : cr[2]);
      const xd wi = i == 0 ? w[0] : (i == 1 ? w[1] : w[2]);
      ti = (ci - Rc + wi * wv) / theta2;
    }
    double* e = Erow + (c * 3 + i) * 4;
    e[0] = Ri[0].v, e[1] = Ri[1].v, e[2] = Ri[2].v, e[3] = ti.v;
  }
  __syncwarp();
  if (active) {
    // row i of init_T * E:  linear = Ra Rb, translation = Ra tb + ta   (isometry_mul_hd)
    const double* E0 = Erow + (c * 3) * 4;
    const xd a0(sh.init_T[i]), a1(sh.init_T[i + 4]), a2(sh.init_T[i + 8]), a3(sh.init_T[i + 12]);
    double T[4];
#pragma unroll
    for (int j = 0; j < 3; j++) T[j] = (a0 * xd(E0[j]) + a1 * xd(E0[4 + j]) + a2 * xd(E0[8 + j])).v;
    T[3] = ((a0 * xd(E0[3]) + a1 * xd(E0[7]) + a2 * xd(E0[11])) + a3).v;
#pragma unroll
    for (int j = 0; j < 4; j++) sh.pose64[c][4 * i + j] = T[j];
    sh.pose32[c][i] = make_float4(static_cast<float>(T[0]), static_cast<float>(T[1]), static_cast<float>(T[2]), static_cast<float>(T[3]));
  }
  __syncwarp();
  if (active && i == 0) {
    const double tmax = fmax(fmax(fabs(sh.pose64[c][3]), fabs(sh.pose64[c][7])), fabs(sh.pose64[c][11]));
    sh.pose32[c][3] = make_float4(nextafterf(static_cast<float>(tmax), INFINITY), 0.f, 0.f, 0.f);  // max|t| rounded up
  }
  __syncwarp();
}

// pose-list mode: pose k of the chunk from its row-major 3x4 doubles
__device__ __forceinline__ void pk_pose_from_list(PkShared& sh, int k, const double* __restrict__ T) {
  double tmax = 0.0;
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 4; c++) sh.pose64[k][4 * r + c] = T[4 * r + c];
    sh.pose32[k][r] = make_float4(static_cast<float>(T[4 * r]), static_cast<float>(T[4 * r + 1]), static_cast<float>(T[4 * r + 2]), static_cast<float>(T[4 * r + 3]));
    tmax = fmax(tmax, fabs(T[4 * r + 3]));
  }
  sh.pose32[k][3] = make_float4(nextafterf(static_cast<float>(tmax), INFINITY), 0.f, 0.f, 0.f);
}

static __device__ __noinline__ int pk_delta_anchor(const PkShared& sh, int n, int lane) {
  // lean_delta_anchor's scores, lane 4i + r taking row r of pose i against every pose, then the lowest-index minimum
  const int i = lane >> 2, r = lane & 3;
  float s = 0.0f;
  if (r < 3 && i < n) {
    const float4 a = sh.pose32[i][r];
    for (int j = 0; j < n; j++) {
      const float4 b = sh.pose32[j][r];
      s = fmaxf(s, lean_delta_row_spread(&a.x, &b.x));
    }
  }
  s = fmaxf(s, __shfl_xor_sync(0xffffffffu, s, 1));
  s = fmaxf(s, __shfl_xor_sync(0xffffffffu, s, 2));
  float m = i < n ? s : INFINITY;
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const unsigned int hit = __ballot_sync(0xffffffffu, r == 0 && i < n && s == m);
  const int anc = hit != 0u ? (__ffs(static_cast<int>(hit)) - 1) >> 2 : 0;
  return anc;
}

// warp 0, once the batch's n poses are in sh.pose64 / sh.pose32: the anchor (lean_delta_anchor), the rows of the delta
// step and the batch's gate (every pose within lean_delta_pose's spread of the anchor, and at least two poses).  K: points
// per lane of the tile loop (a tile's deferral mask holds bit p * K + j for point j of pose p); nb: bins per histogram.
template <int K>
__device__ __forceinline__ void pk_delta_rows(PkShared& sh, int n, int nb, int lane) {
  __syncwarp();
  const int anc = pk_delta_anchor(sh, n, lane);
  // lane k in [1, n): the k-th of the other poses in candidate order
  bool close = true;
  if (lane >= 1 && lane < n) {
    const int p = lane - (lane <= anc ? 1 : 0);
    close = lean_delta_pose(sh.pose64[p], sh.pose64[anc], &sh.dpose[lane][0].x);
    sh.dpose[lane][3].z = __uint_as_float(4u * static_cast<unsigned int>(p * nb));
    sh.dpose[lane][3].w = __uint_as_float(1u << (p * K));
  }
  const bool on = __all_sync(0xffffffffu, close) && n >= 2;
  if (lane < 3) sh.dpose[0][lane] = sh.pose32[anc][lane];
  if (lane == 0) {
    sh.delta_on = on ? 1 : 0;
    sh.dpose[0][3] = make_float4(__int_as_float(anc), 0.0f, __uint_as_float(4u * static_cast<unsigned int>(anc * nb)), __uint_as_float(1u << (anc * K)));
  }
  __syncwarp();
}

// ---- block-uniform waits with a timeout ------------------------------------------------------------------------------

// thread 0 spins until *counter >= expected; returns false (for every thread) if the launch is being aborted
__device__ __forceinline__ bool pk_wait_counter(const PkArgs& a, PkShared& sh, const unsigned int* counter, unsigned int expected) {
  if (threadIdx.x == 0) {
    int failed = 0;
    const unsigned long long t0 = global_ns();
    unsigned int spins = 0;
    while (ld_acquire_u32(counter) < expected) {
      if ((++spins & 255u) == 0) {
        if (ld_acquire_u32(a.abort_flag) != 0u) {
          failed = 1;
          break;
        }
        if (global_ns() - t0 > a.timeout_ns) {
          atomicExch(a.abort_flag, 1u);
          if (a.error_host) *reinterpret_cast<volatile int*>(a.error_host) = 1;
          failed = 1;
          break;
        }
      }
    }
    sh.wait_failed = failed;
  }
  __syncthreads();
  const bool ok = sh.wait_failed == 0;
  __syncthreads();
  return ok;
}

// ---- the NID of one accumulated joint histogram, by a whole block (cost_calculator_nid.cpp:54-64) -----------------------
// Same arithmetic and the same canonical summation order as nid_finalize (nid_kernels.cuh): staged p*log(p + 1e-6) terms,
// lane l of warp 0 adds terms l, l+32, ... in ascending order, then a fixed xor tree -- a function of the histogram alone.
// g: this (bag, pose)'s accumulator [nb]; zeroed again on the way.  scratch: >= nb + 2*bins doubles + 2*bins ints.
constexpr int PK_FIN_CH = (PK_MAX_BINS * PK_MAX_BINS + PK_THREADS - 1) / PK_THREADS;  // joint bins per thread

static __device__ __noinline__ double pk_block_nid(PkShared& sh, int* __restrict__ g, int nb, int bins, int* __restrict__ hist_out, int* scratch) {
  double* s_term = reinterpret_cast<double*>(scratch);  // [nb]
  double* s_mterm = s_term + nb;                        // [2*bins]
  int* s_marg = reinterpret_cast<int*>(s_mterm + 2 * bins);  // [2*bins]: image marginal, then lidar marginal
  __shared__ double s_nid;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int i = t; i < 2 * bins; i += PK_THREADS) s_marg[i] = 0;
  __syncthreads();
  int c[PK_FIN_CH];
  int part = 0;
#pragma unroll
  for (int m = 0; m < PK_FIN_CH; m++) {
    const int k = m * PK_THREADS + t;
    c[m] = k < nb ? __ldcg(g + k) : 0;
  }
#pragma unroll
  for (int m = 0; m < PK_FIN_CH; m++) {
    const int k = m * PK_THREADS + t;
    if (c[m]) {
      atomicAdd(&s_marg[k % bins], c[m]);         // hist_image[image_bin]   (:50)
      atomicAdd(&s_marg[bins + k / bins], c[m]);  // hist_points[lidar_bin]  (:51)
      part += c[m];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) sh.s_cnt[warp] = part;
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int w = 0; w < PK_WARPS; w++) total += sh.s_cnt[w];
  const double sum = static_cast<double>(total);  // :54 sum = hist_image.sum()
#pragma unroll
  for (int m = 0; m < PK_FIN_CH; m++) {
    const int k = m * PK_THREADS + t;
    if (k < nb) {
      const double pr = static_cast<double>(c[m]) / sum;
      s_term[k] = entropy_term(pr);  // :59-61
      if (hist_out) hist_out[k] = c[m];
      if (c[m]) g[k] = 0;
    }
  }
  for (int f = t; f < 2 * bins; f += PK_THREADS) {
    const double pm = static_cast<double>(s_marg[f]) / sum;
    s_mterm[f] = entropy_term(pm);
  }
  __threadfence();  // the zeroed accumulator must be visible before anybody can see the score
  __syncthreads();
  if (warp == 0) {
    double t_rs = 0.0, t_r = 0.0, t_s = 0.0;
    for (int k = lane; k < nb; k += 32) t_rs += s_term[k];
    for (int k = lane; k < bins; k += 32) {
      t_r += s_mterm[k];
      t_s += s_mterm[bins + k];
    }
    const double Hrs = -warp_tree_sum(t_rs), Hr = -warp_tree_sum(t_r), Hs = -warp_tree_sum(t_s);
    if (lane == 0) {
      const double MI = Hr + Hs - Hrs;  // :63
      s_nid = (Hrs - MI) / Hrs;         // :64 (NaN when there are no inliers, as in the reference)
    }
  }
  __syncthreads();
  return s_nid;
}

// Nelder-Mead mode: the NIDs of `count` (bag, pose) items at once, by the whole block -- every block finalizes every item of
// the batch itself instead of waiting for an owner block to publish it.  The blocks merged the marginals and the inlier
// count next to the joint histogram (gmarg), so all count * (nb + 2 bins) entropy terms are independent: one L2 round trip,
// one division and one logarithm per thread, one barrier, then per item the canonical sum of pk_block_nid (lane l of one
// warp adds terms l, l+32, ... in ascending order, then the xor tree) -- identical values.  Reads the accumulators only (this
// mode's triple-buffered accumulators are zeroed two batches ahead).
// Item j is (bag ib, pose ip) = ((first + j) / n_poses, (first + j) % n_poses).
// scratch: count * pk_fin_item_bytes(nb, bins) bytes; out[j] <- NID of item j (written by lane 0 of warp j; count <= PK_WARPS).
__host__ __device__ constexpr int pk_fin_item_bytes(int nb, int bins) { return 8 * (nb + 2 * bins); }

static __device__ __noinline__ void pk_block_nid_items(const int* __restrict__ gbuf, const int* __restrict__ mbuf, int first, int count, int n_poses, int nb, int bins, void* scratch,
                                                       double* out) {
  double* s_term = static_cast<double*>(scratch);  // [count][nb + 2*bins]: joint terms, image-marginal terms, lidar-marginal terms
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int per_item = nb + 2 * bins;
  const int n_terms = count * per_item;
  // two terms per round and thread, loads first: the divisions and logarithms of a thread's terms interleave
  for (int base = t; base < n_terms; base += 2 * PK_THREADS) {
    int c[2];
    double sum[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int idx = base + u * PK_THREADS;
      c[u] = 0, sum[u] = 1.0;
      if (idx < n_terms) {
        const int j = idx / per_item, r = idx - j * per_item;
        const int item = first + j, ib = item / n_poses, ip = item - ib * n_poses;
        const size_t rec = static_cast<size_t>(ib) * PK_MAX_POSES + ip;
        const int* m = mbuf + rec * PK_MARG_STRIDE;
        c[u] = r < nb ? __ldcg(gbuf + rec * nb + r) : __ldcg(m + (r - nb));
        sum[u] = static_cast<double>(__ldcg(m + 2 * PK_MAX_BINS));  // :54 sum = hist_image.sum()
      }
    }
    double e[2];
#pragma unroll
    for (int u = 0; u < 2; u++) e[u] = entropy_term(static_cast<double>(c[u]) / sum[u]);  // :59-61
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int idx = base + u * PK_THREADS;
      if (idx < n_terms) s_term[idx] = e[u];
    }
  }
  __syncthreads();
  if (warp < count) {
    const double* tj = s_term + static_cast<size_t>(warp) * per_item;
    double t_rs = 0.0, t_r = 0.0, t_s = 0.0;
    for (int k = lane; k < nb; k += 32) t_rs += tj[k];
    for (int k = lane; k < bins; k += 32) {
      t_r += tj[nb + k];
      t_s += tj[nb + bins + k];
    }
    const double Hrs = -warp_tree_sum(t_rs), Hr = -warp_tree_sum(t_r), Hs = -warp_tree_sum(t_s);
    if (lane == 0) {
      const double MI = Hr + Hs - Hrs;  // :63
      out[warp] = (Hrs - MI) / Hrs;     // :64 (NaN when there are no inliers, as in the reference)
    }
  }
  __syncthreads();
}

// thread b (< n_bags) spins until bag b's arrival counter reaches expected_per_block * (its block count); false for every
// thread if the launch is being aborted
__device__ __forceinline__ bool pk_wait_arrivals(const PkArgs& a, const unsigned int* counters, unsigned int rounds) {
  int failed = 0;
  if (static_cast<int>(threadIdx.x) < a.n_bags) {
    const unsigned int expected = rounds * static_cast<unsigned int>(a.bag[threadIdx.x].block_count);
    const unsigned long long t0 = global_ns();
    unsigned int spins = 0;
    while (ld_acquire_u32(counters + threadIdx.x) < expected) {
      if ((++spins & 255u) == 0) {
        if (ld_acquire_u32(a.abort_flag) != 0u) {
          failed = 1;
          break;
        }
        if (global_ns() - t0 > a.timeout_ns) {
          atomicExch(a.abort_flag, 1u);
          if (a.error_host) *reinterpret_cast<volatile int*>(a.error_host) = 1;
          failed = 1;
          break;
        }
      }
    }
  }
  return __syncthreads_or(failed) == 0;
}

// ---- hot loop -----------------------------------------------------------------------------------------------------------

__device__ __forceinline__ void sts_u32(unsigned int addr, unsigned int v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_u8(unsigned int addr, unsigned int v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned int lds_u32(unsigned int addr) {
  unsigned int v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int lds_u8(unsigned int addr) {
  unsigned int v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ int atoms_add(unsigned int addr, int v) {
  int old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(addr), "r"(v) : "memory");
  return old;
}

struct PkWarp {
  unsigned int hist_addr;  // shared-memory byte address of this warp's histogram copy [P][nb]
  // the warp's queue of deferred (point, pose) pairs, as shared-window byte addresses (generic pointers would turn the pushes into
  // generic stores / generic atomics)
  unsigned int q_idx;   // unsigned int [PK_QUEUE]
  unsigned int q_pose;  // unsigned char [PK_QUEUE]
  unsigned int q_cnt;   // int: shared-memory copy of qn (the lanes claim queue slots from it)
  int qn;
  int lane;
  unsigned int lt_mask;
};

// the per-bag pointers in registers (PkArgs::bag[] is indexed by a runtime bag number: every use would be an indexed LDC)
struct PkBagRegs {
  const float4* points;
  const uint8_t* bin_image;
};

// the call takes the warp's state by value: a reference would force PkWarp into local memory for the whole hot loop
template <int MODEL>
__device__ __noinline__ void pk_drain32_impl(const PkArgs& a, const PkShared& sh, const float4* points, const uint8_t* bin_image, unsigned int hist_addr, unsigned int q_idx, unsigned int q_pose,
                                             int lane, int first, int count) {
  if (lane < count) {  // one deferred (point, pose) per lane, exact path
    const unsigned int i = lds_u32(q_idx + 4u * static_cast<unsigned int>(first + lane));
    const int p = static_cast<int>(lds_u8(q_pose + static_cast<unsigned int>(first + lane)));
    const float4 q = __ldg(points + i);
    const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, sh.pose64[p], q.x, q.y, q.z);
    if (pix >= 0) {
      const int ib = __ldg(bin_image + pix);  // :43,:46 via the pre-binned image
      const unsigned int addr = hist_addr + 4u * static_cast<unsigned int>(p * a.nb + ib + lidar_bin_of(q.w, a.bins) * a.bins);
      asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(addr) : "memory");  // :49 hist(image_bin, lidar_bin)++
    }
  }
}

template <int MODEL>
__device__ __forceinline__ void pk_drain32(const PkArgs& a, const PkShared& sh, const PkBagRegs& B, const PkWarp& w, int first, int count) {
  pk_drain32_impl<MODEL>(a, sh, B.points, B.bin_image, w.hist_addr, w.q_idx, w.q_pose, w.lane, first, count);
}

// one tile = 32*K consecutive points starting at `tile`, swept over the P poses of the batch; the image-bin gathers of
// pose p stay in flight while pose p+1 is classified and are consumed by the histogram increments one iteration later.
// PARTIAL: the tile may reach past `end` (only the single-row tiles at the end of a warp's slice).
// DPOSE: the kernel instance carries the equirectangular delta step (nid_persistent_kernel).
template <int MODEL, int K, bool PARTIAL, bool DPOSE = false>
__device__ __forceinline__ void pk_tile(const PkArgs& a, const PkShared& sh, const PkBagRegs& B, int n_poses, PkWarp& w, unsigned int tile, unsigned int end, const float4 (&q)[K]) {
  float px[K], py[K], pz[K], dl[K];
  unsigned int lb[K];
  const float tmax = sh.tmax;
  const bool valid0 = !PARTIAL || (tile + w.lane < end);  // PARTIAL tiles have K == 1
#pragma unroll
  for (int j = 0; j < K; j++) {
    px[j] = q[j].x, py[j] = q[j].y, pz[j] = q[j].z;
    dl[j] = (5.25f * F32_U) * (fabsf(q[j].x) + fabsf(q[j].y) + fabsf(q[j].z) + tmax);
    lb[j] = w.hist_addr + 4u * static_cast<unsigned int>(lidar_bin_of(q[j].w, a.bins) * a.bins);
  }
  constexpr bool PACKED = !PARTIAL && (K % 2 == 0) && LeanPacked<MODEL>::value;
  F2 X2[(K + 1) / 2], Y2[(K + 1) / 2], Z2[(K + 1) / 2], D2[(K + 1) / 2];
  if constexpr (PACKED) {
#pragma unroll
    for (int j = 0; j < K; j += 2) {
      X2[j / 2] = f2_pack(px[j], px[j + 1]), Y2[j / 2] = f2_pack(py[j], py[j + 1]);
      Z2[j / 2] = f2_pack(pz[j], pz[j + 1]), D2[j / 2] = f2_pack(dl[j], dl[j + 1]);
    }
  }
  unsigned int unc_mask = 0u, unc_bit = 1u;  // deferred verdicts of this tile: bit p * K + j
  int pend_bin[K];  // image bin of the previous pose's verdict, -1 = not counted
#pragma unroll
  for (int j = 0; j < K; j++) pend_bin[j] = -1;
  unsigned int pend_off = 0;
  // :49 hist(image_bin, lidar_bin)++ for the previous pose's verdicts
  auto count_previous = [&]() {
#pragma unroll
    for (int j = 0; j < K; j++)
      if (pend_bin[j] >= 0) red_shared_inc(lb[j] + pend_off + 4u * static_cast<unsigned int>(pend_bin[j]));
  };
  // the image-bin gathers of a pose's accepted verdicts (off: the byte offset of its histogram), consumed by count_previous
  // one pose later
  auto gather = [&](unsigned int off, const bool (&acc)[K], const int (&pix)[K]) {
    pend_off = off;
#pragma unroll
    for (int j = 0; j < K; j++) pend_bin[j] = ldg_u8_or_neg(acc[j], B.bin_image + pix[j]);
  };
  // verdicts of points j, j + 1 from the packed classifier
  auto record2 = [&](const LeanVerdict2& v, int j, bool (&acc)[K], int (&pix)[K]) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      acc[j + h] = v.accept[h];
      if (v.uncertain[h]) unc_mask |= unc_bit << (j + h);
      pix[j + h] = v.idx[h];
    }
  };
  // Equirectangular batches whose poses lie close together (sh.delta_on, set with the poses): the anchor (pk_delta_rows)
  // goes first through the plain classifier, the other poses are first-order updates from it (classify_lean2_delta; bound
  // and guards in lean_filter.cuh).  Each row carries its pose's histogram offset and deferral bit, so every count and
  // every deferral lands in its own pose's slot.
  constexpr bool DELTA = DPOSE && PK_DELTA_POSES && PACKED && MODEL == CAM_EQUIRECTANGULAR;
  const bool delta_tile = DELTA && sh.delta_on;
  if (delta_tile) {
    if constexpr (DELTA) {
      LeanAnchor2 an[K / 2];
      {
        bool acc[K];
        int pix[K];
        const float4 r0 = sh.dpose[0][0], r1 = sh.dpose[0][1], r2 = sh.dpose[0][2], slot = sh.dpose[0][3];
        const float Pm[12] = {r0.x, r0.y, r0.z, r1.x, r1.y, r1.z, r2.x, r2.y, r2.z, r0.w, r1.w, r2.w};
        unc_bit = __float_as_uint(slot.w);
#pragma unroll
        for (int j = 0; j < K; j += 2)
          record2(classify_lean2_anchor<MODEL>(a.fast, a.lean, a.width, Pm, X2[j / 2], Y2[j / 2], Z2[j / 2], D2[j / 2], an[j / 2]), j, acc, pix);
        gather(__float_as_uint(slot.z), acc, pix);
      }
      for (int k = 1; k < n_poses; k++) {
        bool acc[K];
        int pix[K];
        const float4 q0 = sh.dpose[k][0], q1 = sh.dpose[k][1], q2 = sh.dpose[k][2];
        const float2 q3 = *reinterpret_cast<const float2*>(&sh.dpose[k][3].x);
        const float Q[14] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y};
        LeanVerdict2 v[K / 2];
#pragma unroll
        for (int j = 0; j < K; j += 2) v[j / 2] = classify_lean2_delta<MODEL>(a.lean, a.width, Q, X2[j / 2], Y2[j / 2], Z2[j / 2], D2[j / 2], an[j / 2]);
        // the pose's slot, read once its verdicts are in (not held across the classifier)
        const float2 slot = *reinterpret_cast<const float2*>(&sh.dpose[k][3].z);
        unc_bit = __float_as_uint(slot.y);
#pragma unroll
        for (int j = 0; j < K; j += 2) record2(v[j / 2], j, acc, pix);
        count_previous();
        gather(__float_as_uint(slot.x), acc, pix);
      }
      count_previous();
    }
  } else {
    for (int p = 0; p <= n_poses; p++) {
      bool acc[K];
      int pix[K];
      if (p < n_poses) {
        const float4 r0 = sh.pose32[p][0], r1 = sh.pose32[p][1], r2 = sh.pose32[p][2];
        const float Pm[12] = {r0.x, r0.y, r0.z, r1.x, r1.y, r1.z, r2.x, r2.y, r2.z, r0.w, r1.w, r2.w};
        if constexpr (PACKED) {
#pragma unroll
          for (int j = 0; j < K; j += 2)  // two points per instruction on the packed fp32 pipe (lean_filter2.cuh)
            record2(classify_lean2<MODEL>(a.fast, a.lean, a.width, Pm, X2[j / 2], Y2[j / 2], Z2[j / 2], D2[j / 2]), j, acc, pix);
        } else {
#pragma unroll
          for (int j = 0; j < K; j++) {
            const LeanVerdict v = classify_lean<MODEL>(a.fast, a.lean, a.width, Pm, px[j], py[j], pz[j], dl[j]);
            acc[j] = PARTIAL ? (v.accept & valid0) : v.accept;
            const bool unc = PARTIAL ? (v.uncertain & valid0) : v.uncertain;
            if (unc) unc_mask |= unc_bit << j;
            pix[j] = v.idx;
          }
        }
        unc_bit <<= K;
      }
      count_previous();
      if (p < n_poses) gather(4u * static_cast<unsigned int>(p * a.nb), acc, pix);
    }
  }
  // Deferred (point, pose) pairs of this tile -> the warp's queue for the exact path.  Doing this once per tile instead of inside the pose loop
  // matters: with ~3 % of the point-poses deferred, SOME lane of the 32 x K has one in 5 of 6 pose steps, so the ballot /
  // queue code would run almost every step instead of once per tile.
  // Usual case (the tile defers at most 32 pairs): one warp prefix sum gives every lane the queue slots of its pairs.
  // Otherwise: one ballot per round.
  const int cnt = __popc(unc_mask);
  const int total = __reduce_add_sync(0xffffffffu, cnt);
  if (w.lane == 0 && total > 0) atoms_add(static_cast<unsigned int>(__cvta_generic_to_shared(&sh.deferred[threadIdx.x >> 5][delta_tile ? 1 : 0])), total);
  if (total > 0 && total <= 32) {
    if (w.qn + total > PK_QUEUE) {  // make room first (qn > 32 here): the last 32 queued pairs go to the exact path now
      pk_drain32<MODEL>(a, sh, B, w, w.qn - 32, 32);
      w.qn -= 32;
      if (w.lane == 0) sts_u32(w.q_cnt, static_cast<unsigned int>(w.qn));
      __syncwarp();
    }
    if (unc_mask != 0u) {
      // the queue slots of this lane's pairs: one shared-memory atomic on the warp's fill count (the order of the queue does
      // not matter -- histogram increments commute -- so no prefix sum over the lanes is needed)
      int pos = atoms_add(w.q_cnt, cnt);
      do {
        const int b = __ffs(static_cast<int>(unc_mask)) - 1;  // bit p * K + j
        unc_mask &= unc_mask - 1u;
        sts_u32(w.q_idx + 4u * static_cast<unsigned int>(pos), tile + static_cast<unsigned int>(b % K) * 32u + static_cast<unsigned int>(w.lane));
        sts_u8(w.q_pose + static_cast<unsigned int>(pos), static_cast<unsigned int>(b / K));
        pos++;
      } while (unc_mask != 0u);
    }
    w.qn += total;
    __syncwarp();
    if (w.qn >= 32) {
      pk_drain32<MODEL>(a, sh, B, w, w.qn - 32, 32);
      w.qn -= 32;
      if (w.lane == 0) sts_u32(w.q_cnt, static_cast<unsigned int>(w.qn));
      __syncwarp();
    }
  } else if (total > 32) {
    while (__any_sync(0xffffffffu, unc_mask != 0u)) {
      const bool have = unc_mask != 0u;
      const int b = __ffs(static_cast<int>(unc_mask)) - 1;
      unc_mask &= unc_mask - 1u;
      const unsigned int m = __ballot_sync(0xffffffffu, have);
      if (have) {
        const int pos = w.qn + __popc(m & w.lt_mask);
        sts_u32(w.q_idx + 4u * static_cast<unsigned int>(pos), tile + static_cast<unsigned int>(b % K) * 32u + static_cast<unsigned int>(w.lane));
        sts_u8(w.q_pose + static_cast<unsigned int>(pos), static_cast<unsigned int>(b / K));
      }
      w.qn += __popc(m);
      __syncwarp();
      if (w.qn >= 32) {
        pk_drain32<MODEL>(a, sh, B, w, w.qn - 32, 32);
        w.qn -= 32;
        __syncwarp();
      }
    }
    if (w.lane == 0) sts_u32(w.q_cnt, static_cast<unsigned int>(w.qn));
    __syncwarp();
  }
}

template <int K>
__device__ __forceinline__ void pk_load_tile(const float4* __restrict__ pts, unsigned int tile, unsigned int end, int lane, float4 (&q)[K]) {
#pragma unroll
  for (int j = 0; j < K; j++) {
    const unsigned int i = tile + j * 32 + lane;
    q[j] = make_float4(0.f, 0.f, -1.f, 0.f);
    if (i < end) q[j] = __ldg(pts + i);
  }
}

// points [tpos, end) of the cloud in single-row tiles, the next row in flight
template <int MODEL>
__device__ __forceinline__ void pk_rows(const PkArgs& a, const PkShared& sh, const PkBagRegs& B, int n_poses, PkWarp& w, unsigned int tpos, unsigned int end) {
  const int lane = w.lane;
  float4 q1[1], n1[1];
  if (tpos < end) pk_load_tile<1>(B.points, tpos, end, lane, q1);
  while (tpos < end) {
    const bool more = tpos + 32u < end;
    if (more) pk_load_tile<1>(B.points, tpos + 32u, end, lane, n1);
    pk_tile<MODEL, 1, true>(a, sh, B, n_poses, w, tpos, end, q1);
    tpos += 32u;
    if (more) q1[0] = n1[0];
  }
}

// ---- tile ring: per warp, PK_RING shared-memory slots of one tile each, filled by cp.async -------------------------------
// Every lane copies its own K rows of a tile (16-byte cp.async.cg: L2 -> shared memory, L1 left to the image gathers) and
// later reads back exactly those rows, so a lane only waits for its own copies (cp.async.wait_group): no mbarrier, no
// cross-lane handover, no uniform operands in the tile loop.  One commit group per tile (empty past the end of the pass);
// the slot refilled at a step is the one read at the step before, whose rows the pose loop has consumed by then, so
// PK_RING - 1 tiles are in flight while one is swept over the poses.

// this lane's rows of one tile -> its rows of a slot, as one commit group (no copy when !valid: an empty group)
template <int K>
__device__ __forceinline__ void pk_ring_fill(unsigned int slot_lane, const float4* src_lane, bool valid) {
  if (valid) {
#pragma unroll
    for (int j = 0; j < K; j++) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot_lane + 512u * j), "l"(src_lane + 32 * j) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// shared-memory address of this lane's first row in slot s of the calling warp's ring (recomputed from threadIdx where
// needed: cheaper than keeping it in a register across the pose loop)
template <int K>
__device__ __forceinline__ unsigned int pk_ring_slot(const PkArgs& a, unsigned int smem_base, unsigned int s) {
  return smem_base + a.ring_off + ((threadIdx.x >> 5) * PK_RING + s) * (32u * K * 16u) + 16u * (threadIdx.x & 31u);
}

__device__ __forceinline__ void sts_v4(unsigned int addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(unsigned int addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

__device__ __forceinline__ float pk_tmax(const PkShared& sh, int n_poses) {
  float tm = 0.f;
  for (int p = 0; p < n_poses; p++) tm = fmaxf(tm, sh.pose32[p][3].x);
  return tm;
}

__device__ __forceinline__ void pk_stamp(const PkArgs& a, unsigned long long batch, int slot) {
  if (a.stamps && batch < static_cast<unsigned long long>(a.stamps_cap)) a.stamps[batch * PK_STAMP_SLOTS + slot] = global_ns();
}

// stamps per batch: 0 block 0 enters the batch, 1 block 0 main loop done, 2 block 0 merged + arrived,
//                   3 finalizer of item 0: all blocks arrived, 4 finalizer of item 0: score published,
//                   5 block 0: all scores seen, 7 block 0: Nelder-Mead machine stepped, 6 block 0: next poses ready
// DPOSE: this instance carries the equirectangular delta step (instantiated for equirectangular, K = 2 only; the host
// picks it for Nelder-Mead solves and for pose lists with a chunk inside the gate, see pk_pick).  Its anchor state costs
// registers in the whole kernel, so the plain instance stays for everything else.
// blk, grid: this block's index within the blocks that run the launch's work, and their number -- the whole grid for
// nid_persistent_kernel, one solve's group for nid_persistent_solves_kernel
template <int MODEL, int K, bool DPOSE>
__device__ __forceinline__ void pk_run(const PkArgs& a, const PkArgs& grp, const unsigned int blk, const unsigned int grid) {
  extern __shared__ __align__(128) int smem_hist[];
  __shared__ PkShared sh;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const bool solve_mode = grp.solve != nullptr;

  // block -> bag, warp -> its interleaved tiles of the bag's cloud
  int bag = 0;
  while (bag + 1 < grp.n_bags && static_cast<int>(blk) >= grp.bag[bag + 1].block_begin) bag++;
  const PkBag& Bc = grp.bag[bag];
  PkBagRegs B;
  B.points = Bc.points;
  B.bin_image = Bc.bin_image;
  const unsigned int bag_n = Bc.n, bag_block_begin = static_cast<unsigned int>(Bc.block_begin), bag_block_count = static_cast<unsigned int>(Bc.block_count);
  const unsigned int warps_total = bag_block_count * PK_WARPS;
  const unsigned int warp_global = (blk - bag_block_begin) * PK_WARPS + warp;

  PkWarp w;
  w.lane = lane;
  w.lt_mask = (1u << lane) - 1u;
  w.q_idx = static_cast<unsigned int>(__cvta_generic_to_shared(sh.q_idx[warp]));
  w.q_pose = static_cast<unsigned int>(__cvta_generic_to_shared(sh.q_pose[warp]));
  w.q_cnt = static_cast<unsigned int>(__cvta_generic_to_shared(&sh.q_cnt[warp]));
  if (lane == 0) sh.q_cnt[warp] = 0, sh.deferred[warp][0] = sh.deferred[warp][1] = 0u;
  w.qn = 0;
  const unsigned int smem_base = static_cast<unsigned int>(__cvta_generic_to_shared(smem_hist));
  // tile ring of this warp: this lane's rows of slot s at pk_ring_slot<K>(a, smem_base, s).  The pass's
  // bookkeeping {next tile, tiles left, tile step, slot} lives in sh.ring_state[warp] (every lane writes the same values and
  // reads them back).  While a tile is scored it waits there instead of in registers live across the pose loop.
  constexpr bool DELTA = DPOSE && PK_DELTA_POSES && MODEL == CAM_EQUIRECTANGULAR && K % 2 == 0;  // as in pk_tile
  const unsigned int ring_state = static_cast<unsigned int>(__cvta_generic_to_shared(&sh.ring_state[warp]));
  const int n_items_per_batch = grp.n_bags * (solve_mode ? PK_MAX_POSES : grp.chunk);  // finalizer items of a full pose-list chunk
  const int fin_stride = max(1, static_cast<int>(grid) / (grp.n_bags * PK_MAX_POSES));

  // ---- first batch ----
  if (solve_mode) {
    static_assert(sizeof(NmMachine) % 8 == 0, "NmMachine is copied as 8-byte words");
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&grp.solve->nm);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&sh.nm);
    for (int i = t; i < static_cast<int>(sizeof(NmMachine) / 8); i += PK_THREADS) dst[i] = src[i];
    if (t < 16) sh.init_T[t] = grp.solve->init_T[t];
    __syncthreads();
    if (warp == 0) {
      pk_poses_of_candidates(sh, sh.nm.n_cand, lane);
      if constexpr (DELTA) pk_delta_rows<K>(sh, sh.nm.n_cand, a.nb, lane);
    }
    if (t == 0) sh.n_poses = sh.nm.n_cand;
  } else {
    const int pc = min(grp.chunk, grp.n_total);
    if (t < pc) pk_pose_from_list(sh, t, grp.poses_in + 12 * static_cast<size_t>(t));  // pc <= 8: warp 0
    if (DELTA && warp == 0) pk_delta_rows<K>(sh, pc, a.nb, lane);
    if (t == 0) sh.n_poses = pc;
  }
  for (int i = t; i < PK_MAX_POSES * 2 * PK_MAX_BINS; i += PK_THREADS) (&sh.bmarg[0][0])[i] = 0;
  if (t == 0) {
    sh.seq_base = *grp.seq_counter;
    sh.trace_count = 0;
    sh.poses_scored = 0ull;
  }
  __syncthreads();

  for (unsigned long long batch = 0;; batch++) {
    const int n_poses = sh.n_poses;
    if (n_poses == 0) break;
    // accumulator buffer of this batch: pose-list mode alternates two (each zeroed by its finalizers), Nelder-Mead mode
    // rotates three (every block reads all of them; buffer b is zeroed while batch b + 1 is finalized, see (B))
    const int buf = solve_mode ? static_cast<int>(batch % 3ull) : static_cast<int>(batch & 1ull);
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 0);
    if (DELTA && blk == 0 && t == 0 && sh.delta_on && grp.delta_stats) grp.delta_stats[0] += 1ull, grp.delta_stats[1] += static_cast<unsigned long long>(n_poses);
    // pose-list mode runs ahead of the finalizers: buffer `buf` (accumulators, tile counter) must have been finalized for
    // chunk batch - 2 first.  (Nelder-Mead mode: seeing the scores of batch - 1 already implies it.)
    if (!solve_mode && batch >= 2) {
      if (!pk_wait_counter(grp, sh, grp.fin_done + buf, static_cast<unsigned int>((batch >> 1) * static_cast<unsigned long long>(n_items_per_batch)))) return;
    }
    const bool time_block = grp.block_times != nullptr && batch == static_cast<unsigned long long>(grp.block_times_batch) && t == 0;
    if (time_block) grp.block_times[4 * blk + 0] = global_ns();
    // Nelder-Mead mode, batch > 0: the histogram copies were zeroed and sh.tmax set while warp 0 stepped the simplex (end of
    // the previous batch), so the batch starts without a barrier
    const bool fresh = !solve_mode || batch == 0ull;
    if (fresh && t == 0) sh.tmax = pk_tmax(sh, n_poses);
    // ---- (A) histograms of this block's share of the cloud ----------------------------------------------------------
    const int per_copy = n_poses * a.nb;
    w.hist_addr = smem_base + 4u * static_cast<unsigned int>((warp % a.copies) * per_copy);
    // Interleaved split: tile k (32 * K consecutive points of the tile-ordered cloud) goes to warp k mod W of the bag, so
    // every warp -- and every block: its 24 warps take 24 neighbouring tiles per round -- samples the whole image instead of
    // owning one region.  With contiguous slices the cost of a slice followed its region (deferred rechecks, histogram bin
    // collisions, cache hit rates), so the slowest block finished well after the median one, and every Nelder-Mead batch
    // waits for the slowest.  (Claiming tiles from an atomic counter was tried too: no better than the contiguous split
    // at 256-point claims, and finer claims serialise on the counter.)
    constexpr unsigned int TP = 32u * K;
    // The warp's full tiles stream through its shared-memory ring, PK_RING - 1 of them in flight behind the one being
    // scored.  Serpentine sweep: odd passes walk the warp's tiles backwards, so every pass begins on the tiles that the
    // previous one touched last (still in L2 when the cloud is larger than L2) -- same tiles, other order, same counts.
    {
      const unsigned int n_full = bag_n / TP;
      const unsigned int nt = warp_global < n_full ? (n_full - 1u - warp_global) / warps_total + 1u : 0u;
      const bool backward = (batch & 1ull) != 0ull;
      const unsigned int step = backward ? 0u - warps_total : warps_total;  // tiles between consecutive steps (mod 2^32)
      const unsigned int tile0 = backward ? warp_global + (nt - 1u) * warps_total : warp_global;
#pragma unroll
      for (int s = 0; s + 1 < PK_RING; s++)
        pk_ring_fill<K>(pk_ring_slot<K>(a, smem_base, s), B.points + static_cast<size_t>(tile0 + s * step) * TP + lane, static_cast<unsigned int>(s) < nt);
      sts_v4(ring_state, make_uint4(tile0, nt, step, 0u));
    }
    if (fresh) {
      for (int i = t; i < a.copies * per_copy; i += PK_THREADS) smem_hist[i] = 0;
      __syncthreads();
    }
    if (time_block) grp.block_times[4 * blk + 1] = global_ns();
    for (;;) {
      const uint4 rs = lds_v4(ring_state);  // {tile, tiles left, step, slot}
      if (rs.y == 0u) break;
      // this lane's copies of the tile landed (the later groups may still be in flight)
      asm volatile("cp.async.wait_group %0;" ::"n"(PK_RING - 2) : "memory");
      const unsigned int row0 = pk_ring_slot<K>(a, smem_base, rs.w);
      float4 q[K];
#pragma unroll
      for (int j = 0; j < K; j++) {
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(q[j].x), "=f"(q[j].y), "=f"(q[j].z), "=f"(q[j].w) : "r"(row0 + 512u * j) : "memory");
      }
      // refill the slot read at the step before (its rows went through the pose loop) with the tile PK_RING - 1 steps ahead
      const unsigned int refill = rs.w == 0u ? PK_RING - 1u : rs.w - 1u;
      pk_ring_fill<K>(pk_ring_slot<K>(a, smem_base, refill), B.points + static_cast<size_t>(rs.x + (PK_RING - 1) * rs.z) * TP + lane, rs.y > PK_RING - 1u);
      sts_v4(ring_state, make_uint4(rs.x + rs.z, rs.y - 1u, rs.z, rs.w + 1u == PK_RING ? 0u : rs.w + 1u));
      pk_tile<MODEL, K, false, DPOSE>(a, sh, B, n_poses, w, rs.x * TP, bag_n, q);
    }
    // the cloud's ragged last tile (fewer than 32 * K points, register loads) belongs to the warp whose tile sequence reaches it
    const unsigned int n_full = bag_n / TP;
    if (n_full * TP < bag_n && n_full % warps_total == warp_global) pk_rows<MODEL>(a, sh, B, n_poses, w, n_full * TP, bag_n);
    if (w.qn > 0) {
      pk_drain32<MODEL>(a, sh, B, w, 0, w.qn);
      w.qn = 0;
      if (lane == 0) sts_u32(w.q_cnt, 0u);
    }
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 1);
    __syncthreads();
    if (time_block) grp.block_times[4 * blk + 2] = global_ns();
    // ---- merge into the global accumulators -----------------------------------------------------------------------------
    {
      int* g = grp.ghist + (static_cast<size_t>(buf) * grp.n_bags + bag) * PK_MAX_POSES * a.nb;
      for (int k = t; k < per_copy; k += PK_THREADS) {
        int s = 0;
        for (int c = 0; c < a.copies; c++) s += smem_hist[c * per_copy + k];
        if (s) {
          atomicAdd(g + k, s);
          if (solve_mode) {  // the block's marginals (cost_calculator_nid.cpp:50-51), merged below
            const int p = k / a.nb, kk = k - p * a.nb;
            atomicAdd(&sh.bmarg[p][kk % a.bins], s);
            atomicAdd(&sh.bmarg[p][a.bins + kk / a.bins], s);
          }
        }
      }
      if (solve_mode) {
        __syncthreads();
        int* gm = grp.gmarg + (static_cast<size_t>(buf) * grp.n_bags + bag) * PK_MAX_POSES * PK_MARG_STRIDE;
        for (int i = t; i < n_poses * 2 * a.bins; i += PK_THREADS) {
          const int p = i / (2 * a.bins), f = i - p * 2 * a.bins;
          const int v = sh.bmarg[p][f];
          if (v) atomicAdd(gm + p * PK_MARG_STRIDE + f, v);
        }
        if (warp >= PK_WARPS - n_poses) {  // inlier count of pose p (:54): one of the last warps each (the first ones carry the marginals)
          const int p = PK_WARPS - 1 - warp;
          const int tot = __reduce_add_sync(0xffffffffu, lane < a.bins ? sh.bmarg[p][lane] : 0);  // bins <= 32
          if (lane == 0 && tot) atomicAdd(gm + p * PK_MARG_STRIDE + 2 * PK_MAX_BINS, tot);
        }
      }
    }
    // every thread's reductions are ordered before the barrier, the barrier before thread 0's fence, the fence before the
    // arrival: one gpu-scope fence per block instead of one per thread (the pattern of cooperative-groups grid sync)
    __syncthreads();
    if (t == 0) {
      __threadfence();
      atomicAdd(grp.arrive + buf * PK_MAX_BAGS + bag, 1u);
    }
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 2);
    if (time_block) grp.block_times[4 * blk + 3] = global_ns();
    const unsigned long long seq = sh.seq_base + batch + 1ull;
    const int slot = static_cast<int>(seq & 1ull);
    const unsigned long long tag = ((seq & 0x7fffffffull) | 0x80000000ull) << 32;  // never 0 (mailboxes start zeroed)
    if (!solve_mode) {
      // ---- (B, pose list) finalize the (bag, pose) items this block owns; nobody waits for them but the chunk after next ----
      for (int item = 0; item < grp.n_bags * n_poses; item++) {
        const int ib = item / n_poses, ip = item % n_poses;
        if (static_cast<int>((static_cast<long long>(ib * PK_MAX_POSES + ip) * fin_stride) % grid) != static_cast<int>(blk)) continue;
        const unsigned int expected = static_cast<unsigned int>(((batch >> 1) + 1ull) * static_cast<unsigned long long>(grp.bag[ib].block_count));
        if (!pk_wait_counter(grp, sh, grp.arrive + buf * PK_MAX_BAGS + ib, expected)) return;
        if (item == 0 && t == 0) pk_stamp(grp, batch, 3);
        int* g = grp.ghist + ((static_cast<size_t>(buf) * grp.n_bags + ib) * PK_MAX_POSES + ip) * a.nb;
        int* ho = (grp.hist_out && ib == 0) ? grp.hist_out + (static_cast<size_t>(batch) * grp.chunk + ip) * a.nb : nullptr;
        const double nid = pk_block_nid(sh, g, a.nb, a.bins, ho, smem_hist);
        if (t == 0) {
          // sum over the launch's bags in bag order needs all of them; single-bag launches store directly
          if (grp.n_bags == 1) grp.scores_out[batch * grp.chunk + ip] = nid;
          else grp.scores_out[(batch * grp.chunk + ip) * grp.n_bags + ib] = nid;  // per-bag scores; the host adds them in order
          __threadfence();
          atomicAdd(grp.fin_done + buf, 1u);
        }
        if (item == 0 && t == 0) pk_stamp(grp, batch, 4);
        __syncthreads();
      }
      // ---- next chunk of the pose list (only the last chunk can be partial, and no merge ever waits for it) ----
      const long long next0 = static_cast<long long>(batch + 1ull) * grp.chunk;
      const int pc = static_cast<int>(max(0ll, min(static_cast<long long>(grp.chunk), static_cast<long long>(grp.n_total) - next0)));
      __syncthreads();
      if (t < pc) pk_pose_from_list(sh, t, grp.poses_in + 12 * static_cast<size_t>(next0 + t));
      if (DELTA && warp == 0) pk_delta_rows<K>(sh, pc, a.nb, lane);
      if (t == 0) sh.n_poses = pc;
      __syncthreads();
      continue;
    }
    // ---- (B, Nelder-Mead) every block finalizes every (bag, pose) of the batch itself, one warp per item ---------------------
    // The next step of the solve needs all scores in every block.  An owner block per item (round-2 first version) cost a
    // second hop -- all arrived -> owner computes with the whole block -> fence -> publishes -> everybody polls -- and the zero-on-read accumulator needed that fence.  Here the arrival wait is the only hop:
    // each block reads the merged accumulators (4 KB per item, L2) and computes the same canonical NID per item in one warp.
    // Accumulators rotate over three buffers and are zeroed two batches ahead: buffer (batch + 2) % 3 was last read in
    // batch - 1 (finished by every block before it arrived here) and is next merged in batch + 2, which no block reaches
    // before every block arrived for batch + 1, i.e. after this block's zeroing (ordered by the arrival fence).
    if (!pk_wait_arrivals(grp, grp.arrive + buf * PK_MAX_BAGS, static_cast<unsigned int>(batch / 3ull + 1ull))) return;
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 3);
    {
      const int nz = grp.n_bags * PK_MAX_POSES * a.nb;
      int* z = grp.ghist + static_cast<size_t>((buf + 2) % 3) * nz;
      for (int i = static_cast<int>(blk) * PK_THREADS + t; i < nz; i += static_cast<int>(grid) * PK_THREADS) z[i] = 0;
      const int nm = grp.n_bags * PK_MAX_POSES * PK_MARG_STRIDE;
      int* zm = grp.gmarg + static_cast<size_t>((buf + 2) % 3) * nm;
      // (from the last block down: the first blocks carry most of the joint accumulators)
      for (int i = static_cast<int>(grid - 1u - blk) * PK_THREADS + t; i < nm; i += static_cast<int>(grid) * PK_THREADS) zm[i] = 0;
    }
    {
      const int n_items = grp.n_bags * n_poses;
      const int* gbuf = grp.ghist + static_cast<size_t>(buf) * grp.n_bags * PK_MAX_POSES * a.nb;
      const int* mbuf = grp.gmarg + static_cast<size_t>(buf) * grp.n_bags * PK_MAX_POSES * PK_MARG_STRIDE;
      // items per round: what the dead histogram copies hold of staged terms, at most one item per warp
      const int round_items = min(PK_WARPS, (a.copies * PK_MAX_POSES * a.nb * 4) / pk_fin_item_bytes(a.nb, a.bins));
      for (int first = 0; first < n_items; first += round_items) {
        const int count = min(round_items, n_items - first);
        pk_block_nid_items(gbuf, mbuf, first, count, n_poses, a.nb, a.bins, smem_hist, sh.fin_out);
        if (t < count) {
          const int item = first + t, ib = item / n_poses, ip = item - ib * n_poses;
          const int word = (grp.rank * grp.n_bags + ib) * PK_MAX_POSES + ip;
          const double nid = sh.fin_out[t];
          sh.parts[word] = nid;
          // the other ranks get it from one block (NVLink peer stores, tagged words)
          if (grp.world > 1 && static_cast<unsigned int>(item) % grid == blk) {
            const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(nid));
            for (int r = 0; r < grp.world; r++) {
              if (r == grp.rank) continue;
              volatile unsigned long long* dst = grp.box[r]->w[slot][word];
              dst[0] = tag | (bits & 0xffffffffull);
              dst[1] = tag | (bits >> 32);
            }
          }
        }
      }
    }
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 4);
    // ---- (C) the other ranks' scores -> sum over ranks and bags -> Nelder-Mead step -> next poses ---------------------------
    const int n_words = grp.world * grp.n_bags * n_poses;
    bool timed_out = false;
    if (grp.world > 1 && t < n_words && t / (grp.n_bags * n_poses) != grp.rank) {
      const int src = t / n_poses, p = t % n_poses;  // src = rank * n_bags + bag
      volatile unsigned long long* wsrc = grp.box[grp.rank]->w[slot][src * PK_MAX_POSES + p];
      const unsigned long long t0 = global_ns();
      unsigned int spins = 0;
      unsigned long long wl, wh;
      for (;;) {
        wl = wsrc[0], wh = wsrc[1];
        if ((wl & 0xffffffff00000000ull) == tag && (wh & 0xffffffff00000000ull) == tag) break;
        if ((++spins & 255u) == 0) {
          if (ld_acquire_u32(grp.abort_flag) != 0u) {
            timed_out = true;
            break;
          }
          if (global_ns() - t0 > grp.timeout_ns) {
            atomicExch(grp.abort_flag, 1u);
            if (grp.error_host) *reinterpret_cast<volatile int*>(grp.error_host) = 1;
            timed_out = true;
            break;
          }
        }
      }
      sh.parts[src * PK_MAX_POSES + p] = __longlong_as_double(static_cast<long long>((wh << 32) | (wl & 0xffffffffull)));
    }
    if (__syncthreads_or(timed_out ? 1 : 0)) return;
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 5);
    if (t < n_poses) {
      double total = 0.0;
      for (int s = 0; s < grp.world * grp.n_bags; s++) total += sh.parts[s * PK_MAX_POSES + t];  // (rank, bag) order: identical everywhere
      sh.ys[t] = total;
    }
    __syncthreads();
    if (warp == 0) {
      nm_warp_step(sh.nm, sh.ys, lane);
      if (blk == 0 && lane == 0) pk_stamp(grp, batch, 7);
      if (blk == 0) {  // reference-order evaluations of this batch, for the callback replay on the host (posted writes)
        const int n_obs = sh.nm.n_obs;
        const int base = sh.trace_count;
        for (int k = 0; k < n_obs; k++) {
          if (base + k < grp.trace_cap) {
            double* e = grp.trace_host + static_cast<size_t>(base + k) * (NM_MAX_N + 1);
            if (lane < sh.nm.n) e[lane] = sh.nm.obs_x[k][lane];
            if (lane == 0) e[NM_MAX_N] = sh.nm.obs_y[k];
          }
        }
        __syncwarp();
        if (lane == 0) {
          sh.trace_count = base + n_obs;
          sh.poses_scored += static_cast<unsigned long long>(n_poses);
        }
      }
      const int n_next = sh.nm.n_cand;  // 0 when finished
      pk_poses_of_candidates(sh, n_next, lane);
      if constexpr (DELTA) pk_delta_rows<K>(sh, n_next, a.nb, lane);
      if (lane == 0) {
        sh.n_poses = n_next;
        sh.tmax = pk_tmax(sh, n_next);
      }
    } else {
      // meanwhile the other warps clear the histogram copies for the next batch (all PK_MAX_POSES slots: its pose count is
      // being decided by warp 0); the warp-private finalizer scratch in the same array is dead since the barrier above
      for (int i = t - 32; i < a.copies * PK_MAX_POSES * a.nb; i += PK_THREADS - 32) smem_hist[i] = 0;
      for (int i = t - 32; i < PK_MAX_POSES * 2 * PK_MAX_BINS; i += PK_THREADS - 32) (&sh.bmarg[0][0])[i] = 0;
    }
    __syncthreads();
    if (blk == 0 && t == 0) pk_stamp(grp, batch, 6);
  }

  if (grp.delta_stats && lane == 0) {
    atomicAdd(grp.delta_stats + 2, static_cast<unsigned long long>(sh.deferred[warp][0]));
    atomicAdd(grp.delta_stats + 3, static_cast<unsigned long long>(sh.deferred[warp][1]));
  }
  // ---- results (block 0) ----
  if (blk == 0) {
    if (solve_mode) {
      const unsigned long long batches = static_cast<unsigned long long>(sh.nm.num_batches);
      const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&sh.nm);
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(&grp.result_host->nm);
      for (int i = t; i < static_cast<int>(sizeof(NmMachine) / 8); i += PK_THREADS) dst[i] = src[i];
      if (t == 0) {
        grp.result_host->batches = batches;
        grp.result_host->poses = sh.poses_scored;
        grp.result_host->trace_count = sh.trace_count;
        *grp.seq_counter = sh.seq_base + batches;  // every rank runs the same number of exchanges
      }
    }
    __threadfence_system();
    __syncthreads();
    if (t == 0 && grp.done_host && solve_mode) *reinterpret_cast<volatile unsigned long long*>(grp.done_host) = grp.done_seq;
  }
}

template <int MODEL, int K, bool DPOSE = false>
__global__ void __launch_bounds__(PK_THREADS, 1) nid_persistent_kernel(const __grid_constant__ PkArgs a) {
  pk_run<MODEL, K, DPOSE>(a, a, blockIdx.x, gridDim.x);
}

// ---- solve axis: S independent Nelder-Mead solves in one launch -------------------------------------------------------
// The grid is cut into S groups of consecutive blocks; group s is a whole Nelder-Mead mode launch of its own -- its own
// PkArgs (its bags, their block shares within the group, its PkSolve, its accumulators, arrival counters and result) --
// and never waits for another group.  A solve's scores are functions of its integer histograms alone, which do not depend
// on how many blocks share the cloud, so every solve follows the trajectory of a single-solve launch from the same start
// on the same bags, bit for bit.  A group whose solve has finished leaves the kernel; the launch ends with the slowest.
constexpr int PK_MAX_SOLVES = 64;

struct PkSolvesArgs {
  PkArgs common;                           // camera and image geometry, shared by every group (the hot loop reads it here)
  const PkArgs* group;                     // [n_groups] in device memory
  int n_groups;
  int block_begin[PK_MAX_SOLVES + 1];      // group s: blocks [block_begin[s], block_begin[s + 1])
};

// K = 2 only: a solve's result does not depend on the points per lane, and every instance more costs compile time
template <int MODEL, bool DPOSE = false>
__global__ void __launch_bounds__(PK_THREADS, 1) nid_persistent_solves_kernel(const __grid_constant__ PkSolvesArgs m) {
  // the group's arguments in shared memory, read outside the hot loop; the camera stays in the kernel parameter
  __shared__ PkArgs ga;
  int g = 0;
  while (g + 1 < m.n_groups && static_cast<int>(blockIdx.x) >= m.block_begin[g + 1]) g++;
  static_assert(sizeof(PkArgs) % 8 == 0, "PkArgs is copied as 8-byte words");
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(m.group + g);
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(&ga);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(PkArgs) / 8); i += PK_THREADS) dst[i] = src[i];
  __syncthreads();
  pk_run<MODEL, 2, DPOSE>(m.common, ga, blockIdx.x - static_cast<unsigned int>(m.block_begin[g]), static_cast<unsigned int>(m.block_begin[g + 1] - m.block_begin[g]));
}

// debug / test kernel: the lean classifier AND the exact path on every (point, pose); a.dbg: [0] point-poses,
// [1] verdicts deferred to the exact path, [2] kept verdicts that disagree with the exact path (must be 0),
// [3] max over accepted verdicts of |uv_fp32 - uv_exact| / E as float bits (atomicMax; must stay < 1).
// DELTA (equirectangular, packed): the anchor (lean_delta_anchor) through the anchor step, the other poses through the delta
// step of the hot loop, whatever their spread.
template <int MODEL, bool DELTA = false>
__global__ void __launch_bounds__(NID_THREADS) nid_lean_verify_kernel(const __grid_constant__ NidArgs a, const __grid_constant__ LeanCam lc) {
  const float4* __restrict__ pts = static_cast<const float4*>(a.points);
  unsigned long long total = 0, uncertain = 0, mismatch = 0;
  float tmax = 0.f, max_ratio = 0.f;
  for (int p = 0; p < a.n_poses; p++) tmax = fmaxf(tmax, a.pose32[p][12]);
  float Q[NID_MAX_POSES][16];
  int anc = 0;
  if constexpr (DELTA) {
    anc = lean_delta_anchor(a.pose, a.n_poses);
    for (int p = 0; p < a.n_poses; p++)
      if (p != anc) lean_delta_pose(a.pose[p], a.pose[anc], Q[p]);
  }
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  // points in pairs (2k, 2k + 1), as the hot loop classifies them with the packed classifier
  for (long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; 2 * k < a.n; k += stride) {
    const long long i0 = 2 * k, i1 = min(2 * k + 1, static_cast<long long>(a.n) - 1);
    const int n_here = 2 * k + 1 < a.n ? 2 : 1;
    const float4 q2[2] = {__ldg(pts + i0), __ldg(pts + i1)};
    float delta[2];
    for (int h = 0; h < 2; h++) delta[h] = (5.25f * F32_U) * (fabsf(q2[h].x) + fabsf(q2[h].y) + fabsf(q2[h].z) + tmax);
    LeanAnchor2 an;
    for (int k = 0; k < a.n_poses; k++) {
      const int p = k == 0 ? anc : k - (k <= anc ? 1 : 0);  // the anchor first (p == k without the delta step)
      LeanVerdict v2[2];
      if constexpr (DELTA) {
        const F2 X = f2_pack(q2[0].x, q2[1].x), Y = f2_pack(q2[0].y, q2[1].y), Z = f2_pack(q2[0].z, q2[1].z), D = f2_pack(delta[0], delta[1]);
        const LeanVerdict2 w = k == 0 ? classify_lean2_anchor<MODEL>(a.fast, lc, a.width, a.pose32[anc], X, Y, Z, D, an) : classify_lean2_delta<MODEL>(lc, a.width, Q[p], X, Y, Z, D, an);
        for (int h = 0; h < 2; h++) {
          v2[h].accept = w.accept[h], v2[h].uncertain = w.uncertain[h], v2[h].idx = w.idx[h];
          v2[h].up = w.up[h], v2[h].vp = w.vp[h], v2[h].hx = w.hx[h], v2[h].hy = w.hy[h];
        }
      } else if constexpr (LeanPacked<MODEL>::value) {
        const LeanVerdict2 w = classify_lean2<MODEL>(a.fast, lc, a.width, a.pose32[p], f2_pack(q2[0].x, q2[1].x), f2_pack(q2[0].y, q2[1].y),
                                                     f2_pack(q2[0].z, q2[1].z), f2_pack(delta[0], delta[1]));
        for (int h = 0; h < 2; h++) {
          v2[h].accept = w.accept[h], v2[h].uncertain = w.uncertain[h], v2[h].idx = w.idx[h];
          v2[h].up = w.up[h], v2[h].vp = w.vp[h], v2[h].hx = w.hx[h], v2[h].hy = w.hy[h];
        }
      } else {
        for (int h = 0; h < 2; h++) v2[h] = classify_lean<MODEL>(a.fast, lc, a.width, a.pose32[p], q2[h].x, q2[h].y, q2[h].z, delta[h]);
      }
      for (int h = 0; h < n_here; h++) {
        const LeanVerdict& v = v2[h];
        const float4 q = q2[h];
        total++;
        double ue = 0.0, ve = 0.0;
        const int pe = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, a.pose[p], q.x, q.y, q.z, &ue, &ve);
        if (v.uncertain) {
          uncertain++;
        } else if (v.accept ? (v.idx != pe) : (pe != -1)) {
          mismatch++;
        } else if (v.accept) {
          const float ru = static_cast<float>(fabs(static_cast<double>(v.up) - (ue - 0.5))) / (0.5f - v.hx);
          const float rv = static_cast<float>(fabs(static_cast<double>(v.vp) - (ve - 0.5))) / (0.5f - v.hy);
          max_ratio = fmaxf(max_ratio, fmaxf(ru, rv));
        }
      }
    }
  }
  atomicAdd(a.dbg + 0, total);
  atomicAdd(a.dbg + 1, uncertain);
  atomicAdd(a.dbg + 2, mismatch);
  atomicMax(reinterpret_cast<unsigned int*>(a.dbg + 3), __float_as_uint(max_ratio));  // non-negative floats order like uints
}

}  // namespace vlcal
