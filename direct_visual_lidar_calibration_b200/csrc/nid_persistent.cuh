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

#include <climits>
#include <cstdint>

#include "exact_classify.cuh"
#include "lean_filter.cuh"
#include "lean_filter2.cuh"
#include "nid_kernels.cuh"

namespace vlcal {

// Launch shape: ONE block of 768 threads per SM (24 warps, <= 85 registers).  Three blocks of 256 threads (A/B build,
// `make alt ALTFLAGS="-DPK_THREADS_CFG=256 -DPK_MIN_BLOCKS=3"`) hold the same 24 warps, but the warp scheduler prefers higher warp slots, so the three blocks of an SM
// finish their equal slices at different times and every Nelder-Mead batch waits for the slowest; one block also merges
// once instead of three times and arrives once.
#ifndef PK_THREADS_CFG
#define PK_THREADS_CFG 768
#endif
constexpr int PK_THREADS = PK_THREADS_CFG;
constexpr int PK_WARPS = PK_THREADS / 32;
constexpr int PK_MAX_POSES = 8;
constexpr int PK_MAX_BAGS = 8;
constexpr int PK_MAX_WORDS = 256;  // world x bags x 8 score words per batch, one polling thread each
constexpr int PK_QUEUE = 64;
constexpr int PK_MAX_BINS = 32;  // nb <= 1024
constexpr int PK_MARG_STRIDE = 2 * PK_MAX_BINS + 32;  // ints per (bag, pose) record of PkArgs::gmarg
constexpr int PK_STAMP_SLOTS = 8;
constexpr unsigned int PK_TILE_ROWS = 4;
// TMA variant (A/B, VLCAL_PK_TMA=1): the block's window of the image-bin plane staged in shared memory once per solve
constexpr int PK_TMA_BYTES = 48 * 1024;  // shared memory of the window
constexpr int PK_TMA_BOX_W = 256;        // one TMA box = 256 x 1 bytes of a row (boxes of a row are contiguous in shared memory)
constexpr int PK_TMA_HALO = 12;          // pixels around the bounding box of the block's points at the start pose
struct alignas(64) PkTensorMap {         // a CUtensorMap (cuTensorMapEncodeTiled), opaque here
  unsigned long long opaque[16];
};
#ifndef PK_PACKED_FP32
#define PK_PACKED_FP32 1  // classify two points per lane, interleaved (lean_filter2.cuh); 0: scalar classifier (A/B build)
#endif
#ifndef PK_DIAG_STAMPS
#define PK_DIAG_STAMPS 0  // diagnostic build: stamp 3 moves behind the two-ahead zeroing, stamp 5 to the finalizer's inner barrier
#endif
#ifndef PK_MIN_BLOCKS
#define PK_MIN_BLOCKS 1  // blocks per SM the register allocation must allow (768 threads x 85 registers fill the register file)
#endif

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

struct PkArgs {
  PkTensorMap tmap[PK_MAX_BAGS];  // TMA variant: tensor map of each bag's image-bin plane (u8, W x H, box 256 x 1)
  // camera + image geometry (shared by all bags of the launch: one camera, equal image sizes)
  int width, height, bins, nb;
  double cos_fov;
  CameraParams cam;
  FastCam fast;
  LeanCam lean;
  int n_bags;
  PkBag bag[PK_MAX_BAGS];
  int copies;  // shared-memory histogram copies per block
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
  unsigned long long* tma_stats;    // TMA variant: [0] gathers served from the shared-memory window, [1] gathers that escaped it
  unsigned long long* block_times;  // optional [grid][4]: every block's {enter, hist zeroed, main loop done, arrived} stamps of batch block_times_batch
  int block_times_batch;
};

struct PkShared {
  NmMachine nm;
  double init_T[16];
  double pose64[PK_MAX_POSES][12];
  float4 pose32[PK_MAX_POSES][4];  // rows: [R00 R01 R02 t0] [R10 R11 R12 t1] [R20 R21 R22 t2] [max|t| 0 0 0]
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
  // TMA variant: the staged window [box_h][box_w] of the image-bin plane (origin biased like LeanVerdict::ixb / iyb)
  alignas(8) unsigned long long tma_bar;
  int bb_min_x, bb_max_x, bb_min_y, bb_max_y;
  int box_x0b, box_y0b, box_w, box_h;
  unsigned int q_idx[PK_WARPS][PK_QUEUE];
  unsigned char q_pose[PK_WARPS][PK_QUEUE];
  int q_cnt[PK_WARPS];  // fill count of each warp's queue
};

// ---- small PTX helpers ---------------------------------------------------------------------------------------------

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// histogram increment, two forms (A/B, VLCAL_PK_ATOM):
//   ATOM == 0: `if (counted) atomicAdd(p, 1)` -- ptxas emits BSSY / BRA / ATOMS.POPC.INC / BSYNC (lanes of a warp that hit
//              the same bin are merged by the hardware; predication is not available for this form, hence the branch);
//   ATOM == 1: unconditional red.shared.add of a 0 / 1 register -- one ATOMS.ADD, no branch, same-bin lanes serialise.
__device__ __forceinline__ void red_shared_add(unsigned int smem_addr, int inc) {
  asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(smem_addr), "r"(inc) : "memory");
}
__device__ __forceinline__ void red_shared_inc(unsigned int smem_addr) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(smem_addr) : "memory");
}

// 1-byte read-only gather under a predicate; -1 when off (the sign doubles as the "counted" flag one pose later)
__device__ __forceinline__ int ldg_u8_or_neg(bool pred, const uint8_t* p) {
  int v;
  asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %1, 0;\n\tmov.u32 %0, -1;\n\t@q ld.global.nc.u8 %0, [%2];\n\t}" : "=r"(v) : "r"(static_cast<int>(pred)), "l"(p));
  return v;
}

__device__ __forceinline__ int ldg_u8_or_zero(bool pred, const uint8_t* p) {
  int v;
  asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %1, 0;\n\tmov.u32 %0, 0;\n\t@q ld.global.nc.u8 %0, [%2];\n\t}" : "=r"(v) : "r"(static_cast<int>(pred)), "l"(p));
  return v;
}

// TMA variant: the image bin from the staged window (shared memory) when the pixel lies inside it, from global memory
// otherwise; `neg` = -1 (ATOM == 0: the sign is the "counted" flag) or 0
__device__ __forceinline__ int gather_u8_window(bool in_window, bool outside, unsigned int smem_addr, const uint8_t* p, int neg) {
  int v;
  asm("{\n\t.reg .pred q, r;\n\tsetp.ne.b32 q, %1, 0;\n\tsetp.ne.b32 r, %2, 0;\n\tmov.u32 %0, %5;\n\t@q ld.shared.u8 %0, [%3];\n\t@r ld.global.nc.u8 %0, [%4];\n\t}"
      : "=r"(v)
      : "r"(static_cast<int>(in_window)), "r"(static_cast<int>(outside)), "r"(smem_addr), "l"(p), "r"(neg));
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
  // :57, :60, :66, :75  xo, xr, xe, xc
  if (mine) {
    xd sum(0.0);
    for (int k = 0; k < n; k++) sum = sum + xd(s.x[k][lane]);
    const xd xo = sum / xd(static_cast<double>(n));
    const xd diff = xo - xd(s.x[n][lane]);
    s.cand[0][lane] = xo.v;
    s.cand[1][lane] = (xo + xd(s.params.alpha) * diff).v;
    s.cand[2][lane] = (xo + xd(s.params.gamma) * diff).v;
    s.cand[3][lane] = (xo + xd(s.params.rho) * diff).v;
  }
  if (lane == 0) {
    s.n_cand = 4;
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
    const double y0 = ys[0], y1 = ys[1], y2 = ys[2], y3 = ys[3];
    __syncwarp();
    if (lane == 0) {
      s.cand[0][0] = y0;
      s.cand[1][0] = y1;
    }
    __syncwarp();
    nm_warp_observe(s, lane, s.cand[0], y0);  // :58 evaluated, never used in a decision
    nm_warp_observe(s, lane, s.cand[1], y1);  // :61
    bool shrink = false;
    if (f0 <= y1 && y1 < fn1) {  // :63-64
      if (mine) s.x[n][lane] = s.cand[1][lane];
    } else if (y1 < f0) {  // :65-73 expansion
      if (lane == 0) s.cand[2][0] = y2;
      __syncwarp();
      nm_warp_observe(s, lane, s.cand[2], y2);
      const int pick = (y2 < y1) ? 2 : 1;
      if (mine) s.x[n][lane] = s.cand[pick][lane];
    } else {  // :74-86
      if (lane == 0) s.cand[3][0] = y3;
      __syncwarp();
      nm_warp_observe(s, lane, s.cand[3], y3);
      if (y3 < fn) {
        if (mine) s.x[n][lane] = s.cand[3][lane];
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
                                                       double* out, unsigned long long* diag_stamp) {
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
  if (diag_stamp && t == 0) *diag_stamp = global_ns();
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
  // TMA variant
  unsigned int win_addr;   // shared-memory byte address of the staged image window
  int win_x0b, win_y0b;
  unsigned int win_w, win_h;
  unsigned int n_window, n_escaped;
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

template <int MODEL>
__device__ __noinline__ void pk_drain32(const PkArgs& a, const PkShared& sh, const PkBagRegs& B, PkWarp& w, int first, int count) {
  if (w.lane < count) {  // one deferred (point, pose) per lane, exact path
    const unsigned int i = lds_u32(w.q_idx + 4u * static_cast<unsigned int>(first + w.lane));
    const int p = static_cast<int>(lds_u8(w.q_pose + static_cast<unsigned int>(first + w.lane)));
    const float4 q = __ldg(B.points + i);
    const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, sh.pose64[p], q.x, q.y, q.z);
    if (pix >= 0) {
      const int ib = __ldg(B.bin_image + pix);  // :43,:46 via the pre-binned image
      const unsigned int addr = w.hist_addr + 4u * static_cast<unsigned int>(p * a.nb + ib + lidar_bin_of(q.w, a.bins) * a.bins);
      asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(addr) : "memory");  // :49 hist(image_bin, lidar_bin)++
    }
  }
}

// one tile = 32*K consecutive points starting at `tile`, swept over the P poses of the batch; the image-bin gathers of
// pose p stay in flight while pose p+1 is classified and are consumed by the histogram increments one iteration later.
// PARTIAL: the tile may reach past `end` (only the single-row tiles at the end of a warp's slice).
template <int MODEL, int K, bool PARTIAL, int ATOM, bool TMA>
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
  constexpr bool PACKED = PK_PACKED_FP32 && !PARTIAL && (K % 2 == 0) && LeanPacked<MODEL>::value;
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
  int pend_inc[K];  // ATOM == 1: 0 / 1
#pragma unroll
  for (int j = 0; j < K; j++) pend_bin[j] = -1, pend_inc[j] = 0;
  unsigned int pend_off = 0;
  for (int p = 0; p <= n_poses; p++) {
    bool acc[K];
    int pix[K], wx[K], wy[K];
    if (p < n_poses) {
      const float4 r0 = sh.pose32[p][0], r1 = sh.pose32[p][1], r2 = sh.pose32[p][2];
      const float Pm[12] = {r0.x, r0.y, r0.z, r1.x, r1.y, r1.z, r2.x, r2.y, r2.z, r0.w, r1.w, r2.w};
      if constexpr (PACKED) {
#pragma unroll
        for (int j = 0; j < K; j += 2) {  // two points per instruction on the packed fp32 pipe (lean_filter2.cuh)
          const LeanVerdict2 v = classify_lean2<MODEL>(a.fast, a.lean, a.width, Pm, X2[j / 2], Y2[j / 2], Z2[j / 2], D2[j / 2]);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            acc[j + h] = v.accept[h];
            if (v.uncertain[h]) unc_mask |= unc_bit << (j + h);
            pix[j + h] = v.idx[h];
            if constexpr (TMA) wx[j + h] = v.ixb[h], wy[j + h] = v.iyb[h];
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < K; j++) {
          const LeanVerdict v = classify_lean<MODEL>(a.fast, a.lean, a.width, Pm, px[j], py[j], pz[j], dl[j]);
          acc[j] = PARTIAL ? (v.accept & valid0) : v.accept;
          const bool unc = PARTIAL ? (v.uncertain & valid0) : v.uncertain;
          if (unc) unc_mask |= unc_bit << j;
          pix[j] = v.idx;
          if constexpr (TMA) wx[j] = v.ixb, wy[j] = v.iyb;
        }
      }
      unc_bit <<= K;
    }
#pragma unroll
    for (int j = 0; j < K; j++) {  // :49 hist(image_bin, lidar_bin)++ for the previous pose
      if constexpr (ATOM == 0) {
        if (pend_bin[j] >= 0) red_shared_inc(lb[j] + pend_off + 4u * static_cast<unsigned int>(pend_bin[j]));
      } else {
        red_shared_add(lb[j] + pend_off + 4u * static_cast<unsigned int>(pend_bin[j]), pend_inc[j]);
      }
    }
    if (p < n_poses) {
      pend_off = 4u * static_cast<unsigned int>(p * a.nb);
#pragma unroll
      for (int j = 0; j < K; j++) {
        if constexpr (TMA) {
          const unsigned int dx = static_cast<unsigned int>(wx[j] - w.win_x0b), dy = static_cast<unsigned int>(wy[j] - w.win_y0b);
          const bool inw = acc[j] & (dx < w.win_w) & (dy < w.win_h);
          const bool out = acc[j] & !inw;
          pend_bin[j] = gather_u8_window(inw, out, w.win_addr + dy * w.win_w + dx, B.bin_image + pix[j], ATOM == 0 ? -1 : 0);
          if constexpr (ATOM != 0) pend_inc[j] = acc[j] ? 1 : 0;
          w.n_window += inw ? 1u : 0u;
          w.n_escaped += out ? 1u : 0u;
        } else if constexpr (ATOM == 0) {
          pend_bin[j] = ldg_u8_or_neg(acc[j], B.bin_image + pix[j]);
        } else {
          pend_bin[j] = ldg_u8_or_zero(acc[j], B.bin_image + pix[j]);
          pend_inc[j] = acc[j] ? 1 : 0;
        }
      }
    }
  }
  // Deferred (point, pose) pairs of this tile -> the warp's queue for the exact path.  Doing this once per tile instead of inside the pose loop
  // matters: with ~3 % of the point-poses deferred, SOME lane of the 32 x K has one in 5 of 6 pose steps, so the ballot /
  // queue code would run almost every step instead of once per tile.
  // Usual case (the tile defers at most 32 pairs): one warp prefix sum gives every lane the queue slots of its pairs.
  // Otherwise: one ballot per round.
  const int cnt = __popc(unc_mask);
  const int total = __reduce_add_sync(0xffffffffu, cnt);
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

// points [tpos, end) of the cloud: K-row tiles with the next tile's rows in flight, then single-row tiles for the rest;
// qk holds the first K-row tile when `first_loaded`
template <int MODEL, int K, int ATOM, bool TMA>
__device__ __forceinline__ void pk_range(const PkArgs& a, const PkShared& sh, const PkBagRegs& B, int n_poses, PkWarp& w, unsigned int tpos, unsigned int end, float4 (&qk)[K], bool first_loaded) {
  const int lane = w.lane;
  if (!first_loaded && tpos + 32u * K <= end) pk_load_tile<K>(B.points, tpos, end, lane, qk);
  while (tpos + 32u * K <= end) {
    float4 nxt[K];
    const bool more = tpos + 64u * K <= end;
    if (more) pk_load_tile<K>(B.points, tpos + 32u * K, end, lane, nxt);
    pk_tile<MODEL, K, false, ATOM, TMA>(a, sh, B, n_poses, w, tpos, end, qk);
    tpos += 32u * K;
    if (more) {
#pragma unroll
      for (int j = 0; j < K; j++) qk[j] = nxt[j];
    }
  }
  float4 q1[1], n1[1];
  if (tpos < end) pk_load_tile<1>(B.points, tpos, end, lane, q1);
  while (tpos < end) {
    const bool more = tpos + 32u < end;
    if (more) pk_load_tile<1>(B.points, tpos + 32u, end, lane, n1);
    pk_tile<MODEL, 1, true, ATOM, TMA>(a, sh, B, n_poses, w, tpos, end, q1);
    tpos += 32u;
    if (more) q1[0] = n1[0];
  }
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
template <int MODEL, int K, int ATOM, bool TMA = false>
__global__ void __launch_bounds__(PK_THREADS, PK_MIN_BLOCKS) nid_persistent_kernel(const __grid_constant__ PkArgs a) {
  extern __shared__ __align__(128) int smem_hist[];
  __shared__ PkShared sh;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const bool solve_mode = a.solve != nullptr;

  // block -> bag, warp -> fixed slice of the bag's cloud
  int bag = 0;
  while (bag + 1 < a.n_bags && static_cast<int>(blockIdx.x) >= a.bag[bag + 1].block_begin) bag++;
  const PkBag& Bc = a.bag[bag];
  PkBagRegs B;
  B.points = Bc.points;
  B.bin_image = Bc.bin_image;
  const unsigned int bag_n = Bc.n, bag_block_begin = static_cast<unsigned int>(Bc.block_begin), bag_block_count = static_cast<unsigned int>(Bc.block_count);
  const unsigned int warps_total = bag_block_count * PK_WARPS;
  const unsigned int warp_global = (blockIdx.x - bag_block_begin) * PK_WARPS + warp;
  // points per warp: whole K-row tiles (a warp whose slice ends in single-row tiles runs them without instruction-level
  // parallelism: at C2 that was 2 of its 3 tiles)
  const unsigned int chunk = ((bag_n + warps_total - 1) / warps_total + (32u * K - 1u)) / (32u * K) * (32u * K);
  const unsigned long long lo = static_cast<unsigned long long>(warp_global) * chunk;
  const bool has_work = lo < bag_n;
  const unsigned int end = has_work ? static_cast<unsigned int>(min(static_cast<unsigned long long>(bag_n), lo + chunk)) : 0u;
  const unsigned int begin = static_cast<unsigned int>(has_work ? lo : 0ull);

  PkWarp w;
  w.lane = lane;
  w.lt_mask = (1u << lane) - 1u;
  w.q_idx = static_cast<unsigned int>(__cvta_generic_to_shared(sh.q_idx[warp]));
  w.q_pose = static_cast<unsigned int>(__cvta_generic_to_shared(sh.q_pose[warp]));
  w.q_cnt = static_cast<unsigned int>(__cvta_generic_to_shared(&sh.q_cnt[warp]));
  if (lane == 0) sh.q_cnt[warp] = 0;
  w.qn = 0;
  const unsigned int smem_base = static_cast<unsigned int>(__cvta_generic_to_shared(smem_hist));
  const int n_items_per_batch = a.n_bags * (solve_mode ? PK_MAX_POSES : a.chunk);  // finalizer items of a full pose-list chunk
  const int fin_stride = max(1, static_cast<int>(gridDim.x) / (a.n_bags * PK_MAX_POSES));

  // ---- first batch ----
  if (solve_mode) {
    static_assert(sizeof(NmMachine) % 8 == 0, "NmMachine is copied as 8-byte words");
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&a.solve->nm);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&sh.nm);
    for (int i = t; i < static_cast<int>(sizeof(NmMachine) / 8); i += PK_THREADS) dst[i] = src[i];
    if (t < 16) sh.init_T[t] = a.solve->init_T[t];
    __syncthreads();
    if (warp == 0) pk_poses_of_candidates(sh, sh.nm.n_cand, lane);
    if (t == 0) sh.n_poses = sh.nm.n_cand;
  } else {
    const int pc = min(a.chunk, a.n_total);
    if (t < pc) pk_pose_from_list(sh, t, a.poses_in + 12 * static_cast<size_t>(t));
    if (t == 0) sh.n_poses = pc;
  }
  for (int i = t; i < PK_MAX_POSES * 2 * PK_MAX_BINS; i += PK_THREADS) (&sh.bmarg[0][0])[i] = 0;
  if (t == 0) {
    sh.seq_base = *a.seq_counter;
    sh.trace_count = 0;
    sh.poses_scored = 0ull;
    sh.bb_min_x = sh.bb_min_y = INT_MAX;
    sh.bb_max_x = sh.bb_max_y = INT_MIN;
    sh.box_w = sh.box_h = 0;
  }
  __syncthreads();
  w.win_addr = 0, w.win_x0b = w.win_y0b = 0, w.win_w = w.win_h = 0, w.n_window = w.n_escaped = 0;
  if constexpr (TMA) {
    // ---- stage this block's window of the image-bin plane once for the whole solve (static split, Nelder-Mead mode) ----
    // bounding box of the block's points at the first candidate (= the start pose), grown by a halo for the poses the solve
    // will visit; pixels outside the window fall back to the global gather (counted in tma_stats[1])
    const unsigned int win_base = smem_base + 4u * static_cast<unsigned int>(a.copies * PK_MAX_POSES * a.nb);  // 128-byte aligned (host)
    if (solve_mode) {
      int mnx = INT_MAX, mxx = INT_MIN, mny = INT_MAX, mxy = INT_MIN;
      if (has_work) {
        const float4 r0 = sh.pose32[0][0], r1 = sh.pose32[0][1], r2 = sh.pose32[0][2];
        const float Pm[12] = {r0.x, r0.y, r0.z, r1.x, r1.y, r1.z, r2.x, r2.y, r2.z, r0.w, r1.w, r2.w};
        const float tm = sh.pose32[0][3].x;
        for (unsigned int i = begin + lane; i < end; i += 32u) {
          const float4 q = __ldg(B.points + i);
          const float dl = (5.25f * F32_U) * (fabsf(q.x) + fabsf(q.y) + fabsf(q.z) + tm);
          const LeanVerdict v = classify_lean<MODEL>(a.fast, a.lean, a.width, Pm, q.x, q.y, q.z, dl);
          if (v.accept) mnx = min(mnx, v.ixb), mxx = max(mxx, v.ixb), mny = min(mny, v.iyb), mxy = max(mxy, v.iyb);
        }
      }
      mnx = __reduce_min_sync(0xffffffffu, mnx), mny = __reduce_min_sync(0xffffffffu, mny);
      mxx = __reduce_max_sync(0xffffffffu, mxx), mxy = __reduce_max_sync(0xffffffffu, mxy);
      if (lane == 0 && mnx <= mxx) {
        atomicMin(&sh.bb_min_x, mnx), atomicMax(&sh.bb_max_x, mxx);
        atomicMin(&sh.bb_min_y, mny), atomicMax(&sh.bb_max_y, mxy);
      }
      __syncthreads();
      const unsigned int bar = static_cast<unsigned int>(__cvta_generic_to_shared(&sh.tma_bar));
      if (t == 0 && sh.bb_min_x <= sh.bb_max_x) {
        const int x0 = ((sh.bb_min_x - LEAN_MAGIC_BITS) - PK_TMA_HALO) & ~15;  // pixel coordinates; may be negative: TMA zero-fills
        const int x1 = (sh.bb_max_x - LEAN_MAGIC_BITS) + PK_TMA_HALO;
        const int y0 = (sh.bb_min_y - LEAN_MAGIC_BITS) - PK_TMA_HALO;
        const int y1 = (sh.bb_max_y - LEAN_MAGIC_BITS) + PK_TMA_HALO;
        const int nbx = (x1 - x0 + PK_TMA_BOX_W) / PK_TMA_BOX_W;
        int rows = y1 - y0 + 1;
        if (nbx * PK_TMA_BOX_W <= PK_TMA_BYTES) {
          rows = min(rows, PK_TMA_BYTES / (nbx * PK_TMA_BOX_W));
          sh.box_x0b = x0 + LEAN_MAGIC_BITS, sh.box_y0b = y0 + LEAN_MAGIC_BITS;
          sh.box_w = nbx * PK_TMA_BOX_W, sh.box_h = rows;
          asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
          asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(static_cast<unsigned int>(rows * nbx * PK_TMA_BOX_W)) : "memory");
          const unsigned long long tmap = reinterpret_cast<unsigned long long>(&a.tmap[bag]);
          for (int r = 0; r < rows; r++) {
            for (int bx = 0; bx < nbx; bx++) {
              const unsigned int dst = win_base + static_cast<unsigned int>((r * nbx + bx) * PK_TMA_BOX_W);
              asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(tmap),
                           "r"(x0 + bx * PK_TMA_BOX_W), "r"(y0 + r), "r"(bar)
                           : "memory");
            }
          }
        }
      }
      __syncthreads();
      if (sh.box_w > 0) {  // every thread waits for the bytes (phase 0); bounded, so that a refused descriptor cannot hang the GPU
        unsigned int done = 0;
        for (int spin = 0; spin < (1 << 22) && !done; spin++) {
          asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar) : "memory");
        }
        if (!done) {
          atomicExch(a.abort_flag, 1u);
          if (a.error_host) *reinterpret_cast<volatile int*>(a.error_host) = 2;
        }
        w.win_addr = win_base, w.win_x0b = sh.box_x0b, w.win_y0b = sh.box_y0b;
        w.win_w = static_cast<unsigned int>(sh.box_w), w.win_h = static_cast<unsigned int>(sh.box_h);
      }
    }
  }

  for (unsigned long long batch = 0;; batch++) {
    const int n_poses = sh.n_poses;
    if (n_poses == 0) break;
    // accumulator buffer of this batch: pose-list mode alternates two (each zeroed by its finalizers), Nelder-Mead mode
    // rotates three (every block reads all of them; buffer b is zeroed while batch b + 1 is finalized, see (B))
    const int buf = solve_mode ? static_cast<int>(batch % 3ull) : static_cast<int>(batch & 1ull);
    if (blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 0);
    // pose-list mode runs ahead of the finalizers: buffer `buf` (accumulators, tile counter) must have been finalized for
    // chunk batch - 2 first.  (Nelder-Mead mode: seeing the scores of batch - 1 already implies it.)
    if (!solve_mode && batch >= 2) {
      if (!pk_wait_counter(a, sh, a.fin_done + buf, static_cast<unsigned int>((batch >> 1) * static_cast<unsigned long long>(n_items_per_batch)))) return;
    }
    const bool time_block = a.block_times != nullptr && batch == static_cast<unsigned long long>(a.block_times_batch) && t == 0;
    if (time_block) a.block_times[4 * blockIdx.x + 0] = global_ns();
    // Nelder-Mead mode, batch > 0: the histogram copies were zeroed and sh.tmax set while warp 0 stepped the simplex (end of
    // the previous batch), so the batch starts without a barrier
    const bool fresh = !solve_mode || batch == 0ull;
    if (fresh && t == 0) sh.tmax = pk_tmax(sh, n_poses);
    // ---- (A) histograms of this block's share of the cloud ----------------------------------------------------------
    const int per_copy = n_poses * a.nb;
    w.hist_addr = smem_base + 4u * static_cast<unsigned int>((warp % a.copies) * per_copy);
    if constexpr (TMA) {
      // TMA variant: contiguous slice per warp (its image window must be compact)
      float4 qk[K];
      const bool preloaded = has_work && begin + 32u * K <= end;
      if (preloaded) pk_load_tile<K>(B.points, begin, end, lane, qk);
      if (fresh) {
        for (int i = t; i < a.copies * per_copy; i += PK_THREADS) smem_hist[i] = 0;
        __syncthreads();
      }
      if (time_block) a.block_times[4 * blockIdx.x + 1] = global_ns();
      if (has_work) pk_range<MODEL, K, ATOM, TMA>(a, sh, B, n_poses, w, begin, end, qk, preloaded);
    } else {
      // Interleaved split: tile k (32 * K consecutive points of the tile-ordered cloud) goes to warp k mod W of the bag, so
      // every warp -- and every block: its 24 warps take 24 neighbouring tiles per round -- samples the whole image instead of
      // owning one region.  With contiguous slices the cost of a slice followed its region (deferred rechecks, histogram bin
      // collisions, cache hit rates), so the slowest block finished well after the median one, and every Nelder-Mead batch
      // waits for the slowest.  (Claiming tiles from an atomic counter was tried too: no better than the contiguous split
      // at 256-point claims, and finer claims serialise on the counter.)  The next tile's rows are in flight while the current one is swept over the poses.
      constexpr unsigned int TP = 32u * K;
      unsigned int tile = warp_global;
      float4 qk[K];
      bool full = static_cast<unsigned long long>(tile) * TP + TP <= bag_n;
      if (full) pk_load_tile<K>(B.points, tile * TP, bag_n, lane, qk);
      if (fresh) {
        for (int i = t; i < a.copies * per_copy; i += PK_THREADS) smem_hist[i] = 0;
        __syncthreads();
      }
      if (time_block) a.block_times[4 * blockIdx.x + 1] = global_ns();
      while (full) {
        const unsigned int ntile = tile + warps_total;
        const bool nfull = static_cast<unsigned long long>(ntile) * TP + TP <= bag_n;
        float4 nxt[K];
        if (nfull) pk_load_tile<K>(B.points, ntile * TP, bag_n, lane, nxt);
        pk_tile<MODEL, K, false, ATOM, TMA>(a, sh, B, n_poses, w, tile * TP, bag_n, qk);
        tile = ntile;
        full = nfull;
        if (nfull) {
#pragma unroll
          for (int j = 0; j < K; j++) qk[j] = nxt[j];
        }
      }
      // the cloud's ragged last tile (fewer than 32 * K points) belongs to whichever warp's sequence reaches it
      if (static_cast<unsigned long long>(tile) * TP < bag_n) pk_range<MODEL, K, ATOM, TMA>(a, sh, B, n_poses, w, tile * TP, bag_n, qk, false);
    }
    if (w.qn > 0) {
      pk_drain32<MODEL>(a, sh, B, w, 0, w.qn);
      w.qn = 0;
      if (lane == 0) sts_u32(w.q_cnt, 0u);
    }
    if (blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 1);
    __syncthreads();
    if (time_block) a.block_times[4 * blockIdx.x + 2] = global_ns();
    // ---- merge into the global accumulators -----------------------------------------------------------------------------
    {
      int* g = a.ghist + (static_cast<size_t>(buf) * a.n_bags + bag) * PK_MAX_POSES * a.nb;
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
        int* gm = a.gmarg + (static_cast<size_t>(buf) * a.n_bags + bag) * PK_MAX_POSES * PK_MARG_STRIDE;
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
      atomicAdd(a.arrive + buf * PK_MAX_BAGS + bag, 1u);
    }
    if (blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 2);
    if (time_block) a.block_times[4 * blockIdx.x + 3] = global_ns();
    const unsigned long long seq = sh.seq_base + batch + 1ull;
    const int slot = static_cast<int>(seq & 1ull);
    const unsigned long long tag = ((seq & 0x7fffffffull) | 0x80000000ull) << 32;  // never 0 (mailboxes start zeroed)
    if (!solve_mode) {
      // ---- (B, pose list) finalize the (bag, pose) items this block owns; nobody waits for them but the chunk after next ----
      for (int item = 0; item < a.n_bags * n_poses; item++) {
        const int ib = item / n_poses, ip = item % n_poses;
        if (static_cast<int>((static_cast<long long>(ib * PK_MAX_POSES + ip) * fin_stride) % gridDim.x) != static_cast<int>(blockIdx.x)) continue;
        const unsigned int expected = static_cast<unsigned int>(((batch >> 1) + 1ull) * static_cast<unsigned long long>(a.bag[ib].block_count));
        if (!pk_wait_counter(a, sh, a.arrive + buf * PK_MAX_BAGS + ib, expected)) return;
        if (item == 0 && t == 0) pk_stamp(a, batch, 3);
        int* g = a.ghist + ((static_cast<size_t>(buf) * a.n_bags + ib) * PK_MAX_POSES + ip) * a.nb;
        int* ho = (a.hist_out && ib == 0) ? a.hist_out + (static_cast<size_t>(batch) * a.chunk + ip) * a.nb : nullptr;
        const double nid = pk_block_nid(sh, g, a.nb, a.bins, ho, smem_hist);
        if (t == 0) {
          // sum over the launch's bags in bag order needs all of them; single-bag launches store directly
          if (a.n_bags == 1) a.scores_out[batch * a.chunk + ip] = nid;
          else a.scores_out[(batch * a.chunk + ip) * a.n_bags + ib] = nid;  // per-bag scores; the host adds them in order
          __threadfence();
          atomicAdd(a.fin_done + buf, 1u);
        }
        if (item == 0 && t == 0) pk_stamp(a, batch, 4);
        __syncthreads();
      }
      // ---- next chunk of the pose list (only the last chunk can be partial, and no merge ever waits for it) ----
      const long long next0 = static_cast<long long>(batch + 1ull) * a.chunk;
      const int pc = static_cast<int>(max(0ll, min(static_cast<long long>(a.chunk), static_cast<long long>(a.n_total) - next0)));
      __syncthreads();
      if (t < pc) pk_pose_from_list(sh, t, a.poses_in + 12 * static_cast<size_t>(next0 + t));
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
    if (!pk_wait_arrivals(a, a.arrive + buf * PK_MAX_BAGS, static_cast<unsigned int>(batch / 3ull + 1ull))) return;
    if (!PK_DIAG_STAMPS && blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 3);
    {
      const int nz = a.n_bags * PK_MAX_POSES * a.nb;
      int* z = a.ghist + static_cast<size_t>((buf + 2) % 3) * nz;
      for (int i = static_cast<int>(blockIdx.x) * PK_THREADS + t; i < nz; i += static_cast<int>(gridDim.x) * PK_THREADS) z[i] = 0;
      const int nm = a.n_bags * PK_MAX_POSES * PK_MARG_STRIDE;
      int* zm = a.gmarg + static_cast<size_t>((buf + 2) % 3) * nm;
      // (from the last block down: the first blocks carry most of the joint accumulators)
      for (int i = static_cast<int>(gridDim.x - 1u - blockIdx.x) * PK_THREADS + t; i < nm; i += static_cast<int>(gridDim.x) * PK_THREADS) zm[i] = 0;
    }
    {
      const int n_items = a.n_bags * n_poses;
      const int* gbuf = a.ghist + static_cast<size_t>(buf) * a.n_bags * PK_MAX_POSES * a.nb;
      const int* mbuf = a.gmarg + static_cast<size_t>(buf) * a.n_bags * PK_MAX_POSES * PK_MARG_STRIDE;
      // items per round: what the dead histogram copies hold of staged terms, at most one item per warp
      const int round_items = min(PK_WARPS, (a.copies * PK_MAX_POSES * a.nb * 4) / pk_fin_item_bytes(a.nb, a.bins));
      for (int first = 0; first < n_items; first += round_items) {
        const int count = min(round_items, n_items - first);
        unsigned long long* diag = nullptr;
        if (PK_DIAG_STAMPS && blockIdx.x == 0 && first == 0 && a.stamps && batch < static_cast<unsigned long long>(a.stamps_cap)) {
          diag = a.stamps + batch * PK_STAMP_SLOTS + 5;
          if (t == 0) pk_stamp(a, batch, 3);
        }
        pk_block_nid_items(gbuf, mbuf, first, count, n_poses, a.nb, a.bins, smem_hist, sh.fin_out, diag);
        if (t < count) {
          const int item = first + t, ib = item / n_poses, ip = item - ib * n_poses;
          const int word = (a.rank * a.n_bags + ib) * PK_MAX_POSES + ip;
          const double nid = sh.fin_out[t];
          sh.parts[word] = nid;
          // the other ranks get it from one block (NVLink peer stores, tagged words)
          if (a.world > 1 && static_cast<unsigned int>(item) % gridDim.x == blockIdx.x) {
            const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(nid));
            for (int r = 0; r < a.world; r++) {
              if (r == a.rank) continue;
              volatile unsigned long long* dst = a.box[r]->w[slot][word];
              dst[0] = tag | (bits & 0xffffffffull);
              dst[1] = tag | (bits >> 32);
            }
          }
        }
      }
    }
    if (blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 4);
    // ---- (C) the other ranks' scores -> sum over ranks and bags -> Nelder-Mead step -> next poses ---------------------------
    const int n_words = a.world * a.n_bags * n_poses;
    bool timed_out = false;
    if (a.world > 1 && t < n_words && t / (a.n_bags * n_poses) != a.rank) {
      const int src = t / n_poses, p = t % n_poses;  // src = rank * n_bags + bag
      volatile unsigned long long* wsrc = a.box[a.rank]->w[slot][src * PK_MAX_POSES + p];
      const unsigned long long t0 = global_ns();
      unsigned int spins = 0;
      unsigned long long wl, wh;
      for (;;) {
        wl = wsrc[0], wh = wsrc[1];
        if ((wl & 0xffffffff00000000ull) == tag && (wh & 0xffffffff00000000ull) == tag) break;
        if ((++spins & 255u) == 0) {
          if (ld_acquire_u32(a.abort_flag) != 0u) {
            timed_out = true;
            break;
          }
          if (global_ns() - t0 > a.timeout_ns) {
            atomicExch(a.abort_flag, 1u);
            if (a.error_host) *reinterpret_cast<volatile int*>(a.error_host) = 1;
            timed_out = true;
            break;
          }
        }
      }
      sh.parts[src * PK_MAX_POSES + p] = __longlong_as_double(static_cast<long long>((wh << 32) | (wl & 0xffffffffull)));
    }
    if (__syncthreads_or(timed_out ? 1 : 0)) return;
    if (!PK_DIAG_STAMPS && blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 5);
    if (t < n_poses) {
      double total = 0.0;
      for (int s = 0; s < a.world * a.n_bags; s++) total += sh.parts[s * PK_MAX_POSES + t];  // (rank, bag) order: identical everywhere
      sh.ys[t] = total;
    }
    __syncthreads();
    if (warp == 0) {
      nm_warp_step(sh.nm, sh.ys, lane);
      if (blockIdx.x == 0 && lane == 0) pk_stamp(a, batch, 7);
      if (blockIdx.x == 0) {  // reference-order evaluations of this batch, for the callback replay on the host (posted writes)
        const int n_obs = sh.nm.n_obs;
        const int base = sh.trace_count;
        for (int k = 0; k < n_obs; k++) {
          if (base + k < a.trace_cap) {
            double* e = a.trace_host + static_cast<size_t>(base + k) * (NM_MAX_N + 1);
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
    if (blockIdx.x == 0 && t == 0) pk_stamp(a, batch, 6);
  }

  if constexpr (TMA) {
    if (a.tma_stats) {
      const unsigned int nw = __reduce_add_sync(0xffffffffu, w.n_window), ne = __reduce_add_sync(0xffffffffu, w.n_escaped);
      if (lane == 0) {
        atomicAdd(a.tma_stats + 0, static_cast<unsigned long long>(nw));
        atomicAdd(a.tma_stats + 1, static_cast<unsigned long long>(ne));
      }
    }
  }
  // ---- results (block 0) ----
  if (blockIdx.x == 0) {
    if (solve_mode) {
      const unsigned long long batches = static_cast<unsigned long long>(sh.nm.num_batches);
      const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&sh.nm);
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(&a.result_host->nm);
      for (int i = t; i < static_cast<int>(sizeof(NmMachine) / 8); i += PK_THREADS) dst[i] = src[i];
      if (t == 0) {
        a.result_host->batches = batches;
        a.result_host->poses = sh.poses_scored;
        a.result_host->trace_count = sh.trace_count;
        *a.seq_counter = sh.seq_base + batches;  // every rank runs the same number of exchanges
      }
    }
    __threadfence_system();
    __syncthreads();
    if (t == 0 && a.done_host && solve_mode) *reinterpret_cast<volatile unsigned long long*>(a.done_host) = a.done_seq;
  }
}

// debug / test kernel: the lean classifier AND the exact path on every (point, pose); a.dbg: [0] point-poses,
// [1] verdicts deferred to the exact path, [2] kept verdicts that disagree with the exact path (must be 0),
// [3] max over accepted verdicts of |uv_fp32 - uv_exact| / E as float bits (atomicMax; must stay < 1)
template <int MODEL>
__global__ void __launch_bounds__(NID_THREADS) nid_lean_verify_kernel(const __grid_constant__ NidArgs a, const __grid_constant__ LeanCam lc) {
  const float4* __restrict__ pts = static_cast<const float4*>(a.points);
  unsigned long long total = 0, uncertain = 0, mismatch = 0;
  float tmax = 0.f, max_ratio = 0.f;
  for (int p = 0; p < a.n_poses; p++) tmax = fmaxf(tmax, a.pose32[p][12]);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  // points in pairs (2k, 2k + 1), as the hot loop classifies them when the packed classifier is compiled in
  for (long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; 2 * k < a.n; k += stride) {
    const long long i0 = 2 * k, i1 = min(2 * k + 1, static_cast<long long>(a.n) - 1);
    const int n_here = 2 * k + 1 < a.n ? 2 : 1;
    const float4 q2[2] = {__ldg(pts + i0), __ldg(pts + i1)};
    float delta[2];
    for (int h = 0; h < 2; h++) delta[h] = (5.25f * F32_U) * (fabsf(q2[h].x) + fabsf(q2[h].y) + fabsf(q2[h].z) + tmax);
    for (int p = 0; p < a.n_poses; p++) {
      LeanVerdict v2[2];
      if constexpr (PK_PACKED_FP32 && LeanPacked<MODEL>::value) {
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
