// nid_sweep.cuh -- K1s: the NID of a LONG pose list over SMALL clouds, pose-parallel (sm_90a).
//
// The global initial-guess search (initial_guess_search.py) scores 10^5-10^6 poses on a thinned cloud of 10^4-10^5 points.
// K1p's pose-list mode (nid_persistent.cuh) is point-parallel: 8 poses per pass, ceil(N / 768) blocks, grid-wide
// accumulators handed from scoring blocks to owner blocks -- at N = 16 384 that is 22 blocks and one dependent pass per 8
// poses.  Here the roles are swapped: a block owns a group of SW_POSES poses from start to finish.  It streams every bag's
// cloud (L2-resident at these sizes), classifies each loaded point against its poses (CostCalculatorNID::calculate,
// src/vlcal/calib/cost_calculator_nid.cpp:30-52), keeps the joint histograms in shared memory and reduces them to the NID
// itself (:54-64), in the canonical summation order of nid_finalize / pk_block_nid -- equal histograms give equal bits,
// whichever kernel counted them.  Groups are dealt to the blocks by a grid-stride loop; a plain launch: no block ever
// waits for another one, no global accumulator, no atomics outside shared memory.
//
// Classifier: the lean fp32 filter (lean_filter.cuh, classify_lean) with the exact fp64 arbiter (exact_classify.cuh)
// behind a per-warp queue, i.e. the pair the persistent kernel uses, so the integer histograms are the reference's.
#pragma once

#include <cstdint>

#include "exact_classify.cuh"
#include "lean_filter.cuh"
#include "nid_kernels.cuh"

namespace vlcal {

constexpr int SW_THREADS = 256;
constexpr int SW_WARPS = SW_THREADS / 32;
constexpr int SW_POSES = 4;       // poses that share each loaded point
constexpr int SW_MAX_BAGS = 8;
constexpr int SW_MAX_BINS = 32;   // nb <= 1024
constexpr int SW_QUEUE = 64;      // per-warp queue of (point, pose) pairs waiting for the exact path
constexpr int SW_FIN_CH = (SW_MAX_BINS * SW_MAX_BINS + SW_THREADS - 1) / SW_THREADS;  // joint bins per thread

struct SweepBag {
  const float4* points;
  const uint8_t* bin_image;
  unsigned int n;
};

struct SweepArgs {
  SweepBag bag[SW_MAX_BAGS];
  int n_bags;
  int width, height;
  int bins, nb;
  double cos_fov;
  CameraParams cam;
  FastCam fast;
  LeanCam lean;
  const double* poses;   // [n_poses][12] row-major 3x4 [R|t] of T_camera_lidar
  long long n_poses;
  double* scores;        // [n_poses]: sum over the bags, in bag order
  int* hist_out;         // optional [n_poses][nb] of bag 0, index = image_bin + lidar_bin*bins
  long long* inliers;    // optional [n_poses]: points counted, summed over the bags (hist_image.sum() of :54)
  unsigned long long* deferred;  // optional debug count of the (point, pose) pairs sent to the exact path; nullptr: none
};

struct SweepShared {
  int hist[SW_POSES][SW_MAX_BINS * SW_MAX_BINS];
  double term[SW_MAX_BINS * SW_MAX_BINS];  // staged p*log(p + 1e-6) of the joint histogram
  double mterm[2 * SW_MAX_BINS];           // ... of the two marginals
  int marg[2 * SW_MAX_BINS];               // image marginal, then lidar marginal
  double pose64[SW_POSES][12];
  float pose32[SW_POSES][12];              // R (9, row-major), t (3)
  float tmax;                              // max |t| over the group, rounded up (bound of the fp32 filter)
  double score[SW_POSES];
  long long inliers[SW_POSES];
  double nid;
  int cnt[SW_WARPS];
  unsigned int q_idx[SW_WARPS][SW_QUEUE];
  unsigned char q_pose[SW_WARPS][SW_QUEUE];
};

// the deferred (point, pose) pairs [first, first + count) of this warp's queue, one per lane, through the exact path
template <int MODEL>
__device__ __forceinline__ void sweep_drain32(const SweepArgs& a, SweepShared& sh, const SweepBag& B, int warp, int lane, int first, int count) {
  if (lane < count) {
    const unsigned int i = sh.q_idx[warp][first + lane];
    const int p = sh.q_pose[warp][first + lane];
    const float4 q = __ldg(B.points + i);
    const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, sh.pose64[p], q.x, q.y, q.z);
    if (pix >= 0) atomicAdd(&sh.hist[p][__ldg(B.bin_image + pix) + lidar_bin_of(q.w, a.bins) * a.bins], 1);  // :49
  }
  if (a.deferred && lane == 0) atomicAdd(a.deferred, static_cast<unsigned long long>(count));
}

// The NID of one joint histogram in shared memory, by the whole block (cost_calculator_nid.cpp:54-64): the arithmetic and
// the summation order of pk_block_nid (nid_persistent.cuh) and nid_finalize (nid_kernels.cuh).
static __device__ __noinline__ double sweep_block_nid(SweepShared& sh, const int* __restrict__ h, int nb, int bins, int* __restrict__ hist_out, int* __restrict__ total_out) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int i = t; i < 2 * bins; i += SW_THREADS) sh.marg[i] = 0;
  __syncthreads();
  int c[SW_FIN_CH];
  int part = 0;
#pragma unroll
  for (int m = 0; m < SW_FIN_CH; m++) {
    const int k = m * SW_THREADS + t;
    c[m] = k < nb ? h[k] : 0;
    if (c[m]) {
      atomicAdd(&sh.marg[k % bins], c[m]);         // hist_image[image_bin]   (:50)
      atomicAdd(&sh.marg[bins + k / bins], c[m]);  // hist_points[lidar_bin]  (:51)
      part += c[m];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) sh.cnt[warp] = part;
  __syncthreads();
  int total = 0;
#pragma unroll
  for (int w = 0; w < SW_WARPS; w++) total += sh.cnt[w];
  *total_out = total;
  const double sum = static_cast<double>(total);  // :54 sum = hist_image.sum()
#pragma unroll
  for (int m = 0; m < SW_FIN_CH; m++) {
    const int k = m * SW_THREADS + t;
    if (k < nb) {
      const double pr = static_cast<double>(c[m]) / sum;
      sh.term[k] = entropy_term(pr);  // :59-61
      if (hist_out) hist_out[k] = c[m];
    }
  }
  for (int f = t; f < 2 * bins; f += SW_THREADS) {
    const double pm = static_cast<double>(sh.marg[f]) / sum;
    sh.mterm[f] = entropy_term(pm);
  }
  __syncthreads();
  if (warp == 0) {
    double t_rs = 0.0, t_r = 0.0, t_s = 0.0;
    for (int k = lane; k < nb; k += 32) t_rs += sh.term[k];
    for (int k = lane; k < bins; k += 32) {
      t_r += sh.mterm[k];
      t_s += sh.mterm[bins + k];
    }
    const double Hrs = -warp_tree_sum(t_rs), Hr = -warp_tree_sum(t_r), Hs = -warp_tree_sum(t_s);
    if (lane == 0) {
      const double MI = Hr + Hs - Hrs;  // :63
      sh.nid = (Hrs - MI) / Hrs;        // :64 (NaN when there are no inliers, as in the reference)
    }
  }
  __syncthreads();
  return sh.nid;
}

template <int MODEL>
__global__ void __launch_bounds__(SW_THREADS) nid_pose_sweep_kernel(const __grid_constant__ SweepArgs a) {
  __shared__ SweepShared sh;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const unsigned int lt_mask = (1u << lane) - 1u;
  const long long n_groups = (a.n_poses + SW_POSES - 1) / SW_POSES;
  for (long long group = blockIdx.x; group < n_groups; group += gridDim.x) {
    const long long p0 = group * SW_POSES;
    const int n_p = static_cast<int>(min(static_cast<long long>(SW_POSES), a.n_poses - p0));
    __syncthreads();  // the previous group's shared state is no longer read
    if (t < n_p * 12) {
      const double v = a.poses[p0 * 12 + t];
      sh.pose64[t / 12][t % 12] = v;
      const int r = (t % 12) / 4, c = t % 4;  // pose32: R row-major, then t
      sh.pose32[t / 12][c < 3 ? 3 * r + c : 9 + r] = static_cast<float>(v);
    }
    __syncthreads();
    if (t == 0) {
      double tm = 0.0;
      for (int p = 0; p < n_p; p++)
        for (int r = 0; r < 3; r++) tm = fmax(tm, fabs(sh.pose64[p][4 * r + 3]));
      sh.tmax = nextafterf(static_cast<float>(tm), INFINITY);
    }
    for (int b = 0; b < a.n_bags; b++) {
      const SweepBag B = a.bag[b];
      for (int i = t; i < n_p * a.nb; i += SW_THREADS) sh.hist[i / a.nb][i % a.nb] = 0;
      __syncthreads();
      const float tmax = sh.tmax;
      int qn = 0;  // this warp's queue fill, warp-uniform
      // rows of 32 consecutive points per warp, the next row's load in flight while this one is classified
      unsigned int row = static_cast<unsigned int>(warp) * 32u;
      float4 q = make_float4(0.f, 0.f, -1.f, 0.f);
      if (row + lane < B.n) q = __ldg(B.points + row + lane);
      for (; row < B.n; row += SW_THREADS) {
        const unsigned int i = row + lane;
        const bool valid = i < B.n;
        const float4 cur = q;
        const unsigned int nxt = i + SW_THREADS;
        if (nxt < B.n) q = __ldg(B.points + nxt);
        const float dl = (5.25f * F32_U) * (fabsf(cur.x) + fabsf(cur.y) + fabsf(cur.z) + tmax);
        const int lboff = lidar_bin_of(cur.w, a.bins) * a.bins;
        unsigned int unc_mask = 0u;  // bit p: pose p deferred this point
#pragma unroll
        for (int p = 0; p < SW_POSES; p++) {
          if (p < n_p) {
            const LeanVerdict v = classify_lean<MODEL>(a.fast, a.lean, a.width, sh.pose32[p], cur.x, cur.y, cur.z, dl);
            if (v.accept & valid) atomicAdd(&sh.hist[p][__ldg(B.bin_image + v.idx) + lboff], 1);  // :49 hist(image_bin, lidar_bin)++
            if (v.uncertain & valid) unc_mask |= 1u << p;
          }
        }
        // deferred pairs of this row -> the warp's queue, re-decided 32 at a time so that the fp64 path runs with full warps
        if (__any_sync(0xffffffffu, unc_mask != 0u)) {
#pragma unroll
          for (int p = 0; p < SW_POSES; p++) {
            const bool mine = (unc_mask >> p) & 1u;
            const unsigned int m = __ballot_sync(0xffffffffu, mine);
            if (m) {
              if (mine) {
                const int pos = qn + __popc(m & lt_mask);
                sh.q_idx[warp][pos] = i;
                sh.q_pose[warp][pos] = static_cast<unsigned char>(p);
              }
              qn += __popc(m);
              __syncwarp();
              if (qn >= 32) {
                sweep_drain32<MODEL>(a, sh, B, warp, lane, qn - 32, 32);
                qn -= 32;
                __syncwarp();
              }
            }
          }
        }
      }
      if (qn > 0) sweep_drain32<MODEL>(a, sh, B, warp, lane, 0, qn);
      __syncthreads();
      for (int p = 0; p < n_p; p++) {
        int* ho = (a.hist_out && b == 0) ? a.hist_out + (p0 + p) * a.nb : nullptr;
        int total;
        const double nid = sweep_block_nid(sh, sh.hist[p], a.nb, a.bins, ho, &total);
        // sum_costs over the bags in bag order (visual_camera_calibration.cpp:105-110), as vlcal_nid_score_poses adds them
        if (t == 0) {
          sh.score[p] = a.n_bags == 1 ? nid : (b == 0 ? 0.0 : sh.score[p]) + nid;
          sh.inliers[p] = (b == 0 ? 0ll : sh.inliers[p]) + total;
        }
      }
    }
    __syncthreads();
    if (t < n_p) {
      a.scores[p0 + t] = sh.score[t];
      if (a.inliers) a.inliers[p0 + t] = sh.inliers[t];
    }
  }
}

// ---- search sets: poses generated on the device ------------------------------------------------------------------------------
// Pose i of a set = (base ib, left il, offset io), i = (ib * n_left + il) * n_offset + io:
//   R = left[il] * base[ib],  t = R * (center[ib] + offset[io])
// with every product and sum an explicit round-to-nearest operation in a fixed order, so that a host that does the same
// IEEE operations in the same order (initial_guess.search_set_poses, numpy) gets the same bits.  No transcendental is
// evaluated here: the tables carry them.
struct SearchSetDev {
  const double* left;    // [n_left][9] row-major
  const double* base;    // [n_base][9]
  const double* center;  // [n_base][3]
  const double* offset;  // [n_offset][3]
  const int* indices;    // optional [n_poses] flat indices i; nullptr: pose j is flat index j
  int n_left, n_base, n_offset;
  long long n_poses;
};

static __global__ void search_set_poses_kernel(const SearchSetDev s, double* __restrict__ out) {
  const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= s.n_poses) return;
  const long long i = s.indices ? s.indices[j] : j;
  const int io = static_cast<int>(i % s.n_offset);
  const int il = static_cast<int>((i / s.n_offset) % s.n_left);
  const int ib = static_cast<int>(i / (static_cast<long long>(s.n_offset) * s.n_left));
  const double* L = s.left + 9 * il;
  const double* B = s.base + 9 * ib;
  double v[3];
  for (int k = 0; k < 3; k++) v[k] = __dadd_rn(s.center[3 * ib + k], s.offset[3 * io + k]);
  double* T = out + 12 * j;
  for (int r = 0; r < 3; r++) {
    double R[3];
    for (int c = 0; c < 3; c++) R[c] = __dadd_rn(__dadd_rn(__dmul_rn(L[3 * r], B[c]), __dmul_rn(L[3 * r + 1], B[3 + c])), __dmul_rn(L[3 * r + 2], B[6 + c]));
    T[4 * r] = R[0], T[4 * r + 1] = R[1], T[4 * r + 2] = R[2];
    T[4 * r + 3] = __dadd_rn(__dadd_rn(__dmul_rn(R[0], v[0]), __dmul_rn(R[1], v[1])), __dmul_rn(R[2], v[2]));
  }
}

}  // namespace vlcal
