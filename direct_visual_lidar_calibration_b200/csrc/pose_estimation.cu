// pose_estimation.cu -- PoseEstimation, the solver behind initial_guess_auto
// (reference: src/vlcal/common/estimate_pose.cpp, include/vlcal/common/estimate_pose.hpp, include/vlcal/costs/reprojection_cost.hpp).
//
//   bearings    host: estimate_direction (NelderMead<2>) per keypoint, normalised LiDAR points (:47-51).  NelderMead stops
//               at a simplex spread of ~1e-3 rad, so its result follows last-ulp differences of sin/cos; it stays on the
//               host, where it runs libm's like the reference.
//   hypotheses  host: the index pairs a one-thread reference run draws (:86-106).
//   scoring     device, one launch: every hypothesis's rotation (Umeyama on its two bearing pairs, :55-83) and its inlier
//               count over all correspondences (:108-116), correspondences streamed through shared memory in tiles.
//   winner      host argmax of the counts (count desc, index asc = the first strictly greater count of :118-123);
//               a second launch writes its inlier mask (:127-134).
//   refinement  host Levenberg-Marquardt of the Cauchy-robustified reprojection error on SE(3) (:148-177); M is small.
#include <omp.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <random>
#include <vector>

#include "dual_math.cuh"
#include "host_math.hpp"
#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {

constexpr int POSE_THREADS = 128;  // hypotheses per block
constexpr int POSE_TILE = 256;     // correspondences per shared-memory tile: 5 doubles each, 10 KB
// |d1 - d2|^2 or |d1 + d2|^2 below this on either side (bearings within ~1e-9 rad of parallel / antiparallel), or the same
// index drawn twice: the two pairs do not determine a unique rotation
constexpr double POSE_DEGENERATE_SQ = 1e-18;

// Umeyama's rotation for two bearing pairs (c_k = R l_k), in closed form.  For unit vectors a = c1 + c2 and b = c1 - c2
// are orthogonal, as are p = l1 + l2 and q = l1 - l2, so AB = sum_k c_k l_k^T = (a p^T + b q^T) / 2 is already an SVD:
// U = [a^, b^, a^ x b^], V = [p^, q^, p^ x q^], both proper rotations, so S = I and R = U V^T.  For rank-2 AB this is
// the unique solution JacobiSVD's U S V^T also gives, to rounding.  Only + - * / sqrt, never contracted: the host and the
// device compute the same bits.  Returns false for a degenerate pair (R untouched).
VL_HD bool pair_rotation(const double c1[3], const double c2[3], const double l1[3], const double l2[3], xd R[9]) {
  xd a[3], b[3], p[3], q[3];
  for (int k = 0; k < 3; k++) {
    a[k] = xd(c1[k]) + xd(c2[k]);
    b[k] = xd(c1[k]) - xd(c2[k]);
    p[k] = xd(l1[k]) + xd(l2[k]);
    q[k] = xd(l1[k]) - xd(l2[k]);
  }
  const xd na = sqnorm3(a[0], a[1], a[2]), nb = sqnorm3(b[0], b[1], b[2]);
  const xd np = sqnorm3(p[0], p[1], p[2]), nq = sqnorm3(q[0], q[1], q[2]);
  const xd eps(POSE_DEGENERATE_SQ);
  if (!(na >= eps && nb >= eps && np >= eps && nq >= eps)) return false;  // also rejects NaN
  const xd ia = xd(1.0) / xsqrt(na), ib = xd(1.0) / xsqrt(nb), ip = xd(1.0) / xsqrt(np), iq = xd(1.0) / xsqrt(nq);
  for (int k = 0; k < 3; k++) a[k] = a[k] * ia, b[k] = b[k] * ib, p[k] = p[k] * ip, q[k] = q[k] * iq;
  const xd u3[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
  const xd v3[3] = {p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[3 * r + c] = (a[r] * p[c] + b[r] * q[c]) + u3[r] * v3[c];
  return true;
}

// |kp0 - project(R d_l)|^2 (:110-113): the unit direction is projected, without the FoV test
template <int MODEL>
VL_HD xd pose_sq_error(const CameraParams& cam, const xd R[9], xd x, xd y, xd z, xd kx, xd ky) {
  const xd px = (R[0] * x + R[1] * y) + R[2] * z;
  const xd py = (R[3] * x + R[4] * y) + R[5] * z;
  const xd pz = (R[6] * x + R[7] * y) + R[8] * z;
  xd u, v;
  project_exact<MODEL>(cam, px, py, pz, u, v);
  const xd du = kx - u, dv = ky - v;
  return du * du + dv * dv;
}

struct PoseScoreArgs {
  const double* dl;    // [3][M] LiDAR bearings, structure of arrays
  const double* dc;    // [3][M] camera bearings
  const double* kp;    // [2][M] keypoints
  const int2* pairs;   // [H]
  int m, h;
  double thresh_sq;
  CameraParams cam;
  int* counts;            // [H], zeroed by the caller
  unsigned char* degenerate;  // [H]
};

__device__ __forceinline__ bool load_rotation(const PoseScoreArgs& a, int2 ij, xd R[9]) {
  const long long m = a.m;  // 2m + i exceeds INT_MAX above 2^30 correspondences
  const double c1[3] = {a.dc[ij.x], a.dc[m + ij.x], a.dc[2 * m + ij.x]};
  const double c2[3] = {a.dc[ij.y], a.dc[m + ij.y], a.dc[2 * m + ij.y]};
  const double l1[3] = {a.dl[ij.x], a.dl[m + ij.x], a.dl[2 * m + ij.x]};
  const double l2[3] = {a.dl[ij.y], a.dl[m + ij.y], a.dl[2 * m + ij.y]};
  return ij.x != ij.y && pair_rotation(c1, c2, l1, l2, R);
}

// one thread per hypothesis; blockIdx.y strides over the tiles, so a few hypothesis blocks still fill the GPU.  All threads
// of a block read the same tile entry at once (shared-memory broadcast).  Integer counts: the atomics' order does not matter.
template <int MODEL>
__global__ void __launch_bounds__(POSE_THREADS, 4) pose_score_kernel(const __grid_constant__ PoseScoreArgs a) {
  __shared__ double tile[5][POSE_TILE];
  const int hyp = blockIdx.x * POSE_THREADS + threadIdx.x;
  xd R[9];
  bool ok = false;
  if (hyp < a.h) {
    ok = load_rotation(a, a.pairs[hyp], R);
    if (blockIdx.y == 0) a.degenerate[hyp] = ok ? 0 : 1;
  }
  int count = 0;
  for (long long base = static_cast<long long>(blockIdx.y) * POSE_TILE; base < a.m; base += static_cast<long long>(gridDim.y) * POSE_TILE) {
    const int n = static_cast<int>(min(static_cast<long long>(POSE_TILE), a.m - base));
    __syncthreads();  // the previous tile has been consumed
    for (int k = threadIdx.x; k < n; k += POSE_THREADS) {
      const long long j = base + k;
      tile[0][k] = a.dl[j], tile[1][k] = a.dl[a.m + j], tile[2][k] = a.dl[2LL * a.m + j];
      tile[3][k] = a.kp[j], tile[4][k] = a.kp[a.m + j];
    }
    __syncthreads();
    if (ok) {
      for (int k = 0; k < n; k++) {
        const xd e = pose_sq_error<MODEL>(a.cam, R, tile[0][k], tile[1][k], tile[2][k], tile[3][k], tile[4][k]);
        count += e < xd(a.thresh_sq) ? 1 : 0;
      }
    }
  }
  if (count > 0) atomicAdd(a.counts + hyp, count);
}

template <int MODEL>
__global__ void __launch_bounds__(256) pose_mask_kernel(const __grid_constant__ PoseScoreArgs a, int2 winner, unsigned char* mask) {
  __shared__ double Rs[9];
  if (threadIdx.x == 0) {
    xd R[9];
    load_rotation(a, winner, R);  // the winner has inliers, so it is not degenerate
    for (int k = 0; k < 9; k++) Rs[k] = R[k].v;
  }
  __syncthreads();
  const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  xd R[9];
  for (int k = 0; k < 9; k++) R[k] = Rs[k];
  const xd e = pose_sq_error<MODEL>(a.cam, R, a.dl[j], a.dl[a.m + j], a.dl[2LL * a.m + j], a.kp[j], a.kp[a.m + j]);
  mask[j] = e < xd(a.thresh_sq) ? 1 : 0;
}

using PoseScoreKernel = void (*)(const PoseScoreArgs);
using PoseMaskKernel = void (*)(const PoseScoreArgs, int2, unsigned char*);

template <int MODEL>
static void pick_pose_model(PoseScoreKernel* score, PoseMaskKernel* mask) {
  *score = pose_score_kernel<MODEL>;
  *mask = pose_mask_kernel<MODEL>;
}

static bool pick_pose_kernels(int model, PoseScoreKernel* score, PoseMaskKernel* mask) {
  switch (model) {
    case CAM_PLUMB_BOB: pick_pose_model<CAM_PLUMB_BOB>(score, mask); return true;
    case CAM_FISHEYE: pick_pose_model<CAM_FISHEYE>(score, mask); return true;
    case CAM_ATAN: pick_pose_model<CAM_ATAN>(score, mask); return true;
    case CAM_OMNIDIR: pick_pose_model<CAM_OMNIDIR>(score, mask); return true;
    case CAM_EQUIRECTANGULAR: pick_pose_model<CAM_EQUIRECTANGULAR>(score, mask); return true;
    case CAM_RATIONAL_POLYNOMIAL: pick_pose_model<CAM_RATIONAL_POLYNOMIAL>(score, mask); return true;
    default: return false;
  }
}

namespace {

struct DevBuf {
  void* p = nullptr;
  int device = 0;
  cudaError_t alloc(int dev, size_t bytes) {
    device = dev;
    return MemPool::instance().device_alloc(dev, bytes, &p);
  }
  ~DevBuf() { MemPool::instance().device_free(device, p); }
};

// correspondences as the kernels read them: bearings and keypoints, structure of arrays
struct Bearings {
  int m = 0;
  std::vector<double> dl, dc, kp;  // [3][M], [3][M], [2][M]
};

int check_correspondences(const double* kp0, const double* points, int64_t m) {
  if (m < 2 || m > INT_MAX || !kp0 || !points) {
    set_last_error("pose estimation needs at least 2 correspondences (and at most 2^31-1)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int64_t i = 0; i < m; i++) {
    const double* p = points + 3 * i;
    const bool finite = std::isfinite(kp0[2 * i]) && std::isfinite(kp0[2 * i + 1]) && std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]);
    if (!finite || (p[0] == 0.0 && p[1] == 0.0 && p[2] == 0.0)) {
      set_last_error("correspondence " + std::to_string(i) + ": keypoint and point must be finite and the point non-zero (it has no bearing)");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  return VLCAL_OK;
}

// estimate_pose.cpp:47-51
void compute_bearings(const CameraParams& cam, const double* kp0, const double* points, int m, Bearings* b) {
  b->m = m;
  b->dl.resize(3 * static_cast<size_t>(m));
  b->dc.resize(3 * static_cast<size_t>(m));
  b->kp.resize(2 * static_cast<size_t>(m));
#pragma omp parallel for schedule(dynamic, 64)
  for (int i = 0; i < m; i++) {
    double dc[3];
    estimate_direction_host(cam, kp0 + 2 * i, dc);
    const double* p = points + 3 * i;
    const double n = std::sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);  // Eigen normalized(): v / sqrt(squaredNorm)
    for (int k = 0; k < 3; k++) {
      b->dc[static_cast<size_t>(k) * m + i] = dc[k];
      b->dl[static_cast<size_t>(k) * m + i] = p[k] / n;
    }
    b->kp[i] = kp0[2 * i];
    b->kp[static_cast<size_t>(m) + i] = kp0[2 * i + 1];
  }
}

// :86-106 with omp_get_max_threads() == 1: mts[0] = mt19937(mt() + 8192 * 0), two draws per iteration.  A multi-threaded
// reference run hands each thread its own generator and iterations, so it scores a different set (and picks among equal
// counts in whatever order the threads reach the critical section); one thread is the reproducible run.
void sample_pairs(int m, int iterations, int32_t* out) {
  std::mt19937 mt;
  std::mt19937 mt0(mt() + 8192 * 0);
  for (int i = 0; i < iterations; i++) {
    std::uniform_int_distribution<> udist(0, m - 1);
    out[2 * i] = udist(mt0);
    out[2 * i + 1] = udist(mt0);
  }
}

// the scoring launch (and, with mask != nullptr, the mask of the argmax): counts / degenerate flags per hypothesis
int score_hypotheses(
  int device, const CameraParams& cam, const Bearings& b, const int32_t* pairs, int h, double thresh, int32_t* counts, uint8_t* degenerate, int* best,
  uint8_t* mask, double* kernel_ms = nullptr) {
  PoseScoreKernel score_kernel = nullptr;
  PoseMaskKernel mask_kernel = nullptr;
  if (!pick_pose_kernels(cam.model, &score_kernel, &mask_kernel)) {
    set_last_error("unknown camera model id");
    return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
  }
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available: this library has no CPU fallback");
    return VLCAL_ERR_NO_DEVICE;
  }
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  const int m = b.m;
  DevBuf d_dl, d_dc, d_kp, d_pairs, d_counts, d_degenerate, d_mask;
  VL_CUDA(d_dl.alloc(device, sizeof(double) * 3 * static_cast<size_t>(m)));
  VL_CUDA(d_dc.alloc(device, sizeof(double) * 3 * static_cast<size_t>(m)));
  VL_CUDA(d_kp.alloc(device, sizeof(double) * 2 * static_cast<size_t>(m)));
  VL_CUDA(d_pairs.alloc(device, sizeof(int2) * static_cast<size_t>(h)));
  VL_CUDA(d_counts.alloc(device, sizeof(int) * static_cast<size_t>(h)));
  VL_CUDA(d_degenerate.alloc(device, static_cast<size_t>(h)));
  VL_CUDA(cudaMemcpy(d_dl.p, b.dl.data(), sizeof(double) * b.dl.size(), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_dc.p, b.dc.data(), sizeof(double) * b.dc.size(), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_kp.p, b.kp.data(), sizeof(double) * b.kp.size(), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_pairs.p, pairs, sizeof(int2) * static_cast<size_t>(h), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemset(d_counts.p, 0, sizeof(int) * static_cast<size_t>(h)));

  PoseScoreArgs a;
  std::memset(&a, 0, sizeof(a));
  a.dl = static_cast<const double*>(d_dl.p);
  a.dc = static_cast<const double*>(d_dc.p);
  a.kp = static_cast<const double*>(d_kp.p);
  a.pairs = static_cast<const int2*>(d_pairs.p);
  a.m = m, a.h = h;
  a.thresh_sq = std::pow(thresh, 2);  // :108
  a.cam = cam;
  a.counts = static_cast<int*>(d_counts.p);
  a.degenerate = static_cast<unsigned char*>(d_degenerate.p);
  int num_sms = 1;
  VL_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
  const int hyp_blocks = (h + POSE_THREADS - 1) / POSE_THREADS;
  const long long tiles = (m + POSE_TILE - 1) / POSE_TILE;
  // about four blocks per SM in all: split the correspondences when there are few hypothesis blocks
  const long long split = std::max<long long>(1, std::min<long long>(tiles, (4LL * num_sms + hyp_blocks - 1) / hyp_blocks));
  cudaEvent_t ev[2] = {nullptr, nullptr};
  if (kernel_ms) {
    VL_CUDA(cudaEventCreate(&ev[0]));
    VL_CUDA(cudaEventCreate(&ev[1]));
    VL_CUDA(cudaEventRecord(ev[0]));
  }
  score_kernel<<<dim3(hyp_blocks, static_cast<unsigned int>(split)), POSE_THREADS>>>(a);
  VL_CUDA(cudaGetLastError());
  if (kernel_ms) {
    VL_CUDA(cudaEventRecord(ev[1]));
    VL_CUDA(cudaEventSynchronize(ev[1]));
    float ms = 0.f;
    VL_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    *kernel_ms = ms;
    cudaEventDestroy(ev[0]);
    cudaEventDestroy(ev[1]);
  }
  VL_CUDA(cudaMemcpy(counts, d_counts.p, sizeof(int) * static_cast<size_t>(h), cudaMemcpyDeviceToHost));
  if (degenerate) VL_CUDA(cudaMemcpy(degenerate, d_degenerate.p, static_cast<size_t>(h), cudaMemcpyDeviceToHost));
  if (!best) return VLCAL_OK;

  int w = 0;
  for (int i = 1; i < h; i++)
    if (counts[i] > counts[w]) w = i;
  *best = w;
  if (counts[w] <= 0) {
    set_last_error("RANSAC found no hypothesis with an inlier: no rotation reprojects any correspondence within ransac_error_thresh");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (mask) {
    VL_CUDA(d_mask.alloc(device, static_cast<size_t>(m)));
    mask_kernel<<<static_cast<unsigned int>((m + 255) / 256), 256>>>(a, make_int2(pairs[2 * w], pairs[2 * w + 1]), static_cast<unsigned char*>(d_mask.p));
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cudaMemcpy(mask, d_mask.p, static_cast<size_t>(m), cudaMemcpyDeviceToHost));
  }
  return VLCAL_OK;
}

// ---------------------------------------------------------------------------------------------
// refinement: min 1/2 sum_i rho(|r_i|^2), r_i = project(T p_i) - kp0_i, rho(s) = b log(1 + s / b), b = width^2
// (ceres::CauchyLoss(width), :160-166).  Levenberg-Marquardt with Ceres' defaults (trust region radius 1e4, D = diag(J^T J)
// clamped to [1e-6, 1e32], step accepted at a relative decrease > 1e-3) and its residual scaling for a loss with rho'' < 0:
// plain sqrt(rho') weights.  T is updated on the left, T <- Exp(delta) T, delta = (omega, v) (a chart of SE(3) like
// Sophus' x * exp(delta); the minimiser is the same).  Stops: 50 iterations, |dF| <= 1e-6 F, max|g| <= 1e-10,
// |delta| <= 1e-8 (|x| + 1e-8).  Unlike Ceres an accepted step below the parameter tolerance is applied before stopping.
// ---------------------------------------------------------------------------------------------

struct RefineProblem {
  CameraParams cam;
  const double* kp0;
  const double* points;
  int m;
  double b;  // robust_kernel_width^2
};

template <int MODEL>
double refine_eval_model(const RefineProblem& pr, const double T[16], double g[6], double H[36]) {
  double F = 0.0;
  if (g) std::memset(g, 0, sizeof(double) * 6), std::memset(H, 0, sizeof(double) * 36);
  for (int i = 0; i < pr.m; i++) {
    const double* p = pr.points + 3 * i;
    double pc[3];
    for (int r = 0; r < 3; r++) pc[r] = ((host::m4(T, r, 0) * p[0] + host::m4(T, r, 1) * p[1]) + host::m4(T, r, 2) * p[2]) + host::m4(T, r, 3);
    xj3 u, v;
    project_generic<MODEL, xj3>(pr.cam, xj3(xd(pc[0]), 0), xj3(xd(pc[1]), 1), xj3(xd(pc[2]), 2), u, v);
    const double r0 = u.a.v - pr.kp0[2 * i], r1 = v.a.v - pr.kp0[2 * i + 1];
    const double s = r0 * r0 + r1 * r1;
    const double sum = 1.0 + s / pr.b;
    F += 0.5 * (pr.b * std::log(sum));
    if (!g) continue;
    const double w = std::max(1.0 / sum, DBL_MIN);  // rho'
    // d pc / d delta = [-[pc]x | I]  for delta = (omega, v)
    const double dpc[3][6] = {{0.0, pc[2], -pc[1], 1.0, 0.0, 0.0}, {-pc[2], 0.0, pc[0], 0.0, 1.0, 0.0}, {pc[1], -pc[0], 0.0, 0.0, 0.0, 1.0}};
    double J[2][6];
    for (int k = 0; k < 6; k++) {
      J[0][k] = (u.v[0] * dpc[0][k] + u.v[1] * dpc[1][k]) + u.v[2] * dpc[2][k];
      J[1][k] = (v.v[0] * dpc[0][k] + v.v[1] * dpc[1][k]) + v.v[2] * dpc[2][k];
    }
    for (int k = 0; k < 6; k++) {
      g[k] += w * (J[0][k] * r0 + J[1][k] * r1);
      for (int l = 0; l < 6; l++) H[6 * k + l] += w * (J[0][k] * J[0][l] + J[1][k] * J[1][l]);
    }
  }
  return F;
}

double refine_eval(const RefineProblem& pr, const double T[16], double g[6], double H[36]) {
  switch (pr.cam.model) {
    case CAM_PLUMB_BOB: return refine_eval_model<CAM_PLUMB_BOB>(pr, T, g, H);
    case CAM_FISHEYE: return refine_eval_model<CAM_FISHEYE>(pr, T, g, H);
    case CAM_ATAN: return refine_eval_model<CAM_ATAN>(pr, T, g, H);
    case CAM_OMNIDIR: return refine_eval_model<CAM_OMNIDIR>(pr, T, g, H);
    case CAM_EQUIRECTANGULAR: return refine_eval_model<CAM_EQUIRECTANGULAR>(pr, T, g, H);
    default: return refine_eval_model<CAM_RATIONAL_POLYNOMIAL>(pr, T, g, H);
  }
}

// (A) x = rhs for a symmetric positive definite 6x6 A (Cholesky); false if A is not positive definite
bool solve6(const double A[36], const double rhs[6], double x[6]) {
  double L[36] = {0.0};
  for (int i = 0; i < 6; i++) {
    for (int j = 0; j <= i; j++) {
      double s = A[6 * i + j];
      for (int k = 0; k < j; k++) s -= L[6 * i + k] * L[6 * j + k];
      if (i == j) {
        if (!(s > 0.0)) return false;
        L[6 * i + i] = std::sqrt(s);
      } else {
        L[6 * i + j] = s / L[6 * j + j];
      }
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double s = rhs[i];
    for (int k = 0; k < i; k++) s -= L[6 * i + k] * y[k];
    y[i] = s / L[6 * i + i];
  }
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < 6; k++) s -= L[6 * k + i] * x[k];
    x[i] = s / L[6 * i + i];
  }
  return true;
}

void refine(const RefineProblem& pr, const double init_T[16], double T_out[16], int* iterations, double* final_cost) {
  constexpr int max_iterations = 50;
  constexpr double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  double T[16], g[6], H[36];
  std::memcpy(T, init_T, sizeof(T));
  double F = refine_eval(pr, T, g, H);
  double radius = 1e4, decrease_factor = 2.0;
  int it = 0;
  while (it < max_iterations) {
    double gmax = 0.0;
    for (int k = 0; k < 6; k++) gmax = std::max(gmax, std::fabs(g[k]));
    if (gmax <= gradient_tolerance) break;
    it++;
    double A[36], rhs[6], delta[6];
    std::memcpy(A, H, sizeof(A));
    for (int k = 0; k < 6; k++) {
      A[7 * k] += std::min(std::max(H[7 * k], 1e-6), 1e32) / radius;
      rhs[k] = -g[k];
    }
    if (!solve6(A, rhs, delta)) {
      radius /= decrease_factor, decrease_factor *= 2.0;
      continue;
    }
    double E[16], T_new[16];
    host::se3_expmap_gtsam(delta, E);
    host::isometry_mul(E, T, T_new);
    const double F_new = refine_eval(pr, T_new, nullptr, nullptr);
    double model = 0.0;  // -(g.delta + 1/2 delta^T H delta)
    for (int k = 0; k < 6; k++) {
      double Hd = 0.0;
      for (int l = 0; l < 6; l++) Hd += H[6 * k + l] * delta[l];
      model -= g[k] * delta[k] + 0.5 * delta[k] * Hd;
    }
    double step = 0.0, xnorm = 1.0;
    for (int k = 0; k < 6; k++) step += delta[k] * delta[k];
    for (int r = 0; r < 3; r++) xnorm += host::m4(T, r, 3) * host::m4(T, r, 3);
    const bool small_step = std::sqrt(step) <= parameter_tolerance * (std::sqrt(xnorm) + parameter_tolerance);
    const double ratio = model > 0.0 ? (F - F_new) / model : -1.0;
    if (std::isfinite(F_new) && ratio > 1e-3) {
      const double decrease = F - F_new;
      std::memcpy(T, T_new, sizeof(T));
      F = refine_eval(pr, T, g, H);
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * ratio - 1.0, 3));
      decrease_factor = 2.0;
      if (decrease <= function_tolerance * (F + decrease) || small_step) break;
    } else {
      if (small_step) break;
      radius /= decrease_factor, decrease_factor *= 2.0;
    }
  }
  std::memcpy(T_out, T, sizeof(T));
  if (iterations) *iterations = it;
  if (final_cost) *final_cost = F;
}

void to_colmajor_rotation(const xd R[9], double T[16]) {
  std::memset(T, 0, sizeof(double) * 16);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) host::m4(T, r, c) = R[3 * r + c].v;
  host::m4(T, 3, 3) = 1.0;
}

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" {

void vlcal_pose_estimation_default_params(vlcal_pose_estimation_params* p) {
  // the values estimate_pose.hpp:10-14 sets and the reference always runs (its constructor ignores the params argument)
  p->ransac_iterations = 8192;
  p->ransac_error_thresh = 5.0;
  p->robust_kernel_width = 10.0;
}

int vlcal_estimate_directions(
  int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double* pixels, int64_t n, double* dirs_out) {
  if (n < 0 || (n > 0 && (!pixels || !dirs_out))) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  const int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t i = 0; i < n; i++) estimate_direction_host(cam, pixels + 2 * i, dirs_out + 3 * i);
  return VLCAL_OK;
}

int vlcal_pose_debug_sample_pairs(int64_t n_correspondences, int n_iterations, int32_t* pairs_out) {
  if (n_correspondences < 2 || n_correspondences > INT_MAX || n_iterations < 0 || (n_iterations > 0 && !pairs_out)) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  sample_pairs(static_cast<int>(n_correspondences), n_iterations, pairs_out);
  return VLCAL_OK;
}

int vlcal_pose_debug_score_pairs(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double* kp0, const double* points,
  int64_t n_correspondences, const int32_t* pairs, int n_pairs, double ransac_error_thresh, int32_t* counts_out, uint8_t* degenerate_out, double* kernel_ms_out) {
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  rc = check_correspondences(kp0, points, n_correspondences);
  if (rc != VLCAL_OK) return rc;
  if (n_pairs < 1 || !pairs || !counts_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i < 2 * n_pairs; i++) {
    if (pairs[i] < 0 || pairs[i] >= n_correspondences) {
      set_last_error("pair index out of range");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  Bearings b;
  compute_bearings(cam, kp0, points, static_cast<int>(n_correspondences), &b);
  return score_hypotheses(device, cam, b, pairs, n_pairs, ransac_error_thresh, counts_out, degenerate_out, nullptr, nullptr, kernel_ms_out);
}

int vlcal_pose_debug_refine(
  int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double* kp0, const double* points,
  int64_t n_correspondences, double robust_kernel_width, const double init_T_camera_lidar[16], double T_camera_lidar_out[16], int* iterations_out,
  double* final_cost_out) {
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  rc = check_correspondences(kp0, points, n_correspondences);
  if (rc != VLCAL_OK) return rc;
  if (!(robust_kernel_width > 0.0) || !init_T_camera_lidar || !T_camera_lidar_out) {
    set_last_error("invalid arguments (robust_kernel_width must be > 0)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  const RefineProblem pr{cam, kp0, points, static_cast<int>(n_correspondences), robust_kernel_width * robust_kernel_width};
  refine(pr, init_T_camera_lidar, T_camera_lidar_out, iterations_out, final_cost_out);
  return VLCAL_OK;
}

int vlcal_estimate_pose_from_correspondences(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double* kp0, const double* points,
  int64_t n_correspondences, const vlcal_pose_estimation_params* params, double T_camera_lidar_out[16], uint8_t* inlier_mask_out,
  vlcal_pose_estimation_stats* stats_out) {
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  rc = check_correspondences(kp0, points, n_correspondences);
  if (rc != VLCAL_OK) return rc;
  vlcal_pose_estimation_params p;
  vlcal_pose_estimation_default_params(&p);
  if (params) p = *params;
  if (p.ransac_iterations < 1 || !(p.ransac_error_thresh > 0.0) || !(p.robust_kernel_width > 0.0) || !T_camera_lidar_out) {
    set_last_error("invalid arguments (ransac_iterations >= 1, ransac_error_thresh > 0 and robust_kernel_width > 0)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  const int m = static_cast<int>(n_correspondences);
  Bearings b;
  compute_bearings(cam, kp0, points, m, &b);
  std::vector<int32_t> pairs(2 * static_cast<size_t>(p.ransac_iterations)), counts(p.ransac_iterations);
  std::vector<uint8_t> degenerate(p.ransac_iterations);
  sample_pairs(m, p.ransac_iterations, pairs.data());
  int best = 0;
  rc = score_hypotheses(device, cam, b, pairs.data(), p.ransac_iterations, p.ransac_error_thresh, counts.data(), degenerate.data(), &best, inlier_mask_out);
  if (rc != VLCAL_OK) return rc;

  // [R_ransac | 0] (:24-25), R recomputed on the host: the same operations give the same bits as on the device
  const size_t i1 = static_cast<size_t>(pairs[2 * best]), i2 = static_cast<size_t>(pairs[2 * best + 1]), mm = static_cast<size_t>(m);
  const double c1[3] = {b.dc[i1], b.dc[mm + i1], b.dc[2 * mm + i1]}, c2[3] = {b.dc[i2], b.dc[mm + i2], b.dc[2 * mm + i2]};
  const double l1[3] = {b.dl[i1], b.dl[mm + i1], b.dl[2 * mm + i1]}, l2[3] = {b.dl[i2], b.dl[mm + i2], b.dl[2 * mm + i2]};
  xd R[9];
  pair_rotation(c1, c2, l1, l2, R);
  double T0[16];
  to_colmajor_rotation(R, T0);
  const RefineProblem pr{cam, kp0, points, m, p.robust_kernel_width * p.robust_kernel_width};
  int iterations = 0;
  double cost = 0.0;
  refine(pr, T0, T_camera_lidar_out, &iterations, &cost);
  if (stats_out) {
    stats_out->hypotheses = p.ransac_iterations;
    stats_out->degenerate = 0;
    for (uint8_t d : degenerate) stats_out->degenerate += d;
    stats_out->best_index = best;
    stats_out->best_inliers = counts[best];
    stats_out->lm_iterations = iterations;
    stats_out->final_cost = cost;
  }
  return VLCAL_OK;
}

}  // extern "C"
