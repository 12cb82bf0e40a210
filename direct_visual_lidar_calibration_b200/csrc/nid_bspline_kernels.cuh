// nid_bspline_kernels.cuh -- K2: NIDCost::operator()<double> value ("mode B"), batched over poses.
//
// Reference: include/vlcal/costs/nid_cost.hpp:36-107 -- per point: Sophus SE3 action (quaternion form), projection,
// floor() knot, bounds, hist_points[bin]++ and a 4x4 cubic-B-spline footprint splatted into the joint / image
// histograms with weights beta_x[i]*beta_y[j] (the image itself is never interpolated).  No FoV test on this path.
// Geometry and weights use the exact double path (exact_math.cuh) in the reference's operation order.
// Accumulation: the weights are non-negative and <= 1, so they are accumulated as 2^-F fixed-point integers with
// 64-bit integer atomics -- order independent, hence deterministic run to run.  Every tap is rounded once to the nearest
// multiple of 2^-F, so a bin holding m taps is within m * 2^-(F+1) of the exact sum of the per-tap doubles.
// Headroom: the 16 weights of one point sum to 1, so a joint bin, and an image-marginal row sum in the finalize, holds at
// most n * 2^F (plus m/2 of rounding) for a cloud of n points.  nidb_fixed_bits(n) = min(40, 62 - ceil(log2 n)) keeps
// that below 2^62 < 2^64: F = 40 (4.5e-13 per tap) up to n = 2^22 points, F = 37 (3.6e-12 per tap) at 17.8 M points,
// F = 31 at the 2^31 - 1 point limit of the int hist_points counters.  tests/test_gpu_mode_b_edges.py pins every bin
// against the exact (math.fsum) sum of the reference's taps under that bound.
#pragma once

#include <cstdint>

#include "camera_models.cuh"
#include "dual_math.cuh"

namespace vlcal {

constexpr int NIDB_MAX_POSES = 8;
constexpr int NIDB_THREADS = 256;
constexpr int NIDB_MAX_FIXED_BITS = 40;

// fixed-point fraction bits for a cloud of n points: n * 2^F stays <= 2^62 in every joint bin and image row sum
static inline int nidb_fixed_bits(long long n) {
  int lg = 0;  // ceil(log2(max(n, 1)))
  while (lg < 62 && (1ll << lg) < n) lg++;
  return lg > 62 - NIDB_MAX_FIXED_BITS ? 62 - lg : NIDB_MAX_FIXED_BITS;
}

struct NidBArgs {
  const void* points;        // float4[n] or double4[n]
  const uint8_t* bin_image;  // H x W: min(int(u8 * (1/255.0) * bins), bins-1)  (:78-79 on the CV_64F image)
  long long n;
  int width, height;
  int bins, nb;
  int n_poses;
  int copies;
  CameraParams cam;
  double pose[NIDB_MAX_POSES][8];  // qx qy qz qw tx ty tz (Sophus::SE3d storage, :38)
  double C[4][4];                  // spline_coeffs / 6.0  (:29-33)
  double fixed_one, inv_one;       // 2^F and 2^-F, F = nidb_fixed_bits(n)
  unsigned long long* gjoint;      // [NIDB_MAX_POSES][nb] fixed-point joint histogram accumulators
  int* gpoints;                    // [NIDB_MAX_POSES][bins] hist_points accumulators
  unsigned int* counter;
  double* nid_out;                 // [n_poses]
  int* ok_out;                     // [n_poses] 0 where the reference functor returns false (:98-102)
  double* hist_out;                // optional [n_poses][nb] un-normalised joint histogram, index = bin_image + bin_points*bins
};

static __device__ void nidb_finalize(const NidBArgs& a, unsigned long long* smem_j) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  unsigned long long* h_image = smem_j + static_cast<size_t>(warp) * a.bins;  // fixed-point row sums, per warp
  for (int p = warp; p < a.n_poses; p += n_warps) {
    unsigned long long* g = a.gjoint + static_cast<size_t>(p) * a.nb;
    int* gp = a.gpoints + static_cast<size_t>(p) * a.bins;
    for (int i = lane; i < a.bins; i += 32) h_image[i] = 0ull;
    __syncwarp();
    for (int k = lane; k < a.nb; k += 32) {
      const unsigned long long c = __ldcg(g + k);
      if (c) atomicAdd(&h_image[k % a.bins], c);  // hist_image[bin_image] += w  (:81) == row sum of the joint
    }
    int part = 0;
    for (int k = lane; k < a.bins; k += 32) part += __ldcg(gp + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    __syncwarp();
    const double sum = static_cast<double>(part);  // :86 sum = hist_points.sum()
    const double inv_one = a.inv_one;
    double t_j = 0.0, t_i = 0.0, t_p = 0.0;  // :88-94
    for (int k = lane; k < a.nb; k += 32) {
      const double pr = (static_cast<double>(__ldcg(g + k)) * inv_one) / sum;
      t_j += pr * log(pr + 1e-6);
    }
    for (int k = lane; k < a.bins; k += 32) {
      const double pi = (static_cast<double>(h_image[k]) * inv_one) / sum;
      const double pp = static_cast<double>(__ldcg(gp + k)) / sum;
      t_i += pi * log(pi + 1e-6);
      t_p += pp * log(pp + 1e-6);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      t_j += __shfl_xor_sync(0xffffffffu, t_j, o);
      t_i += __shfl_xor_sync(0xffffffffu, t_i, o);
      t_p += __shfl_xor_sync(0xffffffffu, t_p, o);
    }
    if (lane == 0) {
      const double Hip = -t_j, Hi = -t_i, Hp = -t_p;
      const double MI = Hi + Hp - Hip;
      const double nid = (Hip - MI) / Hip;
      a.nid_out[p] = nid;
      a.ok_out[p] = isfinite(nid) ? 1 : 0;  // :98-102
    }
    for (int k = lane; k < a.nb; k += 32) {
      if (a.hist_out) a.hist_out[static_cast<size_t>(p) * a.nb + k] = static_cast<double>(__ldcg(g + k)) * inv_one;
      g[k] = 0ull;
    }
    for (int k = lane; k < a.bins; k += 32) gp[k] = 0;
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) *a.counter = 0u;
}

template <int MODEL, bool F32>
__global__ void __launch_bounds__(NIDB_THREADS) nid_bspline_kernel(const __grid_constant__ NidBArgs a) {
  extern __shared__ unsigned long long smem_b[];  // [copies][P][nb] joint (fixed point), then [P][bins] hist_points (int)
  __shared__ bool s_is_last;
  const int per_copy = a.n_poses * a.nb;
  int* s_points = reinterpret_cast<int*>(smem_b + static_cast<size_t>(a.copies) * per_copy);
  for (int i = threadIdx.x; i < a.copies * per_copy; i += blockDim.x) smem_b[i] = 0ull;
  for (int i = threadIdx.x; i < a.n_poses * a.bins; i += blockDim.x) s_points[i] = 0;
  __syncthreads();
  unsigned long long* my_joint = smem_b + static_cast<size_t>((threadIdx.x >> 5) % a.copies) * per_copy;

  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    double px, py, pz, pw;
    if constexpr (F32) {
      const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
      px = q.x, py = q.y, pz = q.z, pw = q.w;
    } else {
      const double4 q = static_cast<const double4*>(a.points)[i];
      px = q.x, py = q.y, pz = q.z, pw = q.w;
    }
    // :49 bin_points = max(0, min(bins-1, int(intensity*bins)))
    int bp = cast_int_x86(__dmul_rn(pw, static_cast<double>(a.bins)));
    bp = bp < a.bins - 1 ? bp : a.bins - 1;
    bp = bp > 0 ? bp : 0;
    for (int p = 0; p < a.n_poses; p++) {
      const double* T = a.pose[p];
      // :47 Sophus SO3::operator* (so3.hpp:408-417): uv = q.vec x p; uv += uv; p + w*uv + q.vec x uv; then + t (se3.hpp:319-322)
      const xd qx(T[0]), qy(T[1]), qz(T[2]), qw(T[3]);
      const xd X(px), Y(py), Z(pz);
      xd uvx = qy * Z - qz * Y, uvy = qz * X - qx * Z, uvz = qx * Y - qy * X;
      uvx = uvx + uvx, uvy = uvy + uvy, uvz = uvz + uvz;
      const xd cxv = qy * uvz - qz * uvy, cyv = qz * uvx - qx * uvz, czv = qx * uvy - qy * uvx;
      const xd pcx = (X + qw * uvx + cxv) + xd(T[4]);
      const xd pcy = (Y + qw * uvy + cyv) + xd(T[5]);
      const xd pcz = (Z + qw * uvz + czv) + xd(T[6]);
      xd u, v;
      project_exact<MODEL>(a.cam, pcx, pcy, pcz, u, v);  // :51 no FoV test on this path
      const int kx = cast_int_x86(floor(u.v));            // :52
      const int ky = cast_int_x86(floor(v.v));
      if (kx < 0 || ky < 0 || kx >= a.width || ky >= a.height) continue;  // :55-58
      atomicAdd(&s_points[p * a.bins + bp], 1);                           // :60
      const xd sx = u - xd(static_cast<double>(kx)), sy = v - xd(static_cast<double>(ky));  // :53
      xd bx[4], by[4];  // :62-68 beta = C * [1 s s^2 s^3]^T
      {
        const xd sx2 = sx * sx, sx3 = sx2 * sx, sy2 = sy * sy, sy3 = sy2 * sy;
#pragma unroll
        for (int r = 0; r < 4; r++) {
          bx[r] = ((xd(a.C[r][0]) * xd(1.0) + xd(a.C[r][1]) * sx) + xd(a.C[r][2]) * sx2) + xd(a.C[r][3]) * sx3;
          by[r] = ((xd(a.C[r][0]) * xd(1.0) + xd(a.C[r][1]) * sy) + xd(a.C[r][2]) * sy2) + xd(a.C[r][3]) * sy3;
        }
      }
      unsigned long long* hj = my_joint + p * a.nb + bp * a.bins;
#pragma unroll
      for (int j = 0; j < 4; j++) {  // :70-83
        int yy = ky - 1 + j;
        yy = yy > 0 ? yy : 0;
        yy = yy < a.height - 1 ? yy : a.height - 1;
        const uint8_t* row = a.bin_image + static_cast<size_t>(yy) * a.width;
#pragma unroll
        for (int i2 = 0; i2 < 4; i2++) {
          int xx = kx - 1 + i2;
          xx = xx > 0 ? xx : 0;
          xx = xx < a.width - 1 ? xx : a.width - 1;
          const xd w = bx[i2] * by[j];
          const long long q = __double2ll_rn(w.v * a.fixed_one);
          atomicAdd(&hj[__ldg(row + xx)], static_cast<unsigned long long>(q));  // hist(bin_image, bin_points) += w
        }
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < per_copy; k += blockDim.x) {
    unsigned long long s = 0ull;
    for (int c = 0; c < a.copies; c++) s += smem_b[static_cast<size_t>(c) * per_copy + k];
    if (s) atomicAdd(a.gjoint + k, s);
  }
  for (int k = threadIdx.x; k < a.n_poses * a.bins; k += blockDim.x) {
    const int s = s_points[k];
    if (s) atomicAdd(a.gpoints + k, s);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(a.counter, 1u);
    s_is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_is_last) return;
  __threadfence();
  nidb_finalize(a, smem_b);
}

// ---- K3: value + gradient (NIDCost::operator()<ceres::Jet<double, 7>>) ------------------------------------------
// What ceres::AutoDiffFirstOrderFunction evaluates per bag in the reference's BFGS branch
// (visual_camera_calibration.cpp:211): the mode-B NID and its partials with respect to the 7 ambient pose parameters
// (qx, qy, qz, qw, tx, ty, tz).  Per point:
//   pc(theta) = p + w (2 q x p) + q x (2 q x p) + t               (Sophus SO3 action, polynomial in q as the Jets see it)
//   (u, v), J = d(u, v)/d pc                                       (camera model over xj3 duals)
//   U_k = J_u . d pc/d theta_k,  V_k = J_v . d pc/d theta_k        (k = 0..6)
//   w_ij = bx_i(sx) by_j(sy),  d w_ij/d theta_k = bx'_i by_j U_k + bx_i by'_j V_k
// The joint histogram carries 1 + 7 accumulators per bin: the weights as 2^-F fixed point (deterministic, as in K2),
// the partials as doubles (their range is unbounded; double atomics, so bits may differ run to run at the 1e-13 level).
// The last block turns them into NID and d NID/d theta through the entropy chain rule.
constexpr int NIDG_THREADS = 256;

struct NidGArgs {
  const void* points;
  const uint8_t* bin_image;
  long long n;
  int width, height;
  int bins, nb;
  CameraParams cam;
  double pose[8];
  double C[4][4];
  double fixed_one, inv_one;   // 2^F and 2^-F, F = nidb_fixed_bits(n)
  unsigned long long* gjoint;  // [nb] fixed-point weights
  double* gpart;               // [nb][7] partial sums
  int* gpoints;                // [bins]
  unsigned int* counter;
  double* out;                 // [0] NID, [1..7] gradient, [8] ok (1.0 / 0.0)
};

template <int MODEL, bool F32>
__global__ void __launch_bounds__(NIDG_THREADS) nid_bspline_grad_kernel(const __grid_constant__ NidGArgs a) {
  extern __shared__ unsigned long long smem_g[];  // [nb] weights (u64) | [nb][7] partials (double) | [bins] points (int)
  __shared__ bool s_is_last;
  unsigned long long* s_w = smem_g;
  double* s_d = reinterpret_cast<double*>(smem_g + a.nb);
  int* s_points = reinterpret_cast<int*>(s_d + static_cast<size_t>(a.nb) * 7);
  for (int i = threadIdx.x; i < a.nb; i += blockDim.x) s_w[i] = 0ull;
  for (int i = threadIdx.x; i < a.nb * 7; i += blockDim.x) s_d[i] = 0.0;
  for (int i = threadIdx.x; i < a.bins; i += blockDim.x) s_points[i] = 0;
  __syncthreads();

  const xd qx(a.pose[0]), qy(a.pose[1]), qz(a.pose[2]), qw(a.pose[3]);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    double px, py, pz, pw;
    if constexpr (F32) {
      const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
      px = q.x, py = q.y, pz = q.z, pw = q.w;
    } else {
      const double4 q = static_cast<const double4*>(a.points)[i];
      px = q.x, py = q.y, pz = q.z, pw = q.w;
    }
    int bp = cast_int_x86(__dmul_rn(pw, static_cast<double>(a.bins)));  // :49
    bp = bp < a.bins - 1 ? bp : a.bins - 1;
    bp = bp > 0 ? bp : 0;
    // :47 value of the camera point, in the Jet evaluation's order: ((w uv + p) + q x uv) + t
    const xd X(px), Y(py), Z(pz);
    xd uvx = qy * Z - qz * Y, uvy = qz * X - qx * Z, uvz = qx * Y - qy * X;
    uvx = uvx + uvx, uvy = uvy + uvy, uvz = uvz + uvz;
    const xd cxv = qy * uvz - qz * uvy, cyv = qz * uvx - qx * uvz, czv = qx * uvy - qy * uvx;
    const xd pcx = ((qw * uvx + X) + cxv) + xd(a.pose[4]);
    const xd pcy = ((qw * uvy + Y) + cyv) + xd(a.pose[5]);
    const xd pcz = ((qw * uvz + Z) + czv) + xd(a.pose[6]);
    xj3 u, v;
    project_generic<MODEL, xj3>(a.cam, xj3(pcx, 0), xj3(pcy, 1), xj3(pcz, 2), u, v);  // :51
    const int kx = cast_int_x86(floor(u.a.v));                                          // :52
    const int ky = cast_int_x86(floor(v.a.v));
    if (kx < 0 || ky < 0 || kx >= a.width || ky >= a.height) continue;  // :55-58
    atomicAdd(&s_points[bp], 1);                                        // :60

    // d pc / d theta_k, k = qx qy qz qw tx ty tz
    double D[3][7];
    {
      const double q0 = qx.v, q1 = qy.v, q2 = qz.v, w = qw.v;
      const double uv[3] = {uvx.v, uvy.v, uvz.v};
      const double p[3] = {px, py, pz};
      const double qv[3] = {q0, q1, q2};
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        double e_p[3], e_uv[3];  // e_j x p, e_j x uv
        e_p[j] = 0.0, e_p[j1] = -p[j2], e_p[j2] = p[j1];
        e_uv[j] = 0.0, e_uv[j1] = -uv[j2], e_uv[j2] = uv[j1];
        const double duv[3] = {2.0 * e_p[0], 2.0 * e_p[1], 2.0 * e_p[2]};
        const double cr[3] = {qv[1] * duv[2] - qv[2] * duv[1], qv[2] * duv[0] - qv[0] * duv[2], qv[0] * duv[1] - qv[1] * duv[0]};
#pragma unroll
        for (int c = 0; c < 3; c++) D[c][j] = w * duv[c] + e_uv[c] + cr[c];
      }
#pragma unroll
      for (int c = 0; c < 3; c++) {
        D[c][3] = uv[c];
        D[c][4] = c == 0 ? 1.0 : 0.0;
        D[c][5] = c == 1 ? 1.0 : 0.0;
        D[c][6] = c == 2 ? 1.0 : 0.0;
      }
    }
    double U[7], V[7];
#pragma unroll
    for (int k = 0; k < 7; k++) {
      U[k] = u.v[0] * D[0][k] + u.v[1] * D[1][k] + u.v[2] * D[2][k];
      V[k] = v.v[0] * D[0][k] + v.v[1] * D[1][k] + v.v[2] * D[2][k];
    }
    // :53, :62-68 beta = C [1 s s^2 s^3]^T and d beta / d s
    const xd sx = u.a - xd(static_cast<double>(kx)), sy = v.a - xd(static_cast<double>(ky));
    const xd sx2 = sx * sx, sx3 = sx2 * sx, sy2 = sy * sy, sy3 = sy2 * sy;
    double bx[4], by[4], dbx[4], dby[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      bx[r] = (((xd(a.C[r][0]) * xd(1.0) + xd(a.C[r][1]) * sx) + xd(a.C[r][2]) * sx2) + xd(a.C[r][3]) * sx3).v;
      by[r] = (((xd(a.C[r][0]) * xd(1.0) + xd(a.C[r][1]) * sy) + xd(a.C[r][2]) * sy2) + xd(a.C[r][3]) * sy3).v;
      dbx[r] = a.C[r][1] + 2.0 * a.C[r][2] * sx.v + 3.0 * a.C[r][3] * sx2.v;
      dby[r] = a.C[r][1] + 2.0 * a.C[r][2] * sy.v + 3.0 * a.C[r][3] * sy2.v;
    }
    const int row_base = bp * a.bins;
#pragma unroll
    for (int j = 0; j < 4; j++) {  // :70-83
      int yy = ky - 1 + j;
      yy = yy > 0 ? yy : 0;
      yy = yy < a.height - 1 ? yy : a.height - 1;
      const uint8_t* row = a.bin_image + static_cast<size_t>(yy) * a.width;
      // taps of one footprint row that fall into the same bin are merged before touching shared memory
      int tb[4];
      double tw[4], tgx[4], tgy[4];
#pragma unroll
      for (int i2 = 0; i2 < 4; i2++) {
        int xx = kx - 1 + i2;
        xx = xx > 0 ? xx : 0;
        xx = xx < a.width - 1 ? xx : a.width - 1;
        tb[i2] = __ldg(row + xx);
        tw[i2] = __dmul_rn(bx[i2], by[j]);
        tgx[i2] = dbx[i2] * by[j];
        tgy[i2] = bx[i2] * dby[j];
      }
      unsigned int done = 0;
#pragma unroll
      for (int t = 0; t < 4; t++) {
        if ((done >> t) & 1u) continue;
        long long wq = __double2ll_rn(tw[t] * a.fixed_one);
        double gx = tgx[t], gy = tgy[t];
#pragma unroll
        for (int t2 = t + 1; t2 < 4; t2++) {
          if (tb[t2] == tb[t]) {
            wq += __double2ll_rn(tw[t2] * a.fixed_one);
            gx += tgx[t2], gy += tgy[t2];
            done |= 1u << t2;
          }
        }
        const int bin = row_base + tb[t];
        atomicAdd(&s_w[bin], static_cast<unsigned long long>(wq));
        double* dst = s_d + static_cast<size_t>(bin) * 7;
#pragma unroll
        for (int k = 0; k < 7; k++) atomicAdd(dst + k, gx * U[k] + gy * V[k]);
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < a.nb; k += blockDim.x) {
    if (s_w[k]) atomicAdd(a.gjoint + k, s_w[k]);
  }
  for (int k = threadIdx.x; k < a.nb * 7; k += blockDim.x) {
    if (s_d[k] != 0.0) atomicAdd(a.gpart + k, s_d[k]);
  }
  for (int k = threadIdx.x; k < a.bins; k += blockDim.x) {
    if (s_points[k]) atomicAdd(a.gpoints + k, s_points[k]);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(a.counter, 1u);
    s_is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_is_last) return;
  __threadfence();

  // ---- finalize: entropies and their partials (:86-96 over Jets) -------------------------------------------------
  // shared memory is reused: s_w -> joint values (double), s_d -> joint partials, then marginal scratch
  __shared__ double s_red[NIDG_THREADS];
  __shared__ double s_sum;
  double* jv = reinterpret_cast<double*>(s_w);
  const double inv_one = a.inv_one;
  int part = 0;
  for (int k = threadIdx.x; k < a.bins; k += blockDim.x) part += __ldcg(a.gpoints + k);
  s_red[threadIdx.x] = static_cast<double>(part);
  __syncthreads();
  for (int o = NIDG_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) s_sum = s_red[0];
  __syncthreads();
  const double sum = s_sum;  // :86
  for (int k = threadIdx.x; k < a.nb; k += blockDim.x) jv[k] = (static_cast<double>(__ldcg(a.gjoint + k)) * inv_one) / sum;
  for (int k = threadIdx.x; k < a.nb * 7; k += blockDim.x) s_d[k] = __ldcg(a.gpart + k) / sum;
  __syncthreads();
  // t[0] = sum p log(p + eps) over the joint, t[1..7] its partials; same for the image marginal (row sums over lidar bins)
  double tj[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ti[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tp = 0.0;
  for (int k = threadIdx.x; k < a.nb; k += blockDim.x) {
    const double p = jv[k];
    const double lg = log(p + 1e-6);
    tj[0] += p * lg;
    const double f = lg + p / (p + 1e-6);
    for (int c = 0; c < 7; c++) tj[1 + c] += s_d[static_cast<size_t>(k) * 7 + c] * f;
  }
  for (int b = threadIdx.x; b < a.bins; b += blockDim.x) {
    double p = 0.0, dp[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int l = 0; l < a.bins; l++) {  // hist_image[bin_image] = sum over bin_points (:81)
      const int k = b + l * a.bins;
      p += jv[k];
      for (int c = 0; c < 7; c++) dp[c] += s_d[static_cast<size_t>(k) * 7 + c];
    }
    const double lg = log(p + 1e-6);
    ti[0] += p * lg;
    const double f = lg + p / (p + 1e-6);
    for (int c = 0; c < 7; c++) ti[1 + c] += dp[c] * f;
    const double pp = static_cast<double>(__ldcg(a.gpoints + b)) / sum;
    tp += pp * log(pp + 1e-6);
  }
  double red[17];
  for (int q = 0; q < 17; q++) {
    const double val = q < 8 ? tj[q] : (q < 16 ? ti[q - 8] : tp);
    __syncthreads();
    s_red[threadIdx.x] = val;
    __syncthreads();
    for (int o = NIDG_THREADS / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
      __syncthreads();
    }
    red[q] = s_red[0];
  }
  if (threadIdx.x == 0) {
    const double Hip = -red[0], Hi = -red[8], Hp = -red[16];
    const double MI = Hi + Hp - Hip;
    const double num = Hip - MI;
    const double nid = num / Hip;
    a.out[0] = nid;
    for (int c = 0; c < 7; c++) {
      const double dHip = -red[1 + c], dHi = -red[9 + c];
      const double dnum = dHip - (dHi - dHip);  // d(Hip - MI), MI = Hi + Hp - Hip
      a.out[1 + c] = (dnum - nid * dHip) / Hip;
    }
    a.out[8] = isfinite(nid) ? 1.0 : 0.0;  // :98-102
  }
  __syncthreads();
  for (int k = threadIdx.x; k < a.nb; k += blockDim.x) a.gjoint[k] = 0ull;
  for (int k = threadIdx.x; k < a.nb * 7; k += blockDim.x) a.gpart[k] = 0.0;
  for (int k = threadIdx.x; k < a.bins; k += blockDim.x) a.gpoints[k] = 0;
  if (threadIdx.x == 0) *a.counter = 0u;
}

}  // namespace vlcal
