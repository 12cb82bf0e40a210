// nid_kernels.cuh -- K1: batched NID joint-histogram kernel with fused finalize (sm_90a).
//
// Replaces the serial loop of CostCalculatorNID::calculate (reference:
// src/vlcal/calib/cost_calculator_nid.cpp:30-52) and its entropy/NID tail (:54-64) for P candidate
// poses in ONE pass over the cloud:
//   per point  : one coalesced 16-byte load (x,y,z,intensity as float4 -- lossless, SURVEY D9), prefetched one tile ahead
//   per pose   : SE3 transform, FoV test, camera projection, truncation, bounds test, 1-byte gather from the
//                pre-binned image, one shared-memory histogram increment.  Default kernel: fp32 with a rigorous
//                per-point error bound, anything within the bound of a decision edge re-decided by the exact fp64
//                path (bit-identical histograms); nid_hist_exact_kernel does everything in fp64.
//   per block  : P x bins x bins int32 histogram copies in shared memory, merged into the global accumulator with
//                one red.global.add per non-zero bin
//   last block : marginals (row/column sums), the three entropies, MI and NID for every pose; optionally the sum over
//                ranks (NVLink peer-memory exchange) and the next Nelder-Mead batch (device-resident loop); results
//                published to mapped host memory; accumulators zeroed again so the next launch needs no memset.
// Algorithmic traffic: 16 B/point + W*H B of image per pass regardless of P (DESIGN.md section 5); the active bound is
// instruction issue (108 warp-instructions per point-pose) and, for Nelder-Mead sized batches, the serial tail.
#pragma once

#include <cstdint>

#include "camera_models.cuh"
#include "nm_machine.cuh"
#include "se3_math.cuh"

namespace vlcal {

constexpr int NID_MAX_POSES = 8;   // poses carried by one launch
constexpr int NID_THREADS = 256;   // threads per block
constexpr int NID_MAX_BINS = 128;  // bins*bins*4 B must fit shared memory at least once

// ---- fused bag all-reduce over NVLink peer memory (multi-GPU, one bag per rank) -------------------------------
// The joint objective is sum_bags NID (visual_camera_calibration.cpp:105-110).  With one process per GPU and one bag
// per process, the finalizing block of every rank stores its P scores straight into every peer's mailbox (P2P stores
// through NVLink / NVSwitch, buffers shared with cudaIpc; data words carry a sequence tag), waits for the other ranks'
// words and adds the G contributions in rank order -- so all ranks publish bit-identical sums without a separate collective
// launch and without leaving the kernel.  Two slots (seq & 1) because a rank can be at most one exchange ahead.
constexpr int P2P_MAX_RANKS = 8;
// Each double travels as two 8-byte words {32 data bits | 32-bit sequence tag}: an aligned 8-byte store is never torn,
// so the data IS its own arrival flag -- no fence + separate flag store (one NVLink round trip less per exchange).
struct P2PMailbox {
  unsigned long long ll[P2P_MAX_RANKS][2][8][2];  // [sender][slot][pose][lo, hi]
};

// ---- device-resident Nelder-Mead loop ---------------------------------------------------------------------
// With NidArgs::nm set, a launch takes its candidate poses from this block of device memory instead of from its kernel
// parameters, and the finalizing block -- once the scores of the batch are known -- advances the Nelder-Mead state
// machine (nm_machine.cuh) and writes the NEXT batch of poses T = init_T * Expmap(x) back into it.  The host can then
// enqueue many launches back to back without waiting for any of them: the per-iteration host round trip (launch
// latency + PCIe + wake-up) disappears from the critical path.  Launches enqueued after
// the solver finished see n_poses == 0 and exit at once.
struct NmDevice {
  NmMachine nm;
  double init_T[16];                    // column-major start pose (visual_camera_calibration.cpp:104)
  double pose[NID_MAX_POSES][12];       // pending batch: row-major 3x4 [R|t]
  float pose32[NID_MAX_POSES][16];      // fp32 filter copy (R, t, max|t|)
  int n_poses;                          // poses of the pending batch; 0 once finished
  int trace_cap, trace_count;           // reference-order evaluations (x[6], y) for callback replay on the host
  double* trace;
  unsigned long long steps_done;
};

struct NidArgs {
  const void* points;        // float4[n] (x,y,z,intensity) or double4[n]
  const uint8_t* bin_image;  // H x W image bins: clamp(int(u8/255.0*bins), 0, bins-1)  (:43,:46)
  long long n;
  int width, height;
  int bins, nb;  // nb = bins*bins
  int n_poses;   // poses in this launch (<= NID_MAX_POSES)
  int copies;    // shared-memory histogram copies per block
  int finalize_split;  // 1: the block's shared memory is large enough to stage one pose's terms per warp group (nid_finalize)
  double cos_fov;             // cos(max_fov)  (:32)
  CameraParams cam;
  double pose[NID_MAX_POSES][12];  // row-major 3x4 [R|t] of T_camera_lidar
  float pose32[NID_MAX_POSES][16]; // fp32 filter copy: R (9, row-major), t (3), max|t| (1), pad
  FastCam fast;                    // fp32 filter constants (fast.enabled == 0 -> exact kernel only)
  unsigned long long* dbg;         // verify kernel only: {point-poses, uncertain, mismatches, max ratio bits}
  P2PMailbox* peer_box[P2P_MAX_RANKS];  // peer_box[r]: rank r's mailbox as mapped in this process (self included)
  int p2p_world, p2p_rank;         // p2p_world <= 1: no exchange
  int* p2p_error;                  // mapped host word, set to 1 if a peer never answered
  unsigned long long* p2p_counter; // device word: number of exchanges done (kept on the device so that it only advances
                                   // when an exchange really happens -- launches that exit early do not consume a slot)
  NmDevice* nm;                    // device-resident solver loop (nullptr: poses come from the kernel parameters)
  unsigned long long* timeline;    // optional [16] mapped host words: globaltimer stamps of the launch (vlcal_nid_debug_timeline)
  int* ghist;                 // [NID_MAX_POSES][nb] global accumulators, zero on entry, zero on exit
  unsigned int* counter;      // block ticket, zero on entry, zero on exit
  double* nid_out;            // [n_poses]
  double* nid_host;           // optional zero-copy mirror of nid_out in mapped pinned host memory
  unsigned long long* done_flag;  // optional mapped host word; receives done_seq after the results are visible
  unsigned long long done_seq;
  int* hist_out;              // optional [n_poses][nb], index = image_bin + lidar_bin*bins
};

// where a launch reads its poses from: kernel parameters (constant bank) or, in the device-resident loop, NmDevice
template <bool DEVLOOP>
__device__ __forceinline__ int n_poses_of(const NidArgs& a) {
  if constexpr (DEVLOOP) return a.nm->n_poses;
  else return a.n_poses;
}
template <bool DEVLOOP>
__device__ __forceinline__ const double* pose_of(const NidArgs& a, int p) {
  if constexpr (DEVLOOP) return a.nm->pose[p];
  else return a.pose[p];
}
template <bool DEVLOOP>
__device__ __forceinline__ const float* pose32_of(const NidArgs& a, int p) {
  if constexpr (DEVLOOP) return a.nm->pose32[p];
  else return a.pose32[p];
}

// ---- exact decision for one (point, pose): pixel index iy*W+ix (>= 0), or -1 if the reference skips the point
template <int MODEL>
__device__ __forceinline__ int exact_pixel(const NidArgs& a, const double* __restrict__ T, double x, double y, double z, double* u_out = nullptr, double* v_out = nullptr) {
  // :31 pt_camera = T * p  -> ((m0*x + m1*y) + m2*z) + m3
  const xd X(x), Y(y), Z(z);
  const xd pcx = ((xd(T[0]) * X + xd(T[1]) * Y) + xd(T[2]) * Z) + xd(T[3]);
  const xd pcy = ((xd(T[4]) * X + xd(T[5]) * Y) + xd(T[6]) * Z) + xd(T[7]);
  const xd pcz = ((xd(T[8]) * X + xd(T[9]) * Y) + xd(T[10]) * Z) + xd(T[11]);
  // :32 pt_camera.head<3>().normalized().z() < cos(max_fov)
  const xd n2 = sqnorm3(pcx, pcy, pcz);
  const xd nz = n2 > xd(0.0) ? pcz / xsqrt(n2) : pcz;
  if (nz < xd(a.cos_fov)) {
    return -1;
  }
  // :37 project + cast<int> (truncation; NaN -> INT_MIN)
  xd u, v;
  project_exact<MODEL>(a.cam, pcx, pcy, pcz, u, v);
  if (u_out) *u_out = u.v;
  if (v_out) *v_out = v.v;
  const int ix = cast_int_x86(u.v);
  const int iy = cast_int_x86(v.v);
  // :38
  if (ix < 0 || iy < 0 || ix >= a.width || iy >= a.height) {
    return -1;
  }
  return iy * a.width + ix;
}

template <int MODEL>
__device__ __forceinline__ int classify_exact(const NidArgs& a, const double* __restrict__ T, double x, double y, double z) {
  const int pix = exact_pixel<MODEL>(a, T, x, y, z);
  return pix < 0 ? -1 : static_cast<int>(__ldg(a.bin_image + pix));  // :43,:46 via the pre-binned image
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// timeline slots: 0 first block start, 1 last-block: main loop done, 2 merged+fenced, 3 ticket known, 4 finalize done,
// 5 results published (after the system fence); inside finalize: 7 scratch zeroed, 8 marginals + count known,
// 9 entropy terms staged
__device__ __forceinline__ void stamp(const NidArgs& a, int slot) {
  if (a.timeline && threadIdx.x == 0) a.timeline[slot] = global_ns();
}

// ---- fp32 filter --------------------------------------------------------------------------------------------
constexpr int VERDICT_REJECT = -1;     // certainly skipped by the reference
constexpr int VERDICT_UNCERTAIN = -2;  // within the error bound of a decision edge: ask the exact path

// fp32 classification of one (point, pose), written without data-dependent branches (predicate logic only).
// P = pose32 row: R (9, row-major), t (3), max|t|.  Returns pixel index (>= 0), VERDICT_REJECT or VERDICT_UNCERTAIN.
// Decision order mirrors the reference: FoV (:32), then the two truncated coordinates against the image (:37-38).
template <int MODEL>
__device__ __forceinline__ int classify_fast(const NidArgs& a, const float* __restrict__ P, float x, float y, float z, float a_p) {
  const float pcx = fmaf(P[0], x, fmaf(P[1], y, fmaf(P[2], z, P[9])));
  const float pcy = fmaf(P[3], x, fmaf(P[4], y, fmaf(P[5], z, P[10])));
  const float pcz = fmaf(P[6], x, fmaf(P[7], y, fmaf(P[8], z, P[11])));
  const float n2 = fmaf(pcx, pcx, fmaf(pcy, pcy, pcz * pcz));
  const float nrm = n2 * rsqrtf(n2);
  const float delta = (5.25f * F32_U) * (a_p + P[12]);
  // FoV: sign of g = pcz - cos_fov*|pc| with |g_fp32 - g_exact| <= 2.8 delta + 8.5 u |pc|
  const float g = fmaf(-a.fast.cos_fov, nrm, pcz);
  const float mf = fmaf(3.0f, delta, (12.0f * F32_U) * nrm);
  const bool fov_unc = !(fabsf(g) > mf);  // also catches NaN / n2 == 0
  const bool fov_rej = g < 0.0f;
  float u, v, Eu, Ev;
  const bool proj_ok = project_fast<MODEL>(a.fast, pcx, pcy, pcz, nrm, delta, u, v, Eu, Ev);
  // an integer (truncation edge / image border) within the bound of either coordinate -> uncertain.  |c - rint(c)| <= 0.5,
  // so a bound >= 0.5 (useless) or NaN lands here too, and a coordinate that is NOT near an integer truncates exactly
  // like the reference's, wherever it lies: no separate far-outside test is needed.
  const bool edge = !(fabsf(u - rintf(u)) > Eu) || !(fabsf(v - rintf(v)) > Ev);
  const int ix = __float2int_rz(u), iy = __float2int_rz(v);  // truncation toward zero, like cast<int>()
  const bool inside = static_cast<unsigned int>(ix) < static_cast<unsigned int>(a.width) && static_cast<unsigned int>(iy) < static_cast<unsigned int>(a.height);
  const bool uncertain = fov_unc || (!fov_rej && (edge || !proj_ok));
  const bool accept = !fov_unc && !fov_rej && !edge && proj_ok && inside;
  return accept ? iy * a.width + ix : (uncertain ? VERDICT_UNCERTAIN : VERDICT_REJECT);
}

__device__ __forceinline__ int lidar_bin_of(double intensity, int bins) {
  // :44,:47 lidar_bin = max(0, min(bins-1, int(intensity*bins)))
  int lb = cast_int_x86(__dmul_rn(intensity, static_cast<double>(bins)));
  lb = lb < bins - 1 ? lb : bins - 1;
  return lb > 0 ? lb : 0;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// entropies + NID for every pose of the launch; run by the last block only (:54-64).
// This is the serial tail of every launch, so it is laid out for latency: the block's 8 warps are split evenly over
// the P poses (8/P warps per pose), every lane fetches its joint bins with independent L2 loads, and a lane evaluates
// only nb / (32 * warps_per_pose) logarithms.  Marginals are the row / column sums of the joint (the reference
// increments all three together, :49-51).
// The NID must be a function of the histogram ALONE (Nelder-Mead compares scores that were computed in launches with
// different P; equal histograms must give equal bits): the p*log(p) terms are therefore staged in shared memory and
// reduced by one warp in a canonical order -- lane l adds terms l, l+32, ... in ascending order, then a fixed xor tree.
constexpr int FIN_CH = 8;

// natural logarithm for normal, positive, finite arguments (here p + 1e-6 in [1e-6, 1 + 1e-6]), without the special-case
// branches of the library routine, so that the independent terms a lane evaluates interleave instead of serialising
// (the library log serialised the terms in the launch's serial tail).  Algorithm of fdlibm's __ieee754_log (argument
// reduction to [sqrt(1/2), sqrt(2)), s = f/(2+f), degree-14 even/odd polynomial split, hi/lo ln2), error < 1 ulp.
// Every operation is an explicit round-to-nearest intrinsic: the value is a function of x alone, whatever code the call is
// inlined into (the finalizers of the round-1 kernels and of the persistent kernel must produce the same bits -- the solver
// trajectories are compared evaluation by evaluation -- and left to itself the compiler contracts a*b+c differently from one
// inlining context to the next).
__device__ __forceinline__ double log_pos_normal(double x) {
  const long long bits = __double_as_longlong(x);
  int k = static_cast<int>((bits >> 52) & 0x7ff) - 1023;
  double m = __longlong_as_double((bits & 0x000fffffffffffffLL) | 0x3ff0000000000000LL);  // [1, 2)
  const bool hi = m > 1.4142135623730951;
  m = hi ? __dmul_rn(m, 0.5) : m;
  k += hi ? 1 : 0;
  const double f = __dadd_rn(m, -1.0);
  const double s = __ddiv_rn(f, __dadd_rn(2.0, f));
  const double z = __dmul_rn(s, s);
  const double w = __dmul_rn(z, z);
  const double t1 = __dmul_rn(w, __fma_rn(w, __fma_rn(w, 1.531383769920937332e-01, 2.222219843214978396e-01), 3.999999999940941908e-01));
  const double t2 = __dmul_rn(z, __fma_rn(w, __fma_rn(w, __fma_rn(w, 1.479819860511658591e-01, 1.818357216161805012e-01), 2.857142874366239149e-01), 6.666666666666735130e-01));
  const double R = __dadd_rn(t1, t2);
  const double hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
  const double dk = static_cast<double>(k);
  const double b = __fma_rn(s, __dadd_rn(hfsq, R), __dmul_rn(dk, 1.90821492927058770002e-10));
  const double c = __dadd_rn(__dadd_rn(hfsq, -b), -f);
  return __fma_rn(dk, 6.93147180369123816490e-01, -c);
}

// p * log(p + 1e-6) (cost_calculator_nid.cpp:59-61), rounded after the sum, the logarithm and the product
__device__ __forceinline__ double entropy_term(double p) { return __dmul_rn(p, log_pos_normal(__dadd_rn(p, 1e-6))); }

__device__ __forceinline__ double warp_tree_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// called by the finalizing block after every pose's local score sits in a.nid_out (block-synchronised)
static __device__ void nid_peer_allreduce(const NidArgs& a, int n_poses) {
  __shared__ unsigned long long s_seq;
  __shared__ double s_part[P2P_MAX_RANKS][8];
  stamp(a, 10);
  const int t = threadIdx.x;
  if (t == 0) s_seq = ++(*a.p2p_counter);  // every rank performs the same sequence of exchanges
  __syncthreads();
  const unsigned long long seq = s_seq;
  const int slot = static_cast<int>(seq & 1ull);
  const unsigned long long tag = ((seq & 0x7fffffffull) | 0x80000000ull) << 32;  // never 0 (the mailbox starts zeroed)
  if (t < n_poses * a.p2p_world) {  // one thread per (peer, pose)
    const int g = t / n_poses, p = t % n_poses;
    {  // remote stores over NVLink: our partial sum -> rank g's mailbox
      const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(a.nid_out[p]));
      volatile unsigned long long* dst = a.peer_box[g]->ll[a.p2p_rank][slot][p];
      dst[0] = tag | (bits & 0xffffffffull);
      dst[1] = tag | (bits >> 32);
    }
    {  // wait for rank g's partial sum of pose p to land in OUR mailbox
      volatile unsigned long long* src = a.peer_box[a.p2p_rank]->ll[g][slot][p];
      const unsigned long long t0 = global_ns();
      unsigned int spins = 0;
      unsigned long long lo, hi;
      for (;;) {
        lo = src[0], hi = src[1];
        if ((lo & 0xffffffff00000000ull) == tag && (hi & 0xffffffff00000000ull) == tag) break;
        if ((++spins & 1023u) == 0 && global_ns() - t0 > 2000000000ull) {  // 2 s: a peer died or fell out of lockstep
          if (a.p2p_error) *a.p2p_error = 1;
          break;
        }
      }
      s_part[g][p] = __longlong_as_double(static_cast<long long>((hi << 32) | (lo & 0xffffffffull)));
    }
  }
  __syncthreads();
  stamp(a, 11);
  if (t < n_poses) {
    double total = 0.0;
    for (int r = 0; r < a.p2p_world; r++) total += s_part[r][t];  // rank order: identical on every rank
    a.nid_out[t] = total;
    if (a.nid_host) a.nid_host[t] = total;
  }
  __syncthreads();
}

// T = init_T * Expmap(x) for one candidate of the pending batch (visual_camera_calibration.cpp:104) -> pose / pose32 slot k
VL_HD void nm_pose_of_candidate(const double* cand_vertex, const double* init_T, NmDevice* out, int k) {
  double E[16], T[16];
  se3_expmap_gtsam_hd(cand_vertex + 1, E);
  isometry_mul_hd(init_T, E, T);
  double tmax = 0.0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 4; c++) out->pose[k][4 * r + c] = T[r + 4 * c];
    for (int c = 0; c < 3; c++) out->pose32[k][3 * r + c] = static_cast<float>(T[r + 4 * c]);
    out->pose32[k][9 + r] = static_cast<float>(T[r + 12]);
    tmax = fmax(tmax, fabs(T[r + 12]));
  }
  out->pose32[k][12] = nextafterf(static_cast<float>(tmax), INFINITY);  // max|t| rounded up (fp32 filter bound)
  out->pose32[k][13] = out->pose32[k][14] = out->pose32[k][15] = 0.f;
}

// device-resident solver loop: consume the scores of the batch, advance the state machine, emit the next poses.
// The machine is staged in shared memory: stepping it in place in HBM would be hundreds of dependent L2 round trips.
static __device__ void nm_device_advance(const NidArgs& a) {
  static_assert(sizeof(NmMachine) % 8 == 0, "NmMachine is copied as 8-byte words");
  __shared__ NmMachine s_nm;
  __shared__ double s_init_T[16];
  NmDevice* nm = a.nm;
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&nm->nm);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&s_nm);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(NmMachine) / 8); i += blockDim.x) dst[i] = src[i];
    if (threadIdx.x < 16) s_init_T[threadIdx.x] = nm->init_T[threadIdx.x];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s_nm.step(a.nid_out);
    const int n = s_nm.n;
    int count = nm->trace_count;
    for (int k = 0; k < s_nm.n_obs; k++) {  // reference-order evaluations, replayed by the host for params.callback
      if (count < nm->trace_cap) {
        double* e = nm->trace + static_cast<size_t>(count) * (NM_MAX_N + 1);
        for (int d = 0; d < n; d++) e[d] = s_nm.obs_x[k][d];
        e[NM_MAX_N] = s_nm.obs_y[k];
      }
      count++;
    }
    nm->trace_count = count;
    nm->steps_done++;
  }
  __syncthreads();
  {
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&s_nm);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(&nm->nm);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(NmMachine) / 8); i += blockDim.x) dst[i] = src[i];
  }
  const int n_next = s_nm.n_cand;  // 0 when finished
  if (threadIdx.x < n_next) nm_pose_of_candidate(s_nm.cand[threadIdx.x], s_init_T, nm, threadIdx.x);
  __syncthreads();
  if (threadIdx.x == 0) nm->n_poses = n_next;
}

template <bool DEVLOOP>
static __device__ void nid_finalize(const NidArgs& a, int n_poses, int* smem_i) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  __shared__ int s_cnt[NID_THREADS / 32];  // per-warp partial inlier counts
  // splitting a pose over several warps needs staging room in the block's dynamic shared memory (host checks the size)
  const int wpp = a.finalize_split ? max(1, n_warps / n_poses) : 1;  // warps per pose
  const int ppr = n_warps / wpp;                                     // poses per round
  double* s_term = reinterpret_cast<double*>(smem_i);                // [ppr][nb] staged p*log(p+1e-6) terms (wpp > 1)
  double* s_mterm = s_term + ppr * a.nb;                             // [ppr][2*bins] staged marginal terms (wpp > 1)
  int* s_marg = smem_i + (wpp > 1 ? 2 * ppr * (a.nb + 2 * a.bins) : 0);  // [ppr][2*bins] marginal counts
  for (int p0 = 0; p0 < n_poses; p0 += ppr) {
    const int slot = warp / wpp, sub = warp % wpp;  // pose slot of this warp within the round, rank within the pose
    const int p = p0 + slot;
    const bool active = slot < ppr && p < n_poses;
    int* h_image = s_marg + slot * 2 * a.bins;  // [bins]
    int* h_points = h_image + a.bins;           // [bins]
    for (int i = threadIdx.x; i < ppr * 2 * a.bins; i += blockDim.x) s_marg[i] = 0;
    __syncthreads();
    stamp(a, 7);
    int* g = a.ghist + static_cast<size_t>(active ? p : 0) * a.nb;
    const int span = wpp * 32;  // joint bins covered per step by the warps of one pose
    int part = 0;
    int c[FIN_CH];
    const bool single = a.nb <= span * FIN_CH;  // pass-1 counts stay in registers for pass 2
    if (active) {
      for (int k0 = 0; k0 < a.nb; k0 += span * FIN_CH) {  // pass 1: marginals + inlier count
#pragma unroll
        for (int m = 0; m < FIN_CH; m++) {
          const int k = k0 + m * span + sub * 32 + lane;
          c[m] = k < a.nb ? __ldcg(g + k) : 0;
        }
#pragma unroll
        for (int m = 0; m < FIN_CH; m++) {
          const int k = k0 + m * span + sub * 32 + lane;
          if (c[m]) {
            atomicAdd(&h_image[k % a.bins], c[m]);
            atomicAdd(&h_points[k / a.bins], c[m]);
            part += c[m];
          }
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) s_cnt[warp] = part;
    __syncthreads();
    stamp(a, 8);
    double t_rs = 0.0;  // canonical per-lane partial of the joint entropy (only meaningful when wpp == 1)
    double sum = 0.0;
    if (active) {
      int total = 0;
      for (int w = 0; w < wpp; w++) total += s_cnt[slot * wpp + w];
      sum = static_cast<double>(total);  // :54 sum = hist_image.sum()
      // :59-61  H = -sum p*log(p + 1e-6)
      for (int k0 = 0; k0 < a.nb; k0 += span * FIN_CH) {  // pass 2: joint entropy terms, export, self-clean
        if (!single) {
#pragma unroll
          for (int m = 0; m < FIN_CH; m++) {
            const int k = k0 + m * span + sub * 32 + lane;
            c[m] = k < a.nb ? __ldcg(g + k) : 0;
          }
        }
#pragma unroll
        for (int m = 0; m < FIN_CH; m++) {
          const int k = k0 + m * span + sub * 32 + lane;
          if (k < a.nb) {
            const double pr = static_cast<double>(c[m]) / sum;
            const double term = entropy_term(pr);
            if (wpp > 1) {
              s_term[slot * a.nb + k] = term;
            } else {
              t_rs = __dadd_rn(t_rs, term);  // k ascends with (k0, m): already the canonical order
            }
            if (a.hist_out) a.hist_out[static_cast<size_t>(p) * a.nb + k] = c[m];
            g[k] = 0;
          }
        }
      }
    }
    if (wpp > 1 && active) {  // marginal terms too are spread over the pose's warps (same arithmetic per term)
      for (int f = sub * 32 + lane; f < 2 * a.bins; f += span) {
        const double pm = static_cast<double>(f < a.bins ? h_image[f] : h_points[f - a.bins]) / sum;
        s_mterm[slot * 2 * a.bins + f] = entropy_term(pm);
      }
    }
    if (wpp > 1) __syncthreads();
    stamp(a, 9);
    if (active && sub == 0) {  // one warp per pose: canonical reductions
      double t_r = 0.0, t_s = 0.0;
      if (wpp > 1) {
        for (int k = lane; k < a.nb; k += 32) t_rs += s_term[slot * a.nb + k];
        for (int k = lane; k < a.bins; k += 32) {
          t_r += s_mterm[slot * 2 * a.bins + k];
          t_s += s_mterm[slot * 2 * a.bins + a.bins + k];
        }
      } else {
        for (int k = lane; k < a.bins; k += 32) {
          const double pi = static_cast<double>(h_image[k]) / sum;
          const double pp = static_cast<double>(h_points[k]) / sum;
          t_r = __dadd_rn(t_r, entropy_term(pi));
          t_s = __dadd_rn(t_s, entropy_term(pp));
        }
      }
      const double Hrs = -warp_tree_sum(t_rs), Hr = -warp_tree_sum(t_r), Hs = -warp_tree_sum(t_s);
      if (lane == 0) {
        const double MI = Hr + Hs - Hrs;      // :63
        const double nid = (Hrs - MI) / Hrs;  // :64 (NaN when there are no inliers, as in the reference)
        a.nid_out[p] = nid;
        if (a.nid_host) a.nid_host[p] = nid;
      }
    }
    __syncthreads();
  }
  if (a.p2p_world > 1) nid_peer_allreduce(a, n_poses);
  if constexpr (DEVLOOP) nm_device_advance(a);
  stamp(a, 4);
  if (threadIdx.x == 0) {
    *a.counter = 0u;
    if (a.done_flag) {  // publish to the polling host thread: results first, then the sequence number
      __threadfence_system();
      *reinterpret_cast<volatile unsigned long long*>(a.done_flag) = a.done_seq;
    }
  }
  stamp(a, 5);
}

// block epilogue shared by the histogram kernels: merge copies -> global accumulators -> last block finalizes
template <bool DEVLOOP>
__device__ __forceinline__ void nid_block_epilogue(const NidArgs& a, int n_poses, int* smem_hist, bool* s_is_last) {
  const int per_copy = n_poses * a.nb;
  const unsigned long long t_main = a.timeline ? global_ns() : 0ull;
  __syncthreads();
  for (int k = threadIdx.x; k < per_copy; k += blockDim.x) {
    int s = 0;
    for (int c = 0; c < a.copies; c++) s += smem_hist[c * per_copy + k];
    if (s) atomicAdd(a.ghist + k, s);
  }
  __threadfence();
  __syncthreads();
  const unsigned long long t_merged = a.timeline ? global_ns() : 0ull;
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(a.counter, 1u);
    *s_is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!*s_is_last) return;
  if (a.timeline && threadIdx.x == 0) {
    a.timeline[1] = t_main;
    a.timeline[2] = t_merged;
    a.timeline[3] = global_ns();
  }
  __threadfence();
  nid_finalize<DEVLOOP>(a, n_poses, smem_hist);
}

// DEVLOOP: device-resident solver loop variant (poses from NmDevice, Nelder-Mead step in the finalizing block); kept out of
// the default instantiation so that its register footprint does not cost the hot loop an occupancy step.
template <int MODEL, bool F32, bool DEVLOOP>
__global__ void __launch_bounds__(NID_THREADS) nid_hist_exact_kernel(const __grid_constant__ NidArgs a) {
  extern __shared__ int smem_hist[];
  __shared__ bool s_is_last;
  const int n_poses = n_poses_of<DEVLOOP>(a);
  if (n_poses == 0) return;  // device-resident loop: the solver has finished
  const int per_copy = n_poses * a.nb;
  if (a.timeline && threadIdx.x == 0 && blockIdx.x == 0) a.timeline[0] = global_ns();
  for (int i = threadIdx.x; i < a.copies * per_copy; i += blockDim.x) smem_hist[i] = 0;
  __syncthreads();
  int* my_hist = smem_hist + ((threadIdx.x >> 5) % a.copies) * per_copy;

  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    double x, y, z, w;
    if constexpr (F32) {
      const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
      x = q.x, y = q.y, z = q.z, w = q.w;
    } else {
      const double4 q = static_cast<const double4*>(a.points)[i];
      x = q.x, y = q.y, z = q.z, w = q.w;
    }
    const int lb = lidar_bin_of(w, a.bins);
    for (int p = 0; p < n_poses; p++) {
      const int ib = classify_exact<MODEL>(a, pose_of<DEVLOOP>(a, p), x, y, z);
      if (ib >= 0) {
        atomicAdd(&my_hist[p * a.nb + ib + lb * a.bins], 1);  // :49 hist(image_bin, lidar_bin)++
      }
    }
  }
  nid_block_epilogue<DEVLOOP>(a, n_poses, smem_hist, &s_is_last);
}

constexpr int NID_QUEUE = 64;  // per-warp queue of (point, pose) pairs waiting for the exact path

// per-warp state of the filter kernel's hot loop
struct FilterWarp {
  int* my_hist;            // this warp's histogram copy [P][nb]
  unsigned int* q_idx;     // [NID_QUEUE] deferred point indices
  unsigned char* q_pose;   // [NID_QUEUE] deferred pose slots
  int qn;                  // queue fill, warp-uniform
  int lane;
  unsigned int lt_mask;
};

template <int MODEL, bool DEVLOOP>
__device__ __forceinline__ void filter_drain32(const NidArgs& a, FilterWarp& w, const float4* __restrict__ pts, int first, int count) {
  if (w.lane < count) {  // entries [first, first+count), count <= 32: one deferred (point, pose) per lane, exact path
    const unsigned int i = w.q_idx[first + w.lane];
    const int p = w.q_pose[first + w.lane];
    const float4 q = __ldg(pts + i);
    const int ib = classify_exact<MODEL>(a, pose_of<DEVLOOP>(a, p), q.x, q.y, q.z);
    if (ib >= 0) atomicAdd(&w.my_hist[p * a.nb + ib + lidar_bin_of(q.w, a.bins) * a.bins], 1);
  }
}

// one tile = 32*K consecutive points starting at `tile` (K per lane, warp-coalesced rows), swept over all P poses.
// Software pipeline over the poses: the image-bin gathers of pose p are issued unconditionally (clamped address), stay
// in flight while pose p+1 is classified, and are consumed by the histogram atomics one iteration later.
// the K rows of a tile, one float4 per lane and row (rows beyond `end` come back as a point behind the camera)
template <int K>
__device__ __forceinline__ void filter_load_tile(const float4* __restrict__ pts, unsigned int tile, unsigned int end, int lane, float4 (&q)[K]) {
#pragma unroll
  for (int j = 0; j < K; j++) {
    const unsigned int i = tile + j * 32 + lane;
    q[j] = make_float4(0.f, 0.f, -1.f, 0.f);
    if (i < end) q[j] = __ldg(pts + i);
  }
}

template <int MODEL, int K, bool DEVLOOP>
__device__ __forceinline__ void filter_tile(const NidArgs& a, int n_poses, FilterWarp& w, const float4* __restrict__ pts, unsigned int tile, unsigned int end, const float4 (&q)[K]) {
  float px[K], py[K], pz[K], pa[K];
  int lboff[K];
  unsigned int idx[K];
  unsigned int valid_bits = 0;
#pragma unroll
  for (int j = 0; j < K; j++) {
    idx[j] = tile + j * 32 + w.lane;
    valid_bits |= (idx[j] < end ? 1u : 0u) << j;
    px[j] = q[j].x, py[j] = q[j].y, pz[j] = q[j].z;
    pa[j] = fabsf(q[j].x) + fabsf(q[j].y) + fabsf(q[j].z);
    lboff[j] = lidar_bin_of(q[j].w, a.bins) * a.bins;
  }
  int pend_bin[K];
  unsigned int pend_ok = 0;
  int* pend_hist = w.my_hist;
  for (int p = 0; p <= n_poses; p++) {
    int verdict[K];
    unsigned int unc_bits = 0, ok_bits = 0;
    if (p < n_poses) {
      const float* __restrict__ P = pose32_of<DEVLOOP>(a, p);
#pragma unroll
      for (int j = 0; j < K; j++) {
        int vd = classify_fast<MODEL>(a, P, px[j], py[j], pz[j], pa[j]);
        vd = ((valid_bits >> j) & 1u) ? vd : VERDICT_REJECT;
        verdict[j] = vd;
        ok_bits |= (vd >= 0 ? 1u : 0u) << j;
        unc_bits |= (vd == VERDICT_UNCERTAIN ? 1u : 0u) << j;
      }
    }
#pragma unroll
    for (int j = 0; j < K; j++) {  // consume the previous pose's gathers
      if ((pend_ok >> j) & 1u) atomicAdd(&pend_hist[pend_bin[j] + lboff[j]], 1);  // :49 hist(image_bin, lidar_bin)++
    }
    pend_ok = ok_bits;
    if (p < n_poses) {
      pend_hist = w.my_hist + p * a.nb;
#pragma unroll
      for (int j = 0; j < K; j++) pend_bin[j] = __ldg(a.bin_image + max(verdict[j], 0));
      if (__any_sync(0xffffffffu, unc_bits != 0)) {  // some lane deferred a point: queue it for the exact path
#pragma unroll
        for (int j = 0; j < K; j++) {
          const bool mine = (unc_bits >> j) & 1u;
          const unsigned int m = __ballot_sync(0xffffffffu, mine);
          if (m) {
            if (mine) {
              const int pos = w.qn + __popc(m & w.lt_mask);
              w.q_idx[pos] = idx[j];
              w.q_pose[pos] = static_cast<unsigned char>(p);
            }
            w.qn += __popc(m);
            __syncwarp();
            if (w.qn >= 32) {
              filter_drain32<MODEL, DEVLOOP>(a, w, pts, w.qn - 32, 32);
              w.qn -= 32;
              __syncwarp();
            }
          }
        }
      }
    }
  }
}

// K1 (default): fp32 filter + exact fp64 recheck.
// Every (point, pose) is first classified in fp32 together with a rigorous error bound; verdicts that are farther
// than the bound from every decision edge (FoV cone, integer pixel boundaries, image border) are final.  The rest
// (~2 %) are pushed on a per-warp shared-memory queue and re-decided 32 at a time by the exact double path, so the
// fp64 pipe runs with full warps instead of diverging inside the hot loop.  The histogram is therefore bit-identical
// to the all-fp64 kernel (tests/test_gpu_parity.py::test_filter_kernel_*).
// Work split: the cloud is cut into one contiguous, equally long range per warp (multiple of 32 points), processed as
// NID_KPT-row tiles (NID_KPT points per lane in registers: pose constants fetched once per tile, NID_KPT independent
// chains in flight) plus single-row tiles for the remainder, so no warp does a whole extra tile more than another.
template <int MODEL, bool F32, int NID_KPT, bool DEVLOOP>
__global__ void __launch_bounds__(NID_THREADS) nid_hist_filter_kernel(const __grid_constant__ NidArgs a) {
  extern __shared__ int smem_hist[];
  __shared__ bool s_is_last;
  __shared__ unsigned int q_idx[NID_THREADS / 32][NID_QUEUE];
  __shared__ unsigned char q_pose[NID_THREADS / 32][NID_QUEUE];
  static_assert(F32, "the fp32 filter runs on the float4 cloud layout");
  const int n_poses = n_poses_of<DEVLOOP>(a);
  if (n_poses == 0) return;  // device-resident loop: the solver has finished
  const int per_copy = n_poses * a.nb;
  if (a.timeline && threadIdx.x == 0 && blockIdx.x == 0) a.timeline[0] = global_ns();
  const int warp = threadIdx.x >> 5;
  FilterWarp w;
  w.lane = threadIdx.x & 31;
  w.lt_mask = (1u << w.lane) - 1u;
  w.my_hist = smem_hist + (warp % a.copies) * per_copy;
  w.q_idx = q_idx[warp];
  w.q_pose = q_pose[warp];
  w.qn = 0;
  const float4* __restrict__ pts = static_cast<const float4*>(a.points);
  const unsigned int n = static_cast<unsigned int>(a.n);  // host guarantees n < 2^31 for this kernel

  const unsigned int warps_total = gridDim.x * (NID_THREADS / 32);
  const unsigned int warp_global = blockIdx.x * (NID_THREADS / 32) + warp;
  const unsigned int chunk = ((n + warps_total - 1) / warps_total + 31u) & ~31u;  // points per warp, multiple of 32
  const unsigned long long lo = static_cast<unsigned long long>(warp_global) * chunk;
  const bool has_work = lo < n;
  const unsigned int end = has_work ? static_cast<unsigned int>(min(static_cast<unsigned long long>(n), lo + chunk)) : 0u;
  unsigned int t = static_cast<unsigned int>(has_work ? lo : 0ull);
  // the first tile's points are requested before the histogram copies are zeroed, so that their L2 latency overlaps it
  float4 q4[NID_KPT];
  const bool first_is_k4 = has_work && t + 32u * NID_KPT <= end;
  if (first_is_k4) filter_load_tile<NID_KPT>(pts, t, end, w.lane, q4);
  for (int i = threadIdx.x; i < a.copies * per_copy; i += blockDim.x) smem_hist[i] = 0;
  __syncthreads();
  if (has_work) {
    // NID_KPT-row tiles, the next tile's rows in flight while the current one is swept over the poses
    while (t + 32u * NID_KPT <= end) {
      float4 nxt[NID_KPT];
      const bool more = t + 64u * NID_KPT <= end;
      if (more) filter_load_tile<NID_KPT>(pts, t + 32u * NID_KPT, end, w.lane, nxt);
      filter_tile<MODEL, NID_KPT, DEVLOOP>(a, n_poses, w, pts, t, end, q4);
      t += 32u * NID_KPT;
      if (more) {
#pragma unroll
        for (int j = 0; j < NID_KPT; j++) q4[j] = nxt[j];
      }
    }
    // one-row tiles for what is left of the range, pipelined the same way
    float4 q1[1], n1[1];
    if (t < end) filter_load_tile<1>(pts, t, end, w.lane, q1);
    while (t < end) {
      const bool more = t + 32u < end;
      if (more) filter_load_tile<1>(pts, t + 32u, end, w.lane, n1);
      filter_tile<MODEL, 1, DEVLOOP>(a, n_poses, w, pts, t, end, q1);
      t += 32u;
      if (more) q1[0] = n1[0];
    }
  }
  if (w.qn > 0) filter_drain32<MODEL, DEVLOOP>(a, w, pts, 0, w.qn);
  nid_block_epilogue<DEVLOOP>(a, n_poses, smem_hist, &s_is_last);
}

// debug / test kernel: runs BOTH paths on every (point, pose) and counts, in a.dbg:
//   [0] point-poses, [1] uncertain verdicts, [2] certain verdicts that disagree with the exact path (must be 0),
//   [3] max over certain in-image verdicts of |uv_fp32 - uv_exact| / E, as float bits scaled (atomicMax)
template <int MODEL, bool F32>
__global__ void __launch_bounds__(NID_THREADS) nid_filter_verify_kernel(const __grid_constant__ NidArgs a) {
  static_assert(F32, "the fp32 filter runs on the float4 cloud layout");
  const float4* __restrict__ pts = static_cast<const float4*>(a.points);
  unsigned long long total = 0, uncertain = 0, mismatch = 0;
  float max_ratio = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    const float4 q = __ldg(pts + i);
    const float a_p = fabsf(q.x) + fabsf(q.y) + fabsf(q.z);
    for (int p = 0; p < a.n_poses; p++) {
      total++;
      const int vf = classify_fast<MODEL>(a, a.pose32[p], q.x, q.y, q.z, a_p);
      double ue = 0.0, ve = 0.0;
      const int pe = exact_pixel<MODEL>(a, a.pose[p], q.x, q.y, q.z, &ue, &ve);
      if (vf == VERDICT_UNCERTAIN) {
        uncertain++;
      } else if (vf != pe) {  // both -1, or the same pixel
        mismatch++;
      } else if (vf >= 0) {
        // recompute the fp32 projection to measure how much of the bound is used
        const float* P = a.pose32[p];
        const float pcx = fmaf(P[0], q.x, fmaf(P[1], q.y, fmaf(P[2], q.z, P[9])));
        const float pcy = fmaf(P[3], q.x, fmaf(P[4], q.y, fmaf(P[5], q.z, P[10])));
        const float pcz = fmaf(P[6], q.x, fmaf(P[7], q.y, fmaf(P[8], q.z, P[11])));
        const float n2 = fmaf(pcx, pcx, fmaf(pcy, pcy, pcz * pcz));
        const float nrm = n2 * rsqrtf(n2);
        const float delta = (5.25f * F32_U) * (a_p + P[12]);
        float u, v, Eu, Ev;
        if (project_fast<MODEL>(a.fast, pcx, pcy, pcz, nrm, delta, u, v, Eu, Ev)) {
          const float ru = static_cast<float>(fabs(static_cast<double>(u) - ue)) / Eu;
          const float rv = static_cast<float>(fabs(static_cast<double>(v) - ve)) / Ev;
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

// image -> image-bin LUT pass (:43,:46), once per context
static __global__ void apply_lut_kernel(const uint8_t* __restrict__ src, int src_stride, uint8_t* __restrict__ dst, int width, int height, const uint8_t* __restrict__ lut) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x < width && y < height) {
    dst[static_cast<size_t>(y) * width + x] = lut[src[static_cast<size_t>(y) * src_stride + x]];
  }
}

}  // namespace vlcal
