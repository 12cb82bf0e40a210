// tools/microbench.cu -- micro-measurements that drive the design of the NID kernel (DESIGN.md cites the
// numbers): shared-memory histogram atomics, fp64 vs fp32 issue rates (mul/add, div, sqrt), random 1-byte gathers
// from an L2-resident image.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench tools/microbench.cu
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %d: %s\n", #x, __LINE__, cudaGetErrorString(e));   \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

__device__ __forceinline__ unsigned int hash32(unsigned int x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// MODE 0: warp-private copies atomicAdd; 1: one shared copy per block; 2: __match_any aggregated; 3: no histogram (baseline)
template <int MODE>
__global__ void __launch_bounds__(256) hist_kernel(int iters, int nbins, int* out) {
  extern __shared__ int sm[];
  const int copies = MODE == 0 ? 8 : 1;
  for (int i = threadIdx.x; i < copies * nbins; i += blockDim.x) sm[i] = 0;
  __syncthreads();
  int* h = sm + (MODE == 0 ? (threadIdx.x >> 5) * nbins : 0);
  unsigned int s = blockIdx.x * blockDim.x + threadIdx.x;
  int acc = 0;
  for (int it = 0; it < iters; it++) {
    s = hash32(s + it);
    const int b = s % nbins;
    if (MODE == 0 || MODE == 1) {
      atomicAdd(&h[b], 1);
    } else if (MODE == 2) {
      const unsigned int m = __match_any_sync(0xffffffffu, b);
      if ((__ffs(m) - 1) == (threadIdx.x & 31)) atomicAdd(&h[b], __popc(m));
    } else {
      acc += b;
    }
  }
  __syncthreads();
  int t = acc;
  for (int i = threadIdx.x; i < copies * nbins; i += blockDim.x) t += sm[i];
  if (t == 0x7fffffff) out[0] = t;
}

template <typename T, int OP>
__global__ void __launch_bounds__(256) flop_kernel(int iters, T seed, T* out) {
  T a0 = seed + threadIdx.x, a1 = a0 + T(1), a2 = a0 + T(2), a3 = a0 + T(3);
  const T c = T(1.0000001), d = T(0.9999999);
  for (int it = 0; it < iters; it++) {
    if (OP == 0) {  // independent mul+add chains (no fma)
      if constexpr (sizeof(T) == 8) {
        a0 = __dadd_rn(__dmul_rn(a0, c), d); a1 = __dadd_rn(__dmul_rn(a1, c), d); a2 = __dadd_rn(__dmul_rn(a2, c), d); a3 = __dadd_rn(__dmul_rn(a3, c), d);
      } else {
        a0 = __fadd_rn(__fmul_rn(a0, c), d); a1 = __fadd_rn(__fmul_rn(a1, c), d); a2 = __fadd_rn(__fmul_rn(a2, c), d); a3 = __fadd_rn(__fmul_rn(a3, c), d);
      }
    } else if (OP == 1) {  // fma
      a0 = fma(a0, c, d); a1 = fma(a1, c, d); a2 = fma(a2, c, d); a3 = fma(a3, c, d);
    } else if (OP == 2) {  // IEEE division
      a0 = c / a0 + d; a1 = c / a1 + d; a2 = c / a2 + d; a3 = c / a3 + d;
    } else {  // IEEE sqrt
      a0 = sqrt(a0) + c; a1 = sqrt(a1) + c; a2 = sqrt(a2) + c; a3 = sqrt(a3) + c;
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3;
}

// random / coherent 1-byte gathers from an image
__global__ void __launch_bounds__(256) gather_kernel(const unsigned char* img, int w, int h, int iters, int coherent, int* out) {
  unsigned int s = blockIdx.x * blockDim.x + threadIdx.x;
  int acc = 0;
  const int lane = threadIdx.x & 31;
  for (int it = 0; it < iters; it++) {
    unsigned int r = hash32((coherent ? (s >> 5) : s) * 747796405u + it);
    int x = r % w, y = (r >> 12) % h;
    if (coherent) {  // lanes of a warp fall in an 8x4 pixel patch
      x = min(w - 1, x + (lane & 7));
      y = min(h - 1, y + (lane >> 3));
    }
    acc += __ldg(img + (size_t)y * w + x);
  }
  if (acc == 0x7fffffff) out[0] = acc;
}

template <typename F>
float time_ms(F f, int reps = 5) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  f(); CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int i = 0; i < reps; i++) {
    CK(cudaEventRecord(a)); f(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  const int sms = p.multiProcessorCount;
  printf("device %s, %d SMs, clock %d kHz\n", p.name, sms, p.clockRate);
  int* dout; CK(cudaMalloc(&dout, 1 << 20));
  // ---- histogram atomics
  const int iters = 4096, grid = sms * 4;
  const double n_ops = (double)grid * 256 * iters;
  for (int nbins : {256, 1024}) {
    float t0 = time_ms([&] { hist_kernel<0><<<grid, 256, 8 * nbins * 4>>>(iters, nbins, dout); });
    float t1 = time_ms([&] { hist_kernel<1><<<grid, 256, nbins * 4>>>(iters, nbins, dout); });
    float t2 = time_ms([&] { hist_kernel<2><<<grid, 256, nbins * 4>>>(iters, nbins, dout); });
    float t3 = time_ms([&] { hist_kernel<3><<<grid, 256, nbins * 4>>>(iters, nbins, dout); });
    printf("smem hist %4d bins: warp-private %.3f ms (%.1f Gatom/s, %.2f atom/clk/SM) | block-shared %.3f ms (%.1f G/s) | match_any %.3f ms (%.1f G/s) | no-hist baseline %.3f ms\n",
           nbins, t0, n_ops / t0 * 1e-6, n_ops / (t0 * 1e-3) / sms / (p.clockRate * 1e3), t1, n_ops / t1 * 1e-6, t2, n_ops / t2 * 1e-6, t3);
  }
  // ---- flop rates
  {
    const int it2 = 8192, g2 = sms * 8;
    const double ops = (double)g2 * 256 * it2 * 4;
    double* dd; float* df; CK(cudaMalloc(&dd, g2 * 256 * 8)); CK(cudaMalloc(&df, g2 * 256 * 4));
    const char* names[4] = {"mul+add (2 instr)", "fma", "div+add", "sqrt+add"};
    float t;
    t = time_ms([&] { flop_kernel<double, 0><<<g2, 256>>>(it2, 1.0, dd); }); printf("fp64 %-18s %.3f ms  %.2f Tchain/s\n", names[0], t, ops / t * 1e-9);
    t = time_ms([&] { flop_kernel<float, 0><<<g2, 256>>>(it2, 1.0f, df); }); printf("fp32 %-18s %.3f ms  %.2f Tchain/s\n", names[0], t, ops / t * 1e-9);
    t = time_ms([&] { flop_kernel<double, 1><<<g2, 256>>>(it2, 1.0, dd); }); printf("fp64 %-18s %.3f ms  %.2f Tchain/s\n", names[1], t, ops / t * 1e-9);
    t = time_ms([&] { flop_kernel<float, 1><<<g2, 256>>>(it2, 1.0f, df); }); printf("fp32 %-18s %.3f ms  %.2f Tchain/s\n", names[1], t, ops / t * 1e-9);
    t = time_ms([&] { flop_kernel<double, 2><<<g2, 256>>>(it2 / 8, 1.0, dd); }); printf("fp64 %-18s %.3f ms  %.3f Tchain/s\n", names[2], t, ops / 8 / t * 1e-9);
    t = time_ms([&] { flop_kernel<float, 2><<<g2, 256>>>(it2 / 8, 1.0f, df); }); printf("fp32 %-18s %.3f ms  %.3f Tchain/s\n", names[2], t, ops / 8 / t * 1e-9);
    t = time_ms([&] { flop_kernel<double, 3><<<g2, 256>>>(it2 / 8, 1.0, dd); }); printf("fp64 %-18s %.3f ms  %.3f Tchain/s\n", names[3], t, ops / 8 / t * 1e-9);
    t = time_ms([&] { flop_kernel<float, 3><<<g2, 256>>>(it2 / 8, 1.0f, df); }); printf("fp32 %-18s %.3f ms  %.3f Tchain/s\n", names[3], t, ops / 8 / t * 1e-9);
  }
  // ---- gathers
  {
    const int w = 1920, h = 1080, it3 = 1024, g3 = sms * 8;
    unsigned char* img; CK(cudaMalloc(&img, (size_t)w * h)); CK(cudaMemset(img, 1, (size_t)w * h));
    const double n = (double)g3 * 256 * it3;
    float tr = time_ms([&] { gather_kernel<<<g3, 256>>>(img, w, h, it3, 0, dout); });
    float tc = time_ms([&] { gather_kernel<<<g3, 256>>>(img, w, h, it3, 1, dout); });
    printf("u8 gather 1920x1080 (L2 resident): random %.3f ms (%.1f Ggather/s) | warp-coherent 8x4 patch %.3f ms (%.1f Ggather/s)\n", tr, n / tr * 1e-6, tc, n / tc * 1e-6);
  }
  return 0;
}
