// Micro-benchmarks that calibrate the latency model of the single-CTA band solver on H100:
// dependent-chain latency and per-warp issue interval of DFMA, rsqrt(double), LDS, SHFL, and the cost
// of bar.sync with 5 / 16 warps.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_latency fp64_latency.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ long long clk() { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory"); return t; }

template <int CHAINS>
__global__ void dfma_kernel(double* out, long long* cyc, double a, double b, int iters) {
  double x[CHAINS];
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) x[c] = threadIdx.x + c;
  __syncthreads();
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) x[c] = fma(x[c], a, b);
  }
  double s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) s += x[c];
  const long long t1 = clk();
  out[threadIdx.x] = s;
  if ((threadIdx.x & 31) == 0) cyc[threadIdx.x >> 5] = t1 - t0;
}

__global__ void rsqrt_kernel(double* out, long long* cyc, double a, int iters) {
  double x = a + threadIdx.x;
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) x = rsqrt(x) + a;
  const long long t1 = clk();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void lds_kernel(double* out, long long* cyc, int iters, int stride) {
  __shared__ int next[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) next[i] = (i + stride) & 1023;
  __syncthreads();
  int p = threadIdx.x;
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) p = next[p];
  const long long t1 = clk();
  out[threadIdx.x] = p;
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void shfl_kernel(double* out, long long* cyc, int iters) {
  double x = threadIdx.x;
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) x = __shfl_xor_sync(0xffffffffu, x, 1) + 1.0;
  const long long t1 = clk();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void bar_kernel(double* out, long long* cyc, int iters) {
  __shared__ double s[512];
  double x = threadIdx.x;
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) {
    s[threadIdx.x] = x;
    __syncthreads();
    x = s[(threadIdx.x + 33) % blockDim.x] + 1.0;
    __syncthreads();
  }
  const long long t1 = clk();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

// straight-line code footprint test: executes a long unrolled sequence once per iteration
template <int N>
__global__ void icache_kernel(double* out, long long* cyc, double a, double b, int iters) {
  double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3;
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < N; ++k) { x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b); }
  }
  const long long t1 = clk();
  out[threadIdx.x] = x0 + x1 + x2 + x3;
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

// FP64 tensor-core op (mma.sync m8n8k4 -> DMMA.8x8x4): dependent-accumulator latency and issue interval with
// CHAINS independent accumulators, per warp and with 16 warps on the SM (512 FLOP per instruction).
template <int CHAINS>
__global__ void dmma_kernel(double* out, long long* cyc, double a, double b, int iters) {
  double c0[CHAINS], c1[CHAINS];
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) { c0[c] = threadIdx.x + c; c1[c] = 0.5 * c; }
  __syncthreads();
  const long long t0 = clk();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < CHAINS; ++c)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0[c]), "+d"(c1[c]) : "d"(a), "d"(b));
  }
  double s = 0;
#pragma unroll
  for (int c = 0; c < CHAINS; ++c) s += c0[c] + c1[c];
  const long long t1 = clk();
  out[threadIdx.x] = s;
  if ((threadIdx.x & 31) == 0) cyc[threadIdx.x >> 5] = t1 - t0;
}

int main() {
  double* out; long long* cyc;
  cudaMalloc(&out, 1024 * sizeof(double)); cudaMalloc(&cyc, 64 * sizeof(long long));
  long long h[64];
  const int it = 4096;
  auto rd = [&]() { cudaDeviceSynchronize(); cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost); };
  dfma_kernel<1><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, it); rd(); printf("DFMA dependent latency            : %.2f cycles\n", (double)h[0] / it);
  dfma_kernel<8><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, it); rd(); printf("DFMA issue interval, 1 warp, 8 ILP : %.2f cycles/instr\n", (double)h[0] / (8.0 * it));
  dfma_kernel<8><<<1, 128>>>(out, cyc, 1.0000001, 1e-9, it); rd(); printf("DFMA 4 warps (one per scheduler)   : %.2f cycles/instr/warp\n", (double)h[0] / (8.0 * it));
  dfma_kernel<8><<<1, 512>>>(out, cyc, 1.0000001, 1e-9, it); rd(); printf("DFMA 16 warps (4 per scheduler)    : %.2f cycles/instr/warp  (=> %.2f cycles per warp-instr per scheduler)\n", (double)h[0] / (8.0 * it), (double)h[0] / (8.0 * it) / 4.0);
  dmma_kernel<1><<<1, 32>>>(out, cyc, 1e-3, 1e-3, it); rd(); printf("DMMA.8x8x4 dependent latency (1 chain)       : %.2f cycles\n", (double)h[0] / it);
  dmma_kernel<4><<<1, 32>>>(out, cyc, 1e-3, 1e-3, it); rd(); printf("DMMA.8x8x4 issue interval, 1 warp, 4 chains  : %.2f cycles/instr\n", (double)h[0] / (4.0 * it));
  dmma_kernel<8><<<1, 32>>>(out, cyc, 1e-3, 1e-3, it); rd(); printf("DMMA.8x8x4 issue interval, 1 warp, 8 chains  : %.2f cycles/instr\n", (double)h[0] / (8.0 * it));
  dmma_kernel<8><<<1, 128>>>(out, cyc, 1e-3, 1e-3, it); rd(); printf("DMMA.8x8x4 4 warps x 8 chains                : %.2f cycles/instr/warp\n", (double)h[0] / (8.0 * it));
  dmma_kernel<8><<<1, 512>>>(out, cyc, 1e-3, 1e-3, it); rd(); printf("DMMA.8x8x4 16 warps x 8 chains               : %.2f cycles/instr/warp => %.2f cycles per DMMA per SM (512 FLOP each)\n", (double)h[0] / (8.0 * it), (double)h[0] / (8.0 * it) / 16.0);
  rsqrt_kernel<<<1, 32>>>(out, cyc, 1.5, it); rd(); printf("rsqrt(double)+add dependent        : %.2f cycles\n", (double)h[0] / it);
  lds_kernel<<<1, 32>>>(out, cyc, it, 1); rd(); printf("LDS dependent (pointer chase)      : %.2f cycles\n", (double)h[0] / it);
  shfl_kernel<<<1, 32>>>(out, cyc, it); rd(); printf("SHFL(double)+DADD dependent        : %.2f cycles\n", (double)h[0] / it);
  bar_kernel<<<1, 160>>>(out, cyc, it); rd(); printf("2x __syncthreads + STS/LDS, 5 warps : %.2f cycles/iter\n", (double)h[0] / it);
  bar_kernel<<<1, 512>>>(out, cyc, it); rd(); printf("2x __syncthreads + STS/LDS, 16 warps: %.2f cycles/iter\n", (double)h[0] / it);
  icache_kernel<64><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 256); rd(); printf("straight-line  256 DFMA  (4 KB)  : %.2f cycles/instr\n", (double)h[0] / (256.0 * 256));
  icache_kernel<512><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 64); rd(); printf("straight-line 2048 DFMA (32 KB)  : %.2f cycles/instr\n", (double)h[0] / (64.0 * 2048));
  icache_kernel<2048><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 16); rd(); printf("straight-line 8192 DFMA (128 KB) : %.2f cycles/instr\n", (double)h[0] / (16.0 * 8192));
  icache_kernel<8192><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 8); rd(); printf("straight-line 32768 DFMA (512 KB): %.2f cycles/instr\n", (double)h[0] / (8.0 * 32768));
  // cold vs warm instruction fetch: one pass over 2048 straight-line DFMAs (32 KB of code)
  for (int rep = 0; rep < 3; ++rep) {
    icache_kernel<8192><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 1); cudaDeviceSynchronize();   // evict
    icache_kernel<512><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 1); rd(); printf("single pass 2048 DFMA after another kernel : %.2f cycles/instr\n", (double)h[0] / 2048.0);
    icache_kernel<512><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 1); rd(); printf("single pass 2048 DFMA, same kernel again   : %.2f cycles/instr\n", (double)h[0] / 2048.0);
    icache_kernel<512><<<1, 32>>>(out, cyc, 1.0000001, 1e-9, 2); rd(); printf("two passes                                 : %.2f cycles/instr\n", (double)h[0] / 4096.0);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
