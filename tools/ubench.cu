// Micro-benchmarks that size the kernel design: FP64 FMA vs DMMA (mma.sync m8n8k4 f64) issue
// rate, mixed, shared-memory bandwidth, and fp64 atomic (RED) throughput. Build: nvcc -arch=sm_90a.
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__device__ __forceinline__ void dmma(double &c0, double &c1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <int NACC>
__global__ void k_dfma(double *out, int iters, double a, double b)
{
  double acc[NACC];
  for (int i = 0; i < NACC; i++) acc[i] = threadIdx.x + i;
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int i = 0; i < NACC; i++) acc[i] = fma(acc[i], a, b);
  double s = 0;
  for (int i = 0; i < NACC; i++) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NACC>
__global__ void k_dmma(double *out, int iters, double a, double b)
{
  double c0[NACC], c1[NACC];
  for (int i = 0; i < NACC; i++) { c0[i] = threadIdx.x + i; c1[i] = i; }
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int i = 0; i < NACC; i++) dmma(c0[i], c1[i], a, b);
  double s = 0;
  for (int i = 0; i < NACC; i++) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NACC>
__global__ void k_mixed(double *out, int iters, double a, double b)
{
  double c0[NACC], c1[NACC], acc[NACC * 4];
  for (int i = 0; i < NACC; i++) { c0[i] = threadIdx.x + i; c1[i] = i; }
  for (int i = 0; i < NACC * 4; i++) acc[i] = threadIdx.x - i;
  for (int it = 0; it < iters; it++)
  {
#pragma unroll
    for (int i = 0; i < NACC; i++)
    {
      dmma(c0[i], c1[i], a, b);
#pragma unroll
      for (int j = 0; j < 4; j++) acc[4 * i + j] = fma(acc[4 * i + j], a, b);
    }
  }
  double s = 0;
  for (int i = 0; i < NACC; i++) s += c0[i] + c1[i];
  for (int i = 0; i < NACC * 4; i++) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_smem(double *out, int iters)
{
  extern __shared__ double sm[];
  for (int i = threadIdx.x; i < 4096; i += blockDim.x) sm[i] = i;
  __syncthreads();
  double s = 0;
  int idx = threadIdx.x;
  for (int it = 0; it < iters; it++)
  {
#pragma unroll
    for (int j = 0; j < 8; j++) s += sm[(idx + j * 256) & 4095];
    idx = (idx + 1) & 4095;
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_atomic(double *y, const int *idx, int n, int reps)
{
  for (int r = 0; r < reps; r++)
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n; i += (size_t)gridDim.x * blockDim.x)
      atomicAdd(y + idx[i], 1.0);
}

int main()
{
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("device %s sms=%d clock=%d kHz\n", prop.name, sms, prop.clockRate);
  double *out;
  CK(cudaMalloc(&out, sizeof(double) * sms * 8 * 1024));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms;
  const int iters = 4096;
  for (int blocks_per_sm : {1, 2, 4})
    for (int nt : {128, 256, 512})
    {
      const int grid = sms * blocks_per_sm;
      k_dfma<8><<<grid, nt>>>(out, 64, 1.0000001, 1e-9);
      cudaEventRecord(e0);
      k_dfma<8><<<grid, nt>>>(out, iters, 1.0000001, 1e-9);
      cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
      double fl = 2.0 * grid * nt * 8.0 * iters;
      printf("DFMA  bps=%d nt=%d : %.2f TFLOP/s\n", blocks_per_sm, nt, fl / ms * 1e-9);
      k_dmma<8><<<grid, nt>>>(out, 64, 1.0000001, 1e-9);
      cudaEventRecord(e0);
      k_dmma<8><<<grid, nt>>>(out, iters, 1.0000001, 1e-9);
      cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
      fl = 2.0 * 256.0 * grid * (nt / 32) * 8.0 * iters;
      printf("DMMA  bps=%d nt=%d : %.2f TFLOP/s\n", blocks_per_sm, nt, fl / ms * 1e-9);
      k_mixed<4><<<grid, nt>>>(out, 64, 1.0000001, 1e-9);
      cudaEventRecord(e0);
      k_mixed<4><<<grid, nt>>>(out, iters, 1.0000001, 1e-9);
      cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
      double fl_mma = 2.0 * 256.0 * grid * (nt / 32) * 4.0 * iters, fl_fma = 2.0 * grid * nt * 16.0 * iters;
      printf("MIXED bps=%d nt=%d : dmma %.2f + dfma %.2f = %.2f TFLOP/s\n", blocks_per_sm, nt, fl_mma / ms * 1e-9,
             fl_fma / ms * 1e-9, (fl_mma + fl_fma) / ms * 1e-9);
    }
  // shared memory bandwidth
  {
    const int grid = sms * 4, nt = 256;
    cudaEventRecord(e0);
    k_smem<<<grid, nt, 4096 * 8>>>(out, 4096);
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
    double bytes = 8.0 * grid * nt * 8.0 * 4096;
    printf("SMEM LDS.64: %.1f TB/s = %.1f B/clk/SM @1.9GHz\n", bytes / ms * 1e-9, bytes / ms * 1e-6 / sms / 1.9e3 * 1e-3 * 1e3);
  }
  // atomics
  {
    const int n = 24389 * 144;  // one apply's worth of scatter
    const int L = 2021184;
    std::vector<int> h(n);
    // pattern 1: structured (element-local contiguity like edge/face/interior runs), pattern 2: random
    for (int pat = 0; pat < 3; pat++)
    {
      unsigned long long s = 88172645463325252ull;
      for (int i = 0; i < n; i++)
      {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        if (pat == 0) h[i] = (int)(((long long)i * L) / n);           // sequential, duplicates adjacent
        else if (pat == 1) h[i] = (int)(s % L);                        // fully random
        else h[i] = (int)((((long long)(i / 12) * 12 * L) / n + (i % 12) + (s % 7) * 1000) % L);  // runs of 12
      }
      int *d_idx; double *y;
      CK(cudaMalloc(&d_idx, sizeof(int) * n)); CK(cudaMalloc(&y, sizeof(double) * L));
      CK(cudaMemcpy(d_idx, h.data(), sizeof(int) * n, cudaMemcpyHostToDevice));
      CK(cudaMemset(y, 0, sizeof(double) * L));
      k_atomic<<<sms * 8, 256>>>(y, d_idx, n, 1);
      cudaEventRecord(e0);
      k_atomic<<<sms * 8, 256>>>(y, d_idx, n, 10);
      cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
      printf("RED.F64 pattern %d: %.1f G atomics/s (%.3f ms per %d)\n", pat, 10.0 * n / ms * 1e-6, ms / 10, n);
      cudaFree(d_idx); cudaFree(y);
    }
  }
  return 0;
}
