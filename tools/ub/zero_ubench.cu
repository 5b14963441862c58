// Micro-benchmark (round 2, multi-GPU analysis): how long does a zero-fill of an 8 / 16 MB vector take right after the
// bench's L2 flush (a 256 MB memset that leaves the 50 MB L2 of an H100 full of DIRTY lines) compared with a clean L2?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o zero_ubench zero_ubench.cu && ./zero_ubench
#include <cstdio>
#include <cuda_runtime.h>
constexpr int SMS = 132;  // H100 SXM
__global__ void zero_kernel(double2 *y, long long n2)
{
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += stride) y[i] = make_double2(0.0, 0.0);
}
__global__ void read_kernel(const double2 *x, long long n2, double *out)
{
  const long long stride = (long long)gridDim.x * blockDim.x;
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += stride) s += x[i].x + x[i].y;
  if (s == 123.456) *out = s;
}
int main()
{
  const size_t NF = 256ull << 20;
  double *flush, *y, *out;
  cudaMalloc(&flush, NF);
  cudaMalloc(&y, 32 << 20);
  cudaMalloc(&out, 8);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  for (int mode = 0; mode < 4; mode++)          // 0: dirty L2 (memset flush), 1: flush written then read back (clean L2), 2: no flush, 3: dirty, cudaMemsetAsync
    for (int mb = 8; mb <= 16; mb *= 2)
      for (int grid = SMS * 2; grid <= SMS * 8; grid *= 2)
      {
        float tot = 0.f;
        const int reps = 20;
        for (int r = 0; r < reps + 2; r++)
        {
          if (mode != 2) cudaMemsetAsync(flush, 0, NF);
          if (mode == 1) read_kernel<<<SMS * 8, 256>>>((const double2 *)flush, NF / 16, out);
          cudaEventRecord(a);
          if (mode == 3)
            cudaMemsetAsync(y, 0, (size_t)mb << 20);
          else
            zero_kernel<<<grid, 256>>>((double2 *)y, ((long long)mb << 20) / 16);
          cudaEventRecord(b);
          cudaEventSynchronize(b);
          float ms;
          cudaEventElapsedTime(&ms, a, b);
          if (r >= 2) tot += ms;
        }
        printf("mode %d (%s) %2d MB grid %4d: %.2f us\n", mode, mode == 0 ? "dirty L2" : mode == 1 ? "clean L2" : mode == 2 ? "no flush" : "dirty L2, cudaMemset", mb, grid,
               1e3 * tot / reps);
      }
  return 0;
}
