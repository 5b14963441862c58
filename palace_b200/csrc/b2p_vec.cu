// BLAS-1 style vector kernels and global reductions for the device-resident solver loop.
// Replaces the mfem::forall lambdas of /root/reference/palace/linalg/vector.cpp:276-455,461-591,
// the fused Chebyshev updates of /root/reference/palace/linalg/chebyshev.cpp:70-156 and the
// hypre_SeqVectorInnerProd + MPI_Allreduce reductions (vector.cpp:665-698, vector.hpp:247-253).
// Pure HBM streaming: 128-bit loads/stores, grid = a multiple of the SM count, grid-stride loops.
#include <nccl.h>

#include <algorithm>

#include "b2p_linalg.hpp"
#include "b2p_pipe.cuh"

namespace b2p
{

void DVec::resize(b2p_ctx *c, int64_t n_)
{
  if (p && n == n_ && ctx == c) return;
  release();
  ctx = c;
  n = n_;
  if (n > 0)
  {
    cudaError_t e = cudaMalloc((void **)&p, sizeof(double) * n);
    if (e != cudaSuccess)
    {
      set_error(c, "DVec: cudaMalloc(%lld doubles) failed: %s", (long long)n, cudaGetErrorString(e));
      p = nullptr;
      n = 0;
    }
  }
}
void DVec::release()
{
  if (p) cudaFree(p);
  p = nullptr;
  n = 0;
}

namespace
{

constexpr int NT = 256;
inline int grid_for(b2p_ctx *c, int64_t n)
{
  const int64_t want = (n + 2 * NT - 1) / (2 * NT);
  const int64_t cap = (int64_t)c->sm_count * 8;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

// Elementwise kernels over pairs of doubles (128-bit accesses when the base pointers are 16-byte aligned).
template <typename F>
__global__ void ew_kernel(int64_t n, F f)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) f(i);
}

template <typename F>
void launch_ew(b2p_ctx *c, int64_t n, F f)
{
  if (n <= 0) return;
  B2P_LAUNCH(ew_kernel, grid_for(c, n), NT, 0, c->stream, n, f);
}

// Block reduction of up to MAXM partial sums per thread.
template <int M>
__device__ __forceinline__ void block_reduce_store(double (&acc)[M], double *out, int m_stride)
{
  __shared__ double sh[M][NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < M; j++)
  {
    double v = acc[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sh[j][wid] = v;
  }
  __syncthreads();
  if (wid == 0)
  {
#pragma unroll
    for (int j = 0; j < M; j++)
    {
      double v = lane < NT / 32 ? sh[j][lane] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) out[(size_t)j * m_stride + blockIdx.x] = v;
    }
  }
}

constexpr int RED_BLOCKS = 264;  // 2 x 132 SMs (H100 SXM, the most of any sm_90 part); fixed so the summation order is reproducible
constexpr int MAXM = 8;          // vectors per multi-dot pass

struct VecList
{
  const double *v[MAXM];
};

template <int M>
__global__ void __launch_bounds__(NT) multi_dot_kernel(VecList V, const double *__restrict__ w, int64_t n, int m, double *part)
{
  double acc[M];
#pragma unroll
  for (int j = 0; j < M; j++) acc[j] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    const double wi = w[i];
#pragma unroll
    for (int j = 0; j < M; j++)
      if (j < m) acc[j] += wi * V.v[j][i];
  }
  block_reduce_store<M>(acc, part, RED_BLOCKS);
}

__global__ void __launch_bounds__(NT) sum_kernel(const double *__restrict__ x, int64_t n, double *part)
{
  double acc[1] = {0.0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) acc[0] += x[i];
  block_reduce_store<1>(acc, part, RED_BLOCKS);
}

__global__ void final_reduce_kernel(const double *part, int m, int nblocks, double *out)
{
  // one warp per output, fixed order
  const int j = blockIdx.x;
  double v = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 32) v += part[(size_t)j * RED_BLOCKS + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (threadIdx.x == 0) out[j] = v;
}

__global__ void multi_axpy_kernel(VecList V, const double *__restrict__ coef, int m, double sign, double *__restrict__ w, int64_t n)
{
  __shared__ double sc[MAXM];
  if (threadIdx.x < m) sc[threadIdx.x] = sign * coef[threadIdx.x];
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    double s = w[i];
    for (int j = 0; j < m; j++) s += sc[j] * V.v[j][i];
    w[i] = s;
  }
}

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x)
{
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Partial sums of m dot products live in ctx->d_red: [MAXM][RED_BLOCKS] partials then [MAXM] results.
// Blocks of a reduction pass: two per SM (264 on an H100 SXM), fixed per device so the summation order is reproducible.
int red_grid(b2p_ctx *c) { return std::min(RED_BLOCKS, 2 * std::max(1, c->sm_count)); }
double *red_partials(b2p_ctx *c) { return c->d_red; }
double *red_results(b2p_ctx *c) { return c->d_red + (size_t)MAXM * RED_BLOCKS; }

void reduce_finish(b2p_ctx *c, int m, double *host_out)
{
  B2P_LAUNCH(final_reduce_kernel, m, 32, 0, c->stream, red_partials(c), m, red_grid(c), red_results(c));
  if (c->nranks > 1 && c->comm)
    ncclAllReduce(red_results(c), red_results(c), m, ncclDouble, ncclSum, (ncclComm_t)c->comm, c->stream);
  cudaMemcpyAsync(c->h_red, red_results(c), sizeof(double) * m, cudaMemcpyDeviceToHost, c->stream);
  cudaStreamSynchronize(c->stream);
  for (int j = 0; j < m; j++) host_out[j] = c->h_red[j];
}

}  // namespace

void b2p_allreduce_sum(b2p_ctx *c, double *dbuf, int n)
{
  if (c->nranks > 1 && c->comm) ncclAllReduce(dbuf, dbuf, n, ncclDouble, ncclSum, (ncclComm_t)c->comm, c->stream);
}

namespace vec
{

// Zero-fill as a kernel that releases its dependent launch at once (see griddep_wait in the element kernel).
__global__ void zero_release_kernel(double *y, int64_t n)
{
  griddep_launch_dependents();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = 0.0;
}
void zero_release(b2p_ctx *c, double *y, int64_t n)
{
  if (n > 0) B2P_LAUNCH(zero_release_kernel, grid_for(c, n), NT, 0, c->stream, y, n);
}
void set(b2p_ctx *c, double *y, int64_t n, double v)
{
  if (v == 0.0)
  {
    cudaMemsetAsync(y, 0, sizeof(double) * n, c->stream);
    return;
  }
  launch_ew(c, n, [=] __device__(int64_t i) { y[i] = v; });
}
void copy(b2p_ctx *c, double *y, const double *x, int64_t n)
{
  if (y != x && n > 0) cudaMemcpyAsync(y, x, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream);
}
void scale(b2p_ctx *c, double *y, int64_t n, double a)
{
  launch_ew(c, n, [=] __device__(int64_t i) { y[i] *= a; });
}
void axpy(b2p_ctx *c, double a, const double *x, double *y, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) { y[i] += a * x[i]; });
}
void axpby(b2p_ctx *c, double a, const double *x, double b, double *y, int64_t n)
{
  if (b == 0.0)
    launch_ew(c, n, [=] __device__(int64_t i) { y[i] = a * x[i]; });
  else
    launch_ew(c, n, [=] __device__(int64_t i) { y[i] = a * x[i] + b * y[i]; });
}
void axpbypcz(b2p_ctx *c, double a, const double *x, double b, const double *y, double g, double *z, int64_t n)
{
  if (g == 0.0)
    launch_ew(c, n, [=] __device__(int64_t i) { z[i] = a * x[i] + b * y[i]; });
  else
    launch_ew(c, n, [=] __device__(int64_t i) { z[i] = a * x[i] + b * y[i] + g * z[i]; });
}
void mult_diag(b2p_ctx *c, const double *d, const double *x, double *y, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) { y[i] = d[i] * x[i]; });
}
void reciprocal(b2p_ctx *c, double *y, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) { y[i] = 1.0 / y[i]; });
}
void set_sub(b2p_ctx *c, double *y, const int32_t *idx, int64_t nidx, double v)
{
  launch_ew(c, nidx, [=] __device__(int64_t i) { y[idx[i]] = v; });
}
void set_sub_from(b2p_ctx *c, double *y, const int32_t *idx, int64_t nidx, const double *x)
{
  launch_ew(c, nidx, [=] __device__(int64_t i) { y[idx[i]] = x[idx[i]]; });
}
void axpy_sub(b2p_ctx *c, double a, const double *x, const int32_t *idx, int64_t nidx, double *y)
{
  launch_ew(c, nidx, [=] __device__(int64_t i) { y[idx[i]] += a * x[idx[i]]; });
}
void set_random(b2p_ctx *c, double *y, int64_t n, uint64_t seed)
{
  const uint64_t base = splitmix64(seed * 0x100000001B3ull + (uint64_t)c->rank + 1);
  launch_ew(c, n, [=] __device__(int64_t i)
            {
              const uint64_t r = splitmix64(base + (uint64_t)i);
              y[i] = 2.0 * ((double)(r >> 11) * (1.0 / 9007199254740992.0)) - 1.0;
            });
}
void cheb_first(b2p_ctx *c, double sr, const double *dinv, const double *r, double *d, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) { d[i] = sr * dinv[i] * r[i]; });
}
void cheb_next(b2p_ctx *c, double sd, double sr, const double *dinv, const double *r, double *d, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) { d[i] = sd * d[i] + sr * dinv[i] * r[i]; });
}

// The same with the solution update folded in (one pass instead of cheb_* followed by y += d): y = d or y += d.
void cheb_first_y(b2p_ctx *c, double sr, const double *dinv, const double *r, double *d, double *y, bool assign, int64_t n)
{
  if (assign)
    launch_ew(c, n, [=] __device__(int64_t i) {
      const double di = sr * dinv[i] * r[i];
      d[i] = di;
      y[i] = di;
    });
  else
    launch_ew(c, n, [=] __device__(int64_t i) {
      const double di = sr * dinv[i] * r[i];
      d[i] = di;
      y[i] += di;
    });
}
void cheb_next_y(b2p_ctx *c, double sd, double sr, const double *dinv, const double *r, double *d, double *y, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i) {
    const double di = sd * d[i] + sr * dinv[i] * r[i];
    d[i] = di;
    y[i] += di;
  });
}

void multi_dot(b2p_ctx *c, int m, const double *const *V, const double *w, int64_t n, double *out)
{
  for (int j0 = 0; j0 < m; j0 += MAXM)
  {
    const int mm = std::min(MAXM, m - j0);
    VecList L;
    for (int j = 0; j < MAXM; j++) L.v[j] = j < mm ? V[j0 + j] : nullptr;
    if (mm == 1)
      B2P_LAUNCH(multi_dot_kernel<1>, red_grid(c), NT, 0, c->stream, L, w, n, mm, red_partials(c));
    else if (mm == 2)
      B2P_LAUNCH(multi_dot_kernel<2>, red_grid(c), NT, 0, c->stream, L, w, n, mm, red_partials(c));
    else if (mm <= 4)
      B2P_LAUNCH(multi_dot_kernel<4>, red_grid(c), NT, 0, c->stream, L, w, n, mm, red_partials(c));
    else
      B2P_LAUNCH(multi_dot_kernel<8>, red_grid(c), NT, 0, c->stream, L, w, n, mm, red_partials(c));
    reduce_finish(c, mm, out + j0);
  }
}

// Device-resident scalar variants (sync-free Krylov iterations): the dot product stays in device memory, the vector
// updates read their scalar coefficients from there.
void dot_dev(b2p_ctx *c, const double *x, const double *y, int64_t n, double *d_out)
{
  VecList L;
  for (int j = 0; j < MAXM; j++) L.v[j] = j == 0 ? y : nullptr;
  B2P_LAUNCH(multi_dot_kernel<1>, red_grid(c), NT, 0, c->stream, L, x, n, 1, red_partials(c));
  B2P_LAUNCH(final_reduce_kernel, 1, 32, 0, c->stream, red_partials(c), 1, red_grid(c), d_out);
  if (c->nranks > 1 && c->comm) ncclAllReduce(d_out, d_out, 1, ncclDouble, ncclSum, (ncclComm_t)c->comm, c->stream);
}
// p = z + (num / den) p
void xpay_ratio_dev(b2p_ctx *c, const double *z, const double *d_num, const double *d_den, double *p, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i)
            {
              const double den = *d_den, b = den != 0.0 ? *d_num / den : 0.0;
              p[i] = z[i] + b * p[i];
            });
}
// a = num / den;  x += a p;  r -= a q
void cg_update_dev(b2p_ctx *c, const double *d_num, const double *d_den, const double *p, const double *q, double *x, double *r, int64_t n)
{
  launch_ew(c, n, [=] __device__(int64_t i)
            {
              const double den = *d_den, a = den != 0.0 ? *d_num / den : 0.0;
              x[i] += a * p[i];
              r[i] -= a * q[i];
            });
}

double dot(b2p_ctx *c, const double *x, const double *y, int64_t n)
{
  double out = 0.0;
  const double *V[1] = {y};
  multi_dot(c, 1, V, x, n, &out);
  return out;
}

double sum(b2p_ctx *c, const double *x, int64_t n)
{
  B2P_LAUNCH(sum_kernel, red_grid(c), NT, 0, c->stream, x, n, red_partials(c));
  double out = 0.0;
  reduce_finish(c, 1, &out);
  return out;
}

void multi_axpy(b2p_ctx *c, int m, const double *coef, const double *const *V, double *w, int64_t n, double sign)
{
  // coefficients arrive on the host; stage them through the pinned buffer -> device scratch
  for (int j0 = 0; j0 < m; j0 += MAXM)
  {
    const int mm = std::min(MAXM, m - j0);
    VecList L;
    for (int j = 0; j < MAXM; j++) L.v[j] = j < mm ? V[j0 + j] : nullptr;
    double *dcoef = red_results(c) + MAXM;  // scratch after the results
    cudaMemcpyAsync(dcoef, coef + j0, sizeof(double) * mm, cudaMemcpyHostToDevice, c->stream);
    B2P_LAUNCH(multi_axpy_kernel, grid_for(c, n), NT, 0, c->stream, L, dcoef, mm, sign, w, n);
  }
}

}  // namespace vec

}  // namespace b2p
