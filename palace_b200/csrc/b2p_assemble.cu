// Full assembly of a (sum of) local partially assembled operator(s) into a device-resident CSR matrix on the L-vector:
// the object BilinearForm::FullAssemble / CeedOperatorFullAssemble hands to HYPRE for the coarsest multigrid level and for
// sparse direct solvers (/root/reference/palace/fem/libceed/operator.cpp:262-523, consumed by
// ParOperator::ParallelAssemble, /root/reference/palace/linalg/rap.cpp:84-152). The reference assembles the COO values
// with libCEED, then sorts COO -> CSR on the host for every assembly. Here
//   * symbolic (once per space, host): the CSR pattern follows from the restriction alone; every element-matrix entry
//     (e, i, j) gets its position in the value array (pos[ne][P][P], uploaded once);
//   * numeric (every assembly, device, no sort): the element matrices are obtained from the OPERATOR KERNELS THEMSELVES --
//     the operator is applied through an identity restriction (one private slot per element dof) to the P "local unit
//     vectors" e_j, which yields column j of every element matrix in one launch -- and a scatter kernel adds
//     c * s_i s_j * A_e(i, j) into the CSR values. Whatever the element kernels compute (sum-factorised hex, dense tets
//     with curl-oriented restrictions, assembled or on-the-fly D) is therefore assembled bit-consistently with the
//     matrix-free action; re-assembly after a coefficient change costs P launches and no host work.
// Intended for the coarse levels (p = 1, 2): the position map takes ne * P^2 integers.
#include <algorithm>

#include "b2p_internal.hpp"

struct b2p_csr
{
  b2p_ctx *ctx = nullptr;
  int64_t n = 0, nnz = 0;
  int ne = 0, P = 0, PS = 0;
  int32_t *d_rowptr = nullptr, *d_col = nullptr, *d_pos = nullptr, *d_eidx = nullptr, *d_gidx = nullptr;
  double *d_val = nullptr, *d_x = nullptr, *d_y = nullptr;
  std::vector<int32_t> h_rowptr, h_col;
};

namespace b2p
{
namespace
{
__global__ void set_unit_kernel(double *x, int64_t total, int P, int j)
{
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w < total) x[w] = ((int)(w % P) == j) ? 1.0 : 0.0;
}
// val[pos(e, i, j)] += c * s_i * s_j * y_E[e][i]   (y_E = column j of every element matrix)
__global__ void scatter_column_kernel(const double *__restrict__ yE, const int32_t *__restrict__ pos, const int32_t *__restrict__ gidx,
                                      int64_t total, int P, int PS, int j, double c, double *val)
{
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= total) return;
  const int64_t e = w / P;
  const int i = (int)(w % P);
  const int32_t k = pos[(size_t)w * P + j];
  if (k < 0) return;
  const double si = gidx[e * PS + i] < 0 ? -1.0 : 1.0, sj = gidx[e * PS + j] < 0 ? -1.0 : 1.0;
  atomicAdd(val + k, c * si * sj * yE[w]);
}
// y = A x, CSR_LANES lanes per row: the lanes stride over the row's entries (coalesced val / col reads; the coarse-level
// rows hold 27-81 entries) and fold their partial sums with shuffles.
constexpr int CSR_LANES = 8;
__global__ void csr_mult_kernel(int64_t n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                const double *__restrict__ val, const double *__restrict__ x, double *__restrict__ y)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / CSR_LANES;
  const int sub = (int)(t % CSR_LANES);
  double s = 0.0;
  if (r < n)
    for (int32_t k = rowptr[r] + sub; k < rowptr[r + 1]; k += CSR_LANES) s += val[k] * x[col[k]];
#pragma unroll
  for (int o = CSR_LANES / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);  // stays inside the row's lane group
  if (r < n && sub == 0) y[r] = s;
}
__global__ void csr_diag_kernel(int64_t n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                const double *__restrict__ val, double *__restrict__ d)
{
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  double s = 0.0;
  for (int32_t k = rowptr[r]; k < rowptr[r + 1]; k++)
    if (col[k] == r) s = val[k];
  d[r] = s;
}
// The real 2n x 2n form [[Ar, Ai], [Ai, -Ar]] of a complex matrix whose parts share one pattern, applied without forming it:
// x = [u; w] -> y = [Ar u + Ai w; Ai u - Ar w]. One pass over rowptr / col serves both halves (4 + 8 + 8 bytes per nonzero
// pair, against 2 x (4 + 8) x 2 for the explicit block matrix); lanes as in csr_mult_kernel.
__global__ void csr_block2_mult_kernel(int64_t n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                       const double *__restrict__ vr, const double *__restrict__ vi, const double *__restrict__ x,
                                       double *__restrict__ y)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / CSR_LANES;
  const int sub = (int)(t % CSR_LANES);
  double top = 0.0, bot = 0.0;
  if (r < n)
    for (int32_t k = rowptr[r] + sub; k < rowptr[r + 1]; k += CSR_LANES)
    {
      const int32_t c = col[k];
      const double ar = vr[k], ai = vi[k], u = x[c], w = x[n + c];
      top += ar * u + ai * w;
      bot += ai * u - ar * w;
    }
#pragma unroll
  for (int o = CSR_LANES / 2; o > 0; o >>= 1)
  {
    top += __shfl_xor_sync(0xffffffffu, top, o);
    bot += __shfl_xor_sync(0xffffffffu, bot, o);
  }
  if (r < n && sub == 0)
  {
    y[r] = top;
    y[n + r] = bot;
  }
}
// d = [diag Ar; -diag Ar]
__global__ void csr_block2_diag_kernel(int64_t n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                       const double *__restrict__ vr, double *__restrict__ d)
{
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  double s = 0.0;
  for (int32_t k = rowptr[r]; k < rowptr[r + 1]; k++)
    if (col[k] == r) s = vr[k];
  d[r] = s;
  d[n + r] = -s;
}
// Values of the explicit block matrix on the pattern of csr_block2_pattern: top row r holds Ar(r, :) then Ai(r, :) (columns
// c, then n + c), bottom row n + r holds Ai(r, :) then -Ar(r, :).
__global__ void csr_block2_fill_kernel(int64_t n, int64_t nnz, const int32_t *__restrict__ rowptr, const double *__restrict__ vr,
                                       const double *__restrict__ vi, double *__restrict__ v2)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / CSR_LANES;
  const int sub = (int)(t % CSR_LANES);
  if (r >= n) return;
  const int32_t b = rowptr[r], e = rowptr[r + 1];
  for (int32_t k = b + sub; k < e; k += CSR_LANES)
  {
    const double ar = vr[k], ai = vi[k];
    v2[(int64_t)b + k] = ar;
    v2[(int64_t)e + k] = ai;
    v2[2 * nnz + b + k] = ai;
    v2[2 * nnz + e + k] = -ar;
  }
}
// mfem::HypreParMatrix::EliminateBC semantics on the local matrix: essential rows and columns zeroed, diagonal set to
// one (DIAG_ONE) or zero (DIAG_ZERO)  (rap.cpp:141-146)
__global__ void csr_eliminate_kernel(int64_t n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col, double *val,
                                     const char *__restrict__ ess, int diag_one)
{
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  for (int32_t k = rowptr[r]; k < rowptr[r + 1]; k++)
    if (ess[r] || ess[col[k]]) val[k] = (diag_one && col[k] == r) ? 1.0 : 0.0;
}
__global__ void mark_kernel(const int32_t *__restrict__ idx, int64_t n, char *flag)
{
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w < n) flag[idx[w]] = 1;
}
inline unsigned blocks(int64_t n, int nt) { return (unsigned)((n + nt - 1) / nt); }
}  // namespace

double *csr_values(b2p_csr *A) { return A->d_val; }

// values = sum_t coefs[t] * A_t  (all terms on the space the pattern was built from)
int csr_assemble_values(b2p_csr *A, int n_terms, b2p_op *const *ops, const double *coefs, double *val, cudaStream_t s)
{
  if (!A || !ops || !coefs || !val || n_terms <= 0) return B2P_ERR_ARG;
  b2p_ctx *ctx = A->ctx;
  const int64_t nE = (int64_t)A->ne * A->P;
  B2P_CUDA(ctx, cudaMemsetAsync(val, 0, sizeof(double) * std::max<int64_t>(A->nnz, 1), s));
  for (int t = 0; t < n_terms; t++)
  {
    b2p_op *op = ops[t];
    B2P_CHECK(ctx, op && op->ne == A->ne && op->P == A->P && op->PS == A->PS && op->lsize == A->n, B2P_ERR_ARG,
              "b2p_csr_assemble: term %d lives on another space", t);
    if (coefs[t] == 0.0) continue;
    // Column j of every element matrix is A_e e_j; it lands at pos(e, i, j) for every row i, so non-symmetric operators (the
    // mixed curl kinds, block sums) are assembled as they are applied, not as their transpose.
    for (int j = 0; j < A->P; j++)
    {
      B2P_LAUNCH(set_unit_kernel, blocks(nE, 256), 256, 0, s, A->d_x, nE, A->P, j);
      B2P_CUDA(ctx, cudaMemsetAsync(A->d_y, 0, sizeof(double) * nE, s));
      ApplyRange rg;
      rg.n_owned = nE;  // the whole E-vector is "owned": no ghost segment (nE >= the operator's L-size)
      int rc = apply_range(op, A->d_eidx, 1.0, A->d_x, A->d_y, rg, 0, s);
      if (rc) return rc;
      B2P_LAUNCH(scatter_column_kernel, blocks(nE, 256), 256, 0, s, A->d_y, A->d_pos, A->d_gidx, nE, A->P, A->PS, j, coefs[t], val);
    }
  }
  B2P_CUDA(ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_eliminate_values(b2p_csr *A, const int32_t *ess_dofs, int64_t n_ess, int diag_policy, double *val, cudaStream_t s)
{
  if (!A || !val || (n_ess > 0 && !ess_dofs)) return B2P_ERR_ARG;
  if (n_ess <= 0) return B2P_SUCCESS;
  b2p_ctx *ctx = A->ctx;
  for (int64_t i = 0; i < n_ess; i++)
    B2P_CHECK(ctx, ess_dofs[i] >= 0 && ess_dofs[i] < A->n, B2P_ERR_ARG, "b2p_csr_eliminate: essential dof %d outside the matrix", ess_dofs[i]);
  int32_t *d_ess = nullptr;
  char *d_flag = nullptr;
  int rc = upload(ctx, ess_dofs, (size_t)n_ess, &d_ess);
  if (rc) return rc;
  if (cudaMalloc(&d_flag, (size_t)A->n) != cudaSuccess)
  {
    cudaFree(d_ess);
    set_error(ctx, "b2p_csr_eliminate: out of device memory");
    return B2P_ERR_CUDA;
  }
  cudaMemsetAsync(d_flag, 0, (size_t)A->n, s);
  B2P_LAUNCH(mark_kernel, blocks(n_ess, 256), 256, 0, s, d_ess, n_ess, d_flag);
  B2P_LAUNCH(csr_eliminate_kernel, blocks(A->n, 256), 256, 0, s, A->n, A->d_rowptr, A->d_col, val, d_flag, diag_policy == 1 ? 1 : 0);
  cudaStreamSynchronize(s);
  cudaFree(d_ess);
  cudaFree(d_flag);
  B2P_CUDA(ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_mult_values(b2p_csr *A, const double *val, const double *x, double *y, cudaStream_t s)
{
  if (!A || !val || !x || !y) return B2P_ERR_ARG;
  B2P_LAUNCH(csr_mult_kernel, blocks(A->n * CSR_LANES, 256), 256, 0, s, A->n, A->d_rowptr, A->d_col, val, x, y);
  B2P_CUDA(A->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_diag_values(b2p_csr *A, const double *val, double *d, cudaStream_t s)
{
  if (!A || !val || !d) return B2P_ERR_ARG;
  B2P_LAUNCH(csr_diag_kernel, blocks(A->n, 256), 256, 0, s, A->n, A->d_rowptr, A->d_col, val, d);
  B2P_CUDA(A->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_block2_mult(b2p_csr *A, const double *vr, const double *vi, const double *x, double *y, cudaStream_t s)
{
  if (!A || !vr || !vi || !x || !y) return B2P_ERR_ARG;
  B2P_LAUNCH(csr_block2_mult_kernel, blocks(A->n * CSR_LANES, 256), 256, 0, s, A->n, A->d_rowptr, A->d_col, vr, vi, x, y);
  B2P_CUDA(A->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_block2_diag(b2p_csr *A, const double *vr, double *d, cudaStream_t s)
{
  if (!A || !vr || !d) return B2P_ERR_ARG;
  B2P_LAUNCH(csr_block2_diag_kernel, blocks(A->n, 256), 256, 0, s, A->n, A->d_rowptr, A->d_col, vr, d);
  B2P_CUDA(A->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int csr_block2_pattern(b2p_csr *A, int32_t **rowptr2, int32_t **col2)
{
  if (!A || !rowptr2 || !col2) return B2P_ERR_ARG;
  b2p_ctx *ctx = A->ctx;
  const int64_t n = A->n, nnz = A->nnz;
  B2P_CHECK(ctx, 4 * nnz < 2147483647LL, B2P_ERR_UNSUPPORTED, "csr_block2_pattern: %lld entries need 64-bit row pointers",
            (long long)(4 * nnz));
  std::vector<int32_t> rp((size_t)2 * n + 1), cl((size_t)4 * nnz);
  for (int64_t r = 0; r < n; r++)
  {
    const int32_t b = A->h_rowptr[(size_t)r], e = A->h_rowptr[(size_t)r + 1];
    rp[(size_t)r] = 2 * b;
    rp[(size_t)(n + r)] = (int32_t)(2 * nnz + 2 * b);
    for (int32_t k = b; k < e; k++)
    {
      const int32_t c = A->h_col[(size_t)k];
      cl[(size_t)b + k] = c;
      cl[(size_t)e + k] = (int32_t)(n + c);
      cl[(size_t)(2 * nnz + b + k)] = c;
      cl[(size_t)(2 * nnz + e + k)] = (int32_t)(n + c);
    }
  }
  rp[(size_t)2 * n] = (int32_t)(4 * nnz);
  int rc = upload(ctx, rp.data(), rp.size(), rowptr2);
  if (!rc) rc = upload(ctx, cl.data(), cl.size(), col2);
  return rc;
}

int csr_block2_fill(b2p_csr *A, const double *vr, const double *vi, double *val2, cudaStream_t s)
{
  if (!A || !vr || !vi || !val2) return B2P_ERR_ARG;
  B2P_LAUNCH(csr_block2_fill_kernel, blocks(A->n * CSR_LANES, 256), 256, 0, s, A->n, A->nnz, A->d_rowptr, vr, vi, val2);
  B2P_CUDA(A->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}
}  // namespace b2p

using namespace b2p;

extern "C"
{

int b2p_csr_create(b2p_ctx *ctx, b2p_op *op, b2p_csr **out)
{
  B2P_CHECK(ctx, ctx && op && out, B2P_ERR_ARG, "b2p_csr_create: null argument");
  const int ne = op->ne, P = op->P, PS = op->PS;
  B2P_CHECK(ctx, (double)ne * P * P < 2.0e9, B2P_ERR_UNSUPPORTED,
            "b2p_csr_create: %d elements x %d^2 entries: full assembly is meant for the coarse levels", ne, P);
  B2P_CHECK(ctx, op->lsize < 2147483647LL, B2P_ERR_UNSUPPORTED, "b2p_csr_create: 32-bit row indices");
  std::vector<int32_t> lidx((size_t)ne * PS);
  B2P_CUDA(ctx, cudaMemcpy(lidx.data(), op->lidx, lidx.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  auto gid = [&](int e, int i) -> int32_t
  {
    const int32_t g = lidx[(size_t)e * PS + i];
    if (g == (int32_t)B2P_SKIP_IDX) return -1;
    return g >= 0 ? g : -1 - g;
  };
  // ---- symbolic: rows with duplicates -> sorted unique columns ----
  const int64_t n = op->lsize;
  std::vector<int64_t> cnt((size_t)n + 1, 0);
  for (int e = 0; e < ne; e++)
  {
    int nv = 0;
    for (int i = 0; i < P; i++) nv += gid(e, i) >= 0;
    for (int i = 0; i < P; i++)
      if (gid(e, i) >= 0) cnt[(size_t)gid(e, i) + 1] += nv;
  }
  for (int64_t r = 0; r < n; r++) cnt[r + 1] += cnt[r];
  std::vector<int32_t> dup((size_t)cnt[n]);
  {
    std::vector<int64_t> fill(cnt.begin(), cnt.end() - 1);
    for (int e = 0; e < ne; e++)
      for (int i = 0; i < P; i++)
      {
        const int32_t r = gid(e, i);
        if (r < 0) continue;
        for (int j = 0; j < P; j++)
          if (gid(e, j) >= 0) dup[(size_t)fill[r]++] = gid(e, j);
      }
  }
  auto *A = new b2p_csr;
  A->ctx = ctx;
  A->n = n;
  A->ne = ne;
  A->P = P;
  A->PS = PS;
  A->h_rowptr.assign((size_t)n + 1, 0);
  for (int64_t r = 0; r < n; r++)
  {
    auto b = dup.begin() + cnt[r], en = dup.begin() + cnt[r + 1];
    std::sort(b, en);
    auto u = std::unique(b, en);
    A->h_rowptr[(size_t)r + 1] = A->h_rowptr[(size_t)r] + (int32_t)(u - b);
    A->h_col.insert(A->h_col.end(), b, u);
  }
  A->nnz = (int64_t)A->h_col.size();
  // ---- position of every element-matrix entry ----
  std::vector<int32_t> pos((size_t)ne * P * P, -1);
  for (int e = 0; e < ne; e++)
    for (int i = 0; i < P; i++)
    {
      const int32_t r = gid(e, i);
      if (r < 0) continue;
      const int32_t *cb = A->h_col.data() + A->h_rowptr[(size_t)r], *ce = A->h_col.data() + A->h_rowptr[(size_t)r + 1];
      for (int j = 0; j < P; j++)
      {
        const int32_t c = gid(e, j);
        if (c < 0) continue;
        pos[((size_t)e * P + i) * P + j] = (int32_t)(std::lower_bound(cb, ce, c) - A->h_col.data());
      }
    }
  // identity restriction: element dof l of element e lives in its own slot e * P + l of an E-vector
  std::vector<int32_t> eidx((size_t)ne * PS, (int32_t)B2P_SKIP_IDX);
  for (int e = 0; e < ne; e++)
    for (int i = 0; i < P; i++)
      if (gid(e, i) >= 0) eidx[(size_t)e * PS + i] = e * P + i;
  int rc = 0;
  if ((rc = upload(ctx, A->h_rowptr.data(), A->h_rowptr.size(), &A->d_rowptr)) || (rc = upload(ctx, A->h_col.data(), A->h_col.size(), &A->d_col)) ||
      (rc = upload(ctx, pos.data(), pos.size(), &A->d_pos)) || (rc = upload(ctx, eidx.data(), eidx.size(), &A->d_eidx)) ||
      (rc = upload(ctx, lidx.data(), lidx.size(), &A->d_gidx)))
  {
    b2p_csr_destroy(A);
    return rc;
  }
  const size_t nE = (size_t)ne * P;
  if (cudaMalloc(&A->d_val, sizeof(double) * std::max<int64_t>(A->nnz, 1)) != cudaSuccess || cudaMalloc(&A->d_x, sizeof(double) * nE) != cudaSuccess ||
      cudaMalloc(&A->d_y, sizeof(double) * nE) != cudaSuccess)
  {
    set_error(ctx, "b2p_csr_create: out of device memory");
    b2p_csr_destroy(A);
    return B2P_ERR_CUDA;
  }
  B2P_CUDA(ctx, cudaMemset(A->d_val, 0, sizeof(double) * std::max<int64_t>(A->nnz, 1)));
  *out = A;
  return B2P_SUCCESS;
}

// values = sum_t coefs[t] * A_t  (all terms on the space the pattern was built from)
int b2p_csr_assemble(b2p_csr *A, int n_terms, b2p_op *const *ops, const double *coefs, b2p_stream stream)
{
  return A ? csr_assemble_values(A, n_terms, ops, coefs, A->d_val, (cudaStream_t)stream) : B2P_ERR_ARG;
}

int64_t b2p_csr_rows(const b2p_csr *A) { return A ? A->n : -1; }
int64_t b2p_csr_nnz(const b2p_csr *A) { return A ? A->nnz : -1; }

// Device arrays for the consumer (e.g. hypre_CSRMatrix with device memory): rowptr[n + 1], col[nnz], val[nnz].
int b2p_csr_device_arrays(b2p_csr *A, const int32_t **rowptr, const int32_t **col, const double **val)
{
  if (!A) return B2P_ERR_ARG;
  if (rowptr) *rowptr = A->d_rowptr;
  if (col) *col = A->d_col;
  if (val) *val = A->d_val;
  return B2P_SUCCESS;
}

int b2p_csr_get_host(b2p_csr *A, int32_t *rowptr, int32_t *col, double *val, b2p_stream stream)
{
  if (!A) return B2P_ERR_ARG;
  if (rowptr) std::copy(A->h_rowptr.begin(), A->h_rowptr.end(), rowptr);
  if (col) std::copy(A->h_col.begin(), A->h_col.end(), col);
  if (val)
  {
    B2P_CUDA(A->ctx, cudaMemcpyAsync(val, A->d_val, sizeof(double) * A->nnz, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    B2P_CUDA(A->ctx, cudaStreamSynchronize((cudaStream_t)stream));
  }
  return B2P_SUCCESS;
}

int b2p_csr_eliminate(b2p_csr *A, const int32_t *ess_dofs, int64_t n_ess, int diag_policy, b2p_stream stream)
{
  return A ? csr_eliminate_values(A, ess_dofs, n_ess, diag_policy, A->d_val, (cudaStream_t)stream) : B2P_ERR_ARG;
}

int b2p_csr_mult(b2p_csr *A, const double *x, double *y, b2p_stream stream)
{
  return A ? csr_mult_values(A, A->d_val, x, y, (cudaStream_t)stream) : B2P_ERR_ARG;
}

int b2p_csr_diag(b2p_csr *A, double *d, b2p_stream stream)
{
  return A ? csr_diag_values(A, A->d_val, d, (cudaStream_t)stream) : B2P_ERR_ARG;
}

void b2p_csr_destroy(b2p_csr *A)
{
  if (!A) return;
  cudaFree(A->d_rowptr);
  cudaFree(A->d_col);
  cudaFree(A->d_pos);
  cudaFree(A->d_eidx);
  cudaFree(A->d_gidx);
  cudaFree(A->d_val);
  cudaFree(A->d_x);
  cudaFree(A->d_y);
  delete A;
}

}  // extern "C"
