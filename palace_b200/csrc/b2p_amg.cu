// Algebraic coarse solvers for the assembled coarsest multigrid level: smoothed-aggregation AMG for one SPD matrix, and the
// auxiliary-space Maxwell solver (AMS, cycle type 14) for the eliminated Nedelec p = 1 matrix built from the discrete gradient
// and the vertex coordinates. They stand where the reference hands the coarse matrix to HYPRE in its GPU configuration
// (linalg/ams.cpp, linalg/amg.cpp: l1-Jacobi relaxation, no aggressive coarsening, a direct solve on the coarsest level).
// The AMG inside is smoothed aggregation, not BoomerAMG's classical coarsening (DESIGN §7 records why).
//
// Setup (SetOperator) runs on the host: strength, greedy aggregation, the smoothed prolongation, the Galerkin products and a
// dense LDL^T pseudo-inverse of the coarsest matrix. The products follow the row-by-row (Gustavson) order with exact zeros
// dropped, so the hierarchy is reproducible entry for entry. Everything the solve needs is uploaded there; Mult allocates
// nothing and never synchronises, so it can be captured in a CUDA graph.
#include <algorithm>
#include <chrono>
#include <cmath>

#include "b2p_linalg.hpp"

namespace b2p
{
b2p_solver *wrap_solver(std::unique_ptr<Solver> &&s);
Solver *solver_of(b2p_solver *s);
const Solver *unwrap_coarse_solver(const Solver *s);

namespace
{
// ---------------------------------------------------------------- host sparse algebra (setup)
struct HCsr
{
  int64_t rows = 0, cols = 0;
  std::vector<int32_t> rp{0}, ci;
  std::vector<double> v;
  int64_t nnz() const { return (int64_t)ci.size(); }
};

HCsr transpose(const HCsr &A)
{
  HCsr T;
  T.rows = A.cols;
  T.cols = A.rows;
  T.rp.assign((size_t)A.cols + 1, 0);
  for (int32_t c : A.ci) T.rp[(size_t)c + 1]++;
  for (int64_t i = 0; i < A.cols; i++) T.rp[(size_t)i + 1] += T.rp[(size_t)i];
  T.ci.resize(A.ci.size());
  T.v.resize(A.v.size());
  std::vector<int32_t> fill(T.rp.begin(), T.rp.end() - 1);
  for (int64_t r = 0; r < A.rows; r++)  // rows in order: the columns of T come out sorted
    for (int32_t k = A.rp[(size_t)r]; k < A.rp[(size_t)r + 1]; k++)
    {
      const int32_t d = fill[(size_t)A.ci[(size_t)k]]++;
      T.ci[(size_t)d] = (int32_t)r;
      T.v[(size_t)d] = A.v[(size_t)k];
    }
  return T;
}

// C = A B row by row: entry (i, k) accumulates a_ij b_jk over the entries of row i of A in stored (sorted) order, starting
// from 0; entries that end exactly zero are dropped; columns sorted.
HCsr spgemm(const HCsr &A, const HCsr &B)
{
  HCsr C;
  C.rows = A.rows;
  C.cols = B.cols;
  C.rp.assign((size_t)A.rows + 1, 0);
  std::vector<double> acc((size_t)B.cols, 0.0);
  std::vector<int64_t> mark((size_t)B.cols, -1);
  std::vector<int32_t> touched;
  for (int64_t i = 0; i < A.rows; i++)
  {
    touched.clear();
    for (int32_t ka = A.rp[(size_t)i]; ka < A.rp[(size_t)i + 1]; ka++)
    {
      const int32_t j = A.ci[(size_t)ka];
      const double a = A.v[(size_t)ka];
      for (int32_t kb = B.rp[(size_t)j]; kb < B.rp[(size_t)j + 1]; kb++)
      {
        const int32_t k = B.ci[(size_t)kb];
        if (mark[(size_t)k] != i)
        {
          mark[(size_t)k] = i;
          acc[(size_t)k] = 0.0;
          touched.push_back(k);
        }
        acc[(size_t)k] += a * B.v[(size_t)kb];
      }
    }
    std::sort(touched.begin(), touched.end());
    for (int32_t k : touched)
      if (acc[(size_t)k] != 0.0)
      {
        C.ci.push_back(k);
        C.v.push_back(acc[(size_t)k]);
      }
    C.rp[(size_t)i + 1] = (int32_t)C.ci.size();
  }
  return C;
}

std::vector<double> diagonal(const HCsr &A)
{
  std::vector<double> d((size_t)A.rows, 0.0);
  for (int64_t r = 0; r < A.rows; r++)
    for (int32_t k = A.rp[(size_t)r]; k < A.rp[(size_t)r + 1]; k++)
      if (A.ci[(size_t)k] == r) d[(size_t)r] = A.v[(size_t)k];
  return d;
}

std::vector<double> abs_row_sums(const HCsr &A)
{
  std::vector<double> s((size_t)A.rows, 0.0);
  for (int64_t r = 0; r < A.rows; r++)
    for (int32_t k = A.rp[(size_t)r]; k < A.rp[(size_t)r + 1]; k++) s[(size_t)r] += std::fabs(A.v[(size_t)k]);
  return s;
}

constexpr double kTheta = 0.08;     // strength threshold
constexpr int kCoarseRows = 500;    // direct solve at or below this size
constexpr int kMaxLevels = 10;
constexpr double kMaxKeep = 0.8;    // a coarsening that keeps more of the rows ends the hierarchy
constexpr double kPivotTol = 1e-12; // LDL^T pivots below this fraction of the largest diagonal entry count as zero
constexpr int64_t kMaxDense = 6000; // the coarsest matrix is stored dense

// Three-pass greedy aggregation in increasing row order; agg[i] = -1 for nodes without a strong neighbour.
std::vector<int32_t> aggregate(const HCsr &A, int32_t &n_agg)
{
  const int64_t n = A.rows;
  const std::vector<double> d = diagonal(A);
  auto strong = [&](int64_t i, int32_t k)
  {
    const int32_t j = A.ci[(size_t)k];
    const double a = A.v[(size_t)k];
    return j != i && a != 0.0 && std::fabs(a) >= kTheta * std::sqrt(std::fabs(d[(size_t)i] * d[(size_t)j]));
  };
  std::vector<int32_t> agg((size_t)n, -1);
  std::vector<char> has_strong((size_t)n, 0);
  n_agg = 0;
  // 1: roots whose strong neighbourhood is untouched
  for (int64_t i = 0; i < n; i++)
  {
    bool free_nbhd = true;
    for (int32_t k = A.rp[(size_t)i]; k < A.rp[(size_t)i + 1]; k++)
      if (strong(i, k))
      {
        has_strong[(size_t)i] = 1;
        if (agg[(size_t)A.ci[(size_t)k]] >= 0) free_nbhd = false;
      }
    if (!has_strong[(size_t)i] || agg[(size_t)i] >= 0 || !free_nbhd) continue;
    agg[(size_t)i] = n_agg;
    for (int32_t k = A.rp[(size_t)i]; k < A.rp[(size_t)i + 1]; k++)
      if (strong(i, k)) agg[(size_t)A.ci[(size_t)k]] = n_agg;
    n_agg++;
  }
  // 2: join the aggregate of the strongest strong neighbour aggregated in pass 1 (ties: lowest index)
  const std::vector<int32_t> agg1 = agg;
  for (int64_t i = 0; i < n; i++)
  {
    if (agg[(size_t)i] >= 0 || !has_strong[(size_t)i]) continue;
    double best = -1.0;
    int32_t target = -1;
    for (int32_t k = A.rp[(size_t)i]; k < A.rp[(size_t)i + 1]; k++)
      if (strong(i, k) && agg1[(size_t)A.ci[(size_t)k]] >= 0 && std::fabs(A.v[(size_t)k]) > best)
      {
        best = std::fabs(A.v[(size_t)k]);
        target = agg1[(size_t)A.ci[(size_t)k]];
      }
    agg[(size_t)i] = target;
  }
  // 3: leftovers with their unaggregated strong neighbours
  for (int64_t i = 0; i < n; i++)
  {
    if (agg[(size_t)i] >= 0 || !has_strong[(size_t)i]) continue;
    agg[(size_t)i] = n_agg;
    for (int32_t k = A.rp[(size_t)i]; k < A.rp[(size_t)i + 1]; k++)
      if (strong(i, k) && agg[(size_t)A.ci[(size_t)k]] < 0) agg[(size_t)A.ci[(size_t)k]] = n_agg;
    n_agg++;
  }
  return agg;
}

// P = (I - omega D^-1 A) T with the unit-norm piecewise-constant T and omega = (4/3) / max_i sum_j |a_ij| / |a_ii|.
HCsr smoothed_prolongation(const HCsr &A, const std::vector<int32_t> &agg, int32_t n_agg)
{
  const int64_t n = A.rows;
  std::vector<int64_t> size((size_t)n_agg, 0);
  for (int32_t a : agg)
    if (a >= 0) size[(size_t)a]++;
  HCsr T;
  T.rows = n;
  T.cols = n_agg;
  T.rp.assign((size_t)n + 1, 0);
  for (int64_t i = 0; i < n; i++)
  {
    if (agg[(size_t)i] >= 0)
    {
      T.ci.push_back(agg[(size_t)i]);
      T.v.push_back(1.0 / std::sqrt((double)size[(size_t)agg[(size_t)i]]));
    }
    T.rp[(size_t)i + 1] = (int32_t)T.ci.size();
  }
  const std::vector<double> d = diagonal(A), rs = abs_row_sums(A);
  double lam = 0.0;
  for (int64_t i = 0; i < n; i++)
    if (d[(size_t)i] != 0.0) lam = std::max(lam, rs[(size_t)i] / std::fabs(d[(size_t)i]));
  const double omega = lam > 0.0 ? (4.0 / 3.0) / lam : 0.0;
  const HCsr AT = spgemm(A, T);
  HCsr P;
  P.rows = n;
  P.cols = n_agg;
  P.rp.assign((size_t)n + 1, 0);
  for (int64_t i = 0; i < n; i++)
  {
    const double s = d[(size_t)i] != 0.0 ? omega / d[(size_t)i] : 0.0;
    int32_t a = T.rp[(size_t)i], ae = T.rp[(size_t)i + 1], b = AT.rp[(size_t)i], be = AT.rp[(size_t)i + 1];
    while (a < ae || b < be)
    {
      int32_t c;
      double t = 0.0, x = 0.0;
      if (b >= be || (a < ae && T.ci[(size_t)a] < AT.ci[(size_t)b]))
      {
        c = T.ci[(size_t)a];
        t = T.v[(size_t)a++];
      }
      else if (a >= ae || AT.ci[(size_t)b] < T.ci[(size_t)a])
      {
        c = AT.ci[(size_t)b];
        x = s * AT.v[(size_t)b++];
      }
      else
      {
        c = T.ci[(size_t)a];
        t = T.v[(size_t)a++];
        x = s * AT.v[(size_t)b++];
      }
      const double p = t - x;
      if (p != 0.0)
      {
        P.ci.push_back(c);
        P.v.push_back(p);
      }
    }
    P.rp[(size_t)i + 1] = (int32_t)P.ci.size();
  }
  return P;
}

// Explicit L^-T D^+ L^-1 of A = L D L^T (no pivoting); a pivot at or below kPivotTol * max |a_ii| is dropped together with
// its column, which gives a generalised inverse on a semidefinite matrix (the constant null space of the auxiliary gradient
// problem).
std::vector<double> dense_pseudo_inverse(const HCsr &A)
{
  const int64_t n = A.rows;
  std::vector<double> a((size_t)(n * n), 0.0), L((size_t)(n * n), 0.0), d((size_t)n, 0.0);
  double amax = 0.0;
  for (int64_t r = 0; r < n; r++)
    for (int32_t k = A.rp[(size_t)r]; k < A.rp[(size_t)r + 1]; k++)
    {
      a[(size_t)(r * n + A.ci[(size_t)k])] = A.v[(size_t)k];
      if (A.ci[(size_t)k] == r) amax = std::max(amax, std::fabs(A.v[(size_t)k]));
    }
  const double tol = kPivotTol * amax;
  std::vector<double> ld((size_t)n);
  for (int64_t k = 0; k < n; k++)
  {
    double dk = a[(size_t)(k * n + k)];
    for (int64_t j = 0; j < k; j++)
    {
      ld[(size_t)j] = L[(size_t)(k * n + j)] * d[(size_t)j];
      dk -= L[(size_t)(k * n + j)] * ld[(size_t)j];
    }
    L[(size_t)(k * n + k)] = 1.0;
    if (!(dk > tol)) continue;  // zero pivot: d_k = 0, column k of L stays zero below the diagonal
    d[(size_t)k] = dk;
    for (int64_t i = k + 1; i < n; i++)
    {
      double s = a[(size_t)(i * n + k)];
      for (int64_t j = 0; j < k; j++) s -= L[(size_t)(i * n + j)] * ld[(size_t)j];
      L[(size_t)(i * n + k)] = s / dk;
    }
  }
  // M = L^-1 (unit lower), by columns
  std::vector<double> M((size_t)(n * n), 0.0);
  for (int64_t c = 0; c < n; c++)
  {
    M[(size_t)(c * n + c)] = 1.0;
    for (int64_t i = c + 1; i < n; i++)
    {
      double s = 0.0;
      for (int64_t j = c; j < i; j++) s -= L[(size_t)(i * n + j)] * M[(size_t)(j * n + c)];
      M[(size_t)(i * n + c)] = s;
    }
  }
  std::vector<double> X((size_t)(n * n), 0.0);
  for (int64_t k = 0; k < n; k++)
  {
    if (d[(size_t)k] == 0.0) continue;
    const double inv = 1.0 / d[(size_t)k];
    for (int64_t i = 0; i <= k; i++)
    {
      const double mi = M[(size_t)(k * n + i)] * inv;
      if (mi == 0.0) continue;
      for (int64_t j = 0; j <= k; j++) X[(size_t)(i * n + j)] += mi * M[(size_t)(k * n + j)];
    }
  }
  return X;
}

// ---------------------------------------------------------------- device data and kernels (solve phase)
template <typename T>
struct DBuf  // owning device array
{
  T *p = nullptr;
  DBuf() = default;
  DBuf(const DBuf &) = delete;
  DBuf &operator=(const DBuf &) = delete;
  ~DBuf() { cudaFree(p); }
  int set(b2p_ctx *ctx, const std::vector<T> &h)
  {
    cudaFree(p);
    p = nullptr;
    return upload(ctx, h.data(), std::max<size_t>(h.size(), 1), &p);
  }
};

struct DCsr
{
  int64_t rows = 0, cols = 0, nnz = 0;
  DBuf<int32_t> rp, ci;
  DBuf<double> v;
  int set(b2p_ctx *ctx, const HCsr &A)
  {
    rows = A.rows;
    cols = A.cols;
    nnz = A.nnz();
    std::vector<int32_t> ci_ = A.ci;
    std::vector<double> v_ = A.v;
    if (ci_.empty()) ci_.push_back(0), v_.push_back(0.0);  // (upload needs one element)
    int rc = rp.set(ctx, A.rp);
    if (!rc) rc = ci.set(ctx, ci_);
    if (!rc) rc = v.set(ctx, v_);
    return rc;
  }
};

inline unsigned nblocks(int64_t n, int nt) { return (unsigned)std::max<int64_t>((n + nt - 1) / nt, 1); }

// y = c + s A x (c may be null, or alias y for the in-place add x += P e); LANES lanes per row as in csr_mult_kernel.
template <int LANES>
__global__ void amg_spmv_kernel(int64_t n, const int32_t *__restrict__ rp, const int32_t *__restrict__ ci,
                                const double *__restrict__ v, const double *__restrict__ x, const double *c, double s, double *y)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / LANES;
  const int sub = (int)(t % LANES);
  double acc = 0.0;
  if (r < n)
    for (int32_t k = rp[r] + sub; k < rp[r + 1]; k += LANES) acc += v[k] * x[ci[k]];
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (r < n && sub == 0) y[r] = (c ? c[r] : 0.0) + s * acc;
}

// One l1-Jacobi sweep, residual and update in one pass: xn = xo + dinv .* (b - A xo).
template <int LANES>
__global__ void amg_l1_jacobi_kernel(int64_t n, const int32_t *__restrict__ rp, const int32_t *__restrict__ ci,
                                     const double *__restrict__ v, const double *__restrict__ dinv, const double *__restrict__ b,
                                     const double *__restrict__ xo, double *__restrict__ xn)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / LANES;
  const int sub = (int)(t % LANES);
  double acc = 0.0;
  if (r < n)
    for (int32_t k = rp[r] + sub; k < rp[r + 1]; k += LANES) acc += v[k] * xo[ci[k]];
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (r < n && sub == 0) xn[r] = xo[r] + dinv[r] * (b[r] - acc);
}

// y = X b with the dense coarsest-level pseudo-inverse (row-major): one warp per row.
__global__ void amg_dense_gemv_kernel(int64_t n, const double *__restrict__ X, const double *__restrict__ b, double *__restrict__ y)
{
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = t / 32;
  const int lane = (int)(t % 32);
  double acc = 0.0;
  if (r < n)
    for (int64_t j = lane; j < n; j += 32) acc += X[r * n + j] * b[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (r < n && lane == 0) y[r] = acc;
}

// (Pi_x^T r, Pi_y^T r, Pi_z^T r) in one pass over the G^T pattern: Pi_c(e, v) = |G(e, v)| t_e[c] / 2.
template <int LANES>
__global__ void ams_pi_restrict_kernel(int64_t nv, const int32_t *__restrict__ rp, const int32_t *__restrict__ ci,
                                       const double *__restrict__ v, const double *__restrict__ t, int64_t ne,
                                       const double *__restrict__ r, double *__restrict__ ox, double *__restrict__ oy,
                                       double *__restrict__ oz)
{
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = w / LANES;
  const int sub = (int)(w % LANES);
  double sx = 0.0, sy = 0.0, sz = 0.0;
  if (row < nv)
    for (int32_t k = rp[row] + sub; k < rp[row + 1]; k += LANES)
    {
      const int32_t e = ci[k];
      const double g = 0.5 * fabs(v[k]) * r[e];
      sx += g * t[e];
      sy += g * t[ne + e];
      sz += g * t[2 * ne + e];
    }
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1)
  {
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
    sz += __shfl_xor_sync(0xffffffffu, sz, o);
  }
  if (row < nv && sub == 0)
  {
    ox[row] = sx;
    oy[row] = sy;
    oz[row] = sz;
  }
}

// x += sum_c Pi_c e_c in one pass over the G pattern (two vertices per edge at p = 1).
__global__ void ams_pi_prolong_kernel(int64_t ne, const int32_t *__restrict__ rp, const int32_t *__restrict__ ci,
                                      const double *__restrict__ v, const double *__restrict__ t, const double *__restrict__ ex,
                                      const double *__restrict__ ey, const double *__restrict__ ez, double *__restrict__ x)
{
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  double s = 0.0;
  for (int32_t k = rp[e]; k < rp[e + 1]; k++)
  {
    const int32_t j = ci[k];
    s += 0.5 * fabs(v[k]) * (t[e] * ex[j] + t[ne + e] * ey[j] + t[2 * ne + e] * ez[j]);
  }
  x[e] += s;
}

constexpr int LANES = 8;

void spmv(b2p_ctx *ctx, const DCsr &A, const double *x, const double *c, double s, double *y)
{
  const int64_t n = A.rows;
  const int32_t *rp = A.rp.p, *ci = A.ci.p;
  const double *v = A.v.p;
  B2P_LAUNCH(amg_spmv_kernel<LANES>, nblocks(n * LANES, 256), 256, 0, ctx->stream, n, rp, ci, v, x, c, s, y);
}
void l1_jacobi(b2p_ctx *ctx, const DCsr &A, const double *dinv, const double *b, const double *xo, double *xn)
{
  const int64_t n = A.rows;
  const int32_t *rp = A.rp.p, *ci = A.ci.p;
  const double *v = A.v.p;
  B2P_LAUNCH(amg_l1_jacobi_kernel<LANES>, nblocks(n * LANES, 256), 256, 0, ctx->stream, n, rp, ci, v, dinv, b, xo, xn);
}

// 1 / sum_j |a_ij| (0 for an empty row)
std::vector<double> l1_dinv(const HCsr &A)
{
  std::vector<double> d = abs_row_sums(A);
  for (double &x : d) x = x > 0.0 ? 1.0 / x : 0.0;
  return d;
}

// ---------------------------------------------------------------- one AMG hierarchy
class AmgHierarchy
{
public:
  struct Level
  {
    DCsr A, P, R;  // P: this level -> next coarser (absent on the coarsest)
    DBuf<double> dinv;
    DVec b, x, t, r;  // right-hand side and iterate (levels > 0), sweep partner, residual
  };
  std::vector<std::unique_ptr<Level>> lv;
  DBuf<double> Xc;  // dense pseudo-inverse of the coarsest matrix
  std::vector<int64_t> rows, nnz;
  int smooth_it = 1;

  void Clear()
  {
    lv.clear();
    rows.clear();
    nnz.clear();
  }

  int Setup(b2p_ctx *ctx, HCsr A)
  {
    Clear();
    while (true)
    {
      auto L = std::make_unique<Level>();
      rows.push_back(A.rows);
      nnz.push_back(A.nnz());
      int rc = L->A.set(ctx, A);
      if (!rc) rc = L->dinv.set(ctx, l1_dinv(A));
      if (rc) return rc;
      L->t.resize(ctx, std::max<int64_t>(A.rows, 1));
      L->r.resize(ctx, std::max<int64_t>(A.rows, 1));
      if (!lv.empty())
      {
        L->b.resize(ctx, std::max<int64_t>(A.rows, 1));
        L->x.resize(ctx, std::max<int64_t>(A.rows, 1));
      }
      bool last = A.rows <= kCoarseRows || (int)lv.size() + 1 >= kMaxLevels;
      HCsr P;
      if (!last)
      {
        int32_t n_agg = 0;
        const std::vector<int32_t> agg = aggregate(A, n_agg);
        last = n_agg == 0 || (double)n_agg > kMaxKeep * (double)A.rows;
        if (!last) P = smoothed_prolongation(A, agg, n_agg);
      }
      if (last)
      {
        B2P_CHECK(ctx, A.rows <= kMaxDense, B2P_ERR_UNSUPPORTED,
                  "AMG setup: the coarsest level keeps %lld rows (aggregation stalled); its dense inverse is limited to %lld",
                  (long long)A.rows, (long long)kMaxDense);
        lv.push_back(std::move(L));
        std::vector<double> X = dense_pseudo_inverse(A);
        return Xc.set(ctx, X);
      }
      const HCsr R = transpose(P);
      HCsr Ac = spgemm(R, spgemm(A, P));
      if ((rc = L->P.set(ctx, P)) || (rc = L->R.set(ctx, R))) return rc;
      lv.push_back(std::move(L));
      A = std::move(Ac);
    }
  }

  // x = V-cycle(b) at level l; zero: start from x = 0 (else from the x given). 2 * smooth_it sweeps: the result ends in x.
  void VCycle(b2p_ctx *ctx, int l, const double *b, double *x, bool zero) const
  {
    const Level &L = *lv[(size_t)l];
    const int64_t n = L.A.rows;
    if (l + 1 == (int)lv.size())
    {
      const double *X = Xc.p;
      B2P_LAUNCH(amg_dense_gemv_kernel, nblocks(n * 32, 256), 256, 0, ctx->stream, n, X, b, x);
      return;
    }
    double *cur = x, *oth = L.t.p;
    if (zero) vec::set(ctx, cur, n, 0.0);
    for (int s = 0; s < smooth_it; s++)
    {
      l1_jacobi(ctx, L.A, L.dinv.p, b, cur, oth);
      std::swap(cur, oth);
    }
    const Level &C = *lv[(size_t)l + 1];
    spmv(ctx, L.A, cur, b, -1.0, L.r.p);
    spmv(ctx, L.R, L.r.p, nullptr, 1.0, C.b.p);
    VCycle(ctx, l + 1, C.b.p, C.x.p, true);
    spmv(ctx, L.P, C.x.p, cur, 1.0, cur);
    for (int s = 0; s < smooth_it; s++)
    {
      l1_jacobi(ctx, L.A, L.dinv.p, b, cur, oth);
      std::swap(cur, oth);
    }
  }
};

// The assembled real matrix behind an operator (CsrOperator, CsrValuesOperator) on the host.
int host_matrix(b2p_ctx *ctx, const Operator &op, HCsr &A)
{
  const double *dval = nullptr;
  b2p_csr *csr = op.AssembledMatrix(&dval);
  B2P_CHECK(ctx, csr && dval, B2P_ERR_ARG,
            "AMG / AMS need an assembled real matrix: b2p_operator_csr, or wrap the solver in b2p_solver_assembled / "
            "b2p_csolver_assembled");
  B2P_CHECK(ctx, ctx->nranks == 1, B2P_ERR_UNSUPPORTED, "AMG / AMS: partitioned spaces are not supported");
  A.rows = A.cols = b2p_csr_rows(csr);
  const int64_t nnz = b2p_csr_nnz(csr);
  A.rp.resize((size_t)A.rows + 1);
  A.ci.resize((size_t)nnz);
  A.v.resize((size_t)nnz);
  int rc = b2p_csr_get_host(csr, A.rp.data(), A.ci.data(), nullptr, (b2p_stream)ctx->stream);
  if (rc) return rc;
  B2P_CUDA(ctx, cudaMemcpyAsync(A.v.data(), dval, sizeof(double) * (size_t)nnz, cudaMemcpyDeviceToHost, ctx->stream));
  B2P_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B2P_SUCCESS;
}

// What b2p_solver_amg_levels reports on: the hierarchies of an AMG or AMS solver.
class AlgebraicSolver : public Solver
{
public:
  AlgebraicSolver(b2p_ctx *c, int cycle_it, int smooth_it) : Solver(c), cycle_it(cycle_it), smooth_it(smooth_it) {}
  int Status() const override { return status; }
  virtual const AmgHierarchy *Hierarchy(int h) const = 0;
  double setup_ms = 0.0;

protected:
  int cycle_it, smooth_it;
  int status = B2P_SUCCESS;
  bool Ready() const
  {
    if (height > 0) return true;
    set_error(ctx, "AMG / AMS applied without a successful SetOperator");
    return false;
  }
  void Fail(int rc)
  {
    status = rc;
    height = width = 0;
  }
};

// Smoothed-aggregation AMG: `cycle_it` V-cycles from zero (or from the initial guess).
class AmgSolver : public AlgebraicSolver
{
  AmgHierarchy H;

public:
  AmgSolver(b2p_ctx *c, int cycle_it, int smooth_it) : AlgebraicSolver(c, cycle_it, smooth_it) { H.smooth_it = smooth_it; }
  const AmgHierarchy *Hierarchy(int h) const override { return h == 0 ? &H : nullptr; }
  void SetOperator(const Operator &op) override
  {
    const auto t0 = std::chrono::steady_clock::now();
    HCsr A;
    int rc = host_matrix(ctx, op, A);
    if (!rc) rc = H.Setup(ctx, std::move(A));
    if (rc) return Fail(rc);
    status = B2P_SUCCESS;
    height = width = op.Height();
    setup_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  void Mult(const double *b, double *x) const override
  {
    if (!Ready()) return;
    for (int c = 0; c < cycle_it; c++) H.VCycle(ctx, 0, b, x, c == 0 && !initial_guess);
  }
};

// AMS, cycle "01(3+4+5)10": l1-Jacobi on A, the gradient correction x += G V_G(G^T r), the additive nodal correction
// x += sum_c Pi_c V_c(Pi_c^T r), then the gradient correction and the smoother again. `singular` drops the gradient
// correction (the curl-curl operator without a mass term, whose G^T A G vanishes).
class AmsSolver : public AlgebraicSolver
{
  bool singular;
  int64_t n_e, n_v;
  HCsr G;                  // host copy of the discrete gradient (n_e x n_v)
  std::vector<double> xyz; // [n_v][3]
  AmgHierarchy H[4];       // G, Pi_x, Pi_y, Pi_z
  DCsr A_, G_, Gt_;
  DBuf<double> dinv_, t_;  // l1 diagonal of A; edge vectors t[c][e]
  mutable DVec T_, r_, bv_[3], xv_[3];

public:
  AmsSolver(b2p_ctx *c, int cycle_it, int smooth_it, bool singular, HCsr &&G_host, std::vector<double> &&coords)
    : AlgebraicSolver(c, cycle_it, smooth_it), singular(singular), n_e(G_host.rows), n_v(G_host.cols), G(std::move(G_host)),
      xyz(std::move(coords))
  {
    for (auto &h : H) h.smooth_it = smooth_it;
  }
  const AmgHierarchy *Hierarchy(int h) const override { return h >= 0 && h < 4 ? &H[h] : nullptr; }
  void SetOperator(const Operator &op) override
  {
    const auto t0 = std::chrono::steady_clock::now();
    HCsr A;
    int rc = host_matrix(ctx, op, A);
    if (rc) return Fail(rc);
    if (A.rows != n_e)
    {
      set_error(ctx, "AMS: the matrix has %lld rows, the discrete gradient %lld (one row per edge)", (long long)A.rows, (long long)n_e);
      return Fail(B2P_ERR_ARG);
    }
    // t_e = G [x y z];  Pi_c(e, v) = |G(e, v)| t_e[c] / 2
    std::vector<double> t((size_t)(3 * n_e), 0.0);
    for (int64_t e = 0; e < n_e; e++)
      for (int c = 0; c < 3; c++)
      {
        double s = 0.0;
        for (int32_t k = G.rp[(size_t)e]; k < G.rp[(size_t)e + 1]; k++) s += G.v[(size_t)k] * xyz[(size_t)(3 * G.ci[(size_t)k] + c)];
        t[(size_t)(c * n_e + e)] = s;
      }
    const HCsr Gt = transpose(G);
    const HCsr AG = spgemm(A, G);
    if (!singular && (rc = H[0].Setup(ctx, spgemm(Gt, AG)))) return Fail(rc);
    if (singular) H[0].Clear();
    for (int c = 0; c < 3; c++)
    {
      HCsr Pi = G;
      for (int64_t e = 0; e < n_e; e++)
        for (int32_t k = G.rp[(size_t)e]; k < G.rp[(size_t)e + 1]; k++) Pi.v[(size_t)k] = 0.5 * std::fabs(G.v[(size_t)k]) * t[(size_t)(c * n_e + e)];
      if ((rc = H[c + 1].Setup(ctx, spgemm(transpose(Pi), spgemm(A, Pi))))) return Fail(rc);
    }
    if ((rc = A_.set(ctx, A)) || (rc = G_.set(ctx, G)) || (rc = Gt_.set(ctx, Gt)) || (rc = dinv_.set(ctx, l1_dinv(A))) ||
        (rc = t_.set(ctx, t)))
      return Fail(rc);
    T_.resize(ctx, std::max<int64_t>(n_e, 1));
    r_.resize(ctx, std::max<int64_t>(n_e, 1));
    for (int c = 0; c < 3; c++)
    {
      bv_[c].resize(ctx, std::max<int64_t>(n_v, 1));
      xv_[c].resize(ctx, std::max<int64_t>(n_v, 1));
    }
    status = B2P_SUCCESS;
    height = width = n_e;
    setup_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  void Mult(const double *b, double *x) const override
  {
    if (!Ready()) return;
    double *cur = x, *oth = T_.p;
    auto smooth = [&]()
    {
      for (int s = 0; s < smooth_it; s++)
      {
        l1_jacobi(ctx, A_, dinv_.p, b, cur, oth);
        std::swap(cur, oth);
      }
    };
    auto gradient = [&]()
    {
      if (singular) return;
      spmv(ctx, A_, cur, b, -1.0, r_.p);
      spmv(ctx, Gt_, r_.p, nullptr, 1.0, bv_[0].p);
      H[0].VCycle(ctx, 0, bv_[0].p, xv_[0].p, true);
      spmv(ctx, G_, xv_[0].p, cur, 1.0, cur);
    };
    const int32_t *gt_rp = Gt_.rp.p, *gt_ci = Gt_.ci.p, *g_rp = G_.rp.p, *g_ci = G_.ci.p;
    const double *gt_v = Gt_.v.p, *g_v = G_.v.p, *t = t_.p, *r = r_.p, *ex = xv_[0].p, *ey = xv_[1].p, *ez = xv_[2].p;
    double *bx = bv_[0].p, *by = bv_[1].p, *bz = bv_[2].p;
    const int64_t n_e = this->n_e, n_v = this->n_v;
    if (!initial_guess) vec::set(ctx, cur, n_e, 0.0);
    for (int c = 0; c < cycle_it; c++)
    {
      smooth();
      gradient();
      spmv(ctx, A_, cur, b, -1.0, r_.p);
      B2P_LAUNCH(ams_pi_restrict_kernel<LANES>, nblocks(n_v * LANES, 256), 256, 0, ctx->stream, n_v, gt_rp, gt_ci, gt_v, t, n_e, r,
                 bx, by, bz);
      for (int k = 0; k < 3; k++) H[k + 1].VCycle(ctx, 0, bv_[k].p, xv_[k].p, true);
      B2P_LAUNCH(ams_pi_prolong_kernel, nblocks(n_e, 256), 256, 0, ctx->stream, n_e, g_rp, g_ci, g_v, t, ex, ey, ez, cur);
      gradient();
      smooth();
    }
    // 2 * smooth_it sweeps per cycle: the iterate is back in x
  }
};
}  // namespace
}  // namespace b2p

using namespace b2p;

extern "C"
{

int b2p_solver_amg(b2p_ctx *ctx, int cycle_it, int smooth_it, b2p_solver **out)
{
  B2P_CHECK(ctx, ctx && out && cycle_it >= 1 && smooth_it >= 1, B2P_ERR_ARG, "b2p_solver_amg: bad argument");
  *out = wrap_solver(std::make_unique<AmgSolver>(ctx, cycle_it, smooth_it));
  return B2P_SUCCESS;
}

int b2p_solver_ams(b2p_ctx *ctx, int cycle_it, int smooth_it, int singular, int64_t n_edges, int64_t n_vertices,
                   const int32_t *G_rowptr, const int32_t *G_col, const double *G_val, const double *coords, b2p_solver **out)
{
  B2P_CHECK(ctx, ctx && out && cycle_it >= 1 && smooth_it >= 1 && n_edges > 0 && n_vertices > 0 && G_rowptr && G_col && G_val && coords,
            B2P_ERR_ARG, "b2p_solver_ams: bad argument");
  B2P_CHECK(ctx, n_edges < 2147483647LL && n_vertices < 2147483647LL, B2P_ERR_UNSUPPORTED, "b2p_solver_ams: 32-bit indices");
  HCsr G;
  G.rows = n_edges;
  G.cols = n_vertices;
  G.rp.assign(G_rowptr, G_rowptr + n_edges + 1);
  B2P_CHECK(ctx, G.rp[0] == 0, B2P_ERR_ARG, "b2p_solver_ams: G_rowptr[0] must be 0");
  for (int64_t e = 0; e < n_edges; e++)
    B2P_CHECK(ctx, G.rp[(size_t)e + 1] >= G.rp[(size_t)e], B2P_ERR_ARG, "b2p_solver_ams: G_rowptr decreases at row %lld", (long long)e);
  const int64_t nnz = G.rp[(size_t)n_edges];
  G.ci.assign(G_col, G_col + nnz);
  G.v.assign(G_val, G_val + nnz);
  for (int64_t e = 0; e < n_edges; e++)
    for (int32_t k = G.rp[(size_t)e]; k < G.rp[(size_t)e + 1]; k++)
    {
      B2P_CHECK(ctx, G.ci[(size_t)k] >= 0 && G.ci[(size_t)k] < n_vertices, B2P_ERR_ARG,
                "b2p_solver_ams: G column %d outside the %lld vertices", G.ci[(size_t)k], (long long)n_vertices);
      B2P_CHECK(ctx, k == G.rp[(size_t)e] || G.ci[(size_t)k] > G.ci[(size_t)k - 1], B2P_ERR_ARG,
                "b2p_solver_ams: the columns of G row %lld are not sorted and unique", (long long)e);
    }
  std::vector<double> xyz(coords, coords + 3 * n_vertices);
  *out = wrap_solver(std::make_unique<AmsSolver>(ctx, cycle_it, smooth_it, singular != 0, std::move(G), std::move(xyz)));
  return B2P_SUCCESS;
}

int b2p_solver_amg_levels(b2p_solver *s, int hierarchy, int64_t *rows, int64_t *nnz, int max_levels)
{
  const auto *a = dynamic_cast<const AlgebraicSolver *>(unwrap_coarse_solver(solver_of(s)));
  if (!a || max_levels < 0) return -1;
  const AmgHierarchy *h = a->Hierarchy(hierarchy);
  if (!h) return -1;
  const int n = (int)h->rows.size();
  for (int l = 0; l < n && l < max_levels; l++)
  {
    if (rows) rows[l] = h->rows[(size_t)l];
    if (nnz) nnz[l] = h->nnz[(size_t)l];
  }
  return n;
}

double b2p_solver_amg_setup_ms(b2p_solver *s)
{
  const auto *a = dynamic_cast<const AlgebraicSolver *>(unwrap_coarse_solver(solver_of(s)));
  return a ? a->setup_ms : -1.0;
}

}  // extern "C"
