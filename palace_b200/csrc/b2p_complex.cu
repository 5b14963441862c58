// Complex-valued operators and Krylov solvers on split (real, imag) device vectors, as Palace
// represents them (ComplexVector = two mfem::Vectors, /root/reference/palace/linalg/vector.hpp:23-27):
//   ComplexParOperator   = ComplexParOperator over ComplexWrapperOperator / BuildParSumOperator with complex
//                          coefficients (/root/reference/palace/linalg/rap.cpp:481-517,843-919,
//                          /root/reference/palace/linalg/operator.cpp:98-134): A = sum_i (c_i^r + i c_i^i) A_i
//                          with real partially assembled A_i
//   RealPcSolver         = a real preconditioner applied to the real and imaginary parts, i.e. the
//                          "PCMatReal" configuration (/root/reference/palace/models/spaceoperator.cpp:1098-1105)
//   ComplexIterativeSolver = CgSolver / GmresSolver / FgmresSolver<ComplexOperator>
//                          (/root/reference/palace/linalg/iterative.cpp:361-871, complex Givens :112-226)
// Inner product convention: Dot(x, y) = y^H x (vector.cpp:674-685); Gram-Schmidt calls dot(w, V_j) (orthog.hpp:48-49).
#include <complex>
#include <cstring>
#include <limits>

#include "b2p_givens.hpp"
#include "b2p_linalg.hpp"

namespace b2p
{

using cplx = std::complex<double>;

namespace
{
constexpr int NT = 256;
constexpr int RED_BLOCKS = 264;  // two blocks per SM of an H100 SXM (132 SMs)
constexpr int MAXM = 4;  // complex vectors per multi-dot pass

struct CVecList
{
  const double *re[MAXM], *im[MAXM];
};

// out[2j] = sum wr*vr + wi*vi ; out[2j+1] = sum wi*vr - wr*vi   (= V_j^H w)
__global__ void __launch_bounds__(NT) cmulti_dot_kernel(CVecList V, const double *__restrict__ wr, const double *__restrict__ wi, int64_t n,
                                                        int m, double *part)
{
  double acc[2 * MAXM];
#pragma unroll
  for (int j = 0; j < 2 * MAXM; j++) acc[j] = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    const double a = wr[i], b = wi[i];
#pragma unroll
    for (int j = 0; j < MAXM; j++)
      if (j < m)
      {
        const double vr = V.re[j][i], vi = V.im[j][i];
        acc[2 * j] += a * vr + b * vi;
        acc[2 * j + 1] += b * vr - a * vi;
      }
  }
  __shared__ double sh[2 * MAXM][NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 2 * MAXM; j++)
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
    for (int j = 0; j < 2 * MAXM; j++)
    {
      double v = lane < NT / 32 ? sh[j][lane] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) part[(size_t)j * RED_BLOCKS + blockIdx.x] = v;
    }
  }
}

__global__ void creduce_kernel(const double *part, int nblocks, double *out)
{
  const int j = blockIdx.x;
  double v = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 32) v += part[(size_t)j * RED_BLOCKS + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (threadIdx.x == 0) out[j] = v;
}

// w += sign * sum_j (cr_j + i ci_j) V_j
__global__ void cmulti_axpy_kernel(CVecList V, const double *__restrict__ coef, int m, double sign, double *__restrict__ wr,
                                   double *__restrict__ wi, int64_t n)
{
  __shared__ double sc[2 * MAXM];
  if (threadIdx.x < 2 * m) sc[threadIdx.x] = sign * coef[threadIdx.x];
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    double a = wr[i], b = wi[i];
    for (int j = 0; j < m; j++)
    {
      const double vr = V.re[j][i], vi = V.im[j][i];
      a += sc[2 * j] * vr - sc[2 * j + 1] * vi;
      b += sc[2 * j + 1] * vr + sc[2 * j] * vi;
    }
    wr[i] = a;
    wi[i] = b;
  }
}

// dinv = omega / d (complex reciprocal of the assembled diagonal, jacobi.cpp:75-96)
__global__ void creciprocal_kernel(double *__restrict__ dr, double *__restrict__ di, double omega, int64_t n)
{
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
  {
    const double a = dr[i], b = di[i], m = a * a + b * b;
    dr[i] = omega * a / m;
    di[i] = -omega * b / m;
  }
}
// y = dinv * x (jacobi.cpp:47-63) or y = conj(dinv) * x (transpose branch, :64-72)
__global__ void cdiag_mult_kernel(const double *__restrict__ dr, const double *__restrict__ di, const double *__restrict__ xr,
                                  const double *__restrict__ xi, double *__restrict__ yr, double *__restrict__ yi, double sgn, int64_t n)
{
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
  {
    const double a = dr[i], b = sgn * di[i], u = xr[i], v = xi[i];
    yr[i] = a * u - b * v;
    yi[i] = b * u + a * v;
  }
}

// Chebyshev update with the complex inverse diagonal and the solution update folded in (chebyshev.cpp:81-156):
// d = sd d + sr dinv r, then y = d (assign) or y += d
__global__ void ccheb_kernel(double sd, double sr, const double *__restrict__ ir, const double *__restrict__ ii, const double *__restrict__ rr,
                             const double *__restrict__ ri, double *__restrict__ dr, double *__restrict__ di, double *__restrict__ yr,
                             double *__restrict__ yi, int first, int assign, int64_t n)
{
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
  {
    const double a = ir[i], b = ii[i], u = rr[i], v = ri[i];
    double er = sr * (a * u - b * v), ei = sr * (b * u + a * v);
    if (!first)
    {
      er += sd * dr[i];
      ei += sd * di[i];
    }
    dr[i] = er;
    di[i] = ei;
    if (assign)
    {
      yr[i] = er;
      yi[i] = ei;
    }
    else
    {
      yr[i] += er;
      yi[i] += ei;
    }
  }
}

inline int grid_for(b2p_ctx *c, int64_t n)
{
  const int64_t want = (n + 2 * NT - 1) / (2 * NT), cap = (int64_t)c->sm_count * 8;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

}  // namespace

// ------------------------------------------------------------------------------------ complex vector ops
struct CPtr
{
  double *re, *im;
};
struct CCPtr
{
  const double *re, *im;
};

void cmulti_dot(b2p_ctx *c, int m, const CCPtr *V, CCPtr w, int64_t n, cplx *out)
{
  double *part = c->d_red, *res = c->d_red + (size_t)2 * MAXM * RED_BLOCKS;
  for (int j0 = 0; j0 < m; j0 += MAXM)
  {
    const int mm = std::min(MAXM, m - j0);
    CVecList L;
    for (int j = 0; j < MAXM; j++)
    {
      L.re[j] = j < mm ? V[j0 + j].re : nullptr;
      L.im[j] = j < mm ? V[j0 + j].im : nullptr;
    }
    const int rg = std::min(RED_BLOCKS, 2 * std::max(1, c->sm_count));  // two blocks per SM
    B2P_LAUNCH(cmulti_dot_kernel, rg, NT, 0, c->stream, L, w.re, w.im, n, mm, part);
    B2P_LAUNCH(creduce_kernel, 2 * mm, 32, 0, c->stream, part, rg, res);
    if (c->nranks > 1 && c->comm) b2p_allreduce_sum(c, res, 2 * mm);
    cudaMemcpyAsync(c->h_red, res, sizeof(double) * 2 * mm, cudaMemcpyDeviceToHost, c->stream);
    cudaStreamSynchronize(c->stream);
    for (int j = 0; j < mm; j++) out[j0 + j] = cplx(c->h_red[2 * j], c->h_red[2 * j + 1]);
  }
}

cplx cdot(b2p_ctx *c, CCPtr x, CCPtr y, int64_t n)  // y^H x
{
  cplx out;
  cmulti_dot(c, 1, &y, x, n, &out);
  return out;
}
double cnorm(b2p_ctx *c, CCPtr x, int64_t n) { return std::sqrt(std::abs(cdot(c, x, x, n).real())); }

void cmulti_axpy(b2p_ctx *c, int m, const cplx *coef, const CCPtr *V, CPtr w, int64_t n, double sign)
{
  double *dcoef = c->d_red + (size_t)2 * MAXM * RED_BLOCKS + 2 * MAXM;
  for (int j0 = 0; j0 < m; j0 += MAXM)
  {
    const int mm = std::min(MAXM, m - j0);
    CVecList L;
    double h[2 * MAXM];
    for (int j = 0; j < MAXM; j++)
    {
      L.re[j] = j < mm ? V[j0 + j].re : nullptr;
      L.im[j] = j < mm ? V[j0 + j].im : nullptr;
      if (j < mm)
      {
        h[2 * j] = coef[j0 + j].real();
        h[2 * j + 1] = coef[j0 + j].imag();
      }
    }
    cudaMemcpyAsync(dcoef, h, sizeof(double) * 2 * mm, cudaMemcpyHostToDevice, c->stream);
    cudaStreamSynchronize(c->stream);  // h lives on this stack frame
    B2P_LAUNCH(cmulti_axpy_kernel, grid_for(c, n), NT, 0, c->stream, L, dcoef, mm, sign, w.re, w.im, n);
  }
}
void caxpy(b2p_ctx *c, cplx a, CCPtr x, CPtr y, int64_t n) { cmulti_axpy(c, 1, &a, &x, y, n, 1.0); }

// ------------------------------------------------------------------------------------ ComplexOperator
class ComplexOperator
{
public:
  b2p_ctx *ctx;
  int64_t n;
  ComplexOperator(b2p_ctx *c, int64_t n_) : ctx(c), n(n_) {}
  virtual ~ComplexOperator() = default;
  virtual void Mult(CCPtr x, CPtr y) const = 0;
  virtual void MultHermitianTranspose(CCPtr x, CPtr y) const = 0;
  virtual void AssembleDiagonal(CPtr d) const = 0;
  virtual bool IsReal() const { return false; }  // no imaginary part (operator.hpp:47)
  virtual const int32_t *EssentialTrueDofs() const { return nullptr; }  // device list
  virtual int64_t NumEssential() const { return 0; }
  // y += a A x; the default goes through a temporary, operators that can accumulate straight into y override it
  virtual void AddMult(CCPtr x, CPtr y, cplx a) const
  {
    if (tmp_.n != 2 * n) tmp_.resize(ctx, 2 * n);
    CPtr t{tmp_.p, tmp_.p + n};
    Mult(x, t);
    caxpy(ctx, a, CCPtr{t.re, t.im}, y, n);
  }
  virtual bool NativeAddMult() const { return false; }  // AddMult with a real scalar accumulates into y (no temporary)
  // r = b - A y: with a native AddMult a copy plus one accumulating apply (no zero fill, no AXPBY pass)
  void Residual(CCPtr b, CCPtr y, CPtr r) const
  {
    if (NativeAddMult())
    {
      vec::copy(ctx, r.re, b.re, n);
      vec::copy(ctx, r.im, b.im, n);
      AddMult(y, r, cplx(-1.0, 0.0));
    }
    else
    {
      Mult(y, r);
      vec::axpby(ctx, 1.0, b.re, -1.0, r.re, n);
      vec::axpby(ctx, 1.0, b.im, -1.0, r.im, n);
    }
  }

protected:
  mutable DVec tmp_;
};

class ComplexParOperator : public ComplexOperator
{
public:
  struct Term
  {
    b2p_op *op;
    double cr, ci;
  };
  ComplexParOperator(b2p_ctx *c, int64_t tsize, const std::vector<Term> &terms_, const int32_t *ess, int64_t n_ess_, int diag_policy_)
    : ComplexOperator(c, tsize), terms(terms_), n_ess(n_ess_), diag_policy(diag_policy_)
  {
    if (n_ess > 0) upload(c, ess, (size_t)n_ess, &d_ess);
    for (auto &t : terms)
      if (!t.op->lidx_bc) b2p_op_set_essential(t.op, ess, n_ess);
    build_fused();
  }
  ~ComplexParOperator() override
  {
    cudaFree(d_ess);
    cudaFree(zcoef);
    cudaFree(zcoef_h);
    if (sum_re) b2p_op_destroy(sum_re);
    if (sum_im) b2p_op_destroy(sum_im);
  }

  // Fused path: when every term is a sum-factorised ND operator over the same geometry, space and essential set,
  // the complex sum  sum_i (c_i^r + i c_i^i) A_i  is ONE element operator whose pointwise coefficient is complex:
  // per element {mass Re, mass Im, curl Re, curl Im} 3x3 tensors = sum_i c_i * (material tensor of term i). One
  // kernel launch then replaces the 2-4 real applies per term of the reference's ComplexWrapperOperator
  // (operator.cpp:98-134) and streams the geometry once.
  void build_fused()
  {
    // Default: one pass over the geometry instead of one real apply per term and part (tools/zfused_bench.py times both);
    // parity with the term-by-term path in tests/test_zfused_gpu.py. B2P_COMPLEX_FUSED=0 keeps one real apply per term and part.
    const char *env = std::getenv("B2P_COMPLEX_FUSED");
    if (env && env[0] == '0') return;
    const b2p_op *o0 = terms[0].op;
    bool block = false;
    for (auto &t : terms) block = block || (!t.op->dense && t.op->bcoef);
    if ((o0->dense || block) && terms.size() >= 2)
    {
      // Dense-basis terms (tets, prisms) have no complex element kernel; their sum still collapses to TWO real dense operators,
      // S_re = sum_t c_t^r A_t and S_im = sum_t c_t^i A_t (b2p_op_create_sum: stacked tables, summed per-element tensors), so a
      // complex matvec costs 4 dense applies (2 when every c_t^i = 0) instead of 2-4 per term. Sum-factorised hex terms with a
      // mixed curl kind (Floquet-periodic models) take the same route: S_re and S_im are then two block operators.
      std::vector<b2p_op *> ops;
      std::vector<double> cr, ci;
      for (auto &t : terms)
      {
        ops.push_back(t.op);
        cr.push_back(t.cr);
        ci.push_back(t.ci);
      }
      if (b2p_op_create_sum(ctx, (int)ops.size(), ops.data(), cr.data(), &sum_re) == B2P_SUCCESS &&
          b2p_op_create_sum(ctx, (int)ops.size(), ops.data(), ci.data(), &sum_im) == B2P_SUCCESS)
      {
        // Block sums at q1d = p + 1 with mirror-symmetric tables: one nd_hex_apply7_kernel<..., CPLX> launch reads S_re's and
        // S_im's coefficient blocks (bcoef, or bcoef_t for the Hermitian transpose) instead of 4 applies. S_re / S_im stay:
        // assembly (AssembleValues) reads them, and p = 1 and other tables keep the 4 applies.
        cta = block && !sum_re->dense && sum_re->bcoef && sum_im->bcoef &&
              choose_hex_complex_kernel(sum_re, (int)terms.size()) == HexComplexKernel::ND7Z;
        fused_imag = !IsReal();
        return;
      }
      if (sum_re) b2p_op_destroy(sum_re);
      if (sum_im) b2p_op_destroy(sum_im);
      sum_re = sum_im = nullptr;  // not fusable (mixed kinds / spaces): term by term
      return;
    }
    // the one-pass kernel: choose_hex_complex_kernel (a single term at p >= 4 keeps its real applies)
    const HexComplexKernel zk = choose_hex_complex_kernel(terms[0].op, (int)terms.size());
    for (auto &t : terms)
    {
      b2p_op *o = t.op;
      if (choose_hex_complex_kernel(o, (int)terms.size()) == HexComplexKernel::NONE || o->bcoef || o->geom != o0->geom || o->p != o0->p ||
          o->q1d != o0->q1d || o->ne != o0->ne || o->lsize != o0->lsize || o->PS != o0->PS || !o->ecoef || !o->lidx_bc)
        return;
    }
    const size_t nidx = (size_t)o0->ne * o0->PS;
    std::vector<int32_t> a(nidx), b(nidx);
    if (cudaMemcpy(a.data(), o0->lidx_bc, nidx * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return;
    for (size_t i = 1; i < terms.size(); i++)
    {
      if (cudaMemcpy(b.data(), terms[i].op->lidx_bc, nidx * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess) return;
      if (a != b) return;  // different restriction or essential set
    }
    const int ne = o0->ne;
    fused_e18.assign(terms.size(), std::vector<double>((size_t)18 * ne));
    for (size_t i = 0; i < terms.size(); i++)
      if (cudaMemcpy(fused_e18[i].data(), terms[i].op->ecoef, fused_e18[i].size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess)
        return;
    fused = fill_fused();
    cta = fused && zk == HexComplexKernel::ND7Z;
  }

  // zcoef / zcoef_h from the cached per-term material tensors and the current scalar coefficients
  bool fill_fused()
  {
    const int ne = terms[0].op->ne;
    std::vector<double> z((size_t)36 * ne, 0.0);
    bool mass = false, curl = false;
    fused_imag = false;
    for (size_t ti = 0; ti < terms.size(); ti++)
    {
      const Term &t = terms[ti];
      const std::vector<double> &e18 = fused_e18[ti];
      const bool m = (t.op->kind == B2P_ND_MASS || t.op->kind == B2P_CURLCURL_MASS);
      const bool k = (t.op->kind == B2P_CURLCURL || t.op->kind == B2P_CURLCURL_MASS);
      mass = mass || m;
      curl = curl || k;
      fused_imag = fused_imag || t.ci != 0.0;
      for (int e = 0; e < ne; e++)
        for (int i = 0; i < 9; i++)
        {
          if (m)
          {
            z[(size_t)36 * e + i] += t.cr * e18[(size_t)18 * e + i];
            z[(size_t)36 * e + 9 + i] += t.ci * e18[(size_t)18 * e + i];
          }
          if (k)
          {
            z[(size_t)36 * e + 18 + i] += t.cr * e18[(size_t)18 * e + 9 + i];
            z[(size_t)36 * e + 27 + i] += t.ci * e18[(size_t)18 * e + 9 + i];
          }
        }
    }
    fused_kind = mass && curl ? B2P_CURLCURL_MASS : (mass ? B2P_ND_MASS : B2P_CURLCURL);
    cudaFree(zcoef);
    cudaFree(zcoef_h);
    zcoef = zcoef_h = nullptr;
    if (upload(ctx, z.data(), z.size(), &zcoef)) return false;
    for (int e = 0; e < ne; e++)  // Hermitian transpose: conjugated coefficients (the A_i are real symmetric)
      for (int i = 0; i < 9; i++)
      {
        z[(size_t)36 * e + 9 + i] = -z[(size_t)36 * e + 9 + i];
        z[(size_t)36 * e + 27 + i] = -z[(size_t)36 * e + 27 + i];
      }
    if (upload(ctx, z.data(), z.size(), &zcoef_h)) return false;
    return true;
  }

  // New complex coefficients of the terms (next frequency of a driven sweep): nothing is rebuilt; the fused kernel's
  // per-element complex tensors are refilled from the cached material tensors (36 doubles per element uploaded).
  size_t NumTerms() const { return terms.size(); }
  void SetCoefficients(const double *cr, const double *ci)
  {
    for (size_t t = 0; t < terms.size(); t++)
    {
      terms[t].cr = cr[t];
      terms[t].ci = ci[t];
    }
    if (fused)
    {
      fused = fill_fused();
      cta = cta && fused;
    }
    if (sum_re)
    {
      std::vector<b2p_op *> ops;
      for (auto &t : terms) ops.push_back(t.op);
      b2p_op_sum_set_coefficients(sum_re, (int)ops.size(), ops.data(), cr);
      b2p_op_sum_set_coefficients(sum_im, (int)ops.size(), ops.data(), ci);
      fused_imag = !IsReal();
    }
  }
  // b2p_coperator_fused_path: 0 term by term, 1 two real sums, 2 one pass on nd_hex_apply4_kernel, 3 one pass on
  // nd_hex_apply7_kernel
  int FusedPath() const { return cta ? 3 : fused ? 2 : sum_re ? 1 : 0; }

  // operator.cpp:98-134 with A = sum_i c_i A_i: y_r = sum (c^r A x_r - c^i A x_i), y_i = sum (c^i A x_r + c^r A x_i);
  // essential rows as in ComplexParOperator::Mult (rap.cpp:481-517)
  void apply(CCPtr x, CPtr y, bool herm) const
  {
    vec::set(ctx, y.re, n, 0.0);
    vec::set(ctx, y.im, n, 0.0);
    apply_terms(x, y, 1.0, herm);
    if (n_ess > 0)
    {
      if (diag_policy == 1)
      {
        vec::set_sub_from(ctx, y.re, d_ess, n_ess, x.re);
        vec::set_sub_from(ctx, y.im, d_ess, n_ess, x.im);
      }
      else
      {
        vec::set_sub(ctx, y.re, d_ess, n_ess, 0.0);
        vec::set_sub(ctx, y.im, d_ess, n_ess, 0.0);
      }
    }
  }
  // y += alpha * (masked element operators) x: the essential rows of y are not touched
  void apply_terms(CCPtr x, CPtr y, double alpha, bool herm) const
  {
    cudaStream_t s = ctx->stream;
    b2p_op *o0 = terms[0].op;
    if (cta)
    {
      // one pass over the geometry for all terms and both parts; the Hermitian transpose conjugates the coupling (sgn = -1) and,
      // for block sums, reads the transposed blocks
      int rc;
      if (sum_re)
        rc = launch_nd_hex_apply7z(sum_re, B2P_ND_BLOCK, sum_re->lidx_bc, herm ? sum_re->bcoef_t : sum_re->bcoef,
                                   herm ? sum_im->bcoef_t : sum_im->bcoef, fused_imag ? 1 : 0, herm ? -1.0 : 1.0, alpha, x.re, x.im,
                                   y.re, y.im, s);
      else
        rc = launch_nd_hex_apply7z(o0, fused_kind, o0->lidx_bc, zcoef, nullptr, fused_imag ? 1 : 0, herm ? -1.0 : 1.0, alpha, x.re,
                                   x.im, y.re, y.im, s);
      if (rc == B2P_SUCCESS) n_fused_applies++;
    }
    else if (fused && launch_nd_hex_apply4z(o0, fused_kind, o0->lidx_bc, herm ? zcoef_h : zcoef, fused_imag ? 1 : 0, alpha, x.re, x.im, y.re,
                                       y.im, s) == B2P_SUCCESS)
      n_fused_applies++;
    else if (sum_re)
    {
      bool any_re = false, any_im = false;
      for (auto &t : terms)
      {
        any_re = any_re || t.cr != 0.0;
        any_im = any_im || t.ci != 0.0;
      }
      const double si = herm ? -alpha : alpha;
      // Z^H = S_re^T - i S_im^T: the transpose flag matters for block sums only (dense sums are symmetric)
      const int fl = B2P_APPLY_MASKED | (herm ? B2P_APPLY_TRANSPOSE : 0);
      if (any_re)
      {
        b2p_op_apply_add_ex(sum_re, alpha, x.re, y.re, fl, s);
        b2p_op_apply_add_ex(sum_re, alpha, x.im, y.im, fl, s);
      }
      if (any_im)
      {
        b2p_op_apply_add_ex(sum_im, -si, x.im, y.re, fl, s);
        b2p_op_apply_add_ex(sum_im, si, x.re, y.im, fl, s);
      }
      n_fused_applies++;
    }
    else
    for (auto &t : terms)
    {
      const double ci = herm ? -t.ci : t.ci;
      const int fl = B2P_APPLY_MASKED | (herm ? B2P_APPLY_TRANSPOSE : 0);  // (only the non-symmetric kinds look at the flag)
      if (t.cr != 0.0)
      {
        b2p_op_apply_add_ex(t.op, alpha * t.cr, x.re, y.re, fl, s);
        b2p_op_apply_add_ex(t.op, alpha * t.cr, x.im, y.im, fl, s);
      }
      if (ci != 0.0)
      {
        b2p_op_apply_add_ex(t.op, -alpha * ci, x.im, y.re, fl, s);
        b2p_op_apply_add_ex(t.op, alpha * ci, x.re, y.im, fl, s);
      }
    }
  }
  // y += a A x with a real: the element kernels accumulate straight into y; essential rows: (A x)[ess] = x[ess] (DIAG_ONE) or 0
  bool NativeAddMult() const override { return true; }
  void AddMult(CCPtr x, CPtr y, cplx a) const override
  {
    if (a.imag() != 0.0)
    {
      ComplexOperator::AddMult(x, y, a);
      return;
    }
    apply_terms(x, y, a.real(), false);
    if (n_ess > 0 && diag_policy == 1)
    {
      vec::axpy_sub(ctx, a.real(), x.re, d_ess, n_ess, y.re);
      vec::axpy_sub(ctx, a.real(), x.im, d_ess, n_ess, y.im);
    }
  }
  bool IsReal() const override
  {
    for (auto &t : terms)
      if (t.ci != 0.0) return false;
    return true;
  }
  const int32_t *EssentialTrueDofs() const override { return d_ess; }
  int64_t NumEssential() const override { return n_ess; }
  // Full assembly of both parts into vr / vi [nnz] on a pattern built from PatternOp() (b2p_csr_create): from the fused sums
  // S_re and S_im when they exist (dense or block terms: P launches each), else term by term with the real and then the
  // imaginary coefficients. Essential rows as in ComplexParOperator (rap.cpp:481-517): Ar with the operator's diagonal policy,
  // Ai with DIAG_ZERO.
  b2p_op *PatternOp() const { return terms[0].op; }
  bool HasReal() const
  {
    for (auto &t : terms)
      if (t.cr != 0.0) return true;
    return false;
  }
  int AssembleValues(b2p_csr *A, double *vr, double *vi) const
  {
    cudaStream_t s = ctx->stream;
    int rc;
    if (sum_re)
    {
      const double one = 1.0;
      rc = csr_assemble_values(A, 1, &sum_re, &one, vr, s);
      if (!rc) rc = csr_assemble_values(A, 1, &sum_im, &one, vi, s);
    }
    else
    {
      std::vector<b2p_op *> ops;
      std::vector<double> cr, ci;
      for (auto &t : terms)
      {
        ops.push_back(t.op);
        cr.push_back(t.cr);
        ci.push_back(t.ci);
      }
      rc = csr_assemble_values(A, (int)ops.size(), ops.data(), cr.data(), vr, s);
      if (!rc) rc = csr_assemble_values(A, (int)ops.size(), ops.data(), ci.data(), vi, s);
    }
    if (rc || n_ess <= 0) return rc;
    std::vector<int32_t> ess((size_t)n_ess);
    B2P_CUDA(ctx, cudaMemcpyAsync(ess.data(), d_ess, sizeof(int32_t) * n_ess, cudaMemcpyDeviceToHost, s));
    B2P_CUDA(ctx, cudaStreamSynchronize(s));
    rc = csr_eliminate_values(A, ess.data(), n_ess, diag_policy, vr, s);
    if (!rc) rc = csr_eliminate_values(A, ess.data(), n_ess, 0, vi, s);
    return rc;
  }
  void Mult(CCPtr x, CPtr y) const override { apply(x, y, false); }
  void MultHermitianTranspose(CCPtr x, CPtr y) const override { apply(x, y, true); }
  void AssembleDiagonal(CPtr d) const override
  {
    cudaStream_t s = ctx->stream;
    vec::set(ctx, d.re, n, 0.0);
    vec::set(ctx, d.im, n, 0.0);
    if (tmp_.n != 2 * n) tmp_.resize(ctx, 2 * n);
    for (auto &t : terms)
    {
      vec::set(ctx, tmp_.p, n, 0.0);
      b2p_op_diag_add(t.op, tmp_.p, s);
      if (t.cr != 0.0) vec::axpy(ctx, t.cr, tmp_.p, d.re, n);
      if (t.ci != 0.0) vec::axpy(ctx, t.ci, tmp_.p, d.im, n);
    }
    if (n_ess > 0)
    {
      vec::set_sub(ctx, d.re, d_ess, n_ess, diag_policy == 1 ? 1.0 : 0.0);
      vec::set_sub(ctx, d.im, d_ess, n_ess, 0.0);
    }
  }

private:
  std::vector<Term> terms;
  int32_t *d_ess = nullptr;
  // fused complex element operator (build_fused); cta: its applies (or the block sums') run on nd_hex_apply7_kernel<..., CPLX>
  bool fused = false, fused_imag = false, cta = false;
  // the real and imaginary coefficient sums as two operators: dense-basis terms, or hex terms with a mixed curl kind (block sums)
  b2p_op *sum_re = nullptr, *sum_im = nullptr;
  int fused_kind = 0;
  double *zcoef = nullptr, *zcoef_h = nullptr;
  std::vector<std::vector<double>> fused_e18;  // host copies of the terms' per-element material tensors

public:
  mutable long n_fused_applies = 0;
  int64_t n_ess;
  int diag_policy;
};

// ComplexWrapperOperator (linalg/operator.cpp:98-134): A = Ar + i Ai from two REAL true-dof operators, either may be
// absent. This is the form the reference uses everywhere (ComplexParOperator holds two ParOperators, rap.cpp:481-517): the
// parts may live on partitioned spaces (their own halo exchange), be assembled matrices, or anything else behind Operator.
// Essential dofs: give Ar DIAG_ONE and Ai DIAG_ZERO to get the complex DIAG_ONE rows.
class ComplexWrapperOperator : public ComplexOperator
{
  const Operator *Ar, *Ai;

public:
  ComplexWrapperOperator(b2p_ctx *c, const Operator *ar, const Operator *ai) : ComplexOperator(c, (ar ? ar : ai)->Height()), Ar(ar), Ai(ai) {}
  const Operator *Real() const { return Ar; }
  const Operator *Imag() const { return Ai; }
  void apply(CCPtr x, CPtr y, bool herm) const
  {
    const double si = herm ? -1.0 : 1.0;  // A^H = Ar^T - i Ai^T
    if (Ar)
    {
      if (herm)
      {
        Ar->MultTranspose(x.re, y.re);
        Ar->MultTranspose(x.im, y.im);
      }
      else
      {
        Ar->Mult(x.re, y.re);
        Ar->Mult(x.im, y.im);
      }
    }
    else
    {
      vec::set(ctx, y.re, n, 0.0);
      vec::set(ctx, y.im, n, 0.0);
    }
    if (Ai)
    {
      if (herm)
      {
        Ai->AddMultTranspose(x.im, y.re, -si);
        Ai->AddMultTranspose(x.re, y.im, si);
      }
      else
      {
        Ai->AddMult(x.im, y.re, -si);
        Ai->AddMult(x.re, y.im, si);
      }
    }
  }
  bool IsReal() const override { return Ai == nullptr; }
  const int32_t *EssentialTrueDofs() const override
  {
    return (Ar ? Ar : Ai)->EssentialTrueDofs();  // ParOperator and its general-prolongation form report theirs; others none
  }
  int64_t NumEssential() const override
  {
    return (Ar ? Ar : Ai)->NumEssential();
  }
  void Mult(CCPtr x, CPtr y) const override { apply(x, y, false); }
  void MultHermitianTranspose(CCPtr x, CPtr y) const override { apply(x, y, true); }
  void AssembleDiagonal(CPtr d) const override
  {
    if (Ar)
      Ar->AssembleDiagonal(d.re);
    else
      vec::set(ctx, d.re, n, 0.0);
    if (Ai)
      Ai->AssembleDiagonal(d.im);
    else
      vec::set(ctx, d.im, n, 0.0);
  }
};

// ------------------------------------------------------------------------------------ complex solvers
class ComplexSolver
{
public:
  b2p_ctx *ctx;
  bool initial_guess = false;
  ComplexSolver(b2p_ctx *c) : ctx(c) {}
  virtual ~ComplexSolver() = default;
  virtual void Mult(CCPtr x, CPtr y) const = 0;
  virtual bool SetOperator(const ComplexOperator &) { return false; }  // false: this solver takes no operator
  virtual void MultTranspose(CCPtr x, CPtr y) const { Mult(x, y); }  // smoothers of symmetric operators: the same
};

// JacobiSmoother<ComplexOperator> (jacobi.cpp:75-105): y = omega D^-1 x with the COMPLEX assembled diagonal; the smoother and
// simplest preconditioner of the complex-valued (PCMatReal = false, the reference's default) path.
class ComplexJacobiSmoother : public ComplexSolver
{
  double omega;
  mutable DVec dinv;
  int64_t n = 0;

public:
  ComplexJacobiSmoother(b2p_ctx *c, double omega_) : ComplexSolver(c), omega(omega_) {}
  bool SetOperator(const ComplexOperator &op) override
  {
    n = op.n;
    dinv.resize(ctx, 2 * n);
    op.AssembleDiagonal(CPtr{dinv.p, dinv.p + n});
    B2P_LAUNCH(creciprocal_kernel, grid_for(ctx, n), NT, 0, ctx->stream, dinv.p, dinv.p + n, omega, n);
    return true;
  }
  void Mult(CCPtr x, CPtr y) const override
  {
    B2P_LAUNCH(cdiag_mult_kernel, grid_for(ctx, n), NT, 0, ctx->stream, (const double *)dinv.p, (const double *)(dinv.p + n), x.re, x.im,
               y.re, y.im, 1.0, n);
  }
};

// ChebyshevSmoother<ComplexOperator>, 4th kind (chebyshev.cpp:160-220): complex inverse diagonal, lambda_max =
// sf_max * ||D^-1 A||_2 by the reference's power iteration (operator.cpp:583-631; on (D^-1 A)^H (D^-1 A) unless A is real).
class ComplexChebyshevSmoother : public ComplexSolver
{
  int pc_it, order;
  double sf_max;
  const ComplexOperator *A = nullptr;
  int64_t n = 0;
  mutable DVec d, dinv, r_;

  double SpectralNormDinvA(double tol = 1e-4, int max_it = 1000) const
  {
    const bool herm = A->IsReal();
    DVec u(ctx, 2 * n), v(ctx, 2 * n);
    vec::set_random(ctx, u.p, 2 * n, 0);
    double l = cnorm(ctx, CCPtr{u.p, u.p + n}, n), l0 = 0.0;
    vec::scale(ctx, u.p, 2 * n, 1.0 / l);
    int it = 0;
    for (; it < max_it; it++)
    {
      // w = D^-1 A u  (w is u itself in the Hermitian case, else the work vector d)
      const double *ir = dinv.p, *ii = dinv.p + n;
      double *up = u.p, *vp = v.p;
      A->Mult(CCPtr{up, up + n}, CPtr{vp, vp + n});
      double *w = herm ? up : d.p;
      B2P_LAUNCH(cdiag_mult_kernel, grid_for(ctx, n), NT, 0, ctx->stream, ir, ii, (const double *)vp, (const double *)(vp + n), w, w + n, 1.0,
                 n);
      if (!herm)
      {
        // u = (D^-1 A)^H w = A^H (conj(D^-1) w)
        B2P_LAUNCH(cdiag_mult_kernel, grid_for(ctx, n), NT, 0, ctx->stream, ir, ii, (const double *)w, (const double *)(w + n), vp, vp + n,
                   -1.0, n);
        A->MultHermitianTranspose(CCPtr{vp, vp + n}, CPtr{up, up + n});
      }
      l = cnorm(ctx, CCPtr{u.p, u.p + n}, n);
      vec::scale(ctx, u.p, 2 * n, 1.0 / l);
      if (it > 0 && std::abs(l - l0) / l0 < tol) break;
      l0 = l;
    }
    return herm ? l : std::sqrt(l);
  }

public:
  double lambda_max = 0.0;
  ComplexChebyshevSmoother(b2p_ctx *c, int smooth_it, int poly_order, double sf_max_)
    : ComplexSolver(c), pc_it(smooth_it), order(poly_order), sf_max(sf_max_)
  {
  }
  bool SetOperator(const ComplexOperator &op) override
  {
    A = &op;
    n = op.n;
    d.resize(ctx, 2 * n);
    dinv.resize(ctx, 2 * n);
    r_.resize(ctx, 2 * n);
    op.AssembleDiagonal(CPtr{dinv.p, dinv.p + n});
    B2P_LAUNCH(creciprocal_kernel, grid_for(ctx, n), NT, 0, ctx->stream, dinv.p, dinv.p + n, 1.0, n);
    lambda_max = sf_max * SpectralNormDinvA();
    if (!(lambda_max > 0.0)) set_error(ctx, "Encountered zero maximum eigenvalue in Chebyshev smoother!");
    return lambda_max > 0.0;
  }
  // y = y + p(D^-1 A) D^-1 (x - A y), chebyshev.cpp:190-220
  void Mult(CCPtr x, CPtr y) const override
  {
    CPtr r{r_.p, r_.p + n}, dd{d.p, d.p + n};
    const double *ir = dinv.p, *ii = dinv.p + n;
    for (int it = 0; it < pc_it; it++)
    {
      const bool fresh = !(initial_guess || it > 0);
      if (fresh)
      {
        vec::copy(ctx, r.re, x.re, n);
        vec::copy(ctx, r.im, x.im, n);
      }
      else
      {
        A->Residual(x, CCPtr{y.re, y.im}, r);
      }
      B2P_LAUNCH(ccheb_kernel, grid_for(ctx, n), NT, 0, ctx->stream, 0.0, 4.0 / (3.0 * lambda_max), ir, ii, (const double *)r.re,
                 (const double *)r.im, dd.re, dd.im, y.re, y.im, 1, fresh ? 1 : 0, n);
      for (int k = 1; k < order; k++)
      {
        A->AddMult(CCPtr{dd.re, dd.im}, r, cplx(-1.0, 0.0));
        const double sd = (2.0 * k - 1.0) / (2.0 * k + 3.0);
        const double sr = (8.0 * k + 4.0) / ((2.0 * k + 3.0) * lambda_max);
        B2P_LAUNCH(ccheb_kernel, grid_for(ctx, n), NT, 0, ctx->stream, sd, sr, ir, ii, (const double *)r.re, (const double *)r.im, dd.re,
                   dd.im, y.re, y.im, 0, 0, n);
      }
    }
  }
};

// DistRelaxationSmoother<ComplexOperator> (distrelaxation.cpp:39-151): Hiptmair smoothing of the complex ND operator with the
// complex auxiliary (H1) operator; the discrete gradient G is real and acts on both parts.
class ComplexDistRelaxationSmoother : public ComplexSolver
{
  int pc_it;
  const Operator *G;
  const ComplexOperator *A = nullptr, *A_G = nullptr;
  std::unique_ptr<ComplexChebyshevSmoother> B, B_G;
  int64_t n = 0, nG = 0;
  mutable DVec r_, x_G, y_G;

  void Residual(CCPtr x, CPtr y, CPtr r) const { A->Residual(x, CCPtr{y.re, y.im}, r); }
  void AuxCorrection(CCPtr r, CPtr y, bool transpose) const
  {
    CPtr xg{x_G.p, x_G.p + nG}, yg{y_G.p, y_G.p + nG};
    G->MultTranspose(r.re, xg.re);
    G->MultTranspose(r.im, xg.im);
    if (A_G->NumEssential() > 0)
    {
      vec::set_sub(ctx, xg.re, A_G->EssentialTrueDofs(), A_G->NumEssential(), 0.0);
      vec::set_sub(ctx, xg.im, A_G->EssentialTrueDofs(), A_G->NumEssential(), 0.0);
    }
    B_G->initial_guess = false;
    if (transpose)
      B_G->MultTranspose(CCPtr{xg.re, xg.im}, yg);
    else
      B_G->Mult(CCPtr{xg.re, xg.im}, yg);
    G->AddMult(yg.re, y.re, 1.0);
    G->AddMult(yg.im, y.im, 1.0);
  }

public:
  ComplexDistRelaxationSmoother(b2p_ctx *c, const Operator &G_, int smooth_it, int cheby_smooth_it, int cheby_order, double sf_max)
    : ComplexSolver(c), pc_it(smooth_it), G(&G_)
  {
    B = std::make_unique<ComplexChebyshevSmoother>(c, cheby_smooth_it, cheby_order, sf_max);
    B_G = std::make_unique<ComplexChebyshevSmoother>(c, cheby_smooth_it, cheby_order, sf_max);
  }
  bool SetOperators(const ComplexOperator &op, const ComplexOperator &op_G)
  {
    A = &op;
    A_G = &op_G;
    n = op.n;
    nG = op_G.n;
    r_.resize(ctx, 2 * n);
    x_G.resize(ctx, 2 * nG);
    y_G.resize(ctx, 2 * nG);
    return B->SetOperator(op) && B_G->SetOperator(op_G);
  }
  // distrelaxation.cpp:99-119
  void Mult(CCPtr x, CPtr y) const override
  {
    CPtr r{r_.p, r_.p + n};
    for (int it = 0; it < pc_it; it++)
    {
      B->initial_guess = initial_guess || it > 0;
      B->Mult(x, y);
      Residual(x, y, r);
      AuxCorrection(CCPtr{r.re, r.im}, y, false);
    }
  }
  // distrelaxation.cpp:121-151
  void MultTranspose(CCPtr x, CPtr y) const override
  {
    CPtr r{r_.p, r_.p + n};
    for (int it = 0; it < pc_it; it++)
    {
      if (initial_guess || it > 0)
      {
        Residual(x, y, r);
        AuxCorrection(CCPtr{r.re, r.im}, y, true);
      }
      else
      {
        vec::set(ctx, y.re, n, 0.0);
        vec::set(ctx, y.im, n, 0.0);
        AuxCorrection(x, y, true);
      }
      B->initial_guess = true;
      B->MultTranspose(x, y);
    }
  }
};

// GeometricMultigridSolver<ComplexOperator> (gmg.cpp:16-205): complex level operators and smoothers, REAL prolongations and
// discrete gradients applied to both parts.
class ComplexGeometricMultigridSolver : public ComplexSolver
{
public:
  int pc_it;
  std::vector<const Operator *> P;
  std::vector<const ComplexOperator *> A;
  std::vector<std::unique_ptr<ComplexSolver>> B;
  mutable std::vector<DVec> X, Y, R;
  ComplexGeometricMultigridSolver(b2p_ctx *c, std::unique_ptr<ComplexSolver> &&coarse, const std::vector<const Operator *> &P_,
                                  const std::vector<const Operator *> &G, int cycle_it, int smooth_it, int cheby_order, double sf_max)
    : ComplexSolver(c), pc_it(cycle_it), P(P_), A(P_.size() + 1), B(P_.size() + 1), X(P_.size() + 1), Y(P_.size() + 1), R(P_.size() + 1)
  {
    B[0] = std::move(coarse);
    for (size_t l = 1; l < B.size(); l++)
    {
      if (!G.empty())
        B[l] = std::make_unique<ComplexDistRelaxationSmoother>(c, *G[l], smooth_it, 1, cheby_order, sf_max);  // gmg.cpp:45-50
      else
        B[l] = std::make_unique<ComplexChebyshevSmoother>(c, smooth_it, cheby_order, sf_max);  // gmg.cpp:52-63
    }
  }
  // gmg.cpp:66-123
  bool SetOperators(const std::vector<const ComplexOperator *> &A_, const std::vector<const ComplexOperator *> &A_aux)
  {
    bool ok = true;
    for (size_t l = 0; l < A.size(); l++)
    {
      A[l] = A_[l];
      auto *dist = dynamic_cast<ComplexDistRelaxationSmoother *>(B[l].get());
      if (dist)
        ok = ok && !A_aux.empty() && A_aux[l] && dist->SetOperators(*A_[l], *A_aux[l]);
      else
        ok = B[l]->SetOperator(*A_[l]) && ok;
      const int64_t n = A[l]->n;
      if (l + 1 < A.size())  // the finest level works on the caller's vectors (x is only read there, y is the iterate)
      {
        X[l].resize(ctx, 2 * n);
        Y[l].resize(ctx, 2 * n);
      }
      R[l].resize(ctx, 2 * n);
    }
    return ok;
  }
  void Mult(CCPtr x, CPtr y) const override
  {
    const int top = (int)A.size() - 1;
    x_top = x;
    y_top = y;
    for (int it = 0; it < pc_it; it++) VCycle(top, it > 0);
  }

private:
  mutable CCPtr x_top{nullptr, nullptr};
  mutable CPtr y_top{nullptr, nullptr};
  // gmg.cpp:172-205
  void VCycle(int l, bool initial_guess_) const
  {
    const int64_t n = A[l]->n;
    const bool top = l + 1 == (int)A.size();
    const CCPtr x = top ? x_top : CCPtr{X[l].p, X[l].p + n};
    const CPtr y = top ? y_top : CPtr{Y[l].p, Y[l].p + n}, r{R[l].p, R[l].p + n};
    B[l]->initial_guess = initial_guess_;
    if (l == 0)
    {
      B[l]->Mult(x, y);
      return;
    }
    const int64_t nc = A[l - 1]->n;
    CPtr xc{X[l - 1].p, X[l - 1].p + nc}, yc{Y[l - 1].p, Y[l - 1].p + nc};
    B[l]->Mult(x, y);
    A[l]->Residual(x, CCPtr{y.re, y.im}, r);
    P[l - 1]->MultTranspose(r.re, xc.re);
    P[l - 1]->MultTranspose(r.im, xc.im);
    if (A[l - 1]->NumEssential() > 0)
    {
      vec::set_sub(ctx, xc.re, A[l - 1]->EssentialTrueDofs(), A[l - 1]->NumEssential(), 0.0);
      vec::set_sub(ctx, xc.im, A[l - 1]->EssentialTrueDofs(), A[l - 1]->NumEssential(), 0.0);
    }
    VCycle(l - 1, false);
    P[l - 1]->AddMult(yc.re, y.re, 1.0);
    P[l - 1]->AddMult(yc.im, y.im, 1.0);
    B[l]->initial_guess = true;
    B[l]->MultTranspose(x, y);
  }
};

// PCMatReal: the (real) preconditioner acts on real and imaginary parts separately.
class RealPcSolver : public ComplexSolver
{
public:
  RealPcSolver(b2p_ctx *c, const Solver *B_) : ComplexSolver(c), B(B_) {}
  void Mult(CCPtr x, CPtr y) const override
  {
    B->Mult(x.re, y.re);
    B->Mult(x.im, y.im);
  }
  const Solver *B;
};

namespace
{
// The real matrices a complex coarse solver hands its inner solver. Both are non-symmetric in general (Floquet terms, the
// sum Ar + Ai): only Mult and the diagonal are provided.
class CsrValuesOperator : public Operator
{
  b2p_csr *A;
  const double *val;

public:
  CsrValuesOperator(b2p_ctx *c, b2p_csr *a, const double *v) : Operator(c, b2p_csr_rows(a), b2p_csr_rows(a)), A(a), val(v) {}
  void Mult(const double *x, double *y) const override { csr_mult_values(A, val, x, y, ctx->stream); }
  void MultTranspose(const double *, double *) const override { set_error(ctx, "assembled complex coarse matrix: no transpose"); }
  void AssembleDiagonal(double *d) const override { csr_diag_values(A, val, d, ctx->stream); }
  b2p_csr *AssembledMatrix(const double **v) const override
  {
    *v = val;
    return A;
  }
};
class CsrBlock2Operator : public Operator
{
  b2p_csr *A;
  const double *vr, *vi;

public:
  CsrBlock2Operator(b2p_ctx *c, b2p_csr *a, const double *r, const double *i)
    : Operator(c, 2 * b2p_csr_rows(a), 2 * b2p_csr_rows(a)), A(a), vr(r), vi(i)
  {
  }
  void Mult(const double *x, double *y) const override { csr_block2_mult(A, vr, vi, x, y, ctx->stream); }
  void MultTranspose(const double *, double *) const override { set_error(ctx, "assembled complex coarse matrix: no transpose"); }
  void AssembleDiagonal(double *d) const override { csr_block2_diag(A, vr, d, ctx->stream); }
};
}  // namespace

// MfemWrapperSolver<ComplexOperator> (linalg/solver.cpp:33-177) on the device: SetOperator assembles both parts of the complex
// operator on one CSR pattern and hands a REAL matrix to the inner solver (and its preconditioner):
//   * default: Ar + Ai; Mult applies the real solver to the real and the imaginary part separately;
//   * complex_matrix: the 2n block [[Ar, Ai], [Ai, -Ar]] (applied by csr_block2_mult, never formed), solved once for
//     [xr; -xi] with the right-hand side [br; bi].
// A part that is absent (no real / no imaginary coefficient, or a NULL part of a wrapped operator) leaves the other part alone
// as the matrix. The symbolic phase runs once per operator: a later SetOperator with the same operator (new coefficients)
// only re-assembles the values.
class ComplexAssembledSolver : public ComplexSolver
{
  enum Form { NONE, REAL, IMAG, SUM, BLOCK };
  std::unique_ptr<Solver> inner, pc;
  bool complex_matrix;
  const ComplexOperator *src = nullptr;  // the operator whose pattern `csr` holds
  const b2p_op *src_pattern = nullptr;
  b2p_csr *csr = nullptr;
  DVec vr, vi, vsum;
  Form form = NONE;
  std::unique_ptr<Operator> Ac;
  int32_t *d_rp2 = nullptr, *d_col2 = nullptr;  // explicit block matrix (on request)
  DVec v2;
  bool v2_current = false;
  int64_t n = 0;
  mutable DVec X, Y;

  void release_pattern()
  {
    b2p_csr_destroy(csr);
    csr = nullptr;
    cudaFree(d_rp2);
    cudaFree(d_col2);
    d_rp2 = d_col2 = nullptr;
    src = nullptr;
    src_pattern = nullptr;
  }

public:
  ComplexAssembledSolver(b2p_ctx *c, std::unique_ptr<Solver> &&in, std::unique_ptr<Solver> &&p, bool cm)
    : ComplexSolver(c), inner(std::move(in)), pc(std::move(p)), complex_matrix(cm)
  {
  }
  ~ComplexAssembledSolver() override { release_pattern(); }
  bool SetOperator(const ComplexOperator &op) override
  {
    const auto *par = dynamic_cast<const ComplexParOperator *>(&op);
    const auto *wrap = dynamic_cast<const ComplexWrapperOperator *>(&op);
    const ParOperator *pr = nullptr, *pi = nullptr;
    bool has_re, has_im;
    b2p_op *pattern;
    if (par)
    {
      has_re = par->HasReal();
      has_im = !par->IsReal();
      pattern = par->PatternOp();
    }
    else if (wrap)
    {
      pr = dynamic_cast<const ParOperator *>(wrap->Real());
      pi = dynamic_cast<const ParOperator *>(wrap->Imag());
      if ((wrap->Real() && !pr) || (wrap->Imag() && !pi))
      {
        set_error(ctx, "b2p_csolver_assembled: the parts of a wrapped complex operator must be ParOperators (b2p_operator_par) to be assembled");
        return false;
      }
      has_re = pr != nullptr;
      has_im = pi != nullptr;
      pattern = (pr ? pr : pi)->PatternOp();
      if (pr && pi)
      {
        const b2p_op *a = pr->PatternOp(), *b = pi->PatternOp();
        bool same = a->ne == b->ne && a->P == b->P && a->PS == b->PS && a->lsize == b->lsize;
        if (same && a->lidx != b->lidx)
        {
          std::vector<int32_t> ha((size_t)a->ne * a->PS), hb(ha.size());
          same = cudaMemcpy(ha.data(), a->lidx, ha.size() * sizeof(int32_t), cudaMemcpyDeviceToHost) == cudaSuccess &&
                 cudaMemcpy(hb.data(), b->lidx, hb.size() * sizeof(int32_t), cudaMemcpyDeviceToHost) == cudaSuccess && ha == hb;
        }
        if (!same)
        {
          set_error(ctx, "b2p_csolver_assembled: the real and imaginary parts live on different spaces");
          return false;
        }
      }
    }
    else
    {
      set_error(ctx, "b2p_csolver_assembled must be able to assemble its operator: b2p_coperator_par, or b2p_coperator_wrap of b2p_operator_par parts");
      return false;
    }
    if (!has_re && !has_im)
    {
      set_error(ctx, "Empty ComplexOperator for b2p_csolver_assembled!");
      return false;
    }
    if (src != &op || src_pattern != pattern || !csr)
    {
      release_pattern();
      if (b2p_csr_create(ctx, pattern, &csr) != B2P_SUCCESS) return false;
      src = &op;
      src_pattern = pattern;
    }
    const int64_t nnz = b2p_csr_nnz(csr);
    if (vr.n != nnz) vr.resize(ctx, std::max<int64_t>(nnz, 1));
    if (vi.n != nnz) vi.resize(ctx, std::max<int64_t>(nnz, 1));
    int rc = B2P_SUCCESS;
    if (par)
      rc = par->AssembleValues(csr, vr.p, vi.p);
    else
    {
      if (pr) rc = pr->AssembleValues(csr, vr.p);
      if (!rc && pi) rc = pi->AssembleValues(csr, vi.p);
    }
    if (rc)
    {
      release_pattern();
      form = NONE;
      Ac.reset();
      return false;
    }
    n = b2p_csr_rows(csr);
    if (has_re && has_im && complex_matrix)
    {
      form = BLOCK;
      Ac = std::make_unique<CsrBlock2Operator>(ctx, csr, vr.p, vi.p);
    }
    else if (has_re && has_im)
    {
      form = SUM;
      if (vsum.n != vr.n) vsum.resize(ctx, vr.n);
      vec::axpbypcz(ctx, 1.0, vr.p, 1.0, vi.p, 0.0, vsum.p, nnz);
      Ac = std::make_unique<CsrValuesOperator>(ctx, csr, vsum.p);
    }
    else
    {
      form = has_re ? REAL : IMAG;
      Ac = std::make_unique<CsrValuesOperator>(ctx, csr, has_re ? vr.p : vi.p);
    }
    v2_current = false;
    if (pc) pc->SetOperator(*Ac);
    inner->SetOperator(*Ac);
    return inner->Status() == B2P_SUCCESS;
  }
  void Mult(CCPtr x, CPtr y) const override
  {
    if (form == NONE)
    {
      set_error(ctx, "b2p_csolver_assembled: applied without an assembled operator");
      return;
    }
    inner->SetInitialGuess(initial_guess);
    if (form != BLOCK)
    {
      inner->Mult(x.re, y.re);
      inner->Mult(x.im, y.im);
      return;
    }
    // A [yr; -yi] = [xr; xi]  (solver.cpp:158-176)
    if (X.n != 2 * n) X.resize(ctx, 2 * n);
    if (Y.n != 2 * n) Y.resize(ctx, 2 * n);
    vec::copy(ctx, X.p, x.re, n);
    vec::copy(ctx, X.p + n, x.im, n);
    if (initial_guess)
    {
      vec::copy(ctx, Y.p, y.re, n);
      vec::axpby(ctx, -1.0, y.im, 0.0, Y.p + n, n);
    }
    inner->Mult(X.p, Y.p);
    vec::copy(ctx, y.re, Y.p, n);
    vec::axpby(ctx, -1.0, Y.p + n, 0.0, y.im, n);
  }
  // entries of the real matrix the inner solver sees (4 nnz for the block form)
  int64_t Nnz() const { return form == NONE ? -1 : (form == BLOCK ? 4 : 1) * b2p_csr_nnz(csr); }
  // CSR arrays of that matrix (device, owned here); the block form is built on the first request and refilled after a new
  // assembly.
  int DeviceArrays(int64_t *rows, int64_t *nnz, const int32_t **rowptr, const int32_t **col, const double **val)
  {
    B2P_CHECK(ctx, form != NONE, B2P_ERR_ARG, "b2p_csolver_assembled_device_arrays before set_operator");
    const int32_t *rp, *cl;
    const double *v = nullptr;
    if (form == BLOCK)
    {
      if (!d_rp2)
      {
        int rc = csr_block2_pattern(csr, &d_rp2, &d_col2);
        if (rc) return rc;
      }
      if (v2.n != 4 * b2p_csr_nnz(csr)) v2.resize(ctx, std::max<int64_t>(4 * b2p_csr_nnz(csr), 1));
      if (!v2_current)
      {
        int rc = csr_block2_fill(csr, vr.p, vi.p, v2.p, ctx->stream);
        if (rc) return rc;
        v2_current = true;
      }
      rp = d_rp2;
      cl = d_col2;
      v = v2.p;
    }
    else
    {
      b2p_csr_device_arrays(csr, &rp, &cl, nullptr);
      v = form == SUM ? vsum.p : (form == REAL ? vr.p : vi.p);
    }
    if (rows) *rows = (form == BLOCK ? 2 : 1) * n;
    if (nnz) *nnz = Nnz();
    if (rowptr) *rowptr = rp;
    if (col) *col = cl;
    if (val) *val = v;
    return B2P_SUCCESS;
  }
};

namespace
{
inline void ApplyPlaneRotation(cplx &dx, cplx &dy, const double cs, const cplx sn)
{
  const cplx t = cs * dx + sn * dy;
  dy = -std::conj(sn) * dx + cs * dy;
  dx = t;
}
}  // namespace

class ComplexIterativeSolver : public ComplexSolver
{
public:
  ComplexIterativeSolver(b2p_ctx *c, KspType type_) : ComplexSolver(c), type(type_) {}
  KspType type;
  const ComplexOperator *A = nullptr;
  bool SetOperator(const ComplexOperator &op) override
  {
    A = &op;
    return true;
  }
  const ComplexSolver *B = nullptr;
  double rel_tol = 1e-6, abs_tol = 0.0;
  int max_it = 100, max_dim = -1;
  Orthog gs = Orthog::MGS;
  PcSide pc_side = PcSide::RIGHT;
  mutable bool converged = false;
  mutable double initial_res = 1.0, final_res = 0.0;
  mutable int final_it = 0;

  void Mult(CCPtr b, CPtr x) const override
  {
    if (type == KspType::CG)
      MultCG(b, x);
    else
      MultGMRES(b, x, type == KspType::FGMRES);
  }

private:
  mutable std::vector<std::unique_ptr<DVec>> V, Z;
  mutable DVec r_, z_, p_;
  CPtr cp(DVec &v, int64_t n) const
  {
    if (v.n != 2 * n) v.resize(ctx, 2 * n);
    return CPtr{v.p, v.p + n};
  }
  static CCPtr cc(CPtr p) { return CCPtr{p.re, p.im}; }
  void ccopy(CPtr y, CCPtr x, int64_t n) const
  {
    vec::copy(ctx, y.re, x.re, n);
    vec::copy(ctx, y.im, x.im, n);
  }
  void czero(CPtr y, int64_t n) const
  {
    vec::set(ctx, y.re, n, 0.0);
    vec::set(ctx, y.im, n, 0.0);
  }
  // r = b - r
  void residual(CCPtr b, CPtr r, int64_t n) const
  {
    vec::axpby(ctx, 1.0, b.re, -1.0, r.re, n);
    vec::axpby(ctx, 1.0, b.im, -1.0, r.im, n);
  }

  // iterative.cpp:361-486 with complex scalars
  void MultCG(CCPtr b, CPtr x) const
  {
    const int64_t n = A->n;
    CPtr r = cp(r_, n), z = cp(z_, n), p = cp(p_, n);
    cplx beta, beta_prev = 0.0, alpha, denom;
    double res, eps;
    if (initial_guess)
    {
      A->Mult(cc(x), r);
      residual(b, r, n);
    }
    else
    {
      ccopy(r, b, n);
      czero(x, n);
    }
    if (B)
      B->Mult(cc(r), z);
    else
      ccopy(z, cc(r), n);
    beta = cdot(ctx, cc(z), cc(r), n);
    res = std::sqrt(std::abs(beta));
    if (initial_guess)
    {
      cplx beta_rhs;
      if (B)
      {
        B->Mult(b, p);
        beta_rhs = cdot(ctx, cc(p), b, n);
      }
      else
        beta_rhs = cnorm(ctx, b, n);
      initial_res = std::sqrt(std::abs(beta_rhs));
    }
    else
      initial_res = res;
    eps = std::max(rel_tol * initial_res, abs_tol);
    converged = (res < eps) || res == 0.0;  // a zero residual (zero right-hand side: the imaginary part under PCMatReal) is converged, not 0 / 0
    int it = 0;
    for (; it < max_it && !converged; it++)
    {
      if (!it)
        ccopy(p, cc(z), n);
      else
      {
        // p = z + (beta / beta_prev) p
        const cplx g = beta / beta_prev;
        if (tmp_.n != 2 * n) tmp_.resize(ctx, 2 * n);
        CPtr t{tmp_.p, tmp_.p + n};
        ccopy(t, cc(z), n);
        caxpy(ctx, g, cc(p), t, n);
        ccopy(p, cc(t), n);
      }
      A->Mult(cc(p), z);
      denom = cdot(ctx, cc(z), cc(p), n);
      alpha = beta / denom;
      caxpy(ctx, alpha, cc(p), x, n);
      caxpy(ctx, -alpha, cc(z), r, n);
      beta_prev = beta;
      if (B)
        B->Mult(cc(r), z);
      else
        ccopy(z, cc(r), n);
      beta = cdot(ctx, cc(z), cc(r), n);
      res = std::sqrt(std::abs(beta));
      converged = (res < eps);
    }
    final_res = res;
    final_it = it;
  }

  // iterative.cpp:544-705 / :734-871 with complex scalars
  void MultGMRES(CCPtr b, CPtr x, bool flexible) const
  {
    const int64_t n = A->n;
    const int mdim = (max_dim < 0) ? max_it : max_dim;
    CPtr r = cp(r_, n);
    auto ensure = [&](std::vector<std::unique_ptr<DVec>> &W, int k)
    {
      if ((int)W.size() <= k) W.resize(k + 1);
      if (!W[k]) W[k] = std::make_unique<DVec>(ctx, 2 * n);
      if (W[k]->n != 2 * n) W[k]->resize(ctx, 2 * n);
      return CPtr{W[k]->p, W[k]->p + n};
    };
    std::vector<cplx> H((size_t)(mdim + 1) * mdim, 0.0), s(mdim + 1, 0.0), sn(mdim + 1, 0.0);
    std::vector<double> cs(mdim + 1, 0.0);
    const bool right = flexible || pc_side == PcSide::RIGHT;
    double beta = 0.0, true_beta, eps = 0.0;
    converged = false;
    int it = 0, restart = 0;
    for (; it < max_it; restart++)
    {
      CPtr V0 = ensure(V, 0);
      CPtr rv = flexible ? ensure(Z, 0) : r;
      const bool ig = initial_guess || restart > 0;
      if (B && !right)
      {
        if (ig)
        {
          A->Mult(cc(x), V0);
          residual(b, V0, n);
          B->Mult(cc(V0), rv);
        }
        else
        {
          B->Mult(b, rv);
          czero(x, n);
        }
      }
      else
      {
        if (ig)
        {
          A->Mult(cc(x), rv);
          residual(b, rv, n);
        }
        else
        {
          ccopy(rv, b, n);
          czero(x, n);
        }
      }
      true_beta = cnorm(ctx, cc(rv), n);
      if (it == 0)
      {
        if (initial_guess)
        {
          if (B && !right)
          {
            B->Mult(b, V0);
            initial_res = cnorm(ctx, cc(V0), n);
          }
          else
            initial_res = cnorm(ctx, b, n);
        }
        else
          initial_res = true_beta;
        eps = std::max(rel_tol * initial_res, abs_tol);
      }
      beta = true_beta;
      if (beta < eps || beta == 0.0)  // (a zero residual is converged: 1 / beta below)
      {
        converged = true;
        break;
      }
      vec::axpby(ctx, 1.0 / beta, rv.re, 0.0, V0.re, n);
      vec::axpby(ctx, 1.0 / beta, rv.im, 0.0, V0.im, n);
      std::fill(s.begin(), s.end(), cplx(0.0));
      s[0] = beta;
      int j = 0;
      for (;; j++, it++)
      {
        CPtr Vj = ensure(V, j), w = ensure(V, j + 1);
        if (B && !right)
        {
          A->Mult(cc(Vj), r);
          B->Mult(cc(r), w);
        }
        else if (B)
        {
          CPtr zj = flexible ? ensure(Z, j) : r;
          B->Mult(cc(Vj), zj);
          A->Mult(cc(zj), w);
        }
        else
          A->Mult(cc(Vj), w);
        cplx *Hj = H.data() + (size_t)j * (mdim + 1);
        std::vector<CCPtr> Vp(j + 1);
        for (int k = 0; k <= j; k++) Vp[k] = CCPtr{V[k]->p, V[k]->p + n};
        if (gs == Orthog::MGS)
        {
          for (int k = 0; k <= j; k++)
          {
            Hj[k] = cdot(ctx, cc(w), Vp[k], n);
            caxpy(ctx, -Hj[k], Vp[k], w, n);
          }
        }
        else
        {
          cmulti_dot(ctx, j + 1, Vp.data(), cc(w), n, Hj);
          cmulti_axpy(ctx, j + 1, Hj, Vp.data(), w, n, -1.0);
          if (gs == Orthog::CGS2)
          {
            std::vector<cplx> dH(j + 1);
            cmulti_dot(ctx, j + 1, Vp.data(), cc(w), n, dH.data());
            cmulti_axpy(ctx, j + 1, dH.data(), Vp.data(), w, n, -1.0);
            for (int k = 0; k <= j; k++) Hj[k] += dH[k];
          }
        }
        const double hn = cnorm(ctx, cc(w), n);
        Hj[j + 1] = hn;
        vec::scale(ctx, w.re, n, 1.0 / hn);
        vec::scale(ctx, w.im, n, 1.0 / hn);
        for (int k = 0; k < j; k++) ApplyPlaneRotation(Hj[k], Hj[k + 1], cs[k], sn[k]);
        GeneratePlaneRotation(Hj[j], Hj[j + 1], cs[j], sn[j]);
        ApplyPlaneRotation(Hj[j], Hj[j + 1], cs[j], sn[j]);
        ApplyPlaneRotation(s[j], s[j + 1], cs[j], sn[j]);
        beta = std::abs(s[j + 1]);
        converged = (beta < eps);
        if (converged || j + 1 == mdim || it + 1 == max_it)
        {
          it++;
          break;
        }
      }
      for (int i = j; i >= 0; i--)
      {
        cplx *Hi = H.data() + (size_t)i * (mdim + 1);
        s[i] /= Hi[i];
        for (int k = i - 1; k >= 0; k--) s[k] -= Hi[k] * s[i];
      }
      std::vector<CCPtr> W(j + 1);
      if (flexible)
      {
        for (int k = 0; k <= j; k++) W[k] = CCPtr{Z[k]->p, Z[k]->p + n};
        cmulti_axpy(ctx, j + 1, s.data(), W.data(), x, n, 1.0);
      }
      else
      {
        for (int k = 0; k <= j; k++) W[k] = CCPtr{V[k]->p, V[k]->p + n};
        if (!B || !right)
          cmulti_axpy(ctx, j + 1, s.data(), W.data(), x, n, 1.0);
        else
        {
          czero(r, n);
          cmulti_axpy(ctx, j + 1, s.data(), W.data(), r, n, 1.0);
          CPtr V0b = ensure(V, 0);
          B->Mult(cc(r), V0b);
          caxpy(ctx, 1.0, cc(V0b), x, n);
        }
      }
      if (converged) break;
    }
    final_res = beta;
    final_it = it;
  }
  mutable DVec tmp_;
};

}  // namespace b2p

using namespace b2p;

struct b2p_operator;
struct b2p_solver;
namespace b2p
{
Solver *solver_of(b2p_solver *s);
std::unique_ptr<Solver> take_solver(b2p_solver *s);
Operator *operator_of(b2p_operator *A);
}

struct b2p_coperator
{
  std::unique_ptr<ComplexOperator> op;
};
struct b2p_csolver
{
  std::unique_ptr<ComplexSolver> s;
};

#define B2P_CTRY(ctx, stmt)                                      \
  do                                                             \
  {                                                              \
    stmt;                                                        \
    cudaError_t e__ = cudaPeekAtLastError();                     \
    if (e__ != cudaSuccess)                                      \
    {                                                            \
      set_error(ctx, "CUDA error: %s", cudaGetErrorString(e__)); \
      return B2P_ERR_CUDA;                                       \
    }                                                            \
  } while (0)

extern "C"
{

int b2p_vec_cdot(b2p_ctx *ctx, int64_t n, const double *xr, const double *xi, const double *yr, const double *yi, double out[2])
{
  cplx d;
  B2P_CTRY(ctx, d = cdot(ctx, CCPtr{xr, xi}, CCPtr{yr, yi}, n));
  out[0] = d.real();
  out[1] = d.imag();
  return B2P_SUCCESS;
}
int b2p_vec_caxpy(b2p_ctx *ctx, int64_t n, double ar, double ai, const double *xr, const double *xi, double *yr, double *yi)
{
  B2P_CTRY(ctx, caxpy(ctx, cplx(ar, ai), CCPtr{xr, xi}, CPtr{yr, yi}, n));
  return B2P_SUCCESS;
}

int b2p_coperator_wrap(b2p_ctx *ctx, b2p_operator *Ar, b2p_operator *Ai, b2p_coperator **out)
{
  B2P_CHECK(ctx, ctx && out && (Ar || Ai), B2P_ERR_ARG, "b2p_coperator_wrap: Empty ComplexOperator");
  const Operator *ar = operator_of(Ar), *ai = operator_of(Ai);
  B2P_CHECK(ctx, !ar || !ai || (ar->Height() == ai->Height() && ar->Width() == ai->Width()), B2P_ERR_ARG,
            "b2p_coperator_wrap: mismatch in dimension of real and imaginary matrix parts");
  B2P_CHECK(ctx, (ar ? ar : ai)->Height() == (ar ? ar : ai)->Width(), B2P_ERR_ARG, "b2p_coperator_wrap: square operators only");
  auto *h = new b2p_coperator;
  h->op = std::make_unique<ComplexWrapperOperator>(ctx, ar, ai);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_coperator_par(b2p_ctx *ctx, int64_t tsize, int64_t lsize, int n_terms, b2p_op *const *ops, const double *coef_re,
                      const double *coef_im, const int32_t *ess_tdofs, int64_t n_ess, int diag_policy, b2p_coperator **out)
{
  B2P_CHECK(ctx, ctx && out && n_terms > 0 && ops && coef_re && coef_im, B2P_ERR_ARG, "b2p_coperator_par: bad argument");
  B2P_CHECK(ctx, tsize == lsize, B2P_ERR_UNSUPPORTED, "b2p_coperator_par: single partition only; on partitioned spaces wrap two b2p_operator_par with b2p_coperator_wrap");
  std::vector<ComplexParOperator::Term> terms;
  for (int i = 0; i < n_terms; i++)
  {
    B2P_CHECK(ctx, ops[i] && b2p_op_lsize(ops[i]) == lsize, B2P_ERR_ARG, "b2p_coperator_par: term %d has the wrong L-size", i);
    B2P_CHECK(ctx, ops[i]->kind != B2P_RT_MASS, B2P_ERR_UNSUPPORTED,
              "b2p_coperator_par: term %d is a Raviart-Thomas operator; complex sums of them are not supported", i);
    B2P_CHECK(ctx, !ops[i]->lidx_bc || op_essential_matches(ops[i], ess_tdofs, n_ess), B2P_ERR_ARG,
              "b2p_coperator_par: term %d already carries a different essential-dof mask (one b2p_op = one essential set)", i);
    terms.push_back({ops[i], coef_re[i], coef_im[i]});
  }
  auto *h = new b2p_coperator;
  h->op = std::make_unique<ComplexParOperator>(ctx, tsize, terms, ess_tdofs, n_ess, diag_policy);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_coperator_mult(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi)
{
  if (!A) return B2P_ERR_ARG;
  B2P_CTRY(A->op->ctx, A->op->Mult(CCPtr{xr, xi}, CPtr{yr, yi}));
  return B2P_SUCCESS;
}
int b2p_coperator_mult_hermitian_transpose(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi)
{
  if (!A) return B2P_ERR_ARG;
  B2P_CTRY(A->op->ctx, A->op->MultHermitianTranspose(CCPtr{xr, xi}, CPtr{yr, yi}));
  return B2P_SUCCESS;
}
int b2p_coperator_add_mult(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi, double ar, double ai)
{
  if (!A) return B2P_ERR_ARG;
  B2P_CTRY(A->op->ctx, A->op->AddMult(CCPtr{xr, xi}, CPtr{yr, yi}, cplx(ar, ai)));
  return B2P_SUCCESS;
}
int b2p_coperator_assemble_diagonal(b2p_coperator *A, double *dr, double *di)
{
  if (!A) return B2P_ERR_ARG;
  B2P_CTRY(A->op->ctx, A->op->AssembleDiagonal(CPtr{dr, di}));
  return B2P_SUCCESS;
}
int b2p_coperator_set_coefficients(b2p_coperator *A, int n_terms, const double *coef_re, const double *coef_im)
{
  auto *p = A ? dynamic_cast<ComplexParOperator *>(A->op.get()) : nullptr;
  if (!p || !coef_re || !coef_im || n_terms != (int)p->NumTerms()) return B2P_ERR_ARG;
  p->SetCoefficients(coef_re, coef_im);
  return B2P_SUCCESS;
}
long b2p_coperator_fused_applies(b2p_coperator *A)
{
  auto *p = A ? dynamic_cast<ComplexParOperator *>(A->op.get()) : nullptr;
  return p ? p->n_fused_applies : -1;
}
int b2p_coperator_fused_path(b2p_coperator *A)
{
  auto *p = A ? dynamic_cast<ComplexParOperator *>(A->op.get()) : nullptr;
  return p ? p->FusedPath() : -1;
}
void b2p_coperator_destroy(b2p_coperator *A) { delete A; }

int b2p_csolver_real_pc(b2p_ctx *ctx, b2p_solver *real_pc, b2p_csolver **out)
{
  B2P_CHECK(ctx, ctx && real_pc && out, B2P_ERR_ARG, "b2p_csolver_real_pc: bad argument");
  auto *h = new b2p_csolver;
  h->s = std::make_unique<RealPcSolver>(ctx, solver_of(real_pc));
  *out = h;
  return B2P_SUCCESS;
}
int b2p_csolver_assembled(b2p_ctx *ctx, b2p_solver *inner, b2p_solver *inner_pc, int complex_matrix, b2p_csolver **out)
{
  B2P_CHECK(ctx, ctx && inner && solver_of(inner) && out, B2P_ERR_ARG, "b2p_csolver_assembled: bad argument");
  auto *k = dynamic_cast<IterativeSolver *>(solver_of(inner));
  if (inner_pc)
  {
    B2P_CHECK(ctx, solver_of(inner_pc) && k, B2P_ERR_ARG, "b2p_csolver_assembled: a preconditioner needs a Krylov inner solver");
    k->SetPreconditioner(solver_of(inner_pc));
  }
  auto *h = new b2p_csolver;
  h->s = std::make_unique<ComplexAssembledSolver>(ctx, take_solver(inner), take_solver(inner_pc), complex_matrix != 0);
  *out = h;
  return B2P_SUCCESS;
}
// the assembled solver itself, or the one a complex multigrid took over as its coarse solver
static ComplexAssembledSolver *assembled_of(b2p_csolver *s)
{
  ComplexSolver *p = s ? s->s.get() : nullptr;
  if (auto *g = dynamic_cast<ComplexGeometricMultigridSolver *>(p)) p = g->B[0].get();
  return dynamic_cast<ComplexAssembledSolver *>(p);
}
int64_t b2p_csolver_assembled_nnz(b2p_csolver *s)
{
  auto *a = assembled_of(s);
  return a ? a->Nnz() : -1;
}
int b2p_csolver_assembled_device_arrays(b2p_csolver *s, int64_t *rows, int64_t *nnz, const int32_t **rowptr, const int32_t **col,
                                        const double **val)
{
  auto *a = assembled_of(s);
  if (!a) return B2P_ERR_ARG;
  return a->DeviceArrays(rows, nnz, rowptr, col, val);
}
int b2p_csolver_jacobi(b2p_ctx *ctx, double omega, b2p_csolver **out)
{
  B2P_CHECK(ctx, ctx && out, B2P_ERR_ARG, "b2p_csolver_jacobi: bad argument");
  B2P_CHECK(ctx, omega != 0.0, B2P_ERR_UNSUPPORTED, "b2p_csolver_jacobi: give the damping factor (the estimated optimum, omega == 0, is not built)");
  auto *h = new b2p_csolver;
  h->s = std::make_unique<ComplexJacobiSmoother>(ctx, omega);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_csolver_chebyshev(b2p_ctx *ctx, int smooth_it, int order, double sf_max, b2p_csolver **out)
{
  B2P_CHECK(ctx, ctx && out && smooth_it > 0, B2P_ERR_ARG, "b2p_csolver_chebyshev: bad argument");
  B2P_CHECK(ctx, order > 0, B2P_ERR_ARG, "Polynomial order for Chebyshev smoothing must be positive!");
  auto *h = new b2p_csolver;
  h->s = std::make_unique<ComplexChebyshevSmoother>(ctx, smooth_it, order, sf_max);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_csolver_lambda_max(b2p_csolver *s, double *out)
{
  auto *c = s ? dynamic_cast<ComplexChebyshevSmoother *>(s->s.get()) : nullptr;
  if (!c || !out) return B2P_ERR_ARG;
  *out = c->lambda_max;
  return B2P_SUCCESS;
}
int b2p_csolver_gmg(b2p_ctx *ctx, b2p_csolver *coarse, int n_levels, b2p_operator *const *P, b2p_operator *const *G, int cycle_it,
                    int smooth_it, int cheby_order, double sf_max, b2p_csolver **out)
{
  B2P_CHECK(ctx, ctx && coarse && coarse->s && n_levels >= 1 && out && (n_levels == 1 || P), B2P_ERR_ARG, "b2p_csolver_gmg: bad argument");
  std::vector<const Operator *> Pv, Gv;
  for (int l = 0; l + 1 < n_levels; l++) Pv.push_back(operator_of(P[l]));
  if (G)
    for (int l = 0; l < n_levels; l++) Gv.push_back(G[l] ? operator_of(G[l]) : nullptr);
  auto *h = new b2p_csolver;
  h->s = std::make_unique<ComplexGeometricMultigridSolver>(ctx, std::move(coarse->s), Pv, Gv, cycle_it, smooth_it, cheby_order, sf_max);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_csolver_gmg_set_operators(b2p_csolver *s, b2p_coperator *const *A, b2p_coperator *const *A_aux)
{
  auto *g = s ? dynamic_cast<ComplexGeometricMultigridSolver *>(s->s.get()) : nullptr;
  if (!g || !A) return B2P_ERR_ARG;
  std::vector<const ComplexOperator *> Av, Gv;
  for (size_t l = 0; l < g->A.size(); l++)
  {
    B2P_CHECK(g->ctx, A[l], B2P_ERR_ARG, "b2p_csolver_gmg_set_operators: level %d has no operator", (int)l);
    Av.push_back(A[l]->op.get());
    if (A_aux) Gv.push_back(A_aux[l] ? A_aux[l]->op.get() : nullptr);
  }
  bool ok = false;
  B2P_CTRY(g->ctx, ok = g->SetOperators(Av, Gv));
  return ok ? B2P_SUCCESS : B2P_ERR_ARG;
}
int b2p_csolver_krylov(b2p_ctx *ctx, int type, b2p_csolver **out)
{
  B2P_CHECK(ctx, type >= 0 && type <= 2 && out, B2P_ERR_ARG, "b2p_csolver_krylov: type must be 0 (CG), 1 (GMRES) or 2 (FGMRES)");
  auto *h = new b2p_csolver;
  h->s = std::make_unique<ComplexIterativeSolver>(ctx, (KspType)type);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_csolver_krylov_config(b2p_csolver *s, double rel_tol, double abs_tol, int max_it, int max_dim, int orthog, int pc_side)
{
  auto *k = s ? dynamic_cast<ComplexIterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  k->rel_tol = rel_tol;
  k->abs_tol = abs_tol;
  k->max_it = max_it;
  k->max_dim = max_dim;
  k->gs = (Orthog)orthog;
  k->pc_side = (PcSide)pc_side;
  return B2P_SUCCESS;
}
int b2p_csolver_set_operator(b2p_csolver *s, b2p_coperator *A)
{
  if (!s || !s->s || !A) return B2P_ERR_ARG;
  if (auto *k = dynamic_cast<ComplexIterativeSolver *>(s->s.get()))
  {
    k->A = A->op.get();
    return B2P_SUCCESS;
  }
  b2p_ctx *ctx = s->s->ctx;
  bool ok = false;
  B2P_CTRY(ctx, ok = s->s->SetOperator(*A->op));
  return ok ? B2P_SUCCESS : B2P_ERR_ARG;
}
int b2p_csolver_set_preconditioner(b2p_csolver *s, b2p_csolver *pc)
{
  auto *k = s ? dynamic_cast<ComplexIterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  k->B = pc ? pc->s.get() : nullptr;
  return B2P_SUCCESS;
}
int b2p_csolver_set_initial_guess(b2p_csolver *s, int flag)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  s->s->initial_guess = flag != 0;
  return B2P_SUCCESS;
}
int b2p_csolver_mult(b2p_csolver *s, const double *br, const double *bi, double *xr, double *xi)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  if (auto *k = dynamic_cast<ComplexIterativeSolver *>(s->s.get()))
    B2P_CHECK(k->ctx, k->A && (k->type != KspType::FGMRES || k->B), B2P_ERR_ARG,
              "Operator and preconditioner must be set for FgmresSolver::Mult (operator for the others)!");  // iterative.cpp:738
  B2P_CTRY(s->s->ctx, s->s->Mult(CCPtr{br, bi}, CPtr{xr, xi}));
  return B2P_SUCCESS;
}
int b2p_csolver_stats(b2p_csolver *s, int *its, double *initial_res, double *final_res, int *converged)
{
  auto *k = s ? dynamic_cast<ComplexIterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  if (its) *its = k->final_it;
  if (initial_res) *initial_res = k->initial_res;
  if (final_res) *final_res = k->final_res;
  if (converged) *converged = k->converged ? 1 : 0;
  return B2P_SUCCESS;
}
void b2p_csolver_destroy(b2p_csolver *s) { delete s; }

}  // extern "C"

// ---- outer eigen-solver interface (ArpackEPSSolver::ApplyOp / ApplyOpB, arpack.cpp:631-674) ----
namespace b2p
{
namespace eps_detail
{
// interleaved complex (the host layout, staged in z[2n]) <-> split real / imaginary device vectors
__global__ void csplit_kernel(const double *__restrict__ z, double *__restrict__ re, double *__restrict__ im, int64_t n)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    re[i] = z[2 * i];
    im[i] = z[2 * i + 1];
  }
}
__global__ void cjoin_scaled_kernel(const double *__restrict__ re, const double *__restrict__ im, double s, double *__restrict__ z, int64_t n)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    z[2 * i] = s * re[i];
    z[2 * i + 1] = s * im[i];
  }
}
}  // namespace eps_detail
}  // namespace b2p

struct b2p_eps
{
  b2p_ctx *ctx = nullptr;
  int64_t n = 0;
  const ComplexOperator *K = nullptr, *M = nullptr, *B = nullptr;
  const ComplexSolver *opInv = nullptr;
  bool sinvert = true;
  double gamma = 1.0, delta = 1.0;
  DVec xr, xi, zr, zi, yr, yi, stage;  // x1, z1, y1 of the reference + the interleaved staging vector
  double *h_pin = nullptr;             // pinned host staging [2n]
};

static int eps_run(b2p_eps *e, const double *px, double *py, bool op_b)
{
  using namespace b2p::eps_detail;
  b2p_ctx *ctx = e->ctx;
  cudaStream_t s = ctx->stream;
  const int64_t n = e->n;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8);
  std::memcpy(e->h_pin, px, sizeof(double) * 2 * n);  // x1.Set(px, n): the caller's buffer need not be pinned
  B2P_CUDA(ctx, cudaMemcpyAsync(e->stage.p, e->h_pin, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, s));
  B2P_LAUNCH(csplit_kernel, grid, 256, 0, s, (const double *)e->stage.p, e->xr.p, e->xi.p, n);
  double scale;
  if (op_b)
  {
    B2P_CTRY(ctx, e->B->Mult(CCPtr{e->xr.p, e->xi.p}, CPtr{e->yr.p, e->yi.p}));
    scale = e->delta;
  }
  else
  {
    const ComplexOperator *first = e->sinvert ? e->M : e->K;  // y = gamma opInv (M x)  |  y = opInv (K x) / gamma
    B2P_CTRY(ctx, first->Mult(CCPtr{e->xr.p, e->xi.p}, CPtr{e->zr.p, e->zi.p}));
    B2P_CTRY(ctx, e->opInv->Mult(CCPtr{e->zr.p, e->zi.p}, CPtr{e->yr.p, e->yi.p}));
    scale = e->sinvert ? e->gamma : 1.0 / e->gamma;
  }
  B2P_LAUNCH(cjoin_scaled_kernel, grid, 256, 0, s, (const double *)e->yr.p, (const double *)e->yi.p, scale, e->stage.p, n);
  B2P_CUDA(ctx, cudaMemcpyAsync(e->h_pin, e->stage.p, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, s));
  B2P_CUDA(ctx, cudaStreamSynchronize(s));
  std::memcpy(py, e->h_pin, sizeof(double) * 2 * n);  // y1.Get(py, n)
  return B2P_SUCCESS;
}

extern "C"
{

int b2p_eps_create(b2p_ctx *ctx, int64_t n, b2p_coperator *K, b2p_coperator *M, b2p_csolver *opInv, b2p_coperator *B, int sinvert,
                   double gamma, double delta, b2p_eps **out)
{
  B2P_CHECK(ctx, ctx && out && n > 0 && opInv && opInv->s, B2P_ERR_ARG, "b2p_eps_create: bad argument");
  B2P_CHECK(ctx, sinvert ? (M && M->op) : (K && K->op), B2P_ERR_ARG,
            "b2p_eps_create: shift-and-invert applies M first, the untransformed problem K");
  B2P_CHECK(ctx, gamma != 0.0, B2P_ERR_ARG, "b2p_eps_create: gamma = 0");
  auto e = std::make_unique<b2p_eps>();
  e->ctx = ctx;
  e->n = n;
  e->K = K ? K->op.get() : nullptr;
  e->M = M ? M->op.get() : nullptr;
  e->B = B ? B->op.get() : nullptr;
  e->opInv = opInv->s.get();
  e->sinvert = sinvert != 0;
  e->gamma = gamma;
  e->delta = delta;
  for (DVec *v : {&e->xr, &e->xi, &e->zr, &e->zi, &e->yr, &e->yi}) v->resize(ctx, n);
  e->stage.resize(ctx, 2 * n);
  B2P_CUDA(ctx, cudaMallocHost((void **)&e->h_pin, sizeof(double) * 2 * n));
  *out = e.release();
  return B2P_SUCCESS;
}
int b2p_eps_apply_op(b2p_eps *e, const double *x, double *y)
{
  if (!e || !x || !y) return B2P_ERR_ARG;
  return eps_run(e, x, y, false);
}
int b2p_eps_apply_op_b(b2p_eps *e, const double *x, double *y)
{
  if (!e || !x || !y) return B2P_ERR_ARG;
  B2P_CHECK(e->ctx, e->B, B2P_ERR_ARG, "No B operator for weighted inner product in the eigen-solver interface!");
  return eps_run(e, x, y, true);
}
void b2p_eps_destroy(b2p_eps *e)
{
  if (!e) return;
  cudaFreeHost(e->h_pin);
  delete e;
}

}  // extern "C"
