// Flux error estimator for H(curl) problems: FluxProjector + element-wise error integration
//   /root/reference/palace/linalg/errorestimator.cpp:112-175 (FluxProjector), :180-270 (ComputeErrorEstimates),
//   :400-505 (CurlFluxErrorEstimator: discontinuous flux mu^-1 B, B = curl E in the RT space; smooth flux H in the ND space).
//
//   rhs = Flux B            Flux = (mu^-1 u_RT, v_ND): VectorFEMassIntegrator between an H(div) trial and an H(curl) test space,
//                           quadrature function f_apply_hdivhcurl_33 (qfunctions/33/hcurlhdiv_33_qf.h:33-55):
//                           v^ = w detJ (J^-T)^T C (J / detJ) u^
//   M H = rhs               M = ND mass (VectorFEMassIntegrator without coefficient); PCG, Jacobi with the damping from the
//                           eigenvalue estimate (errorestimator.cpp:69-75), no initial guess, abs tol epsilon (:100-106)
//   eta_K^2 = int_K | C_2 (J^-T H^) - C_1 (J B^ / detJ) |^2       f_apply_hdivhcurl_error_33
//                           (qfunctions/33/hcurlhdiv_error_33_qf.h:46-76), C_1 = sqrt(mu^-1), C_2 = (mu^-1)^(-1/2), summed
//                           over the quadrature points of each element (the all-ones "mesh element basis",
//                           libceed/integrator.cpp:560-574); complex fields add both parts before the square root
//   eta_K <- sqrt(s eta_K^2), s = 0.5 / Et or 1 (errorestimator.cpp:506-513)
//
// The two spaces are described the way libCEED sees non-tensor bases (fem/libceed/basis.cpp:40-85): a dense table
// interp[3][Q][P] of reference-space values at the quadrature points and a signed element restriction. These operators run
// once per solve (post-processing): one CTA per element, dense contractions; they are not on the hot path and make no
// roofline claim.
#include <algorithm>
#include <cmath>
#include <initializer_list>
#include <memory>
#include <utility>
#include <vector>

#include "b2p_linalg.hpp"
#include "b2p_qf.cuh"

struct b2p_operator;
namespace b2p
{
Operator *operator_of(b2p_operator *A);
b2p_operator *wrap_operator(std::unique_ptr<Operator> &&op);
IterativeSolver *ksp_solver_of(b2p_ksp *k);
}

namespace b2p
{
namespace
{

constexpr int FLUX_NT = 128;

struct VecFESpace
{
  int P = 0, map = 0;
  int64_t lsize = 0;
  double *interp = nullptr;  // device [3][Q][P]
  int32_t *sidx = nullptr;   // device [ne][P], sign folded in: >= 0 -> +x[i], < 0 -> -x[-1 - i]
  // device [ne][P][3] row-major tridiagonal element transformation (ND tetrahedra / prisms of order >= 2, restriction.cpp:301-329)
  // or null; with it sidx holds plain indices and x_e = T_e x[idx_e]
  int8_t *co = nullptr;
};

__device__ __forceinline__ double gather_signed(const double *x, int32_t gi) { return gi >= 0 ? x[gi] : -x[-1 - gi]; }

// physical value of a reference-space vector: H(curl): J^-T u^ (A = adjJ^T / detJ), H(div): J u^ / detJ (the cofactor of A)
__device__ __forceinline__ void piola_matrix(int map, const double A[9], double M[9])
{
  if (map == B2P_MAP_HCURL)
  {
#pragma unroll
    for (int i = 0; i < 9; i++) M[i] = A[i];
  }
  else
    cofactor33(A, M);
}

// x_e of element e in shared memory (all threads of the block; ends with a barrier): signs folded into the index, or the tridiagonal
// transformation applied to the raw values (tmp: P doubles of scratch, used only then)
__device__ void load_element_vector(const VecFESpace &sp, int e, const double *__restrict__ x, double *xe, double *tmp)
{
  if (!sp.co)
  {
    for (int j = threadIdx.x; j < sp.P; j += blockDim.x) xe[j] = gather_signed(x, sp.sidx[(size_t)e * sp.P + j]);
    __syncthreads();
    return;
  }
  for (int j = threadIdx.x; j < sp.P; j += blockDim.x) tmp[j] = x[sp.sidx[(size_t)e * sp.P + j]];
  __syncthreads();
  const int8_t *co = sp.co + (size_t)e * sp.P * 3;
  for (int i = threadIdx.x; i < sp.P; i += blockDim.x)
  {
    double v = (double)co[3 * i + 1] * tmp[i];
    if (i > 0) v += (double)co[3 * i] * tmp[i - 1];
    if (i < sp.P - 1) v += (double)co[3 * i + 2] * tmp[i + 1];
    xe[i] = v;
  }
  __syncthreads();
}
// entry j of T_e^T s (s in shared memory)
__device__ __forceinline__ double transposed_entry(const VecFESpace &sp, int e, const double *s, int j)
{
  const int8_t *co = sp.co + (size_t)e * sp.P * 3;
  double v = (double)co[3 * j + 1] * s[j];
  if (j > 0) v += (double)co[3 * (j - 1) + 2] * s[j - 1];
  if (j < sp.P - 1) v += (double)co[3 * (j + 1)] * s[j + 1];
  return v;
}
// value of table row `row` for the j-th GLOBAL-side shape function of element e: column j, or the combination T_e(., j) of columns
__device__ __forceinline__ double transformed_column(const VecFESpace &sp, int e, const double *row, int j)
{
  if (!sp.co) return row[j];
  const int8_t *co = sp.co + (size_t)e * sp.P * 3;
  double v = (double)co[3 * j + 1] * row[j];
  if (j > 0) v += (double)co[3 * (j - 1) + 2] * row[j - 1];
  if (j < sp.P - 1) v += (double)co[3 * (j + 1)] * row[j + 1];
  return v;
}

// values of space `sp` at the quadrature points of element e: u[c * Q + q] = sum_j interp[c][q][j] xe[j]
__device__ void eval_at_points(int Q, int P, const double *__restrict__ interp, const double *xe, double *u)
{
  for (int w = threadIdx.x; w < 3 * Q; w += blockDim.x)
  {
    const double *row = interp + (size_t)w * P;
    double s = 0.0;
    for (int j = 0; j < P; j++) s += row[j] * xe[j];
    u[w] = s;
  }
}

// y_test += E_test^T B_test^T D B_trial E_trial x, D = w detJ P_test^T C P_trial at every point
__global__ void mixed_mass_kernel(int ne, int Q, int q1d, VecFESpace trial, VecFESpace test, const double *__restrict__ qd,
                                  const double *__restrict__ coef, const double *__restrict__ x, double *y)
{
  B2P_DYN_SMEM(double, sm);
  const int PM = max(trial.P, test.P);
  double *xe = sm, *u = sm + PM, *tmp = u + 3 * Q;  // tmp [PM]: raw values / element result of transformed restrictions
  const int e = blockIdx.x;
  if (e >= ne) return;
  load_element_vector(trial, e, x, xe, tmp);
  eval_at_points(Q, trial.P, trial.interp, xe, u);
  __syncthreads();
  const double *C = coef + (size_t)e * 9;
  for (int q = threadIdx.x; q < Q; q += blockDim.x)
  {
    const int slot = q1d > 0 ? qslot_of(q1d, q) : q;  // tensor geometries store their q-data x-slowest
    const double *g = qd + (size_t)e * 10 * Q + slot;
    double A[9], M1[9], M2[9], Cm[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      Cm[i] = C[i];
    }
    piola_matrix(trial.map, A, M1);
    piola_matrix(test.map, A, M2);
    const double uu[3] = {u[q], u[Q + q], u[2 * Q + q]};
    double t[3], z[3], v[3];
    Ax33(M1, uu, t);
    Ax33(Cm, t, z);
    Atx33(M2, z, g[0], v);
    u[q] = v[0];
    u[Q + q] = v[1];
    u[2 * Q + q] = v[2];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < test.P; i += blockDim.x)
  {
    double s = 0.0;
    for (int w = 0; w < 3 * Q; w++) s += test.interp[(size_t)w * test.P + i] * u[w];
    if (test.co)
      tmp[i] = s;
    else
    {
      const int32_t gi = test.sidx[(size_t)e * test.P + i];
      atomicAdd(y + (gi >= 0 ? gi : -1 - gi), gi >= 0 ? s : -s);
    }
  }
  if (test.co)
  {
    __syncthreads();
    for (int j = threadIdx.x; j < test.P; j += blockDim.x) atomicAdd(y + test.sidx[(size_t)e * test.P + j], transposed_entry(test, e, tmp, j));
  }
}

// est[e] += sum_q w detJ | C2 P2 u2 - C1 P1 u1 |^2
__global__ void flux_error_kernel(int ne, int Q, int q1d, VecFESpace s1, VecFESpace s2, const double *__restrict__ qd,
                                  const double *__restrict__ coef1, const double *__restrict__ coef2, const double *__restrict__ x1,
                                  const double *__restrict__ x2, double *est)
{
  B2P_DYN_SMEM(double, sm);
  double *xe1 = sm, *xe2 = xe1 + s1.P, *u1 = xe2 + s2.P, *u2 = u1 + 3 * Q, *red = u2 + 3 * Q, *tmp = red + FLUX_NT;  // tmp [max P]
  const int e = blockIdx.x;
  if (e >= ne) return;
  load_element_vector(s1, e, x1, xe1, tmp);
  load_element_vector(s2, e, x2, xe2, tmp);
  eval_at_points(Q, s1.P, s1.interp, xe1, u1);
  eval_at_points(Q, s2.P, s2.interp, xe2, u2);
  __syncthreads();
  double acc = 0.0;
  for (int q = threadIdx.x; q < Q; q += blockDim.x)
  {
    const int slot = q1d > 0 ? qslot_of(q1d, q) : q;
    const double *g = qd + (size_t)e * 10 * Q + slot;
    double A[9], M1[9], M2[9], C1[9], C2[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C1[i] = coef1[(size_t)e * 9 + i];
      C2[i] = coef2[(size_t)e * 9 + i];
    }
    piola_matrix(s1.map, A, M1);
    piola_matrix(s2.map, A, M2);
    const double a[3] = {u1[q], u1[Q + q], u1[2 * Q + q]}, b[3] = {u2[q], u2[Q + q], u2[2 * Q + q]};
    double t[3], v1[3], v2[3];
    Ax33(M1, a, t);
    Ax33(C1, t, v1);
    Ax33(M2, b, t);
    Ax33(C2, t, v2);
    const double d0 = v2[0] - v1[0], d1 = v2[1] - v1[1], d2 = v2[2] - v1[2];
    acc += g[0] * (d0 * d0 + d1 * d1 + d2 * d2);
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0)  // fixed summation order: the estimate does not depend on the schedule
  {
    double s = 0.0;
    for (int i = 0; i < (int)blockDim.x; i++) s += red[i];
    est[e] += s;
  }
}

__global__ void sqrt_scale_kernel(int64_t n, double s, double *est)
{
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) est[i] = sqrt(s * est[i]);
}

// Flux: the partially assembled mixed mass operator between the two spaces (single partition: T-vectors are L-vectors)
class MixedMassOperator : public Operator
{
public:
  MixedMassOperator(b2p_ctx *c, const b2p_geom *g, const VecFESpace &trial_, const VecFESpace &test_, const double *d_coef_)
    : Operator(c, test_.lsize, trial_.lsize), geom(g), trial(trial_), test(test_), d_coef(d_coef_)
  {
  }
  void Mult(const double *x, double *y) const override
  {
    vec::set(ctx, y, height, 0.0);
    const size_t shmem = (size_t)(2 * std::max(trial.P, test.P) + 3 * geom->Q) * sizeof(double);
    if (shmem > 48 * 1024) cudaFuncSetAttribute(mixed_mass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem);
    B2P_LAUNCH(mixed_mass_kernel, geom->ne, FLUX_NT, shmem, ctx->stream, geom->ne, geom->Q, geom->q1d, trial, test,
               (const double *)geom->qd, d_coef, x, y);
  }
  const b2p_geom *geom;
  VecFESpace trial, test;
  const double *d_coef;
};

// Flux of an estimator on hexahedra (b2p_flux_estimator_create_hex): the sum-factorised mixed mass of b2p_hex_flux.cu
class HexMixedMassOperator : public Operator
{
public:
  HexMixedMassOperator(b2p_ctx *c, int64_t h, int64_t w, const HexFluxArgs &a_) : Operator(c, h, w), a(a_) {}
  void Mult(const double *x, double *y) const override
  {
    vec::set(ctx, y, height, 0.0);
    rc = launch_hex_flux_mixed(a, x, y, ctx->stream);
  }
  HexFluxArgs a;
  mutable int rc = B2P_SUCCESS;
};

// diag[|i|] += sum_q phi_i^T D phi_i (the signs of the restriction cancel)
__global__ void vecfe_mass_diag_kernel(int ne, int Q, int q1d, VecFESpace sp, const double *__restrict__ qd, const double *__restrict__ coef,
                                       double *diag)
{
  const int e = blockIdx.x;
  if (e >= ne) return;
  const double *C = coef + (size_t)e * 9;
  for (int i = threadIdx.x; i < sp.P; i += blockDim.x)
  {
    double s = 0.0;
    for (int q = 0; q < Q; q++)
    {
      const int slot = q1d > 0 ? qslot_of(q1d, q) : q;
      const double *g = qd + (size_t)e * 10 * Q + slot;
      double A[9], M[9], Cm[9];
#pragma unroll
      for (int k = 0; k < 9; k++)
      {
        A[k] = g[(1 + k) * Q];
        Cm[k] = C[k];
      }
      piola_matrix(sp.map, A, M);
      const double u[3] = {transformed_column(sp, e, sp.interp + (size_t)(0 * Q + q) * sp.P, i),
                           transformed_column(sp, e, sp.interp + (size_t)(1 * Q + q) * sp.P, i),
                           transformed_column(sp, e, sp.interp + (size_t)(2 * Q + q) * sp.P, i)};
      double t[3], z[3];
      Ax33(M, u, t);
      Ax33(Cm, t, z);
      s += g[0] * (t[0] * z[0] + t[1] * z[1] + t[2] * z[2]);
    }
    const int32_t gi = sp.sidx[(size_t)e * sp.P + i];
    atomicAdd(diag + (gi >= 0 ? gi : -1 - gi), s);
  }
}

// VectorFEMassIntegrator on ONE table-described space (the mass matrix of a FluxProjector's smooth space when that space has no
// sum-factorised operator in this library, e.g. Raviart-Thomas); owns its device arrays
class VecFEMassOperator : public MixedMassOperator
{
public:
  VecFEMassOperator(b2p_ctx *c, b2p_geom *g, const VecFESpace &sp, double *d_coef_owned)
    : MixedMassOperator(c, g, sp, sp, d_coef_owned), owned_geom(g), owned_coef(d_coef_owned)
  {
    g->refcount++;
  }
  ~VecFEMassOperator() override
  {
    cudaFree(trial.interp);
    cudaFree(trial.sidx);
    cudaFree(trial.co);
    cudaFree(owned_coef);
    b2p_geom_destroy(owned_geom);
  }
  void AssembleDiagonal(double *d) const override
  {
    vec::set(ctx, d, height, 0.0);
    B2P_LAUNCH(vecfe_mass_diag_kernel, geom->ne, FLUX_NT, 0, ctx->stream, geom->ne, geom->Q, geom->q1d, trial, (const double *)geom->qd,
               d_coef, d);
  }
  b2p_geom *owned_geom;
  double *owned_coef;
};

// per-element 3x3 blocks [ne][9] from a per-attribute table (identity without one)
int expand_coef(b2p_ctx *ctx, const b2p_geom *geom, int n_attr, const double *coef, std::vector<double> &c)
{
  const int ne = geom->ne;
  c.assign((size_t)ne * 9, 0.0);
  if (!coef)
    for (int el = 0; el < ne; el++) c[(size_t)el * 9] = c[(size_t)el * 9 + 4] = c[(size_t)el * 9 + 8] = 1.0;
  else
  {
    std::vector<int32_t> attr(ne);
    B2P_CUDA(ctx, cudaMemcpy(attr.data(), geom->attr, sizeof(int32_t) * ne, cudaMemcpyDeviceToHost));
    for (int el = 0; el < ne; el++)
    {
      const int a = attr[el] - 1;  // attributes are 1-based
      B2P_CHECK(ctx, a >= 0 && a < n_attr, B2P_ERR_ARG, "element %d has attribute %d outside 1..%d", el, a + 1, n_attr);
      for (int i = 0; i < 9; i++) c[(size_t)el * 9 + i] = coef[(size_t)a * 9 + i];
    }
  }
  return B2P_SUCCESS;
}

int upload_coef(b2p_ctx *ctx, const b2p_geom *geom, int n_attr, const double *coef, double **out)
{
  std::vector<double> c;
  int rc = expand_coef(ctx, geom, n_attr, coef, c);
  return rc ? rc : upload(ctx, c.data(), c.size(), out);
}

// per-element coefficient blocks of the hexahedral kernels: [ne][stride], the k-th table's 3x3 at offset 9 k, zero padding
int upload_coef_blocks(b2p_ctx *ctx, const b2p_geom *geom, int n_attr, std::initializer_list<const double *> coefs, int stride, double **out)
{
  const int ne = geom->ne;
  std::vector<double> blk((size_t)ne * stride, 0.0), c;
  int k = 0, rc;
  for (const double *coef : coefs)
  {
    if ((rc = expand_coef(ctx, geom, n_attr, coef, c))) return rc;
    for (int el = 0; el < ne; el++)
      for (int i = 0; i < 9; i++) blk[(size_t)el * stride + 9 * k + i] = c[(size_t)el * 9 + i];
    k++;
  }
  return upload(ctx, blk.data(), blk.size(), out);
}

int upload_space(b2p_ctx *ctx, const b2p_vecfe_space_desc *d, int ne, int Q, VecFESpace *out)
{
  B2P_CHECK(ctx, d && d->P > 0 && d->interp && d->idx && d->lsize > 0, B2P_ERR_ARG, "b2p_flux_estimator_create: incomplete space description");
  B2P_CHECK(ctx, d->map_type == B2P_MAP_HCURL || d->map_type == B2P_MAP_HDIV, B2P_ERR_ARG,
            "b2p_flux_estimator_create: map type %d is neither H(curl) nor H(div)", d->map_type);
  out->P = d->P;
  out->map = d->map_type;
  out->lsize = d->lsize;
  std::vector<int32_t> s((size_t)ne * d->P);
  for (size_t i = 0; i < s.size(); i++)
  {
    const int32_t g = d->idx[i];
    B2P_CHECK(ctx, g >= 0 && g < d->lsize, B2P_ERR_ARG, "b2p_flux_estimator_create: restriction index %d outside [0, %lld)", (int)g,
              (long long)d->lsize);
    s[i] = (!d->curl_orient && d->orient && d->orient[i] < 0) ? -1 - g : g;  // (the tridiagonal rows carry the signs themselves)
  }
  int rc = upload(ctx, s.data(), s.size(), &out->sidx);
  if (rc) return rc;
  if (d->curl_orient && (rc = upload(ctx, d->curl_orient, (size_t)ne * d->P * 3, &out->co))) return rc;
  return upload(ctx, d->interp, (size_t)3 * Q * d->P, &out->interp);
}

}  // namespace
}  // namespace b2p

using namespace b2p;

struct b2p_flux_estimator
{
  b2p_ctx *ctx = nullptr;
  b2p_geom *geom = nullptr;
  VecFESpace flux, smooth;
  double *d_coef_flux = nullptr, *d_coef_disc = nullptr, *d_coef_smooth = nullptr;
  std::unique_ptr<Operator> Flux;
  // b2p_flux_estimator_create_hex: sum-factorised spaces (flux = space a, smooth = space b of both argument sets)
  bool hex = false;
  HexFluxArgs hex_err;
  std::vector<double> h_tab;
  double *d_tab = nullptr, *d_hex_coef_flux = nullptr, *d_hex_coef_err = nullptr;
  int32_t *hex_lidx[2] = {nullptr, nullptr};
  const Operator *M = nullptr;
  std::unique_ptr<JacobiSmoother> pc;
  std::unique_ptr<IterativeSolver> pcg;
  b2p_ksp *mg = nullptr;                 // b2p_flux_estimator_set_multigrid: PCG with the geometric multigrid preconditioner
  IterativeSolver *solver = nullptr;     // the projection's solver: pcg, or the one inside mg
  DVec rhs, H;
  int mult = 0, mult_it = 0;
  ~b2p_flux_estimator()
  {
    b2p_ksp_destroy(mg);
    cudaFree(flux.interp);
    cudaFree(flux.sidx);
    cudaFree(flux.co);
    cudaFree(smooth.interp);
    cudaFree(smooth.sidx);
    cudaFree(smooth.co);
    cudaFree(d_coef_flux);
    cudaFree(d_coef_disc);
    cudaFree(d_coef_smooth);
    cudaFree(d_tab);
    cudaFree(d_hex_coef_flux);
    cudaFree(d_hex_coef_err);
    cudaFree(hex_lidx[0]);
    cudaFree(hex_lidx[1]);
    if (geom) b2p_geom_destroy(geom);  // (drops this handle's reference)
  }
};

namespace
{
// ConfigureLinearSolver(use_mg = false) (errorestimator.cpp:63-109), then hand the estimator out
int finish_estimator(std::unique_ptr<b2p_flux_estimator> &e, const Operator *M, double tol, int max_it, const char *who,
                     b2p_flux_estimator **out)
{
  b2p_ctx *ctx = e->ctx;
  e->M = M;
  e->pc = std::make_unique<JacobiSmoother>(ctx, 0.0, 1.0);
  e->pc->SetOperator(*M);
  e->pcg = std::make_unique<IterativeSolver>(ctx, KspType::CG);
  e->pcg->SetInitialGuess(false);
  e->pcg->rel_tol = tol;
  e->pcg->abs_tol = 2.220446049250313e-16;
  e->pcg->max_it = max_it;
  e->pcg->SetOperator(*M);
  e->pcg->SetPreconditioner(e->pc.get());
  e->solver = e->pcg.get();
  cudaError_t err = cudaPeekAtLastError();
  B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "%s: %s", who, cudaGetErrorString(err));
  *out = e.release();
  return B2P_SUCCESS;
}

// restriction and space fields of one validated hexahedral space description (slot 0 = flux, 1 = smooth)
int hex_space(b2p_flux_estimator *e, const b2p_op_desc *d, int slot, const char *role)
{
  b2p_ctx *ctx = e->ctx;
  const char *W = "b2p_flux_estimator_create_hex";
  const int ne = e->geom->ne, p = d->p;
  const int P = d->kind == B2P_ND_MASS ? 3 * p * (p + 1) * (p + 1) : 3 * (p + 1) * p * p;
  char who[96];
  snprintf(who, sizeof(who), "%s: %s space: ", W, role);
  int PS = 0;
  int rc = build_lex_restriction(ctx, who, d, P, d->lsize, ne, &PS, &e->hex_lidx[slot]);
  if (rc) return rc;
  VecFESpace &sp = slot == 0 ? e->flux : e->smooth;
  sp.P = P;
  sp.map = d->kind == B2P_ND_MASS ? B2P_MAP_HCURL : B2P_MAP_HDIV;
  sp.lsize = d->lsize;
  HexFluxArgs &a = e->hex_err;
  (slot == 0 ? a.lidx_a : a.lidx_b) = e->hex_lidx[slot];
  (slot == 0 ? a.PS_a : a.PS_b) = PS;
  return B2P_SUCCESS;
}
}  // namespace

extern "C"
{

int b2p_operator_vecfe_mass(b2p_ctx *ctx, b2p_geom *geom, const b2p_vecfe_space_desc *space, int n_attr, const double *coef,
                            b2p_operator **out)
{
  B2P_CHECK(ctx, ctx && geom && space && out && (!coef || n_attr > 0), B2P_ERR_ARG, "b2p_operator_vecfe_mass: bad argument");
  B2P_CHECK(ctx, ctx->nranks == 1, B2P_ERR_UNSUPPORTED, "b2p_operator_vecfe_mass: partitioned spaces are not supported yet");
  VecFESpace sp;
  int rc = upload_space(ctx, space, geom->ne, geom->Q, &sp);
  if (rc) return rc;
  double *d_coef = nullptr;
  if ((rc = upload_coef(ctx, geom, n_attr, coef, &d_coef))) return rc;
  *out = wrap_operator(std::make_unique<VecFEMassOperator>(ctx, geom, sp, d_coef));
  return B2P_SUCCESS;
}

// estimates[i] = sqrt(s * estimates[i]): the last step of the estimators that add several flux terms before the square root
// (TimeDependentFluxErrorEstimator, errorestimator.cpp:531-545)
int b2p_flux_estimator_sqrt_scale(b2p_ctx *ctx, int64_t n, double s, double *estimates)
{
  if (!ctx || !estimates || n < 0) return B2P_ERR_ARG;
  if (n == 0) return B2P_SUCCESS;
  B2P_LAUNCH(sqrt_scale_kernel, (unsigned)((n + 255) / 256), 256, 0, ctx->stream, n, s, estimates);
  cudaError_t err = cudaPeekAtLastError();
  B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "b2p_flux_estimator_sqrt_scale: %s", cudaGetErrorString(err));
  return B2P_SUCCESS;
}

int b2p_flux_estimator_create(b2p_ctx *ctx, b2p_geom *geom, const b2p_vecfe_space_desc *flux_space,
                              const b2p_vecfe_space_desc *smooth_space, int n_attr, const double *coef_flux, const double *coef_disc,
                              const double *coef_smooth, b2p_operator *smooth_mass, double tol, int max_it, b2p_flux_estimator **out)
{
  B2P_CHECK(ctx, ctx && geom && out && n_attr > 0 && coef_flux && coef_disc && coef_smooth && smooth_mass, B2P_ERR_ARG,
            "b2p_flux_estimator_create: bad argument");
  Operator *M = operator_of(smooth_mass);
  B2P_CHECK(ctx, M && smooth_space && M->Height() == smooth_space->lsize && M->Width() == smooth_space->lsize, B2P_ERR_ARG,
            "b2p_flux_estimator_create: the mass operator of the smooth space has the wrong size");
  B2P_CHECK(ctx, ctx->nranks == 1, B2P_ERR_UNSUPPORTED,
            "b2p_flux_estimator_create: partitioned spaces are not supported yet (T-vectors are taken as L-vectors)");
  auto e = std::make_unique<b2p_flux_estimator>();
  e->ctx = ctx;
  geom->refcount++;
  e->geom = geom;
  const int ne = geom->ne, Q = geom->Q;
  int rc;
  if ((rc = upload_space(ctx, flux_space, ne, Q, &e->flux))) return rc;
  if ((rc = upload_space(ctx, smooth_space, ne, Q, &e->smooth))) return rc;
  // per-element coefficient matrices from the per-attribute tables (coeff/coeff_qf.h: attribute -> material -> matrix)
  if ((rc = upload_coef(ctx, geom, n_attr, coef_flux, &e->d_coef_flux))) return rc;
  if ((rc = upload_coef(ctx, geom, n_attr, coef_disc, &e->d_coef_disc))) return rc;
  if ((rc = upload_coef(ctx, geom, n_attr, coef_smooth, &e->d_coef_smooth))) return rc;
  e->Flux = std::make_unique<MixedMassOperator>(ctx, geom, e->flux, e->smooth, e->d_coef_flux);
  return finish_estimator(e, M, tol, max_it, "b2p_flux_estimator_create", out);
}

int b2p_flux_estimator_create_hex(b2p_ctx *ctx, b2p_geom *geom, const b2p_op_desc *flux_space, const b2p_op_desc *smooth_space, int n_attr,
                                  const double *coef_flux, const double *coef_disc, const double *coef_smooth, b2p_operator *smooth_mass,
                                  double tol, int max_it, b2p_flux_estimator **out)
{
  const char *W = "b2p_flux_estimator_create_hex";
  B2P_CHECK(ctx, ctx && geom && flux_space && smooth_space && out && n_attr > 0 && coef_flux && coef_disc && coef_smooth && smooth_mass,
            B2P_ERR_ARG, "%s: bad argument", W);
  B2P_CHECK(ctx, ctx->nranks == 1, B2P_ERR_UNSUPPORTED, "%s: partitioned spaces are not supported yet (T-vectors are taken as L-vectors)",
            W);
  // what the descriptions are, before what they ask for
  for (const auto &[d, role] : {std::pair{flux_space, "flux"}, std::pair{smooth_space, "smooth"}})
    B2P_CHECK(ctx, d->kind == B2P_ND_MASS || d->kind == B2P_RT_MASS, B2P_ERR_ARG,
              "%s: the %s space has kind %d; a space is B2P_ND_MASS (Nedelec) or B2P_RT_MASS (Raviart-Thomas)", W, role, d->kind);
  B2P_CHECK(ctx, flux_space->kind != smooth_space->kind, B2P_ERR_ARG, "%s: both spaces are %s; one Nedelec and one Raviart-Thomas space "
            "are needed", W, flux_space->kind == B2P_ND_MASS ? "Nedelec" : "Raviart-Thomas");
  B2P_CHECK(ctx, geom->q1d > 0, B2P_ERR_ARG, "%s: the geometry has no tensor q-data (q1d = 0); use b2p_flux_estimator_create", W);
  const int p = flux_space->p, q1d = geom->q1d, ne = geom->ne;
  B2P_CHECK(ctx, smooth_space->p == p, B2P_ERR_ARG, "%s: the flux space has p=%d and the smooth space p=%d; both must be the same", W, p,
            smooth_space->p);
  for (const auto &[d, role] : {std::pair{flux_space, "flux"}, std::pair{smooth_space, "smooth"}})
  {
    B2P_CHECK(ctx, d->ne == ne, B2P_ERR_ARG, "%s: the %s space has %d elements vs %d in the geometry", W, role, d->ne, ne);
    B2P_CHECK(ctx, d->idx && d->lsize > 0 && d->Bo && d->Bc, B2P_ERR_ARG, "%s: the %s space lacks its restriction or its Bo / Bc tables", W,
              role);
  }
  Operator *M = operator_of(smooth_mass);
  B2P_CHECK(ctx, M && M->Height() == smooth_space->lsize && M->Width() == smooth_space->lsize, B2P_ERR_ARG,
            "%s: the mass operator of the smooth space has the wrong size", W);
  for (const auto &[d, role] : {std::pair{flux_space, "flux"}, std::pair{smooth_space, "smooth"}})
    B2P_CHECK(ctx, !d->assemble_qdata, B2P_ERR_UNSUPPORTED, "%s: assembled q-data is not available for the %s space (the flux kernels "
              "apply their coefficients on the fly)", W, role);
  B2P_CHECK(ctx, p >= 1 && p <= 6 && p < q1d && q1d <= 7, B2P_ERR_UNSUPPORTED,
            "%s: unsupported p=%d q1d=%d (hex kernels cover p<=6, p<q1d<=7)", W, p, q1d);
  // both spaces are evaluated with one pair of 1-D tables: the smooth space's must be the flux space's
  {
    const size_t nBo = (size_t)q1d * p, nBc = (size_t)q1d * (p + 1);
    double scale = 0.0, diff = 0.0;
    for (size_t i = 0; i < nBo; i++)
    {
      scale = std::max(scale, std::fabs(flux_space->Bo[i]));
      diff = std::max(diff, std::fabs(flux_space->Bo[i] - smooth_space->Bo[i]));
    }
    for (size_t i = 0; i < nBc; i++)
    {
      scale = std::max(scale, std::fabs(flux_space->Bc[i]));
      diff = std::max(diff, std::fabs(flux_space->Bc[i] - smooth_space->Bc[i]));
    }
    B2P_CHECK(ctx, diff <= 1e-14 * scale, B2P_ERR_ARG,
              "%s: the smooth space's Bo / Bc tables differ from the flux space's by %.3e; both spaces need the same 1-D tables", W, diff);
  }
  auto e = std::make_unique<b2p_flux_estimator>();
  e->ctx = ctx;
  geom->refcount++;
  e->geom = geom;
  e->hex = true;
  int rc;
  if ((rc = hex_space(e.get(), flux_space, 0, "flux")) || (rc = hex_space(e.get(), smooth_space, 1, "smooth"))) return rc;
  // the 1-D tables (the same for both spaces, checked above), packed as b2p_op packs them: Bo[q1d][p] | Bc[q1d][p+1] | Gc
  // (not read: zeros)
  e->h_tab.assign((size_t)q1d * p + 2 * (size_t)q1d * (p + 1), 0.0);
  std::copy(flux_space->Bo, flux_space->Bo + (size_t)q1d * p, e->h_tab.begin());
  std::copy(flux_space->Bc, flux_space->Bc + (size_t)q1d * (p + 1), e->h_tab.begin() + (size_t)q1d * p);
  if ((rc = upload(ctx, e->h_tab.data(), e->h_tab.size(), &e->d_tab))) return rc;
  if ((rc = upload_coef_blocks(ctx, geom, n_attr, {coef_flux}, 10, &e->d_hex_coef_flux))) return rc;
  if ((rc = upload_coef_blocks(ctx, geom, n_attr, {coef_disc, coef_smooth}, 18, &e->d_hex_coef_err))) return rc;
  HexFluxArgs &a = e->hex_err;
  a.ctx = ctx;
  a.geom = geom;
  a.p = p;
  a.h_tab = e->h_tab.data();
  a.tab = e->d_tab;
  a.production = hex_flux_production_eligible(p, q1d, e->h_tab.data());
  a.space_a = flux_space->kind == B2P_ND_MASS ? 0 : 1;
  a.ecoef = e->d_hex_coef_err;
  HexFluxArgs af = a;
  af.ecoef = e->d_hex_coef_flux;
  e->Flux = std::make_unique<HexMixedMassOperator>(ctx, smooth_space->lsize, flux_space->lsize, af);
  return finish_estimator(e, M, tol, max_it, W, out);
}

// rhs = Flux flux_dofs
int b2p_flux_estimator_flux_mult(b2p_flux_estimator *e, const double *flux_dofs, double *rhs)
{
  if (!e || !flux_dofs || !rhs) return B2P_ERR_ARG;
  b2p_ctx *ctx = e->ctx;
  e->Flux->Mult(flux_dofs, rhs);
  if (e->hex)
  {
    const int rc = static_cast<HexMixedMassOperator *>(e->Flux.get())->rc;
    if (rc) return rc;
  }
  cudaError_t err = cudaPeekAtLastError();
  B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "b2p_flux_estimator_flux_mult: %s", cudaGetErrorString(err));
  return B2P_SUCCESS;
}


// FluxProjector::Mult (errorestimator.cpp:166-175)
int b2p_flux_estimator_project(b2p_flux_estimator *e, const double *flux_dofs, double *smooth_dofs)
{
  if (!e || !flux_dofs || !smooth_dofs) return B2P_ERR_ARG;
  b2p_ctx *ctx = e->ctx;
  if (e->rhs.n != e->smooth.lsize) e->rhs.resize(ctx, e->smooth.lsize);
  int rc = b2p_flux_estimator_flux_mult(e, flux_dofs, e->rhs.p);
  if (rc) return rc;
  e->solver->Mult(e->rhs.p, smooth_dofs);
  if (!e->solver->converged)
    set_error(ctx, "Linear solver did not converge, norm(Ax-b)/norm(b) = %.3e (norm(b) = %.3e)!", e->solver->final_res / e->solver->initial_res,
              e->solver->initial_res);
  e->mult++;
  e->mult_it += e->solver->final_it;
  cudaError_t err = cudaPeekAtLastError();
  B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "b2p_flux_estimator_project: %s", cudaGetErrorString(err));
  return B2P_SUCCESS;
}

// estimates[ne] += int_K |C2 smooth - C1 flux|^2 (one part of a field): ComputeErrorEstimates without the projection
int b2p_flux_estimator_integrate(b2p_flux_estimator *e, const double *flux_dofs, const double *smooth_dofs, double *estimates)
{
  if (!e || !flux_dofs || !smooth_dofs || !estimates) return B2P_ERR_ARG;
  b2p_ctx *ctx = e->ctx;
  const b2p_geom *g = e->geom;
  if (e->hex)
  {
    const int rc = launch_hex_flux_error(e->hex_err, flux_dofs, smooth_dofs, estimates, ctx->stream);
    if (rc) return rc;
    cudaError_t err = cudaPeekAtLastError();
    B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "b2p_flux_estimator_integrate: %s", cudaGetErrorString(err));
    return B2P_SUCCESS;
  }
  const size_t shmem = (size_t)(e->flux.P + e->smooth.P + 6 * g->Q + FLUX_NT + std::max(e->flux.P, e->smooth.P)) * sizeof(double);
  if (shmem > 48 * 1024) cudaFuncSetAttribute(flux_error_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem);
  B2P_LAUNCH(flux_error_kernel, g->ne, FLUX_NT, shmem, ctx->stream, g->ne, g->Q, g->q1d, e->flux, e->smooth, (const double *)g->qd,
             (const double *)e->d_coef_disc, (const double *)e->d_coef_smooth, flux_dofs, smooth_dofs, estimates);
  cudaError_t err = cudaPeekAtLastError();
  B2P_CHECK(ctx, err == cudaSuccess, B2P_ERR_CUDA, "b2p_flux_estimator_integrate: %s", cudaGetErrorString(err));
  return B2P_SUCCESS;
}

// CurlFluxErrorEstimator::AddErrorIndicator (errorestimator.cpp:506-513): estimates[ne] = sqrt(s * sum over the parts of eta_K^2)
int b2p_flux_estimator_indicator(b2p_flux_estimator *e, const double *flux_re, const double *flux_im, double Et, double *estimates)
{
  if (!e || !flux_re || !estimates) return B2P_ERR_ARG;
  b2p_ctx *ctx = e->ctx;
  const int ne = e->geom->ne;
  if (e->H.n != e->smooth.lsize) e->H.resize(ctx, e->smooth.lsize);
  vec::set(ctx, estimates, ne, 0.0);
  int rc;
  for (const double *part : {flux_re, flux_im})
  {
    if (!part) continue;
    if ((rc = b2p_flux_estimator_project(e, part, e->H.p))) return rc;
    if ((rc = b2p_flux_estimator_integrate(e, part, e->H.p, estimates))) return rc;
  }
  return b2p_flux_estimator_sqrt_scale(ctx, ne, Et > 0.0 ? 0.5 / Et : 1.0, estimates);
}

int b2p_flux_estimator_stats(b2p_flux_estimator *e, int *num_mult, int *num_mult_its, int *last_its, int *converged)
{
  if (!e) return B2P_ERR_ARG;
  if (num_mult) *num_mult = e->mult;
  if (num_mult_its) *num_mult_its = e->mult_it;
  if (last_its) *last_its = e->solver->final_it;
  if (converged) *converged = e->solver->converged ? 1 : 0;
  return B2P_SUCCESS;
}

// ConfigureLinearSolver(use_mg = true) (errorestimator.cpp:66-100): PCG, no initial guess, the estimator's relative tolerance,
// absolute tolerance epsilon; preconditioner GeometricMultigridSolver(coarse, P, no auxiliary space, 1 cycle, 1 smoothing
// iteration, 4th-kind Chebyshev of order 2, sf_max 1, sf_min 0), or the coarse solver alone on one level.
int b2p_flux_estimator_set_multigrid(b2p_flux_estimator *e, int n_levels, b2p_operator *const *ops, b2p_operator *const *P, int coarse_type,
                                     double coarse_tol, int coarse_max_it, b2p_solver *coarse_solver)
{
  if (!e) return B2P_ERR_ARG;
  b2p_ctx *ctx = e->ctx;
  B2P_CHECK(ctx, n_levels >= 1 && ops && (n_levels == 1 || P), B2P_ERR_ARG, "b2p_flux_estimator_set_multigrid: bad argument");
  B2P_CHECK(ctx, ops[n_levels - 1] && operator_of(ops[n_levels - 1]) == e->M, B2P_ERR_ARG,
            "b2p_flux_estimator_set_multigrid: the finest level operator must be the estimator's smooth-space mass operator");
  b2p_ksp_config cfg;
  b2p_ksp_config_default(&cfg, 1);
  cfg.krylov_solver = 0;
  cfg.tol = e->pcg->rel_tol;
  cfg.max_it = e->pcg->max_it;
  cfg.initial_guess = 0;
  cfg.mg_cycle_it = 1;
  cfg.mg_smooth_aux = 0;
  cfg.mg_smooth_it = 1;
  cfg.mg_smooth_order = 2;
  cfg.mg_smooth_sf_max = 1.0;
  cfg.mg_smooth_sf_min = 0.0;
  cfg.mg_smooth_cheby_4th = 1;
  cfg.coarse_type = coarse_type;
  cfg.coarse_tol = coarse_tol;
  cfg.coarse_max_it = coarse_max_it;
  b2p_ksp *k = nullptr;
  int rc = b2p_ksp_create(ctx, &cfg, n_levels, P, nullptr, coarse_solver, &k);
  if (rc) return rc;
  ksp_solver_of(k)->abs_tol = e->pcg->abs_tol;
  if ((rc = b2p_ksp_set_operators(k, ops[n_levels - 1], ops, nullptr)))
  {
    b2p_ksp_destroy(k);
    return rc;
  }
  b2p_ksp_destroy(e->mg);
  e->mg = k;
  e->solver = ksp_solver_of(k);
  return B2P_SUCCESS;
}

void b2p_flux_estimator_destroy(b2p_flux_estimator *e) { delete e; }

}  // extern "C"
