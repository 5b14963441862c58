// Sum-factorised H(div) work on hexahedra: the Raviart-Thomas mass operator (kind B2P_RT_MASS), and the flux operator and element
// error integrals of the flux error estimators (b2p_flux_estimator_create_hex). The RT mass and Flux are one mixed mass over a trial
// space and a test space, with the 1-D tables of the Nedelec space ND_p and the Raviart-Thomas space RT_{p-1}:
//
//   mixed mass        y_test += alpha sum_e E_test^T B_test^T D B_trial E_trial x_trial,   D = w detJ P_test^T C P_trial
//   error integral    est[e] += sum_q w detJ | C2 P2 u2 - C1 P1 u1 |^2                     (u_i = B_i E_i x_i)
//
// P_HCURL = A (the stored adj(J)^T / detJ), P_HDIV = Jd = cofactor(A); C is a general (possibly non-symmetric) 3x3 per element.
//   RT mass       (RT, RT): VectorFEMassIntegrator on an RT space, D = (w / detJ) J^T C J = w detJ Jd^T C Jd, the quadrature
//                 function f_apply_hdiv_33 (fem/integ/vecfemass.cpp:80-86, qfunctions/33/hdiv_33_qf.h:10-30); the operator inside
//                 the FluxProjector's PCG of GradFluxErrorEstimator (linalg/errorestimator.cpp:272-398). C: the first 9 of b2p_op::ecoef.
//   Flux          (ND, RT) or (RT, ND), and the error integrals: the same linear maps as mixed_mass_kernel / flux_error_kernel of
//                 b2p_flux.cu, with 1-D tables instead of dense [3][Q][P] tables.
// Both spaces share p (the ND-equivalent order), q1d and the tables Bo[q1d][p], Bc[q1d][p+1]. Lexicographic element layouts:
//   ND component c: open (p) along axis c, closed (p + 1) along the other two, offset c p (p+1)^2   (b2p_hex_nd.cu)
//   RT component c: closed along axis c, open along the other two,             offset c (p+1) p^2   (hexspace._rt_lex_layout)
//
// Kernels:
//   flux_hex_mixed7_kernel / flux_hex_error7_kernel   production, p = 2 ... 6 at q1d = p + 1 with mirror-symmetric tables: one CTA
//        per element batch, warps specialised by vector component, one 1-D line per thread, tables in the kernel parameter block,
//        q-data and coefficient blocks staged by TMA bulk copies (L2 evict-first); the mixed mass scatters with an unconditional
//        RED.F64 (masked entries add 0.0 to a sink slot), the error integral runs the forward phases of both spaces over the same
//        staged q-data;
//   flux_hex_mixed_kernel / flux_hex_error_kernel     cross-check, every p <= 6 and p < q1d <= 7 (shared-memory contract<>), and
//        the route wherever the production kernels are not eligible (for the RT mass also under B2P_APPLY_SIMPLE_KERNEL);
//   rt_hex_diag_kernel                                the diagonal of the RT mass, one thread per (element, dof).
// Flux and error-integral launches store their kernel name in the context's launch record (b2p_ctx_last_launch): one batch per
// CTA, grid = batches. RT mass launches leave the record alone.
// The error integrals reduce each element's points in a fixed order (one warp per element: strided lane sums, then a butterfly),
// so two calls give bit-identical estimates whatever the schedule.
#include <cstdlib>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_pipe.cuh"
#include "b2p_contract.cuh"

namespace b2p
{

namespace
{

constexpr int SP_ND = 0, SP_RT = 1;

constexpr int imax(int a, int b) { return a > b ? a : b; }

// extents of component C of space S along the three axes: ND open (p) along axis C and closed (p + 1) along the others, RT the
// other way round
template <int P_, int S, int C>
struct HexComp
{
  static constexpr int p = P_, n = P_ + 1;
  static constexpr bool c0 = (C == 0) == (S == SP_RT), c1 = (C == 1) == (S == SP_RT), c2 = (C == 2) == (S == SP_RT);  // closed?
  static constexpr int d0 = c0 ? n : p, d1 = c1 ? n : p, d2 = c2 ? n : p;
  static constexpr int D3 = d0 * d1 * d2;
  static constexpr int off = C * D3;
};
// element dofs of space S, and the largest line counts over its components after the first contraction (d1 d2) and the second (d2)
template <int P_, int S>
struct HexSpace
{
  using K0 = HexComp<P_, S, 0>;
  using K1 = HexComp<P_, S, 1>;
  using K2 = HexComp<P_, S, 2>;
  static constexpr int P = 3 * K0::D3;
  static constexpr int D12 = imax(imax(K0::d1 * K0::d2, K1::d1 * K1::d2), K2::d1 * K2::d2);
  static constexpr int D2 = imax(imax(K0::d2, K1::d2), K2::d2);
};

// physical value of a reference-space vector: H(curl) A u^, H(div) Jd u^
template <int S>
__device__ __forceinline__ void piola(const double A[9], double M[9])
{
  if constexpr (S == SP_ND)
  {
#pragma unroll
    for (int i = 0; i < 9; i++) M[i] = A[i];
  }
  else
    cofactor33(A, M);
}

// v = w detJ P_test^T C P_trial u
template <int ST, int SS>
__device__ __forceinline__ void mixed_point(const double A[9], const double C[9], double wdetj, const double u[3], double v[3])
{
  double Mt[9], Ms[9], t[3], z[3];
  piola<ST>(A, Mt);
  piola<SS>(A, Ms);
  Ax33(Mt, u, t);
  Ax33(C, t, z);
  Atx33(Ms, z, wdetj, v);
}

// w detJ | C2 P2 b - C1 P1 a |^2
template <int S1>
__device__ __forceinline__ double error_point(const double A[9], const double C1[9], const double C2[9], double wdetj, const double a[3],
                                              const double b[3])
{
  double M1[9], M2[9], t[3], v1[3], v2[3];
  piola<S1>(A, M1);
  piola<1 - S1>(A, M2);
  Ax33(M1, a, t);
  Ax33(C1, t, v1);
  Ax33(M2, b, t);
  Ax33(C2, t, v2);
  const double d0 = v2[0] - v1[0], d1 = v2[1] - v1[1], d2 = v2[2] - v1[2];
  return wdetj * (d0 * d0 + d1 * d1 + d2 * d2);
}

// Sum of the `cnt` values r[0], r[1], ... of one element by the 32 lanes of a warp in a fixed order: lane l adds l, l + 32, ...
// in sequence, then a butterfly. Every lane returns the same total.
__device__ __forceinline__ double warp_fixed_sum(const double *r, int cnt, int lane)
{
  double s = 0.0;
  for (int i = lane; i < cnt; i += 32) s += r[i];
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  return s;
}

// ---- cross-check kernels ------------------------------------------------------------------------------------------------

// SA, SB: the two spaces of the kernel; NV = 1: their element dofs one at a time (mixed mass), NV = 2: both (error integral)
template <int P_, int Q_, int SA, int SB, int NV>
struct HFLayout
{
  using Sa = HexSpace<P_, SA>;
  using Sb = HexSpace<P_, SB>;
  static constexpr int p = P_, q = Q_, n = P_ + 1, Q = q * q * q;
  static constexpr int UE = NV == 1 ? imax(Sa::P, Sb::P) : Sa::P + Sb::P;  // element dofs
  static constexpr int N1 = q * imax(Sa::D12, Sb::D12);                     // after the first contraction
  static constexpr int N2 = q * q * imax(Sa::D2, Sb::D2);                   // after the second
  // per-element shared doubles: U | T1 | T2 | uq[NV][3Q]
  static constexpr int PER_ELEM = UE + N1 + N2 + NV * 3 * Q;
};

struct HFParams
{
  const int32_t *lidx_a, *lidx_b;  // trial / test (mixed mass), space 1 / space 2 (error integral)
  int PS_a, PS_b;
  const double *tab;    // Bo[q][p] | Bc[q][n]
  const double *qd;     // [ne][10][Q]
  const double *ecoef;  // [ne][CE]
  int CE;
  const double *x_a, *x_b;
  double *y;            // the test space's L-vector (mixed mass) or the estimates [ne] (error integral)
  double alpha;         // scale of the mixed mass
  int ne;
};

// element dofs U_C of space S (d0, d1, d2) -> values at the points (q, q, q)
template <typename L, int S, int C, int NEB, int NT>
__device__ __forceinline__ void hf_forward(const double *U, double *T1, double *T2, double *uq, const double *sBo, const double *sBc)
{
  using K = HexComp<L::p, S, C>;
  constexpr int q = L::q, ES = L::PER_ELEM, d0 = K::d0, d1 = K::d1, d2 = K::d2;
  contract<0, d0, d1, d2, d0, q, false, NEB, NT>(U + K::off, ES, T1, ES, K::c0 ? sBc : sBo, d0, 1, 1.0);
  __syncthreads();
  contract<1, q, d1, d2, d1, q, false, NEB, NT>(T1, ES, T2, ES, K::c1 ? sBc : sBo, d1, 1, 1.0);
  __syncthreads();
  contract<2, q, q, d2, d2, q, false, NEB, NT>(T2, ES, uq + C * L::Q, ES, K::c2 ? sBc : sBo, d2, 1, 1.0);
  __syncthreads();
}

// point values (q, q, q) -> element dofs U_C of space S (overwritten)
template <typename L, int S, int C, int NEB, int NT>
__device__ __forceinline__ void hf_transpose(double *U, double *T1, double *T2, const double *uq, const double *sBo, const double *sBc)
{
  using K = HexComp<L::p, S, C>;
  constexpr int q = L::q, ES = L::PER_ELEM, d0 = K::d0, d1 = K::d1, d2 = K::d2;
  contract<2, q, q, q, q, d2, false, NEB, NT>(uq + C * L::Q, ES, T2, ES, K::c2 ? sBc : sBo, 1, d2, 1.0);
  __syncthreads();
  contract<1, q, q, d2, q, d1, false, NEB, NT>(T2, ES, T1, ES, K::c1 ? sBc : sBo, 1, d1, 1.0);
  __syncthreads();
  contract<0, q, d1, d2, q, d0, false, NEB, NT>(T1, ES, U + K::off, ES, K::c0 ? sBc : sBo, 1, d0, 1.0);
  __syncthreads();
}

template <typename L, int S, int NEB, int NT>
__device__ __forceinline__ void hf_gather(const int32_t *lidx, int PS, const double *x, double *U, int e0, int ne)
{
  constexpr int P = HexSpace<L::p, S>::P;
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    U[e * L::PER_ELEM + l] = (e0 + e < ne) ? gather1(x, lidx[(size_t)(e0 + e) * PS + l]) : 0.0;
  }
}

// ST: the trial space, SS: the test space
template <int P_, int Q_, int ST, int SS, int NEB, int NT>
__global__ void __launch_bounds__(NT) flux_hex_mixed_kernel(HFParams prm)
{
  using L = HFLayout<P_, Q_, ST, SS, 1>;
  constexpr int p = L::p, q = L::q, n = L::n, Q = L::Q, ES = L::PER_ELEM, PT = HexSpace<P_, SS>::P;
  B2P_DYN_SMEM(double, smem);
  double *sBo = smem, *sBc = sBo + q * p, *work = sBc + q * n;
  double *U = work, *T1 = U + L::UE, *T2 = T1 + L::N1, *uq = T2 + L::N2;
  for (int i = threadIdx.x; i < q * p + q * n; i += NT) sBo[i] = prm.tab[i];
  const int e0 = blockIdx.x * NEB;
  hf_gather<L, ST, NEB, NT>(prm.lidx_a, prm.PS_a, prm.x_a, U, e0, prm.ne);
  __syncthreads();
  hf_forward<L, ST, 0, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  hf_forward<L, ST, 1, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  hf_forward<L, ST, 2, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  for (int w = threadIdx.x; w < NEB * Q; w += NT)
  {
    const int e = w / Q, iq = w % Q;
    if (e0 + e >= prm.ne) continue;
    const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + qslot_of(q, iq);
    const double *Cm = prm.ecoef + (size_t)prm.CE * (e0 + e);
    double A[9], C[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C[i] = Cm[i];
    }
    double *u = uq + e * ES;
    const double uu[3] = {u[iq], u[Q + iq], u[2 * Q + iq]};
    double v[3];
    mixed_point<ST, SS>(A, C, g[0], uu, v);
    u[iq] = v[0];
    u[Q + iq] = v[1];
    u[2 * Q + iq] = v[2];
  }
  __syncthreads();
  hf_transpose<L, SS, 0, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  hf_transpose<L, SS, 1, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  hf_transpose<L, SS, 2, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  for (int w = threadIdx.x; w < NEB * PT; w += NT)
  {
    const int e = w / PT, l = w % PT;
    if (e0 + e >= prm.ne) continue;
    scatter1(prm.y, prm.lidx_b[(size_t)(e0 + e) * prm.PS_b + l], prm.alpha * U[e * ES + l]);
  }
}

// S1: the space of index 1 (the flux space); index 2 is the other one
template <int P_, int Q_, int S1, int NEB, int NT>
__global__ void __launch_bounds__(NT) flux_hex_error_kernel(HFParams prm)
{
  constexpr int S2 = 1 - S1, P1 = HexSpace<P_, S1>::P;
  using L = HFLayout<P_, Q_, S1, S2, 2>;
  constexpr int p = L::p, q = L::q, n = L::n, Q = L::Q, ES = L::PER_ELEM;
  B2P_DYN_SMEM(double, smem);
  double *sBo = smem, *sBc = sBo + q * p, *work = sBc + q * n;
  double *U1 = work, *U2 = U1 + P1, *T1 = U1 + L::UE, *T2 = T1 + L::N1, *uq1 = T2 + L::N2, *uq2 = uq1 + 3 * Q;
  for (int i = threadIdx.x; i < q * p + q * n; i += NT) sBo[i] = prm.tab[i];
  const int e0 = blockIdx.x * NEB;
  hf_gather<L, S1, NEB, NT>(prm.lidx_a, prm.PS_a, prm.x_a, U1, e0, prm.ne);
  hf_gather<L, S2, NEB, NT>(prm.lidx_b, prm.PS_b, prm.x_b, U2, e0, prm.ne);
  __syncthreads();
  hf_forward<L, S1, 0, NEB, NT>(U1, T1, T2, uq1, sBo, sBc);
  hf_forward<L, S1, 1, NEB, NT>(U1, T1, T2, uq1, sBo, sBc);
  hf_forward<L, S1, 2, NEB, NT>(U1, T1, T2, uq1, sBo, sBc);
  hf_forward<L, S2, 0, NEB, NT>(U2, T1, T2, uq2, sBo, sBc);
  hf_forward<L, S2, 1, NEB, NT>(U2, T1, T2, uq2, sBo, sBc);
  hf_forward<L, S2, 2, NEB, NT>(U2, T1, T2, uq2, sBo, sBc);
  // the contribution of every point replaces its first value of space 1
  for (int w = threadIdx.x; w < NEB * Q; w += NT)
  {
    const int e = w / Q, iq = w % Q;
    if (e0 + e >= prm.ne) continue;
    const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + qslot_of(q, iq);
    const double *Cm = prm.ecoef + (size_t)prm.CE * (e0 + e);
    double A[9], C1[9], C2[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C1[i] = Cm[i];
      C2[i] = Cm[9 + i];
    }
    double *a = uq1 + e * ES, *b = uq2 + e * ES;
    const double ua[3] = {a[iq], a[Q + iq], a[2 * Q + iq]}, ub[3] = {b[iq], b[Q + iq], b[2 * Q + iq]};
    a[iq] = error_point<S1>(A, C1, C2, g[0], ua, ub);  // (only this thread reads or writes point iq of element e)
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = warp; e < NEB; e += NT / 32)
  {
    if (e0 + e >= prm.ne) break;
    const double s = warp_fixed_sum(uq1 + e * ES, Q, lane);
    if (lane == 0) prm.y[e0 + e] += s;
  }
}

// ---- production kernels -------------------------------------------------------------------------------------------------

// the cross-check's parameters (tab and CE unread), the scratch of the branch-free scatter and the tables
template <int P_>
struct HF7Params : HFParams
{
  double *sink;
  double Bo[(P_ + 1) * P_];
  double Bc[(P_ + 1) * (P_ + 1)];
};

// NE elements per batch; per element in shared memory: the q-data [10][Q] and the coefficient block [CE] (TMA destinations), the
// element dofs U [UE] (one space at a time for the mixed mass, both spaces for the error integral), and per component the work
// arrays W1 (q, d1, d2), W2 (q, q, d2) sized for the larger of the spaces SA, SB, and NV sets of point values V (q, q, q).
template <int P_, int NE_, int SA, int SB, int NV, int CE_>
struct HF7Layout
{
  using Sa = HexSpace<P_, SA>;
  using Sb = HexSpace<P_, SB>;
  static constexpr int p = P_, NE = NE_, q = P_ + 1, Q = q * q * q;
  static constexpr int UE = NV == 1 ? imax(Sa::P, Sb::P) : Sa::P + Sb::P;
  static constexpr int GE = 10 * Q, CE = CE_;
  static constexpr int W1 = q * imax(Sa::D12, Sb::D12), W2 = q * q * imax(Sa::D2, Sb::D2);
  static constexpr int OFF_G = 0, OFF_C = OFF_G + NE * GE, OFF_U = OFF_C + NE * CE, OFF_W1 = OFF_U + NE * UE,
                       OFF_W2 = OFF_W1 + 3 * NE * W1, OFF_V = OFF_W2 + 3 * NE * W2, OFF_BAR = (OFF_V + NV * 3 * NE * Q + 1) & ~1;
  static constexpr int SMEM_BYTES = (OFF_BAR + 2) * 8;
  static_assert(GE % 2 == 0 && CE % 2 == 0 && UE % 2 == 0, "16-byte blocks for the bulk copies");
};

template <int P_>
struct HF7Shape;
// elements per batch, warps per component, the CTAs per SM asked of the register allocator for the mixed mass (MINB) and the
// error integral (MINB_E); 192 threads per CTA. Shared memory per CTA and registers: DESIGN section 4.2.
template <> struct HF7Shape<2> { static constexpr int NE = 8, WPC = 2, MINB = 4, MINB_E = 4; };
template <> struct HF7Shape<3> { static constexpr int NE = 4, WPC = 2, MINB = 4, MINB_E = 4; };
template <> struct HF7Shape<4> { static constexpr int NE = 2, WPC = 2, MINB = 3, MINB_E = 3; };
template <> struct HF7Shape<5> { static constexpr int NE = 2, WPC = 2, MINB = 3, MINB_E = 2; };
template <> struct HF7Shape<6> { static constexpr int NE = 1, WPC = 2, MINB = 2, MINB_E = 2; };

// The production kernels' rule: q1d = p + 1, p = 2 ... 6 (HF7Shape), and 1-D tables mirror-symmetric within HF7_SYM_TOL of their
// largest entry.
constexpr double HF7_SYM_TOL = 8e-15;
bool hf7_shape(int p, int q1d) { return q1d == p + 1 && p >= 2 && p <= 6; }

// One phase of component C of space S over the batch: every thread of the component's warps owns one line at a time.
//   PH 0..2: forward along x, y, z (U -> W1 -> W2 -> V);  PH 3..5: transposed along z, y, x (V -> W2 -> W1 -> U)
// U points at the space's dofs of element 0 (element stride UE), V at the space's point values of element 0.
template <typename L, int S, int C, int PH, int NTC>
__device__ __forceinline__ void hf7_phase(const HF7Params<L::p> &prm, double *sm, double *U, double *V, int t)
{
  using K = HexComp<L::p, S, C>;
  constexpr int NE = L::NE, q = L::q, d0 = K::d0, d1 = K::d1, d2 = K::d2, UE = L::UE;
  const double *Mx = K::c0 ? prm.Bc : prm.Bo, *My = K::c1 ? prm.Bc : prm.Bo, *Mz = K::c2 ? prm.Bc : prm.Bo;
  double *Uc = U + K::off, *W1 = sm + L::OFF_W1 + C * NE * L::W1, *W2 = sm + L::OFF_W2 + C * NE * L::W2, *Vc = V + C * NE * L::Q;
  constexpr int NP = PH == 0 ? d1 * d2 : PH == 1 || PH == 4 ? q * d2 : PH == 2 || PH == 3 ? q * q : d1 * d2;
  for (int w = t; w < NE * NP; w += NTC)
  {
    const int e = w / NP, r = w % NP;
    if constexpr (PH == 0) pencil<0, d0, d1, d2, d0, q, false>(r, Uc + e * UE, W1 + e * L::W1, Mx, d0, 1, 1.0);
    if constexpr (PH == 1) pencil<1, q, d1, d2, d1, q, false>(r, W1 + e * L::W1, W2 + e * L::W2, My, d1, 1, 1.0);
    if constexpr (PH == 2) pencil<2, q, q, d2, d2, q, false>(r, W2 + e * L::W2, Vc + e * L::Q, Mz, d2, 1, 1.0);
    if constexpr (PH == 3) pencil<2, q, q, q, q, d2, false>(r, Vc + e * L::Q, W2 + e * L::W2, Mz, 1, d2, 1.0);
    if constexpr (PH == 4) pencil<1, q, q, d2, q, d1, false>(r, W2 + e * L::W2, W1 + e * L::W1, My, 1, d1, 1.0);
    if constexpr (PH == 5) pencil<0, q, d1, d2, q, d0, false>(r, W1 + e * L::W1, Uc + e * UE, Mx, 1, d0, 1.0);
  }
}

template <typename L, int S, int PH, int NTC>
__device__ __forceinline__ void hf7_phase_all(const HF7Params<L::p> &prm, double *sm, double *U, double *V, int comp, int t)
{
  if (comp == 0)
    hf7_phase<L, S, 0, PH, NTC>(prm, sm, U, V, t);
  else if (comp == 1)
    hf7_phase<L, S, 1, PH, NTC>(prm, sm, U, V, t);
  else
    hf7_phase<L, S, 2, PH, NTC>(prm, sm, U, V, t);
  __syncthreads();
}

// Stage the batch's q-data and coefficient blocks behind one mbarrier (thread 0 issues; the caller's next __syncthreads publishes
// the initialised barrier before anyone polls it).
template <typename L>
__device__ __forceinline__ void hf7_stage(const HF7Params<L::p> &prm, double *sm, uint64_t *bar, int e0, int nel)
{
  mbar_init(bar, 1);
  fence_proxy_async();
  const uint64_t once = l2_evict_first_policy();
  mbar_expect_tx(bar, (uint32_t)(nel * (L::GE + L::CE) * sizeof(double)));
  tma_bulk_g2s_hint(sm + L::OFF_G, prm.qd + (size_t)e0 * L::GE, (uint32_t)(nel * L::GE * sizeof(double)), bar, once);
  tma_bulk_g2s_hint(sm + L::OFF_C, prm.ecoef + (size_t)e0 * L::CE, (uint32_t)(nel * L::CE * sizeof(double)), bar, once);
}

// li: the batch's first restriction row. Row offsets within a batch are 32-bit (e < NE), which keeps them apart from the 64-bit
// batch offset; a shared 64-bit (e0 + e) PS costs each access a 64-bit multiply.
template <typename L, int S, int NT>
__device__ __forceinline__ void hf7_gather(const int32_t *li, int PS, const double *x, double *U, int nel, int tid)
{
  constexpr int P = HexSpace<L::p, S>::P;
  for (int w = tid; w < L::NE * P; w += NT)
  {
    const int e = w / P, l = w % P;
    U[e * L::UE + l] = e < nel ? gather1(x, li[e * PS + l]) : 0.0;
  }
}

// ST: the trial space, SS: the test space; CE doubles per coefficient block, C first
template <int P_, int ST, int SS, int CE, int NE, int WPC, int MINB>
__global__ void __launch_bounds__(3 * WPC * 32, MINB) flux_hex_mixed7_kernel(const __grid_constant__ HF7Params<P_> prm)
{
  using L = HF7Layout<P_, NE, ST, SS, 1, CE>;
  constexpr int q = L::q, Q = L::Q, PT = HexSpace<P_, SS>::P, NTC = WPC * 32, NT = 3 * NTC;
  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  double *sm = (double *)smem_raw;
  double *sG = sm + L::OFF_G, *sC = sm + L::OFF_C, *sU = sm + L::OFF_U, *sV = sm + L::OFF_V;
  uint64_t *bar = (uint64_t *)(sm + L::OFF_BAR);
  const int tid = threadIdx.x, comp = (tid >> 5) / WPC, t = tid % NTC;
  const int e0 = blockIdx.x * NE, nel = min(NE, prm.ne - e0);
  if (nel <= 0) return;

  if (tid == 0) hf7_stage<L>(prm, sm, bar, e0, nel);
  hf7_gather<L, ST, NT>(prm.lidx_a + (size_t)e0 * prm.PS_a, prm.PS_a, prm.x_a, sU, nel, tid);
  __syncthreads();

  hf7_phase_all<L, ST, 0, NTC>(prm, sm, sU, sV, comp, t);
  hf7_phase_all<L, ST, 1, NTC>(prm, sm, sU, sV, comp, t);
  hf7_phase_all<L, ST, 2, NTC>(prm, sm, sU, sV, comp, t);

  // D: one thread per point, in the x-slowest order of the q-data
  mbar_wait(bar, 0);
  for (int w = tid; w < nel * Q; w += NT)
  {
    const int e = w / Q, s = w % Q;
    const int qx = s / (q * q), qz = (s / q) % q, qy = s % q, iq = qx + q * (qy + q * qz);
    const double *g = sG + e * L::GE + s, *Cm = sC + e * L::CE;
    double A[9], C[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C[i] = Cm[i];
    }
    double *v0 = sV + e * Q + iq, *v1 = v0 + NE * Q, *v2 = v1 + NE * Q;
    const double u[3] = {*v0, *v1, *v2};
    double v[3];
    mixed_point<ST, SS>(A, C, g[0], u, v);
    *v0 = v[0];
    *v1 = v[1];
    *v2 = v[2];
  }
  __syncthreads();

  hf7_phase_all<L, SS, 3, NTC>(prm, sm, sU, sV, comp, t);
  hf7_phase_all<L, SS, 4, NTC>(prm, sm, sU, sV, comp, t);
  hf7_phase_all<L, SS, 5, NTC>(prm, sm, sU, sV, comp, t);

  // scatter: RED.F64 for every entry; masked entries (and the empty slots of a ragged batch) add 0.0 to this thread's sink slot
  const int32_t *li = prm.lidx_b + (size_t)e0 * prm.PS_b;
  double *my_sink = prm.sink + ((blockIdx.x * NT + tid) & (b2p_ctx::SINK_SLOTS - 1));
  for (int w = tid; w < nel * PT; w += NT)
  {
    const int e = w / PT, l = w % PT;
    const int32_t gi = li[e * prm.PS_b + l];  // (32-bit row offset, as in hf7_gather)
    const double v = prm.alpha * sU[e * L::UE + l];
    const bool skip = gi == (int32_t)B2P_SKIP_IDX;
    const int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
    const double sv = skip ? 0.0 : __hiloint2double(hi, __double2loint(v));
    double *addr = skip ? my_sink : prm.y + (uint32_t)abs_idx(gi);
#ifdef B2P_EMU
    atomicAdd(addr, sv);
#else
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(sv) : "memory");
#endif
  }
}

// S1: the space of index 1 (the flux space); index 2 is the other one
template <int P_, int S1, int NE, int WPC, int MINB>
__global__ void __launch_bounds__(3 * WPC * 32, MINB) flux_hex_error7_kernel(const __grid_constant__ HF7Params<P_> prm)
{
  constexpr int S2 = 1 - S1, P1 = HexSpace<P_, S1>::P;
  using L = HF7Layout<P_, NE, S1, S2, 2, 18>;  // coefficient blocks C1 | C2
  constexpr int q = L::q, Q = L::Q, NTC = WPC * 32, NT = 3 * NTC;
  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  double *sm = (double *)smem_raw;
  double *sG = sm + L::OFF_G, *sC = sm + L::OFF_C, *sU1 = sm + L::OFF_U, *sU2 = sU1 + P1, *sV1 = sm + L::OFF_V, *sV2 = sV1 + 3 * NE * Q;
  uint64_t *bar = (uint64_t *)(sm + L::OFF_BAR);
  const int tid = threadIdx.x, comp = (tid >> 5) / WPC, t = tid % NTC;
  const int e0 = blockIdx.x * NE, nel = min(NE, prm.ne - e0);
  if (nel <= 0) return;

  if (tid == 0) hf7_stage<L>(prm, sm, bar, e0, nel);
  hf7_gather<L, S1, NT>(prm.lidx_a + (size_t)e0 * prm.PS_a, prm.PS_a, prm.x_a, sU1, nel, tid);
  hf7_gather<L, S2, NT>(prm.lidx_b + (size_t)e0 * prm.PS_b, prm.PS_b, prm.x_b, sU2, nel, tid);
  __syncthreads();

  hf7_phase_all<L, S1, 0, NTC>(prm, sm, sU1, sV1, comp, t);
  hf7_phase_all<L, S1, 1, NTC>(prm, sm, sU1, sV1, comp, t);
  hf7_phase_all<L, S1, 2, NTC>(prm, sm, sU1, sV1, comp, t);
  hf7_phase_all<L, S2, 0, NTC>(prm, sm, sU2, sV2, comp, t);
  hf7_phase_all<L, S2, 1, NTC>(prm, sm, sU2, sV2, comp, t);
  hf7_phase_all<L, S2, 2, NTC>(prm, sm, sU2, sV2, comp, t);

  // the contribution of every point, stored over its first value of space 1 (x-fastest order)
  mbar_wait(bar, 0);
  for (int w = tid; w < nel * Q; w += NT)
  {
    const int e = w / Q, s = w % Q;
    const int qx = s / (q * q), qz = (s / q) % q, qy = s % q, iq = qx + q * (qy + q * qz);
    const double *g = sG + e * L::GE + s, *Cm = sC + e * L::CE;
    double A[9], C1[9], C2[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C1[i] = Cm[i];
      C2[i] = Cm[9 + i];
    }
    double *a = sV1 + e * Q + iq, *b = sV2 + e * Q + iq;
    const double ua[3] = {a[0], a[NE * Q], a[2 * NE * Q]}, ub[3] = {b[0], b[NE * Q], b[2 * NE * Q]};
    *a = error_point<S1>(A, C1, C2, g[0], ua, ub);  // (only this thread reads or writes point iq of element e)
  }
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31;
  for (int e = warp; e < nel; e += NT / 32)
  {
    const double s = warp_fixed_sum(sV1 + e * Q, Q, lane);
    if (lane == 0) prm.y[e0 + e] += s;
  }
}

// ---- diagonal -----------------------------------------------------------------------------------------------------------

struct RTParams
{
  const int32_t *lidx;
  const double *tab;    // Bo[q][p] | Bc[q][n] | (Gc, unused)
  const double *qd;     // [ne][10][Q]
  const double *ecoef;  // [ne][18]: the material tensor (first 9)
  double *y;
  int ne;
  int PS;
};

// diag[|gid(l)|] += sum_q phi_l(q)^T D_q phi_l(q); one thread per (element, lexicographic dof)
__global__ void rt_hex_diag_kernel(RTParams prm, int p, int q)
{
  const int n = p + 1, D3 = n * p * p, P = 3 * D3, Q = q * q * q;
  const double *Bo = prm.tab, *Bc = Bo + q * p;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)prm.ne * P) return;
  const int e = (int)(w / P), l = (int)(w % P);
  const int c = l / D3, r = l % D3;
  const int d0 = c == 0 ? n : p, d1 = c == 1 ? n : p;
  const int i = r % d0, j = (r / d0) % d1, k = r / (d0 * d1);
  double C[9];
  for (int t = 0; t < 9; t++) C[t] = prm.ecoef[18 * (size_t)e + t];
  double s = 0.0;
  for (int qz = 0; qz < q; qz++)
    for (int qy = 0; qy < q; qy++)
      for (int qx = 0; qx < q; qx++)
      {
        const double fx = c == 0 ? Bc[qx * n + i] : Bo[qx * p + i];
        const double fy = c == 1 ? Bc[qy * n + j] : Bo[qy * p + j];
        const double fz = c == 2 ? Bc[qz * n + k] : Bo[qz * p + k];
        const double f = fx * fy * fz;
        const double u[3] = {c == 0 ? f : 0.0, c == 1 ? f : 0.0, c == 2 ? f : 0.0};
        double A[9], Jd[9], v[3];
        const double *g = prm.qd + (size_t)e * 10 * Q + qslot(q, qx, qy, qz);
        for (int t = 0; t < 9; t++) A[t] = g[(1 + t) * Q];
        cofactor33(A, Jd);
        AtCAx(Jd, C, u, g[0], v);
        s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
      }
  int gi = prm.lidx[(size_t)e * prm.PS + l];
  if (gi == B2P_SKIP_IDX) return;
  if (gi < 0) gi = -1 - gi;
  atomicAdd(prm.y + gi, s);
}

// ---- launchers ----------------------------------------------------------------------------------------------------------

// The kernel parameters of elements [e_off, e_off + e_cnt): restrictions, q-data and coefficient blocks from element e_off on.
HFParams make_hf_params(const HexFluxArgs &a, int CE, double alpha, const double *xa, const double *xb, double *y, int e_off, int e_cnt)
{
  HFParams prm;
  prm.lidx_a = a.lidx_a + (size_t)e_off * a.PS_a;
  prm.lidx_b = a.lidx_b + (size_t)e_off * a.PS_b;
  prm.PS_a = a.PS_a;
  prm.PS_b = a.PS_b;
  prm.tab = a.tab;
  prm.qd = a.geom->qd + (size_t)e_off * 10 * a.geom->Q;
  prm.ecoef = a.ecoef + (size_t)e_off * CE;
  prm.CE = CE;
  prm.x_a = xa;
  prm.x_b = xb;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  return prm;
}

// One CTA per batch of `per_batch` elements. A non-null `record` names the kernel in the context's launch record.
template <typename K, typename Prm>
int launch_batches(K *kern, const Prm &prm, int threads, size_t shmem, cudaStream_t s, b2p_ctx *ctx, const char *record, int per_batch)
{
  const int grid = (prm.ne + per_batch - 1) / per_batch;
  if (record) return launch_persistent(kern, prm, threads, shmem, s, false, ctx, record, false, false, grid, 1, per_batch, grid);
  B2P_LAUNCH(kern, grid, threads, shmem, s, prm);
  B2P_CUDA(ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

template <int P_, int Q_, int SA, int SB, bool ERR>
int launch_hf_pq(const HexFluxArgs &a, const HFParams &prm, bool record, cudaStream_t s)
{
  constexpr int NV = ERR ? 2 : 1, NT = 256;
  using L = HFLayout<P_, Q_, SA, SB, NV>;
  constexpr int per_elem_bytes = L::PER_ELEM * 8;
  constexpr int NEB = (per_elem_bytes * 8 <= 100 * 1024) ? 8 : (per_elem_bytes * 4 <= 100 * 1024) ? 4 : (per_elem_bytes * 2 <= 200 * 1024) ? 2 : 1;
  const size_t shmem = (size_t)(Q_ * P_ + Q_ * (P_ + 1) + NEB * L::PER_ELEM) * sizeof(double);
  auto kern = [] {
    if constexpr (ERR)
      return flux_hex_error_kernel<P_, Q_, SA, NEB, NT>;
    else
      return flux_hex_mixed_kernel<P_, Q_, SA, SB, NEB, NT>;
  }();
  if (int rc = configure_kernel(a.ctx, kern, shmem)) return rc;
  return launch_batches(kern, prm, NT, shmem, s, a.ctx, record ? (ERR ? "flux_hex_error_kernel" : "flux_hex_mixed_kernel") : nullptr, NEB);
}

template <int P_, int SA, int SB, bool ERR, int CE>
int launch_hf7(const HexFluxArgs &a, const HFParams &base, bool record, cudaStream_t s)
{
  using S = HF7Shape<P_>;
  using L = HF7Layout<P_, S::NE, SA, SB, ERR ? 2 : 1, CE>;
  constexpr int NT = 3 * S::WPC * 32;
  auto kern = [] {
    if constexpr (ERR)
      return flux_hex_error7_kernel<P_, SA, S::NE, S::WPC, S::MINB_E>;
    else
      return flux_hex_mixed7_kernel<P_, SA, SB, CE, S::NE, S::WPC, S::MINB>;
  }();
  if (int rc = configure_kernel(a.ctx, kern, L::SMEM_BYTES)) return rc;
  HF7Params<P_> prm;
  static_cast<HFParams &>(prm) = base;
  prm.sink = a.ctx->d_sink;
  copy_tables(a.h_tab, P_, P_ + 1, P_ + 1, prm.Bo, prm.Bc, nullptr);
  return launch_batches(kern, prm, NT, L::SMEM_BYTES, s, a.ctx, record ? (ERR ? "flux_hex_error7_kernel" : "flux_hex_mixed7_kernel") : nullptr,
                        S::NE);
}

// The mixed mass from space SA to space SB with CE-double coefficient blocks, or (ERR) the error integral with SA the space of
// index 1, on the production kernel (`production`) or the cross-check kernel. `who` and `tag` name the launch in the trace and
// the error message; `record`: store it in the context's launch record.
template <int SA, int SB, bool ERR, int CE>
int launch_hdiv(const HexFluxArgs &a, const HFParams &prm, bool production, bool record, const char *who, const char *tag, cudaStream_t s)
{
  if (prm.ne <= 0) return B2P_SUCCESS;
  static const bool trace = std::getenv("B2P_TRACE_KERNEL") != nullptr;
  const int p = a.p, q1d = a.geom->q1d;
  if (trace) fprintf(stderr, "[b2p] %s%s%s p=%d q1d=%d ne=%d\n", who, production ? "7" : "", tag, p, q1d, prm.ne);
  if (production)
  {
#define B2P_CASE(PP) \
  if (p == PP) return launch_hf7<PP, SA, SB, ERR, CE>(a, prm, record, s);
    B2P_CASE(2) B2P_CASE(3) B2P_CASE(4) B2P_CASE(5) B2P_CASE(6)
#undef B2P_CASE
  }
#define B2P_CASE(PP, QQ) \
  if (p == PP && q1d == QQ) return launch_hf_pq<PP, QQ, SA, SB, ERR>(a, prm, record, s);
  B2P_CASE(1, 2) B2P_CASE(1, 3) B2P_CASE(1, 4) B2P_CASE(1, 5) B2P_CASE(1, 6) B2P_CASE(1, 7)
  B2P_CASE(2, 3) B2P_CASE(2, 4) B2P_CASE(2, 5) B2P_CASE(2, 6) B2P_CASE(2, 7)
  B2P_CASE(3, 4) B2P_CASE(3, 5) B2P_CASE(3, 6) B2P_CASE(3, 7)
  B2P_CASE(4, 5) B2P_CASE(4, 6) B2P_CASE(4, 7)
  B2P_CASE(5, 6) B2P_CASE(5, 7)
  B2P_CASE(6, 7)
#undef B2P_CASE
  set_error(a.ctx, "%s: no kernel for p=%d q1d=%d", who, p, q1d);
  return B2P_ERR_UNSUPPORTED;
}

template <bool ERR>
int launch_hex_flux(const HexFluxArgs &a, const double *xa, const double *xb, double *y, cudaStream_t s)
{
  constexpr int CE = ERR ? 18 : 10;  // C1 | C2, or C (+ 1 pad)
  const HFParams prm = make_hf_params(a, CE, 1.0, xa, xb, y, 0, a.geom->ne);
  const char *who = ERR ? "flux_hex_error" : "flux_hex_mixed";
  if (a.space_a == SP_ND) return launch_hdiv<SP_ND, SP_RT, ERR, CE>(a, prm, a.production, true, who, ERR ? " nd,rt" : " nd->rt", s);
  return launch_hdiv<SP_RT, SP_ND, ERR, CE>(a, prm, a.production, true, who, ERR ? " rt,nd" : " rt->nd", s);
}

}  // namespace

bool hex_flux_production_eligible(int p, int q1d, const double *h_tab)
{
  return hf7_shape(p, q1d) && nd_tables_symmetric(h_tab, p, q1d, HF7_SYM_TOL);
}

int launch_hex_flux_mixed(const HexFluxArgs &a, const double *x, double *y, cudaStream_t s)
{
  return launch_hex_flux<false>(a, x, nullptr, y, s);
}

int launch_hex_flux_error(const HexFluxArgs &a, const double *x1, const double *x2, double *est, cudaStream_t s)
{
  return launch_hex_flux<true>(a, x1, x2, est, s);
}

bool rt_hex_apply7_eligible(b2p_op *op)
{
  if (!op || op->kind != B2P_RT_MASS || op->dense || !op->ecoef) return false;
  return hf7_shape(op->p, op->q1d) && nd_tables_symmetric(op, HF7_SYM_TOL);  // (the symmetry cached on the operator)
}

int launch_rt_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                        bool rt7)
{
  HexFluxArgs a;
  a.ctx = op->ctx;
  a.geom = op->geom;
  a.p = op->p;
  a.h_tab = op->h_tab.data();
  a.tab = op->tab;
  a.lidx_a = a.lidx_b = lidx;
  a.PS_a = a.PS_b = op->PS;
  a.ecoef = op->ecoef;
  const HFParams prm = make_hf_params(a, 18, alpha, x, nullptr, y, rg.e_off, range_count(op, rg));
  return launch_hdiv<SP_RT, SP_RT, false, 18>(a, prm, rt7, false, "rt_hex_apply", "", s);
}

int launch_rt_hex_diag(b2p_op *op, double *diag, cudaStream_t s)
{
  const size_t total = (size_t)op->ne * op->P;
  const int nt = 128;
  const RTParams prm = {op->lidx, op->tab, op->geom->qd, op->ecoef, diag, op->ne, op->PS};
  B2P_LAUNCH(rt_hex_diag_kernel, (unsigned)((total + nt - 1) / nt), nt, 0, s, prm, op->p, op->q1d);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p
