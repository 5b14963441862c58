// Matrix-free Raviart-Thomas (H(div)) hexahedron mass operator: VectorFEMassIntegrator on an RT space
//
//   y_L += alpha * sum_e E_e^T  B^T  D  B  E_e x_L,     D = (w / detJ) J^T C J = w detJ Jd^T C Jd   (Jd = J / detJ)
//
// the quadrature function f_apply_hdiv_33 (/root/reference/palace/fem/integ/vecfemass.cpp:80-86,
// qfunctions/33/hdiv_33_qf.h:10-30); Jd is the cofactor of the stored adj(J)^T / detJ, as in the curl part of the ND kernels.
// It is the operator inside the FluxProjector's PCG of GradFluxErrorEstimator (linalg/errorestimator.cpp:272-398).
//
// Space RT_{p-1} described by the ND-equivalent order p (P = 3 p^2 (p + 1)); lexicographic element layout
// (hexspace._rt_lex_layout), each component CLOSED (p + 1 Gauss-Lobatto nodes, table Bc) along its own axis and OPEN (p
// Gauss-Legendre nodes, table Bo) along the other two -- ND's assignment with the roles exchanged:
//   x-directed dofs Ux[k][j][i], i<=p, j,k<p     offset 0
//   y-directed dofs Uy[k][j][i], j<=p, i,k<p     offset (p+1)p^2
//   z-directed dofs Uz[k][j][i], k<=p, i,j<p     offset 2(p+1)p^2
//
// Kernels:
//   rt_hex_apply7_kernel  production, p = 2 ... 6 at q1d = p + 1 with mirror-symmetric tables: one CTA per element batch,
//                         warps specialised by vector component, one 1-D line per thread, tables in the kernel parameter block,
//                         q-data and coefficient blocks staged by TMA bulk copies (L2 evict-first), unconditional RED.F64 scatter
//                         (masked entries add 0.0 to a sink slot);
//   rt_hex_apply_kernel   cross-check, every p <= 6 and p < q1d <= 7 (B2P_APPLY_SIMPLE_KERNEL, and wherever the production kernel
//                         is not eligible);
//   rt_hex_diag_kernel    the diagonal, one thread per (element, dof).
#include <cstdlib>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

// extents of RT component C along the three axes: closed (n = p + 1) along axis C, open (p) along the others
template <int P_, int C>
struct RTComp
{
  static constexpr int p = P_, n = P_ + 1;
  static constexpr int d0 = C == 0 ? n : p, d1 = C == 1 ? n : p, d2 = C == 2 ? n : p;
  static constexpr int D3 = n * p * p;
  static constexpr int off = C * D3;
};

// ---- cross-check kernel -------------------------------------------------------------------------------------------------

template <int P_, int Q_>
struct RTLayout
{
  static constexpr int p = P_, q = Q_, n = P_ + 1;
  static constexpr int P = 3 * n * p * p, Q = q * q * q;
  static constexpr int N1 = q * n * p;  // after the first contraction (largest over the components)
  static constexpr int N2 = q * q * n;  // after the second
  // per-element shared doubles: U | T1 | T2 | uq[3Q]
  static constexpr int PER_ELEM = P + N1 + N2 + 3 * Q;
};

struct RTParams
{
  const int32_t *lidx;
  const double *tab;    // Bo[q][p] | Bc[q][n] | (Gc, unused)
  const double *qd;     // [ne][10][Q]
  const double *ecoef;  // [ne][18]: the material tensor (first 9)
  const double *x;
  double *y;
  double alpha;
  int ne;
  int PS;
};

// forward contractions of component C: element dofs U_C (d0, d1, d2) -> values at the points (q, q, q)
template <int P_, int Q_, int C, int NEB, int NT>
__device__ __forceinline__ void rt_forward(double *U, double *T1, double *T2, double *uq, const double *sBo, const double *sBc)
{
  using L = RTLayout<P_, Q_>;
  using K = RTComp<P_, C>;
  constexpr int q = Q_, ES = L::PER_ELEM, d0 = K::d0, d1 = K::d1, d2 = K::d2;
  contract<0, d0, d1, d2, d0, q, false, NEB, NT>(U + K::off, ES, T1, ES, C == 0 ? sBc : sBo, d0, 1, 1.0);
  __syncthreads();
  contract<1, q, d1, d2, d1, q, false, NEB, NT>(T1, ES, T2, ES, C == 1 ? sBc : sBo, d1, 1, 1.0);
  __syncthreads();
  contract<2, q, q, d2, d2, q, false, NEB, NT>(T2, ES, uq + C * L::Q, ES, C == 2 ? sBc : sBo, d2, 1, 1.0);
  __syncthreads();
}

// transposed contractions of component C: point values (q, q, q) -> element dofs U_C (overwritten)
template <int P_, int Q_, int C, int NEB, int NT>
__device__ __forceinline__ void rt_transpose(double *U, double *T1, double *T2, const double *uq, const double *sBo, const double *sBc)
{
  using L = RTLayout<P_, Q_>;
  using K = RTComp<P_, C>;
  constexpr int q = Q_, ES = L::PER_ELEM, d0 = K::d0, d1 = K::d1, d2 = K::d2;
  contract<2, q, q, q, q, d2, false, NEB, NT>(uq + C * L::Q, ES, T2, ES, C == 2 ? sBc : sBo, 1, d2, 1.0);
  __syncthreads();
  contract<1, q, q, d2, q, d1, false, NEB, NT>(T2, ES, T1, ES, C == 1 ? sBc : sBo, 1, d1, 1.0);
  __syncthreads();
  contract<0, q, d1, d2, q, d0, false, NEB, NT>(T1, ES, U + K::off, ES, C == 0 ? sBc : sBo, 1, d0, 1.0);
  __syncthreads();
}

template <int P_, int Q_, int NEB, int NT>
__global__ void __launch_bounds__(NT) rt_hex_apply_kernel(RTParams prm)
{
  using L = RTLayout<P_, Q_>;
  constexpr int p = L::p, q = L::q, n = L::n, P = L::P, Q = L::Q, ES = L::PER_ELEM;

  B2P_DYN_SMEM(double, smem);
  double *sBo = smem;         // [q][p]
  double *sBc = sBo + q * p;  // [q][n]
  double *work = sBc + q * n;
  double *U = work, *T1 = U + P, *T2 = T1 + L::N1, *uq = T2 + L::N2;

  for (int i = threadIdx.x; i < q * p + q * n; i += NT) sBo[i] = prm.tab[i];
  const int e0 = blockIdx.x * NEB;
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    U[e * ES + l] = (e0 + e < prm.ne) ? gather1(prm.x, prm.lidx[(size_t)(e0 + e) * prm.PS + l]) : 0.0;
  }
  __syncthreads();

  rt_forward<P_, Q_, 0, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  rt_forward<P_, Q_, 1, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  rt_forward<P_, Q_, 2, NEB, NT>(U, T1, T2, uq, sBo, sBc);

  for (int w = threadIdx.x; w < NEB * Q; w += NT)
  {
    const int e = w / Q, iq = w % Q;
    if (e0 + e >= prm.ne) continue;
    const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + qslot_of(q, iq);
    const double *Cm = prm.ecoef + 18 * (size_t)(e0 + e);
    double A[9], Jd[9], C[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C[i] = Cm[i];
    }
    cofactor33(A, Jd);
    double *u = uq + e * ES;
    const double uu[3] = {u[iq], u[Q + iq], u[2 * Q + iq]};
    double v[3];
    AtCAx(Jd, C, uu, g[0], v);
    u[iq] = v[0];
    u[Q + iq] = v[1];
    u[2 * Q + iq] = v[2];
  }
  __syncthreads();

  rt_transpose<P_, Q_, 0, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  rt_transpose<P_, Q_, 1, NEB, NT>(U, T1, T2, uq, sBo, sBc);
  rt_transpose<P_, Q_, 2, NEB, NT>(U, T1, T2, uq, sBo, sBc);

  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    if (e0 + e >= prm.ne) continue;
    scatter1(prm.y, prm.lidx[(size_t)(e0 + e) * prm.PS + l], prm.alpha * U[e * ES + l]);
  }
}

// ---- production kernel --------------------------------------------------------------------------------------------------

template <int P_>
struct RT7Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction (B2P_SKIP_IDX = masked)
  const double *qd;     // [ne][10][Q], x-slowest point order
  const double *ecoef;  // [ne][18]
  const double *x;
  double *y;
  double *sink;         // scratch of the branch-free scatter
  double alpha;
  int ne, PS;
  double Bo[(P_ + 1) * P_];
  double Bc[(P_ + 1) * (P_ + 1)];
};

// NE elements per batch; per element in shared memory: the q-data [10][Q] and the coefficient block [18] (TMA destinations),
// the element dofs U [P], and per component the work arrays W1 (q, d1, d2), W2 (q, q, d2) and the point values V (q, q, q).
template <int P_, int NE>
struct RT7Layout
{
  static constexpr int p = P_, q = P_ + 1, n = P_ + 1, Q = q * q * q, P = 3 * n * p * p;
  static constexpr int GE = 10 * Q, CE = 18;
  static constexpr int W1 = q * n * p, W2 = q * q * n;
  static constexpr int OFF_G = 0, OFF_C = OFF_G + NE * GE, OFF_U = OFF_C + NE * CE, OFF_W1 = OFF_U + NE * P,
                       OFF_W2 = OFF_W1 + 3 * NE * W1, OFF_V = OFF_W2 + 3 * NE * W2, OFF_BAR = (OFF_V + 3 * NE * Q + 1) & ~1;
  static constexpr int SMEM_BYTES = (OFF_BAR + 2) * 8;
  static_assert(GE % 2 == 0 && CE % 2 == 0, "16-byte blocks for the bulk copies");
};

template <int P_>
struct RT7Shape;
// elements per batch, warps per component, the CTAs per SM asked of the register allocator (192 threads; shared memory per CTA
// 33.8, 40.5, 40.0, 69.8, 55.8 KB at p = 2 ... 6; -Xptxas -v: 66-70 registers, no spills)
template <> struct RT7Shape<2> { static constexpr int NE = 8, WPC = 2, MINB = 4; };
template <> struct RT7Shape<3> { static constexpr int NE = 4, WPC = 2, MINB = 4; };
template <> struct RT7Shape<4> { static constexpr int NE = 2, WPC = 2, MINB = 3; };
template <> struct RT7Shape<5> { static constexpr int NE = 2, WPC = 2, MINB = 3; };
template <> struct RT7Shape<6> { static constexpr int NE = 1, WPC = 2, MINB = 2; };

// One phase of component C over the batch: every thread of the component's warps owns one line (pencil) at a time.
//   PH 0..2: forward along x, y, z (U -> W1 -> W2 -> V);  PH 3..5: transposed along z, y, x (V -> W2 -> W1 -> U)
template <int P_, int NE, int C, int PH, int NTC>
__device__ __forceinline__ void rt7_phase(const RT7Params<P_> &prm, double *sm, int t)
{
  using L = RT7Layout<P_, NE>;
  using K = RTComp<P_, C>;
  constexpr int q = L::q, d0 = K::d0, d1 = K::d1, d2 = K::d2;
  const double *Mx = C == 0 ? prm.Bc : prm.Bo, *My = C == 1 ? prm.Bc : prm.Bo, *Mz = C == 2 ? prm.Bc : prm.Bo;
  double *U = sm + L::OFF_U + K::off, *W1 = sm + L::OFF_W1 + C * NE * L::W1, *W2 = sm + L::OFF_W2 + C * NE * L::W2,
         *V = sm + L::OFF_V + C * NE * L::Q;
  constexpr int NP = PH == 0 ? d1 * d2 : PH == 1 || PH == 4 ? q * d2 : PH == 2 || PH == 3 ? q * q : d1 * d2;
  for (int w = t; w < NE * NP; w += NTC)
  {
    const int e = w / NP, r = w % NP;
    if constexpr (PH == 0) pencil<0, d0, d1, d2, d0, q, false>(r, U + e * L::P, W1 + e * L::W1, Mx, d0, 1, 1.0);
    if constexpr (PH == 1) pencil<1, q, d1, d2, d1, q, false>(r, W1 + e * L::W1, W2 + e * L::W2, My, d1, 1, 1.0);
    if constexpr (PH == 2) pencil<2, q, q, d2, d2, q, false>(r, W2 + e * L::W2, V + e * L::Q, Mz, d2, 1, 1.0);
    if constexpr (PH == 3) pencil<2, q, q, q, q, d2, false>(r, V + e * L::Q, W2 + e * L::W2, Mz, 1, d2, 1.0);
    if constexpr (PH == 4) pencil<1, q, q, d2, q, d1, false>(r, W2 + e * L::W2, W1 + e * L::W1, My, 1, d1, 1.0);
    if constexpr (PH == 5) pencil<0, q, d1, d2, q, d0, false>(r, W1 + e * L::W1, U + e * L::P, Mx, 1, d0, 1.0);
  }
}

template <int P_, int NE, int PH, int NTC>
__device__ __forceinline__ void rt7_phase_all(const RT7Params<P_> &prm, double *sm, int comp, int t)
{
  if (comp == 0)
    rt7_phase<P_, NE, 0, PH, NTC>(prm, sm, t);
  else if (comp == 1)
    rt7_phase<P_, NE, 1, PH, NTC>(prm, sm, t);
  else
    rt7_phase<P_, NE, 2, PH, NTC>(prm, sm, t);
  __syncthreads();
}

template <int P_, int NE, int WPC, int MINB>
__global__ void __launch_bounds__(3 * WPC * 32, MINB) rt_hex_apply7_kernel(const __grid_constant__ RT7Params<P_> prm)
{
  using L = RT7Layout<P_, NE>;
  constexpr int q = L::q, Q = L::Q, P = L::P, NTC = WPC * 32, NT = 3 * NTC;
  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  double *sm = (double *)smem_raw;
  double *sG = sm + L::OFF_G, *sC = sm + L::OFF_C, *sU = sm + L::OFF_U;
  uint64_t *bar = (uint64_t *)(sm + L::OFF_BAR);
  const int tid = threadIdx.x, comp = (tid >> 5) / WPC, t = tid % NTC;
  const int e0 = blockIdx.x * NE, nel = min(NE, prm.ne - e0);
  if (nel <= 0) return;

  // q-data and coefficient blocks of the batch: read once per launch, staged behind one mbarrier while the x values are gathered
  if (tid == 0)
  {
    mbar_init(bar, 1);
    fence_proxy_async();
    const uint64_t once = l2_evict_first_policy();
    mbar_expect_tx(bar, (uint32_t)(nel * (L::GE + L::CE) * sizeof(double)));
    tma_bulk_g2s_hint(sG, prm.qd + (size_t)e0 * L::GE, (uint32_t)(nel * L::GE * sizeof(double)), bar, once);
    tma_bulk_g2s_hint(sC, prm.ecoef + (size_t)e0 * L::CE, (uint32_t)(nel * L::CE * sizeof(double)), bar, once);
  }
  const int32_t *li = prm.lidx + (size_t)e0 * prm.PS;
  for (int w = tid; w < NE * P; w += NT)
  {
    const int e = w / P, l = w % P;
    sU[e * P + l] = e < nel ? gather1(prm.x, li[(size_t)e * prm.PS + l]) : 0.0;
  }
  __syncthreads();  // (also publishes the initialised barrier before anyone polls it)

  rt7_phase_all<P_, NE, 0, NTC>(prm, sm, comp, t);
  rt7_phase_all<P_, NE, 1, NTC>(prm, sm, comp, t);
  rt7_phase_all<P_, NE, 2, NTC>(prm, sm, comp, t);

  // D: one thread per point, in the x-slowest order of the q-data
  mbar_wait(bar, 0);
  double *sV = sm + L::OFF_V;
  for (int w = tid; w < nel * Q; w += NT)
  {
    const int e = w / Q, s = w % Q;
    const int qx = s / (q * q), qz = (s / q) % q, qy = s % q, iq = qx + q * (qy + q * qz);
    const double *g = sG + e * L::GE + s, *Cm = sC + e * L::CE;
    double A[9], Jd[9], C[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
      A[i] = g[(1 + i) * Q];
      C[i] = Cm[i];
    }
    cofactor33(A, Jd);
    double *v0 = sV + e * Q + iq, *v1 = v0 + NE * Q, *v2 = v1 + NE * Q;
    const double u[3] = {*v0, *v1, *v2};
    double v[3];
    AtCAx(Jd, C, u, g[0], v);
    *v0 = v[0];
    *v1 = v[1];
    *v2 = v[2];
  }
  __syncthreads();

  rt7_phase_all<P_, NE, 3, NTC>(prm, sm, comp, t);
  rt7_phase_all<P_, NE, 4, NTC>(prm, sm, comp, t);
  rt7_phase_all<P_, NE, 5, NTC>(prm, sm, comp, t);

  // scatter: RED.F64 for every entry; masked entries (and the empty slots of a ragged batch) add 0.0 to this thread's sink slot
  double *my_sink = prm.sink + ((blockIdx.x * NT + tid) & (b2p_ctx::SINK_SLOTS - 1));
  for (int w = tid; w < nel * P; w += NT)
  {
    const int e = w / P, l = w % P;
    const int32_t gi = li[(size_t)e * prm.PS + l];
    const double v = prm.alpha * sU[e * P + l];
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

// ---- diagonal -----------------------------------------------------------------------------------------------------------

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

RTParams make_rt_params(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, int e_off, int e_cnt)
{
  RTParams prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.tab = op->tab;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.ecoef = op->ecoef + 18 * (size_t)e_off;
  prm.x = x;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  prm.PS = op->PS;
  return prm;
}

template <int P_, int Q_>
int launch_rt_pq(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, int e_off, int e_cnt, cudaStream_t s)
{
  using L = RTLayout<P_, Q_>;
  constexpr int per_elem_bytes = L::PER_ELEM * 8;
  constexpr int NEB = (per_elem_bytes * 8 <= 100 * 1024) ? 8 : (per_elem_bytes * 4 <= 100 * 1024) ? 4
                      : (per_elem_bytes * 2 <= 200 * 1024) ? 2 : 1;
  constexpr int NT = 256;
  const size_t shmem = (size_t)(Q_ * P_ + Q_ * (P_ + 1) + NEB * L::PER_ELEM) * sizeof(double);
  auto kern = rt_hex_apply_kernel<P_, Q_, NEB, NT>;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  B2P_LAUNCH(kern, (e_cnt + NEB - 1) / NEB, NT, shmem, s, make_rt_params(op, lidx, alpha, x, y, e_off, e_cnt));
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

template <int P_>
int launch_rt7(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, int e_off, int e_cnt, cudaStream_t s)
{
  using S = RT7Shape<P_>;
  using L = RT7Layout<P_, S::NE>;
  constexpr int NT = 3 * S::WPC * 32;
  auto kern = rt_hex_apply7_kernel<P_, S::NE, S::WPC, S::MINB>;
  if (int rc = configure_kernel(op->ctx, kern, L::SMEM_BYTES)) return rc;
  RT7Params<P_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * L::GE;
  prm.ecoef = op->ecoef + L::CE * (size_t)e_off;
  prm.x = x;
  prm.y = y;
  prm.sink = op->ctx->d_sink;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  prm.PS = op->PS;
  copy_tables(op->h_tab.data(), P_, P_ + 1, P_ + 1, prm.Bo, prm.Bc, nullptr);
  B2P_LAUNCH(kern, (e_cnt + S::NE - 1) / S::NE, NT, L::SMEM_BYTES, s, prm);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace

bool rt_hex_apply7_eligible(b2p_op *op)
{
  // the same test as nd_hex_apply7_eligible: q1d = p + 1, p = 2 ... 6, tables mirror-symmetric within 8e-15 of the largest entry
  if (!op || op->kind != B2P_RT_MASS || op->dense || !op->ecoef) return false;
  if (!(op->q1d == op->p + 1 && op->p >= 2 && op->p <= 6)) return false;
  return nd_tables_symmetric(op, 8e-15);
}

int launch_rt_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                        bool rt7)
{
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  static const bool trace = std::getenv("B2P_TRACE_KERNEL") != nullptr;
  if (rt7)
  {
    if (trace) fprintf(stderr, "[b2p] rt_hex_apply7 p=%d q1d=%d ne=%d\n", op->p, op->q1d, e_cnt);
#define B2P_CASE(PP) \
  if (op->p == PP) return launch_rt7<PP>(op, lidx, alpha, x, y, e_off, e_cnt, s);
    B2P_CASE(2) B2P_CASE(3) B2P_CASE(4) B2P_CASE(5) B2P_CASE(6)
#undef B2P_CASE
  }
  if (trace) fprintf(stderr, "[b2p] rt_hex_apply p=%d q1d=%d ne=%d\n", op->p, op->q1d, e_cnt);
#define B2P_CASE(PP, QQ) \
  if (op->p == PP && op->q1d == QQ) return launch_rt_pq<PP, QQ>(op, lidx, alpha, x, y, e_off, e_cnt, s);
  B2P_CASE(1, 2) B2P_CASE(1, 3) B2P_CASE(1, 4) B2P_CASE(1, 5) B2P_CASE(1, 6) B2P_CASE(1, 7)
  B2P_CASE(2, 3) B2P_CASE(2, 4) B2P_CASE(2, 5) B2P_CASE(2, 6) B2P_CASE(2, 7)
  B2P_CASE(3, 4) B2P_CASE(3, 5) B2P_CASE(3, 6) B2P_CASE(3, 7)
  B2P_CASE(4, 5) B2P_CASE(4, 6) B2P_CASE(4, 7)
  B2P_CASE(5, 6) B2P_CASE(5, 7)
  B2P_CASE(6, 7)
#undef B2P_CASE
  set_error(op->ctx, "rt_hex_apply: no kernel for p=%d q1d=%d", op->p, op->q1d);
  return B2P_ERR_UNSUPPORTED;
}

int launch_rt_hex_diag(b2p_op *op, double *diag, cudaStream_t s)
{
  const size_t total = (size_t)op->ne * op->P;
  const int nt = 128;
  B2P_LAUNCH(rt_hex_diag_kernel, (unsigned)((total + nt - 1) / nt), nt, 0, s, make_rt_params(op, op->lidx, 1.0, nullptr, diag, 0, op->ne),
             op->p, op->q1d);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p
