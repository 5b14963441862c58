// Matrix-free H1 hexahedron diffusion operator (the auxiliary-space operator of the Hiptmair
// smoother): y_L += sum_e E^T G^T D G E x_L with D = w detJ J^-1 C J^-T, i.e. f_apply_hcurl_33 on
// the reference gradient (/root/reference/palace/fem/integ/diffusion.cpp:16-73,
// /root/reference/palace/fem/qfunctions/33/hcurl_33_qf.h:10-29). Lexicographic tensor restriction
// (/root/reference/palace/fem/libceed/restriction.cpp:113-205), sum-factorised 1-D Gauss-Lobatto basis
// (/root/reference/palace/fem/libceed/basis.cpp:15-38).
#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"

namespace b2p
{

namespace
{

struct H1Params
{
  const int32_t *lidx;
  const double *tab;  // (unused Bo) | Bc[q][n] | Gc[q][n]
  const double *qd;
  const double *mat;
  const int32_t *emat;
  const double *aq;
  const double *x;
  double *y;
  double alpha;
  int64_t aq_estride;
  int ne;
  int PS;  // padded restriction row stride
  VSplit sp;
};

template <int P_, int Q_>
struct H1Layout
{
  static constexpr int p = P_, q = Q_, n = P_ + 1;
  static constexpr int P = n * n * n, Q = q * q * q;
  static constexpr int N1 = q * n * n, N2 = q * q * n;
  // U | T1a T1b | T2a T2b T2c | g[3Q]
  static constexpr int PER_ELEM = P + 2 * N1 + 3 * N2 + 3 * Q;
};

template <int P_, int Q_, bool ASM, int NEB, int NT>
__global__ void __launch_bounds__(NT) h1_hex_diffusion_kernel(H1Params prm)
{
  using L = H1Layout<P_, Q_>;
  constexpr int p = L::p, q = L::q, n = L::n, P = L::P, Q = L::Q, N1 = L::N1, N2 = L::N2, ES = L::PER_ELEM;
  B2P_DYN_SMEM(double, smem);
  double *sBc = smem;
  double *sGc = sBc + q * n;
  double *U = sGc + q * n;
  double *T1a = U + P, *T1b = T1a + N1;
  double *T2a = T1b + N1, *T2b = T2a + N2, *T2c = T2b + N2;
  double *gq = T2c + N2;
  for (int i = threadIdx.x; i < 2 * q * n; i += NT) sBc[i] = prm.tab[q * p + i];
  const int e0 = blockIdx.x * NEB;
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    double v = 0.0;
    if (e0 + e < prm.ne)
    {
      v = gather2(prm.x, prm.sp, prm.lidx[(size_t)(e0 + e) * prm.PS + l]);
    }
    U[e * ES + l] = v;
  }
  __syncthreads();
  // forward gradient
  contract<0, n, n, n, n, q, false, NEB, NT>(U, ES, T1a, ES, sBc, n, 1, 1.0);
  contract<0, n, n, n, n, q, false, NEB, NT>(U, ES, T1b, ES, sGc, n, 1, 1.0);
  __syncthreads();
  contract<1, q, n, n, n, q, false, NEB, NT>(T1a, ES, T2a, ES, sBc, n, 1, 1.0);  // B B
  contract<1, q, n, n, n, q, false, NEB, NT>(T1a, ES, T2c, ES, sGc, n, 1, 1.0);  // B G
  contract<1, q, n, n, n, q, false, NEB, NT>(T1b, ES, T2b, ES, sBc, n, 1, 1.0);  // G B
  __syncthreads();
  contract<2, q, q, n, n, q, false, NEB, NT>(T2b, ES, gq + 0 * Q, ES, sBc, n, 1, 1.0);
  contract<2, q, q, n, n, q, false, NEB, NT>(T2c, ES, gq + 1 * Q, ES, sBc, n, 1, 1.0);
  contract<2, q, q, n, n, q, false, NEB, NT>(T2a, ES, gq + 2 * Q, ES, sGc, n, 1, 1.0);
  __syncthreads();
  for (int w = threadIdx.x; w < NEB * Q; w += NT)
  {
    const int e = w / Q, iq = w % Q, sq = qslot_of(q, iq);
    if (e0 + e >= prm.ne) continue;
    double *ge = gq + e * ES;
    const double u0 = ge[iq], u1 = ge[Q + iq], u2 = ge[2 * Q + iq];
    if (ASM)
    {
      const double *a = prm.aq + (size_t)(e0 + e) * prm.aq_estride + sq;
      ge[iq] = a[0 * Q] * u0 + a[3 * Q] * u1 + a[6 * Q] * u2;
      ge[Q + iq] = a[1 * Q] * u0 + a[4 * Q] * u1 + a[7 * Q] * u2;
      ge[2 * Q + iq] = a[2 * Q] * u0 + a[5 * Q] * u1 + a[8 * Q] * u2;
    }
    else
    {
      const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + sq;
      double A[9], C[9], u[3] = {u0, u1, u2}, v[3];
#pragma unroll
      for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
      const int m = prm.emat[2 * (size_t)(e0 + e)];
#pragma unroll
      for (int i = 0; i < 9; i++) C[i] = __ldg(prm.mat + 9 * m + i);
      AtCAx(A, C, u, g[0], v);
      ge[iq] = v[0];
      ge[Q + iq] = v[1];
      ge[2 * Q + iq] = v[2];
    }
  }
  __syncthreads();
  // transpose
  contract<2, q, q, q, q, n, false, NEB, NT>(gq + 0 * Q, ES, T2b, ES, sBc, 1, n, 1.0);
  contract<2, q, q, q, q, n, false, NEB, NT>(gq + 1 * Q, ES, T2c, ES, sBc, 1, n, 1.0);
  contract<2, q, q, q, q, n, false, NEB, NT>(gq + 2 * Q, ES, T2a, ES, sGc, 1, n, 1.0);
  __syncthreads();
  contract<1, q, q, n, q, n, false, NEB, NT>(T2a, ES, T1a, ES, sBc, 1, n, 1.0);
  contract<1, q, q, n, q, n, true, NEB, NT>(T2c, ES, T1a, ES, sGc, 1, n, 1.0);
  contract<1, q, q, n, q, n, false, NEB, NT>(T2b, ES, T1b, ES, sBc, 1, n, 1.0);
  __syncthreads();
  contract<0, q, n, n, q, n, false, NEB, NT>(T1a, ES, U, ES, sBc, 1, n, 1.0);
  contract<0, q, n, n, q, n, true, NEB, NT>(T1b, ES, U, ES, sGc, 1, n, 1.0);
  __syncthreads();
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    if (e0 + e >= prm.ne) continue;
    scatter2(prm.y, prm.sp, prm.lidx[(size_t)(e0 + e) * prm.PS + l], prm.alpha * U[e * ES + l]);
  }
}

__global__ void h1_hex_diag_kernel(H1Params prm, int p, int q, bool assembled)
{
  const int n = p + 1, P = n * n * n, Q = q * q * q;
  const double *Bc = prm.tab + q * p, *Gc = Bc + q * n;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)prm.ne * P) return;
  const int e = (int)(w / P), l = (int)(w % P);
  const int i = l % n, j = (l / n) % n, k = l / (n * n);
  double C[9];
  if (!assembled)
    for (int t = 0; t < 9; t++) C[t] = prm.mat[9 * prm.emat[2 * (size_t)e] + t];
  double s = 0.0;
  for (int qz = 0; qz < q; qz++)
    for (int qy = 0; qy < q; qy++)
      for (int qx = 0; qx < q; qx++)
      {
        const int iq = qslot(q, qx, qy, qz);
        double u[3] = {Gc[qx * n + i] * Bc[qy * n + j] * Bc[qz * n + k], Bc[qx * n + i] * Gc[qy * n + j] * Bc[qz * n + k],
                       Bc[qx * n + i] * Bc[qy * n + j] * Gc[qz * n + k]};
        if (assembled)
        {
          const double *a = prm.aq + (size_t)e * prm.aq_estride + iq;
          for (int rr = 0; rr < 3; rr++)
            for (int cc = 0; cc < 3; cc++) s += u[rr] * a[(rr + 3 * cc) * Q] * u[cc];
        }
        else
        {
          const double *g = prm.qd + (size_t)e * 10 * Q + iq;
          double A[9], v[3];
          for (int t = 0; t < 9; t++) A[t] = g[(1 + t) * Q];
          AtCAx(A, C, u, g[0], v);
          s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
        }
      }
  int gi = prm.lidx[(size_t)e * prm.PS + l];
  if (gi == B2P_SKIP_IDX) return;
  if (gi < 0) gi = -1 - gi;
  atomicAdd(prm.y + gi, s);
}

H1Params make_params(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg = ApplyRange())
{
  H1Params prm;
  const int e_off = rg.e_off, e_cnt = rg.e_cnt < 0 ? op->ne - rg.e_off : rg.e_cnt;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.alpha = alpha;
  prm.sp.n_owned = rg.n_owned < 0 ? op->lsize : rg.n_owned;
  prm.sp.xg = rg.xg;
  prm.sp.yg = rg.yg;
  prm.aq_estride = op->aq_estride;
  prm.PS = op->PS;
  prm.tab = op->tab;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.mat = op->mat;
  prm.emat = op->emat + 2 * (size_t)e_off;
  prm.aq = op->aq ? op->aq + (size_t)e_off * op->aq_estride : nullptr;
  prm.x = x;
  prm.y = y;
  prm.ne = e_cnt;
  return prm;
}

template <int P_, int Q_, bool ASM>
int launch_pq(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  using L = H1Layout<P_, Q_>;
  constexpr int per_elem_bytes = L::PER_ELEM * 8;
  constexpr int NEB = (per_elem_bytes * 8 <= 100 * 1024) ? 8 : (per_elem_bytes * 4 <= 100 * 1024) ? 4
                      : (per_elem_bytes * 2 <= 200 * 1024) ? 2 : 1;
  constexpr int NT = 256;
  const size_t shmem = (size_t)(2 * Q_ * (P_ + 1) + NEB * L::PER_ELEM) * sizeof(double);
  auto kern = h1_hex_diffusion_kernel<P_, Q_, ASM, NEB, NT>;
  const int ne_run = range_count(op, rg);
  if (ne_run <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  B2P_LAUNCH(kern, (ne_run + NEB - 1) / NEB, NT, shmem, s, make_params(op, lidx, alpha, x, y, rg));
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace

int launch_h1_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
#define B2P_CASE(PP, QQ)                                                                              \
  if (op->p == PP && op->q1d == QQ)                                                                   \
    return op->assembled ? launch_pq<PP, QQ, true>(op, lidx, alpha, x, y, rg, s) : launch_pq<PP, QQ, false>(op, lidx, alpha, x, y, rg, s);
  B2P_CASE(1, 2) B2P_CASE(1, 3) B2P_CASE(1, 4) B2P_CASE(1, 5) B2P_CASE(1, 6) B2P_CASE(1, 7)
  B2P_CASE(2, 3) B2P_CASE(2, 4) B2P_CASE(2, 5) B2P_CASE(2, 6) B2P_CASE(2, 7)
  B2P_CASE(3, 4) B2P_CASE(3, 5) B2P_CASE(3, 6) B2P_CASE(3, 7)
  B2P_CASE(4, 5) B2P_CASE(4, 6) B2P_CASE(4, 7)
  B2P_CASE(5, 6) B2P_CASE(5, 7)
  B2P_CASE(6, 7)
#undef B2P_CASE
  set_error(op->ctx, "h1_hex_apply: no kernel for p=%d q1d=%d", op->p, op->q1d);
  return B2P_ERR_UNSUPPORTED;
}

int launch_h1_hex_diag(b2p_op *op, double *diag, cudaStream_t s)
{
  H1Params prm = make_params(op, op->lidx, 1.0, nullptr, diag);
  const size_t total = (size_t)op->ne * op->P;
  const int nt = 128;
  B2P_LAUNCH(h1_hex_diag_kernel, (unsigned)((total + nt - 1) / nt), nt, 0, s, prm, op->p, op->q1d, op->assembled);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p
