// Element-local tensor-product interpolation between two hexahedral spaces on the same mesh:
// the p-multigrid prolongation (ND->ND, H1->H1) and the discrete gradient (H1->ND).
// Reference: DiscreteLinearOperator::PartialAssemble (/root/reference/palace/fem/bilinearform.cpp:203-282)
// builds one element-dense [P_test x P_trial] matrix from GetTransferMatrix/ProjectGrad
// (/root/reference/palace/fem/libceed/basis.cpp:116-165) and applies it through libCEED with an
// identity QFunction (/root/reference/palace/fem/libceed/integrator.cpp:515-548); the output is scaled
// by the inverse dof multiplicity on Mult and the input on MultTranspose
// (/root/reference/palace/fem/libceed/operator.cpp:182-212). On hexes that dense matrix is a Kronecker
// product of 1-D matrices per vector component; it is applied here in that factored form. The discrete curl ND_p -> RT_{p-1}
// (CurlInterpolator, fespace.cpp:204,216) is a sum of two such products per output component, each reading a different
// input block; it has a kernel of its own (curl_hex_kernel) that applies both in one pass.
#include <algorithm>
#include <cstdlib>

#include "b2p_internal.hpp"
#include "b2p_contract.cuh"


namespace b2p
{

namespace
{

struct InterpParams
{
  int owner;  // Mult: out_lidx keeps every output dof in one element only -> plain read-modify-write, no 1/multiplicity
  const int32_t *in_lidx, *out_lidx;
  const double *inv_mult, *mats, *x;
  double *y;
  double alpha;
  int ne, in_P, out_P, in_PS, out_PS, ncomp, n_mats;
  int in_off[3], in_n[3][3], out_off[3], out_n[3][3], mat_off[3][3];
  int ident[3][3];  // 1-D factor is the identity: skip its loop
};

// y[out] += alpha * inv_mult[out] * sum_e E_out^T (Ax (x) Ay (x) Az) E_in x
template <bool TRANSPOSE>
__global__ void interp_kernel(InterpParams prm, int neb)
{
  B2P_DYN_SMEM(double, sm);
  double *smat = sm;                 // [n_mats]
  double *sv = sm + prm.n_mats;      // [neb][src_P]
  const int src_P = TRANSPOSE ? prm.out_P : prm.in_P;
  const int dst_P = TRANSPOSE ? prm.in_P : prm.out_P;
  const int src_PS = TRANSPOSE ? prm.out_PS : prm.in_PS;
  const int dst_PS = TRANSPOSE ? prm.in_PS : prm.out_PS;
  const int32_t *src_lidx = TRANSPOSE ? prm.out_lidx : prm.in_lidx;
  const int32_t *dst_lidx = TRANSPOSE ? prm.in_lidx : prm.out_lidx;
  for (int i = threadIdx.x; i < prm.n_mats; i += blockDim.x) smat[i] = prm.mats[i];
  const int e0 = blockIdx.x * neb;
  for (int w = threadIdx.x; w < neb * src_P; w += blockDim.x)
  {
    const int e = w / src_P, l = w % src_P;
    double v = 0.0;
    if (e0 + e < prm.ne)
    {
      const int32_t gi = src_lidx[(size_t)(e0 + e) * src_PS + l];
      v = gather1(prm.x, gi);
      if (TRANSPOSE && gi != B2P_SKIP_IDX) v *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
    }
    sv[w] = v;
  }
  __syncthreads();
  for (int w = threadIdx.x; w < neb * dst_P; w += blockDim.x)
  {
    const int e = w / dst_P, l = w % dst_P;
    if (e0 + e >= prm.ne) continue;
    if (!TRANSPOSE && prm.owner && dst_lidx[(size_t)(e0 + e) * dst_PS + l] == B2P_SKIP_IDX) continue;  // another element owns it
    // component of the destination dof
    int c = 0;
    if (!TRANSPOSE)
    {
      while (c + 1 < prm.ncomp && l >= prm.out_off[c + 1]) c++;
    }
    else
    {
      // transposed: destination lives in the input space; with one input block shared by all
      // components (discrete gradient) every component contributes.
      c = -1;
    }
    const double *src = sv + e * src_P;
    double s = 0.0;
    if (!TRANSPOSE)
    {
      const int r = l - prm.out_off[c];
      const int ox = prm.out_n[c][0], oy = prm.out_n[c][1];
      const int i = r % ox, j = (r / ox) % oy, k = r / (ox * oy);
      const int nx = prm.in_n[c][0], ny = prm.in_n[c][1], nz = prm.in_n[c][2];
      const double *Ax = smat + prm.mat_off[c][0] + i * nx;
      const double *Ay = smat + prm.mat_off[c][1] + j * ny;
      const double *Az = smat + prm.mat_off[c][2] + k * nz;
      const double *in = src + prm.in_off[c];
      const bool ix = prm.ident[c][0], iy = prm.ident[c][1], iz = prm.ident[c][2];
      const int k0 = iz ? k : 0, k1 = iz ? k + 1 : nz, j0 = iy ? j : 0, j1 = iy ? j + 1 : ny, i0 = ix ? i : 0, i1 = ix ? i + 1 : nx;
      for (int kk = k0; kk < k1; kk++)
      {
        double sy = 0.0;
        for (int jj = j0; jj < j1; jj++)
        {
          double sx = 0.0;
          for (int ii = i0; ii < i1; ii++) sx += Ax[ii] * in[ii + nx * (jj + ny * kk)];
          sy += Ay[jj] * sx;
        }
        s += Az[kk] * sy;
      }
      const int32_t gi = dst_lidx[(size_t)(e0 + e) * dst_PS + l];
      if (prm.owner)
      {
        // conforming interpolation: every element containing the dof computes the same value; its owner writes it
        if (gi >= 0)
          prm.y[gi] += prm.alpha * s;
        else
          prm.y[-1 - gi] -= prm.alpha * s;
      }
      else
      {
        if (gi != B2P_SKIP_IDX) s *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
        scatter1(prm.y, gi, prm.alpha * s);
      }
    }
    else
    {
      for (int cc = 0; cc < prm.ncomp; cc++)
      {
        const int nx = prm.in_n[cc][0], ny = prm.in_n[cc][1], nz = prm.in_n[cc][2];
        const int r = l - prm.in_off[cc];
        if (r < 0 || r >= nx * ny * nz) continue;
        const int ii = r % nx, jj = (r / nx) % ny, kk = r / (nx * ny);
        const int ox = prm.out_n[cc][0], oy = prm.out_n[cc][1], oz = prm.out_n[cc][2];
        const double *Ax = smat + prm.mat_off[cc][0] + ii;   // column ii, stride nx
        const double *Ay = smat + prm.mat_off[cc][1] + jj;
        const double *Az = smat + prm.mat_off[cc][2] + kk;
        const double *out = src + prm.out_off[cc];
        const bool ix = prm.ident[cc][0], iy = prm.ident[cc][1], iz = prm.ident[cc][2];
        const int k0 = iz ? kk : 0, k1 = iz ? kk + 1 : oz, j0 = iy ? jj : 0, j1 = iy ? jj + 1 : oy, i0 = ix ? ii : 0, i1 = ix ? ii + 1 : ox;
        for (int k = k0; k < k1; k++)
        {
          double sy = 0.0;
          for (int j = j0; j < j1; j++)
          {
            double sx = 0.0;
            for (int i = i0; i < i1; i++) sx += Ax[i * nx] * out[i + ox * (j + oy * k)];
            sy += Ay[j * ny] * sx;
          }
          s += Az[k * nz] * sy;
        }
      }
      scatter1(prm.y, dst_lidx[(size_t)(e0 + e) * dst_PS + l], prm.alpha * s);
    }
  }
}

// Element-dense interpolator for any element type (tets: p-prolongation and discrete gradient from
// GetTransferMatrix / ProjectGrad, basis.cpp:116-165): y_L += alpha * (1/mult) E_out^T ( M E_in x_L ), with the
// restrictions' tridiagonal transformations when the spaces need them (domain side: InvTransformPrimal rows, range side:
// InvTransformDual rows, restriction.cpp:301-329). Transposed: the input is scaled by 1/mult (operator.cpp:224-235).
struct DenseInterpParams
{
  const int32_t *in_lidx, *out_lidx;
  const int8_t *in_co, *out_co;
  const double *inv_mult, *M, *x;
  double *y;
  double alpha;
  int ne, in_P, out_P, in_PS, out_PS;
};
constexpr int DI_NEB = 8;

// v <- T v (rows co[i] = {T(i,i-1), T(i,i), T(i,i+1)}) or v <- T^T v, for the element slots of one block
__device__ __forceinline__ void tri_apply(const int8_t *co, int P, bool transpose, const double *src, double *dst, int ne_blk, int e0, int ne)
{
  for (int w = threadIdx.x; w < ne_blk * P; w += blockDim.x)
  {
    const int e = w / P, i = w % P;
    double v = 0.0;
    if (e0 + e < ne)
    {
      const int8_t *c = co + (size_t)(e0 + e) * P * 3;
      const double *s = src + e * P;
      if (!transpose)
      {
        v = (double)c[3 * i + 1] * s[i];
        if (i > 0) v += (double)c[3 * i + 0] * s[i - 1];
        if (i < P - 1) v += (double)c[3 * i + 2] * s[i + 1];
      }
      else
      {
        v = (double)c[3 * i + 1] * s[i];
        if (i > 0) v += (double)c[3 * (i - 1) + 2] * s[i - 1];
        if (i < P - 1) v += (double)c[3 * (i + 1) + 0] * s[i + 1];
      }
    }
    dst[w] = v;
  }
}

template <bool TRANSPOSE>
__global__ void __launch_bounds__(256) dense_interp_kernel(DenseInterpParams prm)
{
  B2P_DYN_SMEM(double, sm);
  const int src_P = TRANSPOSE ? prm.out_P : prm.in_P, dst_P = TRANSPOSE ? prm.in_P : prm.out_P;
  const int src_PS = TRANSPOSE ? prm.out_PS : prm.in_PS, dst_PS = TRANSPOSE ? prm.in_PS : prm.out_PS;
  const int32_t *src_lidx = TRANSPOSE ? prm.out_lidx : prm.in_lidx, *dst_lidx = TRANSPOSE ? prm.in_lidx : prm.out_lidx;
  // the transformation that acts on the gathered values, and the one that acts before the scatter:
  //   Mult:       u = T_in x_e            ...  z = D_out^T (M u)
  //   Transpose:  u = D_out (x_e / mult)  ...  z = T_in^T (M^T u)
  const int8_t *src_co = TRANSPOSE ? prm.out_co : prm.in_co, *dst_co = TRANSPOSE ? prm.in_co : prm.out_co;
  const int PM = src_P > dst_P ? src_P : dst_P;
  double *a = sm, *b = sm + DI_NEB * PM;  // two [NEB][PM] work vectors
  const int e0 = blockIdx.x * DI_NEB;
  for (int w = threadIdx.x; w < DI_NEB * src_P; w += blockDim.x)
  {
    const int e = w / src_P, l = w % src_P;
    double v = 0.0;
    if (e0 + e < prm.ne)
    {
      const int32_t gi = src_lidx[(size_t)(e0 + e) * src_PS + l];
      v = gather1(prm.x, gi);
      if (TRANSPOSE && gi != B2P_SKIP_IDX) v *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
    }
    a[w] = v;
  }
  __syncthreads();
  const double *u = a;
  if (src_co)
  {
    tri_apply(src_co, src_P, false, a, b, DI_NEB, e0, prm.ne);
    __syncthreads();
    u = b;
  }
  double *r = (u == a) ? b : a;  // result of the dense product
  for (int w = threadIdx.x; w < DI_NEB * dst_P; w += blockDim.x)
  {
    const int e = w / dst_P, i = w % dst_P;
    double s = 0.0;
    if (e0 + e < prm.ne)
    {
      const double *ue = u + e * src_P;
      if (!TRANSPOSE)
      {
        const double *row = prm.M + (size_t)i * prm.in_P;
        for (int j = 0; j < src_P; j++) s += row[j] * ue[j];
      }
      else
      {
        const double *col = prm.M + i;
        for (int j = 0; j < src_P; j++) s += col[(size_t)j * prm.in_P] * ue[j];
      }
    }
    r[w] = s;
  }
  __syncthreads();
  const double *z = r;
  if (dst_co)
  {
    double *t = (r == a) ? b : a;
    tri_apply(dst_co, dst_P, true, r, t, DI_NEB, e0, prm.ne);
    __syncthreads();
    z = t;
  }
  for (int w = threadIdx.x; w < DI_NEB * dst_P; w += blockDim.x)
  {
    const int e = w / dst_P, l = w % dst_P;
    if (e0 + e >= prm.ne) continue;
    const int32_t gi = dst_lidx[(size_t)(e0 + e) * dst_PS + l];
    double v = prm.alpha * z[w];
    if (!TRANSPOSE && gi != B2P_SKIP_IDX) v *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
    scatter1(prm.y, gi, v);
  }
}

// Discrete curl C : ND_p -> RT_{p-1} on hexahedra (mfem ProjectCurl, hexspace.discrete_curl_matrix), lexicographic on both
// sides. ND component b is open (p Gauss-Legendre nodes) along axis b and closed (p + 1 Gauss-Lobatto nodes) along the other
// two; RT component c is closed along c and open along the other two. For (c, a, b) cyclic, RT_c = D_a u_b - D_b u_a, where
// D [p][p+1] is the derivative of the closed 1-D basis at the open nodes acting along one axis, the identity along the rest:
// 2 (p + 1) FMAs per RT dof on Mult, 2 p per ND dof on MultTranspose, no element matrix.
template <int P>
struct CurlHex
{
  static constexpr int N = P + 1;
  static constexpr int ND_BLK = P * N * N, RT_BLK = N * P * P;
  static constexpr int ND_P = 3 * ND_BLK, RT_P = 3 * RT_BLK;
  // extent of ND block b / RT block c along axis d, and its stride (x fastest)
  static constexpr int nd_n(int b, int d) { return d == b ? P : N; }
  static constexpr int rt_n(int c, int d) { return d == c ? N : P; }
  static constexpr int nd_stride(int b, int d) { return d == 0 ? 1 : d == 1 ? nd_n(b, 0) : nd_n(b, 0) * nd_n(b, 1); }
  static constexpr int rt_stride(int c, int d) { return d == 0 ? 1 : d == 1 ? rt_n(c, 0) : rt_n(c, 0) * rt_n(c, 1); }
};
constexpr int CURL_HEX_PMAX = 6;
constexpr int CURL_HEX_NT = 256;
// elements per block: at least two destination dofs per thread
constexpr int curl_hex_neb(int dst_P) { return (2 * CURL_HEX_NT + dst_P - 1) / dst_P; }

// RT component C at offset r inside its block, from the ND element vector u
template <int P, int C>
__device__ __forceinline__ double curl_rt_comp(const double *u, const double *D, int r)
{
  using H = CurlHex<P>;
  constexpr int A = (C + 1) % 3, B = (C + 2) % 3;
  constexpr int n0 = H::rt_n(C, 0), n1 = H::rt_n(C, 1);
  const int ix[3] = {r % n0, (r / n0) % n1, r / (n0 * n1)};
  // D_a u_b runs over u_b's closed index along a; D_b u_a over u_a's closed index along b
  int jb[3] = {ix[0], ix[1], ix[2]}, ja[3] = {ix[0], ix[1], ix[2]};
  jb[A] = 0;
  ja[B] = 0;
  const double *ub = u + B * H::ND_BLK + jb[0] * H::nd_stride(B, 0) + jb[1] * H::nd_stride(B, 1) + jb[2] * H::nd_stride(B, 2);
  const double *ua = u + A * H::ND_BLK + ja[0] * H::nd_stride(A, 0) + ja[1] * H::nd_stride(A, 1) + ja[2] * H::nd_stride(A, 2);
  const double *Da = D + ix[A] * H::N, *Db = D + ix[B] * H::N;
  double s = 0.0;
#pragma unroll
  for (int t = 0; t < H::N; t++) s += Da[t] * ub[t * H::nd_stride(B, A)] - Db[t] * ua[t * H::nd_stride(A, B)];
  return s;
}

// ND component B at offset r inside its block, from the RT element vector v (transpose): u_B feeds RT_{A2} through D_{A1}
// with sign -1 and RT_{A1} through D_{A2} with sign +1, for A1 = B + 1 and A2 = B + 2 (mod 3)
template <int P, int B>
__device__ __forceinline__ double curl_nd_comp(const double *v, const double *D, int r)
{
  using H = CurlHex<P>;
  constexpr int A1 = (B + 1) % 3, A2 = (B + 2) % 3;
  constexpr int n0 = H::nd_n(B, 0), n1 = H::nd_n(B, 1);
  const int ix[3] = {r % n0, (r / n0) % n1, r / (n0 * n1)};
  int jp[3] = {ix[0], ix[1], ix[2]}, jm[3] = {ix[0], ix[1], ix[2]};
  jp[A2] = 0;
  jm[A1] = 0;
  const double *vp = v + A1 * H::RT_BLK + jp[0] * H::rt_stride(A1, 0) + jp[1] * H::rt_stride(A1, 1) + jp[2] * H::rt_stride(A1, 2);
  const double *vm = v + A2 * H::RT_BLK + jm[0] * H::rt_stride(A2, 0) + jm[1] * H::rt_stride(A2, 1) + jm[2] * H::rt_stride(A2, 2);
  const double *Dp = D + ix[A2], *Dm = D + ix[A1];  // column of D, stride N
  double s = 0.0;
#pragma unroll
  for (int t = 0; t < P; t++) s += Dp[t * H::N] * vp[t * H::rt_stride(A1, A2)] - Dm[t * H::N] * vm[t * H::rt_stride(A2, A1)];
  return s;
}

struct CurlParams
{
  const int32_t *nd_lidx, *rt_lidx;  // signed lexicographic restrictions [ne][PS]
  const double *inv_mult, *D, *x;    // inv_mult: of the RT space
  double *y;
  double alpha;
  int ne, nd_PS, rt_PS;
};

// Mult:           y_rt += alpha (1/mult_rt) sum_e E_rt^T C E_nd x
// MultTranspose:  y_nd += alpha sum_e E_nd^T C^T E_rt ((1/mult_rt) x)
template <int P, bool TRANSPOSE>
__global__ void __launch_bounds__(CURL_HEX_NT) curl_hex_kernel(CurlParams prm)
{
  using H = CurlHex<P>;
  constexpr int SRC = TRANSPOSE ? H::RT_P : H::ND_P, DST = TRANSPOSE ? H::ND_P : H::RT_P;
  constexpr int NEB = curl_hex_neb(DST);
  __shared__ double sD[P * H::N];
  __shared__ double sv[NEB * SRC];
  const int32_t *src_lidx = TRANSPOSE ? prm.rt_lidx : prm.nd_lidx, *dst_lidx = TRANSPOSE ? prm.nd_lidx : prm.rt_lidx;
  const int src_PS = TRANSPOSE ? prm.rt_PS : prm.nd_PS, dst_PS = TRANSPOSE ? prm.nd_PS : prm.rt_PS;
  for (int i = threadIdx.x; i < P * H::N; i += CURL_HEX_NT) sD[i] = prm.D[i];
  const int e0 = blockIdx.x * NEB;
#pragma unroll
  for (int k = 0; k < (NEB * SRC + CURL_HEX_NT - 1) / CURL_HEX_NT; k++)
  {
    const int w = threadIdx.x + k * CURL_HEX_NT;
    if (w >= NEB * SRC) break;
    const int e = w / SRC, l = w - e * SRC;
    double v = 0.0;
    if (e0 + e < prm.ne)
    {
      const int32_t gi = src_lidx[(size_t)(e0 + e) * src_PS + l];
      v = gather1(prm.x, gi);
      if (TRANSPOSE && gi != B2P_SKIP_IDX) v *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
    }
    sv[w] = v;
  }
  __syncthreads();
  for (int w = threadIdx.x; w < NEB * DST; w += CURL_HEX_NT)
  {
    const int e = w / DST, l = w - e * DST;
    if (e0 + e >= prm.ne) break;
    const double *src = sv + e * SRC;
    constexpr int BLK = TRANSPOSE ? H::ND_BLK : H::RT_BLK;
    const int c = l / BLK, r = l - c * BLK;
    double s;
    if (!TRANSPOSE)
      s = c == 0 ? curl_rt_comp<P, 0>(src, sD, r) : c == 1 ? curl_rt_comp<P, 1>(src, sD, r) : curl_rt_comp<P, 2>(src, sD, r);
    else
      s = c == 0 ? curl_nd_comp<P, 0>(src, sD, r) : c == 1 ? curl_nd_comp<P, 1>(src, sD, r) : curl_nd_comp<P, 2>(src, sD, r);
    const int32_t gi = dst_lidx[(size_t)(e0 + e) * dst_PS + l];
    if (!TRANSPOSE && gi != B2P_SKIP_IDX) s *= prm.inv_mult[gi >= 0 ? gi : -1 - gi];
    scatter1(prm.y, gi, prm.alpha * s);
  }
}

template <int P, bool TRANSPOSE>
void curl_hex_launch(const CurlParams &prm, cudaStream_t s)
{
  constexpr int NEB = curl_hex_neb(TRANSPOSE ? CurlHex<P>::ND_P : CurlHex<P>::RT_P);
  void (*kern)(CurlParams) = curl_hex_kernel<P, TRANSPOSE>;
  B2P_LAUNCH(kern, (prm.ne + NEB - 1) / NEB, CURL_HEX_NT, 0, s, prm);
}

template <int P>
void curl_hex_launch(bool transpose, const CurlParams &prm, cudaStream_t s)
{
  if (transpose)
    curl_hex_launch<P, true>(prm, s);
  else
    curl_hex_launch<P, false>(prm, s);
}

int curl_hex_apply(const b2p_interp *it, bool transpose, double alpha, const double *x, double *y, cudaStream_t s)
{
  CurlParams prm;
  prm.nd_lidx = it->in_lidx;
  prm.rt_lidx = it->out_lidx;
  prm.inv_mult = it->inv_mult;
  prm.D = it->curl_D;
  prm.x = x;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = it->ne;
  prm.nd_PS = it->in_PS;
  prm.rt_PS = it->out_PS;
  switch (it->curl_p)
  {
    case 1: curl_hex_launch<1>(transpose, prm, s); break;
    case 2: curl_hex_launch<2>(transpose, prm, s); break;
    case 3: curl_hex_launch<3>(transpose, prm, s); break;
    case 4: curl_hex_launch<4>(transpose, prm, s); break;
    case 5: curl_hex_launch<5>(transpose, prm, s); break;
    case 6: curl_hex_launch<6>(transpose, prm, s); break;
    default: B2P_CHECK(it->ctx, false, B2P_ERR_UNSUPPORTED, "curl interpolator: p=%d", it->curl_p);
  }
  B2P_CUDA(it->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

InterpParams make_params(const b2p_interp *it, double alpha, const double *x, double *y)
{
  InterpParams p;
  p.owner = 0;
  p.in_lidx = it->in_lidx;
  p.out_lidx = it->out_lidx;
  p.inv_mult = it->inv_mult;
  p.mats = it->mats;
  p.x = x;
  p.y = y;
  p.alpha = alpha;
  p.ne = it->ne;
  p.in_P = it->in_P;
  p.out_P = it->out_P;
  p.in_PS = it->in_PS;
  p.out_PS = it->out_PS;
  p.ncomp = it->ncomp;
  p.n_mats = it->n_mats;
  for (int c = 0; c < 3; c++)
  {
    p.in_off[c] = it->in_off[c];
    p.out_off[c] = it->out_off[c];
    for (int d = 0; d < 3; d++)
    {
      p.in_n[c][d] = it->in_n[c][d];
      p.out_n[c][d] = it->out_n[c][d];
      p.mat_off[c][d] = it->mat_off[c][d];
      p.ident[c][d] = it->ident[c][d];
    }
  }
  return p;
}

int build_lidx(b2p_ctx *ctx, int ne, int P, int64_t lsize, const int32_t *idx, const int8_t *orient, const int32_t *dof_map,
               int *PS_out, int32_t **d_out, std::vector<int32_t> *host_out)
{
  const int PS = (P + 3) & ~3;
  *PS_out = PS;
  std::vector<int32_t> lidx((size_t)ne * PS, (int32_t)B2P_SKIP_IDX);
  for (int l = 0; l < P; l++)
  {
    int nat = dof_map ? dof_map[l] : l, sg = 1;
    if (nat < 0)
    {
      nat = -1 - nat;
      sg = -1;
    }
    B2P_CHECK(ctx, nat >= 0 && nat < P, B2P_ERR_ARG, "interp: dof_map[%d] out of range", l);
    for (int e = 0; e < ne; e++)
    {
      const int32_t gi = idx[(size_t)e * P + nat];
      B2P_CHECK(ctx, gi >= 0 && gi < lsize, B2P_ERR_ARG, "interp: idx out of range");
      const int s = sg * (orient ? (int)orient[(size_t)e * P + nat] : 1);
      lidx[(size_t)e * PS + l] = s >= 0 ? gi : -1 - gi;
    }
  }
  if (host_out) *host_out = lidx;
  return upload(ctx, lidx.data(), lidx.size(), d_out);
}

// 1 / (local elements touching the dof) of the output space, from its signed restriction
int upload_inv_mult(b2p_ctx *ctx, const std::vector<int32_t> &out_lidx, int64_t out_lsize, double **d_out)
{
  std::vector<double> mult((size_t)out_lsize, 0.0);
  for (int32_t g : out_lidx)
  {
    if (g == (int32_t)B2P_SKIP_IDX) continue;
    mult[g >= 0 ? g : -1 - g] += 1.0;
  }
  for (auto &m : mult) m = m > 0.0 ? 1.0 / m : 0.0;
  return upload(ctx, mult.data(), mult.size(), d_out);
}

}  // namespace

int interp_apply(const b2p_interp *it, bool transpose, double alpha, const double *x, double *y, cudaStream_t s)
{
  if (it->curl_p) return curl_hex_apply(it, transpose, alpha, x, y, s);
  if (it->dense)
  {
    DenseInterpParams dp;
    dp.in_lidx = it->in_lidx;
    dp.out_lidx = it->out_lidx;
    dp.in_co = it->in_co;
    dp.out_co = it->out_co;
    dp.inv_mult = it->inv_mult;
    dp.M = it->dmat;
    dp.x = x;
    dp.y = y;
    dp.alpha = alpha;
    dp.ne = it->ne;
    dp.in_P = it->in_P;
    dp.out_P = it->out_P;
    dp.in_PS = it->in_PS;
    dp.out_PS = it->out_PS;
    const size_t shmem = sizeof(double) * 2 * DI_NEB * (size_t)std::max(it->in_P, it->out_P);
    const int grid = (it->ne + DI_NEB - 1) / DI_NEB;
    if (transpose)
      B2P_LAUNCH(dense_interp_kernel<true>, grid, 256, shmem, s, dp);
    else
      B2P_LAUNCH(dense_interp_kernel<false>, grid, 256, shmem, s, dp);
    B2P_CUDA(it->ctx, cudaGetLastError());
    return B2P_SUCCESS;
  }
  InterpParams prm = make_params(it, alpha, x, y);
  if (!transpose && it->out_owner_lidx)
  {
    prm.owner = 1;
    prm.out_lidx = it->out_owner_lidx;
  }
  const int src_P = transpose ? it->out_P : it->in_P;
  // enough elements per block that every thread has at least two destination dofs
  const int dst_P = transpose ? it->in_P : it->out_P;
  int neb = std::max(1, (2 * 256 + dst_P - 1) / dst_P);
  neb = std::min(neb, 16);
  const size_t shmem = sizeof(double) * ((size_t)it->n_mats + (size_t)neb * src_P);
  const int grid = (it->ne + neb - 1) / neb;
  if (transpose)
    B2P_LAUNCH(interp_kernel<true>, grid, 256, shmem, s, prm, neb);
  else
    B2P_LAUNCH(interp_kernel<false>, grid, 256, shmem, s, prm, neb);
  B2P_CUDA(it->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p

using namespace b2p;

extern "C"
{

int b2p_interp_create(b2p_ctx *ctx, const b2p_interp_desc *d, b2p_interp **out)
{
  B2P_CHECK(ctx, ctx && d && out, B2P_ERR_ARG, "b2p_interp_create: null argument");
  B2P_CHECK(ctx, d->ncomp >= 1 && d->ncomp <= 3, B2P_ERR_ARG, "b2p_interp_create: ncomp must be 1..3");
  b2p_interp *it = new b2p_interp;
  it->ctx = ctx;
  it->ne = d->ne;
  it->in_P = d->in_P;
  it->out_P = d->out_P;
  it->in_lsize = d->in_lsize;
  it->out_lsize = d->out_lsize;
  it->ncomp = d->ncomp;
  int rc;
  std::vector<int32_t> out_host;
  if ((rc = build_lidx(ctx, d->ne, d->in_P, d->in_lsize, d->in_idx, d->in_orient, d->in_dof_map, &it->in_PS, &it->in_lidx, nullptr)))
    return rc;
  if ((rc = build_lidx(ctx, d->ne, d->out_P, d->out_lsize, d->out_idx, d->out_orient, d->out_dof_map, &it->out_PS, &it->out_lidx,
                       &out_host)))
    return rc;
  if ((rc = upload_inv_mult(ctx, out_host, d->out_lsize, &it->inv_mult))) return rc;
  // B2P_INTERP_OWNER=1 (opt-in until measured): Mult computes every output dof in its first element only (the
  // interpolators of a conforming hierarchy give the same value from every element; the reference averages them,
  // operator.cpp:186-189) -- ~44 % fewer outputs to form, no atomics, no multiplicity gather.
  {
    const char *env = std::getenv("B2P_INTERP_OWNER");
    if (env && env[0] == '1')
    {
      std::vector<char> seen((size_t)d->out_lsize, 0);
      std::vector<int32_t> own = out_host;
      for (auto &g : own)
      {
        if (g == (int32_t)B2P_SKIP_IDX) continue;
        const int32_t a = g >= 0 ? g : -1 - g;
        if (seen[a])
          g = (int32_t)B2P_SKIP_IDX;
        else
          seen[a] = 1;
      }
      if ((rc = upload(ctx, own.data(), own.size(), &it->out_owner_lidx))) return rc;
    }
  }
  std::vector<double> mats;
  for (int c = 0; c < d->ncomp; c++)
  {
    const b2p_interp_comp &cc = d->comps[c];
    it->in_off[c] = cc.in_off;
    it->out_off[c] = cc.out_off;
    for (int a = 0; a < 3; a++)
    {
      it->in_n[c][a] = cc.in_n[a];
      it->out_n[c][a] = cc.out_n[a];
      it->mat_off[c][a] = (int)mats.size();
      B2P_CHECK(ctx, cc.A[a], B2P_ERR_ARG, "b2p_interp_create: missing 1-D matrix");
      bool id = cc.out_n[a] == cc.in_n[a];
      for (int r = 0; id && r < cc.out_n[a]; r++)
        for (int q2 = 0; q2 < cc.in_n[a]; q2++) id = id && cc.A[a][(size_t)r * cc.in_n[a] + q2] == (r == q2 ? 1.0 : 0.0);
      it->ident[c][a] = id ? 1 : 0;
      mats.insert(mats.end(), cc.A[a], cc.A[a] + (size_t)cc.out_n[a] * cc.in_n[a]);
    }
  }
  it->n_mats = (int)mats.size();
  if ((rc = upload(ctx, mats.data(), mats.size(), &it->mats))) return rc;
  *out = it;
  return B2P_SUCCESS;
}

int b2p_interp_create_dense(b2p_ctx *ctx, const b2p_dense_interp_desc *d, b2p_interp **out)
{
  B2P_CHECK(ctx, ctx && d && out && d->in_idx && d->out_idx && d->mat, B2P_ERR_ARG, "b2p_interp_create_dense: null argument");
  B2P_CHECK(ctx, d->ne > 0 && d->in_P > 0 && d->out_P > 0, B2P_ERR_ARG, "b2p_interp_create_dense: empty");
  B2P_CHECK(ctx, sizeof(double) * 2 * DI_NEB * (size_t)std::max(d->in_P, d->out_P) <= 48 * 1024, B2P_ERR_UNSUPPORTED,
            "b2p_interp_create_dense: element too large (%d x %d)", d->out_P, d->in_P);
  b2p_interp *it = new b2p_interp;
  it->ctx = ctx;
  it->dense = true;
  it->ne = d->ne;
  it->in_P = d->in_P;
  it->out_P = d->out_P;
  it->in_lsize = d->in_lsize;
  it->out_lsize = d->out_lsize;
  it->ncomp = 0;
  int rc;
  std::vector<int32_t> out_host;
  // with a tridiagonal transformation the signs live in it (restriction.cpp:318-329): plain indices
  if ((rc = build_lidx(ctx, d->ne, d->in_P, d->in_lsize, d->in_idx, d->in_curl_orient ? nullptr : d->in_orient, nullptr, &it->in_PS,
                       &it->in_lidx, nullptr)) ||
      (rc = build_lidx(ctx, d->ne, d->out_P, d->out_lsize, d->out_idx, d->out_curl_orient ? nullptr : d->out_orient, nullptr,
                       &it->out_PS, &it->out_lidx, &out_host)))
  {
    b2p_interp_destroy(it);
    return rc;
  }
  if ((rc = upload_inv_mult(ctx, out_host, d->out_lsize, &it->inv_mult)) ||
      (rc = upload(ctx, d->mat, (size_t)d->out_P * d->in_P, &it->dmat)) ||
      (d->in_curl_orient && (rc = upload(ctx, d->in_curl_orient, (size_t)d->ne * d->in_P * 3, &it->in_co))) ||
      (d->out_curl_orient && (rc = upload(ctx, d->out_curl_orient, (size_t)d->ne * d->out_P * 3, &it->out_co))))
  {
    b2p_interp_destroy(it);
    return rc;
  }
  *out = it;
  return B2P_SUCCESS;
}

int b2p_interp_create_curl_hex(b2p_ctx *ctx, const b2p_curl_interp_desc *d, b2p_interp **out)
{
  B2P_CHECK(ctx, ctx && d && out && d->nd_idx && d->rt_idx && d->D, B2P_ERR_ARG, "b2p_interp_create_curl_hex: null argument");
  B2P_CHECK(ctx, d->ne > 0, B2P_ERR_ARG, "b2p_interp_create_curl_hex: ne=%d, no elements", d->ne);
  B2P_CHECK(ctx, d->p >= 1, B2P_ERR_ARG, "b2p_interp_create_curl_hex: p=%d, must be at least 1", d->p);
  B2P_CHECK(ctx, d->p <= CURL_HEX_PMAX, B2P_ERR_UNSUPPORTED, "b2p_interp_create_curl_hex: p=%d, kernels exist for p = 1..%d", d->p,
            CURL_HEX_PMAX);
  B2P_CHECK(ctx, d->nd_lsize > 0 && d->nd_lsize <= INT32_MAX && d->rt_lsize > 0 && d->rt_lsize <= INT32_MAX, B2P_ERR_ARG,
            "b2p_interp_create_curl_hex: nd_lsize=%lld / rt_lsize=%lld outside 1..2^31-1", (long long)d->nd_lsize,
            (long long)d->rt_lsize);
  const int p = d->p, n = p + 1;
  b2p_interp *it = new b2p_interp;
  it->ctx = ctx;
  it->curl_p = p;
  it->ne = d->ne;
  it->in_P = 3 * p * n * n;
  it->out_P = 3 * n * p * p;
  it->in_lsize = d->nd_lsize;
  it->out_lsize = d->rt_lsize;
  it->ncomp = 0;
  int rc;
  std::vector<int32_t> out_host;
  if ((rc = build_lidx(ctx, d->ne, it->in_P, d->nd_lsize, d->nd_idx, d->nd_orient, d->nd_dof_map, &it->in_PS, &it->in_lidx, nullptr)) ||
      (rc = build_lidx(ctx, d->ne, it->out_P, d->rt_lsize, d->rt_idx, d->rt_orient, d->rt_dof_map, &it->out_PS, &it->out_lidx,
                       &out_host)) ||
      (rc = upload_inv_mult(ctx, out_host, d->rt_lsize, &it->inv_mult)) || (rc = upload(ctx, d->D, (size_t)p * n, &it->curl_D)))
  {
    b2p_interp_destroy(it);
    return rc;
  }
  *out = it;
  return B2P_SUCCESS;
}

int b2p_interp_apply_add(b2p_interp *it, int transpose, double alpha, const double *x, double *y, b2p_stream s)
{
  if (!it || !x || !y) return B2P_ERR_ARG;
  return interp_apply(it, transpose != 0, alpha, x, y, (cudaStream_t)s);
}

void b2p_interp_destroy(b2p_interp *it)
{
  if (!it) return;
  cudaFree(it->in_lidx);
  cudaFree(it->out_lidx);
  cudaFree(it->inv_mult);
  cudaFree(it->mats);
  cudaFree(it->out_owner_lidx);
  cudaFree(it->dmat);
  cudaFree(it->in_co);
  cudaFree(it->out_co);
  cudaFree(it->curl_D);
  delete it;
}

}  // extern "C"
