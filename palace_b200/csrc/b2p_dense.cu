// Dense-basis (non-tensor) element operator: the general path the reference takes for every
// vector-valued element and every simplex (InitNonTensorBasis -> CeedBasisCreateHcurl,
// /root/reference/palace/fem/libceed/basis.cpp:40-85,169-186): per element a dense
// [3Q x P] interp and curl (or grad) table is applied, then the pointwise QFunction, then the
// transposes. Native dof order, orientation by sign (restriction.cpp:281-297) or by the tridiagonal
// "curl-oriented" matrix of ND tets/prisms with p >= 2 (restriction.cpp:301-368). The reference runs
// this through MAGMA batched GEMM on GPUs; here the element batch is one FP64 tensor-core GEMM:
//
//   V[R x NEB] = T[R x P] * U[P x NEB]        (R = rows of interp + deriv tables, NEB = 8 elements)
//   Y[P x NEB] = T^T[P x R] * D(V)[R x NEB]
//
// issued as mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4): A fragments stream from the (L2-resident) table,
// B fragments from the element vectors in shared memory, the 8 elements of the batch are the N
// dimension. wgmma has no FP64 kind, so DMMA is the tensor path for double precision on sm_90a.
// The sum-factorised hex kernels (b2p_hex_nd3.cu) do the same operator in O(p^4) and are ~4x faster;
// this kernel is the fallback that covers every other element type MFEM can describe by tables.
#include <cstdlib>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

struct DenseParams
{
  const int32_t *lidx;        // [ne][PS] signed native restriction
  const int8_t *curl_orient;  // [ne][P][3] row-major tridiagonal or null
  const double *T;            // [Rpad][Ppad] stacked tables (interp rows first when present, then deriv), zero padded
  const double *qd;           // [ne][10][Q] geometry, plain point order
  const double *ecoef;        // [ne][18]
  const double *x;
  double *y;
  double alpha;
  VSplit sp;
  int ne, P, PS, Ppad, Q, Rpad, row_u, row_c;  // row_u / row_c: first row of the interp / deriv block (-1: absent)
  int kind;
  int transpose;  // mixed kinds only: apply A^T (the symmetric kinds ignore it)
};

constexpr int NEB0 = 8;  // elements per MMA n-tile

// NT n-tiles (8 NT elements) per block: every table fragment fetched from L2 feeds NT MMAs (the tables, not HBM, are what the
// NT = 1 kernel waits for); NT = 1 is the hardware-verified default, B2P_DENSE_NT = 2 / 4 opt in while shared memory allows.
template <int NT>
__global__ void __launch_bounds__(256) dense_apply_kernel(DenseParams prm)
{
  constexpr int NEB = NEB0 * NT;
  B2P_DYN_SMEM(double, sm);
  double *U = sm;                       // [Ppad][NEB]
  double *V = U + prm.Ppad * NEB;       // [Rpad][NEB]
  double *X = V + prm.Rpad * NEB;       // [P][NEB] raw gathered values (curl-oriented restriction only)
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int e0 = blockIdx.x * NEB;
  const int P = prm.P, Q = prm.Q;

  // ---- restriction (E): native order, sign or tridiagonal orientation ----
  for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
  {
    const int i = w / NEB, e = w % NEB;
    double v = 0.0;
    if (i < P && e0 + e < prm.ne)
    {
      const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
      if (prm.curl_orient)
        v = (gi == B2P_SKIP_IDX) ? 0.0 : __ldg(split_src(prm.x, prm.sp, gi >= 0 ? gi : -1 - gi));
      else
        v = gather2(prm.x, prm.sp, gi);
    }
    (prm.curl_orient ? X : U)[w] = v;
  }
  if (prm.curl_orient)
  {
    __syncthreads();
    for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
    {
      const int i = w / NEB, e = w % NEB;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P + i) * 3;
        v = (double)co[1] * X[i * NEB + e];
        if (i > 0) v += (double)co[0] * X[(i - 1) * NEB + e];
        if (i < P - 1) v += (double)co[2] * X[(i + 1) * NEB + e];
      }
      U[w] = v;
    }
  }
  __syncthreads();

  // ---- V = T U : m-tiles over table rows, k over dofs ----
  for (int mt = wid; mt < prm.Rpad / 8; mt += nw)
  {
    double c[NT][2];
#pragma unroll
    for (int nt = 0; nt < NT; nt++) c[nt][0] = c[nt][1] = 0.0;
    const double *Arow = prm.T + (size_t)(mt * 8 + lane / 4) * prm.Ppad + (lane % 4);
    const double *Bcol = U + (lane % 4) * NEB + lane / 4;
    for (int k0 = 0; k0 < prm.Ppad; k0 += 4)
    {
      const double a = __ldg(Arow + k0);
#pragma unroll
      for (int nt = 0; nt < NT; nt++) dmma884(c[nt][0], c[nt][1], a, Bcol[k0 * NEB + 8 * nt]);
    }
    double *o = V + (mt * 8 + lane / 4) * NEB + 2 * (lane % 4);
#pragma unroll
    for (int nt = 0; nt < NT; nt++)
    {
      o[8 * nt] = c[nt][0];
      o[8 * nt + 1] = c[nt][1];
    }
  }
  __syncthreads();

  // ---- D at the quadrature points (in place) ----
  const bool MASS = (prm.kind == B2P_ND_MASS || prm.kind == B2P_CURLCURL_MASS);
  const bool CURL = (prm.kind == B2P_CURLCURL || prm.kind == B2P_CURLCURL_MASS);
  const bool H1 = (prm.kind == B2P_H1_DIFFUSION);
  for (int w = tid; w < Q * NEB; w += blockDim.x)
  {
    const int iq = w / NEB, e = w % NEB;
    if (e0 + e >= prm.ne) continue;
    const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + iq;
    const double *C = prm.ecoef + (size_t)(e0 + e) * 18;
    const double wdetJ = prm.alpha * g[0];
    double A[9], Cm[9];
#pragma unroll
    for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
    if (MASS || H1)
    {
      const int r0 = MASS ? prm.row_u : prm.row_c;
      double u[3] = {V[(r0 + iq) * NEB + e], V[(r0 + Q + iq) * NEB + e], V[(r0 + 2 * Q + iq) * NEB + e]}, v[3];
#pragma unroll
      for (int i = 0; i < 9; i++) Cm[i] = C[i];
      AtCAx(A, Cm, u, wdetJ, v);
      V[(r0 + iq) * NEB + e] = v[0];
      V[(r0 + Q + iq) * NEB + e] = v[1];
      V[(r0 + 2 * Q + iq) * NEB + e] = v[2];
    }
    if (CURL)
    {
      const int r0 = prm.row_c;
      double c[3] = {V[(r0 + iq) * NEB + e], V[(r0 + Q + iq) * NEB + e], V[(r0 + 2 * Q + iq) * NEB + e]}, v[3], Jd[9];
#pragma unroll
      for (int i = 0; i < 9; i++) Cm[i] = C[9 + i];
      cofactor33(A, Jd);
      AtCAx(Jd, Cm, c, wdetJ, v);
      V[(r0 + iq) * NEB + e] = v[0];
      V[(r0 + Q + iq) * NEB + e] = v[1];
      V[(r0 + 2 * Q + iq) * NEB + e] = v[2];
    }
  }
  __syncthreads();

  // ---- Y = T^T V : m-tiles over dofs, k over table rows; result overwrites U ----
  for (int mt = wid; mt < prm.Ppad / 8; mt += nw)
  {
    double c[NT][2];
#pragma unroll
    for (int nt = 0; nt < NT; nt++) c[nt][0] = c[nt][1] = 0.0;
    const double *Acol = prm.T + (size_t)(lane % 4) * prm.Ppad + mt * 8 + lane / 4;
    const double *Bcol = V + (lane % 4) * NEB + lane / 4;
    for (int k0 = 0; k0 < prm.Rpad; k0 += 4)
    {
      const double a = __ldg(Acol + (size_t)k0 * prm.Ppad);
#pragma unroll
      for (int nt = 0; nt < NT; nt++) dmma884(c[nt][0], c[nt][1], a, Bcol[k0 * NEB + 8 * nt]);
    }
    double *o = U + (mt * 8 + lane / 4) * NEB + 2 * (lane % 4);
#pragma unroll
    for (int nt = 0; nt < NT; nt++)
    {
      o[8 * nt] = c[nt][0];
      o[8 * nt + 1] = c[nt][1];
    }
  }
  __syncthreads();

  // ---- E^T ----
  if (prm.curl_orient)
  {
    for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
    {
      const int i = w / NEB, e = w % NEB;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P) * 3;
        v = (double)co[3 * i + 1] * U[i * NEB + e];
        if (i > 0) v += (double)co[3 * (i - 1) + 2] * U[(i - 1) * NEB + e];
        if (i < P - 1) v += (double)co[3 * (i + 1) + 0] * U[(i + 1) * NEB + e];
      }
      X[w] = v;
    }
    __syncthreads();
  }
  const double *src = prm.curl_orient ? X : U;
  for (int w = tid; w < P * NEB; w += blockDim.x)
  {
    const int i = w / NEB, e = w % NEB;
    if (e0 + e >= prm.ne) continue;
    const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
    if (prm.curl_orient)
    {
      if (gi != B2P_SKIP_IDX) scatter2(prm.y, prm.sp, gi >= 0 ? gi : -1 - gi, src[w]);
    }
    else
      scatter2(prm.y, prm.sp, gi, src[w]);
  }
}

// Round-2 kernel: the two GEMMs of an element batch are fused over chunks of QC quadrature points, so that
//   * the [6Q x NEB] array of point values never exists -- only a [6 QC x NEB] chunk does, which leaves room for NT = 4
//     n-tiles (32 elements per CTA): every table fragment fetched from L2 / L1 feeds four MMAs (the round-1 kernel streamed
//     the whole table twice per 8 elements and was bound by those loads: 4.4 TFLOP/s, 12 % of the DMMA peak);
//   * the output accumulators Y[Ppad x NEB] stay in registers across the chunks (each warp owns its dof tiles);
//   * table fragments are prefetched four k-steps ahead into registers.
// Chunk rows are ordered [block c][point j], block c < 3: interp component c, c >= 3: deriv component c - 3 (blocks of absent
// parts are skipped); QC is a multiple of 8, so an m-tile never straddles two blocks.
template <int NT, int QC, int MTB>
__global__ void __launch_bounds__(256) dense_apply2_kernel(DenseParams prm)
{
  constexpr int NEB = NEB0 * NT, LS = NEB + 4;  // row stride of the shared arrays: +4 doubles makes the B-fragment reads conflict free
  B2P_DYN_SMEM(double, sm);
  const int P = prm.P, Q = prm.Q, Ppad = prm.Ppad;
  const bool MASS = (prm.kind == B2P_ND_MASS || prm.kind == B2P_CURLCURL_MASS);
  const bool CURL = (prm.kind == B2P_CURLCURL || prm.kind == B2P_CURLCURL_MASS);
  const bool H1 = (prm.kind == B2P_H1_DIFFUSION);
  const int nblk = ((MASS ? 3 : 0) + ((CURL || H1) ? 3 : 0));  // row blocks per chunk
  const int CR = nblk * QC;                                    // chunk rows
  double *U = sm;                 // [Ppad][LS]
  double *V = U + Ppad * LS;      // [6 QC][LS]
  double *X = V + 6 * QC * LS;    // [Ppad][LS] raw gathered values (curl-oriented restriction only)
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int e0 = blockIdx.x * NEB;
  // table row of chunk row r (block c = r / QC, point q0 + r % QC); rows of points >= Q are clamped (their V entries are zeroed)
  auto table_row = [&](int r, int q0) -> int
  {
    const int c = r / QC, iq = min(q0 + r % QC, Q - 1);
    const int base = (MASS && c < 3) ? prm.row_u + c * Q : prm.row_c + (c - (MASS ? 3 : 0)) * Q;
    return base + iq;
  };

  // ---- restriction (E): native order, sign or tridiagonal orientation ----
  // (dof index fastest across threads: the index rows and the int8 orientation rows are read coalesced -- element-fastest
  // threads touched one 32-byte sector per 4-byte index, 8x the restriction's bytes; the shared-memory stores take the
  // bank conflicts instead)
  for (int w = tid; w < Ppad * NEB; w += blockDim.x)
  {
    const int e = w / Ppad, i = w % Ppad;
    double v = 0.0;
    if (i < P && e0 + e < prm.ne)
    {
      const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
      if (prm.curl_orient)
        v = (gi == B2P_SKIP_IDX) ? 0.0 : __ldg(split_src(prm.x, prm.sp, gi >= 0 ? gi : -1 - gi));
      else
        v = gather2(prm.x, prm.sp, gi);
    }
    (prm.curl_orient ? X : U)[i * LS + e] = v;
  }
  if (prm.curl_orient)
  {
    __syncthreads();
    for (int w = tid; w < Ppad * NEB; w += blockDim.x)
    {
      const int e = w / Ppad, i = w % Ppad;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P + i) * 3;
        v = (double)co[1] * X[i * LS + e];
        if (i > 0) v += (double)co[0] * X[(i - 1) * LS + e];
        if (i < P - 1) v += (double)co[2] * X[(i + 1) * LS + e];
      }
      U[i * LS + e] = v;
    }
  }
  __syncthreads();

  // output accumulators: dof tiles wid, wid + nw, ... of this warp, NT n-tiles each
  double acc[MTB][NT][2];
#pragma unroll
  for (int t = 0; t < MTB; t++)
#pragma unroll
    for (int nt = 0; nt < NT; nt++) acc[t][nt][0] = acc[t][nt][1] = 0.0;

  const int KF = Ppad / 4;  // k-steps of the forward GEMM
  for (int q0 = 0; q0 < Q; q0 += QC)
  {
    // ---- V_chunk = T_chunk U : m-tiles over chunk rows, k over dofs ----
    for (int mt = wid; mt < CR / 8; mt += nw)
    {
      double c[NT][2];
#pragma unroll
      for (int nt = 0; nt < NT; nt++) c[nt][0] = c[nt][1] = 0.0;
      const double *Arow = prm.T + (size_t)table_row(mt * 8 + lane / 4, q0) * Ppad + (lane % 4);
      const double *Bcol = U + (lane % 4) * LS + lane / 4;
      double a[4];
#pragma unroll
      for (int j = 0; j < 4; j++) a[j] = (j < KF) ? __ldg(Arow + 4 * j) : 0.0;
      for (int kk = 0; kk < KF; kk += 4)
      {
        double an[4];
#pragma unroll
        for (int j = 0; j < 4; j++) an[j] = (kk + 4 + j < KF) ? __ldg(Arow + 4 * (kk + 4 + j)) : 0.0;
#pragma unroll
        for (int j = 0; j < 4; j++)
          if (kk + j < KF)
          {
#pragma unroll
            for (int nt = 0; nt < NT; nt++) dmma884(c[nt][0], c[nt][1], a[j], Bcol[(size_t)(kk + j) * 4 * LS + 8 * nt]);
          }
#pragma unroll
        for (int j = 0; j < 4; j++) a[j] = an[j];
      }
      double *o = V + (mt * 8 + lane / 4) * LS + 2 * (lane % 4);
#pragma unroll
      for (int nt = 0; nt < NT; nt++)
      {
        o[8 * nt] = c[nt][0];
        o[8 * nt + 1] = c[nt][1];
      }
    }
    __syncthreads();

    // ---- D at the chunk's quadrature points (in place); points beyond Q and elements beyond ne become zero rows ----
    // item -> (point, element): a warp covers 4 consecutive points x 8 elements, so every 32-byte sector of the q-data is
    // used whole (element-fastest threads fetched a sector per 8-byte value: 4x the geometry stream, the largest HBM term)
    // and the shared-memory accesses are at most 2-way conflicted
    for (int w = tid; w < QC * NEB; w += blockDim.x)
    {
      const int rest = w >> 5;
      const int j = (rest % (QC / 4)) * 4 + (w & 3), e = (rest / (QC / 4)) * 8 + ((w >> 2) & 7), iq = q0 + j;
      const bool ok = iq < Q && e0 + e < prm.ne;
      const double *g = prm.qd + (size_t)(e0 + (ok ? e : 0)) * 10 * Q + (ok ? iq : 0);
      const double *C = prm.ecoef + (size_t)(e0 + (ok ? e : 0)) * 18;
      const double wdetJ = ok ? prm.alpha * g[0] : 0.0;
      double A[9], Cm[9];
#pragma unroll
      for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
      if (MASS || H1)
      {
        double *r = V + j * LS + e;  // blocks 0, 1, 2
        double u[3] = {r[0], r[QC * LS], r[2 * QC * LS]}, v[3];
#pragma unroll
        for (int i = 0; i < 9; i++) Cm[i] = C[i];
        AtCAx(A, Cm, u, wdetJ, v);
        r[0] = v[0];
        r[QC * LS] = v[1];
        r[2 * QC * LS] = v[2];
      }
      if (CURL)
      {
        double *r = V + ((MASS ? 3 : 0) * QC + j) * LS + e;
        double c[3] = {r[0], r[QC * LS], r[2 * QC * LS]}, v[3], Jd[9];
#pragma unroll
        for (int i = 0; i < 9; i++) Cm[i] = C[9 + i];
        cofactor33(A, Jd);
        AtCAx(Jd, Cm, c, wdetJ, v);
        r[0] = v[0];
        r[QC * LS] = v[1];
        r[2 * QC * LS] = v[2];
      }
    }
    __syncthreads();

    // ---- Y += T_chunk^T V_chunk : this warp's dof tiles, k over chunk rows ----
#pragma unroll
    for (int t = 0; t < MTB; t++)
    {
      const int mt = wid + t * nw;
      if (mt < Ppad / 8)
      {
        const double *Bcol = V + (lane % 4) * LS + lane / 4;
        const int KB = CR / 4;
        // A[m = dof][k = chunk row]: lane reads T[table_row(4 k + lane % 4)][8 mt + lane / 4]
        auto lda = [&](int k) -> double { return __ldg(prm.T + (size_t)table_row(4 * k + lane % 4, q0) * Ppad + mt * 8 + lane / 4); };
        double a[4];
#pragma unroll
        for (int j = 0; j < 4; j++) a[j] = (j < KB) ? lda(j) : 0.0;
        for (int kk = 0; kk < KB; kk += 4)
        {
          double an[4];
#pragma unroll
          for (int j = 0; j < 4; j++) an[j] = (kk + 4 + j < KB) ? lda(kk + 4 + j) : 0.0;
#pragma unroll
          for (int j = 0; j < 4; j++)
            if (kk + j < KB)
            {
#pragma unroll
              for (int nt = 0; nt < NT; nt++) dmma884(acc[t][nt][0], acc[t][nt][1], a[j], Bcol[(size_t)(kk + j) * 4 * LS + 8 * nt]);
            }
#pragma unroll
          for (int j = 0; j < 4; j++) a[j] = an[j];
        }
      }
    }
    __syncthreads();  // the next chunk's forward GEMM overwrites V
  }

  // ---- accumulators -> U (as Y), then E^T ----
#pragma unroll
  for (int t = 0; t < MTB; t++)
  {
    const int mt = wid + t * nw;
    if (mt < Ppad / 8)
    {
      double *o = U + (mt * 8 + lane / 4) * LS + 2 * (lane % 4);
#pragma unroll
      for (int nt = 0; nt < NT; nt++)
      {
        o[8 * nt] = acc[t][nt][0];
        o[8 * nt + 1] = acc[t][nt][1];
      }
    }
  }
  __syncthreads();
  if (prm.curl_orient)
  {
    for (int w = tid; w < Ppad * NEB; w += blockDim.x)
    {
      const int e = w / Ppad, i = w % Ppad;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P) * 3;
        v = (double)co[3 * i + 1] * U[i * LS + e];
        if (i > 0) v += (double)co[3 * (i - 1) + 2] * U[(i - 1) * LS + e];
        if (i < P - 1) v += (double)co[3 * (i + 1) + 0] * U[(i + 1) * LS + e];
      }
      X[i * LS + e] = v;
    }
    __syncthreads();
  }
  const double *src = prm.curl_orient ? X : U;
  for (int w = tid; w < P * NEB; w += blockDim.x)
  {
    const int e = w / P, i = w % P;
    if (e0 + e >= prm.ne) continue;
    const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
    if (prm.curl_orient)
    {
      if (gi != B2P_SKIP_IDX) scatter2(prm.y, prm.sp, gi >= 0 ? gi : -1 - gi, src[i * LS + e]);
    }
    else
      scatter2(prm.y, prm.sp, gi, src[i * LS + e]);
  }
}

// Mixed kinds on one ND space (the Floquet-periodic terms, models/spaceoperator.cpp:305-309):
//   B2P_ND_WEAKCURL   y = E^T Bc^T [w detJ Jd^T C A ] Bu E x   trial VALUES (H(curl) map A = J^-T) tested with CURLS (H(div) map Jd = J / detJ)
//                     MixedVectorWeakCurlIntegrator -> f_apply_hcurlhdiv_33 (integ/mixedveccurl.cpp:68-117, qfunctions/33/hcurlhdiv_33_qf.h:10-31)
//   B2P_ND_MIXEDCURL  y = E^T Bu^T [w detJ A^T C Jd ] Bc E x   trial CURLS tested with VALUES
//                     MixedVectorCurlIntegrator     -> f_apply_hdivhcurl_33 (integ/mixedveccurl.cpp:23-66, hcurlhdiv_33_qf.h:33-55)
// The forward GEMM runs over the trial block of the stacked table only, D maps the three point values in place, the backward GEMM
// runs over the test block: same two DMMA GEMMs per batch of 8 elements as dense_apply_kernel, half the rows each. The transpose
// of one kind is the other kind with C^T (prm.transpose). Not on the hot path (one extra term of periodic models): the whole
// [3Q x 8] point array stays in shared memory, tables stream from L2.
__global__ void __launch_bounds__(256) dense_mixed_kernel(DenseParams prm)
{
  constexpr int NEB = NEB0;
  B2P_DYN_SMEM(double, sm);
  const int P = prm.P, Q = prm.Q, R3 = 3 * Q, R3pad = (R3 + 7) & ~7;
  double *U = sm;                   // [Ppad][NEB]
  double *V = U + prm.Ppad * NEB;   // [R3pad][NEB]
  double *X = V + R3pad * NEB;      // [Ppad][NEB] raw gathered values (curl-oriented restriction only)
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int e0 = blockIdx.x * NEB;
  const bool trial_curl = (prm.kind == B2P_ND_MIXEDCURL) != (prm.transpose != 0);
  const int trial_row = trial_curl ? prm.row_c : prm.row_u, test_row = trial_curl ? prm.row_u : prm.row_c;

  // ---- restriction (E): native order, sign or tridiagonal orientation ----
  for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
  {
    const int i = w / NEB, e = w % NEB;
    double v = 0.0;
    if (i < P && e0 + e < prm.ne)
    {
      const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
      if (prm.curl_orient)
        v = (gi == B2P_SKIP_IDX) ? 0.0 : __ldg(split_src(prm.x, prm.sp, gi >= 0 ? gi : -1 - gi));
      else
        v = gather2(prm.x, prm.sp, gi);
    }
    (prm.curl_orient ? X : U)[w] = v;
  }
  if (prm.curl_orient)
  {
    __syncthreads();
    for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
    {
      const int i = w / NEB, e = w % NEB;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P + i) * 3;
        v = (double)co[1] * X[i * NEB + e];
        if (i > 0) v += (double)co[0] * X[(i - 1) * NEB + e];
        if (i < P - 1) v += (double)co[2] * X[(i + 1) * NEB + e];
      }
      U[w] = v;
    }
  }
  __syncthreads();

  // ---- V = T_trial U : m-tiles over the trial block's rows (rows past the block read as zero), k over dofs ----
  for (int mt = wid; mt < R3pad / 8; mt += nw)
  {
    double c0 = 0.0, c1 = 0.0;
    const int r = mt * 8 + lane / 4;
    const bool live = r < R3;
    const double *Arow = prm.T + (size_t)(trial_row + (live ? r : 0)) * prm.Ppad + (lane % 4);
    const double *Bcol = U + (lane % 4) * NEB + lane / 4;
    for (int k0 = 0; k0 < prm.Ppad; k0 += 4)
    {
      const double a = live ? __ldg(Arow + k0) : 0.0;
      dmma884(c0, c1, a, Bcol[k0 * NEB]);
    }
    double *o = V + r * NEB + 2 * (lane % 4);
    o[0] = c0;
    o[1] = c1;
  }
  __syncthreads();

  // ---- D at the quadrature points (in place): out = w detJ M2^T C' M1 t ----
  for (int w = tid; w < Q * NEB; w += blockDim.x)
  {
    const int iq = w / NEB, e = w % NEB;
    if (e0 + e >= prm.ne) continue;  // (their U columns are zero, so their V entries already are)
    const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + iq;
    const double *C = prm.ecoef + (size_t)(e0 + e) * 18;
    const double wdetJ = prm.alpha * g[0];
    double A[9], Jd[9], Cm[9];
#pragma unroll
    for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) Cm[i + 3 * j] = prm.transpose ? C[j + 3 * i] : C[i + 3 * j];
    cofactor33(A, Jd);
    const double t[3] = {V[iq * NEB + e], V[(Q + iq) * NEB + e], V[(2 * Q + iq) * NEB + e]};
    double t1[3], z[3], v[3];
    Ax33(trial_curl ? Jd : A, t, t1);
    Ax33(Cm, t1, z);
    Atx33(trial_curl ? A : Jd, z, wdetJ, v);
    V[iq * NEB + e] = v[0];
    V[(Q + iq) * NEB + e] = v[1];
    V[(2 * Q + iq) * NEB + e] = v[2];
  }
  __syncthreads();

  // ---- Y = T_test^T V : m-tiles over dofs, k over the test block's rows; result overwrites U ----
  for (int mt = wid; mt < prm.Ppad / 8; mt += nw)
  {
    double c0 = 0.0, c1 = 0.0;
    const double *Bcol = V + (lane % 4) * NEB + lane / 4;
    for (int k0 = 0; k0 < R3pad; k0 += 4)
    {
      const int r = k0 + lane % 4;
      const double a = r < R3 ? __ldg(prm.T + (size_t)(test_row + r) * prm.Ppad + mt * 8 + lane / 4) : 0.0;
      dmma884(c0, c1, a, Bcol[k0 * NEB]);
    }
    double *o = U + (mt * 8 + lane / 4) * NEB + 2 * (lane % 4);
    o[0] = c0;
    o[1] = c1;
  }
  __syncthreads();

  // ---- E^T ----
  if (prm.curl_orient)
  {
    for (int w = tid; w < prm.Ppad * NEB; w += blockDim.x)
    {
      const int i = w / NEB, e = w % NEB;
      double v = 0.0;
      if (i < P && e0 + e < prm.ne)
      {
        const int8_t *co = prm.curl_orient + ((size_t)(e0 + e) * P) * 3;
        v = (double)co[3 * i + 1] * U[i * NEB + e];
        if (i > 0) v += (double)co[3 * (i - 1) + 2] * U[(i - 1) * NEB + e];
        if (i < P - 1) v += (double)co[3 * (i + 1) + 0] * U[(i + 1) * NEB + e];
      }
      X[w] = v;
    }
    __syncthreads();
  }
  const double *src = prm.curl_orient ? X : U;
  for (int w = tid; w < P * NEB; w += blockDim.x)
  {
    const int i = w / NEB, e = w % NEB;
    if (e0 + e >= prm.ne) continue;
    const int32_t gi = prm.lidx[(size_t)(e0 + e) * prm.PS + i];
    if (prm.curl_orient)
    {
      if (gi != B2P_SKIP_IDX) scatter2(prm.y, prm.sp, gi >= 0 ? gi : -1 - gi, src[w]);
    }
    else
      scatter2(prm.y, prm.sp, gi, src[w]);
  }
}

// diag[g(i)] += sum_q w(q)^T D w(q) with w = the i-th shape function as the global side sees it: for sign
// orientation that is column i of the table (the sign squares away); for the tridiagonal orientation it is
// sum_l T_e(l, i) * column l, which makes the diagonal of T^T A T exact (libCEED assembles it through the unsigned
// restriction, an approximation the reference tolerates, test-libceed.cpp:358-372; the Chebyshev / Jacobi smoothers
// converge visibly better with the exact one).
__global__ void dense_diag_kernel(DenseParams prm)
{
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)prm.ne * prm.P) return;
  const int e = (int)(w / prm.P), i = (int)(w % prm.P), Q = prm.Q, P = prm.P;
  const bool MASS = (prm.kind == B2P_ND_MASS || prm.kind == B2P_CURLCURL_MASS);
  const bool CURL = (prm.kind == B2P_CURLCURL || prm.kind == B2P_CURLCURL_MASS);
  const bool H1 = (prm.kind == B2P_H1_DIFFUSION);
  const bool MIXED = (prm.kind == B2P_ND_WEAKCURL || prm.kind == B2P_ND_MIXEDCURL);
  const double *C = prm.ecoef + (size_t)e * 18;
  double C0[9], C1[9];
  for (int t = 0; t < 9; t++)
  {
    C0[t] = C[t];
    C1[t] = C[9 + t];
  }
  // column combination: tc[l - i + 1] = T_e(l, i) for l = i-1, i, i+1
  double tc[3] = {0.0, 1.0, 0.0};
  if (prm.curl_orient)
  {
    const int8_t *co = prm.curl_orient + (size_t)e * P * 3;
    tc[1] = (double)co[3 * i + 1];
    tc[0] = i > 0 ? (double)co[3 * (i - 1) + 2] : 0.0;      // T(i-1, i)
    tc[2] = i < P - 1 ? (double)co[3 * (i + 1) + 0] : 0.0;  // T(i+1, i)
  }
  auto col = [&](int row) -> double
  {
    const double *r = prm.T + (size_t)row * prm.Ppad;
    double v = tc[1] * r[i];
    if (tc[0] != 0.0) v += tc[0] * r[i - 1];
    if (tc[2] != 0.0) v += tc[2] * r[i + 1];
    return v;
  };
  double s = 0.0;
  for (int iq = 0; iq < Q; iq++)
  {
    const double *g = prm.qd + (size_t)e * 10 * Q + iq;
    double A[9], v[3];
    for (int t = 0; t < 9; t++) A[t] = g[(1 + t) * Q];
    if (MASS || H1)
    {
      const int r0 = MASS ? prm.row_u : prm.row_c;
      double u[3] = {col(r0 + iq), col(r0 + Q + iq), col(r0 + 2 * Q + iq)};
      AtCAx(A, C0, u, g[0], v);
      s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
    }
    if (CURL)
    {
      const int r0 = prm.row_c;
      double c[3] = {col(r0 + iq), col(r0 + Q + iq), col(r0 + 2 * Q + iq)}, Jd[9];
      cofactor33(A, Jd);
      AtCAx(Jd, C1, c, g[0], v);
      s += c[0] * v[0] + c[1] * v[1] + c[2] * v[2];
    }
    if (MIXED)
    {
      // value and curl of the same shape function meet through C: c^T (w detJ Jd^T C A) u (weak curl), u^T (w detJ A^T C Jd) c
      double u[3] = {col(prm.row_u + iq), col(prm.row_u + Q + iq), col(prm.row_u + 2 * Q + iq)};
      double c[3] = {col(prm.row_c + iq), col(prm.row_c + Q + iq), col(prm.row_c + 2 * Q + iq)}, Jd[9], t1[3], z[3];
      cofactor33(A, Jd);
      if (prm.kind == B2P_ND_WEAKCURL)
      {
        Ax33(A, u, t1);
        Ax33(C0, t1, z);
        Atx33(Jd, z, g[0], v);
        s += c[0] * v[0] + c[1] * v[1] + c[2] * v[2];
      }
      else
      {
        Ax33(Jd, c, t1);
        Ax33(C0, t1, z);
        Atx33(A, z, g[0], v);
        s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
      }
    }
  }
  int gi = prm.lidx[(size_t)e * prm.PS + i];
  if (gi == B2P_SKIP_IDX) return;
  if (gi < 0) gi = -1 - gi;
  atomicAdd(prm.y + gi, s);
}

DenseParams make_params(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg)
{
  DenseParams p;
  p.transpose = 0;
  const int e_off = rg.e_off, e_cnt = rg.e_cnt < 0 ? op->ne - rg.e_off : rg.e_cnt;
  p.lidx = lidx + (size_t)e_off * op->PS;
  p.curl_orient = op->curl_orient ? op->curl_orient + (size_t)e_off * op->P * 3 : nullptr;
  p.T = op->dense_T;
  p.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  p.ecoef = op->ecoef + 18 * (size_t)e_off;
  p.x = x;
  p.y = y;
  p.alpha = alpha;
  p.sp.n_owned = rg.n_owned < 0 ? op->lsize : rg.n_owned;
  p.sp.xg = rg.xg;
  p.sp.yg = rg.yg;
  p.ne = e_cnt;
  p.P = op->P;
  p.PS = op->PS;
  p.Ppad = op->dense_Ppad;
  p.Q = op->geom->Q;
  p.Rpad = op->dense_Rpad;
  p.row_u = op->dense_row_u;
  p.row_c = op->dense_row_c;
  p.kind = op->kind;
  return p;
}

}  // namespace

namespace
{
// The fused, chunked kernel: NT n-tiles per CTA, QC points per chunk, up to MTB dof tiles per warp.
template <int NT, int QC, int MTB>
int launch_dense2(b2p_op *op, const DenseParams &prm, int nwarps, cudaStream_t s)
{
  constexpr int NEB = NEB0 * NT, LS = NEB + 4;
  const size_t shmem = sizeof(double) * LS * ((size_t)prm.Ppad + 6 * QC + (op->curl_orient ? prm.Ppad : 0));
  auto kern = dense_apply2_kernel<NT, QC, MTB>;
  static size_t configured = 0;
  if (shmem > configured)
  {
    B2P_CUDA(op->ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem));
    configured = shmem;
  }
  B2P_LAUNCH(kern, (prm.ne + NEB - 1) / NEB, nwarps * 32, shmem, s, prm);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}
}  // namespace

int launch_dense_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg,
                       cudaStream_t s, bool transpose)
{
  DenseParams prm = make_params(op, lidx, alpha, x, y, rg);
  if (prm.ne <= 0) return B2P_SUCCESS;
  if (op->kind == B2P_ND_WEAKCURL || op->kind == B2P_ND_MIXEDCURL)
  {
    prm.transpose = transpose ? 1 : 0;
    const int R3pad = (3 * prm.Q + 7) & ~7;
    const size_t shmem = sizeof(double) * NEB0 * ((size_t)prm.Ppad + R3pad + (op->curl_orient ? prm.Ppad : 0));
    B2P_CHECK(op->ctx, shmem <= 227 * 1024, B2P_ERR_UNSUPPORTED, "dense mixed operator: element too large for shared memory (%zu B)", shmem);
    static size_t configured = 0;
    if (shmem > configured)
    {
      B2P_CUDA(op->ctx, cudaFuncSetAttribute(dense_mixed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem));
      configured = shmem;
    }
    B2P_LAUNCH(dense_mixed_kernel, (prm.ne + NEB0 - 1) / NEB0, 256, shmem, s, prm);
    B2P_CUDA(op->ctx, cudaGetLastError());
    return B2P_SUCCESS;
  }
  // B2P_DENSE_KERNEL=1: the round-1 kernel (whole [6Q x 8] point array in shared memory, table streamed per 8 elements)
  static const int which = []
  {
    const char *e = std::getenv("B2P_DENSE_KERNEL");
    return e ? std::atoi(e) : 2;
  }();
  if (which == 2 && prm.ne >= 32)
  {
    constexpr int QC = 32;
    const int tiles = prm.Ppad / 8;  // dof tiles of the backward GEMM: one warp per tile up to 8 warps, then several per warp
    const int nwarps = tiles < 8 ? (tiles < 4 ? 4 : tiles) : 8;
    const int mtb = (tiles + nwarps - 1) / nwarps;
    const size_t rows = (size_t)prm.Ppad + 6 * QC + (op->curl_orient ? prm.Ppad : 0);
    const size_t need4 = sizeof(double) * 36 * rows, need2 = sizeof(double) * 20 * rows;
    // Two CTAs per SM need <= 113 KB each: large elements (p = 6: 180 KB with four n-tiles) run two n-tiles per CTA instead,
    // 16 elements per CTA, so that 16 warps per SM hide the table-fragment latency (B2P_DENSE_NT=4 forces four).
    static const int force_nt = []
    {
      const char *e = std::getenv("B2P_DENSE_NT");
      return e ? std::atoi(e) : 0;
    }();
    const bool two = force_nt == 2 || (force_nt != 4 && need4 > 113 * 1024 && need2 <= 113 * 1024);
    static const bool trace = std::getenv("B2P_TRACE_KERNEL") != nullptr;
    if (two && need2 <= 227 * 1024 && mtb <= 4 && prm.ne >= 16)
    {
      if (trace) fprintf(stderr, "[b2p] dense_apply2 (2 n-tiles) P=%d Q=%d ne=%d warps=%d tiles/warp=%d\n", prm.P, prm.Q, prm.ne, nwarps, mtb);
      if (mtb <= 1) return launch_dense2<2, QC, 1>(op, prm, nwarps, s);
      if (mtb <= 2) return launch_dense2<2, QC, 2>(op, prm, nwarps, s);
      return launch_dense2<2, QC, 4>(op, prm, nwarps, s);
    }
    if (need4 <= 227 * 1024 && mtb <= 4)
    {
      if (trace) fprintf(stderr, "[b2p] dense_apply2 P=%d Q=%d ne=%d warps=%d tiles/warp=%d\n", prm.P, prm.Q, prm.ne, nwarps, mtb);
      if (mtb <= 1) return launch_dense2<4, QC, 1>(op, prm, nwarps, s);
      if (mtb <= 2) return launch_dense2<4, QC, 2>(op, prm, nwarps, s);
      return launch_dense2<4, QC, 4>(op, prm, nwarps, s);
    }
  }
  const size_t shmem1 = sizeof(double) * NEB0 * ((size_t)prm.Ppad + prm.Rpad + (op->curl_orient ? prm.Ppad : 0));
  B2P_CHECK(op->ctx, shmem1 <= 227 * 1024, B2P_ERR_UNSUPPORTED, "dense operator: element too large for shared memory (%zu B)", shmem1);
  static const int want_nt = []
  {
    const char *e = std::getenv("B2P_DENSE_NT");
    const int v = e ? std::atoi(e) : 1;
    return v >= 4 ? 4 : (v >= 2 ? 2 : 1);
  }();
  int nt = want_nt;
  while (nt > 1 && (shmem1 * nt > 227 * 1024 || prm.ne < NEB0 * nt)) nt /= 2;
  const size_t shmem = shmem1 * nt;
  static size_t configured[3] = {0, 0, 0};
  const int slot = nt == 4 ? 2 : (nt == 2 ? 1 : 0);
  auto kern = nt == 4 ? dense_apply_kernel<4> : (nt == 2 ? dense_apply_kernel<2> : dense_apply_kernel<1>);
  if (shmem > configured[slot])
  {
    B2P_CUDA(op->ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem));
    configured[slot] = shmem;
  }
  const int neb = NEB0 * nt;
  B2P_LAUNCH(kern, (prm.ne + neb - 1) / neb, 256, shmem, s, prm);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int launch_dense_diag(b2p_op *op, double *diag, cudaStream_t s)
{
  DenseParams prm = make_params(op, op->lidx, 1.0, nullptr, diag, ApplyRange());
  const size_t total = (size_t)op->ne * op->P;
  B2P_LAUNCH(dense_diag_kernel, (unsigned)((total + 127) / 128), 128, 0, s, prm);
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p
