// Nedelec hexahedron apply kernel for q1d = 4 (p <= 3): ONE element per warp, half-warp pairs.
//
//   y_L += alpha * sum_e E_e^T  B^T  D  B  E_e x_L          (curl-curl, mass, curl-curl + mass)
//
// Same operator and the same warp-autonomous TMA / cp.async pipeline as b2p_hex_nd4.cu, but a warp owns a
// single element, so its shared-memory footprint is half (13.6 KB at p = 3) and 12-16 warps fit on an SM
// instead of 8: the previous kernel was latency bound with two warps per scheduler.
//
// An element at q1d = 4 only has 16 (qy,qz) lines / 12-16 items per contraction phase, half a warp. The two
// half-warps therefore share every line / item and split the QUADRATURE index of the contracted direction:
// half 0 owns points {0, 1}, half 1 owns points {3, 2}. Because the 1-D tables of a symmetric point set obey
//     Bo[q-1-c][p-1-i] = Bo[c][i],   Bc[q-1-c][n-1-i] = Bc[c][i],   Gc[q-1-c][n-1-i] = -Gc[c][i],
// half 1 evaluates its points with the SAME table entries as half 0 applied to the dofs in reversed order
// (a different shared-memory address, not a different instruction) and a sign on the derivative terms, so
// every table entry stays a warp-uniform constant-bank operand of the DFMA. Transposed contractions produce
// per-half partial sums for mirrored output indices; one __shfl_xor(.,16) per finished output combines them.
// The launcher verifies the table symmetry (exact for MFEM's Gauss-Legendre / Gauss-Lobatto bases and
// Gauss-Legendre quadrature) and falls back to nd_hex_apply4_kernel otherwise.
// The index maps, the mirrored contractions and the bank behaviour of this file were validated lane by lane
// against the oracle in tools/nd5_emulate.py before the kernel went to the GPU.
//
// Reference semantics: ceed::Operator::AddMult over CeedOperatorApplyAdd
// (/root/reference/palace/fem/libceed/operator.cpp:148-178,192-212); D from
// /root/reference/palace/fem/qfunctions/33/{hdiv,hcurl,hdivmass}_33_qf.h.
#include <cmath>
#include <cstdlib>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

template <int P_>
struct ND5Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction, rows padded to 16 bytes (B2P_SKIP_IDX = masked/pad)
  const double *qd;     // [ne][10][Q] geometry, x-slowest point order
  const double *aq;     // [ne][ncomp][Q] assembled D, x-slowest (or null)
  const double *ecoef;  // [ne][18] per-element coefficient matrices (value part, derivative part)
  const double *x;
  double *y;
  double alpha;
  int ne;
  VSplit sp;
  const unsigned long long *wait_flags, *wait_expect;  // peer-memory halo flags (SPLIT kernels only)
  int wait_n, wait_from_elem;
  int iso;  // all coefficient matrices are multiples of the identity
  double Bo[4 * P_];
  double Bc[4 * (P_ + 1)];
  double Gc[4 * (P_ + 1)];
};

constexpr int nd5_pad_to(int len, int target)  // smallest pad with (len + pad) % 16 == target
{
  return ((target - len) % 16 + 16) % 16;
}

template <int P_, int KIND, bool ASM>
struct ND5Layout
{
  static constexpr int p = P_, q = 4, n = P_ + 1, Q = 64, P = 3 * p * n * n, D3 = p * n * n;
  static constexpr int PS = (P + 3) & ~3;
  static constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS);
  static constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS);
  static constexpr int NXA = p * q, NNA = n * q;  // items (qz,i) of one row
  // Z region, group A: rows j < n: [XA][XB][ZA]; row stride = 1 (mod 16) doubles
  static constexpr int A_XA = 0, A_XB = A_XA + NXA, A_ZA = A_XB + (CURL ? NXA : 0), LA = A_ZA + NNA, RSA = LA + nd5_pad_to(LA, 1);
  // Z region, group B: rows j < p: [YA][YB]
  static constexpr int B_YA = 0, B_YB = B_YA + NNA, LB = B_YB + (CURL ? NNA : 0), RSB = LB + nd5_pad_to(LB, 1);
  static constexpr int ZA0 = 0, ZB0 = ZA0 + n * RSA, ZSZ = ZB0 + p * RSB;
  // Y region: rows qy < 4: [X1][X2][X3][Y1][Y2][Z1][Z3]; row stride = 4 (mod 8) doubles
  static constexpr int Y_X1 = 0, Y_X2 = Y_X1 + (MASS ? NXA : 0), Y_X3 = Y_X2 + (CURL ? NXA : 0), Y_Y1 = Y_X3 + (CURL ? NXA : 0),
                       Y_Y2 = Y_Y1 + NNA, Y_Z1 = Y_Y2 + (CURL ? NNA : 0), Y_Z3 = Y_Z1 + NNA, LY = Y_Z3 + (CURL ? NNA : 0),
                       RSY = LY + ((LY % 8 == 4) ? 0 : nd5_pad_to(LY, 4));
  static constexpr int Y0 = ZSZ, WTOT = (Y0 + q * RSY + 1) & ~1;
  static constexpr int GCOMP = ASM ? ((MASS ? 9 : 0) + (CURL ? 9 : 0)) : 10;
  static constexpr int GE = (GCOMP * Q + 1) & ~1;
  static constexpr int CE = 18;
  // per-warp shared memory (bytes), every block 16-byte aligned
  static constexpr int OFF_G = 0;
  static constexpr int OFF_W = OFF_G + GE * 8;
  static constexpr int OFF_U = OFF_W + WTOT * 8;         // [PS] doubles: staged x values
  static constexpr int OFF_I = OFF_U + PS * 8;           // [3][PS] int32: restriction index ring
  static constexpr int OFF_C = OFF_I + 3 * PS * 4;       // [18] doubles
  static constexpr int OFF_B = OFF_C + CE * 8;           // 4 mbarriers
  static constexpr int WS = (OFF_B + 4 * 8 + 15) & ~15;
};

template <int P_, int KIND, bool ASM, bool SPLIT, int NW, int MINB>
__global__ void __launch_bounds__(NW * 32, MINB) nd_hex_apply5_kernel(const __grid_constant__ ND5Params<P_> prm)
{
  using L = ND5Layout<P_, KIND, ASM>;
  constexpr int p = L::p, q = 4, n = L::n, Q = L::Q, D3 = L::D3, GE = L::GE, PS = L::PS, QQ = 16;
  constexpr int RSA = L::RSA, RSB = L::RSB, RSY = L::RSY;
  constexpr bool MASS = L::MASS, CURL = L::CURL;
  constexpr int IPX = p * n, IPZ = n * n, IX = p * q, IN = n * q;
  static_assert(IPX <= 16 && IPZ <= 16 && IX <= 16 && IN <= 16, "one half-warp per item set");

  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int h = lane >> 4, t = lane & 15;
  const double sgn = h ? -1.0 : 1.0;
  unsigned char *wbase = smem_raw + (size_t)wid * L::WS;
  double *sG = (double *)(wbase + L::OFF_G);
  double *sW = (double *)(wbase + L::OFF_W);
  double *sU = (double *)(wbase + L::OFF_U);
  int32_t *sI = (int32_t *)(wbase + L::OFF_I);
  double *sC = (double *)(wbase + L::OFF_C);
  uint64_t *bar_g = (uint64_t *)(wbase + L::OFF_B);
  uint64_t *bar_i = bar_g + 1;  // [3]

  const int nb = prm.ne;          // one element per batch
  const int GW = gridDim.x * NW;  // warps in the grid
  int b = blockIdx.x * NW + wid;
  if (b >= nb) return;            // (whole warp)

  if (lane == 0)
  {
    mbar_init(bar_g, 1);
    mbar_init(bar_i + 0, 1);
    mbar_init(bar_i + 1, 1);
    mbar_init(bar_i + 2, 1);
  }
  __syncwarp();

  auto issue_idx = [&](int bb, int slot)
  {
    constexpr uint32_t bytes = (uint32_t)(PS * sizeof(int32_t));
    mbar_expect_tx(bar_i + slot, bytes);
    tma_bulk_g2s(sI + slot * PS, prm.lidx + (size_t)bb * PS, bytes, bar_i + slot);
  };
  auto issue_geom = [&](int bb)
  {
    constexpr uint32_t bytes = (uint32_t)(GE * sizeof(double));
    constexpr uint32_t cbytes = ASM ? 0u : (uint32_t)(18 * sizeof(double));
    mbar_expect_tx(bar_g, bytes + cbytes);
    tma_bulk_g2s(sG, (ASM ? prm.aq : prm.qd) + (size_t)bb * GE, bytes, bar_g);
    if (!ASM) tma_bulk_g2s(sC, prm.ecoef + (size_t)bb * 18, cbytes, bar_g);
  };
  // x values of element bb -> sU (raw; the sign is applied when they are read)
  auto gather_x = [&](int slot)
  {
    const int32_t *gI = sI + slot * PS;
    constexpr int ITER = (PS + 31) / 32;
#pragma unroll
    for (int r = 0; r < ITER; r++)
    {
      const int l = lane + 32 * r;
      if (l < PS)
      {
        const int32_t gi = gI[l];
        if (gi == B2P_SKIP_IDX)
          sU[l] = 0.0;  // masked / padding: reads as zero
        else if (SPLIT)
          cp_async8(sU + l, split_src_fast(prm.x, prm.sp, abs_idx(gi)));
        else
          cp_async8(sU + l, prm.x + (uint32_t)abs_idx(gi));
      }
    }
    cp_async_commit();
  };

  // Peer-memory halo: ghost values of this step are complete once every neighbour's flag reached the expected epoch.
  bool ghosts_ready = !(SPLIT && prm.wait_n > 0);
  auto wait_ghosts = [&](int bb)
  {
    if (ghosts_ready || (bb + 1) <= prm.wait_from_elem) return;
    if (lane < prm.wait_n)
    {
      const unsigned long long want = prm.wait_expect[lane];
      unsigned long long v;
      do
      {
        v = ld_acquire_sys_u64(prm.wait_flags + lane);
      } while (v < want);
    }
    __syncwarp();
    ghosts_ready = true;
  };

  uint32_t par_g = 0, par_i = 0;
  if (lane == 0)
  {
    issue_idx(b, 0);
    if (b + GW < nb) issue_idx(b + GW, 1);
    if (b + 2 * GW < nb) issue_idx(b + 2 * GW, 2);
    issue_geom(b);
  }
  mbar_wait(bar_i + 0, 0);
  par_i ^= 1u;
  wait_ghosts(b);
  gather_x(0);

  const double alpha = prm.alpha;
  // lane roles that do not change: x-/y-directed item of the Z and Zt phases, z-directed item, (qz,i) items of Y / Yt
  const bool vxy = t < IPX, vz = t < IPZ, vx = t < IX, vn = t < IN;
  const int txy = vxy ? t : 0, tz = vz ? t : 0, wx = vx ? t : 0, wn = vn ? t : 0;
  // half 0: x-directed dof txy = i + p*j -> XA row j ; half 1: y-directed dof txy = i + n*j -> YA row j
  const int rowx_off = h ? (L::ZB0 + (txy / n) * RSB + L::B_YA + q * (txy % n)) : (L::ZA0 + (txy / p) * RSA + L::A_XA + q * (txy % p));
  const int offb = h ? (L::B_YB - L::B_YA) : (L::A_XB - L::A_XA);
  const int rowz_off = L::ZA0 + (tz / n) * RSA + L::A_ZA + q * (tz % n);

  int slot = 0;
  for (; b < nb; b += GW)
  {
    const int nslot = (slot == 2) ? 0 : slot + 1;
    const int bn = b + GW;
    const int32_t *cI = sI + slot * PS;
    const double *cU = sU;

    cp_async_wait<0>();
    __syncwarp();

    // ------------------------------------------------------------------ phase Z (z-contraction)
    {
      double ux[n], uz[p];
#pragma unroll
      for (int k = 0; k < n; k++) ux[k] = staged(cI, cU, h * D3 + txy + IPX * k, true);
#pragma unroll
      for (int k = 0; k < p; k++) uz[k] = staged(cI, cU, 2 * D3 + tz + IPZ * (h ? p - 1 - k : k), true);
      double *rowx = sW + rowx_off;
#pragma unroll
      for (int qz = 0; qz < q; qz++)
      {
        double a = 0.0, bb = 0.0;
#pragma unroll
        for (int k = 0; k < n; k++)
        {
          a += prm.Bc[qz * n + k] * ux[k];
          if (CURL) bb += prm.Gc[qz * n + k] * ux[k];
        }
        if (vxy)
        {
          rowx[qz] = a;
          if (CURL) rowx[offb + qz] = bb;
        }
      }
      // z-directed: this half's two qz (half 1 mirrored: point q-1-c from the reversed dofs)
      double *rowz = sW + rowz_off;
#pragma unroll
      for (int c = 0; c < 2; c++)
      {
        double a = 0.0;
#pragma unroll
        for (int k = 0; k < p; k++) a += prm.Bo[c * p + k] * uz[k];
        if (vz) rowz[h ? q - 1 - c : c] = a;
      }
    }
    __syncwarp();
    // the staged x values are consumed: gather the next element's while this one computes
    if (bn < nb)
    {
      mbar_wait(bar_i + nslot, (par_i >> nslot) & 1u);
      par_i ^= (1u << nslot);
      wait_ghosts(bn);
      gather_x(nslot);
    }

    // ------------------------------------------------------------------ phase Y (y-contraction)
    // item (qz,i) = column of a row; this half's two qy (half 1: rows j read in reversed order)
    {
      const int sA = h ? -RSA : RSA, sB = h ? -RSB : RSB;
      double xa[n], xb[n], ya[p], yb[p], za[n];
      {
        const double *pa = sW + L::ZA0 + (h ? (n - 1) * RSA : 0) + L::A_XA + wx;
        const double *qa = sW + L::ZB0 + (h ? (p - 1) * RSB : 0) + L::B_YA + wn;
        const double *ra = sW + L::ZA0 + (h ? (n - 1) * RSA : 0) + L::A_ZA + wn;
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          xa[j] = pa[sA * j];
          if (CURL) xb[j] = pa[(L::A_XB - L::A_XA) + sA * j];
          za[j] = ra[sA * j];
        }
#pragma unroll
        for (int j = 0; j < p; j++)
        {
          ya[j] = qa[sB * j];
          if (CURL) yb[j] = qa[(L::B_YB - L::B_YA) + sB * j];
        }
      }
#pragma unroll
      for (int c = 0; c < 2; c++)
      {
        double *row = sW + L::Y0 + (h ? q - 1 - c : c) * RSY;
        double s1 = 0.0, s2 = 0.0, s3 = 0.0, v1 = 0.0, v2 = 0.0, t1 = 0.0, t3 = 0.0;
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          if (MASS) s1 += prm.Bc[c * n + j] * xa[j];
          if (CURL) s2 += prm.Bc[c * n + j] * xb[j];
          if (CURL) s3 += prm.Gc[c * n + j] * xa[j];
          t1 += prm.Bc[c * n + j] * za[j];
          if (CURL) t3 += prm.Gc[c * n + j] * za[j];
        }
#pragma unroll
        for (int j = 0; j < p; j++)
        {
          v1 += prm.Bo[c * p + j] * ya[j];
          if (CURL) v2 += prm.Bo[c * p + j] * yb[j];
        }
        if (vx)
        {
          if (MASS) row[L::Y_X1 + wx] = s1;
          if (CURL) row[L::Y_X2 + wx] = s2;
          if (CURL) row[L::Y_X3 + wx] = sgn * s3;
        }
        if (vn)
        {
          row[L::Y_Y1 + wn] = v1;
          if (CURL) row[L::Y_Y2 + wn] = v2;
          row[L::Y_Z1 + wn] = t1;
          if (CURL) row[L::Y_Z3 + wn] = sgn * t3;
        }
      }
    }
    __syncwarp();
    mbar_wait(bar_g, par_g);  // q-data of this element has landed
    par_g ^= 1;

    // ------------------------------------------------------------------ phase XDX
    // line s = qy + 4 qz = t; this half's two qx (half 1: points 3, 2 from the reversed dofs)
    {
      const int qy = t & 3, qz = t >> 2;
      double *WXb = sW + L::Y0 + qy * RSY + qz;
      const int si = h ? -q : q;
      double vv[2][3], cw[2][3];
      {
        const double *Xp = WXb + (h ? q * (p - 1) : 0), *Np = WXb + (h ? q * (n - 1) : 0);
        double x1[p], x2[p], x3[p], y1[n], y2[n], z1[n], z3[n];
#pragma unroll
        for (int i = 0; i < p; i++)
        {
          if (MASS) x1[i] = Xp[L::Y_X1 + si * i];
          if (CURL) x2[i] = Xp[L::Y_X2 + si * i];
          if (CURL) x3[i] = Xp[L::Y_X3 + si * i];
        }
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          y1[i] = Np[L::Y_Y1 + si * i];
          if (CURL) y2[i] = Np[L::Y_Y2 + si * i];
          z1[i] = Np[L::Y_Z1 + si * i];
          if (CURL) z3[i] = Np[L::Y_Z3 + si * i];
        }
#pragma unroll
        for (int c = 0; c < 2; c++)
        {
          double u0 = 0, u1 = 0, u2 = 0, dzux = 0, dyux = 0, dzuy = 0, dxuy = 0, dyuz = 0, dxuz = 0;
#pragma unroll
          for (int i = 0; i < p; i++)
          {
            if (MASS) u0 += prm.Bo[c * p + i] * x1[i];
            if (CURL) dzux += prm.Bo[c * p + i] * x2[i];
            if (CURL) dyux += prm.Bo[c * p + i] * x3[i];
          }
#pragma unroll
          for (int i = 0; i < n; i++)
          {
            if (MASS) u1 += prm.Bc[c * n + i] * y1[i];
            if (CURL) dzuy += prm.Bc[c * n + i] * y2[i];
            if (CURL) dxuy += prm.Gc[c * n + i] * y1[i];
            if (MASS) u2 += prm.Bc[c * n + i] * z1[i];
            if (CURL) dyuz += prm.Bc[c * n + i] * z3[i];
            if (CURL) dxuz += prm.Gc[c * n + i] * z1[i];
          }
          vv[c][0] = u0;
          vv[c][1] = u1;
          vv[c][2] = u2;
          cw[c][0] = dyuz - dzuy;
          cw[c][1] = dzux - sgn * dxuz;  // derivative terms of the mirrored half change sign
          cw[c][2] = sgn * dxuy - dyux;
        }
      }
      // pointwise D in place
      const double *C = sC;
#pragma unroll
      for (int c = 0; c < 2; c++)
      {
        const int qx = h ? q - 1 - c : c;
        const double *gq = sG + QQ * qx + t;
        double v[3] = {0, 0, 0}, w[3] = {0, 0, 0};
        if (ASM)
        {
          const double *a = gq;
          if (MASS)
          {
#pragma unroll
            for (int r = 0; r < 3; r++) v[r] = alpha * (a[(r)*Q] * vv[c][0] + a[(r + 3) * Q] * vv[c][1] + a[(r + 6) * Q] * vv[c][2]);
            a += 9 * Q;
          }
          if (CURL)
          {
#pragma unroll
            for (int r = 0; r < 3; r++) w[r] = alpha * (a[(r)*Q] * cw[c][0] + a[(r + 3) * Q] * cw[c][1] + a[(r + 6) * Q] * cw[c][2]);
          }
        }
        else
        {
          const double wdetJ = alpha * gq[0];  // alpha folded into the quadrature weight
          double A[9];
#pragma unroll
          for (int i = 0; i < 9; i++) A[i] = gq[(1 + i) * Q];
          if (prm.iso)
          {
            if (MASS) AtAx(A, vv[c], wdetJ * C[0], v);
            if (CURL)
            {
              double Jd[9];
              cofactor33(A, Jd);
              AtAx(Jd, cw[c], wdetJ * C[9], w);
            }
          }
          else
          {
            if (MASS) AtCAx(A, C, vv[c], wdetJ, v);
            if (CURL)
            {
              double Jd[9];
              cofactor33(A, Jd);
              AtCAx(Jd, C + 9, cw[c], wdetJ, w);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < 3; r++)
        {
          vv[c][r] = v[r];
          cw[c][r] = w[r];
        }
      }
      // transposed x-contraction: partial sums over this half's two points for the (mirrored) output index;
      // output i of half 0 pairs with output len-1-i of half 1
      const double g1[2] = {sgn * cw[0][1], sgn * cw[1][1]}, g2[2] = {sgn * cw[0][2], sgn * cw[1][2]};
      {
        double a1[p], a2[p], a3[p];
#pragma unroll
        for (int i = 0; i < p; i++)
        {
          a1[i] = a2[i] = a3[i] = 0.0;
#pragma unroll
          for (int c = 0; c < 2; c++)
          {
            if (MASS) a1[i] += prm.Bo[c * p + i] * vv[c][0];
            if (CURL) a2[i] += prm.Bo[c * p + i] * cw[c][1];
            if (CURL) a3[i] -= prm.Bo[c * p + i] * cw[c][2];
          }
        }
        double *Xo = WXb + (h ? q * (p - 1) : 0);
#pragma unroll
        for (int i = 0; i < (p + 1) / 2; i++)
        {
          if (MASS) Xo[L::Y_X1 + si * i] = a1[i] + __shfl_xor_sync(0xffffffffu, a1[p - 1 - i], 16);
          if (CURL) Xo[L::Y_X2 + si * i] = a2[i] + __shfl_xor_sync(0xffffffffu, a2[p - 1 - i], 16);
          if (CURL) Xo[L::Y_X3 + si * i] = a3[i] + __shfl_xor_sync(0xffffffffu, a3[p - 1 - i], 16);
        }
      }
      {
        double b1[n], b2[n], c1[n], c3[n];
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          b1[i] = b2[i] = c1[i] = c3[i] = 0.0;
#pragma unroll
          for (int c = 0; c < 2; c++)
          {
            if (MASS) b1[i] += prm.Bc[c * n + i] * vv[c][1];
            if (CURL) b1[i] += prm.Gc[c * n + i] * g2[c];
            if (CURL) b2[i] -= prm.Bc[c * n + i] * cw[c][0];
            if (MASS) c1[i] += prm.Bc[c * n + i] * vv[c][2];
            if (CURL) c1[i] -= prm.Gc[c * n + i] * g1[c];
            if (CURL) c3[i] += prm.Bc[c * n + i] * cw[c][0];
          }
        }
        double *No = WXb + (h ? q * (n - 1) : 0);
#pragma unroll
        for (int i = 0; i < (n + 1) / 2; i++)
        {
          No[L::Y_Y1 + si * i] = b1[i] + __shfl_xor_sync(0xffffffffu, b1[n - 1 - i], 16);
          if (CURL) No[L::Y_Y2 + si * i] = b2[i] + __shfl_xor_sync(0xffffffffu, b2[n - 1 - i], 16);
          No[L::Y_Z1 + si * i] = c1[i] + __shfl_xor_sync(0xffffffffu, c1[n - 1 - i], 16);
          if (CURL) No[L::Y_Z3 + si * i] = c3[i] + __shfl_xor_sync(0xffffffffu, c3[n - 1 - i], 16);
        }
      }
    }
    __syncwarp();
    if (bn < nb && lane == 0)
    {
      fence_proxy_async();
      issue_geom(bn);  // refill the single q-data buffer for the next element
    }

    // ------------------------------------------------------------------ phase Yt (transposed y-contraction)
    {
      const int sR = h ? -RSY : RSY;
      const double *r0 = sW + L::Y0 + (h ? (q - 1) * RSY : 0);
      double X1[2], X2[2], X3[2], Y1[2], Y2[2], Z1[2], Z3[2];
#pragma unroll
      for (int c = 0; c < 2; c++)
      {
        if (MASS) X1[c] = r0[sR * c + L::Y_X1 + wx];
        if (CURL) X2[c] = r0[sR * c + L::Y_X2 + wx];
        if (CURL) X3[c] = sgn * r0[sR * c + L::Y_X3 + wx];
        Y1[c] = r0[sR * c + L::Y_Y1 + wn];
        if (CURL) Y2[c] = r0[sR * c + L::Y_Y2 + wn];
        Z1[c] = r0[sR * c + L::Y_Z1 + wn];
        if (CURL) Z3[c] = sgn * r0[sR * c + L::Y_Z3 + wn];
      }
      const int sA = h ? -RSA : RSA, sB = h ? -RSB : RSB;
      {
        // x-directed: Za'[j] = sum_qy Bc[qy][j] W1 + Gc[qy][j] W3 ; Zb'[j] = sum_qy Bc[qy][j] W2
        double pa[n], pb[n], ra[n];
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          pa[j] = pb[j] = ra[j] = 0.0;
#pragma unroll
          for (int c = 0; c < 2; c++)
          {
            if (MASS) pa[j] += prm.Bc[c * n + j] * X1[c];
            if (CURL) pa[j] += prm.Gc[c * n + j] * X3[c];
            if (CURL) pb[j] += prm.Bc[c * n + j] * X2[c];
            ra[j] += prm.Bc[c * n + j] * Z1[c];
            if (CURL) ra[j] += prm.Gc[c * n + j] * Z3[c];
          }
        }
        double *za = sW + L::ZA0 + (h ? (n - 1) * RSA : 0) + L::A_XA + wx;
        double *zz = sW + L::ZA0 + (h ? (n - 1) * RSA : 0) + L::A_ZA + wn;
#pragma unroll
        for (int j = 0; j < (n + 1) / 2; j++)
        {
          const double ta = pa[j] + __shfl_xor_sync(0xffffffffu, pa[n - 1 - j], 16);
          const double tb = CURL ? pb[j] + __shfl_xor_sync(0xffffffffu, pb[n - 1 - j], 16) : 0.0;
          const double tr = ra[j] + __shfl_xor_sync(0xffffffffu, ra[n - 1 - j], 16);
          if (vx)
          {
            za[sA * j] = ta;
            if (CURL) za[(L::A_XB - L::A_XA) + sA * j] = tb;
          }
          if (vn) zz[sA * j] = tr;
        }
      }
      {
        // y-directed: Za'[j<p] = sum_qy Bo[qy][j] W1 ; Zb' = sum_qy Bo[qy][j] W2
        double qa[p], qb[p];
#pragma unroll
        for (int j = 0; j < p; j++)
        {
          qa[j] = qb[j] = 0.0;
#pragma unroll
          for (int c = 0; c < 2; c++)
          {
            qa[j] += prm.Bo[c * p + j] * Y1[c];
            if (CURL) qb[j] += prm.Bo[c * p + j] * Y2[c];
          }
        }
        double *ya = sW + L::ZB0 + (h ? (p - 1) * RSB : 0) + L::B_YA + wn;
#pragma unroll
        for (int j = 0; j < (p + 1) / 2; j++)
        {
          const double ta = qa[j] + __shfl_xor_sync(0xffffffffu, qa[p - 1 - j], 16);
          const double tb = CURL ? qb[j] + __shfl_xor_sync(0xffffffffu, qb[p - 1 - j], 16) : 0.0;
          if (vn)
          {
            ya[sB * j] = ta;
            if (CURL) ya[(L::B_YB - L::B_YA) + sB * j] = tb;
          }
        }
      }
    }
    __syncwarp();

    // ------------------------------------------------------------------ phase Zt (transposed z-contraction + scatter)
    {
      double xa[q], xb[q], za[q];
      int32_t gx[n], gz[p];
      {
        const double *rowx = sW + rowx_off, *rowz = sW + rowz_off;
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          xa[qz] = rowx[qz];
          if (CURL) xb[qz] = rowx[offb + qz];
          za[qz] = rowz[qz];
        }
#pragma unroll
        for (int k = 0; k < n; k++) gx[k] = cI[h * D3 + txy + IPX * k];
#pragma unroll
        for (int k = 0; k < p; k++) gz[k] = cI[2 * D3 + tz + IPZ * k];
      }
#pragma unroll
      for (int k = 0; k < n; k++)
      {
        double o = 0.0;
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          o += prm.Bc[qz * n + k] * xa[qz];
          if (CURL) o += prm.Gc[qz * n + k] * xb[qz];
        }
        const int32_t g = vxy ? gx[k] : B2P_SKIP_IDX;
        if (SPLIT) scatter_fast_split(prm.y, prm.sp, g, o); else scatter_fast(prm.y, g, o);
      }
#pragma unroll
      for (int k = 0; k < p; k++)
      {
        double o = 0.0;
#pragma unroll
        for (int qz = 0; qz < q; qz++) o += prm.Bo[qz * p + k] * za[qz];
        const int32_t g = (vz && h == 0) ? gz[k] : B2P_SKIP_IDX;
        if (SPLIT) scatter_fast_split(prm.y, prm.sp, g, o); else scatter_fast(prm.y, g, o);
      }
    }
    __syncwarp();
    if (b + 3 * GW < nb && lane == 0)
    {
      fence_proxy_async();
      issue_idx(b + 3 * GW, slot);  // this element's index slot is free again
    }
    slot = nslot;
  }
}

template <int P_, int KIND, bool ASM, int MINB_WANT>
int launch5(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  using L = ND5Layout<P_, KIND, ASM>;
  constexpr int NW = 4;
  constexpr size_t shmem = (size_t)NW * L::WS;
  constexpr int FIT = (int)((228 * 1024) / (shmem + 1024));  // CTAs per SM that fit in shared memory
  constexpr int MINB = MINB_WANT < FIT ? MINB_WANT : FIT;
  static_assert(MINB >= 1, "shared memory per SM");
  const bool split = range_split(op, rg);
  auto kern = split ? nd_hex_apply5_kernel<P_, KIND, ASM, true, NW, MINB> : nd_hex_apply5_kernel<P_, KIND, ASM, false, NW, MINB>;
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem, cudaSharedmemCarveoutMaxShared)) return rc;
  ND5Params<P_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.aq = op->aq ? op->aq + (size_t)e_off * op->aq_estride : nullptr;
  prm.ecoef = op->ecoef ? op->ecoef + 18 * (size_t)e_off : nullptr;
  prm.x = x;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  set_split_wait(prm, op, rg);
  prm.iso = op->iso ? 1 : 0;
  copy_tables(op->h_tab.data(), P_, 4, 4, prm.Bo, prm.Bc, prm.Gc);
  return launch_persistent(kern, prm, NW * 32, shmem, s, false, op->ctx, "nd_hex_apply5_kernel", false, false, op->ctx->sm_count * MINB, NW, 1,
                           e_cnt);
}

template <int P_, int MINB>
int launch5_kind(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  const bool a = op->assembled;
  switch (op->kind)
  {
    case B2P_CURLCURL:
      return a ? launch5<P_, B2P_CURLCURL, true, MINB>(op, lidx, alpha, x, y, rg, s)
               : launch5<P_, B2P_CURLCURL, false, MINB>(op, lidx, alpha, x, y, rg, s);
    case B2P_ND_MASS:
      return a ? launch5<P_, B2P_ND_MASS, true, MINB>(op, lidx, alpha, x, y, rg, s)
               : launch5<P_, B2P_ND_MASS, false, MINB>(op, lidx, alpha, x, y, rg, s);
    case B2P_CURLCURL_MASS:
      return a ? launch5<P_, B2P_CURLCURL_MASS, true, MINB>(op, lidx, alpha, x, y, rg, s)
               : launch5<P_, B2P_CURLCURL_MASS, false, MINB>(op, lidx, alpha, x, y, rg, s);
  }
  set_error(op->ctx, "nd_hex_apply5: unsupported kind %d", op->kind);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace

// True when this operator can run on the one-element-per-warp kernel.
bool nd_hex_apply5_eligible(b2p_op *op)
{
  return op->q1d == 4 && op->p == 3 && nd_tables_symmetric(op, 1e-13);
}

int launch_nd_hex_apply5(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  static const int minb = []
  {
    const char *e = std::getenv("B2P_ND5_MINB");
    return e ? std::atoi(e) : 3;
  }();
  if (minb == 4) return launch5_kind<3, 4>(op, lidx, alpha, x, y, rg, s);
  return launch5_kind<3, 3>(op, lidx, alpha, x, y, rg, s);
}

}  // namespace b2p
