// H1 hexahedron diffusion apply on the warp-autonomous persistent pipeline (see b2p_hex_nd3.cu for
// the design): y_L += alpha * sum_e E^T G^T D G E x_L, D = w detJ J^-1 C J^-T on the reference gradient.
// This is the auxiliary-space operator of the Hiptmair smoother: with Chebyshev order max(2p, 4) it is
// applied as often as the Nedelec operator inside every V-cycle
// (/root/reference/palace/linalg/distrelaxation.cpp:99-151, /root/reference/palace/fem/integ/diffusion.cpp:16-73,
// /root/reference/palace/fem/qfunctions/33/hcurl_33_qf.h:10-29).
//
// Scalar field, so every phase has exactly n^2 or n*q or q^2 items per element:
//   Z   (i,j) pencils:  a = Bc_z u, b = Gc_z u
//   Y   (i,qz) pencils: V1 = Bc_y a, V2 = Gc_y a, V3 = Bc_y b
//   XDX (qy,qz) lines:  g = (Gc_x V1, Bc_x V2, Bc_x V3) for all qx in registers, D, transpose
//   Yt, Zt mirror Y, Z; Zt scatters with RED.F64.
#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

template <int P_, int Q_>
struct H1V3Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction, rows padded to 16 bytes
  const double *qd;     // [ne][10][Q] geometry (x-slowest) or null
  const double *aq;     // [ne][9][Q] assembled D (x-slowest) or null
  const double *ecoef;  // [ne][18]
  const double *x;
  double *y;
  double alpha;
  int ne;
  VSplit sp;
  double Bc[Q_ * (P_ + 1)];
  double Gc[Q_ * (P_ + 1)];
};

template <int P_, int Q_, bool ASM>
struct H1V3Layout
{
  static constexpr int q = Q_, n = P_ + 1, Q = q * q * q, P = n * n * n;
  static constexpr int PS = (P + 3) & ~3;
  static constexpr int ZA = 0, ZB = ZA + n * n * q, ZSZ = ZB + n * n * q;            // index qz + q*(i + n*j)
  static constexpr int Y1 = ZSZ, Y2 = Y1 + n * q * q, Y3 = Y2 + n * q * q, YEND = Y3 + n * q * q;  // qy + q*(qz + q*i)
  static constexpr int ES = (YEND + 1) & ~1;
  static constexpr int GCOMP = ASM ? 9 : 10;
  static constexpr int GE = (GCOMP * Q + 1) & ~1;
  static constexpr int CE = 18;
  static constexpr int NEW = (q * q >= 32) ? 1 : 32 / (q * q);
  static constexpr int OFF_G = 0;
  static constexpr int OFF_W = OFF_G + NEW * GE * 8;
  static constexpr int OFF_U = OFF_W + NEW * ES * 8;
  static constexpr int OFF_I = OFF_U + NEW * PS * 8;
  static constexpr int OFF_C = OFF_I + 3 * NEW * PS * 4;
  static constexpr int OFF_B = OFF_C + ((NEW * CE * 8 + 15) & ~15);
  static constexpr int WS = (OFF_B + 4 * 8 + 15) & ~15;
};

template <int P_, int Q_, bool ASM, bool SPLIT, int NW, int MINB>
__global__ void __launch_bounds__(NW * 32, MINB) h1_hex_apply3_kernel(const __grid_constant__ H1V3Params<P_, Q_> prm)
{
  using L = H1V3Layout<P_, Q_, ASM>;
  constexpr int q = L::q, n = L::n, Q = L::Q, ES = L::ES, GE = L::GE, PS = L::PS, NEW = L::NEW;
  constexpr int QQ = q * q;

  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned char *wbase = smem_raw + (size_t)wid * L::WS;
  double *sG = (double *)(wbase + L::OFF_G);
  double *sW = (double *)(wbase + L::OFF_W);
  double *sU = (double *)(wbase + L::OFF_U);
  int32_t *sI = (int32_t *)(wbase + L::OFF_I);
  double *sC = (double *)(wbase + L::OFF_C);
  uint64_t *bar_g = (uint64_t *)(wbase + L::OFF_B);
  uint64_t *bar_i = bar_g + 1;

  const int nb = (prm.ne + NEW - 1) / NEW;
  const int GW = gridDim.x * NW;
  int b = blockIdx.x * NW + wid;
  if (b >= nb) return;

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
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const uint32_t bytes = (uint32_t)(nel * PS * sizeof(int32_t));
    mbar_expect_tx(bar_i + slot, bytes);
    tma_bulk_g2s(sI + slot * NEW * PS, prm.lidx + (size_t)e0 * PS, bytes, bar_i + slot);
  };
  auto issue_geom = [&](int bb)
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const uint32_t bytes = (uint32_t)(nel * GE * sizeof(double));
    const uint32_t cbytes = ASM ? 0u : (uint32_t)(nel * 18 * sizeof(double));
    mbar_expect_tx(bar_g, bytes + cbytes);
    tma_bulk_g2s(sG, (ASM ? prm.aq : prm.qd) + (size_t)e0 * GE, bytes, bar_g);
    if (!ASM) tma_bulk_g2s(sC, prm.ecoef + (size_t)e0 * 18, cbytes, bar_g);
  };
  auto gather_x = [&](int bb, int slot)
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const int32_t *gI = sI + slot * NEW * PS;
    constexpr int ITER = (NEW * PS + 31) / 32;
#pragma unroll
    for (int r = 0; r < ITER; r++)
    {
      const int l = lane + 32 * r;
      if (l < nel * PS)
      {
        const int32_t gi = gI[l];
        if (gi == B2P_SKIP_IDX)
          sU[l] = 0.0;
        else if (SPLIT)
          cp_async8(sU + l, split_src_fast(prm.x, prm.sp, abs_idx(gi)));
        else
          cp_async8(sU + l, prm.x + (uint32_t)abs_idx(gi));
      }
    }
    cp_async_commit();
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
  gather_x(b, 0);

  const double alpha = prm.alpha;
  int slot = 0;
  for (; b < nb; b += GW)
  {
    const int nslot = (slot == 2) ? 0 : slot + 1;
    const int bn = b + GW;
    const int e0 = b * NEW, nel = min(NEW, prm.ne - e0);
    const int32_t *cI = sI + slot * NEW * PS;
    const double *cU = sU;

    cp_async_wait<0>();
    __syncwarp();

    // ---------------------------------------------------------------- phase Z: items (e, t = i + n*j)
    {
      constexpr int IT = NEW * n * n, ROUNDS = (IT + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool v = w < IT;
        const int wc = v ? w : 0, e = wc / (n * n), t = wc % (n * n);
        double u[n];
#pragma unroll
        for (int k = 0; k < n; k++) u[k] = staged(cI, cU, e * PS + t + n * n * k, e < nel);
        if (v)
        {
          double *za = sW + e * ES + L::ZA + q * t, *zb = sW + e * ES + L::ZB + q * t;
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            double a = 0.0, bb = 0.0;
#pragma unroll
            for (int k = 0; k < n; k++)
            {
              a += prm.Bc[qz * n + k] * u[k];
              bb += prm.Gc[qz * n + k] * u[k];
            }
            za[qz] = a;
            zb[qz] = bb;
          }
        }
      }
    }
    __syncwarp();
    if (bn < nb)
    {
      mbar_wait(bar_i + nslot, (par_i >> nslot) & 1u);
      par_i ^= (1u << nslot);
      gather_x(bn, nslot);
    }

    // ---------------------------------------------------------------- phase Y: items (e, t = qz + q*i)
    {
      constexpr int IT = NEW * n * q, ROUNDS = (IT + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool v = w < IT;
        const int wc = v ? w : 0, e = wc / (n * q), t = wc % (n * q), qz = t % q, i = t / q;
        const double *pa = sW + e * ES + L::ZA + qz + q * i, *pb = sW + e * ES + L::ZB + qz + q * i;
        double a[n], bb[n];
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          a[j] = pa[q * n * j];
          bb[j] = pb[q * n * j];
        }
        if (v)
        {
          double *v1 = sW + e * ES + L::Y1 + q * t, *v2 = sW + e * ES + L::Y2 + q * t, *v3 = sW + e * ES + L::Y3 + q * t;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            double s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              s1 += prm.Bc[qy * n + j] * a[j];
              s2 += prm.Gc[qy * n + j] * a[j];
              s3 += prm.Bc[qy * n + j] * bb[j];
            }
            v1[qy] = s1;
            v2[qy] = s2;
            v3[qy] = s3;
          }
        }
      }
    }
    __syncwarp();
    mbar_wait(bar_g, par_g);
    par_g ^= 1;

    // ---------------------------------------------------------------- phase XDX: items (e, s = qy + q*qz)
    for (int w = lane; w < NEW * QQ; w += 32)
    {
      const int e = w / QQ, s = w % QQ;
      double *W = sW + e * ES + s;
      double gg[q][3];
      {
        double x1[n], x2[n], x3[n];
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          x1[i] = W[L::Y1 + QQ * i];
          x2[i] = W[L::Y2 + QQ * i];
          x3[i] = W[L::Y3 + QQ * i];
        }
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          double g0 = 0, g1 = 0, g2 = 0;
#pragma unroll
          for (int i = 0; i < n; i++)
          {
            g0 += prm.Gc[qx * n + i] * x1[i];
            g1 += prm.Bc[qx * n + i] * x2[i];
            g2 += prm.Bc[qx * n + i] * x3[i];
          }
          gg[qx][0] = g0;
          gg[qx][1] = g1;
          gg[qx][2] = g2;
        }
      }
      const double *g = sG + e * GE + s;
      const double *C = sC + e * 18;
#pragma unroll
      for (int qx = 0; qx < q; qx++)
      {
        double v[3] = {0, 0, 0};
        if (e < nel)
        {
          const double *gq = g + QQ * qx;
          if (ASM)
          {
#pragma unroll
            for (int r = 0; r < 3; r++) v[r] = alpha * (gq[(r)*Q] * gg[qx][0] + gq[(r + 3) * Q] * gg[qx][1] + gq[(r + 6) * Q] * gg[qx][2]);
          }
          else
          {
            double A[9];
#pragma unroll
            for (int i = 0; i < 9; i++) A[i] = gq[(1 + i) * Q];
            AtCAx(A, C, gg[qx], alpha * gq[0], v);
          }
        }
#pragma unroll
        for (int r = 0; r < 3; r++) gg[qx][r] = v[r];
      }
#pragma unroll
      for (int i = 0; i < n; i++)
      {
        double a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          a1 += prm.Gc[qx * n + i] * gg[qx][0];
          a2 += prm.Bc[qx * n + i] * gg[qx][1];
          a3 += prm.Bc[qx * n + i] * gg[qx][2];
        }
        W[L::Y1 + QQ * i] = a1;
        W[L::Y2 + QQ * i] = a2;
        W[L::Y3 + QQ * i] = a3;
      }
    }
    __syncwarp();
    if (bn < nb && lane == 0)
    {
      fence_proxy_async();
      issue_geom(bn);
    }

    // ---------------------------------------------------------------- phase Yt
    {
      constexpr int IT = NEW * n * q, ROUNDS = (IT + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool v = w < IT;
        const int wc = v ? w : 0, e = wc / (n * q), t = wc % (n * q), qz = t % q, i = t / q;
        const double *v1 = sW + e * ES + L::Y1 + q * t, *v2 = sW + e * ES + L::Y2 + q * t, *v3 = sW + e * ES + L::Y3 + q * t;
        double w1[q], w2[q], w3[q];
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          w1[qy] = v1[qy];
          w2[qy] = v2[qy];
          w3[qy] = v3[qy];
        }
        if (v)
        {
          double *za = sW + e * ES + L::ZA + qz + q * i, *zb = sW + e * ES + L::ZB + qz + q * i;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            double a = 0.0, bb = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              a += prm.Bc[qy * n + j] * w1[qy] + prm.Gc[qy * n + j] * w2[qy];
              bb += prm.Bc[qy * n + j] * w3[qy];
            }
            za[q * n * j] = a;
            zb[q * n * j] = bb;
          }
        }
      }
    }
    __syncwarp();

    // ---------------------------------------------------------------- phase Zt + scatter
    {
      constexpr int IT = NEW * n * n, ROUNDS = (IT + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const int wc = w < IT ? w : 0, e = wc / (n * n), t = wc % (n * n);
        const bool v = w < IT && e < nel;
        const double *pa = sW + e * ES + L::ZA + q * t, *pb = sW + e * ES + L::ZB + q * t;
        double a[q], bb[q];
        int32_t gk[n];
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          a[qz] = pa[qz];
          bb[qz] = pb[qz];
        }
#pragma unroll
        for (int k = 0; k < n; k++) gk[k] = cI[e * PS + t + n * n * k];
        if (v)
        {
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            double o = 0.0;
#pragma unroll
            for (int qz = 0; qz < q; qz++) o += prm.Bc[qz * n + k] * a[qz] + prm.Gc[qz * n + k] * bb[qz];
            if (SPLIT)
              scatter_fast_split(prm.y, prm.sp, gk[k], o);
            else
              scatter_fast(prm.y, gk[k], o);
          }
        }
      }
    }
    __syncwarp();
    if (b + 3 * GW < nb && lane == 0)
    {
      fence_proxy_async();
      issue_idx(b + 3 * GW, slot);
    }
    slot = nslot;
  }
}

template <int P_, int Q_, bool ASM>
int launch_h1v3(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  using L = H1V3Layout<P_, Q_, ASM>;
  constexpr int SMEM_SM = 222 * 1024;
  constexpr int WPS0 = (SMEM_SM / L::WS) < 1 ? 1 : SMEM_SM / L::WS;
  constexpr int WPS = WPS0 > 12 ? 12 : WPS0;
  constexpr int MINB = (WPS >= 12) ? 3 : (WPS >= 8) ? 2 : 1;
  constexpr int NW = (WPS / MINB) < 1 ? 1 : WPS / MINB;
  const size_t shmem = (size_t)NW * L::WS;
  const bool split = range_split(op, rg);
  auto kern = split ? h1_hex_apply3_kernel<P_, Q_, ASM, true, NW, MINB> : h1_hex_apply3_kernel<P_, Q_, ASM, false, NW, MINB>;
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  H1V3Params<P_, Q_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.aq = op->aq ? op->aq + (size_t)e_off * op->aq_estride : nullptr;
  prm.ecoef = op->ecoef ? op->ecoef + 18 * (size_t)e_off : nullptr;
  prm.x = x;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  set_split(prm, op, rg);
  copy_tables(op->h_tab.data(), P_, Q_, Q_, nullptr, prm.Bc, prm.Gc);
  const int nb = (e_cnt + L::NEW - 1) / L::NEW;
  return launch_persistent(kern, prm, NW * 32, shmem, s, false, op->ctx, "h1_hex_apply3_kernel", false, false, op->ctx->sm_count * MINB, NW,
                           L::NEW, nb);
}

}  // namespace

int launch_h1_hex_apply3(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg,
                         cudaStream_t s)
{
#define B2P_CASE(PP, QQ)            \
  if (op->p == PP && op->q1d == QQ) \
    return op->assembled ? launch_h1v3<PP, QQ, true>(op, lidx, alpha, x, y, rg, s) : launch_h1v3<PP, QQ, false>(op, lidx, alpha, x, y, rg, s);
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

}  // namespace b2p
