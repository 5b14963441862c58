// Production Nedelec hexahedron apply kernel: warp-autonomous persistent pipeline.
//
//   y_L += alpha * sum_e E_e^T  B^T  D  B  E_e x_L          (curl-curl, mass, curl-curl + mass)
//
// Same operator as b2p_hex_nd.cu (the simple cross-check kernel), organised as:
//   * persistent grid; every WARP owns a batch of NEW elements through all five phases, so the only
//     synchronisation is __syncwarp() (no CTA barriers, warps drift apart and fill each other's stalls):
//       Z   z-contraction of the gathered dofs          (reads the staged x values)
//       Y   y-contraction
//       XDX x-contraction INTO REGISTERS -> u, curl u on one (qy,qz) line of q-points, pointwise D,
//           transposed x-contraction from registers
//       Yt  transposed y-contraction
//       Zt  transposed z-contraction, scatter-add (RED.F64) straight from registers
//   * a three-deep software pipeline per warp hides HBM/L2 latency behind the arithmetic:
//       - the batch's signed restriction indices arrive by TMA bulk copy (cp.async.bulk, UBLKCP) two
//         batches ahead, behind an mbarrier
//       - the x values are gathered one batch ahead with cp.async (LDGSTS) straight into shared memory
//       - the batch's geometry q-data (one contiguous block in HBM) arrives by TMA bulk copy into a
//         single buffer that is refilled as soon as the XDX phase of the previous batch has read it
//   * q-data is stored x-SLOWEST so the XDX phase reads it conflict-free; the shared work arrays are stored
//     as ROWS over the index the NEXT phase contracts (Z region: rows j, Y region: rows qy) with the
//     consumer's item index contiguous inside a row and the row stride padded (b2p_nd4_pads.inc, found by
//     tools/smem_sim.py) so that both the producer's and the consumer's 64-bit accesses are bank-conflict
//     free: the shared-memory data pipe, not HBM, was the top-utilised unit of the previous layout
//   * the 1-D basis tables travel in the kernel parameter block: every basis entry is a constant-bank
//     operand of the DFMA (no shared/global load per multiply).
//
// Reference semantics: ceed::Operator::AddMult over CeedOperatorApplyAdd
// (/root/reference/palace/fem/libceed/operator.cpp:148-178,192-212); D from
// /root/reference/palace/fem/qfunctions/33/{hdiv,hcurl,hdivmass}_33_qf.h.
#include <cstdlib>
#include <type_traits>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

template <int P_, int Q_>
struct ND4Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction, rows padded to 16 bytes (B2P_SKIP_IDX = masked/pad)
  const double *qd;     // [ne][10][Q] geometry, x-slowest point order
  const double *aq;     // [ne][ncomp][Q] assembled D, x-slowest (or null)
  const double *mat;    // [n_mat][9]
  const int32_t *emat;  // [ne][2]
  const double *ecoef;  // [ne][18] per-element coefficient matrices (value part, derivative part)
  const double *x;
  double *y;
  double alpha;
  int ne;
  VSplit sp;
  const unsigned long long *wait_flags, *wait_expect;  // peer-memory halo flags (SPLIT kernels only)
  int wait_n, wait_from_elem;
  int iso;  // all coefficient matrices are multiples of the identity
  double Bo[Q_ * P_];
  double Bc[Q_ * (P_ + 1)];
  double Gc[Q_ * (P_ + 1)];
};

// Fused complex apply (CPLX kernels): y_r + i y_i += alpha * E^T B^T (D_r + i D_i) B E (x_r + i x_i) in ONE pass
// over the geometry. The two parts of a vector ride in adjacent element slots of a warp, so restriction indices,
// q-data and coefficient block are fetched once for both. zcoef[ne][36] holds the per-element complex coefficient
// tensors {mass Re, mass Im, curl Re, curl Im} (column-major 3x3 each): the sum over the terms of a complex
// operator of (c_r + i c_i) * material tensor, so K, M and every mass-type loss term of
// /root/reference/palace/linalg/operator.cpp:98-134 (ComplexWrapperOperator: four real applies per term)
// cost one kernel launch and one geometry stream.
template <int P_, int Q_>
struct ND4ParamsZ : ND4Params<P_, Q_>
{
  const double *xi;     // imaginary part of the input
  double *yi;           // imaginary part of the output
  const double *zcoef;  // [ne][36]
  int has_imag;         // some coefficient has an imaginary part (otherwise the parts never mix)
};

struct Nd4Pad
{
  int p, q, kind, a, b, y;
};
constexpr Nd4Pad nd4_pad_table[] = {
#include "b2p_nd4_pads.inc"
};
constexpr Nd4Pad nd4_pads(int p, int q, int kind)
{
  for (const Nd4Pad &e : nd4_pad_table)
    if (e.p == p && e.q == q && e.kind == kind) return e;
  return Nd4Pad{p, q, kind, 1, 1, 4};
}
constexpr int nd4_pow2ceil(int x)
{
  int r = 1;
  while (r < x) r *= 2;
  return r;
}
// Lanes per element in the Z / Zt phases: padded to a power of two when that costs no extra round, so an
// element's items do not straddle a half-warp (the 64-bit shared-memory access granule).
constexpr int nd4_lane_stride(int items, int nel)
{
  const int pc = nd4_pow2ceil(items), rounds = (nel * items + 31) / 32;
  return (nel * pc <= 32 * rounds) ? pc : items;
}

template <int P_, int Q_, int KIND, bool ASM, bool CPLX = false>
struct ND4Layout
{
  static constexpr int p = P_, q = Q_, n = P_ + 1, Q = q * q * q, P = 3 * p * n * n, D3 = p * n * n;
  static constexpr int PS = (P + 3) & ~3;  // padded restriction stride (16-byte rows for TMA)
  static constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS);
  static constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS);
  // elements per warp: enough (qy,qz) lines to fill the 32 lanes in the XDX phase
  static constexpr int NEW0 = (q * q >= 32) ? 1 : 32 / (q * q);
  // CPLX: the slots of a warp are (element, part) pairs, parts adjacent -> an even number of slots
  static constexpr int NPART = CPLX ? 2 : 1, NEW = CPLX ? (NEW0 & ~1) : NEW0, NEB = NEW / NPART;
  static constexpr Nd4Pad PAD = nd4_pads(P_, Q_, KIND);
  // items of one element inside a row, in the consumer's order t = qz + q*i
  static constexpr int NXA = p * q, NNA = n * q;
  // Z region, group A: rows j < n (closed direction contracted next): [XA][XB][ZA], each [NEW][t]
  static constexpr int A_XA = 0, A_XB = A_XA + NEW * NXA, A_ZA = A_XB + (CURL ? NEW * NXA : 0), LA = A_ZA + NEW * NNA,
                       RSA = LA + PAD.a;
  // Z region, group B: rows j < p (open direction contracted next): [YA][YB]
  static constexpr int B_YA = 0, B_YB = B_YA + NEW * NNA, LB = B_YB + (CURL ? NEW * NNA : 0), RSB = LB + PAD.b;
  static constexpr int ZA0 = 0, ZB0 = ZA0 + n * RSA, ZSZ = ZB0 + p * RSB;
  // Y region: rows qy < q: [X1][X2][X3][Y1][Y2][Z1][Z3], each [NEW][t]
  static constexpr int Y_X1 = 0, Y_X2 = Y_X1 + (MASS ? NEW * NXA : 0), Y_X3 = Y_X2 + (CURL ? NEW * NXA : 0),
                       Y_Y1 = Y_X3 + (CURL ? NEW * NXA : 0), Y_Y2 = Y_Y1 + NEW * NNA, Y_Z1 = Y_Y2 + (CURL ? NEW * NNA : 0),
                       Y_Z3 = Y_Z1 + NEW * NNA, LY = Y_Z3 + (CURL ? NEW * NNA : 0), RSY = LY + PAD.y;
  static constexpr int Y0 = ZSZ, WTOT = (Y0 + q * RSY + 1) & ~1;  // doubles of work space per warp (even)
  static constexpr int LSX = nd4_lane_stride(p * n, NEW), LSZ = nd4_lane_stride(n * n, NEW);
  static constexpr int GCOMP = ASM ? ((MASS ? 9 : 0) + (CURL ? 9 : 0)) : 10;
  static constexpr int GE = (GCOMP * Q + 1) & ~1;  // doubles of q-data per element (even: 16-byte blocks for TMA)
  static constexpr int CE = CPLX ? 36 : 18;        // coefficient matrices per element
  // per-warp shared memory (bytes), every block 16-byte aligned
  static constexpr int OFF_G = 0;
  static constexpr int OFF_W = OFF_G + NEB * GE * 8;
  static constexpr int OFF_U = OFF_W + WTOT * 8;                 // [NEW*PS] doubles: staged x values
  static constexpr int OFF_I = OFF_U + NEW * PS * 8;             // [3][NEB*PS] int32: restriction index ring
  static constexpr int OFF_C = OFF_I + 3 * NEB * PS * 4;         // [NEB*CE] doubles
  static constexpr int OFF_B = OFF_C + ((NEB * CE * 8 + 15) & ~15);  // 4 mbarriers
  static constexpr int WS = (OFF_B + 4 * 8 + 15) & ~15;
};

template <int P_, int Q_, bool CPLX>
using ND4ParamsT = std::conditional_t<CPLX, ND4ParamsZ<P_, Q_>, ND4Params<P_, Q_>>;

// FWD (experimental, B2P_ND_FWDCHAIN=1): the XDX phase consumes the Z region directly -- every lane does the y-contraction
// of its own (qy, qz) line from broadcast reads -- so the forward Y-region round trip (write + read of 7 arrays) and
// the Y phase disappear; same arithmetic, ~14 % fewer shared-memory wavefronts per element.
template <int P_, int Q_, int KIND, bool ASM, bool SPLIT, int NW, int MINB, bool CPLX = false, bool FWD = false>
__global__ void __launch_bounds__(NW * 32, MINB) nd_hex_apply4_kernel(const __grid_constant__ ND4ParamsT<P_, Q_, CPLX> prm)
{
  using L = ND4Layout<P_, Q_, KIND, ASM, CPLX>;
  static_assert(!CPLX || (!SPLIT && !ASM && L::NEW >= 2), "fused complex apply: single partition, on-the-fly D, two slots per warp");
  constexpr int p = L::p, q = L::q, n = L::n, Q = L::Q, D3 = L::D3, GE = L::GE, PS = L::PS, NEW = L::NEW;
  constexpr int NPART = L::NPART, NEB = L::NEB, CE = L::CE;  // slot e = (element e / NPART, part e % NPART)
  constexpr int RSA = L::RSA, RSB = L::RSB, RSY = L::RSY, NXA = L::NXA, NNA = L::NNA;
  constexpr bool MASS = L::MASS, CURL = L::CURL;
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
  uint64_t *bar_i = bar_g + 1;  // [3]

  const int nb = (prm.ne + NEB - 1) / NEB;  // element batches
  const int GW = gridDim.x * NW;            // warps in the grid
  int b = blockIdx.x * NW + wid;
  griddep_launch_dependents();              // a dependent launched programmatically (the halo POST kernel) may be scheduled as CTAs retire
  if (b >= nb) return;                      // (whole warp)

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
    const int e0 = bb * NEB, nel = min(NEB, prm.ne - e0);
    const uint32_t bytes = (uint32_t)(nel * PS * sizeof(int32_t));
    mbar_expect_tx(bar_i + slot, bytes);
    tma_bulk_g2s(sI + slot * NEB * PS, prm.lidx + (size_t)e0 * PS, bytes, bar_i + slot);
  };
  auto issue_geom = [&](int bb)
  {
    const int e0 = bb * NEB, nel = min(NEB, prm.ne - e0);
    const uint32_t bytes = (uint32_t)(nel * GE * sizeof(double));
    const uint32_t cbytes = ASM ? 0u : (uint32_t)(nel * CE * sizeof(double));
    mbar_expect_tx(bar_g, bytes + cbytes);
    tma_bulk_g2s(sG, (ASM ? prm.aq : prm.qd) + (size_t)e0 * GE, bytes, bar_g);
    if constexpr (CPLX)
      tma_bulk_g2s(sC, prm.zcoef + (size_t)e0 * CE, cbytes, bar_g);
    else if (!ASM)
      tma_bulk_g2s(sC, prm.ecoef + (size_t)e0 * 18, cbytes, bar_g);
  };
  // x values of batch bb -> sU (raw; the sign is applied when they are read)
  auto gather_x = [&](int bb, int slot)
  {
    const int e0 = bb * NEB, nel = NPART * min(NEB, prm.ne - e0);
    const int32_t *gI = sI + slot * NEB * PS;
    constexpr int ITER = (NEW * PS + 31) / 32;
#pragma unroll
    for (int r = 0; r < ITER; r++)
    {
      const int l = lane + 32 * r;
      if (l < nel * PS)
      {
        if constexpr (CPLX)
        {
          // slot (element, part): both parts read through the element's one index row
          const int e = l / PS, t = l % PS;
          const int32_t gi = gI[(e / NPART) * PS + t];
          if (gi == B2P_SKIP_IDX)
            sU[l] = 0.0;
          else
            cp_async8(sU + l, ((e % NPART) ? prm.xi : prm.x) + (uint32_t)abs_idx(gi));
        }
        else
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
    }
    cp_async_commit();
  };

  // Peer-memory halo: ghost values of this step are complete once every neighbour's flag reached the expected epoch.
  bool y_ready = false;  // the grid dependency (zero-fill of y / the halo PRE kernel under programmatic dependent launch) is resolved
  bool ghosts_ready = !(SPLIT && prm.wait_n > 0);
  auto wait_ghosts = [&](int bb)
  {
    if (ghosts_ready || (bb + 1) * NEB <= prm.wait_from_elem) return;
    if (!y_ready)
    {
      griddep_wait();  // the expected epochs are advanced by the PRE kernel this grid may be overlapping
      y_ready = true;
    }
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

  // mbarrier phase parities: bit s of par_i for index slot s
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
  gather_x(b, 0);

  const double alpha = prm.alpha;
  int slot = 0;
  for (; b < nb; b += GW)
  {
    const int nslot = (slot == 2) ? 0 : slot + 1;
    const int bn = b + GW;
    const int e0 = b * NEB, nel = NPART * min(NEB, prm.ne - e0);  // nel: valid slots of this batch
    const int32_t *cI = sI + slot * NEB * PS;
    const double *cU = sU;
    (void)e0;

    cp_async_wait<0>();
    __syncwarp();

    // ------------------------------------------------------------------ phase Z (z-contraction)
    // All loads of a round are issued before any arithmetic or store (shared-memory stores would
    // otherwise fence the next component's loads): x-, y- and z-directed items of lane `w`.
    // Output rows: the index the Y phase contracts (j); inside a row the Y phase's item t = qz + q*i.
    {
      constexpr int IPX = p * n, IPZ = n * n, LSX = L::LSX, LSZ = L::LSZ;
      constexpr int LW = (NEW * LSX > NEW * LSZ) ? NEW * LSX : NEW * LSZ;
      constexpr int ROUNDS = (LW + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool vx = (w / LSX) < NEW && (w % LSX) < IPX, vz = (w / LSZ) < NEW && (w % LSZ) < IPZ;
        const int ex = vx ? w / LSX : 0, tx = vx ? w % LSX : 0;
        const int ez = vz ? w / LSZ : 0, tz = vz ? w % LSZ : 0;
        double ux[n], uy[n], uz[p];
#pragma unroll
        for (int k = 0; k < n; k++)
        {
          ux[k] = staged2(cI, (ex / NPART) * PS + tx + p * n * k, cU, ex * PS + tx + p * n * k, ex < nel);
          uy[k] = staged2(cI, (ex / NPART) * PS + D3 + tx + n * p * k, cU, ex * PS + D3 + tx + n * p * k, ex < nel);
        }
#pragma unroll
        for (int k = 0; k < p; k++)
          uz[k] = staged2(cI, (ez / NPART) * PS + 2 * D3 + tz + n * n * k, cU, ez * PS + 2 * D3 + tz + n * n * k, ez < nel);
        if (vx)
        {
          // x-directed dof tx = i + p*j ; y-directed dof tx = i + n*j
          double *xa = sW + L::ZA0 + (tx / p) * RSA + L::A_XA + ex * NXA + q * (tx % p), *xb = xa + (L::A_XB - L::A_XA);
          double *ya = sW + L::ZB0 + (tx / n) * RSB + L::B_YA + ex * NNA + q * (tx % n), *yb = ya + (L::B_YB - L::B_YA);
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            double a = 0.0, b = 0.0, c = 0.0, d = 0.0;
#pragma unroll
            for (int k = 0; k < n; k++)
            {
              a += prm.Bc[qz * n + k] * ux[k];
              c += prm.Bc[qz * n + k] * uy[k];
              if (CURL) b += prm.Gc[qz * n + k] * ux[k];
              if (CURL) d += prm.Gc[qz * n + k] * uy[k];
            }
            xa[qz] = a;
            ya[qz] = c;
            if (CURL) xb[qz] = b;
            if (CURL) yb[qz] = d;
          }
        }
        if (vz)
        {
          double *za = sW + L::ZA0 + (tz / n) * RSA + L::A_ZA + ez * NNA + q * (tz % n);
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            double a = 0.0;
#pragma unroll
            for (int k = 0; k < p; k++) a += prm.Bo[qz * p + k] * uz[k];
            za[qz] = a;
          }
        }
      }
    }
    __syncwarp();
    // the staged x values are consumed: gather the next batch's while this one computes
    if (bn < nb)
    {
      mbar_wait(bar_i + nslot, (par_i >> nslot) & 1u);
      par_i ^= (1u << nslot);
      wait_ghosts(bn);
      gather_x(bn, nslot);
    }

    // ------------------------------------------------------------------ phase Y (y-contraction)
    // item w = (e, t = qz + q*i): reads row j of the Z region at column w, writes row qy of the Y region at column w
    if constexpr (!FWD)
    {
      constexpr int IX = NEW * p * q, IN = NEW * n * q;  // x-directed items; y- and z-directed items
      constexpr int ROUNDS = (IN + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool vx = w < IX, vn = w < IN;
        const int wx = vx ? w : 0, wn = vn ? w : 0;
        double xa[n], xb[n], ya[p], yb[p], za[n];
        {
          const double *pa = sW + L::ZA0 + L::A_XA + wx, *pb = sW + L::ZA0 + L::A_XB + wx;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            xa[j] = pa[RSA * j];
            if (CURL) xb[j] = pb[RSA * j];
          }
          const double *qa = sW + L::ZB0 + L::B_YA + wn, *qb = sW + L::ZB0 + L::B_YB + wn;
#pragma unroll
          for (int j = 0; j < p; j++)
          {
            ya[j] = qa[RSB * j];
            if (CURL) yb[j] = qb[RSB * j];
          }
          const double *ra = sW + L::ZA0 + L::A_ZA + wn;
#pragma unroll
          for (int j = 0; j < n; j++) za[j] = ra[RSA * j];
        }
        if (vx)
        {
          // x-directed (j<n closed): V1 = Bc_y a, V3 = Gc_y a, V2 = Bc_y b
          double *v1 = sW + L::Y0 + L::Y_X1 + wx, *v2 = sW + L::Y0 + L::Y_X2 + wx, *v3 = sW + L::Y0 + L::Y_X3 + wx;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            double s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              if (MASS) s1 += prm.Bc[qy * n + j] * xa[j];
              if (CURL) s2 += prm.Bc[qy * n + j] * xb[j];
              if (CURL) s3 += prm.Gc[qy * n + j] * xa[j];
            }
            if (MASS) v1[RSY * qy] = s1;
            if (CURL) v2[RSY * qy] = s2;
            if (CURL) v3[RSY * qy] = s3;
          }
        }
        if (vn)
        {
          // y-directed (j<p open): V1 = Bo_y a, V2 = Bo_y b ; z-directed (j<n closed): V1 = Bc_y a, V3 = Gc_y a
          double *v1 = sW + L::Y0 + L::Y_Y1 + wn, *v2 = sW + L::Y0 + L::Y_Y2 + wn;
          double *z1 = sW + L::Y0 + L::Y_Z1 + wn, *z3 = sW + L::Y0 + L::Y_Z3 + wn;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            double s1 = 0.0, s2 = 0.0, t1 = 0.0, t3 = 0.0;
#pragma unroll
            for (int j = 0; j < p; j++)
            {
              s1 += prm.Bo[qy * p + j] * ya[j];
              if (CURL) s2 += prm.Bo[qy * p + j] * yb[j];
            }
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              t1 += prm.Bc[qy * n + j] * za[j];
              if (CURL) t3 += prm.Gc[qy * n + j] * za[j];
            }
            v1[RSY * qy] = s1;
            if (CURL) v2[RSY * qy] = s2;
            z1[RSY * qy] = t1;
            if (CURL) z3[RSY * qy] = t3;
          }
        }
      }
    }
    __syncwarp();
    mbar_wait(bar_g, par_g);  // q-data of this batch has landed
    par_g ^= 1;

    // ------------------------------------------------------------------ phase XDX
    // item s = qy + q*qz: reads V[s + q^2 i]; all qx of this line live in registers.
    // Three sub-steps keep the live register set small: (1) x-contraction of the 7 staged arrays
    // into u, curl u for all qx; (2) pointwise D in place; (3) transposed x-contraction, each
    // output formed from the q values and stored at once.
    for (int w = lane; w < NEW * (QQ); w += 32)
    {
      const int e = w / QQ, s = w % QQ;
      // row qy of the Y region; column (e, t = qz + q*i)
      double *WX = sW + L::Y0 + (s % q) * RSY + e * NXA + s / q;
      double *WN = sW + L::Y0 + (s % q) * RSY + e * NNA + s / q;
      double uu[q][3], cc[q][3];
      {
        double x1[p], x2[p], x3[p], y1[n], y2[n], z1[n], z3[n];
        if constexpr (FWD)
        {
          // y-contraction of this lane's own (qy, qz) line straight from the Z region: the four qy-lanes of a (e, qz)
          // read the same words (broadcast), the table rows of qy are indexed loads from the constant bank
          const int qy = s % q, qz = s / q;
          const double *bo = prm.Bo + qy * p, *bc = prm.Bc + qy * n, *gc = prm.Gc + qy * n;
          const double *ZX = sW + L::ZA0 + e * NXA + qz, *ZY = sW + L::ZB0 + e * NNA + qz, *ZZ = sW + L::ZA0 + L::A_ZA + e * NNA + qz;
#pragma unroll
          for (int i = 0; i < p; i++)
          {
            double s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              const double a = ZX[L::A_XA + RSA * j + q * i];
              if (MASS) s1 += bc[j] * a;
              if (CURL) s3 += gc[j] * a;
              if (CURL) s2 += bc[j] * ZX[L::A_XB + RSA * j + q * i];
            }
            x1[i] = s1;
            x2[i] = s2;
            x3[i] = s3;
          }
#pragma unroll
          for (int i = 0; i < n; i++)
          {
            double s1 = 0.0, s2 = 0.0, t1 = 0.0, t3 = 0.0;
#pragma unroll
            for (int j = 0; j < p; j++)
            {
              s1 += bo[j] * ZY[L::B_YA + RSB * j + q * i];
              if (CURL) s2 += bo[j] * ZY[L::B_YB + RSB * j + q * i];
            }
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              const double a = ZZ[RSA * j + q * i];
              t1 += bc[j] * a;
              if (CURL) t3 += gc[j] * a;
            }
            y1[i] = s1;
            y2[i] = s2;
            z1[i] = t1;
            z3[i] = t3;
          }
        }
        else
        {
#pragma unroll
        for (int i = 0; i < p; i++)
        {
          if (MASS) x1[i] = WX[L::Y_X1 + q * i];
          if (CURL) x2[i] = WX[L::Y_X2 + q * i];
          if (CURL) x3[i] = WX[L::Y_X3 + q * i];
        }
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          y1[i] = WN[L::Y_Y1 + q * i];
          if (CURL) y2[i] = WN[L::Y_Y2 + q * i];
          z1[i] = WN[L::Y_Z1 + q * i];
          if (CURL) z3[i] = WN[L::Y_Z3 + q * i];
        }
        }
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          double u0 = 0, u1 = 0, u2 = 0, dzux = 0, dyux = 0, dzuy = 0, dxuy = 0, dyuz = 0, dxuz = 0;
#pragma unroll
          for (int i = 0; i < p; i++)
          {
            if (MASS) u0 += prm.Bo[qx * p + i] * x1[i];
            if (CURL) dzux += prm.Bo[qx * p + i] * x2[i];
            if (CURL) dyux += prm.Bo[qx * p + i] * x3[i];
          }
#pragma unroll
          for (int i = 0; i < n; i++)
          {
            if (MASS) u1 += prm.Bc[qx * n + i] * y1[i];
            if (CURL) dzuy += prm.Bc[qx * n + i] * y2[i];
            if (CURL) dxuy += prm.Gc[qx * n + i] * y1[i];
            if (MASS) u2 += prm.Bc[qx * n + i] * z1[i];
            if (CURL) dyuz += prm.Bc[qx * n + i] * z3[i];
            if (CURL) dxuz += prm.Gc[qx * n + i] * z1[i];
          }
          uu[qx][0] = u0;
          uu[qx][1] = u1;
          uu[qx][2] = u2;
          cc[qx][0] = dyuz - dzuy;
          cc[qx][1] = dzux - dxuz;
          cc[qx][2] = dxuy - dyux;
        }
      }
      const double *g = sG + (e / NPART) * GE + s;
      const double *C = sC + (e / NPART) * CE;
#pragma unroll
      for (int qx = 0; qx < q; qx++)
      {
        double v[3] = {0, 0, 0}, cw[3] = {0, 0, 0};
        if constexpr (CPLX)
        {
          // z = (C_r + i C_i)(t_r + i t_i) with t = J^-T u (mass) or (J/detJ) curl u (curl): this slot owns one part
          // of t; the partner slot (other part, same element, same point) sends its C_i t and gets ours.
          const double *gq = g + QQ * qx;
          const bool ok = e < nel;
          double A[9], Jd[9], t[3], am[3] = {0, 0, 0}, bm[3] = {0, 0, 0}, ac[3] = {0, 0, 0}, bc[3] = {0, 0, 0};
          const double wdetJ = ok ? alpha * gq[0] : 0.0;
#pragma unroll
          for (int i = 0; i < 9; i++) A[i] = ok ? gq[(1 + i) * Q] : 0.0;
          if (MASS)
          {
            Ax33(A, uu[qx], t);
            Ax33(C, t, am);
            Ax33(C + 9, t, bm);
          }
          if (CURL)
          {
            cofactor33(A, Jd);
            Ax33(Jd, cc[qx], t);
            Ax33(C + 18, t, ac);
            Ax33(C + 27, t, bc);
          }
          if (prm.has_imag)
          {
            constexpr unsigned xmask = (NEW * QQ >= 32) ? 0xffffffffu : ((1u << (NEW * QQ)) - 1u);
            const int partner = (e ^ 1) * QQ + s;
            const double sg = (e & 1) ? 1.0 : -1.0;  // real part: a_r - b_i ; imaginary part: a_i + b_r
#pragma unroll
            for (int r = 0; r < 3; r++)
            {
              if (MASS) am[r] += sg * __shfl_sync(xmask, bm[r], partner);
              if (CURL) ac[r] += sg * __shfl_sync(xmask, bc[r], partner);
            }
          }
          if (MASS) Atx33(A, am, wdetJ, v);
          if (CURL) Atx33(Jd, ac, wdetJ, cw);
        }
        else if (e < nel)
        {
          const double *gq = g + QQ * qx;
          if (ASM)
          {
            const double *a = gq;
            if (MASS)
            {
#pragma unroll
              for (int r = 0; r < 3; r++) v[r] = alpha * (a[(r)*Q] * uu[qx][0] + a[(r + 3) * Q] * uu[qx][1] + a[(r + 6) * Q] * uu[qx][2]);
              a += 9 * Q;
            }
            if (CURL)
            {
#pragma unroll
              for (int r = 0; r < 3; r++) cw[r] = alpha * (a[(r)*Q] * cc[qx][0] + a[(r + 3) * Q] * cc[qx][1] + a[(r + 6) * Q] * cc[qx][2]);
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
              // every material is a multiple of the identity (the common isotropic case): C = c I
              if (MASS) AtAx(A, uu[qx], wdetJ * C[0], v);
              if (CURL)
              {
                double Jd[9];
                cofactor33(A, Jd);
                AtAx(Jd, cc[qx], wdetJ * C[9], cw);
              }
            }
            else
            {
              if (MASS) AtCAx(A, C, uu[qx], wdetJ, v);
              if (CURL)
              {
                double Jd[9];
                cofactor33(A, Jd);
                AtCAx(Jd, C + 9, cc[qx], wdetJ, cw);
              }
            }
          }
        }
#pragma unroll
        for (int r = 0; r < 3; r++)
        {
          uu[qx][r] = v[r];
          cc[qx][r] = cw[r];
        }
      }
      // transposed x-contraction: outputs formed one at a time
#pragma unroll
      for (int i = 0; i < p; i++)
      {
        double a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) a1 += prm.Bo[qx * p + i] * uu[qx][0];
          if (CURL) a2 += prm.Bo[qx * p + i] * cc[qx][1];
          if (CURL) a3 -= prm.Bo[qx * p + i] * cc[qx][2];
        }
        if (MASS) WX[L::Y_X1 + q * i] = a1;
        if (CURL) WX[L::Y_X2 + q * i] = a2;
        if (CURL) WX[L::Y_X3 + q * i] = a3;
      }
#pragma unroll
      for (int i = 0; i < n; i++)
      {
        double b1 = 0, b2 = 0, c1 = 0, c3 = 0;
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) b1 += prm.Bc[qx * n + i] * uu[qx][1];
          if (CURL) b1 += prm.Gc[qx * n + i] * cc[qx][2];
          if (CURL) b2 -= prm.Bc[qx * n + i] * cc[qx][0];
          if (MASS) c1 += prm.Bc[qx * n + i] * uu[qx][2];
          if (CURL) c1 -= prm.Gc[qx * n + i] * cc[qx][1];
          if (CURL) c3 += prm.Bc[qx * n + i] * cc[qx][0];
        }
        WN[L::Y_Y1 + q * i] = b1;
        if (CURL) WN[L::Y_Y2 + q * i] = b2;
        WN[L::Y_Z1 + q * i] = c1;
        if (CURL) WN[L::Y_Z3 + q * i] = c3;
      }
    }
    __syncwarp();
    if (bn < nb && lane == 0)
    {
      fence_proxy_async();
      issue_geom(bn);  // refill the single q-data buffer for the next batch
    }

    // ------------------------------------------------------------------ phase Yt (transposed y-contraction)
    {
      constexpr int IX = NEW * p * q, IN = NEW * n * q;
      constexpr int ROUNDS = (IN + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool vx = w < IX, vn = w < IN;
        const int wx = vx ? w : 0, wn = vn ? w : 0;
        double x1[q], x2[q], x3[q], y1[q], y2[q], z1[q], z3[q];
        {
          const double *v1 = sW + L::Y0 + L::Y_X1 + wx, *v2 = sW + L::Y0 + L::Y_X2 + wx, *v3 = sW + L::Y0 + L::Y_X3 + wx;
          const double *u1 = sW + L::Y0 + L::Y_Y1 + wn, *u2 = sW + L::Y0 + L::Y_Y2 + wn;
          const double *t1 = sW + L::Y0 + L::Y_Z1 + wn, *t3 = sW + L::Y0 + L::Y_Z3 + wn;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            if (MASS) x1[qy] = v1[RSY * qy];
            if (CURL) x2[qy] = v2[RSY * qy];
            if (CURL) x3[qy] = v3[RSY * qy];
            y1[qy] = u1[RSY * qy];
            if (CURL) y2[qy] = u2[RSY * qy];
            z1[qy] = t1[RSY * qy];
            if (CURL) z3[qy] = t3[RSY * qy];
          }
        }
        if (vx)
        {
          // x-directed: Za'[j] = sum_qy Bc[qy][j] W1 + Gc[qy][j] W3 ; Zb'[j] = sum_qy Bc[qy][j] W2
          double *za = sW + L::ZA0 + L::A_XA + wx, *zb = sW + L::ZA0 + L::A_XB + wx;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            double a = 0.0, b = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              if (MASS) a += prm.Bc[qy * n + j] * x1[qy];
              if (CURL) a += prm.Gc[qy * n + j] * x3[qy];
              if (CURL) b += prm.Bc[qy * n + j] * x2[qy];
            }
            za[RSA * j] = a;
            if (CURL) zb[RSA * j] = b;
          }
        }
        if (vn)
        {
          // y-directed: Za'[j<p] = sum_qy Bo[qy][j] W1 ; Zb' = sum_qy Bo[qy][j] W2
          double *ya = sW + L::ZB0 + L::B_YA + wn, *yb = sW + L::ZB0 + L::B_YB + wn;
#pragma unroll
          for (int j = 0; j < p; j++)
          {
            double a = 0.0, b = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              a += prm.Bo[qy * p + j] * y1[qy];
              if (CURL) b += prm.Bo[qy * p + j] * y2[qy];
            }
            ya[RSB * j] = a;
            if (CURL) yb[RSB * j] = b;
          }
          // z-directed: Za'[j] = sum_qy Bc[qy][j] W1 + Gc[qy][j] W3
          double *za = sW + L::ZA0 + L::A_ZA + wn;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            double a = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              a += prm.Bc[qy * n + j] * z1[qy];
              if (CURL) a += prm.Gc[qy * n + j] * z3[qy];
            }
            za[RSA * j] = a;
          }
        }
      }
    }
    __syncwarp();

    // ------------------------------------------------------------------ phase Zt (transposed z-contraction + scatter)
    // First write to y: under programmatic dependent launch the zero-fill of y that precedes this kernel in the stream
    // may still be running -- everything above (index / geometry / x traffic and the arithmetic of the first batch) has
    // overlapped with it.
    if (!y_ready)
    {
      griddep_wait();
      y_ready = true;
    }
    {
      constexpr int IPX = p * n, IPZ = n * n, LSX = L::LSX, LSZ = L::LSZ;
      constexpr int LW = (NEW * LSX > NEW * LSZ) ? NEW * LSX : NEW * LSZ;
      constexpr int ROUNDS = (LW + 31) / 32;
#pragma unroll
      for (int r = 0; r < ROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool ix_ok = (w / LSX) < NEW && (w % LSX) < IPX, iz_ok = (w / LSZ) < NEW && (w % LSZ) < IPZ;
        const int ex = ix_ok ? w / LSX : 0, tx = ix_ok ? w % LSX : 0;
        const int ez = iz_ok ? w / LSZ : 0, tz = iz_ok ? w % LSZ : 0;
        const bool vx = ix_ok && ex < nel, vz = iz_ok && ez < nel;
        double xa[q], xb[q], ya[q], yb[q], za[q];
        int32_t gx[n], gy[n], gz[p];
        {
          const double *pxa = sW + L::ZA0 + (tx / p) * RSA + L::A_XA + ex * NXA + q * (tx % p), *pxb = pxa + (L::A_XB - L::A_XA);
          const double *pya = sW + L::ZB0 + (tx / n) * RSB + L::B_YA + ex * NNA + q * (tx % n), *pyb = pya + (L::B_YB - L::B_YA);
          const double *pza = sW + L::ZA0 + (tz / n) * RSA + L::A_ZA + ez * NNA + q * (tz % n);
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            xa[qz] = pxa[qz];
            ya[qz] = pya[qz];
            za[qz] = pza[qz];
            if (CURL) xb[qz] = pxb[qz];
            if (CURL) yb[qz] = pyb[qz];
          }
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            gx[k] = cI[(ex / NPART) * PS + tx + p * n * k];
            gy[k] = cI[(ex / NPART) * PS + D3 + tx + n * p * k];
          }
#pragma unroll
          for (int k = 0; k < p; k++) gz[k] = cI[(ez / NPART) * PS + 2 * D3 + tz + n * n * k];
        }
        // output vector of this lane's slots (the imaginary part for odd slots of a fused complex apply)
        double *yx = prm.y, *yz = prm.y;
        if constexpr (CPLX)
        {
          yx = (ex % NPART) ? prm.yi : prm.y;
          yz = (ez % NPART) ? prm.yi : prm.y;
        }
        if (vx)
        {
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            double o = 0.0, o2 = 0.0;
#pragma unroll
            for (int qz = 0; qz < q; qz++)
            {
              o += prm.Bc[qz * n + k] * xa[qz];
              o2 += prm.Bc[qz * n + k] * ya[qz];
              if (CURL) o += prm.Gc[qz * n + k] * xb[qz];
              if (CURL) o2 += prm.Gc[qz * n + k] * yb[qz];
            }
            if (SPLIT) scatter_fast_split(prm.y, prm.sp, gx[k], o); else scatter_fast(yx, gx[k], o);
            if (SPLIT) scatter_fast_split(prm.y, prm.sp, gy[k], o2); else scatter_fast(yx, gy[k], o2);
          }
        }
        if (vz)
        {
#pragma unroll
          for (int k = 0; k < p; k++)
          {
            double o = 0.0;
#pragma unroll
            for (int qz = 0; qz < q; qz++) o += prm.Bo[qz * p + k] * za[qz];
            if (SPLIT) scatter_fast_split(prm.y, prm.sp, gz[k], o); else scatter_fast(yz, gz[k], o);
          }
        }
      }
    }
    __syncwarp();
    if (b + 3 * GW < nb && lane == 0)
    {
      fence_proxy_async();
      issue_idx(b + 3 * GW, slot);  // this batch's index slot is free again
    }
    slot = nslot;
  }
}

template <int P_, int Q_, int KIND, bool ASM>
int launch4(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  using L = ND4Layout<P_, Q_, KIND, ASM>;
  // warps per CTA / CTAs per SM from the per-warp shared-memory footprint
  constexpr int SMEM_SM = 222 * 1024;
  constexpr int WPS0 = (SMEM_SM / L::WS) < 1 ? 1 : SMEM_SM / L::WS;  // warps per SM that fit in shared memory
  constexpr int WPS = WPS0 > 10 ? 10 : WPS0;  // register file: 10 warps at ~204 registers
  constexpr int MINB = (WPS >= 8) ? 2 : 1;
  constexpr int NW = (WPS / MINB) < 1 ? 1 : WPS / MINB;
  const size_t shmem = (size_t)NW * L::WS;
  // SPLIT: the L-vector comes in two pieces (owned part in x / y, ghosts in separate buffers)
  const bool split = range_split(op, rg);
  auto kern = split ? nd_hex_apply4_kernel<P_, Q_, KIND, ASM, true, NW, MINB> : nd_hex_apply4_kernel<P_, Q_, KIND, ASM, false, NW, MINB>;
  if constexpr (!ASM && Q_ == P_ + 1)
  {
    static const bool fwd = []() { const char *e = std::getenv("B2P_ND_FWDCHAIN"); return e && e[0] == '1'; }();
    if (fwd && !split) kern = nd_hex_apply4_kernel<P_, Q_, KIND, ASM, false, NW, MINB, false, true>;
  }
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  ND4Params<P_, Q_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.aq = op->aq ? op->aq + (size_t)e_off * op->aq_estride : nullptr;
  prm.mat = op->mat;
  prm.emat = op->emat + 2 * (size_t)e_off;
  prm.ecoef = op->ecoef ? op->ecoef + 18 * (size_t)e_off : nullptr;
  prm.x = x;
  prm.y = y;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  set_split_wait(prm, op, rg);
  prm.iso = op->iso ? 1 : 0;
  copy_tables(op->h_tab.data(), P_, Q_, Q_, prm.Bo, prm.Bc, prm.Gc);
  const int nb = (e_cnt + L::NEW - 1) / L::NEW;
  return launch_persistent(kern, prm, NW * 32, shmem, s, rg.pdl, op->ctx, "nd_hex_apply4_kernel", false, false, op->ctx->sm_count * MINB, NW,
                           L::NEW, nb);
}

template <int P_, int Q_>
int launch4_kind(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
  const bool a = op->assembled;
  switch (op->kind)
  {
    case B2P_CURLCURL:
      return a ? launch4<P_, Q_, B2P_CURLCURL, true>(op, lidx, alpha, x, y, rg, s)
               : launch4<P_, Q_, B2P_CURLCURL, false>(op, lidx, alpha, x, y, rg, s);
    case B2P_ND_MASS:
      return a ? launch4<P_, Q_, B2P_ND_MASS, true>(op, lidx, alpha, x, y, rg, s)
               : launch4<P_, Q_, B2P_ND_MASS, false>(op, lidx, alpha, x, y, rg, s);
    case B2P_CURLCURL_MASS:
      return a ? launch4<P_, Q_, B2P_CURLCURL_MASS, true>(op, lidx, alpha, x, y, rg, s)
               : launch4<P_, Q_, B2P_CURLCURL_MASS, false>(op, lidx, alpha, x, y, rg, s);
  }
  set_error(op->ctx, "nd_hex_apply: unsupported kind %d", op->kind);
  return B2P_ERR_UNSUPPORTED;
}

// Fused complex apply: one launch, geometry streamed once for both parts (see ND4ParamsZ).
template <int P_, int Q_, int KIND>
int launch4z(b2p_op *op, const int32_t *lidx, const double *zcoef, int has_imag, double alpha, const double *xr, const double *xi,
             double *yr, double *yi, cudaStream_t s)
{
  using L = ND4Layout<P_, Q_, KIND, false, true>;
  if constexpr (L::NEW < 2)
  {
    set_error(op->ctx, "fused complex apply: q1d=%d leaves one element slot per warp", Q_);
    return B2P_ERR_UNSUPPORTED;
  }
  else
  {
    constexpr int SMEM_SM = 222 * 1024;
    constexpr int WPS0 = (SMEM_SM / L::WS) < 1 ? 1 : SMEM_SM / L::WS;
    constexpr int WPS = WPS0 > 8 ? 8 : WPS0;  // 8 warps per SM at up to 255 registers, as the real kernel (no spills)
    constexpr int MINB = (WPS >= 8) ? 2 : 1;
    constexpr int NW = (WPS / MINB) < 1 ? 1 : WPS / MINB;
    const size_t shmem = (size_t)NW * L::WS;
    auto kern = nd_hex_apply4_kernel<P_, Q_, KIND, false, false, NW, MINB, true>;
    if (op->ne <= 0) return B2P_SUCCESS;
    if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
    ND4ParamsZ<P_, Q_> prm;
    prm.lidx = lidx;
    prm.qd = op->geom->qd;
    prm.aq = nullptr;
    prm.mat = op->mat;
    prm.emat = op->emat;
    prm.ecoef = nullptr;
    prm.x = xr;
    prm.y = yr;
    prm.alpha = alpha;
    prm.ne = op->ne;
    set_split_wait(prm, op, ApplyRange());
    prm.iso = 0;
    prm.xi = xi;
    prm.yi = yi;
    prm.zcoef = zcoef;
    prm.has_imag = has_imag;
    copy_tables(op->h_tab.data(), P_, Q_, Q_, prm.Bo, prm.Bc, prm.Gc);
    const int nb = (op->ne + L::NEB - 1) / L::NEB;
    return launch_persistent(kern, prm, NW * 32, shmem, s, false, op->ctx, "nd_hex_apply4_kernel", false, true, op->ctx->sm_count * MINB, NW,
                             L::NEB, nb);
  }
}

template <int P_, int Q_>
int launch4z_kind(b2p_op *op, int kind, const int32_t *lidx, const double *zcoef, int has_imag, double alpha, const double *xr,
                  const double *xi, double *yr, double *yi, cudaStream_t s)
{
  switch (kind)
  {
    case B2P_CURLCURL: return launch4z<P_, Q_, B2P_CURLCURL>(op, lidx, zcoef, has_imag, alpha, xr, xi, yr, yi, s);
    case B2P_ND_MASS: return launch4z<P_, Q_, B2P_ND_MASS>(op, lidx, zcoef, has_imag, alpha, xr, xi, yr, yi, s);
    case B2P_CURLCURL_MASS: return launch4z<P_, Q_, B2P_CURLCURL_MASS>(op, lidx, zcoef, has_imag, alpha, xr, xi, yr, yi, s);
  }
  set_error(op->ctx, "fused complex apply: unsupported kind %d", kind);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace

bool nd_hex_apply4z_eligible(const b2p_op *op)
{
  // two (element, part) slots per warp need q1d^2 <= 16; default quadrature (q1d = p + 1) only
  return op && !op->dense && !op->assembled && op->kind != B2P_H1_DIFFUSION && op->q1d == op->p + 1 && op->q1d >= 2 && op->q1d <= 4;
}

// `op` supplies geometry, restriction and tables; `kind` says which parts of the complex coefficient block are used.
int launch_nd_hex_apply4z(b2p_op *op, int kind, const int32_t *lidx, const double *zcoef, int has_imag, double alpha,
                          const double *xr, const double *xi, double *yr, double *yi, cudaStream_t s)
{
#define B2P_CASE(PP, QQ) \
  if (op->p == PP && op->q1d == QQ) return launch4z_kind<PP, QQ>(op, kind, lidx, zcoef, has_imag, alpha, xr, xi, yr, yi, s);
  B2P_CASE(1, 2) B2P_CASE(2, 3) B2P_CASE(3, 4)
#undef B2P_CASE
  set_error(op->ctx, "fused complex apply: no kernel for p=%d q1d=%d", op->p, op->q1d);
  return B2P_ERR_UNSUPPORTED;
}

int launch_nd_hex_apply4(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s)
{
#define B2P_CASE(PP, QQ) \
  if (op->p == PP && op->q1d == QQ) return launch4_kind<PP, QQ>(op, lidx, alpha, x, y, rg, s);
  B2P_CASE(1, 2) B2P_CASE(1, 3) B2P_CASE(1, 4) B2P_CASE(1, 5) B2P_CASE(1, 6) B2P_CASE(1, 7)
  B2P_CASE(2, 3) B2P_CASE(2, 4) B2P_CASE(2, 5) B2P_CASE(2, 6) B2P_CASE(2, 7)
  B2P_CASE(3, 4) B2P_CASE(3, 5) B2P_CASE(3, 6) B2P_CASE(3, 7)
  B2P_CASE(4, 5) B2P_CASE(4, 6) B2P_CASE(4, 7)
  B2P_CASE(5, 6) B2P_CASE(5, 7)
  B2P_CASE(6, 7)
#undef B2P_CASE
  set_error(op->ctx, "nd_hex_apply: no kernel for p=%d q1d=%d", op->p, op->q1d);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace b2p
