// Nedelec hexahedron apply kernel, round-2 pipeline: registers instead of shared-memory staging.
//
//   y_L += alpha * sum_e E_e^T  B^T  D  B  E_e x_L          (curl-curl, mass, curl-curl + mass; D applied on the fly)
//
// Same operator, same warp-autonomous organisation and the same work-array layout as nd_hex_apply4_kernel
// (b2p_hex_nd4.cu): a warp owns a batch of NEW elements through the phases Z, (Y,) XDX, Yt, Zt and only ever
// synchronises with itself. What changed is how the HBM streams reach the arithmetic. ncu of the round-1 kernel
// (profiles/r01_nd_hex_apply4_p3_ncu_details.txt) showed 2 warps per scheduler stalled on fixed-latency and
// shared-memory dependencies with the L1/shared data pipe at 71 %: 27 KB of shared memory and 254 registers per warp
// left no room for more warps, and 80 + 48 of the 337 wavefronts per element only staged data that each lane reads once.
//   * geometry q-data: coalesced LDG (L1 no-allocate) straight into the registers of the lane that owns the
//     (qy,qz) line, one qx ahead of the pointwise D; the batch's 10 KB block was pulled into L2 one batch earlier by a
//     single cp.async.bulk.prefetch.L2 -- no TMA->shared->LDS round trip, no 10 KB buffer per warp
//   * x values: gathered by LDG into registers one batch ahead (11 doubles per lane at p = 3), signs kept in a
//     bit mask -- no LDGSTS staging buffer, no second read of the index row in the Z phase
//   * the restriction indices + the elements' coefficient block still arrive by TMA bulk copy into a 3-slot ring
//   * XDX can consume the Z region directly (FWD): the y-contraction of the lane's own line is accumulated
//     straight into the 24 point accumulators, so neither the 25 line inputs nor the forward Y region exist
// Shared memory per warp drops from 27 KB to ~15 KB and the register budget to <= 168, so 12 warps per SM fit.
// Node geometry (NODES, the symmetric kinds at p = 3 on a trilinear mesh whose geometry object kept its vertices,
// b2p_geom::xe; nd_hex_apply6_reads_nodes): no q-data stream at all. The batch's 8 vertices per element (192 B instead of 80 B per point) ride in the ring slot after the
// coefficient blocks, and the D loop forms J, cof(J) and detJ at each point from them with the definition of the stored q-data
// (b2p_geom1.cuh) and applies D scaled once by alpha w / detJ: the staged q-data buffer, its bulk copy and its mbarrier are gone.
//
// Reference semantics: ceed::Operator::AddMult over CeedOperatorApplyAdd
// (/root/reference/palace/fem/libceed/operator.cpp:148-178,192-212); D from
// /root/reference/palace/fem/qfunctions/33/{hdiv,hcurl,hdivmass}_33_qf.h.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"
#include "b2p_pipe.cuh"
#include "b2p_geom1.cuh"

namespace b2p
{

namespace
{

template <int P_, int Q_>
struct ND6Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction, rows padded to 16 bytes (B2P_SKIP_IDX = masked/pad)
  const double *qd;     // [ne][10][Q] geometry, x-slowest point order
  const double *xe;     // [ne][3][8] element vertices of a trilinear mesh (NODES kernels, instead of qd)
  const double *ecoef;  // [ne][18] per-element coefficient matrices (value part, derivative part)
  const double *x;
  double *y;
  double *sink;  // [SINK_SLOTS] scratch: masked entries scatter 0.0 into the thread's slot (branch-free RED)
  double alpha;
  int ne;
  VSplit sp;
  const unsigned long long *wait_flags, *wait_expect;  // peer-memory halo flags (SPLIT kernels only)
  int wait_n, wait_from_elem;
  int iso;  // all coefficient matrices are multiples of the identity
  // 1-D tables, rows c < H = ceil(q/2) only: the launcher has verified the mirror symmetry of MFEM's Gauss-Legendre /
  // Gauss-Lobatto bases on a symmetric point set, Bo[q-1-c][p-1-i] = Bo[c][i], Bc[q-1-c][n-1-i] = Bc[c][i],
  // Gc[q-1-c][n-1-i] = -Gc[c][i]. ptxas keeps every table entry a DFMA touches in a REGISTER (no constant-bank operand
  // on the FP64 pipe: 0 of 924 DFMA in the round-1 SASS), so half the rows is 40 registers less.
  static constexpr int H = (Q_ + 1) / 2;
  double Bo[H * P_];
  double Bc[H * (P_ + 1)];
  double Gc[H * (P_ + 1)];
  // NODES: the linear nodal basis, its derivative and the weights at the 1-D points (b2p_geom1.cuh)
  double nB[2 * Q_], nG[2 * Q_], qw[Q_];
};

struct Nd6Pad
{
  int p, q, kind, a, b, y;
};
constexpr Nd6Pad nd6_pad_table[] = {
#include "b2p_nd4_pads.inc"
};
constexpr Nd6Pad nd6_pads(int p, int q, int kind)
{
  for (const Nd6Pad &e : nd6_pad_table)
    if (e.p == p && e.q == q && e.kind == kind) return e;
  return Nd6Pad{p, q, kind, 1, 1, 4};
}
constexpr int nd6_pow2ceil(int x)
{
  int r = 1;
  while (r < x) r *= 2;
  return r;
}
constexpr int nd6_lane_stride(int items, int nel)
{
  const int pc = nd6_pow2ceil(items), rounds = (nel * items + 31) / 32;
  return (nel * pc <= 32 * rounds) ? pc : items;
}

// Work-array layout: identical to ND4Layout (b2p_hex_nd4.cu) -- rows over the index the next phase contracts, padded
// row strides from b2p_nd4_pads.inc -- minus the staging buffers.
// ALIAS: the Y region (written by the second half of XDX, read by Yt) lies on top of the Z region (read by the first
// half of XDX, written by Yt) -- two extra __syncwarp() separate the reads of one from the writes of the other.
// GSM: the batch's q-data is staged in shared memory by TMA (as in nd_hex_apply4_kernel) instead of LDG into registers.
// NODES: no q-data; the batch's element vertices ride in the ring slot after the coefficient blocks.
template <int P_, int Q_, int KIND, bool ALIAS = false, bool GSM = false, bool NODES = false>
struct ND6Layout
{
  static constexpr int p = P_, q = Q_, n = P_ + 1, Q = q * q * q, P = 3 * p * n * n, D3 = p * n * n;
  static constexpr int PS = (P + 3) & ~3;
  // B2P_ND_BLOCK: the CURLCURL_MASS data flow (and its row pads) with the four-tensor block of b2p_op::bcoef in the D phase
  static constexpr bool BLOCK = (KIND == B2P_ND_BLOCK);
  static constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS || BLOCK);
  static constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS || BLOCK);
  static constexpr int NEW = (q * q >= 32) ? 1 : 32 / (q * q);
  static constexpr Nd6Pad PAD = nd6_pads(P_, Q_, BLOCK ? B2P_CURLCURL_MASS : KIND);
  static constexpr int NXA = p * q, NNA = n * q;
  static constexpr int A_XA = 0, A_XB = A_XA + NEW * NXA, A_ZA = A_XB + (CURL ? NEW * NXA : 0), LA = A_ZA + NEW * NNA,
                       RSA = LA + PAD.a;
  static constexpr int B_YA = 0, B_YB = B_YA + NEW * NNA, LB = B_YB + (CURL ? NEW * NNA : 0), RSB = LB + PAD.b;
  static constexpr int ZA0 = 0, ZB0 = ZA0 + n * RSA, ZSZ = ZB0 + p * RSB;
  static constexpr int Y_X1 = 0, Y_X2 = Y_X1 + (MASS ? NEW * NXA : 0), Y_X3 = Y_X2 + (CURL ? NEW * NXA : 0),
                       Y_Y1 = Y_X3 + (CURL ? NEW * NXA : 0), Y_Y2 = Y_Y1 + NEW * NNA, Y_Z1 = Y_Y2 + (CURL ? NEW * NNA : 0),
                       Y_Z3 = Y_Z1 + NEW * NNA, LY = Y_Z3 + (CURL ? NEW * NNA : 0), RSY = LY + PAD.y;
  static constexpr int LSX = nd6_lane_stride(p * n, NEW), LSZ = nd6_lane_stride(n * n, NEW);
  // Z-phase lane rounds and the x values a lane keeps per round
  static constexpr int LW = (NEW * LSX > NEW * LSZ) ? NEW * LSX : NEW * LSZ;
  static constexpr int ZROUNDS = (LW + 31) / 32;
  static constexpr int NXR = 2 * n + p;
  // Z-phase dump cells: an idle lane of half-warp h (= w / 16) stores its x / y / z-line results from ZD_X / ZD_Y / ZD_Z + 12 h
  // on instead of into the Z region, so the phase has no divergent region. The cells lie past the Z region, in the Y region or
  // the tail of the work array, which the Z phase leaves free. Their residues modulo 16 doubles keep them out of every bank an
  // active lane of the same half-warp stores to, for all p = 2 and p = 3 layouts (the half-warp model of tools/smem_sim.py).
  static constexpr int ZD_X = ZSZ + ((12 - ZSZ) & 15), ZD_Y = ZSZ + ((3 - ZSZ) & 15), ZD_Z = ZD_Y;
  static constexpr int ZDH = 12 * (2 * ZROUNDS - 1);
  static constexpr int ZDX_END = ZD_X + ZDH + (A_XB - A_XA) + q, ZDY_END = ZD_Y + ZDH + (B_YB - B_YA) + q;
  static constexpr int ZDEND = ZDX_END > ZDY_END ? ZDX_END : ZDY_END;
  static constexpr int Y0 = ALIAS ? 0 : ZSZ, WEND0 = (ALIAS && ZSZ > q * RSY) ? ZSZ : Y0 + q * RSY,
                       WEND = WEND0 > ZDEND ? WEND0 : ZDEND, WTOT = (WEND + 1) & ~1;
  static constexpr int GE = 10 * Q;   // doubles of q-data per element
  static constexpr int CE = BLOCK ? 36 : 18;  // coefficient doubles per element: two 3x3 tensors, four for the block form
  static constexpr int NE8 = 24;     // doubles of vertex coordinates per element (NODES)
  // one ring slot: the batch's index rows followed by its coefficient blocks and, with NODES, its vertices (one mbarrier, one
  // transaction count)
  static constexpr int SLOT_I = NEW * PS * 4, SLOT_C = NEW * CE * 8, SLOT_N = NODES ? NEW * NE8 * 8 : 0,
                       SLOT = (SLOT_I + SLOT_C + SLOT_N + 15) & ~15;
  static constexpr int OFF_G = 0;                     // [NEW * GE] doubles of staged q-data (GSM)
  static constexpr int OFF_W = OFF_G + (GSM ? NEW * GE * 8 : 0);
  static constexpr int OFF_R = OFF_W + WTOT * 8;      // [3] ring slots
  static constexpr int OFF_B = OFF_R + 3 * SLOT;      // 3 ring mbarriers + 1 for the q-data
  static constexpr int WS = (OFF_B + 4 * 8 + 15) & ~15;
};

#ifdef B2P_EMU
inline double ldg_stream_f64(const double *p) { return *p; }
inline void prefetch_l2_bulk(const void *, uint32_t) {}
inline void prefetch_l1(const void *) {}
inline double rcp_f64(double d) { return 1.0 / d; }
#else
// 1/d within 1 ulp for normal, non-zero d whose reciprocal is normal, without the slow-path branch of an IEEE division:
// MUFU.RCP64H and two Newton steps. A degenerate element (detJ = 0) gives inf / NaN, as the division of the stored route does.
__device__ __forceinline__ double rcp_f64(double d)
{
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  double e = fma(-d, r, 1.0);
  r = fma(r, e, r);
  e = fma(-d, r, 1.0);
  return fma(r, e, r);
}
__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// streaming read: the q-data is used exactly once per launch -- keep it out of L1 (the x gathers reuse lines there)
__device__ __forceinline__ double ldg_stream_f64(const double *p)
{
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void prefetch_l2_bulk(const void *p, uint32_t bytes)
{
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
#endif

// FWD: XDX consumes the Z region (no forward Y phase / Y region; the backward Y region aliases the Z region).
// GSM: q-data through shared memory (TMA) instead of LDG into registers.  XLATE: gather the next batch's x values after
// XDX instead of right after the Z phase (their registers are then not live across XDX).
// Scatter-add without a predicate: ptxas turns every predicated RED into a branch region (BSSY / BRA / BSYNC), which cuts
// the Zt phase into basic blocks of two short DFMA chains. Masked entries (B2P_SKIP_IDX; idle lanes and tail slots carry it
// too) add 0.0 to the thread's own slot of a scratch array instead -- distinct addresses, no hot spot.
template <bool SPLIT>
__device__ __forceinline__ void scatter_nb(double *y, const VSplit &sp, double *sink, int32_t gi, double v)
{
  const bool skip = gi == (int32_t)B2P_SKIP_IDX;
  const int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
  const double sv = skip ? 0.0 : __hiloint2double(hi, __double2loint(v));
  const uint32_t a = (uint32_t)abs_idx(gi), no = (uint32_t)sp.n_owned;
  double *addr = SPLIT ? ((a < no) ? y + a : sp.yg + (a - no)) : y + a;
  addr = skip ? sink : addr;
#ifdef B2P_EMU
  atomicAdd(addr, sv);
#else
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(sv) : "memory");
#endif
}

// GL1 (with GSM = false): L1 is the staging buffer -- the batch's q-data lines are pulled into L1 by prefetch.global.L1 one
// batch ahead and the LDGs of the D loop hit there (half the L1 data-pipe wavefronts of TMA -> shared -> LDS, no buffer).
// NODES (with GSM = GL1 = false): trilinear geometry evaluated at each point from the element's 8 vertices (b2p_geom1.cuh), which
// arrive with the batch's ring slot -- 192 bytes per element instead of 80 per point of stored q-data.
template <int P_, int Q_, int KIND, bool SPLIT, int NW, int MINB, bool FWD, bool GSM = false, bool XLATE = false, bool GL1 = false,
          bool NODES = false>
__global__ void __launch_bounds__(NW * 32, MINB) nd_hex_apply6_kernel(const __grid_constant__ ND6Params<P_, Q_> prm)
{
  static_assert(!NODES || (!GSM && !GL1), "node geometry stages no q-data");
  using L = ND6Layout<P_, Q_, KIND, FWD, GSM, NODES>;
  static_assert(!NODES || !L::BLOCK, "the block form runs on stored q-data");
  constexpr bool ALIAS = FWD;
  static_assert(L::NEW * Q_ * Q_ <= 32, "one XDX item per lane");
  constexpr int p = L::p, q = L::q, n = L::n, Q = L::Q, D3 = L::D3, GE = L::GE, PS = L::PS, NEW = L::NEW, CE = L::CE;
  constexpr int RSA = L::RSA, RSB = L::RSB, RSY = L::RSY, NXA = L::NXA, NNA = L::NNA;
  constexpr bool MASS = L::MASS, CURL = L::CURL;
  constexpr int QQ = q * q;
  constexpr int IPX = p * n, IPZ = n * n, LSX = L::LSX, LSZ = L::LSZ, ZROUNDS = L::ZROUNDS, NXR = L::NXR;
  constexpr int H = (q + 1) / 2;
// table entry (row c, column i) from the stored half (indices are compile-time constants after unrolling)
#define TBO(c, i) ((c) < H ? prm.Bo[(c) * p + (i)] : prm.Bo[(q - 1 - (c)) * p + (p - 1 - (i))])
#define TBC(c, i) ((c) < H ? prm.Bc[(c) * n + (i)] : prm.Bc[(q - 1 - (c)) * n + (n - 1 - (i))])
#define TGC(c, i) ((c) < H ? prm.Gc[(c) * n + (i)] : -prm.Gc[(q - 1 - (c)) * n + (n - 1 - (i))])

  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned char *wbase = smem_raw + (size_t)wid * L::WS;
  double *sW = (double *)(wbase + L::OFF_W);
  unsigned char *sR = wbase + L::OFF_R;
  uint64_t *bar_i = (uint64_t *)(wbase + L::OFF_B);  // [3]
  uint64_t *bar_g = bar_i + 3;
  double *sG = (double *)(wbase + L::OFF_G);

  const int nb = (prm.ne + NEW - 1) / NEW;  // element batches
  const int GW = gridDim.x * NW;            // warps in the grid
  int b = blockIdx.x * NW + wid;
  griddep_launch_dependents();              // a dependent launched programmatically (the halo POST kernel) may be scheduled as CTAs retire
  if (b >= nb) return;                      // (whole warp)

  if (lane == 0)
  {
    mbar_init(bar_i + 0, 1);
    mbar_init(bar_i + 1, 1);
    mbar_init(bar_i + 2, 1);
    if (GSM) mbar_init(bar_g, 1);
  }
  __syncwarp();

  const uint64_t once = l2_evict_first_policy();  // the bulk copies below stream data read once per launch
  auto issue_ring = [&](int bb, int slot)
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const uint32_t ib = (uint32_t)(nel * PS * sizeof(int32_t)), cb = (uint32_t)(nel * CE * sizeof(double)),
                   nb8 = NODES ? (uint32_t)(nel * L::NE8 * sizeof(double)) : 0u;
    mbar_expect_tx(bar_i + slot, ib + cb + nb8);
    tma_bulk_g2s_hint(sR + slot * L::SLOT, prm.lidx + (size_t)e0 * PS, ib, bar_i + slot, once);
    tma_bulk_g2s_hint(sR + slot * L::SLOT + L::SLOT_I, prm.ecoef + (size_t)e0 * CE, cb, bar_i + slot, once);
    if constexpr (NODES) tma_bulk_g2s_hint(sR + slot * L::SLOT + L::SLOT_I + L::SLOT_C, prm.xe + (size_t)e0 * L::NE8, nb8, bar_i + slot, once);
  };
  auto prefetch_geom = [&](int bb)
  {
    if (GSM || GL1 || NODES) return;
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    prefetch_l2_bulk(prm.qd + (size_t)e0 * GE, (uint32_t)(nel * GE * sizeof(double)));
  };
  auto prefetch_geom_l1 = [&](int bb)  // (whole warp) one 128-byte line per lane and round
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const char *base = (const char *)(prm.qd + (size_t)e0 * GE);
    const int lines = nel * GE * 8 / 128;
    for (int i = lane; i < lines; i += 32) prefetch_l1(base + (size_t)i * 128);
  };
  auto issue_geom = [&](int bb)
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const uint32_t bytes = (uint32_t)(nel * GE * sizeof(double));
    mbar_expect_tx(bar_g, bytes);
    tma_bulk_g2s_hint(sG, prm.qd + (size_t)e0 * GE, bytes, bar_g, once);
  };

  // x values of the batch whose Z phase comes next, in the registers of the lane that contracts them; `xsign` holds the
  // restriction signs (bit r*NXR + k), masked / padded / out-of-range slots are loaded as zero
  double xr[ZROUNDS][NXR];
  uint32_t xsign[ZROUNDS];
  auto gather_x = [&](int bb, int slot)
  {
    const int e0 = bb * NEW, nel = min(NEW, prm.ne - e0);
    const int32_t *gI = (const int32_t *)(sR + slot * L::SLOT);
#pragma unroll
    for (int r = 0; r < ZROUNDS; r++)
    {
      const int w = lane + 32 * r;
      const bool vx = (w / LSX) < NEW && (w % LSX) < IPX && (w / LSX) < nel, vz = (w / LSZ) < NEW && (w % LSZ) < IPZ && (w / LSZ) < nel;
      const int ex = vx ? w / LSX : 0, tx = vx ? w % LSX : 0;
      const int ez = vz ? w / LSZ : 0, tz = vz ? w % LSZ : 0;
      uint32_t sg = 0;
      auto fetch = [&](int pos, bool valid, int bit) -> double
      {
        const int32_t gi = gI[pos];
        const bool ok = valid && gi != (int32_t)B2P_SKIP_IDX;
        sg |= ((uint32_t)gi >> 31) << bit;
        const int32_t a = ok ? abs_idx(gi) : 0;
        const double *src = SPLIT ? split_src_fast(prm.x, prm.sp, a) : prm.x + (uint32_t)a;
        return ok ? __ldg(src) : 0.0;
      };
#pragma unroll
      for (int k = 0; k < n; k++)
      {
        xr[r][k] = fetch(ex * PS + tx + p * n * k, vx, k);
        xr[r][n + k] = fetch(ex * PS + D3 + tx + n * p * k, vx, n + k);
      }
#pragma unroll
      for (int k = 0; k < p; k++) xr[r][2 * n + k] = fetch(ez * PS + 2 * D3 + tz + n * n * k, vz, 2 * n + k);
      xsign[r] = sg;
    }
  };
  auto signed_x = [&](int r, int k) -> double
  {
    const double v = xr[r][k];
    const int hi = __double2hiint(v) ^ (int)(((xsign[r] >> k) & 1u) << 31);
    return __hiloint2double(hi, __double2loint(v));
  };

  // Peer-memory halo: ghost values of this step are complete once every neighbour's flag reached the expected epoch.
  bool y_ready = false;  // the grid dependency (zero-fill of y / the halo PRE kernel under programmatic dependent launch) is resolved
  bool ghosts_ready = !(SPLIT && prm.wait_n > 0);
  auto wait_ghosts = [&](int bb)
  {
    if (ghosts_ready || (bb + 1) * NEW <= prm.wait_from_elem) return;
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

  uint32_t par_i = 0, par_g = 0;  // mbarrier phase parities: bit s for ring slot s
  if (lane == 0)
  {
    issue_ring(b, 0);
    if (b + GW < nb) issue_ring(b + GW, 1);
    if (b + 2 * GW < nb) issue_ring(b + 2 * GW, 2);
    if (GSM) issue_geom(b);
    prefetch_geom(b);
    if (b + GW < nb) prefetch_geom(b + GW);
  }
  if constexpr (GL1) prefetch_geom_l1(b);
  mbar_wait(bar_i + 0, 0);
  par_i ^= 1u;
  wait_ghosts(b);
  gather_x(b, 0);

  const double alpha = prm.alpha;
  double *my_sink = prm.sink + ((blockIdx.x * (NW * 32) + threadIdx.x) & (b2p_ctx::SINK_SLOTS - 1));
  int slot = 0;
  for (; b < nb; b += GW)
  {
    const int nslot = (slot == 2) ? 0 : slot + 1;
    const int bn = b + GW;
    const int e0 = b * NEW, nel = min(NEW, prm.ne - e0);  // nel: valid element slots of this batch
    const int32_t *cI = (const int32_t *)(sR + slot * L::SLOT);
    const double *cC = (const double *)(sR + slot * L::SLOT + L::SLOT_I);
    const double *cN = (const double *)(sR + slot * L::SLOT + L::SLOT_I + L::SLOT_C);

    // ------------------------------------------------------------------ phase Z (z-contraction, from registers)
    {
#pragma unroll
      for (int r = 0; r < ZROUNDS; r++)
      {
        const int w = lane + 32 * r;
        const bool vx = (w / LSX) < NEW && (w % LSX) < IPX, vz = (w / LSZ) < NEW && (w % LSZ) < IPZ;
        const int ex = vx ? w / LSX : 0, tx = vx ? w % LSX : 0;
        const int ez = vz ? w / LSZ : 0, tz = vz ? w % LSZ : 0;
        double ux[n], uy[n], uz[p];
#pragma unroll
        for (int k = 0; k < n; k++)
        {
          ux[k] = signed_x(r, k);
          uy[k] = signed_x(r, n + k);
        }
#pragma unroll
        for (int k = 0; k < p; k++) uz[k] = signed_x(r, 2 * n + k);
        // No divergent regions: idle lanes run on item 0 and store into their dump cells (ND6Layout::ZD_*). A predicated store
        // would let ptxas sink the contractions into a branch region.
        const int dmp = 12 * (w >> 4);
        {
          double *xa = vx ? sW + L::ZA0 + (tx / p) * RSA + L::A_XA + ex * NXA + q * (tx % p) : sW + L::ZD_X + dmp,
                 *xb = xa + (L::A_XB - L::A_XA);
          double *ya = vx ? sW + L::ZB0 + (tx / n) * RSB + L::B_YA + ex * NNA + q * (tx % n) : sW + L::ZD_Y + dmp,
                 *yb = ya + (L::B_YB - L::B_YA);
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            double a = 0.0, b2 = 0.0, c = 0.0, d = 0.0;
#pragma unroll
            for (int k = 0; k < n; k++)
            {
              a += TBC(qz, k) * ux[k];
              c += TBC(qz, k) * uy[k];
              if (CURL) b2 += TGC(qz, k) * ux[k];
              if (CURL) d += TGC(qz, k) * uy[k];
            }
            xa[qz] = a;
            ya[qz] = c;
            if (CURL) xb[qz] = b2;
            if (CURL) yb[qz] = d;
          }
        }
        {
          double *za = vz ? sW + L::ZA0 + (tz / n) * RSA + L::A_ZA + ez * NNA + q * (tz % n) : sW + L::ZD_Z + dmp;
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            double a = 0.0;
#pragma unroll
            for (int k = 0; k < p; k++) a += TBO(qz, k) * uz[k];
            za[qz] = a;
          }
        }
      }
    }
    __syncwarp();
    // the x registers are free: gather the next batch's values while this one computes; its q-data is already on the
    // way to L2, pull the one after it
    auto next_batch = [&]()
    {
      if (bn < nb)
      {
        mbar_wait(bar_i + nslot, (par_i >> nslot) & 1u);
        par_i ^= (1u << nslot);
        wait_ghosts(bn);
        gather_x(bn, nslot);
        if (lane == 0 && bn + GW < nb) prefetch_geom(bn + GW);
      }
    };
    if constexpr (!XLATE) next_batch();

    // ------------------------------------------------------------------ phase Y (y-contraction)
    if constexpr (!FWD)
    {
      constexpr int IX = NEW * p * q, IN = NEW * n * q;
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
          double *v1 = sW + L::Y0 + L::Y_X1 + wx, *v2 = sW + L::Y0 + L::Y_X2 + wx, *v3 = sW + L::Y0 + L::Y_X3 + wx;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            double s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              if (MASS) s1 += TBC(qy, j) * xa[j];
              if (CURL) s2 += TBC(qy, j) * xb[j];
              if (CURL) s3 += TGC(qy, j) * xa[j];
            }
            if (MASS) v1[RSY * qy] = s1;
            if (CURL) v2[RSY * qy] = s2;
            if (CURL) v3[RSY * qy] = s3;
          }
        }
        if (vn)
        {
          double *v1 = sW + L::Y0 + L::Y_Y1 + wn, *v2 = sW + L::Y0 + L::Y_Y2 + wn;
          double *z1 = sW + L::Y0 + L::Y_Z1 + wn, *z3 = sW + L::Y0 + L::Y_Z3 + wn;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            double s1 = 0.0, s2 = 0.0, t1 = 0.0, t3 = 0.0;
#pragma unroll
            for (int j = 0; j < p; j++)
            {
              s1 += TBO(qy, j) * ya[j];
              if (CURL) s2 += TBO(qy, j) * yb[j];
            }
#pragma unroll
            for (int j = 0; j < n; j++)
            {
              t1 += TBC(qy, j) * za[j];
              if (CURL) t3 += TGC(qy, j) * za[j];
            }
            v1[RSY * qy] = s1;
            if (CURL) v2[RSY * qy] = s2;
            z1[RSY * qy] = t1;
            if (CURL) z3[RSY * qy] = t3;
          }
        }
      }
      __syncwarp();
    }

    // ------------------------------------------------------------------ phase XDX
    // item s = qy + q*qz of element slot e: all qx of this line live in registers.
    if constexpr (GSM)
    {
      mbar_wait(bar_g, par_g);  // q-data of this batch has landed
      par_g ^= 1;
    }
    {
      // one item per lane (NEW * QQ <= 32); lanes beyond the last item run on item 0 and store nothing
      const bool act = lane < NEW * QQ;
      const int w = act ? lane : 0;
      const int e = w / QQ, s = w % QQ;
      const bool ok = act && e < nel;
      // q-data of this lane's line, point qx at g[comp * Q + QQ * qx]; rows of a tail batch read element 0 (discarded)
      const double *g = GSM ? sG + (ok ? e : 0) * GE + s : prm.qd + (size_t)(e0 + (ok ? e : 0)) * GE + s;
      double G[2][10];
      if constexpr (!GSM && !NODES)
      {
#pragma unroll
        for (int c = 0; c < 10; c++) G[0][c] = GL1 ? __ldg(g + c * Q) : ldg_stream_f64(g + c * Q);
      }
      double *WX = sW + L::Y0 + (s % q) * RSY + e * NXA + s / q;
      double *WN = sW + L::Y0 + (s % q) * RSY + e * NNA + s / q;
      double uu[q][3], cc[q][3];
#pragma unroll
      for (int qx = 0; qx < q; qx++)
#pragma unroll
        for (int r = 0; r < 3; r++) uu[qx][r] = cc[qx][r] = 0.0;
      if constexpr (FWD)
      {
        // y-contraction of this lane's own line straight from the Z region (broadcast reads), every line value folded
        // into the point accumulators at once
        const int qy = s % q, qz = s / q;
        // this lane's rows of the y tables (lane-dependent: indexed loads from the parameter block, mirrored rows reversed)
        const bool mir = qy >= H;
        const int cy = mir ? q - 1 - qy : qy;
        const double gsgn = mir ? -1.0 : 1.0;
        double bo[p], bc[n], gc[n];
#pragma unroll
        for (int j = 0; j < p; j++) bo[j] = prm.Bo[cy * p + (mir ? p - 1 - j : j)];
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          bc[j] = prm.Bc[cy * n + (mir ? n - 1 - j : j)];
          gc[j] = gsgn * prm.Gc[cy * n + (mir ? n - 1 - j : j)];
        }
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
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) uu[qx][0] += TBO(qx, i) * s1;
            if (CURL) cc[qx][1] += TBO(qx, i) * s2;
            if (CURL) cc[qx][2] -= TBO(qx, i) * s3;
          }
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
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) uu[qx][1] += TBC(qx, i) * s1;
            if (CURL) cc[qx][0] -= TBC(qx, i) * s2;
            if (CURL) cc[qx][2] += TGC(qx, i) * s1;
            if (MASS) uu[qx][2] += TBC(qx, i) * t1;
            if (CURL) cc[qx][0] += TBC(qx, i) * t3;
            if (CURL) cc[qx][1] -= TGC(qx, i) * t1;
          }
        }
      }
      else
      {
#pragma unroll
        for (int i = 0; i < p; i++)
        {
          double x1 = 0.0, x2 = 0.0, x3 = 0.0;
          if (MASS) x1 = WX[L::Y_X1 + q * i];
          if (CURL) x2 = WX[L::Y_X2 + q * i];
          if (CURL) x3 = WX[L::Y_X3 + q * i];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) uu[qx][0] += TBO(qx, i) * x1;
            if (CURL) cc[qx][1] += TBO(qx, i) * x2;
            if (CURL) cc[qx][2] -= TBO(qx, i) * x3;
          }
        }
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          double y1, y2 = 0.0, z1, z3 = 0.0;
          y1 = WN[L::Y_Y1 + q * i];
          if (CURL) y2 = WN[L::Y_Y2 + q * i];
          z1 = WN[L::Y_Z1 + q * i];
          if (CURL) z3 = WN[L::Y_Z3 + q * i];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) uu[qx][1] += TBC(qx, i) * y1;
            if (CURL) cc[qx][0] -= TBC(qx, i) * y2;
            if (CURL) cc[qx][2] += TGC(qx, i) * y1;
            if (MASS) uu[qx][2] += TBC(qx, i) * z1;
            if (CURL) cc[qx][0] += TBC(qx, i) * z3;
            if (CURL) cc[qx][1] -= TGC(qx, i) * z1;
          }
        }
      }
      if constexpr (ALIAS) __syncwarp();  // every lane has read its Z-region values: the Y region may overwrite them
      const double *C = cC + e * CE;
      // NODES: this lane's line constants from the element's vertices (broadcast reads); rows of a tail batch read element 0
      Hex1KLine gl;
      double wl = 0.0;  // NODES: alpha w_y w_z of the line, 0 on tail slots
      if constexpr (NODES)
      {
        const int qy = s % q, qz = s / q;
        Hex1Line ls;
        hex1_line(cN + (ok ? e : 0) * L::NE8, prm.nB + 2 * qy, prm.nG + 2 * qy, prm.nB + 2 * qz, prm.nG + 2 * qz, ls);
        hex1_kline(ls, prm.nG, gl);  // row 0 of nG serves every qx (b2p_geom_create_hex checks it)
        wl = (ok ? 1.0 : 0.0) * (alpha * prm.qw[qy] * prm.qw[qz]);  // a 0/1 factor: a select would make ptxas branch around the loads
      }
      // ISO is warp-uniform (prm.iso): the branch is taken once around the whole point loop, so each copy is one basic block in
      // which ptxas can interleave the points' dependent chains. A branch per point would split them.
      auto d_points = [&](auto iso_tag)
      {
        [[maybe_unused]] constexpr bool ISO = decltype(iso_tag)::value;  // (the block form has no iso branch)
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if constexpr (NODES)
          {
            // With K = cof(J) = detJ J^-T and f = alpha w / detJ, the stored route's w detJ A^T C_m A u (A = K / detJ) is
            // f K^T C_m (K u) and its w detJ Jd^T C_k Jd c (Jd = J / detJ) is f J^T C_k (J c): the four 3x3 products do not wait
            // on the reciprocal, only the final scaling does. f is formed on every slot (tail slots hold element 0's geometry)
            // and zeroed through wl: a select around the reciprocal would make ptxas branch around it.
            double J[9], K[9], detJ, v[3] = {0, 0, 0}, cw[3] = {0, 0, 0};
            hex1_kjacobian(gl, prm.nB[2 * qx + 1], J, K, detJ);
            const double f = wl * prm.qw[qx] * rcp_f64(detJ);
            if constexpr (ISO)
            {
              if (MASS) AtAx(K, uu[qx], f * C[0], v);
              if (CURL) AtAx(J, cc[qx], f * C[9], cw);
            }
            else
            {
              if (MASS) AtCAx(K, C, uu[qx], f, v);
              if (CURL) AtCAx(J, C + 9, cc[qx], f, cw);
            }
#pragma unroll
            for (int r = 0; r < 3; r++)
            {
              uu[qx][r] = v[r];
              cc[qx][r] = cw[r];
            }
            continue;
          }
          if constexpr (GSM)
          {
#pragma unroll
            for (int c = 0; c < 10; c++) G[qx & 1][c] = g[c * Q + QQ * qx];
          }
          else if (qx + 1 < q)
          {
            // q-data of the next point of the line is requested before this point's arithmetic
#pragma unroll
            for (int c = 0; c < 10; c++) G[(qx + 1) & 1][c] = GL1 ? __ldg(g + c * Q + QQ * (qx + 1)) : ldg_stream_f64(g + c * Q + QQ * (qx + 1));
          }
          const double *gq = G[qx & 1];
          double v[3] = {0, 0, 0}, cw[3] = {0, 0, 0};
          const double wdetJ = ok ? alpha * gq[0] : 0.0;  // alpha folded into the quadrature weight; tail slots contribute zero
          const double *A = gq + 1;
          if constexpr (L::BLOCK)
          {
            // out_val = w A^T (Cm A u + Cx Jd c),  out_curl = w Jd^T (Ck Jd c + Cw A u)
            double Jd[9], t[3], sc[3], a[3], b[3], z[3];
            cofactor33(A, Jd);
            Ax33(A, uu[qx], t);
            Ax33(Jd, cc[qx], sc);
            Ax33(C, t, a);
            Ax33(C + 27, sc, b);
#pragma unroll
            for (int r = 0; r < 3; r++) z[r] = a[r] + b[r];
            Atx33(A, z, wdetJ, v);
            Ax33(C + 9, sc, a);
            Ax33(C + 18, t, b);
#pragma unroll
            for (int r = 0; r < 3; r++) z[r] = a[r] + b[r];
            Atx33(Jd, z, wdetJ, cw);
          }
          else if constexpr (ISO)
          {
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
#pragma unroll
          for (int r = 0; r < 3; r++)
          {
            uu[qx][r] = v[r];
            cc[qx][r] = cw[r];
          }
        }
      };
      if constexpr (L::BLOCK)
        d_points(std::false_type{});
      else if (prm.iso)
        d_points(std::true_type{});
      else
        d_points(std::false_type{});
      // transposed x-contraction: outputs formed one at a time
#pragma unroll
      for (int i = 0; i < p; i++)
      {
        double a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) a1 += TBO(qx, i) * uu[qx][0];
          if (CURL) a2 += TBO(qx, i) * cc[qx][1];
          if (CURL) a3 -= TBO(qx, i) * cc[qx][2];
        }
        if (MASS && act) WX[L::Y_X1 + q * i] = a1;
        if (CURL && act) WX[L::Y_X2 + q * i] = a2;
        if (CURL && act) WX[L::Y_X3 + q * i] = a3;
      }
#pragma unroll
      for (int i = 0; i < n; i++)
      {
        double b1 = 0, b2 = 0, c1 = 0, c3 = 0;
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) b1 += TBC(qx, i) * uu[qx][1];
          if (CURL) b1 += TGC(qx, i) * cc[qx][2];
          if (CURL) b2 -= TBC(qx, i) * cc[qx][0];
          if (MASS) c1 += TBC(qx, i) * uu[qx][2];
          if (CURL) c1 -= TGC(qx, i) * cc[qx][1];
          if (CURL) c3 += TBC(qx, i) * cc[qx][0];
        }
        if (act) WN[L::Y_Y1 + q * i] = b1;
        if (CURL && act) WN[L::Y_Y2 + q * i] = b2;
        if (act) WN[L::Y_Z1 + q * i] = c1;
        if (CURL && act) WN[L::Y_Z3 + q * i] = c3;
      }
    }
    __syncwarp();
    if constexpr (GSM)
    {
      if (bn < nb && lane == 0)
      {
        fence_proxy_async();
        issue_geom(bn);  // refill the single q-data buffer for the next batch
      }
    }
    if constexpr (GL1)
    {
      if (bn < nb) prefetch_geom_l1(bn);
    }
    if constexpr (XLATE) next_batch();

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
        if constexpr (ALIAS)
        {
          static_assert(!ALIAS || ROUNDS == 1, "aliased work arrays: one Yt round (all Y-region reads precede the Z-region writes)");
          __syncwarp();
        }
        {
          double *za = sW + L::ZA0 + L::A_XA + wx, *zb = sW + L::ZA0 + L::A_XB + wx;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            double a = 0.0, b2 = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              if (MASS) a += TBC(qy, j) * x1[qy];
              if (CURL) a += TGC(qy, j) * x3[qy];
              if (CURL) b2 += TBC(qy, j) * x2[qy];
            }
            if (vx) za[RSA * j] = a;
            if (CURL && vx) zb[RSA * j] = b2;
          }
        }
        {
          double *ya = sW + L::ZB0 + L::B_YA + wn, *yb = sW + L::ZB0 + L::B_YB + wn;
#pragma unroll
          for (int j = 0; j < p; j++)
          {
            double a = 0.0, b2 = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              a += TBO(qy, j) * y1[qy];
              if (CURL) b2 += TBO(qy, j) * y2[qy];
            }
            if (vn) ya[RSB * j] = a;
            if (CURL && vn) yb[RSB * j] = b2;
          }
          double *za = sW + L::ZA0 + L::A_ZA + wn;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            double a = 0.0;
#pragma unroll
            for (int qy = 0; qy < q; qy++)
            {
              a += TBC(qy, j) * z1[qy];
              if (CURL) a += TGC(qy, j) * z3[qy];
            }
            if (vn) za[RSA * j] = a;
          }
        }
      }
    }
    __syncwarp();

    // ------------------------------------------------------------------ phase Zt (transposed z-contraction + scatter)
    // First write to y: under programmatic dependent launch the zero-fill of y that precedes this kernel in the stream
    // may still be running.
    if (!y_ready)
    {
      griddep_wait();
      y_ready = true;
    }
    {
#pragma unroll
      for (int r = 0; r < ZROUNDS; r++)
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
          // idle lanes / tail slots carry the "masked" index: the predicated RED skips them (no divergent region)
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            gx[k] = vx ? cI[ex * PS + tx + p * n * k] : (int32_t)B2P_SKIP_IDX;
            gy[k] = vx ? cI[ex * PS + D3 + tx + n * p * k] : (int32_t)B2P_SKIP_IDX;
          }
#pragma unroll
          for (int k = 0; k < p; k++) gz[k] = vz ? cI[ez * PS + 2 * D3 + tz + n * n * k] : (int32_t)B2P_SKIP_IDX;
        }
        {
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            double o = 0.0, o2 = 0.0;
#pragma unroll
            for (int qz = 0; qz < q; qz++)
            {
              o += TBC(qz, k) * xa[qz];
              o2 += TBC(qz, k) * ya[qz];
              if (CURL) o += TGC(qz, k) * xb[qz];
              if (CURL) o2 += TGC(qz, k) * yb[qz];
            }
            scatter_nb<SPLIT>(prm.y, prm.sp, my_sink, gx[k], o);
            scatter_nb<SPLIT>(prm.y, prm.sp, my_sink, gy[k], o2);
          }
        }
        {
#pragma unroll
          for (int k = 0; k < p; k++)
          {
            double o = 0.0;
#pragma unroll
            for (int qz = 0; qz < q; qz++) o += TBO(qz, k) * za[qz];
            scatter_nb<SPLIT>(prm.y, prm.sp, my_sink, gz[k], o);
          }
        }
      }
    }
    __syncwarp();
    if (b + 3 * GW < nb && lane == 0)
    {
      fence_proxy_async();
      issue_ring(b + 3 * GW, slot);  // this batch's ring slot is free again
    }
    slot = nslot;
  }
#undef TBO
#undef TBC
#undef TGC
}

template <int P_, int Q_, int KIND, int NW, int MINB, bool FWD, bool GSM, bool XLATE, bool WITH_SPLIT, bool GL1 = false, bool NODES = false>
int launch6_cfg(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                bool transpose = false)
{
  using L = ND6Layout<P_, Q_, KIND, FWD, GSM, NODES>;
  const size_t shmem = (size_t)NW * L::WS;
  const bool split = range_split(op, rg);
  auto kern = nd_hex_apply6_kernel<P_, Q_, KIND, false, NW, MINB, FWD, GSM, XLATE, GL1, NODES>;
  if constexpr (WITH_SPLIT)
  {
    if (split) kern = nd_hex_apply6_kernel<P_, Q_, KIND, true, NW, MINB, FWD, GSM, XLATE, GL1, NODES>;
  }
  else if (split)
  {
    set_error(op->ctx, "nd_hex_apply6: this experimental configuration has no owned/ghost split variant");
    return B2P_ERR_UNSUPPORTED;
  }
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  // GL1: leave the rest of the 256 KB array to L1, the staging buffer of the q-data
  const int carveout = GL1 ? (int)((MINB * (shmem + 1024) * 100 + 228 * 1024 - 1) / (228 * 1024)) : -1;
  if (int rc = configure_kernel(op->ctx, kern, shmem, carveout)) return rc;
  ND6Params<P_, Q_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.xe = NODES ? op->geom->xe + (size_t)e_off * L::NE8 : nullptr;
  if constexpr (L::BLOCK)
    prm.ecoef = (transpose ? op->bcoef_t : op->bcoef) + L::CE * (size_t)e_off;
  else
    prm.ecoef = op->ecoef + L::CE * (size_t)e_off;
  prm.x = x;
  prm.y = y;
  prm.sink = op->ctx->d_sink;
  prm.alpha = alpha;
  prm.ne = e_cnt;
  set_split_wait(prm, op, rg);
  prm.iso = (op->iso && !L::BLOCK) ? 1 : 0;
  copy_tables(op->h_tab.data(), P_, Q_, ND6Params<P_, Q_>::H, prm.Bo, prm.Bc, prm.Gc);  // the first H rows: the rest mirror them
  for (int i = 0; i < 2 * Q_; i++) prm.nB[i] = NODES ? op->geom->h_nodeB[i] : 0.0;
  for (int i = 0; i < 2 * Q_; i++) prm.nG[i] = NODES ? op->geom->h_nodeG[i] : 0.0;
  for (int i = 0; i < Q_; i++) prm.qw[i] = NODES ? op->geom->h_qw[i] : 0.0;
  const int nb = (e_cnt + L::NEW - 1) / L::NEW;
  return launch_persistent(kern, prm, NW * 32, shmem, s, rg.pdl, op->ctx, "nd_hex_apply6_kernel", L::BLOCK, false, op->ctx->sm_count * MINB, NW,
                           L::NEW, nb, NODES);
}

// B2P_ND6_CFG = "<warps per CTA><CTAs per SM><f|y><g|l|c|n><e|x>" picks another launch shape / variant of the p = 3
// curl-curl+mass kernel for A/B measurements: f = XDX consumes the Z region, y = separate Y phase; g = q-data staged in
// shared memory by TMA, l = LDG into registers, c = L1 as the staging buffer, n = geometry from the element vertices (a
// geometry that kept them only); e = x gathered right after the Z phase, x = after XDX.
inline int nd6_cfg_code()
{
  static const int code = []
  {
    const char *e = std::getenv("B2P_ND6_CFG");
    if (!e || std::strlen(e) < 5) return 0;
    return (e[0] - '0') * 10000 + (e[1] - '0') * 1000 + (e[2] == 'y' ? 100 : 0) + (e[3] == 'g' ? 10 : e[3] == 'c' ? 20 : e[3] == 'n' ? 30 : 0) + (e[4] == 'x' ? 1 : 0);
  }();
  return code;
}

constexpr int ND6_NW = 4, ND6_MINB = 2;
constexpr bool ND6_FWD = true, ND6_GSM = true, ND6_XLATE = true;

template <int P_, int Q_, int KIND>
int launch6(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
            bool transpose = false)
{
#ifdef B2P_ND6_EXPERIMENTS
  if constexpr (P_ == 3 && KIND == B2P_CURLCURL_MASS)
  {
    switch (nd6_cfg_code())
    {
#define B2P_CFG(NWV, MB, FW, GS, XL) \
  case NWV * 10000 + MB * 1000 + (FW ? 0 : 100) + (GS ? 10 : 0) + (XL ? 1 : 0): \
    return launch6_cfg<P_, Q_, KIND, NWV, MB, FW, GS, XL, false>(op, lidx, alpha, x, y, rg, s);
      B2P_CFG(4, 3, true, false, false)
      B2P_CFG(4, 3, true, false, true)
      B2P_CFG(4, 2, true, true, false)
      B2P_CFG(4, 2, true, true, true)
      B2P_CFG(5, 2, true, true, false)
      B2P_CFG(5, 2, true, true, true)
      B2P_CFG(3, 3, true, true, false)
      B2P_CFG(3, 3, true, true, true)
      B2P_CFG(4, 2, false, true, true)
#undef B2P_CFG
      case 42021: return launch6_cfg<P_, Q_, KIND, 4, 2, true, false, true, false, true>(op, lidx, alpha, x, y, rg, s);   // "42fcx"
      case 42020: return launch6_cfg<P_, Q_, KIND, 4, 2, true, false, false, false, true>(op, lidx, alpha, x, y, rg, s);  // "42fce"
      case 43021: return launch6_cfg<P_, Q_, KIND, 4, 3, true, false, true, false, true>(op, lidx, alpha, x, y, rg, s);   // "43fcx"
      case 42031:  // "42fnx"
        if (nd_hex_apply6_reads_nodes(op)) return launch6_cfg<P_, Q_, KIND, 4, 2, true, false, true, false, false, true>(op, lidx, alpha, x, y, rg, s);
        break;
      case 43031:  // "43fnx"
        if (nd_hex_apply6_reads_nodes(op)) return launch6_cfg<P_, Q_, KIND, 4, 3, true, false, true, false, false, true>(op, lidx, alpha, x, y, rg, s);
        break;
    }
  }
#endif
  if constexpr (P_ == 3 && KIND != B2P_ND_BLOCK)
  {
    if (nd_hex_apply6_reads_nodes(op))  // trilinear mesh: geometry from the vertices, no q-data stream
      return launch6_cfg<P_, Q_, KIND, ND6_NW, ND6_MINB, ND6_FWD, false, ND6_XLATE, true, false, true>(op, lidx, alpha, x, y, rg, s);
  }
  return launch6_cfg<P_, Q_, KIND, ND6_NW, ND6_MINB, ND6_FWD, ND6_GSM, ND6_XLATE, true>(op, lidx, alpha, x, y, rg, s, transpose);
}

}  // namespace

bool nd_hex_apply6_eligible(b2p_op *op)
{
  if (!op || op->dense || op->assembled || op->kind == B2P_H1_DIFFUSION || !(op->ecoef || op->bcoef)) return false;
  if (!(op->q1d == op->p + 1 && op->p >= 2 && op->p <= 3)) return false;
  return nd_tables_symmetric(op, 4e-16);  // the kernel substitutes mirrored entries: they must agree to round-off
}

// Node geometry for the symmetric kinds at p = 3 only. The block form is already at 253-255 registers on the stored q-data and
// spills with the 18 line sums of the vertex route; at p = 2 the symmetric kinds run on nd_hex_apply7_kernel unless
// B2P_ND_KERNEL=6 forces this kernel.
bool nd_hex_apply6_reads_nodes(const b2p_op *op) { return op->geom->xe && op->p == 3 && !op->bcoef; }

int launch_nd_hex_apply6(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                         bool transpose)
{
#define B2P_CASE(PP, QQ)                                                                                                  \
  if (op->p == PP && op->q1d == QQ)                                                                                       \
  {                                                                                                                       \
    if (op->bcoef) return launch6<PP, QQ, B2P_ND_BLOCK>(op, lidx, alpha, x, y, rg, s, transpose);                        \
    switch (op->kind)                                                                                                     \
    {                                                                                                                     \
      case B2P_CURLCURL: return launch6<PP, QQ, B2P_CURLCURL>(op, lidx, alpha, x, y, rg, s);                              \
      case B2P_ND_MASS: return launch6<PP, QQ, B2P_ND_MASS>(op, lidx, alpha, x, y, rg, s);                                \
      case B2P_CURLCURL_MASS: return launch6<PP, QQ, B2P_CURLCURL_MASS>(op, lidx, alpha, x, y, rg, s);                    \
    }                                                                                                                     \
  }
  B2P_CASE(3, 4)
#ifndef B2P_ND6_P3_ONLY
  B2P_CASE(2, 3)
#endif
#undef B2P_CASE
  set_error(op->ctx, "nd_hex_apply6: no kernel for p=%d q1d=%d kind=%d", op->p, op->q1d, op->kind);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace b2p
