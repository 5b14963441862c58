// High-order Nedelec hexahedron apply kernel: one CTA per element batch, one 1-D line per thread.
//
//   y_L += alpha * sum_e E_e^T  B^T  D  B  E_e x_L          (curl-curl, mass, curl-curl + mass),   p = 2 ... 6 at q1d = p + 1
// and, in the CPLX instantiations, the complex sum  (y_r + i y_i) += alpha * sum_e E_e^T B^T (D_r + i D_i) B E_e (x_r + i x_i)
// of a ComplexParOperator in one pass (both parts through the phases below, one after the other; DESIGN.md 4.3).
//
// Same operator as nd_hex_apply4_kernel. That kernel gives every WARP whole elements and keeps a (qy,qz) line of u, curl u
// in registers through the pointwise D; at p >= 5 a lane then owns several lines (q1d^2 = 36, 49 > 32), the kernel spills
// and 3-5 warps fit an SM (0.19 / 0.12 of the HBM roofline at p = 5 / 6); at p = 2, 3 its registers and shared memory
// hold it to 8 warps per SM, too few to hide the latency of its dependent FP64 chains.
// Here the CTA owns the batch and the warps are specialised by vector COMPONENT (x-, y-, z-directed dofs):
//   * every phase is a set of independent 1-D contractions ("lines"); a thread owns ONE line of its component, so
//     its live state is one input line, one or two output lines and the table entries in flight (<= 85 registers,
//     no spills, 4+ CTAs per SM);
//   * all threads of a warp run the same component, hence the same 1-D tables: the table entries are constant-bank
//     loads at compile-time offsets, mirrored entries are referenced through the stored half so the compiler
//     loads each value once for the two multiplies that use it;
//   * the index spaces are padded to q1d in every direction (the open directions have p entries: the extra
//     lanes idle), which makes every work array [row over the index the NEXT phase contracts][consumer's line id]:
//     the consumer reads consecutive words, the producer's stores are conflict-free with row strides = q1d (Z -> Y
//     arrays) or 1 (Y -> X arrays) modulo 16 words;
//   * the pointwise D runs one thread per quadrature point over values and curls in shared memory (6 doubles in,
//     6 out); the point order inside a batch is x-slowest, the order of the q-data in HBM, so its loads coalesce;
//   * persistent grid; the signed restriction indices of the NEXT batch are fetched into registers behind the Z phase,
//     its x values behind the X phase (both land while the transposed phases run).
// Phases per batch (a barrier between them, component-wide where the hand-off stays inside a component): Z, Y, X, D, Xt, Yt,
// Zt + scatter (RED.F64).
//
// Reference semantics: ceed::Operator::AddMult over CeedOperatorApplyAdd
// (/root/reference/palace/fem/libceed/operator.cpp:148-178,192-212); D from
// /root/reference/palace/fem/qfunctions/33/{hdiv,hcurl,hdivmass}_33_qf.h.
#include <cmath>
#include <cstdlib>
#include <type_traits>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_pipe.cuh"

namespace b2p
{

namespace
{

template <int P_>
struct ND7Params
{
  const int32_t *lidx;  // [ne][PS] signed lexicographic restriction (B2P_SKIP_IDX = masked / pad)
  const double *qd;     // [ne][10][Q] geometry, x-slowest point order
  const double *ecoef;  // [ne][18] per-element coefficient matrices (value part, derivative part)
  const double *x;
  double *y;
  double *sink;  // scratch for masked restriction entries (branch-free scatter)
  double alpha;
  int ne;
  VSplit sp;
  const unsigned long long *wait_flags, *wait_expect;  // peer-memory halo flags (SPLIT kernels only)
  int wait_n, wait_from_elem;
  int iso;
  double Bo[(P_ + 1) * P_];
  double Bc[(P_ + 1) * (P_ + 1)];
  double Gc[(P_ + 1) * (P_ + 1)];
};

// Complex apply (CPLX kernels): y_r + i y_i += alpha * E^T B^T (D_r + s i D_i) B E (x_r + i x_i), both parts in one pass.
// ecoef: {mass Re, mass Im, curl Re, curl Im} 3x3 tensors per element (symmetric kinds) or the real four-tensor block
// (B2P_ND_BLOCK, with ecoef_i the imaginary one); s = sgn (-1: Hermitian transpose, with the transposed blocks).
template <int P_>
struct ND7ParamsZ : ND7Params<P_>
{
  const double *xi, *ecoef_i;
  double *yi;
  double sgn;
  int has_imag;  // some coefficient has an imaginary part (otherwise the parts never mix)
};
template <int P_, bool CPLX>
using ND7ParamsT = std::conditional_t<CPLX, ND7ParamsZ<P_>, ND7Params<P_>>;

// smallest row stride >= len that is = res modulo 16 words (the 64-bit bank period of a half-warp)
constexpr int nd7_stride(int len, int res)
{
  int r = len;
  while ((r % 16) != (res % 16)) r++;
  return r;
}
constexpr int nd7_max(int a, int b) { return a > b ? a : b; }

template <int P_, int KIND, int NE, bool CPLX = false>
struct ND7Layout
{
  static constexpr int p = P_, q = P_ + 1, n = P_ + 1, QQ = q * q, Q = q * q * q, D3 = p * n * n, P = 3 * D3;
  static constexpr int PS = (P + 3) & ~3;
  // B2P_ND_BLOCK: the CURLCURL_MASS data flow with the four-tensor block of b2p_op::bcoef in the D phase
  static constexpr bool BLOCK = (KIND == B2P_ND_BLOCK);
  static constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS || BLOCK);
  static constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS || BLOCK);
  // coefficient doubles per element and array: two 3x3 tensors, four for the block form and for the complex symmetric kinds
  static constexpr int CEA = (BLOCK || CPLX) ? 36 : 18;
  static constexpr int CE = (BLOCK && CPLX) ? 2 * CEA : CEA;  // complex block form: the imaginary block at + NE CEA
  static constexpr int LQ = NE * QQ;  // line slots of one component (all index extents padded to q)
  // Z -> Y arrays (region A), rows j: written by the Z phase at (j, i + q qz), read by the Y phase along j
  static constexpr int RS1 = nd7_stride(LQ, q);
  static constexpr int A_XA = 0, A_XB = A_XA + n * RS1, A_YA = A_XB + (CURL ? n * RS1 : 0), A_YB = A_YA + p * RS1,
                       A_ZA = A_YB + (CURL ? p * RS1 : 0), A_ZY = A_ZA + n * RS1;
  // values and curls at the quadrature points (region A again): [component][qx][line (qy, qz)]
  static constexpr int A_U = 0, A_C = A_U + (MASS ? 3 * q * LQ : 0), A_QP = A_C + (CURL ? 3 * q * LQ : 0);
  static constexpr int SA = (nd7_max(A_ZY, A_QP) + 1) & ~1;
  // Y -> X arrays (region B), rows i: written by the Y phase at (i, qy + q qz), read by the X phase along i
  static constexpr int RS2 = nd7_stride(LQ, 1);
  static constexpr int B_X1 = 0, B_X2 = B_X1 + (MASS ? p * RS2 : 0), B_X3 = B_X2 + (CURL ? p * RS2 : 0),
                       B_Y1 = B_X3 + (CURL ? p * RS2 : 0), B_Y2 = B_Y1 + n * RS2, B_Z1 = B_Y2 + (CURL ? n * RS2 : 0),
                       B_Z3 = B_Z1 + n * RS2, SB = B_Z3 + (CURL ? n * RS2 : 0);
  // CPLX: the point arrays of the real part (region P, same layout as at A_U), which the imaginary part's Z -> Y arrays would overwrite
  static constexpr int OFF_P = SA + SB, SP = CPLX ? A_QP : 0;
  // GSM: q-data [NE][10][Q] and coefficient blocks [NE][CE] of the batch, staged by TMA bulk copies behind one mbarrier
  static constexpr int GE = 10 * Q, OFF_G = (OFF_P + SP + 1) & ~1, OFF_C = OFF_G + NE * GE, OFF_BAR = OFF_C + NE * CE;
  static_assert(GE % 2 == 0, "16-byte blocks for the bulk copies");
  static constexpr int SMEM_BYTES_LDG = (SA + SB) * 8, SMEM_BYTES_GSM = (OFF_BAR + 2) * 8;
};

// Scatter without a branch: masked entries (B2P_SKIP_IDX; idle lines and tail slots carry it too) add 0.0 to the
// thread's own slot of a scratch array.
template <bool SPLIT>
__device__ __forceinline__ void scatter7(double *y, const VSplit &sp, double *sink, int32_t gi, double v)
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

// NE elements per batch, WPC warps per component (3 WPC warps per CTA), MINB CTAs per SM.
// GSM: the batch's q-data and coefficient blocks are staged in shared memory by TMA bulk copies issued one batch ahead (as
// soon as the D phase of the previous batch has read the buffer); otherwise the D phase loads them with LDG.
// CBAR: the three hand-offs that stay inside one vector component (Z -> Y, Yt -> Zt, Zt -> next Z: producer and consumer lines
// belong to the same component's warps and its own work arrays) synchronise only that component's WPC warps (named barrier,
// __syncwarp() for one warp) instead of the CTA; the components may drift apart by a phase. The other four hand-offs cross
// components (X reads all three, the point arrays alias the Z -> Y arrays) and stay __syncthreads().
// CPLX: the batch's restriction, q-data and coefficient blocks are fetched once for both parts. Z, Y, X run for the real part
// (into region P) and then the imaginary part; D forms the geometric transform once per point and couples the parts; Xt, Yt,
// Zt + scatter run for the imaginary part (its point arrays alias the Z -> Y arrays) and then the real part.
template <int P_, int KIND, bool SPLIT, int NE, int WPC, int MINB, bool GSM, bool CBAR, bool CPLX = false>
__global__ void __launch_bounds__(3 * WPC * 32, MINB) nd_hex_apply7_kernel(const __grid_constant__ ND7ParamsT<P_, CPLX> prm)
{
  using L = ND7Layout<P_, KIND, NE, CPLX>;
  constexpr int p = L::p, q = L::q, n = L::n, QQ = L::QQ, Q = L::Q, D3 = L::D3, LQ = L::LQ, RS1 = L::RS1, RS2 = L::RS2;
  constexpr bool MASS = L::MASS, CURL = L::CURL;
  constexpr int NT = 3 * WPC * 32;
  constexpr int NPART = CPLX ? 2 : 1;
  static_assert(LQ <= WPC * 32, "one line per thread");
  static_assert(!CPLX || (GSM && !SPLIT), "complex apply: single partition, coefficients staged by TMA");
  constexpr int H = (q + 1) / 2;
// table entry (row c, column i) through the stored half (indices are compile-time constants after unrolling)
#define TBO(c, i) ((c) < H ? prm.Bo[(c) * p + (i)] : prm.Bo[(q - 1 - (c)) * p + (p - 1 - (i))])
#define TBC(c, i) ((c) < H ? prm.Bc[(c) * n + (i)] : prm.Bc[(q - 1 - (c)) * n + (n - 1 - (i))])
#define TGC(c, i) ((c) < H ? prm.Gc[(c) * n + (i)] : -prm.Gc[(q - 1 - (c)) * n + (n - 1 - (i))])

  B2P_DYN_SMEM_ALIGNED16(unsigned char, smem_raw);
  double *sA = (double *)smem_raw, *sB = sA + L::SA;
  double *sG = sA + L::OFF_G, *sC = sA + L::OFF_C;
  uint64_t *bar_g = (uint64_t *)(sA + L::OFF_BAR);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int comp = wid / WPC;                 // vector component of this warp
  const int tau = lane + 32 * (wid % WPC);    // line slot inside the component
  const bool slot_ok = tau < LQ;
  const int se = slot_ok ? tau / QQ : 0, sr = slot_ok ? tau % QQ : 0, sa = sr % q, sb = sr / q;  // slot = (element; a, b)
  // Z / Zt line (i, j) = (a, b) holds the dofs l0 + k ls, k < nk; Y / Yt line (i, qz) = (a, b); X / Xt line (qy, qz) = (a, b)
  const bool zv = slot_ok && (comp == 0 ? sa < p : comp == 1 ? sb < p : true);
  const bool yv = slot_ok && (comp == 0 ? sa < p : true);
  const int zl0 = comp == 0 ? sa + p * sb : comp == 1 ? D3 + sa + n * sb : 2 * D3 + sa + n * sb;
  const int zls = comp == 2 ? n * n : p * n;
  const int nk = comp == 2 ? p : n;

  const int nb = (prm.ne + NE - 1) / NE;  // element batches
  int b = blockIdx.x;
  griddep_launch_dependents();  // a dependent launched programmatically (the halo POST kernel) may be scheduled as CTAs retire
  if (b >= nb) return;
  double *my_sink = prm.sink + ((blockIdx.x * NT + tid) & (b2p_ctx::SINK_SLOTS - 1));
  auto comp_sync = [&]()
  {
#ifdef B2P_EMU
    __syncthreads();  // (the emulation has CTA barriers only: stricter, same results)
#else
    if (!CBAR)
      __syncthreads();
    else if (WPC == 1)
      __syncwarp();
    else
      asm volatile("bar.sync %0, %1;" ::"r"(comp + 1), "r"(WPC * 32) : "memory");
#endif
  };

  auto load_idx = [&](int bb, int32_t(&g)[n])
  {
    const int e = bb * NE + se;
    const bool ok = zv && e < prm.ne;
    const int32_t *row = prm.lidx + (size_t)(ok ? e : 0) * L::PS + zl0;
#pragma unroll
    for (int k = 0; k < n; k++) g[k] = (ok && k < nk) ? __ldg(row + k * zls) : (int32_t)B2P_SKIP_IDX;
  };
  auto load_x = [&](const int32_t(&g)[n], double(&v)[n])
  {
#pragma unroll
    for (int k = 0; k < n; k++)
    {
      const int32_t gk = g[k];
      if (gk == (int32_t)B2P_SKIP_IDX)
        v[k] = 0.0;
      else if (SPLIT)
        v[k] = __ldg(split_src_fast(prm.x, prm.sp, abs_idx(gk)));
      else
        v[k] = __ldg(prm.x + (uint32_t)abs_idx(gk));
    }
  };
  // Peer-memory halo: ghost values of this step are complete once every neighbour's flag reached the expected epoch.
  bool y_ready = false;  // the grid dependency (zero-fill of y / the halo PRE kernel under programmatic dependent launch) is resolved
  bool ghosts_ready = !(SPLIT && prm.wait_n > 0);
  auto ensure_ghosts = [&](int bb)  // (CTA-uniform)
  {
    if (ghosts_ready || (bb + 1) * NE <= prm.wait_from_elem) return;
    if (!y_ready)
    {
      griddep_wait();  // the expected epochs are advanced by the PRE kernel this grid may be overlapping
      y_ready = true;
    }
    if (tid < prm.wait_n)
    {
      const unsigned long long want = prm.wait_expect[tid];
      unsigned long long v;
      do
      {
        v = ld_acquire_sys_u64(prm.wait_flags + tid);
      } while (v < want);
    }
    __syncthreads();
    ghosts_ready = true;
  };

  auto issue_geom = [&](int bb)  // (one thread)
  {
    const uint64_t once = l2_evict_first_policy();  // q-data and coefficient blocks are read once per launch
    const int e0 = bb * NE, nel = min(NE, prm.ne - e0);
    mbar_expect_tx(bar_g, (uint32_t)(nel * (L::GE + L::CE) * sizeof(double)));
    tma_bulk_g2s_hint(sG, prm.qd + (size_t)e0 * L::GE, (uint32_t)(nel * L::GE * sizeof(double)), bar_g, once);
    if constexpr (CPLX && L::BLOCK)
    {
      tma_bulk_g2s_hint(sC, prm.ecoef + (size_t)e0 * L::CEA, (uint32_t)(nel * L::CEA * sizeof(double)), bar_g, once);
      tma_bulk_g2s_hint(sC + NE * L::CEA, prm.ecoef_i + (size_t)e0 * L::CEA, (uint32_t)(nel * L::CEA * sizeof(double)), bar_g, once);
    }
    else
      tma_bulk_g2s_hint(sC, prm.ecoef + (size_t)e0 * L::CE, (uint32_t)(nel * L::CE * sizeof(double)), bar_g, once);
  };
  uint32_t par_g = 0;
  if (GSM)
  {
    if (tid == 0)
    {
      mbar_init(bar_g, 1);
      issue_geom(b);
    }
    __syncthreads();  // (the barrier object is initialised before anyone polls it)
  }

  int32_t gi[n], ngi[n];
  double xv[n], xvi[n];  // gathered x (real part; CPLX: imaginary part, fetched behind the real part's Z phase)
  auto load_xi = [&](const int32_t(&g)[n])
  {
    if constexpr (CPLX)
    {
#pragma unroll
      for (int k = 0; k < n; k++) xvi[k] = g[k] == (int32_t)B2P_SKIP_IDX ? 0.0 : __ldg(prm.xi + (uint32_t)abs_idx(g[k]));
    }
  };
  load_idx(b, gi);
  ensure_ghosts(b);
  load_x(gi, xv);
#pragma unroll
  for (int k = 0; k < n; k++) ngi[k] = (int32_t)B2P_SKIP_IDX;

  const double alpha = prm.alpha;
  for (; b < nb; b += gridDim.x)
  {
    const int bn = b + gridDim.x;
    const bool has_next = bn < nb;
    const int e0 = b * NE, nel = min(NE, prm.ne - e0);

#pragma unroll
    for (int part = 0; part < NPART; part++)
    {
    // ------------------------------------------------------------------ phase Z (contract k -> qz)
    if (zv)
    {
      double xs[n];
#pragma unroll
      for (int k = 0; k < n; k++) xs[k] = gi[k] < 0 ? -((CPLX && part) ? xvi[k] : xv[k]) : ((CPLX && part) ? xvi[k] : xv[k]);
      double *oa = sA + sb * RS1 + se * QQ + sa;  // + q qz
      if (comp < 2)
      {
        oa += comp == 0 ? L::A_XA : L::A_YA;
        constexpr int DB = CURL ? L::A_XB - L::A_XA : 0;  // (same distance for the y-directed pair)
        static_assert(!CURL || L::A_YB - L::A_YA == p * RS1, "layout");
        const int db = comp == 0 ? DB : p * RS1;
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          double v = 0.0, d = 0.0;
#pragma unroll
          for (int k = 0; k < n; k++)
          {
            v += TBC(qz, k) * xs[k];
            if (CURL) d += TGC(qz, k) * xs[k];
          }
          oa[q * qz] = v;
          if (CURL) oa[db + q * qz] = d;
        }
      }
      else
      {
        oa += L::A_ZA;
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          double v = 0.0;
#pragma unroll
          for (int k = 0; k < p; k++) v += TBO(qz, k) * xs[k];
          oa[q * qz] = v;
        }
      }
    }
    if (CPLX && part == 0) load_xi(gi);  // lands while the real part's Y and X run
    if (has_next && part == 0) load_idx(bn, ngi);
    comp_sync();

    // ------------------------------------------------------------------ phase Y (contract j -> qy)
    if (yv)
    {
      double *ob = sB + sa * RS2 + se * QQ + q * sb;  // + qy
      if (comp == 0)
      {
        double a[n], g[n];
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          a[j] = sA[L::A_XA + j * RS1 + tau];
          if (CURL) g[j] = sA[L::A_XB + j * RS1 + tau];
        }
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          double v1 = 0.0, v2 = 0.0, v3 = 0.0;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            if (MASS) v1 += TBC(qy, j) * a[j];
            if (CURL) v2 += TGC(qy, j) * a[j];
            if (CURL) v3 += TBC(qy, j) * g[j];
          }
          if (MASS) ob[L::B_X1 + qy] = v1;
          if (CURL) ob[L::B_X2 + qy] = v2;
          if (CURL) ob[L::B_X3 + qy] = v3;
        }
      }
      else if (comp == 1)
      {
        double a[p], g[p];
#pragma unroll
        for (int j = 0; j < p; j++)
        {
          a[j] = sA[L::A_YA + j * RS1 + tau];
          if (CURL) g[j] = sA[L::A_YB + j * RS1 + tau];
        }
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          double v1 = 0.0, v2 = 0.0;
#pragma unroll
          for (int j = 0; j < p; j++)
          {
            v1 += TBO(qy, j) * a[j];
            if (CURL) v2 += TBO(qy, j) * g[j];
          }
          ob[L::B_Y1 + qy] = v1;
          if (CURL) ob[L::B_Y2 + qy] = v2;
        }
      }
      else
      {
        double a[n];
#pragma unroll
        for (int j = 0; j < n; j++) a[j] = sA[L::A_ZA + j * RS1 + tau];
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          double v1 = 0.0, v3 = 0.0;
#pragma unroll
          for (int j = 0; j < n; j++)
          {
            v1 += TBC(qy, j) * a[j];
            if (CURL) v3 += TGC(qy, j) * a[j];
          }
          ob[L::B_Z1 + qy] = v1;
          if (CURL) ob[L::B_Z3 + qy] = v3;
        }
      }
    }
    __syncthreads();

    // ------------------------------------------------------------------ phase X (contract i -> qx): u_c and (curl u)_c
    //   curl_x = dy uz - dz uy = Bc (Z3 - Y2),  curl_y = dz ux - dx uz = Bo X3 - Gc Z1,  curl_z = dx uy - dy ux = Gc Y1 - Bo X2
    if (slot_ok)
    {
      double *const sX = (CPLX && part == 0) ? sA + L::OFF_P : sA;  // point arrays of this part
      double *ou = sX + L::A_U + comp * q * LQ + tau;  // + qx LQ
      double *oc = sX + L::A_C + comp * q * LQ + tau;
      const double *in = sB + tau;  // + array + i RS2
      if (comp == 0)
      {
        if (MASS)
        {
          double a[p];
#pragma unroll
          for (int i = 0; i < p; i++) a[i] = in[L::B_X1 + i * RS2];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            double v = 0.0;
#pragma unroll
            for (int i = 0; i < p; i++) v += TBO(qx, i) * a[i];
            ou[qx * LQ] = v;
          }
        }
        if (CURL)
        {
          double d[n];
#pragma unroll
          for (int i = 0; i < n; i++) d[i] = in[L::B_Z3 + i * RS2] - in[L::B_Y2 + i * RS2];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            double v = 0.0;
#pragma unroll
            for (int i = 0; i < n; i++) v += TBC(qx, i) * d[i];
            oc[qx * LQ] = v;
          }
        }
      }
      else
      {
        // y-directed: u_y = Bc Y1, curl_y = Bo X3 - Gc Z1 ; z-directed: u_z = Bc Z1, curl_z = Gc Y1 - Bo X2
        const int o_val = comp == 1 ? L::B_Y1 : L::B_Z1, o_der = comp == 1 ? L::B_Z1 : L::B_Y1, o_opn = comp == 1 ? L::B_X3 : L::B_X2;
        const double sg = comp == 1 ? 1.0 : -1.0;
        if (MASS)
        {
          double a[n];
#pragma unroll
          for (int i = 0; i < n; i++) a[i] = in[o_val + i * RS2];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            double v = 0.0;
#pragma unroll
            for (int i = 0; i < n; i++) v += TBC(qx, i) * a[i];
            ou[qx * LQ] = v;
          }
        }
        if (CURL)
        {
          double f[n], o[p];
#pragma unroll
          for (int i = 0; i < n; i++) f[i] = -sg * in[o_der + i * RS2];
#pragma unroll
          for (int i = 0; i < p; i++) o[i] = sg * in[o_opn + i * RS2];
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            double v = 0.0;
#pragma unroll
            for (int i = 0; i < n; i++) v += TGC(qx, i) * f[i];
#pragma unroll
            for (int i = 0; i < p; i++) v += TBO(qx, i) * o[i];
            oc[qx * LQ] = v;
          }
        }
      }
    }
    __syncthreads();
    }
    if (has_next)
    {
      ensure_ghosts(bn);
      load_x(ngi, xv);  // lands while the transposed phases run
    }

    // ------------------------------------------------------------------ phase D (one thread per quadrature point, in place)
    if (GSM)
    {
      mbar_wait(bar_g, par_g);
      par_g ^= 1u;
    }
#pragma unroll 1
    for (int iota = tid; iota < NE * Q; iota += NT)
    {
      const int qx = iota / LQ, t = iota % LQ, e = t / QQ, rr = t % QQ;
      if (e >= nel) continue;  // (tail slots hold zeros)
      const double *g = GSM ? sG + e * L::GE + qx * QQ + rr : prm.qd + (size_t)(e0 + e) * L::GE + qx * QQ + rr;
      if constexpr (CPLX)
      {
        // t = A u (value), sc = Jd c (curl) for both parts; then per part  out_val = Cm t + Cx sc,  out_curl = Ck sc + Cw t with
        // C = C_r on the own part and s C_i on the other (real part: - s C_i t_i, imaginary part: + s C_i t_r)
        const double *Cr = sC + e * L::CEA;
        const double *Ci = L::BLOCK ? Cr + NE * L::CEA : Cr + 9;  // symmetric kinds: {mass Re, mass Im, curl Re, curl Im}
        constexpr int OK = L::BLOCK ? 9 : 18;                     // curl tensor
        const double wdetJ = alpha * g[0];
        double A[9], Jd[9], t[2][3], sc[2][3];
#pragma unroll
        for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
        if (CURL) cofactor33(A, Jd);
        double *pp[2] = {sA + L::OFF_P + iota, sA + iota};
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
          double u[3];
#pragma unroll
          for (int r3 = 0; r3 < 3; r3++) u[r3] = pp[h][L::A_U + r3 * NE * Q];
          if (MASS) Ax33(A, u, t[h]);
#pragma unroll
          for (int r3 = 0; r3 < 3; r3++) u[r3] = pp[h][L::A_C + r3 * NE * Q];
          if (CURL) Ax33(Jd, u, sc[h]);
        }
        // v += f (Cm t + Cx sc), w += f (Ck sc + Cw t)
        auto couple = [&](const double *Cp, const double(&tt)[3], const double(&ss)[3], double f, double(&v)[3], double(&w)[3])
        {
          double a[3];
          if (MASS)
          {
            Ax33(Cp, tt, a);
#pragma unroll
            for (int r = 0; r < 3; r++) v[r] += f * a[r];
          }
          if (CURL)
          {
            Ax33(Cp + OK, ss, a);
#pragma unroll
            for (int r = 0; r < 3; r++) w[r] += f * a[r];
          }
          if (L::BLOCK)
          {
            Ax33(Cp + 27, ss, a);
#pragma unroll
            for (int r = 0; r < 3; r++) v[r] += f * a[r];
            Ax33(Cp + 18, tt, a);
#pragma unroll
            for (int r = 0; r < 3; r++) w[r] += f * a[r];
          }
        };
        const double sg = prm.sgn;
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
          double v[3] = {0.0, 0.0, 0.0}, w[3] = {0.0, 0.0, 0.0}, o[3];
          couple(Cr, t[h], sc[h], 1.0, v, w);
          if (prm.has_imag) couple(Ci, t[1 - h], sc[1 - h], h ? sg : -sg, v, w);
          if (MASS)
          {
            Atx33(A, v, wdetJ, o);
#pragma unroll
            for (int r3 = 0; r3 < 3; r3++) pp[h][L::A_U + r3 * NE * Q] = o[r3];
          }
          if (CURL)
          {
            Atx33(Jd, w, wdetJ, o);
#pragma unroll
            for (int r3 = 0; r3 < 3; r3++) pp[h][L::A_C + r3 * NE * Q] = o[r3];
          }
        }
        continue;
      }
      const double *C = GSM ? sC + e * L::CE : prm.ecoef + (size_t)(e0 + e) * L::CE;
      double A[9], Cm[9], wdetJ, cm0, cc0;
      if (GSM)
      {
        wdetJ = alpha * g[0];  // alpha folded into the quadrature weight
#pragma unroll
        for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
        cm0 = C[0];
        cc0 = C[9];
      }
      else
      {
        wdetJ = alpha * __ldg(g);
#pragma unroll
        for (int i = 0; i < 9; i++) A[i] = __ldg(g + (1 + i) * Q);
        cm0 = __ldg(C);
        cc0 = __ldg(C + 9);
      }
      double *pu = sA + L::A_U + iota, *pc = sA + L::A_C + iota;  // + component * NE Q
      double u[3], c[3], v[3], cw[3];
#pragma unroll
      for (int r3 = 0; r3 < 3; r3++)
      {
        if (MASS) u[r3] = pu[r3 * NE * Q];
        if (CURL) c[r3] = pc[r3 * NE * Q];
      }
      if constexpr (L::BLOCK)
      {
        // out_val = w A^T (Cm A u + Cx Jd c),  out_curl = w Jd^T (Ck Jd c + Cw A u)
        double Jd[9], Ck[9], Cw[9], Cx[9], t[3], sc[3], a[3], b[3], z[3];
#pragma unroll
        for (int i = 0; i < 9; i++)
        {
          Cm[i] = GSM ? C[i] : __ldg(C + i);
          Ck[i] = GSM ? C[9 + i] : __ldg(C + 9 + i);
          Cw[i] = GSM ? C[18 + i] : __ldg(C + 18 + i);
          Cx[i] = GSM ? C[27 + i] : __ldg(C + 27 + i);
        }
        cofactor33(A, Jd);
        Ax33(A, u, t);
        Ax33(Jd, c, sc);
        Ax33(Cm, t, a);
        Ax33(Cx, sc, b);
#pragma unroll
        for (int r = 0; r < 3; r++) z[r] = a[r] + b[r];
        Atx33(A, z, wdetJ, v);
        Ax33(Ck, sc, a);
        Ax33(Cw, t, b);
#pragma unroll
        for (int r = 0; r < 3; r++) z[r] = a[r] + b[r];
        Atx33(Jd, z, wdetJ, cw);
      }
      else if (prm.iso)
      {
        if (MASS) AtAx(A, u, wdetJ * cm0, v);
        if (CURL)
        {
          double Jd[9];
          cofactor33(A, Jd);
          AtAx(Jd, c, wdetJ * cc0, cw);
        }
      }
      else
      {
        if (MASS)
        {
#pragma unroll
          for (int i = 0; i < 9; i++) Cm[i] = GSM ? C[i] : __ldg(C + i);
          AtCAx(A, Cm, u, wdetJ, v);
        }
        if (CURL)
        {
          double Jd[9];
#pragma unroll
          for (int i = 0; i < 9; i++) Cm[i] = GSM ? C[9 + i] : __ldg(C + 9 + i);
          cofactor33(A, Jd);
          AtCAx(Jd, Cm, c, wdetJ, cw);
        }
      }
#pragma unroll
      for (int r3 = 0; r3 < 3; r3++)
      {
        if (MASS) pu[r3 * NE * Q] = v[r3];
        if (CURL) pc[r3 * NE * Q] = cw[r3];
      }
    }
    __syncthreads();
    if (GSM && has_next && tid == 0)
    {
      fence_proxy_async();  // the D phase's reads of the staging buffer are ordered before the bulk copy that refills it
      issue_geom(bn);
    }

#pragma unroll
    for (int part = NPART - 1; part >= 0; part--)
    {
    // ------------------------------------------------------------------ phase Xt (transposed x-contraction)
    //   X1' = Bo^T w_x, X2' = -Bo^T cw_z, X3' = Bo^T cw_y ; Y1' = Bc^T w_y + Gc^T cw_z, Y2' = -Bc^T cw_x ;
    //   Z1' = Bc^T w_z - Gc^T cw_y, Z3' = Bc^T cw_x
    if (slot_ok)
    {
      const double *const sX = (CPLX && part == 0) ? sA + L::OFF_P : sA;
      const double *wu = sX + L::A_U + tau, *wc = sX + L::A_C + tau;  // + (component q + qx) LQ
      double *out = sB + tau;                                          // + array + i RS2
      if (comp == 0)
      {
        double w[q], cy[q], cz[q];
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) w[qx] = wu[(0 * q + qx) * LQ];
          if (CURL) cy[qx] = wc[(1 * q + qx) * LQ];
          if (CURL) cz[qx] = wc[(2 * q + qx) * LQ];
        }
#pragma unroll
        for (int i = 0; i < p; i++)
        {
          double v1 = 0.0, v2 = 0.0, v3 = 0.0;
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) v1 += TBO(qx, i) * w[qx];
            if (CURL) v2 -= TBO(qx, i) * cz[qx];
            if (CURL) v3 += TBO(qx, i) * cy[qx];
          }
          if (MASS) out[L::B_X1 + i * RS2] = v1;
          if (CURL) out[L::B_X2 + i * RS2] = v2;
          if (CURL) out[L::B_X3 + i * RS2] = v3;
        }
      }
      else
      {
        // y-directed: Y1' = Bc^T w_y + Gc^T cw_z, Y2' = -Bc^T cw_x ; z-directed: Z1' = Bc^T w_z - Gc^T cw_y, Z3' = Bc^T cw_x
        const int o_1 = comp == 1 ? L::B_Y1 : L::B_Z1, o_2 = comp == 1 ? L::B_Y2 : L::B_Z3;
        const double sg = comp == 1 ? 1.0 : -1.0;
        double w[q], cg[q], cx[q];
#pragma unroll
        for (int qx = 0; qx < q; qx++)
        {
          if (MASS) w[qx] = wu[(comp * q + qx) * LQ];
          if (CURL) cg[qx] = sg * wc[((3 - comp) * q + qx) * LQ];  // y-directed: +cw_z, z-directed: -cw_y
          if (CURL) cx[qx] = -sg * wc[(0 * q + qx) * LQ];          // y-directed: -cw_x, z-directed: +cw_x
        }
#pragma unroll
        for (int i = 0; i < n; i++)
        {
          double v1 = 0.0, v2 = 0.0;
#pragma unroll
          for (int qx = 0; qx < q; qx++)
          {
            if (MASS) v1 += TBC(qx, i) * w[qx];
            if (CURL) v1 += TGC(qx, i) * cg[qx];
            if (CURL) v2 += TBC(qx, i) * cx[qx];
          }
          out[o_1 + i * RS2] = v1;
          if (CURL) out[o_2 + i * RS2] = v2;
        }
      }
    }
    __syncthreads();

    // ------------------------------------------------------------------ phase Yt (transposed y-contraction)
    if (yv)
    {
      const double *in = sB + sa * RS2 + se * QQ + q * sb;  // + array + qy
      double *out = sA + tau;                               // + array + j RS1
      if (comp == 0)
      {
        double a[q], b2[q], b3[q];
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          if (MASS) a[qy] = in[L::B_X1 + qy];
          if (CURL) b2[qy] = in[L::B_X2 + qy];
          if (CURL) b3[qy] = in[L::B_X3 + qy];
        }
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          double v = 0.0, d = 0.0;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            if (MASS) v += TBC(qy, j) * a[qy];
            if (CURL) v += TGC(qy, j) * b2[qy];
            if (CURL) d += TBC(qy, j) * b3[qy];
          }
          out[L::A_XA + j * RS1] = v;
          if (CURL) out[L::A_XB + j * RS1] = d;
        }
      }
      else if (comp == 1)
      {
        double a[q], g[q];
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          a[qy] = in[L::B_Y1 + qy];
          if (CURL) g[qy] = in[L::B_Y2 + qy];
        }
#pragma unroll
        for (int j = 0; j < p; j++)
        {
          double v = 0.0, d = 0.0;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            v += TBO(qy, j) * a[qy];
            if (CURL) d += TBO(qy, j) * g[qy];
          }
          out[L::A_YA + j * RS1] = v;
          if (CURL) out[L::A_YB + j * RS1] = d;
        }
      }
      else
      {
        double a[q], g[q];
#pragma unroll
        for (int qy = 0; qy < q; qy++)
        {
          a[qy] = in[L::B_Z1 + qy];
          if (CURL) g[qy] = in[L::B_Z3 + qy];
        }
#pragma unroll
        for (int j = 0; j < n; j++)
        {
          double v = 0.0;
#pragma unroll
          for (int qy = 0; qy < q; qy++)
          {
            v += TBC(qy, j) * a[qy];
            if (CURL) v += TGC(qy, j) * g[qy];
          }
          out[L::A_ZA + j * RS1] = v;
        }
      }
    }
    comp_sync();

    // ------------------------------------------------------------------ phase Zt (transposed z-contraction) + scatter
    if (!y_ready)
    {
      griddep_wait();
      y_ready = true;
    }
    if (zv)
    {
      double *yp = prm.y;
      if constexpr (CPLX) yp = part == 1 ? prm.yi : prm.y;
      const double *in = sA + sb * RS1 + se * QQ + sa;  // + array + q qz
      if (comp < 2)
      {
        const int o_a = comp == 0 ? L::A_XA : L::A_YA, o_b = comp == 0 ? L::A_XB : L::A_YB;
        double a[q], g[q];
#pragma unroll
        for (int qz = 0; qz < q; qz++)
        {
          a[qz] = in[o_a + q * qz];
          if (CURL) g[qz] = in[o_b + q * qz];
        }
#pragma unroll
        for (int k = 0; k < n; k++)
        {
          double v = 0.0;
#pragma unroll
          for (int qz = 0; qz < q; qz++)
          {
            v += TBC(qz, k) * a[qz];
            if (CURL) v += TGC(qz, k) * g[qz];
          }
          scatter7<SPLIT>(yp, prm.sp, my_sink, gi[k], v);
        }
      }
      else
      {
        double a[q];
#pragma unroll
        for (int qz = 0; qz < q; qz++) a[qz] = in[L::A_ZA + q * qz];
#pragma unroll
        for (int k = 0; k < p; k++)
        {
          double v = 0.0;
#pragma unroll
          for (int qz = 0; qz < q; qz++) v += TBO(qz, k) * a[qz];
          scatter7<SPLIT>(yp, prm.sp, my_sink, gi[k], v);
        }
      }
    }
    if (part == 0)
    {
#pragma unroll
      for (int k = 0; k < n; k++) gi[k] = ngi[k];
    }
    comp_sync();  // the next batch's Z phase (CPLX: the real part's Yt) overwrites the arrays Zt has just read
    }
  }
#undef TBO
#undef TBC
#undef TGC
}

// Launch shape per order: elements per batch, warps per component, CTAs per SM (register cap 65536 / threads per SM), q-data
// staged by TMA, component-wide barriers; chosen by A/B timing of the shapes (tools/nd7_ab.py, B2P_ND7_CFG). MINB_BLOCK is the
// CTAs per SM of the B2P_ND_BLOCK instantiation, whose four-tensor D phase needs more registers than the cap of MINB allows at
// p = 2, 3. MINB_CPLX is that of the complex instantiations (both parts' gathered x live across the batch, and the D phase
// holds both parts' values and curls), chosen so that none spills.
template <int P_>
struct ND7Shape;
template <>
struct ND7Shape<2>
{
  static constexpr int NE = 3, WPC = 1, MINB = 8, MINB_BLOCK = 4, MINB_CPLX = 4;  // 27 of 32 lanes, 96 threads
  static constexpr bool GSM = true, CBAR = true;
};
template <>
struct ND7Shape<3>
{
  static constexpr int NE = 2, WPC = 1, MINB = 8, MINB_BLOCK = 5, MINB_CPLX = 4;  // 32 of 32 lanes, 96 threads
  static constexpr bool GSM = true, CBAR = true;
};
template <>
struct ND7Shape<4>
{
  static constexpr int NE = 1, WPC = 1, MINB = 8, MINB_BLOCK = MINB, MINB_CPLX = 4;  // 25 of 32 lanes, 96 threads
  static constexpr bool GSM = true, CBAR = true;
};
template <>
struct ND7Shape<5>
{
  static constexpr int NE = 2, WPC = 3, MINB = 2, MINB_BLOCK = MINB, MINB_CPLX = 1;  // 72 of 96 lanes, 288 threads
  static constexpr bool GSM = true, CBAR = true;
};
template <>
struct ND7Shape<6>
{
  static constexpr int NE = 1, WPC = 2, MINB = 3, MINB_BLOCK = MINB, MINB_CPLX = 2;  // 49 of 64 lanes, 192 threads
  static constexpr bool GSM = true, CBAR = true;
};

template <int P_, int KIND, int NE, int WPC, int MINB, bool GSM, bool CBAR>
int launch7_cfg(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                bool transpose = false)
{
  using L = ND7Layout<P_, KIND, NE>;
  constexpr int NT = 3 * WPC * 32;
  const size_t shmem = GSM ? L::SMEM_BYTES_GSM : L::SMEM_BYTES_LDG;
  const bool split = range_split(op, rg);
  auto kern = split ? nd_hex_apply7_kernel<P_, KIND, true, NE, WPC, MINB, GSM, CBAR> : nd_hex_apply7_kernel<P_, KIND, false, NE, WPC, MINB, GSM, CBAR>;
  const int e_off = rg.e_off, e_cnt = range_count(op, rg);
  if (e_cnt <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  ND7Params<P_> prm;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
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
  copy_tables(op->h_tab.data(), P_, P_ + 1, P_ + 1, prm.Bo, prm.Bc, prm.Gc);
  const int nb = (e_cnt + NE - 1) / NE;
  return launch_persistent(kern, prm, NT, shmem, s, rg.pdl, op->ctx, "nd_hex_apply7_kernel", L::BLOCK, false, op->ctx->sm_count * MINB, 1, NE,
                           nb);
}

// Complex apply: one launch for both parts (see ND7ParamsZ); `op` supplies geometry, restriction and tables.
template <int P_, int KIND>
int launch7z(b2p_op *op, const int32_t *lidx, const double *coef, const double *coef_i, int has_imag, double sgn, double alpha,
             const double *xr, const double *xi, double *yr, double *yi, cudaStream_t s)
{
  using S = ND7Shape<P_>;
  using L = ND7Layout<P_, KIND, S::NE, true>;
  constexpr int NT = 3 * S::WPC * 32;
  constexpr size_t shmem = L::SMEM_BYTES_GSM;
  auto kern = nd_hex_apply7_kernel<P_, KIND, false, S::NE, S::WPC, S::MINB_CPLX, true, S::CBAR, true>;
  if (op->ne <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  ND7ParamsZ<P_> prm;
  prm.lidx = lidx;
  prm.qd = op->geom->qd;
  prm.ecoef = coef;
  prm.ecoef_i = coef_i;
  prm.x = xr;
  prm.xi = xi;
  prm.y = yr;
  prm.yi = yi;
  prm.sink = op->ctx->d_sink;
  prm.alpha = alpha;
  prm.sgn = sgn;
  prm.has_imag = has_imag;
  prm.ne = op->ne;
  set_split_wait(prm, op, ApplyRange());
  prm.iso = 0;
  copy_tables(op->h_tab.data(), P_, P_ + 1, P_ + 1, prm.Bo, prm.Bc, prm.Gc);
  const int nb = (op->ne + S::NE - 1) / S::NE;
  return launch_persistent(kern, prm, NT, shmem, s, false, op->ctx, "nd_hex_apply7_kernel", L::BLOCK, true, op->ctx->sm_count * S::MINB_CPLX, 1,
                           S::NE, nb);
}

// B2P_ND7_CFG = "<elements per batch><warps per component><CTAs per SM><d | g | c>" picks another launch shape of the
// curl-curl + mass kernel without owned | ghost split (d: q-data by LDG in the D phase, g: staged by TMA, c: staged by TMA and
// component-wide barriers): A/B measurements
// (tools/nd7_ab.py switches it inside one process, so it is read per launch).
inline int nd7_cfg_code()
{
  const char *e = std::getenv("B2P_ND7_CFG");
  if (!e || !e[0] || !e[1] || !e[2] || !e[3]) return -1;
  return (e[0] - '0') * 1000 + (e[1] - '0') * 100 + (e[2] - '0') * 10 + (e[3] == 'c' ? 2 : e[3] == 'g' ? 1 : 0);
}

template <int P_, int KIND>
int launch7(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
            bool transpose = false)
{
  using S = ND7Shape<P_>;
  if constexpr (KIND == B2P_CURLCURL_MASS)
  {
    const bool split = rg.xg || rg.yg || (rg.n_owned >= 0 && rg.n_owned < op->lsize);
    const int code = split ? -1 : nd7_cfg_code();
#define B2P_CFG(PP, NEV, WPCV, MB)                                                                                       \
  if (P_ == PP && code / 10 == NEV * 100 + WPCV * 10 + MB)                                                               \
    return (code % 10) == 2   ? launch7_cfg<P_, KIND, NEV, (P_ == PP ? WPCV : S::WPC), MB, true, true>(op, lidx, alpha, x, y, rg, s)   \
           : (code % 10) == 1 ? launch7_cfg<P_, KIND, NEV, (P_ == PP ? WPCV : S::WPC), MB, true, false>(op, lidx, alpha, x, y, rg, s)  \
                              : launch7_cfg<P_, KIND, NEV, (P_ == PP ? WPCV : S::WPC), MB, false, false>(op, lidx, alpha, x, y, rg, s);
    if constexpr (P_ == 2)
    {
      B2P_CFG(2, 3, 1, 7) B2P_CFG(2, 3, 1, 8) B2P_CFG(2, 3, 1, 9) B2P_CFG(2, 7, 2, 4)
    }
    if constexpr (P_ == 3)
    {
      B2P_CFG(3, 2, 1, 7) B2P_CFG(3, 2, 1, 8) B2P_CFG(3, 2, 1, 9) B2P_CFG(3, 3, 2, 4) B2P_CFG(3, 4, 2, 4)
    }
    if constexpr (P_ == 4)
    {
      B2P_CFG(4, 1, 1, 6) B2P_CFG(4, 1, 1, 8) B2P_CFG(4, 2, 2, 4) B2P_CFG(4, 5, 4, 2)
    }
    if constexpr (P_ == 5)
    {
      B2P_CFG(5, 2, 3, 1) B2P_CFG(5, 2, 3, 2) B2P_CFG(5, 3, 4, 1) B2P_CFG(5, 3, 4, 2)
    }
    if constexpr (P_ == 6)
    {
      B2P_CFG(6, 1, 2, 2) B2P_CFG(6, 1, 2, 3) B2P_CFG(6, 2, 4, 1) B2P_CFG(6, 2, 4, 2)
    }
#undef B2P_CFG
  }
  constexpr int MINB = KIND == B2P_ND_BLOCK ? S::MINB_BLOCK : S::MINB;
  return launch7_cfg<P_, KIND, S::NE, S::WPC, MINB, S::GSM, S::CBAR>(op, lidx, alpha, x, y, rg, s, transpose);
}

}  // namespace

bool nd_hex_apply7_eligible(b2p_op *op)
{
  if (!op || op->dense || op->assembled || op->kind == B2P_H1_DIFFUSION || !(op->ecoef || op->bcoef)) return false;
  if (!(op->q1d == op->p + 1 && op->p >= 2 && op->p <= 6)) return false;
  // The kernel reads mirrored table entries through one stored value. Tables evaluated in floating point (MFEM's, or
  // tests/hexspace.py) mirror to a few ulp of the LARGEST entry (measured 6e-16 ... 9e-16 at p = 4, 5): the substitution
  // changes the operator by less than the tables' own rounding.
  return nd_tables_symmetric(op, 8e-15);
}

int launch_nd_hex_apply7(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                         bool transpose)
{
#define B2P_CASE(PP)                                                                                                  \
  if (op->p == PP && op->q1d == PP + 1)                                                                               \
  {                                                                                                                   \
    if (op->bcoef) return launch7<PP, B2P_ND_BLOCK>(op, lidx, alpha, x, y, rg, s, transpose);                        \
    switch (op->kind)                                                                                                 \
    {                                                                                                                 \
      case B2P_CURLCURL: return launch7<PP, B2P_CURLCURL>(op, lidx, alpha, x, y, rg, s);                              \
      case B2P_ND_MASS: return launch7<PP, B2P_ND_MASS>(op, lidx, alpha, x, y, rg, s);                                \
      case B2P_CURLCURL_MASS: return launch7<PP, B2P_CURLCURL_MASS>(op, lidx, alpha, x, y, rg, s);                    \
    }                                                                                                                 \
  }
  B2P_CASE(2)
  B2P_CASE(3)
  B2P_CASE(4)
  B2P_CASE(5)
  B2P_CASE(6)
#undef B2P_CASE
  set_error(op->ctx, "nd_hex_apply7: no kernel for p=%d q1d=%d kind=%d", op->p, op->q1d, op->kind);
  return B2P_ERR_UNSUPPORTED;
}

int launch_nd_hex_apply7z(b2p_op *op, int kind, const int32_t *lidx, const double *coef, const double *coef_i, int has_imag, double sgn,
                          double alpha, const double *xr, const double *xi, double *yr, double *yi, cudaStream_t s)
{
#define B2P_ZARGS op, lidx, coef, coef_i, has_imag, sgn, alpha, xr, xi, yr, yi, s
  // block sums at p = 2 ... 6; symmetric kinds at p = 4, 5, 6 (p = 2, 3 run nd_hex_apply4_kernel<..., CPLX>)
#define B2P_BLOCK(PP) \
  if (op->p == PP && op->q1d == PP + 1 && kind == B2P_ND_BLOCK) return launch7z<PP, B2P_ND_BLOCK>(B2P_ZARGS);
#define B2P_SYM(PP)                                                                     \
  if (op->p == PP && op->q1d == PP + 1)                                                 \
  {                                                                                     \
    switch (kind)                                                                       \
    {                                                                                   \
      case B2P_CURLCURL: return launch7z<PP, B2P_CURLCURL>(B2P_ZARGS);                  \
      case B2P_ND_MASS: return launch7z<PP, B2P_ND_MASS>(B2P_ZARGS);                    \
      case B2P_CURLCURL_MASS: return launch7z<PP, B2P_CURLCURL_MASS>(B2P_ZARGS);        \
    }                                                                                   \
  }
  B2P_BLOCK(2) B2P_BLOCK(3) B2P_BLOCK(4) B2P_BLOCK(5) B2P_BLOCK(6)
  B2P_SYM(4) B2P_SYM(5) B2P_SYM(6)
#undef B2P_BLOCK
#undef B2P_SYM
#undef B2P_ZARGS
  set_error(op->ctx, "nd_hex_apply7z: no kernel for p=%d q1d=%d kind=%d", op->p, op->q1d, kind);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace b2p
