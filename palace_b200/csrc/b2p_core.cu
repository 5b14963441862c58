// Context, errors, device memory helpers, geometry q-data and operator construction for the C ABI.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <set>
#include <type_traits>

#include <algorithm>

#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_geom1.cuh"

namespace b2p
{

static thread_local std::string tls_error;

void set_error(b2p_ctx *ctx, const char *fmt, ...)
{
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  tls_error = buf;
  if (ctx) ctx->last_error = buf;
}

template <typename T>
int upload(b2p_ctx *ctx, const T *host, size_t n, T **dptr)
{
  *dptr = nullptr;
  if (n == 0) return B2P_SUCCESS;
  B2P_CUDA(ctx, cudaMalloc((void **)dptr, n * sizeof(T)));
  B2P_CUDA(ctx, cudaMemcpy(*dptr, host, n * sizeof(T), cudaMemcpyHostToDevice));
  return B2P_SUCCESS;
}
template int upload<double>(b2p_ctx *, const double *, size_t, double **);
template int upload<int32_t>(b2p_ctx *, const int32_t *, size_t, int32_t **);
template int upload<int8_t>(b2p_ctx *, const int8_t *, size_t, int8_t **);
template int upload<int64_t>(b2p_ctx *, const int64_t *, size_t, int64_t **);

namespace
{

// Geometry factors at quadrature points of order-k hexes (K6 of SURVEY §2d; restates
// qfunctions/33/geom_33_qf.h:9-34 on the device). One thread per (element, point).
__global__ void geom_hex_kernel(int ne, int k, int q, const double *__restrict__ xe, const double *__restrict__ B,
                                const double *__restrict__ G, const double *__restrict__ qw, double *__restrict__ qd)
{
  const int n = k + 1, Nn = n * n * n, Q = q * q * q;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)ne * Q) return;
  const int e = (int)(w / Q), iq = (int)(w % Q);
  const int qx = iq % q, qy = (iq / q) % q, qz = iq / (q * q);
  const double *x = xe + (size_t)e * 3 * Nn;
  double *o = qd + (size_t)e * 10 * Q + qslot(q, qx, qy, qz);
  if (k == 1)  // trilinear: the definition the element kernels on node geometry share (b2p_geom1.cuh)
  {
    Hex1Line L;
    hex1_line(x, B + 2 * qy, G + 2 * qy, B + 2 * qz, G + 2 * qz, L);
    double A[9];
    hex1_point(L, B + 2 * qx, G + 2 * qx, qw[qx], qw[qy], qw[qz], o[0], A);
    for (int t = 0; t < 9; t++) o[(1 + t) * Q] = A[t];
    return;
  }
  double J[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int kk = 0; kk < n; kk++)
    for (int jj = 0; jj < n; jj++)
      for (int ii = 0; ii < n; ii++)
      {
        const int m = ii + n * (jj + n * kk);
        const double gx = G[qx * n + ii] * B[qy * n + jj] * B[qz * n + kk];
        const double gy = B[qx * n + ii] * G[qy * n + jj] * B[qz * n + kk];
        const double gz = B[qx * n + ii] * B[qy * n + jj] * G[qz * n + kk];
        for (int c = 0; c < 3; c++)
        {
          const double xc = x[c * Nn + m];
          J[c + 0] += xc * gx;
          J[c + 3] += xc * gy;
          J[c + 6] += xc * gz;
        }
      }
  double A[9];
  cofactor33(J, A);
  const double detJ = J[0] * A[0] + J[1] * A[1] + J[2] * A[2];
  o[0] = qw[qx] * qw[qy] * qw[qz] * detJ;
  for (int t = 0; t < 9; t++) o[(1 + t) * Q] = A[t] / detJ;
}

}  // namespace

int launch_geom_hex(b2p_ctx *ctx, int ne, int k, int q1d, const double *d_xe, const double *d_B, const double *d_G,
                    const double *d_qw, double *d_qd, cudaStream_t s)
{
  const size_t total = (size_t)ne * q1d * q1d * q1d;
  const int nt = 128;
  B2P_LAUNCH(geom_hex_kernel, (unsigned)((total + nt - 1) / nt), nt, 0, s, ne, k, q1d, d_xe, d_B, d_G, d_qw, d_qd);
  B2P_CUDA(ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p

namespace b2p
{
// B2P_ND_KERNEL = 4 | 5 | 6 | 7 forces one of the sum-factorised ND kernels (0: the default routes)
static int forced_nd_kernel()
{
  static const int k = []
  {
    const char *e = std::getenv("B2P_ND_KERNEL");
    return e ? std::atoi(e) : 0;
  }();
  return k;
}

// Largest deviation of the packed 1-D tables (Bo, Bc even, Gc odd about the centre) from mirror symmetry, and largest |entry|.
static void tables_mirror_deviation(const double *tab, int p, int q, double &dev, double &scale)
{
  const int n = p + 1;
  const double *Bo = tab, *Bc = tab + q * p, *Gc = Bc + q * n;
  scale = 0.0;
  for (int i = 0; i < q * p + 2 * q * n; i++) scale = std::fmax(scale, std::fabs(tab[i]));
  dev = 0.0;
  for (int c = 0; c < q; c++)
  {
    for (int i = 0; i < p; i++) dev = std::fmax(dev, std::fabs(Bo[c * p + i] - Bo[(q - 1 - c) * p + (p - 1 - i)]));
    for (int i = 0; i < n; i++)
    {
      dev = std::fmax(dev, std::fabs(Bc[c * n + i] - Bc[(q - 1 - c) * n + (n - 1 - i)]));
      dev = std::fmax(dev, std::fabs(Gc[c * n + i] + Gc[(q - 1 - c) * n + (n - 1 - i)]));
    }
  }
}

bool nd_tables_symmetric(const double *tab, int p, int q, double rel_tol)
{
  double dev, scale;
  tables_mirror_deviation(tab, p, q, dev, scale);
  return dev <= rel_tol * scale;
}

bool nd_tables_symmetric(b2p_op *op, double rel_tol)
{
  if (op->tab_dev < 0) tables_mirror_deviation(op->h_tab.data(), op->p, op->q1d, op->tab_dev, op->tab_scale);
  return op->tab_dev <= rel_tol * op->tab_scale;
}

// The element kernel of an apply with these flags: the one place that decides it. B2P_ND_KERNEL (`forced` below) and the
// apply flags SIMPLE, HALFWARP, ROUND1, CTA (B2P_APPLY_*_KERNEL) steer the Nedelec routes; "nd6 / nd5 / nd7" below stand for
// nd_hex_apply6_eligible / nd_hex_apply5_eligible / nd_hex_apply7_eligible (q1d = p + 1 and mirror-symmetric tables among others).
//
//   operator                   condition, first match wins                                         kernel
//   dense basis                                                                                   DENSE
//   Raviart-Thomas mass        not SIMPLE and rt_hex_apply7_eligible                              RT7
//                              otherwise                                                          RT_SIMPLE
//   block (bcoef)              SIMPLE, ROUND1 or HALFWARP, or forced 4 or 5                       ND_SIMPLE
//                              neither CTA nor forced 7, and nd6                                  ND6
//                              nd7                                                                ND7
//                              otherwise                                                          ND_SIMPLE
//   H1 diffusion               SIMPLE                                                             H1_SIMPLE
//                              otherwise                                                          H1V3
//   symmetric Nedelec kinds    SIMPLE                                                             ND_SIMPLE
//                              (HALFWARP or forced 5) and nd5                                     ND5
//                              (forced 6, or unset at p = 3), neither ROUND1 nor CTA, and nd6     ND6
//                              (CTA, forced 7 or unset), not ROUND1, and nd7                      ND7
//                              otherwise (forced 6 at p >= 4 included)                            ND4
//
// Why these defaults: DESIGN.md 4.1 and tools/nd7_ab.py time nd_hex_apply6_kernel (p = 3, and the block form at p = 2, 3),
// nd_hex_apply7_kernel (p = 2, 4, 5, 6) and nd_hex_apply4_kernel against each other; nd_hex_apply5_kernel is slower and kept for
// the analysis. The block form exists only in nd_hex_apply_kernel, nd_hex_apply6_kernel and nd_hex_apply7_kernel.
HexKernel choose_hex_kernel(b2p_op *op, int flags)
{
  if (op->dense) return HexKernel::DENSE;
  const bool simple = flags & B2P_APPLY_SIMPLE_KERNEL, half = flags & B2P_APPLY_HALFWARP_KERNEL;
  const bool round1 = flags & B2P_APPLY_ROUND1_KERNEL, cta = flags & B2P_APPLY_CTA_KERNEL;
  if (op->kind == B2P_RT_MASS) return !simple && rt_hex_apply7_eligible(op) ? HexKernel::RT7 : HexKernel::RT_SIMPLE;
  const int forced = forced_nd_kernel();
  if (op->bcoef)
  {
    if (simple || round1 || half || forced == 4 || forced == 5) return HexKernel::ND_SIMPLE;
    if (!(cta || forced == 7) && nd_hex_apply6_eligible(op)) return HexKernel::ND6;
    return nd_hex_apply7_eligible(op) ? HexKernel::ND7 : HexKernel::ND_SIMPLE;
  }
  if (op->kind == B2P_H1_DIFFUSION) return simple ? HexKernel::H1_SIMPLE : HexKernel::H1V3;
  if (simple) return HexKernel::ND_SIMPLE;
  if ((half || forced == 5) && nd_hex_apply5_eligible(op)) return HexKernel::ND5;
  if ((forced == 6 || (forced == 0 && op->p == 3)) && !round1 && !cta && nd_hex_apply6_eligible(op)) return HexKernel::ND6;
  if ((cta || forced == 7 || forced == 0) && !round1 && nd_hex_apply7_eligible(op)) return HexKernel::ND7;
  return HexKernel::ND4;
}

// One pass over the geometry for a complex sum: nd_hex_apply4_kernel<CPLX> at p <= 3 (and for a single term),
// nd_hex_apply7_kernel<CPLX> for two or more terms at p = 4 ... 6 and for block sums.
HexComplexKernel choose_hex_complex_kernel(b2p_op *op, int n_terms)
{
  if (op->bcoef || (op->p >= 4 && n_terms >= 2)) return nd_hex_apply7_eligible(op) ? HexComplexKernel::ND7Z : HexComplexKernel::NONE;
  return nd_hex_apply4z_eligible(op) ? HexComplexKernel::ND4Z : HexComplexKernel::NONE;
}

bool hex_pair_apply_eligible(b2p_op *op)
{
  return !op->bcoef && op->kind != B2P_RT_MASS && nd_hex_apply4z_eligible(op) && op->ecoef;
}

int configure_kernel_once(b2p_ctx *ctx, const void *kern, size_t shmem, int carveout)
{
  static std::mutex m;
  static std::set<std::pair<const void *, int>> done;
  std::lock_guard<std::mutex> lock(m);
  if (done.count({kern, ctx->device})) return B2P_SUCCESS;
  B2P_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shmem));
  if (carveout >= 0) B2P_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
  done.insert({kern, ctx->device});
  return B2P_SUCCESS;
}

int apply_range(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, int flags,
                cudaStream_t s)
{
  static const bool trace = std::getenv("B2P_TRACE_KERNEL") != nullptr;
  const bool tr = (flags & B2P_APPLY_TRANSPOSE) != 0;  // the symmetric kinds, H1 and Raviart-Thomas ignore it
  const HexKernel k = choose_hex_kernel(op, flags);
  switch (k)
  {
    case HexKernel::DENSE: return launch_dense_apply(op, lidx, alpha, x, y, rg, s, tr);
    case HexKernel::RT7:
    case HexKernel::RT_SIMPLE:
      B2P_CHECK(op->ctx, !rg.xg && !rg.yg, B2P_ERR_UNSUPPORTED, "Raviart-Thomas operators: partitioned applies (ghost pieces) are not supported");
      return launch_rt_hex_apply(op, lidx, alpha, x, y, rg, s, k == HexKernel::RT7);
    case HexKernel::ND_SIMPLE: return launch_nd_hex_apply(op, lidx, alpha, x, y, rg, s, tr);
    case HexKernel::ND4: return launch_nd_hex_apply4(op, lidx, alpha, x, y, rg, s);
    case HexKernel::ND5: return launch_nd_hex_apply5(op, lidx, alpha, x, y, rg, s);
    case HexKernel::ND6:
      if (trace && !op->bcoef) fprintf(stderr, "[b2p] nd_hex_apply6 p=%d q1d=%d kind=%d ne=%d\n", op->p, op->q1d, op->kind, op->ne);
      return launch_nd_hex_apply6(op, lidx, alpha, x, y, rg, s, tr);
    case HexKernel::ND7:
      if (trace && !op->bcoef) fprintf(stderr, "[b2p] nd_hex_apply7 p=%d q1d=%d kind=%d ne=%d\n", op->p, op->q1d, op->kind, op->ne);
      return launch_nd_hex_apply7(op, lidx, alpha, x, y, rg, s, tr);
    case HexKernel::H1_SIMPLE: return launch_h1_hex_apply(op, lidx, alpha, x, y, rg, s);
    case HexKernel::H1V3: return launch_h1_hex_apply3(op, lidx, alpha, x, y, rg, s);
  }
  return B2P_ERR_UNSUPPORTED;
}
}  // namespace b2p

using namespace b2p;

namespace b2p
{
// order-free fingerprint of a dof set (splitmix64 finaliser per dof, summed)
inline uint64_t ess_mix(uint64_t z)
{
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
bool op_essential_matches(const b2p_op *op, const int32_t *ess_ldofs, int64_t n)
{
  std::vector<int32_t> v(ess_ldofs, ess_ldofs + (n > 0 ? n : 0));
  std::sort(v.begin(), v.end());
  v.erase(std::unique(v.begin(), v.end()), v.end());
  uint64_t h = 0;
  for (int32_t d : v) h += ess_mix((uint64_t)d);
  if (!op->lidx_bc) return v.empty();
  return op->ess_n == (int64_t)v.size() && op->ess_hash == h;
}

// Compose the native-order restriction + orientation with the lexicographic->native dof map
// (restriction.cpp:134-188,281-297) into one signed lexicographic index array.
int build_lex_restriction(b2p_ctx *ctx, const char *who, const b2p_op_desc *d, int P, int64_t lsize, int ne, int *PS_out, int32_t **out)
{
  const int PS = (P + 3) & ~3;
  *PS_out = PS;
  std::vector<int32_t> lidx((size_t)ne * PS, (int32_t)B2P_SKIP_IDX);
  for (int l = 0; l < P; l++)
  {
    int nat = d->dof_map ? d->dof_map[l] : l;
    int sg = 1;
    if (nat < 0)
    {
      nat = -1 - nat;
      sg = -1;
    }
    B2P_CHECK(ctx, nat >= 0 && nat < P, B2P_ERR_ARG, "%sdof_map[%d] out of range", who, l);
    for (int e = 0; e < ne; e++)
    {
      const int32_t gi = d->idx[(size_t)e * P + nat];
      B2P_CHECK(ctx, gi >= 0 && gi < lsize, B2P_ERR_ARG, "%sidx[%d][%d]=%d outside L-vector of size %lld", who, e, nat, gi,
                (long long)lsize);
      const int s = sg * (d->orient ? (int)d->orient[(size_t)e * P + nat] : 1);
      lidx[(size_t)e * PS + l] = (s >= 0) ? gi : (-1 - gi);
    }
  }
  return upload(ctx, lidx.data(), lidx.size(), out);
}
}  // namespace b2p

extern "C"
{

int b2p_ctx_create(int cuda_device, b2p_ctx **out)
{
  if (!out) return B2P_ERR_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
  {
    set_error(nullptr, "b2p_ctx_create: no CUDA device (%s); there is no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return B2P_ERR_CUDA;
  }
  B2P_CHECK(nullptr, cuda_device >= 0 && cuda_device < count, B2P_ERR_ARG, "b2p_ctx_create: bad device %d", cuda_device);
  B2P_CUDA(nullptr, cudaSetDevice(cuda_device));
  cudaDeviceProp prop;
  B2P_CUDA(nullptr, cudaGetDeviceProperties(&prop, cuda_device));
  // sm_90a code runs on compute capability 9.0 only: the arch-specific ("a") features have no forward compatibility
  B2P_CHECK(nullptr, prop.major == 9 && prop.minor == 0, B2P_ERR_CUDA,
            "b2p_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", cuda_device, prop.major,
            prop.minor);
  b2p_ctx *ctx = new b2p_ctx;
  ctx->device = cuda_device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->red_cap = 4096;
  B2P_CUDA(nullptr, cudaMalloc((void **)&ctx->d_red, ctx->red_cap * sizeof(double)));
  B2P_CUDA(nullptr, cudaMallocHost((void **)&ctx->h_red, ctx->red_cap * sizeof(double)));
  B2P_CUDA(nullptr, cudaMalloc((void **)&ctx->d_sink, b2p_ctx::SINK_SLOTS * sizeof(double)));
  B2P_CUDA(nullptr, cudaMemset(ctx->d_sink, 0, b2p_ctx::SINK_SLOTS * sizeof(double)));
  *out = ctx;
  return B2P_SUCCESS;
}

const char *b2p_last_error(b2p_ctx *ctx) { return ctx ? ctx->last_error.c_str() : tls_error.c_str(); }
int b2p_ctx_rank(b2p_ctx *ctx) { return ctx ? ctx->rank : 0; }
int b2p_ctx_nranks(b2p_ctx *ctx) { return ctx ? ctx->nranks : 1; }

int b2p_ctx_last_launch(b2p_ctx *ctx, b2p_launch_info *out)
{
  if (!ctx || !out) return B2P_ERR_ARG;
  B2P_CHECK(ctx, ctx->last_launch.seq > 0, B2P_ERR_ARG, "b2p_ctx_last_launch: no persistent element kernel launched on this context yet");
  *out = ctx->last_launch;
  return B2P_SUCCESS;
}

int b2p_ctx_sync(b2p_ctx *ctx, b2p_stream s)
{
  B2P_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)s));
  return B2P_SUCCESS;
}

int b2p_malloc(b2p_ctx *ctx, size_t bytes, void **dptr)
{
  B2P_CUDA(ctx, cudaMalloc(dptr, bytes));
  return B2P_SUCCESS;
}
int b2p_free(b2p_ctx *ctx, void *dptr)
{
  B2P_CUDA(ctx, cudaFree(dptr));
  return B2P_SUCCESS;
}
int b2p_memcpy_h2d(b2p_ctx *ctx, void *dst, const void *src, size_t bytes, b2p_stream s)
{
  B2P_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)s));
  return B2P_SUCCESS;
}
int b2p_memcpy_d2h(b2p_ctx *ctx, void *dst, const void *src, size_t bytes, b2p_stream s)
{
  B2P_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)s));
  B2P_CUDA(ctx, cudaStreamSynchronize((cudaStream_t)s));
  return B2P_SUCCESS;
}

// ---- geometry ---------------------------------------------------------------------------------

int b2p_geom_create_hex(b2p_ctx *ctx, int ne, int mesh_order, int q1d, const double *xe, const double *nodeB,
                        const double *nodeG, const double *qw1d, const int32_t *attr, b2p_geom **out)
{
  B2P_CHECK(ctx, ctx && out && xe && nodeB && nodeG && qw1d && attr, B2P_ERR_ARG, "b2p_geom_create_hex: null argument");
  B2P_CHECK(ctx, ne > 0 && mesh_order >= 1 && q1d >= 1, B2P_ERR_ARG, "b2p_geom_create_hex: bad sizes");
  const int n = mesh_order + 1, Nn = n * n * n, Q = q1d * q1d * q1d;
  b2p_geom *g = new b2p_geom;
  g->ctx = ctx;
  g->ne = ne;
  g->q1d = q1d;
  g->Q = Q;
  double *d_xe = nullptr, *d_B = nullptr, *d_G = nullptr, *d_qw = nullptr;
  int rc;
  if ((rc = upload(ctx, xe, (size_t)ne * 3 * Nn, &d_xe))) return rc;
  if ((rc = upload(ctx, nodeB, (size_t)q1d * n, &d_B))) return rc;
  if ((rc = upload(ctx, nodeG, (size_t)q1d * n, &d_G))) return rc;
  if ((rc = upload(ctx, qw1d, (size_t)q1d, &d_qw))) return rc;
  if ((rc = upload(ctx, attr, (size_t)ne, &g->attr))) return rc;
  B2P_CUDA(ctx, cudaMalloc((void **)&g->qd, (size_t)ne * 10 * Q * sizeof(double)));
  if ((rc = launch_geom_hex(ctx, ne, mesh_order, q1d, d_xe, d_B, d_G, d_qw, g->qd, 0))) return rc;
  B2P_CUDA(ctx, cudaDeviceSynchronize());
  // The vertex route forms the x-derivative column of J once per (qy, qz) line from row 0 of nodeG and the other two columns
  // with B_0 = 1 - B_1: keep the vertices only when the derivative of the linear basis is the same at every 1-D point and the
  // basis is a partition of unity (both hold for a Lagrange basis through two nodes).
  bool g_const = mesh_order == 1;
  for (int c = 0; g_const && c < q1d; c++)
    g_const = nodeG[2 * c] == nodeG[0] && nodeG[2 * c + 1] == nodeG[1] && std::fabs(nodeB[2 * c] + nodeB[2 * c + 1] - 1.0) <= 1e-15;
  if (mesh_order == 1 && g_const)
  {
    g->xe = d_xe;
    g->h_nodeB.assign(nodeB, nodeB + (size_t)q1d * n);
    g->h_nodeG.assign(nodeG, nodeG + (size_t)q1d * n);
    g->h_qw.assign(qw1d, qw1d + q1d);
  }
  else
    cudaFree(d_xe);
  cudaFree(d_B);
  cudaFree(d_G);
  cudaFree(d_qw);
  *out = g;
  return B2P_SUCCESS;
}

int b2p_geom_create_qdata(b2p_ctx *ctx, int ne, int q1d, const double *qdata, b2p_geom **out)
{
  B2P_CHECK(ctx, ctx && out && qdata && ne > 0 && q1d > 0, B2P_ERR_ARG, "b2p_geom_create_qdata: bad argument");
  const int Q = q1d * q1d * q1d;
  std::vector<double> qd((size_t)ne * 10 * Q);
  std::vector<int32_t> attr(ne);
  for (int e = 0; e < ne; e++)
  {
    attr[e] = (int32_t)qdata[(size_t)e * 11 * Q];
    for (int c = 0; c < 10; c++)
      for (int iq = 0; iq < Q; iq++)
        qd[((size_t)e * 10 + c) * Q + qslot_of(q1d, iq)] = qdata[((size_t)e * 11 + 1 + c) * Q + iq];
  }
  b2p_geom *g = new b2p_geom;
  g->ctx = ctx;
  g->ne = ne;
  g->q1d = q1d;
  g->Q = Q;
  int rc;
  if ((rc = upload(ctx, qd.data(), qd.size(), &g->qd))) return rc;
  if ((rc = upload(ctx, attr.data(), attr.size(), &g->attr))) return rc;
  *out = g;
  return B2P_SUCCESS;
}

// General (non-tensor) quadrature: any element type; points in the caller's order.
int b2p_geom_create_qdata_general(b2p_ctx *ctx, int ne, int Q, const double *qdata, b2p_geom **out)
{
  B2P_CHECK(ctx, ctx && out && qdata && ne > 0 && Q > 0, B2P_ERR_ARG, "b2p_geom_create_qdata_general: bad argument");
  std::vector<double> qd((size_t)ne * 10 * Q);
  std::vector<int32_t> attr(ne);
  for (int e = 0; e < ne; e++)
  {
    attr[e] = (int32_t)qdata[(size_t)e * 11 * Q];
    std::memcpy(&qd[(size_t)e * 10 * Q], &qdata[((size_t)e * 11 + 1) * Q], sizeof(double) * 10 * Q);
  }
  b2p_geom *g = new b2p_geom;
  g->ctx = ctx;
  g->ne = ne;
  g->q1d = 0;
  g->Q = Q;
  int rc;
  if ((rc = upload(ctx, qd.data(), qd.size(), &g->qd))) return rc;
  if ((rc = upload(ctx, attr.data(), attr.size(), &g->attr))) return rc;
  *out = g;
  return B2P_SUCCESS;
}

int b2p_geom_get_qdata(b2p_geom *g, double *qdata_host)
{
  if (!g || !qdata_host) return B2P_ERR_ARG;
  const int Q = g->Q;
  std::vector<double> qd((size_t)g->ne * 10 * Q);
  std::vector<int32_t> attr(g->ne);
  B2P_CUDA(g->ctx, cudaMemcpy(qd.data(), g->qd, qd.size() * sizeof(double), cudaMemcpyDeviceToHost));
  B2P_CUDA(g->ctx, cudaMemcpy(attr.data(), g->attr, attr.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  for (int e = 0; e < g->ne; e++)
  {
    for (int i = 0; i < Q; i++) qdata_host[(size_t)e * 11 * Q + i] = (double)attr[e];
    for (int c = 0; c < 10; c++)
      for (int iq = 0; iq < Q; iq++)
        qdata_host[((size_t)e * 11 + 1 + c) * Q + iq] = qd[((size_t)e * 10 + c) * Q + qslot_of(g->q1d, iq)];
  }
  return B2P_SUCCESS;
}

void b2p_geom_destroy(b2p_geom *g)
{
  if (!g) return;
  if (--g->refcount > 0) return;
  cudaFree(g->qd);
  cudaFree(g->attr);
  cudaFree(g->xe);
  delete g;
}

// ---- operator ---------------------------------------------------------------------------------

namespace
{

union IntScalar
{
  int first;
  double second;
};

// Decode a coefficient context (coeff_qf.h:7-43): returns per-attribute material index and the
// material matrices; n_attr == 0 means "every attribute -> material 0".
struct DecodedCtx
{
  std::vector<int> attr_mat;
  std::vector<double> mats;  // [n_mat][9]
  size_t entries = 0;        // entries consumed
};

bool decode_ctx(const IntScalar *c, size_t avail, DecodedCtx &d)
{
  if (avail < 2) return false;
  const int na = c[0].first;
  if (na < 0 || (size_t)(2 + na) > avail) return false;
  d.attr_mat.resize(na);
  for (int i = 0; i < na; i++) d.attr_mat[i] = c[1 + i].first;
  const int nm = c[1 + na].first;
  if (nm <= 0 || (size_t)(2 + na + 9 * (size_t)nm) > avail) return false;
  d.mats.resize(9 * (size_t)nm);
  for (size_t i = 0; i < 9 * (size_t)nm; i++) d.mats[i] = c[2 + na + i].second;
  d.entries = 2 + na + 9 * (size_t)nm;
  for (int i = 0; i < na; i++)
    if (d.attr_mat[i] < 0 || d.attr_mat[i] >= nm) return false;
  return true;
}

// Upload the per-element block {Cm, Ck, Cw, Cx} of a block operator and the block of its transpose: (A^T)'s pointwise form
// has every tensor transposed, and the value->curl and curl->value tensors trade places.
int set_block(b2p_op *op, const std::vector<double> &blk)
{
  std::vector<double> blk_t(blk.size());
  static const int from[4] = {0, 1, 3, 2};
  for (int e = 0; e < op->ne; e++)
    for (int k = 0; k < 4; k++)
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) blk_t[36 * (size_t)e + 9 * k + i + 3 * j] = blk[36 * (size_t)e + 9 * from[k] + j + 3 * i];
  if (op->bcoef)  // refill in place: p-coarsened operators share these arrays
  {
    B2P_CUDA(op->ctx, cudaMemcpy(op->bcoef, blk.data(), blk.size() * sizeof(double), cudaMemcpyHostToDevice));
    B2P_CUDA(op->ctx, cudaMemcpy(op->bcoef_t, blk_t.data(), blk_t.size() * sizeof(double), cudaMemcpyHostToDevice));
    return B2P_SUCCESS;
  }
  int rc;
  if ((rc = upload(op->ctx, blk.data(), blk.size(), &op->bcoef)) || (rc = upload(op->ctx, blk_t.data(), blk_t.size(), &op->bcoef_t)))
    return rc;
  return B2P_SUCCESS;
}

int set_coeff(b2p_op *op, const void *blob, size_t bytes)
{
  b2p_ctx *ctx = op->ctx;
  B2P_CHECK(ctx, blob && bytes % 8 == 0 && bytes >= 16, B2P_ERR_ARG, "coefficient context: bad size %zu", bytes);
  const IntScalar *c = (const IntScalar *)blob;
  const size_t avail = bytes / 8;
  DecodedCtx first, second;
  B2P_CHECK(ctx, decode_ctx(c, avail, first), B2P_ERR_ARG, "coefficient context: malformed (first part)");
  const bool pair = (op->kind == B2P_CURLCURL_MASS);
  if (pair)
    B2P_CHECK(ctx, decode_ctx(c + first.entries, avail - first.entries, second), B2P_ERR_ARG,
              "coefficient context: malformed (second part of pair)");
  // material table: first part then second part
  std::vector<double> mats = first.mats;
  const int off2 = (int)(first.mats.size() / 9);
  mats.insert(mats.end(), second.mats.begin(), second.mats.end());
  std::vector<int32_t> attr(op->ne), emat(2 * (size_t)op->ne);
  B2P_CUDA(ctx, cudaMemcpy(attr.data(), op->geom->attr, sizeof(int32_t) * op->ne, cudaMemcpyDeviceToHost));
  auto lookup = [&](const DecodedCtx &d, int a, int &m) -> bool
  {
    if (d.attr_mat.empty())
    {
      m = 0;
      return true;
    }
    if (a < 1 || a > (int)d.attr_mat.size()) return false;
    m = d.attr_mat[a - 1];
    return true;
  };
  for (int e = 0; e < op->ne; e++)
  {
    int m0 = 0, m1 = 0;
    B2P_CHECK(ctx, lookup(first, attr[e], m0), B2P_ERR_ARG, "element %d attribute %d outside coefficient context", e,
              attr[e]);
    if (pair)
    {
      B2P_CHECK(ctx, lookup(second, attr[e], m1), B2P_ERR_ARG, "element %d attribute %d outside coefficient context", e,
                attr[e]);
      m1 += off2;
    }
    else
      m1 = m0;  // single-part kinds read the same table for whichever part they use
    emat[2 * (size_t)e] = m0;
    emat[2 * (size_t)e + 1] = m1;
  }
  if (op->owns_coeff)
  {
    cudaFree(op->mat);
    cudaFree(op->emat);
    cudaFree(op->ecoef);
  }
  op->owns_coeff = true;
  op->n_mat = (int)(mats.size() / 9);
  op->iso = true;
  for (size_t m = 0; m < mats.size() / 9 && op->iso; m++)
    for (int t = 0; t < 9; t++)
    {
      const double v = mats[9 * m + t], d = mats[9 * m];
      if ((t % 4 == 0) ? (v != d) : (v != 0.0)) op->iso = false;
    }
  int rc;
  if ((rc = upload(ctx, mats.data(), mats.size(), &op->mat))) return rc;
  if ((rc = upload(ctx, emat.data(), emat.size(), &op->emat))) return rc;
  std::vector<double> ecoef(18 * (size_t)op->ne);
  for (int e = 0; e < op->ne; e++)
    for (int part = 0; part < 2; part++)
      for (int t = 0; t < 9; t++) ecoef[18 * (size_t)e + 9 * part + t] = mats[9 * (size_t)emat[2 * (size_t)e + part] + t];
  if ((rc = upload(ctx, ecoef.data(), ecoef.size(), &op->ecoef))) return rc;
  if (!op->dense && (op->kind == B2P_ND_WEAKCURL || op->kind == B2P_ND_MIXEDCURL))
  {
    // the context's tensor goes to Cw (weak curl: values -> curls) or Cx (mixed curl: curls -> values), zeros elsewhere
    const int slot = op->kind == B2P_ND_WEAKCURL ? 2 : 3;
    std::vector<double> blk((size_t)36 * op->ne, 0.0);
    for (int e = 0; e < op->ne; e++)
      for (int t = 0; t < 9; t++) blk[36 * (size_t)e + 9 * slot + t] = ecoef[18 * (size_t)e + t];
    return set_block(op, blk);
  }
  return B2P_SUCCESS;
}

int elem_dofs(int kind, int p)
{
  if (kind == B2P_H1_DIFFUSION) return (p + 1) * (p + 1) * (p + 1);
  if (kind == B2P_RT_MASS) return 3 * p * p * (p + 1);  // RT_{p-1}: closed along one axis, open along two
  return 3 * p * (p + 1) * (p + 1);
}

int build_restriction(b2p_op *op, const b2p_op_desc *d)
{
  return build_lex_restriction(op->ctx, "", d, op->P, op->lsize, op->ne, &op->PS, &op->lidx);
}

int build_tables(b2p_op *op, const b2p_op_desc *d)
{
  const int p = op->p, q = op->q1d, n = p + 1;
  std::vector<double> tab((size_t)q * p + 2 * (size_t)q * n, 0.0);
  if (op->kind != B2P_H1_DIFFUSION)
  {
    B2P_CHECK(op->ctx, d->Bo, B2P_ERR_ARG, "Bo table required for ND operators");
    std::memcpy(tab.data(), d->Bo, sizeof(double) * q * p);
  }
  const bool need_g = op->kind != B2P_RT_MASS;  // the RT mass reads values only
  B2P_CHECK(op->ctx, d->Bc && (d->Gc || !need_g), B2P_ERR_ARG, "Bc/Gc tables required");
  std::memcpy(tab.data() + (size_t)q * p, d->Bc, sizeof(double) * q * n);
  if (need_g) std::memcpy(tab.data() + (size_t)q * p + (size_t)q * n, d->Gc, sizeof(double) * q * n);
  op->h_tab = tab;
  return upload(op->ctx, tab.data(), tab.size(), &op->tab);
}

int assemble_qdata(b2p_op *op)
{
  const int parts = (op->kind == B2P_CURLCURL_MASS) ? 2 : 1;
  op->aq_ncomp = 9 * parts;
  op->aq_estride = ((int64_t)op->aq_ncomp * op->geom->Q + 1) & ~(int64_t)1;
  if (!op->aq)
  {
    B2P_CUDA(op->ctx, cudaMalloc((void **)&op->aq, (size_t)op->ne * op->aq_estride * sizeof(double)));
    B2P_CUDA(op->ctx, cudaMemset(op->aq, 0, (size_t)op->ne * op->aq_estride * sizeof(double)));
  }
  int rc = launch_assemble_qdata(op, 0);
  if (rc) return rc;
  B2P_CUDA(op->ctx, cudaDeviceSynchronize());
  return B2P_SUCCESS;
}

}  // namespace

int b2p_op_create(b2p_ctx *ctx, b2p_geom *geom, const b2p_op_desc *d, b2p_op **out)
{
  B2P_CHECK(ctx, ctx && geom && d && out, B2P_ERR_ARG, "b2p_op_create: null argument");
  B2P_CHECK(ctx, d->kind >= B2P_CURLCURL && d->kind <= B2P_RT_MASS, B2P_ERR_ARG, "b2p_op_create: bad kind %d", d->kind);
  B2P_CHECK(ctx, !(d->assemble_qdata && (d->kind == B2P_ND_WEAKCURL || d->kind == B2P_ND_MIXEDCURL)), B2P_ERR_UNSUPPORTED,
            "b2p_op_create: assembled q-data is not available for the mixed curl kinds (apply their coefficient on the fly)");
  B2P_CHECK(ctx, !(d->assemble_qdata && d->kind == B2P_RT_MASS), B2P_ERR_UNSUPPORTED,
            "b2p_op_create: assembled q-data is not available for the Raviart-Thomas mass (apply its coefficient on the fly)");
  B2P_CHECK(ctx, d->ne == geom->ne, B2P_ERR_ARG, "b2p_op_create: %d elements vs %d in geometry", d->ne, geom->ne);
  B2P_CHECK(ctx, d->p >= 1 && d->p <= 6 && d->p < geom->q1d && geom->q1d <= 7, B2P_ERR_UNSUPPORTED,
            "b2p_op_create: unsupported p=%d q1d=%d (hex kernels cover p<=6, p<q1d<=7)", d->p, geom->q1d);
  B2P_CHECK(ctx, d->idx && d->lsize > 0, B2P_ERR_ARG, "b2p_op_create: missing restriction");
  b2p_op *op = new b2p_op;
  op->ctx = ctx;
  op->geom = geom;
  geom->refcount++;
  op->kind = d->kind;
  op->p = d->p;
  op->q1d = geom->q1d;
  op->ne = d->ne;
  op->P = elem_dofs(d->kind, d->p);
  op->lsize = d->lsize;
  op->assembled = d->assemble_qdata;
  int rc;
  if ((rc = build_restriction(op, d)) || (rc = build_tables(op, d)) || (rc = set_coeff(op, d->coeff_ctx, d->coeff_ctx_bytes)))
  {
    b2p_op_destroy(op);
    return rc;
  }
  if (op->assembled && (rc = assemble_qdata(op)))
  {
    b2p_op_destroy(op);
    return rc;
  }
  *out = op;
  return B2P_SUCCESS;
}

namespace
{
// Dense-basis operator on any element type (see b2p_dense.cu). With `fine` set, the new operator shares the coefficient of
// `fine` (the coarse level of a p-hierarchy) instead of reading desc->coeff_ctx.
int create_dense(b2p_ctx *ctx, b2p_geom *geom, const b2p_dense_op_desc *d, b2p_op *fine, b2p_op **out)
{
  B2P_CHECK(ctx, d->kind >= B2P_CURLCURL && d->kind <= B2P_ND_MIXEDCURL, B2P_ERR_ARG, "b2p_op_create_dense: bad kind %d", d->kind);
  B2P_CHECK(ctx, geom->q1d == 0 && geom->Q == d->Q && geom->ne == d->ne, B2P_ERR_ARG,
            "b2p_op_create_dense: needs a general geometry (b2p_geom_create_qdata_general) with matching ne / Q");
  const bool mixed = (d->kind == B2P_ND_WEAKCURL || d->kind == B2P_ND_MIXEDCURL);  // value and curl tables, one coefficient
  const bool need_u = (d->kind == B2P_ND_MASS || d->kind == B2P_CURLCURL_MASS || mixed), need_c = (d->kind != B2P_ND_MASS);
  B2P_CHECK(ctx, (!need_u || d->interp) && (!need_c || d->deriv) && d->idx && d->lsize > 0 && d->P > 0, B2P_ERR_ARG,
            "b2p_op_create_dense: missing tables / restriction");
  b2p_op *op = new b2p_op;
  op->ctx = ctx;
  op->geom = geom;
  geom->refcount++;
  op->dense = true;
  op->kind = d->kind;
  op->p = 0;
  op->q1d = 0;
  op->ne = d->ne;
  op->P = d->P;
  op->lsize = d->lsize;
  const int P = d->P, Q = d->Q;
  op->dense_Ppad = (P + 7) & ~7;
  int rows = 0;
  if (need_u)
  {
    op->dense_row_u = rows;
    rows += 3 * Q;
  }
  if (need_c)
  {
    op->dense_row_c = rows;
    rows += 3 * Q;
  }
  op->dense_Rpad = (rows + 7) & ~7;
  std::vector<double> T((size_t)op->dense_Rpad * op->dense_Ppad, 0.0);
  for (int r = 0; r < 3 * Q; r++)
    for (int i = 0; i < P; i++)
    {
      if (need_u) T[(size_t)(op->dense_row_u + r) * op->dense_Ppad + i] = d->interp[(size_t)r * P + i];
      if (need_c) T[(size_t)(op->dense_row_c + r) * op->dense_Ppad + i] = d->deriv[(size_t)r * P + i];
    }
  b2p_op_desc rd;
  std::memset(&rd, 0, sizeof(rd));
  rd.idx = d->idx;
  rd.orient = d->curl_orient ? nullptr : d->orient;  // the tridiagonal matrix already carries the signs
  rd.dof_map = nullptr;                              // native order
  int rc;
  if (fine)
  {
    op->mat = fine->mat;
    op->emat = fine->emat;
    op->ecoef = fine->ecoef;
    op->iso = fine->iso;
    op->n_mat = fine->n_mat;
    op->owns_coeff = false;
    op->parent = fine;
    fine->refcount++;
  }
  if ((rc = build_restriction(op, &rd)) || (rc = upload(ctx, T.data(), T.size(), &op->dense_T)) ||
      (!fine && (rc = set_coeff(op, d->coeff_ctx, d->coeff_ctx_bytes))))
  {
    b2p_op_destroy(op);
    return rc;
  }
  if (d->curl_orient && (rc = upload(ctx, d->curl_orient, (size_t)d->ne * P * 3, &op->curl_orient)))
  {
    b2p_op_destroy(op);
    return rc;
  }
  *out = op;
  return B2P_SUCCESS;
}
}  // namespace

int b2p_op_create_dense(b2p_ctx *ctx, b2p_geom *geom, const b2p_dense_op_desc *d, b2p_op **out)
{
  B2P_CHECK(ctx, ctx && geom && d && out, B2P_ERR_ARG, "b2p_op_create_dense: null argument");
  return create_dense(ctx, geom, d, nullptr, out);
}

// ceed::CeedOperatorCoarsen for dense-basis operators (fem/libceed/operator.cpp:525-585): same quadrature, geometry and
// coefficient as `fine`, the coarse space's tables (evaluated at the same Q points) and restriction from the descriptor.
int b2p_op_coarsen_dense(b2p_op *fine, const b2p_dense_op_desc *d, b2p_op **out)
{
  B2P_CHECK(fine ? fine->ctx : nullptr, fine && d && out, B2P_ERR_ARG, "b2p_op_coarsen_dense: null argument");
  b2p_ctx *ctx = fine->ctx;
  B2P_CHECK(ctx, fine->dense, B2P_ERR_ARG, "b2p_op_coarsen_dense: the fine operator is sum-factorised: use b2p_op_coarsen");
  B2P_CHECK(ctx, d->P <= fine->P, B2P_ERR_ARG, "b2p_op_coarsen_dense: %d coarse element dofs > %d fine ones", d->P, fine->P);
  b2p_dense_op_desc dd = *d;
  dd.kind = fine->kind;
  return create_dense(ctx, fine->geom, &dd, fine, out);
}

int b2p_op_coarsen(b2p_op *fine, const b2p_op_desc *d, b2p_op **out)
{
  B2P_CHECK(fine ? fine->ctx : nullptr, fine && d && out, B2P_ERR_ARG, "b2p_op_coarsen: null argument");
  b2p_ctx *ctx = fine->ctx;
  B2P_CHECK(ctx, !fine->dense, B2P_ERR_UNSUPPORTED, "b2p_op_coarsen: not available for dense-basis operators");
  B2P_CHECK(ctx, d->p >= 1 && d->p <= fine->p, B2P_ERR_ARG, "b2p_op_coarsen: coarse p=%d must be <= fine p=%d", d->p, fine->p);
  B2P_CHECK(ctx, d->idx && d->lsize > 0, B2P_ERR_ARG, "b2p_op_coarsen: missing restriction");
  b2p_op *op = new b2p_op;
  op->ctx = ctx;
  op->geom = fine->geom;
  fine->geom->refcount++;
  op->kind = fine->kind;
  op->p = d->p;
  op->q1d = fine->q1d;
  op->ne = fine->ne;
  op->P = elem_dofs(fine->kind, d->p);
  op->lsize = d->lsize;
  op->assembled = fine->assembled;
  // share coefficient arrays and assembled q-data with the fine operator (kept alive by refcount)
  op->mat = fine->mat;
  op->emat = fine->emat;
  op->ecoef = fine->ecoef;
  op->bcoef = fine->bcoef;
  op->bcoef_t = fine->bcoef_t;
  op->iso = fine->iso;
  op->n_mat = fine->n_mat;
  op->aq = fine->aq;
  op->aq_ncomp = fine->aq_ncomp;
  op->aq_estride = fine->aq_estride;
  op->owns_coeff = false;
  op->parent = fine;
  fine->refcount++;
  int rc;
  if ((rc = build_restriction(op, d)) || (rc = build_tables(op, d)))
  {
    b2p_op_destroy(op);
    return rc;
  }
  *out = op;
  return B2P_SUCCESS;
}

int b2p_op_apply_add_ex(b2p_op *op, double alpha, const double *x, double *y, int flags, b2p_stream s)
{
  if (!op || !x || !y) return B2P_ERR_ARG;
  const int32_t *lidx = op->lidx;
  if (flags & B2P_APPLY_MASKED)
  {
    B2P_CHECK(op->ctx, op->lidx_bc, B2P_ERR_ARG, "b2p_op_apply_add_ex: masked apply without b2p_op_set_essential");
    lidx = op->lidx_bc;
  }
  return b2p::apply_range(op, lidx, alpha, x, y, ApplyRange(), flags, (cudaStream_t)s);
}

// y0 += alpha A x0 and y1 += alpha A x1 in ONE pass over the geometry (two right-hand sides: the real and imaginary parts
// under a real preconditioner, PCMatReal, spaceoperator.cpp:1098-1105; two Krylov vectors; ...): the two vectors ride in
// adjacent element slots of the fused-complex kernel with a purely real coefficient block. Falls back to two applies when the
// operator is not eligible (dense basis, H1, assembled D, q1d > 4).
int b2p_op_apply_add_pair(b2p_op *op, double alpha, const double *x0, const double *x1, double *y0, double *y1, int flags, b2p_stream s)
{
  if (!op || !x0 || !x1 || !y0 || !y1) return B2P_ERR_ARG;
  const int32_t *lidx = op->lidx;
  if (flags & B2P_APPLY_MASKED)
  {
    B2P_CHECK(op->ctx, op->lidx_bc, B2P_ERR_ARG, "b2p_op_apply_add_pair: masked apply without b2p_op_set_essential");
    lidx = op->lidx_bc;
  }
  if (!hex_pair_apply_eligible(op))
  {
    int rc = b2p::apply_range(op, lidx, alpha, x0, y0, ApplyRange(), flags, (cudaStream_t)s);
    return rc ? rc : b2p::apply_range(op, lidx, alpha, x1, y1, ApplyRange(), flags, (cudaStream_t)s);
  }
  const b2p_op *csrc = op->parent ? op->parent : op;  // coarsened operators share the fine operator's coefficients
  if (!op->pair_zcoef || op->pair_version != csrc->coeff_version)
  {
    cudaFree(op->pair_zcoef);
    op->pair_zcoef = nullptr;
    std::vector<double> e18((size_t)18 * op->ne), z((size_t)36 * op->ne, 0.0);
    B2P_CUDA(op->ctx, cudaMemcpy(e18.data(), op->ecoef, e18.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (int e = 0; e < op->ne; e++)
      for (int i = 0; i < 9; i++)
      {
        z[(size_t)36 * e + i] = e18[(size_t)18 * e + i];
        z[(size_t)36 * e + 18 + i] = e18[(size_t)18 * e + 9 + i];
      }
    int rc = upload(op->ctx, z.data(), z.size(), &op->pair_zcoef);
    if (rc) return rc;
    op->pair_version = csrc->coeff_version;
  }
  return launch_nd_hex_apply4z(op, op->kind, lidx, op->pair_zcoef, 0, alpha, x0, x1, y0, y1, (cudaStream_t)s);
}

int b2p_op_apply_add_split(b2p_op *op, double alpha, const double *x, const double *x_ghost, double *y, double *y_ghost,
                           int64_t n_owned, int e_begin, int e_count, int flags, b2p_stream s)
{
  if (!op || !x || !y) return B2P_ERR_ARG;
  const int32_t *lidx = op->lidx;
  if (flags & B2P_APPLY_MASKED)
  {
    B2P_CHECK(op->ctx, op->lidx_bc, B2P_ERR_ARG, "b2p_op_apply_add_split: masked apply without b2p_op_set_essential");
    lidx = op->lidx_bc;
  }
  B2P_CHECK(op->ctx, e_begin >= 0 && e_begin <= op->ne && (e_count < 0 || e_begin + e_count <= op->ne), B2P_ERR_ARG,
            "b2p_op_apply_add_split: element range outside the operator");
  ApplyRange rg;
  rg.e_off = e_begin;
  rg.e_cnt = e_count;
  rg.n_owned = n_owned;
  rg.xg = x_ghost;
  rg.yg = y_ghost;
  return b2p::apply_range(op, lidx, alpha, x, y, rg, flags, (cudaStream_t)s);
}

int b2p_op_apply_add(b2p_op *op, const double *x, double *y, b2p_stream s) { return b2p_op_apply_add_ex(op, 1.0, x, y, 0, s); }

int b2p_op_apply(b2p_op *op, const double *x, double *y, b2p_stream s)
{
  if (!op || !x || !y) return B2P_ERR_ARG;
  B2P_CUDA(op->ctx, cudaMemsetAsync(y, 0, sizeof(double) * op->lsize, (cudaStream_t)s));
  return b2p_op_apply_add_ex(op, 1.0, x, y, 0, s);
}

int b2p_op_set_essential(b2p_op *op, const int32_t *ess_ldofs, int64_t n)
{
  if (!op || (n > 0 && !ess_ldofs)) return B2P_ERR_ARG;
  std::vector<char> mark((size_t)op->lsize, 0);
  for (int64_t i = 0; i < n; i++)
  {
    B2P_CHECK(op->ctx, ess_ldofs[i] >= 0 && ess_ldofs[i] < op->lsize, B2P_ERR_ARG, "essential dof %d outside the L-vector",
              ess_ldofs[i]);
    mark[ess_ldofs[i]] = 1;
  }
  std::vector<int32_t> lidx((size_t)op->ne * op->PS);
  B2P_CUDA(op->ctx, cudaMemcpy(lidx.data(), op->lidx, lidx.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  for (auto &g : lidx)
  {
    if (g == (int32_t)B2P_SKIP_IDX) continue;
    const int32_t d = g >= 0 ? g : -1 - g;
    if (mark[d]) g = B2P_SKIP_IDX;
  }
  cudaFree(op->lidx_bc);
  op->lidx_bc = nullptr;
  op->ess_n = 0;
  op->ess_hash = 0;
  for (int64_t d = 0; d < op->lsize; d++)
    if (mark[d])
    {
      op->ess_n++;
      op->ess_hash += b2p::ess_mix((uint64_t)d);
    }
  return upload(op->ctx, lidx.data(), lidx.size(), &op->lidx_bc);
}

int b2p_op_diag_add(b2p_op *op, double *diag, b2p_stream s)
{
  if (!op || !diag) return B2P_ERR_ARG;
  if (op->dense) return launch_dense_diag(op, diag, (cudaStream_t)s);
  if (op->kind == B2P_H1_DIFFUSION) return launch_h1_hex_diag(op, diag, (cudaStream_t)s);
  if (op->kind == B2P_RT_MASS) return launch_rt_hex_diag(op, diag, (cudaStream_t)s);
  return launch_nd_hex_diag(op, diag, (cudaStream_t)s);
}

int b2p_op_set_coeff(b2p_op *op, const void *blob, size_t bytes)
{
  if (!op) return B2P_ERR_ARG;
  op->coeff_version++;
  B2P_CHECK(op->ctx, op->parent == nullptr, B2P_ERR_ARG, "b2p_op_set_coeff: set the coefficient on the fine operator");
  int rc = set_coeff(op, blob, bytes);
  if (rc) return rc;
  if (op->assembled) return assemble_qdata(op);
  return B2P_SUCCESS;
}

int64_t b2p_op_lsize(b2p_op *op) { return op ? op->lsize : 0; }

int64_t b2p_op_algorithmic_bytes(b2p_op *op)
{
  if (!op) return 0;
  // x read once + y written once per unique dof, 4-byte index per element dof, geometry.
  const int64_t Q = op->geom->Q;
  if (op->dense)  // + the tables once (L2 resident)
    return 16 * op->lsize + (int64_t)op->ne * (4 * (int64_t)op->PS + 80 * Q + 144) + 8 * (int64_t)op->dense_Rpad * op->dense_Ppad;
  const int64_t per_point = op->assembled ? op->aq_ncomp : 10;
  // q-data, or the 8 vertices (192 bytes) where the element kernel evaluates a trilinear geometry in place
  const int64_t geom_bytes = (choose_hex_kernel(op, 0) == HexKernel::ND6 && nd_hex_apply6_reads_nodes(op)) ? 192 : 8 * per_point * Q;
  // + per-element coefficient block: 144 bytes (two 3x3 tensors), 288 for block operators (four)
  return 16 * op->lsize + (int64_t)op->ne * (4 * (int64_t)op->PS + geom_bytes + (op->assembled ? 0 : (op->bcoef ? 288 : 144)));
}

// One operator for a real sum  sum_t c_t A_t  of sum-factorised ND operators over the same geometry, space and essential
// set (BuildParSumOperator(a0 K + a1 C + a2 M), /root/reference/palace/linalg/rap.cpp:764-829, where every term is applied
// separately and AXPY'd): the terms differ only in their pointwise coefficient, so the sum is the SAME element kernel with the
// per-element tensors  mass = sum_t c_t * (mass tensor of term t),  curl = sum_t c_t * (curl tensor of term t)  -- one
// launch and one geometry stream instead of one per term, in every smoother step that applies the system matrix.
static int sum_fill_coefficients(b2p_op *sum, int n_terms, b2p_op *const *ops, const double *coefs)
{
  b2p_ctx *ctx = sum->ctx;
  const int ne = sum->ne;
  std::vector<double> e18((size_t)18 * ne), z((size_t)18 * ne, 0.0);
  bool block = false;
  for (int t = 0; t < n_terms; t++) block = block || ops[t]->bcoef;
  if (block)
  {
    // a mixed curl term makes the sum a block operator: each term's tensors go to their slots of {Cm, Ck, Cw, Cx}
    std::vector<double> b36((size_t)36 * ne), z36((size_t)36 * ne, 0.0);
    for (int t = 0; t < n_terms; t++)
    {
      const b2p_op *o = ops[t];
      if (o->bcoef)
      {
        B2P_CUDA(ctx, cudaMemcpy(b36.data(), o->bcoef, b36.size() * sizeof(double), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < z36.size(); i++) z36[i] += coefs[t] * b36[i];
        continue;
      }
      B2P_CUDA(ctx, cudaMemcpy(e18.data(), o->ecoef, e18.size() * sizeof(double), cudaMemcpyDeviceToHost));
      const bool m = (o->kind == B2P_ND_MASS || o->kind == B2P_CURLCURL_MASS), k = (o->kind == B2P_CURLCURL || o->kind == B2P_CURLCURL_MASS);
      for (int e = 0; e < ne; e++)
        for (int i = 0; i < 9; i++)
        {
          if (m) z36[(size_t)36 * e + i] += coefs[t] * e18[(size_t)18 * e + i];
          if (k) z36[(size_t)36 * e + 9 + i] += coefs[t] * e18[(size_t)18 * e + 9 + i];
        }
    }
    sum->kind = B2P_ND_BLOCK;
    sum->iso = false;
    return set_block(sum, z36);
  }
  bool mass = false, curl = false;
  for (int t = 0; t < n_terms; t++)
  {
    const b2p_op *o = ops[t];
    B2P_CUDA(ctx, cudaMemcpy(e18.data(), o->ecoef, e18.size() * sizeof(double), cudaMemcpyDeviceToHost));
    const bool m = (o->kind == B2P_ND_MASS || o->kind == B2P_CURLCURL_MASS), k = (o->kind == B2P_CURLCURL || o->kind == B2P_CURLCURL_MASS);
    mass = mass || m;
    curl = curl || k;
    for (int e = 0; e < ne; e++)
      for (int i = 0; i < 9; i++)
      {
        if (m) z[(size_t)18 * e + i] += coefs[t] * e18[(size_t)18 * e + i];
        if (k) z[(size_t)18 * e + 9 + i] += coefs[t] * e18[(size_t)18 * e + 9 + i];
      }
  }
  sum->kind = mass && curl ? B2P_CURLCURL_MASS : (mass ? B2P_ND_MASS : B2P_CURLCURL);
  if (!(mass && curl))  // single-part kinds read whichever part they use: keep both filled
    for (int e = 0; e < ne; e++)
      for (int i = 0; i < 9; i++)
      {
        if (!mass) z[(size_t)18 * e + i] = z[(size_t)18 * e + 9 + i];
        if (!curl) z[(size_t)18 * e + 9 + i] = z[(size_t)18 * e + i];
      }
  sum->iso = true;
  for (size_t m = 0; m < (size_t)2 * ne && sum->iso; m++)
    for (int t = 0; t < 9; t++)
    {
      const double v = z[9 * m + t], d = z[9 * m];
      if ((t % 4 == 0) ? (v != d) : (v != 0.0)) sum->iso = false;
    }
  std::vector<int32_t> emat((size_t)2 * ne);
  for (int e = 0; e < ne; e++)
  {
    emat[2 * (size_t)e] = 2 * e;
    emat[2 * (size_t)e + 1] = 2 * e + 1;
  }
  cudaFree(sum->mat);
  cudaFree(sum->emat);
  cudaFree(sum->ecoef);
  sum->mat = nullptr;
  sum->emat = nullptr;
  sum->ecoef = nullptr;
  sum->n_mat = 2 * ne;
  int rc;
  if ((rc = upload(ctx, z.data(), z.size(), &sum->mat)) || (rc = upload(ctx, emat.data(), emat.size(), &sum->emat)) ||
      (rc = upload(ctx, z.data(), z.size(), &sum->ecoef)))
    return rc;
  return B2P_SUCCESS;
}

int b2p_op_create_sum(b2p_ctx *ctx, int n_terms, b2p_op *const *ops, const double *coefs, b2p_op **out)
{
  B2P_CHECK(ctx, ctx && ops && coefs && out && n_terms >= 1, B2P_ERR_ARG, "b2p_op_create_sum: bad argument");
  const b2p_op *o0 = ops[0];
  const size_t nidx = (size_t)o0->ne * o0->PS;
  std::vector<int32_t> a(nidx), b(nidx);
  const bool dense = o0 && o0->dense;  // dense-basis terms (tets, prisms, faces) fuse the same way: one stacked table, summed tensors
  for (int t = 0; t < n_terms; t++)
  {
    const b2p_op *o = ops[t];
    // sum-factorised block operators (mixed curl kinds) fuse too; dense mixed terms do not
    B2P_CHECK(ctx, o && o->dense == dense && !o->assembled && ((o->kind >= B2P_CURLCURL && o->kind <= B2P_CURLCURL_MASS && o->ecoef) || o->bcoef),
              B2P_ERR_UNSUPPORTED, "b2p_op_create_sum: term %d is not an ND curl-curl / mass / mixed curl operator with on-the-fly coefficients", t);
    B2P_CHECK(ctx, o->geom == o0->geom && o->p == o0->p && o->q1d == o0->q1d && o->ne == o0->ne && o->lsize == o0->lsize && o->PS == o0->PS &&
                       o->P == o0->P && o->dense_Ppad == o0->dense_Ppad && (o->curl_orient != nullptr) == (o0->curl_orient != nullptr) &&
                       (o->lidx_bc != nullptr) == (o0->lidx_bc != nullptr),
              B2P_ERR_UNSUPPORTED, "b2p_op_create_sum: term %d lives on another geometry / space", t);
    if (dense && o->curl_orient && t > 0)
    {
      const size_t nco = (size_t)o0->ne * o0->P * 3;
      std::vector<int8_t> c0(nco), ct(nco);
      B2P_CUDA(ctx, cudaMemcpy(c0.data(), o0->curl_orient, nco, cudaMemcpyDeviceToHost));
      B2P_CUDA(ctx, cudaMemcpy(ct.data(), o->curl_orient, nco, cudaMemcpyDeviceToHost));
      B2P_CHECK(ctx, c0 == ct, B2P_ERR_UNSUPPORTED, "b2p_op_create_sum: term %d has another orientation of its element dofs", t);
    }
    for (int which = 0; which < 2; which++)
    {
      const int32_t *p0 = which ? o0->lidx_bc : o0->lidx, *pt = which ? o->lidx_bc : o->lidx;
      if (!p0 || t == 0) continue;
      B2P_CUDA(ctx, cudaMemcpy(a.data(), p0, nidx * sizeof(int32_t), cudaMemcpyDeviceToHost));
      B2P_CUDA(ctx, cudaMemcpy(b.data(), pt, nidx * sizeof(int32_t), cudaMemcpyDeviceToHost));
      B2P_CHECK(ctx, a == b, B2P_ERR_UNSUPPORTED, "b2p_op_create_sum: term %d has another restriction / essential set", t);
    }
  }
  b2p_op *op = new b2p_op;
  op->ctx = ctx;
  op->geom = o0->geom;
  o0->geom->refcount++;
  op->p = o0->p;
  op->q1d = o0->q1d;
  op->ne = o0->ne;
  op->P = o0->P;
  op->PS = o0->PS;
  op->lsize = o0->lsize;
  op->h_tab = o0->h_tab;
  op->tab_dev = o0->tab_dev;
  op->tab_scale = o0->tab_scale;
  op->ess_n = o0->ess_n;  // the masked restriction is copied below: same essential set
  op->ess_hash = o0->ess_hash;
  int rc = 0;
  auto dup = [&](const auto *src, size_t n, auto **dst) -> int
  {
    using T = std::remove_const_t<std::remove_pointer_t<decltype(src)>>;
    if (!src) return B2P_SUCCESS;
    if (cudaMalloc((void **)dst, n * sizeof(T)) != cudaSuccess) return B2P_ERR_CUDA;
    return cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyDeviceToDevice) == cudaSuccess ? B2P_SUCCESS : B2P_ERR_CUDA;
  };
  if (dense)
  {
    // stacked table of the sum: the value block of a term that has one, then the curl block of a term that has one (the
    // terms tabulate the same element at the same points, so whichever term supplies a block supplies the same numbers)
    const b2p_op *tu = nullptr, *tc = nullptr;
    for (int t = 0; t < n_terms; t++)
    {
      if (!tu && ops[t]->dense_row_u >= 0 && ops[t]->kind != B2P_CURLCURL) tu = ops[t];
      if (!tc && ops[t]->dense_row_c >= 0 && ops[t]->kind != B2P_ND_MASS) tc = ops[t];
    }
    const int Q = o0->geom->Q, Ppad = o0->dense_Ppad, blk = 3 * Q;
    // every term must tabulate the SAME basis: compare each term's blocks with the ones taken over
    {
      std::vector<double> ref((size_t)blk * Ppad), cmp((size_t)blk * Ppad);
      for (int which = 0; which < 2 && !rc; which++)
      {
        const b2p_op *src = which ? tc : tu;
        if (!src) continue;
        const int srow = which ? src->dense_row_c : src->dense_row_u;
        if (cudaMemcpy(ref.data(), src->dense_T + (size_t)srow * Ppad, sizeof(double) * ref.size(), cudaMemcpyDeviceToHost) != cudaSuccess) rc = B2P_ERR_CUDA;
        for (int t = 0; t < n_terms && !rc; t++)
        {
          const int trow = which ? ops[t]->dense_row_c : ops[t]->dense_row_u;
          if (ops[t] == src || trow < 0) continue;
          if (cudaMemcpy(cmp.data(), ops[t]->dense_T + (size_t)trow * Ppad, sizeof(double) * cmp.size(), cudaMemcpyDeviceToHost) != cudaSuccess)
            rc = B2P_ERR_CUDA;
          else if (cmp != ref)
          {
            set_error(ctx, "b2p_op_create_sum: term %d tabulates another basis (its %s table differs)", t, which ? "derivative" : "value");
            b2p_op_destroy(op);
            return B2P_ERR_UNSUPPORTED;
          }
        }
      }
    }
    op->dense = true;
    op->dense_Ppad = Ppad;
    op->dense_row_u = tu ? 0 : -1;
    op->dense_row_c = tc ? (tu ? blk : 0) : -1;
    op->dense_Rpad = (((tu ? blk : 0) + (tc ? blk : 0)) + 7) & ~7;
    std::vector<double> T((size_t)op->dense_Rpad * Ppad, 0.0);
    if (tu && cudaMemcpy(T.data(), tu->dense_T + (size_t)tu->dense_row_u * Ppad, sizeof(double) * blk * Ppad, cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = B2P_ERR_CUDA;
    if (!rc && tc &&
        cudaMemcpy(T.data() + (size_t)op->dense_row_c * Ppad, tc->dense_T + (size_t)tc->dense_row_c * Ppad, sizeof(double) * blk * Ppad,
                   cudaMemcpyDeviceToHost) != cudaSuccess)
      rc = B2P_ERR_CUDA;
    if (!rc) rc = upload(ctx, T.data(), T.size(), &op->dense_T);
    if (!rc) rc = dup(o0->curl_orient, (size_t)o0->ne * o0->P * 3, &op->curl_orient);
  }
  if (rc || (rc = dup(o0->lidx, nidx, &op->lidx)) || (rc = dup(o0->lidx_bc, nidx, &op->lidx_bc)) ||
      (rc = dup(o0->tab, o0->h_tab.size(), &op->tab)) || (rc = sum_fill_coefficients(op, n_terms, ops, coefs)))
  {
    set_error(ctx, "b2p_op_create_sum: device allocation / copy failed");
    b2p_op_destroy(op);
    return rc;
  }
  *out = op;
  return B2P_SUCCESS;
}

// New coefficients c_t (next frequency of a sweep) for an operator made by b2p_op_create_sum from the same terms.
int b2p_op_sum_set_coefficients(b2p_op *sum, int n_terms, b2p_op *const *ops, const double *coefs)
{
  if (!sum || !ops || !coefs || n_terms < 1) return B2P_ERR_ARG;
  return sum_fill_coefficients(sum, n_terms, ops, coefs);
}

void b2p_op_destroy(b2p_op *op)
{
  if (!op) return;
  if (--op->refcount > 0) return;
  cudaFree(op->lidx);
  cudaFree(op->lidx_bc);
  cudaFree(op->tab);
  cudaFree(op->dense_T);
  cudaFree(op->curl_orient);
  cudaFree(op->pair_zcoef);
  if (op->parent)
  {
    b2p_op_destroy(op->parent);
  }
  else
  {
    cudaFree(op->mat);
    cudaFree(op->emat);
    cudaFree(op->ecoef);
    cudaFree(op->bcoef);
    cudaFree(op->bcoef_t);
    cudaFree(op->aq);
  }
  b2p_geom_destroy(op->geom);
  delete op;
}

void b2p_ctx_destroy(b2p_ctx *ctx)
{
  if (!ctx) return;
  cudaFree(ctx->d_red);
  cudaFree(ctx->d_sink);
  cudaFreeHost(ctx->h_red);
  if (ctx->graph_stream) cudaStreamDestroy(ctx->graph_stream);
  delete ctx;
}

}  // extern "C"
