// Internal declarations shared by the b2p translation units (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/b2p.h"

struct ncclComm;

namespace b2p
{

void set_error(b2p_ctx *ctx, const char *fmt, ...);

#define B2P_CUDA(ctx, call)                                                                              \
  do                                                                                                     \
  {                                                                                                      \
    cudaError_t e__ = (call);                                                                            \
    if (e__ != cudaSuccess)                                                                              \
    {                                                                                                    \
      b2p::set_error(ctx, "%s:%d CUDA error %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return B2P_ERR_CUDA;                                                                               \
    }                                                                                                    \
  } while (0)

#define B2P_CHECK(ctx, cond, code, ...)     \
  do                                        \
  {                                         \
    if (!(cond))                            \
    {                                       \
      b2p::set_error(ctx, __VA_ARGS__);     \
      return code;                          \
    }                                       \
  } while (0)

template <typename T>
int upload(b2p_ctx *ctx, const T *host, size_t n, T **dptr);

// Kernel launch and dynamic shared memory go through these two macros so that the kernel SOURCES can also be
// compiled for the host-thread SIMT emulation of tests/emu (test infrastructure: B2P_EMU is defined only by
// tests/emu/Makefile, never for libb2p.so). In the product build they expand to the plain CUDA constructs.
#ifdef B2P_EMU
#define B2P_LAUNCH(kern, grid, block, shmem, stream, ...) \
  ::cuda_emu::launch(dim3(grid), dim3(block), (size_t)(shmem), [=]() { kern(__VA_ARGS__); })
#define B2P_LAUNCH_PDL(kern, grid, block, shmem, stream, ...) B2P_LAUNCH(kern, grid, block, shmem, stream, __VA_ARGS__)
#define B2P_DYN_SMEM(type, name) type *name = reinterpret_cast<type *>(::cuda_emu::dyn_smem())
#define B2P_DYN_SMEM_ALIGNED16(type, name) B2P_DYN_SMEM(type, name)
#else
// launch that may overlap the tail of the previous kernel in the stream (the kernel must call griddep_wait() before it
// touches anything the predecessor writes)
#define B2P_LAUNCH_PDL(kern, grid, block, shmem, strm__, ...)                          \
  do                                                                                   \
  {                                                                                    \
    cudaLaunchConfig_t cfg__ = {};                                                     \
    cfg__.gridDim = dim3(grid);                                                        \
    cfg__.blockDim = dim3(block);                                                      \
    cfg__.dynamicSmemBytes = (shmem);                                                  \
    cfg__.stream = (strm__);                                                           \
    cudaLaunchAttribute attr__[1];                                                     \
    attr__[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                 \
    attr__[0].val.programmaticStreamSerializationAllowed = 1;                          \
    cfg__.attrs = attr__;                                                              \
    cfg__.numAttrs = 1;                                                                \
    cudaLaunchKernelEx(&cfg__, kern, __VA_ARGS__);                                     \
  } while (0)
#define B2P_LAUNCH(kern, grid, block, shmem, stream, ...) kern<<<(grid), (block), (shmem), (stream)>>>(__VA_ARGS__)
#define B2P_DYN_SMEM(type, name) extern __shared__ type name[]
#define B2P_DYN_SMEM_ALIGNED16(type, name) extern __shared__ __align__(16) type name[]
#endif

}  // namespace b2p

struct b2p_ctx
{
  int device = 0;
  int sm_count = 0;
  int rank = 0, nranks = 1;
  ncclComm *comm = nullptr;
  cudaStream_t stream = 0;  // stream of the linear algebra / solver layer (b2p_ctx_set_stream)
  cudaStream_t graph_stream = nullptr;  // internal BLOCKING stream for graph capture when `stream` is the legacy stream
  std::string last_error;
  // scratch for reductions (dot products): device partials + pinned host result
  double *d_red = nullptr;
  double *h_red = nullptr;
  size_t red_cap = 0;
  // sink of the branch-free scatter (nd_hex_apply6_kernel): masked restriction entries add 0.0 to a per-thread slot here
  double *d_sink = nullptr;
  static constexpr int SINK_SLOTS = 1 << 16;
  // what the last persistent element kernel launched on this context was (b2p_ctx_last_launch; host-side stores only)
  b2p_launch_info last_launch = {};
};

// Geometry q-data of one element block, device resident.
//   qd[ne][10][Q]: {w detJ, (adjJ^T/detJ)[9] column-major}, points in qslot() order; attr[ne] int32 (1-based).
// (The reference stores attr as an 11th double per point, mesh.cpp:188-195; it is constant per
// element, so it is kept once per element here.)
// Storage slot of quadrature point (qx,qy,qz) inside one component row of q-data: x SLOWEST, so that
// a thread owning a (qy,qz) line reads consecutive words across the warp (conflict-free LDS, see
// b2p_hex_nd2.cu). Logical point order everywhere else is x fastest (basis.cpp:18-19).
__host__ __device__ inline int qslot(int q, int qx, int qy, int qz) { return qy + q * (qz + q * qx); }
__host__ __device__ inline int qslot_of(int q, int iq) { return qslot(q, iq % q, (iq / q) % q, iq / (q * q)); }

// Sentinel in the signed lexicographic restriction: dof masked out (essential BC) -> gathers 0, no scatter.
#define B2P_SKIP_IDX (-2147483647 - 1)

struct b2p_geom
{
  b2p_ctx *ctx = nullptr;
  int ne = 0, q1d = 0, Q = 0;  // q1d == 0: general (non-tensor) point set in plain order
  double *qd = nullptr;
  int32_t *attr = nullptr;
  // trilinear meshes (b2p_geom_create_hex with mesh_order 1) only, else null / empty: the element vertices xe[ne][3][8] and the
  // host copies of the 1-D tables they were expanded with (nodeB[q1d][2], nodeG[q1d][2], qw1d[q1d]), from which a kernel can
  // evaluate the geometry in place of reading qd (b2p_geom1.cuh)
  double *xe = nullptr;
  std::vector<double> h_nodeB, h_nodeG, h_qw;
  int refcount = 1;
};

struct b2p_op
{
  b2p_ctx *ctx = nullptr;
  b2p_geom *geom = nullptr;  // shared (refcounted)
  int kind = 0, p = 0, q1d = 0, ne = 0, P = 0;
  int PS = 0;  // restriction row stride: P padded to a multiple of 4 (16-byte rows for TMA bulk copies)
  int64_t lsize = 0;
  int assembled = 0;
  // restriction in LEXICOGRAPHIC element order with the sign folded in:
  // lidx[e][l] >= 0 -> +x[lidx], < 0 -> -x[-1-lidx]   (layout [ne][P])
  int32_t *lidx = nullptr;
  int32_t *lidx_bc = nullptr;  // same with essential dofs replaced by B2P_SKIP_IDX (optional)
  int64_t ess_n = -1;          // fingerprint of the essential set behind lidx_bc: number of distinct dofs, order-free hash
  uint64_t ess_hash = 0;
  std::vector<double> h_tab;   // host copy of the packed 1-D tables (kernel parameter block)
  // 1-D tables (device): Bo[q1d][p], Bc[q1d][p+1], Gc[q1d][p+1]
  double *tab = nullptr;  // packed Bo | Bc | Gc
  // coefficients: material tables + per-element material index for the two parts
  double *mat = nullptr;       // [n_mat_total][9] column-major (mass part first, then curl part)
  int32_t *emat = nullptr;     // [ne][2] indices into mat (value part, derivative part)
  int n_mat = 0;
  bool iso = false;            // every material matrix is c * I
  // mirror symmetry of the 1-D tables (nd_tables_symmetric), computed on first use: the largest deviation from it and the
  // largest |entry|; tab_dev < 0: not computed yet
  double tab_dev = -1.0, tab_scale = 0.0;
  double *ecoef = nullptr;     // [ne][18] per-element coefficient matrices (TMA-friendly copy of mat[emat])
  // assembled q-data (optional): aq[ne][ncomp][Q], symmetric 6 per part
  double *aq = nullptr;
  int aq_ncomp = 0;
  int64_t aq_estride = 0;  // doubles per element (even, so every element block is 16-byte aligned for TMA)
  // dense-basis (non-tensor) operators (b2p_dense.cu)
  bool dense = false;
  double *dense_T = nullptr;   // [Rpad][Ppad] stacked interp/deriv tables, zero padded
  int dense_Ppad = 0, dense_Rpad = 0, dense_row_u = -1, dense_row_c = -1;
  int8_t *curl_orient = nullptr;  // [ne][P][3] tridiagonal orientation (ND tets/prisms p >= 2) or null
  // block operators (the mixed kinds B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL on hexes, and sums that contain one): per element the
  // four 3x3 tensors {Cm value->value, Ck curl->curl, Cw value->curl, Cx curl->value}, column-major, and the same block for
  // the transposed operator (every tensor transposed, Cw and Cx swapped). Null for every other operator.
  double *bcoef = nullptr;     // [ne][36]
  double *bcoef_t = nullptr;   // [ne][36]
  double *pair_zcoef = nullptr;  // [ne][36] {mass, 0, curl, 0}: coefficient block of the two-vector apply (built on first use)
  int coeff_version = 0, pair_version = -1;  // b2p_op_set_coeff bumps coeff_version (coarsened operators follow their parent's)
  bool owns_coeff = true;  // coarsened operators share the fine operator's coefficient arrays
  b2p_op *parent = nullptr;
  int refcount = 1;
};

struct b2p_interp
{
  b2p_ctx *ctx = nullptr;
  int ne = 0, in_P = 0, out_P = 0, in_PS = 0, out_PS = 0, ncomp = 0;
  int64_t in_lsize = 0, out_lsize = 0;
  int32_t *in_lidx = nullptr, *out_lidx = nullptr;  // signed lexicographic restrictions [ne][PS]
  int32_t *out_owner_lidx = nullptr;  // out_lidx with every dof kept in ONE element only (owner-computes Mult), or null
  double *inv_mult = nullptr;                       // [out_lsize] 1 / (local elements touching the dof)
  // per component: dims and matrix offsets into `mats`
  int in_off[3], in_n[3][3], out_off[3], out_n[3][3], mat_off[3][3];
  int ident[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  double *mats = nullptr;
  int n_mats = 0;
  // element-dense variant (any element type, b2p_interp_create_dense): one [out_P][in_P] matrix, native dof order,
  // optional tridiagonal transformations of the two restrictions
  bool dense = false;
  double *dmat = nullptr;
  int8_t *in_co = nullptr, *out_co = nullptr;  // [ne][P][3] rows or null
  // hexahedral discrete curl ND_p -> RT_{p-1} (b2p_interp_create_curl_hex) when curl_p > 0: in = ND, out = RT, both lexicographic
  int curl_p = 0;
  double *curl_D = nullptr;  // [p][p+1] closed-basis derivative at the open nodes
};

namespace b2p
{
// Element sub-range and owned/ghost split of one apply (defaults: all elements, no ghosts).
struct ApplyRange
{
  int e_off = 0, e_cnt = -1;
  long long n_owned = -1;      // dofs below this index live in x / y, the rest in xg / yg
  const double *xg = nullptr;
  double *yg = nullptr;
  // peer-memory halo: elements >= wait_from_elem need the ghost values; before touching them a warp
  // waits until flags[k] >= expect[k] for k < wait_n (acquire at system scope)
  const unsigned long long *wait_flags = nullptr, *wait_expect = nullptr;
  int wait_n = 0, wait_from_elem = 0;
  bool pdl = false;  // launch with programmatic stream serialisation (kernels that call griddep_wait() only)
};
// Internal kind of the sum-factorised ND kernels: the pointwise block form of b2p_op::bcoef,
//   out_val = w detJ A^T (Cm A u + Cx Jd c),   out_curl = w detJ Jd^T (Ck Jd c + Cw A u)   (A = J^-T, Jd = J / detJ).
constexpr int B2P_ND_BLOCK = 16;
// Operators that need B2P_APPLY_TRANSPOSE for their transpose (the mixed kinds and block sums).
inline bool op_nonsymmetric(const b2p_op *op)
{
  return op->kind == B2P_ND_WEAKCURL || op->kind == B2P_ND_MIXEDCURL || op->bcoef != nullptr;
}
// Store the launch record of a persistent element kernel on its context (b2p_ctx_last_launch). `block` / `cplx` name the form,
// `nodes` says that the kernel evaluated the geometry from the element vertices instead of reading the stored q-data.
inline void record_launch(b2p_ctx *c, const char *kernel, bool block, bool cplx, int max_grid, int grid, int workers, int elems_per_batch,
                          int64_t batches, bool nodes = false)
{
  b2p_launch_info &r = c->last_launch;
  snprintf(r.kernel, sizeof(r.kernel), "%s%s%s", kernel, block ? ":block" : "", cplx ? ":cplx" : "");
  snprintf(r.geom, sizeof(r.geom), "%s", nodes ? "nodes" : "qdata");
  r.max_grid = max_grid;
  r.grid = grid;
  r.workers = workers;
  r.elems_per_batch = elems_per_batch;
  r.batches = batches;
  r.seq++;
}
// Elements [rg.e_off, rg.e_off + range_count) of an apply range; <= 0: nothing to launch.
inline int range_count(const b2p_op *op, const ApplyRange &rg) { return rg.e_cnt < 0 ? op->ne - rg.e_off : rg.e_cnt; }
// Does the L-vector come in two pieces (owned part in x / y, ghosts in xg / yg)?
inline bool range_split(const b2p_op *op, const ApplyRange &rg) { return rg.xg || rg.yg || (rg.n_owned >= 0 && rg.n_owned < op->lsize); }
// The owned/ghost split of an apply range on a kernel's params struct (ApplyRange(): one piece).
template <typename Prm>
void set_split(Prm &prm, const b2p_op *op, const ApplyRange &rg)
{
  prm.sp.n_owned = rg.n_owned < 0 ? op->lsize : rg.n_owned;
  prm.sp.xg = rg.xg;
  prm.sp.yg = rg.yg;
}
// The split and the peer-memory halo wait (ApplyRange(): one piece, no wait).
template <typename Prm>
void set_split_wait(Prm &prm, const b2p_op *op, const ApplyRange &rg)
{
  set_split(prm, op, rg);
  prm.wait_flags = rg.wait_flags;
  prm.wait_expect = rg.wait_expect;
  prm.wait_n = rg.wait_n;
  prm.wait_from_elem = rg.wait_from_elem;
}
// The first `rows` rows of the packed 1-D tables Bo[q][p] | Bc[q][p+1] | Gc[q][p+1] into a kernel's parameter block; a null
// destination skips that table.
inline void copy_tables(const double *h_tab, int p, int q, int rows, double *Bo, double *Bc, double *Gc)
{
  const int n = p + 1;
  for (int i = 0; Bo && i < rows * p; i++) Bo[i] = h_tab[i];
  for (int i = 0; Bc && i < rows * n; i++) Bc[i] = h_tab[q * p + i];
  for (int i = 0; Gc && i < rows * n; i++) Gc[i] = h_tab[q * p + q * n + i];
}
// Allow `kern` `shmem` bytes of dynamic shared memory and, with carveout >= 0, set its preferred shared-memory carveout (percent
// or a cudaSharedmemCarveout value). The attributes belong to the device current at the call, so this runs once per (kernel, device).
int configure_kernel_once(b2p_ctx *ctx, const void *kern, size_t shmem, int carveout = -1);
template <typename K>
int configure_kernel(b2p_ctx *ctx, K *kern, size_t shmem, int carveout = -1)
{
  return configure_kernel_once(ctx, (const void *)kern, shmem, carveout);
}
// Launch a persistent element kernel: max_grid CTAs clamped to the CTAs the batches fill (`workers` per CTA each walk batch,
// batch + W, ...), the launch record (record_launch's fields), programmatic stream serialisation only with `pdl` (kernels that
// call griddep_wait()).
template <typename K, typename Prm>
int launch_persistent(K *kern, const Prm &prm, int threads, size_t shmem, cudaStream_t s, bool pdl, b2p_ctx *c, const char *kernel,
                      bool block, bool cplx, int max_grid, int workers, int elems_per_batch, int64_t batches, bool nodes = false)
{
  int grid = max_grid;
  if (grid > (batches + workers - 1) / workers) grid = (int)((batches + workers - 1) / workers);
  record_launch(c, kernel, block, cplx, max_grid, grid, workers, elems_per_batch, batches, nodes);
  if (pdl)
    B2P_LAUNCH_PDL(kern, grid, threads, shmem, s, prm);
  else
    B2P_LAUNCH(kern, grid, threads, shmem, s, prm);
  B2P_CUDA(c, cudaGetLastError());
  return B2P_SUCCESS;
}
// The element kernel of an apply (choose_hex_kernel, b2p_core.cu).
enum class HexKernel
{
  DENSE,
  ND_SIMPLE,
  ND4,
  ND5,
  ND6,
  ND7,
  H1_SIMPLE,
  H1V3,
  RT_SIMPLE,
  RT7
};
HexKernel choose_hex_kernel(b2p_op *op, int flags);
// The one-pass kernel of a complex sum of n_terms operators like `op` (b2p_complex.cu plans the sum).
enum class HexComplexKernel
{
  NONE,
  ND4Z,
  ND7Z
};
HexComplexKernel choose_hex_complex_kernel(b2p_op *op, int n_terms);
// Can b2p_op_apply_add_pair run the two vectors through one nd_hex_apply4_kernel<CPLX> launch?
bool hex_pair_apply_eligible(b2p_op *op);
// Kernel launchers (defined in the .cu files).
int launch_nd_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                        bool transpose = false);
int launch_nd_hex_apply4(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s);
int launch_nd_hex_apply5(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s);
bool nd_hex_apply5_eligible(b2p_op *op);
int launch_nd_hex_apply6(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                         bool transpose = false);
bool nd_hex_apply6_eligible(b2p_op *op);
// Does nd_hex_apply6_kernel, when choose_hex_kernel sends op to it, evaluate the geometry from the vertices of a trilinear mesh
// (the symmetric kinds at p = 3) instead of reading the stored q-data?
bool nd_hex_apply6_reads_nodes(const b2p_op *op);
// Are the packed 1-D tables Bo | Bc | Gc mirror-symmetric (Bo, Bc even, Gc odd about the centre) to within rel_tol times their
// largest entry? The kernels that store half the rows or read mirrored entries through one value need it. The second form
// reads op's tables through the deviation cached on op.
bool nd_tables_symmetric(const double *tab, int p, int q, double rel_tol);
bool nd_tables_symmetric(b2p_op *op, double rel_tol);
int launch_nd_hex_apply7(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                         bool transpose = false);
bool nd_hex_apply7_eligible(b2p_op *op);
// complex apply on nd_hex_apply7_kernel (p = 2 ... 6 for B2P_ND_BLOCK, 4 ... 6 for the symmetric kinds): coef is the 36-double
// {mass Re, mass Im, curl Re, curl Im} block per element, or the real four-tensor block with coef_i the imaginary one;
// y_r + i y_i += alpha (D_r + sgn i D_i) (x_r + i x_i) per element
int launch_nd_hex_apply7z(b2p_op *op, int kind, const int32_t *lidx, const double *coef, const double *coef_i, int has_imag, double sgn,
                          double alpha, const double *xr, const double *xi, double *yr, double *yi, cudaStream_t s);
// fused complex apply (b2p_hex_nd4.cu): both parts of a split complex vector in one pass over the geometry
bool nd_hex_apply4z_eligible(const b2p_op *op);
int launch_nd_hex_apply4z(b2p_op *op, int kind, const int32_t *lidx, const double *zcoef, int has_imag, double alpha, const double *xr,
                          const double *xi, double *yr, double *yi, cudaStream_t s);
// Does the op's masked restriction (b2p_op_set_essential) eliminate exactly this set of L dofs?  (No mask <=> empty set.)
bool op_essential_matches(const b2p_op *op, const int32_t *ess_ldofs, int64_t n);
int apply_range(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, int flags,
                cudaStream_t s);
int launch_nd_hex_diag(b2p_op *op, double *diag, cudaStream_t s);
// Raviart-Thomas mass (b2p_hex_flux.cu, the mixed mass with RT as trial and test space): flux_hex_mixed7_kernel with `rt7`, the
// cross-check kernel otherwise
bool rt_hex_apply7_eligible(b2p_op *op);
int launch_rt_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                        bool rt7);
int launch_rt_hex_diag(b2p_op *op, double *diag, cudaStream_t s);
// Signed lexicographic restriction [ne][*PS] of the b2p_op_desc fields idx / orient / dof_map for P dofs per element (the one
// restriction builder: b2p_op_create, b2p_op_coarsen and b2p_flux_estimator_create_hex); rows padded to *PS = P rounded up to 4
// with B2P_SKIP_IDX. `who` prefixes the error messages.
int build_lex_restriction(b2p_ctx *ctx, const char *who, const b2p_op_desc *d, int P, int64_t lsize, int ne, int *PS, int32_t **lidx);
// Flux operator and error integrals of the flux estimator on hexahedra (b2p_hex_flux.cu, which also fills these for the
// Raviart-Thomas mass). Space a is the trial space of the mixed mass (the test space is b) or the space of index 1 of the error
// integral (index 2 is b); space_a: 0 = Nedelec, 1 = Raviart-Thomas.
struct HexFluxArgs
{
  b2p_ctx *ctx = nullptr;
  const b2p_geom *geom = nullptr;
  int p = 0;
  const double *h_tab = nullptr;  // host Bo[q1d][p] | Bc[q1d][p+1] | Gc (zeros), as b2p_op::h_tab (the production kernels' parameter block)
  const double *tab = nullptr;    // the same on the device
  bool production = false;        // hex_flux_production_eligible
  int space_a = 0;
  const int32_t *lidx_a = nullptr, *lidx_b = nullptr;
  int PS_a = 0, PS_b = 0;
  const double *ecoef = nullptr;  // [ne][10] {C, pad} (Flux), [ne][18] {C1, C2} (error integral) or b2p_op::ecoef (RT mass)
};
bool hex_flux_production_eligible(int p, int q1d, const double *h_tab);
// y_b += Flux x_a
int launch_hex_flux_mixed(const HexFluxArgs &a, const double *x, double *y, cudaStream_t s);
// est[e] += int_e |C2 P_b x_b - C1 P_a x_a|^2
int launch_hex_flux_error(const HexFluxArgs &a, const double *x1, const double *x2, double *est, cudaStream_t s);
int launch_h1_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s);
int launch_h1_hex_apply3(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg,
                         cudaStream_t s);
int launch_h1_hex_diag(b2p_op *op, double *diag, cudaStream_t s);
int launch_assemble_qdata(b2p_op *op, cudaStream_t s);
int launch_dense_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg,
                       cudaStream_t s, bool transpose = false);
int launch_dense_diag(b2p_op *op, double *diag, cudaStream_t s);
int launch_geom_hex(b2p_ctx *ctx, int ne, int k, int q1d, const double *d_xe, const double *d_B, const double *d_G,
                    const double *d_qw, double *d_qd, cudaStream_t s);
// CSR assembly on value arrays other than the handle's own (b2p_assemble.cu): the complex coarse solver keeps the real and
// imaginary parts of one operator as two value arrays [nnz] on ONE pattern.
double *csr_values(b2p_csr *A);
int csr_assemble_values(b2p_csr *A, int n_terms, b2p_op *const *ops, const double *coefs, double *val, cudaStream_t s);
int csr_eliminate_values(b2p_csr *A, const int32_t *ess_dofs, int64_t n_ess, int diag_policy, double *val, cudaStream_t s);
int csr_mult_values(b2p_csr *A, const double *val, const double *x, double *y, cudaStream_t s);
int csr_diag_values(b2p_csr *A, const double *val, double *d, cudaStream_t s);
// The real 2n form [[Ar, Ai], [Ai, -Ar]] of Ar + i Ai (values vr, vi on A's pattern): y = B x and d = diag(B) = [diag Ar; -diag Ar]
// without forming B; csr_block2_pattern (host, device arrays owned by the caller) and csr_block2_fill form it explicitly.
int csr_block2_mult(b2p_csr *A, const double *vr, const double *vi, const double *x, double *y, cudaStream_t s);
int csr_block2_diag(b2p_csr *A, const double *vr, double *d, cudaStream_t s);
int csr_block2_pattern(b2p_csr *A, int32_t **rowptr2, int32_t **col2);
int csr_block2_fill(b2p_csr *A, const double *vr, const double *vi, double *val2, cudaStream_t s);
}  // namespace b2p
