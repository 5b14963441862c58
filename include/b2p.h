/* b2p — H100-native (sm_90a) drop-in for Palace's partial-assembly operator path and the
 * smoother / multigrid / Krylov loop that drives it.  Plain C ABI: opaque handles, raw pointers
 * and sizes, no C++/torch types.  Every entry point returns 0 on success or a non-zero code with
 * a message retrievable through b2p_last_error() (mirrors libCEED's CEED_ERROR_SUCCESS +
 * CeedGetErrorMessage contract that Palace wraps in PalaceCeedCall,
 * /root/reference/palace/fem/libceed/ceed.hpp:13-33).
 *
 * Ownership: the creator owns a handle and destroys it; host arrays passed in *_desc structs are
 * copied during the call (CEED_COPY_VALUES semantics, /root/reference/palace/fem/libceed/restriction.cpp:192-204);
 * the caller owns all vectors; device vector pointers are only used in stream order of the call.
 * Threading: one caller thread per b2p_ctx (the reference uses exactly one Ceed context on GPU,
 * /root/reference/palace/fem/libceed/ceed.cpp:35-39). All work is enqueued on the stream given.
 * There is NO CPU fallback: every entry fails with B2P_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef B2P_H
#define B2P_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2p_ctx b2p_ctx;       /* device + (optional) NCCL communicator; ~ Ceed + MPI_Comm      */
typedef struct b2p_geom b2p_geom;     /* geometry q-data of one element block; ~ ceed::CeedGeomFactorData (mesh.cpp:146-209) */
typedef struct b2p_op b2p_op;         /* one local partially-assembled operator; ~ a CeedOperator sub-operator of ceed::Operator */
typedef struct b2p_interp b2p_interp; /* element-dense interpolator (P_l, G); ~ AssembleCeedInterpolator (libceed/integrator.cpp:515-548) */
typedef struct b2p_halo b2p_halo;     /* shared-dof exchange plan; ~ the P / P^T of ParOperator (linalg/rap.cpp:212-222) */
typedef void *b2p_stream;             /* cudaStream_t */

enum
{
  B2P_SUCCESS = 0,
  B2P_ERR_ARG = 1,
  B2P_ERR_CUDA = 2,
  B2P_ERR_UNSUPPORTED = 3,
  B2P_ERR_NCCL = 4
};

/* Which bilinear form (selects D at the quadrature points), /root/reference/palace/fem/integ/ *.cpp */
enum
{
  B2P_CURLCURL = 0,      /* CurlCurlIntegrator        -> f_apply_hdiv_33      (integ/curlcurl.cpp:47-52)     */
  B2P_ND_MASS = 1,       /* VectorFEMassIntegrator    -> f_apply_hcurl_33     (integ/vecfemass.cpp:72-105)   */
  B2P_CURLCURL_MASS = 2, /* CurlCurlMassIntegrator    -> f_apply_hdivmass_33  (integ/curlcurlmass.cpp:37-44) */
  B2P_H1_DIFFUSION = 3,  /* DiffusionIntegrator       -> f_apply_hcurl_33 on grad (integ/diffusion.cpp:37-42) */
  /* The Floquet-periodic terms on one ND space (models/spaceoperator.cpp:305-309); NOT symmetric (their transpose is applied with
   * B2P_APPLY_TRANSPOSE). Dense-basis operators (b2p_op_create_dense with both tables) on any element, and sum-factorised
   * operators on hexahedra (b2p_op_create, on-the-fly coefficients only: assemble_qdata = 1 returns B2P_ERR_UNSUPPORTED). On
   * hexahedra they also fuse with curl-curl / mass terms in b2p_op_create_sum. One coefficient context each, built by the
   * caller as the reference's integrators do (PopulateCoefficientContext with a = -1 for the weak curl, transpose for the curl): */
  B2P_ND_WEAKCURL = 4,   /* MixedVectorWeakCurlIntegrator: values -> curls,  f_apply_hcurlhdiv_33 (integ/mixedveccurl.cpp:68-117) */
  B2P_ND_MIXEDCURL = 5,  /* MixedVectorCurlIntegrator:     curls  -> values, f_apply_hdivhcurl_33 (integ/mixedveccurl.cpp:23-66)  */
  /* VectorFEMassIntegrator on a Raviart-Thomas (H(div)) space of hexahedra -> f_apply_hdiv_33 (integ/vecfemass.cpp:80-86):
   * D = (w / detJ) J^T C J with the ND_MASS coefficient context. b2p_op_desc.p is the ND-equivalent order: the space is RT_{p-1},
   * P = 3 p^2 (p + 1) dofs per element, restriction in the lexicographic RT layout (component c closed along axis c, open along the
   * other two), Bo / Bc as for ND, Gc not read. Sum-factorised only (b2p_op_create, b2p_op_coarsen; b2p_op_create_dense refuses
   * it); on-the-fly coefficients only (assemble_qdata = 1 returns B2P_ERR_UNSUPPORTED); single partition (b2p_op_apply_add_split
   * with ghost pieces returns B2P_ERR_UNSUPPORTED); not a term of b2p_op_create_sum or b2p_coperator_par (B2P_ERR_UNSUPPORTED). */
  B2P_RT_MASS = 6
};

/* ---- context -------------------------------------------------------------------------------- */
int b2p_ctx_create(int cuda_device, b2p_ctx **out);
/* Multi-GPU: one process per GPU. `nccl_unique_id` = 128 bytes from b2p_nccl_unique_id() on rank 0,
 * distributed by the caller (MPI_Bcast in Palace, torch.distributed in the harness). */
int b2p_nccl_unique_id(void *out128);
int b2p_ctx_create_dist(int cuda_device, const void *nccl_unique_id, int rank, int nranks, b2p_ctx **out);
void b2p_ctx_destroy(b2p_ctx *ctx);
const char *b2p_last_error(b2p_ctx *ctx); /* ctx may be NULL: last error of the calling thread */
int b2p_ctx_rank(b2p_ctx *ctx);
int b2p_ctx_nranks(b2p_ctx *ctx);
int b2p_ctx_sync(b2p_ctx *ctx, b2p_stream s);

/* Launch record of the persistent element kernels (nd_hex_apply4/5/6/7_kernel, h1_hex_apply3_kernel). Each of them clamps its
 * grid to the element batches and lets every worker (a warp, or the whole CTA for nd_hex_apply7_kernel) walk batch, batch + W,
 * ... with W workers in the grid. The launcher stores, on the host, what it launched last on this context, whichever operator
 * or complex / true-dof wrapper asked for it: which kernel ran, and whether every worker saw several batches. The kernels of
 * the hexahedral flux estimator (flux_hex_mixed7 / error7 and their cross-check kernels flux_hex_mixed / error, one batch per
 * CTA: grid = max_grid = batches, workers = 1) record themselves too, so a caller can see which route ran. */
typedef struct
{
  char kernel[48];      /* kernel name and form: "nd_hex_apply7_kernel", "nd_hex_apply7_kernel:block", "...:cplx", "...:block:cplx" */
  int max_grid;         /* SM count x CTAs per SM: the grid before clamping to the batches */
  int grid;             /* CTAs launched */
  int workers;          /* batch walkers per CTA: warps (nd4, nd5, nd6, h1v3) or 1 (nd7) */
  int elems_per_batch;  /* elements of one batch */
  int64_t batches;      /* batches of the launch (the last one may be partly filled) */
  int64_t seq;          /* launches recorded on this context so far, this one included */
  char geom[8];         /* where the geometry came from: "qdata" (stored per-point q-data) or "nodes" (evaluated from the
                           vertices of a trilinear mesh inside the kernel) */
} b2p_launch_info;
/* B2P_ERR_ARG before the first persistent launch on ctx. */
int b2p_ctx_last_launch(b2p_ctx *ctx, b2p_launch_info *out);

/* ---- device memory helpers (so a C/C++ host needs no CUDA runtime of its own) ----------------- */
int b2p_malloc(b2p_ctx *ctx, size_t bytes, void **dptr);
int b2p_free(b2p_ctx *ctx, void *dptr);
int b2p_memcpy_h2d(b2p_ctx *ctx, void *dst, const void *src, size_t bytes, b2p_stream s);
int b2p_memcpy_d2h(b2p_ctx *ctx, void *dst, const void *src, size_t bytes, b2p_stream s);

/* ---- geometry q-data (replaces Mesh::GetCeedGeomFactorData, fem/mesh.cpp:146-209,321-333) ----- */
/* Hexahedra of nodal order `mesh_order`; xe[ne][3][(mesh_order+1)^3] element node coordinates
 * (host, lexicographic tensor nodes, component-major); nodeB/nodeG[q1d][mesh_order+1]: the 1-D nodal
 * basis and its derivative at the q1d quadrature points; qw1d[q1d]; attr[ne]: 1-based local
 * attribute. Computes on the device {w detJ, adj(J)^T/detJ} per quadrature point
 * (qfunctions/33/geom_33_qf.h:9-34). */
int b2p_geom_create_hex(b2p_ctx *ctx, int ne, int mesh_order, int q1d, const double *xe, const double *nodeB,
                        const double *nodeG, const double *qw1d, const int32_t *attr, b2p_geom **out);
/* Prebuilt q-data in the reference layout qdata[ne][11][Q] = {attr, w detJ, adjJt/detJ[9]} (host). */
int b2p_geom_create_qdata(b2p_ctx *ctx, int ne, int q1d, const double *qdata, b2p_geom **out);
/* Same for any element type / quadrature rule (Q points per element, caller's point order): feeds the
 * dense-basis operators below. */
int b2p_geom_create_qdata_general(b2p_ctx *ctx, int ne, int Q, const double *qdata, b2p_geom **out);
/* Copy the device q-data back in the reference layout [ne][11][Q] (for parity tests). */
int b2p_geom_get_qdata(b2p_geom *g, double *qdata_host);
void b2p_geom_destroy(b2p_geom *g);

/* ---- local operator (replaces ceed::Operator sub-operators, fem/libceed/operator.hpp:32-65) ---- */
typedef struct
{
  int kind;                /* B2P_CURLCURL ... */
  int p;                   /* element order */
  int ne;                  /* elements in this block (must equal the geometry's) */
  int64_t lsize;           /* L-vector size (GetVSize()) */
  const int32_t *idx;      /* [ne][P] native-order element dofs (InitNativeRestr / InitLexicoRestr) */
  const int8_t *orient;    /* [ne][P] +1/-1 or NULL (restriction.cpp:290-297) */
  const int32_t *dof_map;  /* [P] lexicographic -> native, -1-n for a sign flip (TensorBasisElement::GetDofMap()); NULL = identity */
  const double *Bo;        /* [q1d][p]   open basis at quadrature points (ND only) */
  const double *Bc;        /* [q1d][p+1] closed basis */
  const double *Gc;        /* [q1d][p+1] closed basis derivative */
  const void *coeff_ctx;   /* coefficient context blob, layout of qfunctions/coeff/coeff_qf.h:7-43 (pair ctx for CURLCURL_MASS) */
  size_t coeff_ctx_bytes;
  int assemble_qdata;      /* 0: geometry + coefficient applied on the fly (reference default);
                              1: pre-multiplied symmetric D stored per point (BilinearForm::AssembleQuadratureData) */
} b2p_op_desc;

int b2p_op_create(b2p_ctx *ctx, b2p_geom *geom, const b2p_op_desc *desc, b2p_op **out);
/* Dense-basis (non-tensor) operator: what Palace builds for every vector element and every simplex
 * (InitNonTensorBasis -> CeedBasisCreateHcurl, fem/libceed/basis.cpp:40-85): tables exactly as
 * fe.GetDofToQuad(ir, FULL) supplies them, interp[3][Q][P] and deriv[3][Q][P] (curl for ND kinds, grad for
 * B2P_H1_DIFFUSION) in NATIVE dof order; restriction idx[ne][P] with either sign orientation `orient`
 * (restriction.cpp:290-297) or the row-major tridiagonal `curl_orient[ne][P][3]` of ND tets / prisms with
 * p >= 2 (restriction.cpp:301-368). Applied as one FP64 tensor-core (DMMA) GEMM per batch of 8 elements. */
typedef struct
{
  int kind;
  int P, Q, ne;
  int64_t lsize;
  const int32_t *idx;
  const int8_t *orient;       /* or NULL */
  const int8_t *curl_orient;  /* or NULL */
  const double *interp;       /* [3][Q][P] (ND mass kinds) or NULL */
  const double *deriv;        /* [3][Q][P] */
  const void *coeff_ctx;
  size_t coeff_ctx_bytes;
} b2p_dense_op_desc;
int b2p_op_create_dense(b2p_ctx *ctx, b2p_geom *geom, const b2p_dense_op_desc *desc, b2p_op **out);
/* p-coarsening that shares the fine operator's quadrature, geometry and coefficient
 * (ceed::CeedOperatorCoarsen, fem/libceed/operator.cpp:525-585): only space fields of desc are read
 * (p, lsize, idx, orient, dof_map, Bo/Bc/Gc evaluated at the FINE q1d points). */
int b2p_op_coarsen(b2p_op *fine, const b2p_op_desc *coarse_space, b2p_op **out);
/* The same for dense-basis operators: P, Q, ne, lsize, idx, orient / curl_orient, interp / deriv of the coarse space are
 * read (tables at the fine operator's Q points); kind and coefficient come from `fine`. */
int b2p_op_coarsen_dense(b2p_op *fine, const b2p_dense_op_desc *coarse_space, b2p_op **out);
/* (Dense-basis terms -- b2p_op_create_dense with kinds CURLCURL / ND_MASS / CURLCURL_MASS on one geometry handle, space and
 * orientation -- fuse the same way: one stacked table, summed per-element tensors.)
 * One operator for the real sum  sum_t coefs[t] * A_t  of sum-factorised ND operators over the same geometry, space and
 * essential set (BuildParSumOperator(a0 K + a1 C + a2 M), linalg/rap.cpp:764-829): the terms differ only in their pointwise
 * coefficient, so the sum runs as ONE element-kernel launch (one geometry stream) instead of one per term.
 * b2p_operator_par does this by itself when its terms qualify. The result is independent of the terms afterwards, except
 * that b2p_op_sum_set_coefficients re-reads their material tensors. */
int b2p_op_create_sum(b2p_ctx *ctx, int n_terms, b2p_op *const *ops, const double *coefs, b2p_op **out);
int b2p_op_sum_set_coefficients(b2p_op *sum, int n_terms, b2p_op *const *ops, const double *coefs);
/* y = A x  (ceed::Operator::Mult zero-fills first, operator.cpp:182-190) */
int b2p_op_apply(b2p_op *op, const double *x, double *y, b2p_stream s);
/* y += A x (ceed::Operator::AddMult, a == 1 only, operator.cpp:192-212) */
int b2p_op_apply_add(b2p_op *op, const double *x, double *y, b2p_stream s);
/* y += alpha * A x with options (ParOperator::AddMult scaling, linalg/rap.cpp:277-318):
 *   B2P_APPLY_MASKED         use the restriction with essential dofs masked out (b2p_op_set_essential):
 *                            masked inputs read as 0 and masked outputs are not written, which is what
 *                            ParOperator::Mult does with SetSubVector(tx, dbc_tdof_list, 0.0) before P and
 *                            the overwrite of y at those rows after P^T (rap.cpp:207-233)
 *   B2P_APPLY_SIMPLE_KERNEL  run the simple cross-check kernel instead of the production one
 *   B2P_APPLY_HALFWARP_KERNEL  run the one-element-per-warp ND kernel where it applies (p = 3, q1d = 4,
 *                            mirror-symmetric 1-D tables; ignored otherwise)
 *   B2P_APPLY_ROUND1_KERNEL  run nd_hex_apply4_kernel (the round-1 production kernel) where the default is
 *                            nd_hex_apply6_kernel (p = 3) or nd_hex_apply7_kernel (p = 2, 4, 5, 6), at q1d = p + 1;
 *                            same as B2P_ND_KERNEL=4 for one call
 *   B2P_APPLY_CTA_KERNEL     run nd_hex_apply7_kernel (one CTA per element batch, one 1-D line per thread) where it
 *                            applies (p = 2 ... 6 at q1d = p + 1, mirror-symmetric tables; ignored otherwise); same as
 *                            B2P_ND_KERNEL=7 for one call */
enum
{
  B2P_APPLY_MASKED = 1,
  B2P_APPLY_SIMPLE_KERNEL = 2,
  B2P_APPLY_HALFWARP_KERNEL = 4,
  B2P_APPLY_ROUND1_KERNEL = 8,
  B2P_APPLY_CTA_KERNEL = 16,
  B2P_APPLY_TRANSPOSE = 32 /* y += alpha A^T x; only the non-symmetric kinds (B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL) look at it */
};
int b2p_op_apply_add_ex(b2p_op *op, double alpha, const double *x, double *y, int flags, b2p_stream s);
/* Same over the element sub-range [e_begin, e_begin + e_count) with the L-vector in two pieces: dofs
 * < n_owned in x / y (the true-dof vectors themselves), the rest in x_ghost / y_ghost. This is what lets
 * a partitioned ParOperator run its interior elements while the ghost values are still in flight and
 * never copy a T-vector into an L-vector (e_count < 0: to the end; n_owned < 0: everything owned). */
/* Two right-hand sides in one pass over the geometry: y0 += alpha A x0, y1 += alpha A x1 (falls back to two applies when
 * the operator has no two-slot kernel). flags as b2p_op_apply_add_ex. */
int b2p_op_apply_add_pair(b2p_op *op, double alpha, const double *x0, const double *x1, double *y0, double *y1, int flags, b2p_stream s);
int b2p_op_apply_add_split(b2p_op *op, double alpha, const double *x, const double *x_ghost, double *y, double *y_ghost,
                           int64_t n_owned, int e_begin, int e_count, int flags, b2p_stream s);
/* Essential (Dirichlet / PEC) L-vector dofs for the masked apply. */
int b2p_op_set_essential(b2p_op *op, const int32_t *ess_ldofs, int64_t n);
/* diag += diag(A) (ceed::Operator::AssembleDiagonal, operator.cpp:116-143) */
int b2p_op_diag_add(b2p_op *op, double *diag, b2p_stream s);
/* Replace the coefficient context without touching geometry/restriction (driven sweeps re-coefficient
 * per frequency, drivers/drivensolver.cpp:176-198). */
int b2p_op_set_coeff(b2p_op *op, const void *coeff_ctx, size_t bytes);
int64_t b2p_op_lsize(b2p_op *op);
/* Algorithmic HBM bytes one apply moves (x read + y write + indices + q-data), for roofline reports. */
int64_t b2p_op_algorithmic_bytes(b2p_op *op);
void b2p_op_destroy(b2p_op *op);

/* ---- element-local interpolators (P_l, G): replaces fem/bilinearform.cpp:203-282 + AssembleCeedInterpolator ---- */
typedef struct
{
  int in_off;          /* offset of this component's input block inside the lexicographic input element vector */
  int in_n[3];         /* input block dims (x fastest) */
  int out_off;         /* offset of the output block */
  int out_n[3];        /* output block dims */
  const double *A[3];  /* 1-D matrices A_x, A_y, A_z, row-major [out_n[d]][in_n[d]] */
} b2p_interp_comp;

typedef struct
{
  int ne;
  int in_P;                  /* input (trial) space: native restriction + GetDofMap(), as in b2p_op_desc */
  int64_t in_lsize;
  const int32_t *in_idx;
  const int8_t *in_orient;
  const int32_t *in_dof_map;
  int out_P;                 /* output (test) space */
  int64_t out_lsize;
  const int32_t *out_idx;
  const int8_t *out_orient;
  const int32_t *out_dof_map;
  int ncomp;                 /* output vector components (1: H1, 3: ND) */
  b2p_interp_comp comps[3];
} b2p_interp_desc;

int b2p_interp_create(b2p_ctx *ctx, const b2p_interp_desc *desc, b2p_interp **out);
/* y += alpha * (1/mult) .* I x   (transpose = 0, ceed::Operator::AddMult with dof multiplicity, operator.cpp:182-212)
 * y += alpha * I^T ((1/mult) .* x) (transpose = 1) */
/* Element-dense interpolator for any element type (tetrahedra: p-prolongation / discrete gradient matrices from
 * GetTransferMatrix / ProjectGrad, fem/libceed/basis.cpp:116-165): one [out_P][in_P] row-major matrix in native dof
 * order for every element; restrictions with sign orientation (+1/-1) or with the int8 tridiagonal rows of
 * restriction.cpp:301-329 -- domain side filled from InvTransformPrimal, range side from InvTransformDual. Same Mult /
 * MultTranspose multiplicity scaling as b2p_interp_create (libceed/operator.cpp:182-235). */
typedef struct
{
  int ne, in_P, out_P;
  int64_t in_lsize, out_lsize;
  const int32_t *in_idx;          /* [ne][in_P] */
  const int8_t *in_orient;        /* [ne][in_P] or NULL */
  const int8_t *in_curl_orient;   /* [ne][in_P][3] or NULL */
  const int32_t *out_idx;         /* [ne][out_P] */
  const int8_t *out_orient;       /* [ne][out_P] or NULL */
  const int8_t *out_curl_orient;  /* [ne][out_P][3] (dual rows) or NULL */
  const double *mat;              /* [out_P][in_P] */
} b2p_dense_interp_desc;
int b2p_interp_create_dense(b2p_ctx *ctx, const b2p_dense_interp_desc *desc, b2p_interp **out);
/* Discrete curl C : ND_p -> RT_{p-1} on hexahedra (SpaceOperator::GetCurlMatrix, a DiscreteLinearOperator with a
 * CurlInterpolator, fem/fespace.cpp:204,216), sum-factorised: per element, in lexicographic order, RT component c equals
 * D_a u_b - D_b u_a for (c, a, b) cyclic, with D acting along one axis and the identity along the other two; no element
 * matrix is formed. ND component b is open (p Gauss-Legendre nodes) along axis b and closed (p + 1 Gauss-Lobatto nodes) along
 * the others; RT component c is closed along c and open along the others. The ND space is described as in b2p_op_desc of
 * B2P_ND_MASS (native idx + orient + GetDofMap()), the RT space as in B2P_RT_MASS (lexicographic idx + signs, dof_map NULL).
 * The result is an ordinary b2p_interp with the Mult / MultTranspose multiplicity scaling of b2p_interp_create (1/mult of
 * the RT space), one kernel launch per apply. B2P_ERR_ARG: a null pointer, ne < 1, p < 1, an lsize outside 1..2^31-1, an index
 * outside [0, lsize) or a dof_map entry outside the element; B2P_ERR_UNSUPPORTED: p > 6. */
typedef struct
{
  int ne, p;              /* ND_p -> RT_{p-1}; p as in b2p_op_desc of B2P_ND_MASS / B2P_RT_MASS */
  int64_t nd_lsize;
  const int32_t *nd_idx;  /* [ne][3 p (p+1)^2] native order */
  const int8_t *nd_orient;
  const int32_t *nd_dof_map;
  int64_t rt_lsize;
  const int32_t *rt_idx;  /* [ne][3 p^2 (p+1)] */
  const int8_t *rt_orient;
  const int32_t *rt_dof_map; /* may be NULL */
  const double *D;        /* [p][p+1] row-major: closed-basis derivative at the open nodes (ProjectCurl) */
} b2p_curl_interp_desc;
int b2p_interp_create_curl_hex(b2p_ctx *ctx, const b2p_curl_interp_desc *desc, b2p_interp **out);
int b2p_interp_apply_add(b2p_interp *it, int transpose, double alpha, const double *x, double *y, b2p_stream s);
void b2p_interp_destroy(b2p_interp *it);

/* ---- shared-dof exchange between partitions (P / P^T of ParOperator, linalg/rap.cpp:212-222) ---- */
/* L-vector layout on every rank: [n_true owned | n_ghost ghosts grouped by owner rank in nbr_ranks order].
 * send_idx: owned indices whose values neighbour k holds as ghosts, concatenated (send_counts[k] each), in the
 * same (global dof) order as that neighbour's ghost segment. */
int b2p_halo_create(b2p_ctx *ctx, int64_t n_true, int64_t n_ghost, int n_nbr, const int32_t *nbr_ranks,
                    const int64_t *send_counts, const int32_t *send_idx, const int64_t *recv_counts, b2p_halo **out);
int b2p_halo_forward(b2p_halo *h, double *lvec); /* owners -> ghosts (P) */
int b2p_halo_reverse(b2p_halo *h, double *lvec); /* ghosts added into owners (P^T) */
/* Optional peer-memory (NVLink) exchange for ParOperator::Mult instead of NCCL send/recv: every rank exports a
 * blob (CUDA IPC handle of its mailbox + exchange offsets; call with blob == NULL to get the size), the caller
 * all-gathers the blobs (MPI_Allgather in Palace, torch.distributed in the harness) and every rank imports them. */
int b2p_halo_p2p_export(b2p_halo *h, void *blob, size_t *bytes);
int b2p_halo_p2p_import(b2p_halo *h, const void *blobs, size_t stride, int nranks);
void b2p_halo_destroy(b2p_halo *h);

/* ---- full assembly (coarse levels) ------------------------------------------------------------------------------
 * Device-resident CSR matrix of a sum of local operators on the L-vector: what BilinearForm::FullAssemble /
 * CeedOperatorFullAssemble (fem/libceed/operator.cpp:262-523) produce for ParOperator::ParallelAssemble
 * (linalg/rap.cpp:84-152) -> HYPRE AMS/BoomerAMG or a sparse direct solver on the coarsest multigrid level.
 * b2p_csr_create: symbolic phase from the restriction of `op` (host, once per space; the reference's
 *   CeedOperatorLinearAssembleSymbolic + COO->CSR sort). Any operator on the same space can be assembled into it.
 * b2p_csr_assemble: numeric phase on the device, values = sum_t coefs[t] * A_t (the reference's "set" = false
 *   accumulation). The element matrices come from the operator kernels themselves (applied to local unit vectors
 *   through an identity restriction), so hex / tet / assembled-D operators are all covered; no host work, no sort. Column j
 *   of every element matrix is the apply to e_j, so the non-symmetric hex kinds (B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL) and
 *   block sums that contain them are assembled as A, not A^T.
 * b2p_csr_device_arrays: rowptr[n+1] / col[nnz] (int32, sorted columns) / val[nnz] device pointers, owned by the handle
 *   (wrap them in a hypre_CSRMatrix). b2p_csr_eliminate: essential rows/columns as HypreParMatrix::EliminateBC with
 *   the ParOperator diagonal policy (1 = DIAG_ONE, 0 = DIAG_ZERO), for callers that skip the P^T A P step.
 * b2p_csr_mult: y = A x (verification / standalone coarse solves). */
typedef struct b2p_csr b2p_csr;
int b2p_csr_create(b2p_ctx *ctx, b2p_op *op, b2p_csr **out);
int b2p_csr_assemble(b2p_csr *A, int n_terms, b2p_op *const *ops, const double *coefs, b2p_stream s);
int64_t b2p_csr_rows(const b2p_csr *A);
int64_t b2p_csr_nnz(const b2p_csr *A);
int b2p_csr_device_arrays(b2p_csr *A, const int32_t **rowptr, const int32_t **col, const double **val);
int b2p_csr_get_host(b2p_csr *A, int32_t *rowptr, int32_t *col, double *val, b2p_stream s);
int b2p_csr_eliminate(b2p_csr *A, const int32_t *ess_dofs, int64_t n_ess, int diag_policy, b2p_stream s);
int b2p_csr_mult(b2p_csr *A, const double *x, double *y, b2p_stream s);
int b2p_csr_diag(b2p_csr *A, double *d, b2p_stream stream);   /* d = diag(A) */
void b2p_csr_destroy(b2p_csr *A);

/* ---- device-resident linear algebra (replaces linalg/vector.cpp kernels + MPI_Allreduce) ---- */
int b2p_ctx_set_stream(b2p_ctx *ctx, b2p_stream s); /* stream used by everything below */
int b2p_vec_axpby(b2p_ctx *ctx, int64_t n, double a, const double *x, double b, double *y);                 /* y = a x + b y  (vector.cpp:276-377) */
int b2p_vec_axpbypcz(b2p_ctx *ctx, int64_t n, double a, const double *x, double b, const double *y, double g, double *z);
int b2p_vec_dot(b2p_ctx *ctx, int64_t n, const double *x, const double *y, double *out);                    /* global: all-reduced over ranks */
int b2p_vec_sum(b2p_ctx *ctx, int64_t n, const double *x, double *out);
int b2p_vec_set_sub(b2p_ctx *ctx, double *y, const int32_t *idx_dev, int64_t nidx, double v);               /* vector.cpp:461-527 */
int b2p_vec_set_random(b2p_ctx *ctx, int64_t n, double *y, uint64_t seed);
/* Gram-Schmidt of w against V[0..m) (linalg/orthog.hpp:41-89): type 0 MGS, 1 CGS, 2 CGS2; H[m] on the host */
int b2p_vec_orthogonalize(b2p_ctx *ctx, int type, int64_t n, int m, const double *const *V, double *w, double *H);

/* ---- operators on true-dof vectors ---- */
typedef struct b2p_operator b2p_operator;
/* ParOperator over sum_i coef_i * op_i (BuildParSumOperator, rap.cpp:764-829) with essential true dofs;
 * diag_policy 0 = DIAG_ZERO, 1 = DIAG_ONE; halo may be NULL (single partition).
 * Op sharing: essential dofs are eliminated through the b2p_op's masked restriction (b2p_op_set_essential), one mask per
 * b2p_op. The first single-partition operator built on an op installs the mask from ess_tdofs; building another operator on
 * the same op with a DIFFERENT essential set (including empty vs non-empty) fails with B2P_ERR_ARG -- create a second b2p_op
 * (geometry and tables are shared, refcounted) or re-install the mask. Partitioned callers (halo != NULL) install the mask
 * in L-vector indices, ghost copies included, before this call. */
int b2p_operator_par(b2p_ctx *ctx, int64_t tsize, int64_t lsize, int n_terms, b2p_op *const *ops, const double *coefs,
                     const int32_t *ess_tdofs, int64_t n_ess, int diag_policy, b2p_halo *halo, b2p_operator **out);
int b2p_operator_par_is_fused(b2p_operator *A); /* 1: the terms run as one fused element operator (b2p_op_create_sum) */
/* New coefficients of the sum without rebuilding the operator (frequency sweeps: a0 K + a1 C + a2 M with new a_i). */
int b2p_operator_par_set_coefficients(b2p_operator *A, int n_terms, const double *coefs);
/* Elements [0, ne_interior) of every local operator touch no ghost dof: they are applied while the forward
 * shared-dof exchange is still in flight (element order chosen by the caller; 0 disables the overlap). */
int b2p_operator_par_set_interior(b2p_operator *A, int ne_interior);
/* The assembled matrix as an operator (symmetric; not owned): coarse-level Krylov / Jacobi / Chebyshev solvers run on it. */
int b2p_operator_csr(b2p_ctx *ctx, b2p_csr *A, b2p_operator **out);
/* Interpolator on true-dof vectors (ParOperator(..., use_R) semantics); halos/true sizes of the input
 * and output spaces, NULL / L-size for a single partition. */
int b2p_operator_interp(b2p_ctx *ctx, b2p_interp *it, b2p_halo *in_halo, int64_t in_tsize, b2p_halo *out_halo,
                        int64_t out_tsize, b2p_operator **out);
int b2p_operator_mult(b2p_operator *A, const double *x, double *y);
int b2p_operator_mult_transpose(b2p_operator *A, const double *x, double *y);
int b2p_operator_add_mult(b2p_operator *A, const double *x, double *y, double a);
int b2p_operator_assemble_diagonal(b2p_operator *A, double *d);
int64_t b2p_operator_height(b2p_operator *A);
int64_t b2p_operator_width(b2p_operator *A);
void b2p_operator_destroy(b2p_operator *A);

/* ---- ParOperator with a general conforming prolongation (non-conforming / AMR meshes; linalg/rap.cpp:154-275) ----
 * On a non-conforming mesh the prolongation of a space is a sparse matrix P [lsize x tsize] whose slave rows interpolate from
 * master dofs (mfem::ParFiniteElementSpace::GetProlongationMatrix(), a HypreParMatrix); the reference applies y = P^T A P x with
 * the essential TRUE dofs zeroed before P and overwritten after P^T (rap.cpp:195-234), and assembles the diagonal as |P|^T d_L
 * with entry-wise absolute values (rap.cpp:162-178, HypreParMatrix::AbsMultTranspose).
 * b2p_spmat: device CSR matrix from host arrays (int32 rowptr[rows+1] / col[nnz], double val[nnz]; copied), kept with its
 * transpose. b2p_operator_rap: A_local is the operator on the L-vector (a b2p_operator_par over the local operators with
 * tsize == lsize and NO essential dofs; not owned), P the space's prolongation (shared: reference counted, the caller may destroy
 * its handle), ess_tdofs in TRUE-dof numbering; Mult, MultTranspose, AddMult and AssembleDiagonal as above. Single partition. */
typedef struct b2p_spmat b2p_spmat;
int b2p_spmat_create(b2p_ctx *ctx, int64_t rows, int64_t cols, const int32_t *rowptr, const int32_t *col, const double *val,
                     b2p_spmat **out);
int b2p_spmat_mult(b2p_spmat *m, int transpose, const double *x, double *y); /* y = A x or A^T x on the context's stream */
void b2p_spmat_destroy(b2p_spmat *m);
int b2p_operator_rap(b2p_ctx *ctx, b2p_operator *A_local, b2p_spmat *P, const int32_t *ess_tdofs, int64_t n_ess, int diag_policy,
                     b2p_operator **out);
/* y = L A R x with sparse L and / or R (NULL: absent), transpose R^T A^T L^T: the level prolongations and discrete gradients of
 * non-conforming spaces, ParOperator(interpolator, trial, test, use_R = true) = R_test I P_trial (rap.cpp:195-275,320-345), with
 * A_mid the interpolator on L-vectors (b2p_operator_interp without halos), L the test space's restriction (true-dof selection)
 * and R the trial space's prolongation. A_mid is not owned; the matrices are shared. */
int b2p_operator_triple(b2p_ctx *ctx, b2p_spmat *L, b2p_operator *A_mid, b2p_spmat *R, b2p_operator **out);

/* ---- solvers (palace::Solver<Operator>, linalg/solver.hpp:21-65) ---- */
typedef struct b2p_solver b2p_solver;
int b2p_solver_jacobi(b2p_ctx *ctx, double omega, double sf_max, b2p_solver **out);                                  /* jacobi.cpp */
int b2p_solver_chebyshev(b2p_ctx *ctx, int smooth_it, int order, double sf_max, double sf_min, int fourth_kind,
                         b2p_solver **out);                                                                           /* chebyshev.cpp */
int b2p_solver_distrelax(b2p_ctx *ctx, b2p_operator *G, int smooth_it, int cheby_smooth_it, int cheby_order, double sf_max,
                         double sf_min, int fourth_kind, b2p_solver **out);                                           /* distrelaxation.cpp */
int b2p_solver_distrelax_set_operators(b2p_solver *s, b2p_operator *A, b2p_operator *A_G);
/* coarse: level-0 solver (ownership moves to the multigrid solver); P[n_levels-1]; G[n_levels] or NULL */
int b2p_solver_gmg(b2p_ctx *ctx, b2p_solver *coarse, int n_levels, b2p_operator *const *P, b2p_operator *const *G, int cycle_it,
                   int smooth_it, int cheby_order, double sf_max, double sf_min, int fourth_kind, b2p_solver **out);  /* gmg.cpp */
int b2p_solver_gmg_set_operators(b2p_solver *s, b2p_operator *const *A, b2p_operator *const *A_aux);
/* type 0 CG, 1 GMRES, 2 FGMRES (iterative.cpp) */
/* A solver that runs on the device-ASSEMBLED matrix of the ParOperator it is given at set_operator time
 * (MfemWrapperSolver, linalg/solver.cpp:13-30; single partition): the multigrid's coarse solver. Takes over `inner` (a Krylov
 * or smoother handle) and, optionally, its preconditioner `inner_pc`, which also gets the assembled matrix; the two handles
 * only need b2p_solver_destroy afterwards. b2p_solver_assembled_nnz: entries of the current matrix (s: the solver, or the multigrid that took it over as its coarse
 * solver), -1 before set_operator. */
int b2p_solver_assembled(b2p_ctx *ctx, b2p_solver *inner, b2p_solver *inner_pc, b2p_solver **out);
int64_t b2p_solver_assembled_nnz(b2p_solver *s);
int b2p_solver_krylov(b2p_ctx *ctx, int type, b2p_solver **out);
int b2p_solver_krylov_config(b2p_solver *s, double rel_tol, double abs_tol, int max_it, int max_dim, int orthog, int pc_side);
/* CG only: keep alpha / beta in device memory and read the residual back every `check_every` iterations (1 = the
 * reference's iteration with two host-visible dot products per step, iterative.cpp:361-486). */
int b2p_solver_krylov_set_check_interval(b2p_solver *s, int check_every);
int b2p_solver_set_preconditioner(b2p_solver *s, b2p_solver *pc);
int b2p_solver_set_operator(b2p_solver *s, b2p_operator *A);
int b2p_solver_set_initial_guess(b2p_solver *s, int flag);
int b2p_solver_mult(b2p_solver *s, const double *x, double *y);
int b2p_solver_mult2(b2p_solver *s, const double *x, double *y, double *r);
int b2p_solver_mult_transpose2(b2p_solver *s, const double *x, double *y, double *r);
int b2p_solver_stats(b2p_solver *s, int *its, double *initial_res, double *final_res, int *converged);
int b2p_solver_lambda_max(b2p_solver *s, double *out); /* Chebyshev: estimated lambda_max(D^-1 A) * sf_max */
void b2p_solver_destroy(b2p_solver *s);

/* ---- algebraic coarse solvers (the reference's HypreAmsSolver / BoomerAmgSolver, linalg/{ams,amg}.cpp, GPU configuration) ----
 * Both take an ASSEMBLED real matrix at set_operator: b2p_operator_csr, the matrix b2p_solver_assembled hands its inner solver,
 * or the Ar + Ai matrix of b2p_csolver_assembled; anything else (and a partitioned context) fails with B2P_ERR_ARG /
 * B2P_ERR_UNSUPPORTED. The usual wiring is b2p_solver_assembled(ctx, ams, NULL, &coarse) as the coarse solver of b2p_solver_gmg,
 * or as coarse_type 2 of b2p_ksp_create / b2p_divfree_create / b2p_flux_estimator_set_multigrid. Setup (aggregation, Galerkin
 * products, dense pseudo-inverse of the coarsest level) runs on the host at set_operator; a mult runs on the device without
 * allocation or host synchronisation (CUDA-graph capturable). Both are symmetric and can precondition CG.
 * b2p_solver_amg: smoothed-aggregation AMG (strength 0.08, three-pass greedy aggregation, one Jacobi-smoothed prolongation, stop
 *   at <= 500 rows / 10 levels / a level keeping > 80 % of its rows), l1-Jacobi with smooth_it sweeps before and after; mult =
 *   cycle_it V-cycles from zero, or from the initial guess when set.
 * b2p_solver_ams: AMS cycle type 14 ("01(3+4+5)10") for the eliminated Nedelec p = 1 matrix: G [n_edges x n_vertices] the discrete
 *   gradient (host CSR, sorted unique columns, entries +-1), coords[n_vertices][3] the vertex coordinates (host). The auxiliary
 *   matrices G^T A G and Pi_c^T A Pi_c (Pi_c(e, v) = |G(e, v)| (G x_c)_e / 2) each get an AMG hierarchy with one V-cycle per
 *   correction; singular != 0 drops the gradient correction (curl-curl without mass, the reference's ams_singular_op). mult =
 *   exactly cycle_it cycles, no norm checks.
 * b2p_solver_amg_levels: rows / nnz of each level of hierarchy `hierarchy` (AMG: 0; AMS: 0 = G, 1..3 = Pi_x, Pi_y, Pi_z) of s, of
 *   the inner solver of a b2p_solver_assembled, or of either as a multigrid's coarse solver; returns the number of levels (0
 *   for the skipped gradient hierarchy of a singular AMS), -1 if s has no such hierarchy. b2p_solver_amg_setup_ms: host time of
 *   the last set_operator, -1 likewise. */
int b2p_solver_amg(b2p_ctx *ctx, int cycle_it, int smooth_it, b2p_solver **out);
int b2p_solver_ams(b2p_ctx *ctx, int cycle_it, int smooth_it, int singular, int64_t n_edges, int64_t n_vertices,
                   const int32_t *G_rowptr, const int32_t *G_col, const double *G_val, const double *coords, b2p_solver **out);
int b2p_solver_amg_levels(b2p_solver *s, int hierarchy, int64_t *rows, int64_t *nnz, int max_levels);
double b2p_solver_amg_setup_ms(b2p_solver *s);

/* ---- BaseKspSolver: configuration -> Krylov solver + preconditioner (linalg/ksp.cpp:29-102,131-239,256-328) ----
 * The fields mirror config::LinearSolverData (utils/configfile.hpp:1000-1120) with the defaults iodata.cpp:500-545 derives;
 * b2p_ksp_config_default fills them for a solution space of polynomial order `order`. The composer builds
 *   ConfigureKrylovSolver:          CG / GMRES / FGMRES with restart size, tolerances, orthogonalisation, preconditioner side
 *   ConfigurePreconditionerSolver:  one level  -> the coarse solver alone (Jacobi, or PCG-Jacobi on the assembled matrix)
 *                                   n levels   -> GeometricMultigridSolver(coarse, P, mg_smooth_aux ? G : NULL, mg_cycle_it,
 *                                                  mg_smooth_it, mg_smooth_order, sf_max, sf_min, cheby_4th)
 * and keeps the reference's counters NumTotalMult / NumTotalMultIts. The sparse-direct / HYPRE coarse solvers of the
 * reference stay outside this library: coarse_type 2 takes a caller-supplied b2p_solver instead. */
typedef struct b2p_ksp b2p_ksp;
typedef struct
{
  int krylov_solver;     /* 0 CG, 1 GMRES, 2 FGMRES                                   (KrylovSolver) */
  double tol;            /* relative residual tolerance                               (linear.tol, 1e-6) */
  int max_it;            /* (linear.max_it, 100) */
  int max_size;          /* GMRES / FGMRES restart dimension; <= 0: max_it            (linear.max_size) */
  int initial_guess;     /* use the incoming y as the initial guess                   (linear.initial_guess) */
  int pc_side;           /* -1 default of the solver, 0 right, 1 left                 (PreconditionerSide) */
  int gs_orthog;         /* 0 MGS, 1 CGS, 2 CGS2                                      (Orthogonalization) */
  int mg_cycle_it;       /* V-cycles per preconditioner application                   (linear.mg_cycle_it, 1) */
  int mg_smooth_aux;     /* Hiptmair distributive relaxation on the levels > 0        (linear.mg_smooth_aux) */
  int mg_smooth_it;      /* pre/post smoothing iterations                             (linear.mg_smooth_it, 1) */
  int mg_smooth_order;   /* Chebyshev order; <= 0: max(2 * order, 4)                  (iodata.cpp:533-536) */
  double mg_smooth_sf_max, mg_smooth_sf_min; /* (1.0, 0.0) */
  int mg_smooth_cheby_4th; /* 4th-kind (1) or 1st-kind (0) Chebyshev                  (true) */
  int coarse_type;       /* 0 Jacobi (LinearSolver::JACOBI), 1 Jacobi-PCG on the device-assembled level-0 matrix
                          * (MfemWrapperSolver analogue), 2 caller-supplied solver */
  double coarse_tol;     /* coarse_type 1: relative tolerance of the inner PCG */
  int coarse_max_it;
} b2p_ksp_config;
int b2p_ksp_config_default(b2p_ksp_config *cfg, int order);
/* P[n_levels-1] prolongations, G[n_levels] discrete gradients (read when mg_smooth_aux; G[0] unused), coarse_solver only
 * for coarse_type 2 (ownership moves into the composed solver). n_levels == 1: no multigrid, the coarse solver preconditions. */
int b2p_ksp_create(b2p_ctx *ctx, const b2p_ksp_config *cfg, int n_levels, b2p_operator *const *P, b2p_operator *const *G,
                   b2p_solver *coarse_solver, b2p_ksp **out);
/* KspSolver::SetOperators(op, pc_op): `op` the system operator; pc_ops[n_levels] the preconditioner's level operators and
 * aux_ops[n_levels] their auxiliary-space (H1) operators (BaseMultigridOperator), aux_ops may be NULL without mg_smooth_aux. */
int b2p_ksp_set_operators(b2p_ksp *k, b2p_operator *op, b2p_operator *const *pc_ops, b2p_operator *const *aux_ops);
int b2p_ksp_mult(b2p_ksp *k, const double *x, double *y);
/* NumTotalMult(), NumTotalMultIts() (ksp.hpp:57-58) and the last solve's record */
int b2p_ksp_stats(b2p_ksp *k, int *num_total_mult, int *num_total_mult_its, int *last_its, double *initial_res, double *final_res,
                  int *converged);
void b2p_ksp_destroy(b2p_ksp *k);

/* ---- complex-valued operators and Krylov solvers on split (real, imag) vectors ---------------------
 * Palace's ComplexVector is two real vectors (linalg/vector.hpp:23-27); every entry takes the two device
 * pointers separately. Inner product convention Dot(x, y) = y^H x (linalg/vector.cpp:674-685). */
typedef struct b2p_coperator b2p_coperator;
typedef struct b2p_csolver b2p_csolver;
int b2p_vec_cdot(b2p_ctx *ctx, int64_t n, const double *xr, const double *xi, const double *yr, const double *yi, double out[2]);
int b2p_vec_caxpy(b2p_ctx *ctx, int64_t n, double ar, double ai, const double *xr, const double *xi, double *yr, double *yi);
/* A = sum_i (coef_re[i] + i coef_im[i]) * op_i with real partially assembled op_i: ComplexParOperator over
 * BuildParSumOperator / ComplexWrapperOperator (linalg/rap.cpp:481-517,843-919, linalg/operator.cpp:98-134).
 * Single partition (tsize == lsize); on partitioned spaces use b2p_coperator_wrap over two b2p_operator_par. */
int b2p_coperator_par(b2p_ctx *ctx, int64_t tsize, int64_t lsize, int n_terms, b2p_op *const *ops, const double *coef_re,
                      const double *coef_im, const int32_t *ess_tdofs, int64_t n_ess, int diag_policy, b2p_coperator **out);
/* A = Ar + i Ai from two real true-dof operators (either may be NULL, not owned): ComplexWrapperOperator,
 * linalg/operator.cpp:98-134 — the parts can be ParOperators on PARTITIONED spaces (each with its halo), assembled matrices
 * (b2p_operator_csr), ... For the complex DIAG_ONE rows give Ar DIAG_ONE and Ai DIAG_ZERO (rap.cpp:481-517). */
int b2p_coperator_wrap(b2p_ctx *ctx, b2p_operator *Ar, b2p_operator *Ai, b2p_coperator **out);
int b2p_coperator_mult(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi);
int b2p_coperator_mult_hermitian_transpose(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi);
int b2p_coperator_add_mult(b2p_coperator *A, const double *xr, const double *xi, double *yr, double *yi, double ar, double ai);
int b2p_coperator_assemble_diagonal(b2p_coperator *A, double *dr, double *di);
/* Number of Mult / MultHermitianTranspose calls served by the fused complex element kernel (one pass over the geometry
 * for all terms and both vector parts) instead of 2-4 real applies per term; -1 if A is not a sum operator. */
/* New coefficients of the terms (next frequency of a driven sweep, spaceoperator.cpp:945-1153) without rebuilding the
 * operator: the smoothers / solvers that hold A see the new matrix at their next SetOperator. */
int b2p_coperator_set_coefficients(b2p_coperator *A, int n_terms, const double *coef_re, const double *coef_im);
long b2p_coperator_fused_applies(b2p_coperator *A);
/* Route of a b2p_coperator_par's Mult / MultHermitianTranspose / AddMult: 0 term by term (2-4 real applies per term), 1 two real
 * sums S_re and S_im (4 applies), 2 one pass over the geometry on the nd4 kernel (p <= 3), 3 one pass on the CTA-per-batch
 * kernel (symmetric kinds at p = 4 ... 6, block sums at p = 2 ... 6); -1 if A is not a sum operator. */
int b2p_coperator_fused_path(b2p_coperator *A);
void b2p_coperator_destroy(b2p_coperator *A);
/* A real preconditioner (any b2p_solver, e.g. the multigrid) applied to the real and imaginary parts: the
 * "PCMatReal" configuration (models/spaceoperator.cpp:1098-1105, utils/configfile.hpp:1051). */
int b2p_csolver_real_pc(b2p_ctx *ctx, b2p_solver *real_pc, b2p_csolver **out);
/* MfemWrapperSolver<ComplexOperator> (linalg/solver.cpp:33-177; single partition): a complex solver that runs a REAL solver on
 * the device-assembled matrix of the complex operator given to b2p_csolver_set_operator -- the coarse solver of the complex
 * multigrid (b2p_csolver_gmg hands it A[0]). The operator must be a b2p_coperator_par, or a b2p_coperator_wrap whose parts are
 * single-partition b2p_operator_par on one space; anything else fails at set_operator with b2p_last_error set. Both parts are
 * assembled on one CSR pattern (Ar eliminated with the operator's diagonal policy, Ai with DIAG_ZERO), then
 *   complex_matrix == 0: the inner solver gets Ar + Ai, and mult applies it to the real and the imaginary part separately;
 *   complex_matrix != 0: the inner solver gets the 2n block [[Ar, Ai], [Ai, -Ar]] (applied from the two value arrays, not
 *                        formed) and mult solves it once for [xr; -xi] with the right-hand side [br; bi].
 * With only one part present (no imaginary or no real coefficient, a NULL part) that part alone is the matrix. Takes over
 * `inner` (Krylov or smoother) and, optionally, its preconditioner `inner_pc`, which also gets the matrix; both handles then
 * only need b2p_solver_destroy. mult honours b2p_csolver_set_initial_guess. After b2p_coperator_set_coefficients the next
 * set_operator with the same operator re-assembles the values only (no new symbolic phase).
 * b2p_csolver_assembled_nnz: entries of the real matrix the inner solver sees (4 x the pattern for the block form); s is the
 * solver, or the complex multigrid that took it over; -1 before set_operator.
 * b2p_csolver_assembled_device_arrays: rows, entries and device rowptr[rows+1] / col[nnz] (int32, sorted columns) / val[nnz] of
 * that matrix, owned by the solver and valid until its next set_operator: the input of a sparse direct solver. The explicit
 * block matrix is built on the first request (pattern on the host once, values by a kernel). */
int b2p_csolver_assembled(b2p_ctx *ctx, b2p_solver *inner, b2p_solver *inner_pc, int complex_matrix, b2p_csolver **out);
int64_t b2p_csolver_assembled_nnz(b2p_csolver *s);
int b2p_csolver_assembled_device_arrays(b2p_csolver *s, int64_t *rows, int64_t *nnz, const int32_t **rowptr, const int32_t **col,
                                        const double **val);
/* CgSolver / GmresSolver / FgmresSolver<ComplexOperator> (linalg/iterative.cpp:361-871; type 0/1/2) */
/* JacobiSmoother<ComplexOperator> (linalg/jacobi.cpp:75-105): y = omega D^-1 x with the complex diagonal of the operator given to
 * b2p_csolver_set_operator; omega != 0. The preconditioner of the complex-valued (PCMatReal = false) path. */
int b2p_csolver_jacobi(b2p_ctx *ctx, double omega, b2p_csolver **out);
/* ChebyshevSmoother<ComplexOperator>, 4th kind (linalg/chebyshev.cpp:160-220) on the operator given to b2p_csolver_set_operator:
 * complex inverse diagonal, lambda_max = sf_max * ||D^-1 A||_2 (power iteration, linalg/operator.cpp:583-631). mult applies
 * y = y + p(D^-1 A) D^-1 (x - A y) (y = 0 unless b2p_csolver_set_initial_guess). */
int b2p_csolver_chebyshev(b2p_ctx *ctx, int smooth_it, int order, double sf_max, b2p_csolver **out);
int b2p_csolver_lambda_max(b2p_csolver *s, double *out);
/* GeometricMultigridSolver<ComplexOperator> (linalg/gmg.cpp:16-205), the reference's default (PCMatReal = false) preconditioner
 * of complex systems: complex level operators A[l] (and auxiliary H1 operators A_aux[l] when the discrete gradients G are given:
 * DistRelaxationSmoother<ComplexOperator>, distrelaxation.cpp:39-151), 4th-kind complex Chebyshev smoothing, REAL prolongations P
 * and gradients G applied to both parts. Takes over `coarse` (it is handed A[0] by ..._set_operators). */
int b2p_csolver_gmg(b2p_ctx *ctx, b2p_csolver *coarse, int n_levels, b2p_operator *const *P, b2p_operator *const *G, int cycle_it,
                    int smooth_it, int cheby_order, double sf_max, b2p_csolver **out);
int b2p_csolver_gmg_set_operators(b2p_csolver *s, b2p_coperator *const *A, b2p_coperator *const *A_aux);
int b2p_csolver_krylov(b2p_ctx *ctx, int type, b2p_csolver **out);
int b2p_csolver_krylov_config(b2p_csolver *s, double rel_tol, double abs_tol, int max_it, int max_dim, int orthog, int pc_side);
int b2p_csolver_set_operator(b2p_csolver *s, b2p_coperator *A);
int b2p_csolver_set_preconditioner(b2p_csolver *s, b2p_csolver *pc);
int b2p_csolver_set_initial_guess(b2p_csolver *s, int flag);
int b2p_csolver_mult(b2p_csolver *s, const double *br, const double *bi, double *xr, double *xi);
int b2p_csolver_stats(b2p_csolver *s, int *its, double *initial_res, double *final_res, int *converged);
void b2p_csolver_destroy(b2p_csolver *s);

/* ---- outer eigen-solver interface: the operator applications of ArpackEPSSolver (linalg/arpack.cpp:631-674) --------
 * ARPACK's reverse communication (and SLEPc's shell matrices, slepc.cpp) run on the HOST and hand over host pointers to
 * interleaved complex vectors; the vectors of the applications live on the device. One handle keeps the device work
 * vectors and pinned staging:   apply_op   : y = (1/gamma) opInv (K x)            without spectral transformation
 *                                            y = gamma opInv (M x)                shift-and-invert (opInv = (K - sigma M)^-1)
 *                               apply_op_b : y = delta B x                        weighted inner product
 * K may be NULL with sinvert, B may be NULL (apply_op_b then fails). x, y: n std::complex<double> on the host. */
typedef struct b2p_eps b2p_eps;
int b2p_eps_create(b2p_ctx *ctx, int64_t n, b2p_coperator *K, b2p_coperator *M, b2p_csolver *opInv, b2p_coperator *B, int sinvert,
                   double gamma, double delta, b2p_eps **out);
int b2p_eps_apply_op(b2p_eps *e, const double *x_host_interleaved, double *y_host_interleaved);
int b2p_eps_apply_op_b(b2p_eps *e, const double *x_host_interleaved, double *y_host_interleaved);
void b2p_eps_destroy(b2p_eps *e);

/* ---- DivFreeSolver (linalg/divfree.cpp:42-186): projection of an ND field onto the discretely divergence-free fields ----
 *        rhs = WeakDiv y ;  rhs[h1 essential dofs] = 0 ;  M psi = rhs  (PCG) ;  y += G psi
 * with M the H1 diffusion operator with the permittivity (essential dofs DIAG_ONE), G the discrete gradient and WeakDiv the
 * weak divergence -(eps u, grad v). The reference partially assembles WeakDiv from MixedVectorWeakDivergenceIntegrator
 * (fem/integ/mixedvecgrad.cpp:148-208): the ND mass quadrature function between the ND interpolation and the H1 gradient, negated.
 * grad v_h IS G v for an H1 function, so WeakDiv = -G^T M_eps with M_eps the ND mass operator: `nd_mass` is that operator as a
 * b2p_operator_par WITHOUT essential dofs (one element kernel launch), and no separate mixed operator is set up.
 * Solver as the reference builds it: CG, no initial guess, relative tolerance tol, absolute tolerance epsilon; one level ->
 * the coarse solver alone, n levels -> GeometricMultigridSolver(coarse, h1_P, no auxiliary space, 1 cycle, 1 smoothing
 * iteration, Chebyshev 4th kind of order max(h1_order, 2)). coarse_type / coarse_tol / coarse_max_it / coarse_solver as in
 * b2p_ksp_config (the reference's BoomerAMG stays outside this library). h1_ops[n_levels] carry the essential dofs; when the
 * mesh has no marked boundary the caller constrains one dof (true dof 0 of the first rank) on every level as divfree.cpp:50-81
 * does. Complex fields: one CG iteration on both parts together (ComplexParOperator(M, nullptr)). */
typedef struct b2p_divfree b2p_divfree;
int b2p_divfree_create(b2p_ctx *ctx, b2p_operator *nd_mass, b2p_operator *grad, int n_levels, b2p_operator *const *h1_ops,
                       b2p_operator *const *h1_P, const int32_t *h1_ess_tdofs, int64_t n_ess, int h1_order, double tol, int max_it,
                       int coarse_type, double coarse_tol, int coarse_max_it, b2p_solver *coarse_solver, b2p_divfree **out);
int b2p_divfree_mult(b2p_divfree *d, double *y);                         /* DivFreeSolver<Vector>::Mult, in place */
int b2p_divfree_mult_complex(b2p_divfree *d, double *y_re, double *y_im); /* DivFreeSolver<ComplexVector>::Mult */
int b2p_divfree_stats(b2p_divfree *d, int *num_mult, int *num_mult_its, int *last_its, int *converged);
void b2p_divfree_destroy(b2p_divfree *d);

/* ---- Flux error estimator for H(curl) problems (linalg/errorestimator.cpp:112-270,400-513) ------------------------------------
 * CurlFluxErrorEstimator: the discontinuous flux mu^-1 B (B = curl E, dofs in the RT space) is projected onto the ND space,
 *        M H = Flux B    (FluxProjector: mixed H(div) -> H(curl) mass operator with mu^-1, ND mass matrix, PCG + damped Jacobi),
 * and eta_K^2 = int_K |(mu^-1)^(-1/2) H - (mu^-1)^(1/2) B|^2 is integrated element by element (f_apply_hdivhcurl_error_33); complex
 * fields add the two parts; eta_K = sqrt(s eta_K^2) with s = 0.5 / Et (or 1 when Et <= 0).
 * A space is what libCEED sees of a non-tensor basis (fem/libceed/basis.cpp:40-85, restriction.cpp:281-297): reference-space
 * values interp[3][Q][P] at the quadrature points of `geom` (x fastest for tensor rules), native restriction idx[ne][P] with
 * orient[ne][P] in {+1, -1} (NULL: all +1), and the reference-to-physical map of the values. The three coefficient tables are
 * per ATTRIBUTE, [n_attr][9] column-major: mu^-1, its matrix square root and its inverse square root (linalg::MatrixSqrt /
 * MatrixPow of the reference, computed by the caller). `smooth_mass`: ParOperator of the ND mass integrator (no coefficient, no
 * essential dofs). Single partition only for now (T-vectors = L-vectors); the estimator is post-processing, not hot path. */
enum
{
  B2P_MAP_HCURL = 1, /* u = J^-T u^      (mfem::FiniteElement::H_CURL) */
  B2P_MAP_HDIV = 2   /* u = J u^ / detJ  (mfem::FiniteElement::H_DIV) */
};
typedef struct
{
  int P;                /* dofs per element */
  int map_type;         /* B2P_MAP_HCURL | B2P_MAP_HDIV */
  const double *interp; /* [3][Q][P] */
  const int32_t *idx;   /* [ne][P] */
  const int8_t *orient; /* [ne][P] or NULL */
  int64_t lsize;
  /* [ne][P][3] row-major tridiagonal element transformations of ND tetrahedra / prisms of order >= 2 (restriction.cpp:301-329, as
   * b2p_dense_op_desc.curl_orient) or NULL; when given it carries the signs and `orient` is ignored */
  const int8_t *curl_orient;
} b2p_vecfe_space_desc;
typedef struct b2p_flux_estimator b2p_flux_estimator;
/* VectorFEMassIntegrator on ONE table-described space: y = sum_e E^T B^T (w detJ P^T C P) B E x with the space's map P; coef
 * [n_attr][9] per attribute or NULL (identity). The mass matrix `smooth_mass` of a FluxProjector whose smooth space has no
 * sum-factorised operator here (Raviart-Thomas: GradFluxErrorEstimator, errorestimator.cpp:272-398, with the H(curl) space as
 * the flux space and sqrt(eps), eps^(-1/2) as coef_disc, coef_smooth). Mult and AssembleDiagonal; single partition. */
int b2p_operator_vecfe_mass(b2p_ctx *ctx, b2p_geom *geom, const b2p_vecfe_space_desc *space, int n_attr, const double *coef,
                            b2p_operator **out);
int b2p_flux_estimator_create(b2p_ctx *ctx, b2p_geom *geom, const b2p_vecfe_space_desc *flux_space,
                              const b2p_vecfe_space_desc *smooth_space, int n_attr, const double *coef_flux, const double *coef_disc,
                              const double *coef_smooth, b2p_operator *smooth_mass, double tol, int max_it, b2p_flux_estimator **out);
/* FluxProjector::Mult: smooth_dofs = M^-1 Flux flux_dofs */
int b2p_flux_estimator_project(b2p_flux_estimator *e, const double *flux_dofs, double *smooth_dofs);
/* estimates[ne] += eta_K^2 of one part (device array) */
int b2p_flux_estimator_integrate(b2p_flux_estimator *e, const double *flux_dofs, const double *smooth_dofs, double *estimates);
/* CurlFluxErrorEstimator::AddErrorIndicator: estimates[ne] = sqrt(s (eta_K^2(re) + eta_K^2(im))); flux_im may be NULL */
int b2p_flux_estimator_indicator(b2p_flux_estimator *e, const double *flux_re, const double *flux_im, double Et, double *estimates);
/* estimates[i] = sqrt(s estimates[i]): last step when several flux terms are added before the square root
 * (TimeDependentFluxErrorEstimator: project + integrate of both estimators into one array, errorestimator.cpp:531-545) */
int b2p_flux_estimator_sqrt_scale(b2p_ctx *ctx, int64_t n, double s, double *estimates);
/* FluxProjector with "EstimatorMG" (ConfigureLinearSolver(use_mg = true), errorestimator.cpp:66-100): the projection's PCG is
 * preconditioned by GeometricMultigridSolver(coarse, P, no auxiliary space, 1 cycle, 1 smoothing iteration, 4th-kind Chebyshev of
 * order 2, sf_max 1, sf_min 0) over the smooth space's p-hierarchy -- RT levels for the grad-flux estimator, ND levels for the
 * curl-flux estimator; with one level the coarse solver alone. ops[n_levels] coarse -> fine (ops[n_levels-1] must be the
 * estimator's smooth_mass), P[n_levels-1] the prolongations; coarse_type / coarse_tol / coarse_max_it / coarse_solver as in
 * b2p_ksp_config and b2p_ksp_create. Replaces the Jacobi-preconditioned PCG; tolerances and the statistics stay. */
int b2p_flux_estimator_set_multigrid(b2p_flux_estimator *e, int n_levels, b2p_operator *const *ops, b2p_operator *const *P, int coarse_type,
                                     double coarse_tol, int coarse_max_it, b2p_solver *coarse_solver);
int b2p_flux_estimator_stats(b2p_flux_estimator *e, int *num_mult, int *num_mult_its, int *last_its, int *converged);
void b2p_flux_estimator_destroy(b2p_flux_estimator *e);
/* The flux estimator on hexahedra with sum-factorised spaces: flux_space / smooth_space are b2p_op_desc restricted to their
 * space fields (kind = B2P_ND_MASS or B2P_RT_MASS names the space, one of each; p, ne, lsize, idx, orient, dof_map, Bo, Bc
 * read as b2p_op_create reads them for that kind; coeff_ctx ignored; assemble_qdata must be 0). geom: tensor q-data (q1d > 0).
 * Both spaces are evaluated with the same 1-D tables: the smooth space's Bo / Bc must equal the flux space's (B2P_ERR_ARG otherwise).
 * Coefficient tables, smooth_mass, tol, max_it and the returned handle as b2p_flux_estimator_create. Flux and the error integrals
 * run the sum-factorised kernels of b2p_hex_flux.cu (both directions, general coefficient matrices); project, integrate, indicator,
 * set_multigrid, stats and destroy work on it unchanged. B2P_ERR_ARG: a kind other than ND_MASS / RT_MASS, two spaces of the same
 * type, different p, ne different from the geometry's, a geometry without tensor q-data, smooth_mass of the wrong size, different
 * tables, a restriction index outside [0, lsize); B2P_ERR_UNSUPPORTED: assemble_qdata = 1, nranks > 1, p / q1d outside the hex
 * kernels. The kinds are checked first, so a wrong kind is B2P_ERR_ARG whatever else the description holds. */
int b2p_flux_estimator_create_hex(b2p_ctx *ctx, b2p_geom *geom, const b2p_op_desc *flux_space, const b2p_op_desc *smooth_space,
                                  int n_attr, const double *coef_flux, const double *coef_disc, const double *coef_smooth,
                                  b2p_operator *smooth_mass, double tol, int max_it, b2p_flux_estimator **out);
/* rhs = Flux flux_dofs (the projection's right-hand side), for estimators from either create function */
int b2p_flux_estimator_flux_mult(b2p_flux_estimator *e, const double *flux_dofs, double *rhs);

#ifdef __cplusplus
}
#endif
#endif /* B2P_H */
