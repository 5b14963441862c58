// C ABI of the linear-algebra / solver layer (include/b2p.h): thin handles over the C++ classes.
#include "b2p_linalg.hpp"

using namespace b2p;

struct b2p_halo;
namespace b2p
{
Halo *halo_of(b2p_halo *h);
}

struct b2p_operator
{
  std::unique_ptr<Operator> op;
};
struct b2p_solver
{
  std::unique_ptr<Solver> s;
  bool owned_elsewhere = false;
};

namespace b2p
{
Solver *solver_of(b2p_solver *s) { return s ? s->s.get() : nullptr; }
std::unique_ptr<Solver> take_solver(b2p_solver *s) { return s ? std::move(s->s) : nullptr; }
Operator *operator_of(b2p_operator *A) { return A ? A->op.get() : nullptr; }
b2p_operator *wrap_operator(std::unique_ptr<Operator> &&op)  // (handles of operators built in other translation units)
{
  auto *h = new b2p_operator;
  h->op = std::move(op);
  return h;
}
b2p_solver *wrap_solver(std::unique_ptr<Solver> &&s)
{
  auto *h = new b2p_solver;
  h->s = std::move(s);
  return h;
}
}  // namespace b2p

#define B2P_TRY(ctx, stmt)                                   \
  do                                                         \
  {                                                          \
    stmt;                                                    \
    cudaError_t e__ = cudaPeekAtLastError();                 \
    if (e__ != cudaSuccess)                                  \
    {                                                        \
      set_error(ctx, "CUDA error: %s", cudaGetErrorString(e__)); \
      return B2P_ERR_CUDA;                                   \
    }                                                        \
  } while (0)

extern "C"
{

int b2p_ctx_set_stream(b2p_ctx *ctx, b2p_stream s)
{
  if (!ctx) return B2P_ERR_ARG;
  ctx->stream = (cudaStream_t)s;
  return B2P_SUCCESS;
}

int b2p_vec_axpby(b2p_ctx *ctx, int64_t n, double a, const double *x, double b, double *y)
{
  B2P_TRY(ctx, vec::axpby(ctx, a, x, b, y, n));
  return B2P_SUCCESS;
}
int b2p_vec_axpbypcz(b2p_ctx *ctx, int64_t n, double a, const double *x, double b, const double *y, double g, double *z)
{
  B2P_TRY(ctx, vec::axpbypcz(ctx, a, x, b, y, g, z, n));
  return B2P_SUCCESS;
}
int b2p_vec_dot(b2p_ctx *ctx, int64_t n, const double *x, const double *y, double *out)
{
  B2P_TRY(ctx, *out = vec::dot(ctx, x, y, n));
  return B2P_SUCCESS;
}
int b2p_vec_sum(b2p_ctx *ctx, int64_t n, const double *x, double *out)
{
  B2P_TRY(ctx, *out = vec::sum(ctx, x, n));
  return B2P_SUCCESS;
}
int b2p_vec_set_sub(b2p_ctx *ctx, double *y, const int32_t *idx_dev, int64_t nidx, double v)
{
  B2P_TRY(ctx, vec::set_sub(ctx, y, idx_dev, nidx, v));
  return B2P_SUCCESS;
}
int b2p_vec_set_random(b2p_ctx *ctx, int64_t n, double *y, uint64_t seed)
{
  B2P_TRY(ctx, vec::set_random(ctx, y, n, seed));
  return B2P_SUCCESS;
}
int b2p_vec_orthogonalize(b2p_ctx *ctx, int type, int64_t n, int m, const double *const *V, double *w, double *H)
{
  if (m <= 0) return B2P_SUCCESS;
  if (type == 0)
  {
    for (int j = 0; j < m; j++)
    {
      H[j] = vec::dot(ctx, w, V[j], n);
      vec::axpy(ctx, -H[j], V[j], w, n);
    }
  }
  else
  {
    vec::multi_dot(ctx, m, V, w, n, H);
    vec::multi_axpy(ctx, m, H, V, w, n, -1.0);
    if (type == 2)
    {
      std::vector<double> dH(m);
      vec::multi_dot(ctx, m, V, w, n, dH.data());
      vec::multi_axpy(ctx, m, dH.data(), V, w, n, -1.0);
      for (int j = 0; j < m; j++) H[j] += dH[j];
    }
  }
  cudaError_t e = cudaPeekAtLastError();
  B2P_CHECK(ctx, e == cudaSuccess, B2P_ERR_CUDA, "orthogonalize: %s", cudaGetErrorString(e));
  return B2P_SUCCESS;
}

int b2p_operator_par(b2p_ctx *ctx, int64_t tsize, int64_t lsize, int n_terms, b2p_op *const *ops, const double *coefs,
                     const int32_t *ess_tdofs, int64_t n_ess, int diag_policy, b2p_halo *halo, b2p_operator **out)
{
  B2P_CHECK(ctx, ctx && out && n_terms > 0 && ops, B2P_ERR_ARG, "b2p_operator_par: bad argument");
  std::vector<ParOperator::Term> terms;
  for (int i = 0; i < n_terms; i++)
  {
    B2P_CHECK(ctx, ops[i] && b2p_op_lsize(ops[i]) == lsize, B2P_ERR_ARG, "b2p_operator_par: term %d has the wrong L-size", i);
    // Operators built on one b2p_op share its masked restriction. On a single partition the mask is installed from
    // ess_tdofs by the first operator; a later one with another essential set would silently reuse it (wrong columns
    // eliminated), so it is refused. (Partitioned callers install the mask themselves, with ghost copies, in L indices.)
    B2P_CHECK(ctx, halo || !ops[i]->lidx_bc || op_essential_matches(ops[i], ess_tdofs, n_ess), B2P_ERR_ARG,
              "b2p_operator_par: term %d already carries a different essential-dof mask (one b2p_op = one essential set; "
              "create a second b2p_op or call b2p_op_set_essential again)", i);
    terms.push_back({ops[i], coefs ? coefs[i] : 1.0});
  }
  auto *h = new b2p_operator;
  h->op = std::make_unique<ParOperator>(ctx, tsize, lsize, terms, ess_tdofs, n_ess, diag_policy, halo ? halo_of(halo) : nullptr);
  *out = h;
  return B2P_SUCCESS;
}
namespace
{
// The assembled coarse-level matrix behind the Operator interface, so that the Krylov solvers and smoothers can run on it
// (the reference hands the assembled coarse matrix to its coarse solver, linalg/ksp.cpp:ConfigurePreconditionerSolver).
class CsrOperator : public Operator
{
  b2p_csr *A;

public:
  CsrOperator(b2p_ctx *c, b2p_csr *a) : Operator(c, b2p_csr_rows(a), b2p_csr_rows(a)), A(a) {}
  void Mult(const double *x, double *y) const override { b2p_csr_mult(A, x, y, (b2p_stream)ctx->stream); }
  void AssembleDiagonal(double *d) const override { b2p_csr_diag(A, d, (b2p_stream)ctx->stream); }
  b2p_csr *AssembledMatrix(const double **val) const override
  {
    *val = csr_values(A);
    return A;
  }
};
// A solver that runs on the ASSEMBLED matrix of the ParOperator it is given (MfemWrapperSolver::SetOperator,
// linalg/solver.cpp:13-30: "Operator is always assembled as a HypreParMatrix"): SetOperator assembles and eliminates the
// sum on the device and hands the matrix to the inner solver and its preconditioner. This is how the multigrid's coarse
// solver sees level 0.
class AssembledSolver : public Solver
{
  std::unique_ptr<Solver> inner, pc;
  b2p_csr *csr = nullptr;
  std::unique_ptr<CsrOperator> Ac;

public:
  AssembledSolver(b2p_ctx *c, std::unique_ptr<Solver> &&in, std::unique_ptr<Solver> &&p) : Solver(c), inner(std::move(in)), pc(std::move(p)) {}
  ~AssembledSolver() override { b2p_csr_destroy(csr); }
  void SetOperator(const Operator &op) override
  {
    const auto *pa = dynamic_cast<const ParOperator *>(&op);
    if (!pa)
    {
      set_error(ctx, "AssembledSolver must be able to assemble its operator: ParOperator required");
      return;
    }
    b2p_csr *A = pa->FullAssemble();
    if (!A) return;
    b2p_csr_destroy(csr);
    csr = A;
    Ac = std::make_unique<CsrOperator>(ctx, csr);
    if (pc) pc->SetOperator(*Ac);
    inner->SetOperator(*Ac);
    height = op.Height();
    width = op.Width();
  }
  void Mult(const double *x, double *y) const override
  {
    inner->SetInitialGuess(initial_guess);
    inner->Mult(x, y);
  }
  const b2p_csr *Matrix() const { return csr; }
  const Solver *Inner() const { return inner.get(); }
  int Status() const override { return inner->Status(); }
};
}  // namespace
}  // extern "C"
namespace b2p
{
// The solver that runs on the assembled matrix: s itself, the inner solver of a b2p_solver_assembled, and either of them as
// the coarse solver a multigrid took over.
const Solver *unwrap_coarse_solver(const Solver *s)
{
  if (auto *g = dynamic_cast<const GeometricMultigridSolver *>(s)) s = g->B[0].get();
  if (auto *a = dynamic_cast<const AssembledSolver *>(s)) s = a->Inner();
  return s;
}
}  // namespace b2p
extern "C"
{
int b2p_operator_csr(b2p_ctx *ctx, b2p_csr *A, b2p_operator **out)
{
  B2P_CHECK(ctx, ctx && A && out, B2P_ERR_ARG, "b2p_operator_csr: null argument");
  auto *h = new b2p_operator;
  h->op = std::make_unique<CsrOperator>(ctx, A);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_operator_par_set_coefficients(b2p_operator *A, int n_terms, const double *coefs)
{
  auto *pa = A ? dynamic_cast<ParOperator *>(A->op.get()) : nullptr;
  if (!pa || !coefs || n_terms != (int)pa->NumTerms()) return B2P_ERR_ARG;
  pa->SetCoefficients(coefs);
  return B2P_SUCCESS;
}
int b2p_operator_par_is_fused(b2p_operator *A)
{
  auto *pa = A ? dynamic_cast<ParOperator *>(A->op.get()) : nullptr;
  return pa ? (pa->Fused() ? 1 : 0) : -1;
}
int b2p_operator_par_set_interior(b2p_operator *A, int ne_interior)
{
  auto *pa = A ? dynamic_cast<ParOperator *>(A->op.get()) : nullptr;
  if (!pa || ne_interior < 0) return B2P_ERR_ARG;
  pa->SetInteriorElements(ne_interior);
  return B2P_SUCCESS;
}
int b2p_operator_interp(b2p_ctx *ctx, b2p_interp *it, b2p_halo *in_halo, int64_t in_tsize, b2p_halo *out_halo,
                        int64_t out_tsize, b2p_operator **out)
{
  B2P_CHECK(ctx, ctx && it && out, B2P_ERR_ARG, "b2p_operator_interp: bad argument");
  auto *h = new b2p_operator;
  h->op = std::make_unique<InterpOperator>(ctx, it, in_halo ? halo_of(in_halo) : nullptr, in_tsize,
                                           out_halo ? halo_of(out_halo) : nullptr, out_tsize);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_operator_mult(b2p_operator *A, const double *x, double *y)
{
  if (!A) return B2P_ERR_ARG;
  B2P_TRY(A->op->ctx, A->op->Mult(x, y));
  return B2P_SUCCESS;
}
int b2p_operator_mult_transpose(b2p_operator *A, const double *x, double *y)
{
  if (!A) return B2P_ERR_ARG;
  if (auto *pa = dynamic_cast<ParOperator *>(A->op.get()))
    B2P_CHECK(pa->ctx, pa->TransposeAvailable(), B2P_ERR_UNSUPPORTED,
              "b2p_operator_mult_transpose: non-symmetric terms (B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL) on a partitioned space are not supported");
  B2P_TRY(A->op->ctx, A->op->MultTranspose(x, y));
  return B2P_SUCCESS;
}
int b2p_operator_add_mult(b2p_operator *A, const double *x, double *y, double a)
{
  if (!A) return B2P_ERR_ARG;
  B2P_TRY(A->op->ctx, A->op->AddMult(x, y, a));
  return B2P_SUCCESS;
}
int b2p_operator_assemble_diagonal(b2p_operator *A, double *d)
{
  if (!A) return B2P_ERR_ARG;
  B2P_TRY(A->op->ctx, A->op->AssembleDiagonal(d));
  return B2P_SUCCESS;
}
int64_t b2p_operator_height(b2p_operator *A) { return A ? A->op->Height() : 0; }
int64_t b2p_operator_width(b2p_operator *A) { return A ? A->op->Width() : 0; }
void b2p_operator_destroy(b2p_operator *A) { delete A; }

int b2p_solver_jacobi(b2p_ctx *ctx, double omega, double sf_max, b2p_solver **out)
{
  auto *h = new b2p_solver;
  h->s = std::make_unique<JacobiSmoother>(ctx, omega, sf_max);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_solver_chebyshev(b2p_ctx *ctx, int smooth_it, int order, double sf_max, double sf_min, int fourth_kind, b2p_solver **out)
{
  B2P_CHECK(ctx, order > 0, B2P_ERR_ARG, "Polynomial order for Chebyshev smoothing must be positive!");
  auto *h = new b2p_solver;
  h->s = std::make_unique<ChebyshevSmoother>(ctx, smooth_it, order, sf_max, sf_min, fourth_kind != 0);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_solver_distrelax(b2p_ctx *ctx, b2p_operator *G, int smooth_it, int cheby_smooth_it, int cheby_order, double sf_max,
                         double sf_min, int fourth_kind, b2p_solver **out)
{
  B2P_CHECK(ctx, G, B2P_ERR_ARG, "b2p_solver_distrelax: missing G");
  auto *h = new b2p_solver;
  h->s = std::make_unique<DistRelaxationSmoother>(ctx, *G->op, smooth_it, cheby_smooth_it, cheby_order, sf_max, sf_min,
                                                  fourth_kind != 0);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_solver_distrelax_set_operators(b2p_solver *s, b2p_operator *A, b2p_operator *A_G)
{
  auto *d = s ? dynamic_cast<DistRelaxationSmoother *>(s->s.get()) : nullptr;
  Operator *pa = A ? A->op.get() : nullptr, *pg = A_G ? A_G->op.get() : nullptr;  // ParOperator or its general-prolongation form
  if (!d || !pa || !pg) return B2P_ERR_ARG;
  B2P_TRY(d->ctx, d->SetOperators(*pa, *pg));
  return B2P_SUCCESS;
}
int b2p_solver_gmg(b2p_ctx *ctx, b2p_solver *coarse, int n_levels, b2p_operator *const *P, b2p_operator *const *G, int cycle_it,
                   int smooth_it, int cheby_order, double sf_max, double sf_min, int fourth_kind, b2p_solver **out)
{
  B2P_CHECK(ctx, coarse && coarse->s && n_levels >= 1 && out && (P || n_levels == 1), B2P_ERR_ARG, "b2p_solver_gmg: bad argument");
  std::vector<const Operator *> Pv, Gv;
  for (int l = 0; l + 1 < n_levels; l++)
  {
    B2P_CHECK(ctx, P[l] && P[l]->op, B2P_ERR_ARG, "b2p_solver_gmg: no prolongation between levels %d and %d", l, l + 1);
    Pv.push_back(P[l]->op.get());
  }
  if (G)
    for (int l = 0; l < n_levels; l++)
    {
      // every level above the coarsest gets a DistRelaxationSmoother built on G[l] (gmg.cpp:45-50); G[0] is unused
      B2P_CHECK(ctx, l == 0 || (G[l] && G[l]->op), B2P_ERR_ARG, "b2p_solver_gmg: level %d has no discrete gradient", l);
      Gv.push_back(G[l] ? G[l]->op.get() : nullptr);
    }
  auto *h = new b2p_solver;
  h->s = std::make_unique<GeometricMultigridSolver>(ctx, std::move(coarse->s), Pv, Gv, cycle_it, smooth_it, cheby_order, sf_max,
                                                    sf_min, fourth_kind != 0);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_solver_gmg_set_operators(b2p_solver *s, b2p_operator *const *A, b2p_operator *const *A_aux)
{
  auto *g = s ? dynamic_cast<GeometricMultigridSolver *>(s->s.get()) : nullptr;
  if (!g || !A) return B2P_ERR_ARG;
  std::vector<const Operator *> Av, Gv;
  for (size_t l = 0; l < g->A.size(); l++)
  {
    B2P_CHECK(g->ctx, A[l] && A[l]->op, B2P_ERR_ARG, "b2p_solver_gmg_set_operators: level %d has no operator", (int)l);
    Av.push_back(A[l]->op.get());  // a ParOperator (b2p_operator_par) or its general-prolongation form (b2p_operator_rap)
    Operator *pg = (A_aux && A_aux[l]) ? A_aux[l]->op.get() : nullptr;
    // a level smoothed by DistRelaxationSmoother (the multigrid was built with discrete gradients) needs its auxiliary-space operator
    const bool dist = dynamic_cast<DistRelaxationSmoother *>(g->B[l].get()) != nullptr;
    B2P_CHECK(g->ctx, !dist || pg, B2P_ERR_ARG, "b2p_solver_gmg_set_operators: level %d needs an auxiliary-space ParOperator", (int)l);
    Gv.push_back(pg);
  }
  B2P_TRY(g->ctx, g->SetOperators(Av, Gv));
  return B2P_SUCCESS;
}
int b2p_solver_assembled(b2p_ctx *ctx, b2p_solver *inner, b2p_solver *inner_pc, b2p_solver **out)
{
  B2P_CHECK(ctx, ctx && inner && inner->s && out, B2P_ERR_ARG, "b2p_solver_assembled: bad argument");
  auto *k = dynamic_cast<IterativeSolver *>(inner->s.get());
  if (inner_pc)
  {
    B2P_CHECK(ctx, inner_pc->s && k, B2P_ERR_ARG, "b2p_solver_assembled: a preconditioner needs a Krylov inner solver");
    k->SetPreconditioner(inner_pc->s.get());
  }
  auto *h = new b2p_solver;
  h->s = std::make_unique<AssembledSolver>(ctx, std::move(inner->s), inner_pc ? std::move(inner_pc->s) : nullptr);
  *out = h;
  return B2P_SUCCESS;
}
int64_t b2p_solver_assembled_nnz(b2p_solver *s)
{
  const Solver *p = s ? s->s.get() : nullptr;
  if (auto *g = dynamic_cast<const GeometricMultigridSolver *>(p)) p = g->B[0].get();  // the multigrid took the coarse solver over
  auto *a = dynamic_cast<const AssembledSolver *>(p);
  return a && a->Matrix() ? b2p_csr_nnz(a->Matrix()) : -1;
}
int b2p_solver_krylov(b2p_ctx *ctx, int type, b2p_solver **out)
{
  B2P_CHECK(ctx, type >= 0 && type <= 2, B2P_ERR_ARG, "b2p_solver_krylov: type must be 0 (CG), 1 (GMRES) or 2 (FGMRES)");
  auto *h = new b2p_solver;
  h->s = std::make_unique<IterativeSolver>(ctx, (KspType)type);
  *out = h;
  return B2P_SUCCESS;
}
int b2p_solver_krylov_config(b2p_solver *s, double rel_tol, double abs_tol, int max_it, int max_dim, int orthog, int pc_side)
{
  auto *k = s ? dynamic_cast<IterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  k->rel_tol = rel_tol;
  k->abs_tol = abs_tol;
  k->max_it = max_it;
  k->max_dim = max_dim;
  k->gs = (Orthog)orthog;
  k->pc_side = (PcSide)pc_side;
  return B2P_SUCCESS;
}
int b2p_solver_krylov_set_check_interval(b2p_solver *s, int check_every)
{
  auto *k = s ? dynamic_cast<IterativeSolver *>(s->s.get()) : nullptr;
  if (!k || check_every < 1) return B2P_ERR_ARG;
  k->check_every = check_every;
  return B2P_SUCCESS;
}
int b2p_solver_set_preconditioner(b2p_solver *s, b2p_solver *pc)
{
  auto *k = s ? dynamic_cast<IterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  k->SetPreconditioner(pc ? pc->s.get() : nullptr);
  return B2P_SUCCESS;
}
int b2p_solver_set_operator(b2p_solver *s, b2p_operator *A)
{
  if (!s || !s->s || !A) return B2P_ERR_ARG;
  B2P_TRY(s->s->ctx, s->s->SetOperator(*A->op));
  return s->s->Status();
}
int b2p_solver_set_initial_guess(b2p_solver *s, int flag)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  s->s->SetInitialGuess(flag != 0);
  return B2P_SUCCESS;
}
int b2p_solver_mult(b2p_solver *s, const double *x, double *y)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  B2P_CHECK(s->s->ctx, s->s->Height() > 0, B2P_ERR_ARG, "solver applied before SetOperator (a preconditioner needs its own set_operator call, as in Palace's KspSolver::SetOperators)");
  if (auto *k = dynamic_cast<IterativeSolver *>(s->s.get()))
    B2P_CHECK(k->ctx, k->type != KspType::FGMRES || k->B, B2P_ERR_ARG, "Operator and preconditioner must be set for FgmresSolver::Mult!");  // iterative.cpp:738
  B2P_TRY(s->s->ctx, s->s->Mult(x, y));
  return B2P_SUCCESS;
}
int b2p_solver_mult2(b2p_solver *s, const double *x, double *y, double *r)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  B2P_CHECK(s->s->ctx, s->s->Height() > 0, B2P_ERR_ARG, "solver applied before SetOperator (a preconditioner needs its own set_operator call, as in Palace's KspSolver::SetOperators)");
  B2P_TRY(s->s->ctx, s->s->Mult2(x, y, r));
  return B2P_SUCCESS;
}
int b2p_solver_mult_transpose2(b2p_solver *s, const double *x, double *y, double *r)
{
  if (!s || !s->s) return B2P_ERR_ARG;
  B2P_CHECK(s->s->ctx, s->s->Height() > 0, B2P_ERR_ARG, "solver applied before SetOperator (a preconditioner needs its own set_operator call, as in Palace's KspSolver::SetOperators)");
  B2P_TRY(s->s->ctx, s->s->MultTranspose2(x, y, r));
  return B2P_SUCCESS;
}
int b2p_solver_stats(b2p_solver *s, int *its, double *initial_res, double *final_res, int *converged)
{
  auto *k = s ? dynamic_cast<IterativeSolver *>(s->s.get()) : nullptr;
  if (!k) return B2P_ERR_ARG;
  if (its) *its = k->final_it;
  if (initial_res) *initial_res = k->initial_res;
  if (final_res) *final_res = k->final_res;
  if (converged) *converged = k->converged ? 1 : 0;
  return B2P_SUCCESS;
}
int b2p_solver_lambda_max(b2p_solver *s, double *out)
{
  auto *c = s ? dynamic_cast<ChebyshevSmoother *>(s->s.get()) : nullptr;
  if (!c || !out) return B2P_ERR_ARG;
  *out = c->lambda_max;
  return B2P_SUCCESS;
}
void b2p_solver_destroy(b2p_solver *s) { delete s; }

}  // extern "C"

// BaseKspSolver (ksp.cpp:256-328): owns the Krylov solver and its preconditioner, counts solves and iterations.
struct b2p_ksp
{
  b2p_ctx *ctx = nullptr;
  b2p_ksp_config cfg;
  int n_levels = 1;
  std::unique_ptr<IterativeSolver> ksp;
  std::unique_ptr<Solver> pc;
  int ksp_mult = 0, ksp_mult_it = 0;
};

namespace b2p
{
IterativeSolver *ksp_solver_of(b2p_ksp *k) { return k ? k->ksp.get() : nullptr; }  // (the flux estimator's multigrid PCG)
}

extern "C"
{

int b2p_ksp_config_default(b2p_ksp_config *c, int order)
{
  if (!c || order < 1) return B2P_ERR_ARG;
  c->krylov_solver = 1;  // GMRES for the frequency-domain problems (iodata.cpp:480-498); CG for the SPD ones
  c->tol = 1e-6;
  c->max_it = 100;
  c->max_size = -1;
  c->initial_guess = 1;
  c->pc_side = -1;
  c->gs_orthog = 0;
  c->mg_cycle_it = 1;
  c->mg_smooth_aux = 1;
  c->mg_smooth_it = 1;
  c->mg_smooth_order = std::max(2 * order, 4);  // iodata.cpp:533-536
  c->mg_smooth_sf_max = 1.0;
  c->mg_smooth_sf_min = 0.0;
  c->mg_smooth_cheby_4th = 1;
  c->coarse_type = 1;
  c->coarse_tol = 1e-3;
  c->coarse_max_it = 500;
  return B2P_SUCCESS;
}

int b2p_ksp_create(b2p_ctx *ctx, const b2p_ksp_config *cfg, int n_levels, b2p_operator *const *P, b2p_operator *const *G,
                   b2p_solver *coarse_solver, b2p_ksp **out)
{
  B2P_CHECK(ctx, ctx && cfg && out && n_levels >= 1, B2P_ERR_ARG, "b2p_ksp_create: bad argument");
  B2P_CHECK(ctx, cfg->krylov_solver >= 0 && cfg->krylov_solver <= 2, B2P_ERR_ARG,
            "b2p_ksp_create: Unexpected solver type for Krylov solver configuration!");
  B2P_CHECK(ctx, n_levels == 1 || P, B2P_ERR_ARG, "b2p_ksp_create: a multigrid hierarchy needs its prolongation operators");
  B2P_CHECK(ctx, n_levels == 1 || !cfg->mg_smooth_aux || G, B2P_ERR_ARG,
            "Multigrid with auxiliary space smoothers requires both primary space and auxiliary spaces for construction!");
  auto k = std::make_unique<b2p_ksp>();
  k->ctx = ctx;
  k->cfg = *cfg;
  k->n_levels = n_levels;
  // ConfigureKrylovSolver (ksp.cpp:29-102)
  k->ksp = std::make_unique<IterativeSolver>(ctx, (KspType)cfg->krylov_solver);
  k->ksp->rel_tol = cfg->tol;
  k->ksp->max_it = cfg->max_it;
  k->ksp->max_dim = cfg->max_size > 0 ? cfg->max_size : cfg->max_it;
  k->ksp->gs = (Orthog)cfg->gs_orthog;
  if (cfg->pc_side >= 0 && cfg->krylov_solver != 0) k->ksp->pc_side = (PcSide)cfg->pc_side;  // ignored for CG, as in the reference
  k->ksp->SetInitialGuess(cfg->initial_guess != 0);
  // ConfigurePreconditionerSolver (ksp.cpp:131-239): the coarse solver first ...
  std::unique_ptr<Solver> coarse;
  switch (cfg->coarse_type)
  {
    case 0: coarse = std::make_unique<JacobiSmoother>(ctx, 1.0, 1.0); break;
    case 1:
    {
      auto cg = std::make_unique<IterativeSolver>(ctx, KspType::CG);
      cg->rel_tol = cfg->coarse_tol;
      cg->max_it = cfg->coarse_max_it;
      auto jac = std::make_unique<JacobiSmoother>(ctx, 1.0, 1.0);
      cg->SetPreconditioner(jac.get());
      coarse = std::make_unique<AssembledSolver>(ctx, std::move(cg), std::move(jac));
      break;
    }
    case 2:
      B2P_CHECK(ctx, coarse_solver && coarse_solver->s, B2P_ERR_ARG, "b2p_ksp_create: coarse_type 2 needs a coarse solver");
      coarse = std::move(coarse_solver->s);
      break;
    default: B2P_CHECK(ctx, false, B2P_ERR_ARG, "Unexpected solver type for preconditioner configuration!");
  }
  // ... then the multigrid hierarchy around it when there is more than one level
  if (n_levels > 1)
  {
    std::vector<const Operator *> Pv, Gv;
    for (int l = 0; l + 1 < n_levels; l++)
    {
      B2P_CHECK(ctx, P[l] && P[l]->op, B2P_ERR_ARG, "b2p_ksp_create: no prolongation between levels %d and %d", l, l + 1);
      Pv.push_back(P[l]->op.get());
    }
    if (cfg->mg_smooth_aux)
      for (int l = 0; l < n_levels; l++)
      {
        B2P_CHECK(ctx, l == 0 || (G[l] && G[l]->op), B2P_ERR_ARG, "b2p_ksp_create: level %d has no discrete gradient", l);
        Gv.push_back(G[l] ? G[l]->op.get() : nullptr);
      }
    k->pc = std::make_unique<GeometricMultigridSolver>(ctx, std::move(coarse), Pv, Gv, cfg->mg_cycle_it, cfg->mg_smooth_it,
                                                       cfg->mg_smooth_order, cfg->mg_smooth_sf_max, cfg->mg_smooth_sf_min,
                                                       cfg->mg_smooth_cheby_4th != 0);
  }
  else
    k->pc = std::move(coarse);
  k->ksp->SetPreconditioner(k->pc.get());
  *out = k.release();
  return B2P_SUCCESS;
}

int b2p_ksp_set_operators(b2p_ksp *k, b2p_operator *op, b2p_operator *const *pc_ops, b2p_operator *const *aux_ops)
{
  if (!k || !op || !pc_ops) return B2P_ERR_ARG;
  b2p_ctx *ctx = k->ctx;
  B2P_TRY(ctx, k->ksp->SetOperator(*op->op));  // ksp.cpp:295-297
  if (auto *g = dynamic_cast<GeometricMultigridSolver *>(k->pc.get()))
  {
    std::vector<const Operator *> Av, Gv;
    for (int l = 0; l < k->n_levels; l++)
    {
      B2P_CHECK(ctx, pc_ops[l] && pc_ops[l]->op, B2P_ERR_ARG, "b2p_ksp_set_operators: level %d has no operator", l);
      Av.push_back(pc_ops[l]->op.get());
      Operator *pg = (aux_ops && aux_ops[l]) ? aux_ops[l]->op.get() : nullptr;
      const bool dist = dynamic_cast<DistRelaxationSmoother *>(g->B[l].get()) != nullptr;
      B2P_CHECK(ctx, !dist || pg, B2P_ERR_ARG, "b2p_ksp_set_operators: level %d needs an auxiliary-space ParOperator", l);
      Gv.push_back(pg);
    }
    B2P_TRY(ctx, g->SetOperators(Av, Gv));
  }
  else
  {
    // one level: the finest (only) preconditioner operator goes to the solver itself (ksp.cpp:302-305)
    B2P_CHECK(ctx, pc_ops[0] && pc_ops[0]->op, B2P_ERR_ARG, "b2p_ksp_set_operators: no preconditioner operator");
    B2P_TRY(ctx, k->pc->SetOperator(*pc_ops[0]->op));
  }
  return B2P_SUCCESS;
}

int b2p_ksp_mult(b2p_ksp *k, const double *x, double *y)
{
  if (!k || !x || !y) return B2P_ERR_ARG;
  B2P_CHECK(k->ctx, k->ksp->Height() > 0, B2P_ERR_ARG, "b2p_ksp_mult before b2p_ksp_set_operators");
  B2P_TRY(k->ctx, k->ksp->Mult(x, y));
  if (!k->ksp->converged)
    set_error(k->ctx, "Linear solver did not converge, norm(Ax-b)/norm(b) = %.3e (norm(b) = %.3e)!", k->ksp->final_res / k->ksp->initial_res,
              k->ksp->initial_res);  // a warning in the reference (ksp.cpp:316-322): recorded, not an error code
  k->ksp_mult++;
  k->ksp_mult_it += k->ksp->final_it;
  return B2P_SUCCESS;
}

int b2p_ksp_stats(b2p_ksp *k, int *num_total_mult, int *num_total_mult_its, int *last_its, double *initial_res, double *final_res,
                  int *converged)
{
  if (!k) return B2P_ERR_ARG;
  if (num_total_mult) *num_total_mult = k->ksp_mult;
  if (num_total_mult_its) *num_total_mult_its = k->ksp_mult_it;
  if (last_its) *last_its = k->ksp->final_it;
  if (initial_res) *initial_res = k->ksp->initial_res;
  if (final_res) *final_res = k->ksp->final_res;
  if (converged) *converged = k->ksp->converged ? 1 : 0;
  return B2P_SUCCESS;
}

void b2p_ksp_destroy(b2p_ksp *k) { delete k; }

}  // extern "C"

// ---------------------------------------------------------------- DivFreeSolver (linalg/divfree.cpp)
namespace b2p
{
// The complex instantiation of the reference runs ONE Krylov iteration on the complex vector with the real operators applied to
// both parts (ComplexParOperator(M, nullptr), divfree.cpp:36-41): the same recurrence as real CG on the stacked vector
// [re; im] with diag(M, M) and diag(B, B) (the operator is Hermitian, so every inner product is real).
class TwoPartOperator : public Operator
{
public:
  TwoPartOperator(b2p_ctx *c, const Operator *A_) : Operator(c, 2 * A_->Height(), 2 * A_->Width()), A(A_) {}
  void Mult(const double *x, double *y) const override
  {
    A->Mult(x, y);
    A->Mult(x + A->Width(), y + A->Height());
  }
  const Operator *A;
};
class TwoPartSolver : public Solver
{
public:
  TwoPartSolver(b2p_ctx *c, const Solver *B_, int64_t n_) : Solver(c), B(B_), n(n_) { height = width = 2 * n_; }
  void SetOperator(const Operator &) override {}
  void Mult(const double *x, double *y) const override
  {
    B->Mult(x, y);
    B->Mult(x + n, y + n);
  }
  const Solver *B;
  int64_t n;
};
}  // namespace b2p

struct b2p_divfree
{
  b2p_ctx *ctx = nullptr;
  const Operator *Mnd = nullptr, *Grad = nullptr;
  b2p_ksp *ksp = nullptr;
  std::unique_ptr<TwoPartOperator> A2;
  std::unique_ptr<TwoPartSolver> B2;
  std::unique_ptr<IterativeSolver> ksp2;
  int32_t *d_ess = nullptr;
  int64_t n_ess = 0, n_h1 = 0, n_nd = 0;
  DVec t_nd, rhs, psi;
  int mult = 0, mult_it = 0, last_it = 0;
  bool last_converged = true;
  ~b2p_divfree()
  {
    b2p_ksp_destroy(ksp);
    cudaFree(d_ess);
  }
};

extern "C"
{

int b2p_divfree_create(b2p_ctx *ctx, b2p_operator *nd_mass, b2p_operator *grad, int n_levels, b2p_operator *const *h1_ops,
                       b2p_operator *const *h1_P, const int32_t *h1_ess_tdofs, int64_t n_ess, int h1_order, double tol, int max_it,
                       int coarse_type, double coarse_tol, int coarse_max_it, b2p_solver *coarse_solver, b2p_divfree **out)
{
  B2P_CHECK(ctx, ctx && nd_mass && nd_mass->op && grad && grad->op && h1_ops && out && n_levels >= 1 && h1_order >= 1, B2P_ERR_ARG,
            "b2p_divfree_create: bad argument");
  B2P_CHECK(ctx, n_ess == 0 || h1_ess_tdofs, B2P_ERR_ARG, "b2p_divfree_create: essential dof list missing");
  b2p_operator *fine = h1_ops[n_levels - 1];
  B2P_CHECK(ctx, fine && fine->op, B2P_ERR_ARG, "b2p_divfree_create: no operator on the finest H1 level");
  B2P_CHECK(ctx, grad->op->Width() == fine->op->Height() && grad->op->Height() == nd_mass->op->Height() &&
                     nd_mass->op->Height() == nd_mass->op->Width(),
            B2P_ERR_ARG, "b2p_divfree_create: sizes of the mass operator (%lld), the gradient (%lld x %lld) and the H1 operator (%lld) do not match",
            (long long)nd_mass->op->Height(), (long long)grad->op->Height(), (long long)grad->op->Width(), (long long)fine->op->Height());
  auto d = std::make_unique<b2p_divfree>();
  d->ctx = ctx;
  d->Mnd = nd_mass->op.get();
  d->Grad = grad->op.get();
  d->n_h1 = fine->op->Height();
  d->n_nd = nd_mass->op->Height();
  // PCG, no initial guess, relative tolerance `tol`, absolute tolerance epsilon (divfree.cpp:137-143); preconditioner: the coarse
  // solver alone on one level, else GeometricMultigridSolver(coarse, P, no auxiliary space, 1 cycle, 1 smoothing iteration,
  // Chebyshev order max(p, 2), sf_max 1, sf_min 0, 4th kind) (divfree.cpp:121-135)
  b2p_ksp_config cfg;
  b2p_ksp_config_default(&cfg, h1_order);
  cfg.krylov_solver = 0;
  cfg.tol = tol;
  cfg.max_it = max_it;
  cfg.initial_guess = 0;
  cfg.mg_cycle_it = 1;
  cfg.mg_smooth_aux = 0;
  cfg.mg_smooth_it = 1;
  cfg.mg_smooth_order = std::max(h1_order, 2);
  cfg.mg_smooth_sf_max = 1.0;
  cfg.mg_smooth_sf_min = 0.0;
  cfg.mg_smooth_cheby_4th = 1;
  cfg.coarse_type = coarse_type;
  cfg.coarse_tol = coarse_tol;
  cfg.coarse_max_it = coarse_max_it;
  int rc = b2p_ksp_create(ctx, &cfg, n_levels, h1_P, nullptr, coarse_solver, &d->ksp);
  if (rc) return rc;
  d->ksp->ksp->abs_tol = 2.220446049250313e-16;
  if ((rc = b2p_ksp_set_operators(d->ksp, fine, h1_ops, nullptr))) return rc;  // ksp->SetOperators(*M, *M)
  if (n_ess > 0)
  {
    if ((rc = upload(ctx, h1_ess_tdofs, (size_t)n_ess, &d->d_ess))) return rc;
    d->n_ess = n_ess;
  }
  *out = d.release();
  return B2P_SUCCESS;
}

// rhs = WeakDiv y = -G^T (M_eps y): MixedVectorWeakDivergenceIntegrator is the ND mass quadrature function between the ND
// interpolation and the H1 gradient with the coefficient negated (fem/integ/mixedvecgrad.cpp:148-208), and the gradient of an H1
// function is exactly G applied to its dofs, so the partially assembled weak divergence equals -G^T M_eps to round-off.
static void divfree_rhs(b2p_divfree *d, const double *y, double *rhs)
{
  if (d->t_nd.n != d->n_nd) d->t_nd.resize(d->ctx, d->n_nd);
  d->Mnd->Mult(y, d->t_nd.p);
  d->Grad->MultTranspose(d->t_nd.p, rhs);
  vec::scale(d->ctx, rhs, d->n_h1, -1.0);
  if (d->n_ess > 0) vec::set_sub(d->ctx, rhs, d->d_ess, d->n_ess, 0.0);  // divfree.cpp:168-171
}

int b2p_divfree_mult(b2p_divfree *d, double *y)
{
  if (!d || !y) return B2P_ERR_ARG;
  b2p_ctx *ctx = d->ctx;
  if (d->rhs.n < d->n_h1) d->rhs.resize(ctx, 2 * d->n_h1);
  if (d->psi.n < d->n_h1) d->psi.resize(ctx, 2 * d->n_h1);
  B2P_TRY(ctx, divfree_rhs(d, y, d->rhs.p));
  int rc = b2p_ksp_mult(d->ksp, d->rhs.p, d->psi.p);
  if (rc) return rc;
  B2P_TRY(ctx, d->Grad->AddMult(d->psi.p, y, 1.0));  // divfree.cpp:174-183
  d->mult++;
  d->last_it = d->ksp->ksp->final_it;
  d->mult_it += d->last_it;
  d->last_converged = d->ksp->ksp->converged;
  return B2P_SUCCESS;
}

int b2p_divfree_mult_complex(b2p_divfree *d, double *yr, double *yi)
{
  if (!d || !yr || !yi) return B2P_ERR_ARG;
  b2p_ctx *ctx = d->ctx;
  const int64_t n = d->n_h1;
  if (d->rhs.n < 2 * n) d->rhs.resize(ctx, 2 * n);
  if (d->psi.n < 2 * n) d->psi.resize(ctx, 2 * n);
  if (!d->ksp2)
  {
    d->A2 = std::make_unique<TwoPartOperator>(ctx, d->ksp->ksp->A);
    d->B2 = std::make_unique<TwoPartSolver>(ctx, d->ksp->pc.get(), n);
    d->ksp2 = std::make_unique<IterativeSolver>(ctx, KspType::CG);
    d->ksp2->rel_tol = d->ksp->ksp->rel_tol;
    d->ksp2->abs_tol = d->ksp->ksp->abs_tol;
    d->ksp2->max_it = d->ksp->ksp->max_it;
    d->ksp2->SetInitialGuess(false);
    d->ksp2->SetOperator(*d->A2);
    d->ksp2->SetPreconditioner(d->B2.get());
  }
  B2P_TRY(ctx, divfree_rhs(d, yr, d->rhs.p));
  B2P_TRY(ctx, divfree_rhs(d, yi, d->rhs.p + n));
  B2P_TRY(ctx, d->ksp2->Mult(d->rhs.p, d->psi.p));
  if (!d->ksp2->converged)
    set_error(ctx, "Linear solver did not converge, norm(Ax-b)/norm(b) = %.3e (norm(b) = %.3e)!", d->ksp2->final_res / d->ksp2->initial_res,
              d->ksp2->initial_res);
  B2P_TRY(ctx, d->Grad->AddMult(d->psi.p, yr, 1.0));
  B2P_TRY(ctx, d->Grad->AddMult(d->psi.p + n, yi, 1.0));
  d->mult++;
  d->last_it = d->ksp2->final_it;
  d->mult_it += d->last_it;
  d->last_converged = d->ksp2->converged;
  return B2P_SUCCESS;
}

int b2p_divfree_stats(b2p_divfree *d, int *num_mult, int *num_mult_its, int *last_its, int *converged)
{
  if (!d) return B2P_ERR_ARG;
  if (num_mult) *num_mult = d->mult;
  if (num_mult_its) *num_mult_its = d->mult_it;
  if (last_its) *last_its = d->last_it;
  if (converged) *converged = d->last_converged ? 1 : 0;
  return B2P_SUCCESS;
}

void b2p_divfree_destroy(b2p_divfree *d) { delete d; }

}  // extern "C"
