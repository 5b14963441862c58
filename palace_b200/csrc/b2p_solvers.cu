// Host logic of the device-resident solver loop. Every vector operation is a kernel on ctx->stream;
// the only host synchronisations are the scalar reductions that steer the recurrences.
// Class-by-class restatement of the reference (file:line in each method).
#include <cstdlib>

#include "b2p_linalg.hpp"

namespace b2p
{

int halo_forward(Halo *h, double *lx);
int halo_reverse(Halo *h, double *ly);
int halo_forward_split(Halo *h, const double *x, cudaStream_t s);
int halo_reverse_split(Halo *h, double *y, cudaStream_t s);
int halo_forward_p2p(Halo *h, const double *x, bool in_kernel_wait, cudaStream_t s);
int halo_reverse_p2p(Halo *h, double *y, cudaStream_t s);
int halo_pre_p2p(Halo *h, const double *x, double *y, long long ny, bool in_kernel_wait, cudaStream_t s);
int halo_post_p2p(Halo *h, double *y, cudaStream_t s, bool pdl);
int interp_apply(const b2p_interp *it, bool transpose, double alpha, const double *x, double *y, cudaStream_t s);

// ------------------------------------------------------------------------------------ Operator
void Operator::AddMult(const double *x, double *y, double a) const
{
  if (tmp_.n != height) tmp_.resize(ctx, height);
  Mult(x, tmp_.p);
  vec::axpy(ctx, a, tmp_.p, y, height);
}
void Operator::AddMultTranspose(const double *x, double *y, double a) const
{
  if (tmp_.n != width) tmp_.resize(ctx, width);
  MultTranspose(x, tmp_.p);
  vec::axpy(ctx, a, tmp_.p, y, width);
}
void Operator::AssembleDiagonal(double *) const { set_error(ctx, "AssembleDiagonal not implemented for this operator"); }

// ------------------------------------------------------------------------------------ ParOperator
ParOperator::ParOperator(b2p_ctx *c, int64_t tsize, int64_t lsize_, const std::vector<Term> &terms_, const int32_t *ess_tdofs,
                         int64_t n_ess_, int diag_policy_, Halo *halo_)
  : Operator(c, tsize, tsize), lsize(lsize_), terms(terms_), n_ess(n_ess_), diag_policy(diag_policy_), halo(halo_)
{
  if (n_ess > 0) upload(c, ess_tdofs, (size_t)n_ess, &d_ess);
  // Essential dofs are eliminated inside the element kernels (masked restriction): the masked
  // gather is SetSubVector(tx, dbc_tdof_list, 0.0) before P, the skipped scatter is the row
  // overwrite after P^T (rap.cpp:207-233). Ghost copies of essential dofs are masked by the
  // caller through b2p_op_set_essential with L-vector indices.
  // (multi-partition callers mask ghost copies too by calling b2p_op_set_essential with L indices first)
  for (auto &t : terms)
    if (!t.op->lidx_bc) b2p_op_set_essential(t.op, ess_tdofs, n_ess);
  // Several ND terms on one space: apply their sum as one operator (one launch, one geometry stream per Mult).
  // B2P_SUM_FUSED=0 keeps one apply per term.
  const char *env = getenv("B2P_SUM_FUSED");
  if (terms.size() >= 2 && !(env && env[0] == '0'))
  {
    std::vector<b2p_op *> ops;
    std::vector<double> cf;
    for (auto &t : terms)
    {
      ops.push_back(t.op);
      cf.push_back(t.coef);
    }
    if (b2p_op_create_sum(c, (int)ops.size(), ops.data(), cf.data(), &fused_sum) == B2P_SUCCESS)
    {
      orig_terms = terms;
      terms.assign(1, Term{fused_sum, 1.0});
    }
    else
      fused_sum = nullptr;  // not eligible (mixed element types / spaces): term-by-term as before
  }
}
ParOperator::~ParOperator()
{
  if (fused_sum) b2p_op_destroy(fused_sum);
  cudaFree(d_ess);
  for (auto &g : graphs_) cudaGraphExecDestroy(g.second);
}

void ParOperator::SetCoefficients(const double *coefs)
{
  if (fused_sum)
  {
    std::vector<b2p_op *> ops;
    for (size_t t = 0; t < orig_terms.size(); t++)
    {
      orig_terms[t].coef = coefs[t];
      ops.push_back(orig_terms[t].op);
    }
    b2p_op_sum_set_coefficients(fused_sum, (int)ops.size(), ops.data(), coefs);
  }
  else
    for (size_t t = 0; t < terms.size(); t++) terms[t].coef = coefs[t];
  for (auto &g : graphs_) cudaGraphExecDestroy(g.second);
  graphs_.clear();
}

void ParOperator::MultHaloBody(const double *x, double *y, cudaStream_t s) const
{
  // Owned dofs are read from x and accumulated into y directly; ghosts live in the halo's buffers:
  //   zero y and y_ghost; forward exchange (P); all elements; reverse exchange (P^T) + add into y.
  // With peer mailboxes (b2p_halo_p2p_*) the exchanges are NVLink stores + flags issued from small
  // kernels on this stream; otherwise NCCL grouped send/recv. (An interior/interface split that overlaps
  // the collectives with the element kernel gives nothing: the persistent element kernel fills every SM, so a
  // collective kernel launched beside it only starts when it retires.)
  Halo *h = halo;
  // B2P_HALO_TIMING=1 (diagnostic): CUDA events between the three launches, accumulated per operator and printed by the
  // destructor -- where the time of a partitioned Mult goes on this rank (the events serialise nothing: same stream).
  static const bool timing = []() { const char *e = getenv("B2P_HALO_TIMING"); return e && e[0] == '1'; }();
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  if (timing)
    for (auto &e : ev)
    {
      cudaEventCreate(&e);
    }
  if (timing) cudaEventRecord(ev[0], s);
  // B2P_HALO_FUSED=0 keeps the round-1 sequence (zero-fill, push, element kernel, push, wait+add: five launches)
  static const bool fused_halo = []() { const char *e = getenv("B2P_HALO_FUSED"); return !(e && e[0] == '0'); }();
  const bool fused = h->p2p && fused_halo;
  if (!fused)
  {
    vec::set(ctx, y, height, 0.0);
    if (h->n_ghost > 0 && !h->p2p) cudaMemsetAsync(h->d_yg, 0, sizeof(double) * h->n_ghost, s);  // (the p2p push kernel clears it)
  }
  // In-kernel wait: with elements ordered interior-first (SetInteriorElements) the ND element kernel itself
  // checks the neighbours' flags just before it reaches the first interface element, so the forward exchange
  // costs nothing on the critical path. (H1 operators use the separate wait kernel.)
  bool in_kernel = h->p2p && ne_interior > 0;
  // only the sum-factorised ND kernel polls the flags itself; H1, dense-basis (tet) and block (mixed curl) operators need the
  // separate wait kernel
  for (auto &t : terms) in_kernel = in_kernel && t.op->kind != B2P_H1_DIFFUSION && !t.op->dense && !t.op->bcoef;
  if (fused)
    halo_pre_p2p(h, x, y, height, in_kernel, s);  // forward exchange and both zero-fills: one launch
  else if (h->p2p)
    halo_forward_p2p(h, x, in_kernel, s);
  else
    halo_forward_split(h, x, s);
  // Eager launches of the fused sequence are chained by programmatic dependent launch: the element kernel starts while the
  // PRE kernel still zero-fills (it waits on the grid dependency before its first scatter or ghost read), the POST kernel
  // is scheduled as the element kernel's CTAs retire. (Not inside a stream capture.)
  if (timing) cudaEventRecord(ev[1], s);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  static const bool pdl_env = []() { const char *e = getenv("B2P_PDL"); return !(e && e[0] == '0'); }();
  bool pdl = fused && pdl_env && cap == cudaStreamCaptureStatusNone && terms.size() == 1;
  for (auto &t : terms) pdl = pdl && t.op->kind != B2P_H1_DIFFUSION && !t.op->dense && in_kernel;
  for (auto &t : terms)
  {
    ApplyRange rg;
    rg.n_owned = height;
    rg.xg = h->d_xg;
    rg.yg = h->d_yg;
    rg.pdl = pdl;
    if (in_kernel)
    {
      rg.wait_flags = h->d_flags;
      rg.wait_expect = h->d_epoch + 2 * 32;
      rg.wait_n = (int)h->nbr.size();
      rg.wait_from_elem = ne_interior;
    }
    apply_range(t.op, t.op->lidx_bc ? t.op->lidx_bc : t.op->lidx, t.coef, x, y, rg, 0, s);
  }
  if (timing) cudaEventRecord(ev[2], s);
  if (fused)
    halo_post_p2p(h, y, s, pdl);  // push, wait and add: one launch
  else if (h->p2p)
    halo_reverse_p2p(h, y, s);
  else
    halo_reverse_split(h, y, s);
  if (timing)
  {
    cudaEventRecord(ev[3], s);
    cudaEventSynchronize(ev[3]);
    for (int i = 0; i < 3; i++)
    {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      halo_ms_[i] += ms;
    }
    halo_calls_++;
    for (auto &e : ev) cudaEventDestroy(e);
    if (halo_calls_ % 100 == 0)
    {
      fprintf(stderr, "[b2p] rank %d ParOperator halo timing, last 100 Mults: pre %.2f us, element kernel(s) %.2f us, post %.2f us\n", ctx->rank,
              10.0 * halo_ms_[0], 10.0 * halo_ms_[1], 10.0 * halo_ms_[2]);
      halo_ms_[0] = halo_ms_[1] = halo_ms_[2] = 0.0;
    }
  }
}

// rap.cpp:195-234
void ParOperator::Mult(const double *x, double *y) const
{
  cudaStream_t s = ctx->stream;
  if (!halo)
  {
    // Zero-fill by a kernel that releases its dependent at once, first element kernel launched with programmatic stream
    // serialisation: its prologue and first batch overlap the zero-fill (it waits on the grid dependency just before its
    // first scatter). B2P_PDL=0 goes back to memset + plain launch (bench.py times both).
    static const bool pdl = []() { const char *e = getenv("B2P_PDL"); return !(e && e[0] == '0'); }();
    const b2p_op *o0 = terms[0].op;
    const bool pdl_ok = pdl && !o0->dense && o0->kind != B2P_H1_DIFFUSION && o0->lidx_bc != nullptr;
    if (pdl_ok)
    {
      vec::zero_release(ctx, y, height);
      ApplyRange rg;
      rg.pdl = true;
      apply_range(terms[0].op, o0->lidx_bc, terms[0].coef, x, y, rg, B2P_APPLY_MASKED, s);
      for (size_t t = 1; t < terms.size(); t++) b2p_op_apply_add_ex(terms[t].op, terms[t].coef, x, y, B2P_APPLY_MASKED, s);
    }
    else
    {
      vec::set(ctx, y, height, 0.0);
      for (auto &t : terms) b2p_op_apply_add_ex(t.op, t.coef, x, y, B2P_APPLY_MASKED, s);
    }
  }
  else
  {
    const auto key = std::make_pair(x, y);
    auto it = graphs_.find(key);
    static const bool no_graph = []() { const char *e = getenv("B2P_NO_GRAPH"); return e && e[0] == '1'; }();
    // Stream capture is not allowed on the legacy default stream (what MFEM and b2p_ctx_set_stream(ctx, nullptr) use).
    // Capture and replay on an internal BLOCKING stream instead -- it synchronises implicitly with the legacy stream in
    // both directions, so the caller's ordering is preserved. (B2P_GRAPH_STREAM=0: a legacy-stream context runs the eager
    // sequence, as in round 1.)
    // Replay on the internal blocking stream can cost more in legacy-stream synchronisation than it saves in launches
    // -- opt-in, B2P_GRAPH_STREAM=1.
    static const bool graph_stream = []() { const char *e = getenv("B2P_GRAPH_STREAM"); return e && e[0] == '1'; }();
    if (s == nullptr && graph_stream && !no_graph)
    {
      if (!ctx->graph_stream && cudaStreamCreate(&ctx->graph_stream) != cudaSuccess) ctx->graph_stream = nullptr;
      if (ctx->graph_stream) s = ctx->graph_stream;
    }
    struct StreamSwap  // the body's vector kernels launch on ctx->stream: point it at the capture stream meanwhile
    {
      b2p_ctx *c;
      cudaStream_t keep;
      StreamSwap(b2p_ctx *c_, cudaStream_t s_) : c(c_), keep(c_->stream) { c->stream = s_; }
      ~StreamSwap() { c->stream = keep; }
    } swap(ctx, s);
    if (no_graph || capture_failed_)
    {
      MultHaloBody(x, y, s);
    }
    else if (!warmed_)
    {
      // first call runs eagerly: one-time kernel attribute setup must not happen inside a capture
      warmed_ = true;
      MultHaloBody(x, y, s);
    }
    else if (it == graphs_.end())
    {
      if (graphs_.size() >= 64)
      {
        for (auto &g : graphs_) cudaGraphExecDestroy(g.second);
        graphs_.clear();
      }
      cudaGraph_t graph = nullptr;
      cudaGraphExec_t exec = nullptr;
      if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess)
      {
        MultHaloBody(x, y, s);
        if (cudaStreamEndCapture(s, &graph) == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess)
          it = graphs_.emplace(key, exec).first;
        if (graph) cudaGraphDestroy(graph);
      }
      if (it == graphs_.end())
      {
        cudaGetLastError();
        set_error(ctx, "ParOperator::Mult: CUDA graph capture of the partitioned apply failed (legacy default stream? set B2P_GRAPH_STREAM=1)");
        capture_failed_ = true;  // do not try again on every call
        MultHaloBody(x, y, s);
      }
    }
    if (it != graphs_.end()) cudaGraphLaunch(it->second, s);
  }
  if (n_ess > 0)
  {
    if (diag_policy == 1)
      vec::set_sub_from(ctx, y, d_ess, n_ess, x);  // DIAG_ONE: y[ess] = x[ess]
    else
      vec::set_sub(ctx, y, d_ess, n_ess, 0.0);      // DIAG_ZERO
  }
}

// rap.cpp:236-275
void ParOperator::MultTranspose(const double *x, double *y) const
{
  bool nonsym = false;
  for (auto &t : terms) nonsym = nonsym || op_nonsymmetric(t.op);
  if (!nonsym)
  {
    Mult(x, y);
    return;
  }
  cudaStream_t s = ctx->stream;
  vec::set(ctx, y, height, 0.0);
  if (halo)
  {
    set_error(ctx, "ParOperator::MultTranspose: non-symmetric terms on a partitioned space are not supported");
    return;
  }
  for (auto &t : terms) b2p_op_apply_add_ex(t.op, t.coef, x, y, B2P_APPLY_MASKED | B2P_APPLY_TRANSPOSE, s);
  if (n_ess > 0)
  {
    if (diag_policy == 1)
      vec::set_sub_from(ctx, y, d_ess, n_ess, x);
    else
      vec::set_sub(ctx, y, d_ess, n_ess, 0.0);
  }
}

// rap.cpp:277-318 (y += a * (P^T A P x with the essential rows replaced))
void ParOperator::AddMult(const double *x, double *y, double a) const
{
  cudaStream_t s = ctx->stream;
  if (!halo)
  {
    // masked scatter never touches essential rows, so their contribution is added separately
    for (auto &t : terms) b2p_op_apply_add_ex(t.op, a * t.coef, x, y, B2P_APPLY_MASKED, s);
    if (n_ess > 0 && diag_policy == 1) vec::axpy_sub(ctx, a, x, d_ess, n_ess, y);  // y[ess] += a x[ess]
  }
  else
  {
    Operator::AddMult(x, y, a);
  }
}

// rap.cpp:154-193: diag = |P|^T diag_L, essential rows per the diagonal policy
b2p_csr *ParOperator::FullAssemble() const
{
  if (halo && halo->n_ghost > 0)
  {
    set_error(ctx, "ParOperator::FullAssemble: partitioned spaces are not assembled (the coarse matrix lives on one device)");
    return nullptr;
  }
  b2p_csr *A = nullptr;
  if (b2p_csr_create(ctx, terms[0].op, &A) != B2P_SUCCESS) return nullptr;
  if (AssembleValues(A, csr_values(A)) != B2P_SUCCESS)
  {
    b2p_csr_destroy(A);
    return nullptr;
  }
  return A;
}
int ParOperator::AssembleValues(b2p_csr *A, double *val) const
{
  if (halo && halo->n_ghost > 0)
  {
    set_error(ctx, "ParOperator::FullAssemble: partitioned spaces are not assembled (the coarse matrix lives on one device)");
    return B2P_ERR_UNSUPPORTED;
  }
  std::vector<b2p_op *> ops;
  std::vector<double> cf;
  for (auto &t : terms)
  {
    ops.push_back(t.op);
    cf.push_back(t.coef);
  }
  std::vector<int32_t> ess((size_t)n_ess);
  if (n_ess > 0)
  {
    cudaMemcpyAsync(ess.data(), d_ess, sizeof(int32_t) * n_ess, cudaMemcpyDeviceToHost, ctx->stream);
    cudaStreamSynchronize(ctx->stream);
  }
  int rc = csr_assemble_values(A, (int)ops.size(), ops.data(), cf.data(), val, ctx->stream);
  if (!rc) rc = csr_eliminate_values(A, ess.data(), n_ess, diag_policy, val, ctx->stream);
  return rc;
}
void ParOperator::AssembleDiagonal(double *d) const
{
  cudaStream_t s = ctx->stream;
  double *dl = d;
  if (halo)
  {
    if (ly_.n != lsize) ly_.resize(ctx, lsize);
    dl = ly_.p;
  }
  vec::set(ctx, dl, halo ? lsize : height, 0.0);
  for (auto &t : terms)
  {
    if (t.coef == 1.0)
      b2p_op_diag_add(t.op, dl, s);
    else
    {
      if (tmp_.n != lsize) tmp_.resize(ctx, lsize);
      vec::set(ctx, tmp_.p, lsize, 0.0);
      b2p_op_diag_add(t.op, tmp_.p, s);
      vec::axpy(ctx, t.coef, tmp_.p, dl, lsize);
    }
  }
  if (halo)
  {
    halo_reverse(halo, dl);
    vec::copy(ctx, d, dl, height);
  }
  if (n_ess > 0) vec::set_sub(ctx, d, d_ess, n_ess, diag_policy == 1 ? 1.0 : 0.0);
}

// ------------------------------------------------------------------------------------ Solver base
void Solver::Mult2(const double *x, double *y, double *) const { Mult(x, y); }

// linalg/operator.cpp:583-631 for DinvA (chebyshev.cpp:14-28): power iteration on u <- D^-1 A u,
// lambda = ||u|| after the step, relative change < tol. (The reference wraps the real operator in
// a complex one and starts from a complex random vector; the limit is the same lambda_max.)
double SpectralNormDinvA(b2p_ctx *c, const Operator &A, const double *dinv, double tol, int max_it, uint64_t seed)
{
  const int64_t n = A.Height();
  DVec u(c, n), v(c, n);
  vec::set_random(c, u.p, n, seed);
  double nrm = vec::norml2(c, u.p, n);
  vec::scale(c, u.p, n, 1.0 / nrm);
  double l = 0.0, l0 = 0.0;
  for (int it = 0; it < max_it; it++)
  {
    A.Mult(u.p, v.p);
    vec::mult_diag(c, dinv, v.p, u.p, n);
    l = vec::norml2(c, u.p, n);
    vec::scale(c, u.p, n, 1.0 / l);
    if (it > 0 && std::abs(l - l0) / l0 < tol) break;
    l0 = l;
  }
  return l;
}

// ------------------------------------------------------------------------------------ Jacobi (jacobi.cpp:75-105)
void JacobiSmoother::SetOperator(const Operator &op)
{
  height = op.Height();
  width = op.Width();
  dinv.resize(ctx, height);
  op.AssembleDiagonal(dinv.p);
  vec::reciprocal(ctx, dinv.p, height);
  if (omega == 0.0)
  {
    const double lmax = SpectralNormDinvA(ctx, op, dinv.p);
    const double lmin = (sf_max - 1.0) * lmax;
    omega = 2.0 / (lmin + lmax);
  }
  if (omega != 1.0) vec::scale(ctx, dinv.p, height, omega);
}
void JacobiSmoother::Mult(const double *x, double *y) const { vec::mult_diag(ctx, dinv.p, x, y, height); }

// ------------------------------------------------------------------------------------ Chebyshev
// chebyshev.cpp:170-188 (4th kind) / :233-259 (1st kind)
void ChebyshevSmoother::SetOperator(const Operator &op)
{
  A = &op;
  height = op.Height();
  width = op.Width();
  d.resize(ctx, height);
  dinv.resize(ctx, height);
  op.AssembleDiagonal(dinv.p);
  vec::reciprocal(ctx, dinv.p, height);
  lambda_max = sf_max * SpectralNormDinvA(ctx, op, dinv.p);
  if (!fourth_kind)
  {
    double sfm = sf_min;
    if (sfm <= 0.0) sfm = 1.69 / (std::pow(order, 1.68) + 2.11 * order + 1.98);  // chebyshev.cpp:243-247
    const double lambda_min = sfm * lambda_max;
    theta = 0.5 * (lambda_max + lambda_min);
    delta = 0.5 * (lambda_max - lambda_min);
  }
}

namespace
{
// r = x - A y. With a native AddMult this is a copy and one accumulating apply (no zero fill of r, no separate subtraction
// pass); otherwise Mult followed by r = x - r.
inline void Residual(b2p_ctx *ctx, const Operator &A, const double *x, const double *y, double *r, int64_t n)
{
  if (A.NativeAddMult())
  {
    vec::copy(ctx, r, x, n);
    A.AddMult(y, r, -1.0);
  }
  else
  {
    A.Mult(y, r);
    vec::axpby(ctx, 1.0, x, -1.0, r, n);
  }
}
}  // namespace

// chebyshev.cpp:191-220 and :261-293: y = y + p(D^-1 A) D^-1 (x - A y)
void ChebyshevSmoother::Mult2(const double *x, double *y, double *r) const
{
  // chebyshev.cpp:190-220 (4th kind) / :260-293 (1st kind). Same recurrences; the vector work is arranged so that every
  // step is ONE operator apply and ONE pass over the vectors: r = x - A y accumulates into a copy of x (no zero fill, no
  // separate subtraction), and y += d is folded into the kernel that produces d.
  const int64_t n = height;
  for (int it = 0; it < pc_it; it++)
  {
    const bool fresh = !(initial_guess || it > 0);  // y == 0: r = x, and the first update assigns y
    if (fresh)
      vec::copy(ctx, r, x, n);
    else
      Residual(ctx, *A, x, y, r, n);
    if (fourth_kind)
    {
      vec::cheb_first_y(ctx, 4.0 / (3.0 * lambda_max), dinv.p, r, d.p, y, fresh, n);
      for (int k = 1; k < order; k++)
      {
        A->AddMult(d.p, r, -1.0);
        const double sd = (2.0 * k - 1.0) / (2.0 * k + 3.0);
        const double sr = (8.0 * k + 4.0) / ((2.0 * k + 3.0) * lambda_max);
        vec::cheb_next_y(ctx, sd, sr, dinv.p, r, d.p, y, n);
      }
    }
    else
    {
      vec::cheb_first_y(ctx, 1.0 / theta, dinv.p, r, d.p, y, fresh, n);
      double rhop = delta / theta;
      for (int k = 1; k < order; k++)
      {
        A->AddMult(d.p, r, -1.0);
        const double rho = 1.0 / (2.0 * theta / delta - rhop);
        const double sd = rho * rhop;
        const double sr = 2.0 * rho / delta;
        vec::cheb_next_y(ctx, sd, sr, dinv.p, r, d.p, y, n);
        rhop = rho;
      }
    }
  }
}

// ------------------------------------------------------------------------------------ DistRelaxation
// distrelaxation.cpp:16-37
DistRelaxationSmoother::DistRelaxationSmoother(b2p_ctx *c, const Operator &G_, int smooth_it, int cheby_smooth_it, int cheby_order,
                                               double sf_max, double sf_min, bool fourth_kind)
  : Solver(c), pc_it(smooth_it), G(&G_)
{
  B = std::make_unique<ChebyshevSmoother>(c, cheby_smooth_it, cheby_order, sf_max, sf_min, fourth_kind);
  B_G = std::make_unique<ChebyshevSmoother>(c, cheby_smooth_it, cheby_order, sf_max, sf_min, fourth_kind);
  B_G->SetInitialGuess(false);
}
void DistRelaxationSmoother::SetOperator(const Operator &) { set_error(ctx, "DistRelaxationSmoother needs SetOperators(A, A_G)"); }
// distrelaxation.cpp:39-69
void DistRelaxationSmoother::SetOperators(const Operator &op, const Operator &op_G)
{
  A = &op;
  A_G = &op_G;
  height = op.Height();
  width = op.Width();
  x_G.resize(ctx, op_G.Height());
  y_G.resize(ctx, op_G.Height());
  r_G.resize(ctx, op_G.Height());
  B->SetOperator(op);
  B_G->SetOperator(op_G);
}
void DistRelaxationSmoother::Mult(const double *x, double *y) const
{
  if (r_.n != height) r_.resize(ctx, height);
  Mult2(x, y, r_.p);
}
// distrelaxation.cpp:99-119
void DistRelaxationSmoother::Mult2(const double *x, double *y, double *r) const
{
  for (int it = 0; it < pc_it; it++)
  {
    B->SetInitialGuess(initial_guess || it > 0);
    B->Mult2(x, y, r);
    Residual(ctx, *A, x, y, r, height);
    G->MultTranspose(r, x_G.p);
    if (A_G->NumEssential() > 0) vec::set_sub(ctx, x_G.p, A_G->EssentialTrueDofs(), A_G->NumEssential(), 0.0);
    B_G->Mult2(x_G.p, y_G.p, r_G.p);
    G->AddMult(y_G.p, y, 1.0);
  }
}
// distrelaxation.cpp:121-151
void DistRelaxationSmoother::MultTranspose2(const double *x, double *y, double *r) const
{
  B->SetInitialGuess(true);
  for (int it = 0; it < pc_it; it++)
  {
    if (initial_guess || it > 0)
    {
      Residual(ctx, *A, x, y, r, height);
      G->MultTranspose(r, x_G.p);
    }
    else
    {
      vec::set(ctx, y, height, 0.0);
      G->MultTranspose(x, x_G.p);
    }
    if (A_G->NumEssential() > 0) vec::set_sub(ctx, x_G.p, A_G->EssentialTrueDofs(), A_G->NumEssential(), 0.0);
    B_G->MultTranspose2(x_G.p, y_G.p, r_G.p);
    G->AddMult(y_G.p, y, 1.0);
    B->MultTranspose2(x, y, r);
  }
}

// ------------------------------------------------------------------------------------ GMG (gmg.cpp)
GeometricMultigridSolver::GeometricMultigridSolver(b2p_ctx *c, std::unique_ptr<Solver> &&coarse,
                                                   const std::vector<const Operator *> &P_,
                                                   const std::vector<const Operator *> &G, int cycle_it, int smooth_it,
                                                   int cheby_order, double sf_max, double sf_min, bool fourth_kind)
  : Solver(c), pc_it(cycle_it), P(P_), A(P_.size() + 1), B(P_.size() + 1), X(P_.size() + 1), Y(P_.size() + 1), R(P_.size() + 1)
{
  const size_t n_levels = P.size() + 1;
  B[0] = std::move(coarse);
  for (size_t l = 1; l < n_levels; l++)
  {
    if (!G.empty())
      B[l] = std::make_unique<DistRelaxationSmoother>(c, *G[l], smooth_it, 1, cheby_order, sf_max, sf_min, fourth_kind);  // gmg.cpp:45-50
    else
      B[l] = std::make_unique<ChebyshevSmoother>(c, smooth_it, cheby_order, sf_max, sf_min, fourth_kind);  // gmg.cpp:52-63
  }
}
void GeometricMultigridSolver::SetOperator(const Operator &) { set_error(ctx, "GeometricMultigridSolver needs SetOperators"); }
// gmg.cpp:66-123
void GeometricMultigridSolver::SetOperators(const std::vector<const Operator *> &A_, const std::vector<const Operator *> &A_aux)
{
  const size_t n_levels = A.size();
  for (size_t l = 0; l < n_levels; l++)
  {
    A[l] = A_[l];
    auto *dist = dynamic_cast<DistRelaxationSmoother *>(B[l].get());
    if (dist)
      dist->SetOperators(*A_[l], *A_aux[l]);
    else
      B[l]->SetOperator(*A_[l]);
    X[l].resize(ctx, A[l]->Height());
    Y[l].resize(ctx, A[l]->Height());
    R[l].resize(ctx, A[l]->Height());
  }
  height = A.back()->Height();
  width = A.back()->Width();
}
// gmg.cpp:126-142
void GeometricMultigridSolver::Mult(const double *x, double *y) const
{
  const int n_levels = (int)A.size();
  x_top = x;
  y_top = y;
  for (int it = 0; it < pc_it; it++) VCycle(n_levels - 1, it > 0);
}
// gmg.cpp:172-205
void GeometricMultigridSolver::VCycle(int l, bool initial_guess_) const
{
  B[l]->SetInitialGuess(initial_guess_);
  if (l == 0)
  {
    B[l]->Mult(Xp(l), Yp(l));
    return;
  }
  B[l]->Mult2(Xp(l), Yp(l), R[l].p);
  Residual(ctx, *A[l], Xp(l), Yp(l), R[l].p, A[l]->Height());
  P[l - 1]->MultTranspose(R[l].p, X[l - 1].p);
  if (A[l - 1]->NumEssential() > 0) vec::set_sub(ctx, X[l - 1].p, A[l - 1]->EssentialTrueDofs(), A[l - 1]->NumEssential(), 0.0);
  VCycle(l - 1, false);
  P[l - 1]->AddMult(Y[l - 1].p, Yp(l), 1.0);  // y += P y_c in one pass (no temporary, no zero fill)
  B[l]->SetInitialGuess(true);
  B[l]->MultTranspose2(Xp(l), Yp(l), R[l].p);
}

// ------------------------------------------------------------------------------------ Krylov (iterative.cpp)
namespace
{
// iterative.cpp:73-110 (real GeneratePlaneRotation) and :228-235 (ApplyPlaneRotation)
inline void GeneratePlaneRotation(const double dx, const double dy, double &cs, double &sn)
{
  if (dy == 0.0)
  {
    cs = 1.0;
    sn = 0.0;
    return;
  }
  if (dx == 0.0)
  {
    cs = 0.0;
    sn = std::copysign(1.0, dy);
    return;
  }
  const double safmin = std::numeric_limits<double>::min(), safmax = 1.0 / safmin;
  const double root_min = std::sqrt(safmin), root_max = std::sqrt(safmax / 2);
  const double dx1 = std::abs(dx), dy1 = std::abs(dy);
  if (dx1 > root_min && dx1 < root_max && dy1 > root_min && dy1 < root_max)
  {
    const double d = std::sqrt(dx * dx + dy * dy);
    cs = dx1 / d;
    sn = dy / std::copysign(d, dx);
  }
  else
  {
    const double u = std::min(safmax, std::max(safmin, std::max(dx1, dy1)));
    const double dxs = dx / u, dys = dy / u;
    const double d = std::sqrt(dxs * dxs + dys * dys);
    cs = std::abs(dxs) / d;
    sn = dys / std::copysign(d, dx);
  }
}
inline void ApplyPlaneRotation(double &dx, double &dy, const double cs, const double sn)
{
  const double t = cs * dx + sn * dy;
  dy = -sn * dx + cs * dy;
  dx = t;
}
}  // namespace

void IterativeSolver::Mult(const double *b, double *x) const
{
  if (type == KspType::CG)
    (check_every > 1 ? MultCGDeviceScalars(b, x) : MultCG(b, x));
  else
    MultGMRES(b, x, type == KspType::FGMRES);
}

// iterative.cpp:361-486
void IterativeSolver::MultCG(const double *b, double *x) const
{
  const int64_t n = height;
  r.resize(ctx, n);
  z.resize(ctx, n);
  p.resize(ctx, n);
  res_history.clear();
  double beta, beta_prev = 0.0, alpha, denom, res, eps;
  if (initial_guess)
  {
    A->Mult(x, r.p);
    vec::axpby(ctx, 1.0, b, -1.0, r.p, n);
  }
  else
  {
    vec::copy(ctx, r.p, b, n);
    vec::set(ctx, x, n, 0.0);
  }
  if (B)
    B->Mult(r.p, z.p);
  else
    vec::copy(ctx, z.p, r.p, n);
  beta = vec::dot(ctx, z.p, r.p, n);
  res = std::sqrt(std::abs(beta));
  if (initial_guess)
  {
    double beta_rhs;
    if (B)
    {
      B->Mult(b, p.p);
      beta_rhs = vec::dot(ctx, p.p, b, n);
    }
    else
      beta_rhs = vec::norml2(ctx, b, n);  // (sic) iterative.cpp:408
    initial_res = std::sqrt(std::abs(beta_rhs));
  }
  else
    initial_res = res;
  eps = std::max(rel_tol * initial_res, abs_tol);
  converged = (res < eps) || res == 0.0;  // a zero residual (zero right-hand side: the imaginary part under PCMatReal) is converged, not 0 / 0
  int it = 0;
  for (; it < max_it && !converged; it++)
  {
    res_history.push_back(res);
    if (!it)
      vec::copy(ctx, p.p, z.p, n);
    else
      vec::axpby(ctx, 1.0, z.p, beta / beta_prev, p.p, n);
    A->Mult(p.p, z.p);
    denom = vec::dot(ctx, z.p, p.p, n);
    alpha = beta / denom;
    vec::axpy(ctx, alpha, p.p, x, n);
    vec::axpy(ctx, -alpha, z.p, r.p, n);
    beta_prev = beta;
    if (B)
      B->Mult(r.p, z.p);
    else
      vec::copy(ctx, z.p, r.p, n);
    beta = vec::dot(ctx, z.p, r.p, n);
    res = std::sqrt(std::abs(beta));
    converged = (res < eps);
  }
  res_history.push_back(res);
  final_res = res;
  final_it = it;
}

// The same preconditioned CG recurrence with alpha, beta formed on the device: per iteration no host synchronisation;
// the residual norm sqrt(|z.r|) is read back every check_every iterations.
void IterativeSolver::MultCGDeviceScalars(const double *b, double *x) const
{
  const int64_t n = height;
  r.resize(ctx, n);
  z.resize(ctx, n);
  p.resize(ctx, n);
  if (scal.n != 4) scal.resize(ctx, 4);
  double *d_beta = scal.p, *d_beta_prev = scal.p + 1, *d_denom = scal.p + 2;
  res_history.clear();
  auto read = [&](const double *d) -> double
  {
    double h = 0.0;
    cudaMemcpyAsync(&h, d, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
    cudaStreamSynchronize(ctx->stream);
    return h;
  };
  if (initial_guess)
  {
    A->Mult(x, r.p);
    vec::axpby(ctx, 1.0, b, -1.0, r.p, n);
  }
  else
  {
    vec::copy(ctx, r.p, b, n);
    vec::set(ctx, x, n, 0.0);
  }
  if (B)
    B->Mult(r.p, z.p);
  else
    vec::copy(ctx, z.p, r.p, n);
  vec::dot_dev(ctx, z.p, r.p, n, d_beta);
  double res = std::sqrt(std::abs(read(d_beta)));
  if (initial_guess)
  {
    double beta_rhs;
    if (B)
    {
      B->Mult(b, p.p);
      beta_rhs = vec::dot(ctx, p.p, b, n);
    }
    else
      beta_rhs = vec::norml2(ctx, b, n);
    initial_res = std::sqrt(std::abs(beta_rhs));
  }
  else
    initial_res = res;
  const double eps = std::max(rel_tol * initial_res, abs_tol);
  converged = (res < eps) || res == 0.0;  // a zero residual (zero right-hand side: the imaginary part under PCMatReal) is converged, not 0 / 0
  int it = 0;
  for (; it < max_it && !converged; it++)
  {
    if (!it)
      vec::copy(ctx, p.p, z.p, n);
    else
      vec::xpay_ratio_dev(ctx, z.p, d_beta, d_beta_prev, p.p, n);  // p = z + (beta / beta_prev) p
    A->Mult(p.p, z.p);
    vec::dot_dev(ctx, z.p, p.p, n, d_denom);
    vec::cg_update_dev(ctx, d_beta, d_denom, p.p, z.p, x, r.p, n);  // x += alpha p, r -= alpha A p
    std::swap(d_beta, d_beta_prev);
    if (B)
      B->Mult(r.p, z.p);
    else
      vec::copy(ctx, z.p, r.p, n);
    vec::dot_dev(ctx, z.p, r.p, n, d_beta);
    if ((it + 1) % check_every == 0 || it + 1 == max_it)
    {
      res = std::sqrt(std::abs(read(d_beta)));
      res_history.push_back(res);
      converged = (res < eps);
    }
  }
  final_res = res;
  final_it = it;
}

// iterative.cpp:544-705 (GMRES) and :734-871 (FGMRES)
void IterativeSolver::MultGMRES(const double *b, double *x, bool flexible) const
{
  const int64_t n = height;
  const int mdim = (max_dim < 0) ? max_it : max_dim;
  r.resize(ctx, n);
  auto ensure = [&](std::vector<std::unique_ptr<DVec>> &W, int k)
  {
    if ((int)W.size() <= k) W.resize(k + 1);
    if (!W[k]) W[k] = std::make_unique<DVec>(ctx, n);
    if (W[k]->n != n) W[k]->resize(ctx, n);
    return W[k]->p;
  };
  H.assign((size_t)(mdim + 1) * mdim, 0.0);
  s.assign(mdim + 1, 0.0);
  cs.assign(mdim + 1, 0.0);
  sn.assign(mdim + 1, 0.0);
  res_history.clear();
  const bool right = flexible || pc_side == PcSide::RIGHT;
  double beta = 0.0, true_beta, eps = 0.0;
  converged = false;
  int it = 0, restart = 0;
  for (; it < max_it; restart++)
  {
    double *V0 = ensure(V, 0);
    double *res_vec = flexible ? ensure(Z, 0) : r.p;  // FGMRES keeps the residual in Z[0] (iterative.cpp:757)
    // InitialResidual (iterative.cpp:253-286)
    const bool ig = initial_guess || restart > 0;
    if (B && !right)
    {
      if (ig)
      {
        A->Mult(x, V0);
        vec::axpby(ctx, 1.0, b, -1.0, V0, n);
        B->Mult(V0, res_vec);
      }
      else
      {
        B->Mult(b, res_vec);
        vec::set(ctx, x, n, 0.0);
      }
    }
    else
    {
      if (ig)
      {
        A->Mult(x, res_vec);
        vec::axpby(ctx, 1.0, b, -1.0, res_vec, n);
      }
      else
      {
        vec::copy(ctx, res_vec, b, n);
        vec::set(ctx, x, n, 0.0);
      }
    }
    true_beta = vec::norml2(ctx, res_vec, n);
    if (it == 0)
    {
      if (initial_guess)
      {
        if (B && !right)
        {
          B->Mult(b, V0);
          initial_res = vec::norml2(ctx, V0, n);
        }
        else
          initial_res = vec::norml2(ctx, b, n);
      }
      else
        initial_res = true_beta;
      eps = std::max(rel_tol * initial_res, abs_tol);
    }
    beta = true_beta;
    if (beta < eps || beta == 0.0)  // (a zero residual is converged: 1 / beta below)
    {
      converged = true;
      break;
    }
    vec::axpby(ctx, 1.0 / beta, res_vec, 0.0, V0, n);
    std::fill(s.begin(), s.end(), 0.0);
    s[0] = beta;
    int j = 0;
    for (;; j++, it++)
    {
      res_history.push_back(beta);
      double *Vj = ensure(V, j), *w = ensure(V, j + 1);
      // ApplyBA (iterative.cpp:288-305)
      if (B && !right)
      {
        A->Mult(Vj, r.p);
        B->Mult(r.p, w);
      }
      else if (B)
      {
        double *zj = flexible ? ensure(Z, j) : r.p;
        B->Mult(Vj, zj);
        A->Mult(zj, w);
      }
      else
        A->Mult(Vj, w);
      double *Hj = H.data() + (size_t)j * (mdim + 1);
      std::vector<const double *> Vp(j + 1);
      for (int k = 0; k <= j; k++) Vp[k] = V[k]->p;
      // orthog.hpp:41-89
      if (gs == Orthog::MGS)
      {
        for (int k = 0; k <= j; k++)
        {
          Hj[k] = vec::dot(ctx, w, Vp[k], n);
          vec::axpy(ctx, -Hj[k], Vp[k], w, n);
        }
      }
      else
      {
        vec::multi_dot(ctx, j + 1, Vp.data(), w, n, Hj);
        vec::multi_axpy(ctx, j + 1, Hj, Vp.data(), w, n, -1.0);
        if (gs == Orthog::CGS2)
        {
          std::vector<double> dH(j + 1);
          vec::multi_dot(ctx, j + 1, Vp.data(), w, n, dH.data());
          vec::multi_axpy(ctx, j + 1, dH.data(), Vp.data(), w, n, -1.0);
          for (int k = 0; k <= j; k++) Hj[k] += dH[k];
        }
      }
      Hj[j + 1] = vec::norml2(ctx, w, n);
      vec::scale(ctx, w, n, 1.0 / Hj[j + 1]);
      for (int k = 0; k < j; k++) ApplyPlaneRotation(Hj[k], Hj[k + 1], cs[k], sn[k]);
      GeneratePlaneRotation(Hj[j], Hj[j + 1], cs[j], sn[j]);
      ApplyPlaneRotation(Hj[j], Hj[j + 1], cs[j], sn[j]);
      ApplyPlaneRotation(s[j], s[j + 1], cs[j], sn[j]);
      beta = std::abs(s[j + 1]);
      converged = (beta < eps);
      if (converged || j + 1 == mdim || it + 1 == max_it)
      {
        it++;
        break;
      }
    }
    // back substitution (iterative.cpp:652-662)
    for (int i = j; i >= 0; i--)
    {
      double *Hi = H.data() + (size_t)i * (mdim + 1);
      s[i] /= Hi[i];
      for (int k = i - 1; k >= 0; k--) s[k] -= Hi[k] * s[i];
    }
    if (flexible)
    {
      std::vector<const double *> Zp(j + 1);
      for (int k = 0; k <= j; k++) Zp[k] = Z[k]->p;
      vec::multi_axpy(ctx, j + 1, s.data(), Zp.data(), x, n, 1.0);
    }
    else
    {
      std::vector<const double *> Vp(j + 1);
      for (int k = 0; k <= j; k++) Vp[k] = V[k]->p;
      if (!B || !right)
        vec::multi_axpy(ctx, j + 1, s.data(), Vp.data(), x, n, 1.0);
      else
      {
        vec::set(ctx, r.p, n, 0.0);
        vec::multi_axpy(ctx, j + 1, s.data(), Vp.data(), r.p, n, 1.0);
        B->Mult(r.p, V[0]->p);
        vec::axpy(ctx, 1.0, V[0]->p, x, n);
      }
    }
    if (converged) break;
  }
  res_history.push_back(beta);
  final_res = beta;
  final_it = it;
}

// ------------------------------------------------------------------------------------ InterpOperator
InterpOperator::InterpOperator(b2p_ctx *c, b2p_interp *impl_, Halo *in_halo_, int64_t in_tsize, Halo *out_halo_, int64_t out_tsize)
  : Operator(c, out_halo_ ? out_tsize : impl_->out_lsize, in_halo_ ? in_tsize : impl_->in_lsize), impl(impl_), in_halo(in_halo_),
    out_halo(out_halo_)
{
}
// y_T = R (1/mult) I P x_T   (ParOperator with use_R: no summation over ranks, libceed/operator.cpp:182-190)
void InterpOperator::AddMult(const double *x, double *y, double a) const
{
  const double *lx = x;
  if (in_halo)
  {
    if (lin_.n != impl->in_lsize) lin_.resize(ctx, impl->in_lsize);
    vec::copy(ctx, lin_.p, x, width);
    halo_forward(in_halo, lin_.p);
    lx = lin_.p;
  }
  if (!out_halo)
    interp_apply(impl, false, a, lx, y, ctx->stream);
  else
  {
    if (lout_.n != impl->out_lsize) lout_.resize(ctx, impl->out_lsize);
    vec::set(ctx, lout_.p, impl->out_lsize, 0.0);
    interp_apply(impl, false, a, lx, lout_.p, ctx->stream);
    vec::axpy(ctx, 1.0, lout_.p, y, height);
  }
}
void InterpOperator::Mult(const double *x, double *y) const
{
  vec::set(ctx, y, height, 0.0);
  AddMult(x, y, 1.0);
}
// y_T = P^T I^T (1/mult) R^T x_T  (libceed/operator.cpp:214-240 with RestrictionMatrixMultTranspose)
void InterpOperator::MultTranspose(const double *x, double *y) const
{
  const double *lx = x;
  if (out_halo)
  {
    if (lout_.n != impl->out_lsize) lout_.resize(ctx, impl->out_lsize);
    vec::set(ctx, lout_.p, impl->out_lsize, 0.0);
    vec::copy(ctx, lout_.p, x, height);
    lx = lout_.p;
  }
  if (!in_halo)
  {
    vec::set(ctx, y, width, 0.0);
    interp_apply(impl, true, 1.0, lx, y, ctx->stream);
  }
  else
  {
    if (lin_.n != impl->in_lsize) lin_.resize(ctx, impl->in_lsize);
    vec::set(ctx, lin_.p, impl->in_lsize, 0.0);
    interp_apply(impl, true, 1.0, lx, lin_.p, ctx->stream);
    halo_reverse(in_halo, lin_.p);
    vec::copy(ctx, y, lin_.p, width);
  }
}

}  // namespace b2p
