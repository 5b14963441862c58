// Device-resident linear algebra and solver layer (C++ host logic over sm_90a kernels), mirroring
// the reference's class structure so that the C ABI (and a Palace adapter) maps one to one:
//   palace::Operator / ParOperator / SumOperator        /root/reference/palace/linalg/{operator.hpp,rap.hpp}
//   palace::Solver<OperType>                            /root/reference/palace/linalg/solver.hpp:21-65
//   JacobiSmoother, ChebyshevSmoother(1stKind)          /root/reference/palace/linalg/{jacobi,chebyshev}.cpp
//   DistRelaxationSmoother, GeometricMultigridSolver    /root/reference/palace/linalg/{distrelaxation,gmg}.cpp
//   CgSolver, GmresSolver, FgmresSolver                 /root/reference/palace/linalg/iterative.cpp
// Real-valued (OperType = Operator) instantiation; all vectors are raw device pointers (T-vectors).
#pragma once
#include <cmath>
#include <map>
#include <memory>
#include <vector>

#include "b2p_internal.hpp"

namespace b2p
{

// ---------------------------------------------------------------- vectors / BLAS-1 (b2p_vec.cu)
struct DVec  // owning device vector
{
  b2p_ctx *ctx = nullptr;
  double *p = nullptr;
  int64_t n = 0;
  DVec() = default;
  DVec(b2p_ctx *c, int64_t n_) { resize(c, n_); }
  DVec(const DVec &) = delete;
  DVec &operator=(const DVec &) = delete;
  ~DVec() { release(); }
  void resize(b2p_ctx *c, int64_t n_);
  void release();
  operator double *() { return p; }
  operator const double *() const { return p; }
};

void b2p_allreduce_sum(b2p_ctx *c, double *dbuf, int n);  // in place, on ctx->stream (no-op for one rank)

namespace vec
{
void set(b2p_ctx *c, double *y, int64_t n, double v);
void dot_dev(b2p_ctx *c, const double *x, const double *y, int64_t n, double *d_out);  // result stays on the device
void xpay_ratio_dev(b2p_ctx *c, const double *z, const double *d_num, const double *d_den, double *p, int64_t n);
void cg_update_dev(b2p_ctx *c, const double *d_num, const double *d_den, const double *p, const double *q, double *x, double *r, int64_t n);
void zero_release(b2p_ctx *c, double *y, int64_t n);  // y = 0 by a kernel that lets a PDL-launched successor start early
void copy(b2p_ctx *c, double *y, const double *x, int64_t n);
void scale(b2p_ctx *c, double *y, int64_t n, double a);
void axpy(b2p_ctx *c, double a, const double *x, double *y, int64_t n);                       // y += a x
void axpby(b2p_ctx *c, double a, const double *x, double b, double *y, int64_t n);            // y = a x + b y
void axpbypcz(b2p_ctx *c, double a, const double *x, double b, const double *y, double g, double *z, int64_t n);
void mult_diag(b2p_ctx *c, const double *d, const double *x, double *y, int64_t n);           // y = d .* x
void reciprocal(b2p_ctx *c, double *y, int64_t n);
void set_sub(b2p_ctx *c, double *y, const int32_t *idx, int64_t nidx, double v);              // y[idx] = v
void set_sub_from(b2p_ctx *c, double *y, const int32_t *idx, int64_t nidx, const double *x);  // y[idx] = x[idx]
void axpy_sub(b2p_ctx *c, double a, const double *x, const int32_t *idx, int64_t nidx, double *y);       // y[idx] += a x[idx]
void set_random(b2p_ctx *c, double *y, int64_t n, uint64_t seed);                             // uniform [-1, 1]
// Chebyshev fused updates (chebyshev.cpp:70-156 plus the y += d the reference does separately)
void cheb_first(b2p_ctx *c, double sr, const double *dinv, const double *r, double *d, int64_t n);
void cheb_next(b2p_ctx *c, double sd, double sr, const double *dinv, const double *r, double *d, int64_t n);
void cheb_first_y(b2p_ctx *c, double sr, const double *dinv, const double *r, double *d, double *y, bool assign, int64_t n);
void cheb_next_y(b2p_ctx *c, double sd, double sr, const double *dinv, const double *r, double *d, double *y, int64_t n);
// Global reductions: local device reduction (deterministic order) + NCCL all-reduce + one host sync.
double dot(b2p_ctx *c, const double *x, const double *y, int64_t n);
double sum(b2p_ctx *c, const double *x, int64_t n);
void multi_dot(b2p_ctx *c, int m, const double *const *V, const double *w, int64_t n, double *out);  // out[j] = <w, V_j>
void multi_axpy(b2p_ctx *c, int m, const double *coef, const double *const *V, double *w, int64_t n, double sign);  // w += sign * sum coef_j V_j
inline double norml2(b2p_ctx *c, const double *x, int64_t n) { return std::sqrt(std::abs(dot(c, x, x, n))); }
}  // namespace vec

// ---------------------------------------------------------------- operators
class Operator
{
public:
  b2p_ctx *ctx;
  int64_t height, width;
  Operator(b2p_ctx *c, int64_t h, int64_t w) : ctx(c), height(h), width(w) {}
  virtual ~Operator() = default;
  virtual void Mult(const double *x, double *y) const = 0;
  virtual void MultTranspose(const double *x, double *y) const { Mult(x, y); }
  virtual void AddMult(const double *x, double *y, double a = 1.0) const;           // default: temp + axpy
  virtual void AddMultTranspose(const double *x, double *y, double a = 1.0) const;
  virtual void AssembleDiagonal(double *d) const;
  // true: AddMult accumulates straight into y (no temporary): r = x - A y is then a copy plus one AddMult
  virtual bool NativeAddMult() const { return false; }
  // essential (Dirichlet) true dofs of operators that eliminate them (ParOperator and its general-prolongation form): the
  // multigrid zeroes them in restricted residuals (gmg.cpp:190-194)
  virtual const int32_t *EssentialTrueDofs() const { return nullptr; }
  virtual int64_t NumEssential() const { return 0; }
  // Operators that are an assembled real matrix: its CSR pattern and the device values they apply (*val), else nullptr.
  // The algebraic coarse solvers (b2p_amg.cu) read the matrix through this.
  virtual b2p_csr *AssembledMatrix(const double **val) const { return nullptr; }
  int64_t Height() const { return height; }
  int64_t Width() const { return width; }

protected:
  mutable DVec tmp_;
};

// P / P^T of one finite element space on this rank (linalg/rap.cpp:212-222): owned dofs first,
// then ghosts. nranks == 1 (or no shared dofs): identity, zero copies.
struct Halo
{
  b2p_ctx *ctx = nullptr;
  int64_t n_true = 0, n_ghost = 0;
  std::vector<int> nbr;                 // neighbour ranks
  std::vector<int64_t> send_off, recv_off;  // prefix sums (size n_nbr + 1)
  int32_t *d_send_idx = nullptr;        // owned L-indices to send, concatenated per neighbour
  double *d_buf = nullptr;              // pack / unpack buffer (size send total)
  double *d_xg = nullptr, *d_yg = nullptr;  // ghost pieces of the input / output L-vectors
  // peer-memory mailboxes (optional, b2p_halo_p2p_*): see b2p_halo.cu
  bool p2p = false;
  double *d_mail = nullptr;                     // this rank's mailbox
  double *d_mail_rev = nullptr;                 // = d_mail + n_ghost
  unsigned long long *d_flags = nullptr;        // [64]: fwd flags [0,32), rev flags [32,64)
  int *d_recv_has = nullptr;                    // [32] neighbour k sends me ghosts
  unsigned int *d_done = nullptr;               // [64] block-completion counters of the push kernels
  unsigned long long *d_epoch = nullptr;        // [128]: send-fwd, send-rev, expect-fwd, expect-rev (32 each)
  long long *d_send_off = nullptr, *d_recv_off = nullptr;  // prefix sums on the device
  double **d_peer_fwd = nullptr, **d_peer_rev = nullptr;   // per neighbour: where my data lands in the peer's mailbox
  unsigned long long **d_peer_flag_fwd = nullptr, **d_peer_flag_rev = nullptr;
  std::vector<void *> peer_maps;                // cudaIpcOpenMemHandle results
  cudaStream_t comm_stream = nullptr;   // high-priority stream: the forward exchange overlaps interior elements
  cudaEvent_t ev_in = nullptr, ev_fwd = nullptr;
};

// ParOperator over the local partially assembled operators: y = P^T (sum_i c_i A_i) P x with
// essential-dof elimination (rap.cpp:195-234,277-318,154-193; BuildParSumOperator rap.cpp:764-829).
class ParOperator : public Operator
{
public:
  struct Term
  {
    b2p_op *op;
    double coef;
  };
  ParOperator(b2p_ctx *c, int64_t tsize, int64_t lsize, const std::vector<Term> &terms, const int32_t *ess_tdofs,
              int64_t n_ess, int diag_policy, Halo *halo);
  // New scalar coefficients of the terms (a0 K + a1 C + a2 M at the next frequency of a sweep, spaceoperator.cpp:945-1153)
  // without rebuilding anything; cached CUDA graphs bake the coefficients in, so they are dropped.
  void SetCoefficients(const double *coefs);
  size_t NumTerms() const { return fused_sum ? orig_terms.size() : terms.size(); }
  bool Fused() const { return fused_sum != nullptr; }
  ~ParOperator() override;
  void Mult(const double *x, double *y) const override;
  // Symmetric terms: Mult. With a non-symmetric term (B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL) the local operators are applied
  // transposed (single partition; the reference has no transpose of its BilinearForm operators at all, libceed/operator.cpp:60-99).
  void MultTranspose(const double *x, double *y) const override;
  // false: a non-symmetric term on a partitioned space (the transposed local apply is not plumbed through the halo path)
  bool TransposeAvailable() const
  {
    if (!halo) return true;
    for (auto &t : terms)
      if (op_nonsymmetric(t.op)) return false;
    return true;
  }
  void AddMult(const double *x, double *y, double a = 1.0) const override;
  bool NativeAddMult() const override { return halo == nullptr; }
  void AssembleDiagonal(double *d) const override;
  // elements [0, n) touch no ghost dof. A captured graph bakes in the wait mode that follows from it: drop the cache.
  void SetInteriorElements(int n)
  {
    if (n == ne_interior) return;
    ne_interior = n;
    for (auto &g : graphs_) cudaGraphExecDestroy(g.second);
    graphs_.clear();
    capture_failed_ = false;
  }
  // The eliminated sum as one device CSR matrix (ParOperator::ParallelAssemble, rap.cpp:84-152; coarse levels, single
  // partition); the caller owns the result (b2p_csr_destroy). Throws through set_error + nullptr on failure.
  b2p_csr *FullAssemble() const;
  // The numeric phase of FullAssemble into `val` (nnz entries on a pattern built from PatternOp()): the complex coarse solver
  // re-assembles the parts of a ComplexWrapperOperator without a new symbolic phase.
  int AssembleValues(b2p_csr *A, double *val) const;
  b2p_op *PatternOp() const { return terms[0].op; }
  const int32_t *EssentialTrueDofs() const override { return d_ess; }
  int64_t NumEssential() const override { return n_ess; }
  int64_t lsize;

private:
  std::vector<Term> terms;
  // terms as given by the caller when `terms` has been replaced by their fused sum (b2p_op_create_sum)
  std::vector<Term> orig_terms;
  b2p_op *fused_sum = nullptr;
  int32_t *d_ess = nullptr;
  int64_t n_ess = 0;
  int diag_policy;  // 0 = DIAG_ZERO, 1 = DIAG_ONE
  Halo *halo;
  int ne_interior = 0;
  mutable DVec lx_, ly_;
  // The partitioned Mult is ~a dozen stream operations (events, pack, NCCL groups, memsets, two element
  // kernels, unpack): launch-bound when issued one by one, so it is captured once per (x, y) pair into a
  // CUDA graph and replayed (solver loops reuse a handful of vector pairs).
  void MultHaloBody(const double *x, double *y, cudaStream_t s) const;
  mutable std::map<std::pair<const double *, double *>, cudaGraphExec_t> graphs_;
  mutable double halo_ms_[3] = {0.0, 0.0, 0.0};  // B2P_HALO_TIMING: accumulated event times of pre / element / post
  mutable long halo_calls_ = 0;
  mutable bool warmed_ = false;
  mutable bool capture_failed_ = false;  // stream capture is not possible on this stream: stay on the eager sequence
};

// Element-local tensor-product interpolation between two hex spaces on the same mesh: the
// p-multigrid prolongation P_l and the discrete gradient G (fem/bilinearform.cpp:203-282,
// libceed/integrator.cpp:515-548, basis.cpp:116-165) with the reference's multiplicity scaling
// (libceed/operator.cpp:182-212) and ParOperator(use_R) semantics.
struct InterpDesc;
class InterpOperator : public Operator
{
public:
  InterpOperator(b2p_ctx *c, b2p_interp *impl, Halo *in_halo, int64_t in_tsize, Halo *out_halo, int64_t out_tsize);
  void Mult(const double *x, double *y) const override;
  void MultTranspose(const double *x, double *y) const override;
  void AddMult(const double *x, double *y, double a = 1.0) const override;
  b2p_interp *impl;
  Halo *in_halo, *out_halo;

private:
  mutable DVec lin_, lout_;
};

// ---------------------------------------------------------------- solvers
class Solver : public Operator
{
public:
  bool initial_guess = false;
  Solver(b2p_ctx *c) : Operator(c, 0, 0) {}
  virtual void SetOperator(const Operator &op) = 0;
  void SetInitialGuess(bool g) { initial_guess = g; }
  // Error code of the last SetOperator, for solvers whose setup can refuse the operator they are given
  virtual int Status() const { return B2P_SUCCESS; }
  // y = y + B (x - A y) style application with a caller-supplied residual work vector
  virtual void Mult2(const double *x, double *y, double *r) const;
  virtual void MultTranspose2(const double *x, double *y, double *r) const { Mult2(x, y, r); }

protected:
  mutable DVec r_;
};

double SpectralNormDinvA(b2p_ctx *c, const Operator &A, const double *dinv, double tol = 1e-4, int max_it = 1000,
                         uint64_t seed = 0);

class JacobiSmoother : public Solver
{
public:
  JacobiSmoother(b2p_ctx *c, double omega = 1.0, double sf_max = 1.0) : Solver(c), omega(omega), sf_max(sf_max) {}
  void SetOperator(const Operator &op) override;
  void Mult(const double *x, double *y) const override;
  double omega, sf_max;
  DVec dinv;
};

class ChebyshevSmoother : public Solver
{
public:
  // fourth_kind: ChebyshevSmoother (4th kind, chebyshev.cpp:191-220) else ChebyshevSmoother1stKind (:261-293)
  ChebyshevSmoother(b2p_ctx *c, int smooth_it, int order, double sf_max, double sf_min, bool fourth_kind)
    : Solver(c), pc_it(smooth_it), order(order), sf_max(sf_max), sf_min(sf_min), fourth_kind(fourth_kind)
  {
  }
  void SetOperator(const Operator &op) override;
  void Mult(const double *x, double *y) const override { Mult2(x, y, work()); }
  void Mult2(const double *x, double *y, double *r) const override;
  int pc_it, order;
  double sf_max, sf_min;
  bool fourth_kind;
  const Operator *A = nullptr;
  double lambda_max = 0.0, theta = 0.0, delta = 0.0;
  DVec dinv;
  mutable DVec d;

private:
  double *work() const
  {
    if (r_.n != height) r_.resize(ctx, height);
    return r_.p;
  }
};

class DistRelaxationSmoother : public Solver
{
public:
  DistRelaxationSmoother(b2p_ctx *c, const Operator &G, int smooth_it, int cheby_smooth_it, int cheby_order, double sf_max,
                         double sf_min, bool fourth_kind);
  void SetOperator(const Operator &) override;  // not used: needs both operators
  void SetOperators(const Operator &op, const Operator &op_G);
  void Mult(const double *x, double *y) const override;
  void Mult2(const double *x, double *y, double *r) const override;
  void MultTranspose2(const double *x, double *y, double *r) const override;
  int pc_it;
  const Operator *G;
  const Operator *A = nullptr, *A_G = nullptr;
  std::unique_ptr<ChebyshevSmoother> B, B_G;
  mutable DVec x_G, y_G, r_G;
};

class GeometricMultigridSolver : public Solver
{
public:
  // P[l]: level l -> l+1 prolongation (l = 0 .. n_levels-2); G[l]: aux (H1) -> primary (ND) gradient per level or empty.
  GeometricMultigridSolver(b2p_ctx *c, std::unique_ptr<Solver> &&coarse, const std::vector<const Operator *> &P,
                           const std::vector<const Operator *> &G, int cycle_it, int smooth_it, int cheby_order, double sf_max,
                           double sf_min, bool fourth_kind);
  void SetOperator(const Operator &) override;
  void SetOperators(const std::vector<const Operator *> &A, const std::vector<const Operator *> &A_aux);
  void Mult(const double *x, double *y) const override;
  int pc_it;
  std::vector<const Operator *> P;
  std::vector<const Operator *> A;
  std::vector<std::unique_ptr<Solver>> B;
  mutable std::vector<DVec> X, Y, R;

private:
  void VCycle(int l, bool initial_guess) const;
  // the finest level works on the caller's vectors directly (x is only read there, y is the iterate): no copies in / out
  mutable const double *x_top = nullptr;
  mutable double *y_top = nullptr;
  const double *Xp(int l) const { return l + 1 == (int)A.size() ? x_top : X[l].p; }
  double *Yp(int l) const { return l + 1 == (int)A.size() ? y_top : Y[l].p; }
};

enum class KspType { CG = 0, GMRES = 1, FGMRES = 2 };
enum class Orthog { MGS = 0, CGS = 1, CGS2 = 2 };
enum class PcSide { RIGHT = 0, LEFT = 1 };

class IterativeSolver : public Solver
{
public:
  IterativeSolver(b2p_ctx *c, KspType type) : Solver(c), type(type) {}
  void SetOperator(const Operator &op) override
  {
    A = &op;
    height = op.Height();
    width = op.Width();
  }
  void SetPreconditioner(const Solver *pc) { B = pc; }
  void Mult(const double *b, double *x) const override;
  KspType type;
  const Operator *A = nullptr;
  const Solver *B = nullptr;
  double rel_tol = 1e-6, abs_tol = 0.0;
  int max_it = 100, max_dim = -1;
  // CG only: > 1 keeps the recurrence scalars in device memory and looks at the residual every check_every iterations
  // only (one host synchronisation per check instead of two per iteration); may run up to check_every - 1 iterations
  // past convergence. 1 = the reference's iteration (iterative.cpp:361-486).
  int check_every = 1;
  Orthog gs = Orthog::MGS;
  PcSide pc_side = PcSide::RIGHT;
  int print = 0;
  // results
  mutable bool converged = false;
  mutable double initial_res = 1.0, final_res = 0.0;
  mutable int final_it = 0;
  mutable std::vector<double> res_history;

private:
  void MultCG(const double *b, double *x) const;
  void MultCGDeviceScalars(const double *b, double *x) const;
  mutable DVec scal;  // device scalars of the sync-free CG
  void MultGMRES(const double *b, double *x, bool flexible) const;
  mutable std::vector<std::unique_ptr<DVec>> V, Z;
  mutable DVec r, z, p;
  mutable std::vector<double> H, s, cs, sn;
};

}  // namespace b2p
