// Header-only Palace/MFEM adapters over the C ABI of b2p.h. Compiled only inside a Palace build
// (needs <mfem.hpp> and Palace's own headers); nothing here is built or tested in this repository,
// where MFEM is not available — it documents exactly which reference interface each entry point
// replaces. See INTEGRATION.md.
//
//   b2p::palace::Operator            replaces palace::ceed::Operator   (palace/fem/libceed/operator.hpp:32-65)
//   b2p::palace::ParOperatorAdapter  replaces palace::ParOperator      (palace/linalg/rap.hpp:24-121)
//   b2p::palace::SolverAdapter       wraps any b2p_solver as palace::Solver<palace::Operator>
//                                    (palace/linalg/solver.hpp:21-65): Chebyshev, Jacobi, DistRelaxation,
//                                    GeometricMultigrid, Cg/Gmres/Fgmres.
//   b2p::palace::ComplexParOperatorAdapter  replaces palace::ComplexParOperator over ComplexWrapperOperator
//                                    (palace/linalg/rap.hpp:123-220, operator.cpp:98-134): sum_i (a_i^r + i a_i^i) A_i on split
//                                    real / imaginary vectors, one fused element-kernel launch per matvec when eligible.
//   b2p::palace::KspSolverAdapter    replaces palace::BaseKspSolver<Operator> (palace/linalg/ksp.hpp:24-75): one configuration
//                                    record -> Krylov solver + p-multigrid preconditioner, NumTotalMult / NumTotalMultIterations.
//   b2p::palace::FullAssembly        replaces BilinearForm::FullAssemble / CeedOperatorFullAssemble for the coarse level
//                                    (palace/fem/bilinearform.hpp:72-84, libceed/operator.cpp:262-523): device CSR arrays
//                                    to wrap in a hypre::HypreCSRMatrix.
// tests/test_capi_symbols.py compiles this header against a mock <mfem.hpp> (tests/mock_mfem) so that its use of the C ABI
// stays type-correct.
#pragma once
#if defined(MFEM_VERSION) || __has_include(<mfem.hpp>)
#include <mfem.hpp>

#include <cstdint>
#include <memory>
#include <vector>

#include "b2p.h"

namespace b2p::palace
{

inline void Check(int rc, b2p_ctx *ctx)
{
  if (rc != B2P_SUCCESS)
  {
    MFEM_ABORT("b2p error " << rc << ": " << b2p_last_error(ctx));  // PalaceCeedCall semantics, ceed.hpp:13-33
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Integrator glue: MFEM objects -> the descriptors of b2p.h. This is what BilinearForm::PartialAssemble
// (palace/fem/bilinearform.cpp:27-107) does through InitBasis / InitRestriction / Mesh::GetCeedGeomFactorData for libCEED:
//   1-D tables       fem/libceed/basis.cpp:15-38    (fe.GetDofToQuad(ir, TENSOR) of the closed and open bases)
//   dof map          fem/libceed/restriction.cpp:134-136,413-426 (TensorBasisElement::GetDofMap())
//   element dofs     fem/libceed/restriction.cpp:207-297 (GetElementDofs: index + sign from the -1-d encoding)
//   node coordinates fem/mesh.cpp:146-209           (E-vector of mesh.GetNodes(), attributes)
// tests/mock_mfem/glue_exec.cpp runs these functions on a one-element mesh through the C ABI against the oracle.
// ------------------------------------------------------------------------------------------------------------------
// Host arrays a b2p_op_desc points into (they must outlive b2p_op_create only).
struct HexNDSpaceInputs
{
  int p = 0, q1d = 0, ne = 0;
  long long lsize = 0;
  std::vector<int32_t> idx, dof_map;
  std::vector<int8_t> orient;
  std::vector<double> Bo, Bc, Gc;
};

// DofToQuad tables are column-major [nqpt x ndof] (B[q + nqpt * d]); b2p wants [q1d][ndof] row-major.
inline std::vector<double> RowMajorTable(const std::vector<double> &colmajor, int nqpt, int ndof)
{
  std::vector<double> t((size_t)nqpt * ndof);
  for (int q = 0; q < nqpt; q++)
    for (int d = 0; d < ndof; d++) t[(size_t)q * ndof + d] = colmajor[q + (size_t)nqpt * d];
  return t;
}

inline HexNDSpaceInputs GatherHexNDSpace(const mfem::FiniteElementSpace &fes, const mfem::IntegrationRule &ir1d)
{
  HexNDSpaceInputs in;
  const auto *fe = dynamic_cast<const mfem::VectorTensorFiniteElement *>(fes.GetFE(0));
  MFEM_VERIFY(fe, "GatherHexNDSpace: a tensor-product vector element (ND hexahedron) is required!");
  in.p = fe->GetOrder();
  in.q1d = ir1d.GetNPoints();
  in.ne = fes.GetNE();
  in.lsize = fes.GetVSize();
  const mfem::DofToQuad &mc = fe->GetDofToQuad(ir1d, mfem::DofToQuad::TENSOR);      // closed (Gauss-Lobatto) basis
  const mfem::DofToQuad &mo = fe->GetDofToQuadOpen(ir1d, mfem::DofToQuad::TENSOR);  // open (Gauss-Legendre) basis
  MFEM_VERIFY(mc.ndof == in.p + 1 && mo.ndof == in.p && mc.nqpt == in.q1d && mo.nqpt == in.q1d, "unexpected 1-D table sizes!");
  in.Bc = RowMajorTable(mc.B, in.q1d, in.p + 1);
  in.Gc = RowMajorTable(mc.G, in.q1d, in.p + 1);
  in.Bo = RowMajorTable(mo.B, in.q1d, in.p);
  const mfem::Array<int> &dm = fe->GetDofMap();
  in.dof_map.assign(dm.HostRead(), dm.HostRead() + dm.Size());
  const int P = dm.Size();
  in.idx.resize((size_t)in.ne * P);
  in.orient.resize((size_t)in.ne * P);
  mfem::Array<int> dofs;
  for (int e = 0; e < in.ne; e++)
  {
    fes.GetElementDofs(e, dofs);  // native element order; d < 0 encodes -(d + 1) with a sign flip (restriction.cpp:281-297)
    MFEM_VERIFY(dofs.Size() == P, "element dof count differs from the dof map!");
    for (int i = 0; i < P; i++)
    {
      const int d = dofs[i];
      in.idx[(size_t)e * P + i] = d >= 0 ? d : -1 - d;
      in.orient[(size_t)e * P + i] = d >= 0 ? 1 : -1;
    }
  }
  return in;
}

// Geometry handle of a hexahedral mesh block (Mesh::GetCeedGeomFactorData -> b2p_geom_create_hex): the element node
// coordinates in LEXICOGRAPHIC tensor order, component-major, through the nodal element's dof map; 1-D nodal tables and
// weights of the rule.
inline b2p_geom *CreateHexGeometry(b2p_ctx *ctx, const mfem::Mesh &mesh, const mfem::IntegrationRule &ir1d)
{
  const mfem::GridFunction *nodes = mesh.GetNodes();
  MFEM_VERIFY(nodes, "CreateHexGeometry: the mesh needs a nodal grid function (Mesh::EnsureNodes)!");
  const mfem::FiniteElementSpace *nfes = nodes->FESpace();
  const auto *nfe = dynamic_cast<const mfem::NodalTensorFiniteElement *>(nfes->GetFE(0));
  MFEM_VERIFY(nfe && nfes->GetVDim() == 3, "CreateHexGeometry: H1 tensor-product nodes in 3-D are required!");
  const int k = nfe->GetOrder(), nn = (k + 1) * (k + 1) * (k + 1), ne = mesh.GetNE(), q1d = ir1d.GetNPoints();
  const mfem::DofToQuad &mn = nfe->GetDofToQuad(ir1d, mfem::DofToQuad::TENSOR);
  const std::vector<double> nB = RowMajorTable(mn.B, q1d, k + 1), nG = RowMajorTable(mn.G, q1d, k + 1);
  const mfem::Array<int> &dm = nfe->GetDofMap();  // lexicographic -> native node
  std::vector<double> xe((size_t)ne * 3 * nn);
  std::vector<int32_t> attr(ne);
  mfem::Array<int> vdofs;
  mfem::Vector xv;
  for (int e = 0; e < ne; e++)
  {
    nfes->GetElementVDofs(e, vdofs);  // byNODES: [x of all nodes | y ... | z ...] in native node order
    nodes->GetSubVector(vdofs, xv);
    for (int c = 0; c < 3; c++)
      for (int l = 0; l < nn; l++) xe[((size_t)e * 3 + c) * nn + l] = xv.HostRead()[c * nn + (dm.Size() ? dm[l] : l)];
    attr[e] = mesh.GetAttribute(e);
  }
  std::vector<double> qw(q1d);
  for (int i = 0; i < q1d; i++) qw[i] = ir1d.IntPoint(i).weight;
  b2p_geom *geom = nullptr;
  Check(b2p_geom_create_hex(ctx, ne, k, q1d, xe.data(), nB.data(), nG.data(), qw.data(), attr.data(), &geom), ctx);
  return geom;
}

// One integrator of the form on one hexahedral block: kind from fem/integ/{curlcurl,vecfemass,curlcurlmass}.cpp, or one of
// the Floquet pair of fem/integ/mixedveccurl.cpp (B2P_ND_WEAKCURL / B2P_ND_MIXEDCURL, on-the-fly coefficients only), the
// coefficient context bytes exactly as PopulateCoefficientContext builds them (fem/libceed/coefficient.cpp:51-130).
inline b2p_op *CreateHexNDIntegrator(b2p_ctx *ctx, b2p_geom *geom, int kind, const HexNDSpaceInputs &in, const void *coeff_ctx,
                                     size_t coeff_ctx_bytes, bool assemble_q_data = false)
{
  b2p_op_desc d = {};
  d.kind = kind;
  d.p = in.p;
  d.ne = in.ne;
  d.lsize = in.lsize;
  d.idx = in.idx.data();
  d.orient = in.orient.data();
  d.dof_map = in.dof_map.data();
  d.Bo = in.Bo.data();
  d.Bc = in.Bc.data();
  d.Gc = in.Gc.data();
  d.coeff_ctx = coeff_ctx;
  d.coeff_ctx_bytes = coeff_ctx_bytes;
  d.assemble_qdata = assemble_q_data ? 1 : 0;
  b2p_op *op = nullptr;
  Check(b2p_op_create(ctx, geom, &d, &op), ctx);
  return op;
}

// ---- non-tensor elements (tetrahedra, prisms, pyramids; any vector element libCEED sees through dense tables) --------------
// What InitNonTensorBasis (fem/libceed/basis.cpp:40-85) and InitNativeRestr (fem/libceed/restriction.cpp:207-385) gather, as the
// arrays of a b2p_dense_op_desc: the FULL DofToQuad tables Bt / Gt ARE interp[3][Q][P] / deriv[3][Q][P]; element dofs with the
// -1-d sign encoding; with a DofTransformation (ND tets / prisms of order >= 2) the int8 tridiagonal rows, filled column by
// column from InvTransformPrimal exactly as restriction.cpp:301-329 does.
struct DenseNDSpaceInputs
{
  int P = 0, Q = 0, ne = 0;
  long long lsize = 0;
  std::vector<int32_t> idx;
  std::vector<int8_t> orient, curl_orient;  // one of the two is filled
  std::vector<double> interp, deriv;
};

inline DenseNDSpaceInputs GatherDenseNDSpace(const mfem::FiniteElementSpace &fes, const mfem::IntegrationRule &ir)
{
  DenseNDSpaceInputs in;
  const auto *fe = dynamic_cast<const mfem::VectorFiniteElement *>(fes.GetFE(0));
  MFEM_VERIFY(fe && fe->GetDim() == 3, "GatherDenseNDSpace: a 3-D vector finite element is required!");
  const mfem::DofToQuad &maps = fe->GetDofToQuad(ir, mfem::DofToQuad::FULL);
  in.P = maps.ndof;
  in.Q = maps.nqpt;
  in.ne = fes.GetNE();
  in.lsize = fes.GetVSize();
  MFEM_VERIFY((int)maps.Bt.size() == 3 * in.Q * in.P && (int)maps.Gt.size() == 3 * in.Q * in.P, "unexpected FULL table sizes!");
  in.interp = maps.Bt;
  in.deriv = maps.Gt;
  const int P = in.P;
  in.idx.resize((size_t)in.ne * P);
  mfem::Array<int> dofs;
  mfem::Vector col(P);
  bool any_trans = false;
  for (int e = 0; e < in.ne && !any_trans; e++) any_trans = fes.GetElementDofs(e, dofs, 0) != nullptr;
  if (any_trans)
    in.curl_orient.assign((size_t)in.ne * P * 3, 0);
  else
    in.orient.resize((size_t)in.ne * P);
  for (int e = 0; e < in.ne; e++)
  {
    const mfem::DofTransformation *dt = fes.GetElementDofs(e, dofs, 0);
    MFEM_VERIFY(dofs.Size() == P, "element dof count differs from the table!");
    for (int j = 0; j < P; j++)
    {
      const int d = dofs[j];
      in.idx[(size_t)e * P + j] = d >= 0 ? d : -1 - d;
      if (!any_trans)
      {
        in.orient[(size_t)e * P + j] = d >= 0 ? 1 : -1;
        continue;
      }
      // column j of the element's transformation, scaled by the sign of dof j (restriction.cpp:301-329)
      col = 0.0;
      col[j] = 1.0;
      if (dt) dt->InvTransformPrimal(col);
      const double sj = d >= 0 ? 1.0 : -1.0;
      int8_t *co = in.curl_orient.data() + (size_t)e * P * 3;
      co[3 * j + 1] = (int8_t)(sj * col[j]);
      if (j > 0) co[3 * (j - 1) + 2] = (int8_t)(sj * col[j - 1]);
      if (j < P - 1) co[3 * (j + 1) + 0] = (int8_t)(sj * col[j + 1]);
    }
  }
  return in;
}

// q-data of any element type at the points of `ir` (Mesh::GetCeedGeomFactorData + f_build_geom_factor_33, fem/mesh.cpp:146-209,
// qfunctions/33/geom_33_qf.h:9-34): {attr, w detJ, adj(J)^T / detJ = J^-T column-major} from the element transformations.
inline b2p_geom *CreateGeneralGeometry(b2p_ctx *ctx, const mfem::Mesh &mesh, const mfem::IntegrationRule &ir)
{
  const int ne = mesh.GetNE(), Q = ir.GetNPoints();
  std::vector<double> qd((size_t)ne * 11 * Q);
  for (int e = 0; e < ne; e++)
  {
    mfem::ElementTransformation *T = mesh.GetElementTransformation(e);
    for (int q = 0; q < Q; q++)
    {
      const mfem::IntegrationPoint &ip = ir.IntPoint(q);
      T->SetIntPoint(&ip);
      const mfem::DenseMatrix &J = T->Jacobian();
      const double det = T->Weight();
      double *o = qd.data() + (size_t)e * 11 * Q + q;
      o[0] = mesh.GetAttribute(e);
      o[(size_t)Q] = ip.weight * det;
      // J^-T = cofactor(J) / det, stored column-major: entry (r, c) at 2 + r + 3 c
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++)
        {
          const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
          o[(size_t)(2 + r + 3 * c) * Q] = (J(r1, c1) * J(r2, c2) - J(r1, c2) * J(r2, c1)) / det;
        }
    }
  }
  b2p_geom *geom = nullptr;
  Check(b2p_geom_create_qdata_general(ctx, ne, Q, qd.data(), &geom), ctx);
  return geom;
}

inline b2p_op *CreateDenseNDIntegrator(b2p_ctx *ctx, b2p_geom *geom, int kind, const DenseNDSpaceInputs &in, const void *coeff_ctx,
                                       size_t coeff_ctx_bytes)
{
  b2p_dense_op_desc d = {};
  d.kind = kind;
  d.P = in.P;
  d.Q = in.Q;
  d.ne = in.ne;
  d.lsize = in.lsize;
  d.idx = in.idx.data();
  d.orient = in.orient.empty() ? nullptr : in.orient.data();
  d.curl_orient = in.curl_orient.empty() ? nullptr : in.curl_orient.data();
  d.interp = in.interp.data();
  d.deriv = in.deriv.data();
  d.coeff_ctx = coeff_ctx;
  d.coeff_ctx_bytes = coeff_ctx_bytes;
  b2p_op *op = nullptr;
  Check(b2p_op_create_dense(ctx, geom, &d, &op), ctx);
  return op;
}

// Same five methods as ceed::Operator; sub-operators are b2p_op handles created by the integrator glue.
class Operator : public mfem::Operator
{
protected:
  b2p_ctx *ctx;
  std::vector<b2p_op *> ops;  // owned (AddSubOperator takes ownership, operator.cpp:60-87)

public:
  Operator(b2p_ctx *ctx, int h, int w) : mfem::Operator(h, w), ctx(ctx) {}
  ~Operator() override
  {
    for (auto *op : ops) b2p_op_destroy(op);
  }
  void AddSubOperator(b2p_op *sub_op) { ops.push_back(sub_op); }
  void Finalize() {}
  void DestroyAssemblyData() const {}
  const std::vector<b2p_op *> &SubOperators() const { return ops; }

  void Mult(const mfem::Vector &x, mfem::Vector &y) const override
  {
    y = 0.0;  // operator.cpp:184
    AddMult(x, y, 1.0);
  }
  void AddMult(const mfem::Vector &x, mfem::Vector &y, const double a = 1.0) const override
  {
    const double *xd = x.Read(true);  // zero-copy device pointers, operator.cpp:160-161
    double *yd = y.ReadWrite(true);
    for (auto *op : ops) Check(b2p_op_apply_add_ex(op, a, xd, yd, 0, nullptr), ctx);
  }
  void MultTranspose(const mfem::Vector &x, mfem::Vector &y) const override { Mult(x, y); }  // SymmetricOperator
  void AddMultTranspose(const mfem::Vector &x, mfem::Vector &y, const double a = 1.0) const override { AddMult(x, y, a); }
  void AssembleDiagonal(mfem::Vector &diag) const override
  {
    diag = 0.0;
    double *d = diag.ReadWrite(true);
    for (auto *op : ops) Check(b2p_op_diag_add(op, d, nullptr), ctx);
  }
};

// y = P^T (sum_i c_i A_i) P x with essential-dof elimination done inside the element kernels.
class ParOperatorAdapter : public mfem::Operator
{
  b2p_ctx *ctx;
  b2p_operator *A = nullptr;
  mfem::Array<int> dbc_tdof_list;

public:
  ParOperatorAdapter(b2p_ctx *ctx, int tsize, int lsize, const std::vector<b2p_op *> &ops, const std::vector<double> &coefs,
                     const mfem::Array<int> &dbc, int diag_policy, b2p_halo *halo)
    : mfem::Operator(tsize), ctx(ctx), dbc_tdof_list(dbc)
  {
    Check(b2p_operator_par(ctx, tsize, lsize, (int)ops.size(), ops.data(), coefs.data(), dbc.HostRead(), dbc.Size(), diag_policy,
                           halo, &A),
          ctx);
  }
  ~ParOperatorAdapter() override { b2p_operator_destroy(A); }
  b2p_operator *Handle() const { return A; }
  const mfem::Array<int> *GetEssentialTrueDofs() const { return dbc_tdof_list.Size() ? &dbc_tdof_list : nullptr; }
  void Mult(const mfem::Vector &x, mfem::Vector &y) const override { Check(b2p_operator_mult(A, x.Read(true), y.Write(true)), ctx); }
  void MultTranspose(const mfem::Vector &x, mfem::Vector &y) const override { Mult(x, y); }
  void AddMult(const mfem::Vector &x, mfem::Vector &y, const double a = 1.0) const override
  {
    Check(b2p_operator_add_mult(A, x.Read(true), y.ReadWrite(true), a), ctx);
  }
  void AssembleDiagonal(mfem::Vector &d) const override { Check(b2p_operator_assemble_diagonal(A, d.Write(true)), ctx); }
};

// palace::Solver<Operator> over a b2p_solver handle.
class SolverAdapter : public mfem::Solver
{
protected:
  b2p_ctx *ctx;
  b2p_solver *S;
  bool initial_guess = false;

public:
  SolverAdapter(b2p_ctx *ctx, b2p_solver *S) : mfem::Solver(), ctx(ctx), S(S) {}
  ~SolverAdapter() override { b2p_solver_destroy(S); }
  b2p_solver *Handle() const { return S; }
  void SetInitialGuess(bool guess)
  {
    initial_guess = guess;
    Check(b2p_solver_set_initial_guess(S, guess), ctx);
  }
  void SetOperator(const mfem::Operator &op) override
  {
    const auto *par = dynamic_cast<const ParOperatorAdapter *>(&op);
    MFEM_VERIFY(par, "b2p solvers require a b2p ParOperatorAdapter!");
    Check(b2p_solver_set_operator(S, par->Handle()), ctx);
    height = op.Height();
    width = op.Width();
  }
  void Mult(const mfem::Vector &x, mfem::Vector &y) const override { Check(b2p_solver_mult(S, x.Read(true), y.ReadWrite(true)), ctx); }
  void Mult2(const mfem::Vector &x, mfem::Vector &y, mfem::Vector &r) const
  {
    Check(b2p_solver_mult2(S, x.Read(true), y.ReadWrite(true), r.Write(true)), ctx);
  }
  void MultTranspose2(const mfem::Vector &x, mfem::Vector &y, mfem::Vector &r) const
  {
    Check(b2p_solver_mult_transpose2(S, x.Read(true), y.ReadWrite(true), r.Write(true)), ctx);
  }
};

// The multigrid's coarse solver on the device-assembled level-0 matrix: MfemWrapperSolver<Operator> (palace/linalg/solver.hpp:
// 67-110, solver.cpp:13-30) with a Krylov method (and its preconditioner) from this library inside instead of HYPRE. The
// handles `krylov` and `pc` are consumed; SetOperator assembles the ParOperator it is given.
inline std::unique_ptr<SolverAdapter> MakeAssembledCoarseSolver(b2p_ctx *ctx, b2p_solver *krylov, b2p_solver *pc)
{
  b2p_solver *S = nullptr;
  Check(b2p_solver_assembled(ctx, krylov, pc, &S), ctx);
  b2p_solver_destroy(krylov);
  if (pc) b2p_solver_destroy(pc);
  return std::make_unique<SolverAdapter>(ctx, S);
}

// palace::ComplexOperator interface (palace/linalg/operator.hpp:24-68) on two mfem::Vectors per complex vector
// (palace/linalg/vector.hpp:23-27).
class ComplexParOperatorAdapter
{
  b2p_ctx *ctx;
  b2p_coperator *A = nullptr;
  int n;

public:
  ComplexParOperatorAdapter(b2p_ctx *ctx, int tsize, int lsize, const std::vector<b2p_op *> &ops, const std::vector<double> &coef_re,
                            const std::vector<double> &coef_im, const mfem::Array<int> &dbc, int diag_policy)
    : ctx(ctx), n(tsize)
  {
    Check(b2p_coperator_par(ctx, tsize, lsize, (int)ops.size(), ops.data(), coef_re.data(), coef_im.data(), dbc.HostRead(), dbc.Size(),
                            diag_policy, &A),
          ctx);
  }
  // The reference's own ComplexParOperator(Ar, Ai) form over two real adapters (rap.hpp:123-150): this is the one for
  // PARTITIONED spaces (each part runs its halo exchange); give Ar DIAG_ONE and Ai DIAG_ZERO. Either part may be null.
  ComplexParOperatorAdapter(b2p_ctx *ctx, const ParOperatorAdapter *Ar, const ParOperatorAdapter *Ai)
    : ctx(ctx), n((Ar ? Ar : Ai)->Height())
  {
    Check(b2p_coperator_wrap(ctx, Ar ? Ar->Handle() : nullptr, Ai ? Ai->Handle() : nullptr, &A), ctx);
  }
  ~ComplexParOperatorAdapter() { b2p_coperator_destroy(A); }
  b2p_coperator *Handle() const { return A; }
  int Height() const { return n; }
  // next frequency of a sweep: a0 K + a1 C + a2 M with new a_i, nothing rebuilt (spaceoperator.cpp:945-1153)
  void SetCoefficients(const std::vector<double> &coef_re, const std::vector<double> &coef_im)
  {
    Check(b2p_coperator_set_coefficients(A, (int)coef_re.size(), coef_re.data(), coef_im.data()), ctx);
  }
  void Mult(const mfem::Vector &xr, const mfem::Vector &xi, mfem::Vector &yr, mfem::Vector &yi) const
  {
    Check(b2p_coperator_mult(A, xr.Read(true), xi.Read(true), yr.Write(true), yi.Write(true)), ctx);
  }
  void MultHermitianTranspose(const mfem::Vector &xr, const mfem::Vector &xi, mfem::Vector &yr, mfem::Vector &yi) const
  {
    Check(b2p_coperator_mult_hermitian_transpose(A, xr.Read(true), xi.Read(true), yr.Write(true), yi.Write(true)), ctx);
  }
  void AddMult(const mfem::Vector &xr, const mfem::Vector &xi, mfem::Vector &yr, mfem::Vector &yi, double ar, double ai) const
  {
    Check(b2p_coperator_add_mult(A, xr.Read(true), xi.Read(true), yr.ReadWrite(true), yi.ReadWrite(true), ar, ai), ctx);
  }
  void AssembleDiagonal(mfem::Vector &dr, mfem::Vector &di) const
  {
    Check(b2p_coperator_assemble_diagonal(A, dr.Write(true), di.Write(true)), ctx);
  }
};

// Coarse-level matrix for HYPRE (AMS / BoomerAMG) or a sparse direct solver: symbolic phase once per space, numeric phase
// per coefficient change, device CSR arrays handed out by pointer (wrap with hypre_CSRMatrixCreate + I / J / Data).
class FullAssembly
{
  b2p_ctx *ctx;
  b2p_csr *csr = nullptr;

public:
  FullAssembly(b2p_ctx *ctx, b2p_op *space_op) : ctx(ctx) { Check(b2p_csr_create(ctx, space_op, &csr), ctx); }
  ~FullAssembly() { b2p_csr_destroy(csr); }
  void Assemble(const std::vector<b2p_op *> &ops, const std::vector<double> &coefs)
  {
    Check(b2p_csr_assemble(csr, (int)ops.size(), ops.data(), coefs.data(), nullptr), ctx);
  }
  long long Rows() const { return b2p_csr_rows(csr); }
  long long NNZ() const { return b2p_csr_nnz(csr); }
  void DeviceArrays(const int **I, const int **J, const double **data) const { Check(b2p_csr_device_arrays(csr, I, J, data), ctx); }
};

// palace::BaseKspSolver<Operator> (palace/linalg/ksp.hpp:24-75, ksp.cpp:256-328): the configured Krylov solver together
// with its (multigrid) preconditioner, built from one b2p_ksp_config -- see INTEGRATION.md section 5 for the field mapping
// from config::LinearSolverData. P / G: prolongation and discrete-gradient operators of the space hierarchy
// (fespaces.GetProlongationOperators(), GetDiscreteInterpolators(aux_fespaces)), already wrapped as b2p_operator handles.
class KspSolverAdapter
{
  b2p_ctx *ctx;
  b2p_ksp *K = nullptr;
  int n_levels;

public:
  KspSolverAdapter(b2p_ctx *ctx, const b2p_ksp_config &cfg, const std::vector<b2p_operator *> &P, const std::vector<b2p_operator *> &G,
                   b2p_solver *coarse_plugin = nullptr)
    : ctx(ctx), n_levels((int)P.size() + 1)
  {
    Check(b2p_ksp_create(ctx, &cfg, n_levels, P.data(), G.empty() ? nullptr : G.data(), coarse_plugin, &K), ctx);
  }
  ~KspSolverAdapter() { b2p_ksp_destroy(K); }
  // SetOperators(op, pc_op): pc_levels / aux_levels are the ParOperators of the MultigridOperator, coarsest first
  void SetOperators(const ParOperatorAdapter &op, const std::vector<const ParOperatorAdapter *> &pc_levels,
                    const std::vector<const ParOperatorAdapter *> &aux_levels)
  {
    MFEM_VERIFY((int)pc_levels.size() == n_levels, "one preconditioner operator per multigrid level!");
    std::vector<b2p_operator *> A, Ax;
    for (auto *a : pc_levels) A.push_back(a->Handle());
    for (auto *a : aux_levels) Ax.push_back(a ? a->Handle() : nullptr);
    Check(b2p_ksp_set_operators(K, op.Handle(), A.data(), Ax.empty() ? nullptr : Ax.data()), ctx);
  }
  void Mult(const mfem::Vector &x, mfem::Vector &y) const { Check(b2p_ksp_mult(K, x.Read(true), y.ReadWrite(true)), ctx); }
  int NumTotalMult() const
  {
    int n = 0;
    Check(b2p_ksp_stats(K, &n, nullptr, nullptr, nullptr, nullptr, nullptr), ctx);
    return n;
  }
  int NumTotalMultIterations() const
  {
    int n = 0;
    Check(b2p_ksp_stats(K, nullptr, &n, nullptr, nullptr, nullptr, nullptr), ctx);
    return n;
  }
};

}  // namespace b2p::palace
#endif
