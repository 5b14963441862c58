// Matrix-free Nedelec (H(curl)) hexahedron operators: curl-curl, mass, curl-curl + mass, and the block form of the mixed
// curl kinds and their sums (B2P_ND_BLOCK: value and curl at every point, coupled by four 3x3 tensors per element).
//
//   y_L += sum_e E_e^T  B^T  D  B  E_e x_L
//
// Replaces libCEED's CeedOperatorApplyAdd behind ceed::Operator::AddMult
// (/root/reference/palace/fem/libceed/operator.cpp:148-178) for the integrators
// /root/reference/palace/fem/integ/{curlcurl,vecfemass,curlcurlmass}.cpp on hexes. The reference
// applies a DENSE [3Q x P] interp and curl table per element (fem/libceed/basis.cpp:40-85); here B
// is sum-factorised over the 1-D open (Gauss-Legendre) / closed (Gauss-Lobatto) bases of the ND hex
// element, which is the same linear operator in O(p^4) instead of O(p^6) flops per element.
//
// Lexicographic element layout (restriction pre-composed with TensorBasisElement::GetDofMap()):
//   x-directed dofs Ux[k][j][i], i<p (open),  j,k<=p (closed)   offset 0
//   y-directed dofs Uy[k][j][i], i<=p, j<p (open), k<=p          offset p(p+1)^2
//   z-directed dofs Uz[k][j][i], i,j<=p, k<p (open)              offset 2p(p+1)^2
// Quadrature points x-fastest (basis.cpp:18-19).
#include "b2p_internal.hpp"
#include "b2p_qf.cuh"
#include "b2p_contract.cuh"

namespace b2p
{

namespace
{

template <int P_, int Q_>
struct NDLayout
{
  static constexpr int p = P_, q = Q_, n = P_ + 1;
  static constexpr int P = 3 * p * n * n;
  static constexpr int Q = q * q * q;
  static constexpr int D3 = p * n * n;
  // scratch sizes
  static constexpr int N1 = q * n * n;  // after one contraction (largest)
  static constexpr int N2 = q * q * n;  // after two
  // per-element shared doubles: U | T1a T1b | T2a T2b T2c | uq[3Q] cq[3Q]
  static constexpr int PER_ELEM = P + 2 * N1 + 3 * N2 + 6 * Q;
};

struct NDParams
{
  const int32_t *lidx;
  const double *tab;   // Bo[q][p] | Bc[q][n] | Gc[q][n]
  const double *qd;    // [ne][10][Q]
  const double *mat;   // [n_mat][9]
  const int32_t *emat; // [ne][2]
  const double *aq;    // assembled q-data [ne][ncomp][Q] or null
  const double *x;
  double *y;
  double alpha;
  int64_t aq_estride;
  int ne;
  int PS;  // padded restriction row stride
  VSplit sp;
  const double *bcoef;  // B2P_ND_BLOCK: [ne][36] {Cm, Ck, Cw, Cx} (the transposed block for a transposed apply)
};

// KIND: B2P_CURLCURL / B2P_ND_MASS / B2P_CURLCURL_MASS / B2P_ND_BLOCK. ASM: assembled q-data.
template <int P_, int Q_, int KIND, bool ASM, int NEB, int NT>
__global__ void __launch_bounds__(NT) nd_hex_apply_kernel(NDParams prm)
{
  using L = NDLayout<P_, Q_>;
  constexpr int p = L::p, q = L::q, n = L::n, P = L::P, Q = L::Q, D3 = L::D3, N1 = L::N1, N2 = L::N2;
  constexpr bool BLOCK = (KIND == B2P_ND_BLOCK);
  constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS || BLOCK);
  constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS || BLOCK);
  static_assert(!(BLOCK && ASM), "block operators have no assembled q-data");
  constexpr int ES = L::PER_ELEM;

  B2P_DYN_SMEM(double, smem);
  double *sBo = smem;            // [q][p]
  double *sBc = sBo + q * p;     // [q][n]
  double *sGc = sBc + q * n;     // [q][n]
  double *work = sGc + q * n;
  double *U = work;              // + e*ES
  double *T1a = U + P, *T1b = T1a + N1;
  double *T2a = T1b + N1, *T2b = T2a + N2, *T2c = T2b + N2;
  double *uq = T2c + N2, *cq = uq + 3 * Q;

  for (int i = threadIdx.x; i < q * p + 2 * q * n; i += NT) sBo[i] = prm.tab[i];

  const int e0 = blockIdx.x * NEB;
  // ---- gather (E): lexicographic dofs with sign ----
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    double v = 0.0;
    if (e0 + e < prm.ne)
    {
      v = gather2(prm.x, prm.sp, prm.lidx[(size_t)(e0 + e) * prm.PS + l]);
    }
    U[e * ES + l] = v;
  }
  for (int w = threadIdx.x; w < NEB * 3 * Q; w += NT)
  {
    const int e = w / (3 * Q), i = w % (3 * Q);
    uq[e * ES + i] = 0.0;
    cq[e * ES + i] = 0.0;
  }
  __syncthreads();

  // ---- forward: values and reference curl at quadrature points ----
  // x-directed: Ux dims (p, n, n)
  contract<0, p, n, n, p, q, false, NEB, NT>(U, ES, T1a, ES, sBo, p, 1, 1.0);
  __syncthreads();
  contract<1, q, n, n, n, q, false, NEB, NT>(T1a, ES, T2a, ES, sBc, n, 1, 1.0);
  if (CURL) contract<1, q, n, n, n, q, false, NEB, NT>(T1a, ES, T2b, ES, sGc, n, 1, 1.0);
  __syncthreads();
  if (MASS) contract<2, q, q, n, n, q, true, NEB, NT>(T2a, ES, uq + 0 * Q, ES, sBc, n, 1, 1.0);
  if (CURL)
  {
    contract<2, q, q, n, n, q, true, NEB, NT>(T2a, ES, cq + 1 * Q, ES, sGc, n, 1, 1.0);   // curl_y += dz ux
    contract<2, q, q, n, n, q, true, NEB, NT>(T2b, ES, cq + 2 * Q, ES, sBc, n, 1, -1.0);  // curl_z -= dy ux
  }
  __syncthreads();
  // y-directed: Uy dims (n, p, n)
  contract<0, n, p, n, n, q, false, NEB, NT>(U + D3, ES, T1a, ES, sBc, n, 1, 1.0);
  if (CURL) contract<0, n, p, n, n, q, false, NEB, NT>(U + D3, ES, T1b, ES, sGc, n, 1, 1.0);
  __syncthreads();
  contract<1, q, p, n, p, q, false, NEB, NT>(T1a, ES, T2a, ES, sBo, p, 1, 1.0);
  if (CURL) contract<1, q, p, n, p, q, false, NEB, NT>(T1b, ES, T2b, ES, sBo, p, 1, 1.0);
  __syncthreads();
  if (MASS) contract<2, q, q, n, n, q, true, NEB, NT>(T2a, ES, uq + 1 * Q, ES, sBc, n, 1, 1.0);
  if (CURL)
  {
    contract<2, q, q, n, n, q, true, NEB, NT>(T2a, ES, cq + 0 * Q, ES, sGc, n, 1, -1.0);  // curl_x -= dz uy
    contract<2, q, q, n, n, q, true, NEB, NT>(T2b, ES, cq + 2 * Q, ES, sBc, n, 1, 1.0);   // curl_z += dx uy
  }
  __syncthreads();
  // z-directed: Uz dims (n, n, p)
  contract<0, n, n, p, n, q, false, NEB, NT>(U + 2 * D3, ES, T1a, ES, sBc, n, 1, 1.0);
  if (CURL) contract<0, n, n, p, n, q, false, NEB, NT>(U + 2 * D3, ES, T1b, ES, sGc, n, 1, 1.0);
  __syncthreads();
  contract<1, q, n, p, n, q, false, NEB, NT>(T1a, ES, T2a, ES, sBc, n, 1, 1.0);
  if (CURL)
  {
    contract<1, q, n, p, n, q, false, NEB, NT>(T1a, ES, T2c, ES, sGc, n, 1, 1.0);
    contract<1, q, n, p, n, q, false, NEB, NT>(T1b, ES, T2b, ES, sBc, n, 1, 1.0);
  }
  __syncthreads();
  if (MASS) contract<2, q, q, p, p, q, true, NEB, NT>(T2a, ES, uq + 2 * Q, ES, sBo, p, 1, 1.0);
  if (CURL)
  {
    contract<2, q, q, p, p, q, true, NEB, NT>(T2c, ES, cq + 0 * Q, ES, sBo, p, 1, 1.0);   // curl_x += dy uz
    contract<2, q, q, p, p, q, true, NEB, NT>(T2b, ES, cq + 1 * Q, ES, sBo, p, 1, -1.0);  // curl_y -= dx uz
  }
  __syncthreads();

  // ---- D at quadrature points ----
  for (int w = threadIdx.x; w < NEB * Q; w += NT)
  {
    const int e = w / Q, iq = w % Q, sq = qslot_of(q, iq);
    if (e0 + e >= prm.ne) continue;
    double *uqe = uq + e * ES, *cqe = cq + e * ES;
    if (ASM)
    {
      const double *a = prm.aq + (size_t)(e0 + e) * prm.aq_estride + sq;
      if (MASS)
      {
        const double u0 = uqe[iq], u1 = uqe[Q + iq], u2 = uqe[2 * Q + iq];
        uqe[iq] = a[0 * Q] * u0 + a[3 * Q] * u1 + a[6 * Q] * u2;
        uqe[Q + iq] = a[1 * Q] * u0 + a[4 * Q] * u1 + a[7 * Q] * u2;
        uqe[2 * Q + iq] = a[2 * Q] * u0 + a[5 * Q] * u1 + a[8 * Q] * u2;
        a += 9 * Q;
      }
      if (CURL)
      {
        const double u0 = cqe[iq], u1 = cqe[Q + iq], u2 = cqe[2 * Q + iq];
        cqe[iq] = a[0 * Q] * u0 + a[3 * Q] * u1 + a[6 * Q] * u2;
        cqe[Q + iq] = a[1 * Q] * u0 + a[4 * Q] * u1 + a[7 * Q] * u2;
        cqe[2 * Q + iq] = a[2 * Q] * u0 + a[5 * Q] * u1 + a[8 * Q] * u2;
      }
    }
    else if (BLOCK)
    {
      const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + sq;
      const double *C = prm.bcoef + 36 * (size_t)(e0 + e);
      double A[9], Jd[9], Cm[9], Ck[9], Cw[9], Cx[9];
#pragma unroll
      for (int i = 0; i < 9; i++)
      {
        A[i] = g[(1 + i) * Q];
        Cm[i] = __ldg(C + i);
        Ck[i] = __ldg(C + 9 + i);
        Cw[i] = __ldg(C + 18 + i);
        Cx[i] = __ldg(C + 27 + i);
      }
      cofactor33(A, Jd);
      const double u[3] = {uqe[iq], uqe[Q + iq], uqe[2 * Q + iq]}, c[3] = {cqe[iq], cqe[Q + iq], cqe[2 * Q + iq]};
      double t[3], s[3], a[3], b[3], zv[3], zc[3], v[3], w[3];
      Ax33(A, u, t);
      Ax33(Jd, c, s);
      Ax33(Cm, t, a);
      Ax33(Cx, s, b);
      for (int i = 0; i < 3; i++) zv[i] = a[i] + b[i];
      Ax33(Ck, s, a);
      Ax33(Cw, t, b);
      for (int i = 0; i < 3; i++) zc[i] = a[i] + b[i];
      Atx33(A, zv, g[0], v);
      Atx33(Jd, zc, g[0], w);
      uqe[iq] = v[0];
      uqe[Q + iq] = v[1];
      uqe[2 * Q + iq] = v[2];
      cqe[iq] = w[0];
      cqe[Q + iq] = w[1];
      cqe[2 * Q + iq] = w[2];
    }
    else
    {
      const double *g = prm.qd + (size_t)(e0 + e) * 10 * Q + sq;
      const double wdetJ = g[0];
      double A[9];
#pragma unroll
      for (int i = 0; i < 9; i++) A[i] = g[(1 + i) * Q];
      const int32_t *em = prm.emat + 2 * (size_t)(e0 + e);
      if (MASS)
      {
        double C[9], u[3] = {uqe[iq], uqe[Q + iq], uqe[2 * Q + iq]}, v[3];
#pragma unroll
        for (int i = 0; i < 9; i++) C[i] = __ldg(prm.mat + 9 * em[0] + i);
        AtCAx(A, C, u, wdetJ, v);
        uqe[iq] = v[0];
        uqe[Q + iq] = v[1];
        uqe[2 * Q + iq] = v[2];
      }
      if (CURL)
      {
        double C[9], Jd[9], u[3] = {cqe[iq], cqe[Q + iq], cqe[2 * Q + iq]}, v[3];
#pragma unroll
        for (int i = 0; i < 9; i++) C[i] = __ldg(prm.mat + 9 * em[1] + i);
        cofactor33(A, Jd);
        AtCAx(Jd, C, u, wdetJ, v);
        cqe[iq] = v[0];
        cqe[Q + iq] = v[1];
        cqe[2 * Q + iq] = v[2];
      }
    }
  }
  __syncthreads();

  // ---- transpose: test functions; results overwrite U ----
  // x-directed test function (f,0,0): f vx + dz f wy - dy f wz
  if (MASS) contract<2, q, q, q, q, n, false, NEB, NT>(uq + 0 * Q, ES, T2a, ES, sBc, 1, n, 1.0);
  if (CURL)
  {
    if (MASS)
      contract<2, q, q, q, q, n, true, NEB, NT>(cq + 1 * Q, ES, T2a, ES, sGc, 1, n, 1.0);
    else
      contract<2, q, q, q, q, n, false, NEB, NT>(cq + 1 * Q, ES, T2a, ES, sGc, 1, n, 1.0);
    contract<2, q, q, q, q, n, false, NEB, NT>(cq + 2 * Q, ES, T2b, ES, sBc, 1, n, 1.0);
  }
  __syncthreads();
  contract<1, q, q, n, q, n, false, NEB, NT>(T2a, ES, T1a, ES, sBc, 1, n, 1.0);
  if (CURL) contract<1, q, q, n, q, n, true, NEB, NT>(T2b, ES, T1a, ES, sGc, 1, n, -1.0);
  __syncthreads();
  contract<0, q, n, n, q, p, false, NEB, NT>(T1a, ES, U, ES, sBo, 1, p, 1.0);
  __syncthreads();
  // y-directed (0,f,0): f vy - dz f wx + dx f wz
  if (MASS) contract<2, q, q, q, q, n, false, NEB, NT>(uq + 1 * Q, ES, T2a, ES, sBc, 1, n, 1.0);
  if (CURL)
  {
    if (MASS)
      contract<2, q, q, q, q, n, true, NEB, NT>(cq + 0 * Q, ES, T2a, ES, sGc, 1, n, -1.0);
    else
      contract<2, q, q, q, q, n, false, NEB, NT>(cq + 0 * Q, ES, T2a, ES, sGc, 1, n, -1.0);
    contract<2, q, q, q, q, n, false, NEB, NT>(cq + 2 * Q, ES, T2b, ES, sBc, 1, n, 1.0);
  }
  __syncthreads();
  contract<1, q, q, n, q, p, false, NEB, NT>(T2a, ES, T1a, ES, sBo, 1, p, 1.0);
  if (CURL) contract<1, q, q, n, q, p, false, NEB, NT>(T2b, ES, T1b, ES, sBo, 1, p, 1.0);
  __syncthreads();
  contract<0, q, p, n, q, n, false, NEB, NT>(T1a, ES, U + D3, ES, sBc, 1, n, 1.0);
  if (CURL) contract<0, q, p, n, q, n, true, NEB, NT>(T1b, ES, U + D3, ES, sGc, 1, n, 1.0);
  __syncthreads();
  // z-directed (0,0,f): f vz + dy f wx - dx f wy
  if (MASS) contract<2, q, q, q, q, p, false, NEB, NT>(uq + 2 * Q, ES, T2a, ES, sBo, 1, p, 1.0);
  if (CURL)
  {
    contract<2, q, q, q, q, p, false, NEB, NT>(cq + 0 * Q, ES, T2b, ES, sBo, 1, p, 1.0);
    contract<2, q, q, q, q, p, false, NEB, NT>(cq + 1 * Q, ES, T2c, ES, sBo, 1, p, 1.0);
  }
  __syncthreads();
  if (MASS) contract<1, q, q, p, q, n, false, NEB, NT>(T2a, ES, T1a, ES, sBc, 1, n, 1.0);
  if (CURL)
  {
    if (MASS)
      contract<1, q, q, p, q, n, true, NEB, NT>(T2b, ES, T1a, ES, sGc, 1, n, 1.0);
    else
      contract<1, q, q, p, q, n, false, NEB, NT>(T2b, ES, T1a, ES, sGc, 1, n, 1.0);
    contract<1, q, q, p, q, n, false, NEB, NT>(T2c, ES, T1b, ES, sBc, 1, n, 1.0);
  }
  __syncthreads();
  contract<0, q, n, p, q, n, false, NEB, NT>(T1a, ES, U + 2 * D3, ES, sBc, 1, n, 1.0);
  if (CURL) contract<0, q, n, p, q, n, true, NEB, NT>(T1b, ES, U + 2 * D3, ES, sGc, 1, n, -1.0);
  __syncthreads();

  // ---- scatter-add (E^T) ----
  for (int w = threadIdx.x; w < NEB * P; w += NT)
  {
    const int e = w / P, l = w % P;
    if (e0 + e >= prm.ne) continue;
    scatter2(prm.y, prm.sp, prm.lidx[(size_t)(e0 + e) * prm.PS + l], prm.alpha * U[e * ES + l]);
  }
}

// Diagonal: diag[gid(l)] += sum_q  B_l(q)^T D_q B_l(q). Thread per (element, lexicographic dof).
template <int KIND>
__global__ void nd_hex_diag_kernel(NDParams prm, int p, int q, bool assembled)
{
  const int n = p + 1, P = 3 * p * n * n, Q = q * q * q, D3 = p * n * n;
  constexpr bool BLOCK = (KIND == B2P_ND_BLOCK);
  constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS);
  constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS);
  const double *Bo = prm.tab, *Bc = Bo + q * p, *Gc = Bc + q * n;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)prm.ne * P) return;
  const int e = (int)(w / P), l = (int)(w % P);
  const int c = l / D3, r = l % D3;
  int i, j, k;
  if (c == 0) { i = r % p; j = (r / p) % n; k = r / (p * n); }
  else if (c == 1) { i = r % n; j = (r / n) % p; k = r / (n * p); }
  else { i = r % n; j = (r / n) % n; k = r / (n * n); }
  double C0[9], C1[9];
  const int32_t *em = prm.emat + 2 * (size_t)e;
  if (!assembled && !BLOCK)
  {
    for (int t = 0; t < 9; t++)
    {
      C0[t] = MASS ? prm.mat[9 * em[0] + t] : 0.0;
      C1[t] = CURL ? prm.mat[9 * em[1] + t] : 0.0;
    }
  }
  double s = 0.0;
  for (int qz = 0; qz < q; qz++)
    for (int qy = 0; qy < q; qy++)
      for (int qx = 0; qx < q; qx++)
      {
        const int iq = qslot(q, qx, qy, qz);
        // 1-D factors for this dof at this point: value f and the two non-zero curl entries
        double fx, fy, fz, gx, gy, gz;  // value / derivative of the factor along each axis
        fx = (c == 0) ? Bo[qx * p + i] : Bc[qx * n + i];
        fy = (c == 1) ? Bo[qy * p + j] : Bc[qy * n + j];
        fz = (c == 2) ? Bo[qz * p + k] : Bc[qz * n + k];
        gx = (c == 0) ? 0.0 : Gc[qx * n + i];
        gy = (c == 1) ? 0.0 : Gc[qy * n + j];
        gz = (c == 2) ? 0.0 : Gc[qz * n + k];
        double u[3] = {0, 0, 0}, cu[3] = {0, 0, 0};
        u[c] = fx * fy * fz;
        if (c == 0) { cu[1] = fx * fy * gz; cu[2] = -fx * gy * fz; }
        else if (c == 1) { cu[0] = -fx * fy * gz; cu[2] = gx * fy * fz; }
        else { cu[0] = fx * gy * fz; cu[1] = -gx * fy * fz; }
        if (BLOCK)
        {
          // u^T (w A^T (Cm A u + Cx Jd cu)) + cu^T (w Jd^T (Ck Jd cu + Cw A u))
          const double *g = prm.qd + (size_t)e * 10 * Q + iq, *C = prm.bcoef + 36 * (size_t)e;
          double A[9], Jd[9], t[3], sc[3], a[3], b[3], z[3], v[3];
          for (int tt = 0; tt < 9; tt++) A[tt] = g[(1 + tt) * Q];
          cofactor33(A, Jd);
          Ax33(A, u, t);
          Ax33(Jd, cu, sc);
          Ax33(C, t, a);
          Ax33(C + 27, sc, b);
          for (int d = 0; d < 3; d++) z[d] = a[d] + b[d];
          Atx33(A, z, g[0], v);
          s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
          Ax33(C + 9, sc, a);
          Ax33(C + 18, t, b);
          for (int d = 0; d < 3; d++) z[d] = a[d] + b[d];
          Atx33(Jd, z, g[0], v);
          s += cu[0] * v[0] + cu[1] * v[1] + cu[2] * v[2];
        }
        else if (assembled)
        {
          const double *a = prm.aq + (size_t)e * prm.aq_estride + iq;
          if (MASS)
          {
            for (int rr = 0; rr < 3; rr++)
              for (int cc = 0; cc < 3; cc++) s += u[rr] * a[(rr + 3 * cc) * Q] * u[cc];
            a += 9 * Q;
          }
          if (CURL)
            for (int rr = 0; rr < 3; rr++)
              for (int cc = 0; cc < 3; cc++) s += cu[rr] * a[(rr + 3 * cc) * Q] * cu[cc];
        }
        else
        {
          const double *g = prm.qd + (size_t)e * 10 * Q + iq;
          double A[9], v[3];
          for (int t = 0; t < 9; t++) A[t] = g[(1 + t) * Q];
          if (MASS)
          {
            AtCAx(A, C0, u, g[0], v);
            s += u[0] * v[0] + u[1] * v[1] + u[2] * v[2];
          }
          if (CURL)
          {
            double Jd[9];
            cofactor33(A, Jd);
            AtCAx(Jd, C1, cu, g[0], v);
            s += cu[0] * v[0] + cu[1] * v[1] + cu[2] * v[2];
          }
        }
      }
  int gi = prm.lidx[(size_t)e * prm.PS + l];
  if (gi == B2P_SKIP_IDX) return;
  if (gi < 0) gi = -1 - gi;
  atomicAdd(prm.y + gi, s);
}

// Pre-multiplied D per point (BilinearForm::AssembleQuadratureData -> f_build_*_33):
// aq[e][part*9 + t][Q] = w detJ * (A^T C A)[t]  (mass part first, hdivmass_build_33_qf.h:10-52).
template <int KIND>
__global__ void nd_assemble_qdata_kernel(NDParams prm, int Q, double *aq)
{
  constexpr bool MASS = (KIND == B2P_ND_MASS || KIND == B2P_CURLCURL_MASS || KIND == B2P_H1_DIFFUSION);
  constexpr bool CURL = (KIND == B2P_CURLCURL || KIND == B2P_CURLCURL_MASS);
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= (size_t)prm.ne * Q) return;
  const int e = (int)(w / Q), iq = (int)(w % Q);
  const double *g = prm.qd + (size_t)e * 10 * Q + iq;
  const int32_t *em = prm.emat + 2 * (size_t)e;
  double A[9], C[9], S[9];
  for (int t = 0; t < 9; t++) A[t] = g[(1 + t) * Q];
  double *a = aq + (size_t)e * prm.aq_estride + iq;
  if (MASS)
  {
    for (int t = 0; t < 9; t++) C[t] = prm.mat[9 * em[0] + t];
    AtCA(A, C, g[0], S);
    for (int t = 0; t < 9; t++) a[t * Q] = S[t];
    a += 9 * Q;
  }
  if (CURL)
  {
    double Jd[9];
    cofactor33(A, Jd);
    for (int t = 0; t < 9; t++) C[t] = prm.mat[9 * em[1] + t];
    AtCA(Jd, C, g[0], S);
    for (int t = 0; t < 9; t++) a[t * Q] = S[t];
  }
}

NDParams make_params(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg = ApplyRange(),
                     bool transpose = false)
{
  NDParams prm;
  const double *bc = transpose ? op->bcoef_t : op->bcoef;
  prm.bcoef = bc ? bc + 36 * (size_t)rg.e_off : nullptr;
  const int e_off = rg.e_off, e_cnt = rg.e_cnt < 0 ? op->ne - rg.e_off : rg.e_cnt;
  prm.lidx = lidx + (size_t)e_off * op->PS;
  prm.alpha = alpha;
  prm.sp.n_owned = rg.n_owned < 0 ? op->lsize : rg.n_owned;
  prm.sp.xg = rg.xg;
  prm.sp.yg = rg.yg;
  prm.aq_estride = op->aq_estride;
  prm.PS = op->PS;
  prm.tab = op->tab;
  prm.qd = op->geom->qd + (size_t)e_off * 10 * op->geom->Q;
  prm.mat = op->mat;
  prm.emat = op->emat + 2 * (size_t)e_off;
  prm.aq = op->aq ? op->aq + (size_t)e_off * op->aq_estride : nullptr;
  prm.x = x;
  prm.y = y;
  prm.ne = e_cnt;
  return prm;
}

template <int P_, int Q_, int KIND, bool ASM>
int launch_pq(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
              bool transpose = false)
{
  using L = NDLayout<P_, Q_>;
  // elements per block: keep shared memory under ~96 KB and at least 128 threads of work
  constexpr int per_elem_bytes = L::PER_ELEM * 8;
  constexpr int NEB = (per_elem_bytes * 8 <= 100 * 1024) ? 8 : (per_elem_bytes * 4 <= 100 * 1024) ? 4
                      : (per_elem_bytes * 2 <= 200 * 1024) ? 2 : 1;
  constexpr int NT = 256;
  const size_t shmem = (size_t)(Q_ * P_ + 2 * Q_ * (P_ + 1) + NEB * L::PER_ELEM) * sizeof(double);
  auto kern = nd_hex_apply_kernel<P_, Q_, KIND, ASM, NEB, NT>;
  const int ne_run = range_count(op, rg);
  if (ne_run <= 0) return B2P_SUCCESS;
  if (int rc = configure_kernel(op->ctx, kern, shmem)) return rc;
  const int grid = (ne_run + NEB - 1) / NEB;
  B2P_LAUNCH(kern, grid, NT, shmem, s, make_params(op, lidx, alpha, x, y, rg, transpose));
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

template <int P_, int Q_>
int launch_kind(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                bool transpose)
{
  const bool a = op->assembled;
  if (op->bcoef) return launch_pq<P_, Q_, B2P_ND_BLOCK, false>(op, lidx, alpha, x, y, rg, s, transpose);
  switch (op->kind)
  {
    case B2P_CURLCURL:
      return a ? launch_pq<P_, Q_, B2P_CURLCURL, true>(op, lidx, alpha, x, y, rg, s) : launch_pq<P_, Q_, B2P_CURLCURL, false>(op, lidx, alpha, x, y, rg, s);
    case B2P_ND_MASS:
      return a ? launch_pq<P_, Q_, B2P_ND_MASS, true>(op, lidx, alpha, x, y, rg, s) : launch_pq<P_, Q_, B2P_ND_MASS, false>(op, lidx, alpha, x, y, rg, s);
    case B2P_CURLCURL_MASS:
      return a ? launch_pq<P_, Q_, B2P_CURLCURL_MASS, true>(op, lidx, alpha, x, y, rg, s)
               : launch_pq<P_, Q_, B2P_CURLCURL_MASS, false>(op, lidx, alpha, x, y, rg, s);
  }
  set_error(op->ctx, "nd_hex_apply: unsupported kind %d", op->kind);
  return B2P_ERR_UNSUPPORTED;
}

}  // namespace

int launch_nd_hex_apply(b2p_op *op, const int32_t *lidx, double alpha, const double *x, double *y, const ApplyRange &rg, cudaStream_t s,
                        bool transpose)
{
#define B2P_CASE(PP, QQ) \
  if (op->p == PP && op->q1d == QQ) return launch_kind<PP, QQ>(op, lidx, alpha, x, y, rg, s, transpose);
  // (p, q1d): q1d = p+1 for a stand-alone operator; larger q1d for p-coarsened operators that
  // reuse the fine level's quadrature (CeedOperatorCoarsen, libceed/operator.cpp:525-585).
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

int launch_nd_hex_diag(b2p_op *op, double *diag, cudaStream_t s)
{
  NDParams prm = make_params(op, op->lidx, 1.0, nullptr, diag);
  const size_t total = (size_t)op->ne * op->P;
  const int nt = 128;
  const unsigned grid = (unsigned)((total + nt - 1) / nt);
  if (op->bcoef)
  {
    B2P_LAUNCH(nd_hex_diag_kernel<B2P_ND_BLOCK>, grid, nt, 0, s, prm, op->p, op->q1d, false);
    B2P_CUDA(op->ctx, cudaGetLastError());
    return B2P_SUCCESS;
  }
  switch (op->kind)
  {
    case B2P_CURLCURL: B2P_LAUNCH(nd_hex_diag_kernel<B2P_CURLCURL>, grid, nt, 0, s, prm, op->p, op->q1d, op->assembled); break;
    case B2P_ND_MASS: B2P_LAUNCH(nd_hex_diag_kernel<B2P_ND_MASS>, grid, nt, 0, s, prm, op->p, op->q1d, op->assembled); break;
    case B2P_CURLCURL_MASS:
      B2P_LAUNCH(nd_hex_diag_kernel<B2P_CURLCURL_MASS>, grid, nt, 0, s, prm, op->p, op->q1d, op->assembled);
      break;
    default: set_error(op->ctx, "nd_hex_diag: unsupported kind %d", op->kind); return B2P_ERR_UNSUPPORTED;
  }
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

int launch_assemble_qdata(b2p_op *op, cudaStream_t s)
{
  NDParams prm = make_params(op, op->lidx, 1.0, nullptr, nullptr);
  const int Q = op->geom->Q;
  const size_t total = (size_t)op->ne * Q;
  const int nt = 128;
  const unsigned grid = (unsigned)((total + nt - 1) / nt);
  switch (op->kind)
  {
    case B2P_CURLCURL: B2P_LAUNCH(nd_assemble_qdata_kernel<B2P_CURLCURL>, grid, nt, 0, s, prm, Q, op->aq); break;
    case B2P_ND_MASS: B2P_LAUNCH(nd_assemble_qdata_kernel<B2P_ND_MASS>, grid, nt, 0, s, prm, Q, op->aq); break;
    case B2P_CURLCURL_MASS: B2P_LAUNCH(nd_assemble_qdata_kernel<B2P_CURLCURL_MASS>, grid, nt, 0, s, prm, Q, op->aq); break;
    case B2P_H1_DIFFUSION: B2P_LAUNCH(nd_assemble_qdata_kernel<B2P_H1_DIFFUSION>, grid, nt, 0, s, prm, Q, op->aq); break;
    default: set_error(op->ctx, "assemble_qdata: unsupported kind %d", op->kind); return B2P_ERR_UNSUPPORTED;
  }
  B2P_CUDA(op->ctx, cudaGetLastError());
  return B2P_SUCCESS;
}

}  // namespace b2p
