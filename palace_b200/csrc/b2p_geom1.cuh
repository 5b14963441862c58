// Geometry factors of a trilinear (mesh order 1) hexahedron at a tensor quadrature point, from its 8 vertices: the one definition
// of J behind the stored q-data of order-1 meshes (geom_hex_kernel) and the element kernels that evaluate the geometry in place
// (nd_hex_apply6_kernel on node geometry). Both routes form J from the same line sums; the stored route divides by detJ per entry,
// the vertex route scales the finished quadrature-point operator once by w / detJ, so the two agree to rounding, not bit for bit.
//   x[c * 8 + i + 2 (j + 2 k)]: vertex coordinates (b2p_geom::xe); B[q][2], G[q][2]: the linear nodal basis and its derivative
//   at the 1-D quadrature points; w: the 1-D quadrature weights.
// Along a line of fixed (qy, qz) every column of J is a two-term combination in the qx tables: hex1_line forms the 18 line sums
// once, hex1_jacobian J, K = cof(J) = detJ J^-T and detJ at a point, hex1_point the stored q-data on top of it -- w detJ and
// A = K / detJ, as q-data component 0 and components 1 ... 9.
#pragma once
#include "b2p_qf.cuh"

namespace b2p
{

struct Hex1Line
{
  double s[3][2], t[3][2], u[3][2];  // [c][i]: sum over (j, k) of x[c][i][j][k] times B_y B_z, G_y B_z, B_y G_z
};

__device__ __forceinline__ void hex1_line(const double *x, const double By[2], const double Gy[2], const double Bz[2], const double Gz[2],
                                          Hex1Line &L)
{
  double byz[4], gyz[4], bgz[4];  // (j, k) at j + 2 k
#pragma unroll
  for (int k = 0; k < 2; k++)
#pragma unroll
    for (int j = 0; j < 2; j++)
    {
      byz[j + 2 * k] = By[j] * Bz[k];
      gyz[j + 2 * k] = Gy[j] * Bz[k];
      bgz[j + 2 * k] = By[j] * Gz[k];
    }
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int i = 0; i < 2; i++)
    {
      double s = 0.0, t = 0.0, u = 0.0;
#pragma unroll
      for (int jk = 0; jk < 4; jk++)
      {
        const double v = x[c * 8 + i + 2 * jk];
        s += byz[jk] * v;
        t += gyz[jk] * v;
        u += bgz[jk] * v;
      }
      L.s[c][i] = s;
      L.t[c][i] = t;
      L.u[c][i] = u;
    }
}

// J, K = cof(J) = adj(J)^T (column-major) and detJ at point qx of the line. Column 0 (d/dxi_x) depends on qx only through Gx,
// which is the same at every point for the linear basis.
__device__ __forceinline__ void hex1_jacobian(const Hex1Line &L, const double Bx[2], const double Gx[2], double J[9], double K[9],
                                              double &detJ)
{
#pragma unroll
  for (int c = 0; c < 3; c++)
  {
    J[c + 0] = Gx[0] * L.s[c][0] + Gx[1] * L.s[c][1];
    J[c + 3] = Bx[0] * L.t[c][0] + Bx[1] * L.t[c][1];
    J[c + 6] = Bx[0] * L.u[c][0] + Bx[1] * L.u[c][1];
  }
  cofactor33(J, K);
  detJ = J[0] * K[0] + J[1] * K[1] + J[2] * K[2];
}

// wdetJ = w_x w_y w_z detJ, A = adj(J)^T / detJ (column-major) at point qx of the line
__device__ __forceinline__ void hex1_point(const Hex1Line &L, const double Bx[2], const double Gx[2], double wx, double wy, double wz,
                                           double &wdetJ, double A[9])
{
  double J[9], adj[9], detJ;
  hex1_jacobian(L, Bx, Gx, J, adj, detJ);
  const double r = 1.0 / detJ;
  wdetJ = wx * wy * wz * detJ;
#pragma unroll
  for (int t = 0; t < 9; t++) A[t] = adj[t] * r;
}

// The element kernel's per-point form of the same J. For a Lagrange basis through two nodes B_0 = 1 - B_1, so along the line
// columns 1 and 2 of J are a + B_1(xi_x) d with a = t[c][0], d = t[c][1] - t[c][0] (u likewise). hex1_kline forms those and
// column 0 once per line from hex1_line's sums, which it shares with the stored route; hex1_kjacobian then forms J, K = cof(J)
// and detJ at a point with one FMA per entry of columns 1 and 2 (hex1_jacobian: a product and an FMA). Agrees with
// hex1_jacobian to rounding.
struct Hex1KLine
{
  double j0[3], a1[3], d1[3], a2[3], d2[3];  // [c]: J[c] = j0, J[c + 3] = a1 + B_1 d1, J[c + 6] = a2 + B_1 d2
};

__device__ __forceinline__ void hex1_kline(const Hex1Line &L, const double Gx[2], Hex1KLine &K)
{
#pragma unroll
  for (int c = 0; c < 3; c++)
  {
    K.j0[c] = Gx[0] * L.s[c][0] + Gx[1] * L.s[c][1];
    K.a1[c] = L.t[c][0];
    K.d1[c] = L.t[c][1] - L.t[c][0];
    K.a2[c] = L.u[c][0];
    K.d2[c] = L.u[c][1] - L.u[c][0];
  }
}

__device__ __forceinline__ void hex1_kjacobian(const Hex1KLine &L, double b1, double J[9], double K[9], double &detJ)
{
#pragma unroll
  for (int c = 0; c < 3; c++)
  {
    J[c + 0] = L.j0[c];
    J[c + 3] = fma(b1, L.d1[c], L.a1[c]);
    J[c + 6] = fma(b1, L.d2[c], L.a2[c]);
  }
  cofactor33(J, K);
  detJ = J[0] * K[0] + J[1] * K[1] + J[2] * K[2];
}

}  // namespace b2p
