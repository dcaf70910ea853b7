// Horn's quaternion solve of a weighted rigid superposition from its 17 one-pass sums, shared by the alignment kernels
// (align.cu: one pair list per job; best_align.cu: the best of a job's atom mappings). Both must give the same bits for
// the same sums, so there is one copy of the Jacobi sweep and the solve.
#pragma once

#include <cmath>

namespace b200 {
namespace horn {

__device__ __forceinline__ double warpSum(double v) {  // butterfly: every lane ends with the same bits
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// a[i][j] and a[k][l] of the upper triangle after the plane rotation (s, tau)
__device__ __forceinline__ void rot(double& x, double& y, double s, double tau) {
  const double g = x, h = y;
  x = g - s * (h + g * tau);
  y = h + s * (g - h * tau);
}

// Cyclic Jacobi on the symmetric 4x4 matrix a (upper triangle used, destroyed), at most maxIters sweeps: eigenvalue
// estimates d and eigenvectors in the columns of v. Every index is a compile-time constant, so a, d and v stay in
// registers.
__device__ __forceinline__ void jacobi4(double (&a)[4][4], double (&d)[4], double (&v)[4][4], int maxIters) {
  double b[4], z[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    b[i] = d[i] = a[i][i];
    z[i] = 0.0;
  }
  for (int it = 1; it <= maxIters; ++it) {
    double sm = 0.0;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) sm += fabs(a[p][q]);
    if (sm == 0.0) break;
    const double tresh = it < 4 ? 0.2 * sm / 16.0 : 0.0;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        const double g = 100.0 * fabs(a[p][q]);
        if (it > 4 && fabs(d[p]) + g == fabs(d[p]) && fabs(d[q]) + g == fabs(d[q])) {
          a[p][q] = 0.0;
        } else if (fabs(a[p][q]) > tresh) {
          double       h = d[q] - d[p], t;
          if (fabs(h) + g == fabs(h)) {
            t = a[p][q] / h;
          } else {
            const double theta = 0.5 * h / a[p][q];
            t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
            if (theta < 0.0) t = -t;
          }
          const double c = 1.0 / sqrt(1.0 + t * t), s = t * c, tau = s / (1.0 + c);
          h = t * a[p][q];
          z[p] -= h;
          z[q] += h;
          d[p] -= h;
          d[q] += h;
          a[p][q] = 0.0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j < p) rot(a[j][p], a[j][q], s, tau);
            else if (j > p && j < q) rot(a[p][j], a[j][q], s, tau);
            else if (j > q) rot(a[p][j], a[q][j], s, tau);
            rot(v[j][p], v[j][q], s, tau);
          }
        }
      }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      b[i] += z[i];
      d[i] = b[i];
      z[i] = 0.0;
    }
  }
}

constexpr int kSums = 17;  // W, sum w dp (3), sum w dr (3), sum w (|dp|^2 + |dr|^2), sum w dp dr^T (9, row-major)

// Adds one pair's terms to the 17 sums: w, w dp, w dr, w (|dp|^2 + |dr|^2) and w dp dr^T, in this order.
__device__ __forceinline__ void accumulate(double (&x)[kSums], double w, const double (&dp)[3], const double (&dr)[3]) {
  x[0] += w;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    x[1 + c] += w * dp[c];
    x[4 + c] += w * dr[c];
  }
  x[7] += w * (dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2] + dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) x[8 + 3 * r + c] += w * dp[r] * dr[c];
}

// From a job's 17 sums: R (row-major), the reflected probe centroid offset cp and the reference centroid offset cr
// (relative to the shifts), and the RMSD.
__device__ __forceinline__ double solve(const double (&x)[kSums], int L, int maxIters, double (&R)[9], double (&cp)[3],
                                        double (&cr)[3]) {
  const double W = x[0], iw = 1.0 / W;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    cp[k] = x[1 + k] * iw;
    cr[k] = x[4 + k] * iw;
  }
  const double G = x[7] - (x[1] * cp[0] + x[2] * cp[1] + x[3] * cp[2]) - (x[4] * cr[0] + x[5] * cr[1] + x[6] * cr[2]);
  double       S[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) S[r][c] = x[8 + 3 * r + c] - x[1 + r] * cr[c];
  double N[4][4];
  N[0][0] = S[0][0] + S[1][1] + S[2][2];
  N[0][1] = S[1][2] - S[2][1];
  N[0][2] = S[2][0] - S[0][2];
  N[0][3] = S[0][1] - S[1][0];
  N[1][1] = S[0][0] - S[1][1] - S[2][2];
  N[1][2] = S[0][1] + S[1][0];
  N[1][3] = S[2][0] + S[0][2];
  N[2][2] = -S[0][0] + S[1][1] - S[2][2];
  N[2][3] = S[1][2] + S[2][1];
  N[3][3] = -S[0][0] - S[1][1] + S[2][2];
  N[1][0] = N[2][0] = N[3][0] = N[2][1] = N[3][1] = N[3][2] = 0.0;  // unused lower triangle
  double d[4], v[4][4];
  jacobi4(N, d, v, maxIters);
  int    top = 0;  // the first of equal largest values: N = 0 gives q = (1, 0, 0, 0), R = I
  double lam = d[0];
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (d[i] > lam) lam = d[i], top = i;
  double q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = top == 0 ? v[i][0] : top == 1 ? v[i][1] : top == 2 ? v[i][2] : v[i][3];
  const double qn = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] *= qn;
  R[0] = q[0] * q[0] + q[1] * q[1] - q[2] * q[2] - q[3] * q[3];
  R[1] = 2.0 * (q[1] * q[2] - q[0] * q[3]);
  R[2] = 2.0 * (q[1] * q[3] + q[0] * q[2]);
  R[3] = 2.0 * (q[1] * q[2] + q[0] * q[3]);
  R[4] = q[0] * q[0] - q[1] * q[1] + q[2] * q[2] - q[3] * q[3];
  R[5] = 2.0 * (q[2] * q[3] - q[0] * q[1]);
  R[6] = 2.0 * (q[1] * q[3] - q[0] * q[2]);
  R[7] = 2.0 * (q[2] * q[3] + q[0] * q[1]);
  R[8] = q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3];
  return sqrt(fmax(G - 2.0 * lam, 0.0) / L);
}

}  // namespace horn
}  // namespace b200
