/*
 * oracle_align.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). RDKit's AlignPoints (Numerics/Alignment), restated on the
 * CPU in fp64 for one probe / reference pair list: weighted centroids, the weighted covariance, Horn's 4x4 quaternion
 * matrix, its eigenvectors by the Numerical Recipes cyclic Jacobi capped at maxIters sweeps, the quaternion of the largest
 * eigenvalue estimate as a rotation, the mirror image when reflect is set, and the 4x4 transform; then the transform
 * applied to every atom of a conformer (MolTransforms::transformConformer).
 *
 * Where the product departs from RDKit for accuracy it is checked against a different route here: RDKit forms raw
 * one-pass sums, the product forms one-pass sums of coordinates shifted by the first pair (csrc/align.cu), and this file
 * forms the centroids first and then sums the centred coordinates (two passes), which is accurate at any offset.
 */
#include <math.h>
#include <stdint.h>

static void rot(double* x, double* y, double s, double tau) {
  const double g = *x, h = *y;
  *x = g - s * (h + g * tau);
  *y = h + s * (g - h * tau);
}

/* eigenvalue estimates d and eigenvectors (columns of v) of the symmetric a (upper triangle, destroyed) */
static void jacobi4(double a[4][4], double d[4], double v[4][4], int maxIters) {
  double b[4], z[4];
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < 4; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    b[i] = d[i] = a[i][i];
    z[i] = 0.0;
  }
  for (int it = 1; it <= maxIters; ++it) {
    double sm = 0.0;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) sm += fabs(a[p][q]);
    if (sm == 0.0) return;
    const double tresh = it < 4 ? 0.2 * sm / 16.0 : 0.0;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) {
        const double g = 100.0 * fabs(a[p][q]);
        if (it > 4 && fabs(d[p]) + g == fabs(d[p]) && fabs(d[q]) + g == fabs(d[q])) {
          a[p][q] = 0.0;
          continue;
        }
        if (fabs(a[p][q]) <= tresh) continue;
        double h = d[q] - d[p], t;
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
        for (int j = 0; j < p; ++j) rot(&a[j][p], &a[j][q], s, tau);
        for (int j = p + 1; j < q; ++j) rot(&a[p][j], &a[j][q], s, tau);
        for (int j = q + 1; j < 4; ++j) rot(&a[p][j], &a[q][j], s, tau);
        for (int j = 0; j < 4; ++j) rot(&v[j][p], &v[j][q], s, tau);
      }
    for (int i = 0; i < 4; ++i) {
      b[i] += z[i];
      d[i] = b[i];
      z[i] = 0.0;
    }
  }
}

/* Align probe atoms prb[pairs[2 i]] onto reference atoms ref[pairs[2 i + 1]], i < L, with weights w (NULL = 1).
 * Returns the RMSD sqrt(max(0, SSR) / L); T (16 doubles, row-major) receives [[+-R, t], [0 0 0 1]]. */
double oracle_align(const double* prb, const double* ref, const int32_t* pairs, const double* w, int L, int reflect,
                    int maxIters, double* T) {
  const double sg = reflect ? -1.0 : 1.0;
  double       W = 0.0, pb[3] = {0, 0, 0}, rb[3] = {0, 0, 0};
  for (int i = 0; i < L; ++i) {
    const double wi = w ? w[i] : 1.0;
    W += wi;
    for (int k = 0; k < 3; ++k) {
      pb[k] += wi * sg * prb[3 * pairs[2 * i] + k];
      rb[k] += wi * ref[3 * pairs[2 * i + 1] + k];
    }
  }
  for (int k = 0; k < 3; ++k) pb[k] /= W, rb[k] /= W;
  double S[3][3] = {{0}}, G = 0.0;
  for (int i = 0; i < L; ++i) {
    const double wi = w ? w[i] : 1.0;
    double       x[3], y[3];
    for (int k = 0; k < 3; ++k) {
      x[k] = sg * prb[3 * pairs[2 * i] + k] - pb[k];
      y[k] = ref[3 * pairs[2 * i + 1] + k] - rb[k];
      G += wi * (x[k] * x[k] + y[k] * y[k]);
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) S[r][c] += wi * x[r] * y[c];
  }
  double N[4][4] = {
    {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0]},
    {0.0, S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2]},
    {0.0, 0.0, -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1]},
    {0.0, 0.0, 0.0, -S[0][0] - S[1][1] + S[2][2]}};
  double d[4], v[4][4];
  jacobi4(N, d, v, maxIters);
  int top = 0;
  for (int i = 1; i < 4; ++i)
    if (d[i] > d[top]) top = i;
  double q[4], n2 = 0.0;
  for (int i = 0; i < 4; ++i) q[i] = v[i][top], n2 += q[i] * q[i];
  for (int i = 0; i < 4; ++i) q[i] /= sqrt(n2);
  const double R[3][3] = {
    {q[0] * q[0] + q[1] * q[1] - q[2] * q[2] - q[3] * q[3], 2.0 * (q[1] * q[2] - q[0] * q[3]), 2.0 * (q[1] * q[3] + q[0] * q[2])},
    {2.0 * (q[1] * q[2] + q[0] * q[3]), q[0] * q[0] - q[1] * q[1] + q[2] * q[2] - q[3] * q[3], 2.0 * (q[2] * q[3] - q[0] * q[1])},
    {2.0 * (q[1] * q[3] - q[0] * q[2]), 2.0 * (q[2] * q[3] + q[0] * q[1]), q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3]}};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * r + c] = sg * R[r][c];
    T[4 * r + 3] = rb[r] - (R[r][0] * pb[0] + R[r][1] * pb[1] + R[r][2] * pb[2]);
  }
  T[12] = T[13] = T[14] = 0.0;
  T[15] = 1.0;
  const double ssr = G - 2.0 * d[top];
  return sqrt((ssr > 0.0 ? ssr : 0.0) / L);
}

/* xyz[n][3] <- T xyz (row-major 4x4 acting on column vectors) */
void oracle_apply_transform(const double* T, double* xyz, int n) {
  for (int a = 0; a < n; ++a) {
    const double x = xyz[3 * a], y = xyz[3 * a + 1], z = xyz[3 * a + 2];
    for (int r = 0; r < 3; ++r) xyz[3 * a + r] = T[4 * r] * x + T[4 * r + 1] * y + T[4 * r + 2] * z + T[4 * r + 3];
  }
}
