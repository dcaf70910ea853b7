/*
 * oracle_dg.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). Bounds-matrix triangle smoothing, power-iteration
 * eigensolver, metric-matrix coordinate generation, on the CPU in fp64.
 *
 * Follows (nvMolKit v0.5.0 checkout): src/triangle_smooth.cu:27-129 (one relaxation per pivot k; identical to RDKit
 * DistGeom::triangleSmoothBounds, which the reference's tests compare against, tests/test_triangle_smooth.cu:182-367);
 * src/symmetric_eigensolver.cu:62-192 (port of RDKit PowerEigenSolver: largest-|z| element as eigenvalue estimate,
 * tolerance 1e-3, <= 1000 iterations, deflation); src/forcefields/coord_gen.cu:55-127 (sqrt of eigenvalues,
 * coordinates = sqrt(lambda_j) v_j[i]). The metric matrix from a distance matrix is RDKit's
 * DistGeom::computeInitialCoords (un-vendored RDKit, Code/DistGeom/DistGeomUtils.cpp; published algorithm restated).
 * Pinned by the reference's eigenvalue known answers (tests/test_coordgen.cu:98-135) in tests/test_oracle_golden.py.
 *
 * Bounds matrix layout (RDKit BoundsMatrix): n x n row-major, upper triangle (i<j) = upper bounds, lower triangle
 * (i>j: element [j][i] for the pair i<j) = lower bounds.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* Returns 1 when the bounds are consistent, 0 when smoothing found lb > ub (matrix left partially smoothed). */
int oracle_triangle_smooth(double* b, int n, double tol) {
  for (int k = 0; k < n; ++k) {
    for (int i = 0; i < n - 1; ++i) {
      if (i == k) continue;
      const int    ii = i < k ? i : k, ik = i < k ? k : i;
      const double Uik = b[ii * n + ik], Lik = b[ik * n + ii];
      for (int j = i + 1; j < n; ++j) {
        if (j == k) continue;
        const int    jj = j < k ? j : k, jk = j < k ? k : j;
        const double Ukj = b[jj * n + jk], Ljk = b[jk * n + jj];
        const double sumU = Uik + Ukj, d1 = Lik - Ukj, d2 = Ljk - Uik;
        if (b[i * n + j] > sumU) b[i * n + j] = sumU;
        if (b[j * n + i] < d1) b[j * n + i] = d1;
        else if (b[j * n + i] < d2) b[j * n + i] = d2;
        const double lB = b[j * n + i], uB = b[i * n + j];
        if (tol > 0.0 && (lB - uB) > 0.0 && (lB - uB) / lB < tol) b[i * n + j] = lB;
        else if (lB - uB > 0.0) return 0;
      }
    }
  }
  return 1;
}

/* Top-numEigs eigenpairs of the symmetric n x n matrix `m` (destroyed by deflation). v0[numEigs*n] = start vectors.
 * eigvals[numEigs], eigvecs[numEigs*n] (row e = eigenvector e). Returns the number of eigenpairs that converged.
 * The trace arrays (numEigs each, or NULL) describe every eigenpair attempted, the failed last one included:
 * iters[e] = power iterations run; convMargin[e] = min over iterations of | |eig - prev| - 1e-3 |, zeroMargin[e] = min of
 * | |eig| - 1e-10 |, i.e. how close each stopping decision came to going the other way. */
int oracle_power_eigen_trace(double* m, int n, int numEigs, const double* v0, double* eigvals, double* eigvecs, int* iters,
                             double* convMargin, double* zeroMargin) {
  double* v = (double*)malloc(sizeof(double) * n);
  double* z = (double*)malloc(sizeof(double) * n);
  int     done = 0;
  for (int e = 0; e < numEigs; ++e) {
    double norm = 0.0;
    for (int i = 0; i < n; ++i) norm += v0[e * n + i] * v0[e * n + i];
    norm = sqrt(norm);
    for (int i = 0; i < n; ++i) v[i] = v0[e * n + i] / norm;
    double eig = -1000.0, cm = INFINITY, zm = INFINITY;
    int    converged = 0, it = 0;
    while (it < 1000) {
      ++it;
      const double prev = eig;
      for (int i = 0; i < n; ++i) {
        double a = 0.0;
        for (int j = 0; j < n; ++j) a += m[i * n + j] * v[j];
        z[i] = a;
      }
      eig = z[0];
      for (int i = 1; i < n; ++i)
        if (fabs(z[i]) > fabs(eig)) eig = z[i];
      zm = fmin(zm, fabs(fabs(eig) - 1.0e-10));
      if (fabs(eig) < 1.0e-10) break;
      for (int i = 0; i < n; ++i) v[i] = z[i] / eig;
      cm = fmin(cm, fabs(fabs(eig - prev) - 0.001));
      if (fabs(eig - prev) < 0.001) {
        converged = 1;
        break;
      }
    }
    if (iters) iters[e] = it;
    if (convMargin) convMargin[e] = cm;
    if (zeroMargin) zeroMargin[e] = zm;
    if (!converged) break;
    norm = 0.0;
    for (int i = 0; i < n; ++i) norm += v[i] * v[i];
    norm = sqrt(norm);
    for (int i = 0; i < n; ++i) {
      v[i] /= norm;
      eigvecs[e * n + i] = v[i];
    }
    eigvals[e] = eig;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) m[i * n + j] -= eig * v[i] * v[j];
    ++done;
  }
  free(v);
  free(z);
  return done;
}

int oracle_power_eigen(double* m, int n, int numEigs, const double* v0, double* eigvals, double* eigvecs) {
  return oracle_power_eigen_trace(m, n, numEigs, v0, eigvals, eigvecs, NULL, NULL, NULL);
}

/* dist[n*n] symmetric distances -> metric matrix T (n*n), RDKit computeInitialCoords. */
void oracle_metric_matrix(const double* dist, int n, double* T) {
  double* sq0 = (double*)calloc(n, sizeof(double));
  double  sumSq = 0.0;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) {
      const double d2 = dist[i * n + j] * dist[i * n + j];
      sq0[i] += d2;
      sumSq += d2;
    }
  sumSq /= (double)n * n * 2.0; /* sum over unordered pairs / n^2 */
  for (int i = 0; i < n; ++i) sq0[i] = sq0[i] / n - sumSq;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) T[i * n + j] = 0.5 * (sq0[i] + sq0[j] - dist[i * n + j] * dist[i * n + j]);
  free(sq0);
}

/* coords[n*dim] = sqrt(eigval_j) * eigvec_j[i]; returns 0 if an eigenvalue is not positive (embedding failed). */
int oracle_coords_from_eigen(const double* eigvals, const double* eigvecs, int n, int dim, double* coords) {
  for (int j = 0; j < dim; ++j)
    if (!(eigvals[j] > 0.0)) return 0;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < dim; ++j) coords[i * dim + j] = sqrt(eigvals[j]) * eigvecs[j * n + i];
  return 1;
}
