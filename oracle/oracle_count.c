/*
 * oracle_count.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of the count-vector
 * similarity calls (nvmolkit_b200/csrc: b200mol_count_cross, _topk, _threshold) in tests/ and __graft_entry__.smoke().
 * Nothing under nvmolkit_b200/ may import, link or call this.
 *
 * Rows are int32 count vectors of `bins` bins. With a = the sum of row i of A (group one), b = the sum of row j of B and
 * c = sum over bins of min(A[i][k], B[j][k]) (exact 64-bit integers), the value of the pair is
 *   0                                         if c == 0
 *   c / ((alpha (a - c) + beta (b - c)) + c)  otherwise,
 * each product, sum and the quotient one fp64 operation rounded to nearest, in exactly this order (the Makefile builds
 * with -ffp-contract=off). Tanimoto is (1, 1), Dice (0.5, 0.5). OpenMP over rows. Top-k and threshold are derived from
 * this matrix in NumPy (oracle/count.py), pinned by tests/test_count_similarity.py to RDKit's literal expressions.
 */
#include <stdint.h>
#include <stdlib.h>

static double tversky_counts(long long c, long long a, long long b, double alpha, double beta) {
  if (c == 0) return 0.0;
  const double d1 = alpha * (double)(a - c);
  const double d2 = beta * (double)(b - c);
  const double d  = (d1 + d2) + (double)c;
  return (double)c / d;
}

static long long* row_sums(const int32_t* X, long n, int bins) {
  long long* s = (long long*)malloc(sizeof(long long) * (n > 0 ? n : 1));
  for (long i = 0; i < n; ++i) {
    long long t = 0;
    for (int k = 0; k < bins; ++k) t += X[i * bins + k];
    s[i] = t;
  }
  return s;
}

void oracle_count_cross(const int32_t* A, long nA, const int32_t* B, long nB, int bins, double alpha, double beta,
                        double* out) {
  long long* sa = row_sums(A, nA, bins);
  long long* sb = row_sums(B, nB, bins);
#pragma omp parallel for schedule(dynamic, 4)
  for (long i = 0; i < nA; ++i) {
    const int32_t* x = A + i * bins;
    for (long j = 0; j < nB; ++j) {
      const int32_t* y = B + j * bins;
      long long      c = 0;
      for (int k = 0; k < bins; ++k) c += x[k] < y[k] ? x[k] : y[k];
      out[i * nB + j] = tversky_counts(c, sa[i], sb[j], alpha, beta);
    }
  }
  free(sa);
  free(sb);
}
