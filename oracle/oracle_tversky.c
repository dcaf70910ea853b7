/*
 * oracle_tversky.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of the Dice / Tversky
 * similarity calls (nvmolkit_b200/csrc: b200mol_tversky_cross, _cross_host, _topk, _threshold) in tests/ and
 * __graft_entry__.smoke(). Nothing under nvmolkit_b200/ may import, link or call this.
 *
 * The value of a pair with popcounts a (row, group one), b and intersection c is
 *   0                                         if c == 0
 *   c / ((alpha (a - c) + beta (b - c)) + c)  otherwise,
 * each product, sum and the quotient one fp64 operation rounded to nearest, in exactly this order (the Makefile builds
 * with -ffp-contract=off, so nothing becomes an FMA). Dice is (0.5, 0.5). Exact integer popcounts, OpenMP over rows:
 * the matrix, the top-k (first k columns of each row by value descending, column ascending) and the threshold CSR
 * (columns with value >= t, ascending), the latter two without the matrix. Pinned by tests/test_tversky.py to a NumPy
 * restatement of the same expression, to np.lexsort and to np.nonzero over the matrix.
 */
#include <stdint.h>
#include <stdlib.h>

static inline int popc32(uint32_t v) { return __builtin_popcount(v); }

static int popcount_row(const uint32_t* r, int words) {
  int s = 0;
  for (int w = 0; w < words; ++w) s += popc32(r[w]);
  return s;
}

static int and_count(const uint32_t* x, const uint32_t* y, int words) {
  int c = 0;
  for (int w = 0; w < words; ++w) c += popc32(x[w] & y[w]);
  return c;
}

static double tversky(int c, int a, int b, double alpha, double beta) {
  if (c == 0) return 0.0;
  const double d1 = alpha * (double)(a - c);
  const double d2 = beta * (double)(b - c);
  const double d  = (d1 + d2) + (double)c;
  return (double)c / d;
}

static int* popcounts(const uint32_t* B, long n, int words) {
  int* p = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
  for (long j = 0; j < n; ++j) p[j] = popcount_row(B + j * words, words);
  return p;
}

void oracle_tversky_cross(const uint32_t* A, long nA, const uint32_t* B, long nB, int words, double alpha, double beta,
                          double* out) {
  int* pb = popcounts(B, nB, words);
#pragma omp parallel for schedule(dynamic, 4)
  for (long i = 0; i < nA; ++i) {
    const uint32_t* ai = A + i * words;
    const int       pa = popcount_row(ai, words);
    for (long j = 0; j < nB; ++j) out[i * nB + j] = tversky(and_count(ai, B + j * words, words), pa, pb[j], alpha, beta);
  }
  free(pb);
}

/* Partial selection as oracle_topk: a column enters the sorted list of k only if it beats the last entry (columns come
 * in ascending order, so ties keep the lowest index). */
void oracle_tversky_topk(const uint32_t* Q, long nQ, const uint32_t* B, long nB, int words, double alpha, double beta, int k,
                         double* values, int32_t* indices) {
  int* pb = popcounts(B, nB, words);
#pragma omp parallel for schedule(dynamic, 1)
  for (long i = 0; i < nQ; ++i) {
    double*         v  = values + i * k;
    int32_t*        ix = indices + i * k;
    const uint32_t* qi = Q + i * words;
    const int       pa = popcount_row(qi, words);
    int             n  = 0;
    for (long j = 0; j < nB; ++j) {
      const double s = tversky(and_count(qi, B + j * words, words), pa, pb[j], alpha, beta);
      if (n == k && !(s > v[k - 1])) continue;
      int at = n < k ? n++ : k - 1;
      while (at > 0 && s > v[at - 1]) {
        v[at]  = v[at - 1];
        ix[at] = ix[at - 1];
        --at;
      }
      v[at]  = s;
      ix[at] = (int32_t)j;
    }
  }
  free(pb);
}

/* As oracle_threshold: indices = NULL counts only (indptr[nQ + 1] is always written); returns nnz. */
long oracle_tversky_threshold(const uint32_t* Q, long nQ, const uint32_t* B, long nB, int words, double alpha, double beta,
                              double t, int64_t* indptr, int32_t* indices, double* values) {
  int* pb = popcounts(B, nB, words);
  indptr[0] = 0;
#pragma omp parallel for schedule(dynamic, 4)
  for (long i = 0; i < nQ; ++i) {
    const uint32_t* qi = Q + i * words;
    const int       pa = popcount_row(qi, words);
    long            n  = 0;
    for (long j = 0; j < nB; ++j)
      if (tversky(and_count(qi, B + j * words, words), pa, pb[j], alpha, beta) >= t) ++n;
    indptr[i + 1] = n;
  }
  for (long i = 0; i < nQ; ++i) indptr[i + 1] += indptr[i];
  if (indices) {
#pragma omp parallel for schedule(dynamic, 4)
    for (long i = 0; i < nQ; ++i) {
      const uint32_t* qi = Q + i * words;
      const int       pa = popcount_row(qi, words);
      int64_t         at = indptr[i];
      for (long j = 0; j < nB; ++j) {
        const double s = tversky(and_count(qi, B + j * words, words), pa, pb[j], alpha, beta);
        if (s >= t) {
          indices[at] = (int32_t)j;
          values[at]  = s;
          ++at;
        }
      }
    }
  }
  free(pb);
  return (long)indptr[nQ];
}
