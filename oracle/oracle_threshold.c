/*
 * oracle_threshold.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of the threshold similarity
 * search (nvmolkit_b200/csrc/threshold.cu) in tests/ and __graft_entry__.smoke(). Nothing under nvmolkit_b200/ may import,
 * link or call this.
 *
 * Row i of the CSR result lists, in ascending order, the columns j whose entry of oracle_similarity_cross's matrix
 * (oracle_fp.c) is >= t, with that value: exact integer popcounts and the same fp64 expression (0 when the intersection
 * is empty, else one divide), without the matrix. Two row-parallel OpenMP scans: one counts each row's entries (indptr by
 * a prefix sum), the other writes them. Pinned by tests/test_threshold.py to np.nonzero over oracle_similarity_cross.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static inline int popc32(uint32_t v) { return __builtin_popcount(v); }

/* as sim_from_counts of oracle_fp.c; metric 0 = Tanimoto, 1 = cosine */
static double sim_from_counts(int c, int a, int b, int metric) {
  if (c == 0) return 0.0;
  if (metric == 0) return (double)c / (double)(a + b - c);
  return (double)c / sqrt((double)a * (double)b);
}

static int popcount_row(const uint32_t* r, int words) {
  int s = 0;
  for (int w = 0; w < words; ++w) s += popc32(r[w]);
  return s;
}

/* Pass indices = NULL to count only: indptr[nQ + 1] is always written; returns nnz. With indices / values (room for
 * nnz, as the counting call returned), the entries are written too. */
long oracle_threshold(const uint32_t* Q, long nQ, const uint32_t* B, long nB, int words, int metric, double t, int64_t* indptr,
                      int32_t* indices, double* values) {
  int* pb = (int*)malloc(sizeof(int) * (nB > 0 ? nB : 1));
  for (long j = 0; j < nB; ++j) pb[j] = popcount_row(B + j * words, words);
  indptr[0] = 0;
#pragma omp parallel for schedule(dynamic, 4)
  for (long i = 0; i < nQ; ++i) {
    const uint32_t* qi = Q + i * words;
    const int       pa = popcount_row(qi, words);
    long            n  = 0;
    for (long j = 0; j < nB; ++j) {
      int c = 0;
      for (int w = 0; w < words; ++w) c += popc32(qi[w] & B[j * words + w]);
      if (sim_from_counts(c, pa, pb[j], metric) >= t) ++n;
    }
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
        int c = 0;
        for (int w = 0; w < words; ++w) c += popc32(qi[w] & B[j * words + w]);
        const double s = sim_from_counts(c, pa, pb[j], metric);
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
