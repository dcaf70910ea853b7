/*
 * oracle_topk.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of the top-k similarity search
 * (nvmolkit_b200/csrc/topk.cu) in tests/ and __graft_entry__.smoke(). Nothing under nvmolkit_b200/ may import, link or
 * call this.
 *
 * Row q of values / indices [nQ][k] = the first k columns of row q of oracle_similarity_cross's matrix (oracle_fp.c)
 * ordered by (value descending, column ascending), without the matrix: exact integer popcounts, the same fp64 value
 * (0 when the intersection is empty, else one divide), OpenMP over the queries. Pinned by tests/test_topk.py to
 * np.lexsort over oracle_similarity_cross.
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

/* Partial selection: a sorted list of k; a column enters by insertion only if it beats the list's last entry (columns
 * come in ascending order, so an equal value never does, and ties keep the lowest index). */
void oracle_topk(const uint32_t* Q, long nQ, const uint32_t* B, long nB, int words, int metric, int k, double* values,
                 int32_t* indices) {
  int* pb = (int*)malloc(sizeof(int) * (nB > 0 ? nB : 1));
  for (long j = 0; j < nB; ++j) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(B[j * words + w]);
    pb[j] = s;
  }
#pragma omp parallel for schedule(dynamic, 1)
  for (long i = 0; i < nQ; ++i) {
    double*  v  = values + i * k;
    int32_t* ix = indices + i * k;
    int      pa = 0, n = 0;
    for (int w = 0; w < words; ++w) pa += popc32(Q[i * words + w]);
    for (long j = 0; j < nB; ++j) {
      int c = 0;
      for (int w = 0; w < words; ++w) c += popc32(Q[i * words + w] & B[j * words + w]);
      const double s = sim_from_counts(c, pa, pb[j], metric);
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
