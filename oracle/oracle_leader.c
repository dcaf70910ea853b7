/*
 * oracle_leader.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of Leader (sphere-exclusion)
 * diversity picking (nvmolkit_b200/csrc/leader.cu) in tests/ and __graft_entry__.smoke(). Nothing under nvmolkit_b200/
 * may import, link or call this.
 *
 * oracle_leader_pick restates RDKit's LeaderPicker::lazyPick as a list walk: the remaining pool v in ascending index
 * order; the first picks are applied first, in their order; then each pick is v[0]. Applying a pick p removes p itself
 * from v and compacts the rest to the items with d(i, p) > threshold, in order. Every compaction runs on OpenMP threads
 * over contiguous chunks of v, each thread's kept items placed at an offset from a prefix over the chunk counts, so v
 * keeps its order, as RDKit threads it. The distance is 1 - sim_from_counts of oracle_fp.c (copied here; 0 for an empty
 * intersection), evaluated with the same fp64 operations as the other oracles. Picking stops when v is empty or there are
 * pickSize picks; returns the number of picks written to picks[].
 */
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdlib.h>

static inline int popc32(uint32_t v) { return __builtin_popcount(v); }

static double sim_from_counts(int c, int a, int b, int metric) {
  if (c == 0) return 0.0;
  if (metric == 0) return (double)c / (double)(a + b - c);
  return (double)c / sqrt((double)a * (double)b);
}

static double dist(const uint32_t* fp, const int* pc, int words, int metric, long i, long j) {
  int c = 0;
  for (int w = 0; w < words; ++w) c += popc32(fp[i * words + w] & fp[j * words + w]);
  return 1.0 - sim_from_counts(c, pc[i], pc[j], metric);
}

/* dst = the items of src[0, n) other than p with d(item, p) > threshold, in order; returns their count */
static long compact(const int32_t* src, long n, int32_t* dst, long p, const uint32_t* fp, const int* pc, int words,
                    int metric, double threshold, char* keep, long* offs) {
  long total = 0;
#pragma omp parallel
  {
    const int  t = omp_get_thread_num(), T = omp_get_num_threads();
    const long k0 = n * t / T, k1 = n * (t + 1) / T;
    long       kept = 0;
    for (long k = k0; k < k1; ++k) {
      keep[k] = src[k] != p && dist(fp, pc, words, metric, src[k], p) > threshold;
      kept += keep[k];
    }
    offs[t + 1] = kept;
#pragma omp barrier
#pragma omp single
    {
      offs[0] = 0;
      for (int u = 0; u < T; ++u) offs[u + 1] += offs[u];
      total = offs[T];
    }
    long at = offs[t];
    for (long k = k0; k < k1; ++k)
      if (keep[k]) dst[at++] = src[k];
  }
  return total;
}

long oracle_leader_pick(const uint32_t* fp, int words, int metric, long poolSize, double threshold, long pickSize,
                        const int32_t* first, int nFirst, int32_t* picks) {
  int* pc = (int*)malloc(sizeof(int) * (poolSize > 0 ? poolSize : 1));
  for (long i = 0; i < poolSize; ++i) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(fp[i * words + w]);
    pc[i] = s;
  }
  int32_t* v    = (int32_t*)malloc(sizeof(int32_t) * (poolSize > 0 ? poolSize : 1));
  int32_t* w    = (int32_t*)malloc(sizeof(int32_t) * (poolSize > 0 ? poolSize : 1));
  char*    keep = (char*)malloc(poolSize > 0 ? poolSize : 1);
  long*    offs = (long*)malloc(sizeof(long) * (omp_get_max_threads() + 1));
  long     n = poolSize, np = 0;
  for (long i = 0; i < n; ++i) v[i] = (int32_t)i;
  for (int f = 0; f < nFirst && np < pickSize; ++f) {
    picks[np++] = first[f];
    n           = compact(v, n, w, first[f], fp, pc, words, metric, threshold, keep, offs);
    int32_t* t  = v;
    v = w, w = t;
  }
  while (np < pickSize && n > 0) {
    const long p = v[0];
    picks[np++]  = (int32_t)p;
    n            = compact(v, n, w, p, fp, pc, words, metric, threshold, keep, offs);
    int32_t* t   = v;
    v = w, w = t;
  }
  free(offs);
  free(keep);
  free(w);
  free(v);
  free(pc);
  return np;
}
