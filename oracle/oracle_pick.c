/*
 * oracle_pick.c — TEST INFRASTRUCTURE ONLY, like the rest of this directory: the checker of MaxMin diversity picking
 * (nvmolkit_b200/csrc/maxmin.cu) in tests/ and __graft_entry__.smoke(). Nothing under nvmolkit_b200/ may import, link
 * or call this.
 *
 * oracle_maxmin_lazy restates RDKit's MaxMinPicker::lazyPick step for step: the pool as a list in index order (0
 * ends it, as there), a per-item distance bound and count of picks it covers, the first pass over the first pick, the
 * walk that only looks at items whose bound beats the running max-min (strict >), catches them up through the later
 * picks and leaves as soon as the bound falls to the running max-min, and the threshold stop. oracle_maxmin_dense is the
 * plain definition for large pools: every pick updates every item's min, OpenMP over items, argmax with ties to the
 * lowest index. The distance is 1 - sim_from_counts of oracle_fp.c (copied here; 0 for an empty intersection).
 * Both write picks[pickSize] (-1 past a threshold stop) and return the threshold RDKit returns: the max-min of the last
 * pick the loop added, -1 when it added none.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

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

static int* popcounts(const uint32_t* fp, long n, int words) {
  int* pc = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
  for (long i = 0; i < n; ++i) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(fp[i * words + w]);
    pc[i] = s;
  }
  return pc;
}

typedef struct {
  double       dist_bound;
  unsigned int picks;
  unsigned int next;
} PickInfo;

double oracle_maxmin_lazy(const uint32_t* fp, int words, int metric, unsigned int poolSize, unsigned int pickSize,
                          const int32_t* first, int nFirst, double threshold, int32_t* picks) {
  int*      pc    = popcounts(fp, poolSize, words);
  PickInfo* pinfo = (PickInfo*)calloc(poolSize, sizeof(PickInfo));
  for (unsigned int k = 0; k < pickSize; ++k) picks[k] = -1;
  unsigned int picked = 0, pick = 0;
  for (int f = 0; f < nFirst; ++f) {
    pick           = (unsigned int)first[f];
    picks[picked++] = (int32_t)pick;
    pinfo[pick].picks = 1;
  }
  if (picked >= pickSize) {
    free(pinfo);
    free(pc);
    return -1.0;
  }
  /* the unpicked pool as a list in index order */
  unsigned int  pool_list = 0;
  unsigned int* prev      = &pool_list;
  for (unsigned int i = 0; i < poolSize; ++i)
    if (pinfo[i].picks == 0) {
      *prev = i;
      prev  = &pinfo[i].next;
    }
  *prev = 0;
  /* first pass: every item's bound from the first pick */
  unsigned int poolIdx, pickIdx = (unsigned int)picks[0];
  prev = &pool_list;
  do {
    poolIdx                    = *prev;
    pinfo[poolIdx].dist_bound = dist(fp, pc, words, metric, poolIdx, pickIdx);
    pinfo[poolIdx].picks      = 1;
    prev                       = &pinfo[poolIdx].next;
  } while (*prev != 0);

  double maxOFmin = -1.0, tmpThreshold = -1.0;
  while (picked < pickSize) {
    unsigned int* pick_prev = NULL;
    maxOFmin                = -1.0;
    prev                    = &pool_list;
    do {
      poolIdx       = *prev;
      double minTOi = pinfo[poolIdx].dist_bound;
      if (minTOi > maxOFmin) {
        unsigned int pi = pinfo[poolIdx].picks;
        while (pi < picked) {
          const unsigned int picki = (unsigned int)picks[pi];
          const double       d     = dist(fp, pc, words, metric, poolIdx, picki);
          ++pi;
          if (d <= minTOi) {
            minTOi = d;
            if (minTOi <= maxOFmin) break;
          }
        }
        pinfo[poolIdx].dist_bound = minTOi;
        pinfo[poolIdx].picks      = pi;
        if (minTOi > maxOFmin) {
          maxOFmin  = minTOi;
          pick_prev = prev;
          pick      = poolIdx;
        }
      }
      prev = &pinfo[poolIdx].next;
    } while (*prev != 0);
    if (maxOFmin <= threshold && threshold >= 0.0) break;
    tmpThreshold = maxOFmin;
    *pick_prev   = pinfo[pick].next;
    picks[picked++] = (int32_t)pick;
  }
  free(pinfo);
  free(pc);
  return tmpThreshold;
}

double oracle_maxmin_dense(const uint32_t* fp, int words, int metric, long poolSize, int pickSize, const int32_t* first,
                           int nFirst, double threshold, int32_t* picks) {
  int*    pc  = popcounts(fp, poolSize, words);
  double* mn  = (double*)malloc(sizeof(double) * poolSize);
  char*   pkd = (char*)calloc(poolSize, 1);
  for (int k = 0; k < pickSize; ++k) picks[k] = -1;
  for (long i = 0; i < poolSize; ++i) mn[i] = INFINITY;
  for (int f = 0; f < nFirst; ++f) picks[f] = first[f], pkd[first[f]] = 1;
  int    t = nFirst, applied = 0;
  double last = -1.0;
  while (t < pickSize) {
    double best  = -1.0;
    long   bestI = -1;
#pragma omp parallel
    {
      double lb = -1.0;
      long   li = -1;
#pragma omp for schedule(static)
      for (long i = 0; i < poolSize; ++i) {
        if (pkd[i]) continue;
        for (int p = applied; p < t; ++p) {
          const double d = dist(fp, pc, words, metric, i, picks[p]);
          if (d < mn[i]) mn[i] = d;
        }
        if (mn[i] > lb || (mn[i] == lb && i < li)) lb = mn[i], li = i;
      }
#pragma omp critical
      if (li >= 0 && (lb > best || (lb == best && li < bestI))) best = lb, bestI = li;
    }
    applied = t;
    if (threshold >= 0.0 && best <= threshold) break;
    picks[t++]  = (int32_t)bestI;
    pkd[bestI] = 1;
    last       = best;
  }
  free(pkd);
  free(mn);
  free(pc);
  return last;
}
