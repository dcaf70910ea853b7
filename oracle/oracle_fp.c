/*
 * oracle_fp.c — TEST INFRASTRUCTURE ONLY (CPU restatement used as the checker in tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline leg). Nothing under nvmolkit_b200/ may import, link or call this.
 *
 * Path A: packed-fingerprint Tanimoto / cosine, thresholded neighbour counts, Butina clustering, Morgan fingerprints.
 *
 * What each function follows (paths relative to the nvMolKit v0.5.0 checkout):
 *   - similarity:  src/load_store.cuh:264-276 (0 when the intersection is empty) evaluated in fp64 as RDKit's
 *                  TanimotoSimilarity / CosineSimilarity do (integer popcounts, one divide).
 *   - butina:      RDKit rdkit/ML/Cluster/Butina.py ClusterData(isDistData=True, reordering=True). RDKit is an
 *                  un-vendored dependency (supported 2025.03.1 - 2026.03.1, reference README.md:19); the published
 *                  algorithm is restated here and anchored on the reference's call site
 *                  benchmarks/butina_clustering_bench.py:97-99 and its known answer tests/test_butina.cpp:241-273.
 *   - morgan:      src/morgan_fingerprint_cpu.cpp:61-255 (getEnvironments, literally: sort the (bitset, invariant,
 *                  atom) tuples, then walk them against the set of emitted neighbourhoods) and :257-307; hash =
 *                  RDKit gboost::hash_combine in uint32 (src/morgan_fingerprint_kernels.cu:53-62); bitset order =
 *                  boost::dynamic_bitset operator< (src/data_structures/flat_bit_vect.h:218-237).
 * Pinned by: tests/test_oracle_golden.py (reference known answers) — see DESIGN.md "Oracle pinning".
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

static inline int popc32(uint32_t v) { return __builtin_popcount(v); }

static double sim_from_counts(int c, int a, int b, int metric) {
  if (c == 0) return 0.0;
  if (metric == 0) return (double)c / (double)(a + b - c);
  return (double)c / sqrt((double)a * (double)b);
}

/* out[nA*nB] fp64 similarity. metric 0 = Tanimoto, 1 = cosine. */
void oracle_similarity_cross(const uint32_t* A, long nA, const uint32_t* B, long nB, int words, int metric,
                             double* out) {
  int* pa = (int*)malloc(sizeof(int) * (nA > 0 ? nA : 1));
  int* pb = (int*)malloc(sizeof(int) * (nB > 0 ? nB : 1));
  for (long i = 0; i < nA; ++i) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(A[i * words + w]);
    pa[i] = s;
  }
  for (long j = 0; j < nB; ++j) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(B[j * words + w]);
    pb[j] = s;
  }
#pragma omp parallel for schedule(static)
  for (long i = 0; i < nA; ++i) {
    for (long j = 0; j < nB; ++j) {
      int c = 0;
      for (int w = 0; w < words; ++w) c += popc32(A[i * words + w] & B[j * words + w]);
      out[i * nB + j] = sim_from_counts(c, pa[i], pb[j], metric);
    }
  }
  free(pa);
  free(pb);
}

/* counts[i] += sign * #{ j : 1 - sim(X_i, Y_j) <= cutoff }  (nvmolkit/_fusedButina.py:99-179, in fp64) */
void oracle_count_ge(const uint32_t* X, long nX, const uint32_t* Y, long nY, int words, int metric, double cutoff,
                     int sign, int32_t* counts) {
  int* py = (int*)malloc(sizeof(int) * (nY > 0 ? nY : 1));
  for (long j = 0; j < nY; ++j) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(Y[j * words + w]);
    py[j] = s;
  }
#pragma omp parallel for schedule(static)
  for (long i = 0; i < nX; ++i) {
    int px = 0;
    for (int w = 0; w < words; ++w) px += popc32(X[i * words + w]);
    int hits = 0;
    for (long j = 0; j < nY; ++j) {
      int c = 0;
      for (int w = 0; w < words; ++w) c += popc32(X[i * words + w] & Y[j * words + w]);
      if (1.0 - sim_from_counts(c, px, py[j], metric) <= cutoff) ++hits;
    }
    counts[i] += sign * hits;
  }
  free(py);
}

/* The materialised tensor-core Tanimoto epilogue (nvmolkit_b200/csrc/tanimoto_tc.cu) computes c / u without a division:
 * r = RN(1/u), q0 = RN(c r), q = fma(fma(-q0, u, c), r, q0). Returns the number of pairs 1 <= c <= u <= umax for which
 * q differs from the correctly rounded c / u (every pair is checked; umax = 8192 covers 4096-bit fingerprints).
 * newton = 0 drops the correction step (q = q0), so that a caller can see the check find mismatches where they exist. */
long oracle_recip_quotient_mismatches(int umax, int newton) {
  long bad = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : bad)
  for (int u = 1; u <= umax; ++u) {
    const double du = (double)u, r = 1.0 / du;
    for (int c = 1; c <= u; ++c) {
      const double dc = (double)c, q0 = dc * r;
      const double q  = newton ? fma(fma(-q0, du, dc), r, q0) : q0;
      bad += q != dc / du;
    }
  }
  return bad;
}

/* ---- Butina (ClusterData, reordering=True) on neighbour lists ---- */
typedef struct {
  long* start; /* [n+1] */
  int*  nbr;
} NbrLists;

static int butina_from_lists(long n, const NbrLists* L, int32_t* ids, int32_t* centroids) {
  /* live count of not-yet-assigned neighbours; RDKit keeps tLists sorted by (count, idx) descending and pops the head */
  int*  count = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
  char* seen  = (char*)calloc(n > 0 ? n : 1, 1);
  for (long i = 0; i < n; ++i) {
    count[i] = (int)(L->start[i + 1] - L->start[i]);
    ids[i]   = -1;
  }
  int nClusters = 0;
  for (;;) {
    long best = -1;
    for (long i = 0; i < n; ++i) {
      if (seen[i]) continue;
      if (best < 0 || count[i] > count[best] || (count[i] == count[best] && i > best)) best = i;
    }
    if (best < 0) break;
    /* tRes = [idx] + unseen neighbours */
    seen[best]           = 1;
    ids[best]            = nClusters;
    centroids[nClusters] = (int32_t)best;
    for (long e = L->start[best]; e < L->start[best + 1]; ++e) {
      const int m = L->nbr[e];
      if (seen[m]) continue;
      seen[m] = 1;
      ids[m]  = nClusters;
    }
    /* reordering: every remaining point loses the members of the new cluster from its neighbour list */
    for (long e = L->start[best]; e < L->start[best + 1]; ++e) {
      const int m = L->nbr[e];
      if (ids[m] != nClusters) continue;
      for (long f = L->start[m]; f < L->start[m + 1]; ++f) count[L->nbr[f]] -= 1;
    }
    for (long f = L->start[best]; f < L->start[best + 1]; ++f) count[L->nbr[f]] -= 1;
    ++nClusters;
  }
  free(count);
  free(seen);
  return nClusters;
}

static void build_lists_from_hits(long n, const unsigned char* hit, NbrLists* L) {
  L->start    = (long*)malloc(sizeof(long) * (n + 1));
  L->start[0] = 0;
  for (long i = 0; i < n; ++i) {
    long d = 0;
    for (long j = 0; j < n; ++j) d += (j != i && hit[i * n + j]);
    L->start[i + 1] = L->start[i] + d;
  }
  L->nbr = (int*)malloc(sizeof(int) * (L->start[n] > 0 ? L->start[n] : 1));
  for (long i = 0; i < n; ++i) {
    long at = L->start[i];
    for (long j = 0; j < n; ++j)
      if (j != i && hit[i * n + j]) L->nbr[at++] = (int)j;
  }
}

/* Dense distance matrix (dist <= cutoff are neighbours, src/butina.cu:1043-1051). Returns the number of clusters. */
int oracle_butina_dense(const double* dist, long n, double cutoff, int32_t* ids, int32_t* centroids) {
  unsigned char* hit = (unsigned char*)malloc((size_t)(n > 0 ? n * n : 1));
  for (long k = 0; k < n * n; ++k) hit[k] = dist[k] <= cutoff;
  NbrLists L;
  build_lists_from_hits(n, hit, &L);
  const int k = butina_from_lists(n, &L, ids, centroids);
  free(hit);
  free(L.start);
  free(L.nbr);
  return k;
}

/* Fingerprints in; distance = 1 - sim in fp64, neighbours: dist <= cutoff. Every unordered pair is evaluated once
 * (the matrix is symmetric) with OpenMP over rows; this is also bench.py's CPU baseline. */
int oracle_butina_fp(const uint32_t* fp, long n, int words, int metric, double cutoff, int32_t* ids,
                     int32_t* centroids) {
  int* pc = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
  for (long i = 0; i < n; ++i) {
    int s = 0;
    for (int w = 0; w < words; ++w) s += popc32(fp[i * words + w]);
    pc[i] = s;
  }
  int   nThreads = 1;
#ifdef _OPENMP
  nThreads = omp_get_max_threads();
#endif
  int** ebuf = (int**)calloc(nThreads, sizeof(int*));
  long* ecnt = (long*)calloc(nThreads, sizeof(long));
  long* ecap = (long*)calloc(nThreads, sizeof(long));
#pragma omp parallel
  {
    int t = 0;
#ifdef _OPENMP
    t = omp_get_thread_num();
#endif
#pragma omp for schedule(dynamic, 16)
    for (long i = 0; i < n; ++i) {
      const uint32_t* a = fp + i * words;
      for (long j = i + 1; j < n; ++j) {
        const uint32_t* b = fp + j * words;
        int             c = 0;
        if ((words & 1) == 0) { /* 64-bit popcounts, as RDKit's bit-vector code does */
          for (int w = 0; w < words; w += 2) {
            uint64_t av, bv;
            memcpy(&av, a + w, 8);
            memcpy(&bv, b + w, 8);
            c += __builtin_popcountll(av & bv);
          }
        } else {
          for (int w = 0; w < words; ++w) c += popc32(a[w] & b[w]);
        }
        if (1.0 - sim_from_counts(c, pc[i], pc[j], metric) <= cutoff) {
          if (ecnt[t] + 2 > ecap[t]) {
            ecap[t] = ecap[t] ? 2 * ecap[t] : 4096;
            ebuf[t] = (int*)realloc(ebuf[t], sizeof(int) * ecap[t]);
          }
          ebuf[t][ecnt[t]++] = (int)i;
          ebuf[t][ecnt[t]++] = (int)j;
        }
      }
    }
  }
  NbrLists L;
  L.start = (long*)calloc(n + 2, sizeof(long));
  for (int t = 0; t < nThreads; ++t)
    for (long e = 0; e < ecnt[t]; ++e) L.start[ebuf[t][e] + 1] += 1;
  for (long i = 0; i < n; ++i) L.start[i + 1] += L.start[i];
  L.nbr      = (int*)malloc(sizeof(int) * (L.start[n] > 0 ? L.start[n] : 1));
  long* fill = (long*)malloc(sizeof(long) * (n > 0 ? n : 1));
  for (long i = 0; i < n; ++i) fill[i] = L.start[i];
  for (int t = 0; t < nThreads; ++t) {
    for (long e = 0; e < ecnt[t]; e += 2) {
      const int i = ebuf[t][e], j = ebuf[t][e + 1];
      L.nbr[fill[i]++] = j;
      L.nbr[fill[j]++] = i;
    }
    free(ebuf[t]);
  }
  const int k = butina_from_lists(n, &L, ids, centroids);
  free(pc);
  free(fill);
  free(ebuf);
  free(ecnt);
  free(ecap);
  free(L.start);
  free(L.nbr);
  return k;
}

/* ---- Morgan ---- */
static inline void hash_combine(uint32_t* seed, uint32_t v) { *seed ^= v + 0x9e3779b9u + (*seed << 6) + (*seed >> 2); }

/* Atom invariant: gboost::hash<vector<uint32_t>> over {Z, degree+Hs, Hs incl. H neighbours, charge, deltaMass[, 1 if
 * in ring]} (src/morgan_fingerprint_common.cpp:80-121). */
uint32_t oracle_morgan_atom_invariant(uint32_t z, uint32_t totalDegree, uint32_t totalHs, int32_t charge,
                                      int32_t deltaMass, int inRing) {
  uint32_t seed = 0;
  hash_combine(&seed, z);
  hash_combine(&seed, totalDegree);
  hash_combine(&seed, totalHs);
  hash_combine(&seed, (uint32_t)charge);
  hash_combine(&seed, (uint32_t)deltaMass);
  if (inRing) hash_combine(&seed, 1u);
  return seed;
}

typedef struct {
  const uint32_t* bits; /* bw words */
  uint32_t        invar;
  unsigned        atom;
} EnvTuple;

static int g_bw; /* qsort context (oracle is single-threaded per call) */

static int bitset_cmp(const uint32_t* a, const uint32_t* b, int bw) {
  for (int w = bw - 1; w >= 0; --w) { /* most significant block first, like boost::dynamic_bitset operator< */
    if (a[w] < b[w]) return -1;
    if (a[w] > b[w]) return 1;
  }
  return 0;
}

static int env_cmp(const void* pa, const void* pb) {
  const EnvTuple* a = (const EnvTuple*)pa;
  const EnvTuple* b = (const EnvTuple*)pb;
  const int       c = bitset_cmp(a->bits, b->bits, g_bw);
  if (c) return c;
  if (a->invar != b->invar) return a->invar < b->invar ? -1 : 1;
  if (a->atom != b->atom) return a->atom < b->atom ? -1 : 1;
  return 0;
}

typedef struct {
  int32_t  first;
  uint32_t second;
} NbrPair;
static int pair_cmp(const void* pa, const void* pb) {
  const NbrPair* a = (const NbrPair*)pa;
  const NbrPair* b = (const NbrPair*)pb;
  if (a->first != b->first) return a->first < b->first ? -1 : 1;
  if (a->second != b->second) return a->second < b->second ? -1 : 1;
  return 0;
}

/* One molecule. codes_out (optional, capacity (radius+1)*nAtoms) receives the unfolded environment codes in emission
 * order; returns their number. fp (optional) gets bit (code % fpBits) set. */
int oracle_morgan_one(int nAtoms, int nBonds, const uint32_t* atomInv, const uint32_t* bondInv, const uint16_t* bondA,
                      const uint16_t* bondB, int radius, int fpBits, uint32_t* fp, uint32_t* codes_out) {
  const int bw = (nBonds + 31) / 32 > 0 ? (nBonds + 31) / 32 : 1;
  g_bw         = bw;
  uint32_t* cur      = (uint32_t*)malloc(sizeof(uint32_t) * (nAtoms + 1));
  uint32_t* next     = (uint32_t*)calloc(nAtoms + 1, sizeof(uint32_t));
  uint32_t* nbhd     = (uint32_t*)calloc((size_t)(nAtoms + 1) * bw, sizeof(uint32_t));
  uint32_t* nbhdR    = (uint32_t*)calloc((size_t)(nAtoms + 1) * bw, sizeof(uint32_t));
  uint32_t* emitted  = (uint32_t*)calloc((size_t)(radius + 1) * (nAtoms + 1) * bw, sizeof(uint32_t));
  char*     dead     = (char*)calloc(nAtoms + 1, 1);
  EnvTuple* round    = (EnvTuple*)malloc(sizeof(EnvTuple) * (nAtoms + 1));
  NbrPair*  pairs    = (NbrPair*)malloc(sizeof(NbrPair) * (2 * nBonds + 1));
  int       nEmitted = 0, nCodes = 0;
  if (fp) memset(fp, 0, (size_t)(fpBits / 32) * 4);
  memcpy(cur, atomInv, sizeof(uint32_t) * nAtoms);

  for (int i = 0; i < nAtoms; ++i) { /* round 0 */
    if (codes_out) codes_out[nCodes] = cur[i];
    ++nCodes;
    if (fp) fp[(cur[i] % (uint32_t)fpBits) >> 5] |= 1u << ((cur[i] % (uint32_t)fpBits) & 31);
  }
  for (int layer = 0; layer < radius; ++layer) {
    int nRound = 0;
    for (int a = 0; a < nAtoms; ++a) {
      if (dead[a]) continue;
      int deg = 0;
      for (int b = 0; b < nBonds; ++b) {
        int o = -1;
        if (bondA[b] == a) o = bondB[b];
        else if (bondB[b] == a) o = bondA[b];
        if (o < 0) continue;
        nbhdR[a * bw + (b >> 5)] |= 1u << (b & 31);
        for (int w = 0; w < bw; ++w) nbhdR[a * bw + w] |= nbhd[o * bw + w];
        pairs[deg].first  = (int32_t)bondInv[b];
        pairs[deg].second = cur[o];
        ++deg;
      }
      if (deg == 0) {
        dead[a] = 1;
        continue;
      }
      qsort(pairs, deg, sizeof(NbrPair), pair_cmp);
      uint32_t invar = (uint32_t)layer;
      hash_combine(&invar, cur[a]);
      for (int k = 0; k < deg; ++k) {
        uint32_t h = 0; /* gboost::hash<std::pair<int32,uint32>> */
        hash_combine(&h, (uint32_t)pairs[k].first);
        hash_combine(&h, pairs[k].second);
        hash_combine(&invar, h);
      }
      next[a]             = invar;
      round[nRound].bits  = nbhdR + (size_t)a * bw;
      round[nRound].invar = invar;
      round[nRound].atom  = (unsigned)a;
      ++nRound;
    }
    qsort(round, nRound, sizeof(EnvTuple), env_cmp);
    for (int t = 0; t < nRound; ++t) {
      int found = 0;
      for (int s = 0; s < nEmitted && !found; ++s) found = bitset_cmp(emitted + (size_t)s * bw, round[t].bits, bw) == 0;
      if (!found) {
        if (codes_out) codes_out[nCodes] = round[t].invar;
        ++nCodes;
        if (fp) fp[(round[t].invar % (uint32_t)fpBits) >> 5] |= 1u << ((round[t].invar % (uint32_t)fpBits) & 31);
        memcpy(emitted + (size_t)nEmitted * bw, round[t].bits, sizeof(uint32_t) * bw);
        ++nEmitted;
      } else {
        dead[round[t].atom] = 1;
      }
    }
    uint32_t* t = cur;
    cur         = next;
    next        = t;
    memset(next, 0, sizeof(uint32_t) * (nAtoms + 1));
    memcpy(nbhd, nbhdR, sizeof(uint32_t) * (size_t)nAtoms * bw);
  }
  free(cur);
  free(next);
  free(nbhd);
  free(nbhdR);
  free(emitted);
  free(dead);
  free(round);
  free(pairs);
  return nCodes;
}

/* Batch in the C-ABI's CSR layout (include/b200mol.h b200mol_morgan). out u32[nMols][fpBits/32]. */
void oracle_morgan(const int32_t* atomStarts, const int32_t* bondStarts, const uint32_t* atomInv,
                   const uint32_t* bondInv, const uint16_t* bondA, const uint16_t* bondB, long nMols, int radius,
                   int fpBits, uint32_t* out) {
  for (long m = 0; m < nMols; ++m) {
    const int a0 = atomStarts[m], b0 = bondStarts[m];
    oracle_morgan_one(atomStarts[m + 1] - a0, bondStarts[m + 1] - b0, atomInv + a0, bondInv + b0, bondA + b0,
                      bondB + b0, radius, fpBits, out + (size_t)m * (fpBits / 32), NULL);
  }
}

/* Thread count of the OpenMP teams of this library (bench.py: torchrun exports OMP_NUM_THREADS=1 to its workers; the CPU
 * baseline must say how many threads it really used). Returns the resulting maximum team size. */
int oracle_set_threads(int n) {
  if (n > 0) omp_set_num_threads(n);
  return omp_get_max_threads();
}
