/*
 * oracle_best_align.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). The symmetry-aware alignment of one probe /
 * reference conformer pair in fp64 (RDKit GetBestRMS / GetBestAlignmentTransform / CalcRMS): per mapping k of P to Q_k,
 * mode 0 aligns through oracle_align (oracle_align.c) and mode 1 takes the RMSD on the coordinates as given; the result
 * is the first mapping with the strictly smallest RMSD, as RDKit's `if (rms < best)`.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

double oracle_align(const double* prb, const double* ref, const int32_t* pairs, const double* w, int L, int reflect,
                    int maxIters, double* T);

/* lists: P, then Q_1 .. Q_K, L atoms each; w: L weights or NULL. Returns the best RMSD; *best its first mapping, T (16,
 * mode 0 only) its transform, per_map (optional, K) every mapping's RMSD. */
double oracle_best_align(const double* prb, const double* ref, const int16_t* lists, const double* w, int K, int L,
                         int mode, int reflect, int maxIters, double* T, int* best, double* per_map) {
  int32_t* pairs = malloc(sizeof(int32_t) * 2 * (size_t)L);
  double   bestV = INFINITY, Tk[16];
  *best        = 0;
  for (int k = 0; k < K; ++k) {
    const int16_t* q = lists + (size_t)(k + 1) * L;
    double         v;
    if (mode) {
      double ssd = 0.0;
      for (int i = 0; i < L; ++i) {
        double d2 = 0.0;
        for (int c = 0; c < 3; ++c) {
          const double d = prb[3 * lists[i] + c] - ref[3 * q[i] + c];
          d2 += d * d;
        }
        ssd += (w ? w[i] : 1.0) * d2;
      }
      v = sqrt(ssd / L);
    } else {
      for (int i = 0; i < L; ++i) pairs[2 * i] = lists[i], pairs[2 * i + 1] = q[i];
      v = oracle_align(prb, ref, pairs, w, L, reflect, maxIters, Tk);
    }
    if (per_map) per_map[k] = v;
    if (v < bestV) {
      bestV = v;
      *best = k;
      if (!mode)
        for (int i = 0; i < 16; ++i) T[i] = Tk[i];
    }
  }
  free(pairs);
  return bestV;
}
