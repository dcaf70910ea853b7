/*
 * oracle_rmsd.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). The conformer RMSD matrix of one molecule in fp64, pair
 * by pair: after the best proper superposition through oracle_best_ssd (oracle_prune.c: Horn's quaternion matrix and
 * Jacobi rotations, a different route than the GPU's closed-form singular values of a tensor-core covariance), or,
 * prealigned, the plain sum of squared differences of the raw coordinates. OpenMP over rows.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

double oracle_best_ssd(const double* a, const int16_t* ia, const double* b, const int16_t* ib, int n);

/* conformer k of the molecule is confs[k], whose n atoms start at conf_atom_start[confs[k]] in xyz[.][3];
 * out[i (i - 1) / 2 + j] = RMSD of conformers i > j */
void oracle_rms_matrix(int nConf, const int32_t* confs, const int32_t* conf_atom_start, const double* xyz, int n,
                       int prealigned, double* out) {
#pragma omp parallel for schedule(dynamic, 4)
  for (int i = 1; i < nConf; ++i) {
    const double* a = xyz + 3 * (int64_t)conf_atom_start[confs[i]];
    for (int j = 0; j < i; ++j) {
      const double* b = xyz + 3 * (int64_t)conf_atom_start[confs[j]];
      double        ssd = 0.0;
      if (prealigned) {
        for (int k = 0; k < 3 * n; ++k) ssd += (a[k] - b[k]) * (a[k] - b[k]);
      } else {
        ssd = oracle_best_ssd(a, NULL, b, NULL, n);
      }
      out[(int64_t)i * (i - 1) / 2 + j] = sqrt(ssd / n);
    }
  }
}
