/*
 * oracle_best_rms.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). The mapped conformer RMSD matrix of one molecule in
 * fp64 (RDKit GetAllConformerBestRMS): per pair i > j the minimum over the K mappings of the per-pair definition of
 * oracle_rmsd.c, with conformer i's atoms taken from the probe list P and conformer j's from the reference list Q_k:
 * oracle_best_ssd over the selected atoms, or, prealigned, the plain sum of squared differences. OpenMP over rows.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

double oracle_best_ssd(const double* a, const int16_t* ia, const double* b, const int16_t* ib, int n);

/* conformer k of the molecule is confs[k], whose atoms start at conf_atom_start[confs[k]] in xyz[.][3]; lists holds P,
 * then Q_1 .. Q_K, L atoms each; out[i (i - 1) / 2 + j] = min_k RMSD(x_i[P], x_j[Q_k]) of conformers i > j */
void oracle_rms_matrix_mapped(int nConf, const int32_t* confs, const int32_t* conf_atom_start, const double* xyz, int K,
                              int L, const int16_t* lists, int prealigned, double* out) {
#pragma omp parallel for schedule(dynamic, 4)
  for (int i = 1; i < nConf; ++i) {
    const double* a = xyz + 3 * (int64_t)conf_atom_start[confs[i]];
    for (int j = 0; j < i; ++j) {
      const double* b    = xyz + 3 * (int64_t)conf_atom_start[confs[j]];
      double        best = INFINITY;
      for (int k = 0; k < K; ++k) {
        const int16_t* q   = lists + (size_t)(k + 1) * L;
        double         ssd = 0.0;
        if (prealigned) {
          for (int t = 0; t < L; ++t)
            for (int r = 0; r < 3; ++r) {
              const double d = a[3 * lists[t] + r] - b[3 * q[t] + r];
              ssd += d * d;
            }
        } else {
          ssd = oracle_best_ssd(a, lists, b, q, L);
        }
        const double v = sqrt(ssd / L);
        if (v < best) best = v;
      }
      out[(int64_t)i * (i - 1) / 2 + j] = best;
    }
  }
}
