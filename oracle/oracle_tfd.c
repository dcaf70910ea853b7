/*
 * oracle_tfd.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). Torsion fingerprint deviation between the conformers of
 * each molecule, in fp64, pair by pair straight from the definition (RDKit TorsionFingerprints.CalculateTFD; restated by
 * the reference in src/tfd/tfd_detail.h:62-120 and src/tfd/tfd_kernels.cu:84-166). For conformers I > J and torsion t:
 *   single     d = circdiff(phi_I, phi_J)
 *   symmetric  d = min over quartet pairs (q, q') of circdiff(phi_I[q], phi_J[q'])
 *   ring       d = | mean_q |phi_I[q]| - mean_q |phi_J[q]| |
 * circdiff(a, b) = min(|a - b|, 360 - |a - b|), phi the signed dihedral in (-180, 180], 0 when a cross product is exactly
 * zero; TFD = sum w d / maxDev / sum w, 0 when sum w <= 1e-10. Same flat tables as b200mol_tfd_matrices, no feature rows
 * and no tiles: the dihedrals are recomputed for every pair.
 */
#include <math.h>
#include <stdint.h>

static double dihedral(const double* p0, const double* p1, const double* p2, const double* p3) {
  double v1[3], v2[3], v3[3], n1[3], n2[3], m[3];
  for (int k = 0; k < 3; ++k) {
    v1[k] = p1[k] - p0[k];
    v2[k] = p2[k] - p1[k];
    v3[k] = p3[k] - p2[k];
  }
  n1[0] = v1[1] * v2[2] - v1[2] * v2[1], n1[1] = v1[2] * v2[0] - v1[0] * v2[2], n1[2] = v1[0] * v2[1] - v1[1] * v2[0];
  n2[0] = v2[1] * v3[2] - v2[2] * v3[1], n2[1] = v2[2] * v3[0] - v2[0] * v3[2], n2[2] = v2[0] * v3[1] - v2[1] * v3[0];
  if ((n1[0] == 0.0 && n1[1] == 0.0 && n1[2] == 0.0) || (n2[0] == 0.0 && n2[1] == 0.0 && n2[2] == 0.0)) return 0.0;
  m[0] = n1[1] * n2[2] - n1[2] * n2[1], m[1] = n1[2] * n2[0] - n1[0] * n2[2], m[2] = n1[0] * n2[1] - n1[1] * n2[0];
  const double x = n1[0] * n2[0] + n1[1] * n2[1] + n1[2] * n2[2];
  const double y = (m[0] * v2[0] + m[1] * v2[1] + m[2] * v2[2]) / sqrt(v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2]);
  double phi = atan2(y, x) * (180.0 / M_PI);
  if (phi <= -180.0) phi += 360.0;
  return phi;
}

double oracle_tfd_dihedral(const double* p0, const double* p1, const double* p2, const double* p3) {
  return dihedral(p0, p1, p2, p3);
}

static double circdiff(double a, double b) {
  const double d = fabs(a - b);
  return d < 360.0 - d ? d : 360.0 - d;
}

static double phi_of(const double* xyz, int64_t atom0, const int16_t* q) {
  return dihedral(xyz + 3 * (atom0 + q[0]), xyz + 3 * (atom0 + q[1]), xyz + 3 * (atom0 + q[2]), xyz + 3 * (atom0 + q[3]));
}

/* confs[k] (k < nConf): index into conf_atom_start of the molecule's k-th conformer; torsions [t0, t1) of the global
 * tables; out[I(I-1)/2 + J] for I > J. */
void oracle_tfd_mol(int nConf, const int32_t* confs, const int32_t* conf_atom_start, const double* xyz, int t0, int t1,
                    const int32_t* quartet_start, const int16_t* quartets, const uint8_t* type, const double* weight,
                    const double* maxdev, double* out) {
  double sumW = 0.0;
  for (int t = t0; t < t1; ++t) sumW += weight[t];
#pragma omp parallel for schedule(dynamic, 4)
  for (int I = 1; I < nConf; ++I) {
    const int64_t aI = conf_atom_start[confs[I]];
    for (int J = 0; J < I; ++J) {
      const int64_t aJ  = conf_atom_start[confs[J]];
      double        acc = 0.0;
      for (int t = t0; t < t1; ++t) {
        const int      Q = quartet_start[t + 1] - quartet_start[t];
        const int16_t* q = quartets + 4 * (int64_t)quartet_start[t];
        double         d;
        if (type[t] == 2) { /* ring */
          double mI = 0.0, mJ = 0.0;
          for (int k = 0; k < Q; ++k) {
            mI += fabs(phi_of(xyz, aI, q + 4 * k));
            mJ += fabs(phi_of(xyz, aJ, q + 4 * k));
          }
          d = fabs(mI / Q - mJ / Q);
        } else {
          d = 180.0;
          for (int a = 0; a < Q; ++a)
            for (int b = 0; b < Q; ++b) {
              const double c = circdiff(phi_of(xyz, aI, q + 4 * a), phi_of(xyz, aJ, q + 4 * b));
              if (c < d) d = c;
            }
        }
        acc += weight[t] * d / maxdev[t];
      }
      out[(int64_t)I * (I - 1) / 2 + J] = sumW > 1e-10 ? acc / sumW : 0.0;
    }
  }
}
