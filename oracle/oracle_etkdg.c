/*
 * oracle_etkdg.c — TEST INFRASTRUCTURE ONLY (see oracle_fp.c). The ETKDG attempt pipeline and its acceptance checks on
 * the CPU: same stage list, constants and counter-based random coordinates as nvmolkit_b200/csrc/etkdg.cu, built on the
 * oracle's own force fields and BFGS (oracle_ff.c).
 *
 * Follows (nvMolKit v0.5.0): stage configuration src/etkdg.cpp:325-394; energy acceptance
 * src/etkdg_stage_distgeom_minimize.cu:36-50 (+ .h:34); checks src/etkdg_stage_stereochem_checks.cu:30-440 (and
 * .h:69,122 tolerances); ETK refresh + planarity src/etkdg_stage_etk_minimization.cu:32-86,204-266; random box
 * src/etkdg_stage_coordgen.cu:100-122. Parity against RDKit's EmbedMultipleConfs is statistical by nature (the
 * reference's own tests, tests/test_etkdg.cu:506-651) — "parity unpinned" for coordinates, see DESIGN.md.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  const int32_t* starts;
  const int16_t* idx;
  const double*  par;
} TermTable;
typedef struct {
  int32_t        nMols;
  const int32_t* atomCounts;
  TermTable      dist, chiral, fourth;
} DgSystem;
typedef struct {
  int32_t        nMols;
  const int32_t* atomCounts;
  TermTable      torsion, improper, dist12, dist13, angle13, longrange;
} EtkSystem;
typedef struct {
  TermTable      tetrahedral, chiral, chiralDist, dbStereo, dbGeom;
  const int32_t* numImpropers;
} Checks;
typedef struct {
  uint64_t seed;
  double   boxSize, optimizerForceTol;
  int32_t  enforceChirality, useExpTorsions, useBasicKnowledge, maxAttempts, dgIters, fourthIters, etkIters, maxRestarts;
  int32_t  useMetricStart;
} EmbedParams;

void oracle_metric_matrix(const double* dist, int n, double* T);
int  oracle_power_eigen(double* m, int n, int numEigs, const double* v0, double* eigvals, double* eigvecs);

double oracle_dg_energy_grad(const DgSystem* s, int mol, int dim, double cw, double fw, const double* pos, double* grad);
double oracle_etk_energy_grad_ref(const EtkSystem* s, int mol, const double* pos, double* grad, int plain, const double* ref);
int    oracle_dg_minimize_one(const DgSystem* s, int mol, int dim, double cw, double fw, double* pos, int maxIters,
                              double gradTol, int maxRestarts, double* energy);
int    oracle_etk_minimize_one(const EtkSystem* s, int mol, int plain, const double* ref, double* pos, int maxIters,
                               double gradTol, double* energy);

static uint64_t mix64(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
double oracle_uniform01(uint64_t seed, uint32_t slot, uint32_t attempt, uint32_t element) {
  const uint64_t h = mix64(mix64(seed ^ ((uint64_t)slot << 32 | attempt)) + element);
  return (double)(h >> 11) * (1.0 / 9007199254740992.0);
}

static void sub(const double* a, const double* b, double* c) {
  c[0] = a[0] - b[0];
  c[1] = a[1] - b[1];
  c[2] = a[2] - b[2];
}
static void crs(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
static double dt(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
/* A zero vector stays zero (as in csrc/etkdg.cu): a tetrahedral volume through a zero-length arm is 0 and the row
 * fails the volume test. A division by the zero length would give NaN volumes that pass it, but the centre-in-volume
 * test would still fail the row (the centre lies in three face planes), so the verdict does not depend on it. */
static void   unit(double* v) {
  const double l = sqrt(dt(v, v));
  if (l > 0.0) {
    v[0] /= l;
    v[1] /= l;
    v[2] /= l;
  }
}
static int same_side(double tol, const double* v1, const double* v2, const double* v3, const double* v4, const double* p0) {
  double a[3], b[3], c[3], d[3];
  sub(v2, v1, a);
  sub(v3, v1, b);
  crs(a, b, c);
  sub(v4, v1, d);
  const double d1 = dt(c, d);
  sub(p0, v1, d);
  const double d2 = dt(c, d);
  if (fabs(d1) < tol || fabs(d2) < tol) return 0;
  return !((d1 < 0.) ^ (d2 < 0.));
}

static int tetrahedral_fails(const TermTable* T, int mol, const double* pos, double tol, int volume) {
  for (int t = T->starts[mol]; t < T->starts[mol + 1]; ++t) {
    const int16_t* ix = T->idx + 5 * t;
    const double * p0 = pos + 4 * ix[0], *p1 = pos + 4 * ix[1], *p2 = pos + 4 * ix[2], *p3 = pos + 4 * ix[3],
                 *p4 = pos + 4 * ix[4];
    if (volume) {
      double d1[3], d2[3], d3[3], d4[3], c[3];
      sub(p0, p1, d1);
      sub(p0, p2, d2);
      sub(p0, p3, d3);
      sub(p0, p4, d4);
      unit(d1);
      unit(d2);
      unit(d3);
      unit(d4);
      const double lim = (T->par[t] != 0.0 ? 0.25 : 1.0) * 0.50;
      crs(d1, d2, c);
      if (fabs(dt(c, d3)) < lim || fabs(dt(c, d4)) < lim) return 1;
      crs(d1, d3, c);
      if (fabs(dt(c, d4)) < lim) return 1;
      crs(d2, d3, c);
      if (fabs(dt(c, d4)) < lim) return 1;
    }
    if (ix[0] == ix[4]) continue;
    if (!same_side(tol, p1, p2, p3, p4, p0) || !same_side(tol, p2, p3, p4, p1, p0) || !same_side(tol, p3, p4, p1, p2, p0) ||
        !same_side(tol, p4, p1, p2, p3, p0))
      return 1;
  }
  return 0;
}
static int chirality_fails(const TermTable* T, int mol, const double* pos) {
  for (int t = T->starts[mol]; t < T->starts[mol + 1]; ++t) {
    const int16_t* ix = T->idx + 5 * t;
    const double * p1 = pos + 4 * ix[1], *p2 = pos + 4 * ix[2], *p3 = pos + 4 * ix[3], *p4 = pos + 4 * ix[4];
    double         v1[3], v2[3], v3[3], c[3];
    sub(p1, p4, v1);
    sub(p2, p4, v2);
    sub(p3, p4, v3);
    crs(v2, v3, c);
    const double vol = dt(v1, c), lb = T->par[2 * t], ub = T->par[2 * t + 1];
    if ((lb > 0 && vol < lb && (vol / lb < .8 || (signbit(vol) != 0) != (signbit(lb) != 0))) ||
        (ub < 0 && vol > ub && (vol / ub < .8 || (signbit(vol) != 0) != (signbit(ub) != 0))))
      return 1;
  }
  return 0;
}
static int chiral_dist_fails(const TermTable* T, int mol, const double* pos) {
  for (int t = T->starts[mol]; t < T->starts[mol + 1]; ++t) {
    double d[3];
    sub(pos + 4 * T->idx[2 * t], pos + 4 * T->idx[2 * t + 1], d);
    const double dist = sqrt(dt(d, d)), lb = T->par[2 * t], ub = T->par[2 * t + 1];
    if ((dist < lb && fabs(dist - lb) > 0.1 * ub) || (dist > ub && fabs(dist - ub) > 0.1 * ub)) return 1;
  }
  return 0;
}
static int db_stereo_fails(const TermTable* T, int mol, const double* pos) {
  for (int t = T->starts[mol]; t < T->starts[mol + 1]; ++t) {
    const int16_t* ix = T->idx + 4 * t;
    double         d1[3], d2[3], d3[3], c1[3], c2[3];
    sub(pos + 4 * ix[2], pos + 4 * ix[1], d1);
    sub(pos + 4 * ix[0], pos + 4 * ix[1], d2);
    sub(pos + 4 * ix[3], pos + 4 * ix[2], d3);
    crs(d2, d1, c1);
    crs(d3, d1, c2);
    const double d = dt(c1, c2) / sqrt(dt(c1, c1) * dt(c2, c2));
    double       angle = acos(d);
    if (d <= -1.0) angle = M_PI;
    else if (d >= 1.0) angle = 0.0;
    if ((angle - M_PI_2) * T->par[t] < 0.0) return 1;
  }
  return 0;
}
static int db_geom_fails(const TermTable* T, int mol, const double* pos) {
  for (int t = T->starts[mol]; t < T->starts[mol + 1]; ++t) {
    const int16_t* ix = T->idx + 3 * t;
    double         a[3], b[3];
    sub(pos + 4 * ix[1], pos + 4 * ix[0], a);
    sub(pos + 4 * ix[1], pos + 4 * ix[2], b);
    unit(a);
    unit(b);
    if (dt(a, b) + 1.0 < 1e-3) return 1;
  }
  return 0;
}
static int planarity_fails(const EtkSystem* etk, const Checks* ck, int mol, const double* pos) {
  EtkSystem only = *etk; /* improper terms alone */
  static const int32_t zeros[2] = {0, 0};
  (void)zeros;
  /* evaluate all, subtract the rest: simpler to zero the other ranges by pointing them at an all-zero CSR */
  int32_t* z = (int32_t*)calloc(etk->nMols + 1, sizeof(int32_t));
  only.torsion.starts = only.dist12.starts = only.dist13.starts = only.angle13.starts = only.longrange.starts = z;
  const double e = oracle_etk_energy_grad_ref(&only, mol, pos, NULL, 0, NULL);
  free(z);
  return e > 0.7 * (ck->numImpropers ? ck->numImpropers[mol] : 0);
}
static unsigned final_checks(const EtkSystem* etk, const Checks* ck, const EmbedParams* p, int mol, const double* pos,
                             int stopAtFirst) {
  (void)etk;
  unsigned m = 0;
  if (db_geom_fails(&ck->dbGeom, mol, pos)) m |= 1u << 6;
  if (m && stopAtFirst) return m;
  if (p->enforceChirality) {
    if (chirality_fails(&ck->chiral, mol, pos)) m |= 1u << 7;
    if (m && stopAtFirst) return m;
    if (chiral_dist_fails(&ck->chiralDist, mol, pos)) m |= 1u << 8;
    if (m && stopAtFirst) return m;
    if (tetrahedral_fails(&ck->chiral, mol, pos, 0.1, 0)) m |= 1u << 9;
    if (m && stopAtFirst) return m;
    if (db_stereo_fails(&ck->dbStereo, mol, pos)) m |= 1u << 10;
  }
  return m;
}

unsigned oracle_etkdg_check(const DgSystem* dg, const EtkSystem* etk, const Checks* ck, const EmbedParams* p, int mol,
                            const double* pos4) {
  unsigned     m = 0;
  const double e = oracle_dg_energy_grad(dg, mol, 4, 1.0, 0.1, pos4, NULL);
  if (e / dg->atomCounts[mol] >= 0.05) m |= 1u << 1;
  if (tetrahedral_fails(&ck->tetrahedral, mol, pos4, 0.3, 1)) m |= 1u << 2;
  if (p->enforceChirality && chirality_fails(&ck->chiral, mol, pos4)) m |= 1u << 3;
  if (p->useBasicKnowledge && planarity_fails(etk, ck, mol, pos4)) m |= 1u << 5;
  m |= final_checks(etk, ck, p, mol, pos4, 0);
  return m;
}

/* Stage 0 of one attempt: 4-D start coordinates. Random box (src/etkdg_stage_coordgen.cu:100-122), or with useMetricStart
 * RDKit's useRandomCoords = false start: DistGeom::pickRandomDistMat (d = lb + u (ub - lb)) and computeInitialCoords
 * (Code/DistGeom/DistGeomUtils.cpp of the un-vendored RDKit, restated: sqD0i < 1e-3 fails when N > 3; eigenvalues > 1e-3
 * -> sqrt, |.| < 1e-3 -> zero (one zero fails, numZeroFail = 1, when N > 3), negative -> random coordinate 1 - 2u
 * (randNegEig)) on the reference's power eigensolver (oracle_dg.c). Same random-stream elements as csrc/etkdg.cu.
 * Returns 1 on success. */
int oracle_etkdg_initial_coords(const DgSystem* dg, const EmbedParams* p, int slot, int mol, int attempt, double* pos) {
  const int nA = dg->atomCounts[mol], n = 4 * nA;
  if (!p->useMetricStart) {
    for (int i = 0; i < n; ++i) pos[i] = (oracle_uniform01(p->seed, slot, attempt, i) - 0.5) * p->boxSize;
    return 1;
  }
  double* dist = (double*)calloc((size_t)nA * nA, sizeof(double));
  double* T    = (double*)malloc(sizeof(double) * nA * nA);
  for (int t = dg->dist.starts[mol]; t < dg->dist.starts[mol + 1]; ++t) {
    int i = dg->dist.idx[2 * t], j = dg->dist.idx[2 * t + 1];
    if (i > j) {
      const int k = i;
      i = j;
      j = k;
    }
    const double lb = sqrt(dg->dist.par[3 * t]), ub = sqrt(dg->dist.par[3 * t + 1]);
    const double d  = lb + oracle_uniform01(p->seed, slot, attempt, (uint32_t)(n + i * nA + j)) * (ub - lb);
    dist[i * nA + j] = dist[j * nA + i] = d;
  }
  int ok = 1;
  /* the degenerate-centre test of computeInitialCoords on the same sqD0i the metric matrix is built from */
  double sumSq = 0.0;
  for (int e = 0; e < nA * nA; ++e) sumSq += dist[e] * dist[e];
  sumSq /= (double)nA * nA * 2.0;
  for (int i = 0; i < nA && ok; ++i) {
    double s = 0.0;
    for (int j = 0; j < nA; ++j) s += dist[i * nA + j] * dist[i * nA + j];
    if (s / nA - sumSq < 1.0e-3 && nA > 3) ok = 0;
  }
  const int nEigs = nA < 4 ? nA : 4;
  double    vals[4] = {0, 0, 0, 0};
  double*   vecs = (double*)calloc((size_t)4 * nA, sizeof(double));
  double*   v0   = (double*)malloc(sizeof(double) * 4 * nA);
  if (ok) {
    oracle_metric_matrix(dist, nA, T);
    for (int e = 0; e < nEigs * nA; ++e) v0[e] = oracle_uniform01(p->seed, slot, attempt, (uint32_t)(n + nA * nA + e));
    if (oracle_power_eigen(T, nA, nEigs, v0, vals, vecs) < nEigs) ok = 0;
  }
  if (ok) {
    int zero = 0;
    for (int k = 0; k < nEigs; ++k)
      if (fabs(vals[k]) < 1.0e-3) ++zero;
    if (zero >= 1 && nA > 3) ok = 0;
  }
  if (ok)
    for (int i = 0; i < nA; ++i)
      for (int k = 0; k < 4; ++k) {
        double x = 0.0;
        if (k < nEigs) {
          if (vals[k] > 1.0e-3) x = sqrt(vals[k]) * vecs[k * nA + i];
          else if (fabs(vals[k]) < 1.0e-3) x = 0.0;
          else x = 1.0 - 2.0 * oracle_uniform01(p->seed, slot, attempt, (uint32_t)(2 * n + nA * nA + k * nA + i));
        }
        pos[4 * i + k] = x;
      }
  free(dist);
  free(T);
  free(vecs);
  free(v0);
  return ok;
}

/* One slot. coords3[nAtoms*3] written on success. Returns 1 on success; *attemptsOut attempts used; failStages[11]
 * (optional) incremented per failed attempt. */
int oracle_etkdg_embed_one(const DgSystem* dg, const EtkSystem* etk, const Checks* ck, const EmbedParams* p, int slot,
                           int mol, double* coords3, int32_t* attemptsOut, double* energyOut, int64_t* failStages) {
  const int nA = dg->atomCounts[mol], n = 4 * nA;
  double*   pos = (double*)malloc(sizeof(double) * n);
  double*   ref = (double*)malloc(sizeof(double) * n);
  int       ok = 0, attempt = 0;
  for (attempt = 0; attempt < p->maxAttempts && !ok; ++attempt) {
    int    failed = -1;
    double e = 0.0, e2 = 0.0;
    if (!oracle_etkdg_initial_coords(dg, p, slot, mol, attempt, pos)) failed = 0;
    if (failed < 0) {
      oracle_dg_minimize_one(dg, mol, 4, 1.0, 0.1, pos, p->dgIters, p->optimizerForceTol, p->maxRestarts, &e);
      if (e / nA >= 0.05) failed = 1;
    }
    if (failed < 0 && tetrahedral_fails(&ck->tetrahedral, mol, pos, 0.3, 1)) failed = 2;
    if (failed < 0 && p->enforceChirality && chirality_fails(&ck->chiral, mol, pos)) failed = 3;
    if (failed < 0) oracle_dg_minimize_one(dg, mol, 4, 0.2, 1.0, pos, p->fourthIters, p->optimizerForceTol, 0, &e2);
    if (failed < 0 && (p->useExpTorsions || p->useBasicKnowledge)) {
      memcpy(ref, pos, sizeof(double) * n);
      oracle_etk_minimize_one(etk, mol, p->useBasicKnowledge ? 0 : 1, ref, pos, p->etkIters, p->optimizerForceTol, &e2);
      if (p->useBasicKnowledge && planarity_fails(etk, ck, mol, pos)) failed = 5;
    }
    if (failed < 0) {
      const unsigned m = final_checks(etk, ck, p, mol, pos, 1);
      if (m) failed = __builtin_ffs((int)m) - 1;
    }
    if (failed < 0) {
      ok = 1;
      if (energyOut) *energyOut = e;
    } else if (failStages) {
      failStages[failed] += 1;
    }
  }
  if (ok)
    for (int i = 0; i < nA; ++i)
      for (int c = 0; c < 3; ++c) coords3[3 * i + c] = pos[4 * i + c];
  if (attemptsOut) *attemptsOut = attempt;
  free(pos);
  free(ref);
  return ok;
}

/* All slots, OpenMP over slots (bench.py's CPU baseline). coords3: concatenated [slotAtomStart[s]*3 ...]. */
void oracle_etkdg_embed_batch(const DgSystem* dg, const EtkSystem* etk, const Checks* ck, const EmbedParams* p, int nSlots,
                              const int32_t* slotMol, const int32_t* slotAtomStart, double* coords3, int8_t* ok,
                              int32_t* attempts, double* energies) {
#pragma omp parallel for schedule(dynamic, 1)
  for (int s = 0; s < nSlots; ++s) {
    int32_t att = 0;
    double  en  = 0.0;
    ok[s] = (int8_t)oracle_etkdg_embed_one(dg, etk, ck, p, s, slotMol[s], coords3 + 3 * (size_t)slotAtomStart[s], &att, &en, NULL);
    if (attempts) attempts[s] = att;
    if (energies) energies[s] = en;
  }
}
