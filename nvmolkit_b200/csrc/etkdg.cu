// ETKDG conformer embedding: one CTA carries one conformer slot through the WHOLE attempt pipeline inside one persistent
// kernel — random 4-D coordinates -> DG minimisation (repeat until converged) -> energy / tetrahedral / chirality
// checks -> fourth-dimension collapse -> ETK refinement -> planarity, double-bond and final chirality checks — and
// retries failed attempts itself with a fresh random stream. No host round trip between stages.
//
// Stage list and constants = the reference's production pipeline (src/etkdg.cpp:325-394, SURVEY.md §3.3):
//   0 coordinates: (u - 0.5) * boxSize in all four dimensions           (src/etkdg_stage_coordgen.cu:100-122; on the CPU there)
//     or, useRandomCoords = 0 (the reference refuses it, src/etkdg.cpp:99-101; SURVEY.md 8f-1): RDKit's metric-matrix
//     start - a random distance matrix inside the bounds, its metric matrix, the top four eigenpairs by power iteration
//     (the matrix lives in this CTA's inverse-Hessian slab, which is idle at that point), coordinates sqrt(lambda) v
//   1 DG minimise  chiral 1.0 / 4th-dim 0.1, 400 iterations, repeated until converged; fail if E/atom >= 0.05
//                                                                        (src/etkdg_stage_distgeom_minimize.cu:177-249, .h:34)
//   2 tetrahedral check (volume >= 0.5, x0.25 in fused small rings; centre inside, tol 0.3)   (stereochem_checks.cu:52-168)
//   3 first chirality check                                             (stereochem_checks.cu:219-268)
//   4 DG minimise  chiral 0.2 / 4th-dim 1.0, 200 iterations             (src/etkdg.cpp:365-370)
//   5 ETK minimise 300 iterations on xyz, 1-2 / 1-3 windows re-centred; planarity: improper energy <= 0.7 * nImpropers
//                                                                        (src/etkdg_stage_etk_minimization.cu:66-86,204-266)
//   6 double-bond linearity  7 final chirality  8 chiral distance matrix  9 centre-in-volume (tol 0.1)  10 double-bond stereo
//                                                                        (stereochem_checks.cu:270-440)
// The reference launches each stage as separate kernels over a 500-conformer batch, generates coordinates on the CPU,
// and lets a host Scheduler re-dispatch failures (src/etkdg_impl.cpp:111-159,286-312).
#include "bfgs_device.cuh"
#include "dgprep_device.cuh"
#include "profile.cuh"

namespace b200 {
extern int g_bfgsCtasPerSm;
extern int g_bfgsL2Persist;
int        g_etkdgHessianFp64 = 0;  // option "etkdg_hessian_fp64": the embedder's inverse Hessian in fp64 (default fp32)
unsigned long long* pathBStats();
namespace {

using ff::V3;

struct EmbedArgs {
  b200mol_dg_system       dg;
  b200mol_etk_system      etk;
  b200mol_etkdg_checks    chk;
  b200mol_embed_params    par;
  int                     nSlots;
  const int32_t*          slotMol;        // [nSlots]
  const int32_t*          slotAtomStart;  // [nSlots+1] offsets into coords (atoms)
  double*                 coords;         // [totalAtoms][3]
  int8_t*                 ok;             // [nSlots]
  int32_t*                attempts;       // [nSlots]
  double*                 energy;         // [nSlots] DG energy (first-stage weights) of the accepted attempt
  unsigned long long*     stageFailures;  // [kNumStages] (may be NULL)
  void*                   hessWs;  // inverse-Hessian slabs: fp32 by default (swept in fp32, bfgs_device.cuh; half the
                                   // traffic), fp64 with option "etkdg_hessian_fp64" (the reference's storage type)
  size_t                  hessStride;
  int*                    queue;
  int                     maxN;
  // attempt-level work stealing (see etkdgKernel): per slot, the next attempt index to hand out, the lowest successful
  // attempt so far (kNoAttempt = none), a spin lock for the result write, and the number of attempts that have ended
  int *slotNext, *slotBest, *slotLock, *slotDone;
  unsigned long long* stats;
};
constexpr int kNoAttempt      = 0x7f7f7f7f;  // cudaMemset(0x7f) pattern
constexpr int kMaxSpeculation = 8;           // attempts of one slot in flight at once, at most

constexpr int kNumStages = 11;

__device__ __forceinline__ uint64_t mix64(uint64_t x) {  // splitmix64 finaliser: counter-based, stateless
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// u in [0,1) from (seed, slot, attempt, element)
__device__ __forceinline__ double uniform01(uint64_t seed, uint32_t slot, uint32_t attempt, uint32_t element) {
  const uint64_t h = mix64(mix64(seed ^ (static_cast<uint64_t>(slot) << 32 | attempt)) + element);
  return static_cast<double>(h >> 11) * (1.0 / 9007199254740992.0);
}

__device__ __forceinline__ V3 p3(const double* pos, int a) { return {pos[4 * a], pos[4 * a + 1], pos[4 * a + 2]}; }

__device__ bool anyFail(bool mine);

// Stage 0 of one attempt: 4-D start coordinates pos[4 * nA]. Returns false (block-uniform) when the metric-matrix start
// fails (the attempt is then spent, like RDKit's embedPoints). Random streams are functions of (seed, slot, attempt,
// element): elements [0, 4 nA) the box coordinates; 4 nA + i nA + j (i < j) the distance of pair (i, j);
// 4 nA + nA^2 + e nA + i the start vector of eigenpair e; 8 nA + nA^2 + k nA + i the replacement coordinate of a
// dimension with a negative eigenvalue.
//   work: shared memory, >= 11 nA + 8 doubles.   mat: nA x nA doubles of global scratch (metric start only).
// Metric start = RDKit DistGeom::pickRandomDistMat + computeInitialCoords (Code/DistGeom/DistGeomUtils.cpp of the
// un-vendored RDKit 2025.03, restated: EIGVAL_TOL 1e-3, randNegEig = true, numZeroFail = 1) with the reference's power
// eigensolver (src/symmetric_eigensolver.cu:62-247, dgprep_device.cuh).
__device__ bool initialCoords(const b200mol_embed_params& par, const b200mol_dg_system& dg, int mol, int nA, int slot,
                              int attempt, double* pos, double* work, double* mat, double* red) {
  const int tid = threadIdx.x, n = 4 * nA;
  if (!par.useMetricStart) {
    for (int i = tid; i < n; i += kT) pos[i] = (uniform01(par.seed, slot, attempt, i) - 0.5) * par.boxSize;
    __syncthreads();
    return true;
  }
  double* v = work;                    // nA
  double* z = v + nA;                  // nA
  double* vecs = z + nA;               // 4 nA
  double* v0 = vecs + 4 * nA;          // 4 nA
  double* sq0 = v0 + 4 * nA;           // nA
  double* vals = sq0 + nA;             // 4
  const uint32_t base = static_cast<uint32_t>(n);
  for (int e = tid; e < nA * nA; e += kT) mat[e] = 0.0;
  __syncthreads();
  // squared random distances inside the bounds (every pair is a DG distance term: basinThresh = 1e8)
  for (int t = dg.dist.starts[mol] + tid; t < dg.dist.starts[mol + 1]; t += kT) {
    int i = dg.dist.idx[2 * t], j = dg.dist.idx[2 * t + 1];
    if (i > j) {
      const int k = i;
      i           = j;
      j           = k;
    }
    const double lb = sqrt(dg.dist.par[3 * t]), ub = sqrt(dg.dist.par[3 * t + 1]);
    const double d  = lb + uniform01(par.seed, slot, attempt, base + static_cast<uint32_t>(i * nA + j)) * (ub - lb);
    mat[i * nA + j] = mat[j * nA + i] = d * d;
  }
  __syncthreads();
  double tot = 0.0;
  for (int i = tid; i < nA; i += kT) {
    double s = 0.0;
    for (int j = 0; j < nA; ++j) s += mat[i * nA + j];
    sq0[i] = s;
    tot += s;
  }
  const double sumSq = blockSum(tot, red) / (static_cast<double>(nA) * nA * 2.0);
  bool         bad   = false;
  for (int i = tid; i < nA; i += kT) {
    sq0[i] = sq0[i] / nA - sumSq;
    if (sq0[i] < 1.0e-3 && nA > 3) bad = true;
  }
  if (anyFail(bad)) return false;
  for (int e = tid; e < nA * nA; e += kT) mat[e] = 0.5 * (sq0[e / nA] + sq0[e % nA] - mat[e]);
  const int nEigs = nA < 4 ? nA : 4;
  for (int e = tid; e < nEigs * nA; e += kT) v0[e] = uniform01(par.seed, slot, attempt, base + static_cast<uint32_t>(nA * nA + e));
  __syncthreads();
  const int done = powerEigen(mat, nA, nEigs, v0, 0u, v, z, red, vals, vecs);
  if (done < nEigs) return false;
  int zeroEigs = 0;
  for (int k = 0; k < nEigs; ++k)  // (every thread evaluates the same four numbers)
    if (fabs(vals[k]) < 1.0e-3) ++zeroEigs;
  if (zeroEigs >= 1 && nA > 3) return false;
  for (int e = tid; e < n; e += kT) {
    const int i = e >> 2, k = e & 3;
    double    x = 0.0;
    if (k < nEigs) {
      const double lam = vals[k];
      if (lam > 1.0e-3) x = sqrt(lam) * vecs[k * nA + i];
      else if (fabs(lam) < 1.0e-3) x = 0.0;
      else x = 1.0 - 2.0 * uniform01(par.seed, slot, attempt, 2u * base + static_cast<uint32_t>(nA * nA + k * nA + i));
    }
    pos[e] = x;
  }
  __syncthreads();
  return true;
}

__device__ __forceinline__ bool sameSide(double tol, const V3& v1, const V3& v2, const V3& v3, const V3& v4, const V3& p0) {
  const V3     c  = ff::cross(v2 - v1, v3 - v1);
  const double d1 = ff::dot(c, v4 - v1), d2 = ff::dot(c, p0 - v1);
  if (fabs(d1) < tol || fabs(d2) < tol) return false;
  return !((d1 < 0.) ^ (d2 < 0.));
}

// Each check returns true when the conformer FAILS it. All threads take part; the verdict is block-uniform.
__device__ bool anyFail(bool mine) { return __syncthreads_or(mine ? 1 : 0) != 0; }

template <bool VOLUME>
__device__ bool tetrahedralFails(const b200mol_term_table& T, int mol, const double* pos, double tol) {
  bool bad = false;
  for (int t = T.starts[mol] + threadIdx.x; t < T.starts[mol + 1]; t += kT) {
    const int16_t* ix = T.idx + 5 * t;
    const V3       p0 = p3(pos, ix[0]), p1 = p3(pos, ix[1]), p2 = p3(pos, ix[2]), q3 = p3(pos, ix[3]), p4 = p3(pos, ix[4]);
    if (VOLUME) {
      auto unit = [](V3 v) {
        const double l = sqrt(ff::dot(v, v));
        return l > 0.0 ? v * (1.0 / l) : v;
      };
      const V3     d1 = unit(p0 - p1), d2 = unit(p0 - p2), d3 = unit(p0 - q3), d4 = unit(p0 - p4);
      const double lim = (T.par[t] != 0.0 ? 0.25 : 1.0) * 0.50;
      V3           c   = ff::cross(d1, d2);
      if (fabs(ff::dot(c, d3)) < lim || fabs(ff::dot(c, d4)) < lim) bad = true;
      c = ff::cross(d1, d3);
      if (fabs(ff::dot(c, d4)) < lim) bad = true;
      c = ff::cross(d2, d3);
      if (fabs(ff::dot(c, d4)) < lim) bad = true;
      if (bad) continue;
    }
    if (ix[0] == ix[4]) continue;  // three-coordinate centre
    if (!sameSide(tol, p1, p2, q3, p4, p0) || !sameSide(tol, p2, q3, p4, p1, p0) || !sameSide(tol, q3, p4, p1, p2, p0) ||
        !sameSide(tol, p4, p1, p2, q3, p0))
      bad = true;
  }
  return anyFail(bad);
}

__device__ bool chiralityFails(const b200mol_term_table& T, int mol, const double* pos) {
  bool bad = false;
  for (int t = T.starts[mol] + threadIdx.x; t < T.starts[mol + 1]; t += kT) {
    const int16_t* ix = T.idx + 5 * t;
    const V3       p1 = p3(pos, ix[1]), p2 = p3(pos, ix[2]), q3 = p3(pos, ix[3]), p4 = p3(pos, ix[4]);
    const double   vol = ff::dot(p1 - p4, ff::cross(p2 - p4, q3 - p4));
    const double   lb = T.par[2 * t], ub = T.par[2 * t + 1];
    if ((lb > 0 && vol < lb && (vol / lb < .8 || (signbit(vol) != signbit(lb)))) ||
        (ub < 0 && vol > ub && (vol / ub < .8 || (signbit(vol) != signbit(ub)))))
      bad = true;
  }
  return anyFail(bad);
}

__device__ bool chiralDistFails(const b200mol_term_table& T, int mol, const double* pos) {
  bool bad = false;
  for (int t = T.starts[mol] + threadIdx.x; t < T.starts[mol + 1]; t += kT) {
    const V3     d    = p3(pos, T.idx[2 * t]) - p3(pos, T.idx[2 * t + 1]);
    const double dist = sqrt(ff::dot(d, d)), lb = T.par[2 * t], ub = T.par[2 * t + 1];
    if ((dist < lb && fabs(dist - lb) > 0.1 * ub) || (dist > ub && fabs(dist - ub) > 0.1 * ub)) bad = true;
  }
  return anyFail(bad);
}

__device__ bool doubleBondStereoFails(const b200mol_term_table& T, int mol, const double* pos) {
  bool bad = false;
  for (int t = T.starts[mol] + threadIdx.x; t < T.starts[mol + 1]; t += kT) {
    const int16_t* ix = T.idx + 4 * t;
    const V3       p0 = p3(pos, ix[0]), p1 = p3(pos, ix[1]), p2 = p3(pos, ix[2]), q3 = p3(pos, ix[3]);
    const V3       d1 = p2 - p1, d2 = p0 - p1, d3 = q3 - p2;
    const V3       c1 = ff::cross(d2, d1), c2 = ff::cross(d3, d1);
    double         dt = ff::dot(c1, c2) / sqrt(ff::dot(c1, c1) * ff::dot(c2, c2));
    double         angle = acos(dt);
    if (dt <= -1.0) angle = 3.14159265358979323846;
    else if (dt >= 1.0) angle = 0.0;
    if ((angle - 3.14159265358979323846 / 2.0) * T.par[t] < 0.0) bad = true;
  }
  return anyFail(bad);
}

__device__ bool doubleBondGeometryFails(const b200mol_term_table& T, int mol, const double* pos) {
  bool bad = false;
  for (int t = T.starts[mol] + threadIdx.x; t < T.starts[mol + 1]; t += kT) {
    const int16_t* ix = T.idx + 3 * t;
    V3             a = p3(pos, ix[1]) - p3(pos, ix[0]), b = p3(pos, ix[1]) - p3(pos, ix[2]);
    a                = a * (1.0 / sqrt(ff::dot(a, a)));
    b                = b * (1.0 / sqrt(ff::dot(b, b)));
    if (ff::dot(a, b) + 1.0 < 1e-3) bad = true;
  }
  return anyFail(bad);
}

// Planarity: energy of the improper (inversion) terms alone vs 0.7 * numImpropers.
__device__ bool planarityFails(const b200mol_etk_system& etk, const int32_t* numImpropers, int mol, const double* pos,
                               double* red) {
  ff::Etk::View v = ff::Etk::view(etk, mol, {0, 0});
  v.torsion.end = v.torsion.beg;
  v.d12.end     = v.d12.beg;
  v.d13.end     = v.d13.beg;
  v.a13.end     = v.a13.beg;
  v.lr.end      = v.lr.beg;
  const double e = blockSum(ff::Etk::eval<false>(v, pos, nullptr, threadIdx.x, kT), red);
  return e > 0.7 * (numImpropers ? numImpropers[mol] : 0);
}

// Stage outcomes on given 4-D coordinates as a bit mask (bit s = stage s failed); used by the attempt kernel and by the
// check-only entry point that tests compare against the CPU oracle.
__device__ unsigned finalChecks(const EmbedArgs& a, int mol, const double* pos, double* red, bool stopAtFirst) {
  unsigned m = 0;
  if (doubleBondGeometryFails(a.chk.dbGeom, mol, pos)) m |= 1u << 6;
  if (m && stopAtFirst) return m;
  if (a.par.enforceChirality) {
    if (chiralityFails(a.chk.chiral, mol, pos)) m |= 1u << 7;
    if (m && stopAtFirst) return m;
    if (chiralDistFails(a.chk.chiralDist, mol, pos)) m |= 1u << 8;
    if (m && stopAtFirst) return m;
    if (tetrahedralFails<false>(a.chk.chiral, mol, pos, 0.1)) m |= 1u << 9;
    if (m && stopAtFirst) return m;
    if (doubleBondStereoFails(a.chk.dbStereo, mol, pos)) m |= 1u << 10;
  }
  return m;
}

template <class HT>
__global__ void __launch_bounds__(kT, kMinCtas) etkdgKernel(const EmbedArgs a) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[kRed];
  __shared__ double                     colBuf[kColBuf];
  const BfgsWorkT<HT> w = carveWork<HT>(sm, a.maxN, static_cast<HT*>(a.hessWs) + static_cast<size_t>(blockIdx.x) * a.hessStride, red, colBuf, a.stats);
  double*        ref = sm + kBfgsVectors * a.maxN;  // ETK reference geometry
  const int      tid = threadIdx.x;
  // Work item = one ATTEMPT of one slot. A CTA first works through the slot queue, retrying its own slot while it fails;
  // once the queue is dry it helps slots that are still unfinished by running their NEXT attempts speculatively
  // (attempts are independent: their random streams are functions of (seed, slot, attempt)). The accepted conformer is
  // always the LOWEST successful attempt index, exactly what the sequential retry loop of the reference yields
  // (src/etkdg.cpp:339-394), so a small batch no longer waits on one CTA grinding through a hard molecule.
  __shared__ int                sSlot, sAttempt, sWrite;
  __shared__ unsigned long long sPick;
  int                           mySlot = -1;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      sSlot = -1;
      if (mySlot >= 0 && *reinterpret_cast<volatile int*>(a.slotBest + mySlot) == kNoAttempt) {
        const int at = atomicAdd(a.slotNext + mySlot, 1);
        if (at < a.par.maxAttempts) {
          sSlot    = mySlot;
          sAttempt = at;
        }
      }
      if (sSlot < 0) {
        const int q = atomicAdd(a.queue, 1);
        if (q < a.nSlots) {
          a.ok[q] = 0;
          if (a.attempts) a.attempts[q] = a.par.maxAttempts;
          if (a.energy) a.energy[q] = 0.0;
          __threadfence();
          sSlot    = q;
          sAttempt = atomicAdd(a.slotNext + q, 1);  // 0: nobody can have touched it before
        }
      }
      sPick = ~0ull;
    }
    __syncthreads();
    if (sSlot < 0) {  // queue dry: find an unfinished slot with the fewest attempts handed out
      for (int s = tid; s < a.nSlots; s += kT) {
        const int nx = *reinterpret_cast<volatile int*>(a.slotNext + s);
        if (nx > 0 && nx < a.par.maxAttempts && *reinterpret_cast<volatile int*>(a.slotBest + s) == kNoAttempt &&
            nx - *reinterpret_cast<volatile int*>(a.slotDone + s) < kMaxSpeculation)
          atomicMin(&sPick, static_cast<unsigned long long>(nx) << 32 | static_cast<unsigned>(s));
      }
      __syncthreads();
      if (tid == 0 && sPick != ~0ull) {
        const int s  = static_cast<int>(sPick & 0xffffffffu);
        const int at = atomicAdd(a.slotNext + s, 1);
        if (at < a.par.maxAttempts) {
          sSlot    = s;
          sAttempt = at;
        } else {
          sSlot = -2;  // lost the race for the last attempt: look again
        }
      }
      __syncthreads();
      if (sSlot == -2) continue;
      if (sSlot < 0) break;  // nothing left that another attempt could help
      mySlot = -1;
    } else {
      mySlot = sSlot;
    }
    const int slot = sSlot, attempt = sAttempt;
    const int mol = a.slotMol[slot];
    const int nA  = a.dg.atomCounts[mol];
    const int n   = 4 * nA;
    double    eAccepted = 0.0;
    {
      int failedStage = -1;
      // 0: start coordinates (random box, or the metric-matrix start with the matrix in this CTA's idle Hessian slab)
      if (!initialCoords(a.par, a.dg, mol, nA, slot, attempt, w.pos, sm + a.maxN, reinterpret_cast<double*>(w.H), red)) failedStage = 0;
      // 1: first minimisation
      if (failedStage < 0) {
        const auto        v = ff::Dg<4>::view(a.dg, mol, {1.0, 0.1});
        const BfgsOutcome o = bfgsMinimize<ff::Dg<4>, HT>(v, w, n, a.par.dgIters, a.par.optimizerForceTol, true, a.par.maxRestarts);
        eAccepted           = o.energy;
        if (o.energy / nA >= 0.05) failedStage = 1;
      }
      // 2, 3: tetrahedral + first chirality checks
      if (failedStage < 0 && tetrahedralFails<true>(a.chk.tetrahedral, mol, w.pos, 0.3)) failedStage = 2;
      if (failedStage < 0 && a.par.enforceChirality && chiralityFails(a.chk.chiral, mol, w.pos)) failedStage = 3;
      // 4: fourth-dimension collapse
      if (failedStage < 0) {
        const auto v = ff::Dg<4>::view(a.dg, mol, {0.2, 1.0});
        bfgsMinimize<ff::Dg<4>, HT>(v, w, n, a.par.fourthIters, a.par.optimizerForceTol, true, 0);
      }
      // 5: ETK refinement + planarity
      if (failedStage < 0 && (a.par.useExpTorsions || a.par.useBasicKnowledge)) {
        for (int i = tid; i < n; i += kT) ref[i] = w.pos[i];
        __syncthreads();
        auto v   = ff::Etk::view(a.etk, mol, {a.par.useBasicKnowledge ? 0 : 1, 1});
        v.refPos = ref;
        bfgsMinimize<ff::Etk, HT>(v, w, n, a.par.etkIters, a.par.optimizerForceTol, true, 0);
        if (a.par.useBasicKnowledge && planarityFails(a.etk, a.chk.numImpropers, mol, w.pos, red)) failedStage = 5;
      }
      // 6-10: final checks
      if (failedStage < 0) {
        const unsigned m = finalChecks(a, mol, w.pos, red, true);
        if (m) failedStage = __ffs(m) - 1;
      }
      __syncthreads();
      if (failedStage < 0) {
        // result write under the slot's lock; only a LOWER attempt index than the one already stored may overwrite
        if (tid == 0) {
          while (atomicCAS(a.slotLock + slot, 0, 1) != 0) {}
          __threadfence();
          sWrite = attempt < *reinterpret_cast<volatile int*>(a.slotBest + slot);
        }
        __syncthreads();
        if (sWrite) {
          const int a0 = a.slotAtomStart[slot];
          for (int i = tid; i < nA * 3; i += kT) a.coords[static_cast<size_t>(a0) * 3 + i] = w.pos[(i / 3) * 4 + (i % 3)];
          if (tid == 0) {
            a.ok[slot] = 1;
            if (a.attempts) a.attempts[slot] = attempt + 1;
            if (a.energy) a.energy[slot] = eAccepted;
          }
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
          if (sWrite) atomicExch(a.slotBest + slot, attempt);
          __threadfence();
          atomicExch(a.slotLock + slot, 0);
        }
      } else if (tid == 0 && a.stageFailures) {
        atomicAdd(a.stageFailures + failedStage, 1ull);
      }
      if (tid == 0) {
        atomicAdd(a.slotDone + slot, 1);
        if (a.stats) atomicAdd(a.stats + kStatAttempts, 1ull);
      }
    }
  }
}

// Check-only: evaluates stages 1 (energy per atom), 2, 3, 5 (planarity), 6-10 on given 4-D coordinates.
__global__ void __launch_bounds__(kT) etkdgCheckKernel(const EmbedArgs a, const double* pos4, uint32_t* masks) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[kRed];
  for (int slot = blockIdx.x; slot < a.nSlots; slot += gridDim.x) {
    const int mol = a.slotMol[slot];
    const int nA  = a.dg.atomCounts[mol];
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * nA; i += kT) sm[i] = pos4[static_cast<size_t>(a.slotAtomStart[slot]) * 4 + i];
    __syncthreads();
    unsigned     m = 0;
    const auto   v = ff::Dg<4>::view(a.dg, mol, {1.0, 0.1});
    const double e = energyOf<ff::Dg<4>>(v, sm, red);
    if (e / nA >= 0.05) m |= 1u << 1;
    if (tetrahedralFails<true>(a.chk.tetrahedral, mol, sm, 0.3)) m |= 1u << 2;
    if (a.par.enforceChirality && chiralityFails(a.chk.chiral, mol, sm)) m |= 1u << 3;
    if (a.par.useBasicKnowledge && planarityFails(a.etk, a.chk.numImpropers, mol, sm, red)) m |= 1u << 5;
    m |= finalChecks(a, mol, sm, red, false);
    if (threadIdx.x == 0) masks[slot] = m;
  }
}

// Stage 0 alone (tests, and callers that want the start geometry): one CTA per slot.
__global__ void __launch_bounds__(kT) initialCoordsKernel(const b200mol_dg_system dg, const b200mol_embed_params par, int nSlots,
                                                        const int32_t* slotMol, const int32_t* slotAtomStart, int attempt,
                                                        double* pos4, int8_t* ok, double* matWs, size_t matStride) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[kRed];
  for (int slot = blockIdx.x; slot < nSlots; slot += gridDim.x) {
    const int mol = slotMol[slot], nA = dg.atomCounts[mol];
    __syncthreads();
    const bool good = initialCoords(par, dg, mol, nA, slot, attempt, sm, sm + 4 * nA, matWs + blockIdx.x * matStride, red);
    double*    out  = pos4 + static_cast<size_t>(slotAtomStart[slot]) * 4;
    for (int i = threadIdx.x; i < 4 * nA; i += kT) out[i] = good ? sm[i] : 0.0;
    if (threadIdx.x == 0) ok[slot] = good ? 1 : 0;
  }
}

void validate(const b200mol_embed_params& p) {
  B200_REQUIRE(p.maxAttempts >= 1, "maxAttempts must be >= 1");
  B200_REQUIRE(p.boxSize > 0.0, "boxSize must be positive");
  B200_REQUIRE(p.dgIters >= 0 && p.fourthIters >= 0 && p.etkIters >= 0 && p.maxRestarts >= 0, "negative iteration count");
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_etkdg_embed(const b200mol_dg_system* dg, const b200mol_etk_system* etk,
                                   const b200mol_etkdg_checks* checks, const b200mol_embed_params* params, int32_t nSlots,
                                   const int32_t* d_slot_mol, const int32_t* d_slot_atom_start, int max_atoms,
                                   double* d_coords, int8_t* d_ok, int32_t* d_attempts, double* d_energy,
                                   uint64_t* d_stage_failures, void* stream) {
  return guarded([&] {
    B200_REQUIRE(dg && etk && checks && params, "null system");
    validate(*params);
    ff::requireSchedule(*dg);
    ff::requireSchedule(*etk);
    if (nSlots <= 0) return;
    B200_REQUIRE(d_slot_mol && d_slot_atom_start && d_coords && d_ok, "null pointer");
    cudaStream_t s    = asStream(stream);
    const int    maxN = 4 * max_atoms;
    const size_t smem = static_cast<size_t>(kBfgsVectors + 1) * maxN * sizeof(double);
    B200_REQUIRE(max_atoms > 0 && smem <= 200 * 1024, "molecule too large for the shared-memory embedder (%d atoms)", max_atoms);
    const bool wide = g_etkdgHessianFp64 != 0;
    static bool configured[kMaxDevices] = {};
    if (!configured[currentDeviceSlot()]) {
      B200_CUDA(cudaFuncSetAttribute(etkdgKernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      B200_CUDA(cudaFuncSetAttribute(etkdgKernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      configured[currentDeviceSlot()] = true;
    }
    int perSm = 0;
    if (wide) B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, etkdgKernel<double>, kT, smem));
    else B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, etkdgKernel<float>, kT, smem));
    B200_REQUIRE(perSm >= 1, "embedding kernel does not fit");
    perSm      = perSm > g_bfgsCtasPerSm ? g_bfgsCtasPerSm : perSm;
    int blocks = smCount() * perSm;
    if (blocks > nSlots) blocks = nSlots;
    const size_t    stride  = static_cast<size_t>(maxN) * (wide ? bfgsLd<double>(maxN) : bfgsLd<float>(maxN));  // elements
    const size_t    hessBytes = stride * blocks * (wide ? sizeof(double) : sizeof(float));
    Scratch<uint8_t> hess(hessBytes, s);
    Scratch<int>    queue(1, s);
    B200_CUDA(cudaMemsetAsync(queue.get(), 0, sizeof(int), s));
    if (d_stage_failures) B200_CUDA(cudaMemsetAsync(d_stage_failures, 0, kNumStages * sizeof(uint64_t), s));
    Scratch<int>    state(static_cast<size_t>(4) * nSlots, s);  // next | best | lock | done
    B200_CUDA(cudaMemsetAsync(state.get(), 0, sizeof(int) * 4 * nSlots, s));
    B200_CUDA(cudaMemsetAsync(state.get() + nSlots, 0x7f, sizeof(int) * nSlots, s));
    EmbedArgs a{*dg, *etk, *checks, *params, nSlots, d_slot_mol, d_slot_atom_start, d_coords, d_ok, d_attempts, d_energy,
                reinterpret_cast<unsigned long long*>(d_stage_failures), hess.get(), stride, queue.get(), maxN,
                state.get(), state.get() + nSlots, state.get() + 2 * static_cast<size_t>(nSlots), state.get() + 3 * static_cast<size_t>(nSlots),
                pathBStats()};
    L2Persist  keep(s, hess.get(), hessBytes, g_bfgsL2Persist != 0);
    PhaseTimer t("etkdg", s);
    if (wide) etkdgKernel<double><<<blocks, kT, smem, s>>>(a);
    else etkdgKernel<float><<<blocks, kT, smem, s>>>(a);
    B200_LAUNCHED();
  });
}

extern "C" int b200mol_etkdg_check(const b200mol_dg_system* dg, const b200mol_etk_system* etk,
                                   const b200mol_etkdg_checks* checks, const b200mol_embed_params* params, int32_t nSlots,
                                   const int32_t* d_slot_mol, const int32_t* d_slot_atom_start, int max_atoms,
                                   const double* d_pos4, uint32_t* d_fail_masks, void* stream) {
  return guarded([&] {
    B200_REQUIRE(dg && etk && checks && params, "null system");
    if (nSlots <= 0) return;
    B200_REQUIRE(d_slot_mol && d_slot_atom_start && d_pos4 && d_fail_masks, "null pointer");
    const size_t smem = static_cast<size_t>(4) * max_atoms * sizeof(double);
    B200_REQUIRE(max_atoms > 0 && smem <= 200 * 1024, "molecule too large (%d atoms)", max_atoms);
    static bool configured[kMaxDevices] = {};
    if (!configured[currentDeviceSlot()]) {
      B200_CUDA(cudaFuncSetAttribute(etkdgCheckKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      configured[currentDeviceSlot()] = true;
    }
    int blocks = smCount() * 4;
    if (blocks > nSlots) blocks = nSlots;
    EmbedArgs a{*dg, *etk, *checks, *params, nSlots, d_slot_mol, d_slot_atom_start, nullptr, nullptr, nullptr, nullptr,
                nullptr, nullptr, 0, nullptr, 4 * max_atoms, nullptr, nullptr, nullptr, nullptr, nullptr};
    etkdgCheckKernel<<<blocks, kT, smem, asStream(stream)>>>(a, d_pos4, d_fail_masks);
    B200_LAUNCHED();
  });
}

extern "C" int b200mol_etkdg_initial_coords(const b200mol_dg_system* dg, const b200mol_embed_params* params, int32_t nSlots,
                                            const int32_t* d_slot_mol, const int32_t* d_slot_atom_start, int max_atoms,
                                            int32_t attempt, double* d_pos4, int8_t* d_ok, void* stream) {
  return guarded([&] {
    B200_REQUIRE(dg && params, "null system");
    validate(*params);
    if (nSlots <= 0) return;
    B200_REQUIRE(d_slot_mol && d_slot_atom_start && d_pos4 && d_ok, "null pointer");
    B200_REQUIRE(attempt >= 0, "negative attempt index");
    cudaStream_t s    = asStream(stream);
    const size_t smem = (static_cast<size_t>(15) * max_atoms + 8) * sizeof(double);
    B200_REQUIRE(max_atoms > 0 && smem <= 200 * 1024, "molecule too large (%d atoms)", max_atoms);
    static bool configured[kMaxDevices] = {};
    if (!configured[currentDeviceSlot()]) {
      B200_CUDA(cudaFuncSetAttribute(initialCoordsKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      configured[currentDeviceSlot()] = true;
    }
    int blocks = smCount() * 2;
    if (blocks > nSlots) blocks = nSlots;
    const size_t    stride = static_cast<size_t>(max_atoms) * max_atoms;
    Scratch<double> mats(params->useMetricStart ? stride * blocks : 0, s);
    initialCoordsKernel<<<blocks, kT, smem, s>>>(*dg, *params, nSlots, d_slot_mol, d_slot_atom_start, attempt, d_pos4, d_ok,
                                                  mats.get(), stride);
    B200_LAUNCHED();
  });
}

#ifdef B200_BFGS_TIMING
extern "C" void b200mol_debug_clocks_etkdg(unsigned long long* out8) { b200::readBfgsClocks(out8); }
#endif
