// Flattened force fields, block-cooperative evaluation for ONE conformer held in shared memory (sm_90a).
//
// Every force field exposes   View (this molecule's term ranges),
//                             eval<false>(view, pos, nullptr, tid, nT) -> this thread's partial energy,
//                             eval<true>(view, pos, acc, tid, nT)      -> gradient contributions into `acc`.
// Energy: threads stride over the CSR term ranges; records are [n][K] int16 indices + [n][P] fp64 parameters, so a warp
// reads one contiguous span per term type. All arithmetic is fp64 (the reference drops to fp32 inside most terms,
// src/forcefields/mmff_kernels_device.cuh:37-107,196-237; its own acceptance bars are looser than north_star's 1e-4).
//
// Gradient: NO atomics. The host orders every table's terms into WAVES: at most 32 consecutive terms that share no atom
// (b200mol_schedule_waves: round-robin-tournament rounds (i + j) mod M for the dense pair tables, first-fit colouring
// for the sparse ones). One warp takes one wave at a time - lane = term - and adds the term's contributions with plain
// shared-memory read-modify-writes into the warp's PRIVATE accumulator (`acc` + warp * accStride); atoms are distinct
// within a wave, waves of a warp are ordered by __syncwarp, and the accumulators are summed in a fixed order afterwards
// (bfgs_device.cuh gradOf). So the gradient - hence a whole minimisation - is bit-reproducible run to run, and the
// gradient pass no longer waits on shared-memory fp64 CAS loops (1.4 per clock and SM measured, 6-8 per pair term:
// that alone was ~4 SM-clocks per term against ~2.5 for the term's arithmetic).
// The reference scatters with global atomicAdd(double) (mmff_kernels_device.cuh, dist_geom_kernels_device.cuh:66-94).
//
// Term math follows RDKit as restated by the reference: MMFF src/forcefields/mmff_kernels_device.cuh:28-661,
// DG/ETK src/forcefields/dist_geom_kernels_device.cuh:37-830 (including RDKit's quirks: chiral/4th-dim gradient
// without the factor 2, 6-fold ETK torsion gradient using V5).
#pragma once
#include "common.cuh"

namespace b200 {
namespace ff {

constexpr double kDeg2Rad = 3.14159265358979323846 / 180.0;
constexpr double kRad2Deg = 180.0 / 3.14159265358979323846;

struct V3 {
  double x, y, z;
};
__device__ __forceinline__ V3 operator-(const V3& a, const V3& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 operator+(const V3& a, const V3& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator*(const V3& a, double s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ V3 operator-(const V3& a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ double dot(const V3& a, const V3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(const V3& a, const V3& b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <int DIM>
__device__ __forceinline__ V3 ld(const double* pos, int a) {
  return {pos[a * DIM], pos[a * DIM + 1], pos[a * DIM + 2]};
}
// plain read-modify-write: the caller owns atom `a` for the duration of the wave (see the header comment)
template <int DIM>
__device__ __forceinline__ void acc(double* grad, int a, const V3& g) {
  grad[a * DIM] += g.x;
  grad[a * DIM + 1] += g.y;
  grad[a * DIM + 2] += g.z;
}
__device__ __forceinline__ double clampd(double v, double lo, double hi) { return fmin(hi, fmax(lo, v)); }
__device__ __forceinline__ bool   isZero(double v) { return v < 1.0e-10 && v > -1.0e-10; }

struct Range {
  int beg, end;    // terms
  int wbeg, wend;  // waves (gradient schedule)
};
__device__ __forceinline__ Range range(const b200mol_term_table& t, int mol) {
  return {t.starts[mol], t.starts[mol + 1], t.molWaves ? t.molWaves[mol] : 0, t.molWaves ? t.molWaves[mol + 1] : 0};
}
__device__ __forceinline__ void emptyRange(Range& r) {
  r.end  = r.beg;
  r.wend = r.wbeg;
}
// One term record in registers: K molecule-local atom indices + P parameters.
template <int K, int P>
struct TermRec {
  int16_t ix[K];
  double  q[P > 0 ? P : 1];
};
template <int K, int P>
__device__ __forceinline__ void loadTerm(const b200mol_term_table& T, int t, TermRec<K, P>& r) {
  if constexpr (K == 2) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(T.idx + 2 * t);
    r.ix[0]          = static_cast<int16_t>(u & 0xffffu);
    r.ix[1]          = static_cast<int16_t>(u >> 16);
  } else if constexpr (K == 4) {
    const uint2 u = *reinterpret_cast<const uint2*>(T.idx + 4 * t);
    r.ix[0] = static_cast<int16_t>(u.x & 0xffffu), r.ix[1] = static_cast<int16_t>(u.x >> 16);
    r.ix[2] = static_cast<int16_t>(u.y & 0xffffu), r.ix[3] = static_cast<int16_t>(u.y >> 16);
  } else {
#pragma unroll
    for (int k = 0; k < K; ++k) r.ix[k] = T.idx[K * t + k];
  }
#pragma unroll
  for (int k = 0; k < P; ++k) r.q[k] = T.par[P * t + k];
}
// Energy mode: thread-strided over the terms. Gradient mode: warp-strided over the waves, lane = term of the wave.
// Both loops keep the NEXT term's record in flight while the current one is evaluated: the records stream from L2 / HBM
// (a molecule's tables are 70-120 KB and ten thousand molecules do not fit L2), and a load-then-use loop paid that
// latency once per term and thread - it, not the arithmetic, set the evaluation time.
#ifndef B200_TERM_PREFETCH
#define B200_TERM_PREFETCH 0  // 0 = load-then-use (default); 1 = prefetch.global.L1 of the next record; 2 = next record in registers
#endif
template <int K, int P>
__device__ __forceinline__ void prefetchTerm(const b200mol_term_table& T, int t) {
  asm volatile("prefetch.global.L1 [%0];" ::"l"(T.idx + K * t));
  if constexpr (P > 0) {
    asm volatile("prefetch.global.L1 [%0];" ::"l"(T.par + P * t));
    if constexpr (P * 8 > 32) asm volatile("prefetch.global.L1 [%0];" ::"l"(T.par + P * t + P - 1));  // a record may straddle lines
  }
}
template <bool GRAD, int K, int P, class F>
__device__ __forceinline__ void forTerms(const b200mol_term_table& T, const Range& r, int tid, int nT, F&& f) {
  constexpr bool kRegs = B200_TERM_PREFETCH == 2 && P <= 4;  // (two records of the fat tables do not fit the register budget)
  constexpr bool kL1   = B200_TERM_PREFETCH == 1;
  TermRec<K, P> cur;
  if constexpr (!GRAD) {
    int t = r.beg + tid;
    if constexpr (kRegs) {
      if (t < r.end) loadTerm<K, P>(T, t, cur);
      while (t < r.end) {
        TermRec<K, P> nxt;
        const int     tn = t + nT;
        if (tn < r.end) loadTerm<K, P>(T, tn, nxt);
        f(cur);
        cur = nxt;
        t   = tn;
      }
    } else {
      for (; t < r.end; t += nT) {
        if constexpr (kL1)
          if (t + nT < r.end) prefetchTerm<K, P>(T, t + nT);
        loadTerm<K, P>(T, t, cur);
        f(cur);
      }
    }
  } else {
    const int warp = tid >> 5, lane = tid & 31, nW = nT >> 5;
    int       w = r.wbeg + warp;
    if constexpr (kRegs) {
      int t = 0, tEnd = 0;
      if (w < r.wend) {
        t    = T.waves[w] + lane;
        tEnd = T.waves[w + 1];
        if (t < tEnd) loadTerm<K, P>(T, t, cur);
      }
      while (w < r.wend) {
        TermRec<K, P> nxt;
        const int     wn = w + nW;
        int           tn = 0, tnEnd = 0;
        if (wn < r.wend) {
          tn    = T.waves[wn] + lane;
          tnEnd = T.waves[wn + 1];
          if (tn < tnEnd) loadTerm<K, P>(T, tn, nxt);
        }
        if (t < tEnd) f(cur);
        __syncwarp();
        cur  = nxt;
        t    = tn;
        tEnd = tnEnd;
        w    = wn;
      }
    } else {
      for (; w < r.wend; w += nW) {
        const int t = T.waves[w] + lane;
        if constexpr (kL1)
          if (w + nW < r.wend) prefetchTerm<K, P>(T, T.waves[w + nW] + lane);  // (a lane past the wave's end prefetches the next wave's head: harmless)
        if (t < T.waves[w + 1]) {
          loadTerm<K, P>(T, t, cur);
          f(cur);
        }
        __syncwarp();
      }
    }
  }
}

// ============================================================================================ restraints
// The four restraint ("constraint") term types of RDKit's MMFF / UFF force fields, shared by both
// (src/forcefields/mmff_kernels_device.cuh:673-1036; specs src/forcefields/forcefield_constraints.h:31-73):
//   distance K2 P3 {minLen, maxLen, k}      flat-bottomed  1/2 k (d - bound)^2
//   position K1 P5 {refX, refY, refZ, maxDispl, k}          1/2 k max(|x - ref| - maxDispl, 0)^2
//   angle    K3 P3 {minDeg, maxDeg, k}      k (theta - bound)^2 in DEGREES (no 1/2)
//   torsion  K4 P3 {minDeg, maxDeg, k}      k (phi - nearest bound)^2, signed dihedral in degrees, periodic
struct RestraintRanges {
  Range dist, pos, angle, torsion;
};
__device__ __forceinline__ double normDeg(double a) {
  a = fmod(a, 360.0);
  if (a < -180.0) a += 360.0;
  else if (a > 180.0) a -= 360.0;
  return a;
}
template <bool GRAD>
__device__ __forceinline__ double restraintTerms(const b200mol_term_table& TD, const b200mol_term_table& TP, const b200mol_term_table& TA,
                                                 const b200mol_term_table& TT, const RestraintRanges& r, const double* pos, double* grad,
                                                 int tid, int nT) {
  double e = 0.0;
  forTerms<GRAD, 2, 3>(TD, r.dist, tid, nT, [&](const TermRec<2, 3>& rec) {
    const V3     d  = ld<3>(pos, rec.ix[0]) - ld<3>(pos, rec.ix[1]);
    const double d2 = dot(d, d), mn = rec.q[0], mx = rec.q[1];
    double       bound;
    if (d2 < mn * mn) bound = mn;
    else if (d2 > mx * mx) bound = mx;
    else return;
    const double dist = sqrt(d2);
    if (!GRAD) {
      e += 0.5 * rec.q[2] * (dist - bound) * (dist - bound);
    } else {
      const V3 g = d * ((dist - bound) * rec.q[2] / fmax(1.0e-8, dist));
      acc<3>(grad, rec.ix[0], g);
      acc<3>(grad, rec.ix[1], -g);
    }
  });
  forTerms<GRAD, 1, 5>(TP, r.pos, tid, nT, [&](const TermRec<1, 5>& rec) {
    const V3     d    = ld<3>(pos, rec.ix[0]) - V3{rec.q[0], rec.q[1], rec.q[2]};
    const double dist = sqrt(dot(d, d));
    if (!GRAD) {
      const double t = fmax(dist - rec.q[3], 0.0);
      e += 0.5 * rec.q[4] * t * t;
    } else {
      if (dist <= rec.q[3]) return;
      acc<3>(grad, rec.ix[0], d * ((dist - rec.q[3]) * rec.q[4] / fmax(dist, 1.0e-8)));
    }
  });
  forTerms<GRAD, 3, 3>(TA, r.angle, tid, nT, [&](const TermRec<3, 3>& rec) {
    const V3     r1 = ld<3>(pos, rec.ix[0]) - ld<3>(pos, rec.ix[1]), r2 = ld<3>(pos, rec.ix[2]) - ld<3>(pos, rec.ix[1]);
    const double l1 = fmax(1.0e-5, dot(r1, r1)), l2 = fmax(1.0e-5, dot(r2, r2));
    const double ang = kRad2Deg * acos(clampd(dot(r1, r2) / sqrt(l1 * l2), -1.0, 1.0));
    const double at  = ang < rec.q[0] ? ang - rec.q[0] : (ang > rec.q[1] ? ang - rec.q[1] : 0.0);
    if (!GRAD) {
      e += rec.q[2] * at * at;
    } else {
      if (isZero(at)) return;
      const V3     rp  = cross(r2, r1);
      const double pre = 2.0 * kRad2Deg * rec.q[2] * at / fmax(1.0e-5, sqrt(dot(rp, rp)));
      const V3     a = cross(r1, rp) * (-pre / l1), b = cross(r2, rp) * (pre / l2);
      acc<3>(grad, rec.ix[0], a);
      acc<3>(grad, rec.ix[1], -(a + b));
      acc<3>(grad, rec.ix[2], b);
    }
  });
  forTerms<GRAD, 4, 3>(TT, r.torsion, tid, nT, [&](const TermRec<4, 3>& rec) {
    const V3     p1 = ld<3>(pos, rec.ix[0]), p2 = ld<3>(pos, rec.ix[1]), p3 = ld<3>(pos, rec.ix[2]), p4 = ld<3>(pos, rec.ix[3]);
    const V3     r0 = p1 - p2, r1 = p3 - p2, r2 = -r1, r3 = p4 - p3;
    const V3     tt0 = cross(r0, r1), tt1 = cross(r2, r3);
    const double d0 = fmax(sqrt(dot(tt0, tt0)), 1.0e-5), d1 = fmax(sqrt(dot(tt1, tt1)), 1.0e-5);
    const V3     t0 = tt0 * (1.0 / d0), t1 = tt1 * (1.0 / d1);
    const double cosPhi = clampd(dot(t0, t1), -1.0, 1.0);
    const V3     mv = cross(t0, r1);
    const double phi = kRad2Deg * -atan2(dot(mv, t1) / fmax(sqrt(dot(mv, mv)), 1.0e-5), cosPhi);
    const double mn = rec.q[0], mx = rec.q[1];
    double       target = phi;
    if (!(phi > mn && phi < mx) && !(phi > mn && mn > mx) && !(phi < mx && mn > mx))
      target = fabs(normDeg(phi - mn)) < fabs(normDeg(phi - mx)) ? mn : mx;
    const double term = normDeg(phi - target);
    if (!GRAD) {
      e += rec.q[2] * term * term;
    } else {
      if (isZero(term)) return;
      const V3     d23v = p2 - p3;
      const double pre  = 2.0 * kRad2Deg * rec.q[2] * term / fmax(sqrt(dot(d23v, d23v)), 1.0e-8);
      const V3     dedt0 = cross(tt0, r2) * (pre / fmax(dot(tt0, tt0), 1.0e-8));
      const V3     dedt1 = cross(tt1, r1) * (pre / fmax(dot(tt1, tt1), 1.0e-8));
      acc<3>(grad, rec.ix[0], cross(r2, dedt0));
      acc<3>(grad, rec.ix[1], cross(p3 - p1, dedt0) - cross(r3, dedt1));
      acc<3>(grad, rec.ix[2], cross(r0, dedt0) + cross(p4 - p2, dedt1));
      acc<3>(grad, rec.ix[3], cross(r2, dedt1));
    }
  });
  return e;
}

// ============================================================================================ MMFF94
struct Mmff {
  static constexpr int  kDim    = 3;
  static constexpr bool kHasRef = false;
  using System            = b200mol_mmff_system;
  struct Params {};
  struct View {
    const System*   s;
    Range           bond, angle, strbend, oop, torsion, vdw, ele;
    RestraintRanges rs;
  };
  __device__ static View view(const System& s, int mol, const Params&) {
    return {&s,          range(s.bond, mol),    range(s.angle, mol), range(s.strbend, mol),
            range(s.oop, mol), range(s.torsion, mol), range(s.vdw, mol),   range(s.ele, mol),
            {range(s.distc, mol), range(s.posc, mol), range(s.anglec, mol), range(s.torsc, mol)}};
  }

  // bytes of this molecule's term records (K int16 + P fp64 each): the T of SURVEY.md 8d's per-iteration figure
  __device__ static unsigned termBytes(const View& v) {
    return (v.bond.end - v.bond.beg) * 20u + (v.angle.end - v.angle.beg) * 30u + (v.strbend.end - v.strbend.beg) * 46u +
           (v.oop.end - v.oop.beg) * 16u + (v.torsion.end - v.torsion.beg) * 32u + (v.vdw.end - v.vdw.beg) * 20u +
           (v.ele.end - v.ele.beg) * 28u;
  }
  template <bool GRAD>
  __device__ static double eval(const View& v, const double* pos, double* grad, int tid, int nT) {
    const System& s = *v.s;
    double        e = 0.0;
    // ---- bond stretch ----
    forTerms<GRAD, 2, 2>(s.bond, v.bond, tid, nT, [&](const TermRec<2, 2>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double r0 = rec.q[0], kb = rec.q[1];
      const V3     d    = ld<3>(pos, i) - ld<3>(pos, j);
      const double dist = sqrt(dot(d, d)), dr = dist - r0;
      constexpr double cs = -2.0;
      if (!GRAD) {
        e += 143.9325 / 2.0 * kb * dr * dr * (1.0 + cs * dr + 7.0 / 12.0 * cs * cs * dr * dr);
      } else {
        const double de = 143.9325 * kb * dr * (1.0 + 1.5 * cs * dr + 2.0 * 7.0 / 12.0 * cs * cs * dr * dr);
        const V3     g  = dist > 0.0 ? d * (de / dist) : V3{kb * 0.01, kb * 0.01, kb * 0.01};
        acc<3>(grad, i, g);
        acc<3>(grad, j, -g);
      }
    });
    // ---- angle bend ----
    forTerms<GRAD, 3, 3>(s.angle, v.angle, tid, nT, [&](const TermRec<3, 3>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1], k = rec.ix[2];
      const double theta0 = rec.q[0], ka = rec.q[1];
      const bool   linear = rec.q[2] != 0.0;
      const V3     d1 = ld<3>(pos, i) - ld<3>(pos, j), d2 = ld<3>(pos, k) - ld<3>(pos, j);
      const double l1sq = dot(d1, d1), l2sq = dot(d2, d2), l1 = sqrt(l1sq), l2 = sqrt(l2sq);
      const double cosT = clampd(dot(d1, d2) / (l1 * l2), -1.0, 1.0);
      const double dT   = kRad2Deg * acos(cosT) - theta0;
      if (!GRAD) {
        e += linear ? 143.9325 * ka * (1.0 + cosT)
                    : 0.5 * 143.9325 * kDeg2Rad * kDeg2Rad * ka * dT * dT * (1.0 + (-0.4 * kDeg2Rad) * dT);
      } else {
        const double sinSq = 1.0 - cosT * cosT;
        if (isZero(sinSq) || isZero(l1sq) || isZero(l2sq)) return;
        const double de = linear ? -143.9325 * ka * sqrt(sinSq)
                                 : 143.9325 * kDeg2Rad * ka * dT * (1.0 + (-0.006981317 * 1.5) * dT);
        const double cf = -de / sqrt(sinSq);
        const V3     n1 = d1 * (1.0 / l1), n2 = d2 * (1.0 / l2);
        const V3     a = (n2 - n1 * cosT) * (cf / l1), b = (n1 - n2 * cosT) * (cf / l2);
        acc<3>(grad, i, a);
        acc<3>(grad, j, -(a + b));
        acc<3>(grad, k, b);
      }
    });
    // ---- stretch-bend ----
    forTerms<GRAD, 3, 5>(s.strbend, v.strbend, tid, nT, [&](const TermRec<3, 5>& rec) {
      const int     i = rec.ix[0], j = rec.ix[1], k = rec.ix[2];
      const V3      d1 = ld<3>(pos, i) - ld<3>(pos, j), d2 = ld<3>(pos, k) - ld<3>(pos, j);
      const double  l1 = sqrt(dot(d1, d1)), l2 = sqrt(dot(d2, d2));
      const double  cosT = clampd(dot(d1, d2) / (l1 * l2), -1.0, 1.0);
      const double  dT = kRad2Deg * acos(cosT) - rec.q[0], dr1 = l1 - rec.q[1], dr2 = l2 - rec.q[2];
      if (!GRAD) {
        e += 2.51210 * dT * (dr1 * rec.q[3] + dr2 * rec.q[4]);
      } else {
        constexpr double pre = 143.9325 * kDeg2Rad;
        const double     invSin = fmin(1.0 / sqrt(1.0 - cosT * cosT), 1.0e8);
        const double     bt = kRad2Deg * (rec.q[3] * dr1 + rec.q[4] * dr2) * invSin;
        const V3         n1 = d1 * (1.0 / l1), n2 = d2 * (1.0 / l2);
        const V3         a = (n2 - n1 * cosT) * (1.0 / l1), b = (n1 - n2 * cosT) * (1.0 / l2);
        acc<3>(grad, i, (n1 * (dT * rec.q[3]) - a * bt) * pre);
        acc<3>(grad, j, ((n1 * rec.q[3] + n2 * rec.q[4]) * (-dT) + (a + b) * bt) * pre);
        acc<3>(grad, k, (n2 * (dT * rec.q[4]) - b * bt) * pre);
      }
    });
    // ---- out-of-plane ----
    forTerms<GRAD, 4, 1>(s.oop, v.oop, tid, nT, [&](const TermRec<4, 1>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1], k = rec.ix[2], l = rec.ix[3];
      const double koop = rec.q[0];
      V3           ji = ld<3>(pos, i) - ld<3>(pos, j), jk = ld<3>(pos, k) - ld<3>(pos, j), jl = ld<3>(pos, l) - ld<3>(pos, j);
      const double li = sqrt(dot(ji, ji)), lk = sqrt(dot(jk, jk)), ll = sqrt(dot(jl, jl));
      ji = ji * (1.0 / li);
      jk = jk * (1.0 / lk);
      jl = jl * (1.0 / ll);
      V3 n = cross(-ji, jk);
      n    = n * (1.0 / sqrt(dot(n, n)));
      const double sinChi = clampd(dot(jl, n), -1.0, 1.0);
      const double chi    = kRad2Deg * asin(sinChi);
      if (!GRAD) {
        e += 0.5 * 143.9325 * kDeg2Rad * kDeg2Rad * koop * chi * chi;
      } else {
        const double cosChiSq = 1.0 - sinChi * sinChi;
        const double invCosChi = cosChiSq > 0.0 ? 1.0 / sqrt(cosChiSq) : 1.0e8;
        const double cosT = clampd(dot(ji, jk), -1.0, 1.0);
        const double invSinT = 1.0 / sqrt(fmax(1.0 - cosT * cosT, 1.0e-8));
        const double de = 143.9325 * kDeg2Rad * koop * chi;
        const V3     t1 = cross(jl, jk), t2 = cross(ji, jl), t3 = cross(jk, ji);
        const double term1 = invCosChi * invSinT, term2 = sinChi * invCosChi * invSinT * invSinT;
        const V3     g1 = (t1 * term1 - (ji - jk * cosT) * term2) * (1.0 / li);
        const V3     g3 = (t2 * term1 - (jk - ji * cosT) * term2) * (1.0 / lk);
        const V3     g4 = (t3 * term1 - jl * (sinChi * invCosChi)) * (1.0 / ll);
        acc<3>(grad, i, g1 * de);
        acc<3>(grad, j, (g1 + g3 + g4) * (-de));
        acc<3>(grad, k, g3 * de);
        acc<3>(grad, l, g4 * de);
      }
    });
    // ---- torsion ----
    forTerms<GRAD, 4, 3>(s.torsion, v.torsion, tid, nT, [&](const TermRec<4, 3>& rec) {
      const double   V1 = rec.q[0], V2 = rec.q[1], V3c = rec.q[2];
      const V3       d1 = ld<3>(pos, rec.ix[0]) - ld<3>(pos, rec.ix[1]), d2 = ld<3>(pos, rec.ix[2]) - ld<3>(pos, rec.ix[1]),
               d4 = ld<3>(pos, rec.ix[3]) - ld<3>(pos, rec.ix[2]);
      V3           c1 = cross(d1, d2), c2 = cross(-d2, d4);
      const double n1 = 1.0 / sqrt(dot(c1, c1)), n2 = 1.0 / sqrt(dot(c2, c2));
      if (!GRAD) {
        const double cosPhi = clampd(dot(c1, c2) * n1 * n2, -1.0, 1.0);
        const double phi    = acos(cosPhi);
        e += 0.5 * (V1 * (1.0 + cosPhi) + V2 * (1.0 - cos(2.0 * phi)) + V3c * (1.0 + cos(3.0 * phi)));
      } else {
        const double i1 = fmin(n1, 1.0e5), i2 = fmin(n2, 1.0e5);
        c1 = c1 * i1;
        c2 = c2 * i2;
        const double cosPhi = clampd(dot(c1, c2), -1.0, 1.0);
        const double sinSq  = 1.0 - cosPhi * cosPhi;
        double       sinTerm = 0.0;
        if (sinSq > 0.0) sinTerm = 0.5 * (V1 - 2.0 * V2 * (2.0 * cosPhi) + 3.0 * V3c * (3.0 - 4.0 * sinSq));
        const V3 a = (c2 - c1 * cosPhi) * i1, b = (c1 - c2 * cosPhi) * i2;
        acc<3>(grad, rec.ix[0], V3{a.z * d2.y - a.y * d2.z, a.x * d2.z - a.z * d2.x, a.y * d2.x - a.x * d2.y} * sinTerm);
        acc<3>(grad, rec.ix[1],
               V3{a.y * (d2.z - d1.z) + a.z * (d1.y - d2.y) + b.y * (-d4.z) + b.z * (d4.y),
                  a.x * (d1.z - d2.z) + a.z * (d2.x - d1.x) + b.x * (d4.z) + b.z * (-d4.x),
                  a.x * (d2.y - d1.y) + a.y * (d1.x - d2.x) + b.x * (-d4.y) + b.y * (d4.x)} * sinTerm);
        acc<3>(grad, rec.ix[2],
               V3{a.y * (d1.z) + a.z * (-d1.y) + b.y * (d4.z + d2.z) + b.z * (-d4.y - d2.y),
                  a.x * (-d1.z) + a.z * (d1.x) + b.x * (-d4.z - d2.z) + b.z * (d4.x + d2.x),
                  a.x * (d1.y) + a.y * (-d1.x) + b.x * (d4.y + d2.y) + b.y * (-d4.x - d2.x)} * sinTerm);
        acc<3>(grad, rec.ix[3],
               V3{b.y * (-d2.z) - b.z * (-d2.y), b.z * (-d2.x) - b.x * (-d2.z), b.x * (-d2.y) - b.y * (-d2.x)} * sinTerm);
      }
    });
    // ---- buffered 14-7 van der Waals ----
    forTerms<GRAD, 2, 2>(s.vdw, v.vdw, tid, nT, [&](const TermRec<2, 2>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double R = rec.q[0], eps = rec.q[1];
      const V3     d    = ld<3>(pos, i) - ld<3>(pos, j);
      const double d2   = dot(d, d), dist = sqrt(d2);
      if (!GRAD) {
        const double R2 = R * R, R7 = R2 * R2 * R2 * R, dist7 = d2 * d2 * d2 * dist;
        const double t1 = 1.07 * R / (dist + 0.07 * R), t1sq = t1 * t1, t17 = t1sq * t1sq * t1sq * t1;
        e += eps * t17 * (1.12 * R7 / (dist7 + 0.12 * R7) - 2.0);
      } else {
        const double q = dist / R, q2 = q * q, q6 = q2 * q2 * q2, q7p = q6 * q + 0.12;
        const double tt = 1.07 / (q + 0.07), tt2 = tt * tt, t7 = tt2 * tt2 * tt2 * tt;
        const double de = eps / R * t7 * (-1.12 * 7.0 * q6 / (q7p * q7p) + ((-1.12 * 7.0 / q7p + 14.0) / (q + 0.07)));
        const V3     g  = dist <= 0.0 ? V3{R * 0.01, R * 0.01, R * 0.01} : d * (de / dist);
        acc<3>(grad, i, g);
        acc<3>(grad, j, -g);
      }
    });
    // ---- buffered Coulomb ----
    forTerms<GRAD, 2, 3>(s.ele, v.ele, tid, nT, [&](const TermRec<2, 3>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double ct = rec.q[0];
      const bool   sq = rec.q[1] == 2.0, is14 = rec.q[2] != 0.0;
      const V3     d    = ld<3>(pos, i) - ld<3>(pos, j);
      const double dist = sqrt(dot(d, d)), rb = dist + 0.05;
      if (!GRAD) {
        double en = 332.0716 * ct / (sq ? rb * rb : rb);
        if (is14) en *= 0.75;
        e += en;
      } else {
        double de = sq ? -2.0 * 332.0716 * ct / (rb * rb * rb) : -332.0716 * ct / (rb * rb);
        if (is14) de *= 0.75;
        const V3 g = d * (de / dist);
        acc<3>(grad, i, g);
        acc<3>(grad, j, -g);
      }
    });
    e += restraintTerms<GRAD>(s.distc, s.posc, s.anglec, s.torsc, v.rs, pos, grad, tid, nT);
    return e;
  }
};

// ============================================================================================ distance geometry
template <int DIM>
struct Dg {
  static constexpr int  kDim    = DIM;
  static constexpr bool kHasRef = false;
  using System            = b200mol_dg_system;
  struct Params {
    double chiralWeight, fourthWeight;
  };
  struct View {
    const System* s;
    Range         dist, chiral, fourth;
    double        cw, fw;
  };
  __device__ static View view(const System& s, int mol, const Params& p) {
    return {&s, range(s.dist, mol), range(s.chiral, mol), range(s.fourth, mol), p.chiralWeight, p.fourthWeight};
  }
  __device__ static unsigned termBytes(const View& v) {
    return (v.dist.end - v.dist.beg) * 28u + (v.chiral.end - v.chiral.beg) * 24u + (v.fourth.end - v.fourth.beg) * 2u;
  }
  template <bool GRAD>
  __device__ static double eval(const View& v, const double* pos, double* grad, int tid, int nT) {
    const System& s = *v.s;
    double        e = 0.0;
    forTerms<GRAD, 2, 3>(s.dist, v.dist, tid, nT, [&](const TermRec<2, 3>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double lb2 = rec.q[0], ub2 = rec.q[1], w = rec.q[2];
      double       dd[DIM], d2 = 0.0;
#pragma unroll
      for (int c = 0; c < DIM; ++c) {
        dd[c] = pos[i * DIM + c] - pos[j * DIM + c];
        d2 += dd[c] * dd[c];
      }
      if (d2 > ub2) {
        const double val = d2 / ub2 - 1.0;
        if (!GRAD) {
          if (val > 0.0) e += w * val * val;
        } else {
          const double pre = w * 4.0 * val / ub2;
#pragma unroll
          for (int c = 0; c < DIM; ++c) {
            grad[i * DIM + c] += pre * dd[c];
            grad[j * DIM + c] -= pre * dd[c];
          }
        }
      } else if (d2 < lb2) {
        const double l2d2 = d2 + lb2;
        if (!GRAD) {
          const double val = 2.0 * lb2 / l2d2 - 1.0;
          if (val > 0.0) e += w * val * val;
        } else {
          const double pre = w * 8.0 * lb2 * (1.0 - 2.0 * lb2 / l2d2) / (l2d2 * l2d2);
#pragma unroll
          for (int c = 0; c < DIM; ++c) {
            grad[i * DIM + c] += pre * dd[c];
            grad[j * DIM + c] -= pre * dd[c];
          }
        }
      }
    });
    forTerms<GRAD, 4, 2>(s.chiral, v.chiral, tid, nT, [&](const TermRec<4, 2>& rec) {
      const double   ub = rec.q[0], lb = rec.q[1];
      const V3       p1 = ld<DIM>(pos, rec.ix[0]), p2 = ld<DIM>(pos, rec.ix[1]), p3 = ld<DIM>(pos, rec.ix[2]), p4 = ld<DIM>(pos, rec.ix[3]);
      const V3       v1 = p1 - p4, v2 = p2 - p4, v3 = p3 - p4;
      const double   vol = dot(v1, cross(v2, v3));
      double         diff;
      if (vol < lb) diff = vol - lb;
      else if (vol > ub) diff = vol - ub;
      else return;
      if (!GRAD) {
        e += v.cw * diff * diff;
      } else {
        const double pre = v.cw * diff;  // RDKit: no factor 2
        acc<DIM>(grad, rec.ix[0], cross(v2, v3) * pre);
        acc<DIM>(grad, rec.ix[1], cross(v3, v1) * pre);
        acc<DIM>(grad, rec.ix[2], V3{v2.z * v1.y - v2.y * v1.z, v2.x * v1.z - v2.z * v1.x, v2.y * v1.x - v2.x * v1.y} * pre);
        acc<DIM>(grad, rec.ix[3],
                 V3{p1.z * (p2.y - p3.y) + p2.z * (p3.y - p1.y) + p3.z * (p1.y - p2.y),
                    p1.x * (p2.z - p3.z) + p2.x * (p3.z - p1.z) + p3.x * (p1.z - p2.z),
                    p1.y * (p2.x - p3.x) + p2.y * (p3.x - p1.x) + p3.y * (p1.x - p2.x)} * pre);
      }
    });
    if constexpr (DIM == 4) {
      forTerms<GRAD, 1, 0>(s.fourth, v.fourth, tid, nT, [&](const TermRec<1, 0>& rec) {
        const int    a  = rec.ix[0];
        const double w4 = pos[a * 4 + 3];
        if (!GRAD) e += v.fw * w4 * w4;
        else grad[a * 4 + 3] += v.fw * w4;  // RDKit: no factor 2
      });
    }
    return e;
  }
};

// ============================================================================================ ETK (4-D storage)
struct Etk {
  static constexpr int  kDim    = 4;
  static constexpr bool kHasRef = true;
  using System                  = b200mol_etk_system;
  struct Params {
    int plain;     // 1 = skip improper terms (ETDG variant)
    int recentre;  // 1 = re-centre the 1-2 / free 1-3 windows on the reference (= starting) geometry
  };
  struct View {
    const System* s;
    Range         torsion, improper, d12, d13, a13, lr;
    const double* refPos;  // reference coordinates for the window refresh, or nullptr
  };
  __device__ static View view(const System& s, int mol, const Params& p) {
    Range imp = range(s.improper, mol);
    if (p.plain) emptyRange(imp);
    return {&s, range(s.torsion, mol), imp, range(s.dist12, mol), range(s.dist13, mol), range(s.angle13, mol),
            range(s.longrange, mol), nullptr};
  }
  __device__ static unsigned termBytes(const View& v) {
    return (v.torsion.end - v.torsion.beg) * 104u + (v.improper.end - v.improper.beg) * 40u + (v.d12.end - v.d12.beg) * 36u +
           (v.d13.end - v.d13.beg) * 36u + (v.a13.end - v.a13.beg) * 22u + (v.lr.end - v.lr.beg) * 28u;
  }

  // Flat-bottom distance terms. P = 4 {min, max, k, fixed}: with a reference geometry the window of every term whose
  // `fixed` flag is 0 is re-centred on the reference distance keeping its half-width (ETK stage refresh,
  // src/etkdg_stage_etk_minimization.cu:32-64,176-202); long-range terms (P = 3) are never refreshed.
  template <bool GRAD, int P>
  __device__ static double distTerms(const b200mol_term_table& T, Range r, const double* pos, double* grad, int tid, int nT,
                                     const double* refPos) {
    double e = 0.0;
    forTerms<GRAD, 2, P>(T, r, tid, nT, [&](const TermRec<2, P>& rec) {
      const int i = rec.ix[0], j = rec.ix[1];
      double    mn = rec.q[0], mx = rec.q[1];
      const double fk = rec.q[2];
      if (P == 4 && refPos && rec.q[3] == 0.0) {
        const V3     rd   = ld<4>(refPos, i) - ld<4>(refPos, j);
        const double dref = sqrt(dot(rd, rd)), half = (mx - mn) / 2.0;
        mn                = dref - half;
        mx                = dref + half;
      }
      const V3     d  = ld<4>(pos, i) - ld<4>(pos, j);
      const double d2 = dot(d, d);
      double       ref;
      if (d2 < mn * mn) ref = mn;
      else if (d2 > mx * mx) ref = mx;
      else return;
      const double dist = sqrt(d2);
      if (!GRAD) {
        e += 0.5 * fk * (dist - ref) * (dist - ref);
      } else {
        const V3 g = d * (fk * (dist - ref) / fmax(1.0e-8, dist));
        acc<4>(grad, i, g);
        acc<4>(grad, j, -g);
      }
    });
    return e;
  }

  template <bool GRAD>
  __device__ static double eval(const View& v, const double* pos, double* grad, int tid, int nT) {
    const System& s = *v.s;
    double        e = 0.0;
    forTerms<GRAD, 4, 12>(s.torsion, v.torsion, tid, nT, [&](const TermRec<4, 12>& rec) {
      const double*  fc = rec.q;
      const double*  sg = fc + 6;
      const V3       p1 = ld<4>(pos, rec.ix[0]), p2 = ld<4>(pos, rec.ix[1]), p3 = ld<4>(pos, rec.ix[2]), p4 = ld<4>(pos, rec.ix[3]);
      const V3       r1 = p1 - p2, r2 = p3 - p2, r3 = p2 - p3, r4 = p4 - p3;
      V3             t0 = cross(r1, r2), t1 = cross(r3, r4);
      const double   d02 = dot(t0, t0), d12 = dot(t1, t1);
      if (!GRAD) {
        const double comb = d02 * d12;
        const double c    = isZero(comb) ? 0.0 : clampd(dot(t0, t1) / sqrt(comb), -1.0, 1.0);
        const double c2 = c * c, c3 = c * c2, c4 = c * c3, c5 = c * c4, c6 = c * c5;
        e += fc[0] * (1.0 + sg[0] * c) + fc[1] * (1.0 + sg[1] * (2.0 * c2 - 1.0)) +
             fc[2] * (1.0 + sg[2] * (4.0 * c3 - 3.0 * c)) + fc[3] * (1.0 + sg[3] * (8.0 * c4 - 8.0 * c2 + 1.0)) +
             fc[4] * (1.0 + sg[4] * (16.0 * c5 - 20.0 * c3 + 5.0 * c)) +
             fc[5] * (1.0 + sg[5] * (32.0 * c6 - 48.0 * c4 + 18.0 * c2 - 1.0));
      } else {
        if (isZero(d02) || isZero(d12)) return;
        const double i0 = 1.0 / sqrt(d02), i1 = 1.0 / sqrt(d12);
        t0 = t0 * i0;
        t1 = t1 * i1;
        const double cp = clampd(dot(t0, t1), -1.0, 1.0);
        const double sSq = 1.0 - cp * cp, sp = sSq > 0.0 ? sqrt(sSq) : 0.0;
        const double q2 = cp * cp, q3 = cp * q2, q4 = cp * q3, q5 = cp * q4;
        const double dE = (-fc[0] * sg[0] * sp - 2.0 * fc[1] * sg[1] * (2.0 * cp * sp) -
                           3.0 * fc[2] * sg[2] * (4.0 * q2 * sp - sp) - 4.0 * fc[3] * sg[3] * (8.0 * q3 * sp - 4.0 * cp * sp) -
                           5.0 * fc[4] * sg[4] * (16.0 * q4 * sp - 12.0 * q2 * sp + sp) -
                           6.0 * fc[4] * sg[4] * (32.0 * q5 * sp - 32.0 * q3 * sp + 6.0 * sp));  // V5 twice: RDKit quirk
        const double sinTerm = -dE * (isZero(sp) ? 1.0 / cp : 1.0 / sp);
        const V3     a = (t1 - t0 * cp) * i0, b = (t0 - t1 * cp) * i1;
        acc<4>(grad, rec.ix[0], V3{a.z * r2.y - a.y * r2.z, a.x * r2.z - a.z * r2.x, a.y * r2.x - a.x * r2.y} * sinTerm);
        acc<4>(grad, rec.ix[3], V3{b.y * r3.z - b.z * r3.y, b.z * r3.x - b.x * r3.z, b.x * r3.y - b.y * r3.x} * sinTerm);
        acc<4>(grad, rec.ix[1],
               V3{a.y * (r2.z - r1.z) + a.z * (r1.y - r2.y) + b.y * (-r4.z) + b.z * (r4.y),
                  a.x * (r1.z - r2.z) + a.z * (r2.x - r1.x) + b.x * (r4.z) + b.z * (-r4.x),
                  a.x * (r2.y - r1.y) + a.y * (r1.x - r2.x) + b.x * (-r4.y) + b.y * (r4.x)} * sinTerm);
        acc<4>(grad, rec.ix[2],
               V3{a.y * r1.z + a.z * (-r1.y) + b.y * (r4.z - r3.z) + b.z * (r3.y - r4.y),
                  a.x * (-r1.z) + a.z * r1.x + b.x * (r3.z - r4.z) + b.z * (r4.x - r3.x),
                  a.x * r1.y + a.y * (-r1.x) + b.x * (r4.y - r3.y) + b.y * (r3.x - r4.x)} * sinTerm);
      }
    });
    forTerms<GRAD, 4, 4>(s.improper, v.improper, tid, nT, [&](const TermRec<4, 4>& rec) {
      const double   C0 = rec.q[0], C1 = rec.q[1], C2 = rec.q[2],
                   fk = rec.q[3];
      const V3     ji = ld<4>(pos, rec.ix[0]) - ld<4>(pos, rec.ix[1]), jk = ld<4>(pos, rec.ix[2]) - ld<4>(pos, rec.ix[1]),
               jl = ld<4>(pos, rec.ix[3]) - ld<4>(pos, rec.ix[1]);
      const double l2i = dot(ji, ji), l2k = dot(jk, jk), l2l = dot(jl, jl);
      if (!GRAD) {
        double cosY = 0.0;
        if (!(l2i < 1.0e-16 || l2k < 1.0e-16 || l2l < 1.0e-16)) {
          const V3     n   = cross(ji, jk) * (1.0 / sqrt(l2i * l2k));
          const double l2n = dot(n, n);
          if (!(l2n < 1.0e-16)) cosY = dot(n, jl) / sqrt(l2l) / sqrt(l2n);
        }
        const double sSq = 1.0 - cosY * cosY, sinY = sSq > 0.0 ? sqrt(sSq) : 0.0;
        e += fk * (C0 + C1 * sinY + C2 * (2.0 * sinY * sinY - 1.0));
      } else {
        if (isZero(l2i) || isZero(l2k) || isZero(l2l)) return;
        const double ii = 1.0 / sqrt(l2i), ik = 1.0 / sqrt(l2k), il = 1.0 / sqrt(l2l);
        const V3     a = ji * ii, b = jk * ik, c = jl * il;
        V3           n = cross(-a, b);
        n              = n * (1.0 / sqrt(dot(n, n)));
        const double cY = clampd(dot(n, c), -1.0, 1.0), sY = fmax(sqrt(1.0 - cY * cY), 1.0e-8);
        const double cT = clampd(dot(a, b), -1.0, 1.0), sTsq = 1.0 - cT * cT, sT = fmax(sqrt(sTsq), 1.0e-8);
        const double dE = -fk * (C1 * cY - 4.0 * C2 * cY * sY);
        const V3     t1 = cross(c, b), t2 = cross(a, c), t3 = cross(b, a);
        const double inv1 = 1.0 / (sY * sT), term2 = cY / (sY * sTsq), cOs = cY / sY;
        const V3     g1 = (t1 * inv1 - (a - b * cT) * term2) * ii;
        const V3     g3 = (t2 * inv1 - (b - a * cT) * term2) * ik;
        const V3     g4 = (t3 * inv1 - c * cOs) * il;
        acc<4>(grad, rec.ix[0], g1 * dE);
        acc<4>(grad, rec.ix[1], (g1 + g3 + g4) * (-dE));
        acc<4>(grad, rec.ix[2], g3 * dE);
        acc<4>(grad, rec.ix[3], g4 * dE);
      }
    });
    e += distTerms<GRAD, 4>(s.dist12, v.d12, pos, grad, tid, nT, v.refPos);
    e += distTerms<GRAD, 4>(s.dist13, v.d13, pos, grad, tid, nT, v.refPos);
    e += distTerms<GRAD, 3>(s.longrange, v.lr, pos, grad, tid, nT, nullptr);
    forTerms<GRAD, 3, 2>(s.angle13, v.a13, tid, nT, [&](const TermRec<3, 2>& rec) {
      const double   mn = rec.q[0], mx = rec.q[1];
      const V3       r1 = ld<4>(pos, rec.ix[0]) - ld<4>(pos, rec.ix[1]), r2 = ld<4>(pos, rec.ix[2]) - ld<4>(pos, rec.ix[1]);
      const double   l1 = dot(r1, r1), l2 = dot(r2, r2);
      if (!GRAD) {
        if (isZero(l1 * l2)) return;
        const double ang = kRad2Deg * acos(clampd(dot(r1, r2) / sqrt(l1 * l2), -1.0, 1.0));
        const double at  = ang < mn ? ang - mn : (ang > mx ? ang - mx : 0.0);
        e += at * at;
      } else {
        const double m1 = fmax(1.0e-5, l1), m2 = fmax(1.0e-5, l2);
        const double ang = kRad2Deg * acos(clampd(dot(r1, r2) / sqrt(m1 * m2), -1.0, 1.0));
        const double at  = ang < mn ? ang - mn : (ang > mx ? ang - mx : 0.0);
        const double dE  = 2.0 * kRad2Deg * at;
        const V3     rp  = cross(r2, r1);
        const double pre = dE / sqrt(fmax(dot(rp, rp), 1.0e-10));
        const V3     a = cross(r1, rp) * (-pre / m1), b = cross(r2, rp) * (pre / m2);
        acc<4>(grad, rec.ix[0], a);
        acc<4>(grad, rec.ix[1], -(a + b));
        acc<4>(grad, rec.ix[2], b);
      }
    });
    return e;
  }
};

// ============================================================================================ UFF
// Term math: src/forcefields/uff_kernels_device.cuh:37-590 (RDKit ForceFields::UFF contribs).
struct Uff {
  static constexpr int  kDim    = 3;
  static constexpr bool kHasRef = false;
  using System                  = b200mol_uff_system;
  struct Params {};
  struct View {
    const System*   s;
    Range           bond, angle, torsion, inversion, vdw;
    RestraintRanges rs;
  };
  __device__ static View view(const System& s, int mol, const Params&) {
    return {&s, range(s.bond, mol), range(s.angle, mol), range(s.torsion, mol), range(s.inversion, mol), range(s.vdw, mol),
            {range(s.distc, mol), range(s.posc, mol), range(s.anglec, mol), range(s.torsc, mol)}};
  }
  __device__ static unsigned termBytes(const View& v) {
    return (v.bond.end - v.bond.beg) * 20u + (v.angle.end - v.angle.beg) * 54u + (v.torsion.end - v.torsion.beg) * 32u +
           (v.inversion.end - v.inversion.beg) * 40u + (v.vdw.end - v.vdw.beg) * 28u;
  }
  template <bool GRAD>
  __device__ static double eval(const View& v, const double* pos, double* grad, int tid, int nT) {
    const System& s = *v.s;
    double        e = 0.0;
    forTerms<GRAD, 2, 2>(s.bond, v.bond, tid, nT, [&](const TermRec<2, 2>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double r0 = rec.q[0], k = rec.q[1];
      const V3     d    = ld<3>(pos, i) - ld<3>(pos, j);
      const double dist = sqrt(dot(d, d));
      if (!GRAD) {
        e += 0.5 * k * (dist - r0) * (dist - r0);
      } else {
        const V3 g = dist > 0.0 ? d * (k * (dist - r0) / dist) : V3{k * 0.01, k * 0.01, k * 0.01};
        acc<3>(grad, i, g);
        acc<3>(grad, j, -g);
      }
    });
    forTerms<GRAD, 3, 6>(s.angle, v.angle, tid, nT, [&](const TermRec<3, 6>& rec) {
      const int     i = rec.ix[0], j = rec.ix[1], k = rec.ix[2];
      const int     order = static_cast<int>(rec.q[2]);
      const V3      d1 = ld<3>(pos, i) - ld<3>(pos, j), d2 = ld<3>(pos, k) - ld<3>(pos, j);
      const double  l1sq = dot(d1, d1), l2sq = dot(d2, d2);
      if (l1sq <= 0.0 || l2sq <= 0.0) return;
      const double l1 = sqrt(l1sq), l2 = sqrt(l2sq);
      const double c  = clampd(dot(d1, d2) / (l1 * l2), -1.0, 1.0);
      const double sSq = 1.0 - c * c;
      const bool   corr = order > 0 && order < 5 && c > 0.8660;
      if (!GRAD) {
        const double c2t = c * c - sSq;
        double       term;
        if (order == 0) {
          term = rec.q[3] + rec.q[4] * c + rec.q[5] * c2t;
        } else {
          double r = 0.0;
          if (order == 1) r = -c;
          else if (order == 2) r = c2t;
          else if (order == 3) r = c * (c * c - 3.0 * sSq);
          else if (order == 4) r = c * c * c * c - 6.0 * c * c * sSq + sSq * sSq;
          term = (1.0 - r) / static_cast<double>(order * order);
        }
        double en = rec.q[1] * term;
        if (corr) en += exp(-20.0 * (acos(c) - rec.q[0] + 0.25));
        e += en;
      } else {
        if (isZero(sSq)) return;
        const double sn = fmax(sqrt(sSq), 1.0e-8), s2t = 2.0 * sn * c;
        double       dE;
        if (order == 0) {
          dE = -rec.q[1] * (rec.q[4] * sn + 2.0 * rec.q[5] * s2t);
        } else {
          double r = 0.0;
          if (order == 1) r = -sn;
          else if (order == 2) r = s2t;
          else if (order == 3) r = sn * (3.0 - 4.0 * sn * sn);
          else if (order == 4) r = c * sn * (4.0 - 8.0 * sn * sn);
          dE = (order >= 1 && order <= 4) ? r * rec.q[1] / static_cast<double>(order) : 0.0;
        }
        if (corr) dE += -20.0 * exp(-20.0 * (acos(c) - rec.q[0] + 0.25));
        const double cf = dE / (-sn);
        const V3     n1 = d1 * (1.0 / l1), n2 = d2 * (1.0 / l2);
        const V3     a = (n2 - n1 * c) * (cf / l1), b = (n1 - n2 * c) * (cf / l2);
        acc<3>(grad, i, a);
        acc<3>(grad, j, -(a + b));
        acc<3>(grad, k, b);
      }
    });
    forTerms<GRAD, 4, 3>(s.torsion, v.torsion, tid, nT, [&](const TermRec<4, 3>& rec) {
      const double   fk = rec.q[0], cosTerm = rec.q[2];
      const int      order = static_cast<int>(rec.q[1]);
      const V3       r0 = ld<3>(pos, rec.ix[0]) - ld<3>(pos, rec.ix[1]), r1 = ld<3>(pos, rec.ix[2]) - ld<3>(pos, rec.ix[1]), r2 = -r1,
               r3 = ld<3>(pos, rec.ix[3]) - ld<3>(pos, rec.ix[2]);
      V3           t0 = cross(r0, r1), t1 = cross(r2, r3);
      const double d0 = sqrt(dot(t0, t0)), d1 = sqrt(dot(t1, t1));
      if (!GRAD) {
        const double c = (isZero(d0) || isZero(d1)) ? 0.0 : clampd(dot(t0, t1) / (d0 * d1), -1.0, 1.0);
        const double sSq = 1.0 - c * c;
        double       cn;
        if (order == 2) cn = 1.0 - 2.0 * sSq;
        else if (order == 3) cn = c * (c * c - 3.0 * sSq);
        else if (order == 6) cn = 1.0 + sSq * (-32.0 * sSq * sSq + 48.0 * sSq - 18.0);
        else return;
        e += fk / 2.0 * (1.0 - cosTerm * cn);
      } else {
        if (isZero(d0) || isZero(d1)) return;
        t0 = t0 * (1.0 / d0);
        t1 = t1 * (1.0 / d1);
        const double c = clampd(dot(t0, t1), -1.0, 1.0), sSq = 1.0 - c * c, sn = sSq > 0.0 ? sqrt(sSq) : 0.0;
        double       r;
        if (order == 2) r = 2.0 * sn * c;
        else if (order == 3) r = sn * (3.0 - 4.0 * sSq);
        else if (order == 6) r = c * sn * (32.0 * sSq * (sSq - 1.0) + 6.0);
        else return;
        const double dE = r * fk / 2.0 * cosTerm * -1.0 * static_cast<double>(order);
        const double sinTerm = dE * (isZero(sn) ? (1.0 / fmax(fabs(c), 1.0e-8)) : (1.0 / sn));
        const V3     a = (t1 - t0 * c) * (1.0 / d0), b = (t0 - t1 * c) * (1.0 / d1);
        acc<3>(grad, rec.ix[0], V3{a.z * r1.y - a.y * r1.z, a.x * r1.z - a.z * r1.x, a.y * r1.x - a.x * r1.y} * sinTerm);
        acc<3>(grad, rec.ix[1],
               V3{a.y * (r1.z - r0.z) + a.z * (r0.y - r1.y) + b.y * (-r3.z) + b.z * (r3.y),
                  a.x * (r0.z - r1.z) + a.z * (r1.x - r0.x) + b.x * (r3.z) + b.z * (-r3.x),
                  a.x * (r1.y - r0.y) + a.y * (r0.x - r1.x) + b.x * (-r3.y) + b.y * (r3.x)} * sinTerm);
        acc<3>(grad, rec.ix[2],
               V3{a.y * r0.z + a.z * (-r0.y) + b.y * (r3.z - r2.z) + b.z * (r2.y - r3.y),
                  a.x * (-r0.z) + a.z * r0.x + b.x * (r2.z - r3.z) + b.z * (r3.x - r2.x),
                  a.x * r0.y + a.y * (-r0.x) + b.x * (r3.y - r2.y) + b.y * (r2.x - r3.x)} * sinTerm);
        acc<3>(grad, rec.ix[3], V3{b.y * r2.z - b.z * r2.y, b.z * r2.x - b.x * r2.z, b.x * r2.y - b.y * r2.x} * sinTerm);
      }
    });
    forTerms<GRAD, 4, 4>(s.inversion, v.inversion, tid, nT, [&](const TermRec<4, 4>& rec) {
      const double   fk = rec.q[0], C0 = rec.q[1], C1 = rec.q[2],
                   C2 = rec.q[3];
      const V3     ji = ld<3>(pos, rec.ix[0]) - ld<3>(pos, rec.ix[1]), jk = ld<3>(pos, rec.ix[2]) - ld<3>(pos, rec.ix[1]),
               jl = ld<3>(pos, rec.ix[3]) - ld<3>(pos, rec.ix[1]);
      const double l2i = dot(ji, ji), l2k = dot(jk, jk), l2l = dot(jl, jl);
      if (!GRAD) {
        double cosY = 0.0;
        if (!(l2i < 1.0e-16 || l2k < 1.0e-16 || l2l < 1.0e-16)) {
          const V3     n   = cross(ji, jk) * (1.0 / (sqrt(l2i) * sqrt(l2k)));
          const double l2n = dot(n, n);
          if (!(l2n < 1.0e-16)) cosY = dot(n, jl) / (sqrt(l2l) * sqrt(l2n));
        }
        const double sSq = 1.0 - cosY * cosY, sinY = sSq > 0.0 ? sqrt(sSq) : 0.0;
        e += fk * (C0 + C1 * sinY + C2 * (2.0 * sinY * sinY - 1.0));
      } else {
        const double dI = sqrt(l2i), dK = sqrt(l2k), dL = sqrt(l2l);
        if (isZero(dI) || isZero(dK) || isZero(dL)) return;
        const V3 a = ji * (1.0 / dI), b = jk * (1.0 / dK), c = jl * (1.0 / dL);
        V3       n = cross(-a, b);
        const double nn = sqrt(dot(n, n));
        if (nn <= 0.0) return;
        n = n * (1.0 / nn);
        const double cY = clampd(dot(n, c), -1.0, 1.0), sY = fmax(sqrt(1.0 - cY * cY), 1.0e-8);
        const double cT = clampd(dot(a, b), -1.0, 1.0), sTsq = 1.0 - cT * cT, sT = fmax(sqrt(sTsq), 1.0e-8);
        const double dE = -fk * (C1 * cY - 4.0 * C2 * cY * sY);
        const V3     t1 = cross(c, b), t2 = cross(a, c), t3 = cross(b, a);
        const double term1 = sY * sT, term2 = cY / (sY * sTsq);
        const V3     g1 = (t1 * (1.0 / term1) - (a - b * cT) * term2) * (1.0 / dI);
        const V3     g3 = (t2 * (1.0 / term1) - (b - a * cT) * term2) * (1.0 / dK);
        const V3     g4 = (t3 * (1.0 / term1) - c * (cY / sY)) * (1.0 / dL);
        acc<3>(grad, rec.ix[0], g1 * dE);
        acc<3>(grad, rec.ix[1], (g1 + g3 + g4) * (-dE));
        acc<3>(grad, rec.ix[2], g3 * dE);
        acc<3>(grad, rec.ix[3], g4 * dE);
      }
    });
    forTerms<GRAD, 2, 3>(s.vdw, v.vdw, tid, nT, [&](const TermRec<2, 3>& rec) {
      const int    i = rec.ix[0], j = rec.ix[1];
      const double x = rec.q[0], eps = rec.q[1], thr = rec.q[2];
      const V3     d    = ld<3>(pos, i) - ld<3>(pos, j);
      const double dist = sqrt(dot(d, d));
      if (dist > thr) return;
      if (!GRAD) {
        if (dist <= 0.0) return;
        const double r = x / dist, r2 = r * r, r6 = r2 * r2 * r2;
        e += eps * (r6 * r6 - 2.0 * r6);
      } else {
        V3 g;
        if (dist <= 0.0) {
          g = V3{100.0, 100.0, 100.0};
        } else {
          const double r = x / dist, r2 = r * r, r7 = r * r2 * r2 * r2, r13 = r7 * r2 * r2 * r2;
          g = d * (12.0 * eps / x * (r7 - r13) / dist);
        }
        acc<3>(grad, i, g);
        acc<3>(grad, j, -g);
      }
    });
    e += restraintTerms<GRAD>(s.distc, s.posc, s.anglec, s.torsc, v.rs, pos, grad, tid, nT);
    return e;
  }
};

// ============================================================================================ analytic test potential
struct Poly {
  static constexpr int  kDim    = 1;
  static constexpr bool kHasRef = false;
  struct System {
    int           power;
    const double* w;
    const double* c;
    const int32_t* starts;
  };
  struct Params {};
  struct View {
    const double* w;
    const double* c;
    int           n, power;
  };
  __device__ static View view(const System& s, int sys, const Params&) {
    return {s.w + s.starts[sys], s.c + s.starts[sys], s.starts[sys + 1] - s.starts[sys], s.power};
  }
  __device__ static unsigned termBytes(const View& v) { return v.n * 16u; }
  template <bool GRAD>
  __device__ static double eval(const View& v, const double* x, double* grad, int tid, int nT) {
    double e = 0.0;
    for (int i = tid; i < v.n; i += nT) {
      const double d = x[i] - v.c[i];
      if (v.power == 2) {
        if (!GRAD) e += v.w[i] * d * d;
        else grad[i] += 2.0 * v.w[i] * d;
      } else {
        if (!GRAD) e += v.w[i] * d * d * d * d;
        else grad[i] += 4.0 * v.w[i] * d * d * d;
      }
    }
    return e;
  }
};

// Host-side check: every table with terms must carry its wave schedule before a gradient is evaluated.
inline void needWaves(const b200mol_term_table& t, const char* what) {
  B200_REQUIRE(!t.idx || (t.molWaves && t.waves), "term table '%s' has no gradient schedule (see b200mol_schedule_waves)", what);
}
inline void requireSchedule(const b200mol_mmff_system& s) {
  needWaves(s.bond, "bond"), needWaves(s.angle, "angle"), needWaves(s.strbend, "strbend"), needWaves(s.oop, "oop");
  needWaves(s.torsion, "torsion"), needWaves(s.vdw, "vdw"), needWaves(s.ele, "ele");
  needWaves(s.distc, "distc"), needWaves(s.posc, "posc"), needWaves(s.anglec, "anglec"), needWaves(s.torsc, "torsc");
}
inline void requireSchedule(const b200mol_uff_system& s) {
  needWaves(s.bond, "bond"), needWaves(s.angle, "angle"), needWaves(s.torsion, "torsion");
  needWaves(s.inversion, "inversion"), needWaves(s.vdw, "vdw");
  needWaves(s.distc, "distc"), needWaves(s.posc, "posc"), needWaves(s.anglec, "anglec"), needWaves(s.torsc, "torsc");
}
inline void requireSchedule(const b200mol_dg_system& s) {
  needWaves(s.dist, "dist"), needWaves(s.chiral, "chiral"), needWaves(s.fourth, "fourth");
}
inline void requireSchedule(const b200mol_etk_system& s) {
  needWaves(s.torsion, "torsion"), needWaves(s.improper, "improper"), needWaves(s.dist12, "dist12");
  needWaves(s.dist13, "dist13"), needWaves(s.angle13, "angle13"), needWaves(s.longrange, "longrange");
}
inline void requireSchedule(const Poly::System&) {}

}  // namespace ff
}  // namespace b200
