// Device-side BFGS over a flattened force field for ONE conformer held in shared memory (see bfgs.cu for the design).
#pragma once
#include <type_traits>

#include "ff.cuh"

namespace b200 {

#ifndef B200_BFGS_THREADS
#define B200_BFGS_THREADS 256
#endif
constexpr int kT     = B200_BFGS_THREADS;  // threads per CTA (one conformer per CTA)
constexpr int kWarps = kT / 32;
#ifndef B200_BFGS_MIN_CTAS
#define B200_BFGS_MIN_CTAS 3
#endif
constexpr int kMinCtas = B200_BFGS_MIN_CTAS;  // resident CTAs per SM the minimiser kernels are compiled for (register cap)
constexpr int kRed   = kWarps * 6;  // doubles of shared memory behind `red`

__device__ __forceinline__ double warpSum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warpMaxD(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Block-wide reductions; every thread receives the same value. `red` is kRed doubles of shared memory.
__device__ __forceinline__ double blockSum(double v, double* red) {
  v = warpSum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += red[w];
  return t;
}
// N sums with one barrier pair; `red` holds kRed doubles.
template <int N>
__device__ __forceinline__ void blockSumN(double (&v)[N], double* red) {
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = warpSum(v[k]);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) red[k * kWarps + (threadIdx.x >> 5)] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[k * kWarps + w];
    v[k] = t;
  }
}
__device__ __forceinline__ double blockMax(double v, double* red) {
  v = warpMaxD(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = red[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) t = fmax(t, red[w]);
  return t;
}

// RDKit ForceField::minimize gradient cap (>= 2025.09: |g|), bfgs_minimize.cu:797-851.
__device__ inline double scaleGrad(int n, double* grad, bool scaleGrads, double* red) {
  const int tid       = threadIdx.x;
  double    gradScale = scaleGrads ? 0.1 : 1.0, mx = 0.0;
  for (int i = tid; i < n; i += kT) {
    if (scaleGrads) grad[i] *= gradScale;
    mx = fmax(mx, fabs(grad[i]));
  }
  mx = blockMax(mx, red);
  if (scaleGrads && mx > 10.0) {
    while (mx * gradScale > 10.0) gradScale *= 0.5;
    for (int i = tid; i < n; i += kT) grad[i] *= gradScale;
  }
  __syncthreads();
  return gradScale;
}

template <class FF>
__device__ double energyOf(const typename FF::View& v, const double* x, double* red) {
  return blockSum(FF::template eval<false>(v, x, nullptr, threadIdx.x, kT), red);
}
// Gradient at x into acc[0..n): every warp scatters its waves' contributions into its own accumulator
// acc + warp * accStride (plain shared-memory adds, ff.cuh), then the kWarps accumulators are summed in a fixed order.
// No atomics anywhere: the result does not depend on scheduling, so two runs give the same bits.
template <class FF>
__device__ void gradOf(const typename FF::View& v, const double* x, double* acc, int accStride, int n) {
  for (int w = 0; w < kWarps; ++w)
    for (int i = threadIdx.x; i < n; i += kT) acc[w * accStride + i] = 0.0;
  __syncthreads();
  FF::template eval<true>(v, x, acc + (threadIdx.x >> 5) * accStride, threadIdx.x, kT);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kT) {
    double g = acc[i];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) g += acc[w * accStride + i];
    acc[i] = g;
  }
  __syncthreads();
}

// Shared-memory working set of one CTA: 6 + kWarps vectors of maxN doubles + the per-CTA inverse-Hessian slab (global/L2).
//   pos, dir, dGrad, scratch[3] (the pending update's vectors)      - live across iterations
//   acc[0..kWarps)  the per-warp gradient accumulators; outside a gradient evaluation acc[0] = grad (the reduced
//                   gradient), acc[1] = hdg (H * dGrad), acc[2] = newPos (trial point / H * grad): each of the three is
//                   dead while the gradient is being accumulated, so only kWarps - 3 vectors are extra
// HT = storage type of the inverse Hessian: double (default; bit-for-bit the RDKit recurrence) or float (half the slab
// traffic) for the embedding stages whose trajectories are chaotic anyway. The sweep computes in HT: with float the
// rank-2 update, the products, the per-lane column partials, the row sums and their butterfly are fp32; only the
// cross-warp column reduction and the accumulated H*dGrad / H*grad are fp64.
template <class HT = double>
struct BfgsWorkT {
  double *pos, *grad, *dir, *newPos, *dGrad, *hdg;  // shared memory, maxN each
  HT*     H;                                        // [n*n] global slab of this CTA
  double* red;                                      // kRed doubles of shared memory
  double* scratch;                                  // shared memory, 3 * maxN doubles (scaled vectors of the Hessian passes)
  double* colBuf;                                   // shared memory, kColBuf doubles: per-warp column sums of one sweep chunk
  int     maxN;                                     // stride of the accumulators
  unsigned long long* stats;                        // device counters (kStat*), may be nullptr
};
// Work counters of the conformer kernels (b200mol_stats_read): what bench.py's roofline of this path is computed from.
enum : int { kStatIters = 0, kStatEnergyEvals = 1, kStatGradEvals = 2, kStatAlgoBytes = 3, kStatMinimisations = 4, kStatAttempts = 5, kStatN2Iters = 6, kStatCount = 8 };
constexpr int kBfgsVectors = 6 + kWarps;
constexpr int kColBuf      = 2 * kWarps * 64;  // doubles: 2 products x kWarps x 64 fp64 (= 128 fp32) columns of a chunk
template <class HT>
__host__ __device__ inline int bfgsLd(int n) {
  constexpr int per = 128 / static_cast<int>(sizeof(HT));
  return (n + per - 1) / per * per;
}  // six working vectors + four scratch vectors of maxN doubles
using BfgsWork = BfgsWorkT<double>;
template <class HT = double>
__device__ __forceinline__ BfgsWorkT<HT> carveWork(double* sm, int maxN, HT* H, double* red, double* colBuf,
                                                    unsigned long long* stats = nullptr) {
  double* acc = sm + 6 * maxN;  // accumulators: grad | hdg | newPos | kWarps - 3 more
  return {sm, acc, sm + maxN, acc + 2 * maxN, sm + 2 * maxN, acc + maxN, H, red, sm + 3 * maxN, colBuf, maxN, stats};
}

struct BfgsOutcome {
  int    status;  // 0 converged, 1 not
  int    iters;   // BFGS iterations of the last (re)start
  double energy;  // energy at w.pos (re-evaluated)
};

// Minimises w.pos[0..n) in place. maxRestarts > 0 re-runs (H = I, fresh gradient) while the run ends unconverged:
// RDKit's `while (needMore) needMore = field->minimize(...)` (src/etkdg_stage_distgeom_minimize.cu repeatUntilConverged).
#ifdef B200_BFGS_TIMING
static __device__ unsigned long long g_bfgsClk[8];  // per translation unit
static inline void readBfgsClocks(unsigned long long* out) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, g_bfgsClk, sizeof(g_bfgsClk));
  unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  cudaMemcpyToSymbol(g_bfgsClk, z, sizeof(z));
}
#define B200_T0() const long long t0_ = clock64()
#define B200_T1(slot) tim[slot] += clock64() - t0_
#else
#define B200_T0()
#define B200_T1(slot)
#endif

// One sweep over the upper triangle (j >= i) of the inverse Hessian of one conformer, by the whole CTA:
//   H[i][j] (+)= fac x_i x_j - fad h_i h_j + fae u_i u_j   (if `pending`; a `fresh` H is the identity and is not read)
//   outD += H d,  outG += H g                               (both symmetric products, from the stored half only)
// A lane owns V = 16/sizeof(HT) consecutive columns of a 32*V-wide chunk: one 128-bit load and store per row, the
// column values and column sums stay in registers for all rows of the chunk, the row sums of FOUR rows are reduced
// together by one exchange-halving butterfly (9 shuffles for 8 values instead of 40). Columns [n, ld) hold zeros, so
// only the chunk that contains the diagonal needs per-element masks. The sweep is issue-bound, not latency-bound,
// hence the instruction diet.
#ifndef B200_SWEEP_PREFETCH
#define B200_SWEEP_PREFETCH 0
#endif
constexpr int kSweepPrefetch = B200_SWEEP_PREFETCH;  // batches ahead the sweep asks its rows into L2 (0 = off)
template <class HT, bool FRESH, bool PENDING>
__device__ __noinline__ void hessianSweepT(HT* __restrict__ H, int ld, int n, HT cfac, HT cfad, HT cfae, const HT* px, const HT* ph,
                                           const HT* pu, const HT* vD, const HT* vG, double* outD, double* outG, double* colBuf) {
  constexpr int V  = 16 / static_cast<int>(sizeof(HT));
  constexpr int CW = 32 * V;
  struct alignas(16) Pack {
    HT e[V];
  };
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c0 = 0; c0 < n; c0 += CW) {
    const int  cb     = c0 + V * lane;  // first column of this lane
    const bool laneIn = cb < ld;
    HT         aD[V], aG[V], xj[V], hj[V], uj[V], dj[V], gj[V];
#pragma unroll
    for (int t = 0; t < V; ++t) {
      const bool in = cb + t < n;
      aD[t] = aG[t] = HT(0);
      // the three scalars of the rank-2 update ride on the COLUMN values (once per chunk), not on the row values
      xj[t] = (in && PENDING) ? cfac * px[cb + t] : HT(0);
      hj[t] = (in && PENDING) ? -cfad * ph[cb + t] : HT(0);
      uj[t] = (in && PENDING) ? cfae * pu[cb + t] : HT(0);
      dj[t] = in ? vD[cb + t] : HT(0);
      gj[t] = in ? vG[cb + t] : HT(0);
    }
    const int rowEnd = min(n, c0 + CW);  // rows below have no element with j >= i in this chunk
    auto      batch  = [&](int i0, auto diagTag) {
      constexpr bool DIAG = decltype(diagTag)::value;  // the four rows' diagonal elements lie in this chunk
      Pack           pk[4];
      // the four rows' loads first: they are independent, and the sweep is bound by memory latency (HBM-resident slabs)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = i0 + q;
#pragma unroll
        for (int t = 0; t < V; ++t) pk[q].e[t] = (FRESH && cb + t == i) ? HT(1) : HT(0);
        if constexpr (!FRESH)
          if (laneIn && i < rowEnd) pk[q] = *reinterpret_cast<const Pack*>(H + static_cast<size_t>(i) * ld + cb);
      }
      HT r[8];  // row sums: [0..3] with d, [4..7] with g
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int  i  = i0 + q;
        const bool ok = i < rowEnd;  // rows past the end contribute zeros and are not stored
        const HT   di = ok ? vD[i] : HT(0), gi = ok ? vG[i] : HT(0);
        if constexpr (PENDING) {
          const HT si = ok ? px[i] : HT(0), ti = ok ? ph[i] : HT(0), wi = ok ? pu[i] : HT(0);
#pragma unroll
          for (int t = 0; t < V; ++t) {
            HT v = pk[q].e[t];
            if constexpr (sizeof(HT) == 4) {
              v = __fmaf_rn(si, xj[t], v);
              v = __fmaf_rn(ti, hj[t], v);
              v = __fmaf_rn(wi, uj[t], v);
            } else {
              v = __fma_rn(si, xj[t], v);
              v = __fma_rn(ti, hj[t], v);
              v = __fma_rn(wi, uj[t], v);
            }
            pk[q].e[t] = v;
          }
        }
        if constexpr (DIAG) {
#pragma unroll
          for (int t = 0; t < V; ++t) pk[q].e[t] = (cb + t >= i) ? pk[q].e[t] : HT(0);
        }
        if constexpr (PENDING)
          if (laneIn && ok) *reinterpret_cast<Pack*>(H + static_cast<size_t>(i) * ld + cb) = pk[q];
        HT rd = HT(0), rg = HT(0);
#pragma unroll
        for (int t = 0; t < V; ++t) {
          const HT v = pk[q].e[t];
          aD[t] += v * di;
          aG[t] += v * gi;
          const HT vs = (!DIAG || cb + t > i) ? v : HT(0);
          rd += vs * dj[t];
          rg += vs * gj[t];
        }
        r[q]     = rd;
        r[q + 4] = rg;
      }
      // eight sums over the warp: halve the value set at each of the first three exchange steps
      const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
      HT         s4[4], s2[2];
#pragma unroll
      for (int k = 0; k < 4; ++k) s4[k] = (b4 ? r[k + 4] : r[k]) + __shfl_xor_sync(0xffffffffu, b4 ? r[k] : r[k + 4], 16);
#pragma unroll
      for (int k = 0; k < 2; ++k) s2[k] = (b3 ? s4[k + 2] : s4[k]) + __shfl_xor_sync(0xffffffffu, b3 ? s4[k] : s4[k + 2], 8);
      HT s1 = (b2 ? s2[1] : s2[0]) + __shfl_xor_sync(0xffffffffu, b2 ? s2[0] : s2[1], 4);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      // lane 16 a + 8 b + 4 c holds value index 4 a + 2 b + c : a selects g over d, (2 b + c) the row of the four
      // (row i belongs to this lane in every chunk and the column sums are added between barriers: a plain add)
      if ((lane & 3) == 0) {
        const int i = i0 + ((lane >> 2) & 3);
        if (i < rowEnd) (b4 ? outG : outD)[i] += static_cast<double>(s1);
      }
    };
    // rows above the chunk's diagonal block: no masks; rows inside it (CW is a multiple of 4): masked
    // The slabs live in HBM (444 of them do not fit L2 next to the streaming term tables) and a warp has four row packs
    // in flight. Two ways of getting further ahead were measured and rejected: the next
    // batch in registers spills at the 80-register budget of three CTAs per SM; asking the rows of a later batch into L2
    // with prefetch.global.L2 (B200_SWEEP_PREFETCH = batches ahead) is 3-5 % SLOWER than nothing (0, the default).
    // lanes 8 q + l, l < 4: row q of the batch, 128-byte line l of its 512 bytes in this chunk
    const int  pfCol = c0 + (lane & 7) * static_cast<int>(128 / sizeof(HT));
    const bool pfOn  = !FRESH && kSweepPrefetch > 0 && (lane & 7) < 4 && pfCol < ld;
    const HT*  pfAt  = H + static_cast<size_t>(lane >> 3) * ld + pfCol;
    auto ahead = [&](int i) {
      if (pfOn && i + (lane >> 3) < rowEnd) asm volatile("prefetch.global.L2 [%0];" ::"l"(pfAt + static_cast<size_t>(i) * ld));
    };
    int i0 = 4 * warp;
    for (; i0 < min(c0, rowEnd); i0 += 4 * kWarps) {
      ahead(i0 + kSweepPrefetch * 4 * kWarps);
      batch(i0, std::false_type{});
    }
    for (; i0 < rowEnd; i0 += 4 * kWarps) {
      ahead(i0 + kSweepPrefetch * 4 * kWarps);
      batch(i0, std::true_type{});
    }
    // column sums of the chunk: every warp parks its partials, then one thread per column adds the kWarps of them in a
    // fixed order (no atomics: bit-reproducible)
    HT* colD = reinterpret_cast<HT*>(colBuf);
    HT* colG = colD + kWarps * CW;
#pragma unroll
    for (int t = 0; t < V; ++t) {
      colD[warp * CW + V * lane + t] = aD[t];
      colG[warp * CW + V * lane + t] = aG[t];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < CW && c0 + c < n; c += kT) {
      double sD = 0.0, sG = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        sD += static_cast<double>(colD[w * CW + c]);
        sG += static_cast<double>(colG[w * CW + c]);
      }
      outD[c0 + c] += sD;
      outG[c0 + c] += sG;
    }
    __syncthreads();
  }
}
template <class HT>
__device__ __forceinline__ void hessianSweep(HT* H, int ld, int n, bool fresh, bool pending, HT cfac, HT cfad, HT cfae, const HT* px,
                                             const HT* ph, const HT* pu, const HT* vD, const HT* vG, double* outD, double* outG,
                                             double* colBuf) {
  if (!fresh && pending) hessianSweepT<HT, false, true>(H, ld, n, cfac, cfad, cfae, px, ph, pu, vD, vG, outD, outG, colBuf);
  else if (fresh) hessianSweepT<HT, true, true>(H, ld, n, cfac, cfad, cfae, px, ph, pu, vD, vG, outD, outG, colBuf);  // pending by construction
  else hessianSweepT<HT, false, false>(H, ld, n, cfac, cfad, cfae, px, ph, pu, vD, vG, outD, outG, colBuf);
}

template <class FF, class HT = double>
__device__ BfgsOutcome bfgsMinimize(const typename FF::View& view, const BfgsWorkT<HT>& w, int n, int maxIters,
                                    double gradTol, bool scaleGrads, int maxRestarts) {
  constexpr double FUNCTOL = 1e-4, MOVETOL = 1e-7, TOLX = 4. * 3e-8, EPS = 3e-8;
  double *pos = w.pos, *grad = w.grad, *dir = w.dir, *newPos = w.newPos, *dGrad = w.dGrad, *hdg = w.hdg, *red = w.red;
  HT*     H   = w.H;
  const int tid = threadIdx.x;
  // leading dimension of the slab: rows padded to 128 bytes so that every warp access is whole, aligned cache lines
  const int ld = bfgsLd<HT>(n);
  int       status = 1, iter = 0;
  unsigned  nEvals = 0, nIters = 0, nGrads = 0;  // work counters (thread 0 publishes them)
#ifdef B200_BFGS_TIMING
  long long tim[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const long long tAll = clock64();
#endif
  for (int restart = 0;; ++restart) {
    __syncthreads();
    bool   fresh = true, pending = false;  // H = I (not materialised); no rank-2 update waiting
    double pfac = 0.0, pfad = 0.0, pfae = 0.0;

    double fp = energyOf<FF>(view, pos, red);
    gradOf<FF>(view, pos, grad, w.maxN, n);
    ++nEvals;
    ++nGrads;
    double gradScale = scaleGrad(n, grad, scaleGrads, red);
    double s2        = 0.0;
    for (int i = tid; i < n; i += kT) {
      dir[i] = -grad[i];
      s2 += pos[i] * pos[i];
    }
    const double maxStep = 100.0 * fmax(sqrt(blockSum(s2, red)), static_cast<double>(n));
    status               = 1;
    for (iter = 0; iter < maxIters; ++iter) {
      // ---------------- line search (bfgs_minimize.cu:80-162, 202-356) ----------------
      double t = 0.0;
      for (int i = tid; i < n; i += kT) t += dir[i] * dir[i];
      const double dsum = sqrt(blockSum(t, red));
      if (dsum > maxStep) {
        const double sc = maxStep / dsum;
        for (int i = tid; i < n; i += kT) dir[i] *= sc;
      }
      double sl = 0.0, tst = 0.0;
      for (int i = tid; i < n; i += kT) {
        sl += dir[i] * grad[i];
        tst = fmax(tst, fabs(dir[i]) / fmax(fabs(pos[i]), 1.0));
      }
      const double slope     = blockSum(sl, red);
      const double lambdaMin = MOVETOL / blockMax(tst, red);
      double       lambda = 1.0, lambda2 = 0.0, val2 = 0.0, newVal = fp;
      bool         accepted = false;
      for (int it = 0; it < 1000; ++it) {
        if (lambda < lambdaMin) break;
        for (int i = tid; i < n; i += kT) newPos[i] = pos[i] + lambda * dir[i];
        __syncthreads();
        {
          B200_T0();
          newVal = energyOf<FF>(view, newPos, red);
          B200_T1(0);
        }
        ++nEvals;
        if (newVal - fp <= FUNCTOL * lambda * slope) {
          accepted = true;
          break;
        }
        double tmp;
        if (it == 0) {
          tmp = -slope / (2.0 * (newVal - fp - slope));
        } else {
          const double rhs1 = newVal - fp - lambda * slope, rhs2 = val2 - fp - lambda2 * slope;
          const double a    = (rhs1 / (lambda * lambda) - rhs2 / (lambda2 * lambda2)) / (lambda - lambda2);
          const double bq   = (-lambda2 * rhs1 / (lambda * lambda) + lambda * rhs2 / (lambda2 * lambda2)) / (lambda - lambda2);
          if (a == 0.0) {
            tmp = -slope / (2.0 * bq);
          } else {
            const double disc = bq * bq - 3 * a * slope;
            if (disc < 0.0) tmp = 0.5 * lambda;
            else if (bq <= 0.0) tmp = (-bq + sqrt(disc)) / (3.0 * a);
            else tmp = -slope / (bq + sqrt(disc));
          }
          if (tmp > 0.5 * lambda) tmp = 0.5 * lambda;
        }
        lambda2 = lambda;
        val2    = newVal;
        lambda  = fmax(tmp, 0.1 * lambda);
      }
      __syncthreads();
      if (!accepted)
        for (int i = tid; i < n; i += kT) newPos[i] = pos[i];  // "nothing was done"
      fp = newVal;
      // ---------------- direction, TOLX (bfgs_minimize.cu:732-776) ----------------
      tst = 0.0;
      for (int i = tid; i < n; i += kT) {
        const double xi = newPos[i] - pos[i];
        dir[i]          = xi;
        pos[i]          = newPos[i];
        tst             = fmax(tst, fabs(xi) / fmax(fabs(pos[i]), 1.0));
        dGrad[i]        = grad[i];
      }
      if (blockMax(tst, red) < TOLX) {
        status = 0;
        break;
      }
      {
        B200_T0();
        gradOf<FF>(view, pos, grad, w.maxN, n);
        B200_T1(1);
      }
      ++nGrads;
      gradScale = scaleGrad(n, grad, scaleGrads, red);
      tst       = 0.0;
      for (int i = tid; i < n; i += kT) {
        tst      = fmax(tst, fabs(grad[i]) * fmax(fabs(pos[i]), 1.0));
        dGrad[i] = grad[i] - dGrad[i];
      }
      if (blockMax(tst, red) / fmax(fp * gradScale, 1.0) < gradTol) {
        status = 0;
        break;
      }
      // ---------------- inverse Hessian (bfgs_hessian.cu:37-239) ----------------
      // ONE sweep over the UPPER TRIANGLE of H per iteration. The reference makes three passes over the full matrix
      // (H*dGrad; rank-2 update; -H*grad). Here the rank-2 update of iteration k stays PENDING (three vectors, three
      // scalars) and is applied by the sweep of iteration k+1, which in the same pass accumulates H*dGrad and H*grad;
      // the next direction follows from H*grad and the pending vectors by O(n) algebra:
      //   H' g = H g + fac x (x.g) - fad h (h.g) + fae u (u.g),  u = fac x - fad h.
      // H is symmetric, so only j >= i is stored/streamed: element (i,j) feeds column sums (lane-private registers)
      // and row sums (one shuffle tree per row). Traffic per iteration: n^2/2 read + n^2/2 written instead of
      // 2 n^2 read + n^2 written. A fresh H (= I) is never materialised: the first sweep with a pending update writes it.
      B200_T0();
      using AT             = HT;  // arithmetic type of the sweep = storage type
      AT*           px     = reinterpret_cast<AT*>(w.scratch);  // pending x (step), h (H dGrad), u
      AT*           ph     = px + n;
      AT*           pu     = ph + n;
      double*       hgv    = newPos;  // H * grad (newPos is free here)
      if (fresh && !pending) {
        for (int i = tid; i < n; i += kT) {
          hdg[i] = dGrad[i];
          hgv[i] = grad[i];
        }
        __syncthreads();
      } else {
        const AT *vD, *vG;
        if constexpr (sizeof(AT) == 4) {
          AT* cD = pu + n;
          AT* cG = cD + n;
          for (int i = tid; i < n; i += kT) {
            cD[i] = static_cast<AT>(dGrad[i]);
            cG[i] = static_cast<AT>(grad[i]);
          }
          vD = cD;
          vG = cG;
        } else {
          vD = dGrad;
          vG = grad;
        }
        for (int i = tid; i < n; i += kT) {
          hdg[i] = 0.0;
          hgv[i] = 0.0;
        }
        __syncthreads();
        hessianSweep<HT>(H, ld, n, fresh, pending, static_cast<AT>(pfac), static_cast<AT>(pfad), static_cast<AT>(pfae), px, ph, pu,
                         vD, vG, hdg, hgv, w.colBuf);
        if (pending) fresh = false;
        __syncthreads();
      }
      B200_T1(2);
      double f[6] = {0, 0, 0, 0, 0, 0};
      for (int i = tid; i < n; i += kT) {
        f[0] += dGrad[i] * dir[i];
        f[1] += dGrad[i] * hdg[i];
        f[2] += dGrad[i] * dGrad[i];
        f[3] += dir[i] * dir[i];
        f[4] += dir[i] * grad[i];
        f[5] += hdg[i] * grad[i];
      }
      blockSumN<6>(f, red);
      double       fac      = f[0];
      const double fae      = f[1];
      const bool   update   = fac > sqrt(EPS * f[2] * f[3]);
      if (update) {
        fac             = 1.0 / fac;
        const double fad = 1.0 / fae;
        const double xg = f[4], hg = f[5], ug = fac * xg - fad * hg;
        for (int i = tid; i < n; i += kT) {
          const double x = dir[i], hd = hdg[i];
          const double u = fac * x - fad * hd;
          px[i]          = static_cast<AT>(x);
          ph[i]          = static_cast<AT>(hd);
          pu[i]          = static_cast<AT>(u);
          dir[i]         = -(hgv[i] + (fac * xg) * x - (fad * hg) * hd + (fae * ug) * u);
        }
        pending = true;
        pfac    = fac;
        pfad    = fad;
        pfae    = fae;
      } else {
        for (int i = tid; i < n; i += kT) dir[i] = -hgv[i];
        pending = false;
      }
#ifdef B200_BFGS_TIMING
      tim[4] += 1;
#endif
      __syncthreads();
    }
    nIters += iter < maxIters ? iter + 1 : iter;
    if (status == 0 || restart >= maxRestarts) break;
  }
  __syncthreads();
  if (w.stats && tid == 0) {
    // SURVEY.md 8d: per iteration 3 n^2 x 8 B of inverse Hessian + (1 + k_ls) x T bytes of term records
    const unsigned long long T = FF::termBytes(view);
    atomicAdd(w.stats + kStatIters, static_cast<unsigned long long>(nIters));
    atomicAdd(w.stats + kStatEnergyEvals, static_cast<unsigned long long>(nEvals + 1));
    atomicAdd(w.stats + kStatGradEvals, static_cast<unsigned long long>(nGrads));
    atomicAdd(w.stats + kStatAlgoBytes, 24ull * n * n * nIters + T * (nEvals + 1 + nGrads));
    atomicAdd(w.stats + kStatMinimisations, 1ull);
    atomicAdd(w.stats + kStatN2Iters, static_cast<unsigned long long>(n) * n * nIters);
  }
  BfgsOutcome out;
  out.status = status;
  out.iters  = iter;
  out.energy = energyOf<FF>(view, pos, red);
#ifdef B200_BFGS_TIMING
  if (tid == 0) {
    tim[5] = clock64() - tAll;
    for (int k = 0; k < 6; ++k) atomicAdd(&g_bfgsClk[k], static_cast<unsigned long long>(tim[k]));
  }
#endif
  return out;
}

}  // namespace b200
