// MaxMin diversity picking on packed fingerprints (RDKit MaxMinPicker::LazyBitVectorPick): b200mol_maxmin_pick.
//
// Contract. d(i, j) = 1 - s(i, j), s the fp64 value b200mol_tanimoto_cross / b200mol_cosine_cross store for the pair
// (simFromCounts: 0 for an empty intersection). Picks start with the caller's first picks, in order; every further pick
// is the unpicked pool item with the largest min over the picks of d(i, p), ties to the lowest index. That is what
// RDKit's lazyPick returns: it walks the pool in index order and replaces its candidate only on a strictly larger value,
// and its lazy early exit never drops an item that could win. With threshold >= 0 the loop stops before adding a pick
// whose max-min is <= threshold.
//
// One persistent cooperative kernel runs the whole pick loop; CTA b owns the pool slice [b * slice, (b + 1) * slice).
// Per item it keeps bound (fp64, an upper bound of its min distance, exact over the picks applied so far; -1 = picked),
// applied (how many picks bound covers) and the popcount, in shared memory when the slice fits, else in a per-CTA region
// of global memory. The slice's fingerprints stay in shared memory when they fit too ("resident"); otherwise they are
// read from L2 / HBM. Pick fingerprints are read by index from the pool, so the picks stay hot in L2.
//
// Popcount skip. Before an item's fingerprint is read for pick p, lb = 1 - s(min(|A|, |B|), |A|, |B|) is formed by the
// same fp64 operations as the distance. The intersection c is at most min(|A|, |B|); the real Tanimoto quotient
// c / (|A| + |B| - c) and the cosine c / sqrt(|A||B|) grow with c, correctly rounded division and sqrt are monotone, c = 0
// gives 0 <= any value, and 1 - x rounds monotonically: so lb <= d(i, p) exactly. When lb >= bound the pick cannot lower
// the item's min, and the fingerprint is not read.
//
// Dense mode (maxmin_mode 0), one pick per round: every unpicked item takes the newest pick; each CTA writes its best
// (value, then lowest index) to its slot; grid.sync; every CTA reduces the slots in the same fixed order, so all agree on
// the winner without atomics; CTA 0 records it and applies the threshold stop.
//
// Deferred mode (maxmin_mode 1), RDKit's lazy bound, two grid syncs per pick. After a first pass that applies the first
// pick to every item (as RDKit's does):
//   phase A  each CTA brings its item with the largest stale bound fully up to date (its warps split the missing picks)
//            and publishes that exact value; tau = the max of the published values, a lower bound of this round's max-min;
//   phase B  each CTA catches up only its items with bound >= tau, through picks[applied..t), stopping once bound < tau;
//            its best comes only from items that are fully up to date.
// Why it is exact: the winner has true min M >= tau (tau is some unpicked item's exact min) and its stale bound is >= M,
// so it is never skipped nor cut short, and it ends with its exact value M. An item that exits early or is skipped has a
// true min below tau <= M. Items fully up to date carry exact values, so the reduction by (value, index) finds the winner.
#include <cooperative_groups.h>

#include <algorithm>
#include <vector>

#include "options.cuh"
#include "similarity.cuh"

namespace cg = cooperative_groups;

namespace b200 {

int       g_maxminMode         = 0;   // option "maxmin_mode": 0 dense (measured faster in most workloads, DESIGN §4), 1 deferred
long long g_maxminResidentRows = -1;  // option "maxmin_resident_rows": < 0 automatic, 0 streamed, > 0 largest resident pool
int       g_maxminResidentLast = 0;   // the last call kept the pool in shared memory ("maxmin_resident_last")

namespace {

constexpr int    kThreads  = 512;
constexpr int    kWarps    = kThreads / 32;
constexpr int    kMinSlice = 128;   // items per CTA at least: small pools take fewer CTAs, so the grid barrier stays cheap
constexpr int    kUnroll   = 4;     // items a group loads before it counts, in the dense pass
constexpr double kUnset    = 2.0;   // bound before any pick: above every distance
constexpr double kPicked   = -1.0;
constexpr int    kNone     = 0x7fffffff;

__device__ unsigned long long g_maxminStat[2];  // [0] distances evaluated, [1] skipped by the popcount bound

struct PickArgs {
  const uint4*   fp;   // [n][chunks] the pool
  const int32_t* pop;  // [n]
  int            n, chunks, group, slice;
  bool           cosine;
  int            deferred, nFirst, pickSize;
  double         threshold;  // < 0: none
  int32_t*       picks;      // [pickSize]; [0, nFirst) given
  double*        thresholdOut;
  double*        slotV;  // [3][gridDim.x]: end of round by parity, phase A
  int32_t*       slotI;
  double*        gBound;  // per-CTA state in global memory when it does not fit in shared memory, else null
  int32_t*       gApplied;
  int32_t*       gPop;
};

__device__ __forceinline__ bool better(double v1, int i1, double v2, int i2) { return v1 > v2 || (v1 == v2 && i1 < i2); }

__device__ __forceinline__ double distance(int c, int a, int b, bool cosine) { return __dsub_rn(1.0, simFromCounts(c, a, b, cosine)); }
__device__ __forceinline__ double lowerBound(int a, int b, bool cosine) { return distance(min(a, b), a, b, cosine); }

__device__ __forceinline__ int popAnd(uint4 x, uint4 y) {
  return __popc(x.x & y.x) + __popc(x.y & y.y) + __popc(x.z & y.z) + __popc(x.w & y.w);
}

struct Ctx {
  const PickArgs& a;
  const uint4*    sFp;  // resident slice, or null
  double*         bound;
  int32_t*        applied;
  int32_t*        pop;
  int             lo, cnt;  // slice start, items in it
  int             G, gl, grp, nGroups;
  unsigned        mask;  // lanes of this thread's group
  unsigned long long evaluated = 0, skipped = 0;

  template <bool kRes>
  __device__ __forceinline__ uint4 item(int j, int w) const {
    if (kRes) return sFp[static_cast<size_t>(j) * a.chunks + w];
    return __ldg(a.fp + static_cast<size_t>(lo + j) * a.chunks + w);
  }
  __device__ __forceinline__ int groupSum(int c) const {
    for (int o = G >> 1; o; o >>= 1) c += __shfl_xor_sync(mask, c, o);
    return c;
  }
  // |item j & pool[pick]|, by the group
  template <bool kRes>
  __device__ int count(int j, int pick) const {
    const uint4* pf = a.fp + static_cast<size_t>(pick) * a.chunks;
    int          c  = 0;
    for (int w = gl; w < a.chunks; w += G) c += popAnd(item<kRes>(j, w), __ldg(pf + w));
    return groupSum(c);
  }
};

// picks[p]; the newest pick (p == t - 1) was written this round without a barrier since, so it comes from a register
__device__ __forceinline__ int pickAt(const PickArgs& a, int p, int t, int newest) { return p == t - 1 ? newest : __ldcg(a.picks + p); }

// Every unpicked item of the slice takes pick `pick`.
template <bool kRes>
__device__ void densePass(Ctx& c, int pick) {
  const PickArgs& a   = c.a;
  const uint4*    pf  = a.fp + static_cast<size_t>(pick) * a.chunks;
  const uint4     z   = make_uint4(0, 0, 0, 0);
  const uint4     y0  = c.gl < a.chunks ? __ldg(pf + c.gl) : z;
  const uint4     y1  = c.gl + c.G < a.chunks ? __ldg(pf + c.gl + c.G) : z;
  const int       pp  = __ldg(a.pop + pick);
  for (int base = c.grp; base < c.cnt; base += c.nGroups * kUnroll) {
    uint4  x0[kUnroll], x1[kUnroll];
    double b[kUnroll];
    bool   need[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int j = base + u * c.nGroups;
      x0[u] = x1[u] = z;
      b[u]          = kPicked;
      need[u]       = false;
      if (j < c.cnt) {
        b[u]    = c.bound[j];
        need[u] = b[u] >= 0.0 && lowerBound(c.pop[j], pp, a.cosine) < b[u];
        if (c.gl == 0 && b[u] >= 0.0) (need[u] ? c.evaluated : c.skipped) += 1;
      }
      if (need[u]) {
        if (c.gl < a.chunks) x0[u] = c.template item<kRes>(j, c.gl);
        if (c.gl + c.G < a.chunks) x1[u] = c.template item<kRes>(j, c.gl + c.G);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int n = c.groupSum(popAnd(x0[u], y0) + popAnd(x1[u], y1));
      if (need[u]) {
        const int    j = base + u * c.nGroups;
        const double d = distance(n, c.pop[j], pp, a.cosine);
        if (c.gl == 0 && d < b[u]) c.bound[j] = d;
      }
    }
  }
}

// Best (value, then lowest index) of the threads' (v, i) in every thread; the whole CTA calls it.
__device__ void blockReduce(double v, int i, double* sV, int* sI, double& bv, int& bi) {
  for (int o = 16; o; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int    oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(ov, oi, v, i)) v = ov, i = oi;
  }
  __syncthreads();  // (sV / sI may still be read from the previous call)
  if ((threadIdx.x & 31) == 0) sV[threadIdx.x >> 5] = v, sI[threadIdx.x >> 5] = i;
  __syncthreads();
  v = sV[0], i = sI[0];
  for (int w = 1; w < kWarps; ++w)
    if (better(sV[w], sI[w], v, i)) v = sV[w], i = sI[w];
  bv = v, bi = i;
}

// Best (value, then lowest index) over the unpicked items with applied >= minApplied.
__device__ void blockBest(const Ctx& c, int minApplied, double* sV, int* sI, double& bv, int& bi) {
  double v = -1.0;
  int    i = kNone;
  for (int j = threadIdx.x; j < c.cnt; j += kThreads) {
    const double b = c.bound[j];
    if (b >= 0.0 && (minApplied <= 0 || c.applied[j] >= minApplied) && better(b, c.lo + j, v, i)) v = b, i = c.lo + j;
  }
  blockReduce(v, i, sV, sI, bv, bi);
}

// Best over the slots of one bank. The order (value, then index) is total, so every CTA finds the same winner.
__device__ void reduceSlots(const PickArgs& a, int bank, double* sV, int* sI, double& bv, int& bi) {
  double v = -1.0;
  int    i = kNone;
  for (int b = threadIdx.x; b < static_cast<int>(gridDim.x); b += kThreads) {
    const double sv = __ldcg(a.slotV + bank * gridDim.x + b);
    const int    si = __ldcg(a.slotI + bank * gridDim.x + b);
    if (better(sv, si, v, i)) v = sv, i = si;
  }
  blockReduce(v, i, sV, sI, bv, bi);
}

template <bool kRes>
__global__ void __launch_bounds__(kThreads, 1) maxminKernel(const PickArgs a) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double sV[kWarps];
  __shared__ int    sI[kWarps];
  __shared__ double sMin[kThreads];

  const int lo  = blockIdx.x * a.slice;
  const int cnt = max(0, min(a.n - lo, a.slice));
  const int tid = threadIdx.x, lane = tid & 31, G = a.group;
  Ctx       c{a};
  c.lo = lo, c.cnt = cnt, c.G = G, c.gl = lane & (G - 1), c.grp = tid / G, c.nGroups = kThreads / G;
  c.mask = (G == 32 ? 0xffffffffu : ((1u << G) - 1u)) << (lane & ~(G - 1));
  {
    unsigned char* p = smem;
    if (kRes) {
      c.sFp = reinterpret_cast<const uint4*>(p);
      uint4*       dst = reinterpret_cast<uint4*>(p);
      const uint4* src = a.fp + static_cast<size_t>(lo) * a.chunks;
      for (int w = tid; w < cnt * a.chunks; w += kThreads) dst[w] = __ldg(src + w);
      p += static_cast<size_t>(a.slice) * a.chunks * 16;
    }
    if (a.gBound) {
      c.bound   = a.gBound + static_cast<size_t>(blockIdx.x) * a.slice;
      c.applied = a.gApplied + static_cast<size_t>(blockIdx.x) * a.slice;
      c.pop     = a.gPop + static_cast<size_t>(blockIdx.x) * a.slice;
    } else {
      c.bound   = reinterpret_cast<double*>(p);
      c.applied = reinterpret_cast<int32_t*>(p + static_cast<size_t>(a.slice) * 8);
      c.pop     = reinterpret_cast<int32_t*>(p + static_cast<size_t>(a.slice) * 12);
    }
  }
  const int initApplied = a.deferred ? 1 : 0;  // deferred: the first pass below applies picks[0] to every item
  for (int j = tid; j < cnt; j += kThreads) c.bound[j] = kUnset, c.applied[j] = initApplied, c.pop[j] = __ldg(a.pop + lo + j);
  __syncthreads();
  for (int f = tid; f < a.nFirst; f += kThreads) {
    const int p = __ldcg(a.picks + f);
    if (p >= lo && p < lo + cnt) c.bound[p - lo] = kPicked;
  }
  __syncthreads();

  int    t = a.nFirst, newest = __ldcg(a.picks + a.nFirst - 1), done = 0, round = 0;
  double lastV = -1.0;
  if (a.deferred && t < a.pickSize) {
    densePass<kRes>(c, __ldcg(a.picks));
    __syncthreads();
  }
  while (t < a.pickSize) {
    double bv;
    int    bi;
    if (!a.deferred) {
      for (; done < t; ++done) {
        densePass<kRes>(c, pickAt(a, done, t, newest));
        __syncthreads();
      }
      blockBest(c, 0, sV, sI, bv, bi);
    } else {
      // phase A: the item with the largest stale bound, brought up to date by the whole CTA
      blockBest(c, 0, sV, sI, bv, bi);
      double exact = -1.0;
      if (bi != kNone) {
        const int    j  = bi - lo;
        const int    p0 = c.applied[j];
        const int    pj = c.pop[j];
        const double b0 = bv;
        double       m  = b0;
        for (int p = p0 + c.grp; p < t; p += c.nGroups) {
          const int pick = pickAt(a, p, t, newest), pp = __ldg(a.pop + pick);
          if (!(lowerBound(pj, pp, a.cosine) < m)) {
            if (c.gl == 0) ++c.skipped;
            continue;
          }
          const double d = distance(c.template count<kRes>(j, pick), pj, pp, a.cosine);
          if (c.gl == 0) ++c.evaluated;
          m = d < m ? d : m;
        }
        sMin[tid] = m;
        __syncthreads();
        if (tid == 0) {
          for (int g = 0; g < c.nGroups; ++g) m = sMin[g * G] < m ? sMin[g * G] : m;
          c.bound[j] = m, c.applied[j] = t;
          sMin[0] = m;
        }
        __syncthreads();
        exact = sMin[0];
      }
      if (tid == 0) a.slotV[2 * gridDim.x + blockIdx.x] = exact, a.slotI[2 * gridDim.x + blockIdx.x] = bi;
      grid.sync();
      double tau;
      int    unused;
      reduceSlots(a, 2, sV, sI, tau, unused);
      // phase B: only the items that could still reach tau, each stopping once it falls below
      for (int j = c.grp; j < cnt; j += c.nGroups) {
        double b = c.bound[j];
        if (b < tau) continue;  // (picked items too: their bound is -1)
        int       p  = c.applied[j];
        const int pj = c.pop[j];
        while (p < t) {
          const int pick = pickAt(a, p, t, newest), pp = __ldg(a.pop + pick);
          ++p;
          if (!(lowerBound(pj, pp, a.cosine) < b)) {
            if (c.gl == 0) ++c.skipped;
            continue;
          }
          const double d = distance(c.template count<kRes>(j, pick), pj, pp, a.cosine);
          if (c.gl == 0) ++c.evaluated;
          if (d < b) {
            b = d;
            if (b < tau) break;
          }
        }
        if (c.gl == 0) c.bound[j] = b, c.applied[j] = p;
      }
      __syncthreads();
      blockBest(c, t, sV, sI, bv, bi);
    }
    const int bank = round & 1;
    if (tid == 0) a.slotV[bank * gridDim.x + blockIdx.x] = bv, a.slotI[bank * gridDim.x + blockIdx.x] = bi;
    grid.sync();
    reduceSlots(a, bank, sV, sI, bv, bi);
    if (a.threshold >= 0.0 && bv <= a.threshold) break;  // (every CTA reads the same slots: all leave together)
    if (tid == 0) {
      if (blockIdx.x == 0) a.picks[t] = bi;
      if (bi >= lo && bi < lo + cnt) c.bound[bi - lo] = kPicked;
    }
    __syncthreads();
    lastV = bv, newest = bi;
    ++t, ++round;
  }
  if (blockIdx.x == 0 && tid == 0) *a.thresholdOut = lastV;
  unsigned long long e = c.evaluated, s = c.skipped;
  for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o), s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0 && (e | s)) atomicAdd(&g_maxminStat[0], e), atomicAdd(&g_maxminStat[1], s);
}

template <bool kRes>
void launchPick(const PickArgs& a, int blocks, size_t smemBytes, cudaStream_t s) {
  B200_CUDA(cudaFuncSetAttribute(maxminKernel<kRes>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smemBytes)));
  int perSm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, maxminKernel<kRes>, kThreads, smemBytes));
  B200_REQUIRE(perSm >= 1, "maxmin kernel does not fit on an SM");
  PickArgs arg    = a;
  void*    args[] = {&arg};
  B200_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(maxminKernel<kRes>), dim3(blocks), dim3(kThreads), args, smemBytes, s));
  g_launchCount.fetch_add(1);
}

size_t staticSmem(const void* fn) {
  cudaFuncAttributes fa{};
  B200_CUDA(cudaFuncGetAttributes(&fa, fn));
  return fa.sharedSizeBytes;
}

}  // namespace

unsigned long long readMaxminStat(int i) { return readDeviceCounter(g_maxminStat, i); }

}  // namespace b200

using namespace b200;

extern "C" int b200mol_maxmin_pick(const uint32_t* d_fp, size_t nPool, int words, int metric, const int32_t* h_first, int nFirst,
                                   int pickSize, double threshold, int32_t* d_picks, double* d_threshold, void* stream) {
  return guarded([&] {
    const Measure m = measureOfMetric(metric);
    requireFingerprintWidth(words);
    B200_REQUIRE(nPool >= 1 && nPool < (1ull << 31), "pool size must be in [1, 2^31) (got %zu)", nPool);
    B200_REQUIRE(pickSize >= 1 && static_cast<size_t>(pickSize) <= nPool, "pickSize must be in [1, pool size] (got %d, pool %zu)",
                 pickSize, nPool);
    B200_REQUIRE(nFirst >= 1 && nFirst <= pickSize, "need 1 <= first picks <= pickSize (got %d, pickSize %d)", nFirst, pickSize);
    B200_REQUIRE(h_first && d_fp && d_picks && d_threshold, "null pointer");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(d_fp) & 15) == 0, "fingerprint buffer must be 16-byte aligned");
    {
      std::vector<char> seen(nPool, 0);
      for (int f = 0; f < nFirst; ++f) {
        B200_REQUIRE(h_first[f] >= 0 && static_cast<size_t>(h_first[f]) < nPool, "first pick %d is outside the pool", h_first[f]);
        B200_REQUIRE(!seen[h_first[f]], "first pick %d is repeated", h_first[f]);
        seen[h_first[f]] = 1;
      }
    }
    cudaStream_t s = asStream(stream);
    const int    n = static_cast<int>(nPool), chunks = words / 4;
    int          G = 1;
    while (G * 2 <= chunks && G < 16) G *= 2;  // lanes per fingerprint: every lane takes at most two 16-byte words

    Scratch<int32_t> pop(nPool, s);
    launchRowPopcount(d_fp, nPool, words, pop.get(), s);
    B200_CUDA(cudaMemcpyAsync(d_picks, h_first, sizeof(int32_t) * nFirst, cudaMemcpyHostToDevice, s));
    if (pickSize > nFirst) B200_CUDA(cudaMemsetAsync(d_picks + nFirst, 0xFF, sizeof(int32_t) * (pickSize - nFirst), s));
    resetDeviceCounters(g_maxminStat, s);

    const int blocks = std::max(1, std::min(smCount(), (n + kMinSlice - 1) / kMinSlice));
    const int slice  = (n + blocks - 1) / blocks;
    int       dev = 0, optin = 0;
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const size_t fpBytes = static_cast<size_t>(slice) * chunks * 16, stateBytes = static_cast<size_t>(slice) * 16;
    const size_t budgetRes = static_cast<size_t>(optin) - staticSmem(reinterpret_cast<const void*>(maxminKernel<true>));
    const size_t budget    = static_cast<size_t>(optin) - staticSmem(reinterpret_cast<const void*>(maxminKernel<false>));
    const bool   wantRes   = g_maxminResidentRows < 0 || (g_maxminResidentRows > 0 && nPool <= static_cast<size_t>(g_maxminResidentRows));
    const bool   resident  = wantRes && fpBytes + stateBytes <= budgetRes;
    const bool   stateSh   = resident || stateBytes <= budget;
    g_maxminResidentLast   = resident ? 1 : 0;

    Scratch<double>  slotV(3 * static_cast<size_t>(blocks), s), gBound(stateSh ? 0 : static_cast<size_t>(blocks) * slice, s);
    Scratch<int32_t> slotI(3 * static_cast<size_t>(blocks), s), gApplied(stateSh ? 0 : static_cast<size_t>(blocks) * slice, s),
      gPop(stateSh ? 0 : static_cast<size_t>(blocks) * slice, s);
    PickArgs a{};
    a.fp = reinterpret_cast<const uint4*>(d_fp), a.pop = pop.get();
    a.n = n, a.chunks = chunks, a.group = G, a.slice = slice, a.cosine = m.kind == kCosine;
    a.deferred = g_maxminMode == 1, a.nFirst = nFirst, a.pickSize = pickSize, a.threshold = threshold >= 0.0 ? threshold : -1.0;
    a.picks = d_picks, a.thresholdOut = d_threshold, a.slotV = slotV.get(), a.slotI = slotI.get();
    a.gBound = gBound.get(), a.gApplied = gApplied.get(), a.gPop = gPop.get();
    if (resident) launchPick<true>(a, blocks, fpBytes + stateBytes, s);
    else launchPick<false>(a, blocks, stateSh ? stateBytes : 0, s);
  });
}
