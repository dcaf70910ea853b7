// What the exact top-k searches share (topk.cu on packed bits, count_similarity.cu on count vectors): the order of the
// contract, the CTA-wide bitonic sort of the select and scan kernels, the scan kernels' CTA-local list, and the sizes of
// their lists and candidate slots.
#pragma once
#include <cstdint>

#include "../../include/b200mol.h"

namespace b200 {
namespace {  // (each search's kernels get their own copies, compiled with them)

constexpr int      kTopkMax    = B200MOL_TOPK_MAX;
constexpr int      kSelThreads = 256;
constexpr int      kSelItems   = 2048;  // items a CTA sorts at most: the list (<= kTopkMax) + the candidate slots (<= kCapMax)
constexpr int      kCapMax     = kSelItems - kTopkMax;
constexpr uint32_t kNoCand     = 0xFFFFFFFFu;
constexpr int32_t  kNoIdx      = 0x7fffffff;

// The contract's order: value descending, column ascending. For Tanimoto this is also the order of the integer ratios
// (the tile's filter compares those, see tanimoto_tc.cu): equal ratios round to the same fp64 and distinct ratios with
// denominators <= 8192 differ by far more than an ulp. For cosine the fp64 values themselves are the only order there is.
// Dice, 2c / (|A| + |B|), is an increasing function of Tanimoto's c / (|A| + |B|) ratio as well, with the same ties: a
// Dice search is the Tanimoto search, whose values topkDiceValuesKernel then rewrites. General Tversky orders by the fp64
// value, like cosine (the kernels' WEIGHTED instantiations).
__device__ __forceinline__ bool better(double v1, int32_t i1, double v2, int32_t i2) { return v1 > v2 || (v1 == v2 && i1 < i2); }

// val / idx [0, n2) in shared memory, n2 a power of two, best first. Called by the whole CTA.
__device__ void sortBestFirst(double* val, int32_t* idx, int n2) {
  for (int size = 2; size <= n2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < n2 / 2; t += blockDim.x) {
        const int    lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const double vl = val[lo], vh = val[hi];
        const int32_t il = idx[lo], ih = idx[hi];
        const bool   up = (lo & size) == 0;  // this block ends best first
        if (up ? better(vh, ih, vl, il) : better(vl, il, vh, ih)) {
          val[lo] = vh, idx[lo] = ih;
          val[hi] = vl, idx[hi] = il;
        }
      }
    }
  __syncthreads();
}

__device__ __forceinline__ int nextPow2(int n) {
  int p = 2;
  while (p < n) p <<= 1;
  return p;
}

// The CTA-local list of a scan kernel: columns [c0, c1) of one query, a thread per column, value(col) the column's fp64
// value. A column that beats the bar (barV, barI) is parked in val / idx [k ..); when that fills up, the parked entries
// are sorted with the list [0, k) and cut to k, which raises the bar. A final cut leaves the CTA's k best, best first,
// in val / idx [0, k). nPend (0), barV and barI are in shared memory, set before the call. Called by the whole CTA.
template <class Value>
__device__ __forceinline__ void scanBest(double* val, int32_t* idx, int k, int& nPend, double& barV, int32_t& barI, uint32_t c0,
                                         uint32_t c1, Value value) {
  const int tid  = threadIdx.x;
  const int room = kSelItems - k - kSelThreads;  // pending entries from which a round could run out of slots
  auto cut = [&]() {  // sort list + pending, keep k, raise the bar to the k-th if there is one
    const int n2 = nextPow2(k + nPend);
    for (int i = k + nPend + tid; i < n2; i += kSelThreads) val[i] = -1.0, idx[i] = kNoIdx;
    sortBestFirst(val, idx, n2);
    if (tid == 0) {
      nPend = 0;
      if (idx[k - 1] != kNoIdx && better(val[k - 1], idx[k - 1], barV, barI)) barV = val[k - 1], barI = idx[k - 1];
    }
    __syncthreads();
  };
  for (uint32_t base = c0; base < c1; base += kSelThreads) {
    const uint32_t col = base + tid;
    if (col < c1) {
      const double v = value(col);
      if (better(v, static_cast<int32_t>(col), barV, barI)) {
        const int at = k + atomicAdd(&nPend, 1);
        val[at] = v, idx[at] = static_cast<int32_t>(col);
      }
    }
    __syncthreads();
    const int pending = nPend;
    __syncthreads();  // (every thread has read it before the next round adds to it)
    if (pending > room) cut();
  }
  cut();
}

}  // namespace
}  // namespace b200
