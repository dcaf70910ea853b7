// What the exact top-k searches share (topk.cu on packed bits, count_similarity.cu on count vectors): the order of the
// contract, the CTA-wide bitonic sort of the select and scan kernels, and the sizes of their lists and candidate slots.
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

}  // namespace
}  // namespace b200
