// Lower-triangle tile walk shared by the conformer pair matrices (tfd.cu, conformer_rmsd.cu). A molecule with T tiles
// per side has T(T+1)/2 units (ti, tj), tj <= ti, numbered row-major; the call plans a prefix sum of units over its
// molecules on the host, and persistent CTAs take global unit numbers from an atomic queue and map them back here.
#pragma once
#include <cstdint>

namespace b200 {

// units of a T x T tile grid's lower triangle, diagonal included
__host__ __device__ __forceinline__ int64_t lowerTriangleUnits(int64_t T) { return T * (T + 1) / 2; }

__device__ __forceinline__ int upperIndex(const int64_t* starts, int n, int64_t v) {  // largest m with starts[m] <= v
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (starts[mid] <= v) lo = mid;
    else hi = mid;
  }
  return lo;
}

// a molecule's local unit number -> tile (ti, tj), tj <= ti
__device__ __forceinline__ void lowerTriangleTile(int64_t loc, int& ti, int& tj) {
  ti = static_cast<int>((sqrt(8.0 * static_cast<double>(loc) + 1.0) - 1.0) * 0.5);
  while (static_cast<int64_t>(ti) * (ti + 1) / 2 > loc) --ti;
  while (static_cast<int64_t>(ti + 1) * (ti + 2) / 2 <= loc) ++ti;
  tj = static_cast<int>(loc - static_cast<int64_t>(ti) * (ti + 1) / 2);
}

}  // namespace b200
