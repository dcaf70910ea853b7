// Internal interface of the N x M popcount-similarity tile (used by tanimoto.cu and butina.cu).
#pragma once
#include <cstdint>

#include "common.cuh"

namespace b200 {

// What the tile kernel does with the 128x128 integer intersection counts.
enum SimMode : int {
  kMaterialiseTanimoto = 0,  // fp64 similarity matrix
  kMaterialiseCosine   = 1,
  kCountTanimoto       = 2,  // thresholded neighbour counts (+ optional edge list)
  kCountCosine         = 3,
  kListCosine          = 4,  // edges only: every pair with sim >= cutoff, possibly with false positives (tensor tile:
                             // a float bound, unordered; the SIMT fallback runs kCountCosine and lists exactly)
};

struct SimLaunch {
  const uint32_t* x      = nullptr;  // [nX][words]
  const uint32_t* y      = nullptr;  // [nY][words]
  size_t          nX     = 0;
  size_t          nY     = 0;
  int             words  = 0;
  // materialise
  double* out = nullptr;  // [nX][nY]
  // count
  double   cutoff      = 0.0;      // neighbour iff 1 - sim <= cutoff (fp64)
  bool     atLeast     = false;    // ... or, when set, iff sim >= cutoff (fp64; the threshold search)
  int      sign        = 1;        // counts += sign * hits
  int32_t* rowCounts   = nullptr;  // [nX]
  bool     symmetric   = false;    // x == y: visit tiles tn >= tm only, skip the diagonal pairs, update both endpoints
  uint32_t groupOffset = 0;        // multi-GPU row sharding: this call covers tile-row groups (32 x 128 rows each)
  uint32_t groupStride = 1;        //   groupOffset, groupOffset + groupStride, ...
  int2*    edges       = nullptr;  // optional: neighbour pairs (i, j) appended here (symmetric: i < j)
  unsigned long long* edgeCursor = nullptr;  // device counter; entries beyond edgeCap are dropped (cursor still advances)
  unsigned long long  edgeCap    = 0;
};

// Launch the tile kernel(s). Row popcounts and the threshold table are computed internally (stream-ordered scratch).
void launchSimilarity(SimMode mode, const SimLaunch& p, cudaStream_t stream);

// pop[i] = popcount of row i
void launchRowPopcount(const uint32_t* fp, size_t n, int words, int32_t* pop, cudaStream_t s);

// The similarity of a pair from its integer counts, as the materialise modes store it: 0 for an empty intersection, else
// the correctly rounded fp64 quotient c / (a + b - c) (the tensor tile's reciprocal + Newton step gives the same bits, see
// tanimoto_tc.cu) or c / sqrt(a b) from the same three correctly rounded operations.
__device__ __forceinline__ double simFromCounts(int c, int a, int b, bool cosine) {
  if (c == 0) return 0.0;
  if (cosine) return __ddiv_rn(static_cast<double>(c), __dsqrt_rn(__dmul_rn(static_cast<double>(a), static_cast<double>(b))));
  return __ddiv_rn(static_cast<double>(c), static_cast<double>(a + b - c));
}

// ---- top-k search: what topk.cu uses of the tensor-core tile (tanimoto_tc.cu) ----
// one u8 (0 / 1) per bit of n fingerprints
void launchExpandBits(const uint32_t* fp, size_t n, int words, uint8_t* out, cudaStream_t s);
bool topkTileEligible(int words);  // the tile takes widths that are multiples of 128 bits up to 4096
// One pass of the expanded queries over an expanded column slab of the library (caller's indices colBase ..): for every
// pair that could beat its row's bar[row] = {c, |A| + |B|, column, float bits of a lower bound of the value} of the row's
// current k-th best, the caller's column index goes to cand[row][at], at = count[row]++, while at < cap.
void launchTopkTile(bool cosine, const uint8_t* expQ, size_t nQ, const int32_t* popQ, const uint8_t* expLib, size_t nCols,
                    const int32_t* popCols, int words, const int4* bar, uint32_t* cand, uint32_t* count, uint32_t cap,
                    uint32_t colBase, cudaStream_t s);

}  // namespace b200
