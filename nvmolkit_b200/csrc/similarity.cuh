// Internal interface of the fingerprint-similarity stack: the measure of a call, the N x M popcount tiles that serve it
// (tanimoto.cu: SIMT, tanimoto_tc.cu: wgmma) and the fp64 value of a pair from its integer counts.
#pragma once
#include <cstddef>
#include <cstdint>
#include <functional>

#include "common.cuh"

namespace b200 {

// The similarity measure of a call. A measure is only made by measureOfMetric and measureOfWeights below, the library's
// one place that turns caller input into one.
enum MeasureKind : int { kTanimoto = 0, kCosine = 1, kDice = 2, kTversky = 3 };
struct Measure {
  MeasureKind kind  = kTanimoto;
  double      alpha = 0.0;  // Tversky's weights of the bits only in X (alpha) and only in Y (beta); Dice's are 1/2, 1/2
  double      beta  = 0.0;
};
// Dice and Tversky: the value is tverskyFromCounts of the weights (kernels instantiated for these two take it so)
__host__ __device__ constexpr bool isWeighted(MeasureKind k) { return k == kDice || k == kTversky; }

// A B200MOL_METRIC_* code
inline Measure measureOfMetric(int metric) {
  B200_REQUIRE(metric == B200MOL_METRIC_TANIMOTO || metric == B200MOL_METRIC_COSINE, "unknown metric %d", metric);
  return Measure{metric == B200MOL_METRIC_COSINE ? kCosine : kTanimoto};
}

// Tversky weights: finite, 0 <= alpha, beta <= 1000 (the range the float tile filters are derived for; NaN fails the
// comparisons). (1/2, 1/2) is Dice, which runs on the Tanimoto machinery (integer ratio order, threshold table), and
// (1, 1) Tanimoto itself: the same bits as the general expression in both cases.
inline Measure measureOfWeights(double alpha, double beta) {
  B200_REQUIRE(alpha >= 0.0 && alpha <= 1000.0 && beta >= 0.0 && beta <= 1000.0,
               "Tversky weights must be finite with 0 <= alpha, beta <= 1000 (got alpha = %g, beta = %g)", alpha, beta);
  const MeasureKind kind = alpha == 0.5 && beta == 0.5 ? kDice : alpha == 1.0 && beta == 1.0 ? kTanimoto : kTversky;
  return Measure{kind, alpha, beta};
}

inline void requireFingerprintWidth(int words) {
  B200_REQUIRE(words > 0 && words % 4 == 0 && words <= 128,
               "fingerprint width must be a multiple of 128 bits and at most 4096 bits (got %d words)", words);
}

// What a tile does with the integer intersection counts of its pairs, for the call's measure (SimLaunch::measure).
// Each tile maps (operation, measure kind) to its kernel in one place: launchSimilarity (SIMT), kTensorKernels (wgmma).
enum SimMode : int {
  kMaterialise = 0,  // fp64 similarity matrix
  kCount       = 1,  // thresholded neighbour counts (+ optional edge list); Tanimoto and Dice (atLeast only) test with an
                     // integer threshold table, bit-exact with the fp64 predicate; cosine's runs on SIMT only
  kList        = 2,  // cosine and Tversky, atLeast: edges only, every pair with sim >= cutoff, possibly with false
                     // positives (tensor tile: a float bound, unordered; the SIMT tile lists exactly)
};

struct SimLaunch {
  const uint32_t* x      = nullptr;  // [nX][words]
  const uint32_t* y      = nullptr;  // [nY][words]
  size_t          nX     = 0;
  size_t          nY     = 0;
  int             words  = 0;
  Measure         measure;
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
void launchSimilarity(SimMode op, const SimLaunch& p, cudaStream_t stream);

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

// The Tversky similarity of a pair with popcounts a (the group-one fingerprint), b and intersection c, as every Tversky
// and Dice path stores it: 0 for an empty intersection, else c / ((alpha (a - c) + beta (b - c)) + c) with each product,
// sum and the quotient one fp64 operation rounded to nearest, in that order (never contracted into an FMA). The
// denominator is >= c > 0. Dice is (1/2, 1/2): its intermediates are exact, so it is RN(2c / (a + b)); (1, 1) is
// Tanimoto's RN(c / (a + b - c)) bit for bit.
__device__ __forceinline__ double tverskyFromCounts(int c, int a, int b, double alpha, double beta) {
  if (c == 0) return 0.0;
  return __ddiv_rn(static_cast<double>(c), __dadd_rn(__dadd_rn(__dmul_rn(alpha, static_cast<double>(a - c)),
                                                                 __dmul_rn(beta, static_cast<double>(b - c))),
                                                       static_cast<double>(c)));
}

// The value of a pair under m as every path stores it, in a kernel instantiated for the weighted measures (WEIGHTED:
// Dice and Tversky, from m's weights) or for Tanimoto and cosine (told apart at run time: only those two reach it, so any
// kind but Tanimoto is cosine, a test against zero).
template <bool WEIGHTED>
__device__ __forceinline__ double measureFromCounts(const Measure& m, int c, int a, int b) {
  if constexpr (WEIGHTED) return tverskyFromCounts(c, a, b, m.alpha, m.beta);
  else return simFromCounts(c, a, b, m.kind != kTanimoto);
}

// A float bound for the tile filters of the Tversky searches: can a pair with count c reach a value >= L, L a float
// lower bound of the bar (or threshold) at least 1e-5 (relative) below it? Tested as c - L d >= 0 with
// d = alpha_f (a - c) + (beta_f (b - c) + c) in float (fmaf), alpha_f, beta_f alpha and beta rounded to float.
// Why no pair whose fp64 value v >= V (V >= L (1 + 1e-5)) is dropped: every term of the denominator is >= 0, so
// rounding alpha and beta (2^-24 relative each) and the two fmaf (2^-24 each) give d <= D (1 + 2^-24)^3 < D (1 + 2e-7),
// D the exact real denominator; the fp64 evaluation errs by at most 4 ulp, so v >= V means c >= V D (1 - 5e-16).
// Then L d <= V D (1 - 1e-5 + 2e-7) < c. The final fmaf rounds once and keeps the sign of c - L d exactly. c and the
// popcounts (<= 4096) are exact floats. c = 0 (value 0) never beats a bar (its column comes earlier) nor reaches t > 0.
__device__ __forceinline__ bool tverskyMayReach(int c, int a, int b, float alphaF, float betaF, float L) {
  const float cf = static_cast<float>(c);
  const float d  = fmaf(alphaF, static_cast<float>(a - c), fmaf(betaF, static_cast<float>(b - c), cf));
  return c != 0 && fmaf(-L, d, cf) >= 0.0f;
}

// ---- top-k search: what topk.cu uses of the tensor-core tile (tanimoto_tc.cu) ----
// one u8 (0 / 1) per bit of n fingerprints
void launchExpandBits(const uint32_t* fp, size_t n, int words, uint8_t* out, cudaStream_t s);
bool topkTileEligible(int words);  // the tile takes widths that are multiples of 128 bits up to 4096
// One pass of the expanded queries over an expanded column slab of the library (caller's indices colBase ..): for every
// pair that could beat its row's bar[row] = {c, |A| + |B|, column, float bits of a lower bound of the value} of the row's
// current k-th best, the caller's column index goes to cand[row][at], at = count[row]++, while at < cap. Tanimoto filters
// with the integer ratio (.x, .y), cosine and Tversky with the float bound (.w). A Dice search is Tanimoto's (topk.cu).
void launchTopkTile(const Measure& m, const uint8_t* expQ, size_t nQ, const int32_t* popQ, const uint8_t* expLib, size_t nCols,
                    const int32_t* popCols, int words, const int4* bar, uint32_t* cand, uint32_t* count, uint32_t cap,
                    uint32_t colBase, cudaStream_t s);

// ---- threshold search (threshold.cu): one attempt protocol for packed bits and count vectors ----
// listPairs(list, vals, listCap, stat) enqueues the work that lists the pairs (i, j) of one attempt, at most listCap of
// them, with their values (i = -1: dropped), counting them at stat[0]; it may count kept pairs at stat[1] and non-empty
// rows at stat[2]. stat is zero on entry. nnzOf(stat) is the result size those counts give.
using ListPairs = std::function<void(int2* list, double* vals, unsigned long long listCap, unsigned long long* stat)>;
using ResultSize = std::function<unsigned long long(const unsigned long long* stat)>;
// The pass from a list of listCap entries, rerun once into a list of the exact size when it listed more; one host read
// per attempt. *hNnz = the result size; when it fits `cap` the pairs are written to the caller's CSR, indptr [nX + 1],
// indices / values [nnz], columns ascending: each kept pair, twice in a symmetric search together with one diagonal
// entry per row of popX > 0. nCols: the column count.
void thresholdCsr(unsigned long long listCap, const ListPairs& listPairs, const ResultSize& nnzOf, bool symmetric,
                  const int32_t* popX, size_t nX, size_t nCols, MeasureKind kind, int64_t* indptr, int32_t* indices,
                  double* values, uint64_t cap, uint64_t* hNnz, cudaStream_t s);

// ---- fused Butina (butina.cu): one driver for the bit and the count pass ----
// One pass over the pairs of a neighbour graph: counts[] += the degrees, and the (i < j) pairs appended to edges[] at
// *cursor while below cap (the cursor ends at the pair total).
using EdgePass = std::function<void(int32_t* counts, int2* edges, unsigned long long cap, unsigned long long* cursor)>;
// The pass with a zeroed cursor of its own; *hNEdges (when given) = the pair total, read with a stream synchronise.
void edgePassWithTotal(const EdgePass& pass, int32_t* counts, int2* edges, unsigned long long cap, uint64_t* hNEdges,
                       cudaStream_t s);
// Butina on n > 0 points from their pass: an edge list of 64 per point, one rerun at the exact size for a denser graph,
// then the clusters as b200mol_butina_from_edges makes them (centroids and dNClusters may be NULL).
void fusedButina(size_t n, const EdgePass& pass, int32_t* ids, int32_t* centroids, int32_t* dNClusters, int32_t* hNClusters,
                 cudaStream_t s);
// The result of clustering no points: zero clusters, in *hNClusters and *dNClusters where given.
void noClusters(int32_t* dNClusters, int32_t* hNClusters, cudaStream_t s);

}  // namespace b200
