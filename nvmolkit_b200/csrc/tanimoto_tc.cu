// Popcount similarity on the Hopper tensor cores (wgmma, sm_90a): the thresholded neighbour pass of the fused Butina
// path and the materialised Tanimoto / cosine matrices.
//
// |A & B| of two bit vectors is the dot product of their 0/1 expansions, so the N x M intersection-count matrix is a
// GEMM with exact small-integer sums. The SIMT tile (tanimoto.cu) is bound by the POPC issue rate (64 POPC per
// 2048-bit pair); here the contraction runs on the tensor cores:
//
//   pre-pass   bits -> one u8 per bit (0 / 1) once per fingerprint set, 2 KB per 2048-bit row; for the neighbour pass a
//              row operand is the SUM of S = 4 fingerprints and a column operand the sum of C = 1, 2 or 4 (bytes <= 4,
//              s32 accumulation exact), so one accumulator bounds S * C pair counts. The superposed pass first gathers
//              the fingerprints in popcount order (stable), so that a group sums fingerprints of nearly equal popcount
//              and the pre-filter's bound, set by the group's smallest popcount, is about as tight as a single pair's.
//   tile       128 x 256 accumulators per step of a persistent CTA (optionally a cluster of two CTAs that share the
//              column operand through TMA multicast)
//   warp 0     TMA producer: [128 | 256 rows][128 B] K-chunks, SWIZZLE_128B, mbarrier ring of 4 stages; per tile also
//              the rows' and columns' {popcount, pre-filter term} (computed once per pass by tileMetaKernel) with one
//              bulk copy into a 2-deep metadata ring, so the consumers issue no global load and meet at no barrier
//              between tiles
//   warpgroups 1-2  each issues wgmma.mma_async m64n256k32 .s32.u8.u8 for 64 of the tile's rows (accumulators in
//              registers) and runs the epilogue on them: a fixed-point pre-filter (256 acc - floor(256 alpha |B_j|) >=
//              floor(256 alpha |A_i|)) decides "no pair of this group can reach its threshold"; survivors go to a candidate list that
//              verifyCandidatesKernel re-counts exactly with the integer threshold table (bit-exact with the fp64
//              predicate, see tanimoto.cu) and maps back to the caller's indices. Unsuperposed (S = C = 1) the same warps apply the exact test themselves:
//              neighbour counts for both endpoints + edges. Candidates and edges are staged per warp in shared memory
//              and leave with one global atomic per 128-entry flush. Materialise modes write fp64 Tanimoto / cosine
//              values straight from the accumulator registers.
// A pilot over a prefix sample (itself ordered by popcount) picks C for the data at hand; a candidate-list overflow
// reruns with fewer pairs per accumulator before anything has been counted.
//
// Replaces crossSimilarityKernelTensorOp (src/similarity_kernels.cu:104-240) + the Triton count kernel
// (nvmolkit/_fusedButina.py:99-179) for the fused Butina pass.
#include <cub/device/device_radix_sort.cuh>
#include <tuple>
#include <vector>

#include "options.cuh"
#include "profile.cuh"
#include "similarity.cuh"
#include "tma.cuh"

namespace b200 {
namespace {

constexpr int kTM      = 128;  // tile rows: two consumer warpgroups of 64
constexpr int kTN      = 256;  // tile columns: the N of one wgmma
constexpr int kTK      = 128;  // bytes (= bits of the fingerprint) per K chunk: one 128-byte swizzle row
constexpr int kStages  = 4;    // smem ring depth (48 KB per stage)
constexpr int kThreadsTC = 384;  // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: MMA + epilogue
constexpr int kABytes  = kTM * kTK;
constexpr int kBBytes  = kTN * kTK;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kRunStat      = 16;  // tile columns per unit of the row-stationary tile (the row operand is loaded once per unit)
constexpr int kMaxChunksStat = 8;   // ... whose row operand stays in shared memory: 8 K-chunks x 16 KB (fingerprints <= 1024 bits)
constexpr int kStagesStat   = 2;   // ... and whose ring holds the column operand only (32 KB per stage, next to 128 KB of row operand)
constexpr int kGroupRows = 8192;  // fingerprints per row group: the unit of L2 reuse of the column operand AND of the
                                  // multi-GPU row split (independent of the tile variant and of the superposition factor)

struct TcParams {
  uint32_t        n;  // X == Y (symmetric) or nX/nY
  uint32_t        nY;
  int             kChunks;
  uint32_t        tilesM, tilesN;
  int             symmetric;
  uint32_t        groupOffset, groupStride;  // multi-GPU: this rank owns tile-row groups with group % stride == offset
  const int2*     rowMeta;  // per row of the X operand, whole tiles: {popcount, floor(256 alpha popcount)} (tileMetaKernel)
  const int2*     colMeta;  // per row of the Y operand (tile column), whole tiles: {popcount, -floor(256 alpha popcount)}
  const uint16_t* thresh;
  int             threshLen;
  int             sign;
  int32_t*        counts;
  int32_t*        countsY;  // == counts in symmetric mode; nullptr in X-vs-Y mode (rows only)
  int2*           edges;
  unsigned long long* edgeCursor;
  unsigned long long  edgeCap;
  double*         out;       // materialise modes: [n][nY] fp64
  int             outVec;    // materialise modes: out 16-byte aligned and nY even (two values per store)
  const double*   recipG;    // RN(1/u), u = 0 .. 2 * bits (global memory, 64 KB at most: L1-resident)
  // Row superposition (count mode): a row of the X operand is the SUM of superS consecutive fingerprints (values 0..4),
  // so one accumulator bounds superS pair counts at once; n / tilesM then count SUPER rows, rowMeta holds the smallest
  // popcount of each super row, and the epilogue only lists candidates (super row, column) for the exact verification
  // kernel. rowSpan = fingerprints per tile row = kTM * superS.
  int                 superS;
  int                 superC;   // the same for the columns of the Y operand: one accumulator then bounds superS * superC pair counts
  uint32_t            colSpan;  // fingerprints per tile column = kTN * superC
  float               alpha;    // (1 - cutoff) / (2 - cutoff), rounded down: a pair can only pass with c >= alpha (|A| + |B|)
  uint32_t            rowSpan;
  uint32_t            groupTiles;  // tile rows per row group (a power of two): kGroupRows fingerprints whatever superS is
  int2*               cand;
  unsigned long long* candCursor;
  unsigned long long  candCap;
  // Popcount band (ordered count passes; nullptr elsewhere): per row group, the end of the tile columns that can hold a
  // neighbour of any of its rows (popcountBandKernel). The walk skips the tile columns at and past it.
  const uint32_t*     bandEnd;
  unsigned long long* walked;  // [0] += units walked (once per CTA pair), [1] += tiles a CTA ran; nullptr: not counted
  // Top-k search (topk.cu): per query row its running bar {c, |A| + |B|, column, float bits of a lower bound of the value}
  // of the current k-th best; an accumulator that could beat it leaves as its column index in the row's candidate slots.
  const int4* topkBar;
  uint32_t*   topkCand;   // [n][topkCap] caller's column indices
  uint32_t*   topkCount;  // [n] slots asked for (may pass topkCap: the row is then redone, nothing of it is merged)
  uint32_t    topkCap;
  uint32_t    topkColBase;  // caller's index of the Y operand's first row (the library is searched in column slabs)
  // Tversky modes: the weights in fp64 (the matrix) and rounded to float (the filters, tverskyMayReach), and the list
  // mode's float lower bound of the threshold
  double tvAlpha, tvBeta;
  float  tvAlphaF, tvBetaF, tvBound;
};

// The popcount band. A pair with popcounts a, b and intersection c <= min(a, b) can only be a neighbour if
// c >= thresh[a + b]. thresh is not monotone where no pair reaches a sum (0xFFFF at s < 2, and at small odd s for small
// cutoffs), so the band tests its suffix minimum tmin[s] = min over s' >= s of thresh[s']: tmin[A + b] > A says that no
// column of popcount b' >= b can be a neighbour of a row of popcount A, and then none of a row of popcount a <= A either
// (tests/test_pair_pass_popcount_band_gpu.py checks both against the fp64 predicate for every pair up to 4096 bits). For a
// row group whose largest popcount is A, no column past the first one this cuts can be a neighbour of any of its rows.
__host__ __device__ __forceinline__ bool bandCuts(const uint16_t* tmin, int A, int b) { return tmin[A + b] > A; }

enum TcMode : int {
  kTcCount = 0, kTcTanimoto = 1, kTcCosine = 2, kTcTopkTanimoto = 3, kTcTopkCosine = 4, kTcListCosine = 5,
  kTcDice = 6, kTcTversky = 7, kTcTopkTversky = 8, kTcListTversky = 9
};
}  // namespace
int g_tensorCluster = 1;  // count tile in clusters of two CTAs with a multicast column operand (option "similarity_tensor_cluster":
                          // 0 one CTA per tile, 1 the pair, 2 the pair too (kept for callers written for the CTA-pair MMA
                          // that Hopper lacks), 3 the pair with the row operand stationary)
namespace {

__global__ void expandBitsKernel(const uint32_t* __restrict__ fp, size_t nWords, uint4* __restrict__ out) {
  const size_t w = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (w >= nWords) return;
  const uint32_t x = fp[w];
  uint32_t       b[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {  // 4 bits -> 4 bytes of 0/1 (bit j of the nibble lands in byte j)
    const uint32_t nib = (x >> (4 * q)) & 0xFu;
    b[q]               = (nib * 0x00204081u) & 0x01010101u;
  }
  out[2 * w]     = make_uint4(b[0], b[1], b[2], b[3]);
  out[2 * w + 1] = make_uint4(b[4], b[5], b[6], b[7]);
}

// Superposed operand: byte k of row R = sum over s < S of bit k of fingerprint S R + s (0..4, no carry between bytes).
// One thread per 32 fingerprint bits.
__global__ void expandBitsSuperKernel(const uint32_t* __restrict__ fp, size_t n, int words, int S, size_t nSuper,
                                      uint4* __restrict__ out) {
  const size_t t = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= nSuper * static_cast<size_t>(words)) return;
  const size_t R = t / words;
  const int    w = static_cast<int>(t % words);
  uint32_t     b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int s = 0; s < S; ++s) {
    const size_t i = R * S + s;
    if (i >= n) break;
    const uint32_t x = fp[i * words + w];
#pragma unroll
    for (int q = 0; q < 8; ++q) b[q] += (((x >> (4 * q)) & 0xFu) * 0x00204081u) & 0x01010101u;
  }
  out[2 * t]     = make_uint4(b[0], b[1], b[2], b[3]);
  out[2 * t + 1] = make_uint4(b[4], b[5], b[6], b[7]);
}

// out row i = fp row perm[i]; one thread per 16 bytes
__global__ void gatherRowsKernel(const uint4* __restrict__ fp, const int32_t* __restrict__ perm, size_t n, int chunks,
                                 uint4* __restrict__ out) {
  const size_t t = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * static_cast<size_t>(chunks)) return;
  const size_t i = t / chunks;
  out[t]         = fp[static_cast<size_t>(perm[i]) * chunks + t % chunks];
}

// What the tile epilogue needs of each operand row, computed once per pass and fetched by the producer per tile with
// one bulk copy: .x = the smallest popcount among the S fingerprints summed into the row (the conservative pre-filter
// needs the lowest threshold any pair of the group can have; with S = 1 the popcount itself), .y = dir * floor(256
// alpha .x), the pre-filter's fixed-point term (dir = +1 for rows, -1 for columns). Rows past the end, up to whole
// tiles (nPad), get popcount 0 and dir * 0x3fffffff, which no accumulator passes.
__global__ void tileMetaKernel(const int32_t* __restrict__ pop, size_t n, int S, size_t nSuper, size_t nPad, float alpha, int dir,
                               int2* __restrict__ out) {
  const size_t R = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (R >= nPad) return;
  if (R >= nSuper) {
    out[R] = make_int2(0, dir * 0x3fffffff);
    return;
  }
  int m = 0x3fffffff;
  for (int s = 0; s < S; ++s)
    if (R * S + s < n) m = min(m, pop[R * S + s]);
  out[R] = make_int2(m, dir * static_cast<int>(floorf(__fmul_rd(256.0f * alpha, static_cast<float>(m)))));
}

// Exact verification of the candidates of a superposed pass: one warp per (super row R, super column J), for each of
// the S * C pairs (i = S R + s, j = C J + c) of the group the exact count |X_i & Y_j| and the exact integer threshold
// test; counts for both endpoints and the (i < j) edge list exactly as the unsuperposed epilogue produces them.
// x, y, popX and popY are in the pass's popcount order; permX / permY map a row back to the caller's index, where the
// counts land and the edges are written (symmetric: as (min, max) of the two, so that still i < j).
// A block takes 64 consecutive candidates at a time (one coalesced load; the warp that listed them worked on one quarter
// of a tile row, so their row operands are L1 / L2 hits), a warp one candidate: all of its 128-bit row loads and the two
// popcount loads are in flight together; edges are parked in 64 shared-memory slots per warp that leave with ONE global
// atomic per flush.
__global__ void __launch_bounds__(256) verifyCandidatesKernel(const uint32_t* __restrict__ x, const uint32_t* __restrict__ y, int words,
                                                             const int2* __restrict__ cand, unsigned long long nCand, int S, int C,
                                                             uint32_t nRows, uint32_t nCols, int symmetric,
                                                             const int32_t* __restrict__ popX, const int32_t* __restrict__ popY,
                                                             const int32_t* __restrict__ permX, const int32_t* __restrict__ permY,
                                                             const uint16_t* __restrict__ thresh, int sign, int32_t* counts,
                                                             int32_t* countsY, int2* edges, unsigned long long* edgeCursor,
                                                             unsigned long long edgeCap) {
  constexpr int kStage = 64, kFlight = 1, kChunk = 64;  // a block takes 64 consecutive candidates at a time: the epilogue
  // warp that listed them worked on ONE quarter of a tile row (32 super rows = 32 KB of fingerprints), so most of their
  // row operands are L1 hits for the block
  __shared__ int2 stage[8][kStage];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = 32 / (S * C), sub = lane / G, gl = lane % G;  // S, C are 1, 2 or 4: G lanes per pair
  const int chunks = words / 4;                                // uint4 per fingerprint
  int       nStaged = 0;
  auto flush = [&]() {
    if (nStaged == 0) return;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(edgeCursor, static_cast<unsigned long long>(nStaged));
    base = __shfl_sync(0xffffffffu, base, 0);
    __syncwarp();
    for (int k = lane; k < nStaged; k += 32)
      if (base + k < edgeCap) edges[base + k] = stage[warp][k];
    __syncwarp();
    nStaged = 0;
  };
  __shared__ int2 chunkCand[kChunk];
  for (unsigned long long chunk = static_cast<unsigned long long>(blockIdx.x) * kChunk; chunk < nCand; chunk += static_cast<unsigned long long>(gridDim.x) * kChunk) {
  // the block's 64 candidates in one coalesced load (a warp fetching its own entry would start every candidate with a
  // dependent L2 round trip)
  __syncthreads();
  if (threadIdx.x < kChunk) chunkCand[threadIdx.x] = chunk + threadIdx.x < nCand ? cand[chunk + threadIdx.x] : make_int2(-1, -1);
  __syncthreads();
  for (int it = 0; it < kChunk / (8 * kFlight); ++it) {
    uint32_t     iOf[kFlight], jOf[kFlight];
    bool         live[kFlight];
    int          popSum[kFlight];
    const uint4 *xi[kFlight], *yj[kFlight];
#pragma unroll
    for (int f = 0; f < kFlight; ++f) {
      const int2 rj   = chunkCand[it * 8 * kFlight + warp * kFlight + f];
      const bool have = rj.x >= 0;
      iOf[f]          = static_cast<uint32_t>(rj.x) * S + sub / C;
      jOf[f]          = static_cast<uint32_t>(rj.y) * C + sub % C;
      live[f]         = have && iOf[f] < nRows && jOf[f] < nCols && !(symmetric && iOf[f] >= jOf[f]);
      xi[f]           = reinterpret_cast<const uint4*>(x + static_cast<size_t>(live[f] ? iOf[f] : 0) * words);
      yj[f]           = reinterpret_cast<const uint4*>(y + static_cast<size_t>(live[f] ? jOf[f] : 0) * words);
      popSum[f]       = (gl == 0 && live[f]) ? popX[iOf[f]] + popY[jOf[f]] : 0;  // (in flight together with the rows)
    }
    int cnt[kFlight] = {};
    for (int q = gl; q < chunks; q += 4 * G) {  // (4 chunks per lane and candidate in flight)
      uint4 a[kFlight][4], b4[kFlight][4];
#pragma unroll
      for (int f = 0; f < kFlight; ++f)
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (q + u * G < chunks) a[f][u] = xi[f][q + u * G], b4[f][u] = yj[f][q + u * G];
#pragma unroll
      for (int f = 0; f < kFlight; ++f)
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (q + u * G < chunks)
            cnt[f] += __popc(a[f][u].x & b4[f][u].x) + __popc(a[f][u].y & b4[f][u].y) + __popc(a[f][u].z & b4[f][u].z) +
                      __popc(a[f][u].w & b4[f][u].w);
    }
#pragma unroll
    for (int f = 0; f < kFlight; ++f) {
      int v = cnt[f];
      for (int o = G >> 1; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      const bool hit = gl == 0 && live[f] && v >= thresh[popSum[f]];
      int        i = 0, j = 0;  // the pair in the caller's order
      if (hit) {
        i = permX[iOf[f]], j = permY[jOf[f]];
        if (symmetric && i > j) {
          const int t = i;
          i = j, j = t;
        }
        atomicAdd(counts + i, sign);
        if (countsY) atomicAdd(countsY + j, sign);
      }
      if (edges) {
        const unsigned hits = __ballot_sync(0xffffffffu, hit);
        if (hits) {
          const int total = __popc(hits);  // <= 16
          if (nStaged + total > kStage) flush();
          if (hit) stage[warp][nStaged + __popc(hits & ((1u << lane) - 1u))] = make_int2(i, j);
          nStaged += total;
        }
      }
    }
  }
  }
  if (edges) flush();
}

// The results of an unsuperposed pass over the fingerprints in popcount order, moved to the caller's indices:
// counts[permX[i]] += countsOrd[i] (a permutation: no two threads meet), and the edges the pass appended to the list
// ([*start, *end) within its capacity) renamed in place, as (min, max) when symmetric so that still i < j.
__global__ void mapBackKernel(const int32_t* __restrict__ countsOrd, const int32_t* __restrict__ permX, size_t nX, int32_t* counts,
                              const int32_t* __restrict__ permY, int symmetric, int2* edges, const unsigned long long* start,
                              const unsigned long long* end, unsigned long long cap) {
  const size_t t0 = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x, step = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = t0; i < nX; i += step)
    if (countsOrd[i]) counts[permX[i]] += countsOrd[i];
  if (!edges) return;
  const unsigned long long e1 = min(*end, cap);
  for (unsigned long long e = *start + t0; e < e1; e += step) {
    const int2 v = edges[e];
    int        i = permX[v.x], j = permY[v.y];
    if (symmetric && i > j) {
      const int t = i;
      i = j, j = t;
    }
    edges[e] = make_int2(i, j);
  }
}

// The popcount band of an ordered count pass, in one block: the suffix minimum of thresh (len entries) into shared
// memory, then one thread per row group of kGroupRows fingerprints. popX and popY are in the pass's (ascending) order, so
// the group's largest popcount is its last row's, and bandCuts is monotone along popY: a bisection finds the first column
// jCut it cuts. Tile columns at or past ceil(jCut / colSpan) hold no neighbour of the group, whatever the superposition.
constexpr int kBandThreads = 128;
__global__ void __launch_bounds__(kBandThreads) popcountBandKernel(const int32_t* __restrict__ popX, size_t nX,
                                                                   const int32_t* __restrict__ popY, size_t nY,
                                                                   const uint16_t* __restrict__ thresh, int len, uint32_t colSpan,
                                                                   uint32_t tilesN, uint32_t groups, uint32_t* __restrict__ bandEnd) {
  extern __shared__ uint16_t tmin[];
  __shared__ uint16_t carry[kBandThreads + 1];
  const int t = threadIdx.x, per = (len + kBandThreads - 1) / kBandThreads, i0 = t * per, i1 = min(len, i0 + per);
  uint16_t  m = 0xFFFF;
  for (int i = i1 - 1; i >= i0; --i) tmin[i] = m = min(m, thresh[i]);  // the suffix minimum within this thread's slice
  carry[t] = m;
  if (t == 0) carry[kBandThreads] = 0xFFFF;
  __syncthreads();
  if (t == 0)
    for (int k = kBandThreads - 1; k >= 0; --k) carry[k] = min(carry[k], carry[k + 1]);
  __syncthreads();
  for (int i = i0; i < i1; ++i) tmin[i] = min(tmin[i], carry[t + 1]);  // ... and past it
  __syncthreads();
  for (uint32_t g = t; g < groups; g += kBandThreads) {
    const int A  = popX[min(nX, (static_cast<size_t>(g) + 1) * kGroupRows) - 1];
    size_t    lo = 0, hi = nY;
    while (lo < hi) {
      const size_t mid = (lo + hi) / 2;
      if (bandCuts(tmin, A, popY[mid])) hi = mid;
      else lo = mid + 1;
    }
    bandEnd[g] = static_cast<uint32_t>(min(static_cast<size_t>(tilesN), (lo + colSpan - 1) / colSpan));
  }
}

// The cosine list tile's metadata: {popcount, float bits of scale sqrt(popcount)} per operand row, whole tiles; rows past
// the end get popcount 0 and 3e38, which no count reaches
__global__ void listMetaKernel(const int32_t* __restrict__ pop, size_t n, size_t nPad, float scale, int2* __restrict__ out) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nPad) return;
  if (i >= n) out[i] = make_int2(0, __float_as_int(3.0e38f));
  else out[i] = make_int2(pop[i], __float_as_int(scale * sqrtf(static_cast<float>(pop[i]))));
}

__global__ void recipTableKernel(double* __restrict__ r, int len) {  // r[u] = RN(1 / u), r[0] = 0
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u <= len) r[u] = u ? __drcp_rn(static_cast<double>(u)) : 0.0;
}

// ---- wgmma (sm_90a) ----
// K-major operand with the 128-byte swizzle TMA wrote it with: 8-row groups 1024 B apart (SBO), LBO unused for
// swizzled K-major layouts (1 by convention), layout type 1 = SWIZZLE_128B. Stage bases are 1024-byte aligned, so the
// base-offset field stays 0; a K step of 32 bytes inside the swizzle row is +2 in the 16-byte address field.
__device__ __forceinline__ uint64_t makeSmemDesc(uint32_t smemByteAddr) {
  return static_cast<uint64_t>((smemByteAddr & 0x3FFFFu) >> 4) | (static_cast<uint64_t>(1) << 16) |
         (static_cast<uint64_t>(1024 >> 4) << 32) | (static_cast<uint64_t>(1) << 62);
}

#define B200_WG_R4(i) "+r"(d[i]), "+r"(d[(i) + 1]), "+r"(d[(i) + 2]), "+r"(d[(i) + 3])
#define B200_WG_R16(i) B200_WG_R4(i), B200_WG_R4((i) + 4), B200_WG_R4((i) + 8), B200_WG_R4((i) + 12)
#define B200_WG_R64(i) B200_WG_R16(i), B200_WG_R16((i) + 16), B200_WG_R16((i) + 32), B200_WG_R16((i) + 48)

// D[64 x 256] (+)= A[64 x 32] * B[256 x 32]^T, u8 x u8 -> s32, both operands K-major in shared memory. Thread t of the
// warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1): d[4 j .. 4 j + 3] =
// (row, col), (row, col + 1), (row + 8, col), (row + 8, col + 1).
__device__ __forceinline__ void wgmmaU8(uint32_t (&d)[128], uint64_t aDesc, uint64_t bDesc, uint32_t accumulate) {
  asm volatile(
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
    "wgmma.mma_async.sync.aligned.m64n256k32.s32.u8.u8 {"
    "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
    "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, "
    "%68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, "
    "%90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, "
    "%110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
    "}, %128, %129, p;\n\t}"
    : B200_WG_R64(0), B200_WG_R64(64)
    : "l"(aDesc), "l"(bDesc), "r"(accumulate));
}
#undef B200_WG_R64
#undef B200_WG_R16
#undef B200_WG_R4

// keeps the compiler from moving reads / writes of the accumulators across the asynchronous MMA's fence / wait
__device__ __forceinline__ void fenceAccumulators(uint32_t (&d)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void wgmmaFence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmmaCommit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmmaWait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// 16-byte shared-memory load that the compiler may not merge with another one of the same address: the count epilogue
// reads its column metadata in the pre-filter and again for the survivors, and keeping the pre-filter's 32 int4 alive
// until then would spill
__device__ __forceinline__ int4 ldsFresh(const int4* p) {
  int4 v;
  asm volatile("ld.volatile.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smemAddr(p)));
  return v;
}

// An accumulator the compiler may not share between the Tversky filters' two passes over the tile (the test and the
// listing): kept, the float terms of 128 accumulators would spill
__device__ __forceinline__ int fresh(int a) {
  asm volatile("" : "+r"(a));
  return a;
}

// The list of one epilogue warp of the count tile - candidates when superposed, else edges (if asked for): (row, column)
// pairs are parked in kStagePairs shared-memory slots and leave with ONE global atomic per flush, when the slots are
// full and at the end of the warp's work. The atomic's result (the store address) is waited on once per flush instead
// of once per column block with a hit. Entries past the list's capacity are dropped; the cursor still counts them.
constexpr int kStagePairs = 128;  // >= the 4 x 32 pairs one add() can bring
struct PairStage {
  int n;  // pairs parked in `slot` (the warp's kStagePairs shared-memory slots, passed in: no register holds the address)
  __device__ __forceinline__ void flush(const TcParams& p, int2* slot, int lane) {
    if (n == 0) return;
    const bool               super  = p.superS * p.superC > 1;
    int2* const              list   = super ? p.cand : p.edges;
    const unsigned long long cap    = super ? p.candCap : p.edgeCap;
    __syncwarp();
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(super ? p.candCursor : p.edgeCursor, static_cast<unsigned long long>(n));
    base = __shfl_sync(0xffffffffu, base, 0);
    for (int k = lane; k < n; k += 32)
      if (base + k < cap) list[base + k] = slot[k];
    __syncwarp();
    n = 0;
  }
  // the pairs of `bits` (bit e: row e < 2 ? r0 : r1, column c0 + (e & 1)) of every lane of the warp
  __device__ __forceinline__ void add(const TcParams& p, int2* slot, uint32_t bits, uint32_t r0, uint32_t r1, uint32_t c0, int lane) {
    const int mine = __popc(bits);
    int       incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    if (n + total > kStagePairs) flush(p, slot, lane);
    int at = n + incl - mine;
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if ((bits >> e) & 1u) slot[at++] = make_int2(static_cast<int>(e < 2 ? r0 : r1), static_cast<int>(c0 + (e & 1)));
    n += total;
  }
};

#ifdef B200_TC_TIMING
// clock64() attribution of the tile loop (make tctiming, tools/pair_pass_timing.py). Consumer warps (lane 0, summed over
// warps): 0 the wait for the tile's metadata, 1 fullBar waits, 2 wgmma waits, 3 pre-filter, 4 candidate / edge path
// (with the last flush), 5 warp-tiles, 6 the whole tile loop; 7 the producer thread's emptyBar waits.
__device__ unsigned long long g_tcClk[8];
#define B200_TC_T0(t) const long long t = clock64()
#define B200_TC_T1(t, slot) tcClk[slot] += clock64() - (t)
#else
#define B200_TC_T0(t)
#define B200_TC_T1(t, slot)
#endif

// Work units. A unit = one tile (CL = 0) or two vertically adjacent tiles of one tile column (CTA pairs: unit row r
// holds tile rows 2 r and 2 r + 1, the two CTAs share the column operand). Unit rows come in groups of G (p.groupTiles
// tile rows = kGroupRows fingerprints), a group sweeps the tile columns row-fastest (L2 reuse of the row operand). Only units that can hold a pair
// are enumerated: a rank walks the groups it OWNS, and a group starts at the first tile column that reaches past the
// diagonal for its top tile row (closed form), so that neither the other ranks' groups nor the lower triangle cost
// loop iterations.
// RUN > 1 (the row-stationary tile, CL = 3): a unit is a RUN of consecutive tile columns of one unit row - the row
// operand is loaded once per unit and stays in shared memory - and the units of a group go chunk-major (all rows of the
// group take column chunk q, then q + 1): the CTA pairs of a group stream the same column tiles at about the same time.
// In an ordered pass a group also ends at its popcount band (p.bandEnd): the tile columns past it hold no neighbour of
// any of its rows. The band is per group, so the rule that the upper tile of a pair decides for both still holds.
// Ownership is serpentine over cycles of `groupStride` groups (even cycles: group = cycle * stride + offset, odd
// cycles mirrored), which balances the triangle's shrinking rows across ranks to < 0.1 % (with the band on the bench
// data: tools/pilot_model.py prints the ranks' shares).
// A CTA walks units first, first + step, ... of the concatenated owned groups; (cycle, index in group) are kept
// incrementally, the only divisions are by compile-time constants and happen once per group.
template <bool PAIR, int RUN = 1>
struct UnitWalk {
  uint32_t cycle, inGroup, units, gRows, tn0, group, step, G, gShift;
  bool     done;
  __device__ UnitWalk(const TcParams& p, uint32_t first, uint32_t stepBy)
      : cycle(0), inGroup(first), units(0), gRows(0), tn0(0), group(0), step(stepBy), G(PAIR ? p.groupTiles / 2 : p.groupTiles),
        gShift(0), done(false) {
    while ((1u << gShift) < G) ++gShift;  // G is a power of two
    settle(p);
  }
  __device__ void settle(const TcParams& p) {  // make (cycle, inGroup) point at an existing unit, or set done
    const uint32_t unitRows = PAIR ? (p.tilesM + 1) / 2 : p.tilesM;
    for (;;) {
      if (static_cast<uint64_t>(cycle) * p.groupStride * G >= unitRows) {
        done = true;
        return;
      }
      group = cycle * p.groupStride + ((cycle & 1u) ? p.groupStride - 1 - p.groupOffset : p.groupOffset);
      units = 0;
      if (static_cast<uint64_t>(group) * G < unitRows) {
        gRows = min(G, unitRows - group * G);
        // first tile column holding a pair with row < col for the group's top tile row tm0 = group * groupTiles:
        // (tn + 1) * colSpan - 1 > tm0 * rowSpan   (rowSpan / colSpan = fingerprints per tile row / tile column)
        tn0   = p.symmetric ? (group * p.groupTiles * p.rowSpan + 1u) / p.colSpan : 0u;
        const uint32_t tnLim = limit(p);
        if (tn0 < tnLim) units = gRows * ((tnLim - tn0 + RUN - 1) / RUN);
      }
      if (inGroup < units) return;
      inGroup -= units;
      ++cycle;
    }
  }
  // the end of the group's tile columns: its popcount band, if the pass has one (read again per unit rather than kept in
  // a register: the consumers' 128 accumulators leave none to spare)
  __device__ uint32_t limit(const TcParams& p) const { return p.bandEnd ? min(p.tilesN, __ldg(p.bandEnd + group)) : p.tilesN; }
  __device__ void next(const TcParams& p) {
    inGroup += step;
    if (inGroup >= units) {
      inGroup -= units;
      ++cycle;
      settle(p);
    }
  }
  // tiles [tnBeg, tnEnd) of tile row tm for CTA `rank` of the pair (0 when unpaired); false = nothing to do
  __device__ bool coords(const TcParams& p, uint32_t rank, uint32_t& tm, uint32_t& tnBeg, uint32_t& tnEnd) const {
    uint32_t row, col;
    if (gRows == G) {
      row = inGroup & (G - 1);  // G is a power of two
      col = inGroup >> gShift;
    } else {  // the last, partial group
      row = inGroup % gRows;
      col = inGroup / gRows;
    }
    tnBeg              = tn0 + col * RUN;
    tnEnd              = RUN == 1 ? tnBeg + 1 : min(limit(p), tnBeg + RUN);  // (a unit of one column lies inside the limit)
    const uint32_t tr  = group * G + row;  // unit row
    const uint32_t top = PAIR ? 2 * tr : tr;
    // the upper tile decides for both CTAs of a pair (if it has no pair with row < col, neither has the lower one); a
    // lower tile past the end or below the diagonal still runs - its loads are zero-filled / its predicates reject all.
    // A tile column is useful iff (tn + 1) * colSpan - 1 > top * rowSpan: monotone in tn, so a run is clipped from the left.
    if (p.symmetric) tnBeg = max(tnBeg, (top * p.rowSpan + 1u) / p.colSpan);
    if (tnBeg >= tnEnd) return false;
    tm = top + (PAIR ? rank : 0u);
    return true;
  }
};

// host twin of the walk's unit count (sizes the grid); band = the host copy of p.bandEnd (nullptr when p has none)
template <bool PAIR, int RUN = 1>
uint64_t countUnits(const TcParams& p, const uint32_t* band) {
  const uint32_t G        = PAIR ? p.groupTiles / 2 : p.groupTiles;
  const uint32_t unitRows = PAIR ? (p.tilesM + 1) / 2 : p.tilesM;
  uint64_t       total    = 0;
  for (uint32_t cycle = 0; static_cast<uint64_t>(cycle) * p.groupStride * G < unitRows; ++cycle) {
    const uint32_t group = cycle * p.groupStride + ((cycle & 1u) ? p.groupStride - 1 - p.groupOffset : p.groupOffset);
    if (static_cast<uint64_t>(group) * G >= unitRows) continue;
    const uint32_t gRows = std::min(G, unitRows - group * G);
    const uint32_t tn0   = p.symmetric ? (group * p.groupTiles * p.rowSpan + 1u) / p.colSpan : 0u;
    const uint32_t tnLim = band ? std::min(p.tilesN, band[group]) : p.tilesN;
    if (tn0 < tnLim) total += static_cast<uint64_t>(gRows) * ((tnLim - tn0 + RUN - 1) / RUN);
  }
  return total;
}

// CL: 0 = one CTA per tile; 1 = a cluster of two CTAs on vertically adjacent tiles that share the column operand (each
// CTA loads half of it and TMA multicasts that half to both), so a pair of tiles reads the column operand from L2 once;
// 3 = the same pair with the ROW operand stationary: a unit is a run of kRunStat tile columns of one tile row, the row
// tile's K chunks are loaded once per unit into their own shared-memory region and only the column operand streams
// through the ring (half the L2 -> shared memory bytes per pair). The next unit's row chunks are requested as soon as
// the last tile of the current unit has retired its MMAs.
template <int MODE, int CL>
__global__ void __launch_bounds__(kThreadsTC, 1)
  simTensorKernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smemRaw[];
  static_assert(!CL || MODE == kTcCount, "the two-CTA cluster is wired for the count tile");
  constexpr bool COUNT = MODE == kTcCount;
  constexpr bool TOPK  = MODE == kTcTopkTanimoto || MODE == kTcTopkCosine || MODE == kTcTopkTversky;
  constexpr bool LIST  = MODE == kTcListCosine || MODE == kTcListTversky;  // edges only, through the same per-warp staging
                                                                         // as the count mode
  constexpr bool ST    = CL == 3;  // row operand stationary
  using Walk           = UnitWalk<CL != 0, ST ? kRunStat : 1>;
  constexpr int  kStg       = ST ? kStagesStat : kStages;
  constexpr int  kStgBytes  = ST ? kBBytes : kStageBytes;       // ring stage: column operand (+ row operand unless stationary)
  constexpr int  kAResident = ST ? kMaxChunksStat * kABytes : 0;  // the stationary row tile, ahead of the ring
  __shared__ uint64_t fullBar[kStages], emptyBar[kStages];
  __shared__ uint64_t aFull[ST ? kMaxChunksStat : 1], aEmpty[ST ? kMaxChunksStat : 1];
  // the tile's row and column metadata (tileMetaKernel), two tiles deep: the producer fetches tile t + 1's while the
  // consumers still read tile t's
  __shared__ uint64_t metaFull[2], metaEmpty[2];
  __shared__ __align__(16) int2 colMeta[2][kTN];
  __shared__ __align__(16) int2 rowMeta[2][kTM];
  __shared__ int2 pairSlots[COUNT || LIST ? 8 : 1][COUNT || LIST ? kStagePairs : 1];  // count / list: each epilogue warp's PairStage
  __shared__ uint32_t walkCount[2];  // units the producer walked, tiles it ran (in shared memory: no register to spare)

  const uint32_t rank      = CL ? clusterCtaRank() : 0u;
  const uint32_t firstUnit = CL ? blockIdx.x / 2 : blockIdx.x, unitStep = CL ? gridDim.x / 2 : gridDim.x;
  const uint32_t smemA     = (smemAddr(smemRaw) + 1023u) & ~1023u;  // (stationary tile: the row operand's K chunks)
  const uint32_t smemBase  = smemA + kAResident;                    // the ring
  uint8_t*       smemGen   = smemRaw + (smemBase - smemAddr(smemRaw));
  const int      warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#ifdef B200_TC_TIMING
  unsigned long long tcClk[8] = {};
#endif

  if (threadIdx.x == 0) {
    walkCount[0] = walkCount[1] = 0;
    tmaPrefetchDesc(&tmA);
    tmaPrefetchDesc(&tmB);
    for (int s = 0; s < kStg; ++s) {
      mbarInit(&fullBar[s], 1);
      mbarInit(&emptyBar[s], CL ? 16 : 8);  // one arrival per consumer warp (of both CTAs when the column operand is shared)
    }
    if constexpr (ST)
      for (int s = 0; s < kMaxChunksStat; ++s) {
        mbarInit(&aFull[s], 1);
        mbarInit(&aEmpty[s], 8);  // the row tile is this CTA's own: its eight consumer warps
      }
    for (int s = 0; s < 2; ++s) {
      mbarInit(&metaFull[s], 1);
      mbarInit(&metaEmpty[s], 8);
    }
    fenceBarrierInit();
  }
  __syncthreads();
  if constexpr (CL) clusterSync();  // the peer's barriers exist before anything is multicast at them

  if (warp < 4) {
    // ===================== TMA producer (one thread) =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int      stage = 0, meta = 0;
      uint32_t phase = 0, aPhase = 0, metaPhase = 0;
      for (Walk w(p, firstUnit, unitStep); !w.done; w.next(p)) {
        uint32_t tm, tnBeg, tnEnd;
        atomicAdd(&walkCount[0], 1u);
        if (!w.coords(p, rank, tm, tnBeg, tnEnd)) continue;
        atomicAdd(&walkCount[1], tnEnd - tnBeg);
        for (uint32_t tn = tnBeg; tn < tnEnd; ++tn) {
          mbarWait(&metaEmpty[meta], metaPhase ^ 1);
          mbarExpectTx(&metaFull[meta], (kTN + kTM) * sizeof(int2));
          bulkLoad1D(colMeta[meta], p.colMeta + static_cast<size_t>(tn) * kTN, kTN * sizeof(int2), &metaFull[meta]);
          bulkLoad1D(rowMeta[meta], p.rowMeta + static_cast<size_t>(tm) * kTM, kTM * sizeof(int2), &metaFull[meta]);
          if (++meta == 2) {
            meta = 0;
            metaPhase ^= 1;
          }
          for (int kc = 0; kc < p.kChunks; ++kc) {
            if constexpr (ST) {
              if (tn == tnBeg) {  // this unit's row tile, chunk kc: once the previous unit's last tile is done with it
                mbarWait(&aEmpty[kc], aPhase ^ 1);
                mbarExpectTx(&aFull[kc], kABytes);
                tmaLoad2D(smemRaw + (smemA - smemAddr(smemRaw)) + kc * kABytes, &tmA, kc * kTK, tm * kTM, &aFull[kc]);
              }
            }
            B200_TC_T0(tw);
            mbarWait(&emptyBar[stage], phase ^ 1);
            B200_TC_T1(tw, 7);
            uint8_t* dst = smemGen + stage * kStgBytes;
            mbarExpectTx(&fullBar[stage], kStgBytes);
            if constexpr (!ST) tmaLoad2D(dst, &tmA, kc * kTK, tm * kTM, &fullBar[stage]);
            uint8_t* dstB = ST ? dst : dst + kABytes;
            if constexpr (CL) {
              // half of the shared column operand each, delivered to both CTAs (their barriers count the bytes)
              constexpr int kHalfRows = kTN / 2;
              tmaLoad2DMulticast(dstB + rank * (kHalfRows * kTK), &tmB, kc * kTK, tn * kTN + rank * kHalfRows,
                                 &fullBar[stage], static_cast<uint16_t>(3));
            } else {
              tmaLoad2D(dstB, &tmB, kc * kTK, tn * kTN, &fullBar[stage]);
            }
            if (++stage == kStg) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
        aPhase ^= 1;
      }
      if (p.walked) {  // (both CTAs of a pair walk the same units: rank 0 counts them)
        if (rank == 0) atomicAdd(p.walked, static_cast<unsigned long long>(walkCount[0]));
        atomicAdd(p.walked + 1, static_cast<unsigned long long>(walkCount[1]));
      }
#ifdef B200_TC_TIMING
      atomicAdd(&g_tcClk[7], tcClk[7]);
#endif
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 1 and 2: rows 0..63 and 64..127 of the tile) =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int      ct = threadIdx.x - 128;  // 0..255
    const int      wg = ct >> 7, q = lane & 3;
    uint32_t       acc[128];
    int            stage = 0;
    uint32_t       phase = 0, local = 0, aPhase = 0;
    PairStage      pairs{0};
    auto release = [&](int s) {  // this warp's MMAs on stage s have retired
      if (lane == 0) {
        mbarArrive(&emptyBar[s]);
        if constexpr (CL) mbarArriveRemote(&emptyBar[s], rank ^ 1u);
      }
    };
    B200_TC_T0(tLoop);
    for (Walk w(p, firstUnit, unitStep); !w.done; w.next(p)) {
      uint32_t tm, tnBeg, tnEnd;
      if (!w.coords(p, rank, tm, tnBeg, tnEnd)) continue;
      for (uint32_t tn = tnBeg; tn < tnEnd; ++tn) {
        int prev = -1;
        for (int kc = 0; kc < p.kChunks; ++kc) {
          B200_TC_T0(tFull);
          if constexpr (ST) {
            if (tn == tnBeg) mbarWait(&aFull[kc], aPhase);
          }
          mbarWait(&fullBar[stage], phase);
          B200_TC_T1(tFull, 1);
          fenceAccumulators(acc);
          wgmmaFence();
          const uint32_t sAddr = smemBase + stage * kStgBytes;
          const uint64_t aDesc = makeSmemDesc((ST ? smemA + kc * kABytes : sAddr) + wg * 64 * kTK);
          const uint64_t bDesc = makeSmemDesc(ST ? sAddr : sAddr + kABytes);
#pragma unroll
          for (int k = 0; k < kTK / 32; ++k) wgmmaU8(acc, aDesc + 2 * k, bDesc + 2 * k, (kc | k) != 0 ? 1u : 0u);
          wgmmaCommit();
          if (prev >= 0) {
            B200_TC_T0(tMma);
            wgmmaWait<1>();  // the previous chunk's MMAs have read their stage
            B200_TC_T1(tMma, 2);
            release(prev);
          }
          prev = stage;
          if (++stage == kStg) {
            stage = 0;
            phase ^= 1;
          }
        }
        {
          B200_TC_T0(tMma);
          wgmmaWait<0>();
          B200_TC_T1(tMma, 2);
        }
        fenceAccumulators(acc);
        release(prev);
        if constexpr (ST) {
          if (tn + 1 == tnEnd && lane == 0)  // the unit's last tile: its row chunks may be replaced
            for (int kc = 0; kc < p.kChunks; ++kc) mbarArrive(&aEmpty[kc]);
        }

        const int meta = local & 1;
        {
          B200_TC_T0(tMeta);
          mbarWait(&metaFull[meta], (local >> 1) & 1);  // (long since landed: requested before the tile's first K chunk)
          B200_TC_T1(tMeta, 0);
        }
        const int      rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows rl, rl + 8 of the tile
        const uint32_t r0 = tm * kTM + rl, r1 = r0 + 8;
        const int2     ra0 = rowMeta[meta][rl], ra1 = rowMeta[meta][rl + 8];
        const int      pa0 = ra0.x, pa1 = ra1.x;
        // colMeta[meta][8 j + 2 q + h] = {popcount, pre-filter term} of column c0 + 8 j + h, as one 16-byte load
        const int4*    cm = reinterpret_cast<const int4*>(&colMeta[meta][2 * q]);
        const uint32_t c0 = tn * kTN + 2 * q;  // column of acc[0]; acc[4 j ..] sit 8 j further
        if constexpr (COUNT) {
          // Pre-filter: a pair (or a superposed group of pairs) can only pass with c >= alpha (|A| + |B|) (the exact
          // threshold is the smallest integer the fp64 predicate accepts, never below alpha S - 1e-12), so with both
          // products in 1/256 units and rounded down (acc <= 65,536: no overflow)
          //   256 acc - floor(256 alpha |B_j|)  >=  floor(256 alpha |A_i|)
          // is necessary. The common case is "no survivor in this thread's 128 accumulators": a max per row decides it.
          B200_TC_T0(tPre);
          const int rowI0 = ra0.y, rowI1 = ra1.y;
          int       m0 = -0x3fffffff, m1 = -0x3fffffff;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int4 ci = cm[4 * j];
            m0            = max(m0, max(256 * static_cast<int>(acc[4 * j]) + ci.y, 256 * static_cast<int>(acc[4 * j + 1]) + ci.w));
            m1            = max(m1, max(256 * static_cast<int>(acc[4 * j + 2]) + ci.y, 256 * static_cast<int>(acc[4 * j + 3]) + ci.w));
          }
          const bool super = p.superS * p.superC > 1;
          int        hits0 = 0, hits1 = 0;
          const bool anySurvivor = __any_sync(0xffffffffu, m0 >= rowI0 || m1 >= rowI1);
          B200_TC_T1(tPre, 3);
          B200_TC_T0(tCand);
          if (anySurvivor && super) {
            // The survivors of the pre-filter as bits 4 (j % 8) + e of sv[j / 8], in one unrolled pass over the
            // accumulators; the candidate list then takes them in a ROLLED loop over the column blocks that hold any.
            // (Unrolled 32 times, the list code made the tile loop hundreds of KB of straight-line code that ran from
            // cold instruction caches on every tile with a survivor.)
            uint32_t sv[4] = {0, 0, 0, 0}, blocks = 0;  // blocks: bit j = a survivor in column block j
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int4 ci  = ldsFresh(cm + 4 * j);
              uint32_t   nib = 0;
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (256 * static_cast<int>(acc[4 * j + e]) + ((e & 1) ? ci.w : ci.y) >= (e < 2 ? rowI0 : rowI1)) nib |= 1u << e;
              sv[j >> 3] |= nib << (4 * (j & 7));
              if (nib) blocks |= 1u << j;
            }
            // the column blocks where any lane of the warp has a survivor, one at a time
            for (uint32_t todo = __reduce_or_sync(0xffffffffu, blocks); todo; todo &= todo - 1) {
              const int      j   = __ffs(todo) - 1;
              const uint32_t nib = ((j < 8 ? sv[0] : j < 16 ? sv[1] : j < 24 ? sv[2] : sv[3]) >> (4 * (j & 7))) & 0xFu;
              uint32_t       bits = 0;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint32_t r = e < 2 ? r0 : r1, c = c0 + 8 * j + (e & 1);
                // the exact verification kernel re-examines the group: a pair i < j must exist
                if ((nib >> e) & 1u && r < p.n && c < p.nY &&
                    (!p.symmetric || r * static_cast<uint32_t>(p.superS) + 1u < (c + 1u) * static_cast<uint32_t>(p.superC)))
                  bits |= 1u << e;
              }
              if (__any_sync(0xffffffffu, bits != 0)) pairs.add(p, pairSlots[warp - 4], bits, r0, r1, c0 + 8 * j, lane);
            }
          } else if (anySurvivor) {  // unsuperposed: the exact test, neighbour counts for both endpoints and the edges
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              uint32_t   bits = 0;
              const int4 ci   = ldsFresh(cm + 4 * j);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint32_t r = e < 2 ? r0 : r1, c = c0 + 8 * j + (e & 1);
                const int      a = static_cast<int>(acc[4 * j + e]);
                if (256 * a + ((e & 1) ? ci.w : ci.y) < (e < 2 ? rowI0 : rowI1) || r >= p.n || c >= p.nY) continue;
                if ((!p.symmetric || r < c) && a >= p.thresh[(e < 2 ? pa0 : pa1) + ((e & 1) ? ci.z : ci.x)]) bits |= 1u << e;
              }
              if (!__any_sync(0xffffffffu, bits != 0)) continue;
              hits0 += __popc(bits & 3u);
              hits1 += __popc(bits >> 2);
              if (p.countsY)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  if ((bits >> e) & 1u) atomicAdd(p.countsY + c0 + 8 * j + (e & 1), p.sign);
              if (p.edges) pairs.add(p, pairSlots[warp - 4], bits, r0, r1, c0 + 8 * j, lane);
            }
          }
          if (hits0) atomicAdd(p.counts + r0, p.sign * hits0);
          if (hits1) atomicAdd(p.counts + r1, p.sign * hits1);
          B200_TC_T1(tCand, 4);
        } else if constexpr (TOPK) {
          // Top-k filter: can the pair beat the row's bar, the key of its current k-th best? Conservative - the select
          // kernel (topk.cu) re-counts every survivor and orders them exactly - but tight, so that survivors stay rare.
          // The bar's column lies before the slab (the list holds earlier columns only), so a tie never wins.
          // Tanimoto, in integers: c / (s - c) > cB / (sB - cB)  <=>  c sB > cB s  (s = |A| + |B|; both sides < 2^26).
          // Equal ratios round to equal fp64 values and distinct ratios with denominators <= 8192 differ by more than
          // 2^-26, far above an ulp, so this integer order is the order of the fp64 values the select kernel compares.
          // Cosine, c / sqrt(|A| |B|), has no integer form: float(c) >= tauLow sqrt|A| sqrt|B| with tauLow a few 1e-5
          // (relative) below the bar, which covers the float roundings; ties and near ties survive.
          // Tversky depends on c, |A| and |B| apart: tverskyMayReach (similarity.cuh) with the same float bar. For fixed
          // |A| and |B| the value c / (K + (1 - alpha - beta) c), K = alpha |A| + beta |B|, has derivative K / D^2 >= 0 in c,
          // so the exact select kernel orders by value alone, as for cosine.
          constexpr bool COS = MODE == kTcTopkCosine;
          constexpr bool TV  = MODE == kTcTopkTversky;
          const bool in0 = r0 < p.n, in1 = r1 < p.n;
          // per row: margin(c, column) = c f - g term(column) must exceed t. Past the end nothing does.
          int   f0 = 0, g0 = 0, t0 = 0x7fffffff, f1 = 0, g1 = 0, t1 = 0x7fffffff;
          float rt0 = 3.0e38f, rt1 = 3.0e38f;
          if (in0) {
            const int4 b = __ldg(p.topkBar + r0);
            f0 = b.y, g0 = b.x, t0 = b.x * pa0;
            rt0 = TV ? __int_as_float(b.w) : __int_as_float(b.w) * sqrtf(static_cast<float>(pa0));
          }
          if (in1) {
            const int4 b = __ldg(p.topkBar + r1);
            f1 = b.y, g1 = b.x, t1 = b.x * pa1;
            rt1 = TV ? __int_as_float(b.w) : __int_as_float(b.w) * sqrtf(static_cast<float>(pa1));
          }
          // does accumulator e of a column block (popcount pb, sqrt(pb) as float bits sq) pass? (cosine: the count through
          // the 2^23 trick, exact and no I2F)
          auto pass = [&](int e, int a, int pb, int sq) {
            if constexpr (COS) return fmaf(-(e < 2 ? rt0 : rt1), __int_as_float(sq), __int_as_float(0x4b000000 | a) - 8388608.0f) >= 0.0f;
            else if constexpr (TV) return tverskyMayReach(fresh(a), e < 2 ? pa0 : pa1, pb, p.tvAlphaF, p.tvBetaF, e < 2 ? rt0 : rt1);
            else return a * (e < 2 ? f0 : f1) - (e < 2 ? g0 : g1) * pb > (e < 2 ? t0 : t1);
          };
          bool any = false;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int4 ci = cm[4 * j];
            any |= pass(0, static_cast<int>(acc[4 * j]), ci.x, ci.y) | pass(1, static_cast<int>(acc[4 * j + 1]), ci.z, ci.w) |
                   pass(2, static_cast<int>(acc[4 * j + 2]), ci.x, ci.y) | pass(3, static_cast<int>(acc[4 * j + 3]), ci.z, ci.w);
          }
          if (__any_sync(0xffffffffu, any)) {
            // survivors as bits 4 (j % 8) + e of sv[j / 8] in one unrolled pass; each lane then lists its own in a rolled loop
            uint32_t sv[4] = {0, 0, 0, 0};
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int4 ci  = ldsFresh(cm + 4 * j);
              uint32_t   nib = 0;
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (pass(e, static_cast<int>(acc[4 * j + e]), (e & 1) ? ci.z : ci.x, (e & 1) ? ci.w : ci.y) && (e < 2 ? in0 : in1) &&
                    c0 + 8 * j + (e & 1) < p.nY)
                  nib |= 1u << e;
              sv[j >> 3] |= nib << (4 * (j & 7));
            }
#pragma unroll
            for (int w = 0; w < 4; ++w)
              for (uint32_t bits = sv[w]; bits; bits &= bits - 1) {
                const int      b = __ffs(bits) - 1, e = b & 3;
                const uint32_t r = e < 2 ? r0 : r1, c = c0 + 8 * (8 * w + (b >> 2)) + (e & 1);
                const uint32_t at = atomicAdd(p.topkCount + r, 1u);
                if (at < p.topkCap) p.topkCand[static_cast<size_t>(r) * p.topkCap + at] = p.topkColBase + c;
              }
          }
        } else if constexpr (LIST) {
          // Cosine listing (threshold search, threshold.cu): can c / sqrt(|A| |B|) reach t? Tested as
          // float(c) >= tLow sqrt|A| sqrt|B| with tLow 1e-5 (relative) below t, far more than the few 2^-24 the float
          // square roots and products can err by, so every pair whose fp64 value is >= t is listed; the assembly re-counts
          // each listed pair and drops the near misses. rowMeta .y = float bits of tLow sqrt|A|, colMeta .y = those of
          // sqrt|B| (3e38 past the end). An empty intersection never reaches t > 0.
          // Tversky: tverskyMayReach (similarity.cuh) against p.tvBound = t (1 - 1e-5) rounded down; .x the popcounts.
          const float rt0 = __int_as_float(ra0.y), rt1 = __int_as_float(ra1.y);
          auto pass = [&](int e, int a, int4 ci) {  // (cosine: the count through the 2^23 trick, exact and no I2F)
            if constexpr (MODE == kTcListTversky)
              return tverskyMayReach(fresh(a), e < 2 ? pa0 : pa1, (e & 1) ? ci.z : ci.x, p.tvAlphaF, p.tvBetaF, p.tvBound);
            else
              return a != 0 && fmaf(-(e < 2 ? rt0 : rt1), __int_as_float((e & 1) ? ci.w : ci.y), __int_as_float(0x4b000000 | a) - 8388608.0f) >= 0.0f;
          };
          bool any = false;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int4 ci = cm[4 * j];
            any |= pass(0, static_cast<int>(acc[4 * j]), ci) | pass(1, static_cast<int>(acc[4 * j + 1]), ci) |
                   pass(2, static_cast<int>(acc[4 * j + 2]), ci) | pass(3, static_cast<int>(acc[4 * j + 3]), ci);
          }
          if (__any_sync(0xffffffffu, any)) {
            // survivors as bits 4 (j % 8) + e of sv[j / 8] in one unrolled pass, listed in a rolled loop over the column
            // blocks that hold any (as the superposed count epilogue does)
            uint32_t sv[4] = {0, 0, 0, 0}, blocks = 0;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int4 ci  = ldsFresh(cm + 4 * j);
              uint32_t   nib = 0;
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (pass(e, static_cast<int>(acc[4 * j + e]), ci)) nib |= 1u << e;
              sv[j >> 3] |= nib << (4 * (j & 7));
              if (nib) blocks |= 1u << j;
            }
            for (uint32_t todo = __reduce_or_sync(0xffffffffu, blocks); todo; todo &= todo - 1) {
              const int      j   = __ffs(todo) - 1;
              const uint32_t nib = ((j < 8 ? sv[0] : j < 16 ? sv[1] : j < 24 ? sv[2] : sv[3]) >> (4 * (j & 7))) & 0xFu;
              uint32_t       bits = 0;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const uint32_t r = e < 2 ? r0 : r1, c = c0 + 8 * j + (e & 1);
                if ((nib >> e) & 1u && r < p.n && c < p.nY && (!p.symmetric || r < c)) bits |= 1u << e;
              }
              if (__any_sync(0xffffffffu, bits != 0)) pairs.add(p, pairSlots[warp - 4], bits, r0, r1, c0 + 8 * j, lane);
            }
          }
        } else {
          // fp64 Tanimoto / cosine / Dice / Tversky straight from the accumulators: a quad of lanes writes 64 contiguous
          // bytes of a row
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const uint32_t c = c0 + 8 * j;
            double         v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int cnt = static_cast<int>(acc[4 * j + e]);
              const int pak = e < 2 ? pa0 : pa1, pb = (e & 1) ? cm[4 * j].z : cm[4 * j].x;
              v[e]          = 0.0;
              if (cnt != 0) {
                if constexpr (MODE == kTcTanimoto) {
                  // c / u through one reciprocal + one Newton step: equal to the correctly rounded quotient for every
                  // 1 <= c <= u <= 8192, which oracle_recip_quotient_mismatches (oracle/oracle_fp.c) checks pair by
                  // pair in test_reciprocal_newton_quotient_is_correctly_rounded; int -> double through the 2^52
                  // trick, RN(1/u) from the table
                  const int    u  = pak + pb - cnt;
                  const double dc = __hiloint2double(0x43300000, cnt) - 4503599627370496.0;
                  const double du = __hiloint2double(0x43300000, u) - 4503599627370496.0;
                  const double rc = __ldg(p.recipG + u), q0 = __dmul_rn(dc, rc);
                  v[e]            = __fma_rn(__fma_rn(-q0, du, dc), rc, q0);
                } else if constexpr (MODE == kTcDice) {
                  // 2c / (a + b) = 2 RN(c / u), u = a + b: the same correctly rounded quotient (c <= u / 2 <= 4096), then
                  // an exact doubling; equal to tverskyFromCounts(c, a, b; 1/2, 1/2), whose intermediates are exact
                  const int    u  = pak + pb;
                  const double dc = __hiloint2double(0x43300000, cnt) - 4503599627370496.0;
                  const double du = __hiloint2double(0x43300000, u) - 4503599627370496.0;
                  const double rc = __ldg(p.recipG + u), q0 = __dmul_rn(dc, rc);
                  v[e]            = 2.0 * __fma_rn(__fma_rn(-q0, du, dc), rc, q0);
                } else if constexpr (MODE == kTcTversky) {
                  v[e] = tverskyFromCounts(cnt, pak, pb, p.tvAlpha, p.tvBeta);
                } else {
                  v[e] = __ddiv_rn(static_cast<double>(cnt), __dsqrt_rn(__dmul_rn(static_cast<double>(pak), static_cast<double>(pb))));
                }
              }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t r = h ? r1 : r0;
              if (r >= p.n || c >= p.nY) continue;
              double* o = p.out + static_cast<size_t>(r) * p.nY + c;
              if (p.outVec) __stcs(reinterpret_cast<double2*>(o), make_double2(v[2 * h], v[2 * h + 1]));
              else {
                __stcs(o, v[2 * h]);
                if (c + 1 < p.nY) __stcs(o + 1, v[2 * h + 1]);
              }
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbarArrive(&metaEmpty[meta]);
        ++local;
#ifdef B200_TC_TIMING
        tcClk[5] += 1;
#endif
      }
      aPhase ^= 1;
    }
    if constexpr (COUNT || LIST) {
      B200_TC_T0(tFlush);
      pairs.flush(p, pairSlots[warp - 4], lane);  // (n stays 0 when the pass lists nothing)
      B200_TC_T1(tFlush, 4);
    }
#ifdef B200_TC_TIMING
    B200_TC_T1(tLoop, 6);
    if (lane == 0)
      for (int k = 0; k < 7; ++k) atomicAdd(&g_tcClk[k], tcClk[k]);
#endif
  }
  __syncthreads();
  if constexpr (CL) clusterSync();  // no CTA leaves while its peer may still signal its barriers
}

using TcKernel = void (*)(CUtensorMap, CUtensorMap, TcParams);
// The tensor tile's kernel for each operation (SimMode) and measure kind (MeasureKind); nullptr: the SIMT tile serves it.
// Dice runs on the Tanimoto machinery: its matrix from the reciprocal table, its count on Tanimoto's count tile with its
// own threshold table and pre-filter. The count tile's cluster variants are picked in CountSets::pass.
const TcKernel kTensorKernels[3][4] = {
  // Tanimoto                      cosine                           Dice                          Tversky
  {simTensorKernel<kTcTanimoto, 0>, simTensorKernel<kTcCosine, 0>, simTensorKernel<kTcDice, 0>, simTensorKernel<kTcTversky, 0>},
  {simTensorKernel<kTcCount, 0>, nullptr, simTensorKernel<kTcCount, 0>, nullptr},
  {nullptr, simTensorKernel<kTcListCosine, 0>, nullptr, simTensorKernel<kTcListTversky, 0>},
};
// ... and of the top-k search's tile pass (a Dice search is Tanimoto's: topk.cu)
const TcKernel kTopkKernels[4] = {simTensorKernel<kTcTopkTanimoto, 0>, simTensorKernel<kTcTopkCosine, 0>, nullptr,
                                  simTensorKernel<kTcTopkTversky, 0>};
constexpr size_t kSmemBytesTC = static_cast<size_t>(kStages) * kStageBytes + 1024;

// Every kernel above opts in to the shared memory it runs with, once per device.
void optInTensorKernels() {
  static bool configured[kMaxDevices] = {};
  if (configured[currentDeviceSlot()]) return;
  auto optIn = [](TcKernel kernel) {
    if (kernel) B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBytesTC)));
  };
  for (const auto& row : kTensorKernels)
    for (TcKernel kernel : row) optIn(kernel);
  for (TcKernel kernel : kTopkKernels) optIn(kernel);
  optIn(simTensorKernel<kTcCount, 1>);
  optIn(simTensorKernel<kTcCount, 3>);
  configured[currentDeviceSlot()] = true;
}

}  // namespace

void launchRowPopcount(const uint32_t* fp, size_t n, int words, int32_t* pop, cudaStream_t s);
void launchThreshTable(int maxS, const Measure& m, double cutoff, bool atLeast, uint16_t* thresh, cudaStream_t s);

// A fingerprint set in popcount order: row i of fp is the caller's row perm[i], pop its popcount; ascending, ties in the
// caller's order (CUB's radix sort is stable), so the same input always gives the same order.
struct PopOrder {
  Scratch<uint32_t> fp;
  Scratch<int32_t>  pop, perm;
};
static PopOrder popcountOrder(const uint32_t* fp, const int32_t* pop, size_t n, int words, cudaStream_t s) {
  PopOrder o;
  o.fp   = Scratch<uint32_t>(n * static_cast<size_t>(words), s);
  o.pop  = Scratch<int32_t>(n, s);
  o.perm = Scratch<int32_t>(n, s);
  Scratch<int32_t> index(n, s);
  iotaKernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(index.get(), n);
  B200_LAUNCHED();
  int endBit = 1;  // popcounts are <= 32 words, non-negative: the low bits of the key are enough
  while ((1 << endBit) <= 32 * words) ++endBit;
  size_t tmpBytes = 0;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, pop, o.pop.get(), index.get(), o.perm.get(), static_cast<int>(n), 0,
                                            endBit, s));
  Scratch<uint8_t> tmp(tmpBytes, s);
  B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tmpBytes, pop, o.pop.get(), index.get(), o.perm.get(), static_cast<int>(n), 0,
                                            endBit, s));
  g_launchCount.fetch_add(1);
  const int    chunks = words / 4;
  const size_t t      = n * static_cast<size_t>(chunks);
  gatherRowsKernel<<<static_cast<unsigned>((t + 255) / 256), 256, 0, s>>>(reinterpret_cast<const uint4*>(fp), o.perm.get(), n, chunks,
                                                                          reinterpret_cast<uint4*>(o.fp.get()));
  B200_LAUNCHED();
  return o;
}

int g_superpose = 4;      // fingerprints summed into one row of the count pass (option "similarity_superpose": 1, 2 or 4)
int g_superposeCols = 4;  // ... and into one column ("similarity_superpose_cols": 1, 2 or 4); 4 x 4 sums stay <= 16, exact
int g_superposeLast = 0;  // pairs per accumulator the last graph pass really ran with (1 after an overflow fallback)

constexpr int kMaxPipeline = 8;
int g_pipelineChunks = 4;  // chunks of a superposed pass whose verification overlaps the next chunk's tensor pass
                           // (option "similarity_pipeline_chunks"; 1 = off)
int g_superposeAuto = 1;  // 1: a large graph pass picks rows x cols from a pilot over one row group ("similarity_superpose_auto")
unsigned long long g_candidatesLast = 0;  // candidates the last superposed pass listed ("similarity_candidates_last")
int g_popcountBand = 1;  // ordered passes skip the tile columns past each row group's popcount band ("similarity_popcount_band")
// What the count passes of the last graph call (after its pilot) walked: units the host sized the grids for, and what
// the kernels counted ("similarity_units_planned_last", "similarity_units_last", "similarity_tiles_last").
unsigned long long g_unitsPlanned = 0;
namespace {
__device__ unsigned long long g_walkedDev[2];  // [0] units, [1] tiles (TcParams::walked)
}
static void resetWalkCounters(cudaStream_t s) {
  g_unitsPlanned = 0;
  resetDeviceCounters(g_walkedDev, s);
}
unsigned long long readWalkCounter(int i) { return readDeviceCounter(g_walkedDev, i); }

// Pairs i < j (symmetric) or (i, j) of a pass over all row groups that the popcount band leaves (band = nullptr: all).
static double bandPairs(const TcParams& p, const uint32_t* band, size_t nX, size_t nY) {
  double total = 0.0;
  for (size_t r0 = 0, g = 0; r0 < nX; r0 += kGroupRows, ++g) {
    const size_t r1 = std::min(nX, r0 + kGroupRows);
    const size_t e  = band ? std::min(nY, static_cast<size_t>(band[g]) * p.colSpan) : nY;  // columns [0, e) are visited
    if (!p.symmetric) {
      total += static_cast<double>(r1 - r0) * static_cast<double>(e);
      continue;
    }
    const size_t iEnd = std::min(r1, e > 0 ? e - 1 : 0);  // rows i with a column i < j < e
    if (iEnd <= r0) continue;
    const double m = static_cast<double>(iEnd - r0);
    total += m * static_cast<double>(e - 1) - (static_cast<double>(r0) + static_cast<double>(iEnd) - 1.0) * m / 2.0;
  }
  return total;
}

// The geometry of a tile pass over n x nY fingerprints, S (C) of them summed into one row of the X (Y) operand, over
// every row group
static TcParams tileGeometry(size_t n, size_t nY, int words, int S, int C) {
  const size_t nSuper = (n + S - 1) / S, nSuperY = (nY + C - 1) / C;
  TcParams     p{};
  p.n           = static_cast<uint32_t>(nSuper);
  p.nY          = static_cast<uint32_t>(nSuperY);
  p.kChunks     = words * 32 / kTK;
  p.tilesM      = static_cast<uint32_t>((nSuper + kTM - 1) / kTM);
  p.tilesN      = static_cast<uint32_t>((nSuperY + kTN - 1) / kTN);
  p.superS      = S;
  p.superC      = C;
  p.rowSpan     = static_cast<uint32_t>(kTM * S);
  p.colSpan     = static_cast<uint32_t>(kTN * C);
  p.groupTiles  = static_cast<uint32_t>(kGroupRows / (kTM * S));
  p.groupStride = 1;
  return p;
}

// ... and what the call asks of the pass: its row groups, outputs, measure and pre-filter
static TcParams passParams(const SimLaunch& q, int S, int C) {
  TcParams p    = tileGeometry(q.nX, q.nY, q.words, S, C);
  p.symmetric   = q.symmetric ? 1 : 0;
  p.groupOffset = q.groupOffset;
  p.groupStride = q.groupStride < 1 ? 1 : q.groupStride;
  p.sign        = q.sign;
  p.counts      = q.rowCounts;
  p.countsY     = q.symmetric ? q.rowCounts : nullptr;
  p.edges       = q.edges;
  p.edgeCursor  = q.edgeCursor;
  p.edgeCap     = q.edgeCap;
  p.out         = q.out;
  p.outVec      = (q.nY % 2 == 0 && (reinterpret_cast<uintptr_t>(q.out) & 15) == 0) ? 1 : 0;
  {
    // a pair passes iff 1 - c / (|A| + |B| - c) <= cutoff, i.e. c >= alpha (|A| + |B|) - or, for the threshold search's
    // c / (|A| + |B| - c) >= t, with alpha = t / (1 + t); the pre-filter's alpha is rounded DOWN (and its products
    // too), so it never rejects what the exact fp64 table accepts. Dice's 2c / (|A| + |B|) >= t needs c >= (t / 2) (|A| + |B|).
    const double a  = q.atLeast ? (q.measure.kind == kDice ? q.cutoff / 2.0 : q.cutoff / (1.0 + q.cutoff))
                                : q.cutoff < 2.0 ? (1.0 - q.cutoff) / (2.0 - q.cutoff) : 0.0;
    float        af = static_cast<float>(a);
    if (static_cast<double>(af) > a) af = nextafterf(af, -1.0f);
    p.alpha = nextafterf(af, -1.0f);  // (one more ulp: fp64 rounding inside the table's predicate)
    if (p.alpha < 0.0f) p.alpha = 0.0f;
  }
  p.tvAlpha = q.measure.alpha, p.tvBeta = q.measure.beta;
  p.tvAlphaF = static_cast<float>(q.measure.alpha), p.tvBetaF = static_cast<float>(q.measure.beta);
  return p;
}

// One persistent launch over `units` units (tiles, or vertical tile pairs for the clusters of two CTAs that share the
// column operand): at most one CTA (pair) per SM (pair)
static void launchPersistent(TcKernel kernel, bool cluster, const CUtensorMap& tmA, const CUtensorMap& tmB, const TcParams& p,
                             uint64_t units, cudaStream_t s) {
  optInTensorKernels();
  if (cluster) {
    cudaLaunchConfig_t  cfg{};
    cudaLaunchAttribute attr[1];
    attr[0].id               = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.blockDim             = dim3(kThreadsTC);
    cfg.dynamicSmemBytes     = kSmemBytesTC;
    cfg.stream               = s;
    cfg.attrs                = attr;
    cfg.numAttrs             = 1;
    cfg.gridDim              = dim3(2);
    int maxClusters          = 0;
    B200_CUDA(cudaOccupancyMaxActiveClusters(&maxClusters, kernel, &cfg));
    B200_REQUIRE(maxClusters >= 1, "no CTA pair fits the device");
    uint64_t pairs = maxClusters;  // persistent: one resident cluster per schedulable SM pair
    if (pairs > units) pairs = units;
    cfg.gridDim = dim3(static_cast<unsigned>(2 * pairs));
    B200_CUDA(cudaLaunchKernelEx(&cfg, kernel, tmA, tmB, p));
  } else {
    const int grid = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(smCount()), units));
    kernel<<<grid, kThreadsTC, kSmemBytesTC, s>>>(tmA, tmB, p);
  }
  B200_LAUNCHED();
}

// The 0/1 expansion of both operands (one byte per bit, 2 KB per 2048-bit row); a row of a superposed operand is the sum
// of S (C) consecutive expansions. X and Y share one buffer when they are the same set, summed alike.
struct Operands {
  Scratch<uint8_t> x, yOwn;
  const uint8_t*   y = nullptr;
};
static Operands expandOperands(const uint32_t* fx, size_t nX, int S, const uint32_t* fy, size_t nY, int C, int words, bool same,
                               cudaStream_t s) {
  auto expand = [&](const uint32_t* src, size_t rows, int k, Scratch<uint8_t>& dst) {
    const size_t superRows = (rows + k - 1) / k, nw = superRows * static_cast<size_t>(words);
    dst                    = Scratch<uint8_t>(superRows * static_cast<size_t>(words) * 32, s);
    const auto grid        = static_cast<unsigned>((nw + 255) / 256);
    if (k > 1) expandBitsSuperKernel<<<grid, 256, 0, s>>>(src, rows, words, k, superRows, reinterpret_cast<uint4*>(dst.get()));
    else expandBitsKernel<<<grid, 256, 0, s>>>(src, nw, reinterpret_cast<uint4*>(dst.get()));
    B200_LAUNCHED();
  };
  const bool ownY = !same || S != C;
  Operands   o;
  expand(fx, nX, S, o.x);
  if (ownY) expand(fy, nY, C, o.yOwn);
  o.y = ownY ? o.yOwn.get() : o.x.get();
  return o;
}

// Materialise and list: one unsuperposed pass in the caller's order.
static void launchTileOp(SimMode op, const SimLaunch& q, cudaStream_t s) {
  const MeasureKind kind = q.measure.kind;
  const bool        same = q.x == q.y && q.nX == q.nY;
  TcParams          p    = passParams(q, 1, 1);
  const int         recipLen = 2 * q.words * 32;
  const bool        useRecip = op == kMaterialise && (kind == kTanimoto || kind == kDice);
  Scratch<double>   recip(useRecip ? static_cast<size_t>(recipLen) + 1 : 0, s);
  if (useRecip) {
    recipTableKernel<<<(recipLen + 256) / 256, 256, 0, s>>>(recip.get(), recipLen);
    B200_LAUNCHED();
    p.recipG = recip.get();
  }
  Scratch<int32_t> popX(q.nX, s), popYown(same ? 0 : q.nY, s);
  launchRowPopcount(q.x, q.nX, q.words, popX.get(), s);
  if (!same) launchRowPopcount(q.y, q.nY, q.words, popYown.get(), s);
  const int32_t* popY = same ? popX.get() : popYown.get();
  const Operands e    = expandOperands(q.x, q.nX, 1, q.y, q.nY, 1, q.words, same, s);
  // the epilogue's per-row metadata of both operands, padded to whole tiles for the producer's bulk copies
  const size_t  rowsPad = (static_cast<size_t>(p.tilesM) + 1) * kTM, colsPad = static_cast<size_t>(p.tilesN) * kTN;
  Scratch<int2> rowMeta(rowsPad, s), colMeta(colsPad, s);
  if (op == kList) {
    // the list tile's bound: tLow = t (1 - 1e-5), rounded down
    float tLow = static_cast<float>(q.cutoff * (1.0 - 1e-5));
    if (static_cast<double>(tLow) > q.cutoff * (1.0 - 1e-5)) tLow = nextafterf(tLow, 0.0f);
    p.tvBound = tLow;
    listMetaKernel<<<static_cast<unsigned>((rowsPad + 255) / 256), 256, 0, s>>>(popX.get(), q.nX, rowsPad, tLow, rowMeta.get());
    B200_LAUNCHED();
    listMetaKernel<<<static_cast<unsigned>((colsPad + 255) / 256), 256, 0, s>>>(popY, q.nY, colsPad, 1.0f, colMeta.get());
    B200_LAUNCHED();
  } else {
    tileMetaKernel<<<static_cast<unsigned>((rowsPad + 255) / 256), 256, 0, s>>>(popX.get(), q.nX, 1, q.nX, rowsPad, p.alpha, 1,
                                                                               rowMeta.get());
    B200_LAUNCHED();
    tileMetaKernel<<<static_cast<unsigned>((colsPad + 255) / 256), 256, 0, s>>>(popY, q.nY, 1, q.nY, colsPad, p.alpha, -1,
                                                                               colMeta.get());
    B200_LAUNCHED();
  }
  p.rowMeta = rowMeta.get();
  p.colMeta = colMeta.get();
  CUtensorMap tmA, tmB;
  makeTensorMap2D(&tmA, e.x.get(), q.nX, q.words * 32, kTM, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  makeTensorMap2D(&tmB, e.y, q.nY, q.words * 32, kTN, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  const uint64_t units = countUnits<false>(p, nullptr);
  if (units == 0) return;  // nothing owned by this rank (more ranks than row groups)
  PhaseTimer t(op == kList ? "threshold_list_tc" : "cross_tc", s);
  launchPersistent(kTensorKernels[op][kind], false, tmA, tmB, p, units, s);
}

// ---- the count operation: the thresholded count and the graph passes (Butina's neighbour pass, the threshold search,
// Leader's bulk pass) ----

// Row groups a pass covers: offset, offset + stride, ... (multi-GPU ranks, pipeline chunks)
struct RowGroups {
  uint32_t offset, stride;
  RowGroups chunk(int k, int K) const { return {offset + static_cast<uint32_t>(k) * stride, static_cast<uint32_t>(K) * stride}; }
};

// What one count pass did. Nothing is counted by a pass whose list overflowed: its row groups must be run again.
struct PassResult {
  unsigned long long listed      = 0;      // candidates the superposed pass listed
  bool               overflowed  = false;  // ... more than its list holds
  double             bandedPairs = 0.0;    // pilot passes: the pairs the pass covered, within its band if it walked one
};

// The fingerprints a count call's passes run on and what every pass shares, set up once per call: the caller's order,
// or (ordered) both sets in popcount order with permX / permY mapping a row back to the caller's index.
struct CountSets {
  SimLaunch       q;  // the call, or the pilot's sample of it
  cudaStream_t    s;
  const uint32_t *x, *y;
  const int32_t * popX, *popY, *permX, *permY;
  const uint16_t* thresh;  // [2 bits + 1]
  bool            same;    // X and Y are one set
  bool            ordered;

  // One pass at S x C over `groups`: superposed (a pipeline of chunks from 4 K row groups up, see below) or not. A pilot
  // pass lists candidates and counts nothing (unless unsuperposed), and adds nothing to the call's diagnostics.
  PassResult pass(RowGroups groups, int S, int C, bool pilot) const;

  // Passes over `groups` from S x C down, rows only (S x 1) and then unsuperposed, until one completes; returns the S C
  // of the pass that completed. A pass that overflowed counted nothing, so the next one starts afresh on the same groups.
  int ladder(RowGroups groups, int S, int C) const {
    while (S * C > 1) {
      if (!pass(groups, S, C, false).overflowed) return S * C;
      if (C > 1) C = 1;  // second chance: rows only
      else S = 1;
    }
    pass(groups, 1, 1, false);
    return 1;
  }
};

PassResult CountSets::pass(RowGroups groups, int S, int C, bool pilot) const {
  const bool super = S * C > 1;
  TcParams   p     = passParams(q, S, C);
  p.groupOffset = groups.offset, p.groupStride = groups.stride;
  // An unsuperposed pass in popcount order counts and lists edges in that order; mapBackKernel moves its results to the
  // caller's indices.
  const bool                  mapBack = ordered && !super;
  Scratch<int32_t>            countsOrd(mapBack ? q.nX : 0, s);
  Scratch<unsigned long long> edgeStart(mapBack && q.edges ? 1 : 0, s);
  if (mapBack) {
    B200_CUDA(cudaMemsetAsync(countsOrd.get(), 0, q.nX * sizeof(int32_t), s));
    p.counts  = countsOrd.get();
    p.countsY = q.symmetric ? countsOrd.get() : nullptr;
    if (q.edges) B200_CUDA(cudaMemcpyAsync(edgeStart.get(), q.edgeCursor, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
  }
  const Operands e = expandOperands(x, q.nX, S, y, q.nY, C, q.words, same, s);
  // the epilogue's per-row metadata of both operands, padded to whole tiles for the producer's bulk copies (the lower
  // tile of a CTA pair may lie one tile row past the end)
  const size_t  rowsPad = (static_cast<size_t>(p.tilesM) + 1) * kTM, colsPad = static_cast<size_t>(p.tilesN) * kTN;
  Scratch<int2> rowMeta(rowsPad, s), colMeta(colsPad, s);
  tileMetaKernel<<<static_cast<unsigned>((rowsPad + 255) / 256), 256, 0, s>>>(popX, q.nX, S, p.n, rowsPad, p.alpha, 1, rowMeta.get());
  B200_LAUNCHED();
  tileMetaKernel<<<static_cast<unsigned>((colsPad + 255) / 256), 256, 0, s>>>(popY, q.nY, C, p.nY, colsPad, p.alpha, -1, colMeta.get());
  B200_LAUNCHED();
  p.rowMeta = rowMeta.get();
  p.colMeta = colMeta.get();
  // candidates of a superposed pass: (super row, super column) pairs the exact kernel re-examines. Sized for the
  // neighbour graphs this pass is used on (tens of edges per point); a denser graph overflows it and the caller falls back.
  unsigned long long          candCap = 0;
  Scratch<int2>               cand;
  Scratch<unsigned long long> candCursor;
  if (super) {
    const unsigned long long all = static_cast<unsigned long long>(p.n) * p.nY;
    candCap                      = std::min<unsigned long long>(all, std::max<unsigned long long>(1ull << 22, 64ull * q.nX));
    cand                         = Scratch<int2>(candCap, s);
    candCursor                   = Scratch<unsigned long long>(kMaxPipeline, s);
    B200_CUDA(cudaMemsetAsync(candCursor.get(), 0, kMaxPipeline * sizeof(unsigned long long), s));
    p.cand = cand.get(), p.candCursor = candCursor.get(), p.candCap = candCap;
  }
  const int maxS = 2 * q.words * 32;
  p.thresh       = thresh;
  p.threshLen    = maxS + 1;
  // The popcount band of an ordered pass, with a host copy for the unit count that sizes the grid: one read of a few
  // hundred bytes per pass.
  const uint32_t        nGroups = static_cast<uint32_t>((q.nX + kGroupRows - 1) / kGroupRows);
  const bool            banded  = ordered && g_popcountBand;
  Scratch<uint32_t>     band(banded ? nGroups : 0, s);
  std::vector<uint32_t> bandHost(banded ? nGroups : 0);
  if (banded) {
    popcountBandKernel<<<1, kBandThreads, (maxS + 1) * sizeof(uint16_t), s>>>(popX, q.nX, popY, q.nY, thresh, maxS + 1, p.colSpan,
                                                                              p.tilesN, nGroups, band.get());
    B200_LAUNCHED();
    B200_CUDA(cudaMemcpyAsync(bandHost.data(), band.get(), nGroups * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    p.bandEnd = band.get();
  }
  const uint32_t* bandH = banded ? bandHost.data() : nullptr;
  p.walked              = deviceCounters(g_walkedDev);

  CUtensorMap tmA, tmB;
  makeTensorMap2D(&tmA, e.x.get(), p.n, q.words * 32, kTM, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  // CTA pairs sharing the column operand (TMA multicast); 3 = the same with the row operand stationary, for fingerprints
  // whose 128-row tile fits its shared-memory region (else the plain pair runs)
  const bool cluster    = g_tensorCluster != 0;
  const bool stationary = cluster && g_tensorCluster == 3 && p.kChunks <= kMaxChunksStat;
  makeTensorMap2D(&tmB, e.y, p.nY, q.words * 32, cluster ? kTN / 2 : kTN, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  static_assert(kMaxChunksStat * kABytes + kStagesStat * kBBytes == kStages * kStageBytes, "both layouts take the same shared memory");
  const TcKernel kernel = stationary ? simTensorKernel<kTcCount, 3> : cluster ? simTensorKernel<kTcCount, 1> : simTensorKernel<kTcCount, 0>;
  // units a pass over pk's row groups owns: tiles, or vertical tile pairs (same enumeration as the kernel's UnitWalk)
  auto unitsOf = [&](const TcParams& pk) -> uint64_t {
    return stationary ? countUnits<true, kRunStat>(pk, bandH) : cluster ? countUnits<true>(pk, bandH) : countUnits<false>(pk, bandH);
  };
  auto launchCount = [&](const TcParams& pk) {
    const uint64_t units = unitsOf(pk);
    if (!pilot) g_unitsPlanned += units;
    if (units) launchPersistent(kernel, cluster, tmA, tmB, pk, units, s);
  };
  auto launchVerify = [&](const int2* list, unsigned long long nCand, cudaStream_t on) {
    PhaseTimer         t("verify_candidates", on);
    const unsigned int blocks = static_cast<unsigned int>(std::min<unsigned long long>((nCand + 63) / 64, static_cast<unsigned long long>(smCount()) * 16));
    verifyCandidatesKernel<<<blocks, 256, 0, on>>>(x, y, q.words, list, nCand, S, C, static_cast<uint32_t>(q.nX), static_cast<uint32_t>(q.nY),
                                                   q.symmetric ? 1 : 0, popX, popY, permX, permY, thresh, q.sign, q.rowCounts,
                                                   q.symmetric ? q.rowCounts : nullptr, q.edges, q.edgeCursor, q.edgeCap);
    B200_LAUNCHED();
  };

  // Superposed pass in a PIPELINE of K chunks of the row groups (chunk k = groups k, k + K, ... of this pass's): the
  // exact verification of chunk k runs on a second stream while the tensor pass of chunk k + 1 has the SMs - a pass CTA
  // leaves room for one verify block per SM - so only the last chunk's verification is exposed.
  const uint64_t ownedGroups = (nGroups + groups.stride - 1) / groups.stride;
  const int      K = (super && !pilot && g_pipelineChunks > 1 && ownedGroups >= 4ull * g_pipelineChunks) ? g_pipelineChunks : 1;
  if (K > 1) {
    static cudaStream_t side[kMaxDevices] = {};
    cudaStream_t&       s2 = side[currentDeviceSlot()];
    if (!s2) B200_CUDA(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
    const unsigned long long capK = candCap / K;
    cudaEvent_t              ev[kMaxPipeline];
    {
      PhaseTimer t("neighbor_pass_tc", s);  // the K tensor passes, back to back on the caller's stream
      for (int k = 0; k < K; ++k) {
        TcParams        pk = p;
        const RowGroups g  = groups.chunk(k, K);
        pk.groupOffset = g.offset, pk.groupStride = g.stride;
        pk.cand        = cand.get() + static_cast<size_t>(k) * capK;
        pk.candCursor  = candCursor.get() + k;
        pk.candCap     = capK;
        launchCount(pk);
        B200_CUDA(cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming));
        B200_CUDA(cudaEventRecord(ev[k], s));
      }
    }
    unsigned long long listed = 0;
    int                redo[kMaxPipeline], nRedo = 0;
    for (int k = 0; k < K; ++k) {
      unsigned long long nk = 0;
      B200_CUDA(cudaStreamWaitEvent(s2, ev[k], 0));
      B200_CUDA(cudaMemcpyAsync(&nk, candCursor.get() + k, sizeof(nk), cudaMemcpyDeviceToHost, s2));
      B200_CUDA(cudaStreamSynchronize(s2));  // (waits for chunk k's pass and for the verifications queued before it)
      listed += nk;
      if (nk > capK) redo[nRedo++] = k;
      else if (nk) launchVerify(cand.get() + static_cast<size_t>(k) * capK, nk, s2);
      cudaEventDestroy(ev[k]);
    }
    cudaEvent_t done;
    B200_CUDA(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    B200_CUDA(cudaEventRecord(done, s2));
    B200_CUDA(cudaStreamWaitEvent(s, done, 0));  // the caller's stream continues after the last verification
    cudaEventDestroy(done);
    g_candidatesLast = listed;
    // A chunk whose list overflowed is redone on its own after the others, from rows only (S x 1) with the whole list:
    // its share of the list was a K-th of it, so even at S x C the chunk may fit, but the pipeline has moved on and the
    // rows-only pass needs the fewest candidates of the superposed ones.
    for (int r = 0; r < nRedo; ++r) ladder(groups.chunk(redo[r], K), S, 1);
    return {listed, false, 0.0};
  }

  const uint64_t units = unitsOf(p);
  if (units == 0) return {0, false, pilot ? bandPairs(p, nullptr, q.nX, q.nY) : 0.0};  // nothing owned or left by the band
  {
    PhaseTimer t("neighbor_pass_tc", s);
    launchCount(p);
  }
  if (mapBack) {
    const unsigned grid = static_cast<unsigned>(std::min<size_t>((q.nX + 255) / 256, static_cast<size_t>(smCount()) * 8));
    mapBackKernel<<<grid, 256, 0, s>>>(countsOrd.get(), permX, q.nX, q.rowCounts, permY, p.symmetric, q.edges, edgeStart.get(),
                                       q.edgeCursor, q.edgeCap);
    B200_LAUNCHED();
  }
  if (!super) return {0, false, pilot ? bandPairs(p, nullptr, q.nX, q.nY) : 0.0};
  // the one host read of a superposed pass: how many candidates (the callers synchronise for their edge total anyway)
  unsigned long long nCand = 0;
  B200_CUDA(cudaMemcpyAsync(&nCand, candCursor.get(), sizeof(nCand), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  if (pilot) return {nCand, false, bandPairs(p, bandH, q.nX, q.nY)};
  g_candidatesLast = nCand;
  if (nCand > candCap) return {nCand, true, 0.0};  // nothing has been counted yet
  if (nCand) launchVerify(cand.get(), nCand, s);
  return {nCand, false, 0.0};
}

// How far superposition pays depends on the data: the sum of S C random intersections must stay below the threshold
// ONE true neighbour pair reaches, or every accumulator is a candidate. A pilot over a prefix sample of the fingerprints
// (at most 1/64 of the pairs; candidates listed but nothing counted; the sample is put in popcount order of its own, as
// a prefix of the whole set's order would hold only its lowest popcounts) measures the candidate rate of each column
// factor, widest first; the model
//   time(S, C) = pairs / (S C) * tPair + candidates * S C * tVerify
// picks the cheapest. A narrower factor can only win while the wider one spends more time verifying than multiplying,
// so the search stops as soon as it does not.
// With the popcount band, `pairs` are the pairs the band leaves: the pilot counts them in its sample, at each column
// factor, and the candidate rate is per such pair. The whole set's band is only known after its own sort, so the pass
// is costed at the sample's share of banded pairs; every term of the model scales with that share alike, so the
// choice does not depend on it.
// popX, popY: the call's popcounts in the caller's order. Returns the cheapest (S, C) of (S, C), (S, C / 2), ... and 1 x 1.
static std::pair<int, int> pilotFactors(const SimLaunch& q, const int32_t* popX, const int32_t* popY, const uint16_t* thresh,
                                        cudaStream_t s, int S, int C) {
  const double nX = static_cast<double>(q.nX), nY = static_cast<double>(q.nY);
  SimLaunch    pilot = q;
  pilot.groupOffset  = 0;
  pilot.groupStride  = 1;
  pilot.nX           = std::min<size_t>(32768, std::max<size_t>(2 * kGroupRows, q.nX / 8));
  pilot.nY           = q.symmetric ? pilot.nX : std::min<size_t>(q.nY, std::max<size_t>(pilot.nX, q.nY / 8));
  const bool     same = pilot.x == pilot.y && pilot.nX == pilot.nY;
  const PopOrder ordX = popcountOrder(q.x, popX, pilot.nX, q.words, s);
  const PopOrder ordYown = same ? PopOrder{} : popcountOrder(q.y, popY, pilot.nY, q.words, s);
  const PopOrder& ordY   = same ? ordX : ordYown;
  const CountSets sample{pilot,           s, ordX.fp.get(), ordY.fp.get(), ordX.pop.get(), ordY.pop.get(), ordX.perm.get(),
                         ordY.perm.get(), thresh, same, true};
  const double sX = static_cast<double>(pilot.nX), sY = static_cast<double>(pilot.nY);
  const double pilotPairs = q.symmetric ? sX * (sX - 1) / 2.0 : sX * sY;
  const double totalPairs = (q.symmetric ? nX * (nX - 1) / 2.0 : nX * nY) / (q.groupStride < 1 ? 1 : q.groupStride);
  // seconds per unsuperposed pair / per verified pair; only their ratio (about 1 : 30) steers the choice. tPair is the
  // measured pass: 101.8 ms for the 4.67e11 pairs the popcount band leaves of the 1M bench at S C = 16 (H100 SXM, 400 W
  // limit; 108-110 ms for all 5.0e11 pairs without the band). On the bench data (sample in popcount order) the pilot
  // then costs 4 x 4 at 0.17 s and runs it; tools/pilot_model.py prints these figures for any fingerprint set without
  // a GPU.
  constexpr double tPair = 3.5e-12, tVerify = 0.1e-9;
  double bestT = -1.0;  // unsuperposed, costed at the widest factor's banded share
  int    bestS = 1, bestC = 1;
  for (int c = C; c >= 1; c >>= 1) {
    const PassResult r         = sample.pass({0, 1}, S, c, true);
    const double     left      = r.bandedPairs;
    const double     passPairs = totalPairs * (left / pilotPairs);
    if (bestT < 0.0) bestT = passPairs * tPair;
    const double tPass = passPairs / (S * c) * tPair;
    const double tVer  = left > 0.0 ? static_cast<double>(r.listed) * passPairs / left * S * c * tVerify : 0.0;
    if (tPass + tVer < bestT) bestT = tPass + tVer, bestS = S, bestC = c;
    if (tVer <= tPass) break;
  }
  return {bestS, bestC};
}

static void launchCountOp(const SimLaunch& q, cudaStream_t s) {
  const bool       same = q.x == q.y && q.nX == q.nY;
  Scratch<int32_t> popX(q.nX, s), popYown(same ? 0 : q.nY, s);
  launchRowPopcount(q.x, q.nX, q.words, popX.get(), s);
  if (!same) launchRowPopcount(q.y, q.nY, q.words, popYown.get(), s);
  const int32_t*    popY = same ? popX.get() : popYown.get();
  const int         maxS = 2 * q.words * 32;
  Scratch<uint16_t> thresh(static_cast<size_t>(maxS + 1), s);
  launchThreshTable(maxS, q.measure, q.cutoff, q.atLeast, thresh.get(), s);
  const RowGroups groups{q.groupOffset, q.groupStride < 1 ? 1 : q.groupStride};
  // Superposition serves the graph passes (symmetric and / or with an edge list): they synchronise for their edge
  // total anyway, and the superposed pass needs one host read of its candidate count. The plain thresholded count
  // (b200mol_tanimoto_count_ge) stays asynchronous on the unsuperposed tile.
  const bool graphPass = q.symmetric || q.edges != nullptr;
  if (!graphPass || g_superpose * g_superposeCols == 1) {
    if (graphPass) {
      g_superposeLast = 1;
      resetWalkCounters(s);
    }
    const CountSets call{q, s, q.x, q.y, popX.get(), popY, nullptr, nullptr, thresh.get(), same, false};
    call.pass(groups, 1, 1, false);
    return;
  }
  int S = g_superpose, C = g_superposeCols;
  if (g_superposeAuto && q.nX >= 8 * static_cast<size_t>(kGroupRows) && C > 1) std::tie(S, C) = pilotFactors(q, popX.get(), popY, thresh.get(), s, S, C);
  // A superposed pass runs on the fingerprints ordered by popcount (a stable sort: ties keep the caller's order, so every
  // rank of a sharded pass builds the same order). The S (C) fingerprints summed into one operand row then have nearly
  // the same popcount, and the pre-filter, which must assume the group's smallest, sits at the members' own threshold
  // instead of about a standard deviation below it. Row groups, pipeline chunks and rank ownership all live in this
  // order; the verification maps each pair back (permX / permY). Every pass of the call runs in it, also an unsuperposed
  // fallback (of the whole call, of a rank or of a pipeline chunk): it must cover the same row groups as the superposed
  // pass it replaces or completes, and a sharded call's ranks decide their fallbacks independently, so their row groups
  // must still be groups of ONE order for the union to be every pair once.
  const PopOrder  ordX    = popcountOrder(q.x, popX.get(), q.nX, q.words, s);
  const PopOrder  ordYown = same ? PopOrder{} : popcountOrder(q.y, popY, q.nY, q.words, s);
  const PopOrder& ordY    = same ? ordX : ordYown;
  const CountSets call{q, s, ordX.fp.get(), ordY.fp.get(), ordX.pop.get(), ordY.pop.get(), ordX.perm.get(), ordY.perm.get(),
                       thresh.get(), same, true};
  resetWalkCounters(s);
  g_superposeLast = call.ladder(groups, S, C);
}

// The operations on tensor cores. Returns false when the operation, measure or problem shape is not eligible (caller uses
// the SIMT tile); decided before any device work.
bool launchSimilarityTensor(SimMode op, const SimLaunch& q, cudaStream_t s) {
  const int bits = q.words * 32;
  if (!kTensorKernels[op][q.measure.kind] || bits % kTK != 0 || bits > 4096) return false;
  if (q.symmetric && !(q.x == q.y && q.nX == q.nY)) return false;
  if (op == kCount) launchCountOp(q, s);
  else launchTileOp(op, q, s);
  return true;
}

// ---- top-k search (topk.cu): the 0/1 expansion and one tile pass of the queries over a column slab of the library ----
namespace {
// {popcount, float bits of sqrt(popcount) (cosine) or 0} per operand row, whole tiles; rows past the end: popcount 0 and a
// square root no accumulator reaches
__global__ void topkMetaKernel(const int32_t* __restrict__ pop, size_t n, size_t nPad, int cosine, int2* __restrict__ out) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= nPad) return;
  if (i >= n) out[i] = make_int2(0, cosine ? __float_as_int(3.0e38f) : 0);
  else out[i] = make_int2(pop[i], cosine ? __float_as_int(sqrtf(static_cast<float>(pop[i]))) : 0);
}
}  // namespace

void launchExpandBits(const uint32_t* fp, size_t n, int words, uint8_t* out, cudaStream_t s) {
  const size_t nw = n * static_cast<size_t>(words);
  if (nw == 0) return;
  expandBitsKernel<<<static_cast<unsigned>((nw + 255) / 256), 256, 0, s>>>(fp, nw, reinterpret_cast<uint4*>(out));
  B200_LAUNCHED();
}

bool topkTileEligible(int words) { return (words * 32) % kTK == 0 && words * 32 <= 4096; }

void launchTopkTile(const Measure& m, const uint8_t* expQ, size_t nQ, const int32_t* popQ, const uint8_t* expLib, size_t nCols,
                    const int32_t* popCols, int words, const int4* bar, uint32_t* cand, uint32_t* count, uint32_t cap,
                    uint32_t colBase, cudaStream_t s) {
  const TcKernel kernel = kTopkKernels[m.kind];
  B200_REQUIRE(kernel, "no top-k tile for measure %d", m.kind);
  const bool cosine = m.kind == kCosine;
  TcParams   p      = tileGeometry(nQ, nCols, words, 1, 1);
  p.topkBar         = bar;
  p.topkCand        = cand;
  p.topkCount       = count;
  p.topkCap         = cap;
  p.topkColBase     = colBase;
  p.tvAlphaF        = static_cast<float>(m.alpha);
  p.tvBetaF         = static_cast<float>(m.beta);
  const size_t  rowsPad = static_cast<size_t>(p.tilesM) * kTM, colsPad = static_cast<size_t>(p.tilesN) * kTN;
  Scratch<int2> rowMeta(rowsPad, s), colMeta(colsPad, s);
  topkMetaKernel<<<static_cast<unsigned>((rowsPad + 255) / 256), 256, 0, s>>>(popQ, nQ, rowsPad, 0, rowMeta.get());
  B200_LAUNCHED();
  topkMetaKernel<<<static_cast<unsigned>((colsPad + 255) / 256), 256, 0, s>>>(popCols, nCols, colsPad, cosine ? 1 : 0, colMeta.get());
  B200_LAUNCHED();
  p.rowMeta = rowMeta.get();
  p.colMeta = colMeta.get();
  CUtensorMap tmA, tmB;
  makeTensorMap2D(&tmA, expQ, nQ, words * 32, kTM, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  makeTensorMap2D(&tmB, expLib, nCols, words * 32, kTN, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  const uint64_t units = countUnits<false>(p, nullptr);
  if (units == 0) return;
  launchPersistent(kernel, false, tmA, tmB, p, units, s);
}

}  // namespace b200

#ifdef B200_TC_TIMING
extern "C" void b200mol_debug_clocks_tc(unsigned long long* out8) {  // reads and resets the tile loop's clock counters
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out8, b200::g_tcClk, sizeof(b200::g_tcClk));
  unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  cudaMemcpyToSymbol(b200::g_tcClk, z, sizeof(z));
}
#endif
