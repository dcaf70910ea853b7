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
};

enum TcMode : int { kTcCount = 0, kTcTanimoto = 1, kTcCosine = 2 };
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

__global__ void iotaKernel(int32_t* __restrict__ v, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) v[i] = static_cast<int32_t>(i);
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
// Ownership is serpentine over cycles of `groupStride` groups (even cycles: group = cycle * stride + offset, odd
// cycles mirrored), which balances the triangle's shrinking rows across ranks to < 0.1 %.
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
        if (tn0 < p.tilesN) units = gRows * ((p.tilesN - tn0 + RUN - 1) / RUN);
      }
      if (inGroup < units) return;
      inGroup -= units;
      ++cycle;
    }
  }
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
    tnEnd              = min(p.tilesN, tnBeg + RUN);
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

// host twin of the walk's unit count (sizes the grid)
template <bool PAIR, int RUN = 1>
uint64_t countUnits(const TcParams& p) {
  const uint32_t G        = PAIR ? p.groupTiles / 2 : p.groupTiles;
  const uint32_t unitRows = PAIR ? (p.tilesM + 1) / 2 : p.tilesM;
  uint64_t       total    = 0;
  for (uint32_t cycle = 0; static_cast<uint64_t>(cycle) * p.groupStride * G < unitRows; ++cycle) {
    const uint32_t group = cycle * p.groupStride + ((cycle & 1u) ? p.groupStride - 1 - p.groupOffset : p.groupOffset);
    if (static_cast<uint64_t>(group) * G >= unitRows) continue;
    const uint32_t gRows = std::min(G, unitRows - group * G);
    const uint32_t tn0   = p.symmetric ? (group * p.groupTiles * p.rowSpan + 1u) / p.colSpan : 0u;
    if (tn0 < p.tilesN) total += static_cast<uint64_t>(gRows) * ((p.tilesN - tn0 + RUN - 1) / RUN);
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
  __shared__ int2 pairSlots[COUNT ? 8 : 1][COUNT ? kStagePairs : 1];  // count mode: each epilogue warp's PairStage

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
        if (!w.coords(p, rank, tm, tnBeg, tnEnd)) continue;
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
        } else {
          // fp64 Tanimoto / cosine straight from the accumulators: a quad of lanes writes 64 contiguous bytes of a row
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
    if constexpr (COUNT) {
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

}  // namespace

void launchRowPopcount(const uint32_t* fp, size_t n, int words, int32_t* pop, cudaStream_t s);
void launchThreshTable(int maxS, double cutoff, uint16_t* thresh, cudaStream_t s);

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

static bool launchTensorImpl(SimMode mode, const SimLaunch& q, cudaStream_t s, int superS, int superC, bool ordered,
                             bool* overflow, unsigned long long* pilotCand = nullptr);

// Count / materialise modes on tensor cores. Returns false when the problem shape is not eligible (caller uses the SIMT tile).
bool launchSimilarityTensor(SimMode mode, const SimLaunch& q, cudaStream_t s) {
  // Superposition serves the Butina passes (symmetric and / or with an edge list): they synchronise for their edge
  // total anyway, and the superposed pass needs one host read of its candidate count. The plain thresholded count
  // (b200mol_tanimoto_count_ge) stays asynchronous on the unsuperposed tile.
  const bool graphPass = mode == kCountTanimoto && (q.symmetric || q.edges != nullptr);
  if (!graphPass || g_superpose * g_superposeCols == 1) {
    if (graphPass) g_superposeLast = 1;
    return launchTensorImpl(mode, q, s, 1, 1, false, nullptr);
  }
  int S = g_superpose, C = g_superposeCols;
  // How far superposition pays depends on the data: the sum of S C random intersections must stay below the threshold
  // ONE true neighbour pair reaches, or every accumulator is a candidate. A pilot over a prefix sample of the
  // fingerprints (at most 1/64 of the pairs; candidates listed but nothing counted; launchTensorImpl orders the sample by
  // popcount as it does the whole set, while a prefix of the whole set's order would hold only its lowest popcounts) measures the candidate rate of each
  // column factor, widest first; the model
  //   time(S, C) = pairs / (S C) * tPair + candidates * S C * tVerify
  // picks the cheapest. A narrower factor can only win while the wider one spends more time verifying than multiplying, so the search stops as soon as it does not.
  if (g_superposeAuto && q.nX >= 8 * static_cast<size_t>(kGroupRows) && C > 1) {
    const double nX = static_cast<double>(q.nX), nY = static_cast<double>(q.nY);
    SimLaunch pilot   = q;
    pilot.groupOffset = 0;
    pilot.groupStride = 1;
    pilot.nX          = std::min<size_t>(32768, std::max<size_t>(2 * kGroupRows, q.nX / 8));
    pilot.nY          = q.symmetric ? pilot.nX : std::min<size_t>(q.nY, std::max<size_t>(pilot.nX, q.nY / 8));
    const double sX = static_cast<double>(pilot.nX), sY = static_cast<double>(pilot.nY);
    const double pilotPairs = q.symmetric ? sX * (sX - 1) / 2.0 : sX * sY;
    const double totalPairs = (q.symmetric ? nX * (nX - 1) / 2.0 : nX * nY) / (q.groupStride < 1 ? 1 : q.groupStride);
    // seconds per unsuperposed pair / per verified pair; only their ratio (about 1 : 30) steers the choice. tPair is the
    // measured pass: 108-110 ms for the 5.0e11 pairs of the 1M bench at S C = 16 (H100 SXM, 400 W limit). On the bench
    // data (sample in popcount order) the pilot then costs 4 x 4 at 0.17 s and runs it; tools/pilot_model.py prints
    // these figures for any fingerprint set without a GPU.
    constexpr double tPair = 3.5e-12, tVerify = 0.1e-9;
    double bestT = totalPairs * tPair;  // unsuperposed
    int    bestS = 1, bestC = 1;
    for (int c = C; c >= 1; c >>= 1) {
      unsigned long long got = 0;
      if (!launchTensorImpl(mode, pilot, s, S, c, true, nullptr, &got)) return false;
      const double tPass = totalPairs / (S * c) * tPair;
      const double tVer  = static_cast<double>(got) * totalPairs / pilotPairs * S * c * tVerify;
      if (tPass + tVer < bestT) bestT = tPass + tVer, bestS = S, bestC = c;
      if (tVer <= tPass) break;
    }
    S = bestS, C = bestC;
  }
  while (S * C > 1) {
    bool overflow = false;
    if (!launchTensorImpl(mode, q, s, S, C, true, &overflow)) return false;
    g_superposeLast = S * C;
    if (!overflow) return true;  // else: the candidate list overflowed (dense graph / loose cutoff), nothing was counted yet
    if (C > 1) C = 1;            // second chance: rows only
    else S = 1;
  }
  // The unsuperposed pass that completes a superposed one stays in popcount order: a sharded call's ranks decide their
  // fallbacks independently, and their row groups must still be groups of ONE order for the union to be every pair once.
  g_superposeLast = 1;
  return launchTensorImpl(mode, q, s, 1, 1, true, nullptr);
}

// ordered (graph passes of the count mode): run on the fingerprints in popcount order and map the results back. Every
// pass of a graph pass with superposition on is ordered, also an unsuperposed fallback (of the whole call, of a rank or
// of a pipeline chunk): it must cover the same row groups as the superposed pass it replaces or completes.
static bool launchTensorImpl(SimMode mode, const SimLaunch& q, cudaStream_t s, int superS, int superC, bool ordered,
                             bool* overflow, unsigned long long* pilotCand) {
  if (mode == kCountCosine) return false;
  const int bits = q.words * 32;
  if (bits % kTK != 0 || bits > 4096) return false;
  const bool same = (q.x == q.y && q.nX == q.nY);
  if (q.symmetric && !same) return false;

  const bool count    = mode == kCountTanimoto;
  const int  rowBytes = bits;  // one byte per bit of the fingerprint
  if (!count) superS = superC = 1;  // only the count mode verifies
  const bool   super  = superS * superC > 1;
  ordered             = count && (ordered || super);  // (a superposed pass is always ordered)
  const size_t nSuper = (q.nX + superS - 1) / superS;   // rows of the X operand
  const size_t nSuperY = (q.nY + superC - 1) / superC;  // rows of the Y operand (tile columns)

  TcParams p{};
  p.n         = static_cast<uint32_t>(nSuper);
  p.nY        = static_cast<uint32_t>(nSuperY);
  p.kChunks   = rowBytes / kTK;
  p.tilesM    = static_cast<uint32_t>((nSuper + kTM - 1) / kTM);
  p.superS    = superS;
  p.superC    = superC;
  p.rowSpan   = static_cast<uint32_t>(kTM * superS);
  p.colSpan   = static_cast<uint32_t>(kTN * superC);
  p.groupTiles = static_cast<uint32_t>(kGroupRows / (kTM * superS));
  p.tilesN    = static_cast<uint32_t>((nSuperY + kTN - 1) / kTN);
  p.symmetric = q.symmetric ? 1 : 0;
  p.groupOffset = q.groupOffset;
  p.groupStride = q.groupStride < 1 ? 1 : q.groupStride;
  p.sign      = q.sign;
  p.counts    = q.rowCounts;
  p.countsY   = q.symmetric ? q.rowCounts : nullptr;
  p.edges     = q.edges;
  p.edgeCursor = q.edgeCursor;
  p.edgeCap   = q.edgeCap;
  p.out       = q.out;
  p.outVec    = (q.nY % 2 == 0 && (reinterpret_cast<uintptr_t>(q.out) & 15) == 0) ? 1 : 0;
  const int recipLen = 2 * bits;
  Scratch<double> recip(mode == kMaterialiseTanimoto ? static_cast<size_t>(recipLen) + 1 : 0, s);
  if (mode == kMaterialiseTanimoto) {
    recipTableKernel<<<(recipLen + 256) / 256, 256, 0, s>>>(recip.get(), recipLen);
    B200_LAUNCHED();
    p.recipG = recip.get();
  }
  {
    // a pair passes iff 1 - c / (|A| + |B| - c) <= cutoff, i.e. c >= alpha (|A| + |B|); the pre-filter's alpha is rounded
    // DOWN (and its products too), so it never rejects what the exact fp64 table accepts
    const double a  = q.cutoff < 2.0 ? (1.0 - q.cutoff) / (2.0 - q.cutoff) : 0.0;
    float        af = static_cast<float>(a);
    if (static_cast<double>(af) > a) af = nextafterf(af, -1.0f);
    p.alpha = nextafterf(af, -1.0f);  // (one more ulp: fp64 rounding inside the table's predicate)
    if (p.alpha < 0.0f) p.alpha = 0.0f;
  }

  Scratch<int32_t> popX(q.nX, s), popYown(same ? 0 : q.nY, s);
  launchRowPopcount(q.x, q.nX, q.words, popX.get(), s);
  if (!same) launchRowPopcount(q.y, q.nY, q.words, popYown.get(), s);
  // A superposed pass runs on the fingerprints ordered by popcount (a stable sort: ties keep the caller's order, so every
  // rank of a sharded pass builds the same order). The S (C) fingerprints summed into one operand row then have nearly
  // the same popcount, and the pre-filter, which must assume the group's smallest, sits at the members' own threshold
  // instead of about a standard deviation below it. Row groups, pipeline chunks and rank ownership all live in this
  // order; the verification maps each pair back (permX / permY). An unsuperposed pass in this order counts and lists
  // edges in it, and mapBackKernel moves its results to the caller's indices.
  PopOrder       ordX, ordYown;
  const uint32_t *fx = q.x, *fy = q.y;
  const int32_t * popXs = popX.get(), *popYs = same ? popX.get() : popYown.get(), *permX = nullptr, *permY = nullptr;
  if (ordered) {
    ordX = popcountOrder(q.x, popX.get(), q.nX, q.words, s);
    if (!same) ordYown = popcountOrder(q.y, popYown.get(), q.nY, q.words, s);
    const PopOrder& ordY = same ? ordX : ordYown;
    fx = ordX.fp.get(), fy = ordY.fp.get();
    popXs = ordX.pop.get(), popYs = ordY.pop.get();
    permX = ordX.perm.get(), permY = ordY.perm.get();
  }
  const bool                  mapBack = ordered && !super;
  Scratch<int32_t>            countsOrd(mapBack ? q.nX : 0, s);
  Scratch<unsigned long long> edgeStart(mapBack && q.edges ? 1 : 0, s);
  if (mapBack) {
    B200_CUDA(cudaMemsetAsync(countsOrd.get(), 0, q.nX * sizeof(int32_t), s));
    p.counts  = countsOrd.get();
    p.countsY = q.symmetric ? countsOrd.get() : nullptr;
    if (q.edges) B200_CUDA(cudaMemcpyAsync(edgeStart.get(), q.edgeCursor, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
  }

  // 0/1 expansion of the fingerprints (2 KB per 2048-bit row); a superposed operand is the sum of superS (superC)
  // consecutive expansions. X and Y share one buffer when they are the same set, summed alike.
  const bool       ownY = !same || superS != superC;
  Scratch<uint8_t> expX(nSuper * static_cast<size_t>(rowBytes), s);
  Scratch<uint8_t> expYown(ownY ? nSuperY * static_cast<size_t>(rowBytes) : 0, s);
  auto expand = [&](const uint32_t* src, size_t rows, int S, size_t superRows, uint8_t* dst) {
    const size_t nw = superRows * static_cast<size_t>(q.words);
    const auto   grid = static_cast<unsigned>((nw + 255) / 256);
    if (S > 1) expandBitsSuperKernel<<<grid, 256, 0, s>>>(src, rows, q.words, S, superRows, reinterpret_cast<uint4*>(dst));
    else expandBitsKernel<<<grid, 256, 0, s>>>(src, nw, reinterpret_cast<uint4*>(dst));
    B200_LAUNCHED();
  };
  expand(fx, q.nX, superS, nSuper, expX.get());
  if (ownY) expand(fy, q.nY, superC, nSuperY, expYown.get());
  const uint8_t* expY = ownY ? expYown.get() : expX.get();

  // the epilogue's per-row metadata of both operands, padded to whole tiles for the producer's bulk copies (the lower
  // tile of a CTA pair may lie one tile row past the end)
  const size_t  rowsPad = (static_cast<size_t>(p.tilesM) + 1) * kTM, colsPad = static_cast<size_t>(p.tilesN) * kTN;
  Scratch<int2> rowMeta(rowsPad, s), colMeta(colsPad, s);
  tileMetaKernel<<<static_cast<unsigned>((rowsPad + 255) / 256), 256, 0, s>>>(popXs, q.nX, superS, nSuper, rowsPad, p.alpha, 1,
                                                                             rowMeta.get());
  B200_LAUNCHED();
  tileMetaKernel<<<static_cast<unsigned>((colsPad + 255) / 256), 256, 0, s>>>(popYs, q.nY, superC, nSuperY, colsPad, p.alpha, -1,
                                                                             colMeta.get());
  B200_LAUNCHED();
  p.rowMeta = rowMeta.get();
  p.colMeta = colMeta.get();
  // candidates of a superposed pass: (super row, super column) pairs the exact kernel re-examines. Sized for the
  // neighbour graphs this pass is used on (tens of edges per point); a denser graph overflows it and the caller falls back.
  unsigned long long          candCap = 0;
  Scratch<int2>               cand;
  Scratch<unsigned long long> candCursor;
  if (super) {
    const unsigned long long all = static_cast<unsigned long long>(nSuper) * nSuperY;
    candCap                      = std::min<unsigned long long>(all, std::max<unsigned long long>(1ull << 22, 64ull * q.nX));
    cand                         = Scratch<int2>(candCap, s);
    candCursor                   = Scratch<unsigned long long>(kMaxPipeline, s);
    B200_CUDA(cudaMemsetAsync(candCursor.get(), 0, kMaxPipeline * sizeof(unsigned long long), s));
    p.cand = cand.get(), p.candCursor = candCursor.get(), p.candCap = candCap;
  }
  const int         maxS = 2 * bits;
  Scratch<uint16_t> thresh(static_cast<size_t>(maxS + 1), s);
  if (mode == kCountTanimoto) {
    launchThreshTable(maxS, q.cutoff, thresh.get(), s);
    p.threshLen = maxS + 1;
  }
  p.thresh = thresh.get();

  CUtensorMap tmA, tmB;
  makeTensorMap2D(&tmA, expX.get(), nSuper, rowBytes, kTM, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);
  // CTA pairs sharing the column operand (TMA multicast); 3 = the same with the row operand stationary, for fingerprints
  // whose 128-row tile fits its shared-memory region (else the plain pair runs)
  const bool cluster    = count && g_tensorCluster != 0;
  const bool stationary = cluster && g_tensorCluster == 3 && p.kChunks <= kMaxChunksStat;
  makeTensorMap2D(&tmB, expY, nSuperY, rowBytes, cluster ? kTN / 2 : kTN, kTK, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1);

  static_assert(kMaxChunksStat * kABytes + kStagesStat * kBBytes == kStages * kStageBytes, "both layouts take the same shared memory");
  const size_t smemBytes = static_cast<size_t>(kStages) * kStageBytes + 1024;
  static bool configured[kMaxDevices] = {};
  auto optIn = [&](auto kernel) {
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smemBytes)));
  };
  if (!configured[currentDeviceSlot()]) {
    optIn(simTensorKernel<kTcCount, 0>);
    optIn(simTensorKernel<kTcCount, 1>);
    optIn(simTensorKernel<kTcCount, 3>);
    optIn(simTensorKernel<kTcTanimoto, 0>);
    optIn(simTensorKernel<kTcCosine, 0>);
    configured[currentDeviceSlot()] = true;
  }
  // units a call owns: tiles, or vertical tile pairs (same enumeration as the kernel's UnitWalk)
  auto unitsOf = [&](const TcParams& pk) -> uint64_t {
    return stationary ? countUnits<true, kRunStat>(pk) : cluster ? countUnits<true>(pk) : countUnits<false>(pk);
  };
  // the count kernel over the row groups `pk` selects (false: none of them is owned by this call)
  auto launchCount = [&](const TcParams& pk) -> bool {
    const uint64_t units = unitsOf(pk);
    if (units == 0) return false;
    if (cluster) {
      cudaLaunchConfig_t cfg{};
      cudaLaunchAttribute attr[1];
      attr[0].id               = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = 2;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.blockDim         = dim3(kThreadsTC);
      cfg.dynamicSmemBytes = smemBytes;
      cfg.stream           = s;
      cfg.attrs            = attr;
      cfg.numAttrs         = 1;
      cfg.gridDim          = dim3(2);
      int maxClusters = 0;
      if (stationary) B200_CUDA(cudaOccupancyMaxActiveClusters(&maxClusters, simTensorKernel<kTcCount, 3>, &cfg));
      else B200_CUDA(cudaOccupancyMaxActiveClusters(&maxClusters, simTensorKernel<kTcCount, 1>, &cfg));
      B200_REQUIRE(maxClusters >= 1, "no CTA pair fits the device");
      uint64_t pairs = maxClusters;  // persistent: one resident cluster per schedulable SM pair
      if (pairs > units) pairs = units;
      cfg.gridDim = dim3(static_cast<unsigned>(2 * pairs));
      if (stationary) B200_CUDA(cudaLaunchKernelEx(&cfg, simTensorKernel<kTcCount, 3>, tmA, tmB, pk));
      else B200_CUDA(cudaLaunchKernelEx(&cfg, simTensorKernel<kTcCount, 1>, tmA, tmB, pk));
    } else {
      const int grid = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(smCount()), units));
      simTensorKernel<kTcCount, 0><<<grid, kThreadsTC, smemBytes, s>>>(tmA, tmB, pk);
    }
    B200_LAUNCHED();
    return true;
  };
  auto launchVerify = [&](const int2* list, unsigned long long nCand, cudaStream_t on) {
    PhaseTimer         t("verify_candidates", on);
    const unsigned int blocks2 = static_cast<unsigned int>(std::min<unsigned long long>((nCand + 63) / 64, static_cast<unsigned long long>(smCount()) * 16));
    verifyCandidatesKernel<<<blocks2, 256, 0, on>>>(fx, fy, q.words, list, nCand, superS, superC, static_cast<uint32_t>(q.nX),
                                                    static_cast<uint32_t>(q.nY), q.symmetric ? 1 : 0, popXs, popYs, permX, permY,
                                                    thresh.get(), q.sign, q.rowCounts, q.symmetric ? q.rowCounts : nullptr, q.edges,
                                                    q.edgeCursor, q.edgeCap);
    B200_LAUNCHED();
  };

  // Superposed pass in a PIPELINE of K chunks of the row groups (chunk k = groups k, k + K, ... of this call's): the exact
  // verification of chunk k runs on a second stream while the tensor pass of chunk k + 1 has the SMs - a pass CTA leaves
  // room for one verify block per SM - so only the last chunk's verification is exposed.
  // A chunk whose candidate list overflowed is redone on its own with fewer pairs per accumulator after the others.
  const uint64_t ownedGroups = ((q.nX + kGroupRows - 1) / kGroupRows + p.groupStride - 1) / p.groupStride;
  const int      K = (super && !pilotCand && g_pipelineChunks > 1 && ownedGroups >= 4ull * g_pipelineChunks) ? g_pipelineChunks : 1;
  if (K > 1) {
    static cudaStream_t side[kMaxDevices] = {};
    cudaStream_t&       s2 = side[currentDeviceSlot()];
    if (!s2) B200_CUDA(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
    const unsigned long long capK = candCap / K;
    cudaEvent_t              ev[kMaxPipeline];
    {
      PhaseTimer t("neighbor_pass_tc", s);  // the K tensor passes, back to back on the caller's stream
      for (int k = 0; k < K; ++k) {
        TcParams pk    = p;
        pk.groupOffset = p.groupOffset + static_cast<uint32_t>(k) * p.groupStride;
        pk.groupStride = static_cast<uint32_t>(K) * p.groupStride;
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
    for (int r = 0; r < nRedo; ++r) {
      SimLaunch qk   = q;
      qk.groupOffset = p.groupOffset + static_cast<uint32_t>(redo[r]) * p.groupStride;
      qk.groupStride = static_cast<uint32_t>(K) * p.groupStride;
      bool again     = false;
      if (!launchTensorImpl(mode, qk, s, superS, 1, true, &again)) return false;
      if (again && !launchTensorImpl(mode, qk, s, 1, 1, true, nullptr)) return false;
    }
    return true;
  }

  if (unitsOf(p) == 0) return true;  // nothing owned by this rank (more ranks than row groups)
  int blocks = smCount();
  if (static_cast<uint64_t>(blocks) > unitsOf(p)) blocks = static_cast<int>(unitsOf(p));
  if (mode == kCountTanimoto) {
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
  } else if (mode == kMaterialiseTanimoto) {
    PhaseTimer t("cross_tc", s);
    simTensorKernel<kTcTanimoto, 0><<<blocks, kThreadsTC, smemBytes, s>>>(tmA, tmB, p);
  } else {
    PhaseTimer t("cross_tc", s);
    simTensorKernel<kTcCosine, 0><<<blocks, kThreadsTC, smemBytes, s>>>(tmA, tmB, p);
  }
  if (mode != kCountTanimoto) B200_LAUNCHED();
  if (super) {
    // the one host read of a superposed pass: how many candidates (the callers synchronise for their edge total anyway)
    unsigned long long nCand = 0;
    B200_CUDA(cudaMemcpyAsync(&nCand, candCursor.get(), sizeof(nCand), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    if (pilotCand) {  // dry run over one row group: the candidate count is the result
      *pilotCand = nCand;
      return true;
    }
    g_candidatesLast = nCand;
    if (nCand > candCap) {
      if (overflow) *overflow = true;  // nothing has been counted yet: the caller reruns without superposition
      return true;
    }
    if (nCand) launchVerify(cand.get(), nCand, s);
  }
  return true;
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
