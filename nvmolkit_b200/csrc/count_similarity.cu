// Tanimoto, Dice and Tversky similarity on count vectors (RDKit's SparseIntVect measures): b200mol_count_cross, _topk
// and _threshold. The value of a pair is tverskyFromCounts (similarity.cuh) of c = sum over bins of min(x, y) and the row
// sums a, b: the expression, and the order of its fp64 operations, of every other Tversky path.
//
//   compaction  once per call and group: a warp per row sums it, counts its non-zeros and checks every count against
//               0 .. 65535; a scan gives each row its place; a second warp per row packs its non-zero bins, ascending,
//               as (bin << 16 | count) words, so that a warp reads a row's list with coalesced loads. The range flag and
//               the list sizes are the call's one host read, before anything is written to the caller's outputs.
//   pass        countPassKernel: a CTA keeps a block of QB query rows dense in shared memory, transposed to
//               [bin][query] (u16), so that the lanes of a warp, one query each, read consecutive bytes. A warp streams a
//               library row's list once for the whole block, QB words at a time, broadcast by shuffle, and adds
//               min(query count, library count) per non-zero: about 50 adds for a Morgan count row of 2048 bins against
//               2048 for a dense loop. c is exact, so what follows tests the exact fp64 value:
//     matrix      values staged per warp in shared memory, written as 128-byte row segments;
//     top-k       a pair that beats its row's bar (the running list's k-th entry, the order of topk.cuh) takes a
//                 candidate slot with its value; the protocol of topk.cu: slabs of library columns that double, a
//                 select that merges a row's slots into its list, and a scan (topk.cuh's scanBest) that redoes a slab
//                 for the rows whose candidates did not fit;
//     threshold   a pair with value >= t is listed with its value, in threshold.cu's attempt protocol (thresholdCsr),
//                 whose assembly (keys, one radix sort, indptr by bisection) makes the CSR. A self search runs the full
//                 pass (it needs no diagonal step);
//     neighbours  (Butina: b200mol_count_neighbor_edges, and butina.cu's fusedButina for b200mol_count_butina_fused;
//                 Tanimoto and Dice only) a self pass over the rows compacted
//                 in (row sum, index) order (a stable radix sort; the stats and pack kernels gather through it). Query
//                 block [q0, q0 + QB) visits only columns >= q0, and in its own block only col > row, so each
//                 unordered pair is tested once; a pair with 1 - value <= cutoff (fp64) adds to both degrees and is
//                 written as the caller's (i, j), i < j.
// Query blocks are 32 rows up to 2048 bins and 16 rows above, where a warp takes two library rows at a time (half a
// warp each), so that the block stays within 128 KiB of shared memory.
//
// The sum band of the neighbour pass (exact). For Tanimoto and Dice the value is the correctly rounded quotient of
// exact integers, c / (a + b - c) or c / ((a + b) / 2), every intermediate exact (sums < 2^31). For a row of sum a and
// a column of sum b >= a, c <= min(a, b) = a, and the exact quotient grows with c and, c fixed, falls as a falls, so it
// is at most that of (c = a, a, b), which for A >= a is at most that of (c = A, a = A, b) (A / b, 2A / (A + b): both
// grow with A). Rounding to nearest is monotone, so value(c, a, b) <= value(A, A, b); and RN(1 - s) does not increase
// as s grows. Let A be the largest sum of a query block (its last row, in sum order). Every column past the block has
// b >= A, and value(A, A, b) does not increase as b grows (A / b, 2A / (A + b)). So once
// 1 - value(A, A, b) <= cutoff fails at a sorted column, it fails at every later one, and no row of the block has a
// neighbour there. countBandKernel bisects the sorted sums once per block for the first such column; the block's
// columns end there. (A = 0: every value of the block is 0, and the band is everything at cutoff 1, else nothing past
// the block.) The bound and the kernel's value are the same tverskyFromCounts of intrinsics, never contracted into an
// FMA, and the comparison is __dsub_rn. The band's lengths differ widely from block to block, so the pass takes work
// from a flat list of (block, kUnitCols-column chunk) units, a persistent grid walking it in order.
#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "options.cuh"
#include "similarity.cuh"
#include "topk.cuh"

namespace b200 {
namespace {

constexpr int kMaxBins   = 4096;
constexpr int kMaxCount  = 65535;  // every row sum (<= 4096 * 65535) and a + b - c stay below 2^31
constexpr int kPassWarps = 16;
constexpr int kTileCols  = 16;             // columns a warp stages before writing them (128 bytes of each matrix row)
constexpr int kStagePad  = kTileCols + 1;  // (row stride of the stage, in doubles)
constexpr unsigned kFull = 0xffffffffu;

constexpr uint32_t kUnitCols = 4096;       // columns of a neighbour-pass work unit (a multiple of kPassWarps * kTileCols)
static_assert(kUnitCols % (kPassWarps * kTileCols) == 0, "a unit is whole sweeps of the CTA's warps");

enum CountOp : int { kCountMatrix = 0, kCountTopk = 1, kCountThreshold = 2, kCountNeighbors = 3 };

__device__ unsigned long long g_countStat[1];  // [0] pairs the last neighbour pass compared

// One group in the form the pass reads: row r's non-zero bins, ascending, as (bin << 16 | count) at
// pairs[start[r] .. start[r + 1]), and sum[r] the sum of its counts.
struct CountRows {
  const uint32_t*  pairs = nullptr;
  const long long* start = nullptr;
  const int32_t*   sum   = nullptr;
};

// Row r of a compaction is the caller's row perm[r] (perm = NULL: row r).
__device__ __forceinline__ const int32_t* compactRow(const int32_t* rows, const int32_t* perm, size_t r, int bins) {
  return rows + (perm ? static_cast<size_t>(perm[r]) : r) * bins;
}

// sum[r], nnz[r] (nnz[n] = 0, for the scan) and *bad = 1 if a count lies outside 0 .. kMaxCount; a warp per row
__global__ void __launch_bounds__(256) countStatsKernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ perm, size_t n,
                                                        int bins, int32_t* __restrict__ sum, long long* __restrict__ nnz,
                                                        int* __restrict__ bad) {
  const int    lane  = threadIdx.x & 31;
  const size_t warps = static_cast<size_t>(gridDim.x) * (blockDim.x / 32);
  for (size_t r = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32; r < n; r += warps) {
    const int32_t* row = compactRow(rows, perm, r, bins);
    unsigned       s = 0;
    int            z = 0;
    bool           out = false;
    for (int j = lane; j < bins; j += 32) {
      const int32_t v = row[j];
      out |= v < 0 || v > kMaxCount;
      s += static_cast<unsigned>(v);
      z += v != 0;
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(kFull, s, o), z += __shfl_xor_sync(kFull, z, o);
    out = __any_sync(kFull, out);
    if (lane == 0) {
      sum[r] = static_cast<int32_t>(s);
      nnz[r] = z;
      if (out) atomicExch(bad, 1);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) nnz[n] = 0;
}

// row r's non-zeros, ascending, at pairs[start[r] ..]; a warp per row
__global__ void __launch_bounds__(256) countPackKernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ perm, size_t n,
                                                       int bins, const long long* __restrict__ start, uint32_t* __restrict__ pairs) {
  const int    lane  = threadIdx.x & 31;
  const size_t warps = static_cast<size_t>(gridDim.x) * (blockDim.x / 32);
  for (size_t r = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32; r < n; r += warps) {
    const int32_t* row = compactRow(rows, perm, r, bins);
    long long      at  = start[r];
    for (int base = 0; base < bins; base += 32) {
      const int      j = base + lane;
      const int32_t  v = j < bins ? row[j] : 0;
      const unsigned m = __ballot_sync(kFull, v != 0);
      if (v != 0) pairs[at + __popc(m & ((1u << lane) - 1u))] = (static_cast<uint32_t>(j) << 16) | static_cast<uint32_t>(v);
      at += __popc(m);
    }
  }
}

struct PassArgs {
  CountRows q, lib;
  size_t    nQ         = 0;
  uint32_t  colBeg     = 0;  // the library columns of this pass: [colBeg, colEnd), colsPerCta to a CTA (grid.y)
  uint32_t  colEnd     = 0;
  uint32_t  colsPerCta = 0;
  int       bins       = 0;
  Measure   measure;
  // matrix: out[row * ld + column]
  double* out = nullptr;
  size_t  ld  = 0;
  // top-k: the running lists (their k-th entry is the row's bar) and the candidate slots
  const double*  listV = nullptr;
  const int32_t* listI = nullptr;
  int            k     = 0;
  double*        candV = nullptr;
  uint32_t*      candI = nullptr;
  uint32_t*      count = nullptr;
  uint32_t       cap   = 0;
  // threshold: pairs with value >= t appended at *cursor, while below listCap
  double              t       = 0.0;
  int2*               list    = nullptr;
  double*             vals    = nullptr;
  unsigned long long* cursor  = nullptr;
  unsigned long long  listCap = 0;
  // neighbours (a self pass over rows in sum order): a pair (row, col), col > row, with 1 - value <= cutoff adds one to
  // both rows' degrees and is appended to `list` as the caller's (i, j), i < j, by the cursor protocol of threshold.
  // Query block b (rows [b QB, b QB + QB)) visits the columns [b QB, bandEnd[b]) as units of kUnitCols columns; its
  // units are unitStart[b] .. unitStart[b + 1], and unitStart[nBlocks] is their total.
  double                    cutoff    = 0.0;
  const int32_t*            perm      = nullptr;  // [nQ] the caller's index of each row
  int32_t*                  degrees   = nullptr;  // [nQ] (the caller's indices)
  const unsigned long long* unitStart = nullptr;  // [nBlocks + 1]
  const uint32_t*           bandEnd   = nullptr;  // [nBlocks]
  size_t                    nBlocks   = 0;
};

__host__ __device__ constexpr size_t queryBlockBytes(int bins, int qb) { return (static_cast<size_t>(bins) * qb * 2 + 15) & ~size_t(15); }

// Query rows [q0, q0 + QB) dense in shared memory as qs[bin][query] (u16); every thread of the CTA takes part
template <int QB>
__device__ __forceinline__ void loadQueryBlock(const PassArgs& a, uint16_t* qs, size_t q0, int nq) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < a.bins * QB / 2; i += blockDim.x) reinterpret_cast<uint32_t*>(qs)[i] = 0;
  __syncthreads();
  for (int j = warp; j < nq; j += kPassWarps)
    for (long long p = a.q.start[q0 + j] + lane; p < a.q.start[q0 + j + 1]; p += 32) {
      const uint32_t v = a.q.pairs[p];
      qs[(v >> 16) * QB + j] = static_cast<uint16_t>(v & 0xffffu);
    }
  __syncthreads();
}

// The loaded query block against library columns [c0, c1). Lane `sub` of a group of QB lanes serves query q0 + sub; a
// warp takes 32 / QB library columns at a time, one per group.
template <int QB, int OP>
__device__ __forceinline__ void passColumns(const PassArgs& a, const uint16_t* qs, uint8_t* smem, size_t q0, int nq, uint32_t c0,
                                            uint32_t c1) {
  constexpr int G = 32 / QB;
  const int     lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane % QB, grp = lane / QB;
  const bool    live = sub < nq;
  const size_t  row  = q0 + sub;
  const int     sa   = live ? a.q.sum[row] : 0;
  double        barV = -1.0;
  int32_t       barI = kNoIdx;
  if constexpr (OP == kCountTopk)
    if (live) barV = a.listV[row * a.k + a.k - 1], barI = a.listI[row * a.k + a.k - 1];
  int deg = 0;  // (neighbours) of the lane's row in these columns
  double* stage = reinterpret_cast<double*>(smem + queryBlockBytes(a.bins, QB)) + warp * QB * kStagePad;  // (matrix)
  for (uint32_t tile = c0 + warp * kTileCols; tile < c1; tile += kPassWarps * kTileCols) {
    for (int i = 0; i < kTileCols; i += G) {
      const uint32_t col  = tile + i + grp;
      const bool     have = col < c1;
      long long      beg  = 0;
      int            n    = 0;
      if (have) beg = a.lib.start[col], n = static_cast<int>(a.lib.start[col + 1] - beg);
      int nmax = n;
      if constexpr (G == 2) nmax = max(n, __shfl_xor_sync(kFull, n, 16));
      int c = 0;
      for (int j0 = 0; j0 < nmax; j0 += QB) {  // (warp-uniform)
        const uint32_t p   = j0 + sub < n ? __ldg(a.lib.pairs + beg + j0 + sub) : 0u;  // (count 0 adds nothing)
        const int      lim = min(QB, nmax - j0);
#pragma unroll 4
        for (int t = 0; t < lim; ++t) {
          const uint32_t v = __shfl_sync(kFull, p, t, QB);
          c += min(static_cast<int>(qs[(v >> 16) * QB + sub]), static_cast<int>(v & 0xffffu));
        }
      }
      const double v = have ? measureFromCounts<true>(a.measure, c, sa, a.lib.sum[col]) : 0.0;
      if constexpr (OP == kCountMatrix) {
        stage[sub * kStagePad + i + grp] = v;
      } else if constexpr (OP == kCountTopk) {
        if (live && have && better(v, static_cast<int32_t>(col), barV, barI)) {
          const uint32_t at = atomicAdd(a.count + row, 1u);
          if (at < a.cap) a.candV[row * a.cap + at] = v, a.candI[row * a.cap + at] = col;
        }
      } else {
        bool keep;
        if constexpr (OP == kCountNeighbors) keep = live && have && col > row && __dsub_rn(1.0, v) <= a.cutoff;
        else keep = live && have && v >= a.t;
        const unsigned m = __ballot_sync(kFull, keep);
        if (m) {
          const int          first = __ffs(m) - 1;
          unsigned long long base  = 0;
          if (lane == first) base = atomicAdd(a.cursor, static_cast<unsigned long long>(__popc(m)));
          base = __shfl_sync(kFull, base, first);
          const unsigned long long at = base + __popc(m & ((1u << lane) - 1u));
          if constexpr (OP == kCountNeighbors) {
            deg += keep;
            const unsigned mine = m & (G == 1 ? kFull : 0xffffu << (grp * 16));  // the hits of this group's column
            if (sub == 0 && mine) atomicAdd(a.degrees + a.perm[col], __popc(mine));
            if (keep && at < a.listCap) {
              const int i = a.perm[row], j = a.perm[col];
              a.list[at]  = make_int2(min(i, j), max(i, j));
            }
          } else {
            if (keep && at < a.listCap) a.list[at] = make_int2(static_cast<int>(row), static_cast<int>(col)), a.vals[at] = v;
          }
        }
      }
    }
    if constexpr (OP == kCountMatrix) {
      __syncwarp();
      const uint32_t col = tile + lane % kTileCols;
      for (int r = lane / kTileCols; r < nq; r += 32 / kTileCols)
        if (col < c1) a.out[(q0 + r) * a.ld + col] = stage[r * kStagePad + lane % kTileCols];
      __syncwarp();  // (the stage is read before the next tile overwrites it)
    }
  }
  if constexpr (OP == kCountNeighbors)
    if (deg) atomicAdd(a.degrees + a.perm[row], deg);
}

// Matrix, top-k and threshold: grid (query blocks of QB rows, column parts). Neighbours: a persistent grid; CTA x of X
// walks the units [total x / X, total (x + 1) / X) in order, and reloads the query block only when a unit starts a
// new one.
template <int QB, int OP>
__global__ void __launch_bounds__(kPassWarps * 32) countPassKernel(const PassArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint16_t* qs = reinterpret_cast<uint16_t*>(smem);  // [bins][QB]
  if constexpr (OP == kCountNeighbors) {
    __shared__ unsigned long long u1;  // (in shared memory: it stays live over the whole walk)
    const unsigned long long total = a.unitStart[a.nBlocks];
    const unsigned long long u0    = total * blockIdx.x / gridDim.x;
    if (threadIdx.x == 0) u1 = total * (blockIdx.x + 1) / gridDim.x;
    __syncthreads();
    if (u0 >= u1) return;
    uint32_t lo = 0, hi = static_cast<uint32_t>(a.nBlocks);  // the block of u0: the last b with unitStart[b] <= u0
    while (hi - lo > 1) {                                      // (every block has a unit)
      const uint32_t mid = (lo + hi) / 2;
      if (a.unitStart[mid] <= u0) lo = mid;
      else hi = mid;
    }
    uint32_t b = lo, loaded = ~0u;
    for (unsigned long long u = u0; u < u1; ++u) {
      while (a.unitStart[b + 1] <= u) ++b;
      const size_t q0 = static_cast<size_t>(b) * QB;
      const int    nq = static_cast<int>(min(static_cast<size_t>(QB), a.nQ - q0));
      if (b != loaded) {
        __syncthreads();  // (every warp is done with the previous block)
        loadQueryBlock<QB>(a, qs, q0, nq);
        loaded = b;
      }
      const uint32_t c0 = static_cast<uint32_t>(q0 + (u - a.unitStart[b]) * kUnitCols);
      passColumns<QB, OP>(a, qs, smem, q0, nq, c0, min(a.bandEnd[b], c0 + kUnitCols));
    }
  } else {
    const size_t q0 = static_cast<size_t>(blockIdx.x) * QB;
    const int    nq = static_cast<int>(min(static_cast<size_t>(QB), a.nQ - q0));
    loadQueryBlock<QB>(a, qs, q0, nq);
    const uint32_t c0 = a.colBeg + blockIdx.y * a.colsPerCta;
    passColumns<QB, OP>(a, qs, smem, q0, nq, c0, min(a.colEnd, c0 + a.colsPerCta));
  }
}

size_t passSmemBytes(int op, int bins, int qb) {
  return queryBlockBytes(bins, qb) + (op == kCountMatrix ? static_cast<size_t>(kPassWarps) * qb * kStagePad * sizeof(double) : 0);
}

// 32-row query blocks up to 2048 bins, 16-row ones above
int passQueryRows(int bins) { return bins <= 2048 ? 32 : 16; }

template <int QB, int OP>
void launchPassAs(const PassArgs& a, dim3 grid, cudaStream_t s) {
  const size_t  smem = passSmemBytes(OP, a.bins, QB);
  static size_t configured[kMaxDevices] = {};
  if (smem > configured[currentDeviceSlot()]) {
    B200_CUDA(cudaFuncSetAttribute(countPassKernel<QB, OP>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    configured[currentDeviceSlot()] = smem;
  }
  if constexpr (OP == kCountNeighbors) {  // as many CTAs as the device holds at once
    int perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, countPassKernel<QB, OP>, kPassWarps * 32, smem));
    grid = dim3(static_cast<unsigned>(std::max(1, perSm) * smCount()));
  }
  countPassKernel<QB, OP><<<grid, kPassWarps * 32, smem, s>>>(a);
  B200_LAUNCHED();
}

// The pass over columns [a.colBeg, a.colEnd) (neighbours: over the units of a.unitStart); enough column parts per query
// block to give the device several CTAs per SM.
template <int OP>
void launchPass(PassArgs a, cudaStream_t s) {
  const int qb = passQueryRows(a.bins);
  dim3      grid;
  if constexpr (OP != kCountNeighbors) {
    const size_t   blocks = (a.nQ + qb - 1) / qb;
    const uint32_t cols   = a.colEnd - a.colBeg, unit = kPassWarps * kTileCols;
    const size_t   parts  = std::max<size_t>(1, (8 * static_cast<size_t>(smCount()) + blocks - 1) / blocks);
    uint32_t       per    = static_cast<uint32_t>((cols + parts - 1) / parts);
    per                   = std::max<uint32_t>(per, (cols + 65534) / 65535);  // (grid.y)
    a.colsPerCta          = (per + unit - 1) / unit * unit;
    grid                  = dim3(static_cast<unsigned>(blocks), (cols + a.colsPerCta - 1) / a.colsPerCta);
  }
  if (qb == 32) launchPassAs<32, OP>(a, grid, s);
  else launchPassAs<16, OP>(a, grid, s);
}

// ---- top-k ----

struct TopkState {
  double*   values;   // [nQ][k] the running lists, best first; padded with (-1, kNoIdx) until full
  int32_t*  indices;  // [nQ][k]
  int       k;
  double*   candV;  // [nQ][cap] candidate slots
  uint32_t* candI;
  uint32_t* count;  // [nQ] slots asked for
  uint32_t* redo;   // [nQ] 1: the row's candidates of this slab did not fit
  uint32_t  cap;
};

__global__ void countTopkInitKernel(double* values, int32_t* indices, size_t n) {
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    values[i] = -1.0, indices[i] = kNoIdx;
}

// One CTA per query: the row's candidates (with their values) sorted together with its list by the contract's key, and
// the k best kept. afterScan = 0, after a pass: a row that asked for more slots than there are merges nothing and is
// marked for the scan. afterScan = 1: the slots hold the scan's results, of the marked rows only.
__global__ void __launch_bounds__(kSelThreads) countSelectKernel(const TopkState a, int afterScan) {
  __shared__ double  val[kSelItems];
  __shared__ int32_t idx[kSelItems];
  const uint32_t q = blockIdx.x;
  const int      tid = threadIdx.x, k = a.k;
  const uint32_t asked = a.count[q];
  if (afterScan) {
    if (!a.redo[q]) return;
  } else {
    const bool fits = asked <= a.cap;
    __syncthreads();  // (every thread has read count[q] before thread 0 rewrites redo[q])
    if (tid == 0) a.redo[q] = fits ? 0u : 1u;
    if (!fits) return;
  }
  __syncthreads();
  if (tid == 0) a.count[q] = 0;  // the slots are free for the next pass
  const int n = static_cast<int>(asked);
  if (n == 0) return;
  for (int i = tid; i < k; i += kSelThreads) val[i] = a.values[static_cast<size_t>(q) * k + i], idx[i] = a.indices[static_cast<size_t>(q) * k + i];
  for (int j = tid; j < n; j += kSelThreads) {
    const uint32_t col = a.candI[static_cast<size_t>(q) * a.cap + j];
    val[k + j]         = col == kNoCand ? -1.0 : a.candV[static_cast<size_t>(q) * a.cap + j];
    idx[k + j]         = col == kNoCand ? kNoIdx : static_cast<int32_t>(col);
  }
  const int n2 = nextPow2(k + n);
  for (int i = k + n + tid; i < n2; i += kSelThreads) val[i] = -1.0, idx[i] = kNoIdx;
  sortBestFirst(val, idx, n2);
  for (int i = tid; i < k; i += kSelThreads) a.values[static_cast<size_t>(q) * k + i] = val[i], a.indices[static_cast<size_t>(q) * k + i] = idx[i];
}

// The redo of a slab [colBeg, colEnd) for the marked rows: grid (parts, queries), a thread per column against the query
// row dense in shared memory. What beats the row's bar is parked in shared memory and, when that fills up, sorted and cut
// to k, which raises the CTA's bar; the CTA's k best go to the slots [part * k, part * k + k) with their values.
__global__ void __launch_bounds__(kSelThreads) countScanKernel(const TopkState a, const CountRows qr, const CountRows lib, int bins,
                                                               const Measure m, uint32_t colBeg, uint32_t colEnd) {
  __shared__ double   val[kSelItems];
  __shared__ int32_t  idx[kSelItems];
  __shared__ uint16_t qd[kMaxBins];
  __shared__ int      nPend;
  __shared__ double   barV;
  __shared__ int32_t  barI;
  const uint32_t q = blockIdx.y;
  if (!a.redo[q]) return;
  const int tid = threadIdx.x, k = a.k;
  for (int j = tid; j < bins; j += kSelThreads) qd[j] = 0;
  for (int i = tid; i < k; i += kSelThreads) val[i] = -1.0, idx[i] = kNoIdx;
  if (tid == 0) {
    nPend = 0;
    barV  = a.values[static_cast<size_t>(q) * k + k - 1];
    barI  = a.indices[static_cast<size_t>(q) * k + k - 1];
    if (blockIdx.x == 0) a.count[q] = gridDim.x * k;
  }
  __syncthreads();
  for (long long p = qr.start[q] + tid; p < qr.start[q + 1]; p += kSelThreads) qd[qr.pairs[p] >> 16] = static_cast<uint16_t>(qr.pairs[p] & 0xffffu);
  __syncthreads();
  const uint32_t per = (colEnd - colBeg + gridDim.x - 1) / gridDim.x;
  const uint32_t c0 = min(colEnd, colBeg + blockIdx.x * per), c1 = min(colEnd, c0 + per);
  const int      sa = qr.sum[q];
  scanBest(val, idx, k, nPend, barV, barI, c0, c1, [&](uint32_t col) {
    int c = 0;
    for (long long p = lib.start[col]; p < lib.start[col + 1]; ++p) {
      const uint32_t v = __ldg(lib.pairs + p);
      c += min(static_cast<int>(qd[v >> 16]), static_cast<int>(v & 0xffffu));
    }
    return measureFromCounts<true>(m, c, sa, lib.sum[col]);
  });
  for (int i = tid; i < k; i += kSelThreads) {
    const size_t at = static_cast<size_t>(q) * a.cap + blockIdx.x * k + i;
    a.candV[at]     = val[i];
    a.candI[at]     = idx[i] == kNoIdx ? kNoCand : static_cast<uint32_t>(idx[i]);
  }
}

// ---- compaction and the checks of every entry point ----

// A group's compact rows (storage of a CountRows)
struct CompactRows {
  Scratch<long long> nnz, start;
  Scratch<int32_t>   sum;
  Scratch<uint32_t>  pairs;
  CountRows          view() const { return {pairs.get(), start.get(), sum.get()}; }
};

// Both groups compacted (b = NULL: one group, used as both), after the range check: the call's one host read. bySum
// (one group only): the rows are compacted in (row sum, index) order, compact row r being the caller's row order[r].
struct CountInputs {
  CompactRows      a, bOwn;
  CountRows        q, lib;
  Scratch<int32_t> order;
  CountInputs(const int32_t* da, size_t nA, const int32_t* db, size_t nB, int bins, cudaStream_t s, bool bySum = false) {
    Scratch<int> bad(1, s);
    B200_CUDA(cudaMemsetAsync(bad.get(), 0, sizeof(int), s));
    long long total[2] = {0, 0};
    int       hBad     = 0;
    auto      stats    = [&](const int32_t* d, const int32_t* perm, size_t n, CompactRows& c, long long* hTotal) {
      c.nnz   = Scratch<long long>(n + 1, s);
      c.start = Scratch<long long>(n + 1, s);
      c.sum   = Scratch<int32_t>(n, s);
      countStatsKernel<<<blocksFor(n, 8), 256, 0, s>>>(d, perm, n, bins, c.sum.get(), c.nnz.get(), bad.get());
      B200_LAUNCHED();
      size_t tmpBytes = 0;
      B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, c.nnz.get(), c.start.get(), static_cast<uint32_t>(n + 1), s));
      Scratch<uint8_t> tmp(tmpBytes, s);
      B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tmpBytes, c.nnz.get(), c.start.get(), static_cast<uint32_t>(n + 1), s));
      g_launchCount.fetch_add(1);
      B200_CUDA(cudaMemcpyAsync(hTotal, c.start.get() + n, sizeof(long long), cudaMemcpyDeviceToHost, s));
    };
    if (bySum) {
      // the sums in the caller's order (their stats are then recomputed in sum order), and a stable radix sort of
      // (sum, index); a count out of range gives a meaningless order, refused below before it is used
      CompactRows first;
      first.nnz = Scratch<long long>(nA + 1, s);
      first.sum = Scratch<int32_t>(nA, s);
      countStatsKernel<<<blocksFor(nA, 8), 256, 0, s>>>(da, nullptr, nA, bins, first.sum.get(), first.nnz.get(), bad.get());
      B200_LAUNCHED();
      Scratch<int32_t> index(nA, s), sorted(nA, s);
      order = Scratch<int32_t>(nA, s);
      iotaKernel<<<blocksFor(nA, 256), 256, 0, s>>>(index.get(), nA);
      B200_LAUNCHED();
      size_t tmpBytes = 0;
      B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, first.sum.get(), sorted.get(), index.get(), order.get(),
                                                static_cast<int>(nA), 0, 32, s));
      Scratch<uint8_t> tmp(tmpBytes, s);
      B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tmpBytes, first.sum.get(), sorted.get(), index.get(), order.get(),
                                                static_cast<int>(nA), 0, 32, s));
      g_launchCount.fetch_add(1);
    }
    stats(da, order.get(), nA, a, &total[0]);
    if (db) stats(db, nullptr, nB, bOwn, &total[1]);
    B200_CUDA(cudaMemcpyAsync(&hBad, bad.get(), sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));  // documented sync: the range check and the list sizes
    B200_REQUIRE(hBad == 0, "a count lies outside 0 .. %d", kMaxCount);
    auto pack = [&](const int32_t* d, const int32_t* perm, size_t n, CompactRows& c, long long nnz) {
      c.pairs = Scratch<uint32_t>(static_cast<size_t>(nnz), s);
      countPackKernel<<<blocksFor(n, 8), 256, 0, s>>>(d, perm, n, bins, c.start.get(), c.pairs.get());
      B200_LAUNCHED();
    };
    pack(da, order.get(), nA, a, total[0]);
    if (db) pack(db, nullptr, nB, bOwn, total[1]);
    q   = a.view();
    lib = db ? bOwn.view() : q;
  }
};

void requireCountInputs(const int32_t* d_a, size_t nA, size_t nB, int bins) {
  B200_REQUIRE(bins >= 1 && bins <= kMaxBins, "count vectors must have 1 to %d bins (got %d)", kMaxBins, bins);
  B200_REQUIRE(nA < (1ull << 31) && nB < (1ull << 31), "too many count vectors");
  B200_REQUIRE(nA == 0 || d_a, "null count-vector pointer");
}

// ---- the neighbour pass's band (see the file header) ----

// Block b of QB rows in sum order: bandEnd[b] = the end of the columns it visits, units[b] = their units of kUnitCols
// (units[nBlocks] = 0, for the scan), and g_countStat[0] += the pairs (row, col > row) in them. A thread per block
// bisects the sorted sums for the first column past the block that its largest sum A cannot reach:
// 1 - value(c = A, a = A, b) <= cutoff fails from there on.
__global__ void countBandKernel(const int32_t* __restrict__ sum, size_t n, int qb, const Measure m, double cutoff,
                                uint32_t* __restrict__ bandEnd, unsigned long long* __restrict__ units) {
  const size_t       nBlocks = (n + qb - 1) / qb;
  unsigned long long pairs   = 0;
  for (size_t b = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; b < nBlocks; b += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t q0 = b * qb, e = min(n, q0 + qb);
    const int    A  = sum[e - 1];
    size_t       lo = e, hi = n;
    while (lo < hi) {
      const size_t mid = (lo + hi) / 2;
      if (__dsub_rn(1.0, tverskyFromCounts(A, A, sum[mid], m.alpha, m.beta)) <= cutoff) lo = mid + 1;
      else hi = mid;
    }
    bandEnd[b] = static_cast<uint32_t>(lo);
    units[b]   = (lo - q0 + kUnitCols - 1) / kUnitCols;
    const unsigned long long nq = e - q0;
    pairs += nq * (nq - 1) / 2 + nq * (lo - e);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) units[nBlocks] = 0;
  for (int o = 16; o; o >>= 1) pairs += __shfl_xor_sync(kFull, pairs, o);
  if ((threadIdx.x & 31) == 0 && pairs) atomicAdd(&g_countStat[0], pairs);
}

// counts[] += the degrees and edges[] the (i < j) pairs, caller's indices, of the neighbour graph of x (an EdgePass),
// after the range check
void countNeighborEdges(const int32_t* d_x, size_t n, int bins, const Measure& m, double cutoff, int32_t* counts, int2* edges,
                        unsigned long long cap, unsigned long long* cursor, cudaStream_t s) {
  resetDeviceCounters(g_countStat, s);
  CountInputs                 in(d_x, n, nullptr, n, bins, s, true);
  const int                   qb      = passQueryRows(bins);
  const size_t                nBlocks = (n + qb - 1) / qb;
  Scratch<uint32_t>           bandEnd(nBlocks, s);
  Scratch<unsigned long long> units(nBlocks + 1, s), unitStart(nBlocks + 1, s);
  countBandKernel<<<blocksFor(nBlocks, 256), 256, 0, s>>>(in.q.sum, n, qb, m, cutoff, bandEnd.get(), units.get());
  B200_LAUNCHED();
  size_t tmpBytes = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, units.get(), unitStart.get(), static_cast<uint32_t>(nBlocks + 1), s));
  Scratch<uint8_t> tmp(tmpBytes, s);
  B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tmpBytes, units.get(), unitStart.get(), static_cast<uint32_t>(nBlocks + 1), s));
  g_launchCount.fetch_add(1);
  PassArgs p;
  p.q = in.q, p.lib = in.lib, p.nQ = n, p.bins = bins, p.measure = m;
  p.cutoff = cutoff, p.perm = in.order.get(), p.degrees = counts, p.list = edges, p.cursor = cursor, p.listCap = cap;
  p.unitStart = unitStart.get(), p.bandEnd = bandEnd.get(), p.nBlocks = nBlocks;
  launchPass<kCountNeighbors>(p, s);
}

EdgePass countEdgePass(const int32_t* d_x, size_t n, int bins, const Measure& m, double cutoff, cudaStream_t s) {
  return [=](int32_t* counts, int2* edges, unsigned long long cap, unsigned long long* cursor) {
    countNeighborEdges(d_x, n, bins, m, cutoff, counts, edges, cap, cursor, s);
  };
}

}  // namespace

unsigned long long readCountStat(int i) { return readDeviceCounter(g_countStat, i); }

}  // namespace b200

using namespace b200;

extern "C" int b200mol_count_cross(const int32_t* d_a, size_t nA, const int32_t* d_b, size_t nB, int bins, double alpha, double beta,
                                   double* d_out, void* stream) {
  return guarded([&] {
    const Measure m = measureOfWeights(alpha, beta);
    if (!d_b) nB = nA;
    requireCountInputs(d_a, nA, nB, bins);
    if (nA == 0 || nB == 0) return;
    B200_REQUIRE(d_out, "null output pointer");
    const cudaStream_t s = asStream(stream);
    CountInputs        in(d_a, nA, d_b, nB, bins, s);
    PassArgs           p;
    p.q = in.q, p.lib = in.lib, p.nQ = nA, p.colBeg = 0, p.colEnd = static_cast<uint32_t>(nB), p.bins = bins, p.measure = m;
    p.out = d_out, p.ld = nB;
    launchPass<kCountMatrix>(p, s);
  });
}

extern "C" int b200mol_count_topk(const int32_t* d_q, size_t nQ, const int32_t* d_lib, size_t nLib, int bins, double alpha, double beta,
                                  int k, double* d_values, int32_t* d_indices, void* stream) {
  return guarded([&] {
    const Measure m = measureOfWeights(alpha, beta);
    if (!d_lib) nLib = nQ;
    requireCountInputs(d_q, nQ, nLib, bins);
    B200_REQUIRE(k >= 1 && static_cast<size_t>(k) <= nLib && k <= kTopkMax, "k must be in [1, min(library size, %d)] (got k = %d, library %zu)",
                 kTopkMax, k, nLib);
    if (nQ == 0) return;
    B200_REQUIRE(d_values && d_indices, "null output pointer");
    const cudaStream_t s = asStream(stream);
    CountInputs        in(d_q, nQ, d_lib, nLib, bins, s);

    // the slots of topk.cu: room for several times the k survivors a doubling slab expects
    const uint32_t    cap = nQ <= 4096 ? kCapMax : static_cast<uint32_t>(std::min(kCapMax, std::max(256, 8 * k)));
    Scratch<double>   candV(nQ * cap, s);
    Scratch<uint32_t> candI(nQ * cap, s), count(nQ, s), redo(nQ, s);
    B200_CUDA(cudaMemsetAsync(count.get(), 0, nQ * sizeof(uint32_t), s));
    B200_CUDA(cudaMemsetAsync(redo.get(), 0, nQ * sizeof(uint32_t), s));
    countTopkInitKernel<<<blocksFor(nQ * k, 256), 256, 0, s>>>(d_values, d_indices, nQ * k);
    B200_LAUNCHED();
    const TopkState st{d_values, d_indices, k, candV.get(), candI.get(), count.get(), redo.get(), cap};
    PassArgs        p;
    p.q = in.q, p.lib = in.lib, p.nQ = nQ, p.bins = bins, p.measure = m;
    p.listV = d_values, p.listI = d_indices, p.k = k, p.candV = candV.get(), p.candI = candI.get(), p.count = count.get(), p.cap = cap;
    // slabs: the first of cap columns (no row can ask for more slots), then each as large as everything before it
    for (size_t done = 0; done < nLib;) {
      const size_t cols = std::min(nLib - done, done == 0 ? static_cast<size_t>(cap) : done);
      p.colBeg = static_cast<uint32_t>(done), p.colEnd = static_cast<uint32_t>(done + cols);
      launchPass<kCountTopk>(p, s);
      countSelectKernel<<<static_cast<unsigned>(nQ), kSelThreads, 0, s>>>(st, 0);
      B200_LAUNCHED();
      // the rows whose candidates did not fit (none, as a rule: the CTAs return at once)
      const unsigned parts = static_cast<unsigned>(std::max<size_t>(1, std::min<size_t>(cap / k, (cols + kSelThreads - 1) / kSelThreads)));
      for (size_t r0 = 0; r0 < nQ; r0 += 65535) {  // (grid.y)
        TopkState sr = st;
        sr.values += r0 * k, sr.indices += r0 * k, sr.candV += r0 * cap, sr.candI += r0 * cap, sr.count += r0, sr.redo += r0;
        CountRows qr = in.q;
        qr.start += r0, qr.sum += r0;
        countScanKernel<<<dim3(parts, static_cast<unsigned>(std::min<size_t>(65535, nQ - r0))), kSelThreads, 0, s>>>(
          sr, qr, in.lib, bins, m, p.colBeg, p.colEnd);
        B200_LAUNCHED();
      }
      countSelectKernel<<<static_cast<unsigned>(nQ), kSelThreads, 0, s>>>(st, 1);
      B200_LAUNCHED();
      done += cols;
    }
  });
}

extern "C" int b200mol_count_threshold(const int32_t* d_q, size_t nQ, const int32_t* d_lib, size_t nLib, int bins, double alpha,
                                       double beta, double threshold, int64_t* d_indptr, int32_t* d_indices, double* d_values,
                                       uint64_t cap, uint64_t* h_nnz, void* stream) {
  return guarded([&] {
    const Measure m = measureOfWeights(alpha, beta);
    B200_REQUIRE(threshold > 0.0 && threshold <= 1.0, "threshold must be in (0, 1] (got %g)", threshold);
    if (!d_lib) nLib = nQ;
    requireCountInputs(d_q, nQ, nLib, bins);
    B200_REQUIRE(h_nnz && d_indptr, "null pointer");
    B200_REQUIRE(cap == 0 || (d_indices && d_values), "null output pointer");
    const cudaStream_t s = asStream(stream);
    *h_nnz               = 0;
    if (nQ == 0 || nLib == 0) {  // no pair: every row is empty
      B200_CUDA(cudaMemsetAsync(d_indptr, 0, (nQ + 1) * sizeof(int64_t), s));
      return;
    }
    CountInputs in(d_q, nQ, d_lib, nLib, bins, s);

    // the list: sized for a result that fits `cap`
    const double             allPairs = static_cast<double>(nQ) * static_cast<double>(nLib);
    const uint64_t           want     = std::min<uint64_t>(cap, 1ull << 27);
    const unsigned long long firstCap = std::max<unsigned long long>(1, static_cast<unsigned long long>(
                                          std::min(allPairs, static_cast<double>(std::max<uint64_t>(1ull << 20, want)))));
    auto listPairs = [&](int2* list, double* vals, unsigned long long listCap, unsigned long long* stat) {
      PassArgs p;
      p.q = in.q, p.lib = in.lib, p.nQ = nQ, p.colBeg = 0, p.colEnd = static_cast<uint32_t>(nLib), p.bins = bins, p.measure = m;
      p.t = threshold, p.list = list, p.vals = vals, p.cursor = stat, p.listCap = listCap;
      launchPass<kCountThreshold>(p, s);
    };
    // the pass lists exactly the result
    thresholdCsr(firstCap, listPairs, [](const unsigned long long* h) { return h[0]; }, false, nullptr, nQ, nLib, m.kind, d_indptr,
                 d_indices, d_values, cap, h_nnz, s);
  });
}

extern "C" int b200mol_count_neighbor_edges(const int32_t* d_x, size_t n, int bins, double alpha, double beta, double cutoff,
                                            int32_t* d_counts, int32_t* d_edges, uint64_t edge_cap, uint64_t* h_n_edges,
                                            void* stream) {
  return guarded([&] {
    const Measure m = measureOfWeights(alpha, beta);
    B200_REQUIRE(m.kind == kTanimoto || m.kind == kDice,
                 "count neighbours take Tanimoto (1, 1) or Dice (0.5, 0.5) weights (got alpha = %g, beta = %g)", alpha, beta);
    B200_REQUIRE(cutoff >= 0.0 && cutoff <= 1.0, "cutoff must be in [0, 1], got %g", cutoff);
    requireCountInputs(d_x, n, n, bins);
    const cudaStream_t s = asStream(stream);
    if (h_n_edges) *h_n_edges = 0;
    if (n == 0) return;
    B200_REQUIRE(d_counts && (d_edges || edge_cap == 0), "null pointer");
    edgePassWithTotal(countEdgePass(d_x, n, bins, m, cutoff, s), d_counts, reinterpret_cast<int2*>(d_edges), edge_cap, h_n_edges, s);
  });
}

extern "C" int b200mol_count_butina_fused(const int32_t* d_x, size_t n, int bins, double alpha, double beta, double cutoff,
                                          int32_t* d_cluster_ids, int32_t* d_centroids, int32_t* d_n_clusters,
                                          int32_t* h_n_clusters, void* stream) {
  return guarded([&] {
    const Measure m = measureOfWeights(alpha, beta);  // (checked first, as b200mol_count_neighbor_edges does)
    B200_REQUIRE(m.kind == kTanimoto || m.kind == kDice,
                 "count neighbours take Tanimoto (1, 1) or Dice (0.5, 0.5) weights (got alpha = %g, beta = %g)", alpha, beta);
    B200_REQUIRE(cutoff >= 0.0 && cutoff <= 1.0, "cutoff must be in [0, 1], got %g", cutoff);
    requireCountInputs(d_x, n, n, bins);
    const cudaStream_t s = asStream(stream);
    if (n == 0) return noClusters(d_n_clusters, h_n_clusters, s);
    B200_REQUIRE(d_cluster_ids, "null pointer");
    fusedButina(n, countEdgePass(d_x, n, bins, m, cutoff, s), d_cluster_ids, d_centroids, d_n_clusters, h_n_clusters, s);
  });
}
