// Leader (sphere-exclusion) diversity picking on packed fingerprints (RDKit LeaderPicker::lazyPick): b200mol_leader_pick.
//
// Contract. d(i, j) = 1 - s(i, j), s the fp64 value b200mol_tanimoto_cross / b200mol_cosine_cross store for the pair
// (simFromCounts: 0 for an empty intersection). Item j is covered by pick p iff 1.0 - s(p, j) <= threshold: the
// neighbour predicate of the thresholded count pass with cutoff = threshold. Picks start with the caller's first picks, in
// order; every pool item that is a first pick or is covered by one leaves the pool; then, repeatedly, the lowest-index
// item still in the pool becomes a pick, and it and every item it covers leave the pool, until the pool is empty or there
// are pickSize picks. Equivalently: item i is a further pick iff it is no first pick, no first pick covers it, and no
// further pick of lower index covers it. So further picks come out in ascending index order.
//
// Host loop over windows [lo, hi) of the pool, in index order. A device leader buffer holds the fingerprints and
// popcounts of every pick so far, contiguous (it starts as the first picks). Per window:
//   bulk     one call of the cross count pass (launchSimilarity, kCount, X = the window, Y = the
//            leader buffer, cutoff = threshold; SIMT or the wgmma u8 tile as that pass decides) counts, per item, the
//            picks so far that cover it;
//   select   the survivors, items with count 0 that are no first pick, compacted in index order (flags, an in-place
//            exclusive scan, a scatter);
//   resolve  one cooperative kernel over blocks of kBlock survivors. Per block:
//            (a) all CTAs test the block's items against the picks made earlier in this window (32 x 32 tiles);
//            (b) after a grid barrier, all CTAs compute the lower-triangular cover mask of the block's items that (a)
//                left: bit l of row k set iff item l (l < k) covers item k;
//            (c) after a grid barrier, one warp of CTA 0 walks the rows in order: row k is a pick iff
//                row_k & pickedMask == 0; CTA 0 appends the picks' indices, fingerprints and popcounts to the leader
//                buffer, and stops at pickSize;
//   the host reads the survivor and pick counts (one synchronisation per window) and sizes the next window so that
//   about kTargetSurvivors survive it (option "leader_window_rows" > 0 fixes the window instead).
//
// Why it is exact. Take a survivor i of window w that is no first pick. Every pick p of lower index than i is either a
// first pick or a further pick; all first picks and all further picks before window w were in the leader buffer for the
// bulk pass of window w, so the count pass tested i against them; further picks in window w before i's block were tested
// in (a); further picks in i's block before i are rows l < k of the mask, tested in (b), and (c) applies exactly those
// of them that were picked. So i is tested against every earlier pick exactly once, with the count pass's own predicate
// (for Tanimoto the pass tests c >= thresh[|A| + |B|], the smallest c with 1.0 - c / (|A| + |B| - c) <= cutoff in fp64;
// (a) and (b) evaluate that same fp64 expression through simFromCounts, which is the same quotient for c > 0 and 0 for
// c = 0, as the table's). An item that is covered in the bulk pass or in (a) is no pick and needs no row; an item that is
// a first pick is excluded in the selection. The walk in (c) visits items in index order and the picks of a block are
// final before the next block's (a) starts (grid barrier). A pick always leaves the pool explicitly, so two empty
// fingerprints (distance 1) are never picked twice even at thresholds below 1.
//
// Determinism. The scan is sequential in one warp, every CTA agrees on the pick count through barriers, and the (a)
// verdicts are plain stores of 1, so no atomic decides anything: picks are bitwise repeatable. The only atomics add up
// the read-only pair counters.
//
// Popcount skip in (a) and (b): lb = 1 - s(min(|A|, |B|), |A|, |B|) <= d(A, B) by the argument of maxmin.cu's header, so
// a pair with lb > threshold cannot cover and its fingerprints are not compared.
#include <cooperative_groups.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>
#include <vector>

#include "options.cuh"
#include "similarity.cuh"

namespace cg = cooperative_groups;

namespace b200 {

long long          g_leaderWindowRows     = 0;  // option "leader_window_rows": 0 automatic, > 0 fixed window size
long long          g_leaderWindowsLast    = 0;  // windows the last call walked ("leader_windows_last")
unsigned long long g_leaderBulkPairsLast  = 0;  // window x leader pairs sent through the count pass ("leader_bulk_pairs_last")

namespace {

constexpr int kThreads         = 512;
constexpr int kWarps           = kThreads / 32;
constexpr int kBlock           = 1024;         // survivors per resolver block
constexpr int kMaskWords       = kBlock / 32;  // words of one cover-mask row
constexpr int kTile            = 32;           // tile rows / columns in (a) and (b)
constexpr int kTargetSurvivors = 8 * kBlock;   // survivors a window is sized for
constexpr int kMaxWindow       = 1 << 18;      // rows of an automatic window at most

__device__ unsigned long long g_leaderStat[2];  // pairs compared in (a), in (b)

struct ResolveArgs {
  const uint4*   fp;   // [n][chunks] the pool
  const int32_t* pop;  // [n]
  int            chunks;
  bool           cosine;
  double         threshold;
  const int32_t* surv;   // window survivors, pool indices ascending
  const int32_t* count;  // [0] survivors (written by the selection), [1] picks so far
  int32_t*       nPicks;  // = count + 1, advanced by CTA 0
  int            pickSize;
  int32_t*       picks;      // [pickSize]
  uint4*         leaders;    // [capacity][chunks] pick fingerprints
  int32_t*       leaderPop;  // [capacity]
  uint8_t*       covered;    // [kBlock] (a)'s verdicts, all zero between blocks
  uint32_t*      mask;       // [kBlock][kMaskWords]
};

__device__ __forceinline__ int popAnd(uint4 x, uint4 y) {
  return __popc(x.x & y.x) + __popc(x.y & y.y) + __popc(x.z & y.z) + __popc(x.w & y.w);
}
__device__ __forceinline__ double distance(int c, int a, int b, bool cosine) { return __dsub_rn(1.0, simFromCounts(c, a, b, cosine)); }

struct TileSmem {
  uint4*    rows;  // [kTile][stride]
  uint4*    cols;
  int       stride;
  int*      rowPop;  // [kTile]
  int*      colPop;
  uint32_t* colBits;  // [kTile]: bit r = row r is covered by column c
  uint32_t* rowWord;  // [kTile]: bit c = column c covers row r
};

// One 32 x 32 tile of cover bits. rowSrc(r) / colSrc(c): the fingerprint's address (null = no such row / column);
// rowPopOf / colPopOf: its popcount. lowerOnly: only pairs with c < r count (the diagonal tile of the mask). Leaves
// t.rowWord[r] in shared memory; the whole CTA calls it.
template <class RowSrc, class ColSrc, class RowPop, class ColPop>
__device__ void coverTile(const ResolveArgs& a, const TileSmem& t, RowSrc rowSrc, ColSrc colSrc, RowPop rowPopOf,
                          ColPop colPopOf, bool lowerOnly, unsigned long long& compared) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __syncthreads();  // (the previous tile may still be read)
  for (int idx = tid; idx < 2 * kTile * a.chunks; idx += kThreads) {
    const int    side = idx / (kTile * a.chunks), rem = idx % (kTile * a.chunks), r = rem / a.chunks, w = rem % a.chunks;
    const uint4* src  = side ? colSrc(r) : rowSrc(r);
    (side ? t.cols : t.rows)[r * t.stride + w] = src ? __ldcg(src + w) : make_uint4(0, 0, 0, 0);
  }
  if (tid < kTile) t.rowPop[tid] = rowSrc(tid) ? rowPopOf(tid) : -1;
  else if (tid < 2 * kTile) t.colPop[tid - kTile] = colSrc(tid - kTile) ? colPopOf(tid - kTile) : -1;
  __syncthreads();
  const int pa = t.rowPop[lane];
  for (int c = warp; c < kTile; c += kWarps) {
    const int pb  = t.colPop[c];
    bool      hit = false;
    if (pa >= 0 && pb >= 0 && (!lowerOnly || c < lane) && !(distance(min(pa, pb), pa, pb, a.cosine) > a.threshold)) {
      int n = 0;
      for (int q = 0; q < a.chunks; ++q) n += popAnd(t.rows[lane * t.stride + q], t.cols[c * t.stride + q]);
      hit = distance(n, pa, pb, a.cosine) <= a.threshold;
      ++compared;
    }
    const unsigned bits = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) t.colBits[c] = bits;
  }
  __syncthreads();
  if (tid < kTile) {
    uint32_t w = 0;
    for (int c = 0; c < kTile; ++c) w |= ((t.colBits[c] >> tid) & 1u) << c;
    t.rowWord[tid] = w;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) resolveKernel(const ResolveArgs a) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) unsigned char smem[];  // tile operands; in CTA 0 during (c), the block's cover mask
  __shared__ int      sList[kBlock];                     // block positions of the items (a) left, in order
  __shared__ int      sPick[kBlock];                     // (c): compact positions of the block's picks
  __shared__ int      sWarp[kWarps + 1];
  __shared__ int      sRowPop[kTile], sColPop[kTile];
  __shared__ uint32_t sColBits[kTile], sRowWord[kTile];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  TileSmem  t;
  t.stride  = a.chunks | 1;  // odd: the 32 rows of a column step fall in distinct 16-byte bank groups
  t.rows    = reinterpret_cast<uint4*>(smem);
  t.cols    = t.rows + kTile * t.stride;
  t.rowPop = sRowPop, t.colPop = sColPop, t.colBits = sColBits, t.rowWord = sRowWord;
  uint32_t* sMask = reinterpret_cast<uint32_t*>(smem);

  const int nSurv = __ldcg(a.count), winStart = __ldcg(a.count + 1);
  int       np    = winStart;  // picks so far: the same value in every CTA
  unsigned long long comparedA = 0, comparedB = 0;

  for (int base = 0; base < nSurv && np < a.pickSize; base += kBlock) {
    const int      nb   = min(kBlock, nSurv - base);
    const int32_t* item = a.surv + base;
    // (a) the block's items against this window's earlier picks, leaders[winStart, np)
    if (np > winStart) {
      const int rowTiles = (nb + kTile - 1) / kTile, colTiles = (np - winStart + kTile - 1) / kTile;
      for (int u = blockIdx.x; u < rowTiles * colTiles; u += gridDim.x) {
        const int r0 = (u / colTiles) * kTile, c0 = winStart + (u % colTiles) * kTile;
        coverTile(
          a, t, [&](int r) { return r0 + r < nb ? a.fp + static_cast<size_t>(__ldg(item + r0 + r)) * a.chunks : nullptr; },
          [&](int c) { return c0 + c < np ? a.leaders + static_cast<size_t>(c0 + c) * a.chunks : nullptr; },
          [&](int r) { return __ldg(a.pop + __ldg(item + r0 + r)); }, [&](int c) { return __ldcg(a.leaderPop + c0 + c); },
          false, comparedA);
        if (tid < kTile && t.rowWord[tid]) a.covered[r0 + tid] = 1;
      }
      grid.sync();
    }
    // every CTA lists the items (a) left, in order
    int m = 0;
    for (int k0 = 0; k0 < nb; k0 += kThreads) {
      const int      k    = k0 + tid;
      const bool     keep = k < nb && !__ldcg(a.covered + k);
      const unsigned bal  = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) sWarp[warp] = __popc(bal);
      __syncthreads();
      if (tid == 0) {
        int s = m;
        for (int w = 0; w < kWarps; ++w) {
          const int c = sWarp[w];
          sWarp[w]    = s;
          s += c;
        }
        sWarp[kWarps] = s;
      }
      __syncthreads();
      if (keep) sList[sWarp[warp] + __popc(bal & ((1u << lane) - 1u))] = k;
      m = sWarp[kWarps];
      __syncthreads();
    }
    // (b) the lower-triangular cover mask of those items
    {
      const int T = (m + kTile - 1) / kTile;
      for (int u = blockIdx.x; u < T * (T + 1) / 2; u += gridDim.x) {
        int rt = static_cast<int>((sqrtf(8.0f * u + 1.0f) - 1.0f) * 0.5f);
        while (rt * (rt + 1) / 2 > u) --rt;
        while ((rt + 1) * (rt + 2) / 2 <= u) ++rt;
        const int ct = u - rt * (rt + 1) / 2, r0 = rt * kTile, c0 = ct * kTile;
        auto      at = [&](int k) { return a.fp + static_cast<size_t>(__ldg(item + sList[k])) * a.chunks; };
        coverTile(
          a, t, [&](int r) { return r0 + r < m ? at(r0 + r) : nullptr; }, [&](int c) { return c0 + c < m ? at(c0 + c) : nullptr; },
          [&](int r) { return __ldg(a.pop + __ldg(item + sList[r0 + r])); },
          [&](int c) { return __ldg(a.pop + __ldg(item + sList[c0 + c])); }, ct == rt, comparedB);
        if (tid < kTile && r0 + tid < m) a.mask[static_cast<size_t>(r0 + tid) * kMaskWords + ct] = t.rowWord[tid];
      }
    }
    grid.sync();
    // (c) the greedy walk, in one warp of CTA 0
    if (blockIdx.x == 0) {
      for (int idx = tid; idx < m * kMaskWords; idx += kThreads)
        if ((idx % kMaskWords) <= (idx / kMaskWords) / 32) sMask[idx] = __ldcg(a.mask + idx);
      for (int k = tid; k < nb; k += kThreads) a.covered[k] = 0;  // (every CTA has read the verdicts: barrier above)
      __syncthreads();
      if (warp == 0) {
        const int room   = a.pickSize - np;
        uint32_t  picked = 0;  // lane w: word w of the block's picked set
        int       cnt    = 0;
        for (int k = 0; k < m && cnt < room; ++k) {
          const uint32_t row = lane <= (k >> 5) ? sMask[k * kMaskWords + lane] : 0u;
          if (!__any_sync(0xffffffffu, row & picked)) {
            if (lane == (k >> 5)) picked |= 1u << (k & 31);
            if (lane == 0) sPick[cnt] = k;
            ++cnt;
          }
        }
        if (lane == 0) sWarp[0] = cnt;
      }
      __syncthreads();
      const int cnt = sWarp[0];
      for (int q = tid; q < cnt; q += kThreads) {
        const int i = __ldg(item + sList[sPick[q]]);
        a.picks[np + q] = i, a.leaderPop[np + q] = __ldg(a.pop + i);
      }
      for (int idx = tid; idx < cnt * a.chunks; idx += kThreads) {
        const int q = idx / a.chunks, w = idx % a.chunks, i = __ldg(item + sList[sPick[q]]);
        a.leaders[static_cast<size_t>(np + q) * a.chunks + w] = __ldg(a.fp + static_cast<size_t>(i) * a.chunks + w);
      }
      if (tid == 0) *a.nPicks = np + cnt;
    }
    grid.sync();
    np = __ldcg(a.nPicks);
  }
  for (int o = 16; o; o >>= 1) comparedA += __shfl_xor_sync(0xffffffffu, comparedA, o), comparedB += __shfl_xor_sync(0xffffffffu, comparedB, o);
  if (lane == 0 && (comparedA | comparedB)) atomicAdd(&g_leaderStat[0], comparedA), atomicAdd(&g_leaderStat[1], comparedB);
}

// leaders[k] = fp[idx[k]], leaderPop[k] = pop[idx[k]], isFirst[idx[k]] = 1
__global__ void gatherFirstKernel(const uint4* __restrict__ fp, const int32_t* __restrict__ pop, int chunks, const int32_t* __restrict__ idx,
                                  int n, uint4* __restrict__ leaders, int32_t* __restrict__ leaderPop, uint8_t* __restrict__ isFirst) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * chunks) return;
  const int k = t / chunks, w = t % chunks, i = idx[k];
  leaders[static_cast<size_t>(k) * chunks + w] = fp[static_cast<size_t>(i) * chunks + w];
  if (w == 0) leaderPop[k] = pop[i], isFirst[i] = 1;
}

// flag[k] = 1 iff window item lo + k survives the bulk pass and is no first pick (in place over its count); flag[rows] = 0
__global__ void survivorFlagKernel(int32_t* __restrict__ flag, const uint8_t* __restrict__ isFirst, int lo, int rows) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < rows) flag[k] = flag[k] == 0 && !isFirst[lo + k];
  else if (k == rows) flag[k] = 0;
}

// pos = the exclusive scan of the flags (rows + 1 entries): surv[pos[k]] = lo + k for the flagged k; count[0] = survivors
__global__ void survivorScatterKernel(const int32_t* __restrict__ pos, int lo, int rows, int32_t* __restrict__ surv, int32_t* count) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < rows && pos[k + 1] > pos[k]) surv[pos[k]] = lo + k;
  else if (k == rows) count[0] = pos[rows];
}

size_t resolveSmem(int chunks) {
  const size_t tiles = 2 * static_cast<size_t>(kTile) * (chunks | 1) * 16, mask = static_cast<size_t>(kBlock) * kMaskWords * 4;
  return std::max(tiles, mask);
}

}  // namespace

unsigned long long readLeaderStat(int i) { return readDeviceCounter(g_leaderStat, i); }

}  // namespace b200

using namespace b200;

extern "C" int b200mol_leader_pick(const uint32_t* d_fp, size_t nPool, int words, int metric, double threshold,
                                   const int32_t* h_first, int nFirst, int pickSize, int32_t* d_picks, int32_t* h_n_picks,
                                   void* stream) {
  return guarded([&] {
    const Measure m = measureOfMetric(metric);
    requireFingerprintWidth(words);
    B200_REQUIRE(nPool >= 1 && nPool < (1ull << 31), "pool size must be in [1, 2^31) (got %zu)", nPool);
    B200_REQUIRE(pickSize >= 1 && static_cast<size_t>(pickSize) <= nPool, "pickSize must be in [1, pool size] (got %d, pool %zu)",
                 pickSize, nPool);
    B200_REQUIRE(threshold >= 0.0 && threshold <= 1.0, "threshold must be in [0, 1] (got %g)", threshold);
    B200_REQUIRE(nFirst >= 0 && nFirst <= pickSize, "need 0 <= first picks <= pickSize (got %d, pickSize %d)", nFirst, pickSize);
    B200_REQUIRE(d_fp && d_picks && h_n_picks && (nFirst == 0 || h_first), "null pointer");
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
    const bool   fixed = g_leaderWindowRows > 0;
    const int    maxWindow = static_cast<int>(std::min<long long>(n, fixed ? g_leaderWindowRows : kMaxWindow));
    g_leaderWindowsLast = 0, g_leaderBulkPairsLast = 0;
    resetDeviceCounters(g_leaderStat, s);

    Scratch<int32_t> pop(nPool, s), counts(static_cast<size_t>(maxWindow) + 1, s), surv(maxWindow, s), count(2, s);
    Scratch<uint8_t> isFirst(nPool, s), covered(kBlock, s);
    Scratch<uint32_t> mask(static_cast<size_t>(kBlock) * kMaskWords, s);
    launchRowPopcount(d_fp, nPool, words, pop.get(), s);
    B200_CUDA(cudaMemsetAsync(isFirst.get(), 0, nPool, s));
    B200_CUDA(cudaMemsetAsync(covered.get(), 0, kBlock, s));
    const int32_t startCount[2] = {0, nFirst};
    B200_CUDA(cudaMemcpyAsync(count.get(), startCount, sizeof(startCount), cudaMemcpyHostToDevice, s));

    // the leader buffer grows by doubling; it never needs more than pickSize rows
    size_t           cap = std::min<size_t>(pickSize, std::max<size_t>(nFirst, 4096));
    Scratch<uint4>   leaders(cap * chunks, s);
    Scratch<int32_t> leaderPop(cap, s);
    if (nFirst > 0) {
      B200_CUDA(cudaMemcpyAsync(d_picks, h_first, sizeof(int32_t) * nFirst, cudaMemcpyHostToDevice, s));
      gatherFirstKernel<<<(nFirst * chunks + 255) / 256, 256, 0, s>>>(reinterpret_cast<const uint4*>(d_fp), pop.get(), chunks, d_picks,
                                                                     nFirst, leaders.get(), leaderPop.get(), isFirst.get());
      B200_LAUNCHED();
    }

    // the selection's scan scratch, sized once for the largest window
    size_t tempBytes = 0;
    B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tempBytes, counts.get(), counts.get(), maxWindow + 1, s));
    Scratch<unsigned char> temp(tempBytes, s);

    const size_t smemBytes = resolveSmem(chunks);
    B200_CUDA(cudaFuncSetAttribute(resolveKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smemBytes)));
    int perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, resolveKernel, kThreads, smemBytes));
    B200_REQUIRE(perSm >= 1, "leader resolve kernel does not fit on an SM");
    const int blocks = smCount();

    ResolveArgs ra{};
    ra.fp = reinterpret_cast<const uint4*>(d_fp), ra.pop = pop.get(), ra.chunks = chunks;
    ra.cosine = m.kind == kCosine, ra.threshold = threshold;
    ra.surv = surv.get(), ra.count = count.get(), ra.nPicks = count.get() + 1, ra.pickSize = pickSize, ra.picks = d_picks;
    ra.covered = covered.get(), ra.mask = mask.get();

    int    nPicks = nFirst;
    size_t lo     = 0;
    int    window = fixed ? maxWindow : std::min(n, kTargetSurvivors);
    while (lo < nPool && nPicks < pickSize) {
      const int rows = static_cast<int>(std::min<size_t>(window, nPool - lo));
      // room for every survivor of this window to become a pick
      const size_t need = std::min<size_t>(pickSize, static_cast<size_t>(nPicks) + rows);
      if (need > cap) {
        const size_t     grown = std::min<size_t>(pickSize, std::max(need, 2 * cap));
        Scratch<uint4>   l2(grown * chunks, s);
        Scratch<int32_t> p2(grown, s);
        if (nPicks > 0) {
          B200_CUDA(cudaMemcpyAsync(l2.get(), leaders.get(), sizeof(uint4) * nPicks * chunks, cudaMemcpyDeviceToDevice, s));
          B200_CUDA(cudaMemcpyAsync(p2.get(), leaderPop.get(), sizeof(int32_t) * nPicks, cudaMemcpyDeviceToDevice, s));
        }
        leaders = std::move(l2), leaderPop = std::move(p2), cap = grown;
      }
      B200_CUDA(cudaMemsetAsync(counts.get(), 0, sizeof(int32_t) * rows, s));
      if (nPicks > 0) {
        SimLaunch q;
        q.x = d_fp + lo * words, q.nX = rows;
        q.y = reinterpret_cast<const uint32_t*>(leaders.get()), q.nY = static_cast<size_t>(nPicks);
        q.words = words, q.measure = m, q.cutoff = threshold, q.sign = 1, q.rowCounts = counts.get();
        launchSimilarity(kCount, q, s);
        g_leaderBulkPairsLast += static_cast<unsigned long long>(rows) * static_cast<unsigned long long>(nPicks);
      }
      const unsigned selGrid = static_cast<unsigned>((rows + 1 + 255) / 256);
      survivorFlagKernel<<<selGrid, 256, 0, s>>>(counts.get(), isFirst.get(), static_cast<int>(lo), rows);
      B200_LAUNCHED();
      B200_CUDA(cub::DeviceScan::ExclusiveSum(temp.get(), tempBytes, counts.get(), counts.get(), rows + 1, s));
      survivorScatterKernel<<<selGrid, 256, 0, s>>>(counts.get(), static_cast<int>(lo), rows, surv.get(), count.get());
      B200_LAUNCHED();
      ra.leaders = leaders.get(), ra.leaderPop = leaderPop.get();
      void* args[] = {&ra};
      B200_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(resolveKernel), dim3(blocks), dim3(kThreads), args, smemBytes, s));
      B200_LAUNCHED();
      int32_t got[2];
      B200_CUDA(cudaMemcpyAsync(got, count.get(), sizeof(got), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
      nPicks = got[1];
      lo += rows;
      ++g_leaderWindowsLast;
      if (!fixed) {  // the next window: about kTargetSurvivors survivors at this window's survivor fraction
        // (at most 8 times the last window, at least one resolver block)
        const double next = static_cast<double>(kTargetSurvivors) * rows / std::max(1, got[0]);
        window            = static_cast<int>(std::max<double>(kBlock, std::min({next, 8.0 * rows, static_cast<double>(maxWindow)})));
      }
    }
    *h_n_picks = nPicks;
  });
}
