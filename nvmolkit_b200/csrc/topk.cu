// Exact top-k similarity search: for each query fingerprint the k most similar library fingerprints, ordered by
// (value descending, library index ascending), without the Q x M matrix. b200mol_similarity_topk.
//
// The order is total (no two columns of a row share a key), so the k best of a row are ONE set in ONE order: whatever
// path finds them, in whatever order atomics land, the result is the same bits.
//
//   state      the caller's outputs values[Q][k] / indices[Q][k] are the running lists (sorted), bar[q] the key of row q's
//              current k-th best, cand[Q][cap] column indices waiting to be merged
//   scan       topkScanKernel, SIMT: a CTA takes one query and one part of a column range, a thread one column (AND +
//              POPC over the row, the query in shared memory); what beats the bar is parked in shared memory and, when
//              that fills up, sorted and cut to k, which raises the CTA's bar. Nothing can overflow: it leaves its k
//              best in cand. This is the whole search for small inputs, the warm-up of the bars for large ones, and the
//              redo of the rows whose candidates did not fit
//   tile       launchTopkTile (tanimoto_tc.cu): the wgmma u8 tile of the pair pass over an expanded column slab, with an
//              epilogue that lists the columns whose pair could beat the row's bar
//   select     topkSelectKernel, a CTA per query: re-counts the row's candidates exactly, sorts them with the running
//              list by the key (a bitonic network in shared memory), keeps k, and raises the bar
//
// Large inputs: the bars are warmed on the first kWarmCols columns by the scan; the rest of the library goes through the
// tile in slabs that double (each as large as everything before it, up to 512 MB of expanded operand), so that in a
// library in random order a row expects about k survivors per slab. A row with more survivors than slots merges none of
// them: it is marked, the scan redoes the slab for the marked rows, and the select merges that. The call never reads
// anything back, so all of it is enqueued unconditionally and the redo kernels return at once for unmarked rows.
#include <algorithm>

#include "options.cuh"
#include "similarity.cuh"
#include "topk.cuh"

namespace b200 {

long long          g_topkSlabCols = 0;  // option "topk_slab_cols": columns per slab (and of the warm-up); 0 = automatic
unsigned long long g_topkSlabsLast = 0;  // slabs the last call ran through the tensor tile ("topk_slabs_last")

namespace {

constexpr int kWarmCols   = 4096;  // columns of the warm-up scan (>= kTopkMax: every list is full after it)
static_assert(kWarmCols >= kTopkMax && kCapMax >= kTopkMax, "the warm-up fills the lists; a part's k best fit the slots");

__device__ unsigned long long g_topkStat[2];  // [0] candidates the tile passes listed, [1] rows redone by the scan

struct TopkArgs {
  const uint32_t *q, *lib;  // [nQ][words], [nLib][words]
  const int32_t * popQ, *popLib;
  int             words, k;
  Measure         measure;  // Tanimoto, cosine or Tversky (a Dice search is Tanimoto's)
  double*         values;   // [nQ][k] the running lists
  int32_t*        indices;  // [nQ][k]
  int4*           bar;      // [nQ] {c, |A| + |B|, column, float bits of a lower bound of the value} of the k-th best
  uint32_t*       cand;     // [nQ][cap]
  uint32_t*       count;    // [nQ] candidate slots in use
  uint32_t*       redo;     // [nQ] 1: the row's candidates of this slab did not fit
  uint32_t        cap;
};

// Grid (parts, queries). Columns [colBeg, colEnd) in `parts` equal ranges; the CTA's k best of its range (fewer if the
// bar lets fewer through) go to cand[q][part * k ..], padded with kNoCand. listValid: the row's list holds k entries and
// its last one is a bar to start from. onlyRedo: rows not marked are left alone.
template <bool WEIGHTED>
__global__ void __launch_bounds__(kSelThreads) topkScanKernel(const TopkArgs a, uint32_t colBeg, uint32_t colEnd, int listValid, int onlyRedo) {
  __shared__ double   val[kSelItems];
  __shared__ int32_t  idx[kSelItems];
  __shared__ __align__(16) uint32_t sq[128];
  __shared__ int      nPend;
  __shared__ double   barV;
  __shared__ int32_t  barI;
  const uint32_t q = blockIdx.y;
  if (onlyRedo && !a.redo[q]) return;
  const int tid = threadIdx.x, k = a.k;
  for (int w = tid; w < a.words; w += kSelThreads) sq[w] = a.q[static_cast<size_t>(q) * a.words + w];
  for (int i = tid; i < k; i += kSelThreads) val[i] = -1.0, idx[i] = kNoIdx;  // this CTA's list starts empty
  if (tid == 0) {
    nPend = 0;
    barV  = listValid ? a.values[static_cast<size_t>(q) * k + k - 1] : -1.0;
    barI  = listValid ? a.indices[static_cast<size_t>(q) * k + k - 1] : kNoIdx;
    if (blockIdx.x == 0) a.count[q] = gridDim.x * k;
  }
  __syncthreads();
  const uint32_t per = (colEnd - colBeg + gridDim.x - 1) / gridDim.x;
  const uint32_t c0 = min(colEnd, colBeg + blockIdx.x * per), c1 = min(colEnd, c0 + per);
  const int      pa = a.popQ[q], chunks = a.words / 4;
  scanBest(val, idx, k, nPend, barV, barI, c0, c1, [&](uint32_t col) {
    const uint4* row = reinterpret_cast<const uint4*>(a.lib + static_cast<size_t>(col) * a.words);
    int          c   = 0;
    for (int w = 0; w < chunks; ++w) {
      const uint4 y = __ldg(row + w), x = reinterpret_cast<const uint4*>(sq)[w];
      c += __popc(x.x & y.x) + __popc(x.y & y.y) + __popc(x.z & y.z) + __popc(x.w & y.w);
    }
    return measureFromCounts<WEIGHTED>(a.measure, c, pa, a.popLib[col]);
  });
  for (int i = tid; i < k; i += kSelThreads)
    a.cand[static_cast<size_t>(q) * a.cap + blockIdx.x * k + i] = idx[i] == kNoIdx ? kNoCand : static_cast<uint32_t>(idx[i]);
}

// One CTA per query: the row's candidates (columns not in its list: a slab the list has not seen, or the parts of a scan)
// are re-counted exactly, sorted together with the list by the contract's key, and the k best become the list.
// afterScan = 0, after a tile pass: a row that asked for more slots than there are merges nothing and is marked for the
// scan. afterScan = 1: the slots hold the scan's results; with onlyRedo, of the marked rows only.
template <bool WEIGHTED>
__global__ void __launch_bounds__(kSelThreads) topkSelectKernel(const TopkArgs a, int listValid, int afterScan, int onlyRedo) {
  __shared__ double  val[kSelItems];
  __shared__ int32_t idx[kSelItems];
  const uint32_t q = blockIdx.x;
  const int      tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, k = a.k;
  const uint32_t asked = a.count[q];
  if (afterScan) {
    if (onlyRedo && !a.redo[q]) return;
  } else {
    const bool fits = asked <= a.cap;
    __syncthreads();  // (every thread has read count[q] and redo[q] before thread 0 rewrites them)
    if (tid == 0) {
      a.redo[q] = fits ? 0u : 1u;
      atomicAdd(&g_topkStat[0], static_cast<unsigned long long>(asked));
      if (!fits) atomicAdd(&g_topkStat[1], 1ull);
    }
    if (!fits) return;
  }
  __syncthreads();
  if (tid == 0) a.count[q] = 0;  // the slots are free for the next pass
  const int n = static_cast<int>(asked);
  if (n == 0 && listValid) return;
  const int have = listValid ? k : 0;
  for (int i = tid; i < have; i += kSelThreads) val[i] = a.values[static_cast<size_t>(q) * k + i], idx[i] = a.indices[static_cast<size_t>(q) * k + i];
  const uint32_t* qrow = a.q + static_cast<size_t>(q) * a.words;
  const int       pa   = a.popQ[q];
  auto countWith = [&](uint32_t col) {  // |query & library[col]|, by one warp
    const uint32_t* row = a.lib + static_cast<size_t>(col) * a.words;
    int             c   = 0;
    for (int w = lane; w < a.words; w += 32) c += __popc(qrow[w] & __ldg(row + w));
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    return c;
  };
  for (int j = warp; j < n; j += kSelThreads / 32) {
    const uint32_t col = a.cand[static_cast<size_t>(q) * a.cap + j];
    double         v   = -1.0;
    if (col != kNoCand) v = measureFromCounts<WEIGHTED>(a.measure, countWith(col), pa, a.popLib[col]);
    if (lane == 0) val[have + j] = v, idx[have + j] = col == kNoCand ? kNoIdx : static_cast<int32_t>(col);
  }
  const int n2 = nextPow2(have + n);
  for (int i = have + n + tid; i < n2; i += kSelThreads) val[i] = -1.0, idx[i] = kNoIdx;
  sortBestFirst(val, idx, n2);
  for (int i = tid; i < k; i += kSelThreads) a.values[static_cast<size_t>(q) * k + i] = val[i], a.indices[static_cast<size_t>(q) * k + i] = idx[i];
  if (warp == 0) {  // the bar the tile filters with: the k-th best as integers, and its value rounded down with a margin
    const uint32_t col = static_cast<uint32_t>(idx[k - 1]);
    const int      c   = countWith(col);
    if (lane == 0) {
      float lo = __double2float_rd(val[k - 1]);
      lo       = __fmul_rd(lo, 1.0f - 3.0e-5f);
      a.bar[q] = make_int4(c, pa + a.popLib[col], static_cast<int>(col), __float_as_int(lo));
    }
  }
}

// Dice values of a finished Tanimoto search: entry (q, i) of the lists re-counted (one warp each) and stored as
// tverskyFromCounts(c, |A|, |B|; 1/2, 1/2); the indices stay as they are.
__global__ void __launch_bounds__(256) topkDiceValuesKernel(const uint32_t* __restrict__ q, const uint32_t* __restrict__ lib, int words,
                                                            const int32_t* __restrict__ popQ, const int32_t* __restrict__ popLib,
                                                            size_t nQ, int k, const int32_t* __restrict__ indices, double* values) {
  const int          lane = threadIdx.x & 31;
  const size_t       n = nQ * static_cast<size_t>(k), step = static_cast<size_t>(gridDim.x) * (blockDim.x / 32);
  for (size_t e = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32; e < n; e += step) {
    const size_t    row = e / k;
    const int32_t   col = indices[e];
    const uint32_t* x = q + row * words;
    const uint32_t* y = lib + static_cast<size_t>(col) * words;
    int             c = 0;
    for (int w = lane; w < words; w += 32) c += __popc(x[w] & y[w]);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) values[e] = tverskyFromCounts(c, popQ[row], popLib[col], 0.5, 0.5);
  }
}

}  // namespace

unsigned long long readTopkStat(int i) { return readDeviceCounter(g_topkStat, i); }

static void topkSearch(const uint32_t* q, size_t nQ, const uint32_t* lib, size_t nLib, int words, const Measure& m, int k,
                       double* values, int32_t* indices, cudaStream_t s) {
  const bool    dice   = m.kind == kDice;  // a Tanimoto search whose values are then rewritten as Dice
  const Measure search = dice ? Measure{kTanimoto} : m;
  const auto    scanKernel   = isWeighted(search.kind) ? topkScanKernel<true> : topkScanKernel<false>;
  const auto    selectKernel = isWeighted(search.kind) ? topkSelectKernel<true> : topkSelectKernel<false>;
  Scratch<int32_t> popQ(nQ, s), popLibOwn(lib == q && nLib == nQ ? 0 : nLib, s);
  launchRowPopcount(q, nQ, words, popQ.get(), s);
  if (popLibOwn.get()) launchRowPopcount(lib, nLib, words, popLibOwn.get(), s);

  // Candidate slots per row: room for several times the k survivors a doubling slab expects, and for the k best of each
  // part of a scan; a few queries get all the slots a select can sort, so that many CTAs can share one query's scan.
  const uint32_t cap = nQ <= 4096 ? kCapMax : static_cast<uint32_t>(std::min(kCapMax, std::max(256, 8 * k)));
  Scratch<uint32_t> cand(nQ * cap, s), count(nQ, s), redo(nQ, s);
  Scratch<int4>     bar(nQ, s);
  B200_CUDA(cudaMemsetAsync(count.get(), 0, nQ * sizeof(uint32_t), s));
  B200_CUDA(cudaMemsetAsync(redo.get(), 0, nQ * sizeof(uint32_t), s));
  resetDeviceCounters(g_topkStat, s);
  g_topkSlabsLast = 0;

  TopkArgs a{};
  a.q = q, a.lib = lib, a.popQ = popQ.get(), a.popLib = popLibOwn.get() ? popLibOwn.get() : popQ.get();
  a.words = words, a.k = k, a.measure = search;
  a.values = values, a.indices = indices, a.bar = bar.get();
  a.cand = cand.get(), a.count = count.get(), a.redo = redo.get(), a.cap = cap;
  auto diceValues = [&]() {  // (a Dice search: the Tanimoto lists' values rewritten)
    if (!dice) return;
    const size_t   warps  = nQ * static_cast<size_t>(k);
    const unsigned blocks = static_cast<unsigned>(std::min<size_t>((warps + 7) / 8, static_cast<size_t>(smCount()) * 16));
    topkDiceValuesKernel<<<blocks, 256, 0, s>>>(q, lib, words, a.popQ, a.popLib, nQ, k, indices, values);
    B200_LAUNCHED();
  };

  // scan of [beg, end) + the select that merges it; parts: enough CTAs to fill the device, as far as the slots allow
  auto scanAndSelect = [&](size_t beg, size_t end, int listValid, int onlyRedo) {
    const size_t wanted = (4 * static_cast<size_t>(smCount()) + nQ - 1) / nQ, byCols = (end - beg + kSelThreads - 1) / kSelThreads;
    const unsigned parts = static_cast<unsigned>(std::max<size_t>(1, std::min({wanted, byCols, static_cast<size_t>(cap / k)})));
    for (size_t r0 = 0; r0 < nQ; r0 += 65535) {  // (grid.y)
      TopkArgs ar = a;
      ar.q += r0 * words, ar.popQ += r0, ar.values += r0 * k, ar.indices += r0 * k, ar.bar += r0;
      ar.cand += r0 * cap, ar.count += r0, ar.redo += r0;
      scanKernel<<<dim3(parts, static_cast<unsigned>(std::min<size_t>(65535, nQ - r0))), kSelThreads, 0, s>>>(
        ar, static_cast<uint32_t>(beg), static_cast<uint32_t>(end), listValid, onlyRedo);
      B200_LAUNCHED();
    }
    selectKernel<<<static_cast<unsigned>(nQ), kSelThreads, 0, s>>>(a, listValid, 1, onlyRedo);
    B200_LAUNCHED();
  };

  const size_t warm = g_topkSlabCols > 0 ? std::max<size_t>(kTopkMax, static_cast<size_t>(g_topkSlabCols)) : kWarmCols;
  const bool   tensor = g_tensorMinPairs >= 0 && static_cast<double>(nQ) * static_cast<double>(nLib) >= static_cast<double>(g_tensorMinPairs) &&
                      topkTileEligible(words) && nLib > warm;
  if (!tensor) {
    scanAndSelect(0, nLib, 0, 0);
    diceValues();
    return;
  }
  scanAndSelect(0, warm, 0, 0);
  const size_t rowBytes = static_cast<size_t>(words) * 32;
  const size_t slabMax  = g_topkSlabCols > 0 ? static_cast<size_t>(g_topkSlabCols) : (size_t(512) << 20) / rowBytes;
  Scratch<uint8_t> expQ(nQ * rowBytes, s), expLib(std::min(slabMax, nLib - warm) * rowBytes, s);
  launchExpandBits(q, nQ, words, expQ.get(), s);
  for (size_t done = warm; done < nLib;) {
    const size_t cols = std::min({nLib - done, slabMax, g_topkSlabCols > 0 ? slabMax : done});
    launchExpandBits(lib + done * words, cols, words, expLib.get(), s);
    launchTopkTile(search, expQ.get(), nQ, popQ.get(), expLib.get(), cols, a.popLib + done, words, bar.get(), cand.get(), count.get(), cap,
                   static_cast<uint32_t>(done), s);
    selectKernel<<<static_cast<unsigned>(nQ), kSelThreads, 0, s>>>(a, 1, 0, 0);
    B200_LAUNCHED();
    scanAndSelect(done, done + cols, 1, 1);  // the rows whose candidates did not fit (none, as a rule: the CTAs return at once)
    done += cols;
    ++g_topkSlabsLast;
  }
  diceValues();
}

// both entry points: the checks before any device work, then the search
static void topkEntry(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, const Measure& m, int k,
                      double* d_values, int32_t* d_indices, void* stream) {
  B200_REQUIRE(nQ == 0 || d_q, "null fingerprint pointer");
  if (!d_lib) {
    d_lib = d_q;
    nLib  = nQ;
  }
  requireFingerprintWidth(words);
  B200_REQUIRE(nQ < (1ull << 31) && nLib < (1ull << 31), "too many fingerprints");
  B200_REQUIRE(k >= 1 && static_cast<size_t>(k) <= nLib && k <= kTopkMax, "k must be in [1, min(library size, %d)] (got k = %d, library %zu)",
               kTopkMax, k, nLib);
  if (nQ == 0) return;
  B200_REQUIRE(d_values && d_indices, "null output pointer");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(d_q) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_lib) & 15) == 0,
               "fingerprint buffers must be 16-byte aligned");
  topkSearch(d_q, nQ, d_lib, nLib, words, m, k, d_values, d_indices, asStream(stream));
}

}  // namespace b200

using namespace b200;

extern "C" int b200mol_similarity_topk(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, int metric, int k,
                                       double* d_values, int32_t* d_indices, void* stream) {
  return guarded([&] { topkEntry(d_q, nQ, d_lib, nLib, words, measureOfMetric(metric), k, d_values, d_indices, stream); });
}

extern "C" int b200mol_tversky_topk(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, double alpha,
                                    double beta, int k, double* d_values, int32_t* d_indices, void* stream) {
  return guarded([&] { topkEntry(d_q, nQ, d_lib, nLib, words, measureOfWeights(alpha, beta), k, d_values, d_indices, stream); });
}
