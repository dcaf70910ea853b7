// Threshold (range) similarity search on packed fingerprints: b200mol_similarity_threshold.
//
// Contract. Row q of the CSR result lists exactly the columns j for which the fp64 value the matrix of the measure
// (b200mol_tanimoto_cross, b200mol_cosine_cross, b200mol_tversky_cross) stores for (q, j) is >= t (0 < t <= 1), in
// ascending column order, with those values. Without a library the queries are searched against themselves,
// self-matches included.
//
// The pass lists pairs, the assembly makes them exact and orders them:
//   pass      Tanimoto: the thresholded graph pass (launchSimilarity, kCount with atLeast and an edge list):
//             X = queries, Y = library; symmetric (pairs i < j only, half the tiles) for a self search. On the wgmma tile it
//             runs superposed and in popcount order with the popcount band, as the Butina pass does, and lists exactly the
//             pairs whose integer threshold-table test passes - the fp64 predicate s >= t, bit for bit.
//             Cosine: the list operation kList - on the wgmma tile every pair that passes a float bound with a margin
//             (a superset of the answer, unordered); on the SIMT tile the exact fp64 test.
//             Dice (b200mol_tversky_threshold at (1/2, 1/2)): Tanimoto's graph pass with the Dice table and pre-filter.
//             Tversky: kList as well, a float bound like cosine's. With alpha != beta the value is not
//             symmetric, so a self search runs the full (non-symmetric) pass over the set against itself.
//             All run on SIMT or on the tensor cores as "similarity_tensor_min_pairs" decides.
//   read      the listed-pair total, the pairs the re-count keeps and the non-empty queries: the one host read of an attempt.
//             A list longer than its buffer is rerun once into a buffer of the exact size.
//   assembly  (a) every listed pair is re-counted by popcount and its value computed with measureFromCounts (the
//             matrix's expression), kept iff value >= t [before the read, so the read already knows the result size];
//             (b) kept pairs become 64-bit keys (row << colBits | column) with the value as payload, mirrored in a self
//             search, plus the diagonal (s(q, q) = 1 for a non-empty fingerprint; an empty one is at 0 < t);
//             (c) one CUB radix sort over the key bits in use;
//             (d) indices from the sorted keys, indptr[r] = the first key of row >= r by bisection.
// Keys are distinct, so the sorted result does not depend on the order in which the pass or the atomics listed the
// pairs: the output is a pure function of the inputs, whatever tile, superposition or pipeline ran.
#include <algorithm>
#include <cub/device/device_radix_sort.cuh>

#include "profile.cuh"
#include "similarity.cuh"

namespace b200 {
namespace {

constexpr int kRecountLanes = 8;  // lanes per listed pair in the re-count (up to 4 x 16 B of each row per lane)

// stat[0] listed pairs (the pass's edge cursor), [1] pairs the re-count keeps, [2] non-empty queries, [3] fill cursor

// (a): one group of kRecountLanes lanes per listed pair (i, j) in the caller's indices; a dropped pair gets i = -1.
template <bool WEIGHTED>
__global__ void __launch_bounds__(256) recountKernel(const uint32_t* __restrict__ x, const uint32_t* __restrict__ y, int words,
                                                     const int32_t* __restrict__ popX, const int32_t* __restrict__ popY, Measure m,
                                                     double t, int2* list, unsigned long long cap, double* __restrict__ vals,
                                                     unsigned long long* stat) {
  const unsigned long long n = min(stat[0], cap);
  const int                lane = threadIdx.x & 31, gl = lane % kRecountLanes, chunks = words / 4;
  const unsigned long long step = static_cast<unsigned long long>(gridDim.x) * blockDim.x / kRecountLanes;
  for (unsigned long long base = (static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x - lane) / kRecountLanes;
       base < n; base += step) {  // (warp-uniform: a warp takes 32 / kRecountLanes consecutive pairs)
    const unsigned long long e    = base + lane / kRecountLanes;
    const bool               have = e < n;
    int2                     ij   = make_int2(0, 0);
    int                      c    = 0;
    if (have) {
      ij             = list[e];
      const uint4* a = reinterpret_cast<const uint4*>(x + static_cast<size_t>(ij.x) * words);
      const uint4* b = reinterpret_cast<const uint4*>(y + static_cast<size_t>(ij.y) * words);
      for (int k = gl; k < chunks; k += kRecountLanes) {
        const uint4 u = a[k], v = b[k];
        c += __popc(u.x & v.x) + __popc(u.y & v.y) + __popc(u.z & v.z) + __popc(u.w & v.w);
      }
    }
#pragma unroll
    for (int o = kRecountLanes / 2; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    bool keep = false;
    if (have && gl == 0) {
      const double v = measureFromCounts<WEIGHTED>(m, c, popX[ij.x], popY[ij.y]);
      keep           = v >= t;
      vals[e]        = v;
      if (!keep) list[e].x = -1;
    }
    const unsigned kept = __ballot_sync(0xffffffffu, keep);
    if (lane == 0 && kept) atomicAdd(stat + 1, static_cast<unsigned long long>(__popc(kept)));
  }
}

__global__ void nonEmptyKernel(const int32_t* __restrict__ pop, size_t n, unsigned long long* stat) {
  const size_t   i    = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const unsigned some = __ballot_sync(0xffffffffu, i < n && pop[i] > 0);
  if ((threadIdx.x & 31) == 0 && some) atomicAdd(stat + 2, static_cast<unsigned long long>(__popc(some)));
}

// (b): kept pairs (and, symmetric, their mirror images and the diagonal) as keys + values at slots of one warp-aggregated
// cursor; item e < listed is a listed pair, e >= listed the diagonal entry of query e - listed
__global__ void __launch_bounds__(256) fillKernel(const int2* __restrict__ list, const double* __restrict__ vals,
                                                  unsigned long long listed, int symmetric, const int32_t* __restrict__ popX,
                                                  size_t nX, MeasureKind kind, int colBits, unsigned long long* __restrict__ keys,
                                                  double* __restrict__ out, unsigned long long* stat) {
  const unsigned long long total = listed + (symmetric ? nX : 0);
  const int                lane  = threadIdx.x & 31;
  const unsigned long long step  = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long base = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x - lane; base < total;
       base += step) {
    const unsigned long long e = base + lane;
    unsigned long long       k0 = 0, k1 = 0;
    double                   v  = 0.0;
    int                      m  = 0;
    if (e < listed) {
      const int2 ij = list[e];
      if (ij.x >= 0) {
        v  = vals[e];
        k0 = (static_cast<unsigned long long>(ij.x) << colBits) | static_cast<unsigned long long>(ij.y);
        k1 = (static_cast<unsigned long long>(ij.y) << colBits) | static_cast<unsigned long long>(ij.x);
        m  = symmetric ? 2 : 1;
      }
    } else if (e < total) {
      const size_t i = static_cast<size_t>(e - listed);
      const int    a = popX[i];
      if (a > 0) {
        // 1.0, the matrix's diagonal: every measure's value is exactly 1 at c = |A| = |B| (cosine's c / sqrt(c c) too, so
        // the test is against Tanimoto alone, as in the recount)
        v  = simFromCounts(a, a, a, kind != kTanimoto);
        k0 = (static_cast<unsigned long long>(i) << colBits) | static_cast<unsigned long long>(i);
        m  = 1;
      }
    }
    int incl = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    const int          warpTotal = __shfl_sync(0xffffffffu, incl, 31);
    unsigned long long at        = 0;
    if (lane == 31 && warpTotal) at = atomicAdd(stat + 3, static_cast<unsigned long long>(warpTotal));
    at = __shfl_sync(0xffffffffu, at, 31) + static_cast<unsigned long long>(incl - m);
    if (m >= 1) keys[at] = k0, out[at] = v;
    if (m == 2) keys[at + 1] = k1, out[at + 1] = v;
  }
}

// (d): indices[k] = the column of sorted key k; indptr[r] = the first k whose row is >= r (r = 0 .. nX)
__global__ void csrKernel(const unsigned long long* __restrict__ keys, unsigned long long nnz, size_t nX, int colBits,
                          int32_t* __restrict__ indices, int64_t* __restrict__ indptr) {
  const unsigned long long step = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  const unsigned long long mask = (1ull << colBits) - 1ull;
  for (unsigned long long k = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; k < nnz; k += step)
    indices[k] = static_cast<int32_t>(keys[k] & mask);
  for (unsigned long long r = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; r <= nX; r += step) {
    const unsigned long long want = r << colBits;
    unsigned long long       lo = 0, hi = nnz;
    while (lo < hi) {
      const unsigned long long mid = (lo + hi) / 2;
      if (keys[mid] < want) lo = mid + 1;
      else hi = mid;
    }
    indptr[r] = static_cast<int64_t>(lo);
  }
}

int bitsFor(size_t n) {  // bits that hold 0 .. n - 1
  int b = 0;
  while ((1ull << b) < n) ++b;
  return b;
}

// (b) to (d): list[0 .. listed) the listed pairs (i, j) (i = -1: dropped) with their values vals[], nnz the entries they
// give, written to the caller's CSR; stat[3], zero on entry, is the fill cursor
void assembleThresholdCsr(const int2* list, const double* vals, unsigned long long listed, bool symmetric, const int32_t* popX,
                          size_t nX, size_t nCols, MeasureKind kind, unsigned long long nnz, unsigned long long* stat,
                          int64_t* indptr, int32_t* indices, double* values, cudaStream_t s) {
  const int                   colBits = bitsFor(nCols), endBit = std::max(1, colBits + bitsFor(nX));
  Scratch<unsigned long long> keysIn(nnz, s), keysOut(nnz, s);
  Scratch<double>             valsIn(nnz, s);
  if (listed + (symmetric ? nX : 0) > 0) {
    fillKernel<<<blocksFor(listed + (symmetric ? nX : 0), 256), 256, 0, s>>>(list, vals, listed, symmetric ? 1 : 0, popX, nX, kind,
                                                                             colBits, keysIn.get(), valsIn.get(), stat);
    B200_LAUNCHED();
  }
  if (nnz) {
    const int64_t n        = static_cast<int64_t>(nnz);
    size_t        tmpBytes = 0;
    B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmpBytes, keysIn.get(), keysOut.get(), valsIn.get(), values, n, 0, endBit, s));
    Scratch<uint8_t> tmp(tmpBytes, s);
    B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tmpBytes, keysIn.get(), keysOut.get(), valsIn.get(), values, n, 0, endBit, s));
    g_launchCount.fetch_add(1);
  }
  csrKernel<<<blocksFor(std::max<unsigned long long>(nnz, nX + 1), 256), 256, 0, s>>>(keysOut.get(), nnz, nX, colBits, indices, indptr);
  B200_LAUNCHED();
}

}  // namespace

void thresholdCsr(unsigned long long listCap, const ListPairs& listPairs, const ResultSize& nnzOf, bool symmetric,
                  const int32_t* popX, size_t nX, size_t nCols, MeasureKind kind, int64_t* indptr, int32_t* indices,
                  double* values, uint64_t cap, uint64_t* hNnz, cudaStream_t s) {
  Scratch<unsigned long long> stat(4, s);
  unsigned long long          h[3] = {0, 0, 0};
  Scratch<int2>               list;
  Scratch<double>             vals;
  for (int attempt = 0;; ++attempt) {
    list = Scratch<int2>(listCap, s);
    vals = Scratch<double>(listCap, s);
    B200_CUDA(cudaMemsetAsync(stat.get(), 0, 4 * sizeof(unsigned long long), s));
    listPairs(list.get(), vals.get(), listCap, stat.get());
    // the one host read of an attempt
    B200_CUDA(cudaMemcpyAsync(h, stat.get(), sizeof(h), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    if (h[0] <= listCap) break;
    B200_REQUIRE(attempt == 0, "threshold search: the pass listed %llu pairs, then more than that on a rerun", h[0]);
    listCap = h[0];
  }
  const unsigned long long nnz = nnzOf(h);
  *hNnz                        = nnz;
  if (nnz > cap) return;  // the caller asks again with room for nnz

  PhaseTimer timer("threshold_assembly", s);
  assembleThresholdCsr(list.get(), vals.get(), h[0], symmetric, popX, nX, nCols, kind, nnz, stat.get(), indptr, indices, values, s);
}

namespace {

void thresholdSearch(const uint32_t* q, size_t nQ, const uint32_t* lib, size_t nLib, bool self, int words, const Measure& m, double t,
                     int64_t* indptr, int32_t* indices, double* values, uint64_t cap, uint64_t* hNnz, cudaStream_t s) {
  Scratch<int32_t> popQ(nQ, s), popLibOwn(self ? 0 : nLib, s), counts(nQ, s);
  launchRowPopcount(q, nQ, words, popQ.get(), s);
  if (!self) launchRowPopcount(lib, nLib, words, popLibOwn.get(), s);
  const int32_t* popLib = self ? popQ.get() : popLibOwn.get();

  // The pass's list: sized for a result that fits `cap` (a self search lists each off-diagonal pair once), plus room
  // for the cosine tile's near misses.
  const double   allPairs = self ? static_cast<double>(nQ) * (static_cast<double>(nQ) - 1.0) / 2.0
                                 : static_cast<double>(nQ) * static_cast<double>(nLib);
  const uint64_t want     = std::min<uint64_t>(self ? cap / 2 : cap, 1ull << 27);
  const unsigned long long firstCap = std::max<unsigned long long>(1, static_cast<unsigned long long>(
                                        std::min(allPairs, static_cast<double>(std::max<uint64_t>(1ull << 20, want + want / 8)))));
  auto listPairs = [&](int2* list, double* vals, unsigned long long listCap, unsigned long long* stat) {
    {
      PhaseTimer timer("threshold_pass", s);
      SimLaunch  p;
      p.x         = q;
      p.y         = lib;
      p.nX        = nQ;
      p.nY        = nLib;
      p.words     = words;
      p.measure   = m;
      p.cutoff    = t;
      p.atLeast   = true;
      p.rowCounts = counts.get();
      p.symmetric = self;
      p.edges     = list;
      p.edgeCursor = stat;
      p.edgeCap   = listCap;
      B200_CUDA(cudaMemsetAsync(counts.get(), 0, nQ * sizeof(int32_t), s));
      // Tanimoto and Dice count with their exact tables; cosine and Tversky list by a float bound
      launchSimilarity(m.kind == kCosine || m.kind == kTversky ? kList : kCount, p, s);
    }
    PhaseTimer     timer("threshold_recount", s);
    const unsigned blocks  = blocksFor(listCap * kRecountLanes, 256);
    const auto     recount = isWeighted(m.kind) ? recountKernel<true> : recountKernel<false>;
    recount<<<blocks, 256, 0, s>>>(q, lib, words, popQ.get(), popLib, m, t, list, listCap, vals, stat);
    B200_LAUNCHED();
    if (self) {
      nonEmptyKernel<<<static_cast<unsigned>((nQ + 255) / 256), 256, 0, s>>>(popQ.get(), nQ, stat);
      B200_LAUNCHED();
    }
  };
  // the pairs the re-count keeps, mirrored in a self search together with the non-empty queries' diagonal
  auto nnzOf = [self](const unsigned long long* h) { return self ? 2 * h[1] + h[2] : h[1]; };
  thresholdCsr(firstCap, listPairs, nnzOf, self, popQ.get(), nQ, self ? nQ : nLib, m.kind, indptr, indices, values, cap, hNnz, s);
}

}  // namespace
}  // namespace b200

using namespace b200;

static void thresholdEntry(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, const Measure& m,
                           double threshold, int64_t* d_indptr, int32_t* d_indices, double* d_values, uint64_t cap, uint64_t* h_nnz,
                           void* stream) {
  requireFingerprintWidth(words);
  B200_REQUIRE(threshold > 0.0 && threshold <= 1.0, "threshold must be in (0, 1] (got %g)", threshold);
  const bool self = d_lib == nullptr;
  if (self) nLib = nQ;
  B200_REQUIRE(nQ < (1ull << 31) && nLib < (1ull << 31), "too many fingerprints");
  B200_REQUIRE(h_nnz && d_indptr, "null pointer");
  B200_REQUIRE(nQ == 0 || d_q, "null fingerprint pointer");
  B200_REQUIRE(cap == 0 || (d_indices && d_values), "null output pointer");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(d_q) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_lib) & 15) == 0,
               "fingerprint buffers must be 16-byte aligned");
  const cudaStream_t s = asStream(stream);
  *h_nnz               = 0;
  if (nQ == 0 || nLib == 0) {  // no pair: every row is empty
    B200_CUDA(cudaMemsetAsync(d_indptr, 0, (nQ + 1) * sizeof(int64_t), s));
    return;
  }
  // an asymmetric measure has no symmetric pass: the set is searched against itself as a library, every pair in full
  const bool symmetricPass = self && !(m.kind == kTversky && m.alpha != m.beta);
  thresholdSearch(d_q, nQ, self ? d_q : d_lib, nLib, symmetricPass, words, m, threshold, d_indptr, d_indices, d_values, cap, h_nnz, s);
}

extern "C" int b200mol_similarity_threshold(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, int metric,
                                            double threshold, int64_t* d_indptr, int32_t* d_indices, double* d_values, uint64_t cap,
                                            uint64_t* h_nnz, void* stream) {
  return guarded([&] {
    thresholdEntry(d_q, nQ, d_lib, nLib, words, measureOfMetric(metric), threshold, d_indptr, d_indices, d_values, cap, h_nnz, stream);
  });
}

extern "C" int b200mol_tversky_threshold(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, double alpha,
                                         double beta, double threshold, int64_t* d_indptr, int32_t* d_indices, double* d_values,
                                         uint64_t cap, uint64_t* h_nnz, void* stream) {
  return guarded([&] {
    thresholdEntry(d_q, nQ, d_lib, nLib, words, measureOfWeights(alpha, beta), threshold, d_indptr, d_indices, d_values, cap, h_nnz,
                   stream);
  });
}
