// Butina clustering on a neighbour graph held as CSR in HBM, sm_90a.
//
// Definition (RDKit ML.Cluster.Butina.ClusterData(reordering=True); see include/b200mol.h): repeatedly take the free
// point with the most free neighbours (ties -> highest index), cluster = that point + its free neighbours.
//
// Design (not the reference's): the O(N^2) work happens exactly once — the fused similarity tile
// (tanimoto.cu) emits neighbour counts AND the edge list in one pass, or the dense distance matrix is scanned once —
// and the greedy loop then runs on the CSR graph inside ONE persistent cooperative kernel: no per-cluster host sync
// (the reference's fused_butina does three .item() syncs per cluster, nvmolkit/clustering.py:152-169, and its dense
// path re-reads the N^2 hit matrix every round, src/butina.cu:50-74).
//
// The greedy order is honoured exactly, but not one cluster at a time. A free point whose key (free-neighbour count,
// index) is the largest within TWO hops of itself will be chosen by the sequential algorithm with exactly its present
// free neighbours, whatever happens elsewhere first: every centre chosen before it has a larger key, hence lies more
// than two hops away and touches none of its neighbours; and taking it out early only LOWERS keys that were already
// below its own, so it changes no earlier choice. All such local maxima are therefore committed in the same round
// (butinaRoundsKernel: two passes over the free rows' adjacency for the 2-hop maxima, one to commit). Keys chosen by
// the sequential algorithm decrease strictly, so the creation order of the clusters - their ids - is the descending
// order of the keys the centres had when chosen: one radix sort at the end. Rounds that commit only a handful of
// centres hand over to the one-cluster-per-step loop (butinaLoopKernel): (A) slice-wise arg-max with dirty flags,
// grid.sync, (B) a warp per neighbour of the centroid assigns it and decrements the counts of ITS neighbours, grid.sync.
#include <cooperative_groups.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "profile.cuh"
#include "similarity.cuh"

namespace cg = cooperative_groups;

namespace b200 {
void launchRowPopcount(const uint32_t* fp, size_t n, int words, int32_t* pop, cudaStream_t s);

namespace {

constexpr int kSliceShift = 10;  // arg-max slices of 1024 points
constexpr int kSlice      = 1 << kSliceShift;
constexpr int kLoopThreads = 1024;
}  // namespace
int g_butinaMinCommits = 32;  // a parallel round that commits fewer clusters hands over to the stepwise loop (option "butina_min_round_commits")
namespace {

__global__ void fillAdjacencyKernel(const int2* __restrict__ edges, unsigned long long nEdges,
                                    const long long* __restrict__ offsets, int* __restrict__ fillPos,
                                    int* __restrict__ adj) {
  const unsigned long long e = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= nEdges) return;
  const int2 ij = edges[e];
  adj[offsets[ij.x] + atomicAdd(fillPos + ij.x, 1)] = ij.y;
  adj[offsets[ij.y] + atomicAdd(fillPos + ij.y, 1)] = ij.x;
}

// Dense distance matrix: block per row. pass 0 = count, pass 1 = fill.
template <int PASS>
__global__ void denseRowKernel(const double* __restrict__ dist, int n, double cutoff, int32_t* __restrict__ counts,
                               const long long* __restrict__ offsets, int* __restrict__ adj) {
  const int     row = blockIdx.x;
  const double* d   = dist + static_cast<size_t>(row) * n;
  __shared__ int cursor;
  if (threadIdx.x == 0) cursor = 0;
  __syncthreads();
  int local = 0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const bool hit = (j != row) && (__ldcs(d + j) <= cutoff);
    if (PASS == 0) {
      local += hit;
    } else if (hit) {
      adj[offsets[row] + atomicAdd(&cursor, 1)] = j;
    }
  }
  if (PASS == 0) {
    for (int o = 16; o; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&cursor, local);
    __syncthreads();
    if (threadIdx.x == 0) counts[row] = cursor;
  }
}

__global__ void widenCountsKernel(const int32_t* __restrict__ c, int n, long long* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = c[i];
}

struct LoopState {
  int                 n;
  int                 nSlices;
  const long long*    offsets;  // [n+1]
  const int*          adj;
  int32_t*            counts;   // free-neighbour counts (live)
  int32_t*            ids;      // index of the point's centre while the loops run, -1 = free
  unsigned long long* selKey;   // [n] key a centre had when it was chosen (0 = not a centre)
  unsigned long long* sliceBest;  // [nSlices] key = count<<32 | idx ; 0 = nothing
  int*                sliceDirty;
  int*                nClustersOut;  // += clusters formed (non-singletons; isolated leftovers come later)
  int                 vecOk;         // ids / counts are 16-byte aligned: full slices use vector loads
};

__device__ __forceinline__ unsigned long long warpMax(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v                          = t > v ? t : v;
  }
  return v;
}

__global__ void __launch_bounds__(kLoopThreads, 1) butinaLoopKernel(LoopState st) {
  cg::grid_group grid = cg::this_grid();
  __shared__ unsigned long long warpBest[kLoopThreads / 32];
  __shared__ unsigned long long blockBest;

  const int lane         = threadIdx.x & 31;
  const int warpInBlock  = threadIdx.x >> 5;
  const int warpsPerBlk  = kLoopThreads / 32;
  const int gWarp        = blockIdx.x * warpsPerBlk + warpInBlock;
  const int gWarps       = gridDim.x * warpsPerBlk;
  int       cluster      = 0;

  for (;;) {
    // ---- (A) refresh dirty slices: one warp per slice ----
    for (int sl = gWarp; sl < st.nSlices; sl += gWarps) {
      if (!st.sliceDirty[sl]) continue;
      unsigned long long best = 0;
      const int          base = sl << kSliceShift;
      if (base + kSlice <= st.n && st.vecOk) {
        // full slice: 8 independent 16-byte loads of ids and counts per lane (no dependent-load chain)
        const int4* ids4 = reinterpret_cast<const int4*>(st.ids + base);
        const int4* cnt4 = reinterpret_cast<const int4*>(st.counts + base);
        int4        id[8], ct[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          id[k] = ids4[k * 32 + lane];
          ct[k] = cnt4[k * 32 + lane];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int  i0   = base + (k * 32 + lane) * 4;
          const int  iv[4] = {id[k].x, id[k].y, id[k].z, id[k].w};
          const int  cv[4] = {ct[k].x, ct[k].y, ct[k].z, ct[k].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (iv[q] < 0) {
              const unsigned long long key =
                (static_cast<unsigned long long>(static_cast<unsigned>(cv[q])) << 32) | static_cast<unsigned>(i0 + q);
              best = key > best ? key : best;
            }
          }
        }
      } else {
        for (int k = lane; k < kSlice; k += 32) {
          const int i = base + k;
          if (i < st.n && st.ids[i] < 0) {
            const unsigned long long key =
              (static_cast<unsigned long long>(static_cast<unsigned>(st.counts[i])) << 32) | static_cast<unsigned>(i);
            best = key > best ? key : best;
          }
        }
      }
      best = warpMax(best);
      if (lane == 0) {
        st.sliceBest[sl]  = best;
        st.sliceDirty[sl] = 0;
      }
    }
    grid.sync();

    // ---- global arg-max over slice maxima (every block redundantly; nSlices is ~N/1024) ----
    unsigned long long best = 0;
    for (int sl = threadIdx.x; sl < st.nSlices; sl += kLoopThreads) {
      const unsigned long long k = st.sliceBest[sl];
      best                       = k > best ? k : best;
    }
    best = warpMax(best);
    if (lane == 0) warpBest[warpInBlock] = best;
    __syncthreads();
    if (warpInBlock == 0) {
      unsigned long long b = lane < warpsPerBlk ? warpBest[lane] : 0ull;
      b                    = warpMax(b);
      if (lane == 0) blockBest = b;
    }
    __syncthreads();
    best = blockBest;
    if ((best >> 32) == 0) break;  // nobody has a free neighbour left: the rest are singletons
    const int centre = static_cast<int>(best & 0xffffffffu);

    // ---- (B) assign: a warp per neighbour of the centre ----
    const long long cBeg = st.offsets[centre], cEnd = st.offsets[centre + 1];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      st.ids[centre]                        = centre;
      st.selKey[centre]                     = best;
      st.sliceDirty[centre >> kSliceShift] = 1;
    }
    for (long long e = cBeg + gWarp; e < cEnd; e += gWarps) {
      const int m = st.adj[e];
      if (st.ids[m] >= 0) continue;  // taken in an earlier round (ids of this round's members are written only here)
      if (lane == 0) {
        st.ids[m]                         = centre;
        st.sliceDirty[m >> kSliceShift] = 1;
      }
      const long long mBeg = st.offsets[m], mEnd = st.offsets[m + 1];
      for (long long f = mBeg + lane; f < mEnd; f += 32) {
        const int i = st.adj[f];
        // Decrementing a point that is no longer free (or joins this cluster) is harmless: its count is dead.
        if (i != centre) {
          atomicSub(st.counts + i, 1);
          st.sliceDirty[i >> kSliceShift] = 1;
        }
      }
    }
    ++cluster;
    grid.sync();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(st.nClustersOut, cluster);
}

// ---- many clusters per round: every 2-hop local maximum of the key is committed (see the file header) ----
constexpr int kRoundThreads = 256;
__device__ __forceinline__ unsigned long long liveKey(const LoopState& st, int i) {
  // other SMs change ids / counts between the phases of a round: read through L2
  return __ldcg(st.ids + i) < 0
           ? (static_cast<unsigned long long>(static_cast<unsigned>(__ldcg(st.counts + i))) << 32) | static_cast<unsigned>(i)
           : 0ull;
}
__global__ void __launch_bounds__(kRoundThreads) butinaRoundsKernel(LoopState st, unsigned long long* best1, int minCommits) {
  cg::grid_group grid   = cg::this_grid();
  const int      lane   = threadIdx.x & 31;
  const int      gWarp  = (blockIdx.x * kRoundThreads + threadIdx.x) >> 5;
  const int      gWarps = (gridDim.x * kRoundThreads) >> 5;
  int            done   = 0, round = 0;
  for (;;) {
    // (1) best1[m] = largest key in the closed free neighbourhood of every free row m (0 for taken rows)
    for (int base = gWarp * 32; base < st.n; base += gWarps * 32) {
      const int                row  = base + lane;
      const unsigned long long mine = row < st.n ? liveKey(st, row) : 0ull;
      if (row < st.n && mine == 0ull) best1[row] = 0ull;
      unsigned todo = __ballot_sync(0xffffffffu, mine != 0ull);
      while (todo) {
        const int          src = __ffs(todo) - 1;
        const int          m   = base + src;
        unsigned long long b   = __shfl_sync(0xffffffffu, mine, src);
        todo &= todo - 1;
        const long long beg = st.offsets[m], end = st.offsets[m + 1];
        for (long long e = beg + lane; e < end; e += 32) {
          const unsigned long long k = liveKey(st, st.adj[e]);
          b                          = k > b ? k : b;
        }
        b = warpMax(b);
        if (lane == 0) best1[m] = b;
      }
    }
    grid.sync();
    // (2) a free point with free neighbours whose key tops every best1 of its free neighbours is a 2-hop maximum
    for (int base = gWarp * 32; base < st.n; base += gWarps * 32) {
      const int                row  = base + lane;
      unsigned long long       mine = row < st.n ? liveKey(st, row) : 0ull;
      if ((mine >> 32) == 0) mine = 0ull;  // no free neighbour left: a singleton, later
      unsigned todo = __ballot_sync(0xffffffffu, mine != 0ull);
      while (todo) {
        const int                src = __ffs(todo) - 1;
        const int                p   = base + src;
        const unsigned long long kp  = __shfl_sync(0xffffffffu, mine, src);
        todo &= todo - 1;
        unsigned long long b   = 0ull;
        const long long    beg = st.offsets[p], end = st.offsets[p + 1];
        for (long long e = beg + lane; e < end; e += 32) {
          const unsigned long long k = __ldcg(best1 + st.adj[e]);
          b                          = k > b ? k : b;
        }
        b = warpMax(b);
        if (lane == 0 && b <= kp) st.selKey[p] = kp;  // (b == kp: p itself is in its free neighbours' neighbourhoods)
      }
    }
    grid.sync();
    // (3) commit the new centres: their neighbourhoods are pairwise disjoint, the count updates are atomic
    for (int base = gWarp * 32; base < st.n; base += gWarps * 32) {
      const int  row    = base + lane;
      const bool fresh  = row < st.n && __ldcg(st.selKey + row) != 0ull && __ldcg(st.ids + row) < 0;
      unsigned   todo   = __ballot_sync(0xffffffffu, fresh);
      if (lane == 0 && todo) atomicAdd(st.nClustersOut, __popc(todo));
      while (todo) {
        const int p = base + __ffs(todo) - 1;
        todo &= todo - 1;
        if (lane == 0) st.ids[p] = p;
        const long long beg = st.offsets[p], end = st.offsets[p + 1];
        for (long long e = beg; e < end; ++e) {
          const int m = st.adj[e];
          if (__ldcg(st.ids + m) >= 0) continue;  // taken in an earlier round
          if (lane == 0) st.ids[m] = p;
          const long long mBeg = st.offsets[m], mEnd = st.offsets[m + 1];
          for (long long f = mBeg + lane; f < mEnd; f += 32) {
            const int i = st.adj[f];
            if (i != p) atomicSub(st.counts + i, 1);  // dead counts (members, taken points) may go anywhere
          }
        }
      }
    }
    grid.sync();
    const int total = __ldcg(st.nClustersOut);
#ifdef B200_BUTINA_DEBUG
    if (blockIdx.x == 0 && threadIdx.x == 0) printf("round %d total %d done %d\n", round, total, done);
#endif
    if (total - done < (minCommits > 1 ? minCommits : 1)) break;  // (a round without a commit ends the phase in any case)
    if (++round >= st.n) break;  // cannot happen (every continuing round commits a cluster); a guard against a spin
    done = total;
  }
}

__global__ void iotaKernel(int* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}
// sorted (key descending, point): rank r -> centroids[r], idOf[point] = r
__global__ void rankCentresKernel(const unsigned long long* __restrict__ keys, const int* __restrict__ pts, int n,
                                  int32_t* __restrict__ centroids, int* __restrict__ idOf) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || keys[r] == 0ull) return;
  centroids[r]  = pts[r];
  idOf[pts[r]]  = r;
}
__global__ void remapIdsKernel(int32_t* __restrict__ ids, const int* __restrict__ idOf, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && ids[i] >= 0) ids[i] = idOf[ids[i]];
}

// Leftover free points become singletons in descending index order (RDKit sorts (count, idx) descending).
__global__ void freeFlagsKernel(const int32_t* __restrict__ ids, int n, int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = ids[i] < 0 ? 1 : 0;
}
__global__ void assignSingletonsKernel(int32_t* __restrict__ ids, int32_t* __restrict__ centroids,
                                       const int* __restrict__ flags, const int* __restrict__ rankExcl, int n,
                                       const int* __restrict__ nLoopClusters, int32_t* __restrict__ nClustersOut) {
  const int i         = blockIdx.x * blockDim.x + threadIdx.x;
  const int totalFree = rankExcl[n - 1] + flags[n - 1];
  const int base      = *nLoopClusters;
  if (i == 0 && nClustersOut) *nClustersOut = base + totalFree;
  if (i >= n || !flags[i]) return;
  const int id = base + (totalFree - 1 - rankExcl[i]);
  ids[i]       = id;
  centroids[id] = i;
}

__global__ void fillKernel(int32_t* p, size_t n, int32_t v) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// counts[n] = live degrees; offsets/adj = CSR. Runs the greedy loop + singleton tail. Leaves results in ids/centroids.
void clusterFromCsr(int n, const long long* offsets, const int* adj, int32_t* counts, int32_t* ids, int32_t* centroids,
                    int32_t* dNClusters, cudaStream_t s) {
  const int                   nSlices = (n + kSlice - 1) >> kSliceShift;
  Scratch<unsigned long long> sliceBest(nSlices, s);
  Scratch<int>                sliceDirty(nSlices, s);
  Scratch<int>                nLoop(1, s);
  Scratch<unsigned long long> selKey(n, s), best1(n, s);
  fillKernel<<<(n + 255) / 256, 256, 0, s>>>(ids, n, -1);
  B200_LAUNCHED();
  B200_CUDA(cudaMemsetAsync(selKey.get(), 0, sizeof(unsigned long long) * n, s));
  B200_CUDA(cudaMemsetAsync(nLoop.get(), 0, sizeof(int), s));

  const int vecOk = ((reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(counts)) & 15) == 0;
  LoopState st{n, nSlices, offsets, adj, counts, ids, selKey.get(), sliceBest.get(), sliceDirty.get(), nLoop.get(), vecOk};
  {
    // many clusters per round while a round still commits a few dozen; then one cluster per step
    PhaseTimer          t("cluster_rounds", s);
    int                 perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, butinaRoundsKernel, kRoundThreads, 0));
    B200_REQUIRE(perSm >= 1, "butina rounds kernel does not fit on an SM");
    const int           blocks = smCount() * (perSm > 4 ? 4 : perSm);
    unsigned long long* b1     = best1.get();
    int                 minCommits = g_butinaMinCommits;
    void*               args[] = {&st, &b1, &minCommits};
    B200_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(butinaRoundsKernel), dim3(blocks), dim3(kRoundThreads), args, 0, s));
    g_launchCount.fetch_add(1);
  }
  fillKernel<<<(nSlices + 255) / 256, 256, 0, s>>>(sliceDirty.get(), nSlices, 1);
  B200_LAUNCHED();
  {
    PhaseTimer t("cluster_steps", s);
    int        perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, butinaLoopKernel, kLoopThreads, 0));
    B200_REQUIRE(perSm >= 1, "butina loop kernel does not fit on an SM");
    // The loop is latency-bound (two grid-wide barriers per cluster): a small grid keeps the barrier cheap, and 32 CTAs x
    // 32 warps are plenty for the ~100 dirty slices and ~100 member warps of a round.
    const int blocks = smCount() < 32 ? smCount() : 32;
    void*     args[] = {&st};
    B200_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(butinaLoopKernel), dim3(blocks), dim3(kLoopThreads), args, 0, s));
    g_launchCount.fetch_add(1);
  }
  {
    // cluster ids = rank of the centre's key (descending) = creation order of the sequential algorithm
    Scratch<unsigned long long> keysOut(n, s);
    Scratch<int>                ptsIn(n, s), ptsOut(n, s), idOf(n, s);
    iotaKernel<<<(n + 255) / 256, 256, 0, s>>>(ptsIn.get(), n);
    B200_LAUNCHED();
    size_t sortBytes = 0;
    B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, sortBytes, selKey.get(), keysOut.get(), ptsIn.get(), ptsOut.get(), n,
                                                        0, 64, s));
    Scratch<uint8_t> sortTmp(sortBytes, s);
    B200_CUDA(cub::DeviceRadixSort::SortPairsDescending(sortTmp.get(), sortBytes, selKey.get(), keysOut.get(), ptsIn.get(),
                                                        ptsOut.get(), n, 0, 64, s));
    g_launchCount.fetch_add(1);
    rankCentresKernel<<<(n + 255) / 256, 256, 0, s>>>(keysOut.get(), ptsOut.get(), n, centroids, idOf.get());
    B200_LAUNCHED();
    remapIdsKernel<<<(n + 255) / 256, 256, 0, s>>>(ids, idOf.get(), n);
    B200_LAUNCHED();
  }

  Scratch<int> flags(n, s), rank(n, s);
  freeFlagsKernel<<<(n + 255) / 256, 256, 0, s>>>(ids, n, flags.get());
  B200_LAUNCHED();
  size_t tmpBytes = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, flags.get(), rank.get(), n, s));
  Scratch<uint8_t> tmp(tmpBytes, s);
  B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tmpBytes, flags.get(), rank.get(), n, s));
  g_launchCount.fetch_add(1);
  assignSingletonsKernel<<<(n + 255) / 256, 256, 0, s>>>(ids, centroids, flags.get(), rank.get(), n, nLoop.get(), dNClusters);
  B200_LAUNCHED();
}

void scanOffsets(const int32_t* counts, int n, long long* offsets, cudaStream_t s) {
  // offsets[0..n] = exclusive scan of counts (64-bit: edge totals can exceed 2^31)
  Scratch<long long> wide(static_cast<size_t>(n) + 1, s);
  B200_CUDA(cudaMemsetAsync(wide.get(), 0, (static_cast<size_t>(n) + 1) * sizeof(long long), s));
  widenCountsKernel<<<(n + 255) / 256, 256, 0, s>>>(counts, n, wide.get());
  B200_LAUNCHED();
  size_t tmpBytes = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, wide.get(), offsets, n + 1, s));
  Scratch<uint8_t> tmp(tmpBytes, s);
  B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tmpBytes, wide.get(), offsets, n + 1, s));
  g_launchCount.fetch_add(1);
}

}  // namespace
}  // namespace b200

using namespace b200;

namespace b200 {
namespace {

// counts (+=) and (i<j) edges of the thresholded similarity graph for this rank's tile-row groups.
void neighborEdges(const uint32_t* d_fp, size_t n, int words, int metric, double cutoff, uint32_t groupOffset,
                   uint32_t groupStride, int32_t* counts, int2* edges, unsigned long long cap,
                   unsigned long long* dCursor, cudaStream_t s) {
  SimLaunch q;
  q.x = q.y     = d_fp;
  q.nX = q.nY   = n;
  q.words       = words;
  q.cutoff      = cutoff;
  q.sign        = 1;
  q.rowCounts   = counts;
  q.symmetric   = true;
  q.groupOffset = groupOffset;
  q.groupStride = groupStride;
  q.edges       = edges;
  q.edgeCursor  = dCursor;
  q.edgeCap     = cap;
  launchSimilarity(metric == B200MOL_METRIC_TANIMOTO ? kCountTanimoto : kCountCosine, q, s);
}

void clusterFromEdges(int N, int32_t* counts, const int2* edges, unsigned long long nEdges, int32_t* ids,
                      int32_t* centroids, int32_t* dNCl, cudaStream_t s) {
  const size_t       n = static_cast<size_t>(N);
  Scratch<long long> offsets(n + 1, s);
  Scratch<int>       adj(2 * nEdges + 1, s);
  {
    PhaseTimer t("csr_build", s);
    scanOffsets(counts, N, offsets.get(), s);
    Scratch<int> fillPos(n, s);
    B200_CUDA(cudaMemsetAsync(fillPos.get(), 0, n * sizeof(int), s));
    if (nEdges) {
      fillAdjacencyKernel<<<static_cast<unsigned>((nEdges + 255) / 256), 256, 0, s>>>(edges, nEdges, offsets.get(),
                                                                                     fillPos.get(), adj.get());
      B200_LAUNCHED();
    }
  }
  PhaseTimer t("cluster_loop", s);
  clusterFromCsr(N, offsets.get(), adj.get(), counts, ids, centroids, dNCl, s);
}

}  // namespace
}  // namespace b200

extern "C" int b200mol_neighbor_edges(const uint32_t* d_fp, size_t n, int words, int metric, double cutoff,
                                      uint32_t group_offset, uint32_t group_stride, int32_t* d_counts,
                                      int32_t* d_edges, uint64_t edge_cap, uint64_t* h_n_edges, void* stream) {
  return guarded([&] {
    B200_REQUIRE(metric == B200MOL_METRIC_TANIMOTO || metric == B200MOL_METRIC_COSINE, "unknown metric %d", metric);
    B200_REQUIRE(cutoff >= 0.0 && cutoff <= 1.0, "cutoff must be in [0, 1], got %g", cutoff);
    B200_REQUIRE(n < (1ull << 31), "too many fingerprints");
    B200_REQUIRE(group_stride >= 1 && group_offset < group_stride, "bad row-group sharding %u/%u", group_offset, group_stride);
    cudaStream_t s = asStream(stream);
    if (h_n_edges) *h_n_edges = 0;
    if (n == 0) return;
    B200_REQUIRE(d_fp && d_counts && (d_edges || edge_cap == 0), "null pointer");
    Scratch<unsigned long long> cursor(1, s);
    B200_CUDA(cudaMemsetAsync(cursor.get(), 0, sizeof(unsigned long long), s));
    {
      PhaseTimer t("neighbor_pass", s);
      neighborEdges(d_fp, n, words, metric, cutoff, group_offset, group_stride, d_counts,
                    reinterpret_cast<int2*>(d_edges), edge_cap, cursor.get(), s);
    }
    if (h_n_edges) {
      unsigned long long v = 0;
      B200_CUDA(cudaMemcpyAsync(&v, cursor.get(), sizeof(v), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));  // documented sync: the edge total sizes the CSR
      *h_n_edges = v;
    }
  });
}

extern "C" int b200mol_butina_from_edges(size_t n, int32_t* d_counts, const int32_t* d_edges, uint64_t n_edges,
                                         int32_t* d_cluster_ids, int32_t* d_centroids, int32_t* d_n_clusters,
                                         int32_t* h_n_clusters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n < (1ull << 31), "too many points");
    cudaStream_t s = asStream(stream);
    if (n == 0) {
      if (h_n_clusters) *h_n_clusters = 0;
      if (d_n_clusters) B200_CUDA(cudaMemsetAsync(d_n_clusters, 0, sizeof(int32_t), s));
      return;
    }
    B200_REQUIRE(d_counts && d_cluster_ids && (d_edges || n_edges == 0), "null pointer");
    Scratch<int32_t> centroidsOwn(d_centroids ? 0 : n, s);
    int32_t*         centroids = d_centroids ? d_centroids : centroidsOwn.get();
    Scratch<int32_t> nClOwn(1, s);
    int32_t*         dNCl = d_n_clusters ? d_n_clusters : nClOwn.get();
    clusterFromEdges(static_cast<int>(n), d_counts, reinterpret_cast<const int2*>(d_edges), n_edges, d_cluster_ids,
                     centroids, dNCl, s);
    if (h_n_clusters) {
      B200_CUDA(cudaMemcpyAsync(h_n_clusters, dNCl, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
    }
  });
}

extern "C" int b200mol_butina_fused(const uint32_t* d_fp, size_t n, int words, int metric, double cutoff,
                                    int32_t* d_cluster_ids, int32_t* d_centroids, int32_t* d_n_clusters,
                                    int32_t* h_n_clusters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(metric == B200MOL_METRIC_TANIMOTO || metric == B200MOL_METRIC_COSINE, "unknown metric %d", metric);
    B200_REQUIRE(cutoff >= 0.0 && cutoff <= 1.0, "cutoff must be in [0, 1], got %g", cutoff);
    B200_REQUIRE(n < (1ull << 31), "too many fingerprints");
    cudaStream_t s = asStream(stream);
    if (n == 0) {
      if (h_n_clusters) *h_n_clusters = 0;
      if (d_n_clusters) B200_CUDA(cudaMemsetAsync(d_n_clusters, 0, sizeof(int32_t), s));
      return;
    }
    B200_REQUIRE(d_fp && d_cluster_ids, "null pointer");
    Scratch<int32_t> counts(n, s);
    // One N^2/2 pass: counts + edge list. The capacity grows (and the deterministic pass repeats) only when the graph
    // is denser than 64 neighbours per point on average.
    unsigned long long cap = static_cast<unsigned long long>(n) * 64ull;
    Scratch<int2>      edges;
    uint64_t           nEdges = 0;
    for (int attempt = 0; attempt < 2; ++attempt) {
      edges = Scratch<int2>(cap, s);
      B200_CUDA(cudaMemsetAsync(counts.get(), 0, n * sizeof(int32_t), s));
      const int rc = b200mol_neighbor_edges(d_fp, n, words, metric, cutoff, 0, 1, counts.get(),
                                            reinterpret_cast<int32_t*>(edges.get()), cap, &nEdges, stream);
      if (rc != B200MOL_OK) fail(rc, "%s", g_lastError.c_str());
      if (nEdges <= cap) break;
      B200_REQUIRE(attempt == 0, "edge list overflow after resize");
      cap = nEdges;
    }
    const int rc = b200mol_butina_from_edges(n, counts.get(), reinterpret_cast<const int32_t*>(edges.get()), nEdges,
                                             d_cluster_ids, d_centroids, d_n_clusters, h_n_clusters, stream);
    if (rc != B200MOL_OK) fail(rc, "%s", g_lastError.c_str());
  });
}

extern "C" int b200mol_butina_dense(const double* d_dist, size_t n, double cutoff, int32_t* d_cluster_ids,
                                    int32_t* d_centroids, int32_t* d_n_clusters, int32_t* h_n_clusters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(n < (1ull << 31), "too many points");
    cudaStream_t s = asStream(stream);
    if (n == 0) {
      if (h_n_clusters) *h_n_clusters = 0;
      if (d_n_clusters) B200_CUDA(cudaMemsetAsync(d_n_clusters, 0, sizeof(int32_t), s));
      return;
    }
    B200_REQUIRE(d_dist && d_cluster_ids, "null pointer");
    const int        N = static_cast<int>(n);
    Scratch<int32_t> counts(n, s);
    Scratch<int32_t> centroidsOwn(d_centroids ? 0 : n, s);
    int32_t*         centroids = d_centroids ? d_centroids : centroidsOwn.get();
    Scratch<int32_t> nClOwn(1, s);
    int32_t*         dNCl = d_n_clusters ? d_n_clusters : nClOwn.get();

    denseRowKernel<0><<<N, 256, 0, s>>>(d_dist, N, cutoff, counts.get(), nullptr, nullptr);
    B200_LAUNCHED();
    Scratch<long long> offsets(n + 1, s);
    scanOffsets(counts.get(), N, offsets.get(), s);
    long long total = 0;
    B200_CUDA(cudaMemcpyAsync(&total, offsets.get() + n, sizeof(long long), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));  // documented sync: adjacency size
    Scratch<int> adj(static_cast<size_t>(total) + 1, s);
    denseRowKernel<1><<<N, 256, 0, s>>>(d_dist, N, cutoff, nullptr, offsets.get(), adj.get());
    B200_LAUNCHED();
    clusterFromCsr(N, offsets.get(), adj.get(), counts.get(), d_cluster_ids, centroids, dNCl, s);
    if (h_n_clusters) {
      B200_CUDA(cudaMemcpyAsync(h_n_clusters, dNCl, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
    }
  });
}
