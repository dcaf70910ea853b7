// N x M popcount similarity over packed u32 fingerprints (Tanimoto / cosine), sm_90a.
//
// One CTA = one 128 x 128 tile of pairs. The two fingerprint blocks ([128 rows][<=128 B] per K chunk) are staged into
// shared memory by TMA (cp.async.bulk.tensor.2d, hardware swizzle so that 16-byte LDS is bank-conflict free) and
// signalled through mbarriers; each thread owns an 8 x 8 register tile of integer intersection counts
// (LOP3 + POPC + IADD). Epilogues: fp64 similarity matrix (streaming stores), or thresholded neighbour counts with an
// optional edge list (the fused path that never materialises the matrix).
//
// Replaces src/similarity_kernels.cu:104-409 (tile kernels) and nvmolkit/_fusedButina.py:99-179 of the reference;
// written from scratch (the reference stages with scalar 4-byte loads and an emulated b1 mma.sync).
#include <cub/device/device_scan.cuh>

#include "profile.cuh"
#include "similarity.cuh"
#include "tma.cuh"

namespace b200 {

thread_local std::string g_lastError;
std::atomic<uint64_t>    g_launchCount{0};
bool                               g_profileOn = false;
std::mutex                         g_profileMutex;
std::map<std::string, PhaseEvents> g_phases;

namespace {

constexpr int kBM      = 128;
constexpr int kBN      = 128;
constexpr int kThreads = 256;
constexpr int kStages  = 2;   // K chunks resident at once
constexpr int kChunkW  = 32;  // u32 words per K chunk (128 B)
constexpr int kGroupM  = 32;  // tile rows per L2 reuse group

struct TileParams {
  size_t   nX, nY;
  int      words, innerWords, nChunks, swzMask;
  uint32_t tilesM, tilesN;
  const int32_t* popX;
  const int32_t* popY;
  double*        out;
  const uint16_t* thresh;  // Tanimoto count: min intersection for a hit, indexed by |A|+|B|
  double          cutoff;
  int             sign;
  int32_t*        rowCounts;
  int             symmetric;
  uint32_t        groupOffset, groupStride;  // multi-GPU: this rank owns tile-row groups offset, offset+stride, ...
  int2*           edges;
  unsigned long long* edgeCursor;
  unsigned long long  edgeCap;
};

__global__ void rowPopcountKernel(const uint32_t* __restrict__ fp, size_t n, int words, int32_t* __restrict__ pop) {
  const size_t row  = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int    lane = threadIdx.x & 31;
  if (row >= n) return;
  int s = 0;
  for (int w = lane; w < words; w += 32) s += __popc(fp[row * words + w]);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) pop[row] = s;
}

// thresh[s] = smallest intersection c such that a pair with |A|+|B| = s is a neighbour, i.e. the fp64 predicate
// `1.0 - sim <= cutoff` holds with sim = (c == 0 || u == 0) ? 0 : c/u, u = s - c. 0xFFFF = never.
// The predicate is monotone in c, so the hot loop tests `c >= thresh[s]` with integers and stays bit-identical to the
// fp64 evaluation a CPU makes.
__global__ void threshTableKernel(int maxS, double cutoff, uint16_t* __restrict__ thresh) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > maxS) return;
  // explicit round-to-nearest intrinsics: never contracted into an FMA, so the result is the two-rounding value a CPU
  // computes for `1.0 - c/u`
  auto passes = [&](int c) {
    const int    u   = s - c;
    const double sim = (c == 0 || u == 0) ? 0.0 : __ddiv_rn(static_cast<double>(c), static_cast<double>(u));
    return __dsub_rn(1.0, sim) <= cutoff;
  };
  // c/(s - c) grows with c and correctly rounded division and subtraction keep the order, so the smallest passing c is
  // found by bisection over [0, s/2] (a linear scan cost 0.2 ms per table: 2048 dependent fp64 divisions per thread)
  int found = 0xFFFF;
  int lo = 0, hi = s / 2;
  if (passes(hi)) {
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (passes(mid)) hi = mid;
      else lo = mid + 1;
    }
    found = lo;
  }
  thresh[s] = static_cast<uint16_t>(found);
}

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

template <int MODE>
__global__ void __launch_bounds__(kThreads, 2)
  simTileKernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY, const TileParams p) {
  extern __shared__ __align__(1024) uint8_t smemRaw[];
  __shared__ uint64_t                      fullBar[kStages];
  __shared__ int                           colAcc[kBN];

  // ---- tile coordinates: groups of kGroupM tile-rows sweep all tile-columns (Y tiles reused out of L2) ----
  const uint32_t perGroup = kGroupM * p.tilesN;
  const uint32_t group    = (blockIdx.x / perGroup) * p.groupStride + p.groupOffset;
  const uint32_t inGroup  = blockIdx.x % perGroup;
  if (group * kGroupM >= p.tilesM) return;
  const uint32_t gRows    = min(static_cast<uint32_t>(kGroupM), p.tilesM - group * kGroupM);
  const uint32_t tm       = group * kGroupM + inGroup % gRows;
  const uint32_t tn       = inGroup / gRows;
  if (tn >= p.tilesN) return;
  if (p.symmetric && tn < tm) return;

  const int tid = threadIdx.x;
  const int tx  = tid & 15;
  const int ty  = tid >> 4;

  const uint32_t innerBytes = p.innerWords * 4;
  const uint32_t tileBytes  = kBM * innerBytes;  // one operand, one chunk
  // 1024-byte aligned stage buffers (swizzle atoms need it)
  const uint32_t smemBase   = (smemAddr(smemRaw) + 1023u) & ~1023u;
  const uint32_t stageBytes = 2 * tileBytes;

  if (tid == 0) {
    tmaPrefetchDesc(&tmX);
    tmaPrefetchDesc(&tmY);
    for (int s = 0; s < kStages; ++s) mbarInit(&fullBar[s], 1);
    fenceBarrierInit();
  }
  if (MODE >= kCountTanimoto && tid < kBN) colAcc[tid] = 0;
  __syncthreads();

  uint8_t* smemGeneric = smemRaw + (smemBase - smemAddr(smemRaw));
  auto     issue       = [&](int chunk, int stage) {
    mbarExpectTx(&fullBar[stage], 2 * tileBytes);
    tmaLoad2D(smemGeneric + stage * stageBytes, &tmX, chunk * kChunkW, tm * kBM, &fullBar[stage]);
    tmaLoad2D(smemGeneric + stage * stageBytes + tileBytes, &tmY, chunk * kChunkW, tn * kBN, &fullBar[stage]);
  };
  if (tid == 0) {
    for (int c = 0; c < kStages && c < p.nChunks; ++c) issue(c, c);
  }

  int acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0;

  const int      groups = p.innerWords >> 2;  // 16-byte groups per row per chunk
  const uint32_t swz    = p.swzMask;
  for (int chunk = 0; chunk < p.nChunks; ++chunk) {
    const int stage = chunk % kStages;
    mbarWait(&fullBar[stage], (chunk / kStages) & 1);
    const uint32_t xs = smemBase + stage * stageBytes;
    const uint32_t ys = xs + tileBytes;
    for (int q = 0; q < groups; ++q) {
      uint4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t off = (ty * 8 + i) * innerBytes + q * 16;
        a[i]               = lds128(xs + (off ^ (((off >> 7) & swz) << 4)));
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t off = (tx + 16 * j) * innerBytes + q * 16;
        const uint4    b   = lds128(ys + (off ^ (((off >> 7) & swz) << 4)));
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][j] += __popc(a[i].x & b.x) + __popc(a[i].y & b.y) + __popc(a[i].z & b.z) + __popc(a[i].w & b.w);
        }
      }
    }
    if (chunk + kStages < p.nChunks) {  // refill this stage (only for fingerprints wider than 2 chunks)
      __syncthreads();
      if (tid == 0) issue(chunk + kStages, stage);
    }
  }

  // ---- epilogue ----
  const size_t row0 = static_cast<size_t>(tm) * kBM + ty * 8;
  const size_t col0 = static_cast<size_t>(tn) * kBN + tx;
  int          pa[8], pb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) pa[i] = (row0 + i < p.nX) ? __ldg(p.popX + row0 + i) : 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) pb[j] = (col0 + 16 * j < p.nY) ? __ldg(p.popY + col0 + 16 * j) : 0;

  if constexpr (MODE == kMaterialiseTanimoto || MODE == kMaterialiseCosine) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (row0 + i >= p.nX) break;
      double* orow = p.out + (row0 + i) * p.nY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const size_t col = col0 + 16 * j;
        if (col >= p.nY) continue;
        const int c = acc[i][j];
        double    v = 0.0;
        if (c != 0) {
          if constexpr (MODE == kMaterialiseTanimoto) {
            v = __ddiv_rn(static_cast<double>(c), static_cast<double>(pa[i] + pb[j] - c));
          } else {
            v = __ddiv_rn(static_cast<double>(c),
                          __dsqrt_rn(__dmul_rn(static_cast<double>(pa[i]), static_cast<double>(pb[j]))));
          }
        }
        __stcs(orow + col, v);
      }
    }
  } else {
    const bool diag = p.symmetric && (tm == tn);
    unsigned long long hits = 0ull;  // bit (i*8+j)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const size_t gr = row0 + i, gc = col0 + 16 * j;
        bool         ok = (gr < p.nX) && (gc < p.nY);
        if (p.symmetric) ok = ok && (diag ? (gr < gc) : true);
        const int c = acc[i][j];
        bool      h;
        if constexpr (MODE == kCountTanimoto) {
          h = c >= static_cast<int>(__ldg(p.thresh + pa[i] + pb[j]));
        } else {
          const double sim =
            (c == 0) ? 0.0
                     : __ddiv_rn(static_cast<double>(c),
                                 __dsqrt_rn(__dmul_rn(static_cast<double>(pa[i]), static_cast<double>(pb[j]))));
          h = (__dsub_rn(1.0, sim) <= p.cutoff);
        }
        if (ok && h) hits |= 1ull << (i * 8 + j);
      }
    }
    // In symmetric mode each unordered pair is visited once (gr < gc): credit both endpoints.
    const unsigned anyHit = __ballot_sync(0xffffffffu, hits != 0ull);
    if (anyHit) {
      // rows: reduce over the 16 tx lanes of a half-warp
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int v = __popcll(hits & (0xFFull << (i * 8)));
#pragma unroll
        for (int o = 8; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (tx == 0 && v) atomicAdd(p.rowCounts + row0 + i, p.sign * v);
      }
      if (p.symmetric) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int v = __popcll(hits & (0x0101010101010101ull << j));
          if (v) atomicAdd(&colAcc[tx + 16 * j], v);
        }
      }
      if (p.edges) {
        const int      mine  = __popcll(hits);
        int            incl  = mine;
        const int      lane  = tid & 31;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        const int          total = __shfl_sync(0xffffffffu, incl, 31);
        unsigned long long base  = 0;
        if (lane == 31) base = atomicAdd(p.edgeCursor, static_cast<unsigned long long>(total));
        base                     = __shfl_sync(0xffffffffu, base, 31);
        unsigned long long at    = base + incl - mine;
        unsigned long long h     = hits;
        while (h) {
          const int b = __ffsll(static_cast<long long>(h)) - 1;
          h &= h - 1;
          if (at < p.edgeCap) p.edges[at] = make_int2(static_cast<int>(row0 + (b >> 3)), static_cast<int>(col0 + 16 * (b & 7)));
          ++at;
        }
      }
    }
    if (p.symmetric) {
      __syncthreads();
      if (tid < kBN) {
        const int v = colAcc[tid];
        if (v) atomicAdd(p.rowCounts + static_cast<size_t>(tn) * kBN + tid, p.sign * v);
      }
    }
  }
}

template <int MODE>
void launchTile(const CUtensorMap& tmX, const CUtensorMap& tmY, const TileParams& tp, size_t smemBytes, cudaStream_t s) {
  static bool attrSet[kMaxDevices] = {};  // per instantiation and device
  if (!attrSet[currentDeviceSlot()]) {
    B200_CUDA(cudaFuncSetAttribute(simTileKernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attrSet[currentDeviceSlot()] = true;
  }
  const uint64_t groupsM = (tp.tilesM + kGroupM - 1) / kGroupM;
  if (tp.groupOffset >= groupsM) return;
  const uint64_t myGroups = (groupsM - tp.groupOffset + tp.groupStride - 1) / tp.groupStride;
  const uint64_t blocks   = myGroups * kGroupM * tp.tilesN;
  B200_REQUIRE(blocks < (1ull << 31), "similarity grid too large (%llu tiles)", static_cast<unsigned long long>(blocks));
  simTileKernel<MODE><<<static_cast<unsigned>(blocks), kThreads, smemBytes, s>>>(tmX, tmY, tp);
  B200_LAUNCHED();
}

}  // namespace

bool launchSimilarityTensor(SimMode mode, const SimLaunch& q, cudaStream_t s);
extern int g_bfgsCtasPerSm;
extern int g_bfgsL2Persist;
extern int g_etkdgHessianFp64;
extern int g_butinaMinCommits;
extern int g_tensorCluster;
extern int g_superpose;
extern int g_superposeLast;
extern int g_superposeCols;
extern int g_superposeAuto;
extern int g_pipelineChunks;
extern unsigned long long g_candidatesLast;
long long g_tensorMinPairs = 1ll << 24;  // pair count from which the passes run on the tensor-core tile (< 0: never)

void launchThreshTable(int maxS, double cutoff, uint16_t* thresh, cudaStream_t s) {
  threshTableKernel<<<(maxS + 1 + 127) / 128, 128, 0, s>>>(maxS, cutoff, thresh);
  B200_LAUNCHED();
}

void launchRowPopcount(const uint32_t* fp, size_t n, int words, int32_t* pop, cudaStream_t s) {
  if (n == 0) return;
  const size_t threads = n * 32;
  rowPopcountKernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, s>>>(fp, n, words, pop);
  B200_LAUNCHED();
}

void launchSimilarity(SimMode mode, const SimLaunch& q, cudaStream_t s) {
  B200_REQUIRE(q.words > 0 && q.words % 4 == 0 && q.words <= 128,
               "fingerprint width must be a multiple of 128 bits and at most 4096 bits (got %d words)", q.words);
  if (q.nX == 0 || q.nY == 0) return;
  B200_REQUIRE(q.nX < (1ull << 31) && q.nY < (1ull << 31), "too many fingerprints");
  if (mode != kCountCosine && g_tensorMinPairs >= 0 &&
      static_cast<double>(q.nX) * static_cast<double>(q.nY) >= static_cast<double>(g_tensorMinPairs) &&
      (reinterpret_cast<uintptr_t>(q.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q.y) & 15) == 0) {
    if (launchSimilarityTensor(mode, q, s)) return;
  }
  B200_REQUIRE((reinterpret_cast<uintptr_t>(q.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q.y) & 15) == 0,
               "fingerprint buffers must be 16-byte aligned");

  TileParams tp{};
  tp.nX         = q.nX;
  tp.nY         = q.nY;
  tp.words      = q.words;
  // The box is 4, 8, 16 or 32 words wide (16, 32, 64 or 128 B): exactly the span of the swizzle makeTensorMap2D picks
  // for it, so box rows lie back to back in shared memory as the tile's address arithmetic assumes. A narrower
  // fingerprint (384, 640, 768 or 896 bits) gets the next such box; TMA zero-fills the words past the row end, and
  // they add nothing to the counts, as in the last chunk of a fingerprint wider than 1024 bits.
  tp.innerWords = 4;
  while (tp.innerWords < q.words && tp.innerWords < kChunkW) tp.innerWords <<= 1;
  tp.nChunks    = (q.words + kChunkW - 1) / kChunkW;
  tp.tilesM     = static_cast<uint32_t>((q.nX + kBM - 1) / kBM);
  tp.tilesN     = static_cast<uint32_t>((q.nY + kBN - 1) / kBN);
  tp.out        = q.out;
  tp.cutoff     = q.cutoff;
  tp.sign       = q.sign;
  tp.rowCounts  = q.rowCounts;
  tp.symmetric  = q.symmetric ? 1 : 0;
  tp.groupOffset = q.groupOffset;
  tp.groupStride = q.groupStride < 1 ? 1 : q.groupStride;
  tp.edges      = q.edges;
  tp.edgeCursor = q.edgeCursor;
  tp.edgeCap    = q.edgeCap;
  if (q.symmetric) B200_REQUIRE(q.x == q.y && q.nX == q.nY, "symmetric mode needs x == y");

  CUtensorMap tmX, tmY;
  tp.swzMask = makeTensorMap2D(&tmX, q.x, q.nX, q.words, kBM, tp.innerWords);
  makeTensorMap2D(&tmY, q.y, q.nY, q.words, kBN, tp.innerWords);

  const bool        same = (q.x == q.y && q.nX == q.nY);
  Scratch<int32_t>  popX(q.nX, s);
  Scratch<int32_t>  popYown(same ? 0 : q.nY, s);
  launchRowPopcount(q.x, q.nX, q.words, popX.get(), s);
  if (!same) launchRowPopcount(q.y, q.nY, q.words, popYown.get(), s);
  tp.popX = popX.get();
  tp.popY = same ? popX.get() : popYown.get();

  Scratch<uint16_t> thresh;
  if (mode == kCountTanimoto) {
    const int maxS = 2 * q.words * 32;
    thresh         = Scratch<uint16_t>(maxS + 1, s);
    threshTableKernel<<<(maxS + 1 + 127) / 128, 128, 0, s>>>(maxS, q.cutoff, thresh.get());
    B200_LAUNCHED();
    tp.thresh = thresh.get();
  }

  const int    stages    = tp.nChunks < kStages ? tp.nChunks : kStages;
  const size_t smemBytes = static_cast<size_t>(stages) * 2 * kBM * tp.innerWords * 4 + 1024;
  switch (mode) {
    case kMaterialiseTanimoto: launchTile<kMaterialiseTanimoto>(tmX, tmY, tp, smemBytes, s); break;
    case kMaterialiseCosine: launchTile<kMaterialiseCosine>(tmX, tmY, tp, smemBytes, s); break;
    case kCountTanimoto: launchTile<kCountTanimoto>(tmX, tmY, tp, smemBytes, s); break;
    case kCountCosine: launchTile<kCountCosine>(tmX, tmY, tp, smemBytes, s); break;
  }
}

}  // namespace b200

// ------------------------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------------------------
using namespace b200;

extern "C" const char* b200mol_last_error(void) { return g_lastError.c_str(); }
extern "C" int         b200mol_abi_version(void) { return 2; }
extern "C" uint64_t    b200mol_launch_count(void) { return g_launchCount.load(); }

extern "C" int b200mol_profile_enable(int on) {
  g_profileOn = on != 0;
  return B200MOL_OK;
}
extern "C" int b200mol_profile_read(const char* phase, float* ms) {
  return guarded([&] {
    B200_REQUIRE(phase && ms, "null pointer");
    std::lock_guard<std::mutex> lock(g_profileMutex);
    auto                        it = g_phases.find(phase);
    B200_REQUIRE(it != g_phases.end() && it->second.recorded, "phase '%s' was not recorded", phase);
    B200_CUDA(cudaEventSynchronize(it->second.stop));
    B200_CUDA(cudaEventElapsedTime(ms, it->second.start, it->second.stop));
  });
}

extern "C" int b200mol_set_option(const char* key, long long value) {
  return guarded([&] {
    B200_REQUIRE(key, "null key");
    const std::string k(key);
    if (k == "similarity_tensor_min_pairs") g_tensorMinPairs = value;
    else if (k == "bfgs_ctas_per_sm") {
      B200_REQUIRE(value >= 1 && value <= 8, "bfgs_ctas_per_sm must be in [1, 8]");
      g_bfgsCtasPerSm = static_cast<int>(value);
    }
    else if (k == "bfgs_l2_persist") g_bfgsL2Persist = value != 0;
    else if (k == "etkdg_hessian_fp64") g_etkdgHessianFp64 = value != 0;
    else if (k == "similarity_superpose") {
      B200_REQUIRE(value == 1 || value == 2 || value == 4, "similarity_superpose must be 1, 2 or 4");
      g_superpose = static_cast<int>(value);
    }
    else if (k == "similarity_superpose_cols") {
      B200_REQUIRE(value == 1 || value == 2 || value == 4, "similarity_superpose_cols must be 1, 2 or 4");
      g_superposeCols = static_cast<int>(value);
    }
    else if (k == "similarity_superpose_auto") g_superposeAuto = value != 0;
    else if (k == "similarity_pipeline_chunks") {
      B200_REQUIRE(value >= 1 && value <= 8, "similarity_pipeline_chunks must be in [1, 8]");
      g_pipelineChunks = static_cast<int>(value);
    }
    else if (k == "similarity_tensor_cluster") {
      B200_REQUIRE(value >= 0 && value <= 3, "similarity_tensor_cluster must be 0, 1, 2 or 3");
      g_tensorCluster = static_cast<int>(value);
    }
    else if (k == "butina_min_round_commits") {
      B200_REQUIRE(value >= 0, "butina_min_round_commits must be >= 0");
      g_butinaMinCommits = static_cast<int>(value > 1000000000 ? 1000000000 : value);  // huge = stepwise loop only
    }
    else fail(B200MOL_ERR_INVALID, "unknown option '%s'", key);
  });
}

extern "C" int b200mol_get_option(const char* key, long long* value) {
  return guarded([&] {
    B200_REQUIRE(key && value, "null pointer");
    const std::string k(key);
    if (k == "similarity_tensor_min_pairs") *value = g_tensorMinPairs;
    else if (k == "bfgs_ctas_per_sm") *value = g_bfgsCtasPerSm;
    else if (k == "bfgs_l2_persist") *value = g_bfgsL2Persist;
    else if (k == "etkdg_hessian_fp64") *value = g_etkdgHessianFp64;
    else if (k == "similarity_tensor_cluster") *value = g_tensorCluster;
    else if (k == "similarity_superpose") *value = g_superpose;
    else if (k == "similarity_superpose_cols") *value = g_superposeCols;
    else if (k == "similarity_superpose_auto") *value = g_superposeAuto;
    else if (k == "similarity_pipeline_chunks") *value = g_pipelineChunks;
    else if (k == "similarity_candidates_last") *value = static_cast<long long>(g_candidatesLast);
    else if (k == "similarity_superpose_last") *value = g_superposeLast;  // read-only: pairs per accumulator of the last pass
    else if (k == "butina_min_round_commits") *value = g_butinaMinCommits;
    else fail(B200MOL_ERR_INVALID, "unknown option '%s'", key);
  });
}

// Keep stream-ordered scratch (GBs for the 1M x 1M pass) in the pool across synchronisations instead of returning it to
// the OS at every sync (the default release threshold is 0).
static void retainPoolMemory(int dev) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
}

extern "C" int b200mol_check_device(int dev) {
  return guarded([&] {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || dev < 0 || dev >= n)
      fail(B200MOL_ERR_NODEVICE, "no CUDA device %d visible: libb200mol has no CPU fallback", dev);
    int major = 0, minor = 0;
    B200_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    B200_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0)
      fail(B200MOL_ERR_NODEVICE, "device %d is compute capability %d.%d; libb200mol is built for sm_90a (H100) only", dev, major,
           minor);
    retainPoolMemory(dev);
  });
}

extern "C" int b200mol_free_async(void* d_ptr, void* stream) {
  return guarded([&] {
    if (d_ptr) B200_CUDA(cudaFreeAsync(d_ptr, asStream(stream)));
  });
}

static int crossImpl(SimMode mode, const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words,
                     double* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(nA == 0 || d_a, "null fingerprint pointer");
    if (!d_b) {
      d_b = d_a;
      nB  = nA;
    }
    B200_REQUIRE(nA == 0 || nB == 0 || d_out, "null output pointer");
    SimLaunch q;
    q.x     = d_a;
    q.y     = d_b;
    q.nX    = nA;
    q.nY    = nB;
    q.words = words;
    q.out   = d_out;
    launchSimilarity(mode, q, asStream(stream));
  });
}

extern "C" int b200mol_tanimoto_cross(const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words,
                                      double* d_out, void* stream) {
  return crossImpl(kMaterialiseTanimoto, d_a, nA, d_b, nB, words, d_out, stream);
}
extern "C" int b200mol_cosine_cross(const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words,
                                    double* d_out, void* stream) {
  return crossImpl(kMaterialiseCosine, d_a, nA, d_b, nB, words, d_out, stream);
}

extern "C" int b200mol_tanimoto_count_ge(const uint32_t* d_x, size_t nX, const uint32_t* d_y, size_t nY, int words,
                                         int metric, double cutoff, int sign, int32_t* d_counts, void* stream) {
  return guarded([&] {
    B200_REQUIRE(metric == B200MOL_METRIC_TANIMOTO || metric == B200MOL_METRIC_COSINE, "unknown metric %d", metric);
    B200_REQUIRE(sign == 1 || sign == -1, "sign must be +1 or -1");
    B200_REQUIRE(nX == 0 || (d_x && d_counts), "null pointer");
    if (!d_y) {
      d_y = d_x;
      nY  = nX;
    }
    SimLaunch q;
    q.x         = d_x;
    q.y         = d_y;
    q.nX        = nX;
    q.nY        = nY;
    q.words     = words;
    q.cutoff    = cutoff;
    q.sign      = sign;
    q.rowCounts = d_counts;
    launchSimilarity(metric == B200MOL_METRIC_TANIMOTO ? kCountTanimoto : kCountCosine, q, asStream(stream));
  });
}

// Host-in / host-out: row blocks of A through two device buffers, D2H of block k overlapped with compute of block k+1.
extern "C" int b200mol_similarity_cross_host(const uint32_t* h_a, size_t nA, const uint32_t* h_b, size_t nB, int words,
                                             int metric, double* h_out, size_t maxDeviceBytes) {
  return guarded([&] {
    B200_REQUIRE(metric == B200MOL_METRIC_TANIMOTO || metric == B200MOL_METRIC_COSINE, "unknown metric %d", metric);
    if (!h_b) {
      h_b = h_a;
      nB  = nA;
    }
    if (nA == 0 || nB == 0) return;
    B200_REQUIRE(h_a && h_out, "null pointer");
    if (maxDeviceBytes == 0) maxDeviceBytes = size_t(8) << 30;
    size_t rowsPer = maxDeviceBytes / 2 / (nB * sizeof(double));
    rowsPer        = rowsPer / kBM * kBM;
    if (rowsPer < static_cast<size_t>(kBM)) rowsPer = kBM;
    if (rowsPer > nA) rowsPer = nA;
    cudaStream_t st[2];
    cudaEvent_t  done[2];
    for (int i = 0; i < 2; ++i) {
      B200_CUDA(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
      B200_CUDA(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
    }
    uint32_t *dA = nullptr, *dB = nullptr;
    double*   dOut[2] = {nullptr, nullptr};
    try {
      B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&dA), nA * words * sizeof(uint32_t)));
      B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&dB), nB * words * sizeof(uint32_t)));
      for (int i = 0; i < 2; ++i) B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&dOut[i]), rowsPer * nB * sizeof(double)));
      B200_CUDA(cudaMemcpyAsync(dA, h_a, nA * words * sizeof(uint32_t), cudaMemcpyHostToDevice, st[0]));
      B200_CUDA(cudaMemcpyAsync(dB, h_b, nB * words * sizeof(uint32_t), cudaMemcpyHostToDevice, st[0]));
      B200_CUDA(cudaEventRecord(done[0], st[0]));
      B200_CUDA(cudaStreamWaitEvent(st[1], done[0], 0));
      int buf = 0;
      for (size_t r0 = 0; r0 < nA; r0 += rowsPer, buf ^= 1) {
        const size_t rows = (nA - r0 < rowsPer) ? nA - r0 : rowsPer;
        SimLaunch    q;
        q.x     = dA + r0 * words;
        q.y     = dB;
        q.nX    = rows;
        q.nY    = nB;
        q.words = words;
        q.out   = dOut[buf];
        launchSimilarity(metric == B200MOL_METRIC_TANIMOTO ? kMaterialiseTanimoto : kMaterialiseCosine, q, st[buf]);
        B200_CUDA(cudaMemcpyAsync(h_out + r0 * nB, dOut[buf], rows * nB * sizeof(double), cudaMemcpyDeviceToHost, st[buf]));
      }
      B200_CUDA(cudaStreamSynchronize(st[0]));
      B200_CUDA(cudaStreamSynchronize(st[1]));
    } catch (...) {
      cudaFree(dA);
      cudaFree(dB);
      cudaFree(dOut[0]);
      cudaFree(dOut[1]);
      for (int i = 0; i < 2; ++i) {
        cudaStreamDestroy(st[i]);
        cudaEventDestroy(done[i]);
      }
      throw;
    }
    cudaFree(dA);
    cudaFree(dB);
    cudaFree(dOut[0]);
    cudaFree(dOut[1]);
    for (int i = 0; i < 2; ++i) {
      cudaStreamDestroy(st[i]);
      cudaEventDestroy(done[i]);
    }
  });
}
