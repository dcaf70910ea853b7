// The library's options: b200mol_set_option and b200mol_get_option both look the key up in one table, whose row says
// where the value lives and which values a write accepts. Adding an option is its variable (options.cuh), one row here
// and its documentation in include/b200mol.h.
#include <algorithm>
#include <cstring>

#include "common.cuh"
#include "options.cuh"

namespace b200 {

long long g_tensorMinPairs = 1ll << 24;  // pair count from which the passes run on the tensor-core tile (< 0: never)

namespace {

// Where a value lives: a host variable, or a word of a file's device counters.
struct Value {
  int*                i   = nullptr;
  long long*          ll  = nullptr;
  unsigned long long* ull = nullptr;
  unsigned long long (*counter)(int) = nullptr;
  int word = 0;
  constexpr Value(int* p) : i(p) {}
  constexpr Value(long long* p) : ll(p) {}
  constexpr Value(unsigned long long* p) : ull(p) {}
  constexpr Value(unsigned long long (*read)(int), int w) : counter(read), word(w) {}
  long long get() const {
    if (i) return *i;
    if (ll) return *ll;
    return static_cast<long long>(ull ? *ull : counter(word));
  }
  void set(long long v) const {  // (writable options are int or long long)
    if (i) *i = static_cast<int>(v);
    else *ll = v;
  }
};

enum Accepts {
  kReadOnly,
  kAny,
  kBool,            // stored as value != 0
  kRange,           // lo <= value <= hi
  kOneTwoFour,      // 1, 2 or 4
  kNoneIfNegative,  // any; a negative value is stored as -1
  kClamp,           // value >= lo; stored as min(value, hi)
};

struct Option {
  const char* key;
  Value       value;
  Accepts     accepts;
  long long   lo = 0, hi = 0;
  const char* refusal = nullptr;  // the error for a refused value, after the key
};

constexpr long long kBelow2To31 = (1ll << 31) - 1;

constexpr Option kOptions[] = {
    {"similarity_tensor_min_pairs", &g_tensorMinPairs, kAny},
    {"similarity_tensor_cluster", &g_tensorCluster, kRange, 0, 3, "must be 0, 1, 2 or 3"},
    {"similarity_superpose", &g_superpose, kOneTwoFour, 0, 0, "must be 1, 2 or 4"},
    {"similarity_superpose_cols", &g_superposeCols, kOneTwoFour, 0, 0, "must be 1, 2 or 4"},
    {"similarity_superpose_auto", &g_superposeAuto, kBool},
    {"similarity_pipeline_chunks", &g_pipelineChunks, kRange, 1, 8, "must be in [1, 8]"},
    {"similarity_popcount_band", &g_popcountBand, kBool},
    {"similarity_superpose_last", &g_superposeLast, kReadOnly},
    {"similarity_candidates_last", &g_candidatesLast, kReadOnly},
    {"similarity_units_planned_last", &g_unitsPlanned, kReadOnly},
    {"similarity_units_last", {readWalkCounter, 0}, kReadOnly},
    {"similarity_tiles_last", {readWalkCounter, 1}, kReadOnly},
    {"topk_slab_cols", &g_topkSlabCols, kRange, 0, kBelow2To31, "must be in [0, 2^31)"},
    {"topk_slabs_last", &g_topkSlabsLast, kReadOnly},
    {"topk_candidates_last", {readTopkStat, 0}, kReadOnly},
    {"topk_rows_redone_last", {readTopkStat, 1}, kReadOnly},
    {"maxmin_mode", &g_maxminMode, kRange, 0, 1, "must be 0 (dense) or 1 (deferred)"},
    {"maxmin_resident_rows", &g_maxminResidentRows, kNoneIfNegative},
    {"maxmin_resident_last", &g_maxminResidentLast, kReadOnly},
    {"maxmin_distances_last", {readMaxminStat, 0}, kReadOnly},
    {"maxmin_popcount_skips_last", {readMaxminStat, 1}, kReadOnly},
    {"leader_window_rows", &g_leaderWindowRows, kRange, 0, kBelow2To31, "must be in [0, 2^31)"},
    {"leader_windows_last", &g_leaderWindowsLast, kReadOnly},
    {"leader_bulk_pairs_last", &g_leaderBulkPairsLast, kReadOnly},
    {"leader_window_pairs_last", {readLeaderStat, 0}, kReadOnly},
    {"leader_block_pairs_last", {readLeaderStat, 1}, kReadOnly},
    {"count_neighbor_pairs_last", {readCountStat, 0}, kReadOnly},
    {"rmsd_match_chunk", &g_rmsdMatchChunk, kRange, 0, kBelow2To31, "must be in [0, 2^31)"},
    {"rmsd_match_chunks_last", &g_rmsdMatchChunksLast, kReadOnly},
    {"morgan_global_slab_last", &g_morganGlobalSlabLast, kReadOnly},
    // huge = the stepwise loop only
    {"butina_min_round_commits", &g_butinaMinCommits, kClamp, 0, 1000000000, "must be >= 0"},
    {"bfgs_ctas_per_sm", &g_bfgsCtasPerSm, kRange, 1, 8, "must be in [1, 8]"},
    {"bfgs_l2_persist", &g_bfgsL2Persist, kBool},
    {"etkdg_hessian_fp64", &g_etkdgHessianFp64, kBool},
};

const Option& find(const char* key) {
  for (const Option& o : kOptions)
    if (std::strcmp(o.key, key) == 0) return o;
  fail(B200MOL_ERR_INVALID, "unknown option '%s'", key);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_set_option(const char* key, long long value) {
  return guarded([&] {
    B200_REQUIRE(key, "null key");
    const Option& o = find(key);
    switch (o.accepts) {
      case kReadOnly: fail(B200MOL_ERR_INVALID, "option '%s' is read-only", key);
      case kAny: break;
      case kBool: value = value != 0; break;
      case kRange: B200_REQUIRE(value >= o.lo && value <= o.hi, "%s %s", key, o.refusal); break;
      case kOneTwoFour: B200_REQUIRE(value == 1 || value == 2 || value == 4, "%s %s", key, o.refusal); break;
      case kNoneIfNegative: value = std::max(value, -1ll); break;
      case kClamp:
        B200_REQUIRE(value >= o.lo, "%s %s", key, o.refusal);
        value = std::min(value, o.hi);
        break;
    }
    o.value.set(value);
  });
}

extern "C" int b200mol_get_option(const char* key, long long* value) {
  return guarded([&] {
    B200_REQUIRE(key && value, "null pointer");
    *value = find(key).value.get();
  });
}
