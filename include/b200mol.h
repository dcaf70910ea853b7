/*
 * b200mol.h — C-ABI of libb200mol.so, the H100 (sm_90a) batched-molecule hot path.
 *
 * Every entry point is `extern "C"`, takes plain pointers + sizes + an opaque stream
 * (a cudaStream_t passed as void*), returns an int status (0 = OK) and never throws.
 * `b200mol_last_error()` returns the thread-local message of the last failing call.
 *
 * Pointer naming:  d_* = device memory, h_* = host memory.  Inputs are borrowed.
 * Outputs are caller-allocated unless the comment says "callee-allocated"
 * (then release with b200mol_free_async on the same stream).
 * Nothing here synchronises the stream unless the comment says so.
 *
 * Each declaration cites the interface of the reference (NVIDIA-Digital-Bio/nvMolKit
 * v0.5.0, paths relative to its checkout) that it replaces.
 */
#ifndef B200MOL_H
#define B200MOL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MOL_OK 0
#define B200MOL_ERR_INVALID 1 /* bad argument (maps to ValueError / std::invalid_argument) */
#define B200MOL_ERR_CUDA 2    /* CUDA runtime failure (maps to RuntimeError / CudaBadReturnCode) */
#define B200MOL_ERR_NODEVICE 3 /* no sm_90 device visible: the product path has no CPU fallback */

#define B200MOL_METRIC_TANIMOTO 0
#define B200MOL_METRIC_COSINE 1

const char* b200mol_last_error(void);
/* ABI version, bumped on any signature change. */
int b200mol_abi_version(void);
/* Number of kernel launches issued by this library in this process (bench.py's gpu_launches). */
uint64_t b200mol_launch_count(void);
/* 0 when device `dev` is compute capability 9.0; B200MOL_ERR_NODEVICE otherwise. */
int b200mol_check_device(int dev);
int b200mol_free_async(void* d_ptr, void* stream);
/* Tuning knobs (every setting computes the same results; tests/ run the variants against each other and the oracle):
 *   "similarity_tensor_min_pairs"  pair count (nX * nY) from which the similarity passes run on the wgmma tensor-core
 *                                  tile (u8 0/1 operands) instead of the SIMT popcount tile (default 2^24; 0 = always,
 *                                  < 0 = never)
 *   "similarity_tensor_cluster"    1 (default): the thresholded count pass runs in clusters of two CTAs sharing the
 *                                  column operand through TMA multicast; 3: the same pairs with the ROW operand
 *                                  stationary in shared memory for a run of 16 tile columns (fingerprints up to 1024
 *                                  bits, else as 1; half the L2 -> shared memory bytes per pair); 0: one CTA per tile;
 *                                  2: runs as 1 (kept for callers written for a CTA-pair MMA, which Hopper lacks)
 *   "similarity_superpose"         4 (default), 2 or 1: fingerprints summed into one row operand of the Butina neighbour pass
 *                                  (byte values 0..4): one accumulator then bounds that many pair counts, the
 *                                  few survivors are re-examined exactly by a second kernel; 1 = off
 *   "similarity_superpose_cols"    4 (default), 2 or 1: the same for the column operand (sums of products stay <= 16,
 *                                  exact): one accumulator bounds rows x cols pair counts. A pass whose candidate list
 *                                  overflows (dense graph) reruns with rows only, then unsuperposed - results identical
 *   "similarity_pipeline_chunks"   4 (default): from 16 row groups (131,072 fingerprints) up a superposed pass runs as that
 *                                  many chunks of its row groups; the exact verification of a chunk overlaps the tensor
 *                                  pass of the next on a second stream. 1 = off. Results identical
 *   "similarity_superpose_auto"    1 (default): a pass over >= 65,536 fingerprints first runs a pilot over a prefix
 *                                  sample per column factor and keeps the factor a cost model finds cheapest (the
 *                                  sum of rows x cols random intersections must stay below one true pair's threshold);
 *                                  0: always start from the configured factors
 *   "similarity_popcount_band"     1 (default): a neighbour pass in popcount order (superposed, its fallbacks, the
 *                                  pilot) skips, per row group of 8,192 fingerprints, the tile columns whose popcounts
 *                                  no row of the group can reach a neighbour with; 0: visits them. Results identical
 *   "topk_slab_cols"               0 (default): b200mol_similarity_topk warms its bars on the first 4,096 library
 *                                  fingerprints and sends the rest through the tensor tile in column slabs that double,
 *                                  up to 512 MB of expanded operand; > 0: warm-up (at least B200MOL_TOPK_MAX) and every
 *                                  slab take this many fingerprints. Results identical
 *   "maxmin_mode"                  b200mol_maxmin_pick: 0 (default) dense (every pick updates every item), 1 deferred
 *                                  (RDKit's lazy bound: a round catches up only the items that could still win).
 *                                  Results identical
 *   "maxmin_resident_rows"         -1 (default): b200mol_maxmin_pick keeps the pool's fingerprints in shared memory
 *                                  whenever they fit; 0: always reads them from L2 / HBM; > 0: keeps pools of at most
 *                                  this many rows (that fit). Results identical
 *   "leader_window_rows"           0 (default): b200mol_leader_pick sizes each window of the pool so that about 8,192 items
 *                                  survive its bulk pass; > 0: every window takes this many items. Results identical
 *   "rmsd_match_chunk"             0 (default): b200mol_conformer_rmsd_mapped keeps the column operands of as many mappings
 *                                  per molecule resident at once as fit 1 GiB; > 0: at most this many (fewer passes
 *                                  over the pairs against less scratch). Results identical
 *   "butina_min_round_commits"     a parallel Butina round that commits fewer clusters than this hands over to the
 *                                  one-cluster-per-step loop (default 32; 0 = rounds only, >= 1e9 = stepwise only)
 *   "etkdg_hessian_fp64"           0 (default): the embedder keeps its BFGS inverse Hessian in fp32 and sweeps it in fp32
 *                                  (update, products, row sums and per-lane column sums; only the cross-warp column
 *                                  sums and H*dGrad / H*grad are fp64; half the slab traffic); 1: in fp64, the
 *                                  reference's storage type. The MMFF / UFF minimiser always uses fp64
 *   "bfgs_l2_persist"              1: mark the inverse-Hessian slabs persisting in L2 (default 0)
 *   "bfgs_ctas_per_sm"             resident CTAs per SM of the minimiser / embedder kernels (default 3 = the register
 *                                  budget they are compiled for) */
int b200mol_set_option(const char* key, long long value);
/* Current value of an option; also "similarity_superpose_last": pairs per accumulator the last neighbour pass really ran with
 * (1 after a candidate-list overflow made it fall back), "similarity_candidates_last": how many candidates it listed, and
 * what the tensor-core count passes of the last neighbour pass walked after its pilot: "similarity_units_planned_last"
 * (work units the host sized the grids for), "similarity_units_last" and "similarity_tiles_last" (units and tiles the
 * kernels counted; these two synchronise the device). Of the last b200mol_similarity_topk: "topk_slabs_last" (column slabs
 * that went through the tensor tile), "topk_candidates_last" (pairs its epilogue listed) and "topk_rows_redone_last" (rows
 * of a slab whose candidates did not fit and that the SIMT scan redid); the last two synchronise the device. Of the last
 * b200mol_maxmin_pick: "maxmin_resident_last" (1: the pool was kept in shared memory), "maxmin_distances_last" (pair
 * distances it evaluated) and "maxmin_popcount_skips_last" (pairs the popcount bound ruled out unread); the last two
 * synchronise the device. Of the last b200mol_leader_pick: "leader_windows_last" (windows of the pool it walked),
 * "leader_bulk_pairs_last" (window x pick pairs sent through the count pass), "leader_window_pairs_last" and
 * "leader_block_pairs_last" (pairs the resolver compared against earlier picks of the same window / of the same block;
 * these two synchronise the device). Of the last b200mol_conformer_rmsd_mapped: "rmsd_match_chunks_last" (chunks of
 * mappings it ran). Of the last b200mol_morgan that launched: "morgan_global_slab_last" (1: the per-molecule slabs were
 * in device memory, 0: in shared memory). Of the last b200mol_count_neighbor_edges over at least one vector:
 * "count_neighbor_pairs_last" (pairs (i, j), i < j, its pass compared after the sum band; synchronises the device). */
int b200mol_get_option(const char* key, long long* value);
/* Per-phase CUDA-event timing inside the library (off by default). Phases: "neighbor_pass" (the N^2 tile kernel
 * alone), "csr_build", "cluster_loop", "bfgs". b200mol_profile_read waits for the phase's stop event. */
int b200mol_profile_enable(int on);
int b200mol_profile_read(const char* phase, float* ms);
/* Work counters of the conformer kernels on the current device since the last reset: two banks of 8,
 * h_out16[0..7] the embedder (b200mol_etkdg_embed), h_out16[8..15] the stand-alone minimisers (b200mol_*_minimize):
 *   [0] BFGS iterations  [1] energy evaluations  [2] gradient evaluations
 *   [3] ALGORITHMIC bytes of those iterations by the reference's scheme (SURVEY.md 8d: per iteration 3 n^2 x 8 B of
 *       inverse Hessian + (1 + line-search evaluations) x the molecule's term-record bytes) - bench.py's roofline
 *   [4] minimisations  [5] ETKDG attempts  [6] sum over iterations of n^2 (n = BFGS variables)  [7] reserved.
 * Synchronises `stream`. */
int b200mol_stats_read(uint64_t* h_out16, int reset, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fingerprint similarity.
 * Fingerprints are u32 fp[n][words], bit j of row i = fp[i][j>>5] & (1u << (j&31))
 * (reference wire format: src/data_structures/flat_bit_vect.h:129-144, nvmolkit/fingerprints.py:25-72).
 * ---------------------------------------------------------------------------------------- */

/* S[i][j] = |A_i & B_j| / |A_i | B_j| as fp64, 0 when the intersection is empty; row-major d_out[nA*nB].
 * Integer popcounts and ONE correctly rounded fp64 divide (identical to RDKit TanimotoSimilarity in fp64).
 * Replaces launchCrossTanimotoSimilarity (src/similarity_kernels.h:51-56, .cu:505-582) and
 * crossTanimotoSimilarityGpuResult (src/similarity.cpp:38-58). */
int b200mol_tanimoto_cross(const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words, double* d_out,
                           void* stream);
/* Cosine twin: |A&B| / sqrt(|A||B|), 0 when the intersection is empty.
 * Replaces launchCrossCosineSimilarity (src/similarity_kernels.cu:602-631). */
int b200mol_cosine_cross(const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words, double* d_out,
                         void* stream);
/* Host-in / host-out variant: fingerprints in host memory, result matrix to host memory, row blocks of A
 * streamed through two device buffers with overlapped D2H. Synchronous. metric = B200MOL_METRIC_*.
 * Replaces crossTanimotoSimilarityMemoryConstrained / crossSimilarityImpl (src/similarity.cpp:105-236). */
int b200mol_similarity_cross_host(const uint32_t* h_a, size_t nA, const uint32_t* h_b, size_t nB, int words, int metric,
                                  double* h_out, size_t maxDeviceBytes);

/* Fused threshold count: d_counts[i] (+= or -=, sign = +1/-1) #{ j : 1 - sim(X_i, Y_j) <= cutoff }, the comparison
 * evaluated exactly as fp64 `1.0 - c/u <= cutoff` through an integer threshold table, the similarity matrix never
 * materialised. Replaces the Triton kernel _update_neighbor_count_kernel (nvmolkit/_fusedButina.py:99-179, 249-289). */
int b200mol_tanimoto_count_ge(const uint32_t* d_x, size_t nX, const uint32_t* d_y, size_t nY, int words, int metric,
                              double cutoff, int sign, int32_t* d_counts, void* stream);

/* Exact k-nearest-neighbour search, the similarity matrix never materialised: row q of d_values / d_indices ([nQ][k],
 * caller-allocated) holds the first k columns of row q of the matrix b200mol_tanimoto_cross / b200mol_cosine_cross would
 * write for the same inputs, ordered by (value descending, column index ascending): values bit-identical to the matrix
 * entries, ties to the lowest index, the result a pure function of the inputs. d_lib = NULL searches the queries
 * themselves (self-matches included). 1 <= k <= min(nLib, B200MOL_TOPK_MAX), metric = B200MOL_METRIC_*; inputs are
 * borrowed. Asynchronous on `stream`, no host synchronisation; scratch is stream-ordered: 8 * words bytes per query
 * (expanded operand), at most 512 MB of expanded library slab, and 4 * min(1792, max(256, 8 k)) bytes of candidate slots
 * per query. Inputs of fewer than "similarity_tensor_min_pairs" pairs, or with at most 4,096 library fingerprints, are
 * scanned by a SIMT kernel; larger ones run on the wgmma tile. Both give the same bits. */
#define B200MOL_TOPK_MAX 256
int b200mol_similarity_topk(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, int metric,
                            int k, double* d_values /* [nQ][k] */, int32_t* d_indices /* [nQ][k] */, void* stream);

/* Threshold (range) similarity search, the similarity matrix never materialised: row q of the CSR result (d_indptr
 * [nQ + 1], d_indices / d_values [nnz]) lists exactly the columns j for which the fp64 value b200mol_tanimoto_cross /
 * b200mol_cosine_cross would store for (q, j) is >= threshold, in ascending column order, with values bit-identical to
 * those matrix entries; the result is a pure function of the inputs. d_lib = NULL searches the queries against
 * themselves (nLib is then ignored): the same result as passing them twice, self-matches included (1.0 for a non-empty
 * fingerprint, 0 for an empty one), from the symmetric pass over half the pairs. 0 < threshold <= 1, metric =
 * B200MOL_METRIC_*, nQ, nLib < 2^31, inputs 16-byte aligned and borrowed; arguments are checked before any device work.
 * *h_nnz = the true total nnz, always. d_indptr, d_indices and d_values are written only when nnz <= cap (the caller
 * sizes them for cap); otherwise nothing is written and the caller calls again with cap >= *h_nnz.
 * The output size is data-dependent, so the call SYNCHRONISES `stream`: once to read the listed-pair total, and once
 * more in the rare case that the pass listed more pairs than its buffer held and is rerun; the CSR is then written
 * stream-ordered on `stream`. Tanimoto runs the thresholded graph pass of the fused Butina path (symmetric for a self
 * search; superposed and in popcount order on the tensor-core tile), cosine a list mode of the tile (SIMT below
 * "similarity_tensor_min_pairs" pairs). Scratch is stream-ordered: 16 bytes per listed pair (the pair and its value; a
 * self search lists each off-diagonal pair once), 24 bytes per result entry plus CUB's radix-sort temporary storage
 * (about another 16 bytes per entry), 12 bytes per fingerprint, and what the pass itself takes (the tensor tile: 8 bits
 * per fingerprint bit of expanded operand). */
int b200mol_similarity_threshold(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib /* NULL = self */, size_t nLib, int words,
                                 int metric, double threshold, int64_t* d_indptr /* [nQ + 1] */, int32_t* d_indices /* [cap] */,
                                 double* d_values /* [cap] */, uint64_t cap, uint64_t* h_nnz, void* stream);

/* Tversky similarity, S[i][j] = c / ((alpha (a - c) + beta (b - c)) + c) with a = |A_i| (group one, the rows), b = |B_j|
 * and c = |A_i & B_j|; 0 when c = 0 (two empty fingerprints included). Integer popcounts, then each product, sum and the
 * quotient is one fp64 operation rounded to nearest, in exactly this order, never contracted into an FMA. alpha weights
 * the bits only in the row fingerprint, as RDKit's TverskySimilarity(fp1, fp2, a, b) does, so the matrix of (one, two,
 * alpha, beta) is the transpose of that of (two, one, beta, alpha). Dice, 2c / (a + b), is (0.5, 0.5); (1, 1) gives the
 * bits of b200mol_tanimoto_cross. For dyadic weights (0, 1/4, 1/2, 1, 2, ...) the value is the same for any order of
 * evaluation; for others, such as (0.3, 0.7), it may differ by a few ulp from an expanded form such as
 * alpha a + beta b + (1 - alpha - beta) c. Values lie in [0, 1]; a non-empty fingerprint has 1.0 with itself.
 * 0 <= alpha, beta <= 1000, finite (else B200MOL_ERR_INVALID). Each entry point takes the arguments of its Tanimoto /
 * cosine twin, with (alpha, beta) after `words`, and has the twin's semantics for this value:
 *   b200mol_tversky_cross       the (nA, nB) matrix, as b200mol_tanimoto_cross (d_b = NULL: A against itself)
 *   b200mol_tversky_cross_host  host in / host out in row blocks, as b200mol_similarity_cross_host
 *   b200mol_tversky_topk        exact top-k, as b200mol_similarity_topk: the first k columns of each row of the matrix by
 *                               (value descending, column ascending). In a self search the self-match need not come first
 *                               with alpha != beta: under (1, 0) every superset of the query also scores 1.0, and ties go
 *                               to the lowest index.
 *   b200mol_tversky_threshold   the CSR of the entries >= threshold, as b200mol_similarity_threshold; a self search with
 *                               alpha != beta runs the full pass over the set against itself (the value is not symmetric)
 * Dice (0.5, 0.5) runs on the Tanimoto machinery: the Dice epilogue of the matrix tiles, the Tanimoto top-k search (its
 * order is Dice's order) with the values rewritten, and the thresholded graph pass with a Dice threshold table. Other
 * weights take the cosine design: a float pre-filter on the tile that never drops a pair that could qualify, then an
 * exact fp64 recount. */
int b200mol_tversky_cross(const uint32_t* d_a, size_t nA, const uint32_t* d_b, size_t nB, int words, double alpha, double beta,
                          double* d_out, void* stream);
int b200mol_tversky_cross_host(const uint32_t* h_a, size_t nA, const uint32_t* h_b, size_t nB, int words, double alpha, double beta,
                               double* h_out, size_t maxDeviceBytes);
int b200mol_tversky_topk(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib, size_t nLib, int words, double alpha, double beta,
                         int k, double* d_values /* [nQ][k] */, int32_t* d_indices /* [nQ][k] */, void* stream);
int b200mol_tversky_threshold(const uint32_t* d_q, size_t nQ, const uint32_t* d_lib /* NULL = self */, size_t nLib, int words,
                              double alpha, double beta, double threshold, int64_t* d_indptr /* [nQ + 1] */,
                              int32_t* d_indices /* [cap] */, double* d_values /* [cap] */, uint64_t cap, uint64_t* h_nnz,
                              void* stream);

/* Tanimoto, Dice and Tversky on count vectors (RDKit's SparseIntVect / GetCountFingerprint similarity). A row is bins
 * int32 counts (d_a [nA][bins], row-major, 1 <= bins <= 4096), each in 0 .. 65535. With a = the sum of the row (group
 * one), b = the sum of the column's row and c = the sum over bins of min(row, column), the value of a pair is that of
 * b200mol_tversky_cross: 0 when c = 0, else c / ((alpha (a - c) + beta (b - c)) + c) one rounded fp64 operation at a
 * time. The count bound keeps every sum and a + b - c exact integers below 2^31, so Tanimoto (1, 1) is RDKit's
 * andSum / (v1Sum + v2Sum - andSum) and Dice (0.5, 0.5) its 2 andSum / (v1Sum + v2Sum), bit for bit; for non-dyadic
 * weights the note on b200mol_tversky_cross applies. Each entry point takes the arguments of its b200mol_tversky_* twin
 * with `bins` in place of `words`, and has its contract: the fp64 matrix, the exact top-k ((value descending, column
 * ascending), 1 <= k <= min(nLib, B200MOL_TOPK_MAX)), or the exact CSR of the entries >= threshold (0 < threshold <= 1,
 * the cap / h_nnz protocol of b200mol_similarity_threshold); d_b / d_lib = NULL: group one against itself, self-matches
 * included. Argument errors are refused before any device work; a count outside 0 .. 65535 is refused
 * (B200MOL_ERR_INVALID) after a device check whose flag is read once, so every call SYNCHRONISES `stream`, and nothing
 * is written to the outputs when it fails. Scratch is stream-ordered: each row's non-zeros as 4-byte (bin, count) pairs
 * and 12 bytes per row; top-k adds the candidate slots of b200mol_similarity_topk (12 bytes each), threshold 16 bytes per
 * listed pair and the CSR assembly of b200mol_similarity_threshold. Cosine is not defined on counts. */
int b200mol_count_cross(const int32_t* d_a, size_t nA, const int32_t* d_b, size_t nB, int bins, double alpha, double beta,
                        double* d_out, void* stream);
int b200mol_count_topk(const int32_t* d_q, size_t nQ, const int32_t* d_lib, size_t nLib, int bins, double alpha, double beta,
                       int k, double* d_values /* [nQ][k] */, int32_t* d_indices /* [nQ][k] */, void* stream);
int b200mol_count_threshold(const int32_t* d_q, size_t nQ, const int32_t* d_lib /* NULL = self */, size_t nLib, int bins,
                            double alpha, double beta, double threshold, int64_t* d_indptr /* [nQ + 1] */,
                            int32_t* d_indices /* [cap] */, double* d_values /* [cap] */, uint64_t cap, uint64_t* h_nnz,
                            void* stream);

/* MaxMin diversity picking (RDKit MaxMinPicker::LazyBitVectorPick / LazyBitVectorPickWithThreshold) over the pool
 * d_fp[0 .. nPool) ([nPool][words], 16-byte aligned). d(i, j) = 1 - s(i, j), s the fp64 value b200mol_tanimoto_cross /
 * b200mol_cosine_cross store for the pair (metric = B200MOL_METRIC_*), so two empty fingerprints are at distance 1.
 * d_picks[0 .. nFirst) = h_first (host memory, 1 <= nFirst <= pickSize, distinct pool indices; a seeded random first
 * pick is the caller's to draw); each further pick is the unpicked item with the largest min over the picks of d(i, p),
 * ties to the lowest index. threshold >= 0: the loop stops before adding a pick whose max-min is <= threshold, and
 * d_picks holds -1 past the stop; threshold < 0: no stop. *d_threshold = the max-min of the last pick the loop added,
 * -1 when it added none. 1 <= pickSize <= nPool < 2^31. Asynchronous on `stream`, no host synchronisation (h_first is
 * uploaded by one cudaMemcpyAsync from pageable memory); the pick loop is one cooperative kernel. Scratch is
 * stream-ordered: 4 bytes per pool item (popcounts), 12 bytes per CTA, and, when a CTA's slice of the pool does not fit
 * in shared memory (above about 1.9M items), 16 bytes per pool item of per-item state. */
int b200mol_maxmin_pick(const uint32_t* d_fp, size_t nPool, int words, int metric, const int32_t* h_first, int nFirst,
                        int pickSize, double threshold, int32_t* d_picks /* [pickSize] */, double* d_threshold /* [1] */,
                        void* stream);

/* Leader (sphere-exclusion) diversity picking (RDKit LeaderPicker::LazyBitVectorPick) over the pool d_fp[0 .. nPool)
 * ([nPool][words], 16-byte aligned). d(i, j) = 1 - s(i, j) as for b200mol_maxmin_pick; item j is covered by pick p iff
 * d(p, j) <= threshold (the neighbour predicate of b200mol_tanimoto_count_ge with cutoff = threshold). d_picks[0 .. nFirst)
 * = h_first (host memory, distinct pool indices, 0 <= nFirst <= pickSize; h_first may be null when nFirst = 0); every
 * item that is a first pick or is covered by one leaves the pool; then, repeatedly, the lowest-index item left becomes
 * the next pick, and it and every item it covers leave the pool, until the pool is empty or there are pickSize picks.
 * *h_n_picks = the number of picks; d_picks past it is left as it was. 1 <= pickSize <= nPool < 2^31, 0 <= threshold <= 1.
 * Picks are bitwise repeatable. Stream-ordered on `stream`, but the call synchronises it once per window of the pool
 * (to size the next window from the survivor count) and returns after the last: *h_n_picks is valid on return. Scratch
 * is stream-ordered: 5 bytes per pool item, 8 bytes per window item, 132 KB for the resolver's block, the picks' fingerprints (growing by doubling) and
 * what the count pass takes per window. */
int b200mol_leader_pick(const uint32_t* d_fp, size_t nPool, int words, int metric, double threshold, const int32_t* h_first,
                        int nFirst, int pickSize /* >= 1: the cap */, int32_t* d_picks /* [pickSize] */,
                        int32_t* h_n_picks, void* stream);

/* ------------------------------------------------------------------------------------------
 * Butina clustering.  Definition (RDKit ML.Cluster.Butina.ClusterData(reordering=True), the CPU baseline the
 * reference benchmarks against, benchmarks/butina_clustering_bench.py:97-99): repeatedly take the unassigned point
 * with the most unassigned neighbours (ties -> highest index); the cluster is that point plus its unassigned
 * neighbours; ids are assigned in creation order, so cluster 0 is the largest and sizes are non-increasing;
 * when no unassigned point has a neighbour left the rest become singletons in descending index order.
 * ---------------------------------------------------------------------------------------- */

/* Fingerprints in, cluster ids out, O(N + edges) memory.  d_cluster_ids[N]; d_centroids[N] (first *nClusters valid,
 * may be NULL); *h_n_clusters written after an internal stream synchronisation (may be NULL to stay asynchronous,
 * in which case d_n_clusters (device int32, may be NULL) receives it).
 * Replaces fused_butina (nvmolkit/clustering.py:99-189, nvmolkit/_fusedButina.py:99-346). */
int b200mol_butina_fused(const uint32_t* d_fp, size_t n, int words, int metric, double cutoff, int32_t* d_cluster_ids,
                         int32_t* d_centroids, int32_t* d_n_clusters, int32_t* h_n_clusters, void* stream);
/* The two stages of b200mol_butina_fused, exposed so that the N^2 pass can be sharded over GPUs by tile-row group
 * (a group = 32 x 128 fingerprint rows): rank r of R passes group_offset = r, group_stride = R, then the ranks
 * all-reduce d_counts and all-gather their edge lists, and every rank (or rank 0) clusters.
 *   d_counts[n]  += number of neighbours of each point found in this rank's tiles (caller zeroes it)
 *   d_edges      int32 pairs (i, j), i < j, appended; entries beyond edge_cap are dropped but still counted
 *   *h_n_edges   total found (host, written after an internal stream sync; > edge_cap means: retry with more room) */
int b200mol_neighbor_edges(const uint32_t* d_fp, size_t n, int words, int metric, double cutoff, uint32_t group_offset,
                           uint32_t group_stride, int32_t* d_counts, int32_t* d_edges, uint64_t edge_cap,
                           uint64_t* h_n_edges, void* stream);
/* d_counts[n] = full degrees (consumed: decremented in place), d_edges = all n_edges (i<j) pairs. */
int b200mol_butina_from_edges(size_t n, int32_t* d_counts, const int32_t* d_edges, uint64_t n_edges,
                              int32_t* d_cluster_ids, int32_t* d_centroids, int32_t* d_n_clusters,
                              int32_t* h_n_clusters, void* stream);
/* The two stages and the whole of Butina on COUNT vectors (the rows, bins, count range and refusals of b200mol_count_*):
 * points i != j are neighbours iff 1.0 - s(i, j) <= cutoff in fp64, s the value b200mol_count_cross stores for the pair
 * with (alpha, beta) = (1, 1) (Tanimoto) or (0.5, 0.5) (Dice); any other weights, and a cutoff outside [0, 1], are
 * B200MOL_ERR_INVALID before any device work. Ids and centroids are those of b200mol_butina_dense on the matrix
 * 1.0 - s. No similarity matrix is stored: O(N + edges) memory.
 *   b200mol_count_neighbor_edges  d_counts[n] += degrees, d_edges (i, j), i < j, the caller's indices; the edge_cap /
 *                                 *h_n_edges protocol of b200mol_neighbor_edges. It SYNCHRONISES `stream` once for the
 *                                 range check and the list sizes (as b200mol_count_*; a count out of range is refused
 *                                 then, with nothing written) and, when h_n_edges is not NULL, once for the edge total.
 *   b200mol_count_butina_fused    as b200mol_butina_fused: an edge list of 64 per point, one rerun at the exact size for
 *                                 a denser graph, then b200mol_butina_from_edges; it synchronises for the range check,
 *                                 the edge total and, when h_n_clusters is not NULL, *h_n_clusters.
 * The pass visits each unordered pair at most once, with the rows in (sum, index) order, and skips the pairs that a sum
 * bound rules out (csrc/count_similarity.cu); option "count_neighbor_pairs_last" reports how many it compared. Scratch
 * is stream-ordered: that of b200mol_count_*, about 24 bytes per row for the order and 20 bytes per block of 32 rows (16
 * above 2048 bins) for the band; the fused call adds 8 bytes per edge and 12 per point, and b200mol_butina_from_edges's. */
int b200mol_count_neighbor_edges(const int32_t* d_x, size_t n, int bins, double alpha, double beta, double cutoff,
                                 int32_t* d_counts /* [n], += degrees */, int32_t* d_edges /* [cap][2], i < j */,
                                 uint64_t edge_cap, uint64_t* h_n_edges, void* stream);
int b200mol_count_butina_fused(const int32_t* d_x, size_t n, int bins, double alpha, double beta, double cutoff,
                               int32_t* d_cluster_ids, int32_t* d_centroids, int32_t* d_n_clusters, int32_t* h_n_clusters,
                               void* stream);
/* Dense fp64 distance matrix in (neighbours: dist <= cutoff, src/butina.cu:1043-1051).
 * Replaces butinaGpu (src/butina.h:45-50, src/butina.cu:914-1071). */
int b200mol_butina_dense(const double* d_dist, size_t n, double cutoff, int32_t* d_cluster_ids, int32_t* d_centroids,
                         int32_t* d_n_clusters, int32_t* h_n_clusters, void* stream);

/* ------------------------------------------------------------------------------------------
 * Morgan fingerprints from flattened molecular graphs (the seam below RDKit: atom/bond invariants are the
 * output of RDKit's MorganAtomInvGenerator / bond types, src/morgan_fingerprint_common.cpp:43-124).
 *   d_atom_starts[nMols+1], d_bond_starts[nMols+1]  CSR offsets
 *   d_atom_inv[totalAtoms]  u32 atom invariants;  d_bond_inv[totalBonds] u32 bond invariants (bond type)
 *   d_bond_a / d_bond_b [totalBonds]  molecule-local atom indices (u16)
 *   d_out  u32[nMols][fpBits/32], overwritten.
 * Bond endpoints must be smaller than their molecule's atom count and distinct (no self-loops); MolGraphBatch checks
 * this, the kernel does not. An atom may have up to 16 bonds. Any molecule of up to 1024 atoms and 1024 bonds is accepted
 * at every radius <= 16. Exactly: with A = max(maxAtomsPerMol, 1), B = max(maxBondsPerMol, 1), w = ceil(B / 32),
 * R = max(radius, 1) and r(x) = x rounded up to a multiple of 16, a molecule's working set (slab) is
 *   S = 2 r(4A) + 2 r(4Aw) + r(4RAw) + r(4(A + 1)) + 2 r(4B) + 2 r(A) + r(fpBits / 8)  bytes,
 * and the call is accepted when S <= 256 MiB. Slabs of S <= 200 KiB live in shared memory; larger ones in a device
 * scratch buffer of at most 256 MiB per call (get option "morgan_global_slab_last" says which the last call used).
 * Refusals (B200MOL_ERR_INVALID): fpBits not a positive multiple of 32, radius outside [0, 16], maxAtomsPerMol or
 * maxBondsPerMol outside [0, 65536), S > 256 MiB (all before any launch); after the kernel, a molecule with more atoms
 * or bonds than maxAtomsPerMol / maxBondsPerMol (its row is zero) or, at radius >= 1, an atom with more than 16 bonds.
 * Synchronises `stream`.
 * Replaces launchMorganFingerprintKernelBatch<fpSize> (src/morgan_fingerprint_kernels.h:90-95, .cu:152-432) and its
 * CPU twin for large molecules (src/morgan_fingerprint_cpu.cpp:61-255). */
int b200mol_morgan(const int32_t* d_atom_starts, const int32_t* d_bond_starts, const uint32_t* d_atom_inv,
                   const uint32_t* d_bond_inv, const uint16_t* d_bond_a, const uint16_t* d_bond_b, size_t nMols,
                   int maxAtomsPerMol, int maxBondsPerMol, int radius, int fpBits, uint32_t* d_out, void* stream);
/* Morgan count fingerprints: the arguments, checks, launch shapes and sync of b200mol_morgan, writing
 * d_out int32[nMols][fpBits] (overwritten): d_out[i][j] is the number of accepted environments of molecule i whose code
 * is congruent to j mod fpBits (every atom at radius 0; an environment whose bond set an earlier or equal one already
 * had does not count). A bin is non-zero exactly where b200mol_morgan sets the bit. RDKit's GetCountFingerprintAsNumPy
 * for GetMorganGenerator(radius, fpSize) with the options b200mol_morgan fixes. */
int b200mol_morgan_counts(const int32_t* d_atom_starts, const int32_t* d_bond_starts, const uint32_t* d_atom_inv,
                          const uint32_t* d_bond_inv, const uint16_t* d_bond_a, const uint16_t* d_bond_b, size_t nMols,
                          int maxAtomsPerMol, int maxBondsPerMol, int radius, int fpBits, int32_t* d_out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batched force fields + BFGS (the conformer hot path).
 *
 * Data model (replaces the reference's BatchedMolecularSystemHost/Device, src/forcefields/mmff.h:153-436,
 * src/forcefields/dist_geom.h:31-586): a MOLECULE table holds the flattened terms once per molecule, CSR by
 * molecule, with molecule-LOCAL int16 atom indices [n][K] and fp64 parameter records [n][P]; a CONFORMER batch
 * points into it (conformer c is molecule conf_mol[c], its coordinates start at atom conf_atom_start[c]), so the
 * conformers of one molecule share one term block. All pointers inside the structs are DEVICE pointers; the structs
 * themselves are passed from host memory.
 * ---------------------------------------------------------------------------------------- */
typedef struct b200mol_term_table {
  const int32_t* starts;   /* [nMols+1] */
  const int16_t* idx;      /* [n][K] */
  const double*  par;      /* [n][P] */
  /* Gradient schedule (b200mol_schedule_waves): the terms of molecule m are ordered in WAVES molWaves[m] ..
   * molWaves[m+1]; wave w holds the terms waves[w] .. waves[w+1] (global term indices), at most 32 of them, no atom
   * twice. A warp takes a wave at a time and adds the gradient contributions without atomics. Required by every entry
   * point that evaluates gradients (energy-only calls and the ETKDG check tables ignore it; NULL there is fine). */
  const int32_t* molWaves; /* [nMols+1] */
  const int32_t* waves;    /* [nWaves+1] */
} b200mol_term_table;

/* HOST helper (no device work): orders the terms of one table into atom-disjoint waves of at most 32.
 *   h_starts[nMols+1], h_idx[n][K]   the table (host memory), K in 1..8
 *   h_perm[n]        out: new position p holds old term h_perm[p] (apply to idx AND par before the upload)
 *   h_mol_waves[nMols+1], h_waves[n+1]  out (h_waves gets *n_waves + 1 entries)
 * Dense pair tables (K = 2, >= 2 terms per atom) take the rounds of a round-robin tournament, (i + j) mod M with M the
 * odd number >= the atom count: every round is a perfect matching, so all-pairs tables fill their waves; everything
 * else takes a first-fit colouring. Deterministic. The reference has no counterpart (it scatters with atomics). */
int b200mol_schedule_waves(int32_t nMols, const int32_t* h_starts, const int16_t* h_idx, int K, int32_t* h_perm,
                           int32_t* h_mol_waves, int32_t* h_waves, int64_t* n_waves);

/* MMFF94 (term math: src/forcefields/mmff_kernels_device.cuh:241-661; layout source: src/forcefields/mmff.h:37-145)
 *   bond    K2 P2 {r0, kb}                  angle   K3 P3 {theta0, ka, isLinear}
 *   strbend K3 P5 {theta0, r0_ij, r0_kj, kba_ijk, kba_kji}      oop K4 P1 {koop}   (j = idx[1] is the centre)
 *   torsion K4 P3 {V1, V2, V3}              vdw     K2 P2 {R*_ij, eps_ij}
 *   ele     K2 P3 {q_i q_j / dielectric, dielModel (1 | 2), is14} */
typedef struct b200mol_mmff_system {
  int32_t            nMols;
  const int32_t*     atomCounts; /* [nMols] */
  b200mol_term_table bond, angle, strbend, oop, torsion, vdw, ele;
  /* restraints (RDKit MMFF/UFF "constraints", src/forcefields/mmff_kernels_device.cuh:673-1036); empty tables = none:
   *   distc K2 P3 {minLen, maxLen, k}   posc K1 P5 {refX, refY, refZ, maxDispl, k}
   *   anglec K3 P3 {minDeg, maxDeg, k}  torsc K4 P3 {minDeg, maxDeg, k} (signed dihedral, degrees, periodic) */
  b200mol_term_table distc, posc, anglec, torsc;
} b200mol_mmff_system;

/* Distance geometry (src/forcefields/dist_geom_kernels_device.cuh:37-231; src/forcefields/dist_geom.h:31-56)
 *   dist K2 P3 {lb^2, ub^2, weight}    chiral K4 P2 {volUpper, volLower}    fourth K1 P0 (par may be NULL) */
typedef struct b200mol_dg_system {
  int32_t            nMols;
  const int32_t*     atomCounts;
  b200mol_term_table dist, chiral, fourth;
} b200mol_dg_system;

/* ETK / 3-D refinement terms on 4-D coordinate storage (dist_geom_kernels_device.cuh:237-830; dist_geom.h:73-128)
 *   torsion K4 P12 {V1..V6, sign1..sign6}   improper K4 P4 {C0, C1, C2, k}
 *   dist12 / dist13 K2 P4 {min, max, k, fixed}   longrange K2 P3 {min, max, k}   angle13 K3 P2 {minDeg, maxDeg}
 * `fixed` = the reference's isImproperConstrained: with recentre = 1 every 1-2 / 1-3 window whose fixed flag is 0 is
 * re-centred on the distance in the STARTING geometry keeping its half-width (the refresh the reference does before its
 * ETK minimisation, src/etkdg_stage_etk_minimization.cu:32-64,176-202) — evaluated on the fly, the tables stay
 * read-only and shared by all conformers of the molecule. */
typedef struct b200mol_etk_system {
  int32_t            nMols;
  const int32_t*     atomCounts;
  b200mol_term_table torsion, improper, dist12, dist13, angle13, longrange;
} b200mol_etk_system;

/* UFF (src/forcefields/uff_kernels_device.cuh:37-590; layout source src/forcefields/uff.h:33-97)
 *   bond K2 P2 {restLen, k}    angle K3 P6 {theta0 (rad), k, order, C0, C1, C2}    torsion K4 P3 {k, order, cosTerm}
 *   inversion K4 P4 {k, C0, C1, C2} (idx[1] = centre)    vdw K2 P3 {x_ij, wellDepth, threshold} */
typedef struct b200mol_uff_system {
  int32_t            nMols;
  const int32_t*     atomCounts;
  b200mol_term_table bond, angle, torsion, inversion, vdw;
  b200mol_term_table distc, posc, anglec, torsc; /* restraints, as in b200mol_mmff_system */
} b200mol_uff_system;

/* ------------------------------------------------------------------------------------------
 * Term construction on the HOST from a smoothed bounds matrix (pure arithmetic, no RDKit): the seam just below
 * RDKit's setTopolBounds / getExperimentalTorsions. h_bounds = RDKit BoundsMatrix layout, nAtoms x nAtoms row-major,
 * upper bound at [min][max], lower bound at [max][min]. Outputs are caller-allocated at their maximum sizes:
 * pairs nAtoms*(nAtoms-1)/2, chiral nChiral, fourth nAtoms.
 * Replaces constructForceFieldContribs (rdkit_extensions/dist_geom_flattened_builder.cpp:472-491, :56-122):
 * every pair with ub - lb <= basinSizeTol becomes a distance term {lb^2, ub^2, weight 1} (the pipeline passes 1e8: all
 * pairs), the chiral sets (h_chiral_atoms[n][4], h_chiral_bounds[n][2] = {lower, upper}) become chiral terms, dim = 4
 * adds one fourth-dimension term per atom. h_counts3 = {nDist, nChiral, nFourth}. */
int b200mol_dg_terms_from_bounds(int32_t nAtoms, const double* h_bounds, int32_t nChiral, const int32_t* h_chiral_atoms,
                                 const double* h_chiral_bounds, int dim, double basinSizeTol, int16_t* h_dist_idx,
                                 double* h_dist_par, int16_t* h_chiral_idx, double* h_chiral_par, int16_t* h_fourth_idx,
                                 int32_t* h_counts3);
/* RDKit ForceFields::CrystalFF::CrystalFFDetails as plain arrays (host memory). */
typedef struct b200mol_crystalff_details {
  int32_t        nTorsions;
  const int32_t* torsionAtoms; /* [n][4] expTorsionAtoms */
  const double*  torsionV;     /* [n][6] expTorsionAngles[.].second (force constants), zero-padded */
  const int32_t* torsionSigns; /* [n][6] expTorsionAngles[.].first, zero-padded */
  int32_t        nImpropers;
  const int32_t* improperAtoms; /* [n][6] {a0, centre, a2, a3, Z of the centre, isCBoundToO} */
  int32_t        nBonds;
  const int32_t* bonds; /* [n][2] */
  int32_t        nAngles;
  const int32_t* angles; /* [n][4] {a, centre, b, isTripleBond} */
  double         boundsMatForceScaling;
} b200mol_crystalff_details;
/* Output buffers of b200mol_etk_terms_from_details, sized by the caller: torsion nTorsions, improper 3 * nImpropers,
 * dist12 nBonds, dist13 and angle13 nAngles each, longrange nAtoms*(nAtoms-1)/2 (record layouts: b200mol_etk_system). */
typedef struct b200mol_etk_term_buffers {
  int16_t* torsion_idx;   double* torsion_par;
  int16_t* improper_idx;  double* improper_par;
  int16_t* dist12_idx;    double* dist12_par;
  int16_t* dist13_idx;    double* dist13_par;
  int16_t* angle13_idx;   double* angle13_par;
  int16_t* longrange_idx; double* longrange_par;
} b200mol_etk_term_buffers;
/* Replaces construct3DForceFieldContribs (dist_geom_flattened_builder.cpp:493-541, :124-470): experimental torsions,
 * improper terms (3 permutations per centre, inversion coefficients by element, x10 force scaling; only with
 * useBasicKnowledge), 1-2 windows (+-0.01, k 100), 1-3 windows (triple bond: angle 179..180; improper-constrained
 * centre: the bounds, fixed; else +-0.01), long-range terms for every other pair (the bounds, k = 10 x
 * boundsMatForceScaling). h_counts6 = terms written per table in b200mol_etk_system order; *h_num_impropers = the
 * planarity check's count (improper centres, not terms). */
int b200mol_etk_terms_from_details(int32_t nAtoms, const double* h_bounds, const b200mol_crystalff_details* details,
                                   int useBasicKnowledge, b200mol_etk_term_buffers* out, int32_t* h_counts6,
                                   int32_t* h_num_impropers);

/* Energies (d_energy[nConf]) and, when d_grad != NULL, gradients (d_grad[totalAtoms*dim], overwritten) of a
 * conformer batch. Replaces launch*EnergyKernel / launch*GradientKernel + combinedEnergies/GradKernel
 * (src/forcefields/mmff_kernels.h, mmff_kernels.cu:1067-1125; dist_geom_kernels.cu). */
int b200mol_mmff_energy_grad(const b200mol_mmff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                             const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy, double* d_grad,
                             void* stream);
int b200mol_uff_energy_grad(const b200mol_uff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                            const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy, double* d_grad,
                            void* stream);
int b200mol_dg_energy_grad(const b200mol_dg_system* sys, int dim, double chiralWeight, double fourthDimWeight,
                           int32_t nConf, const int32_t* d_conf_mol, const int32_t* d_conf_atom_start,
                           const double* d_pos, double* d_energy, double* d_grad, void* stream);
int b200mol_etk_energy_grad(const b200mol_etk_system* sys, int plain, int recentre, int32_t nConf,
                            const int32_t* d_conf_mol,
                            const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy, double* d_grad,
                            void* stream);

/* BFGS minimisation of every conformer of the batch (RDKit BFGSOpt.h semantics incl. ForceField::minimize gradient
 * scaling, RDKit >= 2025.09 rule), one CTA per conformer, whole minimisation in one persistent kernel launch.
 *   d_pos      in/out coordinates [totalAtoms*dim]        d_energy  out, energy at the returned coordinates
 *   d_status   out int8[nConf]: 0 = converged, 1 = max_iters reached (same meaning as the reference's statuses)
 *   d_iters    out int32[nConf] BFGS iterations used (may be NULL)
 *   d_active   optional uint8[nConf]: conformers with 0 are skipped (reference: activeThisStage)
 *   max_atoms  largest atom count in the batch (sizes shared memory and the inverse-Hessian slabs)
 * Replaces launchBfgsMinimizePerMolKernel[ETK|DG] (src/minimizer/bfgs_minimize.cu:1086-1146), BfgsBatchMinimizer::
 * minimize (:978-1053) and updateInverseHessianBFGSBatch (src/minimizer/bfgs_hessian.cu:373-438). */
int b200mol_mmff_minimize(const b200mol_mmff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                          const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                          double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                          int32_t* d_iters, void* stream);
/* UFF twin (reference: UFFMinimizeMoleculesConfs, src/minimizer/bfgs_uff.cpp; Python default maxIters 1000). */
int b200mol_uff_minimize(const b200mol_uff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                         const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                         double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                         int32_t* d_iters, void* stream);
int b200mol_dg_minimize(const b200mol_dg_system* sys, int dim, double chiralWeight, double fourthDimWeight,
                        int32_t nConf, const int32_t* d_conf_mol, const int32_t* d_conf_atom_start, int max_atoms,
                        double* d_pos, int max_iters, double grad_tol, const uint8_t* d_active, double* d_energy,
                        int8_t* d_status, int32_t* d_iters, void* stream);
int b200mol_etk_minimize(const b200mol_etk_system* sys, int plain, int recentre, int32_t nConf,
                         const int32_t* d_conf_mol,
                         const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                         double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                         int32_t* d_iters, void* stream);
/* Analytic test potential E = sum_i w_i (x_i - c_i)^power, power in {2, 4}; system s owns x[starts[s]..starts[s+1])
 * (the reference drives its BFGS tests through such a user force field, tests/test_bfgs_minimizer.cu:822-930).
 * hessian_fp32 != 0 keeps the inverse Hessian in fp32, the embedder's default slab type (option
 * "etkdg_hessian_fp64"); 0 in fp64 like the force-field minimisers. */
int b200mol_poly_minimize(int32_t nSys, const int32_t* d_starts, int max_dim, int power, const double* d_w,
                          const double* d_c, double* d_x, int max_iters, double grad_tol, int scale_grads,
                          int hessian_fp32, double* d_energy, int8_t* d_status, int32_t* d_iters, void* stream);

/* ------------------------------------------------------------------------------------------
 * ETKDG conformer embedding (replaces nvMolKit::embedMolecules' device pipeline: ETKDGDriver / Scheduler / stages,
 * src/etkdg.cpp:90-484, src/etkdg_impl.cpp:111-312, src/etkdg_stage_*.cu).
 * Stereo / geometry check tables, CSR by molecule like the force-field tables:
 *   tetrahedral K5 {centre, n1, n2, n3, n4 (= centre for 3-coordinate)} P1 {inFusedSmallRings}
 *   chiral      K5 {centre, a1, a2, a3, a4}  P2 {volLower, volUpper}      (RDKit ChiralSet)
 *   chiralDist  K2 P2 {lower, upper}          dbStereo K4 P1 {sign}        dbGeom K3 P0
 *   numImpropers[nMols]: planarity tolerance count (improper energy must stay <= 0.7 * numImpropers)
 * ---------------------------------------------------------------------------------------- */
typedef struct b200mol_etkdg_checks {
  b200mol_term_table tetrahedral, chiral, chiralDist, dbStereo, dbGeom;
  const int32_t*     numImpropers;
} b200mol_etkdg_checks;

typedef struct b200mol_embed_params {
  uint64_t seed;              /* counter-based RNG key: coordinates depend on (seed, slot, attempt, element) only */
  double   boxSize;           /* 5 * boxSizeMult (or -boxSizeMult when negative), src/etkdg_stage_coordgen.cu:102-107 */
  double   optimizerForceTol; /* RDKit EmbedParameters::optimizerForceTol (1e-3) */
  int32_t  enforceChirality, useExpTorsions, useBasicKnowledge;
  int32_t  maxAttempts;       /* per conformer slot (reference: maxIterations) */
  int32_t  dgIters, fourthIters, etkIters; /* 400, 200, 300 */
  int32_t  maxRestarts;       /* cap on "repeat until converged" of the first minimisation */
  int32_t  useMetricStart;    /* 0: random 4-D box (RDKit useRandomCoords = true, the reference's only mode, src/etkdg.cpp:
                                 99-101). 1: RDKit's useRandomCoords = false start - random distance matrix inside the bounds ->
                                 metric matrix -> top-4 eigenpairs (power iteration) -> coordinates, on the device, per attempt */
} b200mol_embed_params;

/* One conformer per slot: slot s embeds molecule d_slot_mol[s] into d_coords[d_slot_atom_start[s]*3 ...] (xyz fp64).
 * d_ok[s] = 1 on success (else the coordinates are untouched); d_attempts[s] attempts used; d_energy[s] DG energy of
 * the accepted attempt; d_stage_failures[11] (optional) failure counts per stage. Asynchronous. */
int b200mol_etkdg_embed(const b200mol_dg_system* dg, const b200mol_etk_system* etk, const b200mol_etkdg_checks* checks,
                        const b200mol_embed_params* params, int32_t nSlots, const int32_t* d_slot_mol,
                        const int32_t* d_slot_atom_start, int max_atoms, double* d_coords, int8_t* d_ok,
                        int32_t* d_attempts, double* d_energy, uint64_t* d_stage_failures, void* stream);
/* Stage 0 alone: the 4-D start coordinates of attempt `attempt` of every slot, d_pos4[d_slot_atom_start[s]*4 ...];
 * d_ok[s] = 0 when the metric-matrix start fails (degenerate metric matrix, eigensolver not converged, zero eigenvalue).
 * Replaces ETKDGCoordGenStage (src/etkdg_stage_coordgen.cu:100-122, the random box) and adds the eigen start the
 * reference leaves to RDKit (InitialCoordinateGenerator, src/forcefields/coord_gen.cu:133-216, is off the production path). */
int b200mol_etkdg_initial_coords(const b200mol_dg_system* dg, const b200mol_embed_params* params, int32_t nSlots,
                                 const int32_t* d_slot_mol, const int32_t* d_slot_atom_start, int max_atoms, int32_t attempt,
                                 double* d_pos4, int8_t* d_ok, void* stream);
/* The acceptance checks alone on given 4-D coordinates d_pos4[atom*4 ...]: bit s of d_fail_masks[slot] = stage s fails
 * (1 energy/atom, 2 tetrahedral, 3 chirality, 5 planarity, 6 double-bond geometry, 7 chirality, 8 chiral distances,
 * 9 centre-in-volume, 10 double-bond stereo). Replaces the kernels of src/etkdg_stage_stereochem_checks.cu:52-440. */
int b200mol_etkdg_check(const b200mol_dg_system* dg, const b200mol_etk_system* etk, const b200mol_etkdg_checks* checks,
                        const b200mol_embed_params* params, int32_t nSlots, const int32_t* d_slot_mol,
                        const int32_t* d_slot_atom_start, int max_atoms, const double* d_pos4, uint32_t* d_fail_masks,
                        void* stream);

/* RMS pruning of embedded conformers on the device (RDKit EmbedParameters::pruneRmsThresh). Conformers of molecule m are
 * [d_mol_conf_start[m], d_mol_conf_start[m+1]) in embedding order; conformer c owns atoms [d_conf_atom_start[c],
 * d_conf_atom_start[c+1]) of d_xyz[.][3]. d_keep[c] = 1 when conformer c is valid (d_conf_valid[c] != 0, NULL = all) and its
 * best-alignment sum of squared deviations to every conformer kept before it is >= nSel * rms_thresh^2.
 * Atom selection / symmetry: per molecule K_m index lists ("self matches") of L_m atoms each, d_match_atoms
 * [d_match_offset[m] .. d_match_offset[m+1]) = K_m * L_m molecule-local indices, d_match_len[m] = L_m; list 0 selects the
 * atoms of the conformer under test, every list in turn those of an earlier conformer (RDKit useSymmetryForPruning); one
 * list of the heavy atoms = onlyHeavyAtomsForRMS; all three NULL = all atoms, identity mapping.
 * Replaces addConformersToMoleculeWithPruning / _isConfFarFromRest (rdkit_extensions/conformer_pruning.cpp:96-137), which
 * the reference runs on the host and refuses for DEVICE output (src/etkdg.cpp:106-110). */
int b200mol_rms_prune(int32_t nMols, const int32_t* d_mol_conf_start, const int32_t* d_conf_atom_start, const double* d_xyz,
                      const int32_t* d_match_offset, const int32_t* d_match_len, const int16_t* d_match_atoms, double rms_thresh,
                      const uint8_t* d_conf_valid, uint8_t* d_keep, void* stream);

/* Torsion fingerprint deviation (TFD) matrices between the conformers of each molecule (RDKit
 * TorsionFingerprints.GetTFDMatrix). Conformer k of molecule m is conformer d_conf_order[h_mol_conf_start[m] + k]
 * (d_conf_order NULL = identity), which owns atoms [d_conf_atom_start[c], ...) of d_xyz[.][3] (f64).
 * Torsions of molecule m are [h_tors_start[m], h_tors_start[m+1]); torsion t has the quartets
 * [h_quartet_start[t], h_quartet_start[t+1]) of h_quartets[.][4] (molecule-local atom indices), type h_type[t]
 * (B200MOL_TFD_SINGLE: one quartet; _SYMMETRIC: the minimum over quartet pairs; _RING: the ring's consecutive
 * quartets, compared through the mean |phi|), weight h_weight[t] >= 0 and h_maxdev[t] > 0 (degrees).
 * For conformers I > J: TFD = sum_t w_t d_t / maxDev_t / sum_t w_t, 0 when sum w <= 1e-10; d as in RDKit's
 * CalculateTFD, with phi = 0 for a quartet whose cross product i-j x j-k or j-k x k-l is exactly zero.
 * d_out (f32): the lower triangles of all molecules, concatenated: molecule m starts at sum_{m'<m} C(C-1)/2, and
 * holds (I, J) at I(I-1)/2 + J. A molecule with fewer than two conformers contributes nothing; one without torsions
 * gives zeros. The torsion and conformer-count tables are HOST arrays: the call plans its tiles from them and uploads
 * the plan in one cudaMemcpyAsync from pageable memory (which CUDA may stage synchronously, as for any pageable copy);
 * coordinates and output stay on the device and both kernels run on `stream`.
 * Replaces GetTFDMatricesGpuBuffer / tfdMatrixKernel (src/tfd/tfd_gpu.cpp, src/tfd/tfd_kernels.cu:84-166). */
#define B200MOL_TFD_SINGLE 0
#define B200MOL_TFD_SYMMETRIC 1
#define B200MOL_TFD_RING 2
int b200mol_tfd_matrices(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* d_conf_order,
                         const int32_t* d_conf_atom_start, const double* d_xyz, const int32_t* h_tors_start,
                         const int32_t* h_quartet_start, const int16_t* h_quartets, const uint8_t* h_type,
                         const double* h_weight, const double* h_maxdev, float* d_out, void* stream);

/* Conformer RMSD matrices (RDKit AllChem.GetConformerRMSMatrix, over all atoms). Conformer k of molecule m is conformer
 * d_conf_order[h_mol_conf_start[m] + k] (d_conf_order NULL = identity), which owns exactly h_mol_atoms[m] atoms from
 * d_conf_atom_start[c] of d_xyz[.][3] (f64). For conformers I > J:
 *   prealigned == 0: sqrt(max(0, Ga + Gb - 2 (s1 + s2 + sign(det H) s3)) / n), the RMSD after the best proper rigid
 *                    superposition (Ga, Gb: sums of squared centred coordinates; s_i: singular values of the covariance
 *                    H of the centred coordinates). The coordinates are not modified.
 *   prealigned != 0: sqrt(sum_k |a_k - b_k|^2 / n) on the coordinates as given.
 * d_out (f64): the lower triangles of all molecules, concatenated: molecule m starts at sum_{m'<m} C(C-1)/2 (int64), and
 * holds (I, J) at I(I-1)/2 + J. A molecule with fewer than two conformers contributes nothing; one with two or more and
 * no atoms is an error. The conformer and atom-count tables are HOST arrays: the call plans its tiles from them and
 * uploads the plan in one cudaMemcpyAsync from pageable memory; coordinates and output stay on the device and both
 * kernels run on `stream`. Sums run in a fixed order: results are bitwise repeatable and independent of the other
 * molecules of the call.
 * Replaces conformerRmsdBatchMatrixGpu (src/conformer_rmsd.cu, nvmolkit/conformerRmsd.cpp). */
int b200mol_conformer_rmsd(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms,
                           const int32_t* d_conf_order, const int32_t* d_conf_atom_start, const double* d_xyz,
                           int32_t prealigned, double* d_out, void* stream);
/* Symmetry-aware conformer RMSD matrices (RDKit rdMolAlign.GetAllConformerBestRMS; with one mapping, an atom selection as
 * AllChem.GetConformerRMSMatrix(atomIds=...)). The conformer tables, output and stream are as b200mol_conformer_rmsd.
 * Molecule m (fewer than 32768 atoms) has a mapping table of K_m = h_map_count[m] >= 1 mappings of
 * L_m = h_map_len[m] in [1, h_mol_atoms[m]] atoms (L_m = 0 for a molecule without atoms, which has no pairs):
 * h_map_atoms[h_map_start[m] .. h_map_start[m+1]) (int64 offsets) holds the probe list P (L_m molecule-local indices),
 * then the reference lists Q_1 .. Q_K (L_m each); no index twice within a list. For conformers I > J:
 *   min over k of RMSD(x_I[P], x_J[Q_k])
 * with RMSD as b200mol_conformer_rmsd over the L_m selected atoms: after the best proper rigid superposition, each side
 * centred on its own selected atoms, or, prealigned != 0, on the coordinates as given (RDKit CalcRMS). K = 1 with
 * P = Q_1 = 0 .. n-1 gives b200mol_conformer_rmsd's output bit for bit. The tables are HOST arrays, checked before any
 * device work; the call uploads them with its plan. The mappings of a molecule run in chunks of at most
 * "rmsd_match_chunk"; a minimum is exact, so results stay bitwise repeatable and batch-independent. */
int b200mol_conformer_rmsd_mapped(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms,
                                  const int32_t* d_conf_order, const int32_t* d_conf_atom_start, const double* d_xyz,
                                  const int64_t* h_map_start, const int32_t* h_map_count, const int32_t* h_map_len,
                                  const int16_t* h_map_atoms, int32_t prealigned, double* d_out, void* stream);

/* Weighted rigid alignment of conformers (RDKit rdMolAlign.AlignMol / GetAlignmentTransform / AlignMolConformers, i.e.
 * Numerics::Alignment::AlignPoints; the reference library has no alignment). Conformer c owns h_conf_atoms[c] atoms from
 * d_conf_atom_start[c] of d_xyz[.][3] (f64), c < nConfs. Job j aligns probe conformer h_job_probe[j] onto reference
 * conformer h_job_ref[j] through pair list h_job_list[j]: list l holds the L >= 1 pairs
 * h_list_pairs[2 i], h_list_pairs[2 i + 1] (probe atom, reference atom; conformer-local) for
 * i in [h_list_start[l], h_list_start[l+1]) (int64, h_list_start[0] = 0), with weights h_list_weights[i] (finite, >= 0,
 * summing to W > 0 per list; NULL = all 1). Lists are shared by jobs (AlignMolConformers: one list per molecule).
 * With weighted centroids p_bar, r_bar and covariance S = sum w (p - p_bar)(r - r_bar)^T (reflect != 0: every probe
 * point p replaced by -p first), lambda = largest eigenvalue estimate of Horn's quaternion matrix N(S) after at most
 * maxIters >= 1 cyclic Jacobi sweeps (converged in fp64 at 50), q its eigenvector, R = R(q) (N = 0: R = I):
 *   d_rmsd[j] = sqrt(max(0, sum w |p - p_bar|^2 + sum w |r - r_bar|^2 - 2 lambda) / L)   (divided by L, not by W)
 *   d_transform[16 j ..] (optional, NULL = not written) = [[+-R, t], [0 0 0 1]] row-major, acting on column vectors,
 *     t = r_bar - R p_bar (reflected p_bar), the sign - when reflect: RDKit's Transform3D layout.
 * move != 0: every atom of the probe conformer (not just the listed ones) is replaced by its image under the transform,
 * in place in d_xyz; then no conformer may be the probe of two jobs or both a probe and a reference. Sums run on
 * coordinates shifted by each job's first pair, so molecules far from the origin keep their accuracy. All tables are
 * HOST arrays, checked before any device work and uploaded in one cudaMemcpyAsync; the kernel runs on `stream`.
 * Results are bitwise repeatable and independent of the other jobs of the call. */
int b200mol_align(int32_t nJobs, const int32_t* h_job_probe, const int32_t* h_job_ref, const int32_t* h_job_list,
                  int32_t nConfs, const int32_t* h_conf_atoms, const int32_t* d_conf_atom_start, double* d_xyz,
                  int32_t nLists, const int64_t* h_list_start, const int32_t* h_list_pairs, const double* h_list_weights,
                  int32_t reflect, int32_t maxIters, int32_t move, double* d_rmsd, double* d_transform, void* stream);

/* Symmetry-aware alignment of conformers (RDKit rdMolAlign.GetBestRMS / GetBestAlignmentTransform / CalcRMS; the
 * reference library has no alignment). Conformers as in b200mol_align. Job j compares probe conformer h_job_probe[j]
 * with reference conformer h_job_ref[j] through mapping set s = h_job_set[j]: K_s = h_set_count[s] >= 1 mappings of
 * L_s = h_set_len[s] >= 1 atoms, h_set_atoms[h_set_start[s] .. h_set_start[s+1]) (int64 offsets, h_set_start[0] = 0,
 * (K_s + 1) L_s entries) holding the probe list P, then the reference lists Q_1 .. Q_K (conformer-local indices below
 * 32768, none twice within a list; the layout of b200mol_conformer_rmsd_mapped). Mapping k pairs P[i] with Q_k[i],
 * with weight h_set_weights[W_s + i] (W_s = sum of L over the sets before s; finite, >= 0, summing to > 0 per set;
 * NULL = all 1). Sets are shared by jobs: one per molecule pair, whatever its number of conformers.
 *   mode 0 (align): per mapping the RMSD of b200mol_align (reflect, maxIters as there); d_rmsd[j] = the smallest,
 *     d_best[j] (optional) = the first mapping that has it, d_transform[16 j ..] (optional) = its transform, and,
 *     move != 0, every atom of the probe conformer moved by it (then no conformer may be the probe of two jobs or both a
 *     probe and a reference).
 *   mode 1 (in place, RDKit CalcRMS): per mapping sqrt(sum w |p - r|^2 / L) on the coordinates as given, the smallest in
 *     d_rmsd[j] and its first mapping in d_best[j]; move, reflect and d_transform must be 0.
 * All tables are HOST arrays, checked before any device work and uploaded in one cudaMemcpyAsync; the kernel runs on
 * `stream`. Results are bitwise repeatable and independent of the other jobs of the call; K = 1 gives b200mol_align's
 * bits. */
int b200mol_best_align(int32_t nJobs, const int32_t* h_job_probe, const int32_t* h_job_ref, const int32_t* h_job_set,
                       int32_t nConfs, const int32_t* h_conf_atoms, const int32_t* d_conf_atom_start, double* d_xyz,
                       int32_t nSets, const int64_t* h_set_start, const int32_t* h_set_count, const int32_t* h_set_len,
                       const int16_t* h_set_atoms, const double* h_set_weights, int32_t mode, int32_t reflect,
                       int32_t maxIters, int32_t move, double* d_rmsd, int32_t* d_best, double* d_transform,
                       void* stream);

/* ------------------------------------------------------------------------------------------
 * Distance-geometry preparation (per-molecule, matrix resident in shared memory).
 * Matrices are concatenated: matrix m occupies d_x[starts[m] .. starts[m+1]) = n_m * n_m doubles, row-major.
 * ---------------------------------------------------------------------------------------- */
/* In-place triangle-inequality smoothing of RDKit bounds matrices ([i][j], i<j = upper bound; [j][i] = lower bound).
 * d_ok[m] = 1 consistent / 0 inconsistent (lb > ub found: the pivot in which it first appears is completed for every
 * pair, later pivots are not run). tol as in RDKit
 * triangleSmoothBounds (0 = strict). Replaces triangleSmoothBoundsBatch (src/triangle_smooth.cu:132-247) and the CPU
 * call DistGeom::triangleSmoothBounds in src/embedder_utils.cpp:313,324. */
int b200mol_triangle_smooth(double* d_bounds, const int64_t* d_matrix_starts, int32_t nMats, double tol, int8_t* d_ok,
                            void* stream);
/* Top-numEigs eigenpairs by power iteration with deflation (RDKit PowerEigenSolver: tol 1e-3, <= 1000 iterations).
 * d_mats is destroyed. d_v0 (optional) start vectors, numEigs * n_m per matrix at d_v0_starts[m]; NULL = hashed
 * counter sequence from `seed`. d_eigvals[m][numEigs]; d_eigvecs row e of matrix m at d_vec_starts[m] + e * n_m;
 * d_n_converged[m] = number of eigenpairs found; the outputs of eigenpairs past it are left unwritten. The two
 * n-vectors of the iteration stay in shared memory (28160 doubles) even when the matrix itself does not fit there, so
 * n <= 14080: a larger matrix gets d_n_converged[m] = 0 and nothing else is written for it. Replaces
 * BatchedEigenSolver::solve (src/symmetric_eigensolver.cu:62-247). */
int b200mol_eig_topk(double* d_mats, const int64_t* d_matrix_starts, int32_t nMats, int numEigs, const double* d_v0,
                     const int64_t* d_v0_starts, uint32_t seed, double* d_eigvals, double* d_eigvecs,
                     const int64_t* d_vec_starts, int8_t* d_n_converged, void* stream);
/* Distance matrix -> metric matrix -> top-`dim` eigenpairs -> coordinates d_coords[(atom_starts[m]+i)*dim + j] =
 * sqrt(lambda_j) v_j[i]; d_ok[m] = 0 when an eigenvalue is not positive or did not converge (3-D AND 4-D; the
 * reference's InitialCoordinateGenerator is 3-D only, src/forcefields/coord_gen.cu:64,160). d_dist is destroyed.
 * Coordinates of a matrix with d_ok[m] = 0 are left unwritten. The iteration vectors, eigenpairs and row means,
 * (3 + dim) n + dim doubles, stay in shared memory (28160 doubles), so n <= 4692 at dim 3 and n <= 4022 at dim 4:
 * a larger matrix gets d_ok[m] = 0. */
int b200mol_metric_embed(double* d_dist, const int64_t* d_matrix_starts, const int32_t* d_atom_starts, int32_t nMats,
                         int dim, const double* d_v0, const int64_t* d_v0_starts, uint32_t seed, double* d_coords,
                         int8_t* d_ok, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU result exchange (one process per GPU, NCCL over NVLink / NVSwitch): the single collective at the end of a
 * molecule-range-sharded conformer job. `nccl_comm` is the caller's ncclComm_t. NCCL is resolved at run time from the
 * library already loaded in the process (or libnccl.so.2), never linked. Replaces DeviceCoordCollector::finalizeOnTarget
 * + copyDeviceToDeviceAsync (src/conformer/device_coord_collector.cpp:30-145, src/utils/p2p.cpp:56-86): every rank ends
 * up with the whole CSR result instead of one target GPU.
 * Step 1: conformer / atom counts of every rank to the host (h_*[world]); synchronises `stream`. */
int b200mol_allgather_counts(void* nccl_comm, int64_t n_conf_local, int64_t n_atoms_local, int64_t* h_conf_counts,
                             int64_t* h_atom_counts, void* stream);
/* Step 2: the payload, rank-major, exact sizes (one ncclBroadcast per rank and array inside one group):
 *   d_positions[sum atoms][3] f64, d_conf_atoms[sum conf] i32 (atoms per conformer), d_energy[sum conf] f64,
 *   d_converged[sum conf] i8. Any of the four output arrays may be NULL (skipped on every rank alike). Asynchronous. */
int b200mol_allgather_results(void* nccl_comm, const int64_t* h_conf_counts, const int64_t* h_atom_counts,
                              const double* d_positions_local, const int32_t* d_conf_atoms_local, const double* d_energy_local,
                              const int8_t* d_converged_local, double* d_positions, int32_t* d_conf_atoms, double* d_energy,
                              int8_t* d_converged, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200MOL_H */
