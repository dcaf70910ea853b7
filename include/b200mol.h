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
 * (1 after a candidate-list overflow made it fall back), and "similarity_candidates_last": how many candidates it listed. */
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
 * Molecules may have up to 1024 atoms and 1024 bonds, and any atom up to 8 bonds (kMaxBondsPerAtom).
 * Replaces launchMorganFingerprintKernelBatch<fpSize> (src/morgan_fingerprint_kernels.h:90-95, .cu:152-432) and its
 * CPU twin for large molecules (src/morgan_fingerprint_cpu.cpp:61-255). */
int b200mol_morgan(const int32_t* d_atom_starts, const int32_t* d_bond_starts, const uint32_t* d_atom_inv,
                   const uint32_t* d_bond_inv, const uint16_t* d_bond_a, const uint16_t* d_bond_b, size_t nMols,
                   int maxAtomsPerMol, int maxBondsPerMol, int radius, int fpBits, uint32_t* d_out, void* stream);

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

/* ------------------------------------------------------------------------------------------
 * Distance-geometry preparation (per-molecule, matrix resident in shared memory).
 * Matrices are concatenated: matrix m occupies d_x[starts[m] .. starts[m+1]) = n_m * n_m doubles, row-major.
 * ---------------------------------------------------------------------------------------- */
/* In-place triangle-inequality smoothing of RDKit bounds matrices ([i][j], i<j = upper bound; [j][i] = lower bound).
 * d_ok[m] = 1 consistent / 0 inconsistent (lb > ub found; matrix left partially smoothed). tol as in RDKit
 * triangleSmoothBounds (0 = strict). Replaces triangleSmoothBoundsBatch (src/triangle_smooth.cu:132-247) and the CPU
 * call DistGeom::triangleSmoothBounds in src/embedder_utils.cpp:313,324. */
int b200mol_triangle_smooth(double* d_bounds, const int64_t* d_matrix_starts, int32_t nMats, double tol, int8_t* d_ok,
                            void* stream);
/* Top-numEigs eigenpairs by power iteration with deflation (RDKit PowerEigenSolver: tol 1e-3, <= 1000 iterations).
 * d_mats is destroyed. d_v0 (optional) start vectors, numEigs * n_m per matrix at d_v0_starts[m]; NULL = hashed
 * counter sequence from `seed`. d_eigvals[m][numEigs]; d_eigvecs row e of matrix m at d_vec_starts[m] + e * n_m;
 * d_n_converged[m] = number of eigenpairs found. Replaces BatchedEigenSolver::solve
 * (src/symmetric_eigensolver.cu:62-247). */
int b200mol_eig_topk(double* d_mats, const int64_t* d_matrix_starts, int32_t nMats, int numEigs, const double* d_v0,
                     const int64_t* d_v0_starts, uint32_t seed, double* d_eigvals, double* d_eigvecs,
                     const int64_t* d_vec_starts, int8_t* d_n_converged, void* stream);
/* Distance matrix -> metric matrix -> top-`dim` eigenpairs -> coordinates d_coords[(atom_starts[m]+i)*dim + j] =
 * sqrt(lambda_j) v_j[i]; d_ok[m] = 0 when an eigenvalue is not positive or did not converge (3-D AND 4-D; the
 * reference's InitialCoordinateGenerator is 3-D only, src/forcefields/coord_gen.cu:64,160). d_dist is destroyed. */
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
