// Weighted rigid alignment of conformers (RDKit rdMolAlign.AlignMol / GetAlignmentTransform / AlignMolConformers, which
// call Numerics::Alignment::AlignPoints): for every job, the rotation, translation (and optional mirror image) that best
// superpose a probe conformer's listed atoms onto a reference conformer's, its RMSD, and, when asked, the probe conformer
// moved in place. The reference library has no alignment; this is new ground.
//
// Per job (probe atoms p_i, reference atoms r_i, weights w_i, i < L, W = sum w):
//  * pass 1 (one warp per job): lanes stride over the L pairs and accumulate 17 fp64 sums -- W, sum w dp, sum w dr,
//    sum w (|dp|^2 + |dr|^2) and sum w dp dr^T -- of coordinates shifted by the job's first pair, dp = s (p - p_0),
//    dr = r - r_0 (s = -1 for the mirror image). The shift keeps the one-pass sums near-centred, so molecules 1e4 A
//    from the origin lose no more than ones at it; a butterfly reduces them, so every lane ends with the same bits.
//  * solve (one lane per job): the centred covariance S = sum w dp dr^T - (sum w dp)(sum w dr)^T / W, Horn's 4x4
//    quaternion matrix N(S), its eigenvectors by cyclic Jacobi capped at maxIters sweeps (the Numerical Recipes scheme
//    RDKit's AlignPoints uses), and from the eigenvector of the largest diagonal entry lambda: R = R(q),
//    t = r_bar - R s p_bar, SSR = G - 2 lambda (clamped at 0), RMSD = sqrt(SSR / L).
//  * pass 2 (the warp again, per job): R and the centroids are shuffled from the job's lane and lanes stride over ALL
//    atoms of the probe conformer, x' = R (s x - s p_bar) + r_bar.
// A warp takes 32 consecutive jobs: pass 1 runs job by job, lane k keeps job k's sums, the 32 solves run side by side,
// and pass 2 runs job by job. The solve is the only real arithmetic (~10^3 fp64 operations); doing it one job per lane
// instead of redundantly on every lane of a warp per job divides its issue slots by 32. Consecutive jobs that share a
// reference (AlignMolConformers) read its atoms from L2.
//
// Sums run in a fixed order that depends only on L: results are bitwise repeatable and independent of the other jobs.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "horn.cuh"

namespace b200 {
namespace {

using namespace horn;

constexpr int kAT = 128;  // threads per CTA: 4 warps, 128 jobs at a time

struct AlignJob {
  int32_t probe, ref, list, nAtoms;  // nAtoms: atoms of the probe conformer (pass 2)
};

// listStart[nLists + 1], pairs[.][2] (probe atom, reference atom), weights (null = 1). Lane k first loads job k's
// record, list bounds, conformer starts and first pair, so that the per-job loops wait on one level of loads (the pairs
// and their coordinates) instead of five.
__global__ void __launch_bounds__(kAT) alignKernel(int nJobs, const AlignJob* jobs, const int64_t* listStart,
                                                   const int2* pairs, const double* weights,
                                                   const int32_t* confAtomStart, double* xyz, int reflect, int maxIters,
                                                   int move, double* rmsd, double* transform) {
  const int    lane = threadIdx.x & 31;
  const int    nGrp = (nJobs + 31) / 32;
  const double sgn  = reflect ? -1.0 : 1.0;
  for (int grp = blockIdx.x * (kAT / 32) + (threadIdx.x >> 5); grp < nGrp; grp += gridDim.x * (kAT / 32)) {
    const int j0 = grp * 32, nj = min(32, nJobs - j0);
    // lane k: job k's list offset and length, atom offsets of its probe and reference, probe atom count, and the shifts
    // s p_0, r_0 (its first pair)
    int64_t myL0 = 0, myP = 0, myQ = 0;
    int     myL = 0, myA = 0;
    double  s0[6] = {0, 0, 0, 0, 0, 0};
    if (lane < nj) {
      const AlignJob jb = jobs[j0 + lane];
      myL0              = listStart[jb.list];
      myL               = static_cast<int>(listStart[jb.list + 1] - myL0);
      myP               = 3 * static_cast<int64_t>(confAtomStart[jb.probe]);
      myQ               = 3 * static_cast<int64_t>(confAtomStart[jb.ref]);
      myA               = jb.nAtoms;
      const int2 f      = pairs[myL0];
#pragma unroll
      for (int c = 0; c < 3; ++c) s0[c] = xyz[myP + 3 * f.x + c], s0[3 + c] = xyz[myQ + 3 * f.y + c];
    }
    double mine[kSums];  // lane k: the sums of job k
#pragma unroll
    for (int i = 0; i < kSums; ++i) mine[i] = 0.0;
    for (int k = 0; k < nj; ++k) {
      const int64_t l0 = __shfl_sync(0xffffffffu, myL0, k);
      const int     L  = __shfl_sync(0xffffffffu, myL, k);
      const double* P  = xyz + __shfl_sync(0xffffffffu, myP, k);
      const double* Q  = xyz + __shfl_sync(0xffffffffu, myQ, k);
      double        p0[3], r0[3], x[kSums];
#pragma unroll
      for (int c = 0; c < 3; ++c) p0[c] = __shfl_sync(0xffffffffu, s0[c], k), r0[c] = __shfl_sync(0xffffffffu, s0[3 + c], k);
#pragma unroll
      for (int i = 0; i < kSums; ++i) x[i] = 0.0;
      for (int i = lane; i < L; i += 32) {
        const int2   pr = pairs[l0 + i];
        const double w  = weights ? weights[l0 + i] : 1.0;
        double       dp[3], dr[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          dp[c] = sgn * (P[3 * pr.x + c] - p0[c]);
          dr[c] = Q[3 * pr.y + c] - r0[c];
        }
        accumulate(x, w, dp, dr);
      }
#pragma unroll
      for (int i = 0; i < kSums; ++i) {
        x[i] = warpSum(x[i]);
        if (lane == k) mine[i] = x[i];
      }
    }

    // one lane per job: R, and the centroids s p_bar = s p_0 + cp, r_bar = r_0 + cr
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, pc[3] = {0, 0, 0}, rc[3] = {0, 0, 0};
    if (lane < nj) {
      double       cp[3], cr[3];
      const double v = solve(mine, myL, maxIters, R, cp, cr);
#pragma unroll
      for (int c = 0; c < 3; ++c) pc[c] = sgn * s0[c] + cp[c], rc[c] = s0[3 + c] + cr[c];
      rmsd[j0 + lane] = v;
      if (transform) {
        double* T = transform + 16 * static_cast<int64_t>(j0 + lane);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
          for (int c = 0; c < 3; ++c) T[4 * r + c] = sgn * R[3 * r + c];
          T[4 * r + 3] = rc[r] - (R[3 * r] * pc[0] + R[3 * r + 1] * pc[1] + R[3 * r + 2] * pc[2]);
        }
        T[12] = T[13] = T[14] = 0.0;
        T[15] = 1.0;
      }
    }
    if (!move) continue;
    for (int k = 0; k < nj; ++k) {
      double Rk[9], pk[3], rk[3];
#pragma unroll
      for (int i = 0; i < 9; ++i) Rk[i] = __shfl_sync(0xffffffffu, R[i], k);
#pragma unroll
      for (int c = 0; c < 3; ++c) pk[c] = __shfl_sync(0xffffffffu, pc[c], k), rk[c] = __shfl_sync(0xffffffffu, rc[c], k);
      double*   P = xyz + __shfl_sync(0xffffffffu, myP, k);
      const int A = __shfl_sync(0xffffffffu, myA, k);
      for (int a = lane; a < A; a += 32) {
        double y[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) y[c] = sgn * P[3 * a + c] - pk[c];
#pragma unroll
        for (int r = 0; r < 3; ++r) P[3 * a + r] = Rk[3 * r] * y[0] + Rk[3 * r + 1] * y[1] + Rk[3 * r + 2] * y[2] + rk[r];
      }
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_align(int32_t nJobs, const int32_t* h_job_probe, const int32_t* h_job_ref, const int32_t* h_job_list,
                             int32_t nConfs, const int32_t* h_conf_atoms, const int32_t* d_conf_atom_start, double* d_xyz,
                             int32_t nLists, const int64_t* h_list_start, const int32_t* h_list_pairs,
                             const double* h_list_weights, int32_t reflect, int32_t maxIters, int32_t move,
                             double* d_rmsd, double* d_transform, void* stream) {
  return guarded([&] {
    B200_REQUIRE(nJobs >= 0, "negative job count");
    B200_REQUIRE(maxIters >= 1, "maxIters must be >= 1, got %d", maxIters);
    if (nJobs == 0) return;
    B200_REQUIRE(h_job_probe && h_job_ref && h_job_list && h_conf_atoms && h_list_start && h_list_pairs, "null table");
    B200_REQUIRE(nConfs >= 1 && nLists >= 1, "a job needs at least one conformer and one pair list");
    B200_REQUIRE(h_list_start[0] == 0, "pair lists must start at 0");

    // per list: L >= 1, finite weights >= 0 with W > 0, and the largest probe and reference atom index
    std::vector<int32_t> maxP(nLists), maxR(nLists);
    for (int l = 0; l < nLists; ++l) {
      const int64_t a0 = h_list_start[l], a1 = h_list_start[l + 1];
      B200_REQUIRE(a1 > a0, "pair list %d is empty", l);
      double W = 0.0;
      maxP[l] = maxR[l] = -1;
      for (int64_t i = a0; i < a1; ++i) {
        const int32_t p = h_list_pairs[2 * i], r = h_list_pairs[2 * i + 1];
        B200_REQUIRE(p >= 0 && r >= 0, "pair list %d holds a negative atom index", l);
        maxP[l] = std::max(maxP[l], p);
        maxR[l] = std::max(maxR[l], r);
        if (h_list_weights) {
          const double w = h_list_weights[i];
          B200_REQUIRE(std::isfinite(w) && w >= 0.0, "pair list %d: weight %g must be finite and >= 0", l, w);
          W += w;
        }
      }
      B200_REQUIRE(!h_list_weights || W > 0.0, "pair list %d: its weights sum to 0", l);
    }
    for (int c = 0; c < nConfs; ++c) B200_REQUIRE(h_conf_atoms[c] >= 0, "conformer %d: negative atom count", c);
    std::vector<AlignJob> jobs(nJobs);
    for (int j = 0; j < nJobs; ++j) {
      const int p = h_job_probe[j], r = h_job_ref[j], l = h_job_list[j];
      B200_REQUIRE(p >= 0 && p < nConfs && r >= 0 && r < nConfs, "job %d: conformer outside [0, %d)", j, nConfs);
      B200_REQUIRE(l >= 0 && l < nLists, "job %d: pair list %d outside [0, %d)", j, l, nLists);
      B200_REQUIRE(maxP[l] < h_conf_atoms[p], "job %d: pair list %d holds probe atom %d, conformer %d has %d atoms", j, l,
                   maxP[l], p, h_conf_atoms[p]);
      B200_REQUIRE(maxR[l] < h_conf_atoms[r], "job %d: pair list %d holds reference atom %d, conformer %d has %d atoms",
                   j, l, maxR[l], r, h_conf_atoms[r]);
      jobs[j] = AlignJob{p, r, l, h_conf_atoms[p]};
    }
    if (move) {  // a moved conformer is written by one job and read by no other
      std::vector<uint8_t> role(nConfs, 0);  // bit 0: some job's probe, bit 1: some job's reference
      for (int j = 0; j < nJobs; ++j) role[h_job_ref[j]] |= 2;
      for (int j = 0; j < nJobs; ++j) {
        const int p = h_job_probe[j];
        B200_REQUIRE(!(role[p] & 1), "job %d: probe conformer %d is moved by an earlier job too", j, p);
        B200_REQUIRE(!(role[p] & 2), "job %d: probe conformer %d is also a reference", j, p);
        role[p] |= 1;
      }
    }
    B200_REQUIRE(d_conf_atom_start && d_xyz && d_rmsd, "null device pointer");

    // one upload: jobs, list starts, pairs, weights
    const int64_t nPairs = h_list_start[nLists];
    auto          align  = [](size_t b) { return (b + 15) & ~static_cast<size_t>(15); };
    const size_t  oStart = align(sizeof(AlignJob) * nJobs), oPairs = align(oStart + 8 * (static_cast<size_t>(nLists) + 1)),
                 oW = align(oPairs + 8 * static_cast<size_t>(nPairs)),
                 nBytes = oW + (h_list_weights ? 8 * static_cast<size_t>(nPairs) : 0);
    std::vector<unsigned char> host(nBytes, 0);
    auto put = [&](size_t o, const void* p, size_t b) { std::copy_n(static_cast<const unsigned char*>(p), b, host.data() + o); };
    put(0, jobs.data(), sizeof(AlignJob) * nJobs);
    put(oStart, h_list_start, 8 * (static_cast<size_t>(nLists) + 1));
    put(oPairs, h_list_pairs, 8 * static_cast<size_t>(nPairs));
    if (h_list_weights) put(oW, h_list_weights, 8 * static_cast<size_t>(nPairs));
    const cudaStream_t     s = asStream(stream);
    Scratch<unsigned char> plan(nBytes, s);
    B200_CUDA(cudaMemcpyAsync(plan.get(), host.data(), nBytes, cudaMemcpyHostToDevice, s));
    const int64_t warps  = (nJobs + 31) / 32;
    const int     blocks = static_cast<int>(std::min<int64_t>((warps + kAT / 32 - 1) / (kAT / 32), static_cast<int64_t>(smCount()) * 8));
    alignKernel<<<blocks, kAT, 0, s>>>(nJobs, reinterpret_cast<const AlignJob*>(plan.get()),
                                       reinterpret_cast<const int64_t*>(plan.get() + oStart),
                                       reinterpret_cast<const int2*>(plan.get() + oPairs),
                                       h_list_weights ? reinterpret_cast<const double*>(plan.get() + oW) : nullptr,
                                       d_conf_atom_start, d_xyz, reflect ? 1 : 0, maxIters, move ? 1 : 0, d_rmsd,
                                       d_transform);
    B200_LAUNCHED();
  });
}
