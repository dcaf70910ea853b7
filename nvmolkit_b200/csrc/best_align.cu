// Symmetry-aware alignment of conformers (RDKit rdMolAlign.GetBestRMS / GetBestAlignmentTransform / CalcRMS): for every
// job, the best of K atom mappings between a probe conformer and a reference conformer, its RMSD and index and, when
// asked, its transform and the probe conformer moved in place. The reference library has no alignment; this is new
// ground.
//
// A job's mapping set holds the probe list P and K reference lists Q_k, L atoms each; mapping k pairs P[i] with Q_k[i].
// A unit is one (job, mapping). Per unit the arithmetic is that of align.cu, through the same horn.cuh:
//  * sums (the warp, per unit): lanes stride over the L pairs and accumulate the 17 sums of coordinates shifted by the
//    unit's first pair, a butterfly reduces them, and the unit's lane keeps them. CalcRMS (mode 1) sums w |p - r|^2 on
//    the coordinates as given instead.
//  * solve (one lane per unit): Horn's matrix and the Jacobi sweep, or sqrt(sum / L) for CalcRMS.
//  * choice: a segmented scan over the lanes takes each job's first strictly smallest RMSD (RDKit's `if (rms < best)`);
//    the winner's rotation and centroids are shuffled from its lane, and the warp writes the outputs and moves all atoms
//    of the probe.
// A warp runs one task: consecutive jobs whose K add up to at most 32, one unit per lane (K = 1: 32 jobs, as align.cu),
// or one job with K > 32, in groups of 32 mappings whose winners it keeps as it goes. So the solves fill the lanes at
// any K, and the host tables stay O(jobs + sum of set sizes): the K lists of a set are shared by every job that names it.
//
// A unit's sums and solve do not depend on anything else in the call, and the choice compares them in mapping order:
// results are bitwise repeatable, independent of the other jobs, and a job with K = 1 gives b200mol_align's bits.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "horn.cuh"

namespace b200 {
namespace {

using namespace horn;

constexpr int      kBT   = 128;  // threads per CTA: 4 warps, one task each
constexpr unsigned kFull = 0xffffffffu;

struct BestJob {
  int32_t probe, ref, set, nAtoms;  // nAtoms: atoms of the probe conformer (the move)
};
struct MapSet {
  int64_t start, wStart;  // P at atoms[start], Q_k at atoms[start + (k + 1) L]; weights at weights[wStart]
  int32_t K, L;
};
struct Task {
  int32_t job0, nJobs;  // nJobs consecutive jobs with sum K <= 32, or one job with K > 32
};

__global__ void __launch_bounds__(kBT) bestAlignKernel(int nTasks, const Task* tasks, const BestJob* jobs,
                                                       const MapSet* sets, const int16_t* atoms, const double* weights,
                                                       const int32_t* confAtomStart, double* xyz, int mode, int reflect,
                                                       int maxIters, int move, double* rmsd, int32_t* best,
                                                       double* transform) {
  const int    lane = threadIdx.x & 31;
  const double sgn  = reflect ? -1.0 : 1.0;
  for (int t = blockIdx.x * (kBT / 32) + (threadIdx.x >> 5); t < nTasks; t += gridDim.x * (kBT / 32)) {
    const Task tk = tasks[t];
    // lane j < nJobs: job j's record, set and conformer offsets
    int     myK = 0, myL = 0, myA = 0;
    int64_t myStart = 0, myW = 0, myP = 0, myQ = 0;
    if (lane < tk.nJobs) {
      const BestJob jb = jobs[tk.job0 + lane];
      const MapSet  st = sets[jb.set];
      myK = st.K, myL = st.L, myA = jb.nAtoms, myStart = st.start, myW = st.wStart;
      myP = 3 * static_cast<int64_t>(confAtomStart[jb.probe]);
      myQ = 3 * static_cast<int64_t>(confAtomStart[jb.ref]);
    }
    int incl = myK;  // inclusive prefix of K over the task's jobs: job j's units start at lane incl - K
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(kFull, incl, o);
      if (lane >= o) incl += y;
    }
    const int      excl    = incl - myK;
    const int      kTot    = __shfl_sync(kFull, incl, 31);
    const int      nGroups = (kTot + 31) / 32;  // > 1 only for a task of one job
    const unsigned heads   = __reduce_or_sync(kFull, lane < tk.nJobs ? 1u << excl : 0u);
    const unsigned le      = heads & (kFull >> (31 - lane));
    const int      jl      = __popc(le) - 1;        // this lane's job within the task
    const int      seg     = 31 - __clz(le);        // the lane of that job's first unit
    const int      nJobs   = nGroups > 1 ? 1 : tk.nJobs;

    double bestV = 0.0, bR[9], bP[3], bQ[3];  // the winner so far, the same on every lane
    int    bestK = 0;
    for (int g = 0; g < nGroups; ++g) {
      // this lane's unit: mapping k of job jl
      const int     k     = g * 32 + lane - seg;
      const int     Kj    = __shfl_sync(kFull, myK, jl);
      const bool    valid = k < Kj;
      const int     L     = __shfl_sync(kFull, myL, jl);
      const int64_t pOff  = __shfl_sync(kFull, myStart, jl);
      const int64_t qOff  = pOff + (static_cast<int64_t>(k) + 1) * L;
      const int64_t wOff  = __shfl_sync(kFull, myW, jl);
      const int64_t Pb    = __shfl_sync(kFull, myP, jl);
      const int64_t Qb    = __shfl_sync(kFull, myQ, jl);
      double        s0[6] = {0, 0, 0, 0, 0, 0};  // the unit's first pair: p_0, r_0
      if (valid && !mode) {
        const int pa = atoms[pOff], qa = atoms[qOff];
#pragma unroll
        for (int c = 0; c < 3; ++c) s0[c] = xyz[Pb + 3 * pa + c], s0[3 + c] = xyz[Qb + 3 * qa + c];
      }
      const int nUnits = __popc(__ballot_sync(kFull, valid));  // the valid units are lanes 0 .. nUnits - 1

      double mine[kSums];  // lane u: the sums of unit u
#pragma unroll
      for (int i = 0; i < kSums; ++i) mine[i] = 0.0;
      for (int u = 0; u < nUnits; ++u) {
        const int     Lu = __shfl_sync(kFull, L, u);
        const int64_t po = __shfl_sync(kFull, pOff, u), qo = __shfl_sync(kFull, qOff, u);
        const int64_t wo = __shfl_sync(kFull, wOff, u);
        const double* P  = xyz + __shfl_sync(kFull, Pb, u);
        const double* Q  = xyz + __shfl_sync(kFull, Qb, u);
        if (mode) {
          double x = 0.0;
          for (int i = lane; i < Lu; i += 32) {
            const int    pa = atoms[po + i], qa = atoms[qo + i];
            const double w  = weights ? weights[wo + i] : 1.0;
            double       d[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) d[c] = P[3 * pa + c] - Q[3 * qa + c];
            x += w * (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
          }
          x = warpSum(x);
          if (lane == u) mine[0] = x;
          continue;
        }
        double p0[3], r0[3], x[kSums];
#pragma unroll
        for (int c = 0; c < 3; ++c) p0[c] = __shfl_sync(kFull, s0[c], u), r0[c] = __shfl_sync(kFull, s0[3 + c], u);
#pragma unroll
        for (int i = 0; i < kSums; ++i) x[i] = 0.0;
        for (int i = lane; i < Lu; i += 32) {
          const int    pa = atoms[po + i], qa = atoms[qo + i];
          const double w  = weights ? weights[wo + i] : 1.0;
          double       dp[3], dr[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            dp[c] = sgn * (P[3 * pa + c] - p0[c]);
            dr[c] = Q[3 * qa + c] - r0[c];
          }
          accumulate(x, w, dp, dr);
        }
#pragma unroll
        for (int i = 0; i < kSums; ++i) {
          x[i] = warpSum(x[i]);
          if (lane == u) mine[i] = x[i];
        }
      }

      // one lane per unit: its RMSD, R and centroids s p_bar, r_bar
      double v = INFINITY, R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, pc[3] = {0, 0, 0}, rc[3] = {0, 0, 0};
      if (valid) {
        if (mode) {
          v = sqrt(mine[0] / L);
        } else {
          double cp[3], cr[3];
          v = solve(mine, L, maxIters, R, cp, cr);
#pragma unroll
          for (int c = 0; c < 3; ++c) pc[c] = sgn * s0[c] + cp[c], rc[c] = s0[3 + c] + cr[c];
        }
      }
      // segmented inclusive scan of (RMSD, mapping) over each job's lanes: the lower mapping wins a tie, a NaN loses
      double sv = v;
      int    sk = k, ss = lane;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double ov = __shfl_up_sync(kFull, sv, o);
        const int    ok = __shfl_up_sync(kFull, sk, o), os = __shfl_up_sync(kFull, ss, o);
        if (lane - o >= seg && (ov <= sv || sv != sv)) sv = ov, sk = ok, ss = os;
      }

      for (int j = 0; j < nJobs; ++j) {
        const int    e  = min(__shfl_sync(kFull, excl + myK - 1, j) - 32 * g, 31);  // job j's last unit in this group
        const double wv = __shfl_sync(kFull, sv, e);
        const int    wk = __shfl_sync(kFull, sk, e), ws = __shfl_sync(kFull, ss, e);
        if (g == 0 || wv < bestV || bestV != bestV) {
          bestV = wv, bestK = wk;
#pragma unroll
          for (int i = 0; i < 9; ++i) bR[i] = __shfl_sync(kFull, R[i], ws);
#pragma unroll
          for (int c = 0; c < 3; ++c) bP[c] = __shfl_sync(kFull, pc[c], ws), bQ[c] = __shfl_sync(kFull, rc[c], ws);
        }
        if (g < nGroups - 1) continue;
        const int64_t job = tk.job0 + j;
        if (lane == 0) {
          rmsd[job] = bestV;
          if (best) best[job] = bestK;
        }
        if (transform && lane == 0) {
          double* T = transform + 16 * job;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
#pragma unroll
            for (int c = 0; c < 3; ++c) T[4 * r + c] = sgn * bR[3 * r + c];
            T[4 * r + 3] = bQ[r] - (bR[3 * r] * bP[0] + bR[3 * r + 1] * bP[1] + bR[3 * r + 2] * bP[2]);
          }
          T[12] = T[13] = T[14] = 0.0;
          T[15] = 1.0;
        }
        if (!move) continue;
        double*   P = xyz + __shfl_sync(kFull, myP, j);
        const int A = __shfl_sync(kFull, myA, j);
        for (int a = lane; a < A; a += 32) {
          double y[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) y[c] = sgn * P[3 * a + c] - bP[c];
#pragma unroll
          for (int r = 0; r < 3; ++r) P[3 * a + r] = bR[3 * r] * y[0] + bR[3 * r + 1] * y[1] + bR[3 * r + 2] * y[2] + bQ[r];
        }
      }
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_best_align(int32_t nJobs, const int32_t* h_job_probe, const int32_t* h_job_ref,
                                  const int32_t* h_job_set, int32_t nConfs, const int32_t* h_conf_atoms,
                                  const int32_t* d_conf_atom_start, double* d_xyz, int32_t nSets,
                                  const int64_t* h_set_start, const int32_t* h_set_count, const int32_t* h_set_len,
                                  const int16_t* h_set_atoms, const double* h_set_weights, int32_t mode,
                                  int32_t reflect, int32_t maxIters, int32_t move, double* d_rmsd, int32_t* d_best,
                                  double* d_transform, void* stream) {
  return guarded([&] {
    B200_REQUIRE(nJobs >= 0, "negative job count");
    B200_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (align) or 1 (in place), got %d", mode);
    B200_REQUIRE(maxIters >= 1, "maxIters must be >= 1, got %d", maxIters);
    B200_REQUIRE(mode == 0 || (!move && !reflect && !d_transform), "in-place mode takes no move, reflect or transform");
    if (nJobs == 0) return;
    B200_REQUIRE(h_job_probe && h_job_ref && h_job_set && h_conf_atoms && h_set_start && h_set_count && h_set_len &&
                     h_set_atoms,
                 "null table");
    B200_REQUIRE(nConfs >= 1 && nSets >= 1, "a job needs at least one conformer and one mapping set");
    B200_REQUIRE(h_set_start[0] == 0, "mapping sets must start at 0");

    // per set: K >= 1, L >= 1, its size, no index twice in a list, finite weights >= 0 with W > 0, and the largest probe
    // and reference atom index
    std::vector<MapSet>  sets(nSets);
    std::vector<int32_t> maxP(nSets), maxR(nSets);
    std::vector<int64_t> seen(32768, -1);  // the last list that held each atom index
    int64_t              listId = 0, nW = 0;
    for (int s = 0; s < nSets; ++s) {
      const int32_t K = h_set_count[s], L = h_set_len[s];
      B200_REQUIRE(K >= 1 && L >= 1, "mapping set %d: K = %d and L = %d must be >= 1", s, K, L);
      const int64_t a0 = h_set_start[s], a1 = h_set_start[s + 1];
      B200_REQUIRE(a1 - a0 == (static_cast<int64_t>(K) + 1) * L, "mapping set %d holds %lld atoms, (K + 1) L = %lld", s,
                   static_cast<long long>(a1 - a0), static_cast<long long>((static_cast<int64_t>(K) + 1) * L));
      maxP[s] = maxR[s] = -1;
      for (int64_t l = 0; l <= K; ++l, ++listId) {
        for (int64_t i = a0 + l * L; i < a0 + (l + 1) * L; ++i) {
          const int32_t a = h_set_atoms[i];
          B200_REQUIRE(a >= 0, "mapping set %d holds a negative atom index", s);
          B200_REQUIRE(seen[a] != listId, "mapping set %d: list %lld holds atom %d twice", s, static_cast<long long>(l),
                       a);
          seen[a] = listId;
          int32_t& m = l == 0 ? maxP[s] : maxR[s];
          m          = std::max(m, a);
        }
      }
      if (h_set_weights) {
        double W = 0.0;
        for (int i = 0; i < L; ++i) {
          const double w = h_set_weights[nW + i];
          B200_REQUIRE(std::isfinite(w) && w >= 0.0, "mapping set %d: weight %g must be finite and >= 0", s, w);
          W += w;
        }
        B200_REQUIRE(W > 0.0, "mapping set %d: its weights sum to 0", s);
      }
      sets[s] = MapSet{a0, nW, K, L};
      nW += L;
    }
    for (int c = 0; c < nConfs; ++c) B200_REQUIRE(h_conf_atoms[c] >= 0, "conformer %d: negative atom count", c);
    std::vector<BestJob> jobs(nJobs);
    for (int j = 0; j < nJobs; ++j) {
      const int p = h_job_probe[j], r = h_job_ref[j], s = h_job_set[j];
      B200_REQUIRE(p >= 0 && p < nConfs && r >= 0 && r < nConfs, "job %d: conformer outside [0, %d)", j, nConfs);
      B200_REQUIRE(s >= 0 && s < nSets, "job %d: mapping set %d outside [0, %d)", j, s, nSets);
      B200_REQUIRE(maxP[s] < h_conf_atoms[p], "job %d: mapping set %d holds probe atom %d, conformer %d has %d atoms",
                   j, s, maxP[s], p, h_conf_atoms[p]);
      B200_REQUIRE(maxR[s] < h_conf_atoms[r],
                   "job %d: mapping set %d holds reference atom %d, conformer %d has %d atoms", j, s, maxR[s], r,
                   h_conf_atoms[r]);
      jobs[j] = BestJob{p, r, s, h_conf_atoms[p]};
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

    // tasks: runs of consecutive jobs with sum K <= 32, and every job with K > 32 on its own
    std::vector<Task> tasks;
    int               open = 33;  // units of the last task, or 33 when it takes no more jobs
    for (int j = 0; j < nJobs; ++j) {
      const int K = sets[h_job_set[j]].K;
      if (K > 32) {
        tasks.push_back(Task{j, 1});
        open = 33;
      } else if (open + K <= 32) {
        ++tasks.back().nJobs;
        open += K;
      } else {
        tasks.push_back(Task{j, 1});
        open = K;
      }
    }

    // one upload: jobs, sets, tasks, atoms, weights
    const int64_t nAtoms = h_set_start[nSets];
    auto          align  = [](size_t b) { return (b + 15) & ~static_cast<size_t>(15); };
    const size_t  oSets = align(sizeof(BestJob) * nJobs), oTasks = align(oSets + sizeof(MapSet) * nSets),
                 oAtoms = align(oTasks + sizeof(Task) * tasks.size()), oW = align(oAtoms + 2 * static_cast<size_t>(nAtoms)),
                 nBytes = oW + (h_set_weights ? 8 * static_cast<size_t>(nW) : 0);
    std::vector<unsigned char> host(nBytes, 0);
    auto put = [&](size_t o, const void* p, size_t b) { std::copy_n(static_cast<const unsigned char*>(p), b, host.data() + o); };
    put(0, jobs.data(), sizeof(BestJob) * nJobs);
    put(oSets, sets.data(), sizeof(MapSet) * nSets);
    put(oTasks, tasks.data(), sizeof(Task) * tasks.size());
    put(oAtoms, h_set_atoms, 2 * static_cast<size_t>(nAtoms));
    if (h_set_weights) put(oW, h_set_weights, 8 * static_cast<size_t>(nW));
    const cudaStream_t     s = asStream(stream);
    Scratch<unsigned char> plan(nBytes, s);
    B200_CUDA(cudaMemcpyAsync(plan.get(), host.data(), nBytes, cudaMemcpyHostToDevice, s));
    const int64_t nTasks = static_cast<int64_t>(tasks.size());
    const int     blocks = static_cast<int>(std::min<int64_t>((nTasks + kBT / 32 - 1) / (kBT / 32), static_cast<int64_t>(smCount()) * 8));
    bestAlignKernel<<<blocks, kBT, 0, s>>>(
        static_cast<int>(nTasks), reinterpret_cast<const Task*>(plan.get() + oTasks),
        reinterpret_cast<const BestJob*>(plan.get()), reinterpret_cast<const MapSet*>(plan.get() + oSets),
        reinterpret_cast<const int16_t*>(plan.get() + oAtoms),
        h_set_weights ? reinterpret_cast<const double*>(plan.get() + oW) : nullptr, d_conf_atom_start, d_xyz, mode,
        reflect ? 1 : 0, maxIters, move ? 1 : 0, d_rmsd, d_best, d_transform);
    B200_LAUNCHED();
  });
}
