// Torsion fingerprint deviation (TFD) matrices between the conformers of each molecule. Semantics (RDKit's
// TorsionFingerprints.CalculateTFD; the reference restates them in src/tfd/tfd_detail.h:62-120 and
// src/tfd/tfd_kernels.cu:84-166): per torsion a deviation d between conformers I > J,
//   single     d = circdiff(phi_I, phi_J)
//   symmetric  d = min over quartet pairs (q, q') of circdiff(phi_I[q], phi_J[q'])
//   ring       d = | mean_q |phi_I[q]| - mean_q |phi_J[q]| |
// with circdiff(a, b) = min(|a - b|, 360 - |a - b|), phi signed in (-180, 180], and TFD = sum w d / maxDev / sum w
// (0 when sum w <= 1e-10). A quartet whose cross product i-j x j-k or j-k x k-l is exactly zero has phi = 0.
//
// Two passes instead of the reference's one block per molecule and one thread per pair:
//  * feature pass: one thread per (conformer, torsion) computes the torsion's dihedrals once, in fp64 from the fp64
//    coordinates, and stores the conformer's *feature row* in fp32: one angle per single torsion, the Q angles of a
//    symmetric torsion, the already averaged |phi| of a ring torsion; rows padded to 16 B.
//  * pair pass: units are (molecule, R x R tile of the lower triangle); persistent CTAs take units from an atomic
//    queue over the unit prefix sum, so one molecule with thousands of conformers and thousands of molecules with a
//    few each both fill the machine. A unit bulk-copies its row block's and column block's feature rows and the
//    molecule's torsion descriptors (offset, Q, type, w / maxDev) into shared memory; each thread owns one column and
//    up to 16 rows, so a column's features are read once per torsion and a row's are broadcast. Output rows are
//    contiguous in J, so stores coalesce. R is 64 unless the molecule's rows do not fit the shared-memory budget,
//    then the largest power of two that does.
// Every sum runs in a fixed order: two runs give bitwise-equal matrices.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "tiles.cuh"
#include "tma.cuh"

namespace b200 {
namespace {

constexpr int    kPT         = 256;        // threads of both kernels
constexpr int    kMaxR       = 64;         // tile side in conformers
constexpr int    kMaxPairs   = kMaxR * kMaxR / kPT;
constexpr size_t kSmemBudget = 96 * 1024;  // per CTA: two CTAs per SM
constexpr int    kSymRegs    = 9;          // symmetric torsions up to 3 x 3 quartets keep a column's angles in registers

struct MolDesc {
  int64_t featBase;  // float offset of the molecule's first feature row
  int64_t outBase;   // offset of its lower triangle in the output
  int32_t confStart; // first entry of the molecule in the conformer order
  int32_t nConf;
  int32_t F;         // floats per feature row (multiple of 4)
  int32_t R;         // tile side
  int32_t T;         // tiles per side
  int32_t torStart;  // first torsion descriptor
  int32_t nTors;
  float   invSumW;   // 1 / sum w, 0 when sum w <= 1e-10
};

struct TorDesc {  // 16 B: bulk-copied as a block
  int32_t off;    // float offset of the torsion's features in the row
  int32_t Q;      // quartets
  int32_t type;   // B200MOL_TFD_*
  float   wm;     // w / maxDev
};

// a x b with every product rounded on its own (__dmul_rn is never contracted into an FMA): the cross product of
// parallel vectors is then exactly zero, as on the CPU, so the phi = 0 convention sees the same geometries there
__device__ __forceinline__ void cross(const double* a, const double* b, double* c) {
  c[0] = __dmul_rn(a[1], b[2]) - __dmul_rn(a[2], b[1]);
  c[1] = __dmul_rn(a[2], b[0]) - __dmul_rn(a[0], b[2]);
  c[2] = __dmul_rn(a[0], b[1]) - __dmul_rn(a[1], b[0]);
}
__device__ __forceinline__ double dot(const double* a, const double* b) {
  return __dmul_rn(a[0], b[0]) + __dmul_rn(a[1], b[1]) + __dmul_rn(a[2], b[2]);
}

__device__ __forceinline__ double dihedralDeg(const double* p0, const double* p1, const double* p2, const double* p3) {
  const double v1[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
  const double v2[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double v3[3] = {p3[0] - p2[0], p3[1] - p2[1], p3[2] - p2[2]};
  double       n1[3], n2[3], m[3];
  cross(v1, v2, n1);
  cross(v2, v3, n2);
  if ((n1[0] == 0.0 && n1[1] == 0.0 && n1[2] == 0.0) || (n2[0] == 0.0 && n2[1] == 0.0 && n2[2] == 0.0)) return 0.0;
  cross(n1, n2, m);
  const double x = dot(n1, n2);
  const double y = dot(m, v2) / __dsqrt_rn(dot(v2, v2));
  double       phi  = atan2(y, x) * 57.295779513082320876798;
  if (phi <= -180.0) phi += 360.0;
  return phi;
}

// one thread per (conformer entry, torsion) of every molecule; workStart[nMols+1] = prefix of nConf * nTors
__global__ void __launch_bounds__(kPT) tfdFeatureKernel(int nMols, const int64_t* workStart, const MolDesc* mols,
                                                        const TorDesc* tors, const int32_t* torQStart, const int16_t* quartets,
                                                        const int32_t* confOrder, const int32_t* confAtomStart, const double* xyz,
                                                        float* feat) {
  const int64_t total = workStart[nMols];
  for (int64_t w = blockIdx.x * static_cast<int64_t>(kPT) + threadIdx.x; w < total; w += static_cast<int64_t>(gridDim.x) * kPT) {
    const int      m   = upperIndex(workStart, nMols + 1, w);
    const MolDesc  md  = mols[m];
    const int64_t  loc = w - workStart[m];
    const int      k = static_cast<int>(loc / md.nTors), t = static_cast<int>(loc % md.nTors);
    const int      entry = md.confStart + k;
    const int      c     = confOrder ? confOrder[entry] : entry;
    const double*  pos   = xyz + static_cast<int64_t>(confAtomStart[c]) * 3;
    float*         row   = feat + md.featBase + static_cast<int64_t>(k) * md.F;
    const TorDesc  td    = tors[md.torStart + t];
    const int16_t* q     = quartets + static_cast<int64_t>(torQStart[md.torStart + t]) * 4;
    double         ringSum = 0.0;
    for (int j = 0; j < td.Q; ++j) {
      const double phi = dihedralDeg(pos + 3 * q[4 * j], pos + 3 * q[4 * j + 1], pos + 3 * q[4 * j + 2], pos + 3 * q[4 * j + 3]);
      if (td.type == B200MOL_TFD_RING) ringSum += fabs(phi);
      else row[td.off + j] = static_cast<float>(phi);
    }
    if (td.type == B200MOL_TFD_RING) row[td.off] = static_cast<float>(ringSum / td.Q);
    if (t == md.nTors - 1)  // the row's padding
      for (int p = td.off + (td.type == B200MOL_TFD_SYMMETRIC ? td.Q : 1); p < md.F; ++p) row[p] = 0.0f;
  }
}

__device__ __forceinline__ float circDiff(float a, float b) {
  const float d = fabsf(a - b);
  return fminf(d, 360.0f - d);
}

// unitStart[nMols+1]: prefix of T(T+1)/2 lower-triangle tiles per molecule; *queue starts at 0
__global__ void __launch_bounds__(kPT) tfdPairKernel(int nMols, const int64_t* unitStart, const MolDesc* mols,
                                                     const TorDesc* tors, const float* feat, float* out,
                                                     unsigned long long* queue) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint64_t bar;
  __shared__ long long sUnit;
  const int           tid   = threadIdx.x;
  const int64_t       total = unitStart[nMols];
  uint32_t            phase = 0;
  if (tid == 0) {
    mbarInit(&bar, 1);
    fenceBarrierInit();
  }
  __syncthreads();
  for (;;) {
    if (tid == 0) sUnit = static_cast<long long>(atomicAdd(queue, 1ull));
    __syncthreads();
    const int64_t u = sUnit;
    if (u >= total) break;
    const int     m  = upperIndex(unitStart, nMols + 1, u);
    const MolDesc md = mols[m];
    int ti, tj;
    lowerTriangleTile(u - unitStart[m], ti, tj);
    const int R     = md.R, F = md.F;
    const int nRows = min(R, md.nConf - ti * R), nCols = min(R, md.nConf - tj * R);
    float*    sRow  = reinterpret_cast<float*>(smem);
    float*    sCol  = ti == tj ? sRow : sRow + R * F;
    TorDesc*  sTor  = reinterpret_cast<TorDesc*>(sRow + 2 * R * F);
    const uint32_t rowBytes = static_cast<uint32_t>(nRows) * F * 4, colBytes = ti == tj ? 0u : static_cast<uint32_t>(nCols) * F * 4;
    const uint32_t torBytes = static_cast<uint32_t>(md.nTors) * sizeof(TorDesc);
    const uint32_t bytes    = rowBytes + colBytes + torBytes;
    if (bytes) {
      if (tid == 0) {
        fenceProxyAsync();  // the previous unit's generic reads of the buffers come before these async writes
        mbarExpectTx(&bar, bytes);
        const float* base = feat + md.featBase;
        if (rowBytes) bulkLoad1D(sRow, base + static_cast<int64_t>(ti) * R * F, rowBytes, &bar);
        if (colBytes) bulkLoad1D(sCol, base + static_cast<int64_t>(tj) * R * F, colBytes, &bar);
        if (torBytes) bulkLoad1D(sTor, tors + md.torStart, torBytes, &bar);
      }
      mbarWait(&bar, phase);
      phase ^= 1u;
    }
    // thread -> column j, rows i0 + k * S
    const int  j = tid % R, i0 = tid / R, S = kPT / R;
    const int  P = R * R >= kPT ? R * R / kPT : (tid < R * R ? 1 : 0);
    const bool colOk = j < nCols;
    float      acc[kMaxPairs];
#pragma unroll
    for (int k = 0; k < kMaxPairs; ++k) acc[k] = 0.0f;
    if (colOk) {
      const float* cj = sCol + j * F;
      for (int t = 0; t < md.nTors; ++t) {
        const TorDesc td = sTor[t];
        if (td.type == B200MOL_TFD_SYMMETRIC && td.Q <= kSymRegs) {  // the column's angles in registers
          float y[kSymRegs];
#pragma unroll
          for (int b = 0; b < kSymRegs; ++b) y[b] = b < td.Q ? cj[td.off + b] : 0.0f;
#pragma unroll
          for (int k = 0; k < kMaxPairs; ++k) {
            const int i = i0 + k * S;
            if (k < P && i < nRows) {
              const float* ri = sRow + i * F + td.off;
              float        dm = 180.0f;
              for (int a = 0; a < td.Q; ++a) {
                const float x = ri[a];
#pragma unroll
                for (int b = 0; b < kSymRegs; ++b)
                  if (b < td.Q) dm = fminf(dm, circDiff(x, y[b]));
              }
              acc[k] += dm * td.wm;
            }
          }
        } else if (td.type == B200MOL_TFD_SYMMETRIC) {
#pragma unroll
          for (int k = 0; k < kMaxPairs; ++k) {
            const int i = i0 + k * S;
            if (k < P && i < nRows) {
              const float* ri = sRow + i * F + td.off;
              float        dm = 180.0f;
              for (int a = 0; a < td.Q; ++a) {
                const float x = ri[a];
                for (int b = 0; b < td.Q; ++b) dm = fminf(dm, circDiff(x, cj[td.off + b]));
              }
              acc[k] += dm * td.wm;
            }
          }
        } else {
          const float y    = cj[td.off];
          const bool  ring = td.type == B200MOL_TFD_RING;
#pragma unroll
          for (int k = 0; k < kMaxPairs; ++k) {
            const int i = i0 + k * S;
            if (k < P && i < nRows) {
              const float x = sRow[i * F + td.off];
              acc[k] += (ring ? fabsf(x - y) : circDiff(x, y)) * td.wm;
            }
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kMaxPairs; ++k) {
      const int i = i0 + k * S;
      if (k < P && i < nRows && colOk) {
        const int64_t gi = static_cast<int64_t>(ti) * R + i, gj = static_cast<int64_t>(tj) * R + j;
        if (gj < gi) out[md.outBase + gi * (gi - 1) / 2 + gj] = acc[k] * md.invSumW;
      }
    }
    __syncthreads();  // shared buffers and sUnit are reused by the next unit
  }
}

size_t unitSmem(int R, int F, int nTors) {
  return static_cast<size_t>(2) * R * F * 4 + static_cast<size_t>(nTors) * sizeof(TorDesc);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_tfd_matrices(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* d_conf_order,
                                    const int32_t* d_conf_atom_start, const double* d_xyz, const int32_t* h_tors_start,
                                    const int32_t* h_quartet_start, const int16_t* h_quartets, const uint8_t* h_type,
                                    const double* h_weight, const double* h_maxdev, float* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(nMols >= 0, "negative molecule count");
    if (nMols == 0) return;
    B200_REQUIRE(h_mol_conf_start && h_tors_start, "null pointer");
    B200_REQUIRE(h_mol_conf_start[0] >= 0 && h_tors_start[0] == 0, "conformer / torsion tables must start at 0");
    const int32_t nTorsAll = h_tors_start[nMols];
    B200_REQUIRE(nTorsAll >= 0, "torsion table: negative size");
    B200_REQUIRE(nTorsAll == 0 || (h_quartet_start && h_quartets && h_type && h_weight && h_maxdev), "null torsion table");
    B200_REQUIRE(nTorsAll == 0 || h_quartet_start[0] == 0, "quartet table must start at 0");
    const cudaStream_t s = asStream(stream);

    std::vector<MolDesc> mols(nMols);
    std::vector<TorDesc> tors(nTorsAll);
    std::vector<int64_t> workStart(nMols + 1, 0), unitStart(nMols + 1, 0);
    int64_t              featTotal = 0, outTotal = 0;
    size_t               smemMax   = 0;
    for (int m = 0; m < nMols; ++m) {
      const int c0 = h_mol_conf_start[m], c1 = h_mol_conf_start[m + 1], t0 = h_tors_start[m], t1 = h_tors_start[m + 1];
      B200_REQUIRE(c1 >= c0 && t1 >= t0, "molecule %d: conformer / torsion starts decrease", m);
      MolDesc& md = mols[m];
      md.confStart = c0;
      md.nConf     = c1 - c0;
      md.torStart  = t0;
      md.nTors     = t1 - t0;
      int    off = 0;
      double sumW = 0.0;
      for (int t = t0; t < t1; ++t) {
        const int Q    = h_quartet_start[t + 1] - h_quartet_start[t];
        const int type = h_type[t];
        B200_REQUIRE(type == B200MOL_TFD_SINGLE || type == B200MOL_TFD_SYMMETRIC || type == B200MOL_TFD_RING,
                     "torsion %d: unknown type %d", t, type);
        B200_REQUIRE(Q >= 1 && (type != B200MOL_TFD_SINGLE || Q == 1), "torsion %d: %d quartets for its type", t, Q);
        B200_REQUIRE(h_maxdev[t] > 0.0 && std::isfinite(h_maxdev[t]), "torsion %d: maxDev must be positive", t);
        B200_REQUIRE(h_weight[t] >= 0.0 && std::isfinite(h_weight[t]), "torsion %d: negative or non-finite weight", t);
        for (int k = 4 * h_quartet_start[t]; k < 4 * h_quartet_start[t + 1]; ++k)
          B200_REQUIRE(h_quartets[k] >= 0, "torsion %d: negative atom index", t);
        tors[t] = TorDesc{off, Q, type, static_cast<float>(h_weight[t] / h_maxdev[t])};
        off += type == B200MOL_TFD_SYMMETRIC ? Q : 1;
        sumW += h_weight[t];
      }
      md.F       = (off + 3) & ~3;
      md.invSumW = sumW > 1e-10 ? static_cast<float>(1.0 / sumW) : 0.0f;
      md.R       = kMaxR;
      while (md.R > 1 && unitSmem(md.R, md.F, md.nTors) > kSmemBudget) md.R >>= 1;
      B200_REQUIRE(unitSmem(md.R, md.F, md.nTors) <= kSmemBudget, "molecule %d: %d torsions / %d-float feature rows exceed "
                   "the shared-memory budget even one conformer per tile", m, md.nTors, md.F);
      md.T        = md.nConf >= 2 ? (md.nConf + md.R - 1) / md.R : 0;
      md.featBase = featTotal;
      md.outBase  = outTotal;
      featTotal += static_cast<int64_t>(md.nConf) * md.F;
      outTotal += static_cast<int64_t>(md.nConf) * (md.nConf - 1) / 2;
      workStart[m + 1] = workStart[m] + static_cast<int64_t>(md.nConf) * md.nTors;
      unitStart[m + 1] = unitStart[m] + lowerTriangleUnits(md.T);
      if (md.T > 0) smemMax = std::max(smemMax, unitSmem(md.R, md.F, md.nTors));
    }
    if (outTotal == 0) return;
    B200_REQUIRE(d_conf_atom_start && d_xyz && d_out, "null pointer");

    // one upload: descriptors, prefix sums, quartet starts and quartets of the whole call
    const int64_t nQ     = nTorsAll ? h_quartet_start[nTorsAll] : 0;
    auto          align  = [](size_t b) { return (b + 15) & ~static_cast<size_t>(15); };
    const size_t  oMols  = 0, oTors = align(oMols + sizeof(MolDesc) * nMols), oWork = align(oTors + sizeof(TorDesc) * nTorsAll),
                 oUnit = align(oWork + 8 * (nMols + 1)), oQS = align(oUnit + 8 * (nMols + 1)), oQ = align(oQS + 4 * (nTorsAll + 1)),
                 oQueue = align(oQ + 8 * nQ), nBytes = align(oQueue + 8);
    std::vector<unsigned char> host(nBytes, 0);
    std::copy_n(reinterpret_cast<const unsigned char*>(mols.data()), sizeof(MolDesc) * nMols, host.data() + oMols);
    if (nTorsAll) {
      std::copy_n(reinterpret_cast<const unsigned char*>(tors.data()), sizeof(TorDesc) * nTorsAll, host.data() + oTors);
      std::copy_n(reinterpret_cast<const unsigned char*>(h_quartet_start), 4 * (nTorsAll + 1), host.data() + oQS);
      std::copy_n(reinterpret_cast<const unsigned char*>(h_quartets), 8 * nQ, host.data() + oQ);
    }
    std::copy_n(reinterpret_cast<const unsigned char*>(workStart.data()), 8 * (nMols + 1), host.data() + oWork);
    std::copy_n(reinterpret_cast<const unsigned char*>(unitStart.data()), 8 * (nMols + 1), host.data() + oUnit);
    Scratch<unsigned char> plan(nBytes, s);
    Scratch<float>         feat(static_cast<size_t>(featTotal), s);
    B200_CUDA(cudaMemcpyAsync(plan.get(), host.data(), nBytes, cudaMemcpyHostToDevice, s));
    auto at = [&](size_t o) { return plan.get() + o; };

    if (workStart[nMols] > 0) {
      const int64_t want   = (workStart[nMols] + kPT - 1) / kPT;
      const int     blocks = static_cast<int>(std::min<int64_t>(want, static_cast<int64_t>(smCount()) * 16));
      tfdFeatureKernel<<<blocks, kPT, 0, s>>>(nMols, reinterpret_cast<const int64_t*>(at(oWork)),
                                              reinterpret_cast<const MolDesc*>(at(oMols)), reinterpret_cast<const TorDesc*>(at(oTors)),
                                              reinterpret_cast<const int32_t*>(at(oQS)), reinterpret_cast<const int16_t*>(at(oQ)),
                                              d_conf_order, d_conf_atom_start, d_xyz, feat.get());
      B200_LAUNCHED();
    }
    static bool attrSet[kMaxDevices] = {};
    const int   dev                  = currentDeviceSlot();
    if (!attrSet[dev]) {
      B200_CUDA(cudaFuncSetAttribute(tfdPairKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBudget)));
      attrSet[dev] = true;
    }
    int perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, tfdPairKernel, kPT, smemMax));
    const int blocks = static_cast<int>(std::min<int64_t>(unitStart[nMols], static_cast<int64_t>(smCount()) * std::max(perSm, 1)));
    tfdPairKernel<<<blocks, kPT, smemMax, s>>>(nMols, reinterpret_cast<const int64_t*>(at(oUnit)),
                                               reinterpret_cast<const MolDesc*>(at(oMols)), reinterpret_cast<const TorDesc*>(at(oTors)),
                                               feat.get(), d_out, reinterpret_cast<unsigned long long*>(at(oQueue)));
    B200_LAUNCHED();
  });
}
