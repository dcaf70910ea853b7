// Conformer RMSD matrices: for every molecule, the RMSD of every conformer pair (I > J) over all atoms, after the best
// proper rigid superposition (RDKit AllChem.GetConformerRMSMatrix; the reference runs one 128-thread block per pair,
// src/conformer_rmsd.cu) or, prealigned, on the coordinates as given.
//
// For one molecule every pair's 3x3 covariance H_IJ = sum_k a_Ik b_Jk^T is a 3x3 block of one Gram product U U^T, where
// U has three rows (x, y, z) per conformer and one column per atom. Two passes:
//  * operand pass: one warp per conformer writes its three rows once, in fp64, centred on its own centroid (or, when
//    prealigned, shifted by the centroid of the molecule's first conformer: a common shift leaves every difference
//    unchanged), with G = sum |a - shift|^2. Centring before the product keeps near-identical conformers far from the
//    origin from cancelling in the product. Rows are zero-padded to a multiple of 16 atoms (the MMA depth) and
//    conformers to a multiple of R, and stored in the order the pair pass's MMA fragments read them: per (tile, chunk
//    of 16 atoms) one contiguous 12 KB block of 12 groups of 8 rows, each group as [k half][lane][2] with lane
//    4 g + t holding row g at atoms t, t + 4 | t + 8, t + 12. Shared-memory fragment loads are then 16-byte,
//    contiguous across the warp and free of bank conflicts, and a tile's chunk is one bulk copy.
//  * pair pass: persistent CTAs take (molecule, R x R tile of the lower triangle) units from an atomic queue over the
//    unit prefix sum (tiles.cuh, as the TFD pass). A unit streams its row and column operand blocks chunk by chunk
//    through two shared-memory stages (bulk copies on mbarriers; a diagonal tile copies one block), so the atom count
//    is unbounded, and accumulates the 3R x 3R product with fp64 tensor-core MMA (mma.m16n8k16.f64, DMMA in SASS).
//    The accumulators then go through shared memory so that one thread owns one pair's 3x3 block, and the epilogue
//    evaluates SSD = Ga + Gb - 2 (s1 + s2 + sign(det H) s3) or, prealigned, Ga + Gb - 2 tr H, and stores
//    sqrt(SSD / n). Output rows are contiguous in J, so stores coalesce.
//
// The singular values come from a Jacobi eigen-decomposition of H^T H and the column norms of H V (bestTrace), not from
// the trigonometric eigenvalues of H^T H that RMS pruning uses (prune.cu). Those square roots of eigenvalues carry an
// absolute error of ~sqrt(eps) s1 whenever H is rank-deficient or two singular values coincide: two-atom, collinear and
// three-atom conformers, symmetric tops. In an fp64 CPU model of both routes on identical or rigidly moved conformers
// the trigonometric form was off by up to 5e-4 A (collinear) and 5e-3 A (three atoms); the Jacobi route stayed below
// 5e-7 A, the sqrt(eps G) floor of any Ga + Gb - 2 trace form.
//
// R = 32: 3R = 96 is a multiple of 16, and the 96 x 96 fp64 accumulator is 36 doubles (72 registers) per thread at 256
// threads; the eight warps each own a 48 x 24 block (3 x 3 MMA tiles). With its fragments the product takes ~180
// registers: under the 128 that two CTAs per SM allow, ptxas spills the accumulators, so the pass runs one CTA per SM
// and uses the shared memory that frees: 2 stages x 24 KB plus a separate 78 KB accumulator exchange (96 rows, stride
// 104 doubles: conflict-free fragment stores and stride-3 epilogue reads), so the next unit's first chunks load while
// the epilogue runs. R = 48 would need 81 accumulator doubles per thread; R = 16 would double the operand traffic per
// pair, which at n = 100 atoms already exceeds the 8 B of output per pair twenty-fold at R = 32.
//
// Every sum runs in a fixed order (MMA k-steps in atom order, warp reductions by butterfly): two runs give bitwise-equal
// matrices, and a molecule's matrix does not depend on the other molecules of the call.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "tiles.cuh"
#include "tma.cuh"

namespace b200 {
namespace {

constexpr int    kPT     = 256;                  // threads of both kernels
constexpr int    kR      = 32;                   // tile side in conformers
constexpr int    kRows   = 3 * kR;               // operand rows per tile
constexpr int    kKC     = 16;                   // atoms per chunk = MMA depth
constexpr int    kGroups = kRows / 8;            // row groups of 8 per tile
constexpr int    kGroupD = 8 * kKC;              // doubles per (group, chunk)
constexpr int    kBlockD = kGroups * kGroupD;    // doubles per (tile, chunk): 12 KB
constexpr int    kAS     = kRows + 8;            // accumulator row stride in shared memory
constexpr size_t kStageBytes = 2 * kBlockD * sizeof(double);
constexpr size_t kSmem = 2 * kStageBytes + static_cast<size_t>(kRows) * kAS * sizeof(double);  // 126 KB

struct MolDesc {
  int64_t opBase;     // first operand double of the molecule
  int64_t gBase;      // first G entry (= first conformer slot, conformers padded to tiles)
  int64_t outBase;    // offset of its lower triangle in the output
  int32_t confStart;  // first entry of the molecule in the conformer order
  int32_t nConf;
  int32_t nAtoms;
  int32_t nK;         // atom chunks
};

// s1 + s2 + sign(det H) s3 for the singular values s1 >= s2 >= s3 of H (row-major): the largest trace of R H over proper
// rotations R. Cyclic Jacobi on H^T H gives orthonormal right singular vectors V; the singular values are then the column
// norms of H V, never square roots of eigenvalues of H^T H, so each is accurate to ~eps |H| even when H is rank-deficient.
__device__ __forceinline__ double bestTrace(const double* H) {
  double M[3][3], V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) M[r][c] = H[r] * H[c] + H[3 + r] * H[3 + c] + H[6 + r] * H[6 + c];
  for (int sweep = 0; sweep < 10; ++sweep) {
    const double off = M[0][1] * M[0][1] + M[0][2] * M[0][2] + M[1][2] * M[1][2];
    if (off <= 1e-32 * (M[0][0] * M[0][0] + M[1][1] * M[1][1] + M[2][2] * M[2][2])) break;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int p = k == 2 ? 1 : 0, q = k == 0 ? 1 : 2, o = 3 - p - q;
      if (M[p][q] == 0.0) continue;
      const double tau = (M[q][q] - M[p][p]) / (2.0 * M[p][q]);
      const double t   = copysign(1.0, tau) / (fabs(tau) + sqrt(1.0 + tau * tau));
      const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
      const double mop = M[o][p], moq = M[o][q];
      M[p][p] -= t * M[p][q];
      M[q][q] += t * M[p][q];
      M[p][q] = M[q][p] = 0.0;
      M[o][p] = M[p][o] = c * mop - s * moq;
      M[o][q] = M[q][o] = s * mop + c * moq;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double vp = V[r][p], vq = V[r][q];
        V[r][p] = c * vp - s * vq;
        V[r][q] = s * vp + c * vq;
      }
    }
  }
  double sig[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double n2 = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const double b = H[3 * r] * V[0][c] + H[3 * r + 1] * V[1][c] + H[3 * r + 2] * V[2][c];
      n2 += b * b;
    }
    sig[c] = sqrt(n2);
  }
  const double det = H[0] * (H[4] * H[8] - H[5] * H[7]) - H[1] * (H[3] * H[8] - H[5] * H[6]) + H[2] * (H[3] * H[7] - H[4] * H[6]);
  const double sum = sig[0] + sig[1] + sig[2];
  return det < 0.0 ? sum - 2.0 * fmin(sig[0], fmin(sig[1], sig[2])) : sum;
}

__device__ __forceinline__ double warpSum(double v) {  // butterfly: every lane ends with the same bits
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void centroid(const double* a, int n, int lane, double* c) {
  double s[3] = {0.0, 0.0, 0.0};
  for (int k = lane; k < n; k += 32)
#pragma unroll
    for (int r = 0; r < 3; ++r) s[r] += a[3 * k + r];
#pragma unroll
  for (int r = 0; r < 3; ++r) c[r] = warpSum(s[r]) / n;
}

// one warp per conformer slot; slotStart[nMols+1] = prefix of T * R slots per molecule
__global__ void __launch_bounds__(kPT) rmsdOperandKernel(int nMols, const int64_t* slotStart, const MolDesc* mols,
                                                         const int32_t* confOrder, const int32_t* confAtomStart,
                                                         const double* xyz, int prealigned, double* ops, double* G) {
  const int     lane  = threadIdx.x & 31;
  const int64_t total = slotStart[nMols];
  const int64_t step  = static_cast<int64_t>(gridDim.x) * (kPT / 32);
  for (int64_t w = static_cast<int64_t>(blockIdx.x) * (kPT / 32) + (threadIdx.x >> 5); w < total; w += step) {
    const int     m    = upperIndex(slotStart, nMols + 1, w);
    const MolDesc md   = mols[m];
    const int     slot = static_cast<int>(w - slotStart[m]);
    const int     n    = md.nAtoms;
    const bool    real = slot < md.nConf;
    auto          pos  = [&](int k) {
      const int e = md.confStart + k;
      return xyz + 3 * static_cast<int64_t>(confAtomStart[confOrder ? confOrder[e] : e]);
    };
    const double* a     = real ? pos(slot) : nullptr;
    double        sh[3] = {0.0, 0.0, 0.0};
    if (real) centroid(prealigned ? pos(0) : a, n, lane, sh);
    double*   base = ops + md.opBase + static_cast<int64_t>(slot / kR) * md.nK * kBlockD;
    const int lr0  = 3 * (slot % kR);
    double    g    = 0.0;
    for (int k = lane; k < md.nK * kKC; k += 32) {
      double v[3] = {0.0, 0.0, 0.0};
      if (real && k < n) {
#pragma unroll
        for (int r = 0; r < 3; ++r) v[r] = a[3 * k + r] - sh[r];
        g += v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
      }
      const int kc = k / kKC, kk = k % kKC, t = kk & 3, i = kk >> 2;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int lr = lr0 + r;
        base[(kc * kGroups + (lr >> 3)) * kGroupD + (i >> 1) * 64 + ((lr & 7) * 4 + t) * 2 + (i & 1)] = v[r];
      }
    }
    g = warpSum(g);
    if (lane == 0) G[md.gBase + slot] = g;
  }
}

// D += A B: A 16 x 16 row-major (a_i at row g + 8 (i % 2), atom t + 4 (i / 2)), B 16 x 8 column-major (b_i at atom
// t + 4 i, column g), D 16 x 8 (d_0,1 at row g, columns 2t, 2t+1; d_2,3 at row g + 8); g = lane / 4, t = lane % 4
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

struct Unit {
  MolDesc       md;
  int           ti, tj;
  const double* rowSrc;  // the row tile's first operand block
  const double* colSrc;
};

__device__ __forceinline__ Unit decodeUnit(int nMols, const int64_t* unitStart, const MolDesc* mols, const double* ops,
                                           int64_t u) {
  Unit      x;
  const int m = upperIndex(unitStart, nMols + 1, u);
  x.md        = mols[m];
  lowerTriangleTile(u - unitStart[m], x.ti, x.tj);
  x.rowSrc = ops + x.md.opBase + static_cast<int64_t>(x.ti) * x.md.nK * kBlockD;
  x.colSrc = ops + x.md.opBase + static_cast<int64_t>(x.tj) * x.md.nK * kBlockD;
  return x;
}

// thread 0: atom chunk kc of unit x into stage kc % 2 (a diagonal tile copies one block)
__device__ __forceinline__ void issueChunk(const Unit& x, int kc, double* sOp, uint64_t* full) {
  const int      s     = kc & 1;
  const uint32_t block = kBlockD * sizeof(double);
  const bool     diag  = x.ti == x.tj;
  fenceProxyAsync();  // earlier generic reads of the stage come before these async writes
  mbarExpectTx(&full[s], diag ? block : 2 * block);
  bulkLoad1D(sOp + s * 2 * kBlockD, x.rowSrc + static_cast<int64_t>(kc) * kBlockD, block, &full[s]);
  if (!diag) bulkLoad1D(sOp + s * 2 * kBlockD + kBlockD, x.colSrc + static_cast<int64_t>(kc) * kBlockD, block, &full[s]);
}

// unitStart[nMols+1]: prefix of T(T+1)/2 lower-triangle tiles per molecule; *queue starts at 0. One CTA per SM: the
// product needs ~180 registers per thread without spilling. The next unit's first chunks load during the epilogue.
__global__ void __launch_bounds__(kPT, 1) rmsdPairKernel(int nMols, const int64_t* unitStart, const MolDesc* mols,
                                                         const double* ops, const double* G, int prealigned, double* out,
                                                         unsigned long long* queue) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t  full[2];
  __shared__ long long sUnit;
  double*              sOp  = reinterpret_cast<double*>(smem);  // stage s: row block, then column block
  double*              sAcc = sOp + 4 * kBlockD;                // [kRows][kAS] product
  const int            tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  const int64_t        total = unitStart[nMols];
  uint32_t             phase = 0;  // bit s: parity of stage s
  if (tid == 0) {
    mbarInit(&full[0], 1);
    mbarInit(&full[1], 1);
    fenceBarrierInit();
    sUnit = static_cast<long long>(atomicAdd(queue, 1ull));
  }
  __syncthreads();
  int64_t u = sUnit;
  if (u < total && tid == 0) {
    const Unit x = decodeUnit(nMols, unitStart, mols, ops, u);
    issueChunk(x, 0, sOp, full);
    if (x.md.nK > 1) issueChunk(x, 1, sOp, full);
  }
  while (u < total) {
    const Unit     x  = decodeUnit(nMols, unitStart, mols, ops, u);
    const MolDesc& md = x.md;
    const bool     diag = x.ti == x.tj;
    double         acc[3][3][4];
#pragma unroll
    for (int mt = 0; mt < 3; ++mt)
#pragma unroll
      for (int nt = 0; nt < 3; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.0;
    for (int kc = 0; kc < md.nK; ++kc) {
      const int s = kc & 1;
      mbarWait(&full[s], (phase >> s) & 1u);
      phase ^= 1u << s;
      const double* sa = sOp + s * 2 * kBlockD;
      const double* sb = diag ? sa : sa + kBlockD;
      double        b[3][4];
#pragma unroll
      for (int nt = 0; nt < 3; ++nt) {
        const double* p  = sb + (3 * wn + nt) * kGroupD + 2 * lane;
        const double2 lo = *reinterpret_cast<const double2*>(p), hi = *reinterpret_cast<const double2*>(p + 64);
        b[nt][0] = lo.x, b[nt][1] = lo.y, b[nt][2] = hi.x, b[nt][3] = hi.y;
      }
#pragma unroll
      for (int mt = 0; mt < 3; ++mt) {
        const double* p0 = sa + (6 * wm + 2 * mt) * kGroupD + 2 * lane;
        const double* p1 = p0 + kGroupD;
        const double2 x0 = *reinterpret_cast<const double2*>(p0), x1 = *reinterpret_cast<const double2*>(p0 + 64);
        const double2 y0 = *reinterpret_cast<const double2*>(p1), y1 = *reinterpret_cast<const double2*>(p1 + 64);
        const double  a[8] = {x0.x, y0.x, x0.y, y0.y, x1.x, y1.x, x1.y, y1.y};
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) dmma16816(acc[mt][nt], a, b[nt]);
      }
      __syncthreads();  // the stage is read by every warp before it is refilled
      if (tid == 0 && kc + 2 < md.nK) issueChunk(x, kc + 2, sOp, full);
    }
    // accumulators -> shared memory; meanwhile thread 0 takes the next unit
#pragma unroll
    for (int mt = 0; mt < 3; ++mt)
#pragma unroll
      for (int nt = 0; nt < 3; ++nt) {
        const int r = 48 * wm + 16 * mt + (lane >> 2), c = 24 * wn + 8 * nt + 2 * (lane & 3);
        *reinterpret_cast<double2*>(sAcc + r * kAS + c)       = make_double2(acc[mt][nt][0], acc[mt][nt][1]);
        *reinterpret_cast<double2*>(sAcc + (r + 8) * kAS + c) = make_double2(acc[mt][nt][2], acc[mt][nt][3]);
      }
    if (tid == 0) sUnit = static_cast<long long>(atomicAdd(queue, 1ull));
    __syncthreads();
    const int64_t next = sUnit;
    if (next < total && tid == 0) {  // the stages are free: every chunk of this unit was waited for and read
      const Unit y = decodeUnit(nMols, unitStart, mols, ops, next);
      issueChunk(y, 0, sOp, full);
      if (y.md.nK > 1) issueChunk(y, 1, sOp, full);
    }
    // one thread per pair: row i = warp + 8 k, column j = lane
    const int     nRows = min(kR, md.nConf - x.ti * kR), nCols = min(kR, md.nConf - x.tj * kR);
    const int64_t gj    = static_cast<int64_t>(x.tj) * kR + lane;
    const double  invN  = 1.0 / md.nAtoms;
#pragma unroll 1
    for (int i = warp; i < nRows; i += kPT / 32) {
      const int64_t gi = static_cast<int64_t>(x.ti) * kR + i;
      if (lane < nCols && gj < gi) {
        double H[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int c = 0; c < 3; ++c) H[3 * r + c] = sAcc[(3 * i + r) * kAS + 3 * lane + c];
        const double Ga  = G[md.gBase + gi], Gb = G[md.gBase + gj];
        const double ssd = Ga + Gb - 2.0 * (prealigned ? H[0] + H[4] + H[8] : bestTrace(H));
        out[md.outBase + gi * (gi - 1) / 2 + gj] = sqrt(fmax(ssd, 0.0) * invN);
      }
    }
    __syncthreads();  // sAcc and sUnit are reused by the next unit
    u = next;
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_conformer_rmsd(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms,
                                      const int32_t* d_conf_order, const int32_t* d_conf_atom_start, const double* d_xyz,
                                      int32_t prealigned, double* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(nMols >= 0, "negative molecule count");
    if (nMols == 0) return;
    B200_REQUIRE(h_mol_conf_start && h_mol_atoms, "null pointer");
    B200_REQUIRE(h_mol_conf_start[0] >= 0, "conformer table must not start below 0");
    const cudaStream_t s = asStream(stream);

    std::vector<MolDesc> mols(nMols);
    std::vector<int64_t> slotStart(nMols + 1, 0), unitStart(nMols + 1, 0);
    int64_t              opTotal = 0, outTotal = 0;
    for (int m = 0; m < nMols; ++m) {
      const int c0 = h_mol_conf_start[m], c1 = h_mol_conf_start[m + 1];
      B200_REQUIRE(c1 >= c0, "molecule %d: conformer starts decrease", m);
      B200_REQUIRE(h_mol_atoms[m] >= 0, "molecule %d: negative atom count", m);
      MolDesc& md = mols[m];
      md.confStart = c0;
      md.nConf     = c1 - c0;
      md.nAtoms    = h_mol_atoms[m];
      B200_REQUIRE(md.nConf < 2 || md.nAtoms > 0, "molecule %d has conformers but no atoms", m);
      md.nK             = (md.nAtoms + kKC - 1) / kKC;
      const int64_t T   = md.nConf >= 2 ? (md.nConf + kR - 1) / kR : 0;
      md.opBase         = opTotal;
      md.gBase          = slotStart[m];
      md.outBase        = outTotal;
      opTotal          += T * md.nK * kBlockD;
      outTotal         += static_cast<int64_t>(md.nConf) * (md.nConf - 1) / 2;
      slotStart[m + 1]  = slotStart[m] + T * kR;
      unitStart[m + 1]  = unitStart[m] + lowerTriangleUnits(T);
    }
    if (outTotal == 0) return;
    B200_REQUIRE(d_conf_atom_start && d_xyz && d_out, "null pointer");

    // one upload: descriptors, prefix sums and the queue counter
    auto         align  = [](size_t b) { return (b + 15) & ~static_cast<size_t>(15); };
    const size_t oMols  = 0, oSlot = align(sizeof(MolDesc) * nMols), oUnit = align(oSlot + 8 * (nMols + 1)),
                 oQueue = align(oUnit + 8 * (nMols + 1)), nBytes = align(oQueue + 8);
    std::vector<unsigned char> host(nBytes, 0);
    std::copy_n(reinterpret_cast<const unsigned char*>(mols.data()), sizeof(MolDesc) * nMols, host.data() + oMols);
    std::copy_n(reinterpret_cast<const unsigned char*>(slotStart.data()), 8 * (nMols + 1), host.data() + oSlot);
    std::copy_n(reinterpret_cast<const unsigned char*>(unitStart.data()), 8 * (nMols + 1), host.data() + oUnit);
    Scratch<unsigned char> plan(nBytes, s);
    Scratch<double>        ops(static_cast<size_t>(opTotal), s);
    Scratch<double>        G(static_cast<size_t>(slotStart[nMols]), s);
    B200_CUDA(cudaMemcpyAsync(plan.get(), host.data(), nBytes, cudaMemcpyHostToDevice, s));
    auto at = [&](size_t o) { return plan.get() + o; };

    const int64_t wantOp = (slotStart[nMols] + kPT / 32 - 1) / (kPT / 32);
    const int     opBlocks = static_cast<int>(std::min<int64_t>(wantOp, static_cast<int64_t>(smCount()) * 16));
    rmsdOperandKernel<<<opBlocks, kPT, 0, s>>>(nMols, reinterpret_cast<const int64_t*>(at(oSlot)),
                                               reinterpret_cast<const MolDesc*>(at(oMols)), d_conf_order, d_conf_atom_start,
                                               d_xyz, prealigned ? 1 : 0, ops.get(), G.get());
    B200_LAUNCHED();
    static bool attrSet[kMaxDevices] = {};
    const int   dev                  = currentDeviceSlot();
    if (!attrSet[dev]) {
      B200_CUDA(cudaFuncSetAttribute(rmsdPairKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem)));
      attrSet[dev] = true;
    }
    int perSm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, rmsdPairKernel, kPT, kSmem));
    const int blocks = static_cast<int>(std::min<int64_t>(unitStart[nMols], static_cast<int64_t>(smCount()) * std::max(perSm, 1)));
    rmsdPairKernel<<<blocks, kPT, kSmem, s>>>(nMols, reinterpret_cast<const int64_t*>(at(oUnit)),
                                              reinterpret_cast<const MolDesc*>(at(oMols)), ops.get(), G.get(),
                                              prealigned ? 1 : 0, d_out, reinterpret_cast<unsigned long long*>(at(oQueue)));
    B200_LAUNCHED();
  });
}
