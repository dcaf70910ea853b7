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
// Mapped matrices (b200mol_conformer_rmsd_mapped, RDKit GetAllConformerBestRMS): per molecule a probe list P and K
// reference lists Q_1..Q_K of L atoms; pair (I, J) is min_m RMSD(x_I[P], x_J[Q_m]). The same two passes run with:
//  * operand pass: the row operand of a conformer is gathered from P and centred on P's atoms; the column operands of
//    the mappings of the current chunk are gathered from Q_m and centred on their own atoms, in the same fragment-
//    ordered blocks (prealigned: every list shifted by the centroid of conformer 0's P atoms). A plain call is the
//    identity without a table: its column operand is its row operand, as before, so its bits do not change, and an
//    explicit identity table (K = 1, P = Q_1 = all atoms) computes the same operands and products bit for bit.
//  * pair pass: a unit is (molecule, group of the chunk's mappings, tile). It runs one product per mapping of its group
//    on the same pipeline (the chunk sequence is mapping-major, so the next mapping's first chunks load while the
//    previous epilogue runs), keeps the running minimum per pair in shared memory (8 KB; each thread owns its pairs,
//    so it needs no barrier) and stores once. A diagonal tile loads a column block per mapping; its one-block shortcut
//    is for the identity only. Where more than one unit covers a pair (several groups, or K larger than the chunk),
//    the output is first filled with 0x7F bytes (1.4e306) and every unit stores by a 64-bit unsigned atomicMin on the
//    bit pattern, which orders non-negative doubles as their values: exact, whatever order the units run in.
//  * chunks: the column operands of at most "rmsd_match_chunk" mappings per molecule are resident at once (0: as many
//    as fit a 1 GiB operand budget); chunks run in order on the stream and reuse one buffer.
//  * groups: mappings per unit are sized so that a chunk has about 8 units per SM when the work allows (one molecule
//    with a few tiles and K = 1,296 otherwise leaves most SMs idle), and never fewer mappings than one per unit.
// No bound-based skip of a mapping's epilogue is attempted: nothing here proves such a skip exact.
//
// Every sum runs in a fixed order (MMA k-steps in atom order, warp reductions by butterfly) and a minimum is exact:
// two runs give bitwise-equal matrices, and a molecule's matrix does not depend on the other molecules of the call.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "options.cuh"
#include "tiles.cuh"
#include "tma.cuh"

namespace b200 {

long long g_rmsdMatchChunk      = 0;  // option "rmsd_match_chunk": mappings per molecule per chunk, 0 = planned
long long g_rmsdMatchChunksLast = 0;  // chunks the last mapped call ran ("rmsd_match_chunks_last")

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
constexpr size_t kSmemMapped = kSmem + kR * kR * sizeof(double);                                   // + the running minimum

constexpr size_t kMatchBudget = size_t(1) << 30;  // column operand bytes of one planned chunk

// One molecule in one chunk of mappings (a plain call is one chunk of the identity).
struct MolDesc {
  int64_t opBase;     // first row operand double of the molecule
  int64_t gBase;      // first row G entry (= first conformer slot, conformers padded to tiles)
  int64_t colOpBase;  // column operands of the chunk's mappings, one T * nK * kBlockD block each (identity: opBase)
  int64_t colGBase;   // their G entries, T * kR each (identity: gBase)
  int64_t outBase;    // offset of its lower triangle in the output
  int64_t mapBase;    // first index of its lists P, Q_1, ..., Q_K in the atom table (no table: unused)
  int32_t confStart;  // first entry of the molecule in the conformer order
  int32_t nConf;
  int32_t nAtoms;     // L: atoms per list (no table: all atoms)
  int32_t nK;         // atom chunks
  int32_t T;          // tiles per side
  int32_t list0;      // list of the chunk's first mapping (Q_m is list m)
  int32_t nMaps;      // mappings in this chunk (0: none left)
  int32_t group;      // mappings per unit
  int32_t combine;    // 1: other units cover the same pairs, store by atomic minimum
  int32_t pad;
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

// atom k of a list: idx[k], or k without a table
__device__ __forceinline__ int listAtom(const int16_t* idx, int k) { return idx ? idx[k] : k; }

__device__ __forceinline__ void centroid(const double* a, const int16_t* idx, int n, int lane, double* c) {
  double s[3] = {0.0, 0.0, 0.0};
  for (int k = lane; k < n; k += 32) {
    const int at = listAtom(idx, k);
#pragma unroll
    for (int r = 0; r < 3; ++r) s[r] += a[3 * at + r];
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) c[r] = warpSum(s[r]) / n;
}

// One warp per (list, conformer slot); slotStart[nMols+1] = prefix of lists x T * R slots per molecule. !kCol: the
// row operand from list 0 (P) into opBase / gBase; kCol: the chunk's mappings, lists list0 .. list0 + nMaps - 1, into
// colOpBase / colGBase. mapAtoms == nullptr: the identity (all atoms, row pass only).
template <bool kCol>
__global__ void __launch_bounds__(kPT) rmsdOperandKernel(int nMols, const int64_t* slotStart, const MolDesc* mols,
                                                         const int32_t* confOrder, const int32_t* confAtomStart,
                                                         const double* xyz, const int16_t* mapAtoms, int prealigned,
                                                         double* ops, double* G) {
  constexpr bool col = kCol;
  const int     lane  = threadIdx.x & 31;
  const int64_t total = slotStart[nMols];
  const int64_t step  = static_cast<int64_t>(gridDim.x) * (kPT / 32);
  for (int64_t w = static_cast<int64_t>(blockIdx.x) * (kPT / 32) + (threadIdx.x >> 5); w < total; w += step) {
    const int      m     = upperIndex(slotStart, nMols + 1, w);
    const MolDesc  md    = mols[m];
    const int64_t  local = w - slotStart[m], slots = static_cast<int64_t>(md.T) * kR;  // a chunk may pass 2^31
    const int      list  = kCol ? static_cast<int>(local / slots) : 0;
    const int      slot  = static_cast<int>(kCol ? local % slots : local);
    const int      n     = md.nAtoms;
    const bool     real  = slot < md.nConf;
    const int16_t* probe = mapAtoms ? mapAtoms + md.mapBase : nullptr;
    const int16_t* idx   = col ? mapAtoms + md.mapBase + static_cast<int64_t>(md.list0 + list) * n : probe;
    auto           pos   = [&](int k) {
      const int e = md.confStart + k;
      return xyz + 3 * static_cast<int64_t>(confAtomStart[confOrder ? confOrder[e] : e]);
    };
    const double* a     = real ? pos(slot) : nullptr;
    double        sh[3] = {0.0, 0.0, 0.0};
    if (real) {
      if (prealigned) centroid(pos(0), probe, n, lane, sh);
      else centroid(a, idx, n, lane, sh);
    }
    const int64_t listOps = static_cast<int64_t>(md.T) * md.nK * kBlockD;
    double*       base = ops + (col ? md.colOpBase + list * listOps : md.opBase) + static_cast<int64_t>(slot / kR) * md.nK * kBlockD;
    const int     lr0  = 3 * (slot % kR);
    double        g    = 0.0;
    for (int k = lane; k < md.nK * kKC; k += 32) {
      double v[3] = {0.0, 0.0, 0.0};
      if (real && k < n) {
        const int at = listAtom(idx, k);
#pragma unroll
        for (int r = 0; r < 3; ++r) v[r] = a[3 * at + r] - sh[r];
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
    if (lane == 0) G[(col ? md.colGBase + static_cast<int64_t>(list) * md.T * kR : md.gBase) + slot] = g;
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
  int           map0, nMap;  // the unit's mappings: chunk-local map0 .. map0 + nMap - 1
  const double* rowSrc;      // the row tile's first operand block
  const double* colSrc;      // the column tile's first operand block of mapping map0
};

__device__ __forceinline__ int64_t colListOps(const MolDesc& md) { return static_cast<int64_t>(md.T) * md.nK * kBlockD; }

// unitStart: prefix of nGroups x T(T+1)/2 units per molecule, group-major (the identity: one group)
template <bool kMapped>
__device__ __forceinline__ Unit decodeUnit(int nMols, const int64_t* unitStart, const MolDesc* mols, const double* ops,
                                           int64_t u) {
  Unit          x;
  const int     m     = upperIndex(unitStart, nMols + 1, u);
  x.md                = mols[m];
  const int64_t tiles = lowerTriangleUnits(x.md.T), loc = u - unitStart[m];
  const int     grp   = kMapped ? static_cast<int>(loc / tiles) : 0;
  lowerTriangleTile(loc - grp * tiles, x.ti, x.tj);
  x.map0   = grp * x.md.group;
  x.nMap   = kMapped ? min(x.md.group, x.md.nMaps - x.map0) : 1;
  x.rowSrc = ops + x.md.opBase + static_cast<int64_t>(x.ti) * x.md.nK * kBlockD;
  x.colSrc = ops + x.md.colOpBase + x.map0 * colListOps(x.md) + static_cast<int64_t>(x.tj) * x.md.nK * kBlockD;
  return x;
}

// thread 0: step s = (mapping, atom chunk) of unit x, mapping-major, into stage s % 2 (for the identity a diagonal tile
// copies one block)
template <bool kMapped>
__device__ __forceinline__ void issueChunk(const Unit& x, int step, double* sOp, uint64_t* full) {
  const int      s     = step & 1;
  const int      mp    = kMapped ? step / x.md.nK : 0, kc = step - mp * x.md.nK;
  const uint32_t block = kBlockD * sizeof(double);
  const bool     one   = !kMapped && x.ti == x.tj;
  fenceProxyAsync();  // earlier generic reads of the stage come before these async writes
  mbarExpectTx(&full[s], one ? block : 2 * block);
  bulkLoad1D(sOp + s * 2 * kBlockD, x.rowSrc + static_cast<int64_t>(kc) * kBlockD, block, &full[s]);
  if (!one)
    bulkLoad1D(sOp + s * 2 * kBlockD + kBlockD, x.colSrc + mp * colListOps(x.md) + static_cast<int64_t>(kc) * kBlockD,
               block, &full[s]);
}

template <bool kMapped>
__device__ __forceinline__ void issueFirst(const Unit& x, double* sOp, uint64_t* full) {
  issueChunk<kMapped>(x, 0, sOp, full);
  if (x.nMap * x.md.nK > 1) issueChunk<kMapped>(x, 1, sOp, full);
}

// unitStart[nMols+1]: prefix of units per molecule; *queue starts at 0. !kMapped: the column operand is the row operand
// (a plain call), compiled without the mapping loop, the running minimum and its 8 KB, as before the mapped calls. One
// CTA per SM: the product needs ~180 registers per thread without spilling. The next mapping's and the next unit's
// first chunks load during the epilogue.
template <bool kMapped>
__global__ void __launch_bounds__(kPT, 1) rmsdPairKernel(int nMols, const int64_t* unitStart, const MolDesc* mols,
                                                         const double* ops, const double* G, int prealigned, double* out,
                                                         unsigned long long* queue) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t  full[2];
  __shared__ long long sUnit;
  double*              sOp  = reinterpret_cast<double*>(smem);  // stage s: row block, then column block
  double*              sAcc = sOp + 4 * kBlockD;                // [kRows][kAS] product
  double*              sMin = sAcc + kRows * kAS;               // [kR][kR] running minimum over a unit's mappings
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
  if (u < total && tid == 0) issueFirst<kMapped>(decodeUnit<kMapped>(nMols, unitStart, mols, ops, u), sOp, full);
  while (u < total) {
    const Unit     x      = decodeUnit<kMapped>(nMols, unitStart, mols, ops, u);
    const MolDesc& md     = x.md;
    const bool     one    = !kMapped && x.ti == x.tj;
    const int      nSteps = x.nMap * md.nK;
    int64_t        next   = total;
#pragma unroll 1
    for (int mp = 0; mp < x.nMap; ++mp) {
      double acc[3][3][4];
#pragma unroll
      for (int mt = 0; mt < 3; ++mt)
#pragma unroll
        for (int nt = 0; nt < 3; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.0;
      for (int kc = 0; kc < md.nK; ++kc) {
        const int step = mp * md.nK + kc, s = step & 1;
        mbarWait(&full[s], (phase >> s) & 1u);
        phase ^= 1u << s;
        const double* sa = sOp + s * 2 * kBlockD;
        const double* sb = one ? sa : sa + kBlockD;
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
        if (tid == 0 && step + 2 < nSteps) issueChunk<kMapped>(x, step + 2, sOp, full);
      }
      // accumulators -> shared memory; after the last mapping thread 0 takes the next unit meanwhile
#pragma unroll
      for (int mt = 0; mt < 3; ++mt)
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
          const int r = 48 * wm + 16 * mt + (lane >> 2), c = 24 * wn + 8 * nt + 2 * (lane & 3);
          *reinterpret_cast<double2*>(sAcc + r * kAS + c)       = make_double2(acc[mt][nt][0], acc[mt][nt][1]);
          *reinterpret_cast<double2*>(sAcc + (r + 8) * kAS + c) = make_double2(acc[mt][nt][2], acc[mt][nt][3]);
        }
      const bool last = mp == x.nMap - 1;
      if (last && tid == 0) sUnit = static_cast<long long>(atomicAdd(queue, 1ull));
      __syncthreads();
      if (last) {
        next = sUnit;
        // the stages are free: every chunk of this unit was waited for and read
        if (next < total && tid == 0) issueFirst<kMapped>(decodeUnit<kMapped>(nMols, unitStart, mols, ops, next), sOp, full);
      }
      // one thread per pair: row i = warp + 8 k, column j = lane
      const int     nRows = min(kR, md.nConf - x.ti * kR), nCols = min(kR, md.nConf - x.tj * kR);
      const int64_t gj    = static_cast<int64_t>(x.tj) * kR + lane;
      const double  invN  = 1.0 / md.nAtoms;
      const double* Gb    = kMapped ? G + md.colGBase + static_cast<int64_t>(x.map0 + mp) * md.T * kR : G + md.gBase;
#pragma unroll 1
      for (int i = warp; i < nRows; i += kPT / 32) {
        const int64_t gi = static_cast<int64_t>(x.ti) * kR + i;
        if (lane < nCols && gj < gi) {
          double H[9];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) H[3 * r + c] = sAcc[(3 * i + r) * kAS + 3 * lane + c];
          const double Ga  = G[md.gBase + gi];
          const double ssd = Ga + Gb[gj] - 2.0 * (prealigned ? H[0] + H[4] + H[8] : bestTrace(H));
          double       v   = sqrt(fmax(ssd, 0.0) * invN);
          double*      o   = out + md.outBase + gi * (gi - 1) / 2 + gj;
          if (!kMapped) {
            *o = v;
            continue;
          }
          if (mp > 0) v = fmin(v, sMin[i * kR + lane]);
          if (!last) sMin[i * kR + lane] = v;
          else if (md.combine) atomicMin(reinterpret_cast<unsigned long long*>(o), __double_as_longlong(v));
          else *o = v;
        }
      }
      __syncthreads();  // sAcc and sUnit are reused by the next mapping or unit
    }
    u = next;
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

namespace {

// The mapping tables of b200mol_conformer_rmsd_mapped (host arrays); null for a plain call.
struct MapTables {
  const int64_t* start;
  const int32_t* count;
  const int32_t* len;
  const int16_t* atoms;
};

void conformerRmsd(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms, const int32_t* d_conf_order,
                   const int32_t* d_conf_atom_start, const double* d_xyz, const MapTables* maps, int32_t prealigned,
                   double* d_out, void* stream) {
  B200_REQUIRE(nMols >= 0, "negative molecule count");
  if (nMols == 0) return;
  B200_REQUIRE(h_mol_conf_start && h_mol_atoms, "null pointer");
  B200_REQUIRE(h_mol_conf_start[0] >= 0, "conformer table must not start below 0");
  if (maps) {
    B200_REQUIRE(maps->start && maps->count && maps->len && maps->atoms, "null mapping table");
    B200_REQUIRE(maps->start[0] >= 0, "mapping table must not start below 0");
  }
  const cudaStream_t s = asStream(stream);

  // the molecules and their row operands; column operand sizes per mapping
  std::vector<MolDesc> base(nMols);
  std::vector<int64_t> rowSlot(nMols + 1, 0);
  std::vector<int>     K(nMols, 1);
  std::vector<int32_t> stamp;
  int64_t              opTotal = 0, outTotal = 0, perMapBytes = 0;
  int                  maxK = 0;
  for (int m = 0; m < nMols; ++m) {
    const int c0 = h_mol_conf_start[m], c1 = h_mol_conf_start[m + 1];
    B200_REQUIRE(c1 >= c0, "molecule %d: conformer starts decrease", m);
    B200_REQUIRE(h_mol_atoms[m] >= 0, "molecule %d: negative atom count", m);
    MolDesc& md = base[m];
    md          = MolDesc{};
    md.confStart = c0;
    md.nConf     = c1 - c0;
    md.nAtoms    = h_mol_atoms[m];
    B200_REQUIRE(md.nConf < 2 || md.nAtoms > 0, "molecule %d has conformers but no atoms", m);
    if (maps) {
      const int n = h_mol_atoms[m], k = maps->count[m], L = maps->len[m];
      B200_REQUIRE(n < 32768, "molecule %d: %d atoms, mapping tables take fewer than 32768", m, n);
      B200_REQUIRE(k >= 1, "molecule %d: mapping count %d must be >= 1", m, k);
      // a molecule without atoms has nothing to select (and fewer than two conformers): its lists are empty
      if (n == 0) B200_REQUIRE(L == 0, "molecule %d has no atoms: its mapping length %d must be 0", m, L);
      else B200_REQUIRE(L >= 1 && L <= n, "molecule %d: mapping length %d must be in [1, %d]", m, L, n);
      const int64_t a0 = maps->start[m], a1 = maps->start[m + 1];
      B200_REQUIRE(a1 - a0 == static_cast<int64_t>(k + 1) * L,
                   "molecule %d: mapping table holds %lld atoms, (K + 1) L = %lld", m, static_cast<long long>(a1 - a0),
                   static_cast<long long>(k + 1) * L);
      stamp.assign(n, -1);
      for (int l = 0; l <= k; ++l)
        for (int i = 0; i < L; ++i) {
          const int at = maps->atoms[a0 + static_cast<int64_t>(l) * L + i];
          B200_REQUIRE(at >= 0 && at < n, "molecule %d: list %d holds atom %d, outside [0, %d)", m, l, at, n);
          B200_REQUIRE(stamp[at] != l, "molecule %d: list %d holds atom %d twice", m, l, at);
          stamp[at] = l;
        }
      md.nAtoms  = L;
      md.mapBase = a0;
      K[m]       = k;
    }
    md.nK            = (md.nAtoms + kKC - 1) / kKC;
    md.T             = md.nConf >= 2 ? (md.nConf + kR - 1) / kR : 0;
    md.opBase        = opTotal;
    md.gBase         = rowSlot[m];
    md.outBase       = outTotal;
    opTotal         += static_cast<int64_t>(md.T) * md.nK * kBlockD;
    outTotal        += static_cast<int64_t>(md.nConf) * (md.nConf - 1) / 2;
    rowSlot[m + 1]   = rowSlot[m] + static_cast<int64_t>(md.T) * kR;
    if (md.T) {
      maxK         = std::max(maxK, K[m]);
      perMapBytes += (static_cast<int64_t>(md.T) * md.nK * kBlockD + static_cast<int64_t>(md.T) * kR) * 8;
    }
  }
  if (maps) g_rmsdMatchChunksLast = 0;
  if (outTotal == 0) return;
  B200_REQUIRE(d_conf_atom_start && d_xyz && d_out, "null pointer");

  // chunks of mappings; per chunk every molecule's mappings in groups that fill the machine
  const int chunk = !maps ? 1
                    : g_rmsdMatchChunk > 0 ? static_cast<int>(std::min<long long>(g_rmsdMatchChunk, maxK))
                                           : static_cast<int>(std::clamp<int64_t>(static_cast<int64_t>(kMatchBudget) / perMapBytes, 1, maxK));
  const int nChunks = maps ? (maxK + chunk - 1) / chunk : 1;
  const int64_t targetUnits = static_cast<int64_t>(smCount()) * 8;
  std::vector<MolDesc> desc(static_cast<size_t>(nChunks) * nMols);
  std::vector<int64_t> colSlot(static_cast<size_t>(nChunks) * (nMols + 1), 0), unitStart(colSlot.size(), 0);
  int64_t              colOpTotal = opTotal, colGTotal = rowSlot[nMols];  // column buffers follow the row operands
  bool                 combine = false;
  for (int m = 0; m < nMols; ++m) {  // the column buffer holds min(chunk, K) mappings per molecule, reused by every chunk
    MolDesc& md  = base[m];
    const int64_t held = maps ? std::min(chunk, K[m]) : 0;
    md.colOpBase = maps ? colOpTotal : md.opBase;
    md.colGBase  = maps ? colGTotal : md.gBase;
    colOpTotal  += held * md.T * md.nK * kBlockD;
    colGTotal   += held * md.T * kR;
  }
  for (int c = 0; c < nChunks; ++c) {
    int64_t work = 0;
    for (int m = 0; m < nMols; ++m) {
      const MolDesc& md = base[m];
      work += md.T ? lowerTriangleUnits(md.T) * std::clamp(K[m] - c * chunk, 0, chunk) * md.nK : 0;
    }
    const int64_t unitWork = std::max<int64_t>(1, (work + targetUnits - 1) / targetUnits);
    MolDesc*      d        = desc.data() + static_cast<size_t>(c) * nMols;
    int64_t*      cs       = colSlot.data() + static_cast<size_t>(c) * (nMols + 1);
    int64_t*      us       = unitStart.data() + static_cast<size_t>(c) * (nMols + 1);
    for (int m = 0; m < nMols; ++m) {
      d[m]       = base[m];
      MolDesc& md = d[m];
      md.list0    = 1 + c * chunk;
      md.nMaps    = md.T ? std::clamp(K[m] - c * chunk, 0, chunk) : 0;
      md.group    = md.nMaps ? static_cast<int>(std::clamp<int64_t>(unitWork / md.nK, 1, md.nMaps)) : 1;  // nK >= 1 here
      const int nGroups = (md.nMaps + md.group - 1) / md.group;
      md.combine  = nGroups > 1 || K[m] > chunk;
      combine     = combine || (md.nMaps && md.combine);
      cs[m + 1]   = cs[m] + (maps ? static_cast<int64_t>(md.nMaps) * md.T * kR : 0);
      us[m + 1]   = us[m] + nGroups * lowerTriangleUnits(md.T);
    }
  }

  // one upload: descriptors, prefix sums, queue counters and the atom table
  const int64_t nMapAtoms = maps ? maps->start[nMols] : 0;
  auto          align     = [](size_t b) { return (b + 15) & ~static_cast<size_t>(15); };
  const size_t  oMols = 0, oRow = align(sizeof(MolDesc) * desc.size()), oCol = align(oRow + 8 * (nMols + 1)),
               oUnit = align(oCol + 8 * colSlot.size()), oQueue = align(oUnit + 8 * unitStart.size()),
               oAtoms = align(oQueue + 8 * static_cast<size_t>(nChunks)), nBytes = align(oAtoms + 2 * nMapAtoms);
  std::vector<unsigned char> host(nBytes, 0);
  auto put = [&](size_t o, const void* p, size_t b) { std::copy_n(static_cast<const unsigned char*>(p), b, host.data() + o); };
  put(oMols, desc.data(), sizeof(MolDesc) * desc.size());
  put(oRow, rowSlot.data(), 8 * rowSlot.size());
  put(oCol, colSlot.data(), 8 * colSlot.size());
  put(oUnit, unitStart.data(), 8 * unitStart.size());
  if (maps) put(oAtoms, maps->atoms, 2 * nMapAtoms);
  Scratch<unsigned char> plan(nBytes, s);
  Scratch<double>        ops(static_cast<size_t>(colOpTotal), s);
  Scratch<double>        G(static_cast<size_t>(colGTotal), s);
  B200_CUDA(cudaMemcpyAsync(plan.get(), host.data(), nBytes, cudaMemcpyHostToDevice, s));
  auto           at      = [&](size_t o) { return plan.get() + o; };
  const int16_t* d_atoms = maps ? reinterpret_cast<const int16_t*>(at(oAtoms)) : nullptr;
  if (combine) B200_CUDA(cudaMemsetAsync(d_out, 0x7F, sizeof(double) * outTotal, s));

  auto operands = [&](int64_t slots, const int64_t* slotStart, const MolDesc* d, bool col) {
    const int64_t want = (slots + kPT / 32 - 1) / (kPT / 32);
    const int     n    = static_cast<int>(std::min<int64_t>(want, static_cast<int64_t>(smCount()) * 16));
    (col ? rmsdOperandKernel<true> : rmsdOperandKernel<false>)<<<n, kPT, 0, s>>>(
        nMols, slotStart, d, d_conf_order, d_conf_atom_start, d_xyz, d_atoms, prealigned ? 1 : 0, ops.get(), G.get());
    B200_LAUNCHED();
  };
  operands(rowSlot[nMols], reinterpret_cast<const int64_t*>(at(oRow)), reinterpret_cast<const MolDesc*>(at(oMols)), false);
  static bool attrSet[kMaxDevices] = {};
  const int   dev                  = currentDeviceSlot();
  if (!attrSet[dev]) {
    B200_CUDA(cudaFuncSetAttribute(rmsdPairKernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmem)));
    B200_CUDA(cudaFuncSetAttribute(rmsdPairKernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(kSmemMapped)));
    attrSet[dev] = true;
  }
  const size_t smem  = maps ? kSmemMapped : kSmem;
  int          perSm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, maps ? rmsdPairKernel<true> : rmsdPairKernel<false>, kPT,
                                                          smem));
  for (int c = 0; c < nChunks; ++c) {
    const MolDesc* d  = reinterpret_cast<const MolDesc*>(at(oMols)) + static_cast<size_t>(c) * nMols;
    const int64_t* cs = reinterpret_cast<const int64_t*>(at(oCol)) + static_cast<size_t>(c) * (nMols + 1);
    const int64_t* us = reinterpret_cast<const int64_t*>(at(oUnit)) + static_cast<size_t>(c) * (nMols + 1);
    const int64_t  units = unitStart[static_cast<size_t>(c) * (nMols + 1) + nMols];
    if (maps) operands(colSlot[static_cast<size_t>(c) * (nMols + 1) + nMols], cs, d, true);
    if (units == 0) continue;
    const int blocks = static_cast<int>(std::min<int64_t>(units, static_cast<int64_t>(smCount()) * std::max(perSm, 1)));
    auto* queue = reinterpret_cast<unsigned long long*>(at(oQueue)) + c;
    if (maps) rmsdPairKernel<true><<<blocks, kPT, smem, s>>>(nMols, us, d, ops.get(), G.get(), prealigned ? 1 : 0, d_out, queue);
    else rmsdPairKernel<false><<<blocks, kPT, smem, s>>>(nMols, us, d, ops.get(), G.get(), prealigned ? 1 : 0, d_out, queue);
    B200_LAUNCHED();
  }
  if (maps) g_rmsdMatchChunksLast = nChunks;
}

}  // namespace

extern "C" int b200mol_conformer_rmsd(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms,
                                      const int32_t* d_conf_order, const int32_t* d_conf_atom_start, const double* d_xyz,
                                      int32_t prealigned, double* d_out, void* stream) {
  return guarded([&] {
    conformerRmsd(nMols, h_mol_conf_start, h_mol_atoms, d_conf_order, d_conf_atom_start, d_xyz, nullptr, prealigned, d_out,
                  stream);
  });
}

extern "C" int b200mol_conformer_rmsd_mapped(int32_t nMols, const int32_t* h_mol_conf_start, const int32_t* h_mol_atoms,
                                             const int32_t* d_conf_order, const int32_t* d_conf_atom_start,
                                             const double* d_xyz, const int64_t* h_map_start, const int32_t* h_map_count,
                                             const int32_t* h_map_len, const int16_t* h_map_atoms, int32_t prealigned,
                                             double* d_out, void* stream) {
  return guarded([&] {
    const MapTables maps{h_map_start, h_map_count, h_map_len, h_map_atoms};
    conformerRmsd(nMols, h_mol_conf_start, h_mol_atoms, d_conf_order, d_conf_atom_start, d_xyz, &maps, prealigned, d_out,
                  stream);
  });
}
