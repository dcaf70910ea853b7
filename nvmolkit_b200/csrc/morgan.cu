// Morgan (ECFP-style) fingerprints from flattened molecular graphs, one warp per molecule, sm_90a.
//
// Algorithm = RDKit's MorganEnvGenerator as restated by the reference (src/morgan_fingerprint_cpu.cpp:61-255,
// GPU twin src/morgan_fingerprint_kernels.cu:152-432), bit-exact:
//   round 0: every atom sets bit (invariant % fpBits);
//   round r: each live atom ORs its neighbours' bond-neighbourhood bitsets, hashes the sorted (bondType, invariant)
//   pairs of its neighbours into a new invariant, and contributes a bit only if its neighbourhood bitset has not been
//   emitted before (this round by an atom with a smaller (invariant, index), or in any earlier round); otherwise the
//   atom is dead from then on (dead atoms' invariants become 0, their neighbourhoods freeze).
//
// Design: the reference sorts all (bitset, invariant, atom) tuples of a round with a tile-wide CUB merge sort and
// scans earlier rounds linearly in global memory. Only the equivalence classes matter, so this kernel replaces the sort
// with a rank test — "is there an equal bitset with a smaller (invariant, atom) key, or an equal accepted bitset from
// an earlier round" — all in shared memory, and handles molecules of any size that fits shared memory (no CPU twin).
#include "common.cuh"

namespace b200 {
namespace {

constexpr int kMaxDeg = 16;

__device__ __forceinline__ void hashCombine(uint32_t& seed, uint32_t v) {
  seed ^= v + 0x9e3779b9u + (seed << 6) + (seed >> 2);
}

struct MorganLayout {  // byte offsets inside one molecule's shared-memory slab
  int inv, invNext, nbhd, nbhdRound, seen, adjStart, adjBond, adjOther, dead, cand, fp, total;
};

__host__ __device__ inline MorganLayout morganLayout(int maxAtoms, int maxBonds, int radius, int fpWords) {
  const int    bw = (maxBonds + 31) / 32 > 0 ? (maxBonds + 31) / 32 : 1;
  MorganLayout L;
  int          o = 0;
  auto         take = [&](int bytes) {
    const int at = o;
    o += (bytes + 15) & ~15;
    return at;
  };
  L.inv       = take(maxAtoms * 4);
  L.invNext   = take(maxAtoms * 4);
  L.nbhd      = take(maxAtoms * bw * 4);
  L.nbhdRound = take(maxAtoms * bw * 4);
  L.seen      = take((radius > 0 ? radius : 1) * maxAtoms * bw * 4);
  L.adjStart  = take((maxAtoms + 1) * 4);
  L.adjBond   = take(2 * maxBonds * 2);
  L.adjOther  = take(2 * maxBonds * 2);
  L.dead      = take(maxAtoms);
  L.cand      = take(maxAtoms);
  L.fp        = take(fpWords * 4);
  L.total     = o;
  return L;
}

__global__ void morganKernel(const int32_t* __restrict__ atomStarts, const int32_t* __restrict__ bondStarts,
                             const uint32_t* __restrict__ atomInv, const uint32_t* __restrict__ bondInv,
                             const uint16_t* __restrict__ bondA, const uint16_t* __restrict__ bondB, int nMols,
                             int maxAtoms, int maxBonds, int radius, int fpBits, uint32_t* __restrict__ out,
                             int* __restrict__ errFlag) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int          lane = threadIdx.x & 31;
  const int          wib  = threadIdx.x >> 5;
  const int          mol  = blockIdx.x * (blockDim.x >> 5) + wib;
  if (mol >= nMols) return;
  const int          fpWords = fpBits >> 5;
  const MorganLayout L       = morganLayout(maxAtoms, maxBonds, radius, fpWords);
  uint8_t*           slab    = smem + static_cast<size_t>(wib) * L.total;
  uint32_t*          inv       = reinterpret_cast<uint32_t*>(slab + L.inv);
  uint32_t*          invNext   = reinterpret_cast<uint32_t*>(slab + L.invNext);
  uint32_t*          nbhd      = reinterpret_cast<uint32_t*>(slab + L.nbhd);
  uint32_t*          nbhdRound = reinterpret_cast<uint32_t*>(slab + L.nbhdRound);
  uint32_t*          seen      = reinterpret_cast<uint32_t*>(slab + L.seen);
  int*               adjStart  = reinterpret_cast<int*>(slab + L.adjStart);
  uint16_t*          adjBond   = reinterpret_cast<uint16_t*>(slab + L.adjBond);
  uint16_t*          adjOther  = reinterpret_cast<uint16_t*>(slab + L.adjOther);
  uint8_t*           dead      = slab + L.dead;
  uint8_t*           cand      = slab + L.cand;
  uint32_t*          fp        = reinterpret_cast<uint32_t*>(slab + L.fp);

  const int a0 = atomStarts[mol], nA = atomStarts[mol + 1] - a0;
  const int b0 = bondStarts[mol], nB = bondStarts[mol + 1] - b0;
  uint32_t* outRow = out + static_cast<size_t>(mol) * fpWords;
  if (nA > maxAtoms || nB > maxBonds) {
    if (lane == 0) atomicExch(errFlag, 1);
    for (int w = lane; w < fpWords; w += 32) outRow[w] = 0;
    return;
  }
  const int bw = (maxBonds + 31) / 32 > 0 ? (maxBonds + 31) / 32 : 1;

  for (int w = lane; w < fpWords; w += 32) fp[w] = 0;
  for (int a = lane; a <= nA; a += 32) adjStart[a] = 0;
  for (int a = lane; a < nA; a += 32) {
    inv[a]  = atomInv[a0 + a];
    dead[a] = 0;
    for (int w = 0; w < bw; ++w) nbhd[a * bw + w] = 0;
  }
  __syncwarp();
  // adjacency as CSR in shared memory: degree count, warp scan, fill
  for (int b = lane; b < nB; b += 32) {
    atomicAdd(&adjStart[bondA[b0 + b] + 1], 1);
    atomicAdd(&adjStart[bondB[b0 + b] + 1], 1);
  }
  __syncwarp();
  {
    int carry = 0;
    for (int base = 0; base <= nA; base += 32) {
      const int a = base + lane;
      int       v = a <= nA ? adjStart[a] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
      }
      if (a <= nA) adjStart[a] = v + carry;
      carry += __shfl_sync(0xffffffffu, v, 31);
    }
  }
  __syncwarp();
  // fill using cand[] region as nothing else yet: per-atom cursors live in invNext temporarily
  for (int a = lane; a < nA; a += 32) invNext[a] = 0;
  __syncwarp();
  for (int b = lane; b < nB; b += 32) {
    const int u = bondA[b0 + b], v = bondB[b0 + b];
    int       s = adjStart[u] + static_cast<int>(atomicAdd(&invNext[u], 1u));
    adjBond[s]  = static_cast<uint16_t>(b);
    adjOther[s] = static_cast<uint16_t>(v);
    s           = adjStart[v] + static_cast<int>(atomicAdd(&invNext[v], 1u));
    adjBond[s]  = static_cast<uint16_t>(b);
    adjOther[s] = static_cast<uint16_t>(u);
  }
  // round 0
  for (int a = lane; a < nA; a += 32) atomicOr(&fp[(inv[a] % fpBits) >> 5], 1u << ((inv[a] % fpBits) & 31));
  __syncwarp();

  int nSeen = 0;
  for (int layer = 0; layer < radius; ++layer) {
    for (int a = lane; a < nA; a += 32) {
      const int beg = adjStart[a], deg = adjStart[a + 1] - beg;
      cand[a] = 0;
      if (dead[a] || deg == 0) {
        dead[a]    = 1;
        invNext[a] = 0;
        for (int w = 0; w < bw; ++w) nbhdRound[a * bw + w] = nbhd[a * bw + w];
        continue;
      }
      if (deg > kMaxDeg) {
        atomicExch(errFlag, 2);
        dead[a]    = 1;
        invNext[a] = 0;
        for (int w = 0; w < bw; ++w) nbhdRound[a * bw + w] = nbhd[a * bw + w];
        continue;
      }
      int32_t  pf[kMaxDeg];
      uint32_t ps[kMaxDeg];
      for (int w = 0; w < bw; ++w) nbhdRound[a * bw + w] = nbhd[a * bw + w];
      for (int k = 0; k < deg; ++k) {
        const int b = adjBond[beg + k], o = adjOther[beg + k];
        nbhdRound[a * bw + (b >> 5)] |= 1u << (b & 31);
        for (int w = 0; w < bw; ++w) nbhdRound[a * bw + w] |= nbhd[o * bw + w];
        // insertion sort by (int32 bond type, uint32 invariant)
        const int32_t  f = static_cast<int32_t>(bondInv[b0 + b]);
        const uint32_t sc = inv[o];
        int            p = k;
        while (p > 0 && (pf[p - 1] > f || (pf[p - 1] == f && ps[p - 1] > sc))) {
          pf[p] = pf[p - 1];
          ps[p] = ps[p - 1];
          --p;
        }
        pf[p] = f;
        ps[p] = sc;
      }
      uint32_t invar = static_cast<uint32_t>(layer);
      hashCombine(invar, inv[a]);
      for (int k = 0; k < deg; ++k) {
        uint32_t h = 0;
        hashCombine(h, static_cast<uint32_t>(pf[k]));
        hashCombine(h, ps[k]);
        hashCombine(invar, h);
      }
      invNext[a] = invar;
      cand[a]    = 1;
    }
    __syncwarp();
    // rank test instead of a sort
    int newCount = 0;
    for (int base = 0; base < nA; base += 32) {
      const int a      = base + lane;
      bool      accept = false;
      if (a < nA && cand[a]) {
        const uint32_t* mine = nbhdRound + a * bw;
        bool            lose = false;
        for (int s = 0; s < nSeen && !lose; ++s) {
          bool eq = true;
          for (int w = 0; w < bw; ++w) eq = eq && (seen[s * bw + w] == mine[w]);
          lose = eq;
        }
        for (int a2 = 0; a2 < nA && !lose; ++a2) {
          if (a2 == a || !cand[a2]) continue;
          if (invNext[a2] > invNext[a] || (invNext[a2] == invNext[a] && a2 > a)) continue;
          bool eq = true;
          for (int w = 0; w < bw; ++w) eq = eq && (nbhdRound[a2 * bw + w] == mine[w]);
          lose = eq;
        }
        accept = !lose;
        if (lose) dead[a] = 1;
      }
      const unsigned m    = __ballot_sync(0xffffffffu, accept);
      if (accept) {
        const int slot = nSeen + newCount + __popc(m & ((1u << lane) - 1));
        for (int w = 0; w < bw; ++w) seen[slot * bw + w] = nbhdRound[a * bw + w];
        const uint32_t bit = invNext[a] % fpBits;
        atomicOr(&fp[bit >> 5], 1u << (bit & 31));
      }
      newCount += __popc(m);
    }
    __syncwarp();
    nSeen += newCount;
    uint32_t* t = inv;
    inv         = invNext;
    invNext     = t;
    t           = nbhd;
    nbhd        = nbhdRound;
    nbhdRound   = t;
  }
  __syncwarp();
  for (int w = lane; w < fpWords; w += 32) outRow[w] = fp[w];
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_morgan(const int32_t* d_atom_starts, const int32_t* d_bond_starts, const uint32_t* d_atom_inv,
                              const uint32_t* d_bond_inv, const uint16_t* d_bond_a, const uint16_t* d_bond_b,
                              size_t nMols, int maxAtomsPerMol, int maxBondsPerMol, int radius, int fpBits,
                              uint32_t* d_out, void* stream) {
  return guarded([&] {
    B200_REQUIRE(fpBits > 0 && fpBits % 32 == 0, "fpBits must be a positive multiple of 32, got %d", fpBits);
    B200_REQUIRE(radius >= 0 && radius <= 16, "radius out of range: %d", radius);
    B200_REQUIRE(maxAtomsPerMol >= 0 && maxBondsPerMol >= 0 && maxAtomsPerMol < 65536 && maxBondsPerMol < 65536,
                 "molecule size out of range");
    B200_REQUIRE(nMols < (1ull << 31), "too many molecules");
    if (nMols == 0) return;
    B200_REQUIRE(d_atom_starts && d_bond_starts && d_out, "null pointer");
    cudaStream_t       s       = asStream(stream);
    const int          maxA    = maxAtomsPerMol > 0 ? maxAtomsPerMol : 1;
    const int          maxB    = maxBondsPerMol > 0 ? maxBondsPerMol : 1;
    const MorganLayout L       = morganLayout(maxA, maxB, radius, fpBits / 32);
    const size_t       budget  = 200 * 1024;
    B200_REQUIRE(static_cast<size_t>(L.total) <= budget,
                 "molecule too large for the shared-memory Morgan kernel (%d atoms, %d bonds, radius %d need %d bytes)",
                 maxAtomsPerMol, maxBondsPerMol, radius, L.total);
    int warps = static_cast<int>(budget / 2 / L.total);  // two CTAs per SM when the slab is small
    warps     = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
    const size_t smemBytes = static_cast<size_t>(warps) * L.total;
    static size_t configured[kMaxDevices] = {};
    if (smemBytes > configured[currentDeviceSlot()]) {
      B200_CUDA(cudaFuncSetAttribute(morganKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(budget)));
      configured[currentDeviceSlot()] = budget;
    }
    Scratch<int> err(1, s);
    B200_CUDA(cudaMemsetAsync(err.get(), 0, sizeof(int), s));
    const unsigned blocks = static_cast<unsigned>((nMols + warps - 1) / warps);
    morganKernel<<<blocks, warps * 32, smemBytes, s>>>(d_atom_starts, d_bond_starts, d_atom_inv, d_bond_inv, d_bond_a,
                                                      d_bond_b, static_cast<int>(nMols), maxA, maxB, radius, fpBits,
                                                      d_out, err.get());
    B200_LAUNCHED();
    int hErr = 0;
    B200_CUDA(cudaMemcpyAsync(&hErr, err.get(), sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));  // documented sync: input validation result
    B200_REQUIRE(hErr != 1, "a molecule exceeds maxAtomsPerMol/maxBondsPerMol");
    B200_REQUIRE(hErr != 2, "an atom has more than %d bonds", kMaxDeg);
  });
}
