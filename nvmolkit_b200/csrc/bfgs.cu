// Batched BFGS over flattened force fields: one CTA per conformer, the WHOLE minimisation inside one persistent kernel.
//
// Algorithm = RDKit BFGSOpt.h (+ ForceField::minimize gradient scaling) as transcribed by the reference's BATCHED
// backend (src/minimizer/bfgs_minimize.cu:80-918, src/minimizer/bfgs_hessian.cu:37-239), all in fp64.
//
// Design (differs from the reference's bfgsMinimizeKernel, bfgs_minimize_permol_kernels.cu:426-743):
//   * persistent grid (3 CTAs per SM) pulling conformers from an atomic queue -> no tail from uneven convergence and no
//     size buckets / host-driven fallback for molecules above 64 atoms;
//   * term tables are per MOLECULE with local int16 indices, shared by all conformers of that molecule;
//   * positions, gradient, direction, trial point, dGrad and H*dGrad live in shared memory for any molecule size;
//   * the inverse Hessian is a per-CTA slab, ONE sweep over its upper triangle per iteration with the rank-2 update of the
//     previous iteration applied on the way (bfgs_device.cuh);
//   * no atomics at all: gradients are scattered wave by wave (atom-disjoint groups of 32 terms scheduled by the host,
//     b200mol_schedule_waves) into per-warp shared-memory accumulators and reduced in a fixed order, the sweep's
//     row / column sums likewise -> a minimisation is bit-reproducible run to run.
#include "bfgs_device.cuh"
#include "profile.cuh"

namespace b200 {
int g_bfgsCtasPerSm = kMinCtas;  // resident minimisation CTAs per SM (option "bfgs_ctas_per_sm")
int g_bfgsL2Persist = 0;         // mark the inverse-Hessian slabs persisting in L2 (option "bfgs_l2_persist")

// Device-side work counters of the conformer kernels, one small buffer per device, allocated on first use: two banks of
// kStatCount, [0] the embedder (etkdgKernel), [1] the stand-alone minimisers (bfgsKernel<FF>).
unsigned long long* pathBStats() {
  static unsigned long long* buf[kMaxDevices] = {};
  const int                  d               = currentDeviceSlot();
  if (!buf[d]) {
    B200_CUDA(cudaMalloc(reinterpret_cast<void**>(&buf[d]), 2 * kStatCount * sizeof(unsigned long long)));
    B200_CUDA(cudaMemset(buf[d], 0, 2 * kStatCount * sizeof(unsigned long long)));
  }
  return buf[d];
}
namespace {

struct Batch {
  int            nConf;
  const int32_t* confMol;        // may be NULL: conformer c is molecule c
  const int32_t* confAtomStart;  // [nConf+1]
  double*        pos;
  int            maxIters;
  double         gradTol;
  int            scaleGrads;
  int            maxRestarts;
  const uint8_t* active;
  double*        energy;
  int8_t*        status;
  int32_t*       iters;
  void*          hessWs;  // inverse-Hessian slabs of the kernel's storage type HT
  size_t         hessStride;
  int*           queue;
  int            maxN;
  unsigned long long* stats;
};

// HT = storage type of the inverse-Hessian slab: double for the force fields, float as well for the analytic test
// systems (the embedder's default type, bfgs_device.cuh)
template <class FF, class HT>
__global__ void __launch_bounds__(kT, kMinCtas) bfgsKernel(const typename FF::System sys, const typename FF::Params par, const Batch b) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[kRed];
  __shared__ double                     colBuf[kColBuf];
  __shared__ int                        nextConf;
  constexpr int                         DIM = FF::kDim;
  const BfgsWorkT<HT> w =
      carveWork<HT>(sm, b.maxN, static_cast<HT*>(b.hessWs) + static_cast<size_t>(blockIdx.x) * b.hessStride, red, colBuf, b.stats);
  const int      tid = threadIdx.x;
  for (;;) {
    __syncthreads();
    if (tid == 0) nextConf = atomicAdd(b.queue, 1);
    __syncthreads();
    const int conf = nextConf;
    if (conf >= b.nConf) break;
    if (b.active && !b.active[conf]) continue;
    const int  mol  = b.confMol ? b.confMol[conf] : conf;
    const int  a0   = b.confAtomStart[conf];
    const int  n    = DIM * (b.confAtomStart[conf + 1] - a0);
    double*    gpos = b.pos + static_cast<size_t>(a0) * DIM;
    auto       view = FF::view(sys, mol, par);
    for (int i = tid; i < n; i += kT) w.pos[i] = gpos[i];
    if constexpr (FF::kHasRef) {
      if (par.recentre) {  // seventh shared vector: the reference geometry of the window refresh
        double* ref = sm + kBfgsVectors * b.maxN;
        for (int i = tid; i < n; i += kT) ref[i] = gpos[i];
        view.refPos = ref;
      }
    }
    __syncthreads();
    const BfgsOutcome o = bfgsMinimize<FF, HT>(view, w, n, b.maxIters, b.gradTol, b.scaleGrads != 0, b.maxRestarts);
    for (int i = tid; i < n; i += kT) gpos[i] = w.pos[i];
    if (tid == 0) {
      b.energy[conf] = o.energy;
      if (b.status) b.status[conf] = static_cast<int8_t>(o.status);
      if (b.iters) b.iters[conf] = o.iters;
    }
  }
}

// Energies (+ gradients) of a conformer batch: CTA per conformer, coordinates staged in shared memory.
template <class FF>
__global__ void __launch_bounds__(kT) energyGradKernel(const typename FF::System sys, const typename FF::Params par, int nConf,
                                                     const int32_t* confMol, const int32_t* confAtomStart,
                                                     const double* posIn, double* energy, double* gradOut, int maxN) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[kRed];
  constexpr int                         DIM = FF::kDim;
  double*                               pos  = sm;
  double*                               grad = sm + maxN;  // kWarps accumulators; the reduced gradient ends up in the first
  for (int conf = blockIdx.x; conf < nConf; conf += gridDim.x) {
    const int mol = confMol ? confMol[conf] : conf;
    const int a0  = confAtomStart[conf];
    const int n   = DIM * (confAtomStart[conf + 1] - a0);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kT) pos[i] = posIn[static_cast<size_t>(a0) * DIM + i];
    __syncthreads();
    auto view = FF::view(sys, mol, par);
    if constexpr (FF::kHasRef) {
      if (par.recentre) view.refPos = pos;
    }
    const double e = energyOf<FF>(view, pos, red);
    if (threadIdx.x == 0) energy[conf] = e;
    if (gradOut) {
      gradOf<FF>(view, pos, grad, maxN, n);
      for (int i = threadIdx.x; i < n; i += kT) gradOut[static_cast<size_t>(a0) * DIM + i] = grad[i];
    }
  }
}

template <class FF, class HT = double>
void runMinimize(const typename FF::System& sys, const typename FF::Params& par, int nConf, const int32_t* confMol,
                 const int32_t* confAtomStart, int maxAtoms, double* pos, int maxIters, double gradTol, int scaleGrads,
                 const uint8_t* active, double* energy, int8_t* status, int32_t* iters, cudaStream_t s) {
  if (nConf == 0) return;
  B200_REQUIRE(nConf > 0 && maxAtoms > 0 && maxIters >= 0, "bad batch arguments");
  B200_REQUIRE(confAtomStart && pos && energy, "null pointer");
  ff::requireSchedule(sys);
  const int    maxN = FF::kDim * maxAtoms;
  const size_t smem = static_cast<size_t>(kBfgsVectors + (FF::kHasRef ? 1 : 0)) * maxN * sizeof(double);
  B200_REQUIRE(smem <= 200 * 1024, "molecule too large for the shared-memory BFGS (%d atoms)", maxAtoms);
  static bool configured[kMaxDevices] = {};  // per instantiation and device; static + dynamic may pass 48 KB together
  if (!configured[currentDeviceSlot()]) {
    B200_CUDA(cudaFuncSetAttribute(bfgsKernel<FF, HT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured[currentDeviceSlot()] = true;
  }
  int perSm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, bfgsKernel<FF, HT>, kT, smem));
  B200_REQUIRE(perSm >= 1, "BFGS kernel does not fit");
  perSm            = perSm > g_bfgsCtasPerSm ? g_bfgsCtasPerSm : perSm;
  int blocks       = smCount() * perSm;
  if (blocks > nConf) blocks = nConf;
  const size_t       stride = static_cast<size_t>(maxN) * bfgsLd<HT>(maxN);
  Scratch<HT>        hess(stride * blocks, s);
  Scratch<int>       queue(1, s);
  B200_CUDA(cudaMemsetAsync(queue.get(), 0, sizeof(int), s));
  Batch b{nConf, confMol, confAtomStart, pos, maxIters, gradTol, scaleGrads, 0, active, energy, status, iters,
          hess.get(), stride, queue.get(), maxN, pathBStats() + kStatCount};
  L2Persist  keep(s, hess.get(), stride * blocks * sizeof(HT), g_bfgsL2Persist != 0);
  PhaseTimer t("bfgs", s);
  bfgsKernel<FF, HT><<<blocks, kT, smem, s>>>(sys, par, b);
  B200_LAUNCHED();
}

template <class FF>
void runEnergyGrad(const typename FF::System& sys, const typename FF::Params& par, int nConf, const int32_t* confMol,
                   const int32_t* confAtomStart, int maxAtoms, const double* pos, double* energy, double* grad,
                   cudaStream_t s) {
  if (nConf == 0) return;
  B200_REQUIRE(confAtomStart && pos && energy, "null pointer");
  if (grad) ff::requireSchedule(sys);
  const int    maxN = FF::kDim * maxAtoms;
  const size_t smem = static_cast<size_t>(1 + kWarps) * maxN * sizeof(double);
  B200_REQUIRE(smem <= 200 * 1024, "molecule too large (%d atoms)", maxAtoms);
  static bool configured[kMaxDevices] = {};
  if (!configured[currentDeviceSlot()]) {
    B200_CUDA(cudaFuncSetAttribute(energyGradKernel<FF>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured[currentDeviceSlot()] = true;
  }
  int blocks = smCount() * 4;
  if (blocks > nConf) blocks = nConf;
  energyGradKernel<FF><<<blocks, kT, smem, s>>>(sys, par, nConf, confMol, confAtomStart, pos, energy, grad, maxN);
  B200_LAUNCHED();
}

// max atoms of a batch, needed by the energy entry points that do not take it: computed on device, read back.
__global__ void maxSpanKernel(const int32_t* starts, int n, int* out) {
  int m = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = max(m, starts[i + 1] - starts[i]);
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}
int maxSpan(const int32_t* dStarts, int n, cudaStream_t s) {
  Scratch<int> d(1, s);
  B200_CUDA(cudaMemsetAsync(d.get(), 0, sizeof(int), s));
  maxSpanKernel<<<64, 256, 0, s>>>(dStarts, n, d.get());
  B200_LAUNCHED();
  int h = 0;
  B200_CUDA(cudaMemcpyAsync(&h, d.get(), sizeof(int), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  return h;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_mmff_energy_grad(const b200mol_mmff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                                        const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy,
                                        double* d_grad, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    if (nConf <= 0) return;
    const int maxAtoms = maxSpan(d_conf_atom_start, nConf, asStream(stream));
    runEnergyGrad<ff::Mmff>(*sys, {}, nConf, d_conf_mol, d_conf_atom_start, maxAtoms, d_pos, d_energy, d_grad, asStream(stream));
  });
}
extern "C" int b200mol_uff_energy_grad(const b200mol_uff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                                       const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy,
                                       double* d_grad, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    if (nConf <= 0) return;
    const int maxAtoms = maxSpan(d_conf_atom_start, nConf, asStream(stream));
    runEnergyGrad<ff::Uff>(*sys, {}, nConf, d_conf_mol, d_conf_atom_start, maxAtoms, d_pos, d_energy, d_grad, asStream(stream));
  });
}
extern "C" int b200mol_uff_minimize(const b200mol_uff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                                    const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                                    double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                                    int32_t* d_iters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    runMinimize<ff::Uff>(*sys, {}, nConf, d_conf_mol, d_conf_atom_start, max_atoms, d_pos, max_iters, grad_tol, 1, d_active,
                         d_energy, d_status, d_iters, asStream(stream));
  });
}
extern "C" int b200mol_dg_energy_grad(const b200mol_dg_system* sys, int dim, double chiralWeight, double fourthDimWeight,
                                      int32_t nConf, const int32_t* d_conf_mol, const int32_t* d_conf_atom_start,
                                      const double* d_pos, double* d_energy, double* d_grad, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    B200_REQUIRE(dim == 3 || dim == 4, "dim must be 3 or 4");
    if (nConf <= 0) return;
    const int maxAtoms = maxSpan(d_conf_atom_start, nConf, asStream(stream));
    if (dim == 4)
      runEnergyGrad<ff::Dg<4>>(*sys, {chiralWeight, fourthDimWeight}, nConf, d_conf_mol, d_conf_atom_start, maxAtoms, d_pos,
                               d_energy, d_grad, asStream(stream));
    else
      runEnergyGrad<ff::Dg<3>>(*sys, {chiralWeight, fourthDimWeight}, nConf, d_conf_mol, d_conf_atom_start, maxAtoms, d_pos,
                               d_energy, d_grad, asStream(stream));
  });
}
extern "C" int b200mol_etk_energy_grad(const b200mol_etk_system* sys, int plain, int recentre, int32_t nConf, const int32_t* d_conf_mol,
                                       const int32_t* d_conf_atom_start, const double* d_pos, double* d_energy,
                                       double* d_grad, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    if (nConf <= 0) return;
    const int maxAtoms = maxSpan(d_conf_atom_start, nConf, asStream(stream));
    runEnergyGrad<ff::Etk>(*sys, {plain, recentre}, nConf, d_conf_mol, d_conf_atom_start, maxAtoms, d_pos, d_energy, d_grad, asStream(stream));
  });
}

extern "C" int b200mol_mmff_minimize(const b200mol_mmff_system* sys, int32_t nConf, const int32_t* d_conf_mol,
                                     const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                                     double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                                     int32_t* d_iters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    runMinimize<ff::Mmff>(*sys, {}, nConf, d_conf_mol, d_conf_atom_start, max_atoms, d_pos, max_iters, grad_tol, 1, d_active,
                          d_energy, d_status, d_iters, asStream(stream));
  });
}
extern "C" int b200mol_dg_minimize(const b200mol_dg_system* sys, int dim, double chiralWeight, double fourthDimWeight,
                                   int32_t nConf, const int32_t* d_conf_mol, const int32_t* d_conf_atom_start,
                                   int max_atoms, double* d_pos, int max_iters, double grad_tol, const uint8_t* d_active,
                                   double* d_energy, int8_t* d_status, int32_t* d_iters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    B200_REQUIRE(dim == 3 || dim == 4, "dim must be 3 or 4");
    if (dim == 4)
      runMinimize<ff::Dg<4>>(*sys, {chiralWeight, fourthDimWeight}, nConf, d_conf_mol, d_conf_atom_start, max_atoms, d_pos,
                             max_iters, grad_tol, 1, d_active, d_energy, d_status, d_iters, asStream(stream));
    else
      runMinimize<ff::Dg<3>>(*sys, {chiralWeight, fourthDimWeight}, nConf, d_conf_mol, d_conf_atom_start, max_atoms, d_pos,
                             max_iters, grad_tol, 1, d_active, d_energy, d_status, d_iters, asStream(stream));
  });
}
extern "C" int b200mol_etk_minimize(const b200mol_etk_system* sys, int plain, int recentre, int32_t nConf, const int32_t* d_conf_mol,
                                    const int32_t* d_conf_atom_start, int max_atoms, double* d_pos, int max_iters,
                                    double grad_tol, const uint8_t* d_active, double* d_energy, int8_t* d_status,
                                    int32_t* d_iters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(sys, "null system");
    runMinimize<ff::Etk>(*sys, {plain, recentre}, nConf, d_conf_mol, d_conf_atom_start, max_atoms, d_pos, max_iters, grad_tol, 1,
                         d_active, d_energy, d_status, d_iters, asStream(stream));
  });
}
extern "C" int b200mol_poly_minimize(int32_t nSys, const int32_t* d_starts, int max_dim, int power, const double* d_w,
                                     const double* d_c, double* d_x, int max_iters, double grad_tol, int scale_grads,
                                     int hessian_fp32, double* d_energy, int8_t* d_status, int32_t* d_iters, void* stream) {
  return guarded([&] {
    B200_REQUIRE(power == 2 || power == 4, "power must be 2 or 4");
    ff::Poly::System sys{power, d_w, d_c, d_starts};
    if (hessian_fp32)
      runMinimize<ff::Poly, float>(sys, {}, nSys, nullptr, d_starts, max_dim, d_x, max_iters, grad_tol, scale_grads, nullptr,
                                   d_energy, d_status, d_iters, asStream(stream));
    else
      runMinimize<ff::Poly, double>(sys, {}, nSys, nullptr, d_starts, max_dim, d_x, max_iters, grad_tol, scale_grads, nullptr,
                                    d_energy, d_status, d_iters, asStream(stream));
  });
}

extern "C" int b200mol_stats_read(uint64_t* h_out16, int reset, void* stream) {
  return guarded([&] {
    B200_REQUIRE(h_out16, "null pointer");
    cudaStream_t        s = asStream(stream);
    unsigned long long* d = pathBStats();
    B200_CUDA(cudaMemcpyAsync(h_out16, d, 2 * kStatCount * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    if (reset) B200_CUDA(cudaMemsetAsync(d, 0, 2 * kStatCount * sizeof(unsigned long long), s));
    B200_CUDA(cudaStreamSynchronize(s));
  });
}

#ifdef B200_BFGS_TIMING
extern "C" void b200mol_debug_clocks_bfgs(unsigned long long* out8) { b200::readBfgsClocks(out8); }
#endif
