// Distance-geometry preparation kernels: bounds-matrix triangle smoothing, power-iteration eigensolver,
// metric-matrix embedding. One CTA per molecule, the n x n matrix resident in shared memory (sm_90a: up to 227 KB,
// n <= 164 in fp64; larger matrices are processed in place in global memory / L2 by the same code).
//
// Replaces src/triangle_smooth.cu:27-247 (one kernel LAUNCH per pivot k over the whole concatenated batch, all traffic
// through global memory), src/symmetric_eigensolver.cu:62-247 (matrix in global memory, cuRAND start vector) and
// src/forcefields/coord_gen.cu:55-216 of the reference. Here the pivot loop / power iterations run inside one launch
// with the matrix in shared memory, so each matrix is read from HBM once and written once.
#include "dgprep_device.cuh"

namespace b200 {
namespace {

constexpr int kT = kEigT;

// ---------------------------------------------------------------------------------------------- triangle smoothing
// RDKit BoundsMatrix: [i][j], i<j upper bound; [j][i] lower bound.
__global__ void __launch_bounds__(kT) triangleSmoothKernel(double* mats, const long long* starts, int nMats, double tol,
                                                         int smemCapDoubles, int8_t* ok) {
  extern __shared__ __align__(16) double sm[];
  __shared__ int                        bad;
  for (int m = blockIdx.x; m < nMats; m += gridDim.x) {
    double*         g    = mats + starts[m];
    const long long size = starts[m + 1] - starts[m];
    const int       n    = static_cast<int>(sqrt(static_cast<double>(size)) + 0.5);
    const bool      useS = size <= smemCapDoubles;
    double*         b    = useS ? sm : g;
    __syncthreads();
    if (threadIdx.x == 0) bad = 0;
    if (useS)
      for (long long e = threadIdx.x; e < size; e += kT) sm[e] = g[e];
    __syncthreads();
    const int pairs = n * (n - 1) / 2;
    for (int k = 0; k < n; ++k) {
      for (int p = threadIdx.x; p < pairs; p += kT) {
        // unrank p -> (i, j), i < j  (row-major over the strict upper triangle)
        int i = static_cast<int>((2.0 * n - 1.0 - sqrt((2.0 * n - 1.0) * (2.0 * n - 1.0) - 8.0 * p)) * 0.5);
        int rowStart = i * (2 * n - i - 1) / 2;
        while (rowStart > p) {
          --i;
          rowStart = i * (2 * n - i - 1) / 2;
        }
        while (rowStart + (n - i - 1) <= p) {
          rowStart += n - i - 1;
          ++i;
        }
        const int j = i + 1 + (p - rowStart);
        if (i == k || j == k) continue;
        const int    ii = i < k ? i : k, ik = i < k ? k : i, jj = j < k ? j : k, jk = j < k ? k : j;
        const double Uik = b[ii * n + ik], Lik = b[ik * n + ii], Ukj = b[jj * n + jk], Ljk = b[jk * n + jj];
        double       u = b[i * n + j], l = b[j * n + i];
        const double sumU = Uik + Ukj, d1 = Lik - Ukj, d2 = Ljk - Uik;
        if (u > sumU) u = sumU;
        if (l < d1) l = d1;
        else if (l < d2) l = d2;
        if (tol > 0.0 && (l - u) > 0.0 && (l - u) / l < tol) u = l;
        else if (l - u > 0.0) bad = 1;
        b[i * n + j] = u;
        b[j * n + i] = l;
      }
      __syncthreads();
      const int stop = bad;  // uniform read between two barriers
      __syncthreads();
      if (stop) break;
    }
    if (useS)
      for (long long e = threadIdx.x; e < size; e += kT) g[e] = sm[e];
    if (threadIdx.x == 0) ok[m] = bad ? 0 : 1;
  }
}

// mode 0: matrices are symmetric inputs, outputs eigvals [m][numEigs] + eigvecs (CSR: vecStarts[m] = numEigs * sum n)
// mode 1: matrices are distance matrices -> metric matrix -> coords [atomStart*dim] = sqrt(lambda_j) v_j[i]
__global__ void __launch_bounds__(kT) eigenKernel(int mode, double* mats, const long long* starts, int nMats, int numEigs,
                                                const double* v0, const long long* v0Starts, uint32_t seed,
                                                int smemCapDoubles, double* eigvals, double* eigvecs,
                                                const long long* vecStarts, double* coords, const int* atomStarts,
                                                int8_t* ok) {
  extern __shared__ __align__(16) double sm[];
  __shared__ double                     red[16];
  for (int m = blockIdx.x; m < nMats; m += gridDim.x) {
    double*         g    = mats + starts[m];
    const long long size = starts[m + 1] - starts[m];
    const int       n    = static_cast<int>(sqrt(static_cast<double>(size)) + 0.5);
    double*         v    = sm;
    double*         z    = sm + n;
    double*         vecs = sm + 2 * n;  // numEigs * n (mode 1 keeps them on chip)
    const int       head = 2 * n + (mode == 1 ? numEigs * n + numEigs + n : 0);
    const bool      useS = size + head <= smemCapDoubles;
    double*         mat  = useS ? sm + head : g;
    double*         ev   = mode == 1 ? vecs + numEigs * n : eigvals + static_cast<size_t>(m) * numEigs;
    double*         evec = mode == 1 ? vecs : eigvecs + vecStarts[m];
    __syncthreads();
    if (mode == 1) {
      // metric matrix from distances: T_ij = 0.5 (d0i^2 + d0j^2 - d_ij^2), d0i^2 = mean_j d_ij^2 - mean_pairs d^2 / ...
      double* sq0 = ev + numEigs;  // n doubles
      double  tot = 0.0;
      for (int i = threadIdx.x; i < n; i += kT) {
        double s = 0.0;
        for (int j = 0; j < n; ++j) s += g[i * n + j] * g[i * n + j];
        sq0[i] = s;
        tot += s;
      }
      tot = warpSumD(tot);
      __syncthreads();
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = tot;
      __syncthreads();
      double sumSq = 0.0;
      for (int w = 0; w < kT / 32; ++w) sumSq += red[w];
      sumSq /= static_cast<double>(n) * n * 2.0;
      __syncthreads();
      for (int i = threadIdx.x; i < n; i += kT) sq0[i] = sq0[i] / n - sumSq;
      __syncthreads();
      for (int idx = threadIdx.x; idx < n * n; idx += kT) {
        const double d = g[idx];
        mat[idx]       = 0.5 * (sq0[idx / n] + sq0[idx % n] - d * d);
      }
    } else if (useS) {
      for (long long e = threadIdx.x; e < size; e += kT) mat[e] = g[e];
    }
    __syncthreads();
    const double* myV0 = v0 ? v0 + v0Starts[m] : nullptr;
    const int     done = powerEigen(mat, n, numEigs, myV0, seed + 0x632be5abu * m, v, z, red, ev, evec);
    if (mode == 1) {
      bool good = done == numEigs;
      for (int j = 0; j < numEigs && good; ++j) good = ev[j] > 0.0;
      if (good) {
        const int a0 = atomStarts[m];
        for (int idx = threadIdx.x; idx < n * numEigs; idx += kT) {
          const int i = idx / numEigs, j = idx % numEigs;
          coords[static_cast<size_t>(a0 + i) * numEigs + j] = sqrt(ev[j]) * evec[j * n + i];
        }
      }
      if (threadIdx.x == 0) ok[m] = good ? 1 : 0;
    } else {
      if (threadIdx.x == 0) ok[m] = static_cast<int8_t>(done);
    }
  }
}

int smemCap(const void* fn) {
  B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return 220 * 1024 / 8;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200mol_triangle_smooth(double* d_bounds, const int64_t* d_matrix_starts, int32_t nMats, double tol,
                                       int8_t* d_ok, void* stream) {
  return guarded([&] {
    if (nMats <= 0) return;
    B200_REQUIRE(d_bounds && d_matrix_starts && d_ok, "null pointer");
    static int cap = smemCap(reinterpret_cast<const void*>(triangleSmoothKernel));
    int        blocks = smCount() * 2;
    if (blocks > nMats) blocks = nMats;
    triangleSmoothKernel<<<blocks, kT, static_cast<size_t>(cap) * 8, asStream(stream)>>>(
      d_bounds, reinterpret_cast<const long long*>(d_matrix_starts), nMats, tol, cap, d_ok);
    B200_LAUNCHED();
  });
}

extern "C" int b200mol_eig_topk(double* d_mats, const int64_t* d_matrix_starts, int32_t nMats, int numEigs,
                                const double* d_v0, const int64_t* d_v0_starts, uint32_t seed, double* d_eigvals,
                                double* d_eigvecs, const int64_t* d_vec_starts, int8_t* d_n_converged, void* stream) {
  return guarded([&] {
    if (nMats <= 0) return;
    B200_REQUIRE(numEigs >= 1 && numEigs <= 8, "numEigs must be in [1, 8]");
    B200_REQUIRE(d_mats && d_matrix_starts && d_eigvals && d_eigvecs && d_vec_starts && d_n_converged, "null pointer");
    B200_REQUIRE(!d_v0 || d_v0_starts, "d_v0 needs d_v0_starts");
    static int cap = smemCap(reinterpret_cast<const void*>(eigenKernel));
    int        blocks = smCount() * 2;
    if (blocks > nMats) blocks = nMats;
    eigenKernel<<<blocks, kT, static_cast<size_t>(cap) * 8, asStream(stream)>>>(
      0, d_mats, reinterpret_cast<const long long*>(d_matrix_starts), nMats, numEigs, d_v0,
      reinterpret_cast<const long long*>(d_v0_starts), seed, cap, d_eigvals, d_eigvecs,
      reinterpret_cast<const long long*>(d_vec_starts), nullptr, nullptr, d_n_converged);
    B200_LAUNCHED();
  });
}

extern "C" int b200mol_metric_embed(double* d_dist, const int64_t* d_matrix_starts, const int32_t* d_atom_starts,
                                    int32_t nMats, int dim, const double* d_v0, const int64_t* d_v0_starts, uint32_t seed,
                                    double* d_coords, int8_t* d_ok, void* stream) {
  return guarded([&] {
    if (nMats <= 0) return;
    B200_REQUIRE(dim == 3 || dim == 4, "dim must be 3 or 4");
    B200_REQUIRE(d_dist && d_matrix_starts && d_atom_starts && d_coords && d_ok, "null pointer");
    B200_REQUIRE(!d_v0 || d_v0_starts, "d_v0 needs d_v0_starts");
    static int cap = smemCap(reinterpret_cast<const void*>(eigenKernel));
    int        blocks = smCount() * 2;
    if (blocks > nMats) blocks = nMats;
    eigenKernel<<<blocks, kT, static_cast<size_t>(cap) * 8, asStream(stream)>>>(
      1, d_dist, reinterpret_cast<const long long*>(d_matrix_starts), nMats, dim, d_v0,
      reinterpret_cast<const long long*>(d_v0_starts), seed, cap, nullptr, nullptr, nullptr, d_coords, d_atom_starts, d_ok);
    B200_LAUNCHED();
  });
}
