// Device-side pieces of the distance-geometry preparation shared by dgprep.cu (stand-alone entry points) and etkdg.cu
// (metric-matrix initial coordinates inside the embedding kernel): the power-iteration eigensolver.
#pragma once
#include "common.cuh"

namespace b200 {

#ifndef B200_BFGS_THREADS
#define B200_BFGS_THREADS 256
#endif
constexpr int kEigT = B200_BFGS_THREADS;  // threads per CTA of every caller (the embedder's CTA shape)
constexpr int kEigWarps = kEigT / 32;
// Doubles of shared memory behind powerEigen's `red`: one double per warp, then the argmax index of each warp as an int.
constexpr int kEigRed = kEigWarps + (kEigWarps * static_cast<int>(sizeof(int)) + 7) / 8;

__device__ __forceinline__ double warpSumD(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------- power eigensolver
__device__ __forceinline__ uint32_t hash32(uint32_t x) {  // counter-based start vector when the caller gives none
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

// mat: n x n symmetric (destroyed by deflation); v, z: n doubles of shared memory; red: kEigRed doubles.
// Returns (to all threads) the number of converged eigenpairs. eigvecs: [numEigs][n].
__device__ inline int powerEigen(double* mat, int n, int numEigs, const double* v0, uint32_t seed, double* v, double* z,
                          double* red, double* eigvals, double* eigvecs) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nWarps = kEigWarps;
  int*      redIdx = reinterpret_cast<int*>(red + nWarps);
  int       done = 0;
  for (int e = 0; e < numEigs; ++e) {
    double part = 0.0;
    for (int i = tid; i < n; i += kEigT) {
      const double x = v0 ? v0[e * n + i] : (hash32(seed ^ (e * 0x9e3779b9u) ^ (i * 0x85ebca6bu)) + 1.0) * (1.0 / 4294967297.0);
      v[i]           = x;
      part += x * x;
    }
    part = warpSumD(part);
    __syncthreads();
    if (lane == 0) red[warp] = part;
    __syncthreads();
    double norm = 0.0;
    for (int w = 0; w < nWarps; ++w) norm += red[w];
    norm = sqrt(norm);
    for (int i = tid; i < n; i += kEigT) v[i] /= norm;
    double eig       = -1000.0;
    bool   converged = false;
    for (int it = 0; it < 1000; ++it) {
      __syncthreads();
      const double prev = eig;
      for (int r = warp; r < n; r += nWarps) {
        double a = 0.0;
        for (int c = lane; c < n; c += 32) a += mat[r * n + c] * v[c];
        a = warpSumD(a);
        if (lane == 0) z[r] = a;
      }
      __syncthreads();
      // element of largest magnitude (first such index, like a sequential scan)
      double best = 0.0;
      int    bi   = 0x7fffffff;
      for (int i = tid; i < n; i += kEigT)
        if (fabs(z[i]) > fabs(best) || (fabs(z[i]) == fabs(best) && i < bi)) {
          best = z[i];
          bi   = i;
        }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int    oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (fabs(ob) > fabs(best) || (fabs(ob) == fabs(best) && oi < bi)) {
          best = ob;
          bi   = oi;
        }
      }
      if (lane == 0) {
        red[warp]    = best;
        redIdx[warp] = bi;
      }
      __syncthreads();
      best = red[0];
      bi   = redIdx[0];
      for (int w = 1; w < nWarps; ++w) {
        const double ob = red[w];
        const int    oi = redIdx[w];
        if (fabs(ob) > fabs(best) || (fabs(ob) == fabs(best) && oi < bi)) {
          best = ob;
          bi   = oi;
        }
      }
      eig = best;
      if (fabs(eig) < 1.0e-10) break;
      __syncthreads();
      for (int i = tid; i < n; i += kEigT) v[i] = z[i] / eig;
      if (fabs(eig - prev) < 0.001) {
        converged = true;
        break;
      }
    }
    __syncthreads();
    if (!converged) break;
    part = 0.0;
    for (int i = tid; i < n; i += kEigT) part += v[i] * v[i];
    part = warpSumD(part);
    __syncthreads();
    if (lane == 0) red[warp] = part;
    __syncthreads();
    norm = 0.0;
    for (int w = 0; w < nWarps; ++w) norm += red[w];
    norm = sqrt(norm);
    for (int i = tid; i < n; i += kEigT) {
      v[i] /= norm;
      eigvecs[e * n + i] = v[i];
    }
    if (tid == 0) eigvals[e] = eig;
    __syncthreads();
    for (int idx = tid; idx < n * n; idx += kEigT) mat[idx] -= eig * v[idx / n] * v[idx % n];
    __syncthreads();  // the next eigenpair's start vector overwrites v: every thread must be done deflating with it
    ++done;
  }
  __syncthreads();
  return done;
}


}  // namespace b200
