// Shared host/device helpers for libb200mol (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

#include "../../include/b200mol.h"

namespace b200 {

extern thread_local std::string g_lastError;
extern std::atomic<uint64_t>    g_launchCount;

struct Failure {
  int         code;
  std::string msg;
};

[[noreturn]] inline void fail(int code, const char* fmt, ...) {
  char    buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw Failure{code, buf};
}

#define B200_CUDA(expr)                                                                                   \
  do {                                                                                                    \
    cudaError_t e_ = (expr);                                                                              \
    if (e_ != cudaSuccess)                                                                                \
      ::b200::fail(B200MOL_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

#define B200_REQUIRE(cond, ...)                             \
  do {                                                      \
    if (!(cond)) ::b200::fail(B200MOL_ERR_INVALID, __VA_ARGS__); \
  } while (0)

// Count a kernel launch and check it.
#define B200_LAUNCHED()                 \
  do {                                  \
    ::b200::g_launchCount.fetch_add(1); \
    B200_CUDA(cudaGetLastError());      \
  } while (0)

// Wrap the body of an extern "C" entry point.
template <class F>
inline int guarded(F&& f) noexcept {
  try {
    f();
    return B200MOL_OK;
  } catch (const Failure& e) {
    g_lastError = e.msg;
    return e.code;
  } catch (const std::exception& e) {
    g_lastError = e.what();
    return B200MOL_ERR_CUDA;
  } catch (...) {
    g_lastError = "unknown failure";
    return B200MOL_ERR_CUDA;
  }
}

// Stream-ordered scratch allocation (RAII).
template <class T>
struct Scratch {
  T*           p = nullptr;
  cudaStream_t s = nullptr;
  Scratch() = default;
  Scratch(size_t n, cudaStream_t stream) : s(stream) {
    if (n) B200_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p), n * sizeof(T), stream));
  }
  Scratch(const Scratch&)            = delete;
  Scratch& operator=(const Scratch&) = delete;
  Scratch(Scratch&& o) noexcept : p(o.p), s(o.s) { o.p = nullptr; }
  Scratch& operator=(Scratch&& o) noexcept {
    if (this != &o) {
      release();
      p   = o.p;
      s   = o.s;
      o.p = nullptr;
    }
    return *this;
  }
  void release() {
    if (p) cudaFreeAsync(p, s);
    p = nullptr;
  }
  ~Scratch() { release(); }
  T* get() const { return p; }
};

inline int smCount() {  // of the current device
  static int cached[64] = {};
  int        dev        = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int v = 132;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = v > 0 ? v : 132;
  }
  return cached[dev];
}

// Function attributes (dynamic shared-memory limits) belong to the device's context: a process that drives several
// GPUs (HardwareOptions.gpuIds / targetGpu) must set them once per DEVICE, not once per process.
constexpr int kMaxDevices = 64;
inline int currentDeviceSlot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
  return dev;
}

inline cudaStream_t asStream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// RAII: while alive, accesses of kernels launched on `s` to [ptr, ptr + bytes) are marked PERSISTING in L2 (the rest
// streaming): the inverse-Hessian slabs of the minimiser kernels are re-read every iteration while the term tables only
// stream through. Best effort - failures of the attribute calls are ignored (the kernels are correct without it).
struct L2Persist {
  cudaStream_t s      = nullptr;
  bool         active = false;
  L2Persist(cudaStream_t stream, const void* ptr, size_t bytes, bool enable) : s(stream) {
    if (!enable || !ptr || !bytes) return;
    int dev = 0, maxPersist = 0, maxWindow = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return;
    cudaDeviceGetAttribute(&maxPersist, cudaDevAttrMaxPersistingL2CacheSize, dev);
    cudaDeviceGetAttribute(&maxWindow, cudaDevAttrMaxAccessPolicyWindowSize, dev);
    if (maxPersist <= 0 || maxWindow <= 0) return;
    cudaCtxResetPersistingL2Cache();  // lines a previous launch left persisting
    if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, static_cast<size_t>(maxPersist)) != cudaSuccess) return;
    cudaStreamAttrValue v{};
    v.accessPolicyWindow.base_ptr  = const_cast<void*>(ptr);
    v.accessPolicyWindow.num_bytes = bytes < static_cast<size_t>(maxWindow) ? bytes : static_cast<size_t>(maxWindow);
    const double ratio             = static_cast<double>(maxPersist) / static_cast<double>(v.accessPolicyWindow.num_bytes);
    v.accessPolicyWindow.hitRatio  = ratio < 1.0 ? static_cast<float>(ratio) : 1.0f;
    v.accessPolicyWindow.hitProp   = cudaAccessPropertyPersisting;
    v.accessPolicyWindow.missProp  = cudaAccessPropertyStreaming;
    active = cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &v) == cudaSuccess;
    cudaGetLastError();
  }
  ~L2Persist() {
    if (!active) return;
    cudaStreamAttrValue v{};
    v.accessPolicyWindow.num_bytes = 0;
    cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &v);  // (later launches on `s` are unaffected; the
    cudaGetLastError();  // kernel just launched keeps the policy it was launched with; its persisting lines age out)
  }
};

}  // namespace b200
