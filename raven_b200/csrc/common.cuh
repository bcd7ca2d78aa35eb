// raven_b200 — shared device/host helpers for the overlap engine (sm_90a).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace rvn {

struct CudaError : std::runtime_error {
  explicit CudaError(const std::string& m) : std::runtime_error(m) {}
};
struct InvalidArgument : std::runtime_error {
  explicit InvalidArgument(const std::string& m) : std::runtime_error(m) {}
};
struct StateError : std::runtime_error {
  explicit StateError(const std::string& m) : std::runtime_error(m) {}
};
struct LimitError : std::runtime_error {
  explicit LimitError(const std::string& m) : std::runtime_error(m) {}
};

#define RVN_CUDA(expr)                                                        \
  do {                                                                        \
    cudaError_t e_ = (expr);                                                  \
    if (e_ != cudaSuccess) {                                                  \
      throw ::rvn::CudaError(std::string(#expr) + ": " +                      \
                             cudaGetErrorString(e_) + " (" + __FILE__ + ":" + \
                             std::to_string(__LINE__) + ")");                 \
    }                                                                         \
  } while (0)

#define RVN_LAUNCH_CHECK() RVN_CUDA(cudaGetLastError())

// Device bytes held by the DevBufs of one context (Ctx::held_bytes): a buffer charges
// the counter that is current on its thread when it allocates (the C ABI makes the
// calling context's current for the call) and gives the bytes back to that counter.
// The stage-1 memory estimate counts them as reusable.
inline thread_local std::uint64_t* g_devbuf_owner = nullptr;

// Grow-only device buffer: steady-state steps re-use capacity, so no
// cudaMalloc lands inside a timed region after warm-up.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  std::size_t cap = 0;  // elements
  std::uint64_t* owner = nullptr;  // the counter charged with cap * sizeof(T)
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    uncharge();
    p = nullptr;
    cap = 0;
  }
  void charge(std::size_t elems) {
    owner = g_devbuf_owner;
    if (owner) *owner += elems * sizeof(T);
  }
  void uncharge() {
    if (owner) *owner -= cap * sizeof(T);
    owner = nullptr;
  }
  // contents are NOT preserved on growth
  T* reserve(std::size_t n) {
    if (n > cap) {
      release();
      std::size_t want = n + n / 16 + 64;
      RVN_CUDA(cudaMalloc(&p, want * sizeof(T)));
      cap = want;
      charge(want);
    }
    return p;
  }
  // growth keeps the first `keep` elements
  T* reserve_keep(std::size_t n, std::size_t keep, cudaStream_t stream) {
    if (n > cap) {
      std::size_t want = n + n / 16 + 64;
      T* np = nullptr;
      RVN_CUDA(cudaMalloc(&np, want * sizeof(T)));
      if (p && keep) {
        RVN_CUDA(cudaMemcpyAsync(np, p, keep * sizeof(T), cudaMemcpyDeviceToDevice,
                                 stream));
        RVN_CUDA(cudaStreamSynchronize(stream));
      }
      if (p) cudaFree(p);
      uncharge();
      p = np;
      cap = want;
      charge(want);
    }
    return p;
  }
  T* get() const { return p; }
  void swap(DevBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
    std::swap(owner, o.owner);
  }
};

// Minimizer values travel as u32 when 2k <= 30 bits (k <= 15: raven's default)
// and as u64 otherwise; kernels that only read them take this view.
struct ValView {
  const void* p;
  int is32;
#ifdef __CUDACC__
  __device__ __forceinline__ uint64_t operator[](uint64_t i) const {
    return is32 ? static_cast<uint64_t>(static_cast<const uint32_t*>(p)[i])
                : static_cast<const uint64_t*>(p)[i];
  }
#endif
};

// Grow-only pinned host buffer (D2H results, H2D staging).
template <typename T>
struct PinBuf {
  T* p = nullptr;
  std::size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() {
    if (p) cudaFreeHost(p);
  }
  T* reserve(std::size_t n) {
    if (n > cap) {
      if (p) cudaFreeHost(p);
      p = nullptr;
      std::size_t want = n + n / 16 + 64;
      RVN_CUDA(cudaMallocHost(&p, want * sizeof(T)));
      cap = want;
    }
    return p;
  }
  // growth keeps the first `keep` elements
  T* reserve_keep(std::size_t n, std::size_t keep) {
    if (n > cap) {
      T* np = nullptr;
      std::size_t want = n + n / 16 + 64;
      RVN_CUDA(cudaMallocHost(&np, want * sizeof(T)));
      for (std::size_t i = 0; p && i < keep; ++i) np[i] = p[i];
      if (p) cudaFreeHost(p);
      p = np;
      cap = want;
    }
    return p;
  }
  T* get() const { return p; }
  void swap(PinBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
  }
};

inline unsigned CeilDiv(std::uint64_t a, std::uint64_t b) {
  return static_cast<unsigned>((a + b - 1) / b);
}

#ifdef __CUDACC__

// ---- block-wide exclusive scan (sum) over one value per thread ----
// smem: at least 33 x T. Returns the exclusive prefix; *total = block sum.
template <typename T, int THREADS>
__device__ __forceinline__ T BlockExclusiveSum(T v, T* smem, T* total) {
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    constexpr int NW = THREADS / 32;
    T w = lane < NW ? smem[lane] : T(0);
    T wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      T o = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += o;
    }
    if (lane < NW) smem[lane] = wi - w;  // exclusive warp offsets
    if (lane == NW - 1) smem[32] = wi;   // block total
  }
  __syncthreads();
  T res = smem[warp] + incl - v;
  *total = smem[32];
  __syncthreads();  // smem reusable by the caller afterwards
  return res;
}

// ---- block-wide inclusive max-scan ----
template <typename T, int THREADS>
__device__ __forceinline__ T BlockInclusiveMax(T v, T* smem) {
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  T incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl = incl > o ? incl : o;
  }
  if (lane == 31) smem[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    constexpr int NW = THREADS / 32;
    T w = lane < NW ? smem[lane] : T(0);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      T o = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w = w > o ? w : o;
    }
    if (lane < NW) smem[lane] = w;  // inclusive max over warps 0..lane
  }
  __syncthreads();
  T res = incl;
  if (warp > 0) {
    T o = smem[warp - 1];
    res = res > o ? res : o;
  }
  __syncthreads();
  return res;
}

#endif  // __CUDACC__

}  // namespace rvn
