// Shared helpers for the tandem_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>

namespace tdm {

// Error convention of the C-ABI: internal code throws, capi.cu converts to int codes + tdm_last_error().
struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define TDM_CUDA(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      throw ::tdm::Error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " @" + __FILE__ + \
                         ":" + std::to_string(__LINE__));                                           \
  } while (0)

#define TDM_CHECK(cond, msg)                                                    \
  do {                                                                          \
    if (!(cond)) throw ::tdm::Error(std::string("check failed: ") + (msg));     \
  } while (0)

// Owners of CUDA resources: each releases its resource when it goes out of scope, so a throw between two creations leaks
// nothing and no class frees by hand.  The device alias of mapped host memory (cudaHostGetDevicePointer) is a plain pointer.
struct DevFree { void operator()(void* p) const { cudaFree(p); } };
struct HostFree { void operator()(void* p) const { cudaFreeHost(p); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct GraphExecDestroy { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
struct GraphDestroy { void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); } };

template <typename T> using DevPtr = std::unique_ptr<T, DevFree>;
template <typename T> using HostPtr = std::unique_ptr<T, HostFree>;   // cudaMallocHost and cudaHostAlloc memory
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;
using GraphExec = std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, GraphExecDestroy>;
using Graph = std::unique_ptr<std::remove_pointer_t<cudaGraph_t>, GraphDestroy>;

template <typename T = void> DevPtr<T> make_dev(size_t bytes) {
  void* p = nullptr;
  TDM_CUDA(cudaMalloc(&p, bytes));
  return DevPtr<T>(static_cast<T*>(p));
}
// flags 0 is cudaMallocHost; cudaHostAllocMapped for memory the device reads and writes in place
template <typename T = void> HostPtr<T> make_host(size_t bytes, unsigned flags = cudaHostAllocDefault) {
  void* p = nullptr;
  TDM_CUDA(cudaHostAlloc(&p, bytes, flags));
  return HostPtr<T>(static_cast<T*>(p));
}
inline Event make_event(unsigned flags = cudaEventDefault) { cudaEvent_t e; TDM_CUDA(cudaEventCreateWithFlags(&e, flags)); return Event(e); }
inline Stream make_stream(int priority) {   // non-blocking; priority 0 is the default
  cudaStream_t s;
  TDM_CUDA(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, priority));
  return Stream(s);
}
inline Graph make_graph() { cudaGraph_t g; TDM_CUDA(cudaGraphCreate(&g, 0)); return Graph(g); }
inline GraphExec make_graph_exec(cudaGraph_t g) { cudaGraphExec_t x; TDM_CUDA(cudaGraphInstantiate(&x, g, 0)); return GraphExec(x); }

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// storage <-> fp32 conversion for activation types
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// Load N consecutive channels (N*sizeof(T) must be a multiple of 16 B or N==1) into fp32 registers
// with 128-bit loads.
template <typename T, int N>
__device__ __forceinline__ void load_vec(const T* __restrict__ p, float (&out)[N]) {
  constexpr int BYTES = N * (int)sizeof(T);
  if constexpr (BYTES % 16 == 0) {
    constexpr int NV = BYTES / 16;
    constexpr int PER = 16 / (int)sizeof(T);
    const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      uint4 v = __ldg(q + i);
      const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int j = 0; j < PER; ++j) out[i * PER + j] = to_f<T>(e[j]);
    }
  } else if constexpr (BYTES % 8 == 0) {
    constexpr int NV = BYTES / 8;
    constexpr int PER = 8 / (int)sizeof(T);
    const uint2* q = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      uint2 v = __ldg(q + i);
      const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int j = 0; j < PER; ++j) out[i * PER + j] = to_f<T>(e[j]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) out[i] = to_f<T>(p[i]);
  }
}

template <typename T, int N>
__device__ __forceinline__ void store_vec(T* __restrict__ p, const float (&in)[N]) {
  constexpr int BYTES = N * (int)sizeof(T);
  if constexpr (BYTES % 16 == 0) {
    constexpr int NV = BYTES / 16;
    constexpr int PER = 16 / (int)sizeof(T);
    uint4* q = reinterpret_cast<uint4*>(p);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      uint4 v;
      T* e = reinterpret_cast<T*>(&v);
#pragma unroll
      for (int j = 0; j < PER; ++j) e[j] = from_f<T>(in[i * PER + j]);
      q[i] = v;
    }
  } else if constexpr (BYTES % 8 == 0) {
    constexpr int NV = BYTES / 8;
    constexpr int PER = 8 / (int)sizeof(T);
    uint2* q = reinterpret_cast<uint2*>(p);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      uint2 v;
      T* e = reinterpret_cast<T*>(&v);
#pragma unroll
      for (int j = 0; j < PER; ++j) e[j] = from_f<T>(in[i * PER + j]);
      q[i] = v;
    }
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) p[i] = from_f<T>(in[i]);
  }
}

}  // namespace tdm
