// TEST INFRASTRUCTURE ONLY. A minimal host emulation of the CUDA execution model, enough to run the SIMT (non-tensor-core)
// kernels of transfuser_b200/csrc *unchanged* on the CPU in the build container, where there is no GPU: one OS thread per CUDA
// thread of a block (threads are reused across the blocks of a launch, blocks run one after another), __syncthreads() = a
// barrier that threads which already left the kernel no longer take part in, warp shuffles through a per-warp barrier,
// __shared__ = a static, kernel<<<grid, block, smem, stream>>>(...) rewritten to emul_launch(...) by tests/cuda_emul/build_emul.py.
// The .cu files see this header through the stand-in <cuda_runtime.h> / <cuda_bf16.h> next to it, so csrc/common.cuh and the
// C-ABI entry points compile as they are. It checks indexing / control flow / arithmetic of the kernel source; it says nothing
// about performance, memory-model races between blocks, or the device compiler.
#pragma once
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <barrier>
#include <cmath>
#include <new>
#include <thread>
#include <vector>

struct uint3_ { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) double2 { double x, y; };
struct alignas(8) uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
static inline uint2 make_uint2(uint32_t a, uint32_t b) { return uint2{a, b}; }
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }

// bf16 storage type with round-to-nearest-even conversion (NaN kept quiet), as cuda_bf16.h's __float2bfloat16_rn
struct __nv_bfloat16 { uint16_t bits; };
struct alignas(4) __nv_bfloat162 { __nv_bfloat16 x, y; };
static inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return __nv_bfloat16{(uint16_t)0x7fff};
  u += 0x7fffu + ((u >> 16) & 1u);
  return __nv_bfloat16{(uint16_t)(u >> 16)};
}
static inline __nv_bfloat16 __float2bfloat16(float f) { return __float2bfloat16_rn(f); }
static inline float __bfloat162float(__nv_bfloat16 h) { uint32_t u = (uint32_t)h.bits << 16; float f; memcpy(&f, &u, 4); return f; }
static inline __nv_bfloat162 __floats2bfloat162_rn(float a, float b) { return __nv_bfloat162{__float2bfloat16_rn(a), __float2bfloat16_rn(b)}; }

typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0 };
enum { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
enum cudaStreamCaptureMode { cudaStreamCaptureModeGlobal = 0, cudaStreamCaptureModeThreadLocal = 1, cudaStreamCaptureModeRelaxed = 2 };
static inline cudaError_t cudaThreadExchangeStreamCaptureMode(cudaStreamCaptureMode*) { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 2; return cudaSuccess; }   // "2 SMs": keeps grid-stride grids small

static thread_local uint3_ threadIdx, blockIdx;
static thread_local dim3 blockDim, gridDim;
alignas(64) static unsigned char emul_sync_mem[sizeof(std::barrier<>)];
alignas(64) static unsigned char emul_warp_mem[32][sizeof(std::barrier<>)];
static inline std::barrier<>& emul_sync_bar() { return *reinterpret_cast<std::barrier<>*>(emul_sync_mem); }
static inline std::barrier<>& emul_warp_bar(unsigned w) { return *reinterpret_cast<std::barrier<>*>(emul_warp_mem[w]); }
static inline unsigned emul_tid() { return threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z); }

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __constant__ static const
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__

static inline void __syncthreads() { emul_sync_bar().arrive_and_wait(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emul_warp_bar(emul_tid() >> 5).arrive_and_wait(); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T> static inline T __ldg(const T* p) { return *p; }
template <typename T> static inline T __ldcg(const T* p) { return *p; }
static float emul_shfl[1024];
static inline float __shfl_xor_sync(unsigned, float v, int lane_mask) {
  const unsigned t = emul_tid(), n = blockDim.x * blockDim.y * blockDim.z;
  emul_shfl[t] = v;
  emul_warp_bar(t >> 5).arrive_and_wait();
  const unsigned src = (t & ~31u) | ((t & 31u) ^ (unsigned)lane_mask);
  const float r = src < n ? emul_shfl[src] : v;
  emul_warp_bar(t >> 5).arrive_and_wait();
  return r;
}
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <typename T, typename U> static inline T emul_atomic_fadd(T* p, T v) {
  U* ip = reinterpret_cast<U*>(p);
  U old = __atomic_load_n(ip, __ATOMIC_RELAXED), want;
  T f;
  do {
    memcpy(&f, &old, sizeof(T));
    f += v;
    memcpy(&want, &f, sizeof(T));
  } while (!__atomic_compare_exchange_n(ip, &old, want, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
  memcpy(&f, &old, sizeof(T));
  return f;
}
static inline float atomicAdd(float* p, float v) { return emul_atomic_fadd<float, uint32_t>(p, v); }
static inline double atomicAdd(double* p, double v) { return emul_atomic_fadd<double, uint64_t>(p, v); }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float rsqrtf(float v) { return 1.0f / sqrtf(v); }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline int64_t min(int64_t a, int64_t b) { return a < b ? a : b; }
static inline int64_t max(int64_t a, int64_t b) { return a > b ? a : b; }
using std::floor;
using std::fma;
using std::fmax;
using std::fmin;
using std::pow;
using std::sqrt;

template <typename F>
static void emul_launch(dim3 grid, dim3 block, F kernel) {
  const unsigned nt = block.x * block.y * block.z, nwarps = (nt + 31) / 32;
  if (nt == 0 || nt > 1024 || grid.x * grid.y * grid.z == 0) { fprintf(stderr, "emul_launch: bad configuration\n"); return; }
  pthread_barrier_t gate;
  pthread_barrier_init(&gate, nullptr, nt);
  std::vector<std::thread> ts;
  ts.reserve(nt);
  for (unsigned t = 0; t < nt; ++t)
    ts.emplace_back([=, &gate]() {
      threadIdx = uint3_{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
      blockDim = block;
      gridDim = grid;
      for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
          for (unsigned bx = 0; bx < grid.x; ++bx) {
            pthread_barrier_wait(&gate);                       // everyone has left the previous block
            if (t == 0) {
              new (emul_sync_mem) std::barrier<>(nt);
              for (unsigned w = 0; w < nwarps; ++w) new (emul_warp_mem[w]) std::barrier<>(w + 1 < nwarps ? 32 : nt - 32 * w);
            }
            pthread_barrier_wait(&gate);
            blockIdx = uint3_{bx, by, bz};
            kernel();
            emul_sync_bar().arrive_and_drop();                 // a finished thread no longer counts in __syncthreads()
            emul_warp_bar(t >> 5).arrive_and_drop();
          }
    });
  for (auto& th : ts) th.join();
  pthread_barrier_destroy(&gate);
}
