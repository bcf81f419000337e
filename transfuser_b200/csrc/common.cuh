// Shared helpers for the transfuser_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "tfb200.h"  // the C-ABI: every TFB_API definition is checked against its declaration

#define TFB_API TFB_EXPORT

// Returns TFB_ERR_LAUNCH if the preceding launch failed (no device sync: current-stream semantics).
#define TFB_CHECK_LAUNCH()                                        \
  do {                                                            \
    cudaError_t e__ = cudaGetLastError();                         \
    if (e__ != cudaSuccess) { tfb_set_last_error(cudaGetErrorString(e__)); return TFB_ERR_LAUNCH; } \
  } while (0)

#define TFB_REQUIRE(cond)                                         \
  do { if (!(cond)) { tfb_set_last_error("argument check failed: " #cond); return TFB_ERR_ARG; } } while (0)

void tfb_set_last_error(const char* msg);

static inline int tfb_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Per-stream scratch of the fixed-order reductions across CTAs: `floats` fp32 values and `counters` unsigned ints. Counters are
// ZERO on entry: every kernel that takes a ticket resets it before it returns. The buffers persist and are shared by all launches
// on the stream (they run one after another); they only grow, and a grown-out buffer is kept, because a captured CUDA graph goes on
// using the address it was captured with. Defined in api.cu.
struct TfbScratch {
  float* f = nullptr;
  unsigned int* cnt = nullptr;
};
int tfb_scratch(TfbScratch& w, size_t floats, size_t counters, cudaStream_t s);

// Grid for a grid-stride elementwise kernel: enough CTAs to fill the chip a few times, never more than needed.
static inline int tfb_grid(int64_t n, int threads, int waves = 8) {
  int64_t need = ceil_div64(n, threads);
  int64_t cap = (int64_t)tfb_num_sms() * waves;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum; `red` must hold >= 32 floats. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) { r = warp_sum(r); if (lane == 0) red[0] = r; }
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) { r = warp_max(r); if (lane == 0) red[0] = r; }
  __syncthreads();
  return red[0];
}

// Stores four fp32 values as four bf16 (round-to-nearest-even) with one 8-byte access: the "bf16 sidecar" that producers of a
// tensor-core operand write next to their fp32 output, so the consumer needs no separate cast pass. `dst + i4*4` must be 8-byte aligned.
__device__ __forceinline__ void tfb_store_bf16x4(__nv_bfloat16* dst, int64_t i4, float a, float b, float c, float d) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
  uint2 o;
  o.x = *reinterpret_cast<uint32_t*>(&lo);
  o.y = *reinterpret_cast<uint32_t*>(&hi);
  reinterpret_cast<uint2*>(dst)[i4] = o;
}

// The fold of every fixed-order cross-CTA sum. For each group g in [0, ngroups) of V consecutive outputs (partials at
// part + off(g), V-aligned), the rows r in [0, nrows) with take(r) are added in row order, starting from +0 in the accumulator type
// Acc, and emit(g, sum) receives the V sums. Rows with !take(r) are not read and count as +0: a fold that starts at +0 never
// becomes -0, so they do not change the bits. Thread t of nthr takes groups t, t + nthr, ...; each thread loads kFoldBatch rows
// (V * sizeof(P) bytes each, 16 with V = 16 / sizeof(P)) before it adds them, so the loads of a batch are in flight together.
constexpr int kFoldBatch = 8;
template <typename P, int V> struct FoldVec;
template <> struct FoldVec<float, 1> { typedef float T; };
template <> struct FoldVec<float, 4> { typedef float4 T; };
template <> struct FoldVec<double, 1> { typedef double T; };
template <> struct FoldVec<double, 2> { typedef double2 T; };
template <typename Acc, int V, typename P, class Off, class Take, class Emit>
__device__ __forceinline__ void ordered_fold(const P* part, int64_t row_stride, int nrows, int64_t ngroups, Off off, Take take, Emit emit,
                                             int t, int nthr) {
  typedef typename FoldVec<P, V>::T Vec;
  for (int64_t g = t; g < ngroups; g += nthr) {
    const P* p = part + off(g);
    Acc s[V];
#pragma unroll
    for (int v = 0; v < V; ++v) s[v] = Acc(0);
    for (int r0 = 0; r0 < nrows; r0 += kFoldBatch) {
      P x[kFoldBatch][V];
#pragma unroll
      for (int b = 0; b < kFoldBatch; ++b) {
        const int r = r0 + b;
        if (r < nrows && take(r)) {
          const Vec q = __ldcg(reinterpret_cast<const Vec*>(p + (int64_t)r * row_stride));
          memcpy(x[b], &q, sizeof(Vec));
        } else {
#pragma unroll
          for (int v = 0; v < V; ++v) x[b][v] = P(0);
        }
      }
#pragma unroll
      for (int b = 0; b < kFoldBatch; ++b)
#pragma unroll
        for (int v = 0; v < V; ++v) s[v] += (Acc)x[b][v];
    }
    emit(g, s);
  }
}

// Cross-block sums that give the same bits on every run. Every output index i in [0, n_out) gets exactly one contribution from
// each split s in [0, nsplit) (ordered_store); the last block of the grid to finish (ordered_finish, called by every thread of
// every block) adds, for each i, the contributions in split order to out[i]. part / cnt: nsplit * n_out floats and one counter
// of the stream's scratch (TfbScratch).
struct OrderedSum {
  float* part;
  unsigned int* cnt;
  int nsplit;
  int64_t n_out;
};
static __device__ __forceinline__ void ordered_store(const OrderedSum& o, int split, int64_t i, float v) { o.part[(int64_t)split * o.n_out + i] = v; }
// out[i] (+)= the fold of part[0..nsplit)[i] for i in [0, n_out), by thread t of nthr; 16-byte loads when n_out % 4 == 0.
static __device__ __forceinline__ void ordered_sum_range(const float* part, int nsplit, int64_t n_out, float* out, bool assign, int t, int nthr) {
  auto all = [](int) { return true; };
  if (n_out % 4 == 0 && (reinterpret_cast<uintptr_t>(part) & 15) == 0) {
    ordered_fold<float, 4>(part, n_out, nsplit, n_out / 4, [](int64_t g) { return g * 4; }, all, [&](int64_t g, const float (&s)[4]) {
#pragma unroll
      for (int v = 0; v < 4; ++v) out[g * 4 + v] = (assign ? 0.f : out[g * 4 + v]) + s[v];
    }, t, nthr);
  } else {
    ordered_fold<float, 1>(part, n_out, nsplit, n_out, [](int64_t g) { return g; }, all, [&](int64_t g, const float (&s)[1]) {
      out[g] = (assign ? 0.f : out[g]) + s[0];
    }, t, nthr);
  }
}
static __device__ __forceinline__ void ordered_finish(const OrderedSum& o, float* out) {
  if (!o.cnt) return;                 // summed by ordered_sum_kernel after the launch instead (large n_out)
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  const int tid = (threadIdx.z * blockDim.y + threadIdx.y) * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y * blockDim.z;
  if (tid == 0) last = atomicAdd(o.cnt, 1u) == gridDim.x * gridDim.y * gridDim.z - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  ordered_sum_range(o.part, o.nsplit, o.n_out, out, false, tid, nthr);
  if (tid == 0) *o.cnt = 0u;
}
// out[i] += sum over splits k (in order) of part[k][i] (assign: out[i] = +0 + that sum): the last step of an OrderedSum whose n_out
// is too large for one CTA (launched after the kernel that stored the partials, with o.cnt = nullptr there).
static __global__ void __launch_bounds__(256) ordered_sum_kernel(const float* __restrict__ part, int nsplit, int64_t n_out, float* __restrict__ out,
                                                                 bool assign = false) {
  ordered_sum_range(part, nsplit, n_out, out, assign, (int)(blockIdx.x * blockDim.x + threadIdx.x), (int)(gridDim.x * blockDim.x));
}

static inline int ordered_alloc(OrderedSum& o, int nsplit, int64_t n_out, cudaStream_t s) {
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)nsplit * n_out, 1, s);
  o.part = w.f; o.cnt = w.cnt; o.nsplit = nsplit; o.n_out = n_out;
  return rc;
}

// Counter-based RNG for dropout: one 32-bit hash per (seed, element index); regenerated in backward, no mask storage.
__device__ __forceinline__ uint32_t tfb_hash32(uint64_t seed, uint64_t idx) {
  uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (uint32_t)(z >> 32);
}
// keep-scale for dropout probability p: 0 when dropped, 1/(1-p) when kept.
__device__ __forceinline__ float tfb_dropout_scale(uint64_t seed, uint64_t idx, float p) {
  if (p <= 0.f) return 1.f;
  float u = (float)(tfb_hash32(seed, idx) >> 8) * (1.0f / 16777216.0f);
  return u < p ? 0.f : 1.f / (1.f - p);
}
