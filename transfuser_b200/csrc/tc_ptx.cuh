// Inline-PTX wrappers for the Hopper (sm_90a) async machinery: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA
// (wgmma.mma_async with register accumulators, wgmma.cuh) and its shared-memory matrix descriptors, plus the register-fragment
// epilogue shared by the tensor-core kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------- mbarrier ----------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// expect `bytes` more transaction bytes in the current phase without arriving (the arrivals come separately)
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 16-byte cp.async global -> shared; src_bytes = 0 writes 16 zero bytes and reads nothing
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrive on bar once this thread's earlier cp.async copies have landed (counted in the barrier's expected arrivals)
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(addr), "r"(parity) : "memory");
}

// ---------------- TMA ----------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------- wgmma ----------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of the accumulator registers across wgmma_fence / wgmma_wait.
template <int K> __device__ __forceinline__ void fence_acc(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// generic-proxy writes to shared memory (st.shared, cp.async) -> visible to wgmma / TMA (async proxy)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Register fragment of a 64 x N wgmma accumulator: element i of thread t (t = thread index in its warpgroup) holds row
// frag_row(t, i) and column frag_col(t, i); elements 2j and 2j + 1 are adjacent columns of the same row.
__device__ __forceinline__ int frag_row(int t, int i) { return (t >> 5) * 16 + ((t & 31) >> 2) + ((i >> 1) & 1) * 8; }
__device__ __forceinline__ int frag_col(int t, int i) { return (i >> 2) * 8 + (t & 3) * 2 + (i & 1); }

// fp32 vector reduction into global memory (sm_90+): four consecutive floats, 16-byte aligned, one L2 transaction per lane instead of 4
__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Epilogue, part 1: columns [32c, 32c + 32) of this warp's 16 accumulator rows (fragment -> padded smem, row stride 36 floats).
// c must be a compile-time constant after unrolling so that the accumulator stays in registers.
template <int K>
__device__ __forceinline__ void frag_to_stage(float* stage, const float (&acc)[K], int c, int lane) {
  const int r = lane >> 2, cc = (lane & 3) * 2;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = c * 4 + jj;
    if (j * 4 < K) {
      *reinterpret_cast<float2*>(stage + r * 36 + jj * 8 + cc) = make_float2(acc[j * 4], acc[j * 4 + 1]);
      *reinterpret_cast<float2*>(stage + (r + 8) * 36 + jj * 8 + cc) = make_float2(acc[j * 4 + 2], acc[j * 4 + 3]);
    }
  }
  __syncwarp();
}

// Eval-mode BatchNorm in the epilogue (tfb_gemm_bf16_tc_bn_eval, tfb_conv3x3_tc_bn_eval): every pointer is pre-offset to the chunk's
// column 0 (res: to the output's base, like out32). o = fma((v - mean) * invstd, gamma, beta) (+ res) (ReLU), v being the value
// the plain launch stores: the same operations, in the same order and without contraction, as bn_apply_kernel (norm.cu).
struct BnEval {
  const float* mean;
  const float* invstd;
  const float* gamma;
  const float* beta;
  const float* res;     // optional residual with the output's layout
  int relu;
};

__device__ __forceinline__ float bn_eval_one(float v, float mu, float is, float ga, float be) {
  return fmaf(__fmul_rn(__fsub_rn(v, mu), is), ga, be);
}

// Epilogue, part 2: one warp writes the 16 x 32 staged block to global memory with COALESCED row segments (4 rows per
// instruction, 128 bytes of fp32 or 64 bytes of bf16 per row), applying o = alpha*acc + bias (ReLU).
// `row_off(row)` returns the ELEMENT offset of staged row `row` (0..15) in the output (a multiple of 4) or -1 for rows that
// must not be written; columns >= cols_valid are not written. The result goes to out32 (fp32) or, when out16 is given, to out16
// (bf16, round-to-nearest-even) at the same element offsets. atomic: the fp32 values are ADDED to out32 (split-K partial tiles).
// stat_sum / stat_sq (optional, this warp's per-tile buffers in SHARED memory, this chunk's column 0): per-column sum and sum of
// squares of the values written (rows with offset -1 contribute nothing) — the training-mode BatchNorm statistics of a conv / GEMM
// output come out of its epilogue instead of a separate read pass over the tensor. They are STORED (each column of a tile belongs
// to one chunk); stat_fold adds the warps' buffers into the CTA's accumulators in warp order, and stat_flush reduces the CTAs in
// CTA order, so the statistics are the same bits on every run.
// BNE (eval-mode BatchNorm, `bne` set): the normalised value goes to out32 AND, when out16 is given, to out16; no atomic, no
// statistics.
template <bool BNE = false, class RowOff>
__device__ __forceinline__ void stage_to_global(const float* stage, RowOff row_off, int cols_valid, const float* bias, float alpha,
                                                int relu, int lane, float* out32, __nv_bfloat16* out16 = nullptr,
                                                float* stat_sum = nullptr, float* stat_sq = nullptr, int atomic = 0,
                                                const BnEval* bne = nullptr) {
  const int c4 = (lane & 7) * 4, rsub = lane >> 3;
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias) {
    bv.x = c4 + 0 < cols_valid ? bias[c4 + 0] : 0.f;
    bv.y = c4 + 1 < cols_valid ? bias[c4 + 1] : 0.f;
    bv.z = c4 + 2 < cols_valid ? bias[c4 + 2] : 0.f;
    bv.w = c4 + 3 < cols_valid ? bias[c4 + 3] : 0.f;
  }
  float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = i * 4 + rsub;
    float4 v = *reinterpret_cast<const float4*>(stage + row * 36 + c4);
    v.x = fmaf(alpha, v.x, bv.x); v.y = fmaf(alpha, v.y, bv.y); v.z = fmaf(alpha, v.z, bv.z); v.w = fmaf(alpha, v.w, bv.w);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    const int64_t off = row_off(row);
    if constexpr (BNE) {
      if (off >= 0) {
        // the per-channel parameters are re-read per row (L1 hits): held across the rows they push the 96-register tiles into spills
        float* vq = &v.x;
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (c4 + q < cols_valid) vq[q] = bn_eval_one(vq[q], bne->mean[c4 + q], bne->invstd[c4 + q], bne->gamma[c4 + q], bne->beta[c4 + q]);
        const bool full = c4 + 3 < cols_valid;
        if (bne->res) {
          const float* r = bne->res + off + c4;
          float4 rv;
          if (full) {
            rv = *reinterpret_cast<const float4*>(r);
          } else {
            rv.x = c4 + 0 < cols_valid ? r[0] : 0.f;
            rv.y = c4 + 1 < cols_valid ? r[1] : 0.f;
            rv.z = c4 + 2 < cols_valid ? r[2] : 0.f;
            rv.w = 0.f;
          }
          v.x = __fadd_rn(v.x, rv.x); v.y = __fadd_rn(v.y, rv.y); v.z = __fadd_rn(v.z, rv.z); v.w = __fadd_rn(v.w, rv.w);
        }
        if (bne->relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        float* p = out32 + off + c4;
        if (full) {
          *reinterpret_cast<float4*>(p) = v;
        } else {
          if (c4 + 0 < cols_valid) p[0] = v.x;
          if (c4 + 1 < cols_valid) p[1] = v.y;
          if (c4 + 2 < cols_valid) p[2] = v.z;
        }
        if (out16) {
          __nv_bfloat16* p16 = out16 + off + c4;
          if (full) {
            __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
            uint2 o;
            o.x = *reinterpret_cast<uint32_t*>(&lo);
            o.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(p16) = o;
          } else {
            if (c4 + 0 < cols_valid) p16[0] = __float2bfloat16_rn(v.x);
            if (c4 + 1 < cols_valid) p16[1] = __float2bfloat16_rn(v.y);
            if (c4 + 2 < cols_valid) p16[2] = __float2bfloat16_rn(v.z);
          }
        }
      }
      continue;
    }
    if (off >= 0) {
      if (stat_sum) {
        s1[0] += v.x; s1[1] += v.y; s1[2] += v.z; s1[3] += v.w;
        s2[0] = fmaf(v.x, v.x, s2[0]); s2[1] = fmaf(v.y, v.y, s2[1]); s2[2] = fmaf(v.z, v.z, s2[2]); s2[3] = fmaf(v.w, v.w, s2[3]);
      }
      if (out16) {
        __nv_bfloat16* p = out16 + off + c4;
        if (c4 + 3 < cols_valid) {
          __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
          uint2 o;
          o.x = *reinterpret_cast<uint32_t*>(&lo);
          o.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(p) = o;
        } else {
          if (c4 + 0 < cols_valid) p[0] = __float2bfloat16_rn(v.x);
          if (c4 + 1 < cols_valid) p[1] = __float2bfloat16_rn(v.y);
          if (c4 + 2 < cols_valid) p[2] = __float2bfloat16_rn(v.z);
        }
      } else {
        float* p = out32 + off + c4;
        if (atomic) {                 // split-K partial tile: one 16-byte vector reduction per lane (coalesced 128-byte row segments)
          if (c4 + 3 < cols_valid) {
            red_add_v4(p, v);
          } else {
            if (c4 + 0 < cols_valid) atomicAdd(p + 0, v.x);
            if (c4 + 1 < cols_valid) atomicAdd(p + 1, v.y);
            if (c4 + 2 < cols_valid) atomicAdd(p + 2, v.z);
          }
        } else if (c4 + 3 < cols_valid) {
          *reinterpret_cast<float4*>(p) = v;
        } else {
          if (c4 + 0 < cols_valid) p[0] = v.x;
          if (c4 + 1 < cols_valid) p[1] = v.y;
          if (c4 + 2 < cols_valid) p[2] = v.z;
        }
      }
    }
  }
  if (stat_sum) {   // warp-uniform: lanes with equal (lane & 7) hold the same 4 columns for different rows
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      s1[q] += __shfl_xor_sync(0xffffffffu, s1[q], 8);  s2[q] += __shfl_xor_sync(0xffffffffu, s2[q], 8);
      s1[q] += __shfl_xor_sync(0xffffffffu, s1[q], 16); s2[q] += __shfl_xor_sync(0xffffffffu, s2[q], 16);
    }
    if (lane < 8) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (c4 + q < cols_valid) { stat_sum[c4 + q] = s1[q]; stat_sq[c4 + q] = s2[q]; }
    }
  }
  __syncwarp();
}

// Deterministic per-column statistics. The consumer warps (kConsumers threads, named barrier 1) own
//   s_stat[2][n]          the CTA's accumulators (shared), cleared by stat_clear,
//   wstat[8][2][kStatW]   one per-tile buffer per consumer warp (shared), written by stage_to_global.
// stat_fold adds columns [0, ncols) of the eight warp buffers, in warp order, into s_stat + col0 (and s_stat + n + col0);
// stat_flush writes the CTA's accumulators to its row of ws[gridDim.x][2n] and the last CTA to arrive (counter *cnt, zero on
// entry, reset on exit) adds the rows in CTA order, in fp64, into stats[2][n] (global: [sum | sum of squares]).
// t = thread index among the consumer threads.
constexpr int kConsumers = 256;
constexpr int kStatW = 256;                    // widest tile
__device__ __forceinline__ void stat_clear(float* s_stat, int n, int t) {
  for (int i = t; i < 2 * n; i += kConsumers) s_stat[i] = 0.f;
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
}
__device__ __forceinline__ void stat_fold(float* s_stat, const float* wstat, int n, int col0, int ncols, int t) {
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  for (int j = t; j < 2 * ncols; j += kConsumers) {
    const int q = j / ncols, c = j - q * ncols;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += wstat[(w * 2 + q) * kStatW + c];
    s_stat[q * n + col0 + c] += s;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
}
// The columns form blocks (a GEMM tile's columns, a conv tile's channel block) and each of the `total` tiles of the persistent grid
// (tile = blockIdx.x + k * gridDim.x) lies in one block: blk(tile). Block g has tpb tiles, tile(g, i) for i < tpb, and the
// columns [cols(g).x, cols(g).x + cols(g).y). cnt holds one counter per block: each CTA adds one per tile it ran, and the CTA that
// brings block g's counter to tpb folds block g's columns over the CTAs that ran one of its tiles, in CTA order (the other CTAs'
// rows are +0 for these columns and are skipped). So the folds of different blocks run in different CTAs, in parallel.
constexpr int kMaxStatGrid = 1024;
template <class Blk, class Tile, class Cols>
__device__ __forceinline__ void stat_flush(const float* s_stat, double* stats, int n, int t, float* ws, unsigned int* cnt, int total, int tpb,
                                           Blk blk, Tile tile, Cols cols) {
  __shared__ unsigned int s_last[2], s_contrib[kMaxStatGrid / 32];   // s_last by tile parity: written again only two barriers later
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  for (int i = t; i < 2 * n; i += kConsumers) ws[(int64_t)blockIdx.x * 2 * n + i] = s_stat[i];
  __threadfence();
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  for (int k = blockIdx.x, p = 0; k < total; k += gridDim.x, p ^= 1) {
    const int g = blk(k);
    if (t == 0) s_last[p] = atomicAdd(cnt + g, 1u) == (unsigned int)(tpb - 1);
    for (int w = t; w < kMaxStatGrid / 32; w += kConsumers) s_contrib[w] = 0u;
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
    if (!s_last[p]) continue;        // block-uniform
    __threadfence();
    for (int i = t; i < tpb; i += kConsumers) {
      const int b = tile(g, i) % gridDim.x;
      atomicOr(&s_contrib[b >> 5], 1u << (b & 31));
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
    const int2 c = cols(g);
    auto take = [&](int b) { return (s_contrib[b >> 5] >> (b & 31)) & 1u; };
    if ((n & 3) == 0) {              // then c.x and c.y are multiples of 4 too
      const int gq = c.y / 4;
      ordered_fold<double, 4>(ws, 2 * n, (int)gridDim.x, 2 * gq, [&](int64_t j) { return (int64_t)(j / gq) * n + c.x + (j % gq) * 4; }, take,
                              [&](int64_t j, const double (&s)[4]) {
                                double* o = stats + (j / gq) * n + c.x + (j % gq) * 4;
#pragma unroll
                                for (int v = 0; v < 4; ++v) o[v] += s[v];
                              }, t, kConsumers);
    } else {
      ordered_fold<double, 1>(ws, 2 * n, (int)gridDim.x, 2 * c.y, [&](int64_t j) { return (int64_t)(j / c.y) * n + c.x + j % c.y; }, take,
                              [&](int64_t j, const double (&s)[1]) { stats[(j / c.y) * n + c.x + j % c.y] += s[0]; }, t, kConsumers);
    }
    if (t == 0) cnt[g] = 0u;         // the stream's scratch counters are zero on entry
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory");
  }
}

// ---------------- descriptors ----------------
// wgmma shared-memory matrix descriptor (sm_90): start address, leading / stride byte offsets (>> 4), swizzle mode in bits 62-63
// (1 = 128B, 2 = 64B, 3 = 32B); stage buffers are 1024-byte aligned, so the base-offset field stays 0.
//   K-major operand : rows of 128 B (64 B for SWIZZLE_64B), 8-row groups SBO bytes apart; LBO unused (1)
//   MN-major operand: 128 B of MN-contiguous elements per K row, 8-row K groups 1024 B apart (SBO), next 128 B MN chunk at LBO
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, int swizzle_bytes = 128) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(swizzle_bytes == 128 ? 1 : swizzle_bytes == 64 ? 2 : 3) << 62;
  return d;
}

}  // namespace tc
