// Fused multi-head self-attention on the wgmma tensor cores (forward and backward) for the GPT fusion blocks
// (reference: SelfAttention.forward, transfuser.py:510-527: q k^T / sqrt(hs) -> softmax -> attn_drop -> @ v; T = 174 tokens,
// 4 heads, head sizes 18 / 54 / 144 / 378). Nothing of size T x T ever reaches HBM: scores live in the wgmma register
// accumulators, probabilities go through shared memory as the bf16 A operand of the second product.
//
// One CTA = one 128-row tile of one (batch, head); warpgroup g (threads 128g..128g+127) owns rows [64g, 64g + 64).
// Three modes share the kernel body:
//   FWD   rows = queries : S = Q K^T (registers, all 192 columns) -> P = softmax(scale S), Pd = dropout(P) (bf16, smem) -> O = Pd V ;
//                          saves the row log-sum-exp for the backward pass
//   BWD_Q rows = queries : S = Q K^T, dPd = dO V^T -> dS = scale P (dPd drop - D) (smem) -> dQ = dS K
//   BWD_K rows = keys    : S^T = K Q^T, dPd^T = V dO^T -> Pd^T and dS^T (smem) -> dV = Pd^T dO ; dK = dS^T Q
// (P is recomputed from the saved log-sum-exp; D_i = sum_d dO_id O_id comes from a small pre-pass.) The backward score products
// run in two 96-column halves so that both accumulators fit the register file.
// Operands are staged by all threads into 128B-swizzled shared memory (the head slices of the packed [B*T, 3C] q|k|v buffer
// start at 4-byte-aligned columns, which rules out TMA boxes) and described to wgmma with the same K-major / MN-major
// shared-memory descriptors as gemm_tc.cu. fp32 or bf16 inputs (converted while staging), fp32 accumulation.
#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRowsX = 128;                 // tile rows (two wgmma M = 64 halves)
constexpr int kRowsY = 192;                 // padded rows of the column operand (T <= 192)
constexpr int kHalf = 96;                   // score columns per backward pass
constexpr int kXBytes = kRowsX * 128;       // one 64-column bf16 chunk of the row operand
constexpr int kYBytes = kRowsY * 128;       // one 64-column bf16 chunk of the column operand
constexpr int kYHalfBytes = kHalf * 128;
// one streaming stage: X1 | Y1 (FWD: 192 rows, BWD: 96 rows) | X2 | Y2 (BWD only)
constexpr int kOffY1 = kXBytes, kOffX2 = kXBytes + kYHalfBytes, kOffY2 = 2 * kXBytes + kYHalfBytes;
constexpr int kStageBytes = 2 * (kXBytes + kYHalfBytes);         // 57344 (>= kXBytes + kYBytes of the forward stage)
constexpr int kMatBytes = 3 * kXBytes;      // the 128 x 192 bf16 probability / score-gradient matrix (3 K chunks of 64)
constexpr int kZBuf = 2 * kYBytes;          // two 64-wide chunks of the MN-major B operand of the second product
constexpr int kSmemStages = 2 * kStageBytes;                     // two streaming stages; later two Z buffers
constexpr int kSmemTotal = kSmemStages + 2 * kMatBytes + 2 * kRowsY * 4 + 1024;  // + Pd^T / dS^T (BWD_K) + column statistics + slack
static_assert(kXBytes + kYBytes <= kStageBytes && 2 * kZBuf <= kSmemStages, "attention shared-memory layout");

enum { MODE_FWD = 0, MODE_BWD_Q = 1, MODE_BWD_K = 2 };

struct Params {
  const void* qkv;      // [B*T, 3C] q | k | v
  const void* dy;       // [B*T, C]  dO (backward)
  float* out32_a;       // FWD: y [B*T, C]; BWD: dqkv [B*T, 3C]   (fp32, may be null)
  __nv_bfloat16* out16_a;  // same, bf16 (may be null)
  float* lse;           // [B, nh, T]
  const float* dsum;    // [B, nh, T]  D (backward)
  const uint64_t* seed_dev;
  uint64_t seed_off;
  int B, T, nh, hs, C;
  int in_bf16, dy_bf16;
  float scale, p_drop;
  int mode;             // MODE_FWD, or 1 = backward (BWD_K CTAs first, then BWD_Q)
};

// cheap counter-based keep/drop decision for the attention dropout (forward and backward of THIS kernel regenerate it)
__device__ __forceinline__ float drop_scale(uint32_t seed_lo, uint32_t seed_hi, uint32_t idx, float p, float keep_scale) {
  uint32_t x = idx * 0x9E3779B1u + seed_lo;
  x ^= x >> 16; x *= 0x85EBCA6Bu;
  x ^= seed_hi;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  x ^= x >> 16;
  const float u = (float)(x >> 8) * (1.0f / 16777216.0f);
  return u < p ? 0.f : keep_scale;
}

// Stages rows [row0, row0 + rows_pad) x columns [col0, col0 + 64) of a row-major matrix (leading dimension ld elements) as one
// 64-column bf16 chunk in the SWIZZLE_128B layout: row r at (r / 8) * 1024 + (r % 8) * 128, 16-byte unit u at (u ^ (r % 8)) * 16.
// Rows >= rows_valid and columns >= cols_valid are zero-filled. cols_valid and col0 are even.
template <typename TIn>
__device__ __forceinline__ void stage_chunk(uint8_t* dst, const TIn* __restrict__ src, int64_t ld, int64_t row0, int rows_valid,
                                            int rows_pad, int col0, int cols_valid, int tid, int nthreads) {
  for (int idx = tid; idx < rows_pad * 8; idx += nthreads) {
    const int r = idx >> 3, u = idx & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    const int c = u * 8;
    if (r < rows_valid && c < cols_valid) {
      const TIn* p = src + (row0 + r) * ld + col0 + c;
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (c + 2 * j < cols_valid) {
          if (sizeof(TIn) == 4) {
            const float2 f = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p) + 2 * j);
            __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
            w[j] = *reinterpret_cast<uint32_t*>(&b);
          } else {
            w[j] = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const __nv_bfloat16*>(p) + 2 * j);
          }
        } else {
          w[j] = 0u;
        }
      }
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    *reinterpret_cast<uint4*>(dst + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4)) = v;
  }
}

// bf16 source: the same chunk through cp.async (global -> shared without registers, many copies in flight per thread; the copies
// of one call are NOT waited for here — cp_async_wait_all() before the proxy fence). VEC = bytes per copy (16 / 8 / 4): the largest
// power of two that divides the source addresses (the head slices of the packed q|k|v rows are only 4-byte aligned in general).
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int VEC>
__device__ __forceinline__ void stage_chunk_async(uint8_t* dst, const __nv_bfloat16* __restrict__ src, int64_t ld, int64_t row0,
                                                  int rows_valid, int rows_pad, int col0, int cols_valid, int tid, int nthreads) {
  constexpr int PIECES = 16 / VEC, EPP = VEC / 2;      // copies per 16-byte unit, elements per copy
  for (int idx = tid; idx < rows_pad * 8; idx += nthreads) {
    const int r = idx >> 3, u = idx & 7;
    uint8_t* d = dst + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4);
    const int c = u * 8;
    if (r < rows_valid && c < cols_valid) {
      const __nv_bfloat16* p = src + (row0 + r) * ld + col0 + c;
#pragma unroll
      for (int j = 0; j < PIECES; ++j) {
        if (c + (j + 1) * EPP <= cols_valid) {
          const uint32_t da = tc::smem_u32(d + j * VEC);
          if (VEC == 16)     asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(da), "l"(p + j * EPP) : "memory");
          else if (VEC == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(da), "l"(p + j * EPP) : "memory");
          else               asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(da), "l"(p + j * EPP) : "memory");
        } else {                                       // partially valid copy (VEC > 4 only): element pairs, the rest zero
#pragma unroll
          for (int e = 0; e < EPP; e += 2) {
            uint32_t w = 0u;
            if (c + j * EPP + e < cols_valid) w = *reinterpret_cast<const uint32_t*>(p + j * EPP + e);
            *reinterpret_cast<uint32_t*>(d + j * VEC + e * 2) = w;
          }
        }
      }
    } else {
      *reinterpret_cast<uint4*>(d) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

// Issues the staging of one chunk; bf16 sources are asynchronous (see above), fp32 sources are converted synchronously.
__device__ __forceinline__ void stage_any(uint8_t* dst, const void* src, int is_bf16, int64_t ld, int64_t row0, int rows_valid,
                                          int rows_pad, int col0, int cols_valid, int tid, int nthreads) {
  if (is_bf16) {
    const __nv_bfloat16* s16 = (const __nv_bfloat16*)src;
    const uintptr_t a = reinterpret_cast<uintptr_t>(s16 + col0) | (uintptr_t)(ld * 2);
    if ((a & 15) == 0)     stage_chunk_async<16>(dst, s16, ld, row0, rows_valid, rows_pad, col0, cols_valid, tid, nthreads);
    else if ((a & 7) == 0) stage_chunk_async<8>(dst, s16, ld, row0, rows_valid, rows_pad, col0, cols_valid, tid, nthreads);
    else                   stage_chunk_async<4>(dst, s16, ld, row0, rows_valid, rows_pad, col0, cols_valid, tid, nthreads);
  } else {
    stage_chunk<float>(dst, (const float*)src, ld, row0, rows_valid, rows_pad, col0, cols_valid, tid, nthreads);
  }
}

// byte offset of element (row r, column j) of the 128 x 192 K-major bf16 matrix (3 chunks of 64 columns)
__device__ __forceinline__ uint32_t mat_off(int r, int j) {
  const int c = j >> 6, u = (j & 63) >> 3, e = j & 7;
  return (uint32_t)(c * kXBytes + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4) + e * 2);
}

struct Operand {          // a head slice: columns [col, col + hs) of a row-major matrix
  const void* src;
  int bf16;
  int64_t ld;
  int col;
};

// acc1 (+)= X1 Y1^T and, when TWO, acc2 (+)= X2 Y2^T over the head dimension, streamed in 64-wide chunks through two stages:
// X rows [xrow0, xrow0 + 128) (valid: xrows), Y rows [yrow0, yrow0 + NP) (valid: yrows), both K-major.
template <int NP, bool TWO>
__device__ __forceinline__ void score_products(uint8_t* smem, const Operand& x1, const Operand& y1, const Operand& x2, const Operand& y2,
                                               int64_t xrow0, int xrows, int64_t yrow0, int yrows, int hs, int tid, int wg,
                                               float (&acc1)[NP / 2], float (&acc2)[NP / 2]) {
  const int nchunks = (hs + 63) / 64;
  auto issue_loads = [&](int c) {
    uint8_t* st = smem + (c & 1) * kStageBytes;
    const int cv = min(64, hs - c * 64);
    stage_any(st, x1.src, x1.bf16, x1.ld, xrow0, xrows, kRowsX, x1.col + c * 64, cv, tid, kThreads);
    stage_any(st + kOffY1, y1.src, y1.bf16, y1.ld, yrow0, yrows, NP, y1.col + c * 64, cv, tid, kThreads);
    if (TWO) {
      stage_any(st + kOffX2, x2.src, x2.bf16, x2.ld, xrow0, xrows, kRowsX, x2.col + c * 64, cv, tid, kThreads);
      stage_any(st + kOffY2, y2.src, y2.bf16, y2.ld, yrow0, yrows, NP, y2.col + c * 64, cv, tid, kThreads);
    }
    cp_async_commit();
  };
  __syncthreads();                                      // the stages may still be read by the other warpgroup's last MMAs
  issue_loads(0);
  for (int c = 0; c < nchunks; ++c) {
    cp_async_wait_all();
    tc::fence_async_smem();
    __syncthreads();                                    // chunk c staged; both warpgroups' MMAs of chunk c - 1 have retired
    const uint32_t st = tc::smem_u32(smem + (c & 1) * kStageBytes);
    const int ksteps = (min(64, hs - c * 64) + 15) / 16;
    tc::fence_acc(acc1);
    if (TWO) tc::fence_acc(acc2);
    tc::wgmma_fence();
    for (int k = 0; k < ksteps; ++k) {
      const uint32_t accum = (c > 0 || k > 0) ? 1u : 0u;
      tc::wgmma_bf16<0, 0>(acc1, tc::make_smem_desc(st + wg * 8192 + k * 32, 16, 1024), tc::make_smem_desc(st + kOffY1 + k * 32, 16, 1024), accum);
      if (TWO)
        tc::wgmma_bf16<0, 0>(acc2, tc::make_smem_desc(st + kOffX2 + wg * 8192 + k * 32, 16, 1024),
                             tc::make_smem_desc(st + kOffY2 + k * 32, 16, 1024), accum);
    }
    tc::wgmma_commit();
    if (c + 1 < nchunks) issue_loads(c + 1);            // into the stage of chunk c - 1 (retired): overlaps the MMAs of chunk c
    tc::wgmma_wait<0>();
    tc::fence_acc(acc1);
    if (TWO) tc::fence_acc(acc2);
  }
}

// out[64 rows of this warpgroup x NM] = M Z over K = ncols tokens: M (bf16, K-major, 3 chunks of 64 tokens) from the
// element-wise stage, Z (MN-major: token rows x head-dimension columns, two 64-wide chunks). Columns d < dvalid of the rows
// with row_ok are scaled by mul[] and written to o32 / o16 (row stride old).
template <int NM>
__device__ __forceinline__ void value_product(const uint8_t* mat, const uint8_t* zb, int ncols, int wg, int t128, const bool (&row_ok)[2],
                                              const int64_t (&orow)[2], const float (&mul)[2], int dvalid, float* o32, __nv_bfloat16* o16) {
  float o[NM / 2];
  tc::fence_acc(o);
  tc::wgmma_fence();
  const uint32_t sm = tc::smem_u32(mat) + wg * 8192, sz = tc::smem_u32(zb);
  for (int k = 0; k < ncols / 16; ++k)
    tc::wgmma_bf16<0, 1>(o, tc::make_smem_desc(sm + (k >> 2) * kXBytes + (k & 3) * 32, 16, 1024), tc::make_smem_desc(sz + k * 2048, kYBytes, 1024),
                         k > 0 ? 1u : 0u);
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::fence_acc(o);
#pragma unroll
  for (int i = 0; i < NM / 2; i += 2) {
    const int h = (i >> 1) & 1, d = tc::frag_col(t128, i);
    if (row_ok[h] && d < dvalid) {                      // (dvalid is even)
      const float a = o[i] * mul[h], b = o[i + 1] * mul[h];
      if (o32) *reinterpret_cast<float2*>(o32 + orow[h] + d) = make_float2(a, b);
      if (o16) *reinterpret_cast<__nv_bfloat162*>(o16 + orow[h] + d) = __floats2bfloat162_rn(a, b);
    }
  }
}

__device__ __forceinline__ void store_pair(uint8_t* mat, int r, int j, float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  *reinterpret_cast<__nv_bfloat162*>(mat + mat_off(r, j)) = v;
}

__global__ void __launch_bounds__(kThreads, 1) attn_tc_kernel(const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* mat0 = smem + kSmemStages;                    // Pd (FWD) / dS (BWD_Q) / Pd^T (BWD_K)
  uint8_t* mat1 = mat0 + kMatBytes;                      // dS^T (BWD_K)
  float* stat_a = reinterpret_cast<float*>(mat1 + kMatBytes);   // [192] lse of the column tokens (BWD_K)
  float* stat_b = stat_a + kRowsY;                               // [192] D   of the column tokens (BWD_K)

  const int tid = threadIdx.x, wg = tid >> 7, t128 = tid & 127;
  const int T = p.T, nh = p.nh, hs = p.hs, C = p.C;
  const int tiles = (T + kRowsX - 1) / kRowsX;
  int blk = blockIdx.x, mode = MODE_FWD;
  if (p.mode != MODE_FWD) {
    const int half = p.B * nh * tiles;
    mode = blk < half ? MODE_BWD_K : MODE_BWD_Q;
    if (blk >= half) blk -= half;
  }
  const int tile = blk % tiles, bh = blk / tiles, h = bh % nh, b = bh / nh;
  const int m0 = tile * kRowsX;
  const int rows_valid = min(kRowsX, T - m0);
  const int ncols = (T + 15) & ~15;                     // K extent of the second product
  const int64_t tok0 = (int64_t)b * T;                  // first token row of this batch element
  const int64_t ld3 = 3 * (int64_t)C;

  // column offsets (elements) of the operands inside their matrices
  const int colq = h * hs, colk = C + h * hs, colv = 2 * C + h * hs, coly = h * hs;
  const Operand Q{p.qkv, p.in_bf16, ld3, colq}, K{p.qkv, p.in_bf16, ld3, colk}, V{p.qkv, p.in_bf16, ld3, colv}, dO{p.dy, p.dy_bf16, C, coly};

  const uint32_t seed_lo = (uint32_t)((p.seed_dev ? *p.seed_dev : 0ull) + p.seed_off);
  const uint32_t seed_hi = (uint32_t)(((p.seed_dev ? *p.seed_dev : 0ull) + p.seed_off) >> 32);
  const float keep = p.p_drop > 0.f ? 1.f / (1.f - p.p_drop) : 1.f;
  const float sl2 = p.scale * 1.4426950408889634f;
  // the two tile rows of this thread's accumulator fragments (frag_row(t, i) for even / odd i >> 1)
  int row[2];
  bool row_ok[2];
  int tok[2];                                            // token index of the row inside the batch element
  for (int e = 0; e < 2; ++e) {
    row[e] = wg * 64 + tc::frag_row(t128, 2 * e);
    row_ok[e] = row[e] < rows_valid;
    tok[e] = m0 + row[e];
  }
  float mul[2] = {1.f, 1.f};

  if (mode == MODE_BWD_K) {                              // per-column statistics of all query tokens
    for (int i = tid; i < kRowsY; i += kThreads) {
      stat_a[i] = i < T ? p.lse[(int64_t)bh * T + i] * 1.4426950408889634f : 0.f;
      stat_b[i] = i < T ? p.dsum[(int64_t)bh * T + i] : 0.f;
    }
  }

  if (mode == MODE_FWD) {
    float s[kRowsY / 2];
    score_products<kRowsY, false>(smem, Q, K, Q, K, tok0 + m0, rows_valid, tok0, T, hs, tid, wg, s, s);
    float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < kRowsY / 2; ++i)
      if (tc::frag_col(t128, i) < T) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    for (int e = 0; e < 2; ++e) {                        // the 4 lanes of a quad share a row
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
      mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
    }
#pragma unroll
    for (int i = 0; i < kRowsY / 2; i += 2) {
      const int e = (i >> 1) & 1, j = tc::frag_col(t128, i);
      const uint32_t ibase = (uint32_t)(((int64_t)bh * T + tok[e]) * T);
      float v[2] = {0.f, 0.f};
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        if (j + q < T) {
          v[q] = exp2f((s[i + q] - mx[e]) * sl2);
          sum[e] += v[q];
          if (p.p_drop > 0.f) v[q] *= drop_scale(seed_lo, seed_hi, ibase + j + q, p.p_drop, keep);
        }
      }
      store_pair(mat0, row[e], j, v[0], v[1]);
    }
    for (int e = 0; e < 2; ++e) {
      sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 1);
      sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 2);
      mul[e] = 1.f / sum[e];
      if (row_ok[e] && (t128 & 3) == 0 && p.lse) p.lse[(int64_t)bh * T + tok[e]] = mx[e] * p.scale + logf(sum[e]);
    }
  } else {
    float lse2[2], dsum[2];
    for (int e = 0; e < 2; ++e) {
      lse2[e] = (mode == MODE_BWD_Q && row_ok[e]) ? p.lse[(int64_t)bh * T + tok[e]] * 1.4426950408889634f : 0.f;
      dsum[e] = (mode == MODE_BWD_Q && row_ok[e]) ? p.dsum[(int64_t)bh * T + tok[e]] : 0.f;
    }
    for (int hc = 0; hc * kHalf < T; ++hc) {
      const int cbase = hc * kHalf;
      float s[kHalf / 2], g[kHalf / 2];
      if (mode == MODE_BWD_Q)
        score_products<kHalf, true>(smem, Q, K, dO, V, tok0 + m0, rows_valid, tok0 + cbase, T - cbase, hs, tid, wg, s, g);
      else
        score_products<kHalf, true>(smem, K, Q, V, dO, tok0 + m0, rows_valid, tok0 + cbase, T - cbase, hs, tid, wg, s, g);
#pragma unroll
      for (int i = 0; i < kHalf / 2; i += 2) {
        const int e = (i >> 1) & 1, j = cbase + tc::frag_col(t128, i);
        float o0[2] = {0.f, 0.f}, o1[2] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int c = j + q;
          if (c >= T) continue;
          if (mode == MODE_BWD_Q) {                       // rows = queries, columns = keys c
            const float pr = exp2f(s[i + q] * sl2 - lse2[e]);
            const float gd = p.p_drop > 0.f ? g[i + q] * drop_scale(seed_lo, seed_hi, (uint32_t)(((int64_t)bh * T + tok[e]) * T) + c, p.p_drop, keep) : g[i + q];
            o0[q] = p.scale * pr * (gd - dsum[e]);
          } else {                                        // rows = keys (tok), columns = queries c: S^T and dPd^T
            const float pr = exp2f(s[i + q] * sl2 - stat_a[c]);
            const float ds = p.p_drop > 0.f ? drop_scale(seed_lo, seed_hi, (uint32_t)(((int64_t)bh * T + c) * T + tok[e]), p.p_drop, keep) : 1.f;
            o0[q] = pr * ds;
            o1[q] = p.scale * pr * (g[i + q] * ds - stat_b[c]);
          }
        }
        store_pair(mat0, row[e], j, o0[0], o0[1]);
        if (mode == MODE_BWD_K) store_pair(mat1, row[e], j, o1[0], o1[1]);
      }
    }
  }

  // second product(s): out[rows x hs] = M Z, M from the element-wise stage, Z MN-major, in passes of 128 head-dimension columns.
  //   FWD: M = Pd, Z = V -> y.   BWD_Q: M = dS, Z = K -> dQ.   BWD_K: round 0 M = Pd^T, Z = dO -> dV; round 1 M = dS^T, Z = Q -> dK.
  const int nrounds = mode == MODE_BWD_K ? 2 : 1;
  const int npass = (hs + 127) / 128;
  for (int round = 0; round < nrounds; ++round) {
    Operand z;
    int ocol;                                            // output column (in out*_a, leading dimension old)
    int64_t old;
    if (mode == MODE_FWD)        { z = V;  ocol = coly; old = C; }
    else if (mode == MODE_BWD_Q) { z = K;  ocol = colq; old = ld3; }
    else if (round == 0)         { z = dO; ocol = colv; old = ld3; }
    else                         { z = Q;  ocol = colk; old = ld3; }
    const uint8_t* mat = round == 0 ? mat0 : mat1;
    const int64_t orow[2] = {(tok0 + tok[0]) * old + ocol, (tok0 + tok[1]) * old + ocol};

    auto stage_z = [&](int ps) {                         // head-dimension columns [128 ps, 128 ps + 128) as two 64-wide chunks
      uint8_t* zb = smem + (ps & 1) * kZBuf;
      for (int q = 0; q < 2; ++q) {
        const int cv = max(0, min(64, hs - ps * 128 - q * 64));
        if (cv > 0) stage_any(zb + q * kYBytes, z.src, z.bf16, z.ld, tok0, T, kRowsY, z.col + ps * 128 + q * 64, cv, tid, kThreads);
      }
    };
    __syncthreads();                                     // the element-wise stage is complete; the stages / Z buffers are free
    stage_z(0);
    cp_async_wait_all();
    tc::fence_async_smem();
    __syncthreads();
    for (int ps = 0; ps < npass; ++ps) {
      if (ps + 1 < npass) stage_z(ps + 1);               // the other Z buffer (its last pass retired before the barrier below)
      const int dvalid = min(128, hs - ps * 128);        // head-dimension columns of this pass
      float* o32 = p.out32_a ? p.out32_a + ps * 128 : nullptr;
      __nv_bfloat16* o16 = p.out16_a ? p.out16_a + ps * 128 : nullptr;
      if (dvalid > 64) value_product<128>(mat, smem + (ps & 1) * kZBuf, ncols, wg, t128, row_ok, orow, mul, dvalid, o32, o16);
      else             value_product<64>(mat, smem + (ps & 1) * kZBuf, ncols, wg, t128, row_ok, orow, mul, dvalid, o32, o16);
      if (ps + 1 < npass) {
        cp_async_wait_all();
        tc::fence_async_smem();
        __syncthreads();
      }
    }
  }
}

// D[b, h, i] = sum_d dO[b*T + i, h*hs + d] * O[b*T + i, h*hs + d]: one warp per (token row, head); the same pass writes the bf16
// copy of dO that the backward kernel stages with cp.async (hs even).
template <typename TY>
__global__ void __launch_bounds__(256) attn_dsum_kernel(const float* __restrict__ dy, const TY* __restrict__ y, float* __restrict__ dsum,
                                                        __nv_bfloat16* __restrict__ dy16, int B, int T, int nh, int hs) {
  const int64_t w = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)B * T * nh) return;
  const int h = (int)(w % nh);
  const int64_t row = w / nh;
  const int b = (int)(row / T), i = (int)(row % T);
  const int64_t base = row * (int64_t)nh * hs + h * hs;
  float s = 0.f;
  for (int d = lane * 2; d < hs; d += 64) {
    const float2 g = *reinterpret_cast<const float2*>(dy + base + d);
    float y0, y1;
    if (sizeof(TY) == 4) {
      const float2 v = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(y) + base + d);
      y0 = v.x; y1 = v.y;
    } else {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(reinterpret_cast<const __nv_bfloat16*>(y) + base + d);
      y0 = __low2float(v); y1 = __high2float(v);
    }
    s = fmaf(g.x, y0, fmaf(g.y, y1, s));
    if (dy16) *reinterpret_cast<__nv_bfloat162*>(dy16 + base + d) = __floats2bfloat162_rn(g.x, g.y);
  }
  s = warp_sum(s);
  if (lane == 0) dsum[((int64_t)b * nh + h) * T + i] = s;
}

int launch_attn(const Params& p, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal) != cudaSuccess) {
      tfb_set_last_error("cudaFuncSetAttribute(smem) failed for attn_tc_kernel");
      return TFB_ERR_DRIVER;
    }
    attr_done = true;
  }
  const int tiles = (p.T + kRowsX - 1) / kRowsX;
  const int grid = p.B * p.nh * tiles * (p.mode == MODE_FWD ? 1 : 2);
  attn_tc_kernel<<<grid, kThreads, kSmemTotal, stream>>>(p);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

}  // namespace

// Fused attention forward on the packed q|k|v buffer: y[b*T + i, h*hs : (h+1)*hs] = dropout(softmax(scale q k^T)) v for every
// (b, h). qkv: [B*T, 3*nh*hs] fp32 (qkv_bf16 = 0) or bf16 (1). y32 / y16: [B*T, nh*hs] outputs (either may be null).
// lse: [B, nh, T] row log-sum-exp of the scaled scores, saved for tfb_attn_bwd_tc. Dropout: keep-probability 1 - p_drop, mask =
// hash(*seed_dev + seed_off, ((b*nh + h)*T + i)*T + j), regenerated in backward. T <= 192, hs even.
TFB_API int tfb_attn_fwd_tc(const void* qkv, int qkv_bf16, int B, int T, int nh, int hs, float* y32, void* y16, float* lse, float scale,
                            float p_drop, const uint64_t* seed_dev, uint64_t seed_off, cudaStream_t stream) {
  TFB_REQUIRE(qkv && (y32 || y16) && lse && B > 0 && T > 0 && T <= kRowsY && nh > 0 && hs > 0 && hs % 2 == 0);
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && p_drop >= 0.f && p_drop < 1.f);
  Params p{};
  p.qkv = qkv; p.in_bf16 = qkv_bf16; p.out32_a = y32; p.out16_a = (__nv_bfloat16*)y16; p.lse = lse;
  p.seed_dev = seed_dev; p.seed_off = seed_off; p.B = B; p.T = T; p.nh = nh; p.hs = hs; p.C = nh * hs;
  p.scale = scale; p.p_drop = p_drop; p.mode = MODE_FWD;
  return launch_attn(p, stream);
}

// Backward of tfb_attn_fwd_tc: dqkv[B*T, 3C] (fp32 and / or bf16; every element written) from dy[B*T, C] (fp32), the forward's
// q|k|v input, its output y (fp32, or bf16 when y_bf16: for D = rowsum(dy * y)) and lse. Scratch: dsum [B, nh, T] fp32 and
// dy16 [B*T, C] bf16 (the bf16 copy of dy the kernel stages; written by the pre-pass).
TFB_API int tfb_attn_bwd_tc(const void* qkv, int qkv_bf16, const float* dy, const void* y, int y_bf16, const float* lse, float* dsum,
                            void* dy16, int B, int T, int nh, int hs, float* dqkv32, void* dqkv16, float scale, float p_drop,
                            const uint64_t* seed_dev, uint64_t seed_off, cudaStream_t stream) {
  TFB_REQUIRE(qkv && dy && y && lse && dsum && dy16 && (dqkv32 || dqkv16) && B > 0 && T > 0 && T <= kRowsY && nh > 0 && hs > 0 && hs % 2 == 0);
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(dy16) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const int64_t warps = (int64_t)B * T * nh;
  if (y_bf16) attn_dsum_kernel<__nv_bfloat16><<<(int)((warps + 7) / 8), 256, 0, stream>>>(dy, (const __nv_bfloat16*)y, dsum, (__nv_bfloat16*)dy16, B, T, nh, hs);
  else        attn_dsum_kernel<float><<<(int)((warps + 7) / 8), 256, 0, stream>>>(dy, (const float*)y, dsum, (__nv_bfloat16*)dy16, B, T, nh, hs);
  TFB_CHECK_LAUNCH();
  Params p{};
  p.qkv = qkv; p.in_bf16 = qkv_bf16; p.dy = dy16; p.dy_bf16 = 1; p.out32_a = dqkv32; p.out16_a = (__nv_bfloat16*)dqkv16;
  p.lse = const_cast<float*>(lse); p.dsum = dsum;
  p.seed_dev = seed_dev; p.seed_off = seed_off; p.B = B; p.T = T; p.nh = nh; p.hs = hs; p.C = nh * hs;
  p.scale = scale; p.p_drop = p_drop; p.mode = 1;
  return launch_attn(p, stream);
}
