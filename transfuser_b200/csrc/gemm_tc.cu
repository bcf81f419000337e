// wgmma / TMA GEMM for sm_90a:  C[M,N] = alpha * op(A)[M,K] * op(B)[K,N] (+ bias[n]) (+ beta*C) (ReLU)
// Operands fp32 in HBM, fed to the tensor cores as TF32 (wgmma .tf32, fp32 accumulate in registers), or bf16.
// All four transpose combinations are served without materialising a transpose: a K-contiguous operand is a
// "K-major" wgmma operand, an M/N-contiguous operand is an "MN-major" (transposed) one; both are staged by TMA into
// 128B-swizzled shared memory and described to the MMA by a shared-memory matrix descriptor.
//   forward  y = x W^T      : A K-major (x[M,K]),  B K-major (W[N,K])
//   dgrad    dx = dy W      : A K-major (dy[M,N']), B MN-major (W[N',K'] read as [k][n])
//   wgrad    dW = dy^T x    : A MN-major (dy[M',N] read as [k][m]), B MN-major (x[M',K] read as [k][n]); split-K + atomics
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups (wgmma issue on rows 0-63 / 64-127 of the tile, then the
// epilogue registers -> global), warp 8 = TMA producer. One 128 x BN output tile at a time per CTA, STAGES-deep mbarrier ring
// between TMA and the MMAs.
// Replaces cuBLAS/cuDNN behind nn.Linear and 1x1 nn.Conv2d (transfuser.py:510-527,538-543; timm RegNet 1x1 convs).
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

constexpr int BM = 128;

template <typename T> struct Elem;
template <> struct Elem<float> {
  static constexpr int kPerRow = 32;   // elements per 128-byte swizzle row
  static constexpr int kUmmaK = 8;
  static constexpr uint32_t kFmt = 2;  // TF32
  static constexpr CUtensorMapDataType kTmaType = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
};
template <> struct Elem<__nv_bfloat16> {
  static constexpr int kPerRow = 64;
  static constexpr int kUmmaK = 16;
  static constexpr uint32_t kFmt = 1;  // BF16
  static constexpr CUtensorMapDataType kTmaType = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
};

// Shared memory: STAGES x (A tile 128 x 128 B | B tile BN x 128 B), barriers, 8 x (16 x 36 floats) epilogue staging. BN (the tile
// width: a multiple of 32 up to kMaxBN, a multiple of 64 for an MN-major B) is a template parameter because it is the N of the wgmma
// instruction and the size of the register accumulator; the host picks the width that fills whole waves of the persistent grid
// and the deepest ring that fits. STAGES is a runtime value. kMaxBN = 192: with 288 threads ptxas budgets 168 registers per thread
// (warpgroup granularity), and the 224- / 256-wide accumulators (112 / 128 registers) spill around the wgmma.
int g_max_ctas = 0;                                           // tfb_gemm_set_max_ctas: cap of the persistent grid (0 = one CTA per SM)
constexpr int kMaxBN = 192;
constexpr int kThreads = 288;                                 // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int kStageFloats = 16 * 36;                         // one warp's epilogue staging block (16 rows, padded stride 36)
constexpr int kABytes = BM * 128;
constexpr int kSmemMax = 232448 - 64;                         // 227 KB opt-in limit, less the kernel's static shared flags
constexpr int kSmemFixed = 256 + 8 * kStageFloats * 4 + 1024; // barriers + epilogue staging + alignment slack

template <typename T, bool A_MN, bool B_MN, int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, float* __restrict__ Cbase,
               int64_t ldc, int M, int N, int num_kb, int kb_per_split, const float* __restrict__ bias, float alpha, float beta,
               int relu, int atomic_out, int splits, int a_step, int b_step, int64_t c_bstride, int tiles_m, int tiles_n,
               int total_tiles, int STAGES, double* __restrict__ stats, __nv_bfloat16* __restrict__ C16, float* __restrict__ ws,
               unsigned int* __restrict__ ws_cnt) {
  // PERSISTENT: gridDim.x CTAs (<= one per SM) walk the tile list t = blockIdx.x, += gridDim.x. A tile is (m-tile, n-tile, z),
  // z = batch * splits + split; m fastest so that concurrently running CTAs share the same B (weight) tile in L2.
  // Consumer warpgroup g (warps 4g..4g+3) owns rows [64g, 64g + 64) of the 128 x BN tile as a wgmma register accumulator;
  // the TMA producer runs ahead across tile boundaries through the shared-memory ring while the consumers run the epilogue.
  using E = Elem<T>;
  constexpr int BK = E::kPerRow;  // K elements per stage
  constexpr int stage_bytes = kABytes + BN * 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes);
  uint64_t* empty_bar = full_bar + STAGES;
  float* stage_out = reinterpret_cast<float*>(smem + STAGES * stage_bytes + 256);
  float* s_stat = stage_out + 8 * kStageFloats;  // [2][N] per-column statistics accumulators (present only when stats != nullptr)
  float* wstat = s_stat + 2 * N;                 // [8 warps][2][kStatW] per-tile statistics of each consumer warp (likewise)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tma_a);
    tc::tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 8); }   // 8 consumer warps
    tc::mbar_fence_init();
  }
  __syncthreads();

  // decode tile t -> coordinates
  auto decode = [&](int t, int& m0, int& n0, int& bz, int& sz, int& kb_begin, int& nkb) {
    const int tm = t % tiles_m;
    const int tn = (t / tiles_m) % tiles_n;
    const int z = t / (tiles_m * tiles_n);
    bz = z / splits; sz = z % splits;
    m0 = tm * BM; n0 = tn * BN;
    kb_begin = sz * kb_per_split;
    nkb = min(num_kb, kb_begin + kb_per_split) - kb_begin;   // >= 1 by construction
  };

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      int s = 0, ph = 0;
      constexpr int nb_chunks = (BN + E::kPerRow - 1) / E::kPerRow;
      constexpr uint32_t tx_bytes = (uint32_t)(kABytes + (B_MN ? nb_chunks * BK * 128 : BN * 128));
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int m0, n0, bz, sz, kb_begin, nkb;
        decode(t, m0, n0, bz, sz, kb_begin, nkb);
        const int am0 = m0 + bz * a_step, bn0 = n0 + bz * b_step;
        for (int i = 0; i < nkb; ++i) {
          tc::mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * stage_bytes;
          uint8_t* sb = sa + kABytes;
          tc::mbar_expect_tx(&full_bar[s], tx_bytes);
          const int k0 = (kb_begin + i) * BK;
          if (!A_MN) {
            tc::tma_load_2d(&tma_a, &full_bar[s], sa, k0, am0);
          } else {
#pragma unroll
            for (int j = 0; j < BM / E::kPerRow; ++j)
              tc::tma_load_2d(&tma_a, &full_bar[s], sa + j * BK * 128, am0 + j * E::kPerRow, k0);
          }
          if (!B_MN) {
            tc::tma_load_2d(&tma_b, &full_bar[s], sb, k0, bn0);
          } else {
#pragma unroll
            for (int j = 0; j < nb_chunks; ++j)
              tc::tma_load_2d(&tma_b, &full_bar[s], sb + j * BK * 128, bn0 + j * E::kPerRow, k0);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===== consumers: wgmma issue + epilogue =====
    const int wg = warp >> 2, t128 = threadIdx.x & 127;
    float acc[BN / 2];
    int s = 0, ph = 0;
    if (stats) tc::stat_clear(s_stat, N, (int)threadIdx.x);
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int m0, n0, bz, sz, kb_begin, nkb;
      decode(t, m0, n0, bz, sz, kb_begin, nkb);
      int prev = 0;
      for (int i = 0; i < nkb; ++i) {
        tc::mbar_wait(&full_bar[s], ph);
        const uint32_t base = tc::smem_u32(smem + s * stage_bytes);
        // this warpgroup's 64 rows: K-major A: 64 rows of 128 B further; MN-major A: the second 64-element M chunk
        const uint32_t sa = base + (A_MN ? wg * BK * 128 : wg * 64 * 128), sb = base + kABytes;
        tc::fence_acc(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / E::kUmmaK; ++k) {
          // K-major: advance 32 B inside the 128 B swizzle row; MN-major: advance kUmmaK rows of 128 B.
          const uint32_t a_off = A_MN ? k * E::kUmmaK * 128 : k * E::kUmmaK * (int)sizeof(T);
          const uint32_t b_off = B_MN ? k * E::kUmmaK * 128 : k * E::kUmmaK * (int)sizeof(T);
          const uint64_t adesc = tc::make_smem_desc(sa + a_off, A_MN ? BK * 128 : 16, 1024);
          const uint64_t bdesc = tc::make_smem_desc(sb + b_off, B_MN ? BK * 128 : 16, 1024);
          const uint32_t accum = (i > 0 || k > 0) ? 1u : 0u;
          if constexpr (sizeof(T) == 4) tc::wgmma_tf32(acc, adesc, bdesc, accum);
          else                          tc::wgmma_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, accum);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();             // the MMAs of k-block i - 1 have retired: hand their slot back to the producer
        tc::fence_acc(acc);
        if (i > 0) { __syncwarp(); if (lane == 0) tc::mbar_arrive(&empty_bar[prev]); }
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::fence_acc(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);

      // ---- epilogue: this warp's 16-row band of the tile ----
      const int r0 = m0 + wg * 64 + (warp & 3) * 16;
      const bool add_bias = bias != nullptr && sz == 0;
      if (splits > 1) {
        // split-K: the partial tile goes to its own slice of the workspace; the last split of the tile to arrive adds the slices
        // to C in split order (the same bits every run, whatever order the CTAs run in)
        __shared__ unsigned int s_last;
        float* part = ws + (int64_t)(bz * splits + sz) * M * N;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) {
          const int m = m0 + wg * 64 + tc::frag_row(t128, i), n = n0 + tc::frag_col(t128, i);
          if (m < M && n < N) part[(int64_t)m * N + n] = alpha * acc[i] + (add_bias ? bias[n] : 0.f);
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(tc::kConsumers) : "memory");
        const int tile = (m0 / BM) + tiles_m * ((n0 / BN) + tiles_n * bz);
        if (threadIdx.x == 0) s_last = atomicAdd(ws_cnt + tile, 1u) == (unsigned int)(splits - 1);
        asm volatile("bar.sync 1, %0;" ::"n"(tc::kConsumers) : "memory");
        if (s_last) {
          __threadfence();
          if (threadIdx.x == 0) ws_cnt[tile] = 0u;   // the stream's scratch counters are zero on entry
          for (int e = threadIdx.x; e < BM * BN; e += tc::kConsumers) {
            const int m = m0 + e / BN, n = n0 + e % BN;
            if (m < M && n < N) {
              float s = 0.f;
              for (int z = 0; z < splits; ++z) s += __ldcg(ws + ((int64_t)(bz * splits + z) * M + m) * N + n);
              Cbase[(int64_t)bz * c_bstride + (int64_t)m * ldc + n] += s;
            }
          }
        }
        continue;
      }
      float* cwarp = Cbase + (int64_t)bz * c_bstride + (int64_t)r0 * ldc;
      const bool fast = (atomic_out || beta == 0.f) && (ldc & 3) == 0 &&
                        (C16 ? (reinterpret_cast<uintptr_t>(C16) & 7) == 0 : (reinterpret_cast<uintptr_t>(cwarp + n0) & 15) == 0);
      if (fast) {
        // coalesced path: 32-column chunks through this warp's padded smem staging buffer
        float* stage = stage_out + warp * kStageFloats;
        const int rows_valid = M - r0;
#pragma unroll
        for (int c = 0; c < (BN + 31) / 32; ++c) {
          const int c0 = c * 32;
          const int cols_valid = min(N - (n0 + c0), BN - c0);
          if (cols_valid <= 0) break;   // warp-uniform
          const int64_t off0 = (int64_t)bz * c_bstride + (int64_t)r0 * ldc + n0 + c0;
          tc::frag_to_stage(stage, acc, c, lane);
          tc::stage_to_global(stage, [=](int row) -> int64_t { return row < rows_valid ? off0 + (int64_t)row * ldc : (int64_t)-1; },
                              cols_valid, add_bias ? bias + n0 + c0 : nullptr, alpha, relu, lane, Cbase, C16,
                              stats ? wstat + (warp * 2) * tc::kStatW + c0 : nullptr,
                              stats ? wstat + (warp * 2 + 1) * tc::kStatW + c0 : nullptr, atomic_out);
        }
        if (stats) tc::stat_fold(s_stat, wstat, N, n0, min(BN, N - n0), (int)threadIdx.x);
      } else {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) {
          const int m = m0 + wg * 64 + tc::frag_row(t128, i), n = n0 + tc::frag_col(t128, i);
          if (m < M && n < N) {
            float* cp = Cbase + (int64_t)bz * c_bstride + (int64_t)m * ldc + n;
            float o = alpha * acc[i] + (add_bias ? bias[n] : 0.f);
            if (atomic_out) {
              atomicAdd(cp, o);
            } else {
              if (beta != 0.f) o += beta * *cp;
              if (relu) o = fmaxf(o, 0.f);
              *cp = o;
            }
          }
        }
      }
    }
    if (stats) tc::stat_flush(s_stat, stats, N, (int)threadIdx.x, ws, ws_cnt);
  }
}

// ---- host side ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D map over a row-major [rows][cols] matrix with leading dimension ld (elements); box = {box_cols, box_rows}.
template <typename T>
bool make_map_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(T)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, Elem<T>::kTmaType, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

template <typename T, bool A_MN, bool B_MN, int BN>
int launch_bn(int M, int N, int K, const T* A, int64_t lda, const T* B, int64_t ldb, float* C, int64_t ldc, const float* bias,
              int relu, float alpha, float beta, int splits, cudaStream_t stream, int nbatch = 1, int a_step = 0, int b_step = 0,
              int64_t c_bstride = 0, double* stats = nullptr, __nv_bfloat16* C16 = nullptr) {
  using E = Elem<T>;
  if (C16) {     // bf16 output: coalesced epilogue path only
    TFB_REQUIRE(splits <= 1 && beta == 0.f && (ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(C16) & 7) == 0);
  }
  constexpr int BK = E::kPerRow;
  if (stats) {   // the statistics come out of the coalesced epilogue path only: make sure the kernel takes it
    TFB_REQUIRE(splits <= 1 && beta == 0.f && nbatch == 1 && (ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0 && !relu && N <= 4096);
  }
  const int stage_bytes = kABytes + BN * 128;
  // per-column accumulators and the consumer warps' per-tile statistics behind the epilogue staging
  const int stat_bytes = stats ? (2 * N + 8 * 2 * tc::kStatW) * (int)sizeof(float) : 0;
  int stages = (kSmemMax - kSmemFixed - stat_bytes) / stage_bytes;
  if (stages > 8) stages = 8;
  const int smem_total = stages * stage_bytes + kSmemFixed + stat_bytes;
  CUtensorMap ma, mb;
  bool ok;
  const int64_t Mext = (int64_t)(nbatch - 1) * a_step + M, Next = (int64_t)(nbatch - 1) * b_step + N;   // extents of the shared maps
  if (!A_MN) ok = make_map_2d<T>(&ma, A, Mext, K, lda, BK, BM);              // A[m][k]
  else       ok = make_map_2d<T>(&ma, A, K, Mext, lda, E::kPerRow, BK);      // A[k][m]
  if (!ok) { tfb_set_last_error("cuTensorMapEncodeTiled(A) failed"); return TFB_ERR_DRIVER; }
  if (!B_MN) ok = make_map_2d<T>(&mb, B, Next, K, ldb, BK, BN);              // B[n][k]
  else       ok = make_map_2d<T>(&mb, B, K, Next, ldb, E::kPerRow, BK);      // B[k][n]
  if (!ok) { tfb_set_last_error("cuTensorMapEncodeTiled(B) failed"); return TFB_ERR_DRIVER; }
  const int num_kb = (K + BK - 1) / BK;
  if (splits < 1) splits = 1;
  if (splits > num_kb) splits = num_kb;
  int kb_per_split = (num_kb + splits - 1) / splits;
  splits = (num_kb + kb_per_split - 1) / kb_per_split;
  // beta == 1 without an activation (accumulating a further term into C: the multi-term parity modes, q/k/v dgrad sums): the
  // reduction epilogue adds into C with coalesced vector reductions instead of the scalar read-modify-write path
  const bool accumulate = beta == 1.f && !relu && !stats && !C16 && nbatch == 1;
  const int atomic_out = (splits > 1 || accumulate) ? 1 : 0;
  if (atomic_out) {
    if (relu) { tfb_set_last_error("split-K cannot fuse ReLU"); return TFB_ERR_ARG; }
    if (beta == 0.f) {
      if (ldc == N && (nbatch == 1 || c_bstride == (int64_t)M * N)) {   // outputs are one contiguous block: a single memset
        if (cudaMemsetAsync(C, 0, (size_t)nbatch * M * N * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
      } else {
        for (int b = 0; b < nbatch; ++b)
          if (cudaMemset2DAsync(C + (int64_t)b * c_bstride, ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, stream) != cudaSuccess)
            return TFB_ERR_DRIVER;
      }
    } else if (beta != 1.f) { tfb_set_last_error("split-K needs beta in {0,1}"); return TFB_ERR_ARG; }
  }
  auto kern = gemm_tc_kernel<T, A_MN, B_MN, BN>;
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax) != cudaSuccess) {
      tfb_set_last_error("cudaFuncSetAttribute(smem) failed");
      return TFB_ERR_DRIVER;
    }
    attr_done = true;
  }
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  const int64_t total = (int64_t)tiles_m * tiles_n * splits * nbatch;
  if (total > 0x7fffffff) { tfb_set_last_error("too many tiles"); return TFB_ERR_ARG; }
  int grid = (int)(total < tfb_num_sms() ? total : tfb_num_sms());
  if (g_max_ctas > 0 && grid > g_max_ctas) grid = g_max_ctas;
  // workspace of the ordered cross-CTA reductions: split-K partial tiles + one counter per output tile, or the CTAs' statistics
  TfbScratch ws;
  if (splits > 1) {
    const int rc = tfb_scratch(ws, (size_t)nbatch * splits * M * N, (size_t)tiles_m * tiles_n * nbatch, stream);
    if (rc != TFB_OK) return rc;
  } else if (stats) {
    const int rc = tfb_scratch(ws, (size_t)grid * 2 * N, 1, stream);
    if (rc != TFB_OK) return rc;
  }
  kern<<<grid, kThreads, smem_total, stream>>>(ma, mb, C, ldc, M, N, num_kb, kb_per_split, bias, alpha, beta, relu, atomic_out, splits,
                                               a_step, b_step, c_bstride, tiles_m, tiles_n, (int)total, stages, stats, C16, ws.f, ws.cnt);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// Tile widths: multiples of 32 (K-major B), multiples of 64 (MN-major B: whole 128-byte swizzle rows); TF32 only as K-major x K-major.
template <typename T, bool A_MN, bool B_MN>
int launch_tc(int BN, int M, int N, int K, const T* A, int64_t lda, const T* B, int64_t ldb, float* C, int64_t ldc, const float* bias,
              int relu, float alpha, float beta, int splits, cudaStream_t stream, int nbatch = 1, int a_step = 0, int b_step = 0,
              int64_t c_bstride = 0, double* stats = nullptr, __nv_bfloat16* C16 = nullptr) {
#define TFB_BN(bn_) case bn_: return launch_bn<T, A_MN, B_MN, bn_>(M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream, \
                                                                  nbatch, a_step, b_step, c_bstride, stats, C16)
  if constexpr (B_MN) {
    switch (BN) { TFB_BN(64); TFB_BN(128); TFB_BN(192); }
  } else {
    switch (BN) { TFB_BN(32); TFB_BN(64); TFB_BN(96); TFB_BN(128); TFB_BN(160); TFB_BN(192); }
  }
#undef TFB_BN
  tfb_set_last_error("gemm_tc: unsupported tile width");
  return TFB_ERR_ARG;
}

template <typename T>
int dispatch_major(int BN, int transA, int transB, int M, int N, int K, const T* A, int64_t lda, const T* B, int64_t ldb, float* C,
                   int64_t ldc, const float* bias, int relu, float alpha, float beta, int splits, cudaStream_t stream, double* stats = nullptr,
                   __nv_bfloat16* C16 = nullptr) {
  // BLAS-style flags: op(A)[m][k] = transA ? A[k*lda+m] : A[m*lda+k];  op(B)[k][n] = transB ? B[n*ldb+k] : B[k*ldb+n]
  const bool a_mn = transA != 0, b_mn = transB == 0;
  if (!a_mn && !b_mn) return launch_tc<T, false, false>(BN, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream, 1, 0, 0, 0, stats, C16);
  if (!a_mn && b_mn && C16) return launch_tc<T, false, true>(BN, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream, 1, 0, 0, 0, nullptr, C16);
  if (C16) { tfb_set_last_error("bf16 output is wired for the forward / dgrad forms only"); return TFB_ERR_UNSUPPORTED; }
  if (stats) { tfb_set_last_error("column statistics are produced by the y = x W^T form only"); return TFB_ERR_UNSUPPORTED; }
  if (!a_mn && b_mn)  return launch_tc<T, false, true>(BN, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream);
  if (a_mn && b_mn)   return launch_tc<T, true, true>(BN, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream);
  return launch_tc<T, true, false>(BN, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream);
}

// Tile width (and, when auto_split, the split-K factor) for a [M, N] output with `nbatch` independent batches and num_kb k-blocks.
// The kernel is bound by the bytes each CTA pulls from L2 per k-block ((128 + BN) * 128 B against ~42 B/clk per SM), so one CTA
// costs ~ kb_per_split * (128 + BN) plus a fixed prologue / epilogue share (kFixed, in the same unit: ~6 k-blocks of a 128 x 128
// tile) plus, for split-K, the fp32 atomics of its 128 x BN partial tile; the persistent grid runs ceil(CTAs / SMs) waves.
// step = 32 (K-major B) or 64 (MN-major B: whole 128-byte swizzle rows). auto_split: the number of splits that fills one wave of
// SMs while leaving >= 4 k-blocks per CTA (weight gradients: long contraction, few output tiles).
int pick_bn(int M, int N, int zs, int step, int num_kb = 0, bool auto_split = false, int* splits_out = nullptr) {
  static int force_bn = -1, model_c = -2;
  if (force_bn < 0) { const char* e = getenv("TFB_GEMM_BN"); force_bn = e ? atoi(e) : 0; }
  if (model_c == -2) { const char* e = getenv("TFB_GEMM_TILE_MODEL"); model_c = e ? atoi(e) : 64; }
  const int nmax = ((N + step - 1) / step) * step;                 // one tile covers all of N
  const int64_t mt = (M + BM - 1) / BM;
  // the grid this launch may use: all SMs, or the cap set for launches on the weight-gradient stream (tfb_gemm_set_max_ctas)
  const int sms = (g_max_ctas > 0 && g_max_ctas < tfb_num_sms()) ? g_max_ctas : tfb_num_sms();
  int best_bn = 0, best_s = 1;
  int64_t best = -1;
  for (int bn = step; bn <= kMaxBN; bn += step) {
    int use = bn < nmax ? bn : nmax;                               // never wider than the problem
    if (force_bn > 0) { use = ((force_bn + step - 1) / step) * step; if (use > kMaxBN) use = kMaxBN; if (use > nmax) use = nmax; }
    const int64_t tiles = mt * ((N + use - 1) / use) * zs;
    int64_t cost;
    int s = 1;
    if (auto_split && num_kb > 0) {
      s = (int)(sms / tiles);
      if (s > num_kb / 4) s = num_kb / 4;
      if (s < 1) s = 1;
      const int kbs = (num_kb + s - 1) / s;
      s = (num_kb + kbs - 1) / kbs;
      const int64_t waves = (tiles * s + sms - 1) / sms;
      cost = waves * ((int64_t)kbs * (128 + use) + 6 * 256 + (s > 1 ? 4 * use : 0));
    } else {
      cost = ((tiles + sms - 1) / sms) * (128 + use + model_c);
    }
    if (best < 0 || cost < best || (cost == best && use > best_bn)) { best = cost; best_bn = use; best_s = s; }
    if (use == nmax || force_bn > 0) break;
  }
  if (splits_out) *splits_out = best_s;
  return best_bn;
}

template <typename T>
int gemm_tc_any(int transA, int transB, int M, int N, int K, const T* A, int64_t lda, const T* B, int64_t ldb, float* C,
                int64_t ldc, const float* bias, int relu, float alpha, float beta, int splits, cudaStream_t stream, double* stats = nullptr,
                __nv_bfloat16* C16 = nullptr) {
  TFB_REQUIRE(M > 0 && N > 0 && K > 0 && A && B && (C || C16));
  // TMA: 16-byte aligned bases and leading dimensions.
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0);
  TFB_REQUIRE((lda * sizeof(T)) % 16 == 0 && (ldb * sizeof(T)) % 16 == 0);
  const int step = transB == 0 ? 64 : 32;
  const int num_kb = (K + Elem<T>::kPerRow - 1) / Elem<T>::kPerRow;
  if (splits <= 0 && !stats && !C16 && !relu && (beta == 0.f || beta == 1.f)) {      // auto split-K (weight gradients)
    const int bn = pick_bn(M, N, 1, step, num_kb, true, &splits);
    return dispatch_major<T>(bn, transA, transB, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream, stats, C16);
  }
  const int zs = splits < 1 ? 1 : (splits > num_kb ? num_kb : splits);
  return dispatch_major<T>(pick_bn(M, N, zs, step), transA, transB, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream, stats, C16);
}

}  // namespace

// Batched split-K product for grouped-conv wgrad: for b < nbatch,
//   C_b[M,N] (fp32, at C + b*c_bstride, row stride ldc) = A[:, b*a_step : +M]^T (bf16 [K, lda]) * B[:, b*b_step : +N] (bf16 [K, ldb])
// i.e. the transA=1 / transB=0 case of tfb_gemm_bf16_tc with per-batch column windows of the same two matrices.
TFB_API int tfb_gemm_bf16_tc_wgrad_batched(int M, int N, int K, const void* A, int64_t lda, int a_step, const void* B, int64_t ldb,
                                           int b_step, float* C, int64_t ldc, int64_t c_bstride, int nbatch, int splits,
                                           cudaStream_t stream) {
  TFB_REQUIRE(M > 0 && N > 0 && K > 0 && A && B && C && nbatch >= 1);
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0);
  TFB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && a_step % 8 == 0 && b_step % 8 == 0);
  using T = __nv_bfloat16;
  const int num_kb = (K + 63) / 64;
  if (splits <= 0) {                                                                  // auto split-K
    const int bn = pick_bn(M, N, nbatch, 64, num_kb, true, &splits);
    return launch_tc<T, true, true>(bn, M, N, K, (const T*)A, lda, (const T*)B, ldb, C, ldc, nullptr, 0, 1.f, 0.f, splits, stream, nbatch, a_step, b_step, c_bstride);
  }
  const int zs = (splits < 1 ? 1 : (splits > num_kb ? num_kb : splits)) * nbatch;
  return launch_tc<T, true, true>(pick_bn(M, N, zs, 64), M, N, K, (const T*)A, lda, (const T*)B, ldb, C, ldc, nullptr, 0, 1.f, 0.f, splits, stream, nbatch, a_step, b_step, c_bstride);
}

// TF32 operands straight from fp32 storage (wgmma .tf32). Only the K-major x K-major case (y = x W^T) exists: wgmma reads
// TF32 operands K-major only. transA must be 0 and transB 1.
TFB_API int tfb_gemm_tf32_tc(int transA, int transB, int M, int N, int K, const float* A, int64_t lda, const float* B,
                             int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, float alpha, float beta,
                             int splits, cudaStream_t stream) {
  TFB_REQUIRE(M > 0 && N > 0 && K > 0 && A && B && C);
  if (transA || !transB) { tfb_set_last_error("tfb_gemm_tf32_tc: only transA=0, transB=1 is supported"); return TFB_ERR_UNSUPPORTED; }
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 && lda % 4 == 0 && ldb % 4 == 0);
  return launch_tc<float, false, false>(pick_bn(M, N, 1, 32), M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, splits, stream);
}

TFB_API int tfb_gemm_bf16_tc(int transA, int transB, int M, int N, int K, const void* A, int64_t lda, const void* B,
                             int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, float alpha, float beta,
                             int splits, cudaStream_t stream) {
  return gemm_tc_any<__nv_bfloat16>(transA, transB, M, N, K, (const __nv_bfloat16*)A, lda, (const __nv_bfloat16*)B, ldb, C, ldc,
                                    bias, relu, alpha, beta, splits, stream);
}

// y[M,N] (fp32) = x[M,K] W[N,K]^T (bf16 operands) as tfb_gemm_bf16_tc(0, 1, ...), and in the same epilogue the per-column
// statistics of y: stats[n] += sum_m y[m][n], stats[N + n] += sum_m y[m][n]^2 (fp64 atomics; the caller zeroes stats once per
// training step). The training-mode BatchNorm behind every 1x1 conv of the RegNetY trunks (timm BatchNormAct2d) then needs no
// statistics pass of its own (tfb_bn_fwd_stats). ldc % 4 == 0, C 16-byte aligned.
TFB_API int tfb_gemm_bf16_tc_stats(int M, int N, int K, const void* A, int64_t lda, const void* B, int64_t ldb, float* C, int64_t ldc,
                                   double* stats, cudaStream_t stream) {
  TFB_REQUIRE(stats != nullptr);
  return gemm_tc_any<__nv_bfloat16>(0, 1, M, N, K, (const __nv_bfloat16*)A, lda, (const __nv_bfloat16*)B, ldb, C, ldc, nullptr, 0, 1.f, 0.f,
                                    1, stream, stats);
}

// As tfb_gemm_bf16_tc with transA = 0 (forward y = x W^T or dgrad dx = dy W), but the result is written in bf16 (C16, leading
// dimension ldc elements, ldc % 4 == 0): the operand of the next tensor-core GEMM / the fused attention needs no cast pass and
// the epilogue writes half the bytes. No split-K, no beta.
TFB_API int tfb_gemm_bf16_tc_out16(int transB, int M, int N, int K, const void* A, int64_t lda, const void* B, int64_t ldb, void* C16,
                                   int64_t ldc, const float* bias, int relu, float alpha, cudaStream_t stream) {
  TFB_REQUIRE(C16 != nullptr);
  return gemm_tc_any<__nv_bfloat16>(0, transB, M, N, K, (const __nv_bfloat16*)A, lda, (const __nv_bfloat16*)B, ldb, nullptr, ldc, bias, relu,
                                    alpha, 0.f, 1, stream, nullptr, (__nv_bfloat16*)C16);
}

// Caps the persistent grid of the following tensor-core GEMM launches at max_ctas CTAs (0 = no cap: one per SM). The weight-gradient
// GEMMs run on a side stream next to the critical dx chain; with a full-chip grid their split-K takes every SM away from it, with a
// capped grid they use the SMs the chain leaves idle.
// Host-side state (not a stream operation); read at launch time, so a captured CUDA graph keeps the grid it was captured with.
TFB_API int tfb_gemm_set_max_ctas(int max_ctas) {
  g_max_ctas = max_ctas > 0 ? max_ctas : 0;
  return TFB_OK;
}
