// Implicit-GEMM 3x3 convolution (stride 1, pad 1, NHWC) on the wgmma tensor cores — no im2col buffer.
// One CTA = one 8x16 spatial tile (128 output pixels = two wgmma M = 64 halves) of one image x one block of output channels.
// For each of the 9 taps and each input-channel chunk, TMA loads the tap-SHIFTED activation patch straight from the NHWC
// bf16 tensor with a 4-D tensor map (box {KC channels, 16 w, 8 h, 1 n}; halo / image-border pixels are TMA out-of-bounds
// zero fill = the conv's zero padding) into 128B/64B-swizzled shared memory, where it is already a K-major A operand;
// the packed weights (K-major B operand, bf16, zero-padded, block-diagonal for grouped convs) come through a 2-D map.
// All taps / chunks accumulate into ONE fp32 register accumulator per consumer warpgroup; the epilogue adds bias / ReLU and
// writes fp32 NHWC. dgrad (stride 1) is the same kernel on dy with tap-flipped, transposed packed weights.
// Grouped RegNetY convs (group width 24): two groups share one CTA (N = 48 output channels, 64-channel K window).
// Replaces cuDNN behind the grouped 3x3 of timm's RegNetY blocks (transfuser.py:145-184) and the dense 3x3 of the
// decoders / heads (transfuser.py:214-281; model.py:93-99, 581-585). Warp roles as in gemm_tc.cu.
#include "common.cuh"
#include "tc_host.cuh"
#include "tc_ptx.cuh"

namespace {

constexpr int TH = 8, TW = 16, BM = TH * TW;
constexpr int kThreads = 288;                   // warps 0-7: two consumer warpgroups (tile rows 0-3 / 4-7); warp 8: TMA producer
constexpr int kStageFloats = 16 * 36;           // one warp's epilogue staging block

template <int KC, int NB, int STAGES>
__global__ void __launch_bounds__(kThreads, NB <= 64 ? 2 : 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tma_x, const __grid_constant__ CUtensorMap tma_w, float* __restrict__ y,
                  const float* __restrict__ bias, int H, int W, int Cout, int tiles_w, int tiles_h, int c_step, int nchunks,
                  int nb_real, int relu, int gblocks, int total_tiles, int stride, double* __restrict__ stats, float* __restrict__ ws,
                  unsigned int* __restrict__ ws_cnt) {
  // H, W: OUTPUT height / width. stride 2: the activation map steps two pixels per box element, so tile pixel (h, w) reads the
  // input pixel (2h + dy, 2w + dx) of tap (dy, dx).
  // PERSISTENT: tile t = (spatial tile, channel block), channel block fastest (CTAs running together re-use the same activation
  // patch out of L2); the producer loads the next tile's stages while the consumers run the epilogue.
  constexpr int ROWB = KC * 2;                 // bytes per smem row (= swizzle width)
  constexpr int A_BYTES = BM * ROWB, B_BYTES = NB * ROWB, STAGE = A_BYTES + B_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE);
  uint64_t* empty_bar = full_bar + STAGES;
  float* stage_out = reinterpret_cast<float*>(smem + STAGES * STAGE + 256);
  float* s_stat = stage_out + 8 * kStageFloats; // [2][Cout] per-channel statistics accumulators (present only when stats != nullptr)
  float* wstat = s_stat + 2 * Cout;             // [8 warps][2][kStatW] per-tile statistics of each consumer warp (likewise)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int iters = nchunks * 9;

  if (threadIdx.x == 0) {
    tc::tma_prefetch_desc(&tma_x);
    tc::tma_prefetch_desc(&tma_w);
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 8); }   // 8 consumer warps
    tc::mbar_fence_init();
  }
  __syncthreads();

  auto decode = [&](int t, int& gb, int& n, int& h0, int& w0) {
    gb = t % gblocks;
    int sp = t / gblocks;
    const int tw = sp % tiles_w; sp /= tiles_w;
    const int th = sp % tiles_h; sp /= tiles_h;
    n = sp; h0 = th * TH; w0 = tw * TW;
  };

  if (warp == 8) {
    if (lane == 0) {
      int it = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int gb, n, h0, w0;
        decode(t, gb, n, h0, w0);
        for (int i = 0; i < iters; ++i, ++it) {
          const int s = it % STAGES, ph = (it / STAGES) & 1;
          const int chunk = i / 9, tap = i % 9;
          tc::mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * STAGE;
          tc::mbar_expect_tx(&full_bar[s], STAGE);
          tc::tma_load_4d(&tma_x, &full_bar[s], sa, gb * c_step + chunk * KC, w0 * stride + tap % 3 - 1, h0 * stride + tap / 3 - 1, n);
          tc::tma_load_2d(&tma_w, &full_bar[s], sa + A_BYTES, 0, ((gb * nchunks + chunk) * 9 + tap) * NB);
        }
      }
    }
  } else {
    const int wg = warp >> 2, wq = warp & 3;
    float* stage = stage_out + warp * kStageFloats;
    float acc[NB / 2];
    int it = 0;
    if (stats) tc::stat_clear(s_stat, Cout, (int)threadIdx.x);
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int gb, n, h0, w0;
      decode(t, gb, n, h0, w0);
      int prev = 0;
      for (int i = 0; i < iters; ++i, ++it) {
        const int s = it % STAGES, ph = (it / STAGES) & 1;
        tc::mbar_wait(&full_bar[s], ph);
        const uint32_t sa = tc::smem_u32(smem + s * STAGE) + wg * 64 * ROWB, sb = tc::smem_u32(smem + s * STAGE) + A_BYTES;
        tc::fence_acc(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < KC / 16; ++k)
          tc::wgmma_bf16<0, 0>(acc, tc::make_smem_desc(sa + k * 32, 16, ROWB * 8, ROWB), tc::make_smem_desc(sb + k * 32, 16, ROWB * 8, ROWB),
                               (i > 0 || k > 0) ? 1u : 0u);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        tc::fence_acc(acc);
        if (i > 0) { __syncwarp(); if (lane == 0) tc::mbar_arrive(&empty_bar[prev]); }
        prev = s;
      }
      tc::wgmma_wait<0>();
      tc::fence_acc(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&empty_bar[prev]);

      // this warp's 16 accumulator rows = tile row 4 * wg + wq = output pixels (h0 + 4 * wg + wq, w0 + 0..15)  (W fastest in the TMA box)
      const int h = h0 + wg * 4 + wq;
      const int nvalid = min(nb_real, Cout - gb * nb_real);
      float* ytile = y + (int64_t)gb * nb_real;
      const float* bp = bias ? bias + gb * nb_real : nullptr;
      const bool fast = (Cout & 3) == 0 && ((gb * nb_real) & 3) == 0 && ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
      if (fast) {
#pragma unroll
        for (int c = 0; c < (NB + 31) / 32; ++c) {
          const int c0 = c * 32;
          const int cols_valid = min(nvalid - c0, NB - c0);
          if (cols_valid <= 0) break;
          tc::frag_to_stage(stage, acc, c, lane);
          tc::stage_to_global(stage,
                              [=](int row) -> int64_t {
                                const int w = w0 + row;
                                return (h < H && w < W) ? (((int64_t)n * H + h) * W + w) * Cout + c0 : (int64_t)-1;
                              },
                              cols_valid, bp ? bp + c0 : nullptr, 1.f, relu, lane, ytile, nullptr,
                              stats ? wstat + (warp * 2) * tc::kStatW + c0 : nullptr,
                              stats ? wstat + (warp * 2 + 1) * tc::kStatW + c0 : nullptr);
        }
        if (stats) tc::stat_fold(s_stat, wstat, Cout, gb * nb_real, nvalid, (int)threadIdx.x);
      } else {
        const int t128 = threadIdx.x & 127;
#pragma unroll
        for (int i = 0; i < NB / 2; ++i) {
          const int r = tc::frag_row(t128, i) - wq * 16, col = tc::frag_col(t128, i);   // r: row inside this warp's band
          const int w = w0 + r;
          if (h < H && w < W && col < nvalid) {
            float o = acc[i] + (bp ? bp[col] : 0.f);
            if (relu) o = fmaxf(o, 0.f);
            ytile[(((int64_t)n * H + h) * W + w) * Cout + col] = o;
          }
        }
      }
    }
    if (stats) tc::stat_flush(s_stat, stats, Cout, (int)threadIdx.x, ws, ws_cnt);
  }
}

template <int KC, int NB>
int launch_conv(const void* x16, const void* wpack, const float* bias, float* y, int N, int Hin, int Win, int Cx, int Cy, int c_step,
                int nchunks, int nb_real, int gblocks, int relu, int stride, double* stats, cudaStream_t stream) {
  const int H = (Hin - 1) / stride + 1, W = (Win - 1) / stride + 1;       // output size (kernel 3, pad 1)
  constexpr int STAGES = NB <= 64 ? 6 : 4;
  constexpr int STAGE = BM * KC * 2 + NB * KC * 2;
  constexpr int SMEM0 = STAGES * STAGE + 256 + 8 * kStageFloats * 4 + 1024;   // ring + barriers + epilogue staging + alignment slack
  // + per-channel statistics accumulators and the consumer warps' per-tile statistics
  const int SMEM = SMEM0 + (stats ? (2 * Cy + 8 * 2 * tc::kStatW) * (int)sizeof(float) : 0);
  CUtensorMap mx, mw;
  const uint64_t xd[4] = {(uint64_t)Cx, (uint64_t)Win, (uint64_t)Hin, (uint64_t)N};
  const uint64_t xs[3] = {(uint64_t)Cx * 2, (uint64_t)Win * Cx * 2, (uint64_t)Hin * Win * Cx * 2};
  const uint32_t xb[4] = {(uint32_t)KC, (uint32_t)(TW * stride), (uint32_t)(TH * stride), 1};
  const uint32_t xe[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
  const CUtensorMapSwizzle swz = KC == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  if (!tc::make_map(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x16, xd, xs, xb, swz, xe)) {
    tfb_set_last_error("cuTensorMapEncodeTiled(activation, 4-D) failed");
    return TFB_ERR_DRIVER;
  }
  const uint64_t wd[2] = {(uint64_t)KC, (uint64_t)gblocks * nchunks * 9 * NB};
  const uint64_t ws[1] = {(uint64_t)KC * 2};
  const uint32_t wb[2] = {(uint32_t)KC, (uint32_t)NB};
  if (!tc::make_map(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, wpack, wd, ws, wb, swz)) {
    tfb_set_last_error("cuTensorMapEncodeTiled(packed weights) failed");
    return TFB_ERR_DRIVER;
  }
  auto kern = conv3x3_tc_kernel<KC, NB, STAGES>;
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM0 + (2 * 2048 + 8 * 2 * tc::kStatW) * (int)sizeof(float)) != cudaSuccess) return TFB_ERR_DRIVER;
    attr_done = true;
  }
  const int tiles_w = (W + TW - 1) / TW, tiles_h = (H + TH - 1) / TH;
  const int64_t total = (int64_t)tiles_w * tiles_h * N * gblocks;
  if (total > 0x7fffffff) { tfb_set_last_error("too many tiles"); return TFB_ERR_ARG; }
  // NB <= 64 tiles use < 100 KB of shared memory: two persistent CTAs per SM hide each other's pipeline bubbles
  const int per_sm = (SMEM <= 110 * 1024) ? 2 : 1;
  const int64_t cap = (int64_t)tfb_num_sms() * per_sm;
  const int grid = (int)(total < cap ? total : cap);
  TfbScratch wk;                 // the CTAs' statistics, reduced in CTA order by the last one
  if (stats) {
    const int rc = tfb_scratch(wk, (size_t)grid * 2 * Cy, 1, stream);
    if (rc != TFB_OK) return rc;
  }
  kern<<<grid, kThreads, SMEM, stream>>>(mx, mw, y, bias, H, W, Cy, tiles_w, tiles_h, c_step, nchunks, nb_real, relu, gblocks, (int)total, stride, stats,
                                         wk.f, wk.cnt);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

}  // namespace

// y[N,Ho,Wo,Cy] (fp32) = conv3x3(x16[N,H,W,Cx] bf16, packed weights; pad 1, stride 1 or 2) (+bias) (ReLU), Ho = (H-1)/stride + 1.
// Block gb reads channels [gb*c_step + chunk*KC, +KC) for chunk < nchunks and writes channels [gb*nb_real, +min(nb_real, Cy - gb*nb_real)).
// stride 2 (first block of every RegNetY stage): the TMA map traverses the activation with element strides {1, 2, 2, 1}.
// stats (optional, 2*Cy doubles, zeroed by the caller once per step): per-channel sum / sum of squares of y accumulated in the
// epilogue (training-mode BatchNorm statistics without a pass over y); needs Cy % 4 == 0, nb_real % 4 == 0, no bias / ReLU.
TFB_API int tfb_conv3x3_tc_strided(const void* x16, const void* wpack, const float* bias, float* y, int N, int H, int W, int Cx, int Cy,
                                   int NB, int KC, int c_step, int nchunks, int nb_real, int gblocks, int relu, int stride, double* stats,
                                   cudaStream_t stream) {
  TFB_REQUIRE(x16 && wpack && y && N > 0 && H > 0 && W > 0 && Cx > 0 && Cy > 0 && Cx % 8 == 0 && (stride == 1 || stride == 2));
  TFB_REQUIRE(!stats || (Cy % 4 == 0 && Cy <= 2048 && nb_real % 4 == 0 && !bias && !relu && (reinterpret_cast<uintptr_t>(y) & 15) == 0));
  TFB_REQUIRE((reinterpret_cast<uintptr_t>(x16) & 15) == 0 && (reinterpret_cast<uintptr_t>(wpack) & 15) == 0);
#define CASE(KC_, NB_) if (KC == KC_ && NB == NB_) return launch_conv<KC_, NB_>(x16, wpack, bias, y, N, H, W, Cx, Cy, c_step, nchunks, nb_real, gblocks, relu, stride, stats, stream)
  CASE(64, 16); CASE(64, 32); CASE(64, 48); CASE(64, 64); CASE(64, 128);
  CASE(32, 16); CASE(32, 32); CASE(32, 64);
#undef CASE
  tfb_set_last_error("tfb_conv3x3_tc: unsupported (KC, NB) tile");
  return TFB_ERR_UNSUPPORTED;
}

// Stride-1 form of tfb_conv3x3_tc_strided.
TFB_API int tfb_conv3x3_tc(const void* x16, const void* wpack, const float* bias, float* y, int N, int H, int W, int Cx, int Cy,
                           int NB, int KC, int c_step, int nchunks, int nb_real, int gblocks, int relu, cudaStream_t stream) {
  return tfb_conv3x3_tc_strided(x16, wpack, bias, y, N, H, W, Cx, Cy, NB, KC, c_step, nchunks, nb_real, gblocks, relu, 1, nullptr, stream);
}
