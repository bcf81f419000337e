// Direct (CUDA-core, fp32) NHWC convolutions: k in {1,3}, pad = k/2, stride in {1,2}, arbitrary groups.
// forward / dgrad / wgrad. These are the exact-fp32 kernels for every conv that is not a plain GEMM:
// the stems (Cin = 3), grouped 3x3 of the RegNetY blocks (group width 24), strided 1x1 shortcuts, and the
// dense 3x3 of the heads / decoders. Replaces cuDNN behind nn.Conv2d:
//   timm RegNet blocks (transfuser.py:136-146,159-184), SegDecoder/DepthDecoder (transfuser.py:214-281),
//   pred_bev and CenterNet heads (model.py:581-585, 93-99).
// Weights keep the PyTorch layout [Cout][Cin/groups][k][k].
#include "common.cuh"

namespace {

constexpr int kCiChunk = 32;

// ---------------------------------------------------------------- forward
// thread = one output pixel x CO_T output channels of one group; weights of the current ci-chunk live in smem.
template <int KS, int CO_T>
__global__ void __launch_bounds__(128)
conv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int stride, int groups, int relu) {
  constexpr int T = KS * KS, P = KS / 2;
  __shared__ __align__(16) float ws[T * kCiChunk * CO_T];
  const int Cig = Cin / groups, Cog = Cout / groups;
  const int cob_per_g = (Cog + CO_T - 1) / CO_T;
  const int g = blockIdx.y / cob_per_g, cb = blockIdx.y % cob_per_g;
  const int co0 = cb * CO_T;  // within group
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t npix = (int64_t)N * Ho * Wo;
  const bool active = pix < npix;
  int n = 0, ho = 0, wo = 0;
  if (active) { wo = pix % Wo; ho = (pix / Wo) % Ho; n = pix / ((int64_t)Wo * Ho); }
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;

  for (int ci0 = 0; ci0 < Cig; ci0 += kCiChunk) {
    const int cur = min(kCiChunk, Cig - ci0);
    __syncthreads();
    for (int e = threadIdx.x; e < T * cur * CO_T; e += blockDim.x) {
      int co = e % CO_T, ci = (e / CO_T) % cur, tap = e / (CO_T * cur);
      float v = 0.f;
      if (co0 + co < Cog) v = w[((int64_t)(g * Cog + co0 + co) * Cig + ci0 + ci) * T + tap];
      ws[(tap * kCiChunk + ci) * CO_T + co] = v;
    }
    __syncthreads();
    if (active) {
#pragma unroll
      for (int tap = 0; tap < T; ++tap) {
        const int hi = ho * stride - P + tap / KS, wi = wo * stride - P + tap % KS;
        if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;
        const float* xp = x + (((int64_t)n * H + hi) * W + wi) * Cin + g * Cig + ci0;
        const float* wt = ws + tap * kCiChunk * CO_T;
        for (int ci = 0; ci < cur; ++ci) {
          const float xv = __ldg(xp + ci);
          const float* wr = wt + ci * CO_T;
#pragma unroll
          for (int c = 0; c < CO_T; c += 4) {
            const float4 wv = *reinterpret_cast<const float4*>(wr + c);
            acc[c + 0] = fmaf(xv, wv.x, acc[c + 0]);
            acc[c + 1] = fmaf(xv, wv.y, acc[c + 1]);
            acc[c + 2] = fmaf(xv, wv.z, acc[c + 2]);
            acc[c + 3] = fmaf(xv, wv.w, acc[c + 3]);
          }
        }
      }
    }
  }
  if (active) {
    float* yp = y + pix * Cout + g * Cog + co0;
#pragma unroll
    for (int c = 0; c < CO_T; ++c) {
      if (co0 + c < Cog) {
        float v = acc[c] + (bias ? bias[g * Cog + co0 + c] : 0.f);
        if (relu) v = fmaxf(v, 0.f);
        yp[c] = v;
      }
    }
  }
}

// ---------------------------------------------------------------- dgrad
// thread = one input pixel x CI_T input channels of one group; dx = sum over taps/co of dy * w.
template <int KS, int CI_T>
__global__ void __launch_bounds__(128)
conv_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, int N, int H, int W, int Cin,
                  int Ho, int Wo, int Cout, int stride, int groups) {
  constexpr int T = KS * KS, P = KS / 2;
  __shared__ __align__(16) float ws[T * kCiChunk * CI_T];  // [tap][co][ci]
  const int Cig = Cin / groups, Cog = Cout / groups;
  const int cib_per_g = (Cig + CI_T - 1) / CI_T;
  const int g = blockIdx.y / cib_per_g, cb = blockIdx.y % cib_per_g;
  const int ci0 = cb * CI_T;
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t npix = (int64_t)N * H * W;
  const bool active = pix < npix;
  int n = 0, hi = 0, wi = 0;
  if (active) { wi = pix % W; hi = (pix / W) % H; n = pix / ((int64_t)W * H); }
  float acc[CI_T];
#pragma unroll
  for (int c = 0; c < CI_T; ++c) acc[c] = 0.f;

  for (int co0 = 0; co0 < Cog; co0 += kCiChunk) {
    const int cur = min(kCiChunk, Cog - co0);
    __syncthreads();
    for (int e = threadIdx.x; e < T * cur * CI_T; e += blockDim.x) {
      int ci = e % CI_T, co = (e / CI_T) % cur, tap = e / (CI_T * cur);
      float v = 0.f;
      if (ci0 + ci < Cig) v = w[((int64_t)(g * Cog + co0 + co) * Cig + ci0 + ci) * T + tap];
      ws[(tap * kCiChunk + co) * CI_T + ci] = v;
    }
    __syncthreads();
    if (active) {
#pragma unroll
      for (int tap = 0; tap < T; ++tap) {
        const int hn = hi + P - tap / KS, wn = wi + P - tap % KS;  // = ho*stride, wo*stride
        if (hn < 0 || wn < 0 || (hn % stride) || (wn % stride)) continue;
        const int ho = hn / stride, wo = wn / stride;
        if (ho >= Ho || wo >= Wo) continue;
        const float* dyp = dy + (((int64_t)n * Ho + ho) * Wo + wo) * Cout + g * Cog + co0;
        const float* wt = ws + tap * kCiChunk * CI_T;
        for (int co = 0; co < cur; ++co) {
          const float dv = __ldg(dyp + co);
          const float* wr = wt + co * CI_T;
#pragma unroll
          for (int c = 0; c < CI_T; c += 4) {
            const float4 wv = *reinterpret_cast<const float4*>(wr + c);
            acc[c + 0] = fmaf(dv, wv.x, acc[c + 0]);
            acc[c + 1] = fmaf(dv, wv.y, acc[c + 1]);
            acc[c + 2] = fmaf(dv, wv.z, acc[c + 2]);
            acc[c + 3] = fmaf(dv, wv.w, acc[c + 3]);
          }
        }
      }
    }
  }
  if (active) {
    float* dxp = dx + pix * Cin + g * Cig + ci0;
#pragma unroll
    for (int c = 0; c < CI_T; ++c)
      if (ci0 + c < Cig) dxp[c] = acc[c];
  }
}

// ---------------------------------------------------------------- wgrad
// CTA = (pixel range, 32-wide co block x 32-wide ci block of one group); 16x16 threads, each owning a 2x2 (co,ci) patch for
// all taps. Output pixels are staged 32 at a time: dy rows and the tap-shifted x rows go through smem, partial sums leave
// the CTA with one partial per weight, the pixel splits added in split order (OrderedSum; dw / dbias zeroed by the launcher).
template <int KS>
__global__ void __launch_bounds__(256)
conv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw, float* __restrict__ dbias,
                  int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int stride, int groups, int pix_per_cta, OrderedSum osw,
                  OrderedSum osb) {
  constexpr int T = KS * KS, P = KS / 2, PB = 32, CB = 32;
  __shared__ __align__(16) float sdy[PB][CB + 2];
  __shared__ __align__(16) float sx[T][PB][CB + 2];
  const int Cig = Cin / groups, Cog = Cout / groups;
  const int cob = (Cog + CB - 1) / CB, cib = (Cig + CB - 1) / CB;
  int by = blockIdx.y;
  const int ib = by % cib; by /= cib;
  const int ob = by % cob; by /= cob;
  const int g = by;
  const int co0 = ob * CB, ci0 = ib * CB;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;  // tx -> ci pair, ty -> co pair
  const int64_t npix = (int64_t)N * Ho * Wo;
  const int64_t p_begin = (int64_t)blockIdx.x * pix_per_cta;
  const int64_t p_end = min(npix, p_begin + pix_per_cta);
  float acc[T][4];
#pragma unroll
  for (int t = 0; t < T; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  float bsum = 0.f;  // dbias partial: threads with ty == 0 ... handled via sdy column sums below

  for (int64_t p0 = p_begin; p0 < p_end; p0 += PB) {
    __syncthreads();
    // stage dy[p][co]
    for (int e = threadIdx.x; e < PB * CB; e += 256) {
      int c = e % CB, pp = e / CB;
      int64_t p = p0 + pp;
      float v = 0.f;
      if (p < p_end && co0 + c < Cog) v = dy[p * Cout + g * Cog + co0 + c];
      sdy[pp][c] = v;
    }
    // stage x[tap][p][ci]
    for (int e = threadIdx.x; e < T * PB * CB; e += 256) {
      int c = e % CB, pp = (e / CB) % PB, tap = e / (CB * PB);
      int64_t p = p0 + pp;
      float v = 0.f;
      if (p < p_end && ci0 + c < Cig) {
        int wo = p % Wo, ho = (p / Wo) % Ho, n = p / ((int64_t)Wo * Ho);
        int hi = ho * stride - P + tap / KS, wi = wo * stride - P + tap % KS;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W) v = x[(((int64_t)n * H + hi) * W + wi) * Cin + g * Cig + ci0 + c];
      }
      sx[tap][pp][c] = v;
    }
    __syncthreads();
    if (dbias && ib == 0 && threadIdx.x < CB) {
      float s = 0.f;
#pragma unroll 8
      for (int pp = 0; pp < PB; ++pp) s += sdy[pp][threadIdx.x];
      bsum += s;
    }
#pragma unroll 4
    for (int pp = 0; pp < PB; ++pp) {
      const float2 d = *reinterpret_cast<const float2*>(&sdy[pp][ty * 2]);
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const float2 xv = *reinterpret_cast<const float2*>(&sx[t][pp][tx * 2]);
        acc[t][0] = fmaf(d.x, xv.x, acc[t][0]);
        acc[t][1] = fmaf(d.x, xv.y, acc[t][1]);
        acc[t][2] = fmaf(d.y, xv.x, acc[t][2]);
        acc[t][3] = fmaf(d.y, xv.y, acc[t][3]);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < T; ++t) {
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        int co = co0 + ty * 2 + a, ci = ci0 + tx * 2 + b;
        if (co < Cog && ci < Cig) ordered_store(osw, blockIdx.x, ((int64_t)(g * Cog + co) * Cig + ci) * T + t, acc[t][a * 2 + b]);
      }
    }
  }
  if (dbias && ib == 0 && threadIdx.x < CB && co0 + threadIdx.x < Cog) ordered_store(osb, blockIdx.x, g * Cog + co0 + threadIdx.x, bsum);
  ordered_finish(osw, dw);
  if (dbias) ordered_finish(osb, dbias);
}

// ---------------------------------------------------------------- wgrad, few input channels (the two stems: Cin = 3)
// The generic kernel above tiles 32 ci x 32 co per CTA: with 3 input channels 29/32 of its lanes and of its smem staging are padding
// (0.5 TFLOP/s measured on the 160x704 stem). Here a WARP owns one output pixel at a time and its 32 lanes own 32 output channels:
// dy[p][co] is one coalesced 128-byte load, the <= 4 x KS*KS tap-shifted inputs are warp-uniform (broadcast) loads, and every lane keeps
// its [ci][tap] accumulators in registers. The 8 warps of a CTA meet in shared memory; one partial per weight and CTA (OrderedSum).
template <int KS>
__global__ void __launch_bounds__(256)
conv_wgrad_smallcin_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw, float* __restrict__ dbias,
                           int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int stride, int pix_per_cta, OrderedSum osw,
                           OrderedSum osb) {
  constexpr int T = KS * KS, P = KS / 2, CI = 4, NW = 8;
  __shared__ float red[NW][32][CI * T + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int co = blockIdx.y * 32 + lane;
  const bool co_ok = co < Cout;
  const int64_t npix = (int64_t)N * Ho * Wo;
  const int64_t p_begin = (int64_t)blockIdx.x * pix_per_cta;
  const int64_t p_end = min(npix, p_begin + pix_per_cta);
  float acc[CI][T];
#pragma unroll
  for (int c = 0; c < CI; ++c)
#pragma unroll
    for (int t = 0; t < T; ++t) acc[c][t] = 0.f;
  float bsum = 0.f;
  for (int64_t p = p_begin + warp; p < p_end; p += NW) {
    const int wo = (int)(p % Wo), ho = (int)((p / Wo) % Ho), n = (int)(p / ((int64_t)Wo * Ho));
    const float d = co_ok ? dy[p * Cout + co] : 0.f;
    bsum += d;
#pragma unroll
    for (int t = 0; t < T; ++t) {
      const int hi = ho * stride - P + t / KS, wi = wo * stride - P + t % KS;
      if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;          // warp-uniform branch
      const float* xp = x + (((int64_t)n * H + hi) * W + wi) * Cin;
#pragma unroll
      for (int c = 0; c < CI; ++c)
        if (c < Cin) acc[c][t] = fmaf(d, __ldg(xp + c), acc[c][t]);
    }
  }
#pragma unroll
  for (int c = 0; c < CI; ++c)
#pragma unroll
    for (int t = 0; t < T; ++t) red[warp][lane][c * T + t] = acc[c][t];
  red[warp][lane][CI * T] = bsum;
  __syncthreads();
  const int nout = 32 * (CI * T + 1);
  for (int e = threadIdx.x; e < nout; e += blockDim.x) {
    const int l = e / (CI * T + 1), k = e % (CI * T + 1);
    const int oc = blockIdx.y * 32 + l;
    if (oc >= Cout) continue;
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < NW; ++w8) s += red[w8][l][k];
    if (k == CI * T) {
      if (dbias) ordered_store(osb, blockIdx.x, oc, s);
    } else {
      const int c = k / T, t = k % T;
      if (c < Cin) ordered_store(osw, blockIdx.x, ((int64_t)oc * Cin + c) * T + t, s);
    }
  }
  ordered_finish(osw, dw);
  if (dbias) ordered_finish(osb, dbias);
}

// ---------------------------------------------------------------- wgrad of a 1x1 conv with few OUTPUT channels (CenterNet head
// outputs: 64 -> {1, 2, 3, 12}). dW[co][ci] = sum_p dy[p][co] x[p][ci]: the generic 32 x 32 tile wastes up to 31/32 of its lanes
// (0.09 TFLOP/s measured for Cout = 1). Here 64 consecutive threads own 64 input channels (x[p][ci..] is one coalesced 256-byte
// load), the <= 16 dy values of the pixel are block-uniform (broadcast) loads, each thread keeps its [co] accumulators in registers;
// the 4 pixel phases of a CTA meet in shared memory, one partial per weight and CTA (OrderedSum).
__global__ void __launch_bounds__(256)
conv1x1_wgrad_narrowout_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw,
                               float* __restrict__ dbias, int64_t npix, int Cin, int Cout, int pix_per_cta, OrderedSum osw, OrderedSum osb) {
  constexpr int CO = 16, CB = 64, NP = 4;
  __shared__ float red[NP][CB][CO + 1];
  const int cl = threadIdx.x % CB, ph = threadIdx.x / CB;
  const int ci = blockIdx.y * CB + cl;
  const bool ci_ok = ci < Cin;
  const int64_t p_begin = (int64_t)blockIdx.x * pix_per_cta;
  const int64_t p_end = min(npix, p_begin + pix_per_cta);
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
  for (int64_t p = p_begin + ph; p < p_end; p += NP) {
    const float xv = ci_ok ? x[p * Cin + ci] : 0.f;
    const float* d = dy + p * Cout;
#pragma unroll
    for (int c = 0; c < CO; ++c)
      if (c < Cout) acc[c] = fmaf(__ldg(d + c), xv, acc[c]);
  }
#pragma unroll
  for (int c = 0; c < CO; ++c) red[ph][cl][c] = acc[c];
  __syncthreads();
  for (int e = threadIdx.x; e < CB * CO; e += blockDim.x) {
    const int c = e / CB, l = e % CB;                    // l fastest: consecutive threads -> consecutive ci of one co row
    const int cc = blockIdx.y * CB + l;
    if (c >= Cout || cc >= Cin) continue;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NP; ++j) s += red[j][l][c];
    ordered_store(osw, blockIdx.x, (int64_t)c * Cin + cc, s);
  }
  if (dbias && blockIdx.y == 0) {                        // dbias[co] = sum_p dy[p][co]: the CTA's pixel range, 16 threads x strided pixels
    __syncthreads();
    float* bs = &red[0][0][0];
    if (threadIdx.x < 256) {
      const int c = threadIdx.x % CO, q = threadIdx.x / CO;   // 16 pixel phases
      float s = 0.f;
      if (c < Cout)
        for (int64_t p = p_begin + q; p < p_end; p += 16) s += dy[p * Cout + c];
      bs[q * CO + c] = s;
    }
    __syncthreads();
    if (threadIdx.x < Cout) {
      float s = 0.f;
      for (int q = 0; q < 16; ++q) s += bs[q * CO + threadIdx.x];
      ordered_store(osb, blockIdx.x, threadIdx.x, s);
    }
  }
  ordered_finish(osw, dw);
  if (dbias) ordered_finish(osb, dbias);
}

template <int KS>
int launch_fwd(const float* x, const float* w, const float* bias, float* y, int N, int H, int W, int Cin, int Ho, int Wo, int Cout,
               int stride, int groups, int relu, cudaStream_t stream) {
  const int Cog = Cout / groups;
  const int64_t npix = (int64_t)N * Ho * Wo;
  const unsigned gx = (unsigned)ceil_div64(npix, 128);
#define FWD(CT)                                                                                                   \
  {                                                                                                               \
    dim3 grid(gx, groups * ((Cog + CT - 1) / CT));                                                                \
    conv_fwd_kernel<KS, CT><<<grid, 128, 0, stream>>>(x, w, bias, y, N, H, W, Cin, Ho, Wo, Cout, stride, groups, relu); \
  }
  if (Cog <= 8) FWD(8) else if (Cog <= 16) FWD(16) else if (Cog % 24 == 0 && Cog % 32 != 0) FWD(24) else FWD(32)
#undef FWD
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

template <int KS>
int launch_dgrad(const float* dy, const float* w, float* dx, int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int stride,
                 int groups, cudaStream_t stream) {
  const int Cig = Cin / groups;
  const int64_t npix = (int64_t)N * H * W;
  const unsigned gx = (unsigned)ceil_div64(npix, 128);
#define DG(CT)                                                                                             \
  {                                                                                                        \
    dim3 grid(gx, groups * ((Cig + CT - 1) / CT));                                                         \
    conv_dgrad_kernel<KS, CT><<<grid, 128, 0, stream>>>(dy, w, dx, N, H, W, Cin, Ho, Wo, Cout, stride, groups); \
  }
  if (Cig <= 8) DG(8) else if (Cig <= 16) DG(16) else if (Cig % 24 == 0 && Cig % 32 != 0) DG(24) else DG(32)
#undef DG
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

template <int KS>
int launch_wgrad(const float* x, const float* dy, float* dw, float* dbias, int N, int H, int W, int Cin, int Ho, int Wo, int Cout,
                 int stride, int groups, cudaStream_t stream) {
  const int Cig = Cin / groups, Cog = Cout / groups;
  const int64_t npix = (int64_t)N * Ho * Wo;
  const int by = groups * ((Cog + 31) / 32) * ((Cig + 31) / 32);
  // enough pixel splits for ~4 waves of CTAs, each CTA at least 256 pixels
  int64_t splits = (4LL * tfb_num_sms() + by - 1) / by;
  int64_t ppc = ceil_div64(npix, splits);
  if (ppc < 256) ppc = 256;
  ppc = ceil_div64(ppc, 32) * 32;
  splits = ceil_div64(npix, ppc);
  if (cudaMemsetAsync(dw, 0, (size_t)Cout * Cig * KS * KS * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  if (dbias && cudaMemsetAsync(dbias, 0, (size_t)Cout * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  // the pixel splits' partial weight / bias gradients, added in split order (the same bits every run)
  TfbScratch wk;
  OrderedSum osw, osb;
  auto partials = [&](int64_t nsplit) -> int {
    const int64_t ndw = (int64_t)Cout * Cig * KS * KS;
    const int rc = tfb_scratch(wk, (size_t)(nsplit * (ndw + Cout)), 2, stream);
    // weight gradients larger than one CTA's share are summed by a grid-wide ordered_sum_kernel after the launch
    osw = OrderedSum{wk.f, ndw > 16384 ? nullptr : wk.cnt, (int)nsplit, ndw};
    osb = OrderedSum{wk.f + nsplit * ndw, wk.cnt + 1, (int)nsplit, Cout};
    return rc;
  };
  auto finish = [&]() -> int {
    TFB_CHECK_LAUNCH();
    if (!osw.cnt) {
      ordered_sum_kernel<<<tfb_grid(osw.n_out, 256), 256, 0, stream>>>(osw.part, osw.nsplit, osw.n_out, dw);
      TFB_CHECK_LAUNCH();
    }
    return TFB_OK;
  };
  if (groups == 1 && KS == 1 && stride == 1 && Cout <= 16) {
    // narrow-output 1x1 conv (head outputs): threads over input channels, dy broadcast (see conv1x1_wgrad_narrowout_kernel)
    const int cib64 = (Cin + 63) / 64;
    int64_t sp = (4LL * tfb_num_sms() + cib64 - 1) / cib64;
    int64_t pp = ceil_div64(npix, sp);
    if (pp < 128) pp = 128;
    pp = ceil_div64(pp, 16) * 16;
    dim3 grid2((unsigned)ceil_div64(npix, pp), cib64);
    const int rc = partials(grid2.x);
    if (rc != TFB_OK) return rc;
    conv1x1_wgrad_narrowout_kernel<<<grid2, 256, 0, stream>>>(x, dy, dw, dbias, npix, Cin, Cout, (int)pp, osw, osb);
    return finish();
  }
  if (groups == 1 && Cin <= 4 && KS == 3) {
    // stems: one warp per pixel, lanes over output channels (see conv_wgrad_smallcin_kernel); ~4 waves of CTAs, >= 256 pixels each
    const int cob32 = (Cout + 31) / 32;
    int64_t sp = (4LL * tfb_num_sms() + cob32 - 1) / cob32;
    int64_t pp = ceil_div64(npix, sp);
    if (pp < 256) pp = 256;
    pp = ceil_div64(pp, 8) * 8;
    dim3 grid2((unsigned)ceil_div64(npix, pp), cob32);
    const int rc = partials(grid2.x);
    if (rc != TFB_OK) return rc;
    conv_wgrad_smallcin_kernel<KS><<<grid2, 256, 0, stream>>>(x, dy, dw, dbias, N, H, W, Cin, Ho, Wo, Cout, stride, (int)pp, osw, osb);
    return finish();
  }
  dim3 grid((unsigned)splits, by);
  const int rc = partials(grid.x);
  if (rc != TFB_OK) return rc;
  conv_wgrad_kernel<KS><<<grid, 256, 0, stream>>>(x, dy, dw, dbias, N, H, W, Cin, Ho, Wo, Cout, stride, groups, (int)ppc, osw, osb);
  return finish();
}

bool conv_args_ok(int N, int H, int W, int Cin, int Cout, int ksize, int stride, int groups) {
  return N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && (ksize == 1 || ksize == 3) && (stride == 1 || stride == 2) &&
         groups > 0 && Cin % groups == 0 && Cout % groups == 0;
}

}  // namespace

TFB_API int tfb_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int N, int H, int W, int Cin, int Cout,
                           int ksize, int stride, int groups, int relu, cudaStream_t stream) {
  TFB_REQUIRE(x && w && y && conv_args_ok(N, H, W, Cin, Cout, ksize, stride, groups));
  const int Ho = (H + 2 * (ksize / 2) - ksize) / stride + 1, Wo = (W + 2 * (ksize / 2) - ksize) / stride + 1;
  if (ksize == 3) return launch_fwd<3>(x, w, bias, y, N, H, W, Cin, Ho, Wo, Cout, stride, groups, relu, stream);
  return launch_fwd<1>(x, w, bias, y, N, H, W, Cin, Ho, Wo, Cout, stride, groups, relu, stream);
}

TFB_API int tfb_conv2d_dgrad(const float* dy, const float* w, float* dx, int N, int H, int W, int Cin, int Cout, int ksize,
                             int stride, int groups, cudaStream_t stream) {
  TFB_REQUIRE(dy && w && dx && conv_args_ok(N, H, W, Cin, Cout, ksize, stride, groups));
  const int Ho = (H + 2 * (ksize / 2) - ksize) / stride + 1, Wo = (W + 2 * (ksize / 2) - ksize) / stride + 1;
  if (ksize == 3) return launch_dgrad<3>(dy, w, dx, N, H, W, Cin, Ho, Wo, Cout, stride, groups, stream);
  return launch_dgrad<1>(dy, w, dx, N, H, W, Cin, Ho, Wo, Cout, stride, groups, stream);
}

TFB_API int tfb_conv2d_wgrad(const float* x, const float* dy, float* dw, float* dbias, int N, int H, int W, int Cin, int Cout,
                             int ksize, int stride, int groups, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dw && conv_args_ok(N, H, W, Cin, Cout, ksize, stride, groups));
  const int Ho = (H + 2 * (ksize / 2) - ksize) / stride + 1, Wo = (W + 2 * (ksize / 2) - ksize) / stride + 1;
  if (ksize == 3) return launch_wgrad<3>(x, dy, dw, dbias, N, H, W, Cin, Ho, Wo, Cout, stride, groups, stream);
  return launch_wgrad<1>(x, dy, dw, dbias, N, H, W, Cin, Ho, Wo, Cout, stride, groups, stream);
}
