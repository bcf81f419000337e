// The ResNet stem (timm resnet18 / resnet34: conv1 -> bn1 -> act1 -> maxpool, transfuser.py:136-143), NHWC fp32:
//   - the 7x7 / stride-2 / pad-3 convolution of an input with at most 4 channels: forward and weight gradient. The generic direct
//     kernels of conv_simt.cu stage 32-channel weight chunks per tap, which at 49 taps is far beyond the shared memory a CTA has;
//     with <= 4 input channels the whole [tap][ci][32 co] slice fits (25 KB). No dgrad: neither trunk input needs a gradient.
//   - the 3x3 / stride-2 / pad-1 max-pool with PyTorch's semantics, forward (fp32 output, optional bf16 copy, one-byte argmax tap)
//     and backward as a gather over the <= 4 windows that can select an input element.
// Exact fp32 on the CUDA cores in every numerics mode, as the 3x3 stems of the RegNet trunk.
#include "common.cuh"

namespace {

constexpr int kKS = 7, kTaps = kKS * kKS, kPad = 3, kCinMax = 4, kCoT = 32;

// forward: thread = one output pixel x 32 output channels; the CTA's 32-channel weight slice lives in shared memory as
// [tap][ci][co], so each fused multiply-add pair of the inner loop reads one broadcast float4.
template <int CIN>
__global__ void __launch_bounds__(128)
stem7_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int N, int H, int W, int Ho, int Wo,
                 int Cout) {
  __shared__ __align__(16) float ws[kTaps * CIN * kCoT];
  const int co0 = blockIdx.y * kCoT;
  for (int e = threadIdx.x; e < kTaps * CIN * kCoT; e += blockDim.x) {
    const int co = e % kCoT, ci = (e / kCoT) % CIN, tap = e / (kCoT * CIN);
    ws[e] = co0 + co < Cout ? w[((int64_t)(co0 + co) * CIN + ci) * kTaps + tap] : 0.f;
  }
  __syncthreads();
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (int64_t)N * Ho * Wo) return;
  const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), n = (int)(pix / ((int64_t)Wo * Ho));
  float acc[kCoT];
#pragma unroll
  for (int c = 0; c < kCoT; ++c) acc[c] = 0.f;
  for (int kh = 0; kh < kKS; ++kh) {
    const int hi = ho * 2 - kPad + kh;
    if (hi < 0 || hi >= H) continue;
    for (int kw = 0; kw < kKS; ++kw) {
      const int wi = wo * 2 - kPad + kw;
      if (wi < 0 || wi >= W) continue;
      const float* xp = x + (((int64_t)n * H + hi) * W + wi) * CIN;
      const float* wt = ws + (kh * kKS + kw) * CIN * kCoT;
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        const float xv = __ldg(xp + ci);
#pragma unroll
        for (int c = 0; c < kCoT; c += 4) {
          const float4 wv = *reinterpret_cast<const float4*>(wt + ci * kCoT + c);
          acc[c + 0] = fmaf(xv, wv.x, acc[c + 0]);
          acc[c + 1] = fmaf(xv, wv.y, acc[c + 1]);
          acc[c + 2] = fmaf(xv, wv.z, acc[c + 2]);
          acc[c + 3] = fmaf(xv, wv.w, acc[c + 3]);
        }
      }
    }
  }
  float* yp = y + pix * Cout + co0;
#pragma unroll
  for (int c = 0; c < kCoT; ++c)
    if (co0 + c < Cout) yp[c] = acc[c];
}

// weight gradient: dW[co][ci][kh][kw] = sum_p dy[p][co] x[p shifted by (kh, kw)][ci]. CTA = (pixel split, 32 output channels, one
// kernel row kh); a warp takes one output pixel at a time and its 32 lanes the 32 output channels (dy[p][co] is one coalesced
// 128-byte load, the 7 x CIN inputs are warp-uniform loads), each lane keeps its [ci][kw] accumulators in registers. The 8 warps
// meet in shared memory in warp order; one partial per weight and split, folded in split order after the launch.
template <int CIN>
__global__ void __launch_bounds__(256)
stem7_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ part, int N, int H, int W, int Ho,
                   int Wo, int Cout, int pix_per_cta) {
  constexpr int NW = 8, K = CIN * kKS;
  __shared__ float red[NW][32][K + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, kh = blockIdx.z;
  const int co = blockIdx.y * 32 + lane;
  const bool co_ok = co < Cout;
  const int64_t npix = (int64_t)N * Ho * Wo;
  const int64_t p_begin = (int64_t)blockIdx.x * pix_per_cta;
  const int64_t p_end = min(npix, p_begin + pix_per_cta);
  float acc[CIN][kKS];
#pragma unroll
  for (int c = 0; c < CIN; ++c)
#pragma unroll
    for (int t = 0; t < kKS; ++t) acc[c][t] = 0.f;
  for (int64_t p = p_begin + warp; p < p_end; p += NW) {
    const int wo = (int)(p % Wo), ho = (int)((p / Wo) % Ho), n = (int)(p / ((int64_t)Wo * Ho));
    const int hi = ho * 2 - kPad + kh;
    if (hi < 0 || hi >= H) continue;                                   // warp-uniform
    const float d = co_ok ? dy[p * Cout + co] : 0.f;
    const float* xr = x + ((int64_t)n * H + hi) * W * CIN;
#pragma unroll
    for (int kw = 0; kw < kKS; ++kw) {
      const int wi = wo * 2 - kPad + kw;
      if (wi < 0 || wi >= W) continue;                                 // warp-uniform
#pragma unroll
      for (int c = 0; c < CIN; ++c) acc[c][kw] = fmaf(d, __ldg(xr + (int64_t)wi * CIN + c), acc[c][kw]);
    }
  }
#pragma unroll
  for (int c = 0; c < CIN; ++c)
#pragma unroll
    for (int t = 0; t < kKS; ++t) red[warp][lane][c * kKS + t] = acc[c][t];
  __syncthreads();
  const int64_t n_out = (int64_t)Cout * CIN * kTaps;
  for (int e = threadIdx.x; e < 32 * K; e += blockDim.x) {
    const int l = e / K, k = e % K;
    const int oc = blockIdx.y * 32 + l;
    if (oc >= Cout) continue;
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < NW; ++w8) s += red[w8][l][k];
    const int c = k / kKS, kw = k % kKS;
    part[(int64_t)blockIdx.x * n_out + ((int64_t)oc * CIN + c) * kTaps + kh * kKS + kw] = s;
  }
}

template <int CIN>
int stem7_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Ho, int Wo, int Cout, cudaStream_t stream) {
  dim3 grid((unsigned)ceil_div64((int64_t)N * Ho * Wo, 128), (Cout + kCoT - 1) / kCoT);
  stem7_fwd_kernel<CIN><<<grid, 128, 0, stream>>>(x, w, y, N, H, W, Ho, Wo, Cout);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

template <int CIN>
int stem7_wgrad(const float* x, const float* dy, float* dw, int N, int H, int W, int Ho, int Wo, int Cout, cudaStream_t stream) {
  const int64_t npix = (int64_t)N * Ho * Wo;
  const int cob32 = (Cout + 31) / 32;
  // ~4 waves of CTAs over (split, channel block, kernel row), at least 256 pixels per CTA
  int64_t sp = (4LL * tfb_num_sms() + cob32 * kKS - 1) / (cob32 * kKS);
  int64_t pp = ceil_div64(npix, sp);
  if (pp < 256) pp = 256;
  pp = ceil_div64(pp, 8) * 8;
  const int64_t nsplit = ceil_div64(npix, pp);
  const int64_t n_out = (int64_t)Cout * CIN * kTaps;
  TfbScratch wk;
  const int rc = tfb_scratch(wk, (size_t)(nsplit * n_out), 0, stream);
  if (rc != TFB_OK) return rc;
  dim3 grid((unsigned)nsplit, cob32, kKS);
  stem7_wgrad_kernel<CIN><<<grid, 256, 0, stream>>>(x, dy, wk.f, N, H, W, Ho, Wo, Cout, (int)pp);
  TFB_CHECK_LAUNCH();
  // the splits' partials added in split order, starting from +0 (assign): the same bits every run, no clearing pass over dw
  ordered_sum_kernel<<<tfb_grid(n_out, 256), 256, 0, stream>>>(wk.f, (int)nsplit, n_out, dw, true);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// max-pool forward: thread = one output pixel x 4 channels. Taps in row-major window order; a value replaces the running maximum
// when it is greater or NaN (PyTorch's rule: padding is -inf and never wins, the first of equal maxima is kept, NaN propagates).
// The argmax starts at the first in-bounds tap, as in PyTorch, so a window of -inf values selects that tap.
__global__ void __launch_bounds__(256)
maxpool3s2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, __nv_bfloat16* __restrict__ y16, uint8_t* __restrict__ arg,
                      int N, int H, int W, int C, int Ho, int Wo) {
  const int C4 = C / 4;
  const int64_t total = (int64_t)N * Ho * Wo * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t pix = i / C4;
    const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), n = (int)(pix / ((int64_t)Wo * Ho));
    const int first = (ho == 0 ? 3 : 0) + (wo == 0 ? 1 : 0);          // the first in-bounds tap (row 0 / column 0 is padding)
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int a[4] = {first, first, first, first};
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = ho * 2 - 1 + kh;
      if (hi < 0 || hi >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wo * 2 - 1 + kw;
        if (wi < 0 || wi >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((int64_t)n * H + hi) * W + wi) * C) + c4);
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (vv[j] > m[j] || vv[j] != vv[j]) {          // greater, or NaN
            m[j] = vv[j];
            a[j] = kh * 3 + kw;
          }
        }
      }
    }
    reinterpret_cast<float4*>(y)[i] = make_float4(m[0], m[1], m[2], m[3]);
    if (y16) tfb_store_bf16x4(y16, i, m[0], m[1], m[2], m[3]);
    reinterpret_cast<uint32_t*>(arg)[i] = (uint32_t)a[0] | (uint32_t)a[1] << 8 | (uint32_t)a[2] << 16 | (uint32_t)a[3] << 24;
  }
}

// max-pool backward as a gather: thread = one input pixel x 4 channels. The windows (ho, wo) whose 3x3 / stride-2 / pad-1 window
// holds (hi, wi) are ho in [(hi - 1) / 2 rounded up, (hi + 1) / 2] (<= 2 per axis). Their gradients are added to +0 in increasing
// (ho, wo) order when their argmax tap is this element: the order in which PyTorch's CPU backward accumulates into a zeroed dx.
__global__ void __launch_bounds__(256)
maxpool3s2_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ arg, float* __restrict__ dx, int N, int H, int W, int C,
                      int Ho, int Wo) {
  const int C4 = C / 4;
  const int64_t total = (int64_t)N * H * W * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t pix = i / C4;
    const int wi = (int)(pix % W), hi = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    const int ho0 = hi / 2, wo0 = wi / 2;               // = ceil((hi - 1) / 2) for hi >= 0
    for (int ho = ho0; ho <= min((hi + 1) / 2, Ho - 1); ++ho) {
      const int kh = hi - (ho * 2 - 1);
      for (int wo = wo0; wo <= min((wi + 1) / 2, Wo - 1); ++wo) {
        const int tap = kh * 3 + (wi - (wo * 2 - 1));
        const int64_t o = (((int64_t)n * Ho + ho) * Wo + wo) * C4 + c4;
        const uint32_t t = __ldg(reinterpret_cast<const uint32_t*>(arg) + o);     // the 4 channels' taps, one byte each
        const bool hit[4] = {(t & 0xff) == (uint32_t)tap, (t >> 8 & 0xff) == (uint32_t)tap, (t >> 16 & 0xff) == (uint32_t)tap,
                             (t >> 24) == (uint32_t)tap};
        if (!(hit[0] || hit[1] || hit[2] || hit[3])) continue;
        const float4 g = __ldg(reinterpret_cast<const float4*>(dy) + o);
        if (hit[0]) s[0] += g.x;
        if (hit[1]) s[1] += g.y;
        if (hit[2]) s[2] += g.z;
        if (hit[3]) s[3] += g.w;
      }
    }
    reinterpret_cast<float4*>(dx)[i] = make_float4(s[0], s[1], s[2], s[3]);
  }
}

// p is a multiple of `bytes` (a null optional operand counts as aligned)
inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

}  // namespace

TFB_API int tfb_conv7x7s2_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, cudaStream_t stream) {
  TFB_REQUIRE(x && w && y && N > 0 && H > 0 && W > 0 && Cin >= 1 && Cin <= kCinMax && Cout > 0);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  switch (Cin) {
    case 1: return stem7_fwd<1>(x, w, y, N, H, W, Ho, Wo, Cout, stream);
    case 2: return stem7_fwd<2>(x, w, y, N, H, W, Ho, Wo, Cout, stream);
    case 3: return stem7_fwd<3>(x, w, y, N, H, W, Ho, Wo, Cout, stream);
    default: return stem7_fwd<4>(x, w, y, N, H, W, Ho, Wo, Cout, stream);
  }
}

TFB_API int tfb_conv7x7s2_wgrad(const float* x, const float* dy, float* dw, int N, int H, int W, int Cin, int Cout, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dw && N > 0 && H > 0 && W > 0 && Cin >= 1 && Cin <= kCinMax && Cout > 0);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  switch (Cin) {
    case 1: return stem7_wgrad<1>(x, dy, dw, N, H, W, Ho, Wo, Cout, stream);
    case 2: return stem7_wgrad<2>(x, dy, dw, N, H, W, Ho, Wo, Cout, stream);
    case 3: return stem7_wgrad<3>(x, dy, dw, N, H, W, Ho, Wo, Cout, stream);
    default: return stem7_wgrad<4>(x, dy, dw, N, H, W, Ho, Wo, Cout, stream);
  }
}

// C % 4 == 0; x and y 16-byte aligned, argmax_u8 4-byte aligned, y16_bf16 8-byte aligned (four channels per access).
TFB_API int tfb_maxpool3x3s2_fwd(const float* x, float* y, void* y16_bf16, void* argmax_u8, int N, int H, int W, int C, cudaStream_t stream) {
  TFB_REQUIRE(x && y && argmax_u8 && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(aligned(x, 16) && aligned(y, 16) && aligned(argmax_u8, 4) && aligned(y16_bf16, 8));
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  maxpool3s2_fwd_kernel<<<tfb_grid((int64_t)N * Ho * Wo * (C / 4), 256), 256, 0, stream>>>(
      x, y, static_cast<__nv_bfloat16*>(y16_bf16), static_cast<uint8_t*>(argmax_u8), N, H, W, C, Ho, Wo);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// C % 4 == 0; dy and dx 16-byte aligned, argmax_u8 4-byte aligned (four channels per access).
TFB_API int tfb_maxpool3x3s2_bwd(const float* dy, const void* argmax_u8, float* dx, int N, int H, int W, int C, cudaStream_t stream) {
  TFB_REQUIRE(dy && argmax_u8 && dx && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(aligned(dy, 16) && aligned(dx, 16) && aligned(argmax_u8, 4));
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  maxpool3s2_bwd_kernel<<<tfb_grid((int64_t)N * H * W * (C / 4), 256), 256, 0, stream>>>(
      dy, static_cast<const uint8_t*>(argmax_u8), dx, N, H, W, C, Ho, Wo);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
