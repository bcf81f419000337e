// HBM-bound NHWC elementwise / gather kernels of the TransFuser backbone, forward + backward:
// residual add+ReLU, SE pooling / gating, input normalisation, layout transposes, adaptive-avg-pool token build,
// the GPT-output "view quirk" + bilinear upsample + add, generic bilinear upsample, dropout, row softmax, bf16 cast.
// Reference call sites: transfuser.py:129-130 (normalize_imagenet), 150-157 (avgpool, GPT, interpolate, add),
// 346-364 (token build / output view), 519-522 (softmax, dropout); timm SEModule / Bottleneck add+ReLU.
#include <assert.h>

#include "common.cuh"

namespace {

// p is a multiple of `bytes` (a null optional operand counts as aligned)
inline bool tfb_aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

__global__ void __launch_bounds__(256) add_relu_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y,
                                                       int64_t n, int relu, __nv_bfloat16* __restrict__ y16) {
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
    float4 o = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    reinterpret_cast<float4*>(y)[i] = o;
    if (y16) tfb_store_bf16x4(y16, i, o.x, o.y, o.z, o.w);
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float o = a[i] + b[i];
    o = relu ? fmaxf(o, 0.f) : o;
    y[i] = o;
    if (y16) y16[i] = __float2bfloat16_rn(o);
  }
}

// MODE 0: dx = dy * (y > 0)   MODE 1: dx = dy * y * (1 - y)   MODE 2: y = sigmoid(x) (dy unused)
template <int MODE>
__global__ void __launch_bounds__(256) act_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx,
                                                  int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[i];
    if (MODE == 0) dx[i] = v > 0.f ? dy[i] : 0.f;
    else if (MODE == 1) dx[i] = dy[i] * v * (1.f - v);
    else dx[i] = 1.f / (1.f + expf(-v));
  }
}

// out[n][c] (+)= scale * sum_p x[n][p][c] (MODE 0)  or  sum_p x[n][p][c] * z[n][p][c] (MODE 1: SE gate gradient)
// block (32 channel quads, 8 row phases); grid (quad slabs, n, HW splits); the splits' partial sums are added in split order
// (OrderedSum; out zeroed).
template <int MODE>
__global__ void __launch_bounds__(256) pool_hw_kernel(const float* __restrict__ x, const float* __restrict__ z, float* __restrict__ out,
                                                      int HW, int C, float scale, OrderedSum os) {
  __shared__ float4 sm[8][33];
  const int n = blockIdx.y, c = (blockIdx.x * 32 + threadIdx.x) * 4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const float* xp = x + (int64_t)n * HW * C + c;
    const float* zp = MODE == 1 ? z + (int64_t)n * HW * C + c : nullptr;
    for (int p = blockIdx.z * 8 + threadIdx.y; p < HW; p += gridDim.z * 8) {
      const float4 v = *reinterpret_cast<const float4*>(xp + (int64_t)p * C);
      if (MODE == 0) { a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
      else {
        const float4 w = *reinterpret_cast<const float4*>(zp + (int64_t)p * C);
        a.x = fmaf(v.x, w.x, a.x); a.y = fmaf(v.y, w.y, a.y); a.z = fmaf(v.z, w.z, a.z); a.w = fmaf(v.w, w.w, a.w);
      }
    }
  }
  sm[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = sm[j][threadIdx.x]; t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w; }
    const int64_t o = (int64_t)n * C + c;
    ordered_store(os, blockIdx.z, o + 0, t.x * scale); ordered_store(os, blockIdx.z, o + 1, t.y * scale);
    ordered_store(os, blockIdx.z, o + 2, t.z * scale); ordered_store(os, blockIdx.z, o + 3, t.w * scale);
  }
  ordered_finish(os, out);
}

// pool_hw_kernel for narrow maps (C / 4 <= 128 channel quads): a block covers 256 / C4 whole pixel rows of ONE sample per iteration,
// consecutive threads read consecutive 16-byte quads (every lane busy: the 32-quad slabs above idle 44 % of the lanes at C = 72);
// grid (splits over the pixels, n).
template <int MODE>
__global__ void __launch_bounds__(256) pool_hw_flat_kernel(const float* __restrict__ x, const float* __restrict__ z, float* __restrict__ out,
                                                           int HW, int C, float scale, OrderedSum os) {
  const int C4 = C / 4, RPB = 256 / C4;
  const int t = threadIdx.x, q = t % C4, rr = t / C4, n = blockIdx.y;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rr < RPB) {
    const float* xp = x + (int64_t)n * HW * C + q * 4;
    const float* zp = MODE == 1 ? z + (int64_t)n * HW * C + q * 4 : nullptr;
    for (int p = blockIdx.x * RPB + rr; p < HW; p += gridDim.x * RPB) {
      const float4 v = *reinterpret_cast<const float4*>(xp + (int64_t)p * C);
      if (MODE == 0) { a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
      else {
        const float4 w = *reinterpret_cast<const float4*>(zp + (int64_t)p * C);
        a.x = fmaf(v.x, w.x, a.x); a.y = fmaf(v.y, w.y, a.y); a.z = fmaf(v.z, w.z, a.z); a.w = fmaf(v.w, w.w, a.w);
      }
    }
  }
  __shared__ float4 sm[256];
  sm[t] = rr < RPB ? a : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  if (t < C4) {
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < RPB; ++j) { const float4 v = sm[j * C4 + t]; s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w; }
    const int64_t o = (int64_t)n * C + t * 4;
    ordered_store(os, blockIdx.x, o + 0, s4.x * scale); ordered_store(os, blockIdx.x, o + 1, s4.y * scale);
    ordered_store(os, blockIdx.x, o + 2, s4.z * scale); ordered_store(os, blockIdx.x, o + 3, s4.w * scale);
  }
  ordered_finish(os, out);
}

// y[n][p][c] = x[n][p][c] * gate[n][c]  (+ add[n][c] * add_scale); VEC = 4 when C % 4 == 0 (16-byte accesses)
template <int VEC>
__global__ void __launch_bounds__(256) scale_nc_kernel(const float* __restrict__ x, const float* __restrict__ gate,
                                                       const float* __restrict__ add, float add_scale, float* __restrict__ y,
                                                       int64_t total, int HW, int C, __nv_bfloat16* __restrict__ y16) {
  const int Cv = C / VEC;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total / VEC; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cv) * VEC;
    const int64_t n = i / ((int64_t)HW * Cv);
    if (VEC == 4) {
      float4 v = reinterpret_cast<const float4*>(x)[i];
      const float4 g = *reinterpret_cast<const float4*>(gate + n * C + c);
      v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
      if (add) {
        const float4 a = *reinterpret_cast<const float4*>(add + n * C + c);
        v.x = fmaf(a.x, add_scale, v.x); v.y = fmaf(a.y, add_scale, v.y); v.z = fmaf(a.z, add_scale, v.z); v.w = fmaf(a.w, add_scale, v.w);
      }
      reinterpret_cast<float4*>(y)[i] = v;
      if (y16) tfb_store_bf16x4(y16, i, v.x, v.y, v.z, v.w);
    } else {
      float v = x[i] * gate[n * C + c];
      if (add) v = fmaf(add[n * C + c], add_scale, v);
      y[i] = v;
      if (y16) y16[i] = __float2bfloat16_rn(v);
    }
  }
}

// dx[n][p][c] (+)= d[n][c] * s
__global__ void __launch_bounds__(256) bcast_nc_kernel(const float* __restrict__ d, float s, float* __restrict__ dx, int64_t total,
                                                       int HW, int C, int accumulate) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t n = i / ((int64_t)HW * C);
    const float v = d[n * C + c] * s;
    dx[i] = accumulate ? dx[i] + v : v;
  }
}

// NCHW uint8-range float image -> NHWC, ImageNet-normalised: ((x/255) - mean) / std   (transfuser.py:419-428)
__global__ void __launch_bounds__(256) image_prep_kernel(const float* __restrict__ img, float* __restrict__ out, int64_t npix_total,
                                                         int HW) {
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix_total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / HW, p = i % HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[i * 3 + c] = ((img[(n * 3 + c) * HW + p] / 255.0f) - mean[c]) / stdv[c];
  }
}

// y[n][b][a] = x[n][a][b]
__global__ void transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int A, int B) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const float* xp = x + (int64_t)n * A * B;
  float* yp = y + (int64_t)n * A * B;
  const int a0 = blockIdx.y * 32, b0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int a = a0 + j, b = b0 + threadIdx.x;
    tile[j][threadIdx.x] = (a < A && b < B) ? xp[(int64_t)a * B + b] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int b = b0 + j, a = a0 + threadIdx.x;
    if (a < A && b < B) yp[(int64_t)b * A + a] = tile[threadIdx.x][j];
  }
}

// tokens[n][t][c] = dropout(pos[t][c] + window_mean(feature)) ; t < gi: image grid (gh_i x gw_i), else lidar grid.
__global__ void __launch_bounds__(256)
tokens_fwd_kernel(const float* __restrict__ img, int Hi, int Wi, int ghi, int gwi, const float* __restrict__ lid, int Hl, int Wl,
                  int ghl, int gwl, const float* __restrict__ pos, float* __restrict__ out, int N, int C, float p_drop,
                  const uint64_t* __restrict__ seed_dev, uint64_t seed_off) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int T = ghi * gwi + ghl * gwl;
  const int64_t total = (int64_t)N * T * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int t = (int)((i / C) % T);
    const int n = (int)(i / ((int64_t)C * T));
    const float* src; int H, W, gw, tt, gh;
    if (t < ghi * gwi) { src = img; H = Hi; W = Wi; gh = ghi; gw = gwi; tt = t; }
    else { src = lid; H = Hl; W = Wl; gh = ghl; gw = gwl; tt = t - ghi * gwi; }
    const int wh = H / gh, ww = W / gw, gy = tt / gw, gx = tt % gw;
    const float* sp = src + (((int64_t)n * H + gy * wh) * W + gx * ww) * C + c;
    float s = 0.f;
    for (int yy = 0; yy < wh; ++yy)
      for (int xx = 0; xx < ww; ++xx) s += sp[((int64_t)yy * W + xx) * C];
    const float v = pos[(int64_t)t * C + c] + s / (float)(wh * ww);
    out[i] = v * tfb_dropout_scale(seed, (uint64_t)i, p_drop);
  }
}

// gradient of the token build w.r.t. one feature map: d[n][y][x][c] (+)= g[n][t(y,x)][c] * drop / window
__global__ void __launch_bounds__(256)
tokens_bwd_feat_kernel(const float* __restrict__ g, float* __restrict__ d, int N, int H, int W, int gh, int gw, int t_off, int T, int C,
                       float p_drop, const uint64_t* __restrict__ seed_dev, uint64_t seed_off, int accumulate) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t total = (int64_t)N * H * W * C;
  const int wh = H / gh, ww = W / gw;
  const float inv = 1.f / (float)(wh * ww);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int x = (int)((i / C) % W);
    const int y = (int)((i / ((int64_t)C * W)) % H);
    const int n = (int)(i / ((int64_t)C * W * H));
    const int t = t_off + (y / wh) * gw + (x / ww);
    const int64_t gi = ((int64_t)n * T + t) * C + c;
    const float v = g[gi] * tfb_dropout_scale(seed, (uint64_t)gi, p_drop) * inv;
    d[i] = accumulate ? d[i] + v : v;
  }
}

// dpos[t][c] = sum_n g[n][t][c] * drop
__global__ void __launch_bounds__(256) tokens_bwd_pos_kernel(const float* __restrict__ g, float* __restrict__ dpos, int N, int T, int C,
                                                             float p_drop, const uint64_t* __restrict__ seed_dev, uint64_t seed_off) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t total = (int64_t)T * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) {
      const int64_t gi = (int64_t)n * total + i;
      s += g[gi] * tfb_dropout_scale(seed, (uint64_t)gi, p_drop);
    }
    dpos[i] = s;
  }
}

struct Lerp { int i0, i1; float l0, l1; };
__device__ __forceinline__ Lerp lerp_coord(int dst, int in, int out, int align_corners) {
  // PyTorch upsample_bilinear2d source index (area_pixel_compute_source_index)
  float src;
  if (align_corners) {
    const float scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
    src = scale * (float)dst;
  } else {
    const float scale = (float)in / (float)out;
    src = scale * ((float)dst + 0.5f) - 0.5f;
    if (src < 0.f) src = 0.f;
  }
  Lerp r;
  r.i0 = (int)src;
  if (r.i0 > in - 1) r.i0 = in - 1;
  r.i1 = r.i0 + (r.i0 < in - 1 ? 1 : 0);
  r.l1 = src - (float)r.i0;
  r.l0 = 1.f - r.l1;
  return r;
}

// Conservative range [lo, hi] of destination indices whose interpolation can touch source cell g (lerp_coord's i0 or i1 == g): the
// source coordinate is monotone in the destination index, so the touching set is contiguous; callers re-check membership exactly.
__device__ __forceinline__ void lerp_window(int g, int in, int out, int align_corners, int* lo, int* hi) {
  float a, b;
  if (align_corners) {
    const float scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
    if (scale <= 0.f) { *lo = 0; *hi = out - 1; return; }
    a = ((float)g - 1.f) / scale;
    b = ((float)g + 1.f) / scale;
  } else {
    const float inv = (float)out / (float)in;
    a = ((float)g - 0.5f) * inv - 0.5f;
    b = ((float)g + 1.5f) * inv - 0.5f;
  }
  int l = (int)floorf(a) - 1, h = (int)ceilf(b) + 1;
  *lo = l < 0 ? 0 : l;
  *hi = h > out - 1 ? out - 1 : h;
}

// sum over destination pixels (y, x) of w_y(y -> gy) * w_x(x -> gx) * d[y * row_stride + x * col_stride]: the adjoint of bilinear
// interpolation for ONE source cell (gy, gx) of a [gh, gw] grid interpolated to [H, W]. The x weights of the (conservative) window
// are computed once into registers (windows up to GATHER_W pixels: scale factors up to ~10), zero-weight pixels are skipped.
constexpr int GATHER_W = 24;
__device__ __forceinline__ float bilinear_adjoint_gather(const float* __restrict__ d, int64_t row_stride, int64_t col_stride, int gy, int gh,
                                                         int H, int gx, int gw, int W, int align_corners) {
  int y0, y1, x0, x1;
  lerp_window(gy, gh, H, align_corners, &y0, &y1);
  lerp_window(gx, gw, W, align_corners, &x0, &x1);
  const int nx = x1 - x0 + 1;
  float acc = 0.f;
  if (nx <= GATHER_W) {
    float wxs[GATHER_W];
#pragma unroll
    for (int j = 0; j < GATHER_W; ++j) {
      float w = 0.f;
      if (j < nx) {
        const Lerp lx = lerp_coord(x0 + j, gw, W, align_corners);
        w = (lx.i0 == gx ? lx.l0 : 0.f) + (lx.i1 == gx ? lx.l1 : 0.f);
      }
      wxs[j] = w;
    }
    for (int y = y0; y <= y1; ++y) {
      const Lerp ly = lerp_coord(y, gh, H, align_corners);
      const float wy = (ly.i0 == gy ? ly.l0 : 0.f) + (ly.i1 == gy ? ly.l1 : 0.f);
      if (wy == 0.f) continue;
      const float* row = d + (int64_t)y * row_stride + (int64_t)x0 * col_stride;
      float racc = 0.f;
#pragma unroll
      for (int j = 0; j < GATHER_W; ++j)
        if (wxs[j] != 0.f) racc = fmaf(wxs[j], row[(int64_t)j * col_stride], racc);
      acc = fmaf(wy, racc, acc);
    }
  } else {
    for (int y = y0; y <= y1; ++y) {
      const Lerp ly = lerp_coord(y, gh, H, align_corners);
      const float wy = (ly.i0 == gy ? ly.l0 : 0.f) + (ly.i1 == gy ? ly.l1 : 0.f);
      if (wy == 0.f) continue;
      const float* row = d + (int64_t)y * row_stride;
      float racc = 0.f;
      for (int x = x0; x <= x1; ++x) {
        const Lerp lx = lerp_coord(x, gw, W, align_corners);
        const float wx = (lx.i0 == gx ? lx.l0 : 0.f) + (lx.i1 == gx ? lx.l1 : 0.f);
        if (wx != 0.f) racc = fmaf(wx, row[(int64_t)x * col_stride], racc);
      }
      acc = fmaf(wy, racc, acc);
    }
  }
  return acc;
}

// GPT output slab [gh*gw][C] of sample n, *viewed* as (C, gh, gw) without permuting (transfuser.py:363-364), bilinearly
// upsampled (align_corners=False) to (H, W) and added to the NHWC feature map.
// MODE 0: out = feat + up(view(tok))      MODE 1 (backward): dtok += up^T(dy)  (atomics; dtok zeroed by the caller)
template <int MODE>
__global__ void __launch_bounds__(256)
gpt_up_add_kernel(const float* __restrict__ feat, float* __restrict__ tok, float* __restrict__ out, int N, int H, int W, int C, int gh,
                  int gw, int t_off, int T, __nv_bfloat16* __restrict__ out16) {
  const int64_t total = (int64_t)N * H * W * C;
  const int G = gh * gw;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int x = (int)((i / C) % W);
    const int y = (int)((i / ((int64_t)C * W)) % H);
    const int n = (int)(i / ((int64_t)C * W * H));
    const Lerp ly = lerp_coord(y, gh, H, 0), lx = lerp_coord(x, gw, W, 0);
    float* slab = tok + ((int64_t)n * T + t_off) * C + (int64_t)c * G;
    const int i00 = ly.i0 * gw + lx.i0, i01 = ly.i0 * gw + lx.i1, i10 = ly.i1 * gw + lx.i0, i11 = ly.i1 * gw + lx.i1;
    if (MODE == 0) {
      const float v = ly.l0 * (lx.l0 * slab[i00] + lx.l1 * slab[i01]) + ly.l1 * (lx.l0 * slab[i10] + lx.l1 * slab[i11]);
      const float o = feat[i] + v;
      out[i] = o;
      if (out16) out16[i] = __float2bfloat16_rn(o);      // bf16 sidecar for the next stage's 1x1 conv
    } else {
      const float g = feat[i];  // dy
      atomicAdd(slab + i00, ly.l0 * lx.l0 * g);
      atomicAdd(slab + i01, ly.l0 * lx.l1 * g);
      atomicAdd(slab + i10, ly.l1 * lx.l0 * g);
      atomicAdd(slab + i11, ly.l1 * lx.l1 * g);
    }
  }
}

// Backward of the upsample + add w.r.t. the token slab as a GATHER: one thread per slab element (n, c, cell) sums the bilinear
// weights x dy over the pixels whose interpolation touches the cell (a ~2s x 2s window for scale s) — no atomics (the scatter
// version issued 4 strided atomicAdds per pixel and channel, up to 20 M per call, all pixels of a cell colliding), every slab
// element is written exactly once, so dtok needs no zero fill. c is the fastest thread index: dy reads are coalesced.
__global__ void __launch_bounds__(256)
gpt_up_add_bwd_gather_kernel(const float* __restrict__ dy, float* __restrict__ dtok, int N, int H, int W, int C, int gh, int gw, int t_off,
                             int T) {
  const int G = gh * gw;
  const int64_t total = (int64_t)N * G * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int cell = (int)((i / C) % G);
    const int n = (int)(i / ((int64_t)C * G));
    const int gy = cell / gw, gx = cell % gw;
    const float acc = bilinear_adjoint_gather(dy + (int64_t)n * H * W * C + c, (int64_t)W * C, C, gy, gh, H, gx, gw, W, 0);
    dtok[((int64_t)n * T + t_off) * C + (int64_t)c * G + cell] = acc;
  }
}

// generic NHWC bilinear upsample. MODE 0: y = up(x)   MODE 1: dx += up^T(dy) (atomics, dx zeroed by the launcher)
template <int MODE>
__global__ void __launch_bounds__(256) upsample_kernel(float* __restrict__ x, float* __restrict__ y, int N, int Hi, int Wi, int Ho,
                                                       int Wo, int C, int align_corners, __nv_bfloat16* __restrict__ y16) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int xo = (int)((i / C) % Wo);
    const int yo = (int)((i / ((int64_t)C * Wo)) % Ho);
    const int n = (int)(i / ((int64_t)C * Wo * Ho));
    const Lerp ly = lerp_coord(yo, Hi, Ho, align_corners), lx = lerp_coord(xo, Wi, Wo, align_corners);
    float* xp = x + (int64_t)n * Hi * Wi * C + c;
    const int64_t o00 = ((int64_t)ly.i0 * Wi + lx.i0) * C, o01 = ((int64_t)ly.i0 * Wi + lx.i1) * C;
    const int64_t o10 = ((int64_t)ly.i1 * Wi + lx.i0) * C, o11 = ((int64_t)ly.i1 * Wi + lx.i1) * C;
    if (MODE == 0) {
      const float v = ly.l0 * (lx.l0 * xp[o00] + lx.l1 * xp[o01]) + ly.l1 * (lx.l0 * xp[o10] + lx.l1 * xp[o11]);
      y[i] = v;
      if (y16) y16[i] = __float2bfloat16_rn(v);      // bf16 sidecar: the operand of the 3x3 conv that follows every upsample
    } else {
      const float g = y[i];
      atomicAdd(xp + o00, ly.l0 * lx.l0 * g);
      atomicAdd(xp + o01, ly.l0 * lx.l1 * g);
      atomicAdd(xp + o10, ly.l1 * lx.l0 * g);
      atomicAdd(xp + o11, ly.l1 * lx.l1 * g);
    }
  }
}

// Backward of the bilinear upsample as a gather (see gpt_up_add_bwd_gather_kernel): one thread per INPUT element (n, yi, xi, c) sums
// weight x dy over the output pixels that interpolate from it; no atomics, no zero fill, dx written exactly once.
__global__ void __launch_bounds__(256)
upsample_bwd_gather_kernel(const float* __restrict__ dy, float* __restrict__ dx, int N, int Hi, int Wi, int Ho, int Wo, int C,
                           int align_corners) {
  const int64_t total = (int64_t)N * Hi * Wi * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int xi = (int)((i / C) % Wi);
    const int yi = (int)((i / ((int64_t)C * Wi)) % Hi);
    const int n = (int)(i / ((int64_t)C * Wi * Hi));
    const float acc = bilinear_adjoint_gather(dy + (int64_t)n * Ho * Wo * C + c, (int64_t)Wo * C, C, yi, Hi, Ho, xi, Wi, Wo, align_corners);
    dx[i] = acc;
  }
}

// ---- float4 forms of the GPT upsample-add (forward, and the gather backward) and of the zero-dilation: the same 32-bit index
// arithmetic / 16-byte access pattern as upsample4_kernel below. The token slab keeps the reference's view quirk (channel c of cell p
// sits at slab[c * G + p]), so the four slab values of a channel quad are gathered separately (the slab is tiny and L1 resident).
__global__ void __launch_bounds__(256) gpt_up_add4_kernel(const float4* __restrict__ feat, const float* __restrict__ tok, float4* __restrict__ out,
                                                          int N, int H, int W, int C4, int gh, int gw, int t_off, int T,
                                                          __nv_bfloat16* __restrict__ out16) {
  const uint32_t total = (uint32_t)N * H * W * C4;
  const int G = gh * gw, C = C4 * 4;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % (uint32_t)C4, pix = i / (uint32_t)C4;
    const int x = (int)(pix % (uint32_t)W);
    const uint32_t t = pix / (uint32_t)W;
    const int y = (int)(t % (uint32_t)H), n = (int)(t / (uint32_t)H);
    const Lerp ly = lerp_coord(y, gh, H, 0), lx = lerp_coord(x, gw, W, 0);
    const float* slab = tok + ((int64_t)n * T + t_off) * C + (int64_t)(c4 * 4) * G;
    const int i00 = ly.i0 * gw + lx.i0, i01 = ly.i0 * gw + lx.i1, i10 = ly.i1 * gw + lx.i0, i11 = ly.i1 * gw + lx.i1;
    const float w00 = ly.l0 * lx.l0, w01 = ly.l0 * lx.l1, w10 = ly.l1 * lx.l0, w11 = ly.l1 * lx.l1;
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float* sq = slab + q * G;
      v[q] = w00 * sq[i00] + w01 * sq[i01] + w10 * sq[i10] + w11 * sq[i11];
    }
    const float4 f = feat[i];
    const float4 o = make_float4(f.x + v[0], f.y + v[1], f.z + v[2], f.w + v[3]);
    out[i] = o;
    if (out16) tfb_store_bf16x4(out16, i, o.x, o.y, o.z, o.w);
  }
}

// MODE 1 of stride2_kernel (zero-dilation of a [N, Ho, Wo, C] map into [N, H, W, C], bf16 output), four channels per thread
__global__ void __launch_bounds__(256) dilate2_bf16x4_kernel(const float4* __restrict__ src, __nv_bfloat16* __restrict__ dst, int N, int H, int W,
                                                             int Ho, int Wo, int C4) {
  const uint32_t total = (uint32_t)N * H * W * C4;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % (uint32_t)C4, pix = i / (uint32_t)C4;
    const int w = (int)(pix % (uint32_t)W);
    const uint32_t t = pix / (uint32_t)W;
    const int h = (int)(t % (uint32_t)H), n = (int)(t / (uint32_t)H);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (((h | w) & 1) == 0 && h / 2 < Ho && w / 2 < Wo) v = src[(((int64_t)n * Ho + h / 2) * Wo + w / 2) * C4 + c4];
    tfb_store_bf16x4(dst, i, v.x, v.y, v.z, v.w);
  }
}

// ---- 4-channel (float4) forms of the two kernels above for C % 4 == 0 and < 2^31 quads: 32-bit index arithmetic, one set of
// interpolation weights per 16 bytes, 16-byte loads / stores and an 8-byte bf16 store. The scalar forward kernel was instruction-bound
// (three 64-bit divisions, four scalar loads and a 2-byte store per ELEMENT: 719 us for the 160x704x64 decoder map, 7 % of the HBM
// rate under ncu); these are the HBM-bound versions the decoders (transfuser.py:239-246, 273-281), the FPN top-down path and the BEV
// head actually run.
__global__ void __launch_bounds__(256) upsample4_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int Hi, int Wi, int Ho,
                                                        int Wo, int C4, int align_corners, __nv_bfloat16* __restrict__ y16) {
  const uint32_t total = (uint32_t)N * Ho * Wo * C4;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % (uint32_t)C4, pix = i / (uint32_t)C4;
    const int xo = (int)(pix % (uint32_t)Wo);
    const uint32_t t = pix / (uint32_t)Wo;
    const int yo = (int)(t % (uint32_t)Ho), n = (int)(t / (uint32_t)Ho);
    const Lerp ly = lerp_coord(yo, Hi, Ho, align_corners), lx = lerp_coord(xo, Wi, Wo, align_corners);
    const float4* xp = x + (int64_t)n * Hi * Wi * C4 + c4;
    const float4 a = xp[(int64_t)(ly.i0 * Wi + lx.i0) * C4], b = xp[(int64_t)(ly.i0 * Wi + lx.i1) * C4];
    const float4 c = xp[(int64_t)(ly.i1 * Wi + lx.i0) * C4], d = xp[(int64_t)(ly.i1 * Wi + lx.i1) * C4];
    float4 o;
    o.x = ly.l0 * (lx.l0 * a.x + lx.l1 * b.x) + ly.l1 * (lx.l0 * c.x + lx.l1 * d.x);
    o.y = ly.l0 * (lx.l0 * a.y + lx.l1 * b.y) + ly.l1 * (lx.l0 * c.y + lx.l1 * d.y);
    o.z = ly.l0 * (lx.l0 * a.z + lx.l1 * b.z) + ly.l1 * (lx.l0 * c.z + lx.l1 * d.z);
    o.w = ly.l0 * (lx.l0 * a.w + lx.l1 * b.w) + ly.l1 * (lx.l0 * c.w + lx.l1 * d.w);
    y[i] = o;
    if (y16) tfb_store_bf16x4(y16, i, o.x, o.y, o.z, o.w);
  }
}

// adjoint of the bilinear interpolation for one source cell and FOUR channels (d points at the cell's channel quad of pixel (0, 0);
// strides in float4 units); same window / weight logic as bilinear_adjoint_gather
__device__ __forceinline__ float4 bilinear_adjoint_gather4(const float4* __restrict__ d, int64_t row_stride, int64_t col_stride, int gy, int gh,
                                                           int H, int gx, int gw, int W, int align_corners) {
  int y0, y1, x0, x1;
  lerp_window(gy, gh, H, align_corners, &y0, &y1);
  lerp_window(gx, gw, W, align_corners, &x0, &x1);
  const int nx = x1 - x0 + 1;
  assert(nx <= GATHER_W);                              // tfb_upsample_bilinear_bwd launches this form only for such windows
  float wxs[GATHER_W];
#pragma unroll
  for (int j = 0; j < GATHER_W; ++j) {
    float w = 0.f;
    if (j < nx) {
      const Lerp lx = lerp_coord(x0 + j, gw, W, align_corners);
      w = (lx.i0 == gx ? lx.l0 : 0.f) + (lx.i1 == gx ? lx.l1 : 0.f);
    }
    wxs[j] = w;
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int y = y0; y <= y1; ++y) {
    const Lerp ly = lerp_coord(y, gh, H, align_corners);
    const float wy = (ly.i0 == gy ? ly.l0 : 0.f) + (ly.i1 == gy ? ly.l1 : 0.f);
    if (wy == 0.f) continue;
    const float4* row = d + (int64_t)y * row_stride + (int64_t)x0 * col_stride;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < GATHER_W; ++j) {
      if (wxs[j] != 0.f) {
        const float4 v = row[(int64_t)j * col_stride];
        r.x = fmaf(wxs[j], v.x, r.x); r.y = fmaf(wxs[j], v.y, r.y); r.z = fmaf(wxs[j], v.z, r.z); r.w = fmaf(wxs[j], v.w, r.w);
      }
    }
    acc.x = fmaf(wy, r.x, acc.x); acc.y = fmaf(wy, r.y, acc.y); acc.z = fmaf(wy, r.z, acc.z); acc.w = fmaf(wy, r.w, acc.w);
  }
  return acc;
}

__global__ void __launch_bounds__(256)
upsample_bwd_gather4_kernel(const float4* __restrict__ dy, float4* __restrict__ dx, int N, int Hi, int Wi, int Ho, int Wo, int C4,
                            int align_corners) {
  const uint32_t total = (uint32_t)N * Hi * Wi * C4;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t c4 = i % (uint32_t)C4, pix = i / (uint32_t)C4;
    const int xi = (int)(pix % (uint32_t)Wi);
    const uint32_t t = pix / (uint32_t)Wi;
    const int yi = (int)(t % (uint32_t)Hi), n = (int)(t / (uint32_t)Hi);
    dx[i] = bilinear_adjoint_gather4(dy + (int64_t)n * Ho * Wo * C4 + c4, (int64_t)Wo * C4, C4, yi, Hi, Ho, xi, Wi, Wo, align_corners);
  }
}

// y = (res ? res : 0) + x * keep_scale(seed, element index): dropout, optionally fused with the residual add that follows it in
// the GPT block (x + drop(branch), transfuser.py:546-547). 4 elements per thread (16-byte accesses), scalar tail.
__global__ void __launch_bounds__(256) dropout_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n, float p,
                                                      const uint64_t* __restrict__ seed_dev, uint64_t seed_off,
                                                      const float* __restrict__ res) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 o;
    o.x = v.x * tfb_dropout_scale(seed, (uint64_t)(4 * i + 0), p);
    o.y = v.y * tfb_dropout_scale(seed, (uint64_t)(4 * i + 1), p);
    o.z = v.z * tfb_dropout_scale(seed, (uint64_t)(4 * i + 2), p);
    o.w = v.w * tfb_dropout_scale(seed, (uint64_t)(4 * i + 3), p);
    if (res) {
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    reinterpret_cast<float4*>(y)[i] = o;
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float o = x[i] * tfb_dropout_scale(seed, (uint64_t)i, p);
    y[i] = res ? res[i] + o : o;
  }
}

// one warp per row of length L: P = softmax(scale * S); Pd = dropout(P). P and Pd may alias S when p == 0.
__global__ void __launch_bounds__(128) softmax_fwd_kernel(const float* __restrict__ S, float* __restrict__ P, float* __restrict__ Pd,
                                                          int64_t rows, int L, float scale, float p_drop, const uint64_t* __restrict__ seed_dev,
                                                          uint64_t seed_off) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* s = S + r * L;
  float m = -INFINITY;
  for (int j = lane; j < L; j += 32) m = fmaxf(m, s[j] * scale);
  m = warp_max(m);
  float sum = 0.f;
  for (int j = lane; j < L; j += 32) sum += expf(s[j] * scale - m);
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  for (int j = lane; j < L; j += 32) {
    const float pv = expf(s[j] * scale - m) * inv;
    P[r * L + j] = pv;
    if (Pd != P) Pd[r * L + j] = pv * tfb_dropout_scale(seed, (uint64_t)(r * L + j), p_drop);
  }
}

// dS = scale * P * (g - sum_j g_j P_j), g = dPd * dropout_scale
__global__ void __launch_bounds__(128) softmax_bwd_kernel(const float* __restrict__ P, const float* __restrict__ dPd, float* __restrict__ dS,
                                                          int64_t rows, int L, float scale, float p_drop, const uint64_t* __restrict__ seed_dev,
                                                          uint64_t seed_off) {
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t r = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  float dot = 0.f;
  for (int j = lane; j < L; j += 32) {
    const float g = dPd[r * L + j] * tfb_dropout_scale(seed, (uint64_t)(r * L + j), p_drop);
    dot = fmaf(g, P[r * L + j], dot);
  }
  dot = warp_sum(dot);
  for (int j = lane; j < L; j += 32) {
    const float g = dPd[r * L + j] * tfb_dropout_scale(seed, (uint64_t)(r * L + j), p_drop);
    dS[r * L + j] = scale * P[r * L + j] * (g - dot);
  }
}

// Stride-2 sampling of an NHWC map and its transpose.
// MODE 0: dst[n][ho][wo][c] = src[n][2ho][2wo][c]           (the input view of a 1x1 / stride-2 conv)
// MODE 1: dst[n][h][w][c]   = (h, w both even) ? src[n][h/2][w/2][c] : 0   (zero-dilation: gradient of MODE 0, and the
//         stride-1 equivalent input of a stride-2 conv's dgrad); TO = float or bf16.
template <int MODE, typename TO>
__global__ void __launch_bounds__(256) stride2_kernel(const float* __restrict__ src, TO* __restrict__ dst, int N, int H, int W, int Ho,
                                                      int Wo, int C, __nv_bfloat16* __restrict__ dst16) {
  const int64_t total = MODE == 0 ? (int64_t)N * Ho * Wo * C : (int64_t)N * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v;
    if (MODE == 0) {
      const int wo = (int)((i / C) % Wo), ho = (int)((i / ((int64_t)C * Wo)) % Ho), n = (int)(i / ((int64_t)C * Wo * Ho));
      v = src[(((int64_t)n * H + 2 * ho) * W + 2 * wo) * C + c];
    } else {
      const int w = (int)((i / C) % W), h = (int)((i / ((int64_t)C * W)) % H), n = (int)(i / ((int64_t)C * W * H));
      v = ((h | w) & 1) == 0 && h / 2 < Ho && w / 2 < Wo ? src[(((int64_t)n * Ho + h / 2) * Wo + w / 2) * C + c] : 0.f;
    }
    if (sizeof(TO) == 4) reinterpret_cast<float*>(dst)[i] = v;
    else reinterpret_cast<__nv_bfloat16*>(dst)[i] = __float2bfloat16_rn(v);
    if (dst16) dst16[i] = __float2bfloat16_rn(v);          // optional bf16 sidecar of an fp32 result
  }
}

__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n) {
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    reinterpret_cast<uint2*>(y)[i] = o;
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16_rn(x[i]);
}

// x = t0 + t1 (+ t2) with t0 = bf16(x), t1 = bf16(x - t0), t2 = bf16(x - t0 - t1): 16 (24) mantissa bits of x in bf16 terms.
// The operands of the multi-term tensor-core parity modes.
__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int cols,
                                                         __nv_bfloat16* __restrict__ a16, __nv_bfloat16* __restrict__ b16,
                                                         __nv_bfloat16* __restrict__ c16, float* __restrict__ a32,
                                                         float* __restrict__ b32, float* __restrict__ c32) {
  const int64_t n = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[(i / cols) * ldx + (i % cols)];
    const __nv_bfloat16 t0 = __float2bfloat16_rn(v);
    const float r1 = v - __bfloat162float(t0);                 // exact (Sterbenz / the residual fits in fp32)
    const __nv_bfloat16 t1 = __float2bfloat16_rn(r1);
    const float r2 = r1 - __bfloat162float(t1);
    const __nv_bfloat16 t2 = __float2bfloat16_rn(r2);
    if (a16) a16[i] = t0;
    if (b16) b16[i] = t1;
    if (c16) c16[i] = t2;
    if (a32) a32[i] = __bfloat162float(t0);
    if (b32) b32[i] = __bfloat162float(t1);
    if (c32) c32[i] = __bfloat162float(t2);
  }
}

// y[n][t][c] = x[n][t][c] + v[n][c]: a per-sample vector added to every token (the GPT velocity embedding, transfuser.py:352-355)
__global__ void __launch_bounds__(256) bcast_add_nc_kernel(const float* __restrict__ x, const float* __restrict__ v, float* __restrict__ y,
                                                           int64_t total, int T, int C) {
  const int64_t tc = (int64_t)T * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = x[i] + v[(i / tc) * C + i % C];
}

// y_k[b][t][c] = x_k[b][t][c] + fmaf(v[b], w[c], bias[c]) for one or two tensors x_k [B, T_k, C]: one CTA per (k, b, t) row, the
// threads stride over the channels.
__global__ void __launch_bounds__(128) vel_emb_add_kernel(const float* __restrict__ v, const float* __restrict__ w,
                                                          const float* __restrict__ bias, const float* __restrict__ x0,
                                                          float* __restrict__ y0, int T0, const float* __restrict__ x1,
                                                          float* __restrict__ y1, int T1, int B, int C) {
  int row = blockIdx.x;
  const float* x = x0;
  float* y = y0;
  int T = T0;
  if (row >= B * T0) { row -= B * T0; x = x1; y = y1; T = T1; }
  const float vb = v[row / T];
  const int64_t off = (int64_t)row * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) y[off + c] = x[off + c] + fmaf(vb, w[c], bias[c]);
}

// dbias[c] = sum_b s_b[c], dw[c] = sum_b v[b] s_b[c], s_b[c] = sum_k sum_t dy_k[b][t][c]. One CTA owns VEB_CW channels whole: no
// cross-CTA fold, no atomics. Thread row ty sums t = ty, ty + VEB_TR, ... in increasing t; the VEB_TR row partials are folded in
// ty order; then k, then b in increasing order (the exact order is spelled out at tfb_vel_emb_bwd).
constexpr int VEB_CW = 32, VEB_TR = 16;
__global__ void __launch_bounds__(VEB_CW * VEB_TR) vel_emb_bwd_kernel(const float* __restrict__ v, const float* __restrict__ dy0, int T0,
                                                                      const float* __restrict__ dy1, int T1, int B, int C,
                                                                      float* __restrict__ dw, float* __restrict__ dbias) {
  __shared__ float part[2][VEB_TR][VEB_CW];
  const int tx = threadIdx.x, ty = threadIdx.y, c = blockIdx.x * VEB_CW + tx;
  const bool live = c < C;
  float acc_b = 0.f, acc_w = 0.f;
  for (int b = 0; b < B; ++b) {
    float p0 = 0.f, p1 = 0.f;
    if (live) {
      const float* d0 = dy0 + (int64_t)b * T0 * C + c;
#pragma unroll 4
      for (int t = ty; t < T0; t += VEB_TR) p0 += d0[(int64_t)t * C];
      if (dy1) {
        const float* d1 = dy1 + (int64_t)b * T1 * C + c;
#pragma unroll 4
        for (int t = ty; t < T1; t += VEB_TR) p1 += d1[(int64_t)t * C];
      }
    }
    part[0][ty][tx] = p0;
    part[1][ty][tx] = p1;
    __syncthreads();
    if (ty == 0) {
      float s0 = 0.f, s1 = 0.f;
      for (int r = 0; r < VEB_TR; ++r) { s0 += part[0][r][tx]; s1 += part[1][r][tx]; }
      const float s = dy1 ? s0 + s1 : s0;
      acc_b += s;
      acc_w = fmaf(v[b], s, acc_w);
    }
    __syncthreads();
  }
  if (ty == 0 && live) { dbias[c] = acc_b; dw[c] = acc_w; }
}

// y = x * (*s) * k  (device-resident scalar: no host sync)  /  y += ...
__global__ void __launch_bounds__(256) scale_dev_kernel(const float* __restrict__ x, const float* __restrict__ s, float k,
                                                        float* __restrict__ y, int64_t n, int accumulate) {
  const float f = (s ? *s : 1.f) * k;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = accumulate ? fmaf(x[i], f, y[i]) : x[i] * f;
}

// ---------------- squeeze-excite MLP backward, fused (batch N <= 16) ----------------
// gate = sigmoid(fc2(h)), h = relu(fc1(pooled)). Given dgate[N,C] (from se_bwd_reduce) the chain
//   ds = dgate*gate*(1-gate);  dw2 = ds^T h;  db2 = colsum ds;  dh = (ds w2) * (h > 0);  dw1 = dh^T pooled;  db1 = colsum dh;
//   dpool = dh w1
// used to be eight launches of [N,C]-sized kernels (sigmoid', 2 weight-gradient GEMMs, 2 column sums, 2 skinny GEMMs, relu'). It is
// two: both run one CTA per 16-channel chunk of C; the only cross-chunk quantity, dh (a sum over all of C), is accumulated by
// kernel 1 into a zeroed [N, Cr] buffer with fp32 atomics (C / 16 <= 95 per address) and read back by every CTA of kernel 2.
constexpr int SE_CHUNK = 16;    // channels of C per CTA: C / 16 CTAs (36 for the 576-channel stage) — these kernels are latency-bound
constexpr int SE_SLICES = 256 / SE_CHUNK;   // se_mlp_bwd2: slices of the Cr range that share one channel
constexpr int SE_MAX_N = 16;
constexpr int SE_MAX_CR = 512;   // static shared memory: (16 + 512) * 16 floats = 33 KiB (+ 15 KiB of partial sums in kernel 2)

__global__ void __launch_bounds__(256) se_mlp_bwd1_kernel(const float* __restrict__ dgate, const float* __restrict__ gate,
                                                          const float* __restrict__ h, const float* __restrict__ w2,
                                                          float* __restrict__ dw2, float* __restrict__ db2, float* __restrict__ dh_acc,
                                                          int N, int C, int Cr) {
  // one CTA per 64-channel chunk of C. dh_acc[chunk][N][Cr] receives this chunk's share of ds w2; se_mlp_bwd2_kernel adds the chunks
  // in chunk order (the same bits every run).
  __shared__ float ds[SE_MAX_N * SE_CHUNK];  // [N][SE_CHUNK]
  __shared__ float hs[SE_MAX_N * SE_MAX_CR]; // [N][Cr]
  const int c0 = blockIdx.x * SE_CHUNK;
  const int cw = min(SE_CHUNK, C - c0);
  for (int i = threadIdx.x; i < N * SE_CHUNK; i += blockDim.x) {
    const int n = i / SE_CHUNK, j = i % SE_CHUNK;
    float v = 0.f;
    if (j < cw) {
      const float g = gate[(int64_t)n * C + c0 + j];
      v = dgate[(int64_t)n * C + c0 + j] * g * (1.f - g);
    }
    ds[i] = v;
  }
  for (int i = threadIdx.x; i < N * Cr; i += blockDim.x) hs[i] = h[i];
  __syncthreads();
  if (threadIdx.x < cw) {
    float t = 0.f;
    for (int n = 0; n < N; ++n) t += ds[n * SE_CHUNK + threadIdx.x];
    db2[c0 + threadIdx.x] = t;
  }
  for (int i = threadIdx.x; i < cw * Cr; i += blockDim.x) {          // dw2[c][r] = sum_n ds[n][c] h[n][r]   (shared-memory operands)
    const int j = i / Cr, r = i % Cr;
    float t = 0.f;
    for (int n = 0; n < N; ++n) t = fmaf(ds[n * SE_CHUNK + j], hs[n * Cr + r], t);
    dw2[(int64_t)(c0 + j) * Cr + r] = t;
  }
  // dh[n][r] += sum_{c in chunk} ds[n][c] w2[c][r]: a thread owns column r, streams the chunk's weights of that column ONCE (coalesced
  // across the threads, 8 loads in flight) and feeds all N rows from registers; the first version re-read each weight per row
  for (int r = threadIdx.x; r < Cr; r += blockDim.x) {
    float acc[SE_MAX_N];
#pragma unroll
    for (int n = 0; n < SE_MAX_N; ++n) acc[n] = 0.f;
    const float* wp = w2 + (int64_t)c0 * Cr + r;
#pragma unroll 8
    for (int j = 0; j < cw; ++j) {
      const float w = wp[(int64_t)j * Cr];
#pragma unroll
      for (int n = 0; n < SE_MAX_N; ++n) acc[n] = fmaf(ds[n * SE_CHUNK + j], w, acc[n]);   // (rows >= N are zero in ds)
    }
#pragma unroll
    for (int n = 0; n < SE_MAX_N; ++n)
      if (n < N) dh_acc[((int64_t)blockIdx.x * N + n) * Cr + r] = acc[n];
  }
}

__global__ void __launch_bounds__(256) se_mlp_bwd2_kernel(const float* __restrict__ dh_acc, const float* __restrict__ h,
                                                          const float* __restrict__ pooled, const float* __restrict__ w1,
                                                          float* __restrict__ dw1, float* __restrict__ db1, float* __restrict__ dpool,
                                                          int N, int C, int Cr) {
  __shared__ float ps[SE_MAX_N * SE_CHUNK];  // [N][SE_CHUNK] pooled chunk
  __shared__ float dh[SE_MAX_N * SE_MAX_CR]; // [N][Cr]
  __shared__ float red[SE_SLICES - 1][SE_MAX_N][SE_CHUNK];   // slices 1.. (slice 0 keeps its sums in registers): 48 KiB of static smem in total
  const int c0 = blockIdx.x * SE_CHUNK;
  const int cw = min(SE_CHUNK, C - c0);
  for (int i = threadIdx.x; i < SE_MAX_N * Cr; i += blockDim.x) {
    float s = 0.f;
    if (i < N * Cr && h[i] > 0.f)
      for (int k = 0; k < (int)gridDim.x; ++k) s += dh_acc[(int64_t)k * N * Cr + i];
    dh[i] = s;
  }
  for (int i = threadIdx.x; i < N * SE_CHUNK; i += blockDim.x) {
    const int n = i / SE_CHUNK, j = i % SE_CHUNK;
    ps[i] = j < cw ? pooled[(int64_t)n * C + c0 + j] : 0.f;
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int r = threadIdx.x; r < Cr; r += blockDim.x) {
      float t = 0.f;
      for (int n = 0; n < N; ++n) t += dh[n * Cr + r];
      db1[r] = t;
    }
  }
  for (int i = threadIdx.x; i < Cr * SE_CHUNK; i += blockDim.x) {    // dw1[r][c] = sum_n dh[n][r] pooled[n][c]   (shared-memory operands)
    const int r = i / SE_CHUNK, j = i % SE_CHUNK;
    if (j >= cw) continue;
    float t = 0.f;
    for (int n = 0; n < N; ++n) t = fmaf(dh[n * Cr + r], ps[n * SE_CHUNK + j], t);
    dw1[(int64_t)r * C + c0 + j] = t;
  }
  // dpool[n][c] = sum_r dh[n][r] w1[r][c]: thread = (channel j, slice q of the r range): each weight is loaded once and used for
  // all N rows; the slices meet in shared memory
  {
    const int j = threadIdx.x % SE_CHUNK, q = threadIdx.x / SE_CHUNK;
    float acc[SE_MAX_N];
#pragma unroll
    for (int n = 0; n < SE_MAX_N; ++n) acc[n] = 0.f;
    if (j < cw) {
      const int r_lo = (Cr * q) / SE_SLICES, r_hi = (Cr * (q + 1)) / SE_SLICES;
      const float* wp = w1 + c0 + j;
#pragma unroll 8
      for (int r = r_lo; r < r_hi; ++r) {
        const float w = wp[(int64_t)r * C];
#pragma unroll
        for (int n = 0; n < SE_MAX_N; ++n) acc[n] = fmaf(dh[n * Cr + r], w, acc[n]);         // (rows >= N are zero in dh)
      }
    }
    if (q > 0) {
#pragma unroll
      for (int n = 0; n < SE_MAX_N; ++n) red[q - 1][n][j] = acc[n];
    }
    __syncthreads();
    if (q == 0 && j < cw) {
#pragma unroll
      for (int n = 0; n < SE_MAX_N; ++n)
        if (n < N) {
          float t = acc[n];
#pragma unroll
          for (int k = 0; k < SE_SLICES - 1; ++k) t += red[k][n][j];
          dpool[(int64_t)n * C + c0 + j] = t;
        }
    }
  }
}


}  // namespace

// y16_bf16 (optional, here and in tfb_se_scale_fwd): bf16 copy of y written in the same pass.
// a, b and y 16-byte aligned, y16_bf16 8-byte aligned (four elements per access).
TFB_API int tfb_add_relu(const float* a, const float* b, float* y, int64_t n, int relu, void* y16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(a && b && y && n >= 0);
  TFB_REQUIRE(tfb_aligned(a, 16) && tfb_aligned(b, 16) && tfb_aligned(y, 16) && tfb_aligned(y16_bf16, 8));
  if (n == 0) return TFB_OK;
  add_relu_kernel<<<tfb_grid(n / 4 + 1, 256), 256, 0, stream>>>(a, b, y, n, relu, (__nv_bfloat16*)y16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_relu_bwd(const float* y, const float* dy, float* dx, int64_t n, cudaStream_t stream) {
  TFB_REQUIRE(y && dy && dx && n >= 0);
  if (n == 0) return TFB_OK;
  act_kernel<0><<<tfb_grid(n, 256), 256, 0, stream>>>(y, dy, dx, n);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_sigmoid_bwd(const float* y, const float* dy, float* dx, int64_t n, cudaStream_t stream) {
  TFB_REQUIRE(y && dy && dx && n >= 0);
  if (n == 0) return TFB_OK;
  act_kernel<1><<<tfb_grid(n, 256), 256, 0, stream>>>(y, dy, dx, n);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_sigmoid_fwd(const float* x, float* y, int64_t n, cudaStream_t stream) {
  TFB_REQUIRE(x && y && n >= 0);
  if (n == 0) return TFB_OK;
  act_kernel<2><<<tfb_grid(n, 256), 256, 0, stream>>>(x, nullptr, y, n);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// out[n][c] = mean over the HW pixels of x[n][.][c]. C % 4 == 0, x 16-byte aligned.
TFB_API int tfb_pool_hw_fwd(const float* x, float* out, int N, int HW, int C, cudaStream_t stream) {
  TFB_REQUIRE(x && out && N > 0 && HW > 0 && C > 0);
  TFB_REQUIRE(C % 4 == 0 && tfb_aligned(x, 16));
  if (cudaMemsetAsync(out, 0, (size_t)N * C * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  int splits = (HW + 255) / 256;
  if (splits > 32) splits = 32;
  dim3 grid((C / 4 + 31) / 32, N, splits), block(32, 8);
  OrderedSum os;
  const int rc = ordered_alloc(os, splits, (int64_t)N * C, stream);
  if (rc != TFB_OK) return rc;
  pool_hw_kernel<0><<<grid, block, 0, stream>>>(x, nullptr, out, HW, C, 1.f / (float)HW, os);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_pool_hw_bwd(const float* dout, float* dx, int N, int HW, int C, int accumulate, cudaStream_t stream) {
  TFB_REQUIRE(dout && dx && N > 0 && HW > 0 && C > 0);
  const int64_t total = (int64_t)N * HW * C;
  bcast_nc_kernel<<<tfb_grid(total, 256), 256, 0, stream>>>(dout, 1.f / (float)HW, dx, total, HW, C, accumulate);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// y[n][p][c] = x[n][p][c] * gate[n][c]. Four channels per access when C % 4 == 0, x, gate and y are 16-byte aligned and y16_bf16
// 8-byte aligned; one otherwise (the same bits).
TFB_API int tfb_se_scale_fwd(const float* x, const float* gate, float* y, int N, int HW, int C, void* y16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(x && gate && y && N > 0 && HW > 0 && C > 0);
  const int64_t total = (int64_t)N * HW * C;
  __nv_bfloat16* y16 = (__nv_bfloat16*)y16_bf16;
  if (C % 4 == 0 && tfb_aligned(x, 16) && tfb_aligned(gate, 16) && tfb_aligned(y, 16) && tfb_aligned(y16, 8)) scale_nc_kernel<4><<<tfb_grid(total / 4, 256), 256, 0, stream>>>(x, gate, nullptr, 0.f, y, total, HW, C, y16);
  else            scale_nc_kernel<1><<<tfb_grid(total, 256), 256, 0, stream>>>(x, gate, nullptr, 0.f, y, total, HW, C, y16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// dgate[n][c] = sum over the HW pixels of x[n][.][c] * dy[n][.][c]. C % 4 == 0, x and dy 16-byte aligned.
TFB_API int tfb_se_bwd_reduce(const float* x, const float* dy, float* dgate, int N, int HW, int C, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dgate && N > 0 && HW > 0 && C > 0);
  TFB_REQUIRE(C % 4 == 0 && tfb_aligned(x, 16) && tfb_aligned(dy, 16));
  if (cudaMemsetAsync(dgate, 0, (size_t)N * C * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  int splits = (HW + 255) / 256;
  if (splits > 32) splits = 32;
  dim3 grid((C / 4 + 31) / 32, N, splits), block(32, 8);
  if (C / 4 <= 128 && HW >= 1024) {
    const int rpb = 256 / (C / 4);
    int sp = (HW + rpb * 16 - 1) / (rpb * 16);                      // >= 16 pixel rows per thread
    const int cap = (4 * tfb_num_sms() + N - 1) / N;
    if (sp > cap) sp = cap;
    if (sp < 1) sp = 1;
    OrderedSum os;
    const int rc = ordered_alloc(os, sp, (int64_t)N * C, stream);
    if (rc != TFB_OK) return rc;
    pool_hw_flat_kernel<1><<<dim3(sp, N), 256, 0, stream>>>(x, dy, dgate, HW, C, 1.f, os);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  OrderedSum os;
  const int rc = ordered_alloc(os, splits, (int64_t)N * C, stream);
  if (rc != TFB_OK) return rc;
  pool_hw_kernel<1><<<grid, block, 0, stream>>>(x, dy, dgate, HW, C, 1.f, os);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// Fused backward of the squeeze-excite MLP (see se_mlp_bwd1_kernel): dgate, gate, pooled [N,C]; h [N,Cr]; w1 [Cr,C]; w2 [C,Cr] ->
// dw1 [Cr,C], db1 [Cr], dw2 [C,Cr], db2 [C], dpool [N,C] (all overwritten). N <= 16, Cr <= 512.
// dh_part: unused (kept for the C-ABI); the per-chunk partial sums live in a per-launch workspace.
TFB_API int tfb_se_mlp_bwd(const float* dgate, const float* gate, const float* h, const float* pooled, const float* w1, const float* w2,
                           float* dw1, float* db1, float* dw2, float* db2, float* dpool, float* dh_part, int N, int C, int Cr,
                           cudaStream_t stream) {
  TFB_REQUIRE(dgate && gate && h && pooled && w1 && w2 && dw1 && db1 && dw2 && db2 && dpool && dh_part);
  TFB_REQUIRE(N > 0 && N <= SE_MAX_N && C > 0 && Cr > 0 && Cr <= SE_MAX_CR);
  const int nchunks = (C + SE_CHUNK - 1) / SE_CHUNK;
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)nchunks * N * Cr, 0, stream);
  if (rc != TFB_OK) return rc;
  se_mlp_bwd1_kernel<<<nchunks, 256, 0, stream>>>(dgate, gate, h, w2, dw2, db2, w.f, N, C, Cr);
  TFB_CHECK_LAUNCH();
  se_mlp_bwd2_kernel<<<nchunks, 256, 0, stream>>>(w.f, h, pooled, w1, dw1, db1, dpool, N, C, Cr);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// dx[n][p][c] = dy[n][p][c] * gate[n][c] + dpool[n][c] / HW. Four channels per access when C % 4 == 0 and dy, gate, dpool and dx are
// 16-byte aligned; one otherwise (the same bits).
TFB_API int tfb_se_bwd_apply(const float* dy, const float* gate, const float* dpool, float* dx, int N, int HW, int C,
                             cudaStream_t stream) {
  TFB_REQUIRE(dy && gate && dpool && dx && N > 0 && HW > 0 && C > 0);
  const int64_t total = (int64_t)N * HW * C;
  if (C % 4 == 0 && tfb_aligned(dy, 16) && tfb_aligned(gate, 16) && tfb_aligned(dpool, 16) && tfb_aligned(dx, 16)) scale_nc_kernel<4><<<tfb_grid(total / 4, 256), 256, 0, stream>>>(dy, gate, dpool, 1.f / (float)HW, dx, total, HW, C, nullptr);
  else            scale_nc_kernel<1><<<tfb_grid(total, 256), 256, 0, stream>>>(dy, gate, dpool, 1.f / (float)HW, dx, total, HW, C, nullptr);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_image_prep(const float* img_nchw, float* out_nhwc, int N, int H, int W, cudaStream_t stream) {
  TFB_REQUIRE(img_nchw && out_nhwc && N > 0 && H > 0 && W > 0);
  const int64_t npix = (int64_t)N * H * W;
  image_prep_kernel<<<tfb_grid(npix, 256), 256, 0, stream>>>(img_nchw, out_nhwc, npix, H * W);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_transpose_last2(const float* x, float* y, int N, int A, int B, cudaStream_t stream) {
  TFB_REQUIRE(x && y && N > 0 && A > 0 && B > 0 && N <= 65535);
  dim3 grid((B + 31) / 32, (A + 31) / 32, N), block(32, 8);
  TFB_REQUIRE(grid.y <= 65535);
  transpose_kernel<<<grid, block, 0, stream>>>(x, y, A, B);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_tokens_fwd(const float* img, int Hi, int Wi, int ghi, int gwi, const float* lid, int Hl, int Wl, int ghl, int gwl,
                           const float* pos, float* out, int N, int C, float p_drop, const uint64_t* seed_dev, uint64_t seed_off,
                           cudaStream_t stream) {
  TFB_REQUIRE(img && lid && pos && out && N > 0 && C > 0);
  TFB_REQUIRE(Hi % ghi == 0 && Wi % gwi == 0 && Hl % ghl == 0 && Wl % gwl == 0);  // exact adaptive-avg-pool windows only
  const int64_t total = (int64_t)N * (ghi * gwi + ghl * gwl) * C;
  tokens_fwd_kernel<<<tfb_grid(total, 256), 256, 0, stream>>>(img, Hi, Wi, ghi, gwi, lid, Hl, Wl, ghl, gwl, pos, out, N, C, p_drop, seed_dev, seed_off);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_tokens_bwd(const float* g, float* dimg, int Hi, int Wi, int ghi, int gwi, float* dlid, int Hl, int Wl, int ghl,
                           int gwl, float* dpos, int N, int C, float p_drop, const uint64_t* seed_dev, uint64_t seed_off, int accumulate_feat,
                           cudaStream_t stream) {
  TFB_REQUIRE(g && dimg && dlid && dpos && N > 0 && C > 0);
  const int T = ghi * gwi + ghl * gwl;
  const int64_t ti = (int64_t)N * Hi * Wi * C, tl = (int64_t)N * Hl * Wl * C;
  tokens_bwd_feat_kernel<<<tfb_grid(ti, 256), 256, 0, stream>>>(g, dimg, N, Hi, Wi, ghi, gwi, 0, T, C, p_drop, seed_dev, seed_off, accumulate_feat);
  TFB_CHECK_LAUNCH();
  tokens_bwd_feat_kernel<<<tfb_grid(tl, 256), 256, 0, stream>>>(g, dlid, N, Hl, Wl, ghl, gwl, ghi * gwi, T, C, p_drop, seed_dev, seed_off, accumulate_feat);
  TFB_CHECK_LAUNCH();
  tokens_bwd_pos_kernel<<<tfb_grid((int64_t)T * C, 256), 256, 0, stream>>>(g, dpos, N, T, C, p_drop, seed_dev, seed_off);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// out16_bf16 (optional): bf16 copy of out written in the same pass.
TFB_API int tfb_gpt_up_add_fwd(const float* feat, const float* tok, float* out, int N, int H, int W, int C, int gh, int gw, int t_off,
                               int T, void* out16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(feat && tok && out && N > 0);
  const int64_t total = (int64_t)N * H * W * C;
  if (C % 4 == 0 && total / 4 < 0x7fffffffLL && ((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 &&
      (!out16_bf16 || (reinterpret_cast<uintptr_t>(out16_bf16) & 7) == 0)) {
    gpt_up_add4_kernel<<<tfb_grid(total / 4, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(feat), tok, reinterpret_cast<float4*>(out), N, H, W,
                                                                    C / 4, gh, gw, t_off, T, (__nv_bfloat16*)out16_bf16);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  gpt_up_add_kernel<0><<<tfb_grid(total, 256), 256, 0, stream>>>(feat, const_cast<float*>(tok), out, N, H, W, C, gh, gw, t_off, T,
                                                                 (__nv_bfloat16*)out16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_gpt_up_add_bwd(const float* dy, float* dtok, int N, int H, int W, int C, int gh, int gw, int t_off, int T,
                               cudaStream_t stream) {
  TFB_REQUIRE(dy && dtok && N > 0 && H > 0 && W > 0 && C > 0 && gh > 0 && gw > 0);
  // overwrites dtok[n][t_off .. t_off + gh*gw)[:] (every element exactly once): no zero fill, no atomics
  gpt_up_add_bwd_gather_kernel<<<tfb_grid((int64_t)N * gh * gw * C, 256), 256, 0, stream>>>(dy, dtok, N, H, W, C, gh, gw, t_off, T);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// y16_bf16 (optional): bf16 copy of y written in the same pass.
TFB_API int tfb_upsample_bilinear_fwd(const float* x, float* y, int N, int Hi, int Wi, int Ho, int Wo, int C, int align_corners,
                                      void* y16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(x && y && N > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0);
  const int64_t total = (int64_t)N * Ho * Wo * C;
  const bool vec = C % 4 == 0 && total / 4 < 0x7fffffffLL && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 &&
                   (!y16_bf16 || (reinterpret_cast<uintptr_t>(y16_bf16) & 7) == 0);
  if (vec) {
    upsample4_kernel<<<tfb_grid(total / 4, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), N, Hi, Wi, Ho, Wo,
                                                                  C / 4, align_corners, (__nv_bfloat16*)y16_bf16);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  upsample_kernel<0><<<tfb_grid(total, 256), 256, 0, stream>>>(const_cast<float*>(x), y, N, Hi, Wi, Ho, Wo, C, align_corners,
                                                               (__nv_bfloat16*)y16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_upsample_bilinear_bwd(const float* dy, float* dx, int N, int Hi, int Wi, int Ho, int Wo, int C, int align_corners,
                                      cudaStream_t stream) {
  TFB_REQUIRE(dy && dx && N > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0);
  // the float4 form needs every interpolation window to fit the register array of x weights (scale factors up to ~10). A window
  // spans at most 2 * sx + 5 destination pixels, sx the inverse scale lerp_window divides by: (Wo - 1) / (Wi - 1) with align_corners
  // (Wo / Wi bounds the whole-row window of Wi == 1 too), Wo / Wi without.
  const double sx = align_corners && Wi > 1 && Wo > 1 ? (double)(Wo - 1) / (double)(Wi - 1) : (double)Wo / (double)Wi;
  const bool vec = C % 4 == 0 && (int64_t)N * Hi * Wi * C / 4 < 0x7fffffffLL && sx * 2.0 + 5.0 <= (double)GATHER_W &&
                   ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  if (vec) {
    upsample_bwd_gather4_kernel<<<tfb_grid((int64_t)N * Hi * Wi * C / 4, 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(dy), reinterpret_cast<float4*>(dx), N, Hi, Wi, Ho, Wo, C / 4, align_corners);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  upsample_bwd_gather_kernel<<<tfb_grid((int64_t)N * Hi * Wi * C, 256), 256, 0, stream>>>(dy, dx, N, Hi, Wi, Ho, Wo, C, align_corners);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// Dropout mask = f(*seed_dev + seed_off, element index): the base seed lives in device memory (advanced by tfb_step_tick once
// per step, also inside a captured CUDA graph), seed_off identifies the call site; the backward regenerates the same mask.
// y = dropout(x) (+ residual when given): the mask is a hash of (*seed_dev + seed_off, element index), regenerated in backward.
// x, y and residual 16-byte aligned (four elements per access).
TFB_API int tfb_dropout(const float* x, float* y, int64_t n, float p, const uint64_t* seed_dev, uint64_t seed_off, const float* residual,
                        cudaStream_t stream) {
  TFB_REQUIRE(x && y && n >= 0 && p >= 0.f && p < 1.f);
  TFB_REQUIRE(tfb_aligned(x, 16) && tfb_aligned(y, 16) && tfb_aligned(residual, 16));
  if (n == 0) return TFB_OK;
  dropout_kernel<<<tfb_grid(n / 4 + 1, 256), 256, 0, stream>>>(x, y, n, p, seed_dev, seed_off, residual);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_softmax_fwd(const float* S, float* P, float* Pd, int64_t rows, int L, float scale, float p_drop, const uint64_t* seed_dev,
                            uint64_t seed_off, cudaStream_t stream) {
  TFB_REQUIRE(S && P && Pd && rows > 0 && L > 0);
  softmax_fwd_kernel<<<(unsigned)ceil_div64(rows, 4), 128, 0, stream>>>(S, P, Pd, rows, L, scale, p_drop, seed_dev, seed_off);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_softmax_bwd(const float* P, const float* dPd, float* dS, int64_t rows, int L, float scale, float p_drop, const uint64_t* seed_dev,
                            uint64_t seed_off, cudaStream_t stream) {
  TFB_REQUIRE(P && dPd && dS && rows > 0 && L > 0);
  softmax_bwd_kernel<<<(unsigned)ceil_div64(rows, 4), 128, 0, stream>>>(P, dPd, dS, rows, L, scale, p_drop, seed_dev, seed_off);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// y = bf16(x). x 16-byte aligned, y 8-byte aligned (four elements per access).
TFB_API int tfb_cast_bf16(const float* x, void* y, int64_t n, cudaStream_t stream) {
  TFB_REQUIRE(x && y && n >= 0);
  TFB_REQUIRE(tfb_aligned(x, 16) && tfb_aligned(y, 8));
  if (n == 0) return TFB_OK;
  cast_bf16_kernel<<<tfb_grid(n / 4 + 1, 256), 256, 0, stream>>>(x, (__nv_bfloat16*)y, n);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// (No reference counterpart: operand preparation of the tensor-core parity modes, which replace cuBLAS fp32 behind nn.Linear / 1x1 /
// dense 3x3 nn.Conv2d — transfuser.py:498-506, 538-543, 214-281, model.py:93-99.)
// The bf16 terms of x[rows, cols] (row stride ldx): t0 = bf16(x), t1 = bf16(x - t0), t2 = bf16(x - t0 - t1), written contiguously as
// bf16 (t0_16 / t1_16 / t2_16) and / or as the same values in fp32 (t0_32 / ...); any output may be null. Two terms carry 16 mantissa
// bits of x, three terms all 24: the tensor-core parity modes of gemm.py multiply term by term ("bf16x3": 3 products of 2 terms,
// ~1e-5 relative; "bf16x6": 6 products of 3 terms, fp32-grade) with fp32 accumulation.
TFB_API int tfb_split_bf16(const float* x, int64_t ldx, int64_t rows, int cols, void* t0_16, void* t1_16, void* t2_16, float* t0_32,
                           float* t1_32, float* t2_32, cudaStream_t stream) {
  TFB_REQUIRE(x && rows >= 0 && cols > 0 && ldx >= cols);
  if (rows == 0) return TFB_OK;
  split_bf16_kernel<<<tfb_grid(rows * cols, 256), 256, 0, stream>>>(x, ldx, rows, cols, (__nv_bfloat16*)t0_16, (__nv_bfloat16*)t1_16,
                                                                   (__nv_bfloat16*)t2_16, t0_32, t1_32, t2_32);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// y[N, T, C] = x[N, T, C] + v[N, C] broadcast over T — GPT.forward with use_velocity (reference team_code_transfuser/transfuser.py:352-355:
// pos_emb + token_embeddings + velocity_embeddings.unsqueeze(1)); the gradient of v is the sum of dy over T (tfb_pool_hw_fwd x T).
TFB_API int tfb_bcast_add_nc(const float* x, const float* v, float* y, int N, int T, int C, cudaStream_t stream) {
  TFB_REQUIRE(x && v && y && N > 0 && T > 0 && C > 0);
  const int64_t total = (int64_t)N * T * C;
  bcast_add_nc_kernel<<<tfb_grid(total, 256), 256, 0, stream>>>(x, v, y, total, T, C);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// The ego-speed embedding Linear(1, C) added to one or two feature tensors (reference late_fusion.py:107-109: the fused vector;
// geometric_fusion.py:142-271: the LiDAR and the image map of one scale). v [B] speeds, w [C] (the [C, 1] weight), bias [C];
// x0 / y0 [B, T0, C] and optionally x1 / y1 [B, T1, C] (x1 = y1 = null, T1 = 0 for one tensor).
//   y_k[b, t, c] = x_k[b, t, c] + e[b, c],   e[b, c] = fmaf(v[b], w[c], bias[c])   (__fmaf_rn: one rounding; then one fp32 add)
// No e tensor is formed.
TFB_API int tfb_vel_emb_add(const float* v, const float* w, const float* bias, const float* x0, float* y0, int T0, const float* x1, float* y1,
                            int T1, int B, int C, cudaStream_t stream) {
  TFB_REQUIRE(v && w && bias && x0 && y0 && T0 > 0 && B > 0 && C > 0 && T1 >= 0);
  TFB_REQUIRE(T1 == 0 ? (!x1 && !y1) : (x1 && y1));
  const int64_t rows = (int64_t)B * (T0 + T1);
  TFB_REQUIRE(rows <= 0x7fffffffLL);
  vel_emb_add_kernel<<<(unsigned)rows, 128, 0, stream>>>(v, w, bias, x0, y0, T0, x1, y1, T1, B, C);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// Backward of tfb_vel_emb_add for the embedding's parameters (dx_k = dy_k needs no kernel): dw [C] (the [C, 1] weight's gradient)
// and dbias [C], both overwritten. Deterministic fixed-order fp32 sums, for every channel c:
//   p_k[r]  = sum over t = r, r + 16, r + 32, ... < T_k of dy_k[b, t, c], in increasing t            (r = 0 .. 15)
//   S_k     = sum over r = 0 .. 15 of p_k[r], in increasing r
//   s_b     = S_0 + S_1   (S_0 alone with one tensor)
//   dbias   = sum over b of s_b, in increasing b;   dw = fmaf(v[b], s_b, dw) over increasing b, from 0
// every sum starting from 0.f. One CTA per 32 channels; no atomics, the same bits on every run.
TFB_API int tfb_vel_emb_bwd(const float* v, const float* dy0, int T0, const float* dy1, int T1, int B, int C, float* dw, float* dbias,
                            cudaStream_t stream) {
  TFB_REQUIRE(v && dy0 && dw && dbias && T0 > 0 && B > 0 && C > 0 && T1 >= 0);
  TFB_REQUIRE(T1 == 0 ? !dy1 : dy1 != nullptr);
  vel_emb_bwd_kernel<<<(C + VEB_CW - 1) / VEB_CW, dim3(VEB_CW, VEB_TR), 0, stream>>>(v, dy0, T0, dy1, T1, B, C, dw, dbias);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_scale_dev(const float* x, const float* s_dev, float k, float* y, int64_t n, int accumulate, cudaStream_t stream) {
  TFB_REQUIRE(x && y && n >= 0);
  if (n == 0) return TFB_OK;
  scale_dev_kernel<<<tfb_grid(n, 256), 256, 0, stream>>>(x, s_dev, k, y, n, accumulate);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// xs[N,Ho,Wo,C] = x[N, ::2, ::2, C] with Ho = (H+1)/2, Wo = (W+1)/2.
// xs16_bf16 (optional): bf16 copy of xs written in the same pass.
TFB_API int tfb_subsample2(const float* x, float* xs, int N, int H, int W, int C, void* xs16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(x && xs && N > 0 && H > 0 && W > 0 && C > 0);
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  stride2_kernel<0, float><<<tfb_grid((int64_t)N * Ho * Wo * C, 256), 256, 0, stream>>>(x, xs, N, H, W, Ho, Wo, C, (__nv_bfloat16*)xs16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
// dst[N,H,W,C] = zero-dilated src[N,Ho,Wo,C] (values at even (h, w)); out_bf16 selects the output type.
TFB_API int tfb_dilate2(const float* src, void* dst, int N, int H, int W, int C, int out_bf16, cudaStream_t stream) {
  TFB_REQUIRE(src && dst && N > 0 && H > 0 && W > 0 && C > 0);
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int grid = tfb_grid((int64_t)N * H * W * C, 256);
  if (out_bf16 && C % 4 == 0 && (int64_t)N * H * W * C / 4 < 0x7fffffffLL && (reinterpret_cast<uintptr_t>(src) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
    dilate2_bf16x4_kernel<<<tfb_grid((int64_t)N * H * W * C / 4, 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(src), (__nv_bfloat16*)dst, N, H, W,
                                                                                        Ho, Wo, C / 4);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  if (out_bf16) stride2_kernel<1, __nv_bfloat16><<<grid, 256, 0, stream>>>(src, (__nv_bfloat16*)dst, N, H, W, Ho, Wo, C, nullptr);
  else          stride2_kernel<1, float><<<grid, 256, 0, stream>>>(src, (float*)dst, N, H, W, Ho, Wo, C, nullptr);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
