// Loss kernels of LidarCenterNet.forward (model.py:759-788) and LidarCenterNetHead.get_targets / loss (model.py:149-374),
// forward + backward, fused reductions; no host synchronisation anywhere (the reference's get_targets loops in Python with
// device syncs). Restated third-party semantics (mmdet 2.25 — GaussianFocalLoss, L1Loss, SmoothL1Loss, CrossEntropyLoss,
// gaussian_radius, gen_gaussian_target) follow oracle/shims/mmdet.
//   - cross entropy over the channel dim of NHWC logits, optional class weights, optional per-position weight that is
//     broadcast over the batch (the reference's (B,H,W)*(B,1,H,W) -> (B,B,H,W) broadcast, model.py:220-224,235-239)
//   - L1 with optional fused sigmoid (depth head, model.py:788; waypoints, model.py:765)
//   - CenterNet: target rasterisation, then all 7 head losses in one pass over the [M,21] prediction matrix
#include "common.cuh"

namespace {

constexpr int kMaxC = 16;

// Loss sums that give the same bits every run: block b stores its sum of term k in part[b * nacc + k] (block_partial); the last
// block (blocks_finish, called by every thread) adds the blocks' sums in block order, in fp64, to acc[k] (zeroed by the caller).
__device__ __forceinline__ void block_partial(float* part, int nacc, int k, float v, float* red) {
  const float s = block_sum(v, red);
  if (threadIdx.x == 0) part[(int64_t)blockIdx.x * nacc + k] = s;
}
__device__ __forceinline__ void blocks_finish(const float* part, int nacc, double* acc, unsigned int* cnt) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(cnt, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int k = threadIdx.x; k < nacc; k += blockDim.x) {
    double s = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) s += (double)__ldcg(part + (int64_t)b * nacc + k);
    acc[k] += s;
  }
  if (threadIdx.x == 0) *cnt = 0u;      // the stream's scratch counters are zero on entry
}

// ---------------- cross entropy ----------------
// acc[0] += sum_m w_m * nll_m, acc[1] += sum_m w_m, w_m = class_w[t_m] * pos_w[m % HW]
__global__ void __launch_bounds__(256) ce_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target, int64_t M, int C,
                                                     const float* __restrict__ class_w, const float* __restrict__ pos_w, int HW,
                                                     double* __restrict__ acc, float* __restrict__ part, unsigned int* __restrict__ cnt) {
  __shared__ float red[32];
  float ls = 0.f, ws = 0.f;
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
    const float* l = logits + m * C;
    float mx = -INFINITY;
    float v[kMaxC];
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c < C) { v[c] = l[c]; mx = fmaxf(mx, v[c]); }
    float se = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c < C) se += expf(v[c] - mx);
    const int t = (int)target[m];
    float lt = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c == t) lt = v[c];
    float w = class_w ? class_w[t] : 1.f;
    if (pos_w) w *= pos_w[m % HW];
    ls = fmaf(w, (logf(se) + mx - lt), ls);
    ws += w;
  }
  block_partial(part, 2, 0, ls, red);
  block_partial(part, 2, 1, ws, red);
  blocks_finish(part, 2, acc, cnt);
}

// dlogits = coef * w_m * (softmax - onehot), coef = (*gout) * k / (den ? max(*den, den_min) : 1)
__global__ void __launch_bounds__(256) ce_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ target, int64_t M, int C,
                                                     const float* __restrict__ class_w, const float* __restrict__ pos_w, int HW,
                                                     const float* __restrict__ gout, const double* __restrict__ den, float den_min, float k,
                                                     float* __restrict__ dlogits) {
  float coef = (gout ? *gout : 1.f) * k;
  if (den) coef = (float)((double)coef / fmax(*den, (double)den_min));
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
    const float* l = logits + m * C;
    float mx = -INFINITY;
    float v[kMaxC];
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c < C) { v[c] = l[c]; mx = fmaxf(mx, v[c]); }
    float se = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c < C) { v[c] = expf(v[c] - mx); se += v[c]; }
    const int t = (int)target[m];
    float w = class_w ? class_w[t] : 1.f;
    if (pos_w) w *= pos_w[m % HW];
    const float f = coef * w, inv = 1.f / se;
    float* d = dlogits + m * C;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) if (c < C) d[c] = f * (v[c] * inv - (c == t ? 1.f : 0.f));
  }
}

// ---------------- L1 (optionally on sigmoid(x)) ----------------
__global__ void __launch_bounds__(256) l1_fwd_kernel(const float* __restrict__ x, const float* __restrict__ t, int64_t n, int sigmoid,
                                                     double* __restrict__ acc, float* __restrict__ part, unsigned int* __restrict__ cnt) {
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = x[i];
    if (sigmoid) v = 1.f / (1.f + expf(-v));
    s += fabsf(v - t[i]);
  }
  block_partial(part, 1, 0, s, red);
  blocks_finish(part, 1, acc, cnt);
}
__global__ void __launch_bounds__(256) l1_bwd_kernel(const float* __restrict__ x, const float* __restrict__ t, int64_t n, int sigmoid,
                                                     const float* __restrict__ gout, float k, float* __restrict__ dx) {
  const float coef = (gout ? *gout : 1.f) * k;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = x[i], dv = 1.f;
    if (sigmoid) { v = 1.f / (1.f + expf(-v)); dv = v * (1.f - v); }
    const float d = v - t[i];
    dx[i] = coef * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * dv;
  }
}

// ---------------- CenterNet targets (model.py:285-374) ----------------
// label [B][K][7] = cx, cy, w, h, yaw, speed, brake in 256-px BEV coordinates; all-zero rows are ignored (model.py:774).
// tgt planes [B][10][H][W]: 0 heat, 1 w, 2 h, 3 off_x, 4 off_y, 5 yaw_res, 6 velocity, 7 weight, 8 yaw_class, 9 brake.
__device__ __forceinline__ float py_remainder(float a, float b) {
  float r = fmodf(a, b);
  if (r != 0.f && ((r < 0.f) != (b < 0.f))) r += b;
  return r;
}
__device__ __forceinline__ float gaussian_radius_f(float height, float width, float min_overlap) {
  // fp32 tensor arithmetic with a double sqrt in between, as mmdet evaluates it on 0-dim fp32 tensors
  const float mo = min_overlap;
  const float b1 = height + width;
  const float c1 = width * height * (1.f - mo) / (1.f + mo);
  const float sq1 = (float)sqrt((double)(b1 * b1 - 4.f * c1));
  const float r1 = (b1 - sq1) / 2.f;
  const float b2 = 2.f * (height + width);
  const float c2 = (1.f - mo) * width * height;
  const float sq2 = (float)sqrt((double)(b2 * b2 - 16.f * c2));
  const float r2 = (b2 - sq2) / 8.f;
  const float a3 = 4.f * mo;
  const float b3 = -2.f * mo * (height + width);
  const float c3 = (mo - 1.f) * width * height;
  const float sq3 = (float)sqrt((double)(b3 * b3 - 4.f * a3 * c3));
  const float r3 = (b3 + sq3) / (2.f * a3);
  return fminf(r1, fminf(r2, r3));
}

__global__ void __launch_bounds__(256) centernet_targets_kernel(const float* __restrict__ label, int K, float* __restrict__ tgt, int H, int W,
                                                                float ratio_w, float ratio_h, int num_dir_bins, int* __restrict__ count) {
  const int b = blockIdx.x;
  const int HW = H * W;
  float* T = tgt + (int64_t)b * 10 * HW;
  for (int i = threadIdx.x; i < 10 * HW; i += blockDim.x) T[i] = 0.f;
  __syncthreads();
  for (int j = 0; j < K; ++j) {
    const float* L = label + ((int64_t)b * K + j) * 7;
    float sum = 0.f;
    for (int q = 0; q < 7; ++q) sum += L[q];
    if (sum == 0.f) continue;  // uniform over the block
    const float ctx = L[0] * ratio_w, cty = L[1] * ratio_w;  // y also uses width_ratio (model.py:331)
    const int x = (int)ctx, y = (int)cty;
    if (x < 0 || x >= W || y < 0 || y >= H) continue;
    const float box_h = L[3] * ratio_h, box_w = L[2] * ratio_w;
    int r = (int)gaussian_radius_f(box_h, box_w, 0.1f);
    if (r < 2) r = 2;
    const float sigma = (float)((double)(2 * r + 1) / 6.0);
    const float denom = (float)(2.0 * ((double)(2 * r + 1) / 6.0) * ((double)(2 * r + 1) / 6.0));
    (void)sigma;
    const int left = min(x, r), right = min(W - x, r + 1), top = min(y, r), bottom = min(H - y, r + 1);
    const int bw = left + right, bh = top + bottom;
    for (int e = threadIdx.x; e < bw * bh; e += blockDim.x) {
      const int dx = e % bw - left, dy = e / bw - top;
      float g = expf(-(float)(dx * dx + dy * dy) / denom);
      if (g < 1.1920928955078125e-07f) g = 0.f;
      float* h = &T[(y + dy) * W + x + dx];
      *h = fmaxf(*h, g);
    }
    if (threadIdx.x == 0) {
      const int p = y * W + x;
      T[1 * HW + p] = box_w;
      T[2 * HW + p] = box_h;
      T[3 * HW + p] = ctx - (float)x;
      T[4 * HW + p] = cty - (float)y;
      // angle2class (model.py:250-267)
      const float two_pi = 6.283185307179586f;
      const float apc = (float)(6.283185307179586 / (double)num_dir_bins);
      const float half = (float)(6.283185307179586 / (double)num_dir_bins / 2.0);
      const float ang = py_remainder(L[4], two_pi);
      const float shifted = py_remainder(ang + half, two_pi);
      const float cls = truncf(shifted / apc);
      T[5 * HW + p] = shifted - (cls * apc + half);
      T[8 * HW + p] = cls;
      T[6 * HW + p] = L[5];
      T[9 * HW + p] = truncf(L[6]);
      T[7 * HW + p] = 1.f;
    }
    __syncthreads();
  }
  __shared__ int scount;
  if (threadIdx.x == 0) scount = 0;
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) c += (T[i] == 1.f) ? 1 : 0;
  if (c) atomicAdd(&scount, c);
  __syncthreads();
  if (threadIdx.x == 0 && scount) atomicAdd(count, scount);
}

// pred [M][21]: 0 heat logit, 1-2 wh, 3-4 offset, 5-16 yaw class, 17 yaw res, 18 velocity, 19-20 brake.
// acc[7] (sums before normalisation): heat focal, wh L1, offset L1, yaw-class CE, yaw-res SmoothL1, velocity L1, brake CE.
// MODE 0: forward sums.  MODE 1: dpred = d(sum_k coef_k * loss_k)/dpred, coef_k = gout[k] * lw_k / (avg * div_k).
template <int MODE>
__global__ void __launch_bounds__(256) centernet_loss_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, int B, int HW,
                                                             const int* __restrict__ count, double* __restrict__ acc,
                                                             const float* __restrict__ gout, float* __restrict__ dpred,
                                                             float* __restrict__ part = nullptr, unsigned int* __restrict__ cnt = nullptr) {
  __shared__ float red[32];
  constexpr int NP = 21;
  const int64_t M = (int64_t)B * HW;
  float coef[7];
  if (MODE == 1) {
    const float avg = fmaxf(1.f, (float)(*count));
    const float lw[7] = {1.f, 0.1f, 1.f, 1.f, 1.f, 1.f, 1.f};
    const float dv[7] = {1.f, 2.f, 2.f, 1.f, 1.f, 1.f, 1.f};
#pragma unroll
    for (int k = 0; k < 7; ++k) coef[k] = gout[k] * lw[k] / (avg * dv[k]);
  }
  float s[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) s[k] = 0.f;
  for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(m / HW), p = (int)(m % HW);
    const float* P = pred + m * NP;
    const float* T = tgt + (int64_t)b * 10 * HW + p;
    float* D = MODE == 1 ? dpred + m * NP : nullptr;
    const float wt = T[7 * HW];
    float Wsum = 0.f;  // sum over the batch of the weight map at this position (quirk Q2)
    for (int bb = 0; bb < B; ++bb) Wsum += tgt[((int64_t)bb * 10 + 7) * HW + p];
    // --- gaussian focal on sigmoid(heat)
    {
      const float t = T[0];
      const float pr = 1.f / (1.f + expf(-P[0]));
      const float eps = 1e-12f;
      if (MODE == 0) {
        if (t == 1.f) s[0] += -logf(pr + eps) * (1.f - pr) * (1.f - pr);
        const float nw = (1.f - t) * (1.f - t) * (1.f - t) * (1.f - t);
        s[0] += -logf(1.f - pr + eps) * pr * pr * nw;
      } else {
        float dp = 0.f;
        if (t == 1.f) dp += -(1.f - pr) * (1.f - pr) / (pr + eps) + 2.f * (1.f - pr) * logf(pr + eps);
        const float nw = (1.f - t) * (1.f - t) * (1.f - t) * (1.f - t);
        dp += (pr * pr / (1.f - pr + eps) - 2.f * pr * logf(1.f - pr + eps)) * nw;
        D[0] = coef[0] * dp * pr * (1.f - pr);
      }
    }
    // --- L1 terms: wh (1,2), offset (3,4), velocity (18); SmoothL1 yaw res (17)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float d = P[1 + q] - T[(1 + q) * HW];
      const int k = q < 2 ? 1 : 2;
      if (MODE == 0) s[k] += fabsf(d) * wt;
      else D[1 + q] = coef[k] * wt * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
    }
    {
      const float d = P[17] - T[5 * HW];
      const float ad = fabsf(d);
      if (MODE == 0) s[4] += (ad < 1.f ? 0.5f * ad * ad : ad - 0.5f) * wt;
      else D[17] = coef[4] * wt * (ad < 1.f ? d : (d > 0.f ? 1.f : -1.f));
    }
    {
      const float d = P[18] - T[6 * HW];
      if (MODE == 0) s[5] += fabsf(d) * wt;
      else D[18] = coef[5] * wt * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
    }
    // --- CE terms with the batch-summed weight
    {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 12; ++c) mx = fmaxf(mx, P[5 + c]);
      float se = 0.f;
#pragma unroll
      for (int c = 0; c < 12; ++c) se += expf(P[5 + c] - mx);
      const int t = (int)T[8 * HW];
      if (MODE == 0) s[3] += Wsum * (logf(se) + mx - P[5 + t]);
      else {
#pragma unroll
        for (int c = 0; c < 12; ++c) D[5 + c] = coef[3] * Wsum * (expf(P[5 + c] - mx) / se - (c == t ? 1.f : 0.f));
      }
    }
    {
      const float a = P[19], bq = P[20];
      const float mx = fmaxf(a, bq);
      const float ea = expf(a - mx), eb = expf(bq - mx), se = ea + eb;
      const int t = (int)T[9 * HW];
      if (MODE == 0) s[6] += Wsum * (logf(se) + mx - (t == 0 ? a : bq));
      else {
        D[19] = coef[6] * Wsum * (ea / se - (t == 0 ? 1.f : 0.f));
        D[20] = coef[6] * Wsum * (eb / se - (t == 1 ? 1.f : 0.f));
      }
    }
  }
  if (MODE == 0) {
#pragma unroll
    for (int k = 0; k < 7; ++k) block_partial(part, 7, k, s[k], red);
    blocks_finish(part, 7, acc, cnt);
  }
}

// out[k] = lw_k * acc[k] / (max(1,count) * div_k)
__global__ void centernet_finalize_kernel(const double* __restrict__ acc, const int* __restrict__ count, float* __restrict__ out) {
  const int k = threadIdx.x;
  if (k >= 7) return;
  const double avg = fmax(1.0, (double)(*count));
  const double lw[7] = {1.0, 0.1, 1.0, 1.0, 1.0, 1.0, 1.0};
  const double dv[7] = {1.0, 2.0, 2.0, 1.0, 1.0, 1.0, 1.0};
  out[k] = (float)(lw[k] * acc[k] / (avg * dv[k]));
}

// out = k * num / (den ? max(den, den_min) : 1)
__global__ void ratio_kernel(const double* __restrict__ num, const double* __restrict__ den, float den_min, float k, float* __restrict__ out) {
  double v = (double)k * (*num);
  if (den) v /= fmax(*den, (double)den_min);
  *out = (float)v;
}

}  // namespace

TFB_API int tfb_ce_fwd(const float* logits, const int64_t* target, int64_t M, int C, const float* class_w, const float* pos_w, int HW,
                       double* acc2, cudaStream_t stream) {
  TFB_REQUIRE(logits && target && acc2 && M > 0 && C > 0 && C <= kMaxC && HW > 0);
  if (cudaMemsetAsync(acc2, 0, 2 * sizeof(double), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  const int grid = tfb_grid(M, 256, 4);
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)grid * 2, 1, stream);
  if (rc != TFB_OK) return rc;
  ce_fwd_kernel<<<grid, 256, 0, stream>>>(logits, target, M, C, class_w, pos_w, HW, acc2, w.f, w.cnt);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_ce_bwd(const float* logits, const int64_t* target, int64_t M, int C, const float* class_w, const float* pos_w, int HW,
                       const float* gout_dev, const double* den_dev, float den_min, float k, float* dlogits, cudaStream_t stream) {
  TFB_REQUIRE(logits && target && dlogits && M > 0 && C > 0 && C <= kMaxC && HW > 0);
  ce_bwd_kernel<<<tfb_grid(M, 256), 256, 0, stream>>>(logits, target, M, C, class_w, pos_w, HW, gout_dev, den_dev, den_min, k, dlogits);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_l1_fwd(const float* x, const float* t, int64_t n, int sigmoid, double* acc1, cudaStream_t stream) {
  TFB_REQUIRE(x && t && acc1 && n > 0);
  if (cudaMemsetAsync(acc1, 0, sizeof(double), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  const int grid = tfb_grid(n, 256, 4);
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)grid, 1, stream);
  if (rc != TFB_OK) return rc;
  l1_fwd_kernel<<<grid, 256, 0, stream>>>(x, t, n, sigmoid, acc1, w.f, w.cnt);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_l1_bwd(const float* x, const float* t, int64_t n, int sigmoid, const float* gout_dev, float k, float* dx,
                       cudaStream_t stream) {
  TFB_REQUIRE(x && t && dx && n > 0);
  l1_bwd_kernel<<<tfb_grid(n, 256), 256, 0, stream>>>(x, t, n, sigmoid, gout_dev, k, dx);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_ratio(const double* num_dev, const double* den_dev, float den_min, float k, float* out, cudaStream_t stream) {
  TFB_REQUIRE(num_dev && out);
  ratio_kernel<<<1, 1, 0, stream>>>(num_dev, den_dev, den_min, k, out);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_centernet_targets(const float* label, int B, int K, float* tgt, int H, int W, float ratio_w, float ratio_h,
                                  int num_dir_bins, int* count, cudaStream_t stream) {
  TFB_REQUIRE(label && tgt && count && B > 0 && K >= 0 && H > 0 && W > 0);
  if (cudaMemsetAsync(count, 0, sizeof(int), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  centernet_targets_kernel<<<B, 256, 0, stream>>>(label, K, tgt, H, W, ratio_w, ratio_h, num_dir_bins, count);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_centernet_loss_fwd(const float* pred, const float* tgt, int B, int HW, const int* count, double* acc7, float* out7,
                                   cudaStream_t stream) {
  TFB_REQUIRE(pred && tgt && count && acc7 && out7 && B > 0 && HW > 0);
  if (cudaMemsetAsync(acc7, 0, 7 * sizeof(double), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  const int grid = tfb_grid((int64_t)B * HW, 256, 2);
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)grid * 7, 1, stream);
  if (rc != TFB_OK) return rc;
  centernet_loss_kernel<0><<<grid, 256, 0, stream>>>(pred, tgt, B, HW, count, acc7, nullptr, nullptr, w.f, w.cnt);
  TFB_CHECK_LAUNCH();
  centernet_finalize_kernel<<<1, 32, 0, stream>>>(acc7, count, out7);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
TFB_API int tfb_centernet_loss_bwd(const float* pred, const float* tgt, int B, int HW, const int* count, const float* gout7,
                                   float* dpred, cudaStream_t stream) {
  TFB_REQUIRE(pred && tgt && count && gout7 && dpred && B > 0 && HW > 0);
  centernet_loss_kernel<1><<<tfb_grid((int64_t)B * HW, 256, 2), 256, 0, stream>>>(pred, tgt, B, HW, count, nullptr, gout7, dpred);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
