// (1) GRU waypoint decoder of LidarCenterNet.forward_gru (model.py:611-646): 4 autoregressive GRUCell(4 -> 64) steps +
//     Linear(64 -> 3) + cumulative sum, forward and full BPTT backward, one CTA per sample (CUDA cores; tiny).
// (2) Fused AdamW over one flat fp32 parameter buffer (replaces torch.optim.AdamW's foreach kernels, train.py:142,314),
//     optionally emitting the bf16 copy of the weights used by the tensor-core GEMMs. HBM-bound: 28 B/param (+2 B bf16).
#include "common.cuh"

namespace {

constexpr int HID = 64, G3 = 192, XIN = 4, SAVE = 5 * HID + XIN;  // per (sample, step): r, z, n, hn_lin, h_prev, x_in

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

__global__ void __launch_bounds__(G3)
gru_fwd_kernel(const float* __restrict__ z0, const float* __restrict__ target_point, const float* __restrict__ w_ih,
               const float* __restrict__ w_hh, const float* __restrict__ b_ih, const float* __restrict__ b_hh,
               const float* __restrict__ w_out, const float* __restrict__ b_out, int steps, float x_shift, float* __restrict__ pred_wp,
               float* __restrict__ save) {
  __shared__ float h[HID], gi[G3], gh[G3], xin[XIN], xcur[2], dxo[3];
  const int b = blockIdx.x, k = threadIdx.x;
  if (k < HID) h[k] = z0[(int64_t)b * HID + k];
  if (k == 0) {
    xcur[0] = 0.f; xcur[1] = 0.f;
    xin[2] = target_point[b * 2 + 0];
    xin[3] = -target_point[b * 2 + 1];  // y of the target point is negated (model.py:619-620)
  }
  __syncthreads();
  for (int t = 0; t < steps; ++t) {
    if (k == 0) { xin[0] = xcur[0]; xin[1] = xcur[1]; }
    __syncthreads();
    float a = b_ih[k], c = b_hh[k];
#pragma unroll
    for (int j = 0; j < XIN; ++j) a = fmaf(w_ih[k * XIN + j], xin[j], a);
    for (int j = 0; j < HID; ++j) c = fmaf(w_hh[k * HID + j], h[j], c);
    gi[k] = a; gh[k] = c;
    __syncthreads();
    float* sv = save + ((int64_t)b * steps + t) * SAVE;
    float hnew = 0.f;
    if (k < HID) {
      const float r = sigmoidf_(gi[k] + gh[k]);
      const float z = sigmoidf_(gi[HID + k] + gh[HID + k]);
      const float n = tanhf(gi[2 * HID + k] + r * gh[2 * HID + k]);
      hnew = (1.f - z) * n + z * h[k];
      sv[k] = r; sv[HID + k] = z; sv[2 * HID + k] = n; sv[3 * HID + k] = gh[2 * HID + k]; sv[4 * HID + k] = h[k];
    }
    if (k < XIN) sv[5 * HID + k] = xin[k];
    __syncthreads();
    if (k < HID) h[k] = hnew;
    __syncthreads();
    if (k < 3) {
      float o = b_out[k];
      for (int j = 0; j < HID; ++j) o = fmaf(w_out[k * HID + j], h[j], o);
      dxo[k] = o;
    }
    __syncthreads();
    if (k == 0) {
      xcur[0] += dxo[0]; xcur[1] += dxo[1];
      pred_wp[((int64_t)b * steps + t) * 2 + 0] = xcur[0] - x_shift;  // vehicle -> lidar frame (model.py:639)
      pred_wp[((int64_t)b * steps + t) * 2 + 1] = xcur[1];
    }
    __syncthreads();
  }
}

// Parameter gradients: block b accumulates its sample's share in its own slice of `part` (every element owned by one thread),
// and the last block adds the slices in sample order into the outputs (the same bits every run).
constexpr int O_WHH = G3 * XIN, O_BIH = O_WHH + G3 * HID, O_BHH = O_BIH + G3, O_WOUT = O_BHH + G3, O_BOUT = O_WOUT + 3 * HID,
              P_GRU = O_BOUT + 3;
__global__ void __launch_bounds__(G3)
gru_bwd_kernel(const float* __restrict__ d_wp, const float* __restrict__ save, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
               const float* __restrict__ w_out, int steps, float* __restrict__ dz0, float* __restrict__ dw_ih_out, float* __restrict__ dw_hh_out,
               float* __restrict__ db_ih_out, float* __restrict__ db_hh_out, float* __restrict__ dw_out_out, float* __restrict__ db_out_out,
               float* __restrict__ part, unsigned int* __restrict__ cnt) {
  __shared__ float dh[HID], dgi[G3], dgh[G3], hnew[HID], dxacc[2], dxin[XIN];
  const int b = blockIdx.x, k = threadIdx.x;
  float* pb = part + (int64_t)b * P_GRU;
  for (int i = k; i < P_GRU; i += blockDim.x) pb[i] = 0.f;
  float *dw_ih = pb, *dw_hh = pb + O_WHH, *db_ih = pb + O_BIH, *db_hh = pb + O_BHH, *dw_out = pb + O_WOUT, *db_out = pb + O_BOUT;
  if (k < HID) dh[k] = 0.f;
  if (k < 2) dxacc[k] = 0.f;
  __syncthreads();
  for (int t = steps - 1; t >= 0; --t) {
    const float* sv = save + ((int64_t)b * steps + t) * SAVE;
    if (k < 2) dxacc[k] += d_wp[((int64_t)b * steps + t) * 2 + k];
    if (k < HID) hnew[k] = (1.f - sv[HID + k]) * sv[2 * HID + k] + sv[HID + k] * sv[4 * HID + k];
    __syncthreads();
    // output Linear: only rows 0,1 of dxo are used
    if (k < HID) {
      dh[k] += w_out[k] * dxacc[0] + w_out[HID + k] * dxacc[1];
      dw_out[k] += dxacc[0] * hnew[k];
      dw_out[HID + k] += dxacc[1] * hnew[k];
    }
    if (k < 2) db_out[k] += dxacc[k];
    __syncthreads();
    if (k < HID) {
      const float r = sv[k], z = sv[HID + k], n = sv[2 * HID + k], hn = sv[3 * HID + k], hp = sv[4 * HID + k];
      const float g = dh[k];
      const float dn_pre = g * (1.f - z) * (1.f - n * n);
      const float dz_pre = g * (hp - n) * z * (1.f - z);
      const float dr_pre = dn_pre * hn * r * (1.f - r);
      dgi[k] = dr_pre; dgi[HID + k] = dz_pre; dgi[2 * HID + k] = dn_pre;
      dgh[k] = dr_pre; dgh[HID + k] = dz_pre; dgh[2 * HID + k] = dn_pre * r;
      dh[k] = g * z;  // direct path to h_prev
    }
    __syncthreads();
    // parameter gradients
    {
      const float gi_k = dgi[k], gh_k = dgh[k];
#pragma unroll
      for (int j = 0; j < XIN; ++j) dw_ih[k * XIN + j] += gi_k * sv[5 * HID + j];
      db_ih[k] += gi_k;
      db_hh[k] += gh_k;
      for (int j = 0; j < HID; ++j) dw_hh[k * HID + j] += gh_k * sv[4 * HID + j];
    }
    // input gradients
    if (k < XIN) {
      float s = 0.f;
      for (int q = 0; q < G3; ++q) s = fmaf(w_ih[q * XIN + k], dgi[q], s);
      dxin[k] = s;
    }
    float dhp = 0.f;
    if (k < HID) {
      for (int q = 0; q < G3; ++q) dhp = fmaf(w_hh[q * HID + k], dgh[q], dhp);
    }
    __syncthreads();
    if (k < HID) dh[k] += dhp;
    if (k < 2) dxacc[k] += dxin[k];  // x_t feeds both the identity path (already in dxacc) and the GRU input
    __syncthreads();
  }
  if (k < HID) dz0[(int64_t)b * HID + k] = dh[k];
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (k == 0) last = atomicAdd(cnt, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int i = k; i < P_GRU; i += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < (int)gridDim.x; ++q) s += __ldcg(part + (int64_t)q * P_GRU + i);
    if (i < O_WHH) dw_ih_out[i] = s;
    else if (i < O_BIH) dw_hh_out[i - O_WHH] = s;
    else if (i < O_BHH) db_ih_out[i - O_BIH] = s;
    else if (i < O_WOUT) db_hh_out[i - O_BHH] = s;
    else if (i < O_BOUT) dw_out_out[i - O_WOUT] = s;
    else db_out_out[i - O_BOUT] = s;
  }
  if (k == 0) *cnt = 0u;                // the stream's scratch counters are zero on entry
}

// torch.optim.AdamW semantics, scalar preparation included: torch derives 1-beta, 1-lr*wd, lr/bias_correction1 and
// sqrt(bias_correction2) in float64 from the Python floats and rounds each to fp32 once; the hyper-parameters therefore arrive
// here as doubles (1.f - 0.999f would be 4.7e-5 off the 0.001 torch uses).
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n, double lr,
             double beta1, double beta2, float eps, double wd, int step_host, float grad_scale, __nv_bfloat16* __restrict__ p_bf16,
             int zero_grad, const int* __restrict__ step_dev, const double* __restrict__ hp_dev) {
  // step count in device memory when given (valid under CUDA-graph replay), else the host's
  const double t = step_dev ? (double)(*step_dev) : (double)step_host;
  // hyper-parameters in device memory when given ([lr, beta1, beta2, eps, weight_decay]): a learning-rate schedule (train.py:194-199)
  // then takes effect inside a replayed CUDA graph, where the host scalars are frozen at capture time
  if (hp_dev) { lr = hp_dev[0]; beta1 = hp_dev[1]; beta2 = hp_dev[2]; eps = (float)hp_dev[3]; wd = hp_dev[4]; }
  const float step = (float)(lr / (1.0 - pow(beta1, t)));
  const float bc2_sqrt = (float)sqrt(1.0 - pow(beta2, t));
  const float decay = (float)(1.0 - lr * wd);
  const float b1 = (float)beta1, b2 = (float)beta2, omb1 = (float)(1.0 - beta1), omb2 = (float)(1.0 - beta2);
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i], G = reinterpret_cast<float4*>(g)[i];
    float4 Mv = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
    float* pp = &P.x; float* gg = &G.x; float* mm = &Mv.x; float* vv = &V.x;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float gr = gg[q] * grad_scale;
      pp[q] *= decay;
      mm[q] = b1 * mm[q] + omb1 * gr;
      vv[q] = b2 * vv[q] + omb2 * gr * gr;
      pp[q] -= step * (mm[q] / (sqrtf(vv[q]) / bc2_sqrt + eps));
    }
    reinterpret_cast<float4*>(p)[i] = P;
    reinterpret_cast<float4*>(m)[i] = Mv;
    reinterpret_cast<float4*>(v)[i] = V;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p_bf16) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(P.x, P.y), hi = __floats2bfloat162_rn(P.z, P.w);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&lo);
      o.y = *reinterpret_cast<uint32_t*>(&hi);
      reinterpret_cast<uint2*>(p_bf16)[i] = o;
    }
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gr = g[i] * grad_scale;
    float P = p[i] * decay;
    const float Mv = b1 * m[i] + omb1 * gr;
    const float V = b2 * v[i] + omb2 * gr * gr;
    P -= step * (Mv / (sqrtf(V) / bc2_sqrt + eps));
    p[i] = P; m[i] = Mv; v[i] = V;
    if (zero_grad) g[i] = 0.f;
    if (p_bf16) p_bf16[i] = __float2bfloat16_rn(P);
  }
}

}  // namespace

TFB_API int tfb_gru_fwd(const float* z0, const float* target_point, const float* w_ih, const float* w_hh, const float* b_ih,
                        const float* b_hh, const float* w_out, const float* b_out, int B, int steps, float x_shift, float* pred_wp,
                        float* save, cudaStream_t stream) {
  TFB_REQUIRE(z0 && target_point && w_ih && w_hh && b_ih && b_hh && w_out && b_out && pred_wp && save && B > 0 && steps > 0);
  gru_fwd_kernel<<<B, G3, 0, stream>>>(z0, target_point, w_ih, w_hh, b_ih, b_hh, w_out, b_out, steps, x_shift, pred_wp, save);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

TFB_API int tfb_gru_bwd(const float* d_wp, const float* save, const float* w_ih, const float* w_hh, const float* w_out, int B, int steps,
                        float* dz0, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh, float* dw_out, float* db_out,
                        cudaStream_t stream) {
  TFB_REQUIRE(d_wp && save && w_ih && w_hh && w_out && dz0 && dw_ih && dw_hh && db_ih && db_hh && dw_out && db_out && B > 0 && steps > 0);
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)B * P_GRU, 1, stream);
  if (rc != TFB_OK) return rc;
  gru_bwd_kernel<<<B, G3, 0, stream>>>(d_wp, save, w_ih, w_hh, w_out, steps, dz0, dw_ih, dw_hh, db_ih, db_hh, dw_out, db_out, w.f, w.cnt);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// zero_grad != 0: the gradient buffer is cleared in the same pass. step_dev (optional): optimizer step count in device memory
// (incremented by tfb_step_tick) — used instead of `step`, so a captured CUDA graph stays valid across replays.
// hp_dev (optional): [lr, beta1, beta2, eps, weight_decay] as doubles in device memory, used instead of the scalar arguments.
TFB_API int tfb_adamw_step(float* p, float* g, float* m, float* v, int64_t n, double lr, double beta1, double beta2, double eps,
                           double weight_decay, int step, const int* step_dev, float grad_scale, void* p_bf16, int zero_grad,
                           const double* hp_dev, cudaStream_t stream) {
  TFB_REQUIRE(p && g && m && v && n >= 0 && (step >= 1 || step_dev));
  if (n == 0) return TFB_OK;
  adamw_kernel<<<tfb_grid(n / 4 + 1, 256), 256, 0, stream>>>(p, g, m, v, n, lr, beta1, beta2, (float)eps, weight_decay, step, grad_scale,
                                                              (__nv_bfloat16*)p_bf16, zero_grad, step_dev, hp_dev);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

namespace {
__global__ void step_tick_kernel(unsigned long long* seed_dev, int* step_dev) {
  if (seed_dev) *seed_dev += 0x9E3779B97F4A7C15ull;
  if (step_dev) *step_dev += 1;
}
}  // namespace

// Once per training step: advances the device-resident dropout base seed and / or the optimizer step counter.
TFB_API int tfb_step_tick(uint64_t* seed_dev, int* step_dev, cudaStream_t stream) {
  step_tick_kernel<<<1, 1, 0, stream>>>((unsigned long long*)seed_dev, step_dev);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
