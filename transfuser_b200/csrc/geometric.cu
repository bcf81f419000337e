// Kernels specific to GeometricFusionBackbone (geometric_fusion.py:98-296): the anchor-grid average pool and the
// "gather 5 projected correspondences and sum" that the reference writes as a B x B advanced index + torch.diagonal +
// permute + sum (geometric_fusion.py:145-148 and the 7 copies of it). Everything else in that backbone (1x1 embeds, the
// 3-layer projection MLPs, bilinear upsample, residual adds) runs on the shared GEMM / upsample / add kernels.
// Layout: NHWC fp32. Both ops are HBM-bound streaming kernels; channels are the fastest dim so every access is a
// coalesced float4 row segment.
#include "common.cuh"

namespace {

// out[n,gy,gx,:] = mean over the (H/gh) x (W/gw) window; accumulation order = rows then columns, then one division
// (the order ATen's CPU adaptive_avg_pool2d uses, so uniform windows reproduce it bit for bit).
template <int VEC>
__global__ void __launch_bounds__(256) avgpool_grid_fwd_kernel(const float* __restrict__ x, float* __restrict__ out, int N, int H, int W, int C,
                                                               int gh, int gw) {
  const int kh = H / gh, kw = W / gw, CV = C / VEC;
  const int64_t total = (int64_t)N * gh * gw * CV;
  const float cnt = (float)(kh * kw);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    int64_t r = i / CV;
    const int gx = (int)(r % gw); r /= gw;
    const int gy = (int)(r % gh);
    const int n = (int)(r / gh);
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
    for (int dy = 0; dy < kh; ++dy)
      for (int dx = 0; dx < kw; ++dx) {
        const float* s = x + (((int64_t)n * H + gy * kh + dy) * W + gx * kw + dx) * C + cv * VEC;
        if (VEC == 4) {
          const float4 t = *reinterpret_cast<const float4*>(s);
          acc[0] += t.x; acc[1] += t.y; acc[2] += t.z; acc[3] += t.w;
        } else {
          acc[0] += s[0];
        }
      }
    float* o = out + i * VEC;
#pragma unroll
    for (int v = 0; v < VEC; ++v) o[v] = acc[v] / cnt;
  }
}

// dx[n,y,x,:] (+)= dout[n, y/kh, x/kw, :] / (kh*kw)
template <int VEC>
__global__ void __launch_bounds__(256) avgpool_grid_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dx, int N, int H, int W, int C,
                                                               int gh, int gw, int accumulate) {
  const int kh = H / gh, kw = W / gw, CV = C / VEC;
  const int64_t total = (int64_t)N * H * W * CV;
  const float cnt = (float)(kh * kw);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    int64_t r = i / CV;
    const int xx = (int)(r % W); r /= W;
    const int yy = (int)(r % H);
    const int n = (int)(r / H);
    const float* g = dout + (((int64_t)n * gh + yy / kh) * gw + xx / kw) * C + cv * VEC;
    float* d = dx + i * VEC;
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      const float t = g[v] / cnt;
      d[v] = accumulate ? d[v] + t : t;
    }
  }
}

__device__ __forceinline__ bool resolve_cell(const int64_t* pt, int h, int w, int* cell) {
  int64_t px = pt[0], py = pt[1];       // (x, y): the reference indexes [:, pts[:,1], pts[:,0]] on an [B,h,w,C] view
  if (px < 0) px += w;                  // python-style negative indices, like the advanced index it replaces
  if (py < 0) py += h;
  if (px < 0 || px >= w || py < 0 || py >= h) return false;
  *cell = (int)(py * w + px);
  return true;
}

// out[b,m,:] = sum_{j<P} emb[b, pts[b,m,j].y, pts[b,m,j].x, :]   (added in j order, as torch.sum over the last dim does)
__global__ void __launch_bounds__(256) gather_sum_fwd_kernel(const float* __restrict__ emb, const int64_t* __restrict__ pts, float* __restrict__ out,
                                                             int B, int h, int w, int C, int M, int P) {
  const int CV = C >> 2;
  const int64_t total = (int64_t)B * M * CV;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    const int64_t bm = i / CV;
    const int b = (int)(bm / M);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < P; ++j) {
      int cell;
      if (!resolve_cell(pts + (bm * P + j) * 2, h, w, &cell)) continue;
      const float4 t = *reinterpret_cast<const float4*>(emb + ((int64_t)b * h * w + cell) * C + cv * 4);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    *reinterpret_cast<float4*>(out + i * 4) = acc;
  }
}

// demb[b, cell(b,m,j), :] += dout[b,m,:]   (demb zeroed by the entry point). Duplicate cells are the common case: one thread per
// (b, c) owns column c of sample b's demb and adds the correspondences in (m, j) order, so the sums are the same bits every run
// (consecutive threads = consecutive channels: the dout reads and demb updates stay coalesced).
__global__ void __launch_bounds__(256) gather_sum_bwd_kernel(const float* __restrict__ dout, const int64_t* __restrict__ pts, float* __restrict__ demb,
                                                             int B, int h, int w, int C, int M, int P) {
  const int64_t total = (int64_t)B * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C), b = (int)(i / C);
    float* col = demb + (int64_t)b * h * w * C + c;
    for (int m = 0; m < M; ++m) {
      const int64_t bm = (int64_t)b * M + m;
      const float g = dout[bm * C + c];
      for (int j = 0; j < P; ++j) {
        int cell;
        if (!resolve_cell(pts + (bm * P + j) * 2, h, w, &cell)) continue;
        col[(int64_t)cell * C] += g;
      }
    }
  }
}

}  // namespace

// AdaptiveAvgPool2d((gh,gw)) on NHWC for maps that divide evenly (geometric_fusion.py:19-20 on 40x176..5x22 / 64..8 maps).
TFB_API int tfb_avgpool_grid_fwd(const float* x, float* out, int N, int H, int W, int C, int gh, int gw, cudaStream_t stream) {
  TFB_REQUIRE(x && out && N > 0 && C > 0 && gh > 0 && gw > 0 && H >= gh && W >= gw && H % gh == 0 && W % gw == 0);
  if (C % 4 == 0)
    avgpool_grid_fwd_kernel<4><<<tfb_grid((int64_t)N * gh * gw * (C / 4), 256), 256, 0, stream>>>(x, out, N, H, W, C, gh, gw);
  else
    avgpool_grid_fwd_kernel<1><<<tfb_grid((int64_t)N * gh * gw * C, 256), 256, 0, stream>>>(x, out, N, H, W, C, gh, gw);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

TFB_API int tfb_avgpool_grid_bwd(const float* dout, float* dx, int N, int H, int W, int C, int gh, int gw, int accumulate, cudaStream_t stream) {
  TFB_REQUIRE(dout && dx && N > 0 && C > 0 && gh > 0 && gw > 0 && H >= gh && W >= gw && H % gh == 0 && W % gw == 0);
  if (C % 4 == 0)
    avgpool_grid_bwd_kernel<4><<<tfb_grid((int64_t)N * H * W * (C / 4), 256), 256, 0, stream>>>(dout, dx, N, H, W, C, gh, gw, accumulate);
  else
    avgpool_grid_bwd_kernel<1><<<tfb_grid((int64_t)N * H * W * C, 256), 256, 0, stream>>>(dout, dx, N, H, W, C, gh, gw, accumulate);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// emb [B,h,w,C], pts [B,M,P,2] int64 (x,y) -> out [B,M,C]. Out-of-range correspondences contribute nothing (the
// reference would raise); negative ones wrap like Python indices.
TFB_API int tfb_gather_sum_fwd(const float* emb, const int64_t* pts, float* out, int B, int h, int w, int C, int M, int P, cudaStream_t stream) {
  TFB_REQUIRE(emb && pts && out && B > 0 && h > 0 && w > 0 && C > 0 && C % 4 == 0 && M > 0 && P > 0);
  gather_sum_fwd_kernel<<<tfb_grid((int64_t)B * M * (C / 4), 256), 256, 0, stream>>>(emb, pts, out, B, h, w, C, M, P);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

TFB_API int tfb_gather_sum_bwd(const float* dout, const int64_t* pts, float* demb, int B, int h, int w, int C, int M, int P, cudaStream_t stream) {
  TFB_REQUIRE(dout && pts && demb && B > 0 && h > 0 && w > 0 && C > 0 && M > 0 && P > 0);
  if (cudaMemsetAsync(demb, 0, (size_t)B * h * w * C * sizeof(float), stream) != cudaSuccess) return TFB_ERR_DRIVER;
  gather_sum_bwd_kernel<<<tfb_grid((int64_t)B * C, 256), 256, 0, stream>>>(dout, pts, demb, B, h, w, C, M, P);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
