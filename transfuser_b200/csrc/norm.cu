// BatchNorm2d (training mode, NHWC as a [M, C] matrix) and LayerNorm, forward + backward. HBM-bound.
// Replaces cuDNN/ATen batch_norm inside timm's BatchNormAct2d (every conv of the RegNetY trunks, transfuser.py:136-184)
// and nn.LayerNorm in Block / GPT.ln_f (transfuser.py:533-534, 321).
//   BN fwd : stats (per-channel sum, sum of squares; fp32 partials combined in fp64) -> normalise (+ReLU) + running stats
//   BN bwd : reduce (sum g, sum g*xhat with the ReLU mask recomputed from x) -> dx, dgamma, dbeta
#include <cstdlib>
#include "common.cuh"

namespace {

// "Last block finalises" epilogue of the column reductions. The workspace `sums` (doubles) is ZERO on entry to every kernel
// that uses it and is zeroed again here by the last block, together with the arrival counter stored right behind it, so no
// memset / convert / finalize launches are needed and one workspace serves every layer on a stream.
//   kind 0: nothing (no reduction output requested)
//   kind 1: BatchNorm forward  -> save_mean, save_invstd, running statistics        (sums = [sum x | sum x^2])
//   kind 2: BatchNorm backward -> dgamma = sum g*xhat, dbeta = sum g                 (sums = [sum g | sum g*xhat])
//   kind 3: column sum         -> out[c] = sum                                        (sums = [sum])
//   kind 4: BatchNorm forward of one rank of a synchronized BatchNorm -> `slice` only, + slice[2C] = M   (sums = [sum x | sum x^2])
struct Finalize {
  int kind;
  int nsums;             // doubles in use (C or 2C); the counter lives at sums[nsums]
  int64_t M;
  float eps, momentum;
  float* o0;             // save_mean | dbeta  | out
  float* o1;             // save_invstd | dgamma
  float* running_mean;
  float* running_var;
  float* zero_buf;       // optional: zero_n floats cleared by the last block (the SE pooling accumulator of the NEXT kernel on the
  int zero_n;            // stream, tfb_bn_fwd with pooling: saves the memset node)
  double* part;          // [nsplit][nsums]: each row split's partial sums; the last block of a slab adds them in split order, so the
                         // result is the same bits on every run (set by the launcher, see alloc_partials)
  unsigned int* cnt;     // one arrival counter per channel slab, in the stream's scratch (alloc_partials)
  double* slice;         // optional: the folded sums are also written here in fp64 (a rank's slice of a synchronized BatchNorm)
};

// save_mean / save_invstd / running statistics of channel c from its sums over N rows (N = M, or the count summed over the ranks of a
// synchronized BatchNorm); returns invstd. Null save_mean / running_mean: not written.
__device__ __forceinline__ float bn_publish(int c, double s0, double s1, double N, float eps, float momentum, float* __restrict__ save_mean,
                                            float* __restrict__ save_invstd, float* __restrict__ running_mean, float* __restrict__ running_var,
                                            double* mean_out = nullptr) {
  const double mean = s0 / N;
  double var = s1 / N - mean * mean;
  if (var < 0.0) var = 0.0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  if (save_mean) { save_mean[c] = (float)mean; save_invstd[c] = invstd; }
  if (running_mean) {
    const double unbiased = N > 1.0 ? var * N / (N - 1.0) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
  if (mean_out) *mean_out = mean;
  return invstd;
}

// The partials of channel slab `slab` (channels [slab * slab_w, +slab_w)) come from the nsplit blocks of that slab; the last of them
// to arrive (arrival counter f.cnt[slab]) folds the slab's channels in split order and finalises them, so the slabs finish in parallel.
// MAXW >= slab_w: 32 or 128 for the slabs of the 2-D grids, 512 for colreduce_flat_kernel (all channels, C / 4 <= 128).
template <int MAXW>
__device__ __forceinline__ void finalize_last_block(double* sums, int C, const Finalize& f, int nsplit, int slab, int slab_w) {
  if (f.kind == 0) return;
  __shared__ bool is_last;
  __shared__ double fs[2][MAXW];
  __threadfence();
  __syncthreads();
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
  if (tid == 0) is_last = atomicAdd(f.cnt + slab, 1u) == (unsigned int)(nsplit - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int lo = slab * slab_w, w = min(slab_w, C - lo), nq = f.nsums > C ? 2 : 1;
  auto all = [](int) { return true; };
  if ((C & 1) == 0) {                // then lo and w are even: pairs of channels, 16-byte loads
    const int hw = w / 2;
    ordered_fold<double, 2>(f.part, f.nsums, nsplit, (int64_t)nq * hw, [&](int64_t g) { return (g / hw) * C + lo + (g % hw) * 2; }, all,
                            [&](int64_t g, const double (&s)[2]) { fs[g / hw][(g % hw) * 2] = s[0]; fs[g / hw][(g % hw) * 2 + 1] = s[1]; },
                            tid, nthr);
  } else {
    ordered_fold<double, 1>(f.part, f.nsums, nsplit, (int64_t)nq * w, [&](int64_t g) { return (g / w) * C + lo + g % w; }, all,
                            [&](int64_t g, const double (&s)[1]) { fs[g / w][g % w] = s[0]; }, tid, nthr);
  }
  __syncthreads();
  for (int i = tid; i < w; i += nthr) {
    const int c = lo + i;
    const double s0 = fs[0][i], s1 = nq > 1 ? fs[1][i] : 0.0;
    if (f.slice) {
      f.slice[c] = s0;
      if (nq > 1) f.slice[C + c] = s1;
    }
    if (f.kind == 1) {
      bn_publish(c, s0, s1, (double)f.M, f.eps, f.momentum, f.o0, f.o1, f.running_mean, f.running_var);
    } else if (f.kind == 2) {
      f.o0[c] = (float)s0;
      f.o1[c] = (float)s1;
    } else if (f.kind == 3) {
      f.o0[c] = (float)s0;
    }
    sums[c] = 0.0;
    if (f.nsums > C) sums[C + c] = 0.0;
  }
  if (slab == 0)
    for (int i = tid; i < f.zero_n; i += nthr) f.zero_buf[i] = 0.f;
  if (f.kind == 4 && slab == 0 && tid == 0) f.slice[f.nsums] = (double)f.M;
  if (tid == 0) f.cnt[slab] = 0u;    // the stream's scratch counters are zero on entry
}

// Gradient entering a BatchNorm whose output feeds a squeeze-excite gate (y = bn_out * gate[n][c]): with dy the gradient of the SE
// OUTPUT, the gradient of the BatchNorm output is dy * gate[n][c] + dpool[n][c] / HW (dpool: gradient of the pooled vector through the
// SE MLP). Folding it into the BatchNorm backward kernels removes the separate se_bwd_apply pass (one write + one read of the map).
__device__ __forceinline__ void se_grad4(float g[4], const float* __restrict__ gate, const float* __restrict__ dpool, int64_t nc, float inv_hw) {
  const float4 ga = *reinterpret_cast<const float4*>(gate + nc), dp = *reinterpret_cast<const float4*>(dpool + nc);
  g[0] = fmaf(g[0], ga.x, dp.x * inv_hw); g[1] = fmaf(g[1], ga.y, dp.y * inv_hw);
  g[2] = fmaf(g[2], ga.z, dp.z * inv_hw); g[3] = fmaf(g[3], ga.w, dp.w * inv_hw);
}

// ---------------- per-channel column reductions over a [M, C] matrix ----------------
// block (32, 8): threadIdx.x -> channel inside a 32-wide slab, threadIdx.y -> row phase. grid (slabs, row splits).
// MODE 0: (sum x, sum x^2)            MODE 1: BN backward (sum g, sum g*xhat), g = dy * relu_mask
template <int MODE>
__global__ void __launch_bounds__(256)
colreduce_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dy, int64_t M, int C, double* __restrict__ out,
                 const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                 const float* __restrict__ beta, int relu, const float* __restrict__ ymask, Finalize fin) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a0 = 0.f, a1 = 0.f;
  double d0 = 0.0, d1 = 0.0;
  if (c < C) {
    float mu = 0.f, is = 0.f, ga = 0.f, be = 0.f;
    if (MODE == 1) { mu = mean[c]; is = invstd[c]; ga = gamma[c]; be = beta[c]; }
    int cnt = 0;
    for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < M; r += (int64_t)gridDim.y * 8) {
      const float v = x[r * ldx + c];
      if (MODE == 0) {
        a0 += v; a1 = fmaf(v, v, a1);
      } else {
        const float xh = (v - mu) * is;
        float g = dy[r * C + c];
        if (ymask) { if (!(ymask[r * C + c] > 0.f)) g = 0.f; }
        else if (relu && !(fmaf(xh, ga, be) > 0.f)) g = 0.f;
        a0 += g; a1 = fmaf(g, xh, a1);
      }
      if (++cnt == 64) { d0 += a0; d1 += a1; a0 = a1 = 0.f; cnt = 0; }  // bound fp32 partial length
    }
    d0 += a0; d1 += a1;
  }
  // combine the 8 row phases in fp64
  __shared__ double sd0[8][33], sd1[8][33];
  sd0[threadIdx.y][threadIdx.x] = d0;
  sd1[threadIdx.y][threadIdx.x] = d1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double t0 = 0.0, t1 = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { t0 += sd0[j][threadIdx.x]; t1 += sd1[j][threadIdx.x]; }
    fin.part[(int64_t)blockIdx.y * fin.nsums + c] = t0;
    if (fin.nsums > C) fin.part[(int64_t)blockIdx.y * fin.nsums + C + c] = t1;
  }
  finalize_last_block<32>(out, C, fin, gridDim.y, blockIdx.x, 32);
}

// float4 variant (C % 4 == 0, 16-byte aligned rows): threadIdx.x -> one channel QUAD inside a 128-channel slab, two rows in
// flight per iteration. Same MODE semantics as colreduce_kernel.
template <int MODE>
__global__ void __launch_bounds__(256)
colreduce4_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dy, int64_t M, int C, double* __restrict__ out,
                  const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                  const float* __restrict__ beta, int relu, const float* __restrict__ ymask, Finalize fin,
                  const float* __restrict__ se_gate = nullptr, const float* __restrict__ se_dpool = nullptr, int hw = 1) {
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
  double d0[4] = {0.0, 0.0, 0.0, 0.0}, d1[4] = {0.0, 0.0, 0.0, 0.0};
  if (c < C) {
    float mu[4] = {0.f, 0.f, 0.f, 0.f}, is[4] = {0.f, 0.f, 0.f, 0.f}, ga[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
    if (MODE == 1) {
#pragma unroll
      for (int q = 0; q < 4; ++q) { mu[q] = mean[c + q]; is[q] = invstd[c + q]; ga[q] = gamma[c + q]; be[q] = beta[c + q]; }
    }
    int cnt = 0;
    const int64_t step = (int64_t)gridDim.y * 8;
    for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < M; r += 2 * step) {
      const bool two = r + step < M;
      const float4 v0 = *reinterpret_cast<const float4*>(x + r * ldx + c);
      const float4 v1 = two ? *reinterpret_cast<const float4*>(x + (r + step) * ldx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
      float4 m0 = make_float4(1.f, 1.f, 1.f, 1.f), m1 = m0;       // mask source (output of the fused add + ReLU), when given
      if (MODE == 1) {
        g0 = *reinterpret_cast<const float4*>(dy + r * C + c);
        if (two) g1 = *reinterpret_cast<const float4*>(dy + (r + step) * C + c);
        if (ymask) {
          m0 = *reinterpret_cast<const float4*>(ymask + r * C + c);
          if (two) m1 = *reinterpret_cast<const float4*>(ymask + (r + step) * C + c);
        }
      }
      const float xv[2][4] = {{v0.x, v0.y, v0.z, v0.w}, {v1.x, v1.y, v1.z, v1.w}};
      float gv[2][4] = {{g0.x, g0.y, g0.z, g0.w}, {g1.x, g1.y, g1.z, g1.w}};
      if (MODE == 1 && se_gate) {
        se_grad4(gv[0], se_gate, se_dpool, (int64_t)((int)r / hw) * C + c, 1.f / (float)hw);
        if (two) se_grad4(gv[1], se_gate, se_dpool, (int64_t)((int)(r + step) / hw) * C + c, 1.f / (float)hw);
      }
      const float mv[2][4] = {{m0.x, m0.y, m0.z, m0.w}, {m1.x, m1.y, m1.z, m1.w}};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (h == 1 && !two) break;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (MODE == 0) {
            a0[q] += xv[h][q]; a1[q] = fmaf(xv[h][q], xv[h][q], a1[q]);
          } else {
            const float xh = (xv[h][q] - mu[q]) * is[q];
            float g = gv[h][q];
            if (ymask) { if (!(mv[h][q] > 0.f)) g = 0.f; }
            else if (relu && !(fmaf(xh, ga[q], be[q]) > 0.f)) g = 0.f;
            a0[q] += g; a1[q] = fmaf(g, xh, a1[q]);
          }
        }
      }
      if (++cnt == 32) {
#pragma unroll
        for (int q = 0; q < 4; ++q) { d0[q] += a0[q]; d1[q] += a1[q]; a0[q] = a1[q] = 0.f; }
        cnt = 0;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) { d0[q] += a0[q]; d1[q] += a1[q]; }
  }
  __shared__ double sd[8][32][8];
#pragma unroll
  for (int q = 0; q < 4; ++q) { sd[threadIdx.y][threadIdx.x][q] = d0[q]; sd[threadIdx.y][threadIdx.x][4 + q] = d1[q]; }
  __syncthreads();
  // 256 threads finish 32 quads x 8 values
  const int tq = threadIdx.x, tv = threadIdx.y;   // value index 0..7 handled by row-phase thread tv
  const int cc = (blockIdx.x * 32 + tq) * 4;
  if (cc < C) {
    double t = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += sd[j][tq][tv];
    if (tv < 4) fin.part[(int64_t)blockIdx.y * fin.nsums + cc + tv] = t;
    else if (fin.nsums > C) fin.part[(int64_t)blockIdx.y * fin.nsums + C + cc + tv - 4] = t;
  }
  finalize_last_block<128>(out, C, fin, gridDim.y, blockIdx.x, 128);
}

// Narrow matrices (C / 4 <= 128 channel quads: the 32-, 72- and 216-channel maps of the stem / stage 1 / stage 2, i.e. the LARGEST
// tensors of the trunks): the 32-quad slabs of colreduce4_kernel leave 44 % (C = 72) of the lanes idle. Here a block of 256 threads
// covers RPB = 256 / C4 whole rows per iteration — consecutive threads read consecutive 16-byte quads of consecutive rows, every lane
// busy (252 of 256 for C = 72) — each thread owns ONE quad column, and the RPB row phases meet in shared memory. Same MODE /
// Finalize semantics as colreduce4_kernel.
template <int MODE>
__global__ void __launch_bounds__(256)
colreduce_flat_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t M, int C, double* __restrict__ out,
                      const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                      const float* __restrict__ beta, int relu, const float* __restrict__ ymask, Finalize fin,
                      const float* __restrict__ se_gate = nullptr, const float* __restrict__ se_dpool = nullptr, int hw = 1) {
  const int C4 = C / 4, RPB = 256 / C4;
  const int t = threadIdx.x, q = t % C4, rr = t / C4;
  const bool active = rr < RPB;
  float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
  double d0[4] = {0.0, 0.0, 0.0, 0.0}, d1[4] = {0.0, 0.0, 0.0, 0.0};
  if (active) {
    float mu[4] = {0.f, 0.f, 0.f, 0.f}, is[4] = {0.f, 0.f, 0.f, 0.f}, ga[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
    if (MODE == 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) { mu[k] = mean[q * 4 + k]; is[k] = invstd[q * 4 + k]; ga[k] = gamma[q * 4 + k]; be[k] = beta[q * 4 + k]; }
    }
    int cnt = 0;
    const int64_t step = (int64_t)gridDim.x * RPB;
    for (int64_t r = (int64_t)blockIdx.x * RPB + rr; r < M; r += step) {
      const float4 v = *reinterpret_cast<const float4*>(x + r * C + q * 4);
      const float xv[4] = {v.x, v.y, v.z, v.w};
      if (MODE == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { a0[k] += xv[k]; a1[k] = fmaf(xv[k], xv[k], a1[k]); }
      } else {
        const float4 g4 = *reinterpret_cast<const float4*>(dy + r * C + q * 4);
        float gv[4] = {g4.x, g4.y, g4.z, g4.w};
        if (MODE == 1 && se_gate) se_grad4(gv, se_gate, se_dpool, (int64_t)((int)r / hw) * C + q * 4, 1.f / (float)hw);
        float mv[4] = {1.f, 1.f, 1.f, 1.f};
        if (ymask) {
          const float4 m4 = *reinterpret_cast<const float4*>(ymask + r * C + q * 4);
          mv[0] = m4.x; mv[1] = m4.y; mv[2] = m4.z; mv[3] = m4.w;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float xh = (xv[k] - mu[k]) * is[k];
          float g = gv[k];
          if (ymask) { if (!(mv[k] > 0.f)) g = 0.f; }
          else if (relu && !(fmaf(xh, ga[k], be[k]) > 0.f)) g = 0.f;
          a0[k] += g; a1[k] = fmaf(g, xh, a1[k]);
        }
      }
      if (++cnt == 64) {           // bound the fp32 partial length
#pragma unroll
        for (int k = 0; k < 4; ++k) { d0[k] += a0[k]; d1[k] += a1[k]; a0[k] = a1[k] = 0.f; }
        cnt = 0;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { d0[k] += a0[k]; d1[k] += a1[k]; }
  }
  __shared__ double sd[256][8];
#pragma unroll
  for (int k = 0; k < 4; ++k) { sd[t][k] = active ? d0[k] : 0.0; sd[t][4 + k] = active ? d1[k] : 0.0; }
  __syncthreads();
  // thread (q, value v): sum the RPB row phases of quad q; 8 values per quad
  for (int i = t; i < C4 * 8; i += 256) {
    const int qq = i >> 3, v = i & 7;
    double sum = 0.0;
    for (int j = 0; j < RPB; ++j) sum += sd[j * C4 + qq][v];
    if (v < 4) fin.part[(int64_t)blockIdx.x * fin.nsums + qq * 4 + v] = sum;
    else if (fin.nsums > C) fin.part[(int64_t)blockIdx.x * fin.nsums + C + qq * 4 + v - 4] = sum;
  }
  finalize_last_block<512>(out, C, fin, gridDim.x, 0, C);
}

// y = (x - mean) * invstd * gamma + beta (ReLU); 4 channels per thread (C % 4 == 0).
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t total4, int C4, const float* __restrict__ mean,
                const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                __nv_bfloat16* __restrict__ y16, const float* __restrict__ res) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 mu = *reinterpret_cast<const float4*>(mean + c);
    const float4 is = *reinterpret_cast<const float4*>(invstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    float4 o;
    o.x = fmaf((v.x - mu.x) * is.x, ga.x, be.x);
    o.y = fmaf((v.y - mu.y) * is.y, ga.y, be.y);
    o.z = fmaf((v.z - mu.z) * is.z, ga.z, be.z);
    o.w = fmaf((v.w - mu.w) * is.w, ga.w, be.w);
    if (res) {                                    // Bottleneck shortcut: act(bn(x) + residual) in one pass
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    reinterpret_cast<float4*>(y)[i] = o;
    if (y16) tfb_store_bf16x4(y16, i, o.x, o.y, o.z, o.w);
  }
}

// BatchNorm apply (+ReLU) that also accumulates the squeeze-excite pooling of its own output: pooled[n][c] += mean_hw(y[n][:, c]).
// Thread mapping of pool_hw_kernel (elementwise.cu): block (32 channel quads, 8 row phases), grid (quad slabs, n, HW splits);
// `pooled` was zeroed by the statistics kernel that runs right before this one (Finalize::zero_buf).
__global__ void __launch_bounds__(256)
bn_apply_pool_kernel(const float* __restrict__ x, float* __restrict__ y, int HW, int C, const float* __restrict__ mean,
                     const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                     float* __restrict__ pooled, float inv_hw, OrderedSum os) {
  __shared__ float4 sm[8][33];
  const int n = blockIdx.y, c = (blockIdx.x * 32 + threadIdx.x) * 4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const float4 mu = *reinterpret_cast<const float4*>(mean + c);
    const float4 is = *reinterpret_cast<const float4*>(invstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    const int64_t base = (int64_t)n * HW * C + c;
    for (int p = blockIdx.z * 8 + threadIdx.y; p < HW; p += gridDim.z * 8) {
      const float4 v = *reinterpret_cast<const float4*>(x + base + (int64_t)p * C);
      float4 o;
      o.x = fmaf((v.x - mu.x) * is.x, ga.x, be.x);
      o.y = fmaf((v.y - mu.y) * is.y, ga.y, be.y);
      o.z = fmaf((v.z - mu.z) * is.z, ga.z, be.z);
      o.w = fmaf((v.w - mu.w) * is.w, ga.w, be.w);
      if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      *reinterpret_cast<float4*>(y + base + (int64_t)p * C) = o;
      a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
    }
  }
  sm[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = sm[j][threadIdx.x]; t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w; }
    const int64_t o = (int64_t)n * C + c;
    ordered_store(os, blockIdx.z, o + 0, t.x * inv_hw); ordered_store(os, blockIdx.z, o + 1, t.y * inv_hw);
    ordered_store(os, blockIdx.z, o + 2, t.z * inv_hw); ordered_store(os, blockIdx.z, o + 3, t.w * inv_hw);
  }
  ordered_finish(os, pooled);
}

// ---- BatchNorm forward when the statistics were accumulated by the PRODUCER's epilogue (tfb_gemm_bf16_tc_stats, tfb_conv3x3_tc_strided):
// stats = [sum x | sum x^2] in fp64. Every block derives scale / shift for all channels into shared memory (C doubles of math per
// block: nothing next to the pass over x), block 0 also publishes save_mean / save_invstd and updates the running statistics.
constexpr int kBnStatsMaxC = 2048;   // RegNetY-3.2GF: 1512 at most

__device__ __forceinline__ void bn_params_from_stats(const double* __restrict__ stats, int C, int64_t M, float eps, float momentum,
                                                     const float* __restrict__ gamma, const float* __restrict__ beta, float* s_scale,
                                                     float* s_shift, bool publish, float* __restrict__ save_mean,
                                                     float* __restrict__ save_invstd, float* __restrict__ running_mean,
                                                     float* __restrict__ running_var, const double* __restrict__ count) {
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
  const double N = count ? *count : (double)M;      // count: the rows of every rank of a synchronized BatchNorm
  for (int c = tid; c < C; c += nthr) {
    double mean;
    const float invstd = bn_publish(c, stats[c], stats[C + c], N, eps, momentum, publish ? save_mean : nullptr, save_invstd,
                                    publish ? running_mean : nullptr, running_var, &mean);
    const float sc = gamma[c] * invstd;
    s_scale[c] = sc;
    s_shift[c] = fmaf(-(float)mean, sc, beta[c]);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256)
bn_apply_stats_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t total4, int C, int64_t M, const double* __restrict__ stats,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum, int relu,
                      float* __restrict__ save_mean, float* __restrict__ save_invstd, float* __restrict__ running_mean,
                      float* __restrict__ running_var, __nv_bfloat16* __restrict__ y16, const float* __restrict__ res,
                      const double* __restrict__ count) {
  __shared__ __align__(16) float s_par[2 * kBnStatsMaxC];
  float* s_scale = s_par;
  float* s_shift = s_par + kBnStatsMaxC;
  bn_params_from_stats(stats, C, M, eps, momentum, gamma, beta, s_scale, s_shift, blockIdx.x == 0, save_mean, save_invstd, running_mean, running_var,
                       count);
  const int C4 = C / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 sc = *reinterpret_cast<const float4*>(s_scale + c);
    const float4 sh = *reinterpret_cast<const float4*>(s_shift + c);
    float4 o = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
    if (res) {
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    reinterpret_cast<float4*>(y)[i] = o;
    if (y16) tfb_store_bf16x4(y16, i, o.x, o.y, o.z, o.w);
  }
}

// the pooling variant (thread mapping of bn_apply_pool_kernel); `pooled` must be zero on entry (the caller's per-step arena)
__global__ void __launch_bounds__(256)
bn_apply_pool_stats_kernel(const float* __restrict__ x, float* __restrict__ y, int HW, int C, int64_t M, const double* __restrict__ stats,
                           const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum, int relu,
                           float* __restrict__ save_mean, float* __restrict__ save_invstd, float* __restrict__ running_mean,
                           float* __restrict__ running_var, float* __restrict__ pooled, float inv_hw, OrderedSum os,
                           const double* __restrict__ count) {
  __shared__ __align__(16) float s_par[2 * kBnStatsMaxC];
  float* s_scale = s_par;
  float* s_shift = s_par + kBnStatsMaxC;
  bn_params_from_stats(stats, C, M, eps, momentum, gamma, beta, s_scale, s_shift, blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0,
                       save_mean, save_invstd, running_mean, running_var, count);
  __shared__ float4 sm[8][33];
  const int n = blockIdx.y, c = (blockIdx.x * 32 + threadIdx.x) * 4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const float4 sc = *reinterpret_cast<const float4*>(s_scale + c);
    const float4 sh = *reinterpret_cast<const float4*>(s_shift + c);
    const int64_t base = (int64_t)n * HW * C + c;
    for (int p = blockIdx.z * 8 + threadIdx.y; p < HW; p += gridDim.z * 8) {
      const float4 v = *reinterpret_cast<const float4*>(x + base + (int64_t)p * C);
      float4 o = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
      if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      *reinterpret_cast<float4*>(y + base + (int64_t)p * C) = o;
      a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
    }
  }
  sm[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float4 v = sm[j][threadIdx.x]; t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w; }
    const int64_t o = (int64_t)n * C + c;
    ordered_store(os, blockIdx.z, o + 0, t.x * inv_hw); ordered_store(os, blockIdx.z, o + 1, t.y * inv_hw);
    ordered_store(os, blockIdx.z, o + 2, t.z * inv_hw); ordered_store(os, blockIdx.z, o + 3, t.w * inv_hw);
  }
  ordered_finish(os, pooled);
}

// bn_apply_pool_stats_kernel for narrow maps (C / 4 <= 128): whole pixel rows of one sample per block iteration, every lane busy
// (same mapping as colreduce_flat_kernel); grid (splits over the pixels, n).
__global__ void __launch_bounds__(256)
bn_apply_pool_stats_flat_kernel(const float* __restrict__ x, float* __restrict__ y, int HW, int C, int64_t M, const double* __restrict__ stats,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum, int relu,
                                float* __restrict__ save_mean, float* __restrict__ save_invstd, float* __restrict__ running_mean,
                                float* __restrict__ running_var, float* __restrict__ pooled, float inv_hw, OrderedSum os,
                                const double* __restrict__ count) {
  __shared__ __align__(16) float s_par[2 * 512];
  float* s_scale = s_par;
  float* s_shift = s_par + 512;
  bn_params_from_stats(stats, C, M, eps, momentum, gamma, beta, s_scale, s_shift, blockIdx.x == 0 && blockIdx.y == 0, save_mean, save_invstd,
                       running_mean, running_var, count);
  const int C4 = C / 4, RPB = 256 / C4;
  const int t = threadIdx.x, q = t % C4, rr = t / C4, n = blockIdx.y;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rr < RPB) {
    const float4 sc = *reinterpret_cast<const float4*>(s_scale + q * 4);
    const float4 sh = *reinterpret_cast<const float4*>(s_shift + q * 4);
    const int64_t base = (int64_t)n * HW * C + q * 4;
    for (int p = blockIdx.x * RPB + rr; p < HW; p += gridDim.x * RPB) {
      const float4 v = *reinterpret_cast<const float4*>(x + base + (int64_t)p * C);
      float4 o = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
      if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      *reinterpret_cast<float4*>(y + base + (int64_t)p * C) = o;
      a.x += o.x; a.y += o.y; a.z += o.z; a.w += o.w;
    }
  }
  __shared__ float4 sm[256];
  sm[t] = rr < RPB ? a : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  if (t < C4) {
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < RPB; ++j) { const float4 v = sm[j * C4 + t]; s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w; }
    const int64_t o = (int64_t)n * C + t * 4;
    ordered_store(os, blockIdx.x, o + 0, s4.x * inv_hw); ordered_store(os, blockIdx.x, o + 1, s4.y * inv_hw);
    ordered_store(os, blockIdx.x, o + 2, s4.z * inv_hw); ordered_store(os, blockIdx.x, o + 3, s4.w * inv_hw);
  }
  ordered_finish(os, pooled);
}

// dx = gamma * invstd * (g - sum_g/M - xhat * sum_gx/M);  block 0 also writes dgamma = sum_gx, dbeta = sum_g.
// 4 channels per thread (C % 4 == 0, 16-byte aligned rows).
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int64_t M, int C,
                    const double* __restrict__ sums, const float* __restrict__ mean, const float* __restrict__ invstd,
                    const float* __restrict__ gamma, const float* __restrict__ beta, int relu, const float* __restrict__ dgamma,
                    const float* __restrict__ dbeta, __nv_bfloat16* __restrict__ dx16, const float* __restrict__ ymask,
                    float* __restrict__ gout, const float* __restrict__ se_gate, const float* __restrict__ se_dpool, int hw,
                    const double* __restrict__ count) {
  const int C4 = C / 4;
  const int64_t total4 = M * C4;
  const double invM = 1.0 / (count ? *count : (double)M);     // count: the rows of every rank of a synchronized BatchNorm
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const float4 xv = reinterpret_cast<const float4*>(x)[i];
    const float4 gv = reinterpret_cast<const float4*>(dy)[i];
    const float4 mu = *reinterpret_cast<const float4*>(mean + c);
    const float4 is = *reinterpret_cast<const float4*>(invstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    float gs[4] = {gv.x, gv.y, gv.z, gv.w};
    if (se_gate) se_grad4(gs, se_gate, se_dpool, (int64_t)((int)(i / C4) / hw) * C + c, 1.f / (float)hw);
    const float mus[4] = {mu.x, mu.y, mu.z, mu.w}, iss[4] = {is.x, is.y, is.z, is.w};
    const float gas[4] = {ga.x, ga.y, ga.z, ga.w}, bes[4] = {be.x, be.y, be.z, be.w};
    float4 mk = make_float4(1.f, 1.f, 1.f, 1.f);
    if (ymask) mk = reinterpret_cast<const float4*>(ymask)[i];
    const float ms[4] = {mk.x, mk.y, mk.z, mk.w};
    float o[4], gm[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float xh = (xs[q] - mus[q]) * iss[q];
      float g = gs[q];
      if (ymask) { if (!(ms[q] > 0.f)) g = 0.f; }
      else if (relu && !(fmaf(xh, gas[q], bes[q]) > 0.f)) g = 0.f;
      gm[q] = g;
      const float mg = (float)((double)dbeta[c + q] * invM), mgx = (float)((double)dgamma[c + q] * invM);
      o[q] = gas[q] * iss[q] * (g - mg - xh * mgx);
    }
    reinterpret_cast<float4*>(dx)[i] = make_float4(o[0], o[1], o[2], o[3]);
    if (dx16) tfb_store_bf16x4(dx16, i, o[0], o[1], o[2], o[3]);
    if (gout) reinterpret_cast<float4*>(gout)[i] = make_float4(gm[0], gm[1], gm[2], gm[3]);
  }
}

// ---------------- LayerNorm over the last dim of [R, C] ----------------
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int C, const float* __restrict__ gamma,
              const float* __restrict__ beta, float eps, float* __restrict__ save_mean, float* __restrict__ save_rstd,
              __nv_bfloat16* __restrict__ y16) {
  __shared__ float red[32];
  const int64_t r = blockIdx.x;
  const float* xr = x + r * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s += xr[c];
  const float mean = block_sum(s, red) / (float)C;
  float v = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = xr[c] - mean; v = fmaf(d, d, v); }
  const float var = block_sum(v, red) / (float)C;
  const float rstd = rsqrtf(var + eps);
  float* yr = y + r * C;
  __nv_bfloat16* hr = y16 ? y16 + r * C : nullptr;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float o = fmaf((xr[c] - mean) * rstd, gamma[c], beta[c]);
    yr[c] = o;
    if (hr) hr[c] = __float2bfloat16_rn(o);
  }
  if (threadIdx.x == 0) { save_mean[r] = mean; save_rstd[r] = rstd; }
}

// dx = rstd * (g*gamma - mean_c(g*gamma) - xhat * mean_c(g*gamma*xhat))
__global__ void __launch_bounds__(256)
ln_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int C,
                 const float* __restrict__ gamma, const float* __restrict__ save_mean, const float* __restrict__ save_rstd,
                 int accumulate) {
  __shared__ float red[32];
  const int64_t r = blockIdx.x;
  const float mean = save_mean[r], rstd = save_rstd[r];
  const float* xr = x + r * C;
  const float* gr = dy + r * C;
  float s1 = 0.f, s2 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float gg = gr[c] * gamma[c];
    s1 += gg;
    s2 = fmaf(gg, (xr[c] - mean) * rstd, s2);
  }
  const float m1 = block_sum(s1, red) / (float)C;
  const float m2 = block_sum(s2, red) / (float)C;
  float* dr = dx + r * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float xh = (xr[c] - mean) * rstd;
    const float v = rstd * (gr[c] * gamma[c] - m1 - xh * m2);
    dr[c] = accumulate ? dr[c] + v : v;
  }
}

// ---- GPT block glue fused (transfuser.py:546-547 followed by the next LayerNorm, transfuser.py:533-534 / 321):
//   xnew = res + dropout(x, p)          (the residual connection)          h = LayerNorm(xnew)   (+ bf16 copy for the next GEMM)
// one CTA per token row, three passes over the L1-resident row (as ln_fwd_kernel); dropout mask = tfb_dropout_scale(seed, flat index).
__global__ void __launch_bounds__(256)
add_dropout_ln_fwd_kernel(const float* __restrict__ res, const float* __restrict__ x, float* __restrict__ xnew, float* __restrict__ h, int C,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float p,
                          const uint64_t* __restrict__ seed_dev, uint64_t seed_off, float* __restrict__ save_mean, float* __restrict__ save_rstd,
                          __nv_bfloat16* __restrict__ h16) {
  __shared__ float red[32];
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t r = blockIdx.x;
  const float* rr = res + r * C;
  const float* xr = x + r * C;
  float* nr = xnew + r * C;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = __fadd_rn(rr[c], __fmul_rn(xr[c], tfb_dropout_scale(seed, (uint64_t)(r * C + c), p)));   // (no FMA: as tfb_dropout + add)
    nr[c] = v;
    s += v;
  }
  const float mean = block_sum(s, red) / (float)C;
  float q = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = nr[c] - mean; q = fmaf(d, d, q); }   // (own writes: same thread)
  const float rstd = rsqrtf(block_sum(q, red) / (float)C + eps);
  float* hr = h + r * C;
  __nv_bfloat16* h16r = h16 ? h16 + r * C : nullptr;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float o = fmaf((nr[c] - mean) * rstd, gamma[c], beta[c]);
    hr[c] = o;
    if (h16r) h16r[c] = __float2bfloat16_rn(o);
  }
  if (threadIdx.x == 0) { save_mean[r] = mean; save_rstd[r] = rstd; }
}

// backward: total = gx (gradient reaching xnew from its other consumer, may be null) + LayerNorm'(dh);  dres = total;  dx = total * mask
__global__ void __launch_bounds__(256)
add_dropout_ln_bwd_kernel(const float* __restrict__ xnew, const float* __restrict__ dh, const float* __restrict__ gx, float* __restrict__ dres,
                          float* __restrict__ dx, int C, const float* __restrict__ gamma, const float* __restrict__ save_mean,
                          const float* __restrict__ save_rstd, float p, const uint64_t* __restrict__ seed_dev, uint64_t seed_off) {
  __shared__ float red[32];
  const uint64_t seed = (seed_dev ? *seed_dev : 0ull) + seed_off;
  const int64_t r = blockIdx.x;
  const float mean = save_mean[r], rstd = save_rstd[r];
  const float* xr = xnew + r * C;
  const float* gr = dh + r * C;
  float s1 = 0.f, s2 = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float gg = gr[c] * gamma[c];
    s1 += gg;
    s2 = fmaf(gg, (xr[c] - mean) * rstd, s2);
  }
  const float m1 = block_sum(s1, red) / (float)C;
  const float m2 = block_sum(s2, red) / (float)C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float xh = (xr[c] - mean) * rstd;
    float t = rstd * (gr[c] * gamma[c] - m1 - xh * m2);
    if (gx) t += gx[r * C + c];
    dres[r * C + c] = t;
    dx[r * C + c] = t * tfb_dropout_scale(seed, (uint64_t)(r * C + c), p);
  }
}

// dgamma[c] = sum_r dy*xhat, dbeta[c] = sum_r dy  (column reduction; rows are few thousand). Partial sums meet in the self-cleaning
// fp64 workspace (sums = [sum dy | sum dy*xhat]) and the last block writes dbeta / dgamma: no memsets of the outputs.
__global__ void __launch_bounds__(256)
ln_bwd_param_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t R, int C, const float* __restrict__ save_mean,
                    const float* __restrict__ save_rstd, double* __restrict__ sums, Finalize fin) {
  __shared__ float sg[8][33], sb[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f, b = 0.f;
  if (c < C) {
    for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < R; r += (int64_t)gridDim.y * 8) {
      const float g = dy[r * C + c];
      a = fmaf(g, (x[r * C + c] - save_mean[r]) * save_rstd[r], a);
      b += g;
    }
  }
  sg[threadIdx.y][threadIdx.x] = a;
  sb[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float ta = 0.f, tb = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { ta += sg[j][threadIdx.x]; tb += sb[j][threadIdx.x]; }
    fin.part[(int64_t)blockIdx.y * fin.nsums + c] = (double)tb;
    fin.part[(int64_t)blockIdx.y * fin.nsums + C + c] = (double)ta;
  }
  finalize_last_block<32>(sums, C, fin, gridDim.y, blockIdx.x, 32);
}

// Backward prologue of a dense layer, one pass over dy [M, C]:  g = relu ? dy * (y > 0) : dy;  optional outputs: g in fp32, g in
// bf16 (operand of the tensor-core dgrad / wgrad GEMMs), and dbias[c] = sum_m g[m][c] (fp32 partials per thread, fp64 atomics).
__global__ void __launch_bounds__(256)
grad_prep_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ g32, __nv_bfloat16* __restrict__ g16,
                 double* __restrict__ sums, int64_t M, int C, Finalize fin) {
  __shared__ float sm[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f;
  if (c < C) {
    for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < M; r += (int64_t)gridDim.y * 8) {
      const int64_t i = r * C + c;
      float g = dy[i];
      if (y && !(y[i] > 0.f)) g = 0.f;
      if (g32) g32[i] = g;
      if (g16) g16[i] = __float2bfloat16_rn(g);
      a += g;
    }
  }
  if (sums) {
    sm[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
      float t = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
      fin.part[(int64_t)blockIdx.y * fin.nsums + c] = (double)t;
    }
    finalize_last_block<32>(sums, C, fin, gridDim.y, blockIdx.x, 32);
  }
}

template <int MODE>
int launch_colreduce(const float* x, int64_t ldx, const float* dy, int64_t M, int C, double* out, const float* mean, const float* invstd,
                     const float* gamma, const float* beta, int relu, const float* ymask, Finalize fin, cudaStream_t stream);

// ---- synchronized BatchNorm: the W ranks' slices [W][stride] (gathered in rank order) folded per value in rank order from +0, the
// rule of ordered_fold, so every rank derives the same bits whatever the collective's algorithm, and one rank gives +0 + s = s.
//   forward  (stride 2C + 1, [sum x | sum x^2 | count]): folded = the sums over all ranks (count included); save_mean / save_invstd and
//            the running statistics from them (bn_publish with N = the total count); `zero_buf` cleared (the SE pooling accumulator).
//   backward (stride 2C, [sum g | sum g*xhat]): gsum = the folded sums rounded to fp32, as tfb_bn_bwd's dbeta / dgamma are.
__global__ void __launch_bounds__(256)
bn_sync_fold_kernel(const double* __restrict__ g, int W, int C, int fwd, float eps, float momentum, float* __restrict__ save_mean,
                    float* __restrict__ save_invstd, float* __restrict__ running_mean, float* __restrict__ running_var,
                    double* __restrict__ folded, float* __restrict__ gsum, float* __restrict__ zero_buf, int zero_n) {
  const int stride = fwd ? 2 * C + 1 : 2 * C;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
  for (int c = tid; c < C; c += nthr) {
    double s0 = 0.0, s1 = 0.0, n = 0.0;
    for (int w = 0; w < W; ++w) {
      const double* sl = g + (int64_t)w * stride;
      s0 += sl[c];
      s1 += sl[C + c];
      if (fwd) n += sl[2 * C];
    }
    if (fwd) {
      folded[c] = s0;
      folded[C + c] = s1;
      if (c == 0) folded[2 * C] = n;
      bn_publish(c, s0, s1, n, eps, momentum, save_mean, save_invstd, running_mean, running_var);
    } else {
      gsum[c] = (float)s0;
      gsum[C + c] = (float)s1;
    }
  }
  for (int i = tid; i < zero_n; i += nthr) zero_buf[i] = 0.f;
}

// a rank's forward slice from statistics its producer's epilogue accumulated: [stats (2C) | M]
__global__ void __launch_bounds__(256) bn_sync_slice_copy_kernel(const double* __restrict__ stats, int C, int64_t M, double* __restrict__ slice) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= 2 * C; i += gridDim.x * blockDim.x) slice[i] = i < 2 * C ? stats[i] : (double)M;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
// Alignment of the operands the BatchNorm apply passes access as float4 (16 bytes) and of the bf16 sidecars they store four at a time
// (8 bytes); a null optional operand passes.
inline bool opt16(const void* p) { return !p || aligned16(p); }
inline bool opt8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

// fin.part for a reduction with nsplit row splits and fin.cnt for `slabs` channel slabs, in the stream's scratch.
int alloc_partials(Finalize& fin, int64_t nsplit, int slabs, cudaStream_t stream) {
  TfbScratch w;
  const int rc = tfb_scratch(w, (size_t)(2 * nsplit * fin.nsums), (size_t)slabs, stream);   // doubles = 2 floats each
  fin.part = reinterpret_cast<double*>(w.f);
  fin.cnt = w.cnt;
  return rc;
}

int colreduce_min_rows() {           // rows per thread below which a column reduction is not split further
  static int v = -1;
  if (v < 0) { const char* e = getenv("TFB_COLREDUCE_ROWS"); v = e ? atoi(e) : 16; if (v < 1) v = 1; }
  return v;
}

int colreduce_splits(int64_t M, int slabs) {
  int64_t want = (4LL * tfb_num_sms() + slabs - 1) / slabs;
  int64_t maxs = ceil_div64(M, 8 * colreduce_min_rows());
  if (want > maxs) want = maxs;
  if (want < 1) want = 1;
  if (want > 65535) want = 65535;
  return (int)want;
}

template <int MODE>
int launch_colreduce(const float* x, int64_t ldx, const float* dy, int64_t M, int C, double* out, const float* mean, const float* invstd,
                     const float* gamma, const float* beta, int relu, const float* ymask, Finalize fin, cudaStream_t stream) {
  const bool vec = C % 4 == 0 && ldx % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (!dy || (reinterpret_cast<uintptr_t>(dy) & 15) == 0) &&
                   (!ymask || (reinterpret_cast<uintptr_t>(ymask) & 15) == 0);
  dim3 block(32, 8);
  int rc;
  if (vec && C / 4 <= 128 && ldx == C && M >= 4096) {
    // narrow and tall: whole rows per block, every lane busy (see colreduce_flat_kernel)
    const int rpb = 256 / (C / 4);
    int64_t blocks = ceil_div64(M, (int64_t)rpb * 8);              // >= 8 rows per thread
    const int64_t cap = (int64_t)tfb_num_sms() * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if ((rc = alloc_partials(fin, blocks, 1, stream)) != TFB_OK) return rc;
    colreduce_flat_kernel<MODE><<<(int)blocks, 256, 0, stream>>>(x, dy, M, C, out, mean, invstd, gamma, beta, relu, ymask, fin);
  } else if (vec) {
    const int slabs = (C / 4 + 31) / 32;
    dim3 grid(slabs, colreduce_splits(M, slabs));
    if ((rc = alloc_partials(fin, grid.y, grid.x, stream)) != TFB_OK) return rc;
    colreduce4_kernel<MODE><<<grid, block, 0, stream>>>(x, ldx, dy, M, C, out, mean, invstd, gamma, beta, relu, ymask, fin);
  } else {
    const int slabs = (C + 31) / 32;
    dim3 grid(slabs, colreduce_splits(M, slabs));
    if ((rc = alloc_partials(fin, grid.y, grid.x, stream)) != TFB_OK) return rc;
    colreduce_kernel<MODE><<<grid, block, 0, stream>>>(x, ldx, dy, M, C, out, mean, invstd, gamma, beta, relu, ymask, fin);
  }
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

}  // namespace

static int bn_apply_launch(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, int relu, const float* save_mean,
                           const float* save_invstd, void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream);
static int bn_apply_stats_launch(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, float eps, float momentum,
                                 int relu, float* running_mean, float* running_var, float* save_mean, float* save_invstd, const double* stats,
                                 const double* count, void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream);

// sums_ws: (2*C + 1) doubles, ZERO on entry, left zero on exit (shared by all layers of a stream; no memset launches).
// y16_bf16 (optional): bf16 copy of y written in the same pass (operand of the next layer's tensor-core GEMM / conv).
// residual (optional, [M, C]): y = act(bn(x) + residual) — the Bottleneck's last BatchNorm + shortcut add + ReLU in one pass.
// pooled (optional, [pool_batch, C], M = pool_batch * HW): also the squeeze-excite pooling of the output, pooled[n][c] =
// mean over the HW pixels of sample n of y — cleared by the statistics kernel, accumulated by the apply kernel (no memset, no
// separate pooling pass); excludes y16_bf16 / residual.
// x, y, residual, gamma, beta, save_mean and save_invstd 16-byte aligned, y16_bf16 8-byte aligned (the normalise pass reads and
// writes four channels at a time); other operands are refused.
TFB_API int tfb_bn_fwd(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, float eps,
                       float momentum, int relu, float* running_mean, float* running_var, float* save_mean, float* save_invstd,
                       double* sums_ws, void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream) {
  TFB_REQUIRE(x && y && gamma && beta && save_mean && save_invstd && sums_ws && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(!pooled || (pool_batch > 0 && M % pool_batch == 0 && !y16_bf16 && !residual));
  TFB_REQUIRE(aligned16(x) && aligned16(y) && opt16(residual) && opt8(y16_bf16) && aligned16(gamma) && aligned16(beta) && aligned16(save_mean) &&
              aligned16(save_invstd));
  Finalize fin = {1, 2 * C, M, eps, momentum, save_mean, save_invstd, running_mean, running_var, pooled, pooled ? pool_batch * C : 0};
  const int rc = launch_colreduce<0>(x, C, nullptr, M, C, sums_ws, nullptr, nullptr, nullptr, nullptr, 0, nullptr, fin, stream);
  if (rc != TFB_OK) return rc;
  return bn_apply_launch(x, y, M, C, gamma, beta, relu, save_mean, save_invstd, y16_bf16, residual, pooled, pool_batch, stream);
}

// The normalise pass of tfb_bn_fwd from save_mean / save_invstd; `pooled` zero on entry.
static int bn_apply_launch(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, int relu, const float* save_mean,
                           const float* save_invstd, void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream) {
  if (pooled) {
    const int HW = (int)(M / pool_batch);
    int splits = (HW + 255) / 256;
    if (splits > 32) splits = 32;
    dim3 grid((C / 4 + 31) / 32, pool_batch, splits), block(32, 8);
    OrderedSum os;
    const int rc2 = ordered_alloc(os, splits, (int64_t)pool_batch * C, stream);
    if (rc2 != TFB_OK) return rc2;
    bn_apply_pool_kernel<<<grid, block, 0, stream>>>(x, y, HW, C, save_mean, save_invstd, gamma, beta, relu, pooled, 1.f / (float)HW, os);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  const int64_t total4 = M * C / 4;
  bn_apply_kernel<<<tfb_grid(total4, 256), 256, 0, stream>>>(x, y, total4, C / 4, save_mean, save_invstd, gamma, beta, relu,
                                                             (__nv_bfloat16*)y16_bf16, residual);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// Training-mode BatchNorm forward from statistics the producing conv / GEMM accumulated in its epilogue: stats = [sum x | sum x^2]
// (2*C doubles, read only). One launch: no reduction pass over x. pooled (optional): must be ZERO on entry (it is accumulated).
// Everything else as tfb_bn_fwd; x, y and residual 16-byte aligned, y16_bf16 8-byte aligned. C <= 2048.
TFB_API int tfb_bn_fwd_stats(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, float eps, float momentum,
                             int relu, float* running_mean, float* running_var, float* save_mean, float* save_invstd, const double* stats,
                             void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream) {
  TFB_REQUIRE(x && y && gamma && beta && save_mean && save_invstd && stats && M > 0 && C > 0 && C % 4 == 0 && C <= kBnStatsMaxC);
  TFB_REQUIRE(!pooled || (pool_batch > 0 && M % pool_batch == 0 && !y16_bf16 && !residual));
  TFB_REQUIRE(aligned16(x) && aligned16(y) && opt16(residual) && opt8(y16_bf16));
  return bn_apply_stats_launch(x, y, M, C, gamma, beta, eps, momentum, relu, running_mean, running_var, save_mean, save_invstd, stats, nullptr,
                               y16_bf16, residual, pooled, pool_batch, stream);
}

// The body of tfb_bn_fwd_stats; count (optional, device): the row count the statistics were summed over, in place of M.
static int bn_apply_stats_launch(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, float eps, float momentum,
                                 int relu, float* running_mean, float* running_var, float* save_mean, float* save_invstd, const double* stats,
                                 const double* count, void* y16_bf16, const float* residual, float* pooled, int pool_batch, cudaStream_t stream) {
  if (pooled) {
    const int HW = (int)(M / pool_batch);
    int splits = (HW + 255) / 256;
    if (splits > 32) splits = 32;
    if (C / 4 <= 128 && HW >= 1024) {
      const int rpb = 256 / (C / 4);
      int sp = (HW + rpb * 16 - 1) / (rpb * 16);
      const int cap = (4 * tfb_num_sms() + pool_batch - 1) / pool_batch;
      if (sp > cap) sp = cap;
      if (sp < 1) sp = 1;
      OrderedSum os;
      const int rc = ordered_alloc(os, sp, (int64_t)pool_batch * C, stream);
      if (rc != TFB_OK) return rc;
      bn_apply_pool_stats_flat_kernel<<<dim3(sp, pool_batch), 256, 0, stream>>>(x, y, HW, C, M, stats, gamma, beta, eps, momentum, relu, save_mean,
                                                                               save_invstd, running_mean, running_var, pooled, 1.f / (float)HW, os,
                                                                               count);
      TFB_CHECK_LAUNCH();
      return TFB_OK;
    }
    dim3 grid((C / 4 + 31) / 32, pool_batch, splits), block(32, 8);
    OrderedSum os;
    const int rc = ordered_alloc(os, splits, (int64_t)pool_batch * C, stream);
    if (rc != TFB_OK) return rc;
    bn_apply_pool_stats_kernel<<<grid, block, 0, stream>>>(x, y, HW, C, M, stats, gamma, beta, eps, momentum, relu, save_mean, save_invstd,
                                                              running_mean, running_var, pooled, 1.f / (float)HW, os, count);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  const int64_t total4 = M * C / 4;
  bn_apply_stats_kernel<<<tfb_grid(total4, 256, 4), 256, 0, stream>>>(x, y, total4, C, M, stats, gamma, beta, eps, momentum, relu, save_mean,
                                                                         save_invstd, running_mean, running_var,
                                                                         (__nv_bfloat16*)y16_bf16, residual, count);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// eval-mode BN: normalise with the running statistics (mean, 1/sqrt(var+eps) computed by the caller into save_*).
// x, y, residual, gamma, beta, mean and invstd 16-byte aligned, y16_bf16 8-byte aligned.
TFB_API int tfb_bn_apply(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, const float* mean,
                         const float* invstd, int relu, void* y16_bf16, const float* residual, cudaStream_t stream) {
  TFB_REQUIRE(x && y && gamma && beta && mean && invstd && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(aligned16(x) && aligned16(y) && opt16(residual) && opt8(y16_bf16) && aligned16(gamma) && aligned16(beta) && aligned16(mean) &&
              aligned16(invstd));
  const int64_t total4 = M * C / 4;
  bn_apply_kernel<<<tfb_grid(total4, 256), 256, 0, stream>>>(x, y, total4, C / 4, mean, invstd, gamma, beta, relu,
                                                             (__nv_bfloat16*)y16_bf16, residual);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// The column reduction of BatchNorm backward (sum g, sum g*xhat per channel) -> dbeta, dgamma; slice (optional): the same sums in fp64.
static int bn_bwd_reduce(const float* x, const float* dy, int64_t M, int C, const float* gamma, const float* beta, const float* save_mean,
                         const float* save_invstd, int relu, float* dgamma, float* dbeta, double* sums_ws, const float* ymask,
                         const float* se_gate, const float* se_dpool, int hw, double* slice, cudaStream_t stream) {
  Finalize fin = {2, 2 * C, M, 0.f, 0.f, dbeta, dgamma, nullptr, nullptr};
  fin.slice = slice;
  if (se_gate) {
    int rc;
    if (C / 4 <= 128 && M >= 4096) {            // as launch_colreduce picks
      const int rpb = 256 / (C / 4);
      int64_t blocks = ceil_div64(M, (int64_t)rpb * 8);
      const int64_t cap = (int64_t)tfb_num_sms() * 4;
      if (blocks > cap) blocks = cap;
      if (blocks < 1) blocks = 1;
      if ((rc = alloc_partials(fin, blocks, 1, stream)) != TFB_OK) return rc;
      colreduce_flat_kernel<1><<<(int)blocks, 256, 0, stream>>>(x, dy, M, C, sums_ws, save_mean, save_invstd, gamma, beta, relu, ymask, fin,
                                                               se_gate, se_dpool, hw);
    } else {
      const int slabs = (C / 4 + 31) / 32;
      dim3 grid(slabs, colreduce_splits(M, slabs)), block(32, 8);
      if ((rc = alloc_partials(fin, grid.y, grid.x, stream)) != TFB_OK) return rc;
      colreduce4_kernel<1><<<grid, block, 0, stream>>>(x, C, dy, M, C, sums_ws, save_mean, save_invstd, gamma, beta, relu, ymask, fin, se_gate,
                                                       se_dpool, hw);
    }
    TFB_CHECK_LAUNCH();
  } else {
    const int rc = launch_colreduce<1>(x, C, dy, M, C, sums_ws, save_mean, save_invstd, gamma, beta, relu, ymask, fin, stream);
    if (rc != TFB_OK) return rc;
  }
  return TFB_OK;
}

// Common body of tfb_bn_bwd / tfb_bn_bwd_se: column reduction (sum g, sum g*xhat per channel) + apply pass.
static int bn_bwd_impl(const float* x, const float* dy, float* dx, int64_t M, int C, const float* gamma, const float* beta,
                       const float* save_mean, const float* save_invstd, int relu, float* dgamma, float* dbeta, double* sums_ws,
                       void* dx16_bf16, const float* ymask, float* gmasked, const float* se_gate, const float* se_dpool, int hw,
                       cudaStream_t stream) {
  const int rc = bn_bwd_reduce(x, dy, M, C, gamma, beta, save_mean, save_invstd, relu, dgamma, dbeta, sums_ws, ymask, se_gate, se_dpool, hw,
                               nullptr, stream);
  if (rc != TFB_OK) return rc;
  bn_bwd_apply_kernel<<<tfb_grid(M * C / 4, 256), 256, 0, stream>>>(x, dy, dx, M, C, sums_ws, save_mean, save_invstd, gamma, beta, relu,
                                                                dgamma, dbeta, (__nv_bfloat16*)dx16_bf16, ymask, gmasked, se_gate, se_dpool, hw,
                                                                nullptr);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// sums_ws: as for tfb_bn_fwd. dx16_bf16 (optional): bf16 copy of dx written in the same pass (operand of the tensor-core dgrad /
// wgrad of the convolution in front of this BatchNorm).
// ymask / gmasked (optional, [M, C]): backward of y = relu(bn(x) + residual) (tfb_bn_fwd with a residual): the ReLU mask is
// (ymask > 0) with ymask = that y, the masked gradient g = dy * mask drives the BatchNorm backward (pass relu = 0) and is also
// written to gmasked — it is the gradient of the residual branch.
// Training-mode BatchNorm backward (timm BatchNormAct2d behind transfuser.py:136-184): dx, dgamma, dbeta (overwritten).
// x, dy, dx, ymask, gmasked, gamma, beta, save_mean and save_invstd 16-byte aligned, dx16_bf16 8-byte aligned.
TFB_API int tfb_bn_bwd(const float* x, const float* dy, float* dx, int64_t M, int C, const float* gamma, const float* beta,
                       const float* save_mean, const float* save_invstd, int relu, float* dgamma, float* dbeta, double* sums_ws,
                       void* dx16_bf16, const float* ymask, float* gmasked, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dx && gamma && beta && save_mean && save_invstd && dgamma && dbeta && sums_ws && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(!gmasked || ymask);
  TFB_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx) && opt16(ymask) && opt16(gmasked) && opt8(dx16_bf16) && aligned16(gamma) &&
              aligned16(beta) && aligned16(save_mean) && aligned16(save_invstd));
  return bn_bwd_impl(x, dy, dx, M, C, gamma, beta, save_mean, save_invstd, relu, dgamma, dbeta, sums_ws, dx16_bf16, ymask, gmasked,
                     nullptr, nullptr, 1, stream);
}

// tfb_bn_bwd for a BatchNorm whose output feeds a squeeze-excite gate (timm Bottleneck conv2.bn -> se inside the RegNetY trunks,
// reference team_code_transfuser/transfuser.py:136-184 via timm.create_model at :382-384): dy is the gradient of the SE
// OUTPUT [M = batch * hw, C]; the gradient of the BatchNorm output, dy * se_gate[n][c] + se_dpool[n][c] / hw, is formed inside the
// two BatchNorm passes (se_gate: the sigmoid gate [batch, C]; se_dpool: gradient of the pooled vector [batch, C], tfb_se_mlp_bwd),
// replacing tfb_se_bwd_apply (one launch, one write and one read of the map fewer). Alignment as for tfb_bn_bwd, and se_gate,
// se_dpool 16-byte aligned.
TFB_API int tfb_bn_bwd_se(const float* x, const float* dy, float* dx, int64_t M, int C, const float* gamma, const float* beta,
                          const float* save_mean, const float* save_invstd, int relu, float* dgamma, float* dbeta, double* sums_ws,
                          void* dx16_bf16, const float* se_gate, const float* se_dpool, int hw, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dx && gamma && beta && save_mean && save_invstd && dgamma && dbeta && sums_ws && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(se_gate && se_dpool && hw > 0 && M % hw == 0 && M < (int64_t)1 << 31);
  TFB_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx) && aligned16(se_gate) && aligned16(se_dpool) && opt8(dx16_bf16) && aligned16(gamma) &&
              aligned16(beta) && aligned16(save_mean) && aligned16(save_invstd));
  return bn_bwd_impl(x, dy, dx, M, C, gamma, beta, save_mean, save_invstd, relu, dgamma, dbeta, sums_ws, dx16_bf16, nullptr, nullptr,
                     se_gate, se_dpool, hw, stream);
}

// Synchronized BatchNorm (torch.nn.SyncBatchNorm semantics over the ranks of a process group), forward, step 1 of 2: this rank's
// slice = [sum x | sum x^2 | M] (2*C + 1 doubles). stats (optional): the sums the producing conv / GEMM epilogue accumulated (as for
// tfb_bn_fwd_stats), copied; else one statistics pass over x (sums_ws as for tfb_bn_fwd). The caller gathers the W ranks' slices.
TFB_API int tfb_bn_sync_slice(const float* x, int64_t M, int C, const double* stats, double* slice, double* sums_ws, cudaStream_t stream) {
  TFB_REQUIRE(slice && M > 0 && C > 0 && C % 4 == 0 && (stats || (x && sums_ws)));
  if (stats) {
    bn_sync_slice_copy_kernel<<<(2 * C + 256) / 256, 256, 0, stream>>>(stats, C, M, slice);
    TFB_CHECK_LAUNCH();
    return TFB_OK;
  }
  Finalize fin = {4, 2 * C, M, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr};
  fin.slice = slice;
  return launch_colreduce<0>(x, C, nullptr, M, C, sums_ws, nullptr, nullptr, nullptr, nullptr, 0, nullptr, fin, stream);
}

// Synchronized BatchNorm forward, step 2 of 2: gathered = the W ranks' slices [W][2*C + 1] in rank order. Folds them in rank order
// (folded: the sums and the total count N, 2*C + 1 doubles, kept for backward), then normalises with the global mean / biased variance;
// the running statistics take the unbiased variance over N. from_stats = 0: the normalise pass of tfb_bn_fwd, 1: that of
// tfb_bn_fwd_stats (with one rank, the same bits as that entry point). pooled (optional): cleared here, then accumulated.
// Everything else as tfb_bn_fwd (with from_stats = 1, the alignment of tfb_bn_fwd_stats).
TFB_API int tfb_bn_fwd_sync(const float* x, float* y, int64_t M, int C, const float* gamma, const float* beta, float eps, float momentum,
                            int relu, float* running_mean, float* running_var, float* save_mean, float* save_invstd, const double* gathered,
                            int world, double* folded, int from_stats, void* y16_bf16, const float* residual, float* pooled, int pool_batch,
                            cudaStream_t stream) {
  TFB_REQUIRE(x && y && gamma && beta && save_mean && save_invstd && gathered && folded && world > 0 && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(!pooled || (pool_batch > 0 && M % pool_batch == 0 && !y16_bf16 && !residual));
  TFB_REQUIRE(!from_stats || C <= kBnStatsMaxC);
  TFB_REQUIRE(aligned16(x) && aligned16(y) && opt16(residual) && opt8(y16_bf16) &&
              (from_stats || (aligned16(gamma) && aligned16(beta) && aligned16(save_mean) && aligned16(save_invstd))));
  bn_sync_fold_kernel<<<(C + 255) / 256, 256, 0, stream>>>(gathered, world, C, 1, eps, momentum, save_mean, save_invstd, running_mean,
                                                           running_var, folded, nullptr, pooled, pooled ? pool_batch * C : 0);
  TFB_CHECK_LAUNCH();
  if (from_stats)
    return bn_apply_stats_launch(x, y, M, C, gamma, beta, eps, momentum, relu, nullptr, nullptr, save_mean, save_invstd, folded, folded + 2 * C,
                                 y16_bf16, residual, pooled, pool_batch, stream);
  return bn_apply_launch(x, y, M, C, gamma, beta, relu, save_mean, save_invstd, y16_bf16, residual, pooled, pool_batch, stream);
}

// Synchronized BatchNorm backward, step 1 of 2: the reduction pass of tfb_bn_bwd (ymask) / tfb_bn_bwd_se (se_gate, se_dpool, hw),
// writing this rank's dgamma / dbeta (local, as torch.nn.SyncBatchNorm returns them) and its slice = [sum g | sum g*xhat] (2*C doubles).
// x, dy, ymask, se_gate and se_dpool 16-byte aligned.
TFB_API int tfb_bn_bwd_sync_reduce(const float* x, const float* dy, int64_t M, int C, const float* gamma, const float* beta, const float* save_mean,
                                   const float* save_invstd, int relu, float* dgamma, float* dbeta, double* sums_ws, const float* ymask,
                                   const float* se_gate, const float* se_dpool, int hw, double* slice, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && gamma && beta && save_mean && save_invstd && dgamma && dbeta && sums_ws && slice && M > 0 && C > 0 && C % 4 == 0);
  TFB_REQUIRE(!se_gate || (se_dpool && hw > 0 && M % hw == 0 && M < (int64_t)1 << 31 && !ymask && aligned16(se_gate) && aligned16(se_dpool)));
  TFB_REQUIRE(aligned16(x) && aligned16(dy) && opt16(ymask));
  return bn_bwd_reduce(x, dy, M, C, gamma, beta, save_mean, save_invstd, relu, dgamma, dbeta, sums_ws, ymask, se_gate, se_dpool, hw, slice,
                       stream);
}

// Synchronized BatchNorm backward, step 2 of 2: gathered = the W ranks' slices [W][2*C] in rank order, folded in rank order into
// gsum (2*C floats of scratch: [sum g | sum g*xhat] over every rank); count = the total row count N of the forward (folded[2*C] of
// tfb_bn_fwd_sync). dx = gamma * invstd * (g - sum_g/N - xhat * sum_gx/N); dx16_bf16 / ymask / gmasked / se_* as for tfb_bn_bwd(_se),
// alignment included.
TFB_API int tfb_bn_bwd_sync_apply(const float* x, const float* dy, float* dx, int64_t M, int C, const float* gamma, const float* beta,
                                  const float* save_mean, const float* save_invstd, int relu, const double* gathered, int world, const double* count,
                                  float* gsum, void* dx16_bf16, const float* ymask, float* gmasked, const float* se_gate, const float* se_dpool,
                                  int hw, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dx && gamma && beta && save_mean && save_invstd && gathered && count && gsum && world > 0 && M > 0 && C > 0 &&
              C % 4 == 0);
  TFB_REQUIRE((!gmasked || ymask) && (!se_gate || (se_dpool && hw > 0 && M % hw == 0 && M < (int64_t)1 << 31)));
  TFB_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dx) && opt16(ymask) && opt16(gmasked) && opt16(se_gate) && opt16(se_dpool) &&
              opt8(dx16_bf16) && aligned16(gamma) && aligned16(beta) && aligned16(save_mean) && aligned16(save_invstd));
  bn_sync_fold_kernel<<<(C + 255) / 256, 256, 0, stream>>>(gathered, world, C, 0, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, gsum,
                                                           nullptr, 0);
  TFB_CHECK_LAUNCH();
  bn_bwd_apply_kernel<<<tfb_grid(M * C / 4, 256), 256, 0, stream>>>(x, dy, dx, M, C, nullptr, save_mean, save_invstd, gamma, beta, relu,
                                                                gsum + C, gsum, (__nv_bfloat16*)dx16_bf16, ymask, gmasked, se_gate, se_dpool, hw,
                                                                count);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// out[c] = sum_r x[r][c]  (bias gradients of Linear / 1x1 conv layers)
// x is [M, C] with row stride ldx (elements).
TFB_API int tfb_colsum(const float* x, int64_t ldx, int64_t M, int C, float* out, double* sums_ws, cudaStream_t stream) {
  TFB_REQUIRE(x && out && sums_ws && M > 0 && C > 0 && ldx >= C);
  Finalize fin = {3, C, M, 0.f, 0.f, out, nullptr, nullptr, nullptr};
  return launch_colreduce<0>(x, ldx, nullptr, M, C, sums_ws, nullptr, nullptr, nullptr, nullptr, 0, nullptr, fin, stream);
}

// See grad_prep_kernel. Any of y / g32 / g16_bf16 / dbias may be null; sums_ws (C doubles) is needed when dbias is given.
TFB_API int tfb_grad_prep(const float* dy, const float* y, float* g32, void* g16_bf16, float* dbias, double* sums_ws, int64_t M, int C,
                          cudaStream_t stream) {
  TFB_REQUIRE(dy && M > 0 && C > 0 && (!dbias || sums_ws));
  const int slabs = (C + 31) / 32;
  dim3 grid(slabs, colreduce_splits(M, slabs)), block(32, 8);
  Finalize fin = {dbias ? 3 : 0, C, M, 0.f, 0.f, dbias, nullptr, nullptr, nullptr};
  if (dbias) {
    const int rc = alloc_partials(fin, grid.y, grid.x, stream);
    if (rc != TFB_OK) return rc;
  }
  grad_prep_kernel<<<grid, block, 0, stream>>>(dy, y, g32, (__nv_bfloat16*)g16_bf16, dbias ? sums_ws : nullptr, M, C, fin);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

TFB_API int tfb_layernorm_fwd(const float* x, float* y, int64_t R, int C, const float* gamma, const float* beta, float eps,
                              float* save_mean, float* save_rstd, void* y16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(x && y && gamma && beta && save_mean && save_rstd && R > 0 && C > 0);
  ln_fwd_kernel<<<(unsigned)R, 256, 0, stream>>>(x, y, C, gamma, beta, eps, save_mean, save_rstd, (__nv_bfloat16*)y16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// dx (+)= LN backward; dgamma/dbeta are overwritten. sums_ws: (2*C + 1) doubles, zero on entry, left zero on exit (as for tfb_bn_fwd).
TFB_API int tfb_layernorm_bwd(const float* x, const float* dy, float* dx, int64_t R, int C, const float* gamma,
                              const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta, int accumulate_dx,
                              double* sums_ws, cudaStream_t stream) {
  TFB_REQUIRE(x && dy && dx && gamma && save_mean && save_rstd && dgamma && dbeta && sums_ws && R > 0 && C > 0);
  ln_bwd_dx_kernel<<<(unsigned)R, 256, 0, stream>>>(x, dy, dx, C, gamma, save_mean, save_rstd, accumulate_dx);
  TFB_CHECK_LAUNCH();
  const int slabs = (C + 31) / 32;
  int splits = (int)ceil_div64(R, 8 * 8);
  if (splits > 64) splits = 64;
  if (splits < 1) splits = 1;
  dim3 grid(slabs, splits), block(32, 8);
  Finalize fin = {2, 2 * C, R, 0.f, 0.f, dbeta, dgamma, nullptr, nullptr};
  const int rc = alloc_partials(fin, grid.y, grid.x, stream);
  if (rc != TFB_OK) return rc;
  ln_bwd_param_kernel<<<grid, block, 0, stream>>>(x, dy, R, C, save_mean, save_rstd, sums_ws, fin);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// Replaces the GPT Block's residual connection and the LayerNorm that reads it (reference team_code_transfuser/transfuser.py:546-547, then
// :533-534 of the same / next Block, or ln_f at :321): xnew = res + dropout(x, p);  h = LayerNorm(xnew) (gamma, beta, eps);  h16 (optional):
// bf16 copy of h. One launch. [R, C] row-major.
TFB_API int tfb_add_dropout_ln_fwd(const float* res, const float* x, float* xnew, float* h, int64_t R, int C, const float* gamma, const float* beta,
                                   float eps, float p, const uint64_t* seed_dev, uint64_t seed_off, float* save_mean, float* save_rstd,
                                   void* h16_bf16, cudaStream_t stream) {
  TFB_REQUIRE(res && x && xnew && h && gamma && beta && save_mean && save_rstd && R > 0 && C > 0 && p >= 0.f && p < 1.f);
  add_dropout_ln_fwd_kernel<<<(unsigned)R, 256, 0, stream>>>(res, x, xnew, h, C, gamma, beta, eps, p, seed_dev, seed_off, save_mean, save_rstd,
                                                             (__nv_bfloat16*)h16_bf16);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// Backward of tfb_add_dropout_ln_fwd: dres, dx (both overwritten) from dh (gradient of h) and gx (gradient of xnew from its other consumer,
// may be null); dgamma / dbeta overwritten (sums_ws as for tfb_layernorm_bwd). Two launches (row kernel + parameter reduction).
TFB_API int tfb_add_dropout_ln_bwd(const float* xnew, const float* dh, const float* gx, float* dres, float* dx, int64_t R, int C, const float* gamma,
                                   const float* save_mean, const float* save_rstd, float p, const uint64_t* seed_dev, uint64_t seed_off,
                                   float* dgamma, float* dbeta, double* sums_ws, cudaStream_t stream) {
  TFB_REQUIRE(xnew && dh && dres && dx && gamma && save_mean && save_rstd && dgamma && dbeta && sums_ws && R > 0 && C > 0);
  add_dropout_ln_bwd_kernel<<<(unsigned)R, 256, 0, stream>>>(xnew, dh, gx, dres, dx, C, gamma, save_mean, save_rstd, p, seed_dev, seed_off);
  TFB_CHECK_LAUNCH();
  const int slabs = (C + 31) / 32;
  int splits = (int)ceil_div64(R, 8 * 8);
  if (splits > 64) splits = 64;
  if (splits < 1) splits = 1;
  dim3 grid(slabs, splits), block(32, 8);
  Finalize fin = {2, 2 * C, R, 0.f, 0.f, dbeta, dgamma, nullptr, nullptr};
  const int rc = alloc_partials(fin, grid.y, grid.x, stream);
  if (rc != TFB_OK) return rc;
  ln_bwd_param_kernel<<<grid, block, 0, stream>>>(xnew, dh, R, C, save_mean, save_rstd, sums_ws, fin);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
