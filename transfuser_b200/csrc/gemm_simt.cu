// fp32 CUDA-core GEMM (exact-fp32 path): C = alpha * op(A) * op(B) + beta * C (+ bias[n]) (ReLU optional),
// row-major, arbitrary leading dimensions, two-level strided batching (used for per-(sample, head) attention
// products and for every shape the tensor-core path does not take: tiny M, odd leading dimensions, parity mode).
// Replaces the cuBLAS calls behind nn.Linear / 1x1 nn.Conv2d / torch.matmul in the reference
// (team_code_transfuser/transfuser.py:510-527, 538-543; model.py:592-605).
// 128x64x16 tiles, 256 threads, 8x4 outputs per thread, register-prefetched double buffering, 8-byte vector loads when the
// operand's contiguous dimension allows it (head offsets of the packed q|k|v buffer are only 8-byte aligned).
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4, NT = 256;

// Loads a [ROWS x BK] (K-contiguous source, TR = false) or [BK x ROWS] (row-contiguous source, TR = true) slab of the
// operand into registers; element (r, k) of the logical tile lives at src[r * ld + k] (TR = false) or src[k * ld + r].
template <int ROWS, int VEC, bool TR>
struct TileLoader {
  static constexpr int kElems = ROWS * BK / NT;   // per thread
  static constexpr int kVecs = kElems / VEC;
  float v[kElems];
  __device__ __forceinline__ void load(const float* __restrict__ src, int64_t ld, int r0, int k0, int R, int K) {
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
      const int e = (threadIdx.x + i * NT) * VEC;   // linear element index inside the slab, contiguous dim fastest
      int r, k;
      if (!TR) { k = e % BK; r = e / BK; } else { r = e % ROWS; k = e / ROWS; }
      const int gr = r0 + r, gk = k0 + k;
      const float* p = TR ? src + (int64_t)gk * ld + gr : src + (int64_t)gr * ld + gk;
      const bool row_ok = gr < R, k_ok = gk < K;
      if (VEC == 2) {
        const bool full = TR ? (k_ok && gr + 1 < R) : (row_ok && gk + 1 < K);
        if (full) {
          const float2 t = *reinterpret_cast<const float2*>(p);
          v[i * 2] = t.x; v[i * 2 + 1] = t.y;
        } else {
          v[i * 2] = (row_ok && k_ok) ? p[0] : 0.f;
          const bool ok1 = TR ? (k_ok && gr + 1 < R) : (row_ok && gk + 1 < K);
          v[i * 2 + 1] = ok1 ? p[1] : 0.f;
        }
      } else {
        v[i] = (row_ok && k_ok) ? p[0] : 0.f;
      }
    }
  }
  // smem layout: s[k][r] with row stride LDS
  template <int LDS>
  __device__ __forceinline__ void store(float* s) const {
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
      const int e = (threadIdx.x + i * NT) * VEC;
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        int r, k;
        if (!TR) { k = (e + j) % BK; r = (e + j) / BK; } else { r = (e + j) % ROWS; k = (e + j) / ROWS; }
        s[k * LDS + r] = v[i * VEC + j];
      }
    }
  }
};

template <bool TA, bool TB, int VEC>
__global__ void __launch_bounds__(NT)
gemm_simt_kernel(int M, int N, int K, const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb,
                 float* __restrict__ C, int64_t ldc, const float* __restrict__ bias, int relu, float alpha, float beta,
                 int nbi, int64_t sAo, int64_t sAi, int64_t sBo, int64_t sBi, int64_t sCo, int64_t sCi) {
  constexpr int LDA = BM + 4, LDB = BN + 4;
  __shared__ __align__(16) float As[2][BK * LDA];
  __shared__ __align__(16) float Bs[2][BK * LDB];
  const int z = blockIdx.z, zo = z / nbi, zi = z % nbi;
  A += zo * sAo + zi * sAi;
  B += zo * sBo + zi * sBi;
  C += zo * sCo + zi * sCi;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // op(A)[m][k]: TA ? A[k*lda+m] : A[m*lda+k]  -> "rows" = m.   op(B)[k][n]: TB ? B[n*ldb+k] : B[k*ldb+n] -> "rows" = n.
  TileLoader<BM, VEC, TA> la;
  TileLoader<BN, VEC, !TB> lb;
  la.load(A, lda, m0, 0, M, K);
  lb.load(B, ldb, n0, 0, N, K);
  la.template store<LDA>(As[0]);
  lb.template store<LDB>(Bs[0]);
  __syncthreads();
  const int nk = (K + BK - 1) / BK;
  for (int t = 0; t < nk; ++t) {
    const int cur = t & 1;
    if (t + 1 < nk) {
      la.load(A, lda, m0, (t + 1) * BK, M, K);
      lb.load(B, ldb, n0, (t + 1) * BK, N, K);
    }
    const float* as = As[cur];
    const float* bs = Bs[cur];
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(as + kk * LDA + ty * TM);
      const float4 a1 = *reinterpret_cast<const float4*>(as + kk * LDA + ty * TM + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(bs + kk * LDB + tx * TN);
      const float a[TM] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[TN] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (t + 1 < nk) {
      la.template store<LDA>(As[cur ^ 1]);
      lb.template store<LDB>(Bs[cur ^ 1]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= N) continue;
      float v = alpha * acc[i][j];
      if (bias) v += bias[n];
      float* c = C + (int64_t)m * ldc + n;
      if (beta != 0.f) v += beta * (*c);
      if (relu) v = fmaxf(v, 0.f);
      *c = v;
    }
  }
}

template <int VEC>
void launch_all(int transA, int transB, dim3 grid, cudaStream_t stream, int M, int N, int K, const float* A, int64_t lda,
                const float* B, int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, float alpha, float beta, int nbi,
                int64_t sAo, int64_t sAi, int64_t sBo, int64_t sBi, int64_t sCo, int64_t sCi) {
#define LAUNCH(TA, TB) gemm_simt_kernel<TA, TB, VEC><<<grid, NT, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, \
                                                                               nbi, sAo, sAi, sBo, sBi, sCo, sCi)
  if (!transA && !transB) LAUNCH(false, false);
  else if (!transA && transB) LAUNCH(false, true);
  else if (transA && !transB) LAUNCH(true, false);
  else LAUNCH(true, true);
#undef LAUNCH
}

}  // namespace

TFB_API int tfb_gemm_f32_simt(int transA, int transB, int M, int N, int K, const float* A, int64_t lda, const float* B,
                              int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, float alpha, float beta,
                              int batch_outer, int batch_inner, int64_t sAo, int64_t sAi, int64_t sBo, int64_t sBi,
                              int64_t sCo, int64_t sCi, cudaStream_t stream) {
  TFB_REQUIRE(M >= 0 && N >= 0 && K >= 0 && batch_outer >= 1 && batch_inner >= 1);
  if (M == 0 || N == 0) return TFB_OK;
  TFB_REQUIRE(A && B && C);
  int64_t nz = (int64_t)batch_outer * batch_inner;
  TFB_REQUIRE(nz <= 65535);
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, (unsigned)nz);
  TFB_REQUIRE(grid.y <= 65535);
  // 8-byte vector loads need every operand address that is formed to be 8-byte aligned
  const bool even = ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) % 8 == 0) && lda % 2 == 0 && ldb % 2 == 0 &&
                    sAo % 2 == 0 && sAi % 2 == 0 && sBo % 2 == 0 && sBi % 2 == 0;
  if (even) launch_all<2>(transA, transB, grid, stream, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, batch_inner, sAo, sAi, sBo, sBi, sCo, sCi);
  else      launch_all<1>(transA, transB, grid, stream, M, N, K, A, lda, B, ldb, C, ldc, bias, relu, alpha, beta, batch_inner, sAo, sAi, sBo, sBi, sCo, sCi);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Small-M products (M <= 16 rows: SE bottleneck fc layers on pooled [B, C] vectors, the `join` MLP of the waypoint head):
//   C[m][n] = act( sum_k A[m][k] * op(B)[k][n] + bias[n] ),  op(B)[k][n] = transB ? B[n*ldb+k] : B[k*ldb+n]
// transB: one warp per output column (coalesced row of B, shuffle reduction); !transB: one thread per column, coalesced
// over n. A (<= 16 x K) is read through L1. act: 0 none, 1 ReLU, 2 sigmoid.
namespace {

// transB: a block of 8 warps covers 8 / KS output columns, KS warps sharing the K range of one column (KS = 1, 2, 4, 8 picked by the
// host so that a lane walks <= ~6 k steps: these products are latency-bound — a few hundred KB of weights read once — so the loads
// of a column are spread over more warps and unrolled rather than walked by one warp). Lanes read consecutive k (coalesced rows of
// A and B); the warp sums meet in shared memory.
template <int KS>
__global__ void __launch_bounds__(256)
small_m_tb_kernel(int M, int N, int K, const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb,
                  float* __restrict__ C, int64_t ldc, const float* __restrict__ bias, int act) {
  constexpr int COLS = 8 / KS;
  __shared__ float red[8][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = warp / KS, slice = warp % KS;
  const int n = blockIdx.x * COLS + col;
  float acc[16];
#pragma unroll
  for (int m = 0; m < 16; ++m) acc[m] = 0.f;
  if (n < N) {
    const float* b = B + (int64_t)n * ldb;
#pragma unroll 4
    for (int k = slice * 32 + lane; k < K; k += 32 * KS) {
      const float bv = b[k];
#pragma unroll
      for (int m = 0; m < 16; ++m)
        if (m < M) acc[m] = fmaf(A[(int64_t)m * lda + k], bv, acc[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    if (m < M) {
      const float v = warp_sum(acc[m]);
      if (lane == 0) red[warp][m] = v;
    }
  }
  __syncthreads();
  const int t = threadIdx.x;                 // thread (column c, row m) finishes one output
  if (t < COLS * 16) {
    const int c = t >> 4, m = t & 15, nn = blockIdx.x * COLS + c;
    if (m < M && nn < N) {
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < KS; ++j) v += red[c * KS + j][m];
      if (bias) v += bias[nn];
      if (act == 1) v = fmaxf(v, 0.f);
      else if (act == 2) v = 1.f / (1.f + expf(-v));
      C[(int64_t)m * ldc + nn] = v;
    }
  }
}

// !transB: block = 32 output columns x 8 K-slices; each thread accumulates its K slice for all rows, slices are reduced
// through shared memory (B reads are coalesced over n; the K loop is 8x shorter than one-thread-per-column).
__global__ void __launch_bounds__(256)
small_m_nt_kernel(int M, int N, int K, const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb,
                  float* __restrict__ C, int64_t ldc, const float* __restrict__ bias, int act) {
  __shared__ float red[8][16][33];
  const int tx = threadIdx.x & 31, ky = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + tx;
  float acc[16];
#pragma unroll
  for (int m = 0; m < 16; ++m) acc[m] = 0.f;
  if (n < N) {
#pragma unroll 4
    for (int k = ky; k < K; k += 8) {
      const float bv = B[(int64_t)k * ldb + n];
#pragma unroll
      for (int m = 0; m < 16; ++m)
        if (m < M) acc[m] = fmaf(A[(int64_t)m * lda + k], bv, acc[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < 16; ++m) red[ky][m][tx] = acc[m];
  __syncthreads();
  // 256 threads finish the 16 x 32 outputs: thread -> (m = ky*2 + {0,1}, n = tx)
#pragma unroll
  for (int mm = 0; mm < 2; ++mm) {
    const int m = ky * 2 + mm;
    if (m < M && n < N) {
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) v += red[j][m][tx];
      if (bias) v += bias[n];
      if (act == 1) v = fmaxf(v, 0.f);
      else if (act == 2) v = 1.f / (1.f + expf(-v));
      C[(int64_t)m * ldc + n] = v;
    }
  }
}

}  // namespace

TFB_API int tfb_gemm_small_m(int transB, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, float* C,
                             int64_t ldc, const float* bias, int act, cudaStream_t stream) {
  TFB_REQUIRE(A && B && C && M >= 1 && M <= 16 && N >= 1 && K >= 1);
  if (transB) {
    const int ks = K > 32 * 6 * 4 ? 8 : K > 32 * 6 * 2 ? 4 : K > 32 * 6 ? 2 : 1;      // <= 6 k steps per lane (K <= 1536)
    if (ks == 8)      small_m_tb_kernel<8><<<N, 256, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, act);
    else if (ks == 4) small_m_tb_kernel<4><<<(N + 1) / 2, 256, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, act);
    else if (ks == 2) small_m_tb_kernel<2><<<(N + 3) / 4, 256, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, act);
    else              small_m_tb_kernel<1><<<(N + 7) / 8, 256, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, act);
  }
  else        small_m_nt_kernel<<<(N + 31) / 32, 256, 0, stream>>>(M, N, K, A, lda, B, ldb, C, ldc, bias, act);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
