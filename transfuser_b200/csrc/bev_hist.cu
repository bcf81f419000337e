// LiDAR point cloud -> 2-bin BEV histogram (2,256,256), bit-exact with the reference's numpy path
// (team_code_transfuser/data.py:446-470, `lidar_to_histogram_features`).
//
// Semantics restated (np.histogramdd with explicit edges = searchsorted(side='right') + last-edge rule):
//   x edges = -16 + k/8, y edges = -32 + k/8 (k = 0..256; all exactly representable),
//   bin k  iff  edge[k] <= v < edge[k+1];  v == edge[256] -> bin 255;  anything else is dropped;
//   channel 0 = points with z > -2.3 ("above"), channel 1 = z <= -2.3 ("below") (data.py:463-468);
//   out[c][row][col] = min(count_c[xbin = 255 - col][ybin = row], 5) / 5  (transpose + rot90(k=-1), data.py:467-469).
// HBM-bound integer scatter: 16 B (fp32) or 32 B (fp64) read per point, 512 KiB written per sample.
#include "common.cuh"

namespace {

constexpr int kGrid = 256;

template <typename T>
__device__ __forceinline__ int bev_bin(T v, T lo) {
  // Exact bin: estimate in double, then correct against the exact edges in the input precision.
  if (!(v >= lo) || !(v <= lo + (T)32)) return -1;  // also rejects NaN
  int k = (int)floor(((double)v - (double)lo) * 8.0);
  k = k < 0 ? 0 : (k > kGrid ? kGrid : k);
  while (k > 0 && v < lo + (T)k * (T)0.125) --k;
  while (k < kGrid && v >= lo + (T)(k + 1) * (T)0.125) ++k;
  if (k == kGrid) k = kGrid - 1;  // v == last edge -> last bin
  return k;
}

// points: [B][N][4] (x, y, z, intensity); n_valid[b] (optional) limits the points of sample b.
template <typename T>
__global__ void bev_scatter_kernel(const T* __restrict__ points, const int* __restrict__ n_valid, int n_max,
                                   unsigned int* __restrict__ counts) {
  const int b = blockIdx.y;
  const int n = n_valid ? min(n_valid[b], n_max) : n_max;
  const T* p = points + (size_t)b * n_max * 4;
  unsigned int* cnt = counts + (size_t)b * 2 * kGrid * kGrid;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    T x, y, z;
    if (sizeof(T) == 4) {
      float4 q = reinterpret_cast<const float4*>(p)[i];  // 16 B coalesced
      x = q.x; y = q.y; z = q.z;
    } else {
      double2 q0 = reinterpret_cast<const double2*>(p)[2 * i];
      double2 q1 = reinterpret_cast<const double2*>(p)[2 * i + 1];
      x = q0.x; y = q0.y; z = q1.x;
    }
    int xb = bev_bin<T>(x, (T)-16), yb = bev_bin<T>(y, (T)-32);
    if (xb < 0 || yb < 0) continue;
    int c;
    if (z > (T)-2.3) c = 0; else if (z <= (T)-2.3) c = 1; else continue;  // NaN z: in neither set
    atomicAdd(&cnt[(c * kGrid + xb) * kGrid + yb], 1u);
  }
}

// align() (data.py:411-443) fused into the scatter: every point is mapped through the sample's 4x4 float64 transform
// (Tr_vehicle_to_lidar @ inv(ego_1) @ ego_0 @ Tr_lidar_to_vehicle, pre-multiplied by the augmentation rotation — computed on
// the host exactly as the reference does) with the y sign flips of data.py:432-439, then binned in float64 like the
// reference's float64 result. The intermediate aligned cloud (32 B / point) never exists in HBM.
template <typename T>
__global__ void bev_scatter_aligned_kernel(const T* __restrict__ points, const double* __restrict__ transforms, const int* __restrict__ n_valid,
                                           int n_max, unsigned int* __restrict__ counts) {
  const int b = blockIdx.y;
  const int n = n_valid ? min(n_valid[b], n_max) : n_max;
  const T* p = points + (size_t)b * n_max * 4;
  unsigned int* cnt = counts + (size_t)b * 2 * kGrid * kGrid;
  __shared__ double m[12];
  if (threadIdx.x < 12) m[threadIdx.x] = transforms[(size_t)b * 16 + threadIdx.x];
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x, y, z;
    if (sizeof(T) == 4) {
      float4 q = reinterpret_cast<const float4*>(p)[i];
      x = q.x; y = q.y; z = q.z;
    } else {
      double2 q0 = reinterpret_cast<const double2*>(p)[2 * i];
      double2 q1 = reinterpret_cast<const double2*>(p)[2 * i + 1];
      x = q0.x; y = q0.y; z = q1.x;
    }
    y = -y;                                                    // data.py:434
    // row . (x, y, z, 1), accumulated left to right with FMAs (the order of a k=4 dgemm micro-kernel)
    const double ax = fma(m[3], 1.0, fma(m[2], z, fma(m[1], y, m[0] * x)));
    const double ay = -fma(m[7], 1.0, fma(m[6], z, fma(m[5], y, m[4] * x)));   // data.py:439
    const double az = fma(m[11], 1.0, fma(m[10], z, fma(m[9], y, m[8] * x)));
    int xb = bev_bin<double>(ax, -16.0), yb = bev_bin<double>(ay, -32.0);
    if (xb < 0 || yb < 0) continue;
    int c;
    if (az > -2.3) c = 0; else if (az <= -2.3) c = 1; else continue;
    atomicAdd(&cnt[(c * kGrid + xb) * kGrid + yb], 1u);
  }
}

__global__ void bev_finalize_kernel(const unsigned int* __restrict__ counts, float* __restrict__ out, int total) {
  // out[b][c][row][col] <- counts[b][c][xbin = 255 - col][ybin = row]; 32x32 tile transpose through smem
  __shared__ unsigned int tile[32][33];
  const int bc = blockIdx.z;
  const int row0 = blockIdx.y * 32, col0 = blockIdx.x * 32;
  const unsigned int* src = counts + (size_t)bc * kGrid * kGrid;
  float* dst = out + (size_t)bc * kGrid * kGrid;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int xbin = 255 - (col0 + j), ybin = row0 + threadIdx.x;
    tile[j][threadIdx.x] = src[xbin * kGrid + ybin];  // coalesced along ybin
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    unsigned int c = tile[threadIdx.x][j];
    c = c > 5u ? 5u : c;
    dst[(row0 + j) * kGrid + col0 + threadIdx.x] = (float)((double)c / 5.0);  // coalesced along col
  }
}

}  // namespace

// See include/tfb200.h
TFB_API int tfb_bev_histogram(const void* points, int is_f64, const int* n_valid, int batch, int n_max,
                              unsigned int* counts_ws, float* out, cudaStream_t stream) {
  TFB_REQUIRE(points && counts_ws && out && batch >= 0 && n_max >= 0);
  if (batch == 0) return TFB_OK;
  size_t cbytes = (size_t)batch * 2 * kGrid * kGrid * sizeof(unsigned int);
  if (cudaMemsetAsync(counts_ws, 0, cbytes, stream) != cudaSuccess) return TFB_ERR_DRIVER;
  if (n_max > 0) {
    int threads = 256;
    int bx = (n_max + threads - 1) / threads;
    if (bx > 160) bx = 160;
    dim3 grid(bx, batch);
    if (is_f64) bev_scatter_kernel<double><<<grid, threads, 0, stream>>>((const double*)points, n_valid, n_max, counts_ws);
    else        bev_scatter_kernel<float><<<grid, threads, 0, stream>>>((const float*)points, n_valid, n_max, counts_ws);
    TFB_CHECK_LAUNCH();
  }
  dim3 fgrid(kGrid / 32, kGrid / 32, batch * 2), fblock(32, 8);
  bev_finalize_kernel<<<fgrid, fblock, 0, stream>>>(counts_ws, out, batch);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}

// transforms: [batch][16] float64 row-major (one per sample). Otherwise as tfb_bev_histogram.
TFB_API int tfb_bev_histogram_aligned(const void* points, int is_f64, const double* transforms, const int* n_valid, int batch, int n_max,
                                      unsigned int* counts_ws, float* out, cudaStream_t stream) {
  TFB_REQUIRE(points && transforms && counts_ws && out && batch >= 0 && n_max >= 0 && batch <= 65535);
  if (batch == 0) return TFB_OK;
  size_t cbytes = (size_t)batch * 2 * kGrid * kGrid * sizeof(unsigned int);
  if (cudaMemsetAsync(counts_ws, 0, cbytes, stream) != cudaSuccess) return TFB_ERR_DRIVER;
  if (n_max > 0) {
    int threads = 256;
    int bx = (n_max + threads - 1) / threads;
    if (bx > 160) bx = 160;
    dim3 grid(bx, batch);
    if (is_f64) bev_scatter_aligned_kernel<double><<<grid, threads, 0, stream>>>((const double*)points, transforms, n_valid, n_max, counts_ws);
    else        bev_scatter_aligned_kernel<float><<<grid, threads, 0, stream>>>((const float*)points, transforms, n_valid, n_max, counts_ws);
    TFB_CHECK_LAUNCH();
  }
  dim3 fgrid(kGrid / 32, kGrid / 32, batch * 2), fblock(32, 8);
  bev_finalize_kernel<<<fgrid, fblock, 0, stream>>>(counts_ws, out, batch);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
