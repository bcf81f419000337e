// LiDAR <-> camera correspondences of the geometric-fusion backbone on the GPU: lidar_bev_cam_correspondences (data.py:675-842)
// and correspondences_at_one_scale (data.py:632-673) for a whole batch, one CTA per sample. The host ships the raw sweep with y
// negated (dataset.CarlaRawDataset; the reference feeds the raw, unaligned, unrotated [..., :3], data.py:160, 256, 273), so y is
// negated back here (exact). Restated per point, in the precisions numpy 2 (NEP 50) evaluates the reference in:
//   x <- -x; keep |x| < 16, y < 32, y > 0; z <- z + float32(2.5 - 2.3)                     float32 (data.py:712-718)
//   centre view    u = (fx * x) / y + 176, v = (fy * z) / y + 80                         float64 (data.py:727-729)
//   left / right   (x', y', z') = R (x, y, z), each row ((r0*x + r1*y) + r2*z) without FMA, then the same pinhole with y' as depth;
//                  no depth test, so points behind those cameras project mirrored and are kept; y' == 0 gives inf / NaN, which
//                  the image tests drop (data.py:740-783)
//   image tests    0 < u < 352 and 0 < v < 160; left keeps u >= 176 and shifts by -176, centre shifts by +176, right keeps u < 176
//                  and shifts by (+176) + 352 (data.py:733-737, 755-760, 778-783)
//   candidate      bev = (int(float32(x + 16) * 8), 255 - int(y * 8)), cam = (int(u'), 159 - int(v)) (data.py:802-814), in the order
//                  left, centre, right, each in sweep order (data.py:786)
//   cells          bev_points[bx/32][by/32] collects cam/32 ([8,8,5,2]), cam_points[cx/32][cy/32] collects bev/32 ([22,5,5,2]);
//                  a cell's slots hold its first candidates in order, zeros after them (data.py:649-671)
// Two points the reference cannot index (it raises IndexError) are dropped: x = 16 - 2^-20, whose float32 x + 16 rounds to 32
// (bx = 256), and a right-view u within an ulp of 176, whose (u + 176) + 352 rounds to 704.
// A cell with more than 5 candidates stores 5 of them in place of random.sample(list, 5), by a rule that does not depend on the
// order threads run in: candidate (view, index) of list L (0 = bev_points, 1 = cam_points) gets the key
// (h, view, index), h = splitmix64(seed[b] ^ (L << 62 | view << 32 | index)), and the 5 smallest keys fill the slots in ascending
// order, a uniform ordered sample without replacement. Cells with at most 5 candidates use h = 0: the reference's order.
// Phases per CTA: (A) integer counts per cell in shared memory, (B) the cells' offsets into `work`, (C) every candidate written
// to its two cells' lists there (slot order within a list is free: the keys decide), (D) one warp per cell keeps a sorted top 5
// per lane, and lane 0 merges the 32 lanes' lists.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kBevCells = 64;                 // 8 x 8: the 256 x 256 BEV grid in 32-pixel cells
constexpr int kCamCells = 110;                // 22 x 5: three 352 x 160 images side by side (704 wide), in 32-pixel cells
constexpr int kCells = kBevCells + kCamCells;
constexpr int kSlots = 5;
constexpr int kIndexBits = 20;                // a list entry: index << 9 | view << 7 | the other list's cell

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Pinhole projection of data.py:728-729 (centre) / 750-751 / 773-774: (f * a) / depth + c.
__device__ __forceinline__ double pinhole(double f, double a, double depth, double c) { return __dadd_rn(__ddiv_rn(__dmul_rn(f, a), depth), c); }

// Row of R.dot(lidar.T) (data.py:746, 769), without FMA.
__device__ __forceinline__ double rot_row(const double* r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(r[0], x), __dmul_rn(r[1], y)), __dmul_rn(r[2], z));
}

// Candidate of point p in view v (0 left, 1 centre, 2 right): true with its BEV cell (bx/32 * 8 + by/32) and camera cell
// (cx/32 * 5 + cy/32). k: focal_x, focal_y, then the left and right rotation matrices row-major (3x3 each).
__device__ __forceinline__ bool candidate(const float* __restrict__ p, const double* __restrict__ k, float dz, int v, int* bcell, int* ccell) {
  const float x = -p[0], y = -p[1];            // x: data.py:712; y: undoes the negation the reader ships
  if (!(fabsf(x) < 16.f) || !(y < 32.f) || !(y > 0.f)) return false;
  const float z = __fadd_rn(p[2], dz);
  const int bx = (int)__fmul_rn(__fadd_rn(x, 16.f), 8.f);
  const int by = 255 - (int)__fmul_rn(y, 8.f);
  if (bx > 255) return false;
  const double X = (double)x, Y = (double)y, Z = (double)z;
  double u, w;
  if (v == 1) {
    u = pinhole(k[0], X, Y, 176.0);
    w = pinhole(k[1], Z, Y, 80.0);
  } else {
    const double* r = k + (v == 0 ? 2 : 11);
    const double rx = rot_row(r, X, Y, Z), ry = rot_row(r + 3, X, Y, Z), rz = rot_row(r + 6, X, Y, Z);
    u = pinhole(k[0], rx, ry, 176.0);
    w = pinhole(k[1], rz, ry, 80.0);
  }
  if (!(u > 0.0 && u < 352.0 && w > 0.0 && w < 160.0)) return false;
  if (v == 0) {
    if (!(u >= 176.0)) return false;
    u = __dsub_rn(u, 176.0);
  } else if (v == 1) {
    u = __dadd_rn(u, 176.0);
  } else {
    if (!(u < 176.0)) return false;
    u = __dadd_rn(__dadd_rn(u, 176.0), 352.0);
  }
  const int cx = (int)u, cy = 159 - (int)w;
  if (cx > 703) return false;
  *bcell = (bx >> 5) * 8 + (by >> 5);
  *ccell = (cx >> 5) * 5 + (cy >> 5);
  return true;
}

// (h, view << 20 | index) lexicographic
__device__ __forceinline__ bool key_less(uint64_t ha, unsigned va, uint64_t hb, unsigned vb) { return ha < hb || (ha == hb && va < vb); }
__device__ __forceinline__ unsigned entry_vi(unsigned e) { return ((e >> 7) & 3u) << kIndexBits | (e >> 9); }

__global__ void __launch_bounds__(kThreads) correspondences_kernel(const float* __restrict__ points, const int* __restrict__ n_valid,
                                                                   const uint64_t* __restrict__ seed, const double* __restrict__ k,
                                                                   float dz, int N, unsigned* __restrict__ work,
                                                                   int64_t* __restrict__ bev_points, int64_t* __restrict__ cam_points) {
  __shared__ int cnt[kCells], off[kCells], cur[kCells];
  __shared__ uint64_t top_h[kWarps][32 * kSlots];
  __shared__ unsigned top_e[kWarps][32 * kSlots];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = n_valid ? min(max(n_valid[b], 0), N) : N;
  const float* pts = points + (int64_t)b * N * 4;
  unsigned* list = work + (int64_t)b * 6 * N;
  for (int c = tid; c < kCells; c += kThreads) cnt[c] = 0;
  __syncthreads();
  // (A) counts
  for (int i = tid; i < n; i += kThreads)
    for (int v = 0; v < 3; ++v) {
      int bc, cc;
      if (candidate(pts + (int64_t)i * 4, k, dz, v, &bc, &cc)) {
        atomicAdd(&cnt[bc], 1);
        atomicAdd(&cnt[kBevCells + cc], 1);
      }
    }
  __syncthreads();
  // (B) offsets: the BEV cells' lists, then the camera cells'
  if (tid == 0) {
    int s = 0;
    for (int c = 0; c < kCells; ++c) { off[c] = s; cur[c] = s; s += cnt[c]; }
  }
  __syncthreads();
  // (C) list entries
  for (int i = tid; i < n; i += kThreads)
    for (int v = 0; v < 3; ++v) {
      int bc, cc;
      if (candidate(pts + (int64_t)i * 4, k, dz, v, &bc, &cc)) {
        const unsigned e = (unsigned)i << 9 | (unsigned)v << 7;
        list[atomicAdd(&cur[bc], 1)] = e | (unsigned)cc;
        list[atomicAdd(&cur[kBevCells + cc], 1)] = e | (unsigned)bc;
      }
    }
  __syncthreads();
  // (D) selection, one warp per cell
  const uint64_t s = seed[b];
  for (int c = warp; c < kCells; c += kWarps) {
    const int m = cnt[c];
    const uint64_t L = c < kBevCells ? 0ull : 1ull;
    uint64_t h5[kSlots] = {};
    unsigned e5[kSlots] = {};
    int have = 0;
    for (int j = lane; j < m; j += 32) {
      const unsigned e = list[off[c] + j];
      const unsigned vi = entry_vi(e);
      const uint64_t h = m > kSlots ? splitmix64(s ^ (L << 62 | (uint64_t)((e >> 7) & 3u) << 32 | (uint64_t)(e >> 9))) : 0ull;
      if (have == kSlots && !key_less(h, vi, h5[kSlots - 1], entry_vi(e5[kSlots - 1]))) continue;
      int q = have < kSlots ? have++ : kSlots - 1;
      while (q > 0 && key_less(h, vi, h5[q - 1], entry_vi(e5[q - 1]))) { h5[q] = h5[q - 1]; e5[q] = e5[q - 1]; --q; }
      h5[q] = h;
      e5[q] = e;
    }
    for (int q = 0; q < kSlots; ++q) {
      top_h[warp][lane * kSlots + q] = h5[q];
      top_e[warp][lane * kSlots + q] = q < have ? e5[q] : 0xffffffffu;
    }
    __syncwarp();
    if (lane == 0) {
      int head[32];
      for (int l = 0; l < 32; ++l) head[l] = 0;
      int64_t* out = c < kBevCells ? bev_points + ((int64_t)b * kBevCells + c) * kSlots * 2
                                   : cam_points + ((int64_t)b * kCamCells + (c - kBevCells)) * kSlots * 2;
      for (int r = 0; r < kSlots; ++r) {
        int best = -1;
        for (int l = 0; l < 32; ++l) {
          if (head[l] == kSlots) continue;
          const unsigned e = top_e[warp][l * kSlots + head[l]];
          if (e == 0xffffffffu) continue;
          if (best < 0 || key_less(top_h[warp][l * kSlots + head[l]], entry_vi(e), top_h[warp][best * kSlots + head[best]],
                                   entry_vi(top_e[warp][best * kSlots + head[best]])))
            best = l;
        }
        int64_t ox = 0, oy = 0;
        if (best >= 0) {
          const unsigned other = top_e[warp][best * kSlots + head[best]] & 127u;
          ++head[best];
          if (c < kBevCells) { ox = other / 5; oy = other % 5; }   // camera cell (cx/32, cy/32)
          else { ox = other >> 3; oy = other & 7; }                // BEV cell (bx/32, by/32)
        }
        out[r * 2] = ox;
        out[r * 2 + 1] = oy;
      }
    }
    __syncwarp();
  }
}

}  // namespace

// points [B,N,4] fp32 (x, y, z, intensity; y negated, as dataset.CarlaRawDataset ships the sweep), n_valid [B] int32 (optional:
// points of sample b beyond n_valid[b] are ignored), seed [B] uint64 (selection in cells with > 5 candidates), consts [20] fp64 on
// the device (focal_x, focal_y, the left and the right camera's rotation matrices row-major, pipeline.correspondence_constants),
// dz = float32(2.5 - 2.3), work [B, 6N] int32 scratch -> bev_points [B,8,8,5,2] and cam_points [B,22,5,5,2] int64, every
// element written.
TFB_API int tfb_lidar_cam_correspondences(const float* points, const int* n_valid, const uint64_t* seed, const double* consts, float dz, int B,
                                          int N, int* work, int64_t* bev_points, int64_t* cam_points, cudaStream_t stream) {
  TFB_REQUIRE(seed && consts && bev_points && cam_points && ((points && work) || N == 0));
  TFB_REQUIRE(B > 0 && B <= 65535 && N >= 0 && N < (1 << kIndexBits));
  correspondences_kernel<<<B, kThreads, 0, stream>>>(points, n_valid, seed, consts, dz, N, reinterpret_cast<unsigned*>(work), bev_points,
                                                     cam_points);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
