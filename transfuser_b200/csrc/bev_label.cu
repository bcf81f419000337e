// BEV semantic label of the reference's data augmentation on the GPU: load_crop_bev_npy (data.py:586-612) for a whole batch.
// The host ships the one uint8 plane of topdown/encoded_*.png that decode_pil_to_npy reads (data.py:844-856: channel 10 = bit 7,
// channel 11 = bit 6 of RGB plane 2) and the 2x3 matrix of skimage's rotate (pipeline.bev_rotation_matrix); one thread per output
// pixel restates, in double and without contraction to FMA, what skimage 0.16.2 computes for that pixel:
//   the 7-row shift         bev_shift[7:] = bev_array[:-7]          (a tap in rows 0..6 reads 0)
//   warp / _warp_fast       (c', r') = ((M0*C + M1*R) + M2, (M3*C + M4*R) + M5) at output (R, C) of the full H x W frame
//   bilinear_interpolation  floor / ceil taps, constant mode with cval 0, top = (1-dc)*TL + dc*TR, (1-dr)*top + dr*bottom
//   _clip_warp_output       clip to [min, max] of the input = [0, 1]: the shifted-in rows make the minimum 0, and an input
//                           without a set bit interpolates to 0 everywhere, so the clip is min(v, 1) in every case
//   crop + argmax           rows 90..249, columns 170..329; class = first maximum of (+0, a, a + b), a + b added in double
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kOut = 160;     // 32 m * 5 px/m (data.py:591-592)
constexpr int kRow0 = 90;     // start_y = 250 - 160
constexpr int kCol0 = 170;    // start_x = 250 - 160 / 2
constexpr int kShift = 7;     // "the lidar is + 1.3 in x" (data.py:596-599)
constexpr double kFar = 1073741824.0;   // |coordinate| beyond which every tap is outside any frame (keeps the long casts defined)

// The two channel bits of tap (r, c) of the shifted frame: bit 0 = channel 10, bit 1 = channel 11; 0 outside the frame.
__device__ __forceinline__ unsigned tap(const uint8_t* __restrict__ p, int H, int W, long r, long c) {
  if (r < kShift || r >= H || c < 0 || c >= W) return 0u;
  const unsigned v = p[(int64_t)(r - kShift) * W + c];
  return ((v >> 7) & 1u) | (((v >> 6) & 1u) << 1);
}

__device__ __forceinline__ double lerp2(double d, double a, double b) {
  return __dadd_rn(__dmul_rn(__dsub_rn(1.0, d), a), __dmul_rn(d, b));
}

__global__ void __launch_bounds__(256) bev_label_kernel(const uint8_t* __restrict__ plane, const double* __restrict__ matrix, int B, int H,
                                                        int W, int64_t* __restrict__ out) {
  const int64_t total = (int64_t)B * kOut * kOut;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % kOut);
    const int k = (int)((i / kOut) % kOut);
    const int b = (int)(i / (kOut * kOut));
    const double* m = matrix + 6 * (int64_t)b;
    const double R = (double)(kRow0 + k), C = (double)(kCol0 + j);
    const double c = __dadd_rn(__dadd_rn(__dmul_rn(m[0], C), __dmul_rn(m[1], R)), m[2]);
    const double r = __dadd_rn(__dadd_rn(__dmul_rn(m[3], C), __dmul_rn(m[4], R)), m[5]);
    double a = 0.0, s = 0.0;
    if (fabs(r) < kFar && fabs(c) < kFar) {
      const long minr = (long)floor(r), minc = (long)floor(c), maxr = (long)ceil(r), maxc = (long)ceil(c);
      const double dr = __dsub_rn(r, (double)minr), dc = __dsub_rn(c, (double)minc);
      const uint8_t* p = plane + (int64_t)b * H * W;
      const unsigned tl = tap(p, H, W, minr, minc), tr = tap(p, H, W, minr, maxc);
      const unsigned bl = tap(p, H, W, maxr, minc), br = tap(p, H, W, maxr, maxc);
      double ch[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const double top = lerp2(dc, (double)((tl >> q) & 1u), (double)((tr >> q) & 1u));
        const double bottom = lerp2(dc, (double)((bl >> q) & 1u), (double)((br >> q) & 1u));
        ch[q] = fmin(lerp2(dr, top, bottom), 1.0);
      }
      a = ch[0];
      s = __dadd_rn(ch[0], ch[1]);
    }
    // np.argmax over (+0, a, a + b): the first maximum wins, so a tie of a + b with a stays class 1
    int64_t cls = 0;
    double best = 0.0;
    if (a > best) { cls = 1; best = a; }
    if (s > best) cls = 2;
    out[i] = cls;
  }
}

}  // namespace

// plane: [B,H,W] uint8 (RGB plane 2 of topdown/encoded_*.png), matrix: [B,6] float64 (rows 0 and 1 of skimage's rotate matrix,
// output -> input coordinates; the third row is [0, 0, 1]) -> out [B,160,160] int64 classes {0, 1, 2}. H >= 250 and W >= 330:
// the 160 x 160 window at rows 90.., columns 170.. lies inside the rotated frame, which has the input's shape.
TFB_API int tfb_bev_label_prep(const uint8_t* plane, const double* matrix, int B, int H, int W, int64_t* out, cudaStream_t stream) {
  TFB_REQUIRE(plane && matrix && out);
  TFB_REQUIRE(B > 0 && B <= 65535 && H >= kRow0 + kOut && W >= kCol0 + kOut && H <= 32768 && W <= 32768);
  const int64_t total = (int64_t)B * kOut * kOut;
  bev_label_kernel<<<tfb_grid(total, 256), 256, 0, stream>>>(plane, matrix, B, H, W, out);
  TFB_CHECK_LAUNCH();
  return TFB_OK;
}
