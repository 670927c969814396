// cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT 0) sampling of a uint8 HWC image, restated from OpenCV's
// fixed-point algorithm (imgwarp.cpp): coordinates on a 1/1024 grid from the INVERTED matrix `minv` (cvRound =
// round half to even), +16, >> 5 -> integer pixel + 5-bit phase; weights 32 * (32 - fy | fy) * (32 - fx | fx)
// (sum 32768); value = (sum w * p + 2^14) >> 15 with out-of-image taps reading the border value 0.
// Shared by the detector pre-process (post.cu) and the training batch builder (train_input.cu).
#pragma once
#include <cuda_runtime.h>

namespace cnb {

// The four taps of output pixel (x, y): top-left source pixel (sx, sy), which of the two rows / columns lie inside
// the H x W image, and the four 15-bit weights.
struct WarpTaps {
  int sx, sy, w0, w1, w2, w3;
  bool y0ok, y1ok, x0ok, x1ok;
};

__device__ __forceinline__ WarpTaps warp_taps(const double *__restrict__ minv, int x, int y, int H, int W) {
  const double m0 = minv[0], m1 = minv[1], m2 = minv[2], m3 = minv[3], m4 = minv[4], m5 = minv[5];
  const long long adelta = (long long)__double2ll_rn(__dmul_rn(__dmul_rn(m0, (double)x), 1024.0));
  const long long bdelta = (long long)__double2ll_rn(__dmul_rn(__dmul_rn(m3, (double)x), 1024.0));
  const long long X0 = (long long)__double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(m1, (double)y), m2), 1024.0)) + 16;
  const long long Y0 = (long long)__double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(m4, (double)y), m5), 1024.0)) + 16;
  auto sat_int = [](long long v) { return v > 2147483647ll ? 2147483647ll : (v < -2147483648ll ? -2147483648ll : v); };
  const int X = (int)((sat_int(X0 - 16) + 16 + sat_int(adelta)) >> 5);   // saturate_cast<int> of each rounded term
  const int Y = (int)((sat_int(Y0 - 16) + 16 + sat_int(bdelta)) >> 5);
  WarpTaps t;
  t.sx = X >> 5;
  t.sy = Y >> 5;
  t.sx = min(max(t.sx, -32768), 32767);
  t.sy = min(max(t.sy, -32768), 32767);
  const int fx = X & 31, fy = Y & 31;
  t.w0 = (32 - fy) * (32 - fx) * 32;
  t.w1 = (32 - fy) * fx * 32;
  t.w2 = fy * (32 - fx) * 32;
  t.w3 = fy * fx * 32;
  t.y0ok = t.sy >= 0 && t.sy < H;
  t.y1ok = t.sy + 1 >= 0 && t.sy + 1 < H;
  t.x0ok = t.sx >= 0 && t.sx < W;
  t.x1ok = t.sx + 1 >= 0 && t.sx + 1 < W;
  return t;
}

}  // namespace cnb
