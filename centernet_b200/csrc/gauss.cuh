// draw_umich_gaussian's values (utils/image.py:118-141): gaussian2D of diameter 2r + 1 and sigma (2r + 1) / 6 in
// float64, rounded to fp32 as np.maximum(..., out=fp32 map) stores them.  Shared by the focal loss / target splat
// (focal.cu) and the ddd heat map of the training sampler (train_input.cu).
#pragma once
#include <cuda_runtime.h>

namespace cnb {

__device__ __forceinline__ float gauss_value(int dx, int dy, int r) {
  // gaussian2D (utils/image.py:118-124) in float64, cast to fp32 like np.maximum(..., out=fp32 map)
  // d2 in float64 (exact, as in numpy): with the centre outside the map |dx| may exceed the map size
  const double sigma = (double)(2 * r + 1) / 6.0;
  return (float)exp(-((double)dx * dx + (double)dy * dy) / (2.0 * sigma * sigma));
}

}  // namespace cnb
