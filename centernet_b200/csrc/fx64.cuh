// Two-limb fixed-point accumulation of float64 gradients (the float64 DCNv2 dX and the float64 PSROI grad_data).
//
// A value v of an accumulator whose elements are bounded by `bound` is held as v * 2^(e + L), e chosen so that
// bound * 2^e < 2^60, and split exactly into hi = floor(v * 2^e), a signed integer added in two's complement, and
// lo = floor(frac * 2^L) in [0, 2^L), added into its own unsigned limb.  Both are integer atomics
// (red.global.add.u64), and integer addition is associative: the sums do not depend on the order the adds land, so
// the gradient is bit-identical run to run for any grid.  With fewer than 2^lc contributions per element,
// L = min(40, 64 - lc) keeps the lo sum below 2^64.  The resolution is about bound * 2^-100, far below the float64
// rounding of the result, and the integers are converted to double once, at the end (fx_finish_launch).
#pragma once
#include "common.cuh"
#include <math.h>

namespace cnb {

struct FxParam {
  int e, L, bad;   // bad: the bound is not finite (inf / NaN among the inputs) -> the result is NaN
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long abs_bits64(double v) {
  return (unsigned long long)__double_as_longlong(v) & 0x7fffffffffffffffull;
}

// bits of a non-negative double (abs_bits64) at or above this are inf or NaN; below it, integer order is value order
constexpr unsigned long long kInfBits64 = 0x7ff0000000000000ull;

__device__ __forceinline__ FxParam fx_param(double bound, double count, bool finite) {
  FxParam f;
  f.bad = !finite || !(bound < INFINITY);
  int x = 0;
  if (bound > 0 && !f.bad) frexp(bound, &x);   // bound < 2^x
  f.e = 60 - x;
  int lc = 0;
  frexp(count > 1 ? count : 1.0, &lc);          // count < 2^lc
  f.L = min(40, 64 - lc);
  return f;
}

__device__ __forceinline__ void fx_add(unsigned long long *hi, unsigned long long *lo, long long i, double v,
                                       const FxParam &f) {
  const double s = scalbn(v, f.e);
  const double h = floor(s);
  const unsigned long long l = (unsigned long long)scalbn(s - h, f.L);
  const long long hv = (long long)h;
  if (hv) atomicAdd(hi + i, (unsigned long long)hv);
  if (l) atomicAdd(lo + i, l);
}
#endif

// bits[i] = max(bits[i], abs_bits64 of every element of image i), for the nimg images of per_img elements in v
// (an order-free maximum: integer max of the bits; NaN > inf > finite).  bits must start at 0 or a previous max.
void absmax_bits_launch(const double *v, long long per_img, int nimg, unsigned long long *bits, cudaStream_t st);

// out[i] += hi[i] + lo[i] * 2^-L, scaled back by 2^-e with the parameters of element i's image
// (prm[i / per_img]); NaN for an image whose bound is not finite.
int fx_finish_launch(const unsigned long long *hi, const unsigned long long *lo, const FxParam *prm,
                     long long per_img, long long n, double *out, cudaStream_t st);

}  // namespace cnb
