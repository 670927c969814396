// Fused inference of one IDA up-sampling step of DLASeg (pose_dla_dcn.py IDAUp.forward):
//
//   out = conv_transpose2d(p, w, stride f, padding f / 2, groups C) + skip      (kernel 2f x 2f, f in {2, 4, 8})
//
// in one pass: the up-sampled map never reaches HBM.  The step is memory-bound; per output element the kernel reads
// skip once and writes out once (16-byte vectors), and reads p (1/f^2 of the output, each pixel reused by (2f)^2
// outputs) and the (2f)^2 weights of the channel through L1 / L2.
//
//   block   = (image, output row y, 32 channels, 64 output columns); 256 threads, 8 consecutive elements each
//   phase 1 the skip tile is loaded in skip's layout (NCHW: 8 columns of one channel a thread; channels_last: 8
//           channels of one pixel) into shared memory as fp32
//   phase 2 every thread computes 8 consecutive elements of out's layout: the 2 x 2 valid taps of the depthwise
//           transposed conv as one fp32 FMA chain in a fixed order, + skip from shared memory, one RN rounding to the
//           output dtype, one store
// Taps: output row y receives source rows q - 1 and q, q = (y + f/2) / f, at kernel rows ky + f and ky,
// ky = y + f/2 - q f; rows outside [0, Hp) are skipped (not multiplied by anything).  Columns likewise.  Staging the
// skip tile lets p, skip and out each take either layout with coalesced accesses.  No atomics and no workspace: the
// output is bit-identical run to run.
#include "common.cuh"

namespace cnb {
namespace {

constexpr int IU_TX = 64;                          // output columns of a block
constexpr int IU_TC = 32;                          // channels of a block
constexpr int IU_V = 8;                            // consecutive elements a thread
constexpr int IU_THREADS = IU_TX * IU_TC / IU_V;   // 256

struct IdaShape {
  int B, C, Hp, Wp, H, W;
  int p_cl, skip_cl, out_cl;
  int tiles_x, tiles_c;
};

__device__ __forceinline__ void load8(const float *src, float v[8]) {
  const float4 a = *reinterpret_cast<const float4 *>(src), b = *reinterpret_cast<const float4 *>(src + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void load8(const __nv_bfloat16 *src, float v[8]) {
  const uint4 a = *reinterpret_cast<const uint4 *>(src);
  const uint32_t u[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u[i]));
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void store8(float *dst, const float v[8]) {
  *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4 *>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void store8(__nv_bfloat16 *dst, const float v[8]) {
  uint32_t u[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    u[i] = *reinterpret_cast<const uint32_t *>(&h);
  }
  *reinterpret_cast<uint4 *>(dst) = make_uint4(u[0], u[1], u[2], u[3]);
}
__device__ __forceinline__ void store1(float *dst, float v) { *dst = v; }
__device__ __forceinline__ void store1(__nv_bfloat16 *dst, float v) { *dst = __float2bfloat16_rn(v); }

// The first of a thread's 8 elements within the block's [IU_TC][IU_TX] tile: along the columns of one channel
// (NCHW) or along the channels of one pixel (channels_last)
__device__ __forceinline__ void thread_origin(int t, int cl, int &c, int &x) {
  if (cl) {
    x = t >> 2;
    c = (t & 3) * IU_V;
  } else {
    c = t >> 3;
    x = (t & 7) * IU_V;
  }
}

template <typename T, int F>
__global__ void __launch_bounds__(IU_THREADS) k_ida_up_add(const T *__restrict__ p, const float *__restrict__ w,
                                                           const T *__restrict__ skip, T *__restrict__ out,
                                                           const IdaShape s) {
  __shared__ float tile[IU_TC][IU_TX + 1];
  long long blk = blockIdx.x;
  const int tx = (int)(blk % s.tiles_x);
  blk /= s.tiles_x;
  const int tc = (int)(blk % s.tiles_c);
  blk /= s.tiles_c;
  const int y = (int)(blk % s.H), b = (int)(blk / s.H);
  const int x0 = tx * IU_TX, c0 = tc * IU_TC;
  const long long HW = (long long)s.H * s.W;

  {   // phase 1: skip tile -> shared memory
    int c, x;
    thread_origin(threadIdx.x, s.skip_cl, c, x);
    const int gc = c0 + c, gx = x0 + x;
    float v[IU_V];
    if (!s.skip_cl) {
      if (gc < s.C && gx < s.W) {
        const T *src = skip + ((long long)b * s.C + gc) * HW + (long long)y * s.W + gx;
        if (s.W % IU_V == 0) {
          load8(src, v);
        } else {
#pragma unroll
          for (int j = 0; j < IU_V; ++j) v[j] = gx + j < s.W ? to_f32(src[j]) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < IU_V; ++j) tile[c][x + j] = v[j];
      }
    } else if (gc < s.C && gx < s.W) {
      const T *src = skip + (((long long)b * s.H + y) * s.W + gx) * s.C + gc;
      if (s.C % IU_V == 0) {
        load8(src, v);
      } else {
#pragma unroll
        for (int j = 0; j < IU_V; ++j) v[j] = gc + j < s.C ? to_f32(src[j]) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < IU_V; ++j) tile[c + j][x] = v[j];
    }
  }
  __syncthreads();

  // phase 2: up + skip in out's layout
  int c, x;
  thread_origin(threadIdx.x, s.out_cl, c, x);
  const int gc = c0 + c, gx = x0 + x;
  if (gc >= s.C || gx >= s.W) return;
  constexpr int K = 2 * F, H2 = F / 2;
  const int qy = (y + H2) / F, ky = y + H2 - qy * F;
  const bool row0 = qy >= 1, row1 = qy < s.Hp;
  // p of this image at (channel, iy, ix) is pb[channel * sc + iy * sy + ix * sx]; an image is within 32-bit indexing
  const T *pb = p + (long long)b * s.Hp * s.Wp * s.C;
  const int sx = s.p_cl ? s.C : 1, sy = s.p_cl ? s.Wp * s.C : s.Wp, sc = s.p_cl ? 1 : s.Hp * s.Wp;
  float o[IU_V];
#pragma unroll
  for (int j = 0; j < IU_V; ++j) {
    const int cc = s.out_cl ? gc + j : gc, xx = s.out_cl ? gx : gx + j;
    o[j] = 0.f;
    if (cc >= s.C || xx >= s.W) continue;
    const int qx = (xx + H2) / F, kx = xx + H2 - qx * F;
    const bool col0 = qx >= 1, col1 = qx < s.Wp;
    const float *wc = w + cc * K * K;
    const T *pc = pb + cc * sc + qy * sy + qx * sx;   // tap (q, q); only valid taps are read
    // fixed order: (q-1, q-1), (q-1, q), (q, q-1), (q, q) as (row, column)
    float acc = 0.f;
    if (row0 && col0) acc = fmaf(to_f32(__ldg(pc - sy - sx)), __ldg(wc + (ky + F) * K + kx + F), acc);
    if (row0 && col1) acc = fmaf(to_f32(__ldg(pc - sy)), __ldg(wc + (ky + F) * K + kx), acc);
    if (row1 && col0) acc = fmaf(to_f32(__ldg(pc - sx)), __ldg(wc + ky * K + kx + F), acc);
    if (row1 && col1) acc = fmaf(to_f32(__ldg(pc)), __ldg(wc + ky * K + kx), acc);
    o[j] = acc + tile[cc - c0][xx - x0];
  }
  if (!s.out_cl) {
    T *dst = out + ((long long)b * s.C + gc) * HW + (long long)y * s.W + gx;
    if (s.W % IU_V == 0) {
      store8(dst, o);
    } else {
#pragma unroll
      for (int j = 0; j < IU_V; ++j)
        if (gx + j < s.W) store1(dst + j, o[j]);
    }
  } else {
    T *dst = out + (((long long)b * s.H + y) * s.W + gx) * s.C + gc;
    if (s.C % IU_V == 0) {
      store8(dst, o);
    } else {
#pragma unroll
      for (int j = 0; j < IU_V; ++j)
        if (gc + j < s.C) store1(dst + j, o[j]);
    }
  }
}

template <typename T>
int launch_ida(const void *p, const float *w, int f, const void *skip, void *out, const IdaShape &s,
               cudaStream_t st) {
  const long long blocks = (long long)s.B * s.H * s.tiles_c * s.tiles_x;
  const T *pp = reinterpret_cast<const T *>(p), *sp = reinterpret_cast<const T *>(skip);
  T *op = reinterpret_cast<T *>(out);
  switch (f) {
    case 2: k_ida_up_add<T, 2><<<(unsigned)blocks, IU_THREADS, 0, st>>>(pp, w, sp, op, s); break;
    case 4: k_ida_up_add<T, 4><<<(unsigned)blocks, IU_THREADS, 0, st>>>(pp, w, sp, op, s); break;
    default: k_ida_up_add<T, 8><<<(unsigned)blocks, IU_THREADS, 0, st>>>(pp, w, sp, op, s); break;
  }
  CNB_CHECK_LAUNCH("cnb_ida_up_add");
  count_launch();
  return CNB_OK;
}

}  // namespace
}  // namespace cnb

using namespace cnb;

extern "C" int cnb_ida_up_add(const void *p, int dtype, int p_channels_last, const float *w, int f, const void *skip,
                              int skip_channels_last, void *out, int out_channels_last, int b, int c, int hp, int wp,
                              void *stream) {
  const char *fn = "cnb_ida_up_add";
  CNB_REQUIRE(p && w && skip && out, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE(dtype == CNB_DTYPE_F32 || dtype == CNB_DTYPE_BF16, CNB_EINVAL,
              "%s: dtype must be CNB_DTYPE_F32 or CNB_DTYPE_BF16 (got %d)", fn, dtype);
  CNB_REQUIRE((unsigned)p_channels_last <= 1u && (unsigned)skip_channels_last <= 1u &&
                  (unsigned)out_channels_last <= 1u,
              CNB_EINVAL, "%s: the channels_last flags must be 0 or 1", fn);
  CNB_REQUIRE(b > 0 && c > 0 && hp > 0 && wp > 0, CNB_EINVAL, "%s: bad shape (b %d, c %d, hp %d, wp %d)", fn, b, c,
              hp, wp);
  const size_t esz = dtype == CNB_DTYPE_F32 ? 4 : 2;
  CNB_REQUIRE(((reinterpret_cast<uintptr_t>(skip) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(p) & (esz - 1)) == 0 && (reinterpret_cast<uintptr_t>(w) & 3u) == 0,
              CNB_EINVAL, "%s: skip and out must be 16-byte aligned, p and w aligned to their element", fn);
  CNB_REQUIRE(f == 2 || f == 4 || f == 8, CNB_EUNSUPPORTED, "%s: up factor must be 2, 4 or 8 (got %d)", fn, f);
  CNB_REQUIRE((long long)b * c * hp * f * wp * f < (1ll << 31), CNB_EUNSUPPORTED,
              "%s: tensors beyond 32-bit indexing", fn);
  IdaShape s;
  s.B = b; s.C = c; s.Hp = hp; s.Wp = wp; s.H = hp * f; s.W = wp * f;
  s.p_cl = p_channels_last; s.skip_cl = skip_channels_last; s.out_cl = out_channels_last;
  s.tiles_x = (s.W + IU_TX - 1) / IU_TX;
  s.tiles_c = (c + IU_TC - 1) / IU_TC;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == CNB_DTYPE_F32 ? launch_ida<float>(p, w, f, skip, out, s, st)
                                : launch_ida<__nv_bfloat16>(p, w, f, skip, out, s, st);
}
