// ExtremeNet edge aggregation (what BASELINE.json calls "corner_pool t/l/b/r"):
// models/decode.py:17-77.  Along a row (left/right) or column (top/bottom)
//     ret[i] = heat[i] + ret[i-1] * [heat[i] >= heat[i-1]],   dir = ret - heat
//     _h_aggregate = w*left + w*right + heat,  _v_aggregate = w*top + w*bottom + heat.
// The fp32 additions are strictly sequential in the reference, so each row/column is
// scanned by ONE thread in that order (a tree/warp scan would re-associate the sums and
// break bit parity); parallelism comes from the B*C*H rows (or B*C*W columns).
//
// Tiled kernels (the normal path): one warp per tile, the tile lives in shared memory so HBM sees
// every byte once (read heat, write out) and all global traffic is full 128-byte lines.
//   rows   : tile = 32 consecutive rows, one TMA bulk copy per row into a row pitch of W+4 floats
//            (== 4 mod 32), so lane l walks row l with 16-byte shared accesses and every quarter-warp
//            covers the 32 banks exactly once.  The reverse pass parks ret-heat in a second buffer,
//            the forward pass combines in place, then the warp streams the buffer out with 16-byte stores.
//   columns: tile = H rows x 32 columns; lane l owns column l (coalesced 128-byte global rows,
//            conflict-free [row][lane] shared layout), same two passes; the tile arrives as one TMA
//            bulk copy per 128-byte row piece, all in flight at once.
// The older thread-per-line kernels below remain as the fallback for shapes the tiles do not cover
// (W % 4 != 0, unaligned bases, very long lines).
//
// Every kernel is templated on the map's element type T (fp32, fp16, bf16) and on SIG (the map holds logits):
// each element is turned into its fp32 score as it is loaded (score_f32: exact widening, then torch's sigmoid with
// SIG), so the scans run on exactly the fp32 values of the .float() upcast -- or of torch.sigmoid of it -- in the
// same strictly sequential order, and the result is the same fp32 map bit for bit.  A 16-bit row reaches shared
// memory by TMA only when it is a whole number of 16-byte pieces (W % 8 == 0).
#include "select.cuh"

namespace cnb {

constexpr int AG_R = 64;    // rows per CTA (one thread each)
constexpr int AG_CW = 128;  // columns per tile

// mode: 0 both directions weighted (+heat), 1 forward only (left/top), 2 reverse only (right/bottom)
__device__ __forceinline__ float combine(int mode, float w, float fwd, float rev, float h) {
  if (mode == 1) return fwd;
  if (mode == 2) return rev;
  return __fadd_rn(__fadd_rn(__fmul_rn(w, fwd), __fmul_rn(w, rev)), h);  // decode.py:72-73 order
}

// Four consecutive elements as fp32 scores: one 16-byte (fp32) or 8-byte (fp16 / bf16) load, then score_f32.
template <bool SIG>
__device__ __forceinline__ float4 sig4(float4 v) {
  if (SIG) {
    v.x = score_f32<true>(v.x); v.y = score_f32<true>(v.y); v.z = score_f32<true>(v.z); v.w = score_f32<true>(v.w);
  }
  return v;
}
template <bool SIG, typename T>
__device__ __forceinline__ float4 ldg4(const T *p) {   // global memory, read-only path
  return sig4<SIG>(widen4<T>(__ldg(reinterpret_cast<const typename Raw4<T>::type *>(p))));
}
template <bool SIG, typename T>
__device__ __forceinline__ float4 lds4(const T *p) {   // shared memory
  return sig4<SIG>(widen4<T>(ld_raw4<T>(p)));
}

// Rows: one thread walks one row with 16-byte accesses.  Neighbouring threads touch different 128-byte
// lines, but every thread consumes each of its lines completely over 8 consecutive steps, so the lines
// live in L1 for that long and DRAM still sees each byte once; 2048 threads per SM hide the latency.
template <typename T, bool SIG, bool VEC>
__global__ void __launch_bounds__(256) k_aggr_rows(const T *__restrict__ heat, float *__restrict__ out,
                                                   long long nrows, int W, float w, int mode) {
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= nrows) return;
  const T *hp = heat + row * W;
  float *op = out + row * W;
  float ret = 0.0f, hn = 0.0f;
  if (mode != 1) {  // right aggregate (decode.py:30-41): from the right edge inwards, parked in `out`
    if (VEC) {
      for (int c = W - 4; c >= 0; c -= 4) {
        const float4 h4 = ldg4<SIG>(hp + c);
        float4 r4;
        float h;
        h = h4.w; ret = (c + 3 == W - 1) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h); hn = h; r4.w = __fsub_rn(ret, h);
        h = h4.z; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; r4.z = __fsub_rn(ret, h);
        h = h4.y; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; r4.y = __fsub_rn(ret, h);
        h = h4.x; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; r4.x = __fsub_rn(ret, h);
        *reinterpret_cast<float4 *>(op + c) = r4;
      }
    } else {
      for (int c = W - 1; c >= 0; --c) {
        const float h = score_f32<SIG>(__ldg(hp + c));
        ret = (c == W - 1) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h);
        hn = h;
        op[c] = __fsub_rn(ret, h);
      }
    }
    if (mode == 2) return;
  }
  // left aggregate (decode.py:17-28) + combine
  if (VEC) {
    for (int c = 0; c < W; c += 4) {
      const float4 h4 = ldg4<SIG>(hp + c);
      float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (mode == 0) rv = *reinterpret_cast<const float4 *>(op + c);
      float4 o4;
      float h;
      h = h4.x; ret = (c == 0) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h); hn = h; o4.x = combine(mode, w, __fsub_rn(ret, h), rv.x, h);
      h = h4.y; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; o4.y = combine(mode, w, __fsub_rn(ret, h), rv.y, h);
      h = h4.z; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; o4.z = combine(mode, w, __fsub_rn(ret, h), rv.z, h);
      h = h4.w; ret = (h >= hn) ? __fadd_rn(h, ret) : h; hn = h; o4.w = combine(mode, w, __fsub_rn(ret, h), rv.w, h);
      *reinterpret_cast<float4 *>(op + c) = o4;
    }
  } else {
    for (int c = 0; c < W; ++c) {
      const float h = score_f32<SIG>(__ldg(hp + c));
      ret = (c == 0) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h);
      hn = h;
      const float rv = (mode == 0) ? op[c] : 0.0f;
      op[c] = combine(mode, w, __fsub_rn(ret, h), rv, h);
    }
  }
}

template <typename T, bool SIG>
__global__ void __launch_bounds__(128) k_aggr_cols(const T *__restrict__ heat, float *__restrict__ out,
                                                   long long planes, int H, int W, float w, int mode) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int xchunks = (W + 127) / 128;
  const long long plane = blockIdx.x / xchunks;
  const int x = (int)(blockIdx.x - plane * xchunks) * 128 + threadIdx.x;
  (void)gid;
  if (plane >= planes || x >= W) return;
  const T *hp = heat + plane * (long long)H * W + x;
  float *op = out + plane * (long long)H * W + x;
  float ret = 0.0f, hn = 0.0f;
  if (mode != 1) {  // bottom aggregate (decode.py:57-69)
#pragma unroll 4
    for (int y = H - 1; y >= 0; --y) {
      const float h = score_f32<SIG>(__ldg(hp + (long long)y * W));
      ret = (y == H - 1) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h);
      hn = h;
      op[(long long)y * W] = __fsub_rn(ret, h);
    }
    if (mode == 2) return;
  }
#pragma unroll 4
  for (int y = 0; y < H; ++y) {  // top aggregate (decode.py:43-55) + combine
    const float h = score_f32<SIG>(__ldg(hp + (long long)y * W));
    ret = (y == 0) ? h : ((h >= hn) ? __fadd_rn(h, ret) : h);
    hn = h;
    const float rev = (mode == 0) ? op[(long long)y * W] : 0.0f;
    op[(long long)y * W] = combine(mode, w, __fsub_rn(ret, h), rev, h);
  }
}

// ---------------------------------------------------------------- tiled kernels (one warp per tile)
constexpr int AGT_LINES = 32;          // lines per tile == lanes
constexpr int AGT_MAX_LEN = 512;       // longest line the tiles take (2 x 32 x 512 x 4 B = 128 KiB of smem)

// step of the segmented running sum (decode.py:21-27): first element starts the sum
__device__ __forceinline__ float aggr_step(bool first, float h, float hn, float ret) {
  return first ? h : ((h >= hn) ? __fadd_rn(h, ret) : h);
}

template <typename T, bool SIG>
__global__ void __launch_bounds__(32) k_aggr_rows_tile(const T *__restrict__ heat, float *__restrict__ out,
                                                       long long nrows, int W, float w, int mode) {
  extern __shared__ __align__(128) float agt_smem[];
  const int S = W + 4;                         // row pitch: == 4 (mod 32) floats -> the 16-byte accesses of a
                                               // quarter-warp (8 lanes, 8 rows) cover all 32 banks once
  const int SH = sizeof(T) == 4 ? S : W / 2 + 4;   // pitch of the loaded rows in floats (16-bit rows: 16 B pad)
  float *Hs = agt_smem;                        // the rows as loaded
  float *Rs = agt_smem + AGT_LINES * SH;       // reverse pass / result, fp32 pitch S
  __shared__ __align__(8) uint64_t bar;
  const int lane = threadIdx.x;
  const long long row0 = (long long)blockIdx.x * AGT_LINES;
  const int rows = (int)min((long long)AGT_LINES, nrows - row0);
  const bool mine = lane < rows;
  if (lane == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
    mbar_expect_tx(&bar, (uint32_t)rows * (uint32_t)W * (uint32_t)sizeof(T));
  }
  __syncwarp();
  if (mine) bulk_g2s(Hs + lane * SH, heat + (row0 + lane) * W, (uint32_t)W * (uint32_t)sizeof(T), &bar);   // one TMA row each
  mbar_wait(&bar, 0);
  const T *hrow = reinterpret_cast<const T *>(Hs + lane * SH);
  float *rrow = Rs + lane * S;
  float ret = 0.0f, hn = 0.0f;
  if (mine && mode != 1) {  // right aggregate (decode.py:30-41): from the right edge inwards
#pragma unroll 2
    for (int c = W - 4; c >= 0; c -= 4) {
      const float4 h4 = lds4<SIG>(hrow + c);
      float4 r4;
      float h;
      h = h4.w; ret = aggr_step(c + 3 == W - 1, h, hn, ret); hn = h; r4.w = __fsub_rn(ret, h);
      h = h4.z; ret = aggr_step(false, h, hn, ret); hn = h; r4.z = __fsub_rn(ret, h);
      h = h4.y; ret = aggr_step(false, h, hn, ret); hn = h; r4.y = __fsub_rn(ret, h);
      h = h4.x; ret = aggr_step(false, h, hn, ret); hn = h; r4.x = __fsub_rn(ret, h);
      *reinterpret_cast<float4 *>(rrow + c) = r4;
    }
  }
  if (mine && mode != 2) {  // left aggregate (decode.py:17-28) + combine, in place over the reverse result
#pragma unroll 2
    for (int c = 0; c < W; c += 4) {
      const float4 h4 = lds4<SIG>(hrow + c);
      float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (mode == 0) rv = *reinterpret_cast<const float4 *>(rrow + c);
      float4 o4;
      float h;
      h = h4.x; ret = aggr_step(c == 0, h, hn, ret); hn = h; o4.x = combine(mode, w, __fsub_rn(ret, h), rv.x, h);
      h = h4.y; ret = aggr_step(false, h, hn, ret); hn = h; o4.y = combine(mode, w, __fsub_rn(ret, h), rv.y, h);
      h = h4.z; ret = aggr_step(false, h, hn, ret); hn = h; o4.z = combine(mode, w, __fsub_rn(ret, h), rv.z, h);
      h = h4.w; ret = aggr_step(false, h, hn, ret); hn = h; o4.w = combine(mode, w, __fsub_rn(ret, h), rv.w, h);
      *reinterpret_cast<float4 *>(rrow + c) = o4;
    }
  }
  __syncwarp();
  // stream the tile out: consecutive lanes write consecutive 16-byte pieces of a row
  float4 *dst = reinterpret_cast<float4 *>(out + row0 * W);
  const int w4 = W >> 2, n4 = rows * w4;
#pragma unroll 4
  for (int i = lane; i < n4; i += 32) {
    const int r = i / w4, c4 = i - r * w4;
    dst[i] = *reinterpret_cast<const float4 *>(Rs + r * S + c4 * 4);
  }
}

template <typename T, bool SIG, bool TMA>
__global__ void __launch_bounds__(32) k_aggr_cols_tile(const T *__restrict__ heat, float *__restrict__ out,
                                                       long long planes, int H, int W, float w, int mode) {
  extern __shared__ __align__(128) float agt_smem[];
  T *Hs = reinterpret_cast<T *>(agt_smem);                         // [H][32] as loaded
  float *Rs = agt_smem + AGT_LINES * H * (int)sizeof(T) / 4;       // [H][32] fp32
  const int lane = threadIdx.x;
  const int xchunks = (W + AGT_LINES - 1) / AGT_LINES;
  const long long plane = blockIdx.x / xchunks;
  const int x = (int)(blockIdx.x - plane * xchunks) * AGT_LINES + lane;
  const bool mine = x < W;
  const T *hp = heat + plane * (long long)H * W + x;
  float *op = out + plane * (long long)H * W + x;
  if (TMA) {
    // bring the tile in: one TMA bulk copy per 128-byte row piece, all of them in flight at once
    __shared__ __align__(8) uint64_t bar;
    const int cw = min(AGT_LINES, W - (x - lane));   // columns in this chunk (a whole number of 16-byte pieces)
    if (lane == 0) {
      mbar_init(&bar, 1);
      mbar_fence_init();
      mbar_expect_tx(&bar, (uint32_t)H * (uint32_t)cw * (uint32_t)sizeof(T));
    }
    __syncwarp();
    for (int y = lane; y < H; y += 32) bulk_g2s(Hs + y * AGT_LINES, hp - lane + (long long)y * W, (uint32_t)cw * (uint32_t)sizeof(T), &bar);
    mbar_wait(&bar, 0);
  } else if (mine) {
#pragma unroll 16
    for (int y = 0; y < H; ++y) Hs[y * AGT_LINES + lane] = __ldg(hp + (long long)y * W);
  }
  float ret = 0.0f, hn = 0.0f;
  if (mine && mode != 1) {  // bottom aggregate (decode.py:57-69)
#pragma unroll 8
    for (int y = H - 1; y >= 0; --y) {
      const float h = score_f32<SIG>(Hs[y * AGT_LINES + lane]);
      ret = aggr_step(y == H - 1, h, hn, ret);
      hn = h;
      Rs[y * AGT_LINES + lane] = __fsub_rn(ret, h);
    }
  }
  if (mine) {
    if (mode == 2) {
#pragma unroll 16
      for (int y = 0; y < H; ++y) op[(long long)y * W] = Rs[y * AGT_LINES + lane];
    } else {  // top aggregate (decode.py:43-55) + combine, streamed straight out
#pragma unroll 8
      for (int y = 0; y < H; ++y) {
        const float h = score_f32<SIG>(Hs[y * AGT_LINES + lane]);
        ret = aggr_step(y == 0, h, hn, ret);
        hn = h;
        const float rev = (mode == 0) ? Rs[y * AGT_LINES + lane] : 0.0f;
        op[(long long)y * W] = combine(mode, w, __fsub_rn(ret, h), rev, h);
      }
    }
  }
}

// horizontal: 1 = _h_aggregate, 0 = _v_aggregate, 2 = left, 3 = right, 4 = top, 5 = bottom (raw ret - heat)
template <typename T, bool SIG>
static int launch_aggr(const T *heat, float *out, int n, int c, int h, int w, float weight, int horizontal,
                       cudaStream_t stream) {
  const long long planes = (long long)n * c;
  const bool rows = (horizontal == 1 || horizontal == 2 || horizontal == 3);
  const int mode = (horizontal <= 1) ? 0 : ((horizontal == 2 || horizontal == 4) ? 1 : 2);
  const bool pieces = ((long long)w * (long long)sizeof(T)) % 16 == 0;   // a row is whole 16-byte pieces
  if (rows && pieces && w <= AGT_MAX_LEN && ((((uintptr_t)heat | (uintptr_t)out) & 15u) == 0)) {
    const long long nrows = planes * h;
    const size_t smem = (size_t)AGT_LINES * (w * sizeof(T) + 16) + (size_t)AGT_LINES * (w + 4) * 4;
    static thread_local int cfg_dev = -1, cfg_bytes = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    if (cfg_dev != dev || cfg_bytes < (int)smem) {
      CNB_CUDA(cudaFuncSetAttribute(k_aggr_rows_tile<T, SIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * AGT_LINES * (AGT_MAX_LEN + 4) * 4));
      cfg_dev = dev; cfg_bytes = 2 * AGT_LINES * (AGT_MAX_LEN + 4) * 4;
    }
    k_aggr_rows_tile<T, SIG><<<(unsigned)((nrows + AGT_LINES - 1) / AGT_LINES), 32, smem, stream>>>(heat, out, nrows, w, weight, mode);
  } else if (!rows && h <= AGT_MAX_LEN) {
    const size_t smem = (size_t)AGT_LINES * h * sizeof(T) + (size_t)AGT_LINES * h * 4;
    static thread_local int cfg_dev = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (cfg_dev != dev) {
      CNB_CUDA(cudaFuncSetAttribute(k_aggr_cols_tile<T, SIG, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * AGT_LINES * AGT_MAX_LEN * 4));
      CNB_CUDA(cudaFuncSetAttribute(k_aggr_cols_tile<T, SIG, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * AGT_LINES * AGT_MAX_LEN * 4));
      cfg_dev = dev;
    }
    const long long blocks = planes * ((w + AGT_LINES - 1) / AGT_LINES);
    const bool tma = pieces && ((((uintptr_t)heat) & 15u) == 0);
    if (tma) k_aggr_cols_tile<T, SIG, true><<<(unsigned)blocks, 32, smem, stream>>>(heat, out, planes, h, w, weight, mode);
    else k_aggr_cols_tile<T, SIG, false><<<(unsigned)blocks, 32, smem, stream>>>(heat, out, planes, h, w, weight, mode);
  } else if (rows) {
    const long long nrows = planes * h;
    // four elements per load: 16 bytes of fp32 / 8 of fp16 / bf16, aligned to their size
    const bool vec = (w % 4 == 0) && ((((uintptr_t)heat & (4 * sizeof(T) - 1)) | ((uintptr_t)out & 15u)) == 0);
    if (vec)
      k_aggr_rows<T, SIG, true><<<(unsigned)((nrows + 255) / 256), 256, 0, stream>>>(heat, out, nrows, w, weight, mode);
    else
      k_aggr_rows<T, SIG, false><<<(unsigned)((nrows + 255) / 256), 256, 0, stream>>>(heat, out, nrows, w, weight, mode);
  } else {
    const long long blocks = planes * ((w + 127) / 128);
    k_aggr_cols<T, SIG><<<(unsigned)blocks, 128, 0, stream>>>(heat, out, planes, h, w, weight, mode);
  }
  CNB_CHECK_LAUNCH("cnb_edge_aggregate");
  count_launch();
  return CNB_OK;
}

int launch_edge_aggregate(const float *heat, float *out, int n, int c, int h, int w, float weight, int horizontal,
                          cudaStream_t stream) {
  return launch_aggr<float, false>(heat, out, n, c, h, w, weight, horizontal, stream);
}

// The same for a map of dtype code dt, holding logits when sigmoid (any dt; the caller checked dt)
int launch_edge_aggregate_ex(const void *heat, int dt, bool sigmoid, float *out, int n, int c, int h, int w,
                             float weight, int horizontal, cudaStream_t stream) {
  if (dt == CNB_DTYPE_BF16) {
    const __nv_bfloat16 *p = reinterpret_cast<const __nv_bfloat16 *>(heat);
    return sigmoid ? launch_aggr<__nv_bfloat16, true>(p, out, n, c, h, w, weight, horizontal, stream)
                   : launch_aggr<__nv_bfloat16, false>(p, out, n, c, h, w, weight, horizontal, stream);
  }
  if (dt == CNB_DTYPE_F16) {
    const __half *p = reinterpret_cast<const __half *>(heat);
    return sigmoid ? launch_aggr<__half, true>(p, out, n, c, h, w, weight, horizontal, stream)
                   : launch_aggr<__half, false>(p, out, n, c, h, w, weight, horizontal, stream);
  }
  const float *p = reinterpret_cast<const float *>(heat);
  return sigmoid ? launch_aggr<float, true>(p, out, n, c, h, w, weight, horizontal, stream)
                 : launch_aggr<float, false>(p, out, n, c, h, w, weight, horizontal, stream);
}

}  // namespace cnb

extern "C" int cnb_edge_aggregate(const float *heat, float *out, int n, int c, int h, int w, float aggr_weight,
                                  int horizontal, void *stream) {
  CNB_REQUIRE(heat && out, CNB_EINVAL, "cnb_edge_aggregate: null pointer");
  CNB_REQUIRE(heat != out, CNB_EINVAL, "cnb_edge_aggregate: in-place operation is not supported");
  CNB_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_edge_aggregate: non-positive dimension");
  CNB_REQUIRE(horizontal >= 0 && horizontal <= 5, CNB_EINVAL, "cnb_edge_aggregate: bad direction code %d", horizontal);
  return cnb::launch_edge_aggregate(heat, out, n, c, h, w, aggr_weight, horizontal, (cudaStream_t)stream);
}

extern "C" int cnb_edge_aggregate_ex(const void *heat, int dtype, int apply_sigmoid, float *out, int n, int c, int h,
                                     int w, float aggr_weight, int horizontal, void *stream) {
  CNB_REQUIRE(cnb::dtype_known(dtype), CNB_EINVAL, "cnb_edge_aggregate_ex: unknown dtype code %d", dtype);
  CNB_REQUIRE(heat && out, CNB_EINVAL, "cnb_edge_aggregate_ex: null pointer");
  CNB_REQUIRE(heat != (const void *)out, CNB_EINVAL, "cnb_edge_aggregate_ex: in-place operation is not supported");
  CNB_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, CNB_EINVAL, "cnb_edge_aggregate_ex: non-positive dimension");
  CNB_REQUIRE(horizontal >= 0 && horizontal <= 5, CNB_EINVAL, "cnb_edge_aggregate_ex: bad direction code %d",
              horizontal);
  return cnb::launch_edge_aggregate_ex(heat, dtype, apply_sigmoid != 0, out, n, c, h, w, aggr_weight, horizontal,
                                       (cudaStream_t)stream);
}
