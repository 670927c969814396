// Fused bf16 inference of a CenterNet output head: Conv2d(Cin, Cmid, 3, padding=1) -> ReLU -> Conv2d(Cmid, C, 1), the
// `nn.Sequential` every DLASeg / PoseResNet head is built from (pose_dla_dcn.py:448-459, resnet_dcn.py:157-165,
// msra_resnet.py:135-143), in one persistent, warp-specialised wgmma kernel.  The Cmid-channel intermediate never
// leaves shared memory.
//
//   work item   = (image, 16 x 8 pixel tile [128 pixels = 2 x wgmma M]); every item computes all Cmid and all C
//   input       = bf16 channels-last [B][H][W][Cin] (the caller's tensor, or the one-pass copy k_head_nhwc /
//                 k_head_cl_to_bf16 makes of any other input)
//   TMA warp    streams, per GEMM 1 pass and 32-channel block, the 18 x 10 halo of the tile as four 8-channel slabs
//               (a 4-D tensor-map load each; the zero padding of the conv is the TMA's out-of-bounds fill), then the
//               nine W1 tiles of that block, and after the last pass the CMID / 32 W2 tiles (cp.async.bulk of
//               pre-tiled weights)
//   consumers   two warpgroups, 64 pixels (8 rows x 8 columns) each:
//               GEMM 1  D1[64, Cmid] += A . W1^T with wgmma m64nNk16 bf16 -> fp32, in passes of N <= 128 columns
//                       (at most 64 accumulators a thread).  A of tap (dy, dx) is the halo slab itself, read through a
//                       descriptor shifted by (dy * 10 + dx) * 16 bytes: the 8 pixels of a core-matrix row group are
//                       8 consecutive halo pixels, and the row groups are one halo row (160 bytes) apart -- the
//                       im2col is never built
//               epilogue 1  + b1 (fp32), ReLU (NaN kept, as torch.relu), one RN rounding to bf16, into this
//                       warpgroup's K-major intermediate tile in shared memory
//               GEMM 2  D2[64, N2] += inter . W2^T (wgmma m64nN2k16), + b2, stored as the input's dtype and layout
// Cmid is padded to CMID in {64, 128, 256} and C to N2 in {8, ..., 256}: padded weight rows are zero and the padded
// intermediate channels are forced to zero, so they add exact zeros (no Inf * 0) and are never stored.
// Every sum is in a fixed order and there are no atomics: the output is bit-identical run to run.
#include <cuda_bf16.h>

#include "halo.cuh"

namespace cnb {
namespace {

constexpr int HD_TW = 8, HD_TH = 16;                 // tile: 8 columns x 16 rows; warpgroup i owns rows 8i..8i+7
constexpr int HD_HX = HD_TW + 2, HD_HY = HD_TH + 2;  // halo
constexpr uint32_t HD_SLAB = HD_HX * HD_HY * 16;     // 2880: one 8-channel k-chunk of the halo, [y][x][8 ch]
constexpr uint32_t HD_SLAB_PITCH = 2944;             // slabs 128-byte aligned (TMA destination)
constexpr uint32_t HD_HALO_BYTES = 4 * HD_SLAB_PITCH;   // one 32-channel block
constexpr int HD_HSTAGES = 2;                        // halo ring
constexpr int HD_WSTAGES = 6;                        // weight-tile ring
constexpr int HD_WARP_TMA = 8;
constexpr int HD_THREADS = 9 * 32;

struct HeadShape {
  int B, Cin, H, W, Cmid, Cout;
  int tiles_x, tiles_y, n_items, ncb;   // ncb: 32-channel blocks of the input
  int out_bf16, out_cl;
};

// Padded GEMM widths of a head: CMID for Cmid, N2 for C
inline int head_cmid_pad(int cmid) { return cmid <= 64 ? 64 : cmid <= 128 ? 128 : 256; }
// GEMM 1 runs in CMID / NT1 passes over K of NT1 <= 128 columns each: a 64-register accumulator a thread
__host__ __device__ constexpr int head_nt1(int cmid_pad) { return cmid_pad > 128 ? 128 : cmid_pad; }
inline int head_n2_pad(int cout) {
  int n = 8;
  while (n < cout) n *= 2;
  return n;
}

__device__ __forceinline__ uint32_t pack2_bf16(float lo, float hi) {   // lo -> lower address
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&v);
}
// torch.relu: NaN stays NaN (fmaxf(NaN, 0) would give 0)
__device__ __forceinline__ float relu_nan(float v) { return v > 0.f ? v : (v != v ? v : 0.f); }

// W1 [Cmid][Cin][3][3] -> per (GEMM 1 pass, channel block cb, tap) one bf16 tile [NT1][32] (k = channel within the
// block) in the dense K-major layout of bf_tile_off, tile index (pass * Cin / 32 + cb) * 9 + tap; W2 [C][Cmid] -> per 32-channel block kc of the
// intermediate one tile [N2][32].  Rows and k beyond the real sizes are zero.  One block per tile.
__global__ void __launch_bounds__(256) k_head_prep(const float *__restrict__ w1, const float *__restrict__ w2, int cin,
                                                   int cmid, int cout, int CMIDp, int N2p,
                                                   unsigned char *__restrict__ w1t, unsigned char *__restrict__ w2t) {
  const int nt1 = head_nt1(CMIDp), per_pass = (cin / 32) * 9, n1 = (CMIDp / nt1) * per_pass;
  const int tile = blockIdx.x;
  if (tile < n1) {
    const int pass = tile / per_pass, cb = (tile % per_pass) / 9, tap = tile % 9;
    unsigned char *dst = w1t + (size_t)tile * nt1 * 64;
    for (int i = threadIdx.x; i < nt1 * 32; i += blockDim.x) {
      const int o = pass * nt1 + (i >> 5), k = i & 31;
      const float v = o < cmid ? w1[((size_t)o * cin + cb * 32 + k) * 9 + tap] : 0.f;
      *reinterpret_cast<__nv_bfloat16 *>(dst + bf_tile_off(i >> 5, k)) = __float2bfloat16_rn(v);
    }
  } else {

    const int kc = tile - n1;
    unsigned char *dst = w2t + (size_t)kc * N2p * 64;
    for (int i = threadIdx.x; i < N2p * 32; i += blockDim.x) {
      const int o = i >> 5, m = kc * 32 + (i & 31);
      const float v = (o < cout && m < cmid) ? w2[(size_t)o * cmid + m] : 0.f;
      *reinterpret_cast<__nv_bfloat16 *>(dst + bf_tile_off(o, i & 31)) = __float2bfloat16_rn(v);
    }
  }
}

// x [B][C][HW] (fp32 or bf16) -> bf16 [B][HW][C] (RN), C a multiple of 32.  grid (pixel blocks of 32, C / 32, B)
template <typename T>
__global__ void __launch_bounds__(256) k_head_nhwc(const T *__restrict__ x, __nv_bfloat16 *__restrict__ xt, int C,
                                                   long long HW) {
  __shared__ float tile[32][33];
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32, b = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c = ty; c < 32; c += 8)
    if (p0 + tx < HW) tile[c][tx] = to_f32(x[((long long)b * C + c0 + c) * HW + p0 + tx]);
  __syncthreads();
  for (int p = ty; p < 32; p += 8)
    if (p0 + p < HW) xt[((long long)b * HW + p0 + p) * C + c0 + tx] = __float2bfloat16_rn(tile[tx][p]);
}

// fp32 channels-last -> bf16 channels-last (RN), 8 values a thread
__global__ void __launch_bounds__(256) k_head_cl_to_bf16(const float4 *__restrict__ x, uint4 *__restrict__ xt,
                                                         long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = __ldg(x + 2 * i), b = __ldg(x + 2 * i + 1);
    xt[i] = make_uint4(pack2_bf16(a.x, a.y), pack2_bf16(a.z, a.w), pack2_bf16(b.x, b.y), pack2_bf16(b.z, b.w));
  }
}

template <int CMID, int N2>
struct HeadSmem {
  static constexpr int NT1 = head_nt1(CMID);
  static constexpr uint32_t W_BYTES = (NT1 > N2 ? NT1 : N2) * 64;     // one weight tile: [rows][32] bf16
  static constexpr uint32_t HALO = 0;
  static constexpr uint32_t RING = HALO + HD_HSTAGES * HD_HALO_BYTES;
  static constexpr uint32_t INTER = RING + HD_WSTAGES * W_BYTES;       // [2 warpgroups][64 px][CMID] bf16
  static constexpr uint32_t INTER_WG = 64 * CMID * 2;
  static constexpr uint32_t BYTES = INTER + 2 * INTER_WG + 128;        // + 128: alignment slack
};

template <int CMID, int N2>
__global__ void __launch_bounds__(HD_THREADS, 1)
k_head_fwd_bf16(const __grid_constant__ CUtensorMap xmap, const __nv_bfloat16 *__restrict__ w1t,
                const float *__restrict__ b1, const __nv_bfloat16 *__restrict__ w2t, const float *__restrict__ b2,
                void *__restrict__ out, const HeadShape s) {
  using L = HeadSmem<CMID, N2>;
  extern __shared__ unsigned char hd_smem_raw[];
  unsigned char *sm = hd_smem_raw + ((128u - (smem_u32(hd_smem_raw) & 127u)) & 127u);
  __shared__ __align__(8) uint64_t h_full[HD_HSTAGES], h_empty[HD_HSTAGES], w_full[HD_WSTAGES], w_empty[HD_WSTAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles = s.tiles_x * s.tiles_y;
  if (tid == 0) {
    for (int i = 0; i < HD_HSTAGES; ++i) {
      mbar_init(&h_full[i], 1);
      mbar_init(&h_empty[i], 2);
    }
    for (int i = 0; i < HD_WSTAGES; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], 2);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == HD_WARP_TMA) {
    // ============================================================ producer: halo slabs and weight tiles
    if (lane == 0) {
      int hs = 0, hph = 0, ws = 0, wph = 0;
      auto put_w = [&](const __nv_bfloat16 *src, uint32_t bytes) {
        mbar_wait(&w_empty[ws], (uint32_t)(wph ^ 1));
        mbar_expect_tx(&w_full[ws], bytes);
        bulk_g2s(sm + L::RING + (size_t)ws * L::W_BYTES, src, bytes, &w_full[ws]);
        if (++ws == HD_WSTAGES) { ws = 0; wph ^= 1; }
      };
      for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
        const int b = item / tiles, t = item - b * tiles;
        const int y0 = (t / s.tiles_x) * HD_TH, x0 = (t % s.tiles_x) * HD_TW;
        for (int pass = 0; pass < CMID / L::NT1; ++pass) {
          for (int cb = 0; cb < s.ncb; ++cb) {
            mbar_wait(&h_empty[hs], (uint32_t)(hph ^ 1));
            mbar_expect_tx(&h_full[hs], 4 * HD_SLAB);
            unsigned char *h = sm + L::HALO + (size_t)hs * HD_HALO_BYTES;
#pragma unroll
            for (int kc = 0; kc < 4; ++kc)
              tma_load_4d(h + kc * HD_SLAB_PITCH, &xmap, cb * 32 + kc * 8, x0 - 1, y0 - 1, b, &h_full[hs]);
            if (++hs == HD_HSTAGES) { hs = 0; hph ^= 1; }
            for (int tap = 0; tap < 9; ++tap)
              put_w(w1t + (size_t)((pass * s.ncb + cb) * 9 + tap) * L::NT1 * 32, L::NT1 * 64);
          }
        }
        for (int kc = 0; kc < CMID / 32; ++kc) put_w(w2t + (size_t)kc * N2 * 32, N2 * 64);
      }
    }
    return;
  }

  // ============================================================== consumers
  const int wg = warp >> 2, wq = warp & 3;
  unsigned char *inter = sm + L::INTER + (size_t)wg * L::INTER_WG;
  const uint32_t inter_u = smem_u32(inter);
  int hs = 0, hph = 0, ws = 0, wph = 0;
  for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
    const int b = item / tiles, t = item - b * tiles;
    const int y0 = (t / s.tiles_x) * HD_TH, x0 = (t % s.tiles_x) * HD_TW;
    for (int pass = 0; pass < CMID / L::NT1; ++pass) {
      float d[L::NT1 / 2];
#pragma unroll
      for (int i = 0; i < L::NT1 / 2; ++i) d[i] = 0.f;
      for (int cb = 0; cb < s.ncb; ++cb) {
        mbar_wait(&h_full[hs], (uint32_t)hph);
        // this warpgroup's first pixel row sits at halo row 8 * wg
        const uint32_t h = smem_u32(sm + L::HALO + (size_t)hs * HD_HALO_BYTES) + (uint32_t)(wg * 8 * HD_HX) * 16u;
        for (int tap = 0; tap < 9; ++tap) {
          mbar_wait(&w_full[ws], (uint32_t)wph);
          const uint32_t a = h + (uint32_t)((tap / 3) * HD_HX + tap % 3) * 16u;
          const uint32_t bw = smem_u32(sm + L::RING + (size_t)ws * L::W_BYTES);
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 2; ++ks)   // one k16 step = two 8-channel slabs
            wgmma_bf16<L::NT1>(d, wg_desc(a + (uint32_t)ks * 2u * HD_SLAB_PITCH, HD_SLAB_PITCH, HD_HX * 16),
                               wg_desc(bw + (uint32_t)ks * 2u * BF_B_LBO, BF_B_LBO, BF_B_SBO),
                               (cb > 0 || tap > 0 || ks > 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait_all();
          if ((tid & 127) == 0) mbar_arrive_tc(&w_empty[ws]);
          if (++ws == HD_WSTAGES) { ws = 0; wph ^= 1; }
        }
        if ((tid & 127) == 0) mbar_arrive_tc(&h_empty[hs]);
        if (++hs == HD_HSTAGES) { hs = 0; hph ^= 1; }
      }
      // epilogue 1: d[4j + 2h + e] is row wq * 16 + lane / 4 + 8h, channel pass * NT1 + 8j + 2 * (lane % 4) + e.
      // The intermediate is K-major: core matrix (row group r / 8, k-chunk kc) at (r / 8) * CMID * 16 + kc * 128
#pragma unroll
      for (int j = 0; j < L::NT1 / 8; ++j) {
        const int c = pass * L::NT1 + 8 * j + 2 * (lane & 3);
        const float bb0 = c < s.Cmid ? __ldg(b1 + c) : 0.f, bb1 = c + 1 < s.Cmid ? __ldg(b1 + c + 1) : 0.f;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = wq * 16 + (lane >> 2) + 8 * hh;
          const float v0 = c < s.Cmid ? relu_nan(d[4 * j + 2 * hh] + bb0) : 0.f;
          const float v1 = c + 1 < s.Cmid ? relu_nan(d[4 * j + 2 * hh + 1] + bb1) : 0.f;
          *reinterpret_cast<uint32_t *>(inter + (r >> 3) * (CMID * 16) + (c >> 3) * 128 + (r & 7) * 16 +
                                        (lane & 3) * 4) =
              pack2_bf16(v0, v1);
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> async proxy (wgmma reads)
    named_bar_sync(1 + wg, 128);

    float e[N2 / 2];
#pragma unroll
    for (int i = 0; i < N2 / 2; ++i) e[i] = 0.f;
    for (int kc = 0; kc < CMID / 32; ++kc) {
      mbar_wait(&w_full[ws], (uint32_t)wph);
      const uint32_t a = inter_u + (uint32_t)kc * 4u * 128u;
      const uint32_t bw = smem_u32(sm + L::RING + (size_t)ws * L::W_BYTES);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
        wgmma_bf16<N2>(e, wg_desc(a + (uint32_t)ks * 256u, 128, CMID * 16),
                       wg_desc(bw + (uint32_t)ks * 2u * BF_B_LBO, BF_B_LBO, BF_B_SBO), (kc > 0 || ks > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait_all();
      if ((tid & 127) == 0) mbar_arrive_tc(&w_empty[ws]);
      if (++ws == HD_WSTAGES) { ws = 0; wph ^= 1; }
    }
    // epilogue 2: + b2, stored as the input's dtype in the input's layout
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = wq * 16 + (lane >> 2) + 8 * hh;
      const int y = y0 + wg * 8 + (r >> 3), x = x0 + (r & 7);
      if (y >= s.H || x >= s.W) continue;
      const size_t pix = ((size_t)b * s.H + y) * s.W + x;
#pragma unroll
      for (int j = 0; j < N2 / 8; ++j) {
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
          const int o = 8 * j + 2 * (lane & 3) + e2;
          if (o >= s.Cout) continue;
          const float v = e[4 * j + 2 * hh + e2] + __ldg(b2 + o);
          const size_t idx = s.out_cl ? pix * s.Cout + o
                                      : (((size_t)b * s.Cout + o) * s.H + y) * s.W + x;
          if (s.out_bf16) reinterpret_cast<__nv_bfloat16 *>(out)[idx] = __float2bfloat16_rn(v);
          else reinterpret_cast<float *>(out)[idx] = v;
        }
      }
    }
  }
}

template <int CMID, int N2>
int launch_head(const CUtensorMap &map, const void *w1t, const float *b1, const void *w2t, const float *b2, void *out,
                const HeadShape &s, cudaStream_t stream) {
  const size_t smem = HeadSmem<CMID, N2>::BYTES;
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_head_fwd_bf16<CMID, N2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dev_done = dev;
  }
  const int grid = s.n_items < num_sms() ? s.n_items : num_sms();
  k_head_fwd_bf16<CMID, N2><<<grid, HD_THREADS, smem, stream>>>(
      map, reinterpret_cast<const __nv_bfloat16 *>(w1t), b1, reinterpret_cast<const __nv_bfloat16 *>(w2t), b2, out, s);
  CNB_CHECK_LAUNCH("cnb_head_forward_bf16 (wgmma)");
  count_launch();
  return CNB_OK;
}

template <int CMID>
int launch_head_n2(const CUtensorMap &map, const void *w1t, const float *b1, const void *w2t, const float *b2,
                   void *out, const HeadShape &s, cudaStream_t stream) {
  switch (head_n2_pad(s.Cout)) {
    case 8: return launch_head<CMID, 8>(map, w1t, b1, w2t, b2, out, s, stream);
    case 16: return launch_head<CMID, 16>(map, w1t, b1, w2t, b2, out, s, stream);
    case 32: return launch_head<CMID, 32>(map, w1t, b1, w2t, b2, out, s, stream);
    case 64: return launch_head<CMID, 64>(map, w1t, b1, w2t, b2, out, s, stream);
    case 128: return launch_head<CMID, 128>(map, w1t, b1, w2t, b2, out, s, stream);
    default: return launch_head<CMID, 256>(map, w1t, b1, w2t, b2, out, s, stream);
  }
}

// The checks every entry shares: CNB_EINVAL for a bad shape, CNB_EUNSUPPORTED outside the kernel's range
int head_check(const char *fn, int b, int cin, int h, int w, int cmid, int cout) {
  CNB_REQUIRE(b > 0 && cin > 0 && h > 0 && w > 0 && cmid > 0 && cout > 0, CNB_EINVAL, "%s: bad shape", fn);
  CNB_REQUIRE(cin % 32 == 0 && cmid % 32 == 0 && cmid <= 256 && cout <= 256, CNB_EUNSUPPORTED,
              "%s: needs cin and head_conv multiples of 32, head_conv <= 256 and 1 <= C <= 256 (got cin %d, "
              "head_conv %d, C %d)", fn, cin, cmid, cout);
  const long long px = (long long)b * h * w;
  const int cmax = cin > cout ? cin : cout;
  CNB_REQUIRE(px * cmax < (1ll << 31) && (long long)h * w * cin < (1ll << 31), CNB_EUNSUPPORTED,
              "%s: tensors beyond 32-bit indexing", fn);
  return CNB_OK;
}

}  // namespace
}  // namespace cnb

using namespace cnb;

extern "C" {

size_t cnb_head_w1t_bytes(int cin, int cmid) {
  if (head_check("cnb_head_w1t_bytes", 1, cin, 1, 1, cmid, 1) != CNB_OK) return 0;
  return (size_t)(cin / 32) * 9 * head_cmid_pad(cmid) * 64;
}

size_t cnb_head_w2t_bytes(int cmid, int cout) {
  if (head_check("cnb_head_w2t_bytes", 1, 32, 1, 1, cmid, cout) != CNB_OK) return 0;
  return (size_t)(head_cmid_pad(cmid) / 32) * head_n2_pad(cout) * 64;
}

int cnb_head_prepare_weights_bf16(const float *w1, const float *w2, int cin, int cmid, int cout, void *w1t,
                                  size_t w1t_bytes, void *w2t, size_t w2t_bytes, void *stream) {
  const char *fn = "cnb_head_prepare_weights_bf16";
  CNB_REQUIRE(w1 && w2 && w1t && w2t, CNB_EINVAL, "%s: null pointer", fn);
  const int rc = head_check(fn, 1, cin, 1, 1, cmid, cout);
  if (rc != CNB_OK) return rc;
  CNB_REQUIRE(w1t_bytes >= cnb_head_w1t_bytes(cin, cmid) && w2t_bytes >= cnb_head_w2t_bytes(cmid, cout),
              CNB_EWORKSPACE, "%s: weight-tile buffer too small", fn);
  CNB_REQUIRE(((reinterpret_cast<uintptr_t>(w1t) | reinterpret_cast<uintptr_t>(w2t)) & 15u) == 0, CNB_EINVAL,
              "%s: tile buffers must be 16-byte aligned", fn);
  const int CMIDp = head_cmid_pad(cmid);
  const int tiles = (CMIDp / head_nt1(CMIDp)) * (cin / 32) * 9 + CMIDp / 32;
  k_head_prep<<<tiles, 256, 0, (cudaStream_t)stream>>>(w1, w2, cin, cmid, cout, CMIDp, head_n2_pad(cout),
                                                      reinterpret_cast<unsigned char *>(w1t),
                                                      reinterpret_cast<unsigned char *>(w2t));
  CNB_CHECK_LAUNCH("cnb_head_prepare_weights_bf16");
  count_launch();
  return CNB_OK;
}

size_t cnb_head_workspace_bytes(int b, int cin, int h, int w, int input_dtype, int input_channels_last) {
  if (head_check("cnb_head_workspace_bytes", b, cin, h, w, 32, 1) != CNB_OK) return 0;
  if (input_dtype == CNB_DTYPE_BF16 && input_channels_last) return 0;   // read in place
  return (size_t)b * h * w * cin * 2;
}

int cnb_head_forward_bf16(const void *input, int input_dtype, int input_channels_last, const void *w1t,
                          const float *b1, const void *w2t, const float *b2, void *out, int b, int cin, int h, int w,
                          int cmid, int cout, void *ws, size_t ws_bytes, void *stream) {
  const char *fn = "cnb_head_forward_bf16";
  CNB_REQUIRE(input && w1t && b1 && w2t && b2 && out, CNB_EINVAL, "%s: null pointer", fn);
  CNB_REQUIRE(input_dtype == CNB_DTYPE_F32 || input_dtype == CNB_DTYPE_BF16, CNB_EINVAL,
              "%s: input dtype must be CNB_DTYPE_F32 or CNB_DTYPE_BF16 (got %d)", fn, input_dtype);
  const int rc = head_check(fn, b, cin, h, w, cmid, cout);
  if (rc != CNB_OK) return rc;
  const size_t need = cnb_head_workspace_bytes(b, cin, h, w, input_dtype, input_channels_last);
  CNB_REQUIRE(need == 0 || ws, CNB_EINVAL, "%s: null workspace", fn);
  CNB_REQUIRE(ws_bytes >= need, CNB_EWORKSPACE, "%s: workspace %zu < %zu", fn, ws_bytes, need);
  CNB_REQUIRE(((reinterpret_cast<uintptr_t>(input) | reinterpret_cast<uintptr_t>(w1t) |
                reinterpret_cast<uintptr_t>(w2t) | reinterpret_cast<uintptr_t>(ws)) & 15u) == 0,
              CNB_EINVAL, "%s: input, tile buffers and workspace must be 16-byte aligned", fn);
  CNB_REQUIRE(tensor_map_encoder() != nullptr, CNB_ECUDA, "%s: the driver has no cuTensorMapEncodeTiled", fn);

  cudaStream_t st = (cudaStream_t)stream;
  const long long HW = (long long)h * w;
  const void *xt = input;
  if (need) {   // one pass to bf16 channels-last
    __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(ws);
    if (input_channels_last) {
      const long long n8 = (long long)b * HW * cin / 8;
      const int grid = (int)((n8 + 255) / 256 < 4096 ? (n8 + 255) / 256 : 4096);
      k_head_cl_to_bf16<<<grid, 256, 0, st>>>(reinterpret_cast<const float4 *>(input), reinterpret_cast<uint4 *>(dst),
                                              n8);
    } else {
      const dim3 grid((unsigned)((HW + 31) / 32), (unsigned)(cin / 32), (unsigned)b);
      if (input_dtype == CNB_DTYPE_BF16)
        k_head_nhwc<__nv_bfloat16><<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16 *>(input), dst, cin, HW);
      else
        k_head_nhwc<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float *>(input), dst, cin, HW);
    }
    CNB_CHECK_LAUNCH("cnb_head_forward_bf16 channels-last copy");
    count_launch();
    xt = dst;
  }

  CUtensorMap map;
  const CUresult cr = encode_halo_map(&map, xt, b, cin, h, w, HD_HX, HD_HY);
  CNB_REQUIRE(cr == CUDA_SUCCESS, CNB_ECUDA, "%s: cuTensorMapEncodeTiled failed (%d)", fn, (int)cr);

  HeadShape s;
  s.B = b; s.Cin = cin; s.H = h; s.W = w; s.Cmid = cmid; s.Cout = cout;
  s.tiles_x = (w + HD_TW - 1) / HD_TW;
  s.tiles_y = (h + HD_TH - 1) / HD_TH;
  s.n_items = b * s.tiles_x * s.tiles_y;
  s.ncb = cin / 32;
  s.out_bf16 = input_dtype == CNB_DTYPE_BF16;
  s.out_cl = input_channels_last != 0;
  switch (head_cmid_pad(cmid)) {
    case 64: return launch_head_n2<64>(map, w1t, b1, w2t, b2, out, s, st);
    case 128: return launch_head_n2<128>(map, w1t, b1, w2t, b2, out, s, st);
    default: return launch_head_n2<256>(map, w1t, b1, w2t, b2, out, s, st);
  }
}

}  // extern "C"
