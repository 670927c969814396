// DCNv2 forward with the dense contraction on the Hopper tensor cores (wgmma) -- a persistent,
// warp-specialised pipeline (reference: dcn_v2_cuda.c:10-102 + dcn_v2_im2col_cuda.cu:118-180).
//
//   work item   = (image, 8x16 output-pixel tile [128 pixels = 2 x wgmma M], Cout tile of 64|128, K split)
//   chunk       = 32 input channels x one tap: K = 32 of the contraction; chunks of an item run over
//                 (channel block OUTER, tap INNER), so the ~40 KB input neighbourhood of a channel block is
//                 fetched from L2 once and then re-read by all 9 taps x 4 bilinear corners out of L1
//   sampler warps (16)  build the column tile col[128 px, 32 ch] of a chunk directly in shared memory
//                 (never in HBM -- the reference writes and re-reads a 37.7 MB column matrix per sample),
//                 split into TF32 hi/lo, in the canonical no-swizzle K-major layout; 2|3-deep ring
//   TMA warp      streams the matching pre-split weight tile (hi+lo) with cp.async.bulk (UBLKCP)
//   consumer warpgroups (2)  each issues wgmma.m64nCo_t k8 .tf32 on its 64 rows: D[64, Cout_t] += col . W^T,
//                 three MMAs per k-step (lo.hi + hi.lo + hi.hi = "3xTF32", fp32-accurate: the reference is an fp32
//                 SGEMM and plain TF32 misses the 1e-4 bar at K = Cin*9 <= 4608), waits for them and frees the ring
//                 slot; the accumulator lives in registers, and the same warpgroup adds the bias and stores NCHW
//                 while the samplers are already filling the ring for the next item
// Nobody waits on anybody except through mbarriers; the only CTA-wide barriers are at start and end.
//
// Sampling: the input is read from a channels-last copy [B][H*W][Cin/32][32] (k_dcn_nhwc; skipped when the
// caller's tensor already is channels-last).  A warp gather covers 4 pixels x 32 channels with
// lane = pixel * 8 + quad, so each quarter-warp -- the unit the L1 data pipe serves for 16-byte accesses --
// reads ONE fully used 128-byte line (4 wavefronts per gather).  Each lane then holds exactly one 16-byte k-chunk of
// the K-major A tile; the tile's k-chunks are pitched 144 bytes (LBO in the descriptor) instead of 128, which puts
// the eight chunks a quarter-warp stores into eight different bank groups -- conflict-free without a transpose
// (round 1 transposed across the warp with 16 shuffles; same speed, fewer instructions).
//
// Small maps (16x16, 8x8): too few tiles to fill 132 SMs, so the channel blocks of an item are split over
// several CTAs (split-K); the partial sums go to the workspace and k_dcn_reduce adds them in a fixed order
// (deterministic, no atomics).
//
// The weight tiles are pre-split / pre-tiled by k_dcn_prep_weights: once per call through the plain
// cnb_dcnv2_forward, or once per weight version through cnb_dcnv2_prepare_weights +
// cnb_dcnv2_forward_prepared (what the Python module does).
//
// k_dcn_forward is templated on the operand format (Tf32x3 / Bf16, dcnv2_tc.cuh).  Its Bf16 form is the opt-in bf16
// forward: one bf16 tile per operand, wgmma k16 bf16 -> fp32, samplers with 8-channel lanes.  Its OM variant (the DCN
// block, bf16 only) also computes the 3x3 conv_offset_mask inside the kernel.
#include <cuda_bf16.h>

#include <type_traits>

#include "halo.cuh"

namespace cnb {

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {   // lo -> lower address (smaller k)
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&v);
}
__device__ __forceinline__ void store_out(float *p, float v) { *p = v; }
__device__ __forceinline__ void store_out(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ float load_in(const float *p) { return __ldg(p); }
__device__ __forceinline__ float load_in(const __nv_bfloat16 *p) { return __bfloat162float(p[0]); }

// W[Cout][Cin][KT] (fp32) -> per (cout tile, channel block bi, tap) one operand tile [co_t][32] (k = channel within
// the block; TF32: hi tile then lo tile).  Tile index = (cot * nb + bi) * 9 + tap.
template <typename F>
__global__ void __launch_bounds__(256) k_dcn_prep_weights(const float *__restrict__ w, const DcnShapeTc s,
                                                          unsigned char *__restrict__ ws) {
  const int KT = s.kh * s.kw;
  const int cpg = s.Cin / s.dg;
  const int tile = blockIdx.x;
  const int tap = tile % TC_NT, r = tile / TC_NT;
  const int bi = r % s.nb, cot = r / s.nb;
  const int g = bi / s.cbs_pg, cbi = bi - g * s.cbs_pg;
  const size_t tile_elems = (size_t)s.co_t * TC_K;
  unsigned char *dst = ws + (size_t)tile * tile_elems * F::ELEM;
  for (int i = threadIdx.x; i < s.co_t * TC_K; i += blockDim.x) {
    const int o = i / TC_K, k = i - o * TC_K;
    const int cw = cbi * TC_CB + k;                    // channel within the group
    float v = 0.f;
    const int oc = cot * s.co_t + o;
    if (oc < s.Cout && cw < cpg && tap < KT) v = w[((size_t)oc * s.Cin + g * cpg + cw) * KT + tap];
    F::put(dst, tile_elems * 4, o, k, v);
  }
}

// x [B][Cin][HW] -> xt [B][HW][nb][32] (fp32 or bf16 either side; bf16 out is rounded RN, bf16 in widens exactly);
// channel ch of group g sits in block g*cbs_pg + (ch - g*cpg)/32, slot (ch - g*cpg) % 32 (identity when Cin/dg is a
// multiple of 32; pad slots are zero-filled by the caller).  grid (pixel blocks of 32, channel blocks of 64, B), 256
// threads.
template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256) k_dcn_nhwc(const TIn *__restrict__ x, TOut *__restrict__ xt,
                                                  const DcnShapeTc s) {
  __shared__ float tile[64][33];
  const long long HW = (long long)s.H * s.W;
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 64, b = blockIdx.z;
  const int Cp = s.nb * TC_CB;
  const int cpg = s.Cin / s.dg;
  {
    const int px = threadIdx.x & 31, cr = threadIdx.x >> 5;
    for (int c = cr; c < 64; c += 8) {
      float v = 0.f;
      if (c0 + c < s.Cin && p0 + px < HW) v = load_in(x + ((long long)b * s.Cin + c0 + c) * HW + p0 + px);
      tile[c][px] = v;
    }
  }
  __syncthreads();
  {
    const int c = threadIdx.x & 63, pr = threadIdx.x >> 6;
    const int ch = c0 + c;
    if (ch < s.Cin) {
      const int g = ch / cpg, within = ch - g * cpg;
      const int slot = (g * s.cbs_pg + within / TC_CB) * TC_CB + within % TC_CB;
      for (int px = pr; px < 32; px += 4)
        if (p0 + px < HW) store_out(xt + ((long long)b * HW + p0 + px) * Cp + slot, tile[c][px]);
    }
  }
}

// y[b][o][p] = epilogue(bias[o] + sum_s part[s][b][o][p]), s ascending (deterministic split-K epilogue), stored as
// fp32 or rounded (RN) to bf16
template <typename TOut>
__global__ void __launch_bounds__(256) k_dcn_reduce(const float *__restrict__ part, const float *__restrict__ bias,
                                                    TOut *__restrict__ y, int splits, int cout, long long hwo,
                                                    long long total, const float *__restrict__ epi_scale,
                                                    const float *__restrict__ epi_shift, int relu) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)((i / hwo) % cout);
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += __ldg(part + (long long)s * total + i);
    if (bias) v += __ldg(bias + o);
    if (epi_scale) v = fmaf(v, __ldg(epi_scale + o), __ldg(epi_shift + o));
    if (relu) v = v < 0.f ? 0.f : v;   // keeps NaN, as torch.relu (fmaxf would make it 0)
    store_out(y + i, v);
  }
}

// fp32 channels-last [B][HW][Cin] with whole 32-channel blocks (so slot == channel) -> bf16 xt, 8 values a thread
__global__ void __launch_bounds__(256) k_dcn_cl_to_bf16(const float4 *__restrict__ x, uint4 *__restrict__ xt,
                                                        long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = __ldg(x + 2 * i), b = __ldg(x + 2 * i + 1);
    xt[i] = make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
  }
}

// bf16 channels-last [B][HW][Cin] with whole 32-channel blocks (slot == channel) -> fp32 xt, 8 values a thread
__global__ void __launch_bounds__(256) k_dcn_cl_widen(const uint4 *__restrict__ x, float4 *__restrict__ xt, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u = __ldg(x + i);
    xt[2 * i] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                            __uint_as_float(u.y & 0xffff0000u));
    xt[2 * i + 1] = make_float4(__uint_as_float(u.z << 16), __uint_as_float(u.z & 0xffff0000u),
                                __uint_as_float(u.w << 16), __uint_as_float(u.w & 0xffff0000u));
  }
}

struct ItemTc {
  int b, cot, b0, b1;     // image, Cout tile, channel blocks [b0, b1)
  int ty0, tx0, split;
};
__device__ __forceinline__ ItemTc tc_item(const DcnShapeTc &s, int item) {
  ItemTc it;
  it.split = item % s.splits;
  int r = item / s.splits;
  it.cot = r % s.n_cot;
  r /= s.n_cot;
  const int tiles = s.tiles_x * s.tiles_y;
  const int t = r % tiles;
  it.b = r / tiles;
  it.ty0 = (t / s.tiles_x) * s.th;
  it.tx0 = (t % s.tiles_x) * s.tw;
  it.b0 = (int)((long long)it.split * s.nb / s.splits);
  it.b1 = (int)((long long)(it.split + 1) * s.nb / s.splits);
  return it;
}

// Bilinear geometry of every (tap, pixel) of item `it` in deformable group g, the mask folded into the corner weights
// (dcn_v2_im2col_cuda.cu:18-47, :165); st = this thread's index among the sampler threads.  load(t, pp, p, dy, dx, m)
// fetches the offsets and the mask (a logit when s.mask_logit) of tap t at tile pixel pp, image pixel p.  Shared by the
// fp32, the bf16 and the block forward, so all of them sample at bit-identical fp32 weights for the same offsets.
template <typename Load>
__device__ __forceinline__ void tc_build_meta_from(const DcnShapeTc &s, const ItemTc &it, int st, int KT,
                                                   TapMetaTc *meta, Load load) {
  for (int idx = st; idx < TC_NT * TC_TP; idx += TC_SAMPLERS * 32) {
    const int t = idx / TC_TP, pp = idx - t * TC_TP;
    const int ho = it.ty0 + pp / s.tw, wo = it.tx0 + pp % s.tw;
    TapMetaTc mt;   // o = -1: corner out of range, not read (the samplers select 0)
#pragma unroll
    for (int q = 0; q < 4; ++q) { mt.o[q] = -1; mt.w[q] = 0.f; }
    if (ho < s.Ho && wo < s.Wo && t < KT) {
      const long long p = (long long)ho * s.Wo + wo;
      const int i = t / s.kw, j = t - i * s.kw;
      float dy, dx, m;
      load(t, pp, p, dy, dx, m);
      if (s.mask_logit) m = 1.0f / (1.0f + expf(-m));        // torch.sigmoid(mask), dcn_v2.py:68
      const float h_im = (float)(ho * s.sh - s.ph + i * s.dh) + dy;
      const float w_im = (float)(wo * s.sw - s.pw + j * s.dw) + dx;
      if (h_im > -1.f && w_im > -1.f && h_im < (float)s.H && w_im < (float)s.W) {   // dcn_v2_im2col_cuda.cu:165
        const float hf = floorf(h_im), wf = floorf(w_im);
        const int hl = (int)hf, wl = (int)wf;
        const float lh = h_im - hf, lw = w_im - wf, hh = 1.f - lh, hw = 1.f - lw;
        const int base = hl * s.W + wl;
        if (hl >= 0 && wl >= 0) { mt.o[0] = base; mt.w[0] = hh * hw * m; }                       // :31-41
        if (hl >= 0 && wl + 1 <= s.W - 1) { mt.o[1] = base + 1; mt.w[1] = hh * lw * m; }
        if (hl + 1 <= s.H - 1 && wl >= 0) { mt.o[2] = base + s.W; mt.w[2] = lh * hw * m; }
        if (hl + 1 <= s.H - 1 && wl + 1 <= s.W - 1) { mt.o[3] = base + s.W + 1; mt.w[3] = lh * lw * m; }
      } else {
        mt.w[0] = 0.f * m;   // outside: the column value is 0 * mask (:174), NaN for a NaN mask
      }
    }
    meta[idx] = mt;
  }
}

// ... with the offsets and the mask read from global memory
__device__ __forceinline__ void tc_build_meta(const DcnShapeTc &s, const float *__restrict__ offset,
                                              const float *__restrict__ mask, const ItemTc &it, int g, int st,
                                              int KT, long long HWo, TapMetaTc *meta) {
  const float *op = offset + (long long)it.b * s.off_bs + (long long)g * 2 * KT * HWo;
  const float *mp = mask + (long long)it.b * s.mask_bs + (long long)g * KT * HWo;
  tc_build_meta_from(s, it, st, KT, meta, [&](int t, int, long long p, float &dy, float &dx, float &m) {
    dy = __ldg(op + (2 * t) * HWo + p);
    dx = __ldg(op + (2 * t + 1) * HWo + p);
    m = __ldg(mp + t * HWo + p);
  });
}

// DCN block variant (OM = true, cnb_dcnv2_forward_block_bf16): the 3x3 conv_offset_mask runs inside the kernel.
// For every item the TMA warp streams, per 32-channel block, the (tw + 2) x (th + 2) halo of the tile as four 8-channel
// slabs (4-D tensor-map loads; the out-of-bounds fill is the conv's zero padding, halo.cuh) and the nine [32][32] W_om
// tiles of the block into a ring of its own.  The consumer warpgroups compute om[128 px][27 -> 32] with wgmma m64n32k16
// straight from the halo (shifted descriptors, no im2col), add b_om in fp32 and leave the 27 fp32 values of every pixel
// in one of two shared buffers; the samplers build the item's tap geometry from that buffer (tc_build_meta_from, the
// mask logit through the same sigmoid).  The consumers compute the offsets of the CTA's NEXT item before the main loop
// of the current one, so the samplers find them ready when they reach the item boundary.  Every item computes its own
// offsets (Cout tiles and K splits of one pixel tile recompute them).  Warpgroup wg's 64 GEMM rows are the tile's
// column half wg (8 x 16 tiles: 8 rows of 8 pixels, one halo row apart) or row half wg (16 x 8 tiles).
constexpr int OM_N = 32;                             // 27 offset / mask channels, padded to the wgmma N
constexpr int OM_C = 27;                             // dg * 3 * 9 with dg = 1
constexpr int OM_PITCH = TC_TP + 4;                  // fp32 om of one channel: 128 pixels (+4: conflict-free stores)
constexpr uint32_t OM_SLAB = 180 * 16;               // one 8-channel slab of a 10 x 18 (or 18 x 10) halo
constexpr uint32_t OM_SLAB_PITCH = 2944;             // slabs 128-byte aligned (TMA destination)
constexpr uint32_t OM_HALO_BYTES = 4 * OM_SLAB_PITCH;
constexpr uint32_t OM_W_BYTES = TC_NT * OM_N * TC_K * 2;   // the nine W_om tiles of one channel block
constexpr uint32_t OM_STAGE_BYTES = OM_HALO_BYTES + OM_W_BYTES;
constexpr int OM_STAGES = 2;
constexpr uint32_t OM_BUF_BYTES = (OM_C * OM_PITCH * 4 + 127) / 128 * 128;
constexpr uint32_t OM_SMEM_BYTES = OM_STAGES * OM_STAGE_BYTES + 2 * OM_BUF_BYTES + 128;   // + 128: alignment slack

template <typename F, int CO_T, typename TOut, bool OM>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_dcn_forward(const typename F::X *__restrict__ xt, const float *__restrict__ offset, const float *__restrict__ mask,
              const unsigned char *__restrict__ wtiles, const float *__restrict__ bias, TOut *__restrict__ y,
              float *__restrict__ part, const DcnShapeTc s, const __grid_constant__ CUtensorMap xmap,
              const __nv_bfloat16 *__restrict__ womt, const float *__restrict__ bom) {
  static_assert(!OM || F::KE == 8, "k_dcn_forward: the DCN block variant is bf16 only");
  extern __shared__ __align__(128) unsigned char tc_smem_raw[];
  // the block variant's TMA halo needs a 128-byte aligned destination
  unsigned char *tc_smem = OM ? tc_smem_raw + ((128u - (smem_u32(tc_smem_raw) & 127u)) & 127u) : tc_smem_raw;
  constexpr int STAGES = F::fw_stages(CO_T);
  constexpr int B_BYTES = CO_T * TC_K * F::ELEM;          // one weight operand tile
  constexpr int STAGE_BYTES = F::FW_A + B_BYTES;
  static_assert(TC_SAMPLER_ROUNDS == 2, "k_dcn_forward: two row groups a sampler warp");
  TapMetaTc *meta = reinterpret_cast<TapMetaTc *>(tc_smem + (size_t)STAGES * STAGE_BYTES);     // [9][128]
  unsigned char *om_ring = tc_smem + (size_t)STAGES * STAGE_BYTES + sizeof(TapMetaTc) * TC_NT * TC_TP;
  float *om_buf = reinterpret_cast<float *>(om_ring + OM_STAGES * OM_STAGE_BYTES);   // [2][27][OM_PITCH]
  __shared__ __align__(8) uint64_t a_full[STAGES], b_full[STAGES], empty[STAGES];
  __shared__ __align__(8) uint64_t om_full[OM ? OM_STAGES : 1], om_empty[OM ? OM_STAGES : 1], om_ready[2], om_free[2];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KT = s.kh * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int Cp = s.nb * TC_CB;

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&a_full[i], TC_SAMPLERS);
      mbar_init(&b_full[i], 1);
      mbar_init(&empty[i], TC_MMA_WGS);
    }
    if (OM) {
      for (int i = 0; i < OM_STAGES; ++i) {
        mbar_init(&om_full[i], 1);
        mbar_init(&om_empty[i], TC_MMA_WGS);
      }
      for (int i = 0; i < 2; ++i) {
        mbar_init(&om_ready[i], TC_MMA_WGS * 128);
        mbar_init(&om_free[i], 1);
      }
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= TC_WARP_S0) {
    // =========================================================== samplers: A operand of every chunk
    // lane = (pixel sp, k-chunk sq): TF32 4 pixels x 8 k-chunks of 4 channels, bf16 8 pixels x 4 k-chunks of 8
    constexpr int KC = TC_K / F::KE;
    const int sw = warp - TC_WARP_S0, st = tid - TC_WARP_S0 * 32;
    const int sp = lane / KC, sq = lane % KC;
    int stage = 0, ph = 0, n = 0;
    for (int item = blockIdx.x; item < s.n_items; item += gridDim.x, ++n) {
      const ItemTc it = tc_item(s, item);
      const typename F::X *xbat = xt + (long long)it.b * HW * Cp + sq * F::KE;
      int cur_g = -1;
      for (int bi = it.b0; bi < it.b1; ++bi) {
        const int g = bi / s.cbs_pg;
        if (g != cur_g) {
          cur_g = g;
          named_bar_sync(1, TC_SAMPLERS * 32);   // everybody is done reading the previous geometry
          if constexpr (OM) {
            // dg == 1: one geometry an item, from the offsets the consumers left in buffer n % 2
            mbar_wait(&om_ready[n & 1], (uint32_t)((n >> 1) & 1));
            const float *ob = om_buf + (n & 1) * (OM_BUF_BYTES / 4);
            tc_build_meta_from(s, it, st, KT, meta, [&](int t, int pp, long long, float &dy, float &dx, float &m) {
              dy = ob[(2 * t) * OM_PITCH + pp];
              dx = ob[(2 * t + 1) * OM_PITCH + pp];
              m = ob[(2 * TC_NT + t) * OM_PITCH + pp];
            });
          } else {
            tc_build_meta(s, offset, mask, it, g, st, KT, HWo, meta);
          }
          named_bar_sync(1, TC_SAMPLERS * 32);
          if (OM && st == 0) mbar_arrive_tc(&om_free[n & 1]);   // the buffer may take the offsets of item n + 2
        }
        const typename F::X *xb = xbat + (long long)bi * TC_CB;
        for (int tap = 0; tap < TC_NT; ++tap) {
          if constexpr (F::KE == 4) {
          // TF32: warp item = 4 pixels: every lane gathers the 4 corners of its pixel as 16-byte pieces (4 channels);
          // a warp fills TC_SAMPLER_ROUNDS 8-pixel row groups, one after the other; both items of a group (pixels
          // 8r..8r+3 and 8r+4..8r+7) are gathered before either is reduced
#pragma unroll 1
          for (int rnd = 0; rnd < TC_SAMPLER_ROUNDS; ++rnd) {
          const int rgp = sw * TC_SAMPLER_ROUNDS + rnd;
          const int pp0 = rgp * 8 + sp, pp1 = pp0 + 4;
          const TapMetaTc m0 = meta[tap * TC_TP + pp0], m1 = meta[tap * TC_TP + pp1];
          float4 u0[4], u1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) u0[q] = m0.o[q] >= 0 ? __ldg(reinterpret_cast<const float4 *>(xb + (long long)m0.o[q] * Cp)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int q = 0; q < 4; ++q) u1[q] = m1.o[q] >= 0 ? __ldg(reinterpret_cast<const float4 *>(xb + (long long)m1.o[q] * Cp)) : make_float4(0.f, 0.f, 0.f, 0.f);
          auto reduce = [&](const TapMetaTc &mt, const float4 (&u)[4]) {
            float4 v;
            v.x = fmaf(mt.w[3], u[3].x, fmaf(mt.w[2], u[2].x, fmaf(mt.w[1], u[1].x, mt.w[0] * u[0].x)));
            v.y = fmaf(mt.w[3], u[3].y, fmaf(mt.w[2], u[2].y, fmaf(mt.w[1], u[1].y, mt.w[0] * u[0].y)));
            v.z = fmaf(mt.w[3], u[3].z, fmaf(mt.w[2], u[2].z, fmaf(mt.w[1], u[1].z, mt.w[0] * u[0].z)));
            v.w = fmaf(mt.w[3], u[3].w, fmaf(mt.w[2], u[2].w, fmaf(mt.w[1], u[1].w, mt.w[0] * u[0].w)));
            return v;
          };
          const float4 v0 = reduce(m0, u0), v1 = reduce(m1, u1);   // (row sp, quad sq) and (row 4 + sp, quad sq)
          // the ring slot must have been drained by the MMAs that last read it
          if (rnd == 0) mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
          unsigned char *a_hi = tc_smem + (size_t)stage * STAGE_BYTES;
          unsigned char *a_lo = a_hi + FW_A_BYTES;
          // each lane already holds one 16-byte k-chunk of the K-major tile: (row, chunk sq).  The k-chunks of the A tile
          // are pitched FW_LBO = 144 bytes (not 128), so the eight chunks of a row -- one quarter-warp -- fall into eight
          // different 16-byte bank groups: conflict-free stores without a transpose
          {
            const float4 h0 = make_float4(tf32_hi(v0.x), tf32_hi(v0.y), tf32_hi(v0.z), tf32_hi(v0.w));
            const float4 h1 = make_float4(tf32_hi(v1.x), tf32_hi(v1.y), tf32_hi(v1.z), tf32_hi(v1.w));
            const uint32_t off0 = (uint32_t)rgp * FW_SBO + (uint32_t)sq * FW_LBO + (uint32_t)sp * 16u, off1 = off0 + 64u;
            *reinterpret_cast<float4 *>(a_hi + off0) = h0;
            *reinterpret_cast<float4 *>(a_lo + off0) = make_float4(v0.x - h0.x, v0.y - h0.y, v0.z - h0.z, v0.w - h0.w);
            *reinterpret_cast<float4 *>(a_hi + off1) = h1;
            *reinterpret_cast<float4 *>(a_lo + off1) = make_float4(v1.x - h1.x, v1.y - h1.y, v1.z - h1.z, v1.w - h1.w);
          }
          }
          } else {
          // bf16: warp item = one 8-row group of the A tile (8 pixels): every lane gathers the 4 corners of its pixel as
          // 16-byte pieces (8 bf16 channels), interpolates in fp32 and stores one rounded 16-byte k-chunk; each warp
          // fills two row groups a chunk, both gathered before either is reduced
          const int rg0 = sw * TC_SAMPLER_ROUNDS, rg1 = rg0 + 1;
          const TapMetaTc m0 = meta[tap * TC_TP + rg0 * 8 + sp], m1 = meta[tap * TC_TP + rg1 * 8 + sp];
          uint4 u0[4], u1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) u0[q] = m0.o[q] >= 0 ? __ldg(reinterpret_cast<const uint4 *>(xb + (long long)m0.o[q] * Cp)) : make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int q = 0; q < 4; ++q) u1[q] = m1.o[q] >= 0 ? __ldg(reinterpret_cast<const uint4 *>(xb + (long long)m1.o[q] * Cp)) : make_uint4(0, 0, 0, 0);
          // fp32 value of channel 2e (lower half) / 2e + 1 (upper half) of a 4 x 32-bit piece: exact widening
          auto reduce = [&](const TapMetaTc &mt, const uint4 (&u)[4]) {
            uint32_t r[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              float v[2];
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float c[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const uint32_t word = e == 0 ? u[q].x : e == 1 ? u[q].y : e == 2 ? u[q].z : u[q].w;
                  c[q] = __uint_as_float(h == 0 ? word << 16 : word & 0xffff0000u);
                }
                v[h] = fmaf(mt.w[3], c[3], fmaf(mt.w[2], c[2], fmaf(mt.w[1], c[1], mt.w[0] * c[0])));
              }
              r[e] = pack_bf16x2(v[0], v[1]);
            }
            return make_uint4(r[0], r[1], r[2], r[3]);
          };
          const uint4 v0 = reduce(m0, u0), v1 = reduce(m1, u1);
          mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));   // drained by the MMAs that last read it
          unsigned char *a = tc_smem + (size_t)stage * STAGE_BYTES;
          const uint32_t off = (uint32_t)sq * BF_LBO + (uint32_t)sp * 16u;
          *reinterpret_cast<uint4 *>(a + (uint32_t)rg0 * BF_SBO + off) = v0;
          *reinterpret_cast<uint4 *>(a + (uint32_t)rg1 * BF_SBO + off) = v1;
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> async proxy (wgmma reads)
          __syncwarp();
          if (lane == 0) mbar_arrive_tc(&a_full[stage]);
          if (++stage == STAGES) { stage = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp == TC_WARP_TMA) {
    // =========================================================== B operand: weight tiles by TMA bulk copy
    if (lane == 0) {
      int stage = 0, ph = 0, os = 0, oph = 0;
      // block variant: the halo slabs and W_om tiles of every channel block of item `item`, in consumer order
      auto put_om = [&](int item) {
        const ItemTc it = tc_item(s, item);
        for (int cb = 0; cb < s.nb; ++cb) {
          mbar_wait(&om_empty[os], (uint32_t)(oph ^ 1));
          unsigned char *h = om_ring + (size_t)os * OM_STAGE_BYTES;
          mbar_expect_tx(&om_full[os], 4u * OM_SLAB + OM_W_BYTES);
#pragma unroll
          for (int kc = 0; kc < 4; ++kc)
            tma_load_4d(h + kc * OM_SLAB_PITCH, &xmap, cb * TC_CB + kc * 8, it.tx0 - 1, it.ty0 - 1, it.b, &om_full[os]);
          bulk_g2s(h + OM_HALO_BYTES, womt + (size_t)cb * (OM_W_BYTES / 2), OM_W_BYTES, &om_full[os]);
          if (++os == OM_STAGES) { os = 0; oph ^= 1; }
        }
      };
      if constexpr (OM) {
        if ((int)blockIdx.x < s.n_items) put_om(blockIdx.x);
      }
      for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
        if constexpr (OM) {
          if (item + (int)gridDim.x < s.n_items) put_om(item + gridDim.x);
        }
        const ItemTc it = tc_item(s, item);
        for (int bi = it.b0; bi < it.b1; ++bi) {
          for (int tap = 0; tap < TC_NT; ++tap) {
            mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
            unsigned char *b = tc_smem + (size_t)stage * STAGE_BYTES + F::FW_A;
            const unsigned char *src = wtiles + (((size_t)it.cot * s.nb + bi) * TC_NT + tap) * (size_t)B_BYTES;
            mbar_expect_tx(&b_full[stage], (uint32_t)B_BYTES);
            F::fetch(b, src, (uint32_t)B_BYTES, &b_full[stage]);
            if (++stage == STAGES) { stage = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    // =========================================================== consumers: wgmma over the ring, epilogue from registers
    const int wgi = warp >> 2, wq = warp & 3;
    int stage = 0, ph = 0, n = 0;
    // block variant: om of the CTA's k-th item into buffer k % 2 -- fp32 sums of exact bf16 products, + b_om.  The
    // k-th item takes offset-ring slots k * nb .. k * nb + nb - 1 (no ring state stays live across the main loop)
    auto om_gemm = [&](int k) {
      const uint32_t hx16 = (uint32_t)(s.tw + 2) * 16u;               // one halo row
      const uint32_t half = s.tw == 16 ? (uint32_t)wgi * 128u : (uint32_t)wgi * 8u * hx16;
      float q[OM_N / 2];
#pragma unroll
      for (int i = 0; i < OM_N / 2; ++i) q[i] = 0.f;
      for (int cb = 0; cb < s.nb; ++cb) {
        const int slot = k * s.nb + cb, os = slot % OM_STAGES;
        mbar_wait(&om_full[os], (uint32_t)((slot / OM_STAGES) & 1));
        const uint32_t h = smem_u32(om_ring + (size_t)os * OM_STAGE_BYTES) + half;
        const uint32_t wb = smem_u32(om_ring + (size_t)os * OM_STAGE_BYTES + OM_HALO_BYTES);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < TC_NT; ++tap) {
          const uint32_t a = h + (uint32_t)((tap / 3) * (int)hx16 + (tap % 3) * 16);
#pragma unroll
          for (int ks = 0; ks < 2; ++ks)   // one k16 step = two 8-channel slabs
            wgmma_bf16<OM_N>(q, wg_desc(a + (uint32_t)ks * 2u * OM_SLAB_PITCH, OM_SLAB_PITCH, hx16),
                           wg_desc(wb + (uint32_t)tap * (OM_N * TC_K * 2) + (uint32_t)ks * 2u * BF_B_LBO, BF_B_LBO,
                                   BF_B_SBO),
                           (cb > 0 || tap > 0 || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        if ((tid & 127) == 0) mbar_arrive_tc(&om_empty[os]);
      }
      mbar_wait(&om_free[k & 1], (uint32_t)(((k >> 1) & 1) ^ 1));   // the samplers are done with item k - 2
      float *ob = om_buf + (k & 1) * (OM_BUF_BYTES / 4);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int m = wq * 16 + (lane >> 2) + 8 * hh;                 // GEMM row: pixel (m / 8, m % 8) of the half
        const int pp = s.tw == 16 ? (m >> 3) * 16 + wgi * 8 + (m & 7) : wgi * 64 + m;
#pragma unroll
        for (int j = 0; j < OM_N / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * (lane & 3) + e;
            if (c < OM_C) ob[c * OM_PITCH + pp] = bom ? q[4 * j + 2 * hh + e] + __ldg(bom + c) : q[4 * j + 2 * hh + e];
          }
        }
      }
      mbar_arrive_tc(&om_ready[k & 1]);
    };
    if constexpr (OM) {
      if ((int)blockIdx.x < s.n_items) om_gemm(0);
    }
    for (int item = blockIdx.x; item < s.n_items; item += gridDim.x, ++n) {
      if constexpr (OM) {
        if (item + (int)gridDim.x < s.n_items) om_gemm(n + 1);
      }
      const ItemTc it = tc_item(s, item);
      float d[CO_T / 2];
#pragma unroll
      for (int i = 0; i < CO_T / 2; ++i) d[i] = 0.f;
      const int n_ch = (it.b1 - it.b0) * TC_NT;
      for (int ch = 0; ch < n_ch; ++ch) {
        mbar_wait(&a_full[stage], (uint32_t)ph);
        mbar_wait(&b_full[stage], (uint32_t)ph);
        const uint32_t base = smem_u32(tc_smem + (size_t)stage * STAGE_BYTES);
        wgmma_fence();   // A: this warpgroup's 64 rows
        F::template mma_k32<CO_T>(d, base + (uint32_t)wgi * 8u * F::FW_A_SBO, F::FW_A / 2, F::FW_A_LBO, F::FW_A_SBO,
                                  base + F::FW_A, B_BYTES / 2, ch > 0);
        wgmma_commit();
        wgmma_wait_all();
        if ((tid & 127) == 0) mbar_arrive_tc(&empty[stage]);
        if (++stage == STAGES) { stage = 0; ph ^= 1; }
      }
      // epilogue: d[4j + r] = (row wq*16 + lane/4 + 8*(r/2), column 8j + 2*(lane%4) + r%2) of this warpgroup's 64
      // rows; split-K partials stay fp32
      const long long img = (long long)it.b * s.Cout * HWo;
      float *pdst = s.splits > 1 ? part + (long long)it.split * s.B * s.Cout * HWo + img : nullptr;
      TOut *ydst = y + img;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pp = wgi * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int ho = it.ty0 + pp / s.tw, wo = it.tx0 + pp % s.tw;
        if (ho >= s.Ho || wo >= s.Wo) continue;
        const long long p = (long long)ho * s.Wo + wo;
#pragma unroll
        for (int j = 0; j < CO_T / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int o = it.cot * CO_T + 8 * j + 2 * (lane & 3) + e;
            if (o < s.Cout) {
              float r = d[4 * j + 2 * h + e];
              if (pdst) {
                pdst[(long long)o * HWo + p] = r;
              } else {
                if (bias) r += __ldg(bias + o);
                if (s.epi_scale) r = fmaf(r, __ldg(s.epi_scale + o), __ldg(s.epi_shift + o));
                if (s.relu) r = r < 0.f ? 0.f : r;   // keeps NaN, as torch.relu
                store_out(ydst + (long long)o * HWo + p, r);
              }
            }
          }
        }
      }
    }
  }
}


// ------------------------------------------------------------------ host
// Weight tiles of one format, one tile a (cout tile, channel block, tap) of the shape s
template <typename F>
static int prep_weights(const float *weight, const DcnShapeTc &s, void *wtiles, cudaStream_t stream) {
  k_dcn_prep_weights<F><<<s.n_cot * s.nb * TC_NT, 256, 0, stream>>>(weight, s, reinterpret_cast<unsigned char *>(wtiles));
  CNB_CHECK_LAUNCH("cnb_dcnv2 weight tiles");
  count_launch();
  return CNB_OK;
}

int dcn_prepare_weights_tc(const float *weight, int cin, int cout, int kh, int kw, int dg, float *wtiles,
                           cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg);
  return prep_weights<Tf32x3>(weight, s, wtiles, stream);
}

int dcn_prepare_weights_bf16(const float *weight, int cin, int cout, int kh, int kw, int dg, void *wtiles,
                             cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg);
  return prep_weights<Bf16>(weight, s, wtiles, stream);
}

// W_om [27][Cin][3][3] (fp32) -> per channel block nine bf16 tiles [32][32] (rows 27..31 zero), tile index bi * 9 + tap:
// the bf16 weight tiles of one Cout tile of 32 rows
int dcn_prepare_om_weights_bf16(const float *w_om, int cin, void *om_tiles, cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, OM_C, 3, 3, 1, 1, 1, 1, 1, 1, 1);
  s.co_t = OM_N;
  s.n_cot = 1;
  return prep_weights<Bf16>(w_om, s, om_tiles, stream);
}

size_t dcn_om_tiles_bytes(int cin) { return (size_t)(cin / TC_CB) * OM_W_BYTES; }

// x -> channels-last copy xt [B][HW][nb][32] in xt's element type.  x_cl: x is [B][HW][Cin] with whole 32-channel
// blocks (slot == channel) in the other element type, converted flat; else x is NCHW
template <typename TIn, typename TOut>
static int to_channels_last(const TIn *x, bool x_cl, TOut *xt, const DcnShapeTc &s, cudaStream_t stream) {
  const long long HW = (long long)s.H * s.W;
  if (x_cl) {
    const long long n8 = (long long)s.B * HW * s.Cin / 8;
    const int grid = (int)((n8 + 255) / 256 < 4096 ? (n8 + 255) / 256 : 4096);
    if constexpr (std::is_same_v<TOut, float>)
      k_dcn_cl_widen<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint4 *>(x), reinterpret_cast<float4 *>(xt), n8);
    else
      k_dcn_cl_to_bf16<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4 *>(x), reinterpret_cast<uint4 *>(xt), n8);
  } else {
    if ((s.Cin / s.dg) % TC_CB != 0)   // pad slots of the last channel block of every group must read as zero
      CNB_CUDA(cudaMemsetAsync(xt, 0, (size_t)s.B * HW * s.nb * TC_CB * sizeof(TOut), stream));
    dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((s.Cin + 63) / 64), (unsigned)s.B);
    k_dcn_nhwc<TIn, TOut><<<tgrid, 256, 0, stream>>>(x, xt, s);
  }
  CNB_CHECK_LAUNCH("cnb_dcnv2 channels-last copy");
  count_launch();
  return CNB_OK;
}

int dcn_to_channels_last(const float *x, float *xt, const DcnShapeTc &s, cudaStream_t stream) {
  return to_channels_last(x, false, xt, s, stream);
}

int dcn_to_channels_last(const __nv_bfloat16 *x, bool x_cl, float *xt, const DcnShapeTc &s, cudaStream_t stream) {
  return to_channels_last(x, x_cl, xt, s, stream);
}

// The channels-last source [B][HW][nb][32] the forward of format F samples: a channels-last input of F's element type
// in place, else a copy into the workspace region xt (l.xt)
template <typename F>
static int fwd_source(const DcnPlan &p, const DcnFwdLayout &l, const DcnShapeTc &s, const void *input, bool in_bf16,
                      void *workspace, cudaStream_t stream, const typename F::X **xsrc) {
  using X = typename F::X;
  X *xt = reinterpret_cast<X *>(reinterpret_cast<char *>(workspace) + l.xt);
  *xsrc = xt;
  if (p.x_cl && in_bf16 == std::is_same_v<X, __nv_bfloat16>) {
    *xsrc = reinterpret_cast<const X *>(input);   // sampled in place
    return CNB_OK;
  }
  if (in_bf16) return to_channels_last(reinterpret_cast<const __nv_bfloat16 *>(input), p.x_cl, xt, s, stream);
  return to_channels_last(reinterpret_cast<const float *>(input), p.x_cl, xt, s, stream);
}

// The operands of the block variant (OM); the other forwards pass none
struct OmArgs {
  CUtensorMap xmap;
  const __nv_bfloat16 *womt;
  const float *bom;
};

template <typename F, int CO_T, typename TOut, bool OM>
static int launch_fwd(const typename F::X *xt, const float *offset, const float *mask, const void *wtiles,
                      const float *bias, void *output, float *part, const DcnShapeTc &s, const OmArgs &om,
                      cudaStream_t stream) {
  const size_t smem = (size_t)F::fw_stages(CO_T) * (F::FW_A + CO_T * TC_K * F::ELEM) +
                      sizeof(TapMetaTc) * TC_NT * TC_TP + (OM ? OM_SMEM_BYTES : 0);
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_forward<F, CO_T, TOut, OM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    dev_done = dev;
  }
  const int grid = s.n_items < num_sms() ? s.n_items : num_sms();
  k_dcn_forward<F, CO_T, TOut, OM><<<grid, TC_THREADS, smem, stream>>>(
      xt, offset, mask, reinterpret_cast<const unsigned char *>(wtiles), bias, reinterpret_cast<TOut *>(output), part,
      s, om.xmap, om.womt, om.bom);
  CNB_CHECK_LAUNCH("cnb_dcnv2 forward (wgmma)");
  count_launch();
  return CNB_OK;
}

// The kernel for the Cout tile, then the split-K reduce on small maps
template <typename F, typename TOut, bool OM>
static int run_fwd(const typename F::X *xsrc, const float *offset, const float *mask, const void *wtiles,
                   const float *bias, void *output, float *part, const DcnShapeTc &s, const OmArgs &om,
                   cudaStream_t stream) {
  const int rc = s.co_t == 64 ? launch_fwd<F, 64, TOut, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream)
                              : launch_fwd<F, 128, TOut, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream);
  if (rc != CNB_OK) return rc;
  if (s.splits > 1) {
    const long long total = (long long)s.B * s.Cout * s.Ho * s.Wo;
    const int grid = (int)((total + 255) / 256 < 1184 ? (total + 255) / 256 : 1184);
    k_dcn_reduce<TOut><<<grid, 256, 0, stream>>>(part, bias, reinterpret_cast<TOut *>(output), s.splits, s.Cout,
                                                 (long long)s.Ho * s.Wo, total, s.epi_scale, s.epi_shift, s.relu);
    CNB_CHECK_LAUNCH("cnb_dcnv2 forward split-K reduce");
    count_launch();
  }
  return CNB_OK;
}

// The call's shape: fused_offset_mask: `offset` is the raw [b, 3*kt*dg, ho, wo] output of conv_offset_mask and *mask
// becomes its last third (mask logits); epi_scale / epi_shift / relu: the folded BatchNorm + ReLU epilogue
static DcnShapeTc call_shape(const DcnPlan &p, int fused_offset_mask, const float *offset, const float **mask,
                             const float *epi_scale, const float *epi_shift, int relu) {
  DcnShapeTc s = p.s;
  if (fused_offset_mask) {
    s.off_bs = s.mask_bs = (long long)s.dg * 3 * s.kh * s.kw * s.Ho * s.Wo;
    s.mask_logit = 1;
    *mask = offset + (long long)s.dg * 2 * s.kh * s.kw * s.Ho * s.Wo;
  }
  s.epi_scale = epi_scale;
  s.epi_shift = epi_scale ? epi_shift : nullptr;
  s.relu = relu;
  return s;
}

// Tensor-core forward from pre-tiled weights.  p.x_cl: `input` already is [B][H*W][Cin] (torch channels_last) with
// Cin/dg a multiple of 32 -- no re-layout pass.
int dcn_forward_tc_prepared(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                            const float *wtiles, const float *bias, float *output, void *workspace, cudaStream_t stream,
                            int fused_offset_mask, const float *epi_scale, const float *epi_shift, int relu) {
  const DcnShapeTc s = call_shape(p, fused_offset_mask, offset, &mask, epi_scale, epi_shift, relu);
  const float *xsrc;
  const int rc = fwd_source<Tf32x3>(p, p.fwd, s, input, false, workspace, stream, &xsrc);
  if (rc != CNB_OK) return rc;
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.fwd.part);
  return run_fwd<Tf32x3, float, false>(xsrc, offset, mask, wtiles, bias, output, part, s, OmArgs{}, stream);
}

int dcn_forward_bf16(const DcnPlan &p, const void *input, bool in_bf16, const float *offset, const float *mask,
                     const void *wtiles, const float *bias, void *output, bool out_bf16, void *workspace,
                     cudaStream_t stream, int fused_offset_mask, const float *epi_scale, const float *epi_shift,
                     int relu) {
  const DcnShapeTc s = call_shape(p, fused_offset_mask, offset, &mask, epi_scale, epi_shift, relu);
  const __nv_bfloat16 *xsrc;
  const int rc = fwd_source<Bf16>(p, p.bf16, s, input, in_bf16, workspace, stream, &xsrc);
  if (rc != CNB_OK) return rc;
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.bf16.part);
  return out_bf16 ? run_fwd<Bf16, __nv_bfloat16, false>(xsrc, offset, mask, wtiles, bias, output, part, s, OmArgs{},
                                                        stream)
                  : run_fwd<Bf16, float, false>(xsrc, offset, mask, wtiles, bias, output, part, s, OmArgs{}, stream);
}

int dcn_forward_block_bf16(const DcnPlan &p, const void *input, bool in_bf16, const void *om_tiles,
                           const float *om_bias, const void *wtiles, const float *bias, void *output,
                           void *workspace, cudaStream_t stream, const float *epi_scale, const float *epi_shift,
                           int relu) {
  const float *mask = nullptr;
  DcnShapeTc s = call_shape(p, 0, nullptr, &mask, epi_scale, epi_shift, relu);
  s.mask_logit = 1;   // the last 9 of the 27 offset-conv channels are mask logits
  const __nv_bfloat16 *xsrc;
  const int rc = fwd_source<Bf16>(p, p.bf16, s, input, in_bf16, workspace, stream, &xsrc);
  if (rc != CNB_OK) return rc;
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.bf16.part);
  OmArgs om;
  const CUresult cr = encode_halo_map(&om.xmap, xsrc, s.B, s.Cin, s.H, s.W, s.tw + 2, s.th + 2);
  CNB_REQUIRE(cr == CUDA_SUCCESS, CNB_ECUDA, "cnb_dcnv2_forward_block_bf16: cuTensorMapEncodeTiled failed (%d)",
              (int)cr);
  om.womt = reinterpret_cast<const __nv_bfloat16 *>(om_tiles);
  om.bom = om_bias;
  return in_bf16 ? run_fwd<Bf16, __nv_bfloat16, true>(xsrc, nullptr, nullptr, wtiles, bias, output, part, s, om, stream)
                 : run_fwd<Bf16, float, true>(xsrc, nullptr, nullptr, wtiles, bias, output, part, s, om, stream);
}

// Workspace of one forward format: channels-last copy of the input (+ split-K partial sums); the plain fp32 forward
// puts the weight tiles in front of it
template <typename F>
static void plan_fwd(const DcnShapeTc &s, DcnFwdLayout &l) {
  const size_t part_bytes = s.splits > 1 ? align_up((size_t)s.splits * s.B * s.Cout * s.Ho * s.Wo * 4, 256) : 0;
  l.xt = 0;
  l.xt_bytes = align_up((size_t)s.B * s.H * s.W * s.nb * TC_CB * sizeof(typename F::X), 256);
  l.part = l.xt + l.xt_bytes;
  l.prepared_bytes = l.part + part_bytes;
  l.wtiles_bytes = align_up((size_t)s.n_cot * s.nb * TC_NT * s.co_t * TC_K * F::ELEM, 256);
  l.bytes = l.wtiles_bytes + l.prepared_bytes;
}

void plan_forward_tc(DcnPlan *p) {
  plan_fwd<Tf32x3>(p->s, p->fwd);
  plan_fwd<Bf16>(p->s, p->bf16);
}

}  // namespace cnb
