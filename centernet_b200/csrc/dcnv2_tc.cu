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
// k_dcn_forward_bf16 (further down) is the opt-in bf16 form of the forward: bf16 tiles, wgmma k16 bf16 -> fp32.
// Its OM variant (the DCN block) also computes the 3x3 conv_offset_mask inside the kernel.
#include <cuda_bf16.h>

#include "halo.cuh"

namespace cnb {

// W[Cout][Cin][KT] -> per (cout tile, channel block bi, tap): hi tile then lo tile, each [co_t][32] in the K-major
// layout; k = channel within the block.  Tile index = (cot * nb + bi) * 9 + tap.
__global__ void __launch_bounds__(256) k_dcn_prep_weights(const float *__restrict__ w, const DcnShapeTc s,
                                                          float *__restrict__ ws) {
  const int KT = s.kh * s.kw;
  const int cpg = s.Cin / s.dg;
  const int tile = blockIdx.x;
  const int tap = tile % TC_NT, r = tile / TC_NT;
  const int bi = r % s.nb, cot = r / s.nb;
  const int g = bi / s.cbs_pg, cbi = bi - g * s.cbs_pg;
  const size_t tile_floats = (size_t)s.co_t * TC_K;
  unsigned char *hi = reinterpret_cast<unsigned char *>(ws + (size_t)tile * 2 * tile_floats);
  unsigned char *lo = hi + tile_floats * 4;
  for (int i = threadIdx.x; i < s.co_t * TC_K; i += blockDim.x) {
    const int o = i / TC_K, k = i - o * TC_K;
    const int cw = cbi * TC_CB + k;                    // channel within the group
    float v = 0.f;
    const int oc = cot * s.co_t + o;
    if (oc < s.Cout && cw < cpg && tap < KT) v = w[((size_t)oc * s.Cin + g * cpg + cw) * KT + tap];
    const float h = tf32_hi(v);
    *reinterpret_cast<float *>(hi + tc_tile_off(o, k)) = h;
    *reinterpret_cast<float *>(lo + tc_tile_off(o, k)) = v - h;
  }
}

// x [B][Cin][HW] -> xt [B][HW][nb][32]; channel ch of group g sits in block g*cbs_pg + (ch - g*cpg)/32,
// slot (ch - g*cpg) % 32 (identity when Cin/dg is a multiple of 32; pad slots are zero-filled by the caller).
// grid (pixel blocks of 32, channel blocks of 64, B), 256 threads.
__global__ void __launch_bounds__(256) k_dcn_nhwc(const float *__restrict__ x, float *__restrict__ xt,
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
      if (c0 + c < s.Cin && p0 + px < HW) v = __ldg(x + ((long long)b * s.Cin + c0 + c) * HW + p0 + px);
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
        if (p0 + px < HW) xt[((long long)b * HW + p0 + px) * Cp + slot] = tile[c][px];
    }
  }
}

// y[b][o][p] = bias[o] + sum_s part[s][b][o][p], s ascending (deterministic split-K epilogue)
__global__ void __launch_bounds__(256) k_dcn_reduce(const float *__restrict__ part, const float *__restrict__ bias,
                                                    float *__restrict__ y, int splits, int cout, long long hwo,
                                                    long long total, const float *__restrict__ epi_scale,
                                                    const float *__restrict__ epi_shift, int relu) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)((i / hwo) % cout);
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += __ldg(part + (long long)s * total + i);
    if (bias) v += __ldg(bias + o);
    if (epi_scale) v = fmaf(v, __ldg(epi_scale + o), __ldg(epi_shift + o));
    if (relu) v = fmaxf(v, 0.f);
    y[i] = v;
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
    TapMetaTc mt;
#pragma unroll
    for (int q = 0; q < 4; ++q) { mt.o[q] = 0; mt.w[q] = 0.f; }
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

template <int CO_T, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_dcn_forward_tc(const float *__restrict__ xt, const float *__restrict__ offset, const float *__restrict__ mask,
                 const float *__restrict__ wtiles, const float *__restrict__ bias, float *__restrict__ y,
                 float *__restrict__ part, const DcnShapeTc s) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  constexpr int B_BYTES = CO_T * TC_K * 4;                  // one hi or lo weight tile
  constexpr int STAGE_BYTES = 2 * FW_A_BYTES + 2 * B_BYTES;
  TapMetaTc *meta = reinterpret_cast<TapMetaTc *>(tc_smem + (size_t)STAGES * STAGE_BYTES);     // [9][128]
  __shared__ __align__(8) uint64_t a_full[STAGES], b_full[STAGES], empty[STAGES];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KT = s.kh * s.kw;
  const long long HWo = (long long)s.Ho * s.Wo, HW = (long long)s.H * s.W;
  const int Cp = s.nb * TC_CB;       // channel pitch of the channels-last copy

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&a_full[i], TC_SAMPLERS);
      mbar_init(&b_full[i], 1);
      mbar_init(&empty[i], TC_MMA_WGS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= TC_WARP_S0) {
    // =========================================================== samplers: A operand of every chunk
    const int sw = warp - TC_WARP_S0, st = tid - TC_WARP_S0 * 32;
    const int sp = lane >> 3, sq = lane & 7;
    int stage = 0, ph = 0;
    for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
      const ItemTc it = tc_item(s, item);
      const float *xbat = xt + (long long)it.b * HW * Cp + sq * 4;
      int cur_g = -1;
      for (int bi = it.b0; bi < it.b1; ++bi) {
        const int g = bi / s.cbs_pg;
        if (g != cur_g) {
          // ---- bilinear geometry of every (tap, pixel) of this deformable group (mask folded into the weights)
          cur_g = g;
          named_bar_sync(1, TC_SAMPLERS * 32);   // everybody is done reading the previous geometry
          tc_build_meta(s, offset, mask, it, g, st, KT, HWo, meta);
          named_bar_sync(1, TC_SAMPLERS * 32);
        }
        const float *xb = xbat + (long long)bi * TC_CB;
        for (int tap = 0; tap < TC_NT; ++tap) {
          // warp item = 4 pixels: every lane gathers the 4 corners of its pixel as 16-byte pieces (4 channels);
          // a warp fills TC_SAMPLER_ROUNDS 8-pixel row groups, one after the other; both items of a group (pixels
          // 8r..8r+3 and 8r+4..8r+7) are gathered before either is reduced
#pragma unroll 1
          for (int rnd = 0; rnd < TC_SAMPLER_ROUNDS; ++rnd) {
          const int rgp = sw * TC_SAMPLER_ROUNDS + rnd;
          const int pp0 = rgp * 8 + sp, pp1 = pp0 + 4;
          const TapMetaTc m0 = meta[tap * TC_TP + pp0], m1 = meta[tap * TC_TP + pp1];
          float4 u0[4], u1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) u0[q] = __ldg(reinterpret_cast<const float4 *>(xb + (long long)m0.o[q] * Cp));
#pragma unroll
          for (int q = 0; q < 4; ++q) u1[q] = __ldg(reinterpret_cast<const float4 *>(xb + (long long)m1.o[q] * Cp));
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
      int stage = 0, ph = 0;
      for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
        const ItemTc it = tc_item(s, item);
        for (int bi = it.b0; bi < it.b1; ++bi) {
          for (int tap = 0; tap < TC_NT; ++tap) {
            mbar_wait(&empty[stage], (uint32_t)(ph ^ 1));
            unsigned char *b_hi = tc_smem + (size_t)stage * STAGE_BYTES + 2 * FW_A_BYTES;
            const float *src = wtiles + (((size_t)it.cot * s.nb + bi) * TC_NT + tap) * 2 * (size_t)CO_T * TC_K;
            mbar_expect_tx(&b_full[stage], 2u * B_BYTES);
            for (uint32_t off = 0; off < 2u * B_BYTES; off += 8192u)
              bulk_g2s(b_hi + off, reinterpret_cast<const unsigned char *>(src) + off, 8192u, &b_full[stage]);
            if (++stage == STAGES) { stage = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    // =========================================================== consumers: wgmma over the ring, epilogue from registers
    const int wgi = warp >> 2, wq = warp & 3;
    int stage = 0, ph = 0;
    for (int item = blockIdx.x; item < s.n_items; item += gridDim.x) {
      const ItemTc it = tc_item(s, item);
      float d[CO_T / 2];
#pragma unroll
      for (int i = 0; i < CO_T / 2; ++i) d[i] = 0.f;
      const int n_ch = (it.b1 - it.b0) * TC_NT;
      for (int ch = 0; ch < n_ch; ++ch) {
        mbar_wait(&a_full[stage], (uint32_t)ph);
        mbar_wait(&b_full[stage], (uint32_t)ph);
        const uint32_t base = smem_u32(tc_smem + (size_t)stage * STAGE_BYTES);
        const uint32_t ah = base + (uint32_t)wgi * 8u * FW_SBO, al = ah + FW_A_BYTES;   // this warpgroup's 64 rows
        const uint32_t bh = base + 2u * FW_A_BYTES, bl = bh + B_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TC_K / 8; ++ks) {   // one k8 step = two 16-byte k-chunks
          const uint32_t koff = (uint32_t)ks * 2u * TC_LBO, koff_a = (uint32_t)ks * 2u * FW_LBO;
          wgmma_3xtf32<CO_T>(d, fw_desc_a(ah + koff_a), fw_desc_a(al + koff_a), tc_desc(bh + koff), tc_desc(bl + koff),
                             (ch > 0 || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();          // the slot is read: hand it back to the samplers and the TMA warp
        if ((tid & 127) == 0) mbar_arrive_tc(&empty[stage]);
        if (++stage == STAGES) { stage = 0; ph ^= 1; }
      }
      // epilogue: d[4j + r] = (row wq*16 + lane/4 + 8*(r/2), column 8j + 2*(lane%4) + r%2) of this warpgroup's 64 rows
      float *dst = (s.splits > 1 ? part + (long long)it.split * s.B * s.Cout * HWo : y) + (long long)it.b * s.Cout * HWo;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pp = wgi * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int ho = it.ty0 + pp / s.tw, wo = it.tx0 + pp % s.tw;
        if (ho >= s.Ho || wo >= s.Wo) continue;
        float *dp = dst + (long long)ho * s.Wo + wo;
#pragma unroll
        for (int j = 0; j < CO_T / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int o = it.cot * CO_T + 8 * j + 2 * (lane & 3) + e;
            if (o < s.Cout) {
              float r = d[4 * j + 2 * h + e];
              if (s.splits == 1) {
                if (bias) r += __ldg(bias + o);
                if (s.epi_scale) r = fmaf(r, __ldg(s.epi_scale + o), __ldg(s.epi_shift + o));
                if (s.relu) r = fmaxf(r, 0.f);
              }
              dp[(long long)o * HWo] = r;
            }
          }
        }
      }
    }
  }
}

// =====================================================================================================================
// bf16 forward: the same pipeline with one bf16 A tile and one bf16 B tile a chunk and wgmma k16 bf16 -> fp32.
// Numeric contract (include/centernet_b200.h): the geometry and the 4-corner interpolation are the fp32 kernel's
// (tc_build_meta, the same fmaf chain), the masked column value is rounded once to bf16 (RN); the weights were
// rounded once (RN) by k_dcn_prep_weights_bf16; the contraction accumulates in fp32, split-K partials are added in
// split order, bias / BN / ReLU are applied in fp32 and the result is stored as fp32 or rounded (RN) to bf16.

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {   // lo -> lower address (smaller k)
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&v);
}
__device__ __forceinline__ void store_out(float *p, float v) { *p = v; }
__device__ __forceinline__ void store_out(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ float load_in(const float *p) { return __ldg(p); }
__device__ __forceinline__ float load_in(const __nv_bfloat16 *p) { return __bfloat162float(p[0]); }

// W[Cout][Cin][KT] (fp32) -> per (cout tile, channel block, tap) one bf16 tile [co_t][32] (k = channel within the
// block), the layout of bf_tile_off; tile index = (cot * nb + bi) * 9 + tap, as k_dcn_prep_weights
__global__ void __launch_bounds__(256) k_dcn_prep_weights_bf16(const float *__restrict__ w, const DcnShapeTc s,
                                                               unsigned char *__restrict__ ws) {
  const int KT = s.kh * s.kw;
  const int cpg = s.Cin / s.dg;
  const int tile = blockIdx.x;
  const int tap = tile % TC_NT, r = tile / TC_NT;
  const int bi = r % s.nb, cot = r / s.nb;
  const int g = bi / s.cbs_pg, cbi = bi - g * s.cbs_pg;
  unsigned char *dst = ws + (size_t)tile * s.co_t * TC_K * 2;
  for (int i = threadIdx.x; i < s.co_t * TC_K; i += blockDim.x) {
    const int o = i / TC_K, k = i - o * TC_K;
    const int cw = cbi * TC_CB + k;
    const int oc = cot * s.co_t + o;
    float v = 0.f;
    if (oc < s.Cout && cw < cpg && tap < KT) v = w[((size_t)oc * s.Cin + g * cpg + cw) * KT + tap];
    *reinterpret_cast<__nv_bfloat16 *>(dst + bf_tile_off(o, k)) = __float2bfloat16_rn(v);
  }
}

// x [B][Cin][HW] (fp32 or bf16) -> bf16 xt [B][HW][nb][32], the slot mapping of k_dcn_nhwc
template <typename T>
__global__ void __launch_bounds__(256) k_dcn_nhwc_bf16(const T *__restrict__ x, __nv_bfloat16 *__restrict__ xt,
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
        if (p0 + px < HW) xt[((long long)b * HW + p0 + px) * Cp + slot] = __float2bfloat16_rn(tile[c][px]);
    }
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

// bf16 x [B][Cin][HW] -> fp32 xt [B][HW][nb][32] (exact widening): k_dcn_nhwc reading bf16, for the bf16 backward
__global__ void __launch_bounds__(256) k_dcn_nhwc_widen(const __nv_bfloat16 *__restrict__ x, float *__restrict__ xt,
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
        if (p0 + px < HW) xt[((long long)b * HW + p0 + px) * Cp + slot] = tile[c][px];
    }
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

// y[b][o][p] = epilogue(bias[o] + sum_s part[s][b][o][p]), s ascending, stored as bf16 (k_dcn_reduce writes fp32)
__global__ void __launch_bounds__(256) k_dcn_reduce_bf16(const float *__restrict__ part, const float *__restrict__ bias,
                                                         __nv_bfloat16 *__restrict__ y, int splits, int cout,
                                                         long long hwo, long long total,
                                                         const float *__restrict__ epi_scale,
                                                         const float *__restrict__ epi_shift, int relu) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)((i / hwo) % cout);
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += __ldg(part + (long long)s * total + i);
    if (bias) v += __ldg(bias + o);
    if (epi_scale) v = fmaf(v, __ldg(epi_scale + o), __ldg(epi_shift + o));
    if (relu) v = fmaxf(v, 0.f);
    y[i] = __float2bfloat16_rn(v);
  }
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

// Warp roles, items and mbarrier hand-over as k_dcn_forward_tc.  Sampler warp item = one 8-row group of the A tile
// (8 pixels): lane = pixel * 4 + k-chunk, every lane gathers the 4 corners of its pixel as 16-byte pieces (8 bf16
// channels), interpolates in fp32 and stores one rounded 16-byte k-chunk; each warp fills two row groups a chunk, both
// gathered before either is reduced.
template <int CO_T, int STAGES, typename TOut, bool OM>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_dcn_forward_bf16(const __nv_bfloat16 *__restrict__ xt, const float *__restrict__ offset,
                   const float *__restrict__ mask, const __nv_bfloat16 *__restrict__ wtiles,
                   const float *__restrict__ bias, TOut *__restrict__ y, float *__restrict__ part, const DcnShapeTc s,
                   const __grid_constant__ CUtensorMap xmap, const __nv_bfloat16 *__restrict__ womt,
                   const float *__restrict__ bom) {
  extern __shared__ __align__(128) unsigned char tc_smem_raw[];
  // the block variant's TMA halo needs a 128-byte aligned destination
  unsigned char *tc_smem = OM ? tc_smem_raw + ((128u - (smem_u32(tc_smem_raw) & 127u)) & 127u) : tc_smem_raw;
  constexpr int B_BYTES = CO_T * TC_K * 2;
  constexpr int STAGE_BYTES = BF_A_BYTES + B_BYTES;
  constexpr int ROWGROUPS = TC_TP / 8 / TC_SAMPLERS;   // 2 row groups a sampler warp
  static_assert(ROWGROUPS == 2, "k_dcn_forward_bf16: two row groups a sampler warp");
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
    const int sw = warp - TC_WARP_S0, st = tid - TC_WARP_S0 * 32;
    const int sp = lane >> 2, sq = lane & 3;
    const int rg0 = sw * ROWGROUPS, rg1 = rg0 + 1;
    int stage = 0, ph = 0, n = 0;
    for (int item = blockIdx.x; item < s.n_items; item += gridDim.x, ++n) {
      const ItemTc it = tc_item(s, item);
      const __nv_bfloat16 *xbat = xt + (long long)it.b * HW * Cp + sq * 8;
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
        const __nv_bfloat16 *xb = xbat + (long long)bi * TC_CB;
        for (int tap = 0; tap < TC_NT; ++tap) {
          const TapMetaTc m0 = meta[tap * TC_TP + rg0 * 8 + sp], m1 = meta[tap * TC_TP + rg1 * 8 + sp];
          uint4 u0[4], u1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) u0[q] = __ldg(reinterpret_cast<const uint4 *>(xb + (long long)m0.o[q] * Cp));
#pragma unroll
          for (int q = 0; q < 4; ++q) u1[q] = __ldg(reinterpret_cast<const uint4 *>(xb + (long long)m1.o[q] * Cp));
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
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> async proxy (wgmma reads)
          __syncwarp();
          if (lane == 0) mbar_arrive_tc(&a_full[stage]);
          if (++stage == STAGES) { stage = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp == TC_WARP_TMA) {
    // =========================================================== B operand: one bf16 weight tile by TMA bulk copy
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
            unsigned char *b = tc_smem + (size_t)stage * STAGE_BYTES + BF_A_BYTES;
            const __nv_bfloat16 *src = wtiles + (((size_t)it.cot * s.nb + bi) * TC_NT + tap) * (size_t)CO_T * TC_K;
            mbar_expect_tx(&b_full[stage], (uint32_t)B_BYTES);
            bulk_g2s(b, src, (uint32_t)B_BYTES, &b_full[stage]);
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
            wgmma_ss<OM_N>(q, wg_desc(a + (uint32_t)ks * 2u * OM_SLAB_PITCH, OM_SLAB_PITCH, hx16),
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
        const uint32_t a = base + (uint32_t)wgi * 8u * BF_SBO;   // this warpgroup's 64 rows
        const uint32_t b = base + (uint32_t)BF_A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < TC_K / 16; ++ks)   // one k16 step = two 16-byte k-chunks
          wgmma_bf16<CO_T>(d, wg_desc(a + (uint32_t)ks * 2u * BF_LBO, BF_LBO, BF_SBO),
                           wg_desc(b + (uint32_t)ks * 2u * BF_B_LBO, BF_B_LBO, BF_B_SBO), (ch > 0 || ks > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        if ((tid & 127) == 0) mbar_arrive_tc(&empty[stage]);
        if (++stage == STAGES) { stage = 0; ph ^= 1; }
      }
      // epilogue: the accumulator fragment of k_dcn_forward_tc; split-K partials stay fp32
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
                if (s.relu) r = fmaxf(r, 0.f);
                store_out(ydst + (long long)o * HWo + p, r);
              }
            }
          }
        }
      }
    }
  }
}

int dcn_prepare_weights_bf16(const float *weight, int cin, int cout, int kh, int kw, int dg, void *wtiles,
                             cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg);
  k_dcn_prep_weights_bf16<<<s.n_cot * s.nb * TC_NT, 256, 0, stream>>>(weight, s,
                                                                       reinterpret_cast<unsigned char *>(wtiles));
  CNB_CHECK_LAUNCH("cnb_dcnv2 bf16 weight tiles");
  count_launch();
  return CNB_OK;
}

// W_om [27][Cin][3][3] (fp32) -> per channel block nine bf16 tiles [32][32] (rows 27..31 zero), tile index bi * 9 + tap:
// k_dcn_prep_weights_bf16 with one Cout tile of 32 rows
int dcn_prepare_om_weights_bf16(const float *w_om, int cin, void *om_tiles, cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, OM_C, 3, 3, 1, 1, 1, 1, 1, 1, 1);
  s.co_t = OM_N;
  s.n_cot = 1;
  k_dcn_prep_weights_bf16<<<s.nb * TC_NT, 256, 0, stream>>>(w_om, s, reinterpret_cast<unsigned char *>(om_tiles));
  CNB_CHECK_LAUNCH("cnb_dcnv2 bf16 offset-conv weight tiles");
  count_launch();
  return CNB_OK;
}

size_t dcn_om_tiles_bytes(int cin) { return (size_t)(cin / TC_CB) * OM_W_BYTES; }

// The operands of the block variant (OM); the plain bf16 forward passes none
struct OmArgs {
  CUtensorMap xmap;
  const __nv_bfloat16 *womt;
  const float *bom;
};

template <int CO_T, typename TOut, bool OM>
static int launch_fwd_bf16(const __nv_bfloat16 *xt, const float *offset, const float *mask, const void *wtiles,
                           const float *bias, void *output, float *part, const DcnShapeTc &s, const OmArgs &om,
                           cudaStream_t stream) {
  constexpr int STAGES = BF_STAGES;
  const size_t smem = (size_t)STAGES * (BF_A_BYTES + CO_T * TC_K * 2) + sizeof(TapMetaTc) * TC_NT * TC_TP +
                      (OM ? OM_SMEM_BYTES : 0);
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_forward_bf16<CO_T, STAGES, TOut, OM>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dev_done = dev;
  }
  const int grid = s.n_items < num_sms() ? s.n_items : num_sms();
  k_dcn_forward_bf16<CO_T, STAGES, TOut, OM><<<grid, TC_THREADS, smem, stream>>>(
      xt, offset, mask, reinterpret_cast<const __nv_bfloat16 *>(wtiles), bias, reinterpret_cast<TOut *>(output), part,
      s, om.xmap, om.womt, om.bom);
  CNB_CHECK_LAUNCH(OM ? "cnb_dcnv2_forward_block_bf16 (wgmma)" : "cnb_dcnv2_forward_bf16 (wgmma)");
  count_launch();
  return CNB_OK;
}

// The bf16 channels-last source [B][HW][nb][32] the kernel samples: a bf16 channels-last input in place, else a copy
// into the workspace (p.bf16.xt)
static int bf16_source(const DcnPlan &p, const DcnShapeTc &s, const void *input, bool in_bf16, void *workspace,
                       cudaStream_t stream, const __nv_bfloat16 **xsrc) {
  __nv_bfloat16 *xt = reinterpret_cast<__nv_bfloat16 *>(reinterpret_cast<char *>(workspace) + p.bf16.xt);
  const long long HW = (long long)s.H * s.W;
  *xsrc = xt;
  if (p.x_cl && in_bf16) {
    *xsrc = reinterpret_cast<const __nv_bfloat16 *>(input);   // sampled in place
  } else if (p.x_cl) {
    const long long n8 = (long long)s.B * HW * s.Cin / 8;
    const int grid = (int)((n8 + 255) / 256 < 4096 ? (n8 + 255) / 256 : 4096);
    k_dcn_cl_to_bf16<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4 *>(input), reinterpret_cast<uint4 *>(xt), n8);
    CNB_CHECK_LAUNCH("cnb_dcnv2_forward_bf16 bf16 copy");
    count_launch();
  } else {
    if ((s.Cin / s.dg) % TC_CB != 0)   // pad slots of the last channel block of every group must read as zero
      CNB_CUDA(cudaMemsetAsync(xt, 0, (size_t)s.B * HW * s.nb * TC_CB * 2, stream));
    dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((s.Cin + 63) / 64), (unsigned)s.B);
    if (in_bf16)
      k_dcn_nhwc_bf16<__nv_bfloat16><<<tgrid, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16 *>(input), xt, s);
    else
      k_dcn_nhwc_bf16<float><<<tgrid, 256, 0, stream>>>(reinterpret_cast<const float *>(input), xt, s);
    CNB_CHECK_LAUNCH("cnb_dcnv2_forward_bf16 channels-last copy");
    count_launch();
  }
  return CNB_OK;
}

// The kernel for the Cout tile and output dtype, then the split-K reduce on small maps
template <bool OM>
static int run_fwd_bf16(const __nv_bfloat16 *xsrc, const float *offset, const float *mask, const void *wtiles,
                        const float *bias, void *output, bool out_bf16, float *part, const DcnShapeTc &s,
                        const OmArgs &om, cudaStream_t stream) {
  int rc;
  if (s.co_t == 64)
    rc = out_bf16 ? launch_fwd_bf16<64, __nv_bfloat16, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream)
                  : launch_fwd_bf16<64, float, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream);
  else
    rc = out_bf16 ? launch_fwd_bf16<128, __nv_bfloat16, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream)
                  : launch_fwd_bf16<128, float, OM>(xsrc, offset, mask, wtiles, bias, output, part, s, om, stream);
  if (rc != CNB_OK) return rc;
  if (s.splits > 1) {
    const long long total = (long long)s.B * s.Cout * s.Ho * s.Wo;
    const int grid = (int)((total + 255) / 256 < 1184 ? (total + 255) / 256 : 1184);
    if (out_bf16)
      k_dcn_reduce_bf16<<<grid, 256, 0, stream>>>(part, bias, reinterpret_cast<__nv_bfloat16 *>(output), s.splits,
                                                  s.Cout, (long long)s.Ho * s.Wo, total, s.epi_scale, s.epi_shift,
                                                  s.relu);
    else
      k_dcn_reduce<<<grid, 256, 0, stream>>>(part, bias, reinterpret_cast<float *>(output), s.splits, s.Cout,
                                             (long long)s.Ho * s.Wo, total, s.epi_scale, s.epi_shift, s.relu);
    CNB_CHECK_LAUNCH("cnb_dcnv2_forward_bf16 split-K reduce");
    count_launch();
  }
  return CNB_OK;
}

int dcn_forward_bf16(const DcnPlan &p, const void *input, bool in_bf16, const float *offset, const float *mask,
                     const void *wtiles, const float *bias, void *output, bool out_bf16, void *workspace,
                     cudaStream_t stream, int fused_offset_mask, const float *epi_scale, const float *epi_shift,
                     int relu) {
  DcnShapeTc s = p.s;
  if (fused_offset_mask) {   // `offset` is the raw [b, 3*kt*dg, ho, wo] output of conv_offset_mask; mask = its last third
    s.off_bs = s.mask_bs = (long long)s.dg * 3 * s.kh * s.kw * s.Ho * s.Wo;
    s.mask_logit = 1;
    mask = offset + (long long)s.dg * 2 * s.kh * s.kw * s.Ho * s.Wo;
  }
  s.epi_scale = epi_scale;
  s.epi_shift = epi_scale ? epi_shift : nullptr;
  s.relu = relu;
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.bf16.part);
  const __nv_bfloat16 *xsrc;
  const int rc = bf16_source(p, s, input, in_bf16, workspace, stream, &xsrc);
  if (rc != CNB_OK) return rc;
  OmArgs none;
  memset(&none, 0, sizeof(none));
  return run_fwd_bf16<false>(xsrc, offset, mask, wtiles, bias, output, out_bf16, part, s, none, stream);
}

int dcn_forward_block_bf16(const DcnPlan &p, const void *input, bool in_bf16, const void *om_tiles,
                           const float *om_bias, const void *wtiles, const float *bias, void *output,
                           void *workspace, cudaStream_t stream, const float *epi_scale, const float *epi_shift,
                           int relu) {
  DcnShapeTc s = p.s;
  s.mask_logit = 1;   // the last 9 of the 27 offset-conv channels are mask logits
  s.epi_scale = epi_scale;
  s.epi_shift = epi_scale ? epi_shift : nullptr;
  s.relu = relu;
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.bf16.part);
  const __nv_bfloat16 *xsrc;
  int rc = bf16_source(p, s, input, in_bf16, workspace, stream, &xsrc);
  if (rc != CNB_OK) return rc;
  OmArgs om;
  const CUresult cr = encode_halo_map(&om.xmap, xsrc, s.B, s.Cin, s.H, s.W, s.tw + 2, s.th + 2);
  CNB_REQUIRE(cr == CUDA_SUCCESS, CNB_ECUDA, "cnb_dcnv2_forward_block_bf16: cuTensorMapEncodeTiled failed (%d)",
              (int)cr);
  om.womt = reinterpret_cast<const __nv_bfloat16 *>(om_tiles);
  om.bom = om_bias;
  return run_fwd_bf16<true>(xsrc, nullptr, nullptr, wtiles, bias, output, in_bf16, part, s, om, stream);
}

// Workspace of the prepared forward: channels-last copy of the input (+ split-K partial sums); the plain forward puts
// the weight tiles in front of it.  The bf16 forward's workspace has the same regions with a bf16 copy.
void plan_forward_tc(DcnPlan *p) {
  const DcnShapeTc &s = p->s;
  const size_t part_bytes = s.splits > 1 ? align_up((size_t)s.splits * s.B * s.Cout * s.Ho * s.Wo * 4, 256) : 0;
  p->xt_bytes = align_up((size_t)s.B * s.H * s.W * s.nb * TC_CB * 4, 256);
  p->fwd.xt = 0;
  p->fwd.part = p->fwd.xt + p->xt_bytes;
  p->fwd.prepared_bytes = p->fwd.part + part_bytes;
  p->fwd.wtiles_bytes = align_up((size_t)s.n_cot * s.nb * TC_NT * 2 * s.co_t * TC_K * 4, 256);
  p->fwd.bytes = p->fwd.wtiles_bytes + p->fwd.prepared_bytes;
  p->bf16.xt = 0;
  p->bf16.xt_bytes = align_up((size_t)s.B * s.H * s.W * s.nb * TC_CB * 2, 256);
  p->bf16.part = p->bf16.xt + p->bf16.xt_bytes;
  p->bf16.bytes = p->bf16.part + part_bytes;
  p->bf16.wtiles_bytes = align_up((size_t)s.n_cot * s.nb * TC_NT * s.co_t * TC_K * 2, 256);
}

int dcn_prepare_weights_tc(const float *weight, int cin, int cout, int kh, int kw, int dg, float *wtiles,
                           cudaStream_t stream) {
  DcnShapeTc s;
  fill_shape(&s, 1, cin, 8, 8, cout, kh, kw, 1, 1, 1, 1, 1, 1, dg);
  k_dcn_prep_weights<<<s.n_cot * s.nb * TC_NT, 256, 0, stream>>>(weight, s, wtiles);
  CNB_CHECK_LAUNCH("cnb_dcnv2 weight tiles");
  count_launch();
  return CNB_OK;
}

int dcn_to_channels_last(const float *x, float *xt, const DcnShapeTc &s, cudaStream_t stream) {
  const long long HW = (long long)s.H * s.W;
  if ((s.Cin / s.dg) % TC_CB != 0)   // pad slots of the last channel block of every group must read as zero
    CNB_CUDA(cudaMemsetAsync(xt, 0, (size_t)s.B * HW * s.nb * TC_CB * 4, stream));
  dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((s.Cin + 63) / 64), (unsigned)s.B);
  k_dcn_nhwc<<<tgrid, 256, 0, stream>>>(x, xt, s);
  CNB_CHECK_LAUNCH("cnb_dcnv2 channels-last copy");
  count_launch();
  return CNB_OK;
}

int dcn_to_channels_last(const __nv_bfloat16 *x, bool x_cl, float *xt, const DcnShapeTc &s, cudaStream_t stream) {
  const long long HW = (long long)s.H * s.W;
  if (x_cl) {
    const long long n8 = (long long)s.B * HW * s.Cin / 8;
    const int grid = (int)((n8 + 255) / 256 < 4096 ? (n8 + 255) / 256 : 4096);
    k_dcn_cl_widen<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint4 *>(x), reinterpret_cast<float4 *>(xt), n8);
    CNB_CHECK_LAUNCH("cnb_dcnv2 channels-last fp32 copy of a bf16 input");
    count_launch();
    return CNB_OK;
  }
  if ((s.Cin / s.dg) % TC_CB != 0)
    CNB_CUDA(cudaMemsetAsync(xt, 0, (size_t)s.B * HW * s.nb * TC_CB * 4, stream));
  dim3 tgrid((unsigned)((HW + 31) / 32), (unsigned)((s.Cin + 63) / 64), (unsigned)s.B);
  k_dcn_nhwc_widen<<<tgrid, 256, 0, stream>>>(x, xt, s);
  CNB_CHECK_LAUNCH("cnb_dcnv2 channels-last fp32 copy of a bf16 input");
  count_launch();
  return CNB_OK;
}

template <int CO_T, int STAGES>
static int launch_fwd(const float *xt, const float *offset, const float *mask, const float *wtiles, const float *bias,
                      float *output, float *part, const DcnShapeTc &s, cudaStream_t stream) {
  const size_t smem = (size_t)STAGES * (2 * FW_A_BYTES + 2 * CO_T * TC_K * 4) + sizeof(TapMetaTc) * TC_NT * TC_TP;
  static thread_local int dev_done = -1;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev_done != dev) {
    CNB_CUDA(cudaFuncSetAttribute(k_dcn_forward_tc<CO_T, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dev_done = dev;
  }
  const int grid = s.n_items < num_sms() ? s.n_items : num_sms();
  k_dcn_forward_tc<CO_T, STAGES><<<grid, TC_THREADS, smem, stream>>>(xt, offset, mask, wtiles, bias, output, part, s);
  CNB_CHECK_LAUNCH("cnb_dcnv2_forward (wgmma)");
  count_launch();
  return CNB_OK;
}

// Tensor-core forward from pre-tiled weights.  p.x_cl: `input` already is [B][H*W][Cin] (torch channels_last) with
// Cin/dg a multiple of 32 -- no re-layout pass.
int dcn_forward_tc_prepared(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                            const float *wtiles, const float *bias, float *output, void *workspace, cudaStream_t stream,
                            int fused_offset_mask, const float *epi_scale, const float *epi_shift, int relu) {
  DcnShapeTc s = p.s;
  if (fused_offset_mask) {   // `offset` is the raw [b, 3*kt*dg, ho, wo] output of conv_offset_mask; mask = its last third
    s.off_bs = s.mask_bs = (long long)s.dg * 3 * s.kh * s.kw * s.Ho * s.Wo;
    s.mask_logit = 1;
    mask = offset + (long long)s.dg * 2 * s.kh * s.kw * s.Ho * s.Wo;
  }
  s.epi_scale = epi_scale;
  s.epi_shift = epi_scale ? epi_shift : nullptr;
  s.relu = relu;
  float *xt = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.fwd.xt);
  float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + p.fwd.part);
  const float *xsrc = xt;
  if (p.x_cl) {
    xsrc = input;
  } else {
    const int rc_t = dcn_to_channels_last(input, xt, s, stream);
    if (rc_t != CNB_OK) return rc_t;
  }
  int rc;
  if (s.co_t == 64) rc = launch_fwd<64, 3>(xsrc, offset, mask, wtiles, bias, output, part, s, stream);
  else rc = launch_fwd<128, 2>(xsrc, offset, mask, wtiles, bias, output, part, s, stream);
  if (rc != CNB_OK) return rc;
  if (s.splits > 1) {
    const long long total = (long long)s.B * s.Cout * s.Ho * s.Wo;
    const int grid = (int)((total + 255) / 256 < 1184 ? (total + 255) / 256 : 1184);
    k_dcn_reduce<<<grid, 256, 0, stream>>>(part, bias, output, s.splits, s.Cout, (long long)s.Ho * s.Wo, total,
                                           s.epi_scale, s.epi_shift, s.relu);
    CNB_CHECK_LAUNCH("cnb_dcnv2_forward split-K reduce");
    count_launch();
  }
  return CNB_OK;
}

}  // namespace cnb
