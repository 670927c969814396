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
#include "dcnv2_tc.cuh"

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
          for (int idx = st; idx < TC_NT * TC_TP; idx += TC_SAMPLERS * 32) {
            const int t = idx / TC_TP, pp = idx - t * TC_TP;
            const int ho = it.ty0 + pp / s.tw, wo = it.tx0 + pp % s.tw;
            TapMetaTc mt;
#pragma unroll
            for (int q = 0; q < 4; ++q) { mt.o[q] = 0; mt.w[q] = 0.f; }
            if (ho < s.Ho && wo < s.Wo && t < KT) {
              const long long p = (long long)ho * s.Wo + wo;
              const int i = t / s.kw, j = t - i * s.kw;
              const float *op = offset + (long long)it.b * s.off_bs + (long long)g * 2 * KT * HWo;
              const float dy = __ldg(op + (2 * t) * HWo + p), dx = __ldg(op + (2 * t + 1) * HWo + p);
              float m = __ldg(mask + (long long)it.b * s.mask_bs + ((long long)g * KT + t) * HWo + p);
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

// Workspace of the prepared forward: channels-last copy of the input (+ split-K partial sums); the plain forward puts
// the weight tiles in front of it
void plan_forward_tc(DcnPlan *p) {
  const DcnShapeTc &s = p->s;
  p->xt_bytes = align_up((size_t)s.B * s.H * s.W * s.nb * TC_CB * 4, 256);
  p->fwd.xt = 0;
  p->fwd.part = p->fwd.xt + p->xt_bytes;
  p->fwd.prepared_bytes = p->fwd.part;
  if (s.splits > 1) p->fwd.prepared_bytes += align_up((size_t)s.splits * s.B * s.Cout * s.Ho * s.Wo * 4, 256);
  p->fwd.wtiles_bytes = align_up((size_t)s.n_cot * s.nb * TC_NT * 2 * s.co_t * TC_K * 4, 256);
  p->fwd.bytes = p->fwd.wtiles_bytes + p->fwd.prepared_bytes;
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
