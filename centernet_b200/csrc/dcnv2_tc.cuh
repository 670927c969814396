// Shared by the wgmma DCNv2 kernels (dcnv2_tc.cu: forward, dcnv2_bwd_tc.cu: backward): the shared-memory tile
// layout (K-major, no swizzle), the wgmma descriptor and instruction wrappers and the shape / work decomposition.
#pragma once
#include "common.cuh"

namespace cnb {

constexpr int TC_TP = 128;        // pixels per item (two warpgroups x wgmma M = 64)
constexpr int TC_CB = 32;         // input channels per chunk = one 128-byte line of the channels-last copy
constexpr int TC_NT = 9;          // taps (3x3 kernel; fewer taps leave zero weight tiles)
constexpr int TC_K = TC_CB;       // K per chunk
constexpr int TC_KC = TC_K / 4;   // 16-byte k-chunks
constexpr int TC_MMA_WGS = 2;     // warps 0-7: two consumer warpgroups, warpgroup i owns rows 64i..64i+63 of the tile
constexpr int TC_WARP_TMA = 8;
constexpr int TC_WARP_S0 = 9;     // first sampler warp
constexpr int TC_SAMPLERS = 8;    // sampler warps of the forward: 2 rounds x 2 warp items (4 pixels each) per chunk
constexpr int TC_SAMPLER_ROUNDS = TC_TP / 8 / TC_SAMPLERS;
constexpr int TC_THREADS = (TC_WARP_S0 + TC_SAMPLERS) * 32;   // 544: the consumers hold up to 64 accumulators each
constexpr uint32_t TC_LBO = 128;            // bytes between consecutive k-chunks (one 8 x 16 B core matrix)
constexpr uint32_t TC_SBO = TC_KC * 128;    // bytes between 8-row groups (1024)
constexpr int TC_A_BYTES = TC_TP * TC_K * 4;  // 16384 per hi / lo tile

// A tile of the forward sampler: the same K-major core-matrix layout with the k-chunks pitched 144 bytes apart
constexpr uint32_t FW_LBO = 144;                    // bytes between consecutive k-chunks (8 rows x 16 B + 16 B of padding)
constexpr uint32_t FW_SBO = TC_KC * FW_LBO;         // bytes between 8-row groups (1152)
constexpr int FW_A_BYTES = (TC_TP / 8) * FW_SBO;    // 18432 per hi / lo tile

struct DcnShapeTc {
  int B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
  int co_t;       // output channels per item (64 or 128)
  int n_cot;      // Cout tiles
  int cbs_pg;     // 32-channel blocks per deformable group
  int nb;         // channel blocks in total = dg * cbs_pg
  int tw, th;     // pixel tile (tw * th == 128)
  int tiles_x, tiles_y;
  int splits;     // K splits (channel-block ranges) per item; > 1 -> partial sums + k_dcn_reduce
  int n_items;    // B * tiles * n_cot * splits
  // fused prologue / epilogue (N3, dcn_v2.py:64-70 + pose_dla_dcn.py:345-357)
  long long off_bs, mask_bs;   // batch strides (floats) of the offset / mask tensors
  int mask_logit;              // mask holds the raw conv_offset_mask output: sigmoid applied on the fly
  int relu;                    // epilogue: y = relu(scale[o] * (acc + bias[o]) + shift[o])
  const float *epi_scale, *epi_shift;   // folded inference BatchNorm (nullable)
};

struct __align__(16) TapMetaTc {
  int o[4];
  float w[4];
};

__device__ __forceinline__ uint32_t tc_tile_off(int row, int k) {  // byte offset of element (row, k) in a K-major tile
  return (uint32_t)(row >> 3) * TC_SBO + (uint32_t)(k >> 2) * TC_LBO + (uint32_t)(row & 7) * 16u + (uint32_t)(k & 3) * 4u;
}
// sm_90 shared-memory matrix descriptor: start address, leading (k-chunk) and stride (8-row group) byte offsets,
// base offset 0, layout type 0 = no swizzle
__device__ __forceinline__ uint64_t wg_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((addr >> 4) & 0x3fff) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}
__device__ __forceinline__ uint64_t tc_desc(uint32_t addr) { return wg_desc(addr, TC_LBO, TC_SBO); }
__device__ __forceinline__ uint64_t fw_desc_a(uint32_t addr) { return wg_desc(addr, FW_LBO, FW_SBO); }

// wgmma (warpgroup-wide, asynchronous): D[64 x N] (+)= A[64 x 8] . B[N x 8]^T in TF32, both operands K-major in
// shared memory, D in registers: d[4j + r] holds row (warp % 4) * 16 + lane / 4 + 8 * (r / 2), column
// 8j + 2 * (lane % 4) + r % 2.  scale_d == 0 overwrites D.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,"
      "%26,%27,%28,%29,%30,%31}"
      ", %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,"
      "%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,"
      "%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
      ", %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(N == 64 || N == 128, "wgmma_tf32: N is 64 or 128");
  if constexpr (N == 64) wgmma_tf32_n64(d, da, db, scale_d);
  else wgmma_tf32_n128(d, da, db, scale_d);
}
// 3xTF32 step of one 8-wide k slice: lo.hi + hi.lo + hi.hi (small terms first) -- fp32-accurate products
template <int N>
__device__ __forceinline__ void wgmma_3xtf32(float (&d)[N / 2], uint64_t dah, uint64_t dal, uint64_t dbh, uint64_t dbl,
                                             uint32_t scale_d) {
  wgmma_tf32<N>(d, dal, dbh, scale_d);
  wgmma_tf32<N>(d, dah, dbl, 1u);
  wgmma_tf32<N>(d, dah, dbh, 1u);
}
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ void mbar_arrive_tc(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

inline void fill_shape(DcnShapeTc *s, int b, int cin, int h, int w, int cout, int kh, int kw, int sh, int sw, int ph,
                       int pw, int dh, int dw, int dg) {
  s->B = b; s->Cin = cin; s->H = h; s->W = w; s->Cout = cout; s->kh = kh; s->kw = kw; s->sh = sh; s->sw = sw;
  s->ph = ph; s->pw = pw; s->dh = dh; s->dw = dw; s->dg = dg;
  s->Ho = (h + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
  s->Wo = (w + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
  s->co_t = cout > 64 ? 128 : 64;
  s->n_cot = (cout + s->co_t - 1) / s->co_t;
  const int cpg = cin / dg;
  s->cbs_pg = (cpg + TC_CB - 1) / TC_CB;
  s->nb = dg * s->cbs_pg;
  s->tw = s->Wo >= 12 ? 16 : 8;          // 8 x 16 pixel tiles; 16 x 8 on narrow maps
  s->th = TC_TP / s->tw;
  s->tiles_x = (s->Wo + s->tw - 1) / s->tw;
  s->tiles_y = (s->Ho + s->th - 1) / s->th;
  const long long base_items = (long long)b * s->tiles_x * s->tiles_y * s->n_cot;
  int splits = 1;
  const int sms = num_sms();
  if (base_items < sms) {                 // small maps: split the channel blocks so every SM gets an item
    splits = (int)((sms + base_items - 1) / base_items);
    if (splits > s->nb) splits = s->nb;
    if (splits > 8) splits = 8;
    if (splits < 1) splits = 1;
  }
  s->splits = splits;
  s->n_items = (int)(base_items * splits);
  s->off_bs = (long long)dg * 2 * kh * kw * s->Ho * s->Wo;
  s->mask_bs = (long long)dg * kh * kw * s->Ho * s->Wo;
  s->mask_logit = 0;
  s->relu = 0;
  s->epi_scale = s->epi_shift = nullptr;
}

// Host-side plan of one fp32 DCNv2 call or workspace query (dcn_plan in dcnv2.cu, after the one validation): the
// shape, the path decisions and the byte offset of every workspace region.  Each size and offset is worked out once,
// by plan_forward_tc and plan_backward_tc; the hosts of the kernels read their pointers from here.
struct DcnPlan {
  DcnShapeTc s;        // the validated shape and the tensor-core decomposition (fill_shape)
  bool det;            // deterministic mode (cnb_dcnv2_set_deterministic), read once per call
  bool fwd_tc;         // the tensor-core forward covers the shape: isotropic stride/pad/dilation
  bool bwd_tc;         // so does the tensor-core backward: isotropic and within its 32-bit in-image indexing
  bool dw_tc;          // and its weight pass: cout <= 256 (above, dW runs on the fp32 kernel)
  bool x_cl, gx_cl;    // input / grad_input are channels-last [b][h*w][cin] (whole 32-channel blocks) and used as such
  bool xt_ready;       // weight pass: the data pass already wrote the channels-last input copy on this stream
  int fp32_dw_splits;  // pixel-range splits of the fp32 dW kernel
  size_t xt_bytes;     // channels-last copy of the input [B][HW][nb][32], in both workspaces
  struct {             // the prepared forward's workspace is [xt][part]; the plain forward's is [wtiles][that], so the
                       // prepared one starts at wtiles_bytes there
    size_t xt, part, prepared_bytes, wtiles_bytes, bytes;
  } fwd;
  struct {             // [xt][dxt][wtt][max(gyt + dcol of one batch chunk, gyk + wpart + bpart)]: the data and the
                       // weight passes run one after the other on the stream and share the tail.  Deterministic mode
                       // appends [bnd][dxi] or, at the same offset and for cout > 256, the fp32 dW partials wpart32
    size_t xt, dxt, wtt, gyt, dcol, gyk, wpart, bpart, bnd, dxi, wpart32, bytes;
    int chunk;         // images per pass of the data pass
  } bwd;
};
void plan_forward_tc(DcnPlan *p);    // dcnv2_tc.cu: xt_bytes and fwd
void plan_backward_tc(DcnPlan *p);   // dcnv2_bwd_tc.cu: bwd_tc, dw_tc and bwd (after plan_forward_tc)

// x [B][Cin][HW] -> channels-last copy xt [B][HW][nb][32] (dcnv2_tc.cu)
int dcn_to_channels_last(const float *x, float *xt, const DcnShapeTc &s, cudaStream_t stream);
int dcn_prepare_weights_tc(const float *weight, int cin, int cout, int kh, int kw, int dg, float *wtiles,
                           cudaStream_t stream);
// Tensor-core forward from pre-tiled weights into the prepared forward's workspace (p.fwd).  fused_offset_mask:
// `offset` is the raw conv_offset_mask output; epi_scale / epi_shift / relu: the folded BatchNorm + ReLU epilogue
int dcn_forward_tc_prepared(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                            const float *wtiles, const float *bias, float *output, void *workspace, cudaStream_t stream,
                            int fused_offset_mask, const float *epi_scale, const float *epi_shift, int relu);
// Tensor-core backward (dcnv2_bwd_tc.cu) into the workspace of p.bwd: dX, dOffset, dMask; then dW and dBias
int dcn_backward_data_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                         const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                         float *grad_mask, void *workspace, cudaStream_t stream);
int dcn_backward_weight_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                           const float *grad_output, float *grad_weight, float *grad_bias, void *workspace,
                           cudaStream_t stream);

}  // namespace cnb
