// Shared by the wgmma DCNv2 kernels (dcnv2_tc.cu: forward, dcnv2_bwd_tc.cu: backward): the shared-memory tile
// layout (K-major, no swizzle), the wgmma descriptor and instruction wrappers and the shape / work decomposition.
#pragma once
#include <cuda_bf16.h>
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

// bf16 forward (k_dcn_forward<Bf16>): a 32-channel block is a 64-byte line of the bf16 channels-last copy and one row
// of a tile is four 16-byte k-chunks (8 channels each).  A tile: k-chunks pitched 160 bytes, so the eight 16-byte
// stores of a quarter-warp (2 rows x 4 k-chunks) land in eight different bank groups (DESIGN 4.4).  B tile: dense.
constexpr uint32_t BF_LBO = 160;                    // A: bytes between consecutive k-chunks (8 rows x 16 B + 32 B)
constexpr uint32_t BF_SBO = 4 * BF_LBO;             // A: bytes between 8-row groups (640)
constexpr int BF_A_BYTES = (TC_TP / 8) * BF_SBO;    // 10240
constexpr uint32_t BF_B_LBO = 128;                  // B: bytes between consecutive k-chunks
constexpr uint32_t BF_B_SBO = 4 * BF_B_LBO;         // B: bytes between 8-row groups (512)
constexpr int BF_STAGES = 4;                        // ring depth: (10240 + 64 * co_t) bytes a stage

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
__device__ __forceinline__ uint32_t bf_tile_off(int row, int k) {   // byte offset of (row, k) in a dense bf16 tile
  return (uint32_t)(row >> 3) * BF_B_SBO + (uint32_t)(k >> 3) * BF_B_LBO + (uint32_t)(row & 7) * 16u +
         (uint32_t)(k & 7) * 2u;
}
// sm_90 shared-memory matrix descriptor: start address, leading (k-chunk) and stride (8-row group) byte offsets,
// base offset 0, layout type 0 = no swizzle
__device__ __forceinline__ uint64_t wg_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((addr >> 4) & 0x3fff) | ((uint64_t)((lbo >> 4) & 0x3fff) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fff) << 32);
}
__device__ __forceinline__ uint64_t tc_desc(uint32_t addr) { return wg_desc(addr, TC_LBO, TC_SBO); }

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
// bf16 operands, fp32 accumulate: D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, both K-major (imm-trans-a/b = 0); the
// accumulator fragment is the one of the TF32 form above
__device__ __forceinline__ void wgmma_bf16_n8(float (&d)[4], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3}"
      ", %4, %5, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}"
      ", %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
      ", %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,"
      "%26,%27,%28,%29,%30,%31}"
      ", %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,"
      "%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,"
      "%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
      ", %64, %65, p, 1, 1, 0, 0;\n\t}"
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
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,"
      "%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,"
      "%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,"
      "%120,%121,%122,%123,%124,%125,%126,%127}"
      ", %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(N == 8 || N == 16 || N == 32 || N == 64 || N == 128 || N == 256, "wgmma_bf16: no such N");
  if constexpr (N == 8) wgmma_bf16_n8(d, da, db, scale_d);
  else if constexpr (N == 16) wgmma_bf16_n16(d, da, db, scale_d);
  else if constexpr (N == 32) wgmma_bf16_n32(d, da, db, scale_d);
  else if constexpr (N == 64) wgmma_bf16_n64(d, da, db, scale_d);
  else if constexpr (N == 128) wgmma_bf16_n128(d, da, db, scale_d);
  else wgmma_bf16_n256(d, da, db, scale_d);
}
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ void mbar_arrive_tc(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Operand formats of the wgmma passes (forward, column gradient, weight gradient).  Each pass is one kernel body
// templated on the format; the format carries only what differs between them: the bytes of an operand tile, the A
// pitches and ring depths of each pass, how a value is written into a tile and the MMA over one 32-wide K slice.
//   Tf32x3  the default fp32 path: an operand tile is a TF32 hi tile followed by its lo tile (tc_tile_off), three
//           MMAs a k8 step (lo.hi + hi.lo + hi.hi: fp32-accurate products)
//   Bf16    the opt-in bf16 path: one bf16 tile rounded RN (bf_tile_off), one MMA a k16 step
// The dense tiles of both have 128-byte k-chunks (8 of them a row in TF32, 4 in bf16); a k step is two k-chunks.
struct Tf32x3 {
  using X = float;                                      // element of the channels-last input copy the forward samples
  static constexpr int ELEM = 8;                        // bytes of one element of an operand tile: hi + lo
  static constexpr int KE = 4;                          // elements of one 16-byte k-chunk
  static constexpr uint32_t SBO = TC_SBO;               // dense tile: bytes between 8-row groups
  static constexpr uint32_t FW_A_LBO = FW_LBO, FW_A_SBO = FW_SBO;   // forward: sampler A tile
  static constexpr int FW_A = 2 * FW_A_BYTES;
  __host__ __device__ static constexpr int fw_stages(int co_t) { return co_t == 64 ? 3 : 2; }
  static constexpr int BW_STAGES = 3;                   // column-gradient ring
  static constexpr uint32_t WG_A_SBO = 1040;            // weight pass: A tile 8-row groups (conflict-free scalar stores)
  static constexpr int WG_A = 2 * (TC_TP / 8) * WG_A_SBO;
  static constexpr int WG_STAGES = 3;

  // v at (row, k) of the dense tile at t whose lo tile starts lo bytes further
  __device__ static __forceinline__ void put(unsigned char *t, size_t lo, int row, int k, float v) {
    const float h = tf32_hi(v);
    *reinterpret_cast<float *>(t + tc_tile_off(row, k)) = h;
    *reinterpret_cast<float *>(t + lo + tc_tile_off(row, k)) = v - h;
  }
  // v.x .. v.w at rows r .. r + 3 of one k (16 bytes apart) from byte off of a tile whose lo tile starts lo bytes further
  __device__ static __forceinline__ void put_rows4(unsigned char *t, size_t lo, uint32_t off, const float4 v) {
    const float4 h4 = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    float *dh = reinterpret_cast<float *>(t + off), *dl = reinterpret_cast<float *>(t + lo + off);
    dh[0] = h4.x; dh[4] = h4.y; dh[8] = h4.z; dh[12] = h4.w;
    dl[0] = v.x - h4.x; dl[4] = v.y - h4.y; dl[8] = v.z - h4.z; dl[12] = v.w - h4.w;
  }
  __device__ static __forceinline__ float bound_value(float v) { return v; }   // deterministic-mode bounds
  // one operand tile (hi + lo) by TMA bulk copies of 8 KB
  __device__ static __forceinline__ void fetch(unsigned char *dst, const unsigned char *src, uint32_t bytes,
                                               uint64_t *bar) {
    for (uint32_t off = 0; off < bytes; off += 8192u) bulk_g2s(dst + off, src + off, 8192u, bar);
  }
  // D[64 x N] (+)= A[64 x 32] . B[N x 32]^T: A at a (lo tile a_lo further) with its k-chunk and 8-row group pitches,
  // B dense at b (lo tile b_lo further); acc == false overwrites D
  template <int N>
  __device__ static __forceinline__ void mma_k32(float (&d)[N / 2], uint32_t a, uint32_t a_lo, uint32_t a_lbo,
                                                 uint32_t a_sbo, uint32_t b, uint32_t b_lo, bool acc) {
#pragma unroll
    for (int ks = 0; ks < TC_K / 8; ++ks) {
      const uint32_t ka = (uint32_t)ks * 2u * a_lbo, kb = (uint32_t)ks * 2u * TC_LBO;
      wgmma_3xtf32<N>(d, wg_desc(a + ka, a_lbo, a_sbo), wg_desc(a + a_lo + ka, a_lbo, a_sbo), tc_desc(b + kb),
                      tc_desc(b + b_lo + kb), (acc || ks > 0) ? 1u : 0u);
    }
  }
};

struct Bf16 {
  using X = __nv_bfloat16;
  static constexpr int ELEM = 2;
  static constexpr int KE = 8;
  static constexpr uint32_t SBO = BF_B_SBO;
  static constexpr uint32_t FW_A_LBO = BF_LBO, FW_A_SBO = BF_SBO;
  static constexpr int FW_A = BF_A_BYTES;
  __host__ __device__ static constexpr int fw_stages(int) { return BF_STAGES; }
  static constexpr int BW_STAGES = 4;
  static constexpr uint32_t WG_A_SBO = 528;             // 512 + 16 bytes (DESIGN 4.4.3)
  static constexpr int WG_A = (TC_TP / 8) * WG_A_SBO;
  static constexpr int WG_STAGES = 4;

  __device__ static __forceinline__ void put(unsigned char *t, size_t, int row, int k, float v) {
    *reinterpret_cast<__nv_bfloat16 *>(t + bf_tile_off(row, k)) = __float2bfloat16_rn(v);
  }
  __device__ static __forceinline__ void put_rows4(unsigned char *t, size_t, uint32_t off, const float4 v) {
    __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(t + off);
    dst[0] = __float2bfloat16_rn(v.x);
    dst[8] = __float2bfloat16_rn(v.y);
    dst[16] = __float2bfloat16_rn(v.z);
    dst[24] = __float2bfloat16_rn(v.w);
  }
  __device__ static __forceinline__ float bound_value(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
  __device__ static __forceinline__ void fetch(unsigned char *dst, const unsigned char *src, uint32_t bytes,
                                               uint64_t *bar) {
    bulk_g2s(dst, src, bytes, bar);
  }
  template <int N>
  __device__ static __forceinline__ void mma_k32(float (&d)[N / 2], uint32_t a, uint32_t, uint32_t a_lbo,
                                                 uint32_t a_sbo, uint32_t b, uint32_t, bool acc) {
#pragma unroll
    for (int ks = 0; ks < TC_K / 16; ++ks) {
      const uint32_t ka = (uint32_t)ks * 2u * a_lbo, kb = (uint32_t)ks * 2u * BF_B_LBO;
      wgmma_bf16<N>(d, wg_desc(a + ka, a_lbo, a_sbo), wg_desc(b + kb, BF_B_LBO, BF_B_SBO), (acc || ks > 0) ? 1u : 0u);
    }
  }
};

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

// Workspace of one forward format: [xt: channels-last copy of the input][part: fp32 split-K partials] (prepared_bytes);
// the weight tiles live in a buffer of their own (wtiles_bytes), or, in the plain fp32 forward, in front of it (bytes)
struct DcnFwdLayout {
  size_t xt, xt_bytes, part, prepared_bytes, wtiles_bytes, bytes;
};
// Workspace of one backward format (plan_bwd in dcnv2_bwd_tc.cu): [xt][dxt][wtt][max(gyt + dcol of one batch chunk,
// gyk + wpart + bpart)], then in deterministic mode [bnd][dxi] or, at the same offset and for cout > 256, the fp32 dW
// partials wpart32.  bytes == 0 where the pass does not run.
struct DcnBwdLayout {
  size_t xt, dxt, wtt, gyt, dcol, gyk, wpart, bpart, bnd, dxi, wpart32, bytes;
  int chunk;           // images per pass of the data pass
};

// Host-side plan of one DCNv2 call or workspace query (dcn_plan in dcnv2.cu, after the one validation): the shape, the
// path decisions and the byte offset of every workspace region.  Each size and offset is worked out once, by
// plan_forward_tc and plan_backward_tc; the hosts of the kernels read their pointers from here.
struct DcnPlan {
  DcnShapeTc s;        // the validated shape and the tensor-core decomposition (fill_shape)
  bool det;            // deterministic mode (cnb_dcnv2_set_deterministic), read once per call
  bool fwd_tc;         // the tensor-core forward covers the shape: isotropic stride/pad/dilation
  bool bwd_tc;         // so does the tensor-core backward: isotropic and within its 32-bit in-image indexing
  bool dw_tc;          // and its weight pass: cout <= 256 (above, dW runs on the fp32 kernel)
  bool x_cl, gx_cl;    // input / grad_input are channels-last [b][h*w][cin] (whole 32-channel blocks) and used as such
  bool xt_ready;       // weight pass: the data pass already wrote the channels-last input copy on this stream
  int fp32_dw_splits;  // pixel-range splits of the fp32 dW kernel
  DcnFwdLayout fwd, bf16;   // 3xTF32 and bf16 forward
  DcnBwdLayout bwd, bwd16;  // 3xTF32 and bf16 backward; both sample an fp32 channels-last input copy (fwd.xt_bytes)
};
void plan_forward_tc(DcnPlan *p);     // dcnv2_tc.cu: fwd and bf16
void plan_backward_tc(DcnPlan *p);    // dcnv2_bwd_tc.cu: bwd_tc, dw_tc, bwd and bwd16 (after plan_forward_tc)

// x [B][Cin][HW] -> channels-last copy xt [B][HW][nb][32] (dcnv2_tc.cu)
int dcn_to_channels_last(const float *x, float *xt, const DcnShapeTc &s, cudaStream_t stream);
// the same fp32 copy from a bf16 x (exact widening): NCHW, or x_cl: [B][HW][Cin] with whole 32-channel blocks
int dcn_to_channels_last(const __nv_bfloat16 *x, bool x_cl, float *xt, const DcnShapeTc &s, cudaStream_t stream);
int dcn_prepare_weights_tc(const float *weight, int cin, int cout, int kh, int kw, int dg, float *wtiles,
                           cudaStream_t stream);
// Tensor-core forward from pre-tiled weights into the prepared forward's workspace (p.fwd).  fused_offset_mask:
// `offset` is the raw conv_offset_mask output; epi_scale / epi_shift / relu: the folded BatchNorm + ReLU epilogue
int dcn_forward_tc_prepared(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                            const float *wtiles, const float *bias, float *output, void *workspace, cudaStream_t stream,
                            int fused_offset_mask, const float *epi_scale, const float *epi_shift, int relu);
// bf16 forward (dcnv2_tc.cu): bf16 weight tiles of one chunk each, [co_t][32] K-major, from an fp32 weight (RN)
int dcn_prepare_weights_bf16(const float *weight, int cin, int cout, int kh, int kw, int dg, void *wtiles,
                             cudaStream_t stream);
// bf16 forward into the workspace of p.bf16.  in_bf16 / out_bf16: input / output are bf16 (else fp32); p.x_cl: the
// input is channels-last and read in place when it is bf16 (an fp32 one is rounded into p.bf16.xt by a flat pass)
int dcn_forward_bf16(const DcnPlan &p, const void *input, bool in_bf16, const float *offset, const float *mask,
                     const void *wtiles, const float *bias, void *output, bool out_bf16, void *workspace,
                     cudaStream_t stream, int fused_offset_mask, const float *epi_scale, const float *epi_shift,
                     int relu);
// DCN block (dcnv2_tc.cu): the 3x3 conv_offset_mask inside the bf16 forward.  Offset-conv weight tiles of a
// [27][cin][3][3] W_om (dcn_om_tiles_bytes), then the forward into the workspace of p.bf16 with the input's dtype out;
// the caller has checked the range (3x3, stride 1, pad 1, dilation 1, dg 1, cin % 32 == 0)
size_t dcn_om_tiles_bytes(int cin);
int dcn_prepare_om_weights_bf16(const float *w_om, int cin, void *om_tiles, cudaStream_t stream);
int dcn_forward_block_bf16(const DcnPlan &p, const void *input, bool in_bf16, const void *om_tiles,
                           const float *om_bias, const void *wtiles, const float *bias, void *output,
                           void *workspace, cudaStream_t stream, const float *epi_scale, const float *epi_shift,
                           int relu);
// Tensor-core backward (dcnv2_bwd_tc.cu) into the workspace of p.bwd: dX, dOffset, dMask; then dW and dBias
int dcn_backward_data_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                         const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                         float *grad_mask, void *workspace, cudaStream_t stream);
int dcn_backward_weight_tc(const DcnPlan &p, const float *input, const float *offset, const float *mask,
                           const float *grad_output, float *grad_weight, float *grad_bias, void *workspace,
                           cudaStream_t stream);
// bf16 backward (dcnv2_bwd_tc.cu) into the workspace of p.bwd16: all five gradients (each nullable, fp32, accumulated
// into).  in_bf16 / gy_bf16: input / grad_output are bf16 (else fp32); offset, mask and weight are fp32
int dcn_backward_bf16(const DcnPlan &p, const void *input, bool in_bf16, const float *offset, const float *mask,
                      const float *weight, const void *grad_output, bool gy_bf16, float *grad_input, float *grad_offset,
                      float *grad_mask, float *grad_weight, float *grad_bias, void *workspace, cudaStream_t stream);

}  // namespace cnb
