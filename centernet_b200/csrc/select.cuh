// Fused 3x3 peak-NMS + exact top-K selection over [n_img, C, H, W] score maps.
// Replaces models/decode.py:9-15 (_nms) + :92-119 (_topk / _topk_channel).
// The score map is fp32, or fp16 / bf16 in the hot geometry (k_select_hot widens each element to fp32 in
// registers, exactly, so a half map selects what its .float() upcast selects).
#pragma once
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "common.cuh"

namespace cnb {

constexpr int SEL_THREADS = 1024;
constexpr int SEL_WARPS = SEL_THREADS / 32;
constexpr int SEL_STAGES = 3;           // stage ring depth (the hot kernel's too, for fp16 / bf16 maps as well)
constexpr int SEL_STAGE_BYTES = 65536;  // one 128x128 fp32 plane
constexpr int SEL_CAP = 2048;           // per-CTA candidate buffer (64-bit keys)
constexpr int SEL_HIST_FINE = 2048;     // running-threshold histogram: 128 bins per octave over [2^-16, 1)
constexpr int SEL_HIST_COARSE = 64;      // 64 fine bins each (only the first FINE/64 are used)
constexpr int SEL_MASK_WORDS = 512;     // qualifying-pixel bitmask of one unit
constexpr int SEL_RW = 4;               // rows per warp work item
constexpr int SEL_MAX_K = 1024;
constexpr int SEL_MAX_CTA = 192;        // stage-1 grid limit (one CTA per SM; H100 has 132)
constexpr int SEL_FIN_MAX = 8192;       // separate-finalize sort capacity (keys); the fused finalize uses SEL_CAP

struct SelectPlan {
  int n_img, C, H, W, K;
  int Wp;         // shared-memory row pitch (floats), W rounded up to 4
  int ncb;        // 128-column blocks per row
  int rb;         // rows per unit (a unit = one strip of one plane, plus halo rows)
  int upp;        // units per plane
  int n_cta;      // stage-1 grid
  int max_slots;  // candidate segments an image can receive (<= CTAs overlapping it)
  int use_tma;
  int nms;
  int logits;     // src holds pre-sigmoid logits; scores are sigmoid(src) (hot geometry only, detectors/ctdet.py:31)
  int clamp_one;  // order by min(score, 1): exct_decode clamps the NMS'd maps before _topk (decode.py:299-302)
  int fused_finalize;  // last CTA of an image merges its segments inside stage 1
  int seg_cap;    // keys per candidate segment (>= K; the hot kernel delivers unsorted supersets)
  int hot;        // 128x128 planes, TMA, NMS, fused finalize, K <= 256: warp-asynchronous kernel
  int wb;         // partition weight of an image boundary, in planes (flush + bootstrap + finalize cost)
  long long P;    // planes = n_img * C
  int cta_start[SEL_MAX_CTA + 1];  // first plane of every CTA's contiguous range (host-computed partition)
#ifdef CNB_SELECT_STATS
  int stat_call;  // tuning build: launch number of the hot kernel (slot of its per-CTA timestamps)
#endif
};

// Raw top-K outputs ([n_img, K] each, any pointer may be null) plus the fused ctdet epilogue.
struct FinalizeOut {
  float *scores;
  int64_t *inds;
  int32_t *clses;
  float *ys;
  float *xs;
  // ctdet epilogue (models/decode.py:472-493); dets == null -> raw only
  const void *wh;   // element type: wh_dtype / reg_dtype (CNB_DTYPE_*; zero-initialised = fp32)
  const void *reg;
  int cat_spec_wh;
  float *dets;
  int wh_dtype, reg_dtype;
};

// Returns CNB_OK or an error; fills `pl`.  elem_size (4, or 2 for fp16 / bf16) and the alignment of src decide
// whether the map can be loaded with TMA bulk copies.
int make_select_plan(const void *src, int n_img, int C, int H, int W, int K, int nms, SelectPlan *pl,
                     int elem_size = 4);
size_t select_workspace_bytes(const SelectPlan &pl);
// select_workspace_bytes for an fp32 map at any address (0 when no plan exists): an aligned 128x128 map takes the hot
// plan, a misaligned one the generic plan, whose grid and segment count differ, so neither bounds the other.
size_t select_workspace_bytes_any_align(int n_img, int C, int H, int W, int K);
// Enqueue stage 1 + finalize.  `ws` must hold select_workspace_bytes(pl).  src_dtype other than CNB_DTYPE_F32 is
// only accepted for a hot plan (pl.hot) made with elem_size 2.
int run_select(const void *src, const SelectPlan &pl, const FinalizeOut &out, void *ws, cudaStream_t stream,
               int src_dtype = CNB_DTYPE_F32);

inline int dtype_bytes(int dt) { return dt == CNB_DTYPE_F32 ? 4 : 2; }
// out = n elements of src (dtype code dt) widened to fp32, or (sigmoid) torch's CUDA sigmoid of them.  A plain
// widening needs a 16-bit src.
int launch_to_f32(const void *src, int dt, bool sigmoid, float *out, long long n, cudaStream_t stream);

// The selection over one score map of dtype code dt as the multi-head decodes run it (logits: the map holds the
// pre-sigmoid logits).  The hot kernel reads the map in place, and so does every fp32 selection of an fp32 heat map;
// otherwise one launch_to_f32 pass writes an fp32 copy (map_bytes, in the caller's workspace) that the fp32 selection
// then reads.  `copy` is where that copy goes (null in the workspace queries: a 16-byte aligned place).
struct MapSelect {
  SelectPlan pl;     // plan of what the selection reads: the map itself, or its fp32 copy
  int widen;         // 1: the fp32 copy is made first
  size_t sel_bytes;  // selection scratch of pl
  size_t map_bytes;  // the fp32 copy (0 when !widen)
};
int plan_map_select(const void *src, int dt, int logits, int n_img, int C, int H, int W, int K, const float *copy,
                    MapSelect *m);
// Enqueue the selection planned by m; `ws` holds at least m.sel_bytes of scratch.
int run_map_select(const void *src, int dt, int logits, const MapSelect &m, float *copy, const FinalizeOut &out,
                   void *ws, cudaStream_t stream);

#ifdef __CUDACC__
// A score-map element as fp32: the exact widening, or (SIG: the element is a logit) torch's CUDA sigmoid of it,
// 1 / (1 + exp(-x)) on the widened value (the expression of k_sigmoid).
template <bool SIG, typename T>
__device__ __forceinline__ float score_f32(T v) {
  const float x = to_f32(v);
  return SIG ? 1.0f / (1.0f + expf(-x)) : x;
}
// Element i of a head of dtype code dt, widened (the decode epilogues gather K rows per image: a runtime switch, no
// template instances).
__device__ __forceinline__ float ld_head(const void *p, int dt, size_t i) {
  if (dt == CNB_DTYPE_BF16) return __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16 *>(p) + i));
  if (dt == CNB_DTYPE_F16) return __half2float(__ldg(reinterpret_cast<const __half *>(p) + i));
  return __ldg(reinterpret_cast<const float *>(p) + i);
}
// Four consecutive map elements as loaded from shared memory (16 bytes of fp32, 8 of fp16 / bf16: the 16-bit sweep
// keeps its row window in half the registers) and their exact widening to fp32.
template <typename T> struct Raw4;
template <> struct Raw4<float> { typedef float4 type; };
template <> struct Raw4<__half> { typedef uint2 type; };
template <> struct Raw4<__nv_bfloat16> { typedef uint2 type; };
template <typename T>
__device__ __forceinline__ typename Raw4<T>::type ld_raw4(const T *p) {
  return *reinterpret_cast<const typename Raw4<T>::type *>(p);
}
template <typename T> __device__ __forceinline__ typename Raw4<T>::type raw4_ninf();   // four -inf
template <> __device__ __forceinline__ float4 raw4_ninf<float>() {
  return make_float4(CNB_NEG_INF, CNB_NEG_INF, CNB_NEG_INF, CNB_NEG_INF);
}
template <> __device__ __forceinline__ uint2 raw4_ninf<__half>() { return make_uint2(0xfc00fc00u, 0xfc00fc00u); }
template <> __device__ __forceinline__ uint2 raw4_ninf<__nv_bfloat16>() { return make_uint2(0xff80ff80u, 0xff80ff80u); }
template <typename T> __device__ __forceinline__ float4 widen4(typename Raw4<T>::type r);
template <> __device__ __forceinline__ float4 widen4<float>(float4 r) { return r; }
template <> __device__ __forceinline__ float4 widen4<__half>(uint2 u) {
  return make_float4(__half2float(__ushort_as_half((unsigned short)(u.x & 0xffffu))),
                     __half2float(__ushort_as_half((unsigned short)(u.x >> 16))),
                     __half2float(__ushort_as_half((unsigned short)(u.y & 0xffffu))),
                     __half2float(__ushort_as_half((unsigned short)(u.y >> 16))));
}
template <> __device__ __forceinline__ float4 widen4<__nv_bfloat16>(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xffff0000u));
}
#endif

}  // namespace cnb
