// Fused 3x3 peak-NMS + exact top-K selection over [n_img, C, H, W] score maps.
// Replaces models/decode.py:9-15 (_nms) + :92-119 (_topk / _topk_channel).
#pragma once
#include "common.cuh"

namespace cnb {

constexpr int SEL_THREADS = 1024;
constexpr int SEL_WARPS = SEL_THREADS / 32;
constexpr int SEL_STAGES = 3;
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
};

// Raw top-K outputs ([n_img, K] each, any pointer may be null) plus the fused ctdet epilogue.
struct FinalizeOut {
  float *scores;
  int64_t *inds;
  int32_t *clses;
  float *ys;
  float *xs;
  // ctdet epilogue (models/decode.py:472-493); dets == null -> raw only
  const float *wh;
  const float *reg;
  int cat_spec_wh;
  float *dets;
};

// Returns CNB_OK or an error; fills `pl`.
int make_select_plan(const float *src, int n_img, int C, int H, int W, int K, int nms, SelectPlan *pl);
size_t select_workspace_bytes(const SelectPlan &pl);
// Enqueue stage 1 + finalize.  `ws` must hold select_workspace_bytes(pl).
int run_select(const float *src, const SelectPlan &pl, const FinalizeOut &out, void *ws, cudaStream_t stream);

}  // namespace cnb
