// Host side of the TMA-fed tensor-core GEMM family (dz_umma.cuh): tensor-map encoding and the per-launch tables
// (CTA descriptors, TMA programs).  A UmPlan is built once per learner and replayed every step.
#pragma once
#include <vector>

#include "dz_umma.cuh"

namespace dz {

// MMA path of a launch: the warp-level mma.sync kernels (every operand layout) or the wgmma kernel (K-major, pre-split).
// On the mma.sync path, launches that fc_eligible() accepts run on umma_fc_kernel, all others on umma_gemm_kernel.
// UM_PATH_CONVERTERS (tests only) keeps umma_gemm_kernel, with its converter warps, where umma_fc_kernel would run.
enum : int { UM_PATH_AUTO = 0, UM_PATH_MMA_SYNC = 1, UM_PATH_WGMMA = 2, UM_PATH_CONVERTERS = 3 };

// One launch of umma_gemm_kernel / umma_fc_kernel / wgmma_gemm_kernel: a contiguous range of CTA descriptors sharing NJT / stage geometry.
struct UmLaunch {
  int cta0 = 0, nctas = 0;
  int njt = 64;
  int stages = 4;
  uint32_t stage_bytes = 0;
  int nmaps = 0;
  int map_ids[um::kMaxMapsPerLaunch] = {0};   // plan map index of the launch-local map slot (the ops of this launch use slots)
};

struct UmPlan {
  std::vector<CUtensorMap> maps;
  std::vector<UmProblem> probs;
  std::vector<UmCta> ctas;
  std::vector<UmTmaOp> ops;
  // device copies
  CUtensorMap* d_maps = nullptr;
  UmProblem* d_probs = nullptr;
  UmCta* d_ctas = nullptr;
  UmTmaOp* d_ops = nullptr;

  // 5-D fp32 tensor map with SWIZZLE_128B; dims/strides innermost first (strides in BYTES for dims 1..4; dims beyond
  // `rank` are 1).  Returns the map index or -1 (error string set).
  int add_map(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);
  // Rewrites the `map` field of the ops of launch `l` (ctas [cta0, cta0 + nctas)) from plan indices to launch-local slots.
  int localize_maps(UmLaunch& l);
  int upload();          // (re)allocates and copies all four tables
  void release();
  // d_trace: 512 clock stamps of CTA 0 (debug).  path: UM_PATH_AUTO picks wgmma_gemm_kernel when wgmma_eligible(l), else
  // the mma.sync path; UM_PATH_MMA_SYNC / UM_PATH_WGMMA force one (forcing wgmma on a launch that is not eligible fails).
  int launch(const char* tag, const UmLaunch& l, void* stream, long long* d_trace = nullptr, int path = UM_PATH_AUTO) const;
  // Every CTA of the launch has both operands K-major tf32 hi/lo pairs that need no conversion, four k-steps per stage.
  bool wgmma_eligible(const UmLaunch& l) const;
  // Every CTA has an MN-major raw fp32 A (convert 1 without scale_r, or 2) of 128 / nprob rows and 32 reduction rows per
  // stage, nprob <= 2, a K-major pre-split B, four k-steps per stage and the direct partial epilogue.
  bool fc_eligible(const UmLaunch& l) const;
  int path_of(const UmLaunch& l) const { return wgmma_eligible(l) ? UM_PATH_WGMMA : UM_PATH_MMA_SYNC; }
  static int configure();   // one-time kernel attributes (outside any stream capture)
};

// Operand format helpers
inline UmOperand um_kmajor(int rows, bool hi_lo, bool convert, const float* scale_r = nullptr) {
  UmOperand o;
  memset(&o, 0, sizeof(o));
  o.part_bytes = (uint32_t)(((rows * 128) + 1023) / 1024 * 1024);
  o.nparts = hi_lo ? 2 : 1; o.convert = convert ? 1 : 0; o.mn_major = 0; o.lbo = 0; o.scale_r = scale_r;
  return o;
}
inline UmOperand um_mnmajor(int mn, int r_rows, bool convert, const float* scale_r = nullptr) {
  UmOperand o;
  memset(&o, 0, sizeof(o));
  o.lbo = (uint32_t)(r_rows * 128);
  o.part_bytes = (uint32_t)((mn / 32) * o.lbo);
  o.nparts = 2; o.convert = convert ? 1 : 0; o.mn_major = 1; o.scale_r = scale_r;
  return o;
}

}  // namespace dz
