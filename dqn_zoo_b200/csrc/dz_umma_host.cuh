// Host side of the TMA-fed tensor-core GEMM family (dz_umma.cuh): tensor-map encoding and the per-launch tables
// (CTA descriptors, TMA programs).  A UmPlan is built once per learner and replayed every step.
#pragma once
#include <algorithm>
#include <vector>

#include "dz_umma.cuh"

namespace dz {

// Dynamic shared memory of a launch with `stages` stages: alignment slack, control block, stage ring.
inline size_t um_smem_bytes(int stages, uint32_t stage_bytes) { return 1024 + um::kCtlBytes + (size_t)stages * stage_bytes; }
// Depth of a launch's stage ring: as many stages as fit in 226 KB of shared memory, at least one and at most kStagesMax.
inline int um_stages_for(uint32_t stage_bytes) {
  return std::max(1, std::min<int>(um::kStagesMax, (int)((226 * 1024 - um_smem_bytes(0, 0)) / stage_bytes)));
}
// The wgmma kernel reads 128 rows (both m64 halves) of every A part from inside the stage.
inline uint32_t um_wgmma_min_stage(uint32_t a_part_bytes) { return a_part_bytes + 16384u; }

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
  std::vector<uint32_t> box_bytes;   // bytes one box of maps[i] lands in shared memory
  std::vector<UmProblem> probs;
  std::vector<UmCta> ctas;
  std::vector<UmTmaOp> ops;
  std::vector<uint32_t> stage_op0;   // while a CTA is being built: index of the first op of each of its stages
  uint32_t build_stage_bytes = 0;    // stage_bytes of the launch being built
  // device copies
  CUtensorMap* d_maps = nullptr;
  UmProblem* d_probs = nullptr;
  UmCta* d_ctas = nullptr;
  UmTmaOp* d_ops = nullptr;

  // 5-D fp32 tensor map with SWIZZLE_128B; dims/strides innermost first (strides in BYTES for dims 1..4; dims beyond
  // `rank` are 1).  Returns the map index or -1 (error string set).
  int add_map(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);
  // The maps of the hi / lo pair of one source, same geometry: ids[0] hi, ids[1] lo.  DZ_OK or DZ_EINVAL.
  int add_map_pair(const float* hi, const float* lo, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int ids[2]);

  // Table builder.  A launch is a run of consecutive CTAs; a CTA's TMA program is a sequence of stages, each a list of
  // ops.  end_cta derives the CTA's nstages, ops_per_stage and tx_bytes from its ops, so the byte count the consumers
  // wait for always matches what the ops deliver.
  void begin_launch(UmLaunch& l, int njt, uint32_t stage_bytes) {   // cta0, njt, stage_bytes and the stage count
    l.cta0 = (int)ctas.size(); l.njt = njt; l.stage_bytes = stage_bytes; l.stages = um_stages_for(stage_bytes);
    build_stage_bytes = stage_bytes;
  }
  void end_launch(UmLaunch& l) { l.nctas = (int)ctas.size() - l.cta0; }
  int add_problem(const UmProblem& p) { probs.push_back(p); return (int)probs.size() - 1; }
  UmCta& begin_cta(int prob) {       // the new CTA, zero but for prob and op0: the caller sets its other fields
    ctas.push_back(UmCta{(uint32_t)prob, (uint32_t)ops.size()});
    stage_op0.clear();
    return ctas.back();
  }
  void stage() { stage_op0.push_back((uint32_t)ops.size()); }   // opens the CTA's next stage
  void op(int map, uint32_t smem_off, int c0, int c1 = 0, int c2 = 0, int c3 = 0, int c4 = 0) {
    ops.push_back(UmTmaOp{(uint32_t)map, smem_off, {c0, c1, c2, c3, c4}, 0u});
  }
  // The same box of a hi / lo map pair into two parts: hi at smem_off, lo part_bytes further.
  void op_pair(const int map[2], uint32_t smem_off, uint32_t part_bytes, int c0, int c1 = 0, int c2 = 0, int c3 = 0, int c4 = 0) {
    op(map[0], smem_off, c0, c1, c2, c3, c4);
    op(map[1], smem_off + part_bytes, c0, c1, c2, c3, c4);
  }
  // DZ_EINVAL when the stages differ in op count or bytes, a stage has more than 32 ops, or a box overruns the stage.
  int end_cta();
  // Rewrites the `map` field of the ops of launch `l` (ctas [cta0, cta0 + nctas)) from plan indices to launch-local slots.
  int localize_maps(UmLaunch& l);
  int upload();          // (re)allocates and copies all four tables
  void release();
  // d_trace: 512 clock stamps of CTA 0 (debug).  path: UM_PATH_AUTO picks wgmma_gemm_kernel when wgmma_eligible(l), else
  // the mma.sync path; UM_PATH_MMA_SYNC / UM_PATH_WGMMA force one (forcing wgmma on a launch that is not eligible fails).
  int launch(const char* tag, const UmLaunch& l, void* stream, long long* d_trace = nullptr, int path = UM_PATH_AUTO) const;
  // Every CTA of the launch has both operands K-major tf32 hi/lo pairs that need no conversion, four k-steps per stage.
  bool wgmma_eligible(const UmLaunch& l) const;
  // Every CTA has a raw fp32 A (convert 1 without scale_r, or 2), either MN-major of 128 / nprob rows and 32 reduction
  // rows per stage, nprob <= 2, or K-major of 128 rows, nprob 1 (the same layout in every CTA of the launch), a K-major
  // pre-split B, four k-steps per stage and the direct partial epilogue.
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
