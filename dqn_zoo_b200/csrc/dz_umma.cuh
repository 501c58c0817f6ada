// TMA-fed tensor-core GEMM family for the batch-32 learner step (sm_90a): every conv / 512-wide FC contraction of
// networks.py:181-221 (dqn_torso, dqn_value_head) and :137-178 (noisy_linear), forward and input-gradient, as
//
//     D[i, j] = sum_r A(i, r) * B(j, r)          fp32 in, fp32-grade out (error-compensated 3xTF32)
//
// Operand tiles live in shared memory in 128-byte-swizzled layouts and are delivered by TMA
// (cp.async.bulk.tensor, SWIZZLE_128B tensor maps) straight from the tensors' natural layouts:
//
//   K-major  (reduction index contiguous in the source): a stage is [rows][32 r] = rows x 128 B; convolutions get
//            their implicit im2col from the tensor map itself — a box over (channels, ox, oy, image) of the NHWC
//            activation lands as dense 128-byte rows, negative / out-of-range coordinates are zero-filled by the TMA
//            unit (that is the zero padding of the input-gradient convolutions).
//   MN-major (row index contiguous in the source, e.g. W[k][n] for y = xW): a stage is [32 r][32 mn] slabs, LBO
//            apart; the MMA warps' fragment loads do the transposition — no shuffles, no transposed copies.  (This is
//            why these launches use the warp-level m16n8k8 MMA, umma_gemm_kernel: tf32 wgmma only reads K-major
//            operands from shared memory.  Launches whose operands are all K-major and pre-split run on warpgroup
//            MMAs that read the staged tiles through shared-memory descriptors, wgmma_gemm_kernel.)
//
// Precision: activations are stored ONCE as tf32 hi/lo pairs by the producing epilogue (x = hi + lo, both exactly
// representable), fp32 weights are split in place in shared memory by converter warps (raw tile -> hi in place, lo
// in the sibling buffer; the split is position-wise, so it is swizzle-agnostic) or, for the fc forward and input
// gradient, in the MMA warps' registers (umma_fc_kernel), D += Al*Bh + Ah*Bl + Ah*Bh.  The
// tensor core truncates its fp32 accumulator, so each k-step's products are added into the fp32 sums with
// round-to-nearest adds (dz_tc.cuh, warp_kstep_3xtf32 / wgmma_kstep_3xtf32).
//
// The TMA "program" of every CTA (which boxes of which tensor map go where in each stage) is a table built once on
// the host (dz_umma.cu): the device side is geometry-free.
#pragma once
#include <cuda.h>

#include "dz_async.cuh"
#include "dz_internal.cuh"
#include "dz_tc.cuh"

namespace dz {

struct UmTmaOp {          // one TMA box load of one stage (32 bytes)
  uint32_t map;           // index into the tensor-map array
  uint32_t smem_off;      // byte offset inside the stage
  int32_t c[5];           // box start coordinates (innermost first)
  uint32_t pad;
};

struct UmOperand {
  uint32_t part_bytes;    // bytes of one part (hi or lo) of a stage; multiple of 1024
  uint32_t nparts;        // 2: hi + lo;  1: exact operand (values are tf32 numbers, no lo part)
  uint32_t convert;       // 1: TMA delivers raw fp32 into part 0; converter warps split it into hi (in place) / lo (part 1)
                          // 2: TMA delivers TWO raw tiles, mu into part 0 and sigma into part 1 (noisy layers, networks.py:
                          //    137-178); the converters form w = mu + sigma * scale_r[r] * scale_i[i] and split THAT in place
  uint32_t mn_major;      // 0: K-major [rows][32 r];  1: MN-major slabs of [r rows][32 mn]
  uint32_t lbo;           // MN-major: bytes between 32-wide slabs (= r rows per stage * 128)
  const float* scale_r;   // convert only: element *= scale_r[reduction index] before the split (noisy sigma weights)
  const float* scale_i;   // convert == 2 only: ... *= scale_i[row index of D / of the operand] (factorised noise, other factor)
};

enum : uint32_t { UM_EPI_PARTIAL = 0, UM_EPI_ROWS = 1 };

struct UmProblem {
  UmOperand A, B;
  uint32_t ksteps;          // MMA k-steps per stage
  uint32_t red_per_stage;   // reduction elements per stage
  uint32_t epi;
  int32_t MI, NJ;           // valid extents of D
  // UM_EPI_PARTIAL: C[split * split_stride + i * sc_i + j * sc_j] = acc * (scale_i ? scale_i[i] : 1)
  float* C;
  long long sc_i, sc_j, split_stride;
  const float* scale_i;
  // UM_EPI_ROWS: one D row = one pixel / sample with NJ channels:
  //   v = acc (+ bias[j]) (relu) (mask[dst * out_ld + j] > 0 ? v : 0)  ->  out_hi / out_lo (tf32 split) and out_f32
  float* out_hi; float* out_lo; float* out_f32;
  const float* bias;
  const float* mask;
  int32_t relu;
  int32_t out_ld;           // floats between consecutive dst rows of out_* / mask (>= NJ; the pointers may be column-offset)
  int32_t pw;               // tile row r -> (r / pw, r % pw); dst row = row_base + (r / pw) * rs_outer + (r % pw) * rs_inner
  int32_t rs_outer, rs_inner;
};

struct UmCta {              // one per CTA
  uint32_t prob;
  uint32_t op0;             // first UmTmaOp
  uint32_t nstages;
  uint32_t ops_per_stage;
  uint32_t tx_bytes;        // bytes landing per stage
  int32_t r0;               // reduction index of stage 0 (for scale_r)
  int32_t i0;               // UM_EPI_PARTIAL: first D row of this tile
  int32_t split;
  int32_t row_base;         // UM_EPI_ROWS
  int32_t ph_valid, pw_valid;   // valid (r / pw) and (r % pw) extents
  uint32_t nprob;           // umma_fc_kernel: problems prob, prob + 1, ... sharing the staged A tile (0 or 1: one)
};

namespace um {

using namespace tc;

constexpr int kStagesMax = 8;
constexpr int kConvWarps = 8;
constexpr int kThreadsU = (2 + 4 + kConvWarps) * 32;   // producer, barrier set-up, 4 MMA / epilogue, 8 converter warps

// In-place hi/lo split of one raw operand part (a sequence of 128-byte swizzled rows).  i0: MN index of the part's row 0.
__device__ __forceinline__ void convert_part(const UmOperand& o, uint8_t* part0, int r0, int i0, int ct) {
  const int nchunks = (int)(o.part_bytes >> 4);
  const float* __restrict__ sc = o.scale_r;
  const float* __restrict__ si = o.scale_i;
  const int rows_per_slab = (int)(o.lbo >> 7);
  const bool dual = o.convert == 2;
  for (int idx = ct; idx < nchunks; idx += kConvWarps * 32) {
    float4* p = reinterpret_cast<float4*>(part0 + ((size_t)idx << 4));
    float4* p1 = reinterpret_cast<float4*>(part0 + o.part_bytes + ((size_t)idx << 4));
    float4 x = *p;
    if (sc || dual) {
      const int row = idx >> 3;
      float4 f = make_float4(1.f, 1.f, 1.f, 1.f);
      if (o.mn_major) {          // rows are reduction indices, the 128 bytes of a row are 32 consecutive MN indices
        const int slab = row / rows_per_slab, rr = row - slab * rows_per_slab;
        if (sc) { const float s = sc[r0 + rr]; f.x = s; f.y = s; f.z = s; f.w = s; }
        if (dual && si) {        // 16-byte chunks XOR-ed with (row & 7): logical chunk of this physical one
          const int cl = (idx & 7) ^ (row & 7);
          const float4 t = *reinterpret_cast<const float4*>(si + i0 + slab * 32 + cl * 4);
          f.x *= t.x; f.y *= t.y; f.z *= t.z; f.w *= t.w;
        }
      } else {                   // columns are reduction indices; logical 16-byte chunk = physical ^ (row & 7)
        const int c = (idx & 7) ^ (row & 7);
        if (sc) f = *reinterpret_cast<const float4*>(sc + r0 + c * 4);
        if (dual && si) { const float t = si[i0 + row]; f.x *= t; f.y *= t; f.z *= t; f.w *= t; }
      }
      if (dual) {
        const float4 g = *p1;
        x.x = fmaf(g.x, f.x, x.x); x.y = fmaf(g.y, f.y, x.y); x.z = fmaf(g.z, f.z, x.z); x.w = fmaf(g.w, f.w, x.w);
      } else {
        x.x *= f.x; x.y *= f.y; x.z *= f.z; x.w *= f.w;
      }
    }
    float4 h, l;
    split_tf32(x, h, l);
    *p = h;
    *p1 = l;
  }
}

// Fast path for a 16 KB operand part (128 x 32 tile: every 3136 -> 512 weight tile): 4 chunks per converter thread,
// fully unrolled.  With 256 threads striding by 256 chunks, a thread's row-within-slab (MN-major) / 16-byte column
// (K-major) never changes, so the reduction-index factor is ONE load per stage and the row-index factors (si_*) are
// loop invariants of the whole kernel (hoisted by the caller).
struct ConvHoist { float4 si4[4]; float si1[4]; };
__device__ __forceinline__ void convert_hoist(const UmOperand& o, int i0, int i_limit, int ct, ConvHoist& h) {
  const float* __restrict__ si = o.convert == 2 ? o.scale_i : nullptr;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h.si4[j] = make_float4(1.f, 1.f, 1.f, 1.f);
    h.si1[j] = 1.f;
    if (si) {
      if (o.mn_major) {   // slab j, logical 16-byte chunk cl of the 128-byte swizzle
        const int cl = (ct & 7) ^ ((ct >> 3) & 7);
        const int i = min(i0 + j * 32 + cl * 4, i_limit - 4);
        h.si4[j] = *reinterpret_cast<const float4*>(si + i);
      } else {
        h.si1[j] = si[min(i0 + (ct >> 3) + j * 32, i_limit - 1)];
      }
    }
  }
}
__device__ __forceinline__ void convert_part16k(const UmOperand& o, uint8_t* part0, int r0, int ct, const ConvHoist& h) {
  const float* __restrict__ sc = o.scale_r;
  const bool dual = o.convert == 2;
  float4 fr = make_float4(1.f, 1.f, 1.f, 1.f);
  if (sc) {
    if (o.mn_major) { const float s = sc[r0 + (ct >> 3)]; fr = make_float4(s, s, s, s); }
    else fr = *reinterpret_cast<const float4*>(sc + r0 + (((ct & 7) ^ ((ct >> 3) & 7)) << 2));
  }
  float4 x[4], g[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    x[j] = *reinterpret_cast<const float4*>(part0 + ((size_t)(ct + j * 256) << 4));
    if (dual) g[j] = *reinterpret_cast<const float4*>(part0 + 16384 + ((size_t)(ct + j * 256) << 4));
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float4 f = fr;
    if (o.mn_major) { f.x *= h.si4[j].x; f.y *= h.si4[j].y; f.z *= h.si4[j].z; f.w *= h.si4[j].w; }
    else { f.x *= h.si1[j]; f.y *= h.si1[j]; f.z *= h.si1[j]; f.w *= h.si1[j]; }
    float4 v = x[j];
    if (dual) { v.x = fmaf(g[j].x, f.x, v.x); v.y = fmaf(g[j].y, f.y, v.y); v.z = fmaf(g[j].z, f.z, v.z); v.w = fmaf(g[j].w, f.w, v.w); }
    else if (sc) { v.x *= f.x; v.y *= f.y; v.z *= f.z; v.w *= f.w; }
    float4 hh, ll;
    split_tf32(v, hh, ll);
    *reinterpret_cast<float4*>(part0 + ((size_t)(ct + j * 256) << 4)) = hh;
    *reinterpret_cast<float4*>(part0 + 16384 + ((size_t)(ct + j * 256) << 4)) = ll;
  }
}

constexpr int kMaxMapsPerLaunch = 12;
struct UmMaps { CUtensorMap m[kMaxMapsPerLaunch]; };   // passed as a __grid_constant__ kernel parameter: the TMA unit's
                                                        // descriptor cache is fed from the constant bank (descriptors left in
                                                        // plain global memory cost a dependent fetch per TMA operation)
constexpr int kMaxOpsPerCta = 256;     // TMA ops of one CTA staged in shared memory (8 KB)
constexpr int kCtlBytes = 1024 + 1024 + kMaxOpsPerCta * 32;   // barriers | problem copy | op table

// Named barrier over the 12 non-producer/non-MMA warps (epilogue + converter warps): the cooperative store phase.
__device__ __forceinline__ void bar_sync_coop() { asm volatile("bar.sync 1, 384;" ::: "memory"); }

// Staging tile of the cooperative store phase: fp32 [128 rows][NJT], 16-byte chunks XOR-swizzled inside every 128-byte
// group so that row-per-thread writes and chunk-per-thread reads are both bank-conflict free.
template <int NJT>
__device__ __forceinline__ float4* stage_chunk(uint8_t* base, int r, int c) {
  return reinterpret_cast<float4*>(base + (size_t)r * (NJT * 4) + (size_t)(((c & ~7) | ((c ^ r) & 7)) << 4));
}

// Cooperative store phase: the fp32 tile staged by stage_chunk<NJT> at stage_base goes out through the row epilogue
// (bias, ReLU, mask, tf32 hi/lo split; one D row = one output pixel / sample) or the partial epilogue.  tid: 0..383,
// the thread's index among the 384 threads that take part.
template <int NJT>
__device__ __forceinline__ void store_tile(const UmProblem& p, const UmCta& cta, uint8_t* stage_base, int tid) {
  const int NJ = p.NJ, cpr = NJ >> 2;
  const int items = 128 * cpr;
  // idx -> (row, chunk) and row -> (outer, inner) without integer divisions: rows < 128, so a 16-bit reciprocal is exact
  const uint32_t inv_cpr = (65536u + (uint32_t)cpr - 1u) / (uint32_t)cpr;
  constexpr int kIters = (128 * (NJT / 4) + 383) / 384;
  if (p.epi == UM_EPI_ROWS) {
    const int pw = p.pw;
    const long long ld = p.out_ld;
    const bool relu = p.relu != 0;
    const float* __restrict__ maskp = p.mask;
    const float* __restrict__ bias = p.bias;
    float* __restrict__ of = p.out_f32; float* __restrict__ oh = p.out_hi; float* __restrict__ ol = p.out_lo;
    const uint32_t inv_pw = pw >= 128 ? 0u : (65536u + (uint32_t)pw - 1u) / (uint32_t)pw;
#pragma unroll
    for (int j = 0; j < kIters; ++j) {
      const int idx = tid + j * 384;
      if (idx >= items) continue;
      const int r = (int)(((uint32_t)idx * inv_cpr) >> 16), c = idx - r * cpr;
      const int ro = (int)(((uint32_t)r * inv_pw) >> 16), ri = r - ro * pw;
      if (ro >= cta.ph_valid || ri >= cta.pw_valid) continue;
      const long long o = ((long long)cta.row_base + (long long)ro * p.rs_outer + (long long)ri * p.rs_inner) * ld + 4 * c;
      float4 v = *stage_chunk<NJT>(stage_base, r, c);
      if (bias) { const float4 b4 = *reinterpret_cast<const float4*>(bias + 4 * c); v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w; }
      if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      if (maskp) {
        const float4 m4 = *reinterpret_cast<const float4*>(maskp + o);
        v.x = m4.x > 0.f ? v.x : 0.f; v.y = m4.y > 0.f ? v.y : 0.f; v.z = m4.z > 0.f ? v.z : 0.f; v.w = m4.w > 0.f ? v.w : 0.f;
      }
      if (of) *reinterpret_cast<float4*>(of + o) = v;
      if (oh) {
        float4 h, l;
        split_tf32(v, h, l);
        *reinterpret_cast<float4*>(oh + o) = h;
        *reinterpret_cast<float4*>(ol + o) = l;
      }
    }
  } else {
    float* __restrict__ C = p.C + (long long)cta.split * p.split_stride;
    const float* __restrict__ scale_i = p.scale_i;
    const long long sc_i = p.sc_i, sc_j = p.sc_j;
    const bool vec = sc_j == 1 && (sc_i & 3) == 0 && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
#pragma unroll
    for (int j = 0; j < kIters; ++j) {
      const int idx = tid + j * 384;
      if (idx >= items) continue;
      const int r = (int)(((uint32_t)idx * inv_cpr) >> 16), c = idx - r * cpr;
      const int i = cta.i0 + r;
      if (i >= p.MI) continue;
      float4 v = *stage_chunk<NJT>(stage_base, r, c);
      if (scale_i) { const float s = scale_i[i]; v.x *= s; v.y *= s; v.z *= s; v.w *= s; }
      float* dst = C + (long long)i * sc_i + (long long)(4 * c) * sc_j;
      if (vec) *reinterpret_cast<float4*>(dst) = v;
      else { dst[0] = v.x; dst[sc_j] = v.y; dst[2 * sc_j] = v.z; dst[3 * sc_j] = v.w; }
    }
  }
}

// grid = number of CTA descriptors; dynamic smem = kCtlBytes + stages * stage_bytes + 1024 (alignment slack).
// Warp roles: 0 TMA producer | 1 barrier set-up | 2-5 MMA (warp 2 + q owns D rows [32q, 32q + 32), all NJT columns, as
// m16n8k8 fragments read straight from the staged tiles) | 6-13 operand converters.  All twelve warps 2-13 take part in the
// final store phase (tile staged in shared memory, written out in full rows).
template <int NJT>
__global__ void __launch_bounds__(kThreadsU, 1)
    umma_gemm_kernel(const __grid_constant__ UmMaps maps, const UmCta* __restrict__ ctas, const UmProblem* __restrict__ probs,
                     const UmTmaOp* __restrict__ ops, int nmaps, int stages, uint32_t stage_bytes, long long* __restrict__ trace) {
  if (threadIdx.x < nmaps) prefetch_tensormap(&maps.m[threadIdx.x]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const bool tr = trace != nullptr && blockIdx.x == 0;
  // The plan tables (CTA descriptors, problems, TMA programs) are written once at plan upload, never by a kernel of the
  // step: the whole set-up below runs BEFORE griddepcontrol.wait, i.e. it overlaps the tail of the previous kernel
  // whenever that kernel has triggered its dependents.
  const UmCta cta = ctas[blockIdx.x];
  const int ST = stages;
  const int nst = (int)cta.nstages;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);      // [ST] TMA landed
  uint64_t* ready = full + kStagesMax;                      // [ST] converters done (only with convert)
  uint64_t* empty = ready + kStagesMax;                     // [ST] MMA warps consumed the stage
  UmProblem* p_smem = reinterpret_cast<UmProblem*>(smem + 1024);
  UmTmaOp* ops_smem = reinterpret_cast<UmTmaOp*>(smem + 2048);
  uint8_t* stage_base = smem + kCtlBytes;
  static_assert(sizeof(UmProblem) <= 1024 && sizeof(UmProblem) % 16 == 0, "problem copy does not fit its slot");
  static_assert(kCtlBytes % 1024 == 0, "stage base must stay 1024-byte aligned");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // The CTA's problem and its whole TMA program go to shared memory once (coalesced): the producer's per-stage
  // work is then a shared-memory read, not a dependent global load per stage.
  {
    const uint4* src = reinterpret_cast<const uint4*>(probs + cta.prob);
    uint4* dst = reinterpret_cast<uint4*>(p_smem);
    for (int i = threadIdx.x; i < (int)(sizeof(UmProblem) / 16); i += kThreadsU) dst[i] = src[i];
    const int nvec = min(nst * (int)cta.ops_per_stage, kMaxOpsPerCta) * 2;
    const uint4* osrc = reinterpret_cast<const uint4*>(ops + cta.op0);
    uint4* odst = reinterpret_cast<uint4*>(ops_smem);
    for (int i = threadIdx.x; i < nvec; i += kThreadsU) odst[i] = osrc[i];
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&ready[s], kConvWarps); mbar_init(&empty[s], 4); }
    fence_mbarrier_init();
  }
  __syncthreads();
  // griddepcontrol.wait is executed per role, right before the role's first access to data an earlier kernel may have
  // produced.
  const UmProblem& p = *p_smem;
  const bool conv_a = p.A.convert != 0, conv_b = p.B.convert != 0;
  const bool any_conv = conv_a || conv_b;
  const uint32_t a_bytes = p.A.part_bytes * p.A.nparts;
  // stores that stay coalesced along i (unit stride) are written straight from the MMA fragments
  const bool direct = p.epi == UM_EPI_PARTIAL && p.sc_i == 1;
  constexpr int NT = NJT / 8;
  float sum[2][NT][4];

  // TMA producers.  Issuing a tensor load costs the issuing warp ~130-300 cycles of operand set-up (shared-memory read of the
  // op, address arithmetic, moves to uniform registers), far more than the TMA unit needs — so the ops of a stage are spread
  // over warps: warp 0 always; when no operand needs conversion the eight converter warps have nothing else to do and
  // each takes ops too (op q -> producer q % nprod).  Every producer waits for the slot itself; warp 0 posts the byte
  // count (bytes may land before the expect_tx arrive: the phase cannot complete without that arrive).
  const int nops = (int)cta.ops_per_stage;
  const int nprod = any_conv ? 1 : min(nops, 1 + kConvWarps);
  const int pidx = warp == 0 ? 0 : (warp >= 6 && warp < 14 ? warp - 5 : 99);
  if (pidx < nprod) {
    int s = 0;
    uint32_t ph = 0;
    uint32_t st_addr = smem_u32(stage_base);
    int oi = 0;
    dz::pdl_enter();
    if (tr && warp == 0 && lane == 0) { trace[323] = clock64(); trace[324] = clock64(); }
    const int my_ops = (nops - pidx + nprod - 1) / nprod;      // ops pidx, pidx + nprod, ...
    for (int it = 0; it < nst; ++it) {
      mbar_wait(&empty[s], ph ^ 1u);
      if (pidx == 0 && lane == 0) mbar_expect_tx(&full[s], cta.tx_bytes);
      __syncwarp();
      if (lane < my_ops) {   // lanes prepare their ops SIMD; only the UTMALDG instructions themselves are serialised
        const int o = oi + pidx + lane * nprod;
        const UmTmaOp op = o < kMaxOpsPerCta ? ops_smem[o] : ops[cta.op0 + o];   // long programs spill to the global table
        tma_load_5d(st_addr + op.smem_off, &maps.m[op.map], &full[s], op.c[0], op.c[1], op.c[2], op.c[3], op.c[4]);
      }
      if (tr && warp == 0 && lane == 0 && it < 64) trace[it] = clock64();                          // [0,64): TMA issued
      __syncwarp();
      oi += nops;
      ++s; st_addr += stage_bytes;
      if (s == ST) { s = 0; ph ^= 1u; st_addr = smem_u32(stage_base); }
    }
  }
  if (warp >= 2 && warp < 6) {
    // ---------------------------------------------------------------- MMA warps
    const int m0 = (warp - 2) * 32;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) sum[mt][nt][e] = 0.f;
    const uint32_t a_lbo = p.A.lbo, b_lbo = p.B.lbo;
    const bool a_mn = p.A.mn_major != 0, b_mn = p.B.mn_major != 0;
    auto a_off = [&](int m, int k) { return a_mn ? sw128_mnmajor(m, k, a_lbo) : sw128_kmajor(m, k); };
    auto b_off = [&](int n, int k) { return b_mn ? sw128_mnmajor(n, k, b_lbo) : sw128_kmajor(n, k); };
    const int ksteps = (int)p.ksteps;
    int s = 0;
    uint32_t ph = 0;
    for (int it = 0; it < nst; ++it) {
      mbar_wait(any_conv ? &ready[s] : &full[s], ph);
      if (tr && warp == 2 && lane == 0 && it < 64) trace[64 + it] = clock64();                     // [64,128): stage data ready
      const uint8_t* st = stage_base + (size_t)s * stage_bytes;
      const uint8_t* bh = st + a_bytes;
      for (int k = 0; k < ksteps; ++k)
        warp_kstep_3xtf32<2, NT>(sum, st, st + p.A.part_bytes, bh, bh + p.B.part_bytes, m0, 0, 8 * k, a_off, b_off);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (tr && warp == 2 && lane == 0 && it < 64) trace[128 + it] = clock64();                    // [128,192): stage consumed
      if (++s == ST) { s = 0; ph ^= 1u; }
    }
    if (warp == 2 && lane == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel's set-up overlaps our epilogue
    dz::pdl_enter();
    if (tr && warp == 2 && lane == 0) trace[320] = clock64();                                       // store phase starts
    if (direct) {
      float* dst = p.C + (long long)cta.split * p.split_stride;
      const long long sc_j = p.sc_j;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; e += 2) {
          const int i = cta.i0 + m0 + frag_row(mt, e);
          if (i >= p.MI) continue;
          const float sc = p.scale_i ? p.scale_i[i] : 1.0f;
#pragma unroll
          for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int j = frag_col(nt, e + h);
              if (j < p.NJ) dst[i + (long long)j * sc_j] = sum[mt][nt][e + h] * sc;
            }
        }
    }
  } else if (warp >= 6 && any_conv) {
    // ---------------------------------------------------------------- converter warps: raw fp32 -> hi / lo in place
    const int ct = threadIdx.x - 6 * 32;
    const UmOperand oa = p.A, ob = p.B;
    const int red = (int)p.red_per_stage;
    int s = 0, r0 = cta.r0;
    uint32_t ph = 0;
    uint8_t* st = stage_base;
    dz::pdl_enter();
    const bool fast_a = conv_a && oa.part_bytes == 16384u && (!oa.mn_major || oa.lbo == 4096u);
    ConvHoist hoist;
    if (fast_a) convert_hoist(oa, cta.i0, p.MI, ct, hoist);
    for (int it = 0; it < nst; ++it) {
      mbar_wait(&full[s], ph);
      if (fast_a) convert_part16k(oa, st, r0, ct, hoist);
      else if (conv_a) convert_part(oa, st, r0, cta.i0, ct);
      if (conv_b) convert_part(ob, st + a_bytes, r0, 0, ct);
      fence_proxy_async_shared();   // before the TMA unit refills the slot
      __syncwarp();
      if (lane == 0) mbar_arrive(&ready[s]);
      r0 += red;
      ++s; st += stage_bytes;
      if (s == ST) { s = 0; ph ^= 1u; st = stage_base; }
    }
  }
  if (!direct && warp >= 2 && warp < 14) {
    // ---------------------------------------------------------------- cooperative store phase (warps 2-13, 384 threads)
    if (warp >= 6 && !any_conv) dz::pdl_enter();          // idle converter warps: first access to global data is here
    // every MMA warp is done reading the stage buffers (and with it every TMA write has landed): they become the staging tile
    bar_sync_coop();
    if (warp < 6) {
      const int m0 = (warp - 2) * 32;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int e = 0; e < 4; e += 2) {
            const int r = m0 + frag_row(mt, e), c = frag_col(nt, e);
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(stage_chunk<NJT>(stage_base, r, c >> 2)) + (c & 3)) =
                make_float2(sum[mt][nt][e], sum[mt][nt][e + 1]);
          }
    }
    bar_sync_coop();
    store_tile<NJT>(p, cta, stage_base, threadIdx.x - 64);
  }
  if (tr && warp == 2 && lane == 0) trace[321] = clock64();                                         // stores issued
  if (tr && threadIdx.x == 0) trace[322] = clock64();
}

// Clock stamp *addr = clock64() where `pred` holds, without a branch (see mbar_arrive_if).
__device__ __forceinline__ void stamp_if(long long* addr, bool pred) {
  asm volatile("{\n.reg .pred p;\n.reg .b64 c;\nsetp.ne.b32 p, %1, 0;\nmov.u64 c, %%clock64;\n@p st.global.b64 [%0], c;\n}\n" ::"l"(addr),
               "r"((int)pred)
               : "memory");
}

// ---------------------------------------------------------------------------------------------------------------------
// Sibling of umma_gemm_kernel for the fc1 / noisy1 forward and input gradient: A = raw fp32 weights W[k][n] (mu, plus
// sigma for noisy layers), B = activations / output gradients, K-major tf32 hi/lo pairs.  The forward stages A
// MN-major (D row = n, reduction = k), the input gradient K-major (AK: D row = k, reduction = n; W's rows are
// contiguous in n).  There are no converter warps: every MMA warp loads raw mu / sigma fragments from the staged tile
// at the addresses umma_gemm_kernel reads hi fragments from, forms
//     w = fmaf(sigma, scale_r[r] * scale_i[i], mu)       (noisy; the operations and their order of convert_part16k)
// (scale_r: the noise factor of the reduction index, scale_i: that of the D row; eps_in[k] * eps_out[n] either way)
// and its tf32 hi/lo split in registers, and issues the k-step of warp_kstep_3xtf32.  Each output element therefore sees
// the same operands and the same sequence of k-steps as on umma_gemm_kernel: the partials are bit-identical.
//
// One CTA serves cta.nprob (1 or 2) consecutive problems that read the same weight tile: the passes of the learner
// that apply the same parameters (online net on s_tm1 and on s_t) stage each mu / sigma tile once.  The tile spans
// 128 / nprob D rows; the stage holds the A parts (A.part_bytes each) followed by one B hi/lo pair per problem.
// Warp roles: 0 TMA producer (and barrier set-up) | 1-8 MMA, 8 / nprob warps per problem, 16 D rows x NJT columns each.
// Only the direct partial epilogue (UM_EPI_PARTIAL, sc_i == 1) is supported: the warps store from their fragments.
constexpr int kFcMmaWarps = 8;
constexpr int kThreadsF = (1 + kFcMmaWarps) * 32;
constexpr int kFcMaxProbs = 2;

template <int NJT, bool AK>
__global__ void __launch_bounds__(kThreadsF, 1)
    umma_fc_kernel(const __grid_constant__ UmMaps maps, const UmCta* __restrict__ ctas, const UmProblem* __restrict__ probs,
                   const UmTmaOp* __restrict__ ops, int nmaps, int stages, uint32_t stage_bytes, long long* __restrict__ trace) {
  if (threadIdx.x < nmaps) prefetch_tensormap(&maps.m[threadIdx.x]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const bool tr = trace != nullptr && blockIdx.x == 0;
  const UmCta cta = ctas[blockIdx.x];
  const int ST = stages;
  const int nst = (int)cta.nstages;
  const int P = cta.nprob > 1 ? 2 : 1;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);      // [ST] TMA landed
  uint64_t* empty = full + 2 * kStagesMax;                  // [ST] MMA warps consumed the stage
  UmProblem* p_smem = reinterpret_cast<UmProblem*>(smem + 1024);
  UmTmaOp* ops_smem = reinterpret_cast<UmTmaOp*>(smem + 2048);
  uint8_t* stage_base = smem + kCtlBytes;
  static_assert(kFcMaxProbs * sizeof(UmProblem) <= 1024, "problem copies do not fit their slot");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {
    const uint4* src = reinterpret_cast<const uint4*>(probs + cta.prob);
    uint4* dst = reinterpret_cast<uint4*>(p_smem);
    for (int i = threadIdx.x; i < P * (int)(sizeof(UmProblem) / 16); i += kThreadsF) dst[i] = src[i];
    const int nvec = min(nst * (int)cta.ops_per_stage, kMaxOpsPerCta) * 2;
    const uint4* osrc = reinterpret_cast<const uint4*>(ops + cta.op0);
    uint4* odst = reinterpret_cast<uint4*>(ops_smem);
    for (int i = threadIdx.x; i < nvec; i += kThreadsF) odst[i] = osrc[i];
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kFcMmaWarps); }
    fence_mbarrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ---------------------------------------------------------------- TMA producer (as in umma_gemm_kernel, one warp)
    const int nops = (int)cta.ops_per_stage;
    int s = 0;
    uint32_t ph = 0;
    uint32_t st_addr = smem_u32(stage_base);
    int oi = 0;
    dz::pdl_enter();
    if (tr && lane == 0) { trace[323] = clock64(); trace[324] = clock64(); }
    for (int it = 0; it < nst; ++it) {
      mbar_wait(&empty[s], ph ^ 1u);
      if (lane == 0) mbar_expect_tx(&full[s], cta.tx_bytes);
      __syncwarp();
      if (lane < nops) {
        const int o = oi + lane;
        const UmTmaOp op = o < kMaxOpsPerCta ? ops_smem[o] : ops[cta.op0 + o];
        tma_load_5d(st_addr + op.smem_off, &maps.m[op.map], &full[s], op.c[0], op.c[1], op.c[2], op.c[3], op.c[4]);
      }
      if (tr && lane == 0 && it < 64) trace[it] = clock64();                                        // [0,64): TMA issued
      __syncwarp();
      oi += nops;
      ++s; st_addr += stage_bytes;
      if (s == ST) { s = 0; ph ^= 1u; st_addr = smem_u32(stage_base); }
    }
    return;
  }

  // ---------------------------------------------------------------- MMA warps
  const int w = warp - 1, wpp = kFcMmaWarps / P;
  const int q = w / wpp, m0 = 16 * (w - q * wpp);         // problem (pass) of this warp, its first D row in the tile
  const bool lead = w == 0 && lane == 0;
  const UmProblem& p = p_smem[q];
  const int g = lane >> 2, t = lane & 3;
  const uint32_t a_part = p.A.part_bytes, a_lbo = p.A.lbo;
  const uint8_t* b_first = stage_base + a_part * 2 + (uint32_t)q * 2u * p.B.part_bytes;
  const uint32_t b_part = p.B.part_bytes;
  const bool noisy = p.A.convert == 2;
  const float* __restrict__ eps_r = p.A.scale_r;
  constexpr int NT = NJT / 8;
  float sum[1][NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) sum[0][nt][e] = 0.f;
  auto b_off = [](int n, int k) { return sw128_kmajor(n, k); };
  dz::pdl_enter();                                          // the noise vectors may come from an earlier kernel
  // noise factor of the thread's two D rows (g, g + 8): loop invariants.  Rows past MI (the zero-filled tail of the
  // input gradient's last tile, never stored) read the last row's factor, as the converters do.
  float eo[2] = {1.f, 1.f};
  if (noisy) {
    eo[0] = p.A.scale_i[min(cta.i0 + m0 + g, p.MI - 1)];
    eo[1] = p.A.scale_i[min(cta.i0 + m0 + g + 8, p.MI - 1)];
  }
  // Noise factors of a stage's 32 reduction indices: lane L holds the one of index r0 + L and the k-steps take theirs
  // by shuffle.  The next stage's load is issued before the current stage's barrier wait, so its global-load latency
  // is hidden behind a stage of MMAs instead of sitting at the head of every stage's dependency chain.
  float er_next = noisy ? eps_r[cta.r0 + lane] : 1.f;
  int s = 0, r0 = cta.r0;
  uint32_t ph = 0;
  for (int it = 0; it < nst; ++it) {
    const float er = er_next;
    if (noisy && it + 1 < nst) er_next = eps_r[r0 + 32 + lane];
    mbar_wait(&full[s], ph);
    stamp_if(trace + 64 + it, tr && lead && it < 64);                                               // [64,128): stage data ready
    const uint8_t* mu = stage_base + (size_t)s * stage_bytes;
    const uint8_t* sg = mu + a_part;
    const uint8_t* bh = b_first + (size_t)s * stage_bytes;
    // NJT 64: a stage's k-steps unrolled in pairs, so that the loads hoisted ahead of the MMAs fit the 168 registers a
    // thread of a nine-warp CTA has (three warps share one sub-partition's register file)
#pragma unroll(NJT == 32 ? 4 : 2)
    for (int ks = 0; ks < 4; ++ks) {
      uint32_t ah[1][4], al[1][4];
      // noise factors of the thread's reduction indices r0 + 8 ks + t + 4 h; shuffled unconditionally (1 on plain
      // layers), so that no branch splits the stage's straight-line k-steps
      const float ei[2] = {__shfl_sync(0xffffffffu, er, 8 * ks + t), __shfl_sync(0xffffffffu, er, 8 * ks + t + 4)};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = m0 + g + (e & 1) * 8, k = 8 * ks + t + (e >> 1) * 4;
        const uint32_t o = AK ? sw128_kmajor(m, k) : sw128_mnmajor(m, k, a_lbo);
        float v = *reinterpret_cast<const float*>(mu + o);
        if (noisy) {
          const float f = ei[e >> 1] * eo[e & 1];
          v = fmaf(*reinterpret_cast<const float*>(sg + o), f, v);
        }
        float hh, ll;
        split_tf32(v, hh, ll);
        ah[0][e] = __float_as_uint(hh);
        al[0][e] = __float_as_uint(ll);
      }
      warp_mma_3xtf32<1, NT>(sum, ah, al, true, bh, bh + b_part, 0, 8 * ks, b_off);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    stamp_if(trace + 128 + it, tr && lead && it < 64);                                              // [128,192): stage consumed
    r0 += 32;
    if (++s == ST) { s = 0; ph ^= 1u; }
  }
  if (lead) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel's set-up overlaps our epilogue
  if (tr && lead) trace[320] = clock64();                                                           // store phase starts
  float* dst = p.C + (long long)cta.split * p.split_stride;
  const long long sc_j = p.sc_j;
#pragma unroll
  for (int e = 0; e < 4; e += 2) {
    const int i = cta.i0 + m0 + frag_row(0, e);
    if (i >= p.MI) continue;
    const float sc = p.scale_i ? p.scale_i[i] : 1.0f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = frag_col(nt, e + h);
        if (j < p.NJ) dst[i + (long long)j * sc_j] = sum[0][nt][e + h] * sc;
      }
  }
  if (tr && lead) { trace[321] = clock64(); trace[322] = clock64(); }                             // stores issued / exit
}

// ---------------------------------------------------------------------------------------------------------------------
// Warpgroup-MMA sibling of umma_gemm_kernel for problems whose operands are both K-major tf32 hi/lo pairs that need no
// conversion (conv2 / conv3 forward and input gradient): the staged tiles are already in the layout wgmma reads, so
// the MMAs take their operands straight from shared-memory descriptors, with no fragment loads.  TMA program, stage
// ring, PDL points, clock stamps and both epilogues are those of umma_gemm_kernel.
constexpr int kThreadsW = 3 * 128;   // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;

// Rows of the CTA's 128-row tile that reach the output: the tail beyond them (padding, TMA zero fill) is never stored,
// so an m64 half that lies entirely in it needs no MMAs.
__device__ __forceinline__ int tile_rows_out(const UmProblem& p, const UmCta& c) {
  if (p.epi == UM_EPI_ROWS) {
    if (c.ph_valid <= 0 || c.pw_valid <= 0) return 0;
    const long long n = (long long)(c.ph_valid - 1) * p.pw + min(c.pw_valid, p.pw);
    return (int)min(n, 128LL);
  }
  return max(0, min(128, p.MI - c.i0));
}

// grid = number of CTA descriptors; dynamic smem as for umma_gemm_kernel.  Warp roles: 0-3 TMA producers (warp 1 also
// sets up the barriers) | warpgroup 1 (warps 4-7) D rows [0, 64), warpgroup 2 (warps 8-11) D rows [64, 128), all NJT
// columns.  All twelve warps take part in the store phase.  A stage holds 32 reduction elements (128-byte K-major
// rows), i.e. ksteps == 4.
template <int NJT>
__global__ void __launch_bounds__(kThreadsW, 1)
    wgmma_gemm_kernel(const __grid_constant__ UmMaps maps, const UmCta* __restrict__ ctas, const UmProblem* __restrict__ probs,
                      const UmTmaOp* __restrict__ ops, int nmaps, int stages, uint32_t stage_bytes, long long* __restrict__ trace) {
  if (threadIdx.x < nmaps) prefetch_tensormap(&maps.m[threadIdx.x]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  const bool tr = trace != nullptr && blockIdx.x == 0;
  const UmCta cta = ctas[blockIdx.x];
  const int ST = stages;
  const int nst = (int)cta.nstages;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);      // [ST] TMA landed
  uint64_t* empty = full + 2 * kStagesMax;                  // [ST] consumer warps retired every MMA reading the stage
  UmProblem* p_smem = reinterpret_cast<UmProblem*>(smem + 1024);
  UmTmaOp* ops_smem = reinterpret_cast<UmTmaOp*>(smem + 2048);
  uint8_t* stage_base = smem + kCtlBytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {
    const uint4* src = reinterpret_cast<const uint4*>(probs + cta.prob);
    uint4* dst = reinterpret_cast<uint4*>(p_smem);
    for (int i = threadIdx.x; i < (int)(sizeof(UmProblem) / 16); i += kThreadsW) dst[i] = src[i];
    const int nvec = min(nst * (int)cta.ops_per_stage, kMaxOpsPerCta) * 2;
    const uint4* osrc = reinterpret_cast<const uint4*>(ops + cta.op0);
    uint4* odst = reinterpret_cast<uint4*>(ops_smem);
    for (int i = threadIdx.x; i < nvec; i += kThreadsW) odst[i] = osrc[i];
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    fence_mbarrier_init();
  }
  __syncthreads();
  const UmProblem& p = *p_smem;
  const uint32_t a_bytes = p.A.part_bytes * 2;
  const bool direct = p.epi == UM_EPI_PARTIAL && p.sc_i == 1;
  constexpr int NA = NJT / 2;   // accumulator floats per thread of an m64 x NJT tile
  float sum[NA];

  // consumer warpgroup 0 / 1 (D rows [64 wg, 64 wg + 64)); -1: producer warpgroup.  The values the MMA loop branches on
  // are broadcast from lane 0 so that ptxas sees them warp-uniform.
  const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0);
  if (wg < 0) {
    // TMA producers: the ops of a stage are spread over the producer warpgroup (op q -> warp q % nprod), as in umma_gemm_kernel.
    const int nops = (int)cta.ops_per_stage;
    const int nprod = min(nops, 4);
    if (warp < nprod) {
      const int pidx = warp;
      int s = 0;
      uint32_t ph = 0;
      uint32_t st_addr = smem_u32(stage_base);
      int oi = 0;
      dz::pdl_enter();
      if (tr && warp == 0 && lane == 0) { trace[323] = clock64(); trace[324] = clock64(); }
      const int my_ops = (nops - pidx + nprod - 1) / nprod;
      for (int it = 0; it < nst; ++it) {
        mbar_wait(&empty[s], ph ^ 1u);
        if (pidx == 0 && lane == 0) mbar_expect_tx(&full[s], cta.tx_bytes);
        __syncwarp();
        if (lane < my_ops) {
          const int o = oi + pidx + lane * nprod;
          const UmTmaOp op = o < kMaxOpsPerCta ? ops_smem[o] : ops[cta.op0 + o];
          tma_load_5d(st_addr + op.smem_off, &maps.m[op.map], &full[s], op.c[0], op.c[1], op.c[2], op.c[3], op.c[4]);
        }
        if (tr && warp == 0 && lane == 0 && it < 64) trace[it] = clock64();                          // [0,64): TMA issued
        __syncwarp();
        oi += nops;
        ++s; st_addr += stage_bytes;
        if (s == ST) { s = 0; ph ^= 1u; st_addr = smem_u32(stage_base); }
      }
    } else {
      dz::pdl_enter();                                      // idle producer warps: first access to global data is in the store phase
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups
    // Every k-step is one wgmma group into a scratch accumulator, acc0 / acc1 alternating: while the tensor cores run
    // k-step k + 1, k-step k is retired (wgmma_wait<1>) and added into `sum`.  A stage's four k-steps are straight-line
    // code and its last group is retired before the stage is released to the producers, so no group is in flight
    // across a branch or a loop edge (ptxas would serialise the MMAs); the other consumer warpgroup keeps the tensor
    // cores busy across that drain.
    const bool active = __shfl_sync(0xffffffffu, (int)(64 * wg < tile_rows_out(p, cta)), 0) != 0;
    const bool lead = warp == 4 && lane == 0;
#pragma unroll
    for (int e = 0; e < NA; ++e) sum[e] = 0.f;
    float acc0[NA], acc1[NA];
#pragma unroll
    for (int e = 0; e < NA; ++e) { acc0[e] = 0.f; acc1[e] = 0.f; }
    const uint32_t a_lo_off = p.A.part_bytes, b_lo_off = p.B.part_bytes;
    auto retire = [&](float (&d)[NA]) {
      wgmma_fence_acc(d);
#pragma unroll
      for (int e = 0; e < NA; ++e) sum[e] += d[e];
    };
    int s = 0;
    uint32_t ph = 0;
    for (int it = 0; it < nst; ++it) {
      mbar_wait(&full[s], ph);
      stamp_if(trace + 64 + it, tr && lead && it < 64);                                         // [64,128): stage data ready
      if (active) {
        const uint32_t a = smem_u32(stage_base) + (uint32_t)s * stage_bytes + 8192u * (uint32_t)wg;
        const uint32_t b = smem_u32(stage_base) + (uint32_t)s * stage_bytes + a_bytes;
        wgmma_kstep_3xtf32(acc0, a, a + a_lo_off, b, b + b_lo_off, 0);
        wgmma_kstep_3xtf32(acc1, a, a + a_lo_off, b, b + b_lo_off, 8);
        wgmma_wait<1>();
        retire(acc0);
        wgmma_kstep_3xtf32(acc0, a, a + a_lo_off, b, b + b_lo_off, 16);
        wgmma_wait<1>();
        retire(acc1);
        wgmma_kstep_3xtf32(acc1, a, a + a_lo_off, b, b + b_lo_off, 24);
        wgmma_wait<1>();
        retire(acc0);
        wgmma_wait<0>();
        mbar_arrive_if(&empty[s], lane == 0);
        retire(acc1);
      } else {
        mbar_arrive_if(&empty[s], lane == 0);
      }
      stamp_if(trace + 128 + it, tr && lead && it < 64);                                        // [128,192): stage consumed
      if (++s == ST) { s = 0; ph ^= 1u; }
    }
    if (lead) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel's set-up overlaps our epilogue
    dz::pdl_enter();
    if (tr && lead) trace[320] = clock64();                                                         // store phase starts
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
    if (direct) {
      float* dst = p.C + (long long)cta.split * p.split_stride;
      const long long sc_j = p.sc_j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = cta.i0 + r0 + 8 * h;
        if (i >= p.MI) continue;
        const float sc = p.scale_i ? p.scale_i[i] : 1.0f;
#pragma unroll
        for (int nt = 0; nt < NJT / 8; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 8 * nt + c0 + e;
            if (j < p.NJ) dst[i + (long long)j * sc_j] = sum[4 * nt + 2 * h + e] * sc;
          }
      }
    }
  }
  if (!direct) {
    // ---------------------------------------------------------------- cooperative store phase (all 384 threads)
    // every consumer warp has retired its last MMA (and with it every TMA write has landed): the stage buffers become the staging tile
    __syncthreads();
    if (wg >= 0) {
      const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int nt = 0; nt < NJT / 8; ++nt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 8 * h, c = 8 * nt + c0;
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(stage_chunk<NJT>(stage_base, r, c >> 2)) + (c & 3)) =
              make_float2(sum[4 * nt + 2 * h], sum[4 * nt + 2 * h + 1]);
        }
    }
    __syncthreads();
    store_tile<NJT>(p, cta, stage_base, threadIdx.x);
  }
  if (tr && warp == 4 && lane == 0) trace[321] = clock64();                                         // stores issued
  if (tr && threadIdx.x == 0) trace[322] = clock64();
}

}  // namespace um
}  // namespace dz
