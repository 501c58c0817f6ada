// Packed-operand tensor-core GEMM for the LARGE contractions of the learner (IQN's 3136->512 layer runs at
// M = batch * tau_samples = 2048 rows per network apply; networks.py:264-292, iqn/agent.py:178-214).
//
//     D[i,j] = sum_r A(i,r) * B(j,r)        fp32 in, fp32-grade out (error-compensated 3xTF32, see dz_tc.cuh)
//
// The hi/lo TF32 split is taken OUT of the GEMM: a bandwidth-bound pack kernel writes each operand once as two
// "tile images" (hi and lo parts) in a shared-memory layout whose m16n8k8 fragment loads are bank-conflict free,
// so that the GEMM's producer is ONE thread issuing cp.async.bulk copies that complete on an mbarrier and the
// MMA warps read the stages as they landed.
//
// Image layout: pk_index (dz_internal.cuh).
//
// Accuracy: the tensor core adds into its fp32 accumulator with round-towards-zero, so the products of each
// k-step are added into the fp32 sums with ordinary round-to-nearest adds (dz_tc.cuh, warp_kstep_3xtf32).
#pragma once
#include "dz_async.cuh"
#include "dz_internal.cuh"
#include "dz_tc.cuh"

namespace dz {

namespace tcp {

using namespace tc;

constexpr int kEpiWarps = 8;
constexpr int kThreadsP = (2 + kEpiWarps) * 32;

// ---- pack: fp32 matrix -> hi/lo tile images -----------------------------------------------------------------
// One block = one 64-row x 64-deep tile, staged through shared memory so that both the source reads (either
// orientation) and the image writes (512-byte runs) are coalesced.
__global__ void __launch_bounds__(256) tc_pack_kernel(const __grid_constant__ PackBatch pb) {
  dz::pdl_enter();
  __shared__ float tile[64][65];
  int j = 0;
  while (j + 1 < pb.n && (int)blockIdx.x >= pb.job[j + 1].block0) ++j;
  const PackJob& J = pb.job[j];
  const int t = (int)blockIdx.x - J.block0;
  const int row0 = (t % J.tiles_r) * 64, red0 = (t / J.tiles_r) * 64;
  const int tid = threadIdx.x;
  const bool vec = (J.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(J.src) & 15) == 0);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int idx = tid + q * 256;
    const int a = idx >> 4, b4 = (idx & 15) * 4;         // a: index along the strided source dim, b4: along the contiguous one
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (J.red_contig) {
      const int row = row0 + a, red = red0 + b4;
      if (row < J.rows && red < J.red) {
        const float* s = J.src + (long long)row * J.ld + red;
        if (vec && red + 3 < J.red) { float4 x = *reinterpret_cast<const float4*>(s); v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; }
        else { for (int e = 0; e < 4; ++e) if (red + e < J.red) v[e] = s[e]; }
      }
      if (row == J.ones_row) for (int e = 0; e < 4; ++e) v[e] = red + e < J.red ? 1.f : 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) tile[a][b4 + e] = v[e];
    } else {
      const int red = red0 + a, row = row0 + b4;
      if (red < J.red && row < J.rows) {
        const float* s = J.src + (long long)red * J.ld + row;
        if (vec && row + 3 < J.rows) { float4 x = *reinterpret_cast<const float4*>(s); v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; }
        else { for (int e = 0; e < 4; ++e) if (row + e < J.rows) v[e] = s[e]; }
      }
      if (red < J.red) for (int e = 0; e < 4; ++e) if (row + e == J.ones_row) v[e] = 1.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) tile[b4 + e][a] = v[e];
    }
  }
  __syncthreads();
  const int RG = J.rows_pad >> 3;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int id = tid + q * 256;
    const int r = id & 7, c = (id >> 3) & 3, rg = (id >> 5) & 7, kbl = id >> 8;
    const int row = row0 + rg * 8 + r, red = red0 + kbl * 16 + c * 4;
    if (row < J.rows_pad && red < J.red_pad) {
      const float* s = &tile[rg * 8 + r][kbl * 16 + c * 4];
      float4 x = make_float4(s[0], s[1], s[2], s[3]);
      float4 h, l;
      split_tf32(x, h, l);
      const long long off = pk_index(row, red, RG);
      *reinterpret_cast<float4*>(J.hi + off) = h;
      *reinterpret_cast<float4*>(J.lo + off) = l;
    }
  }
}

// ---- GEMM -----------------------------------------------------------------------------------------------------
template <int BNJ, int EPI>
struct PkSmem {
  static constexpr int kA = 128 * kPkKB * 4, kB = BNJ * kPkKB * 4;     // bytes of one part (hi or lo) of one stage
  static constexpr int kStage = 2 * kA + 2 * kB;
  static constexpr int kStages = EPI ? 2 : 4;      // EPI 1: short reduction (<= 8 k-blocks)
  static constexpr int kBars = 1024;
  static constexpr int kTotal = kBars + kStages * kStage;
};

// grid = (tiles_j, tiles_i * splits, problems); dynamic smem = PkSmem<BNJ, EPI>::kTotal; 320 threads:
//   warp 0: producer (one lane issues the bulk copies)      warp 1: barrier set-up
//   warps 2..9: MMA + epilogue, D rows [32 q, 32 q + 32) (q = warp % 4) x columns [BNJ/2 h, BNJ/2 (h + 1)) (h = (warp - 2) / 4)
// EPI 0: plain output (split partials, or + bias / ReLU).
// EPI 1: IQN embedding epilogue (networks.py:279-284) for a SHORT reduction (splits == 1):
//        v = relu(acc + bias[j]) -> e0 (fp32, optional);  h = v * mul[i / mul_div][j] -> written straight as the
//        hi/lo tile images of the NEXT GEMMs' operands (rows i, and optionally the transposed rows j).
// The epilogues work on one D row per lane: the fragments are transposed 32 columns at a time through shared memory.
template <int BNJ, int EPI>
__global__ void __launch_bounds__(kThreadsP, 1) tc_pgemm_kernel(const __grid_constant__ PkBatch batch) {
  dz::pdl_enter();
  extern __shared__ __align__(128) uint8_t smem[];
  using L = PkSmem<BNJ, EPI>;
  constexpr int ST = L::kStages;
  const PkProblem& p = batch.p[blockIdx.z];
  const int tiles_i = (p.MI + 127) / 128;
  const int tile_i = blockIdx.y % tiles_i, split = blockIdx.y / tiles_i;
  const int i0 = tile_i * 128, j0 = blockIdx.x * BNJ;
  if ((int)blockIdx.y >= tiles_i * p.splits || j0 >= p.NJ) return;
  const int per = (p.nkb + p.splits - 1) / p.splits;
  const int kb0 = split * per;
  const int nkb = max(min(p.nkb, kb0 + per) - kb0, 0);

  uint64_t* full = reinterpret_cast<uint64_t*>(smem);      // [ST]  bulk copies landed       (tx-count barrier)
  uint64_t* empty = full + ST;                              // [ST]  MMA warps consumed the stage
  uint8_t* stage_base = smem + L::kBars;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kCols = BNJ / 2;                // columns per MMA warp
  constexpr int NT = kCols / 8;

  if (warp == 1 && lane == 0) {
    for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kEpiWarps); }
    fence_mbarrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ---------------------------------------------------------------- producer
    if (elect_one()) {
      const float* a_hi = p.A.hi; const float* a_lo = p.A.lo; const float* b_hi = p.B.hi; const float* b_lo = p.B.lo;
      for (int it = 0; it < nkb; ++it) {
        const int s = it % ST;
        const uint32_t ph = (uint32_t)(it / ST) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        mbar_expect_tx(&full[s], (uint32_t)L::kStage);
        const int r = (kb0 + it) * kPkKB;
        const long long a_off = pk_index(i0, r, p.A.rg_total), b_off = pk_index(j0, r, p.B.rg_total);
        const uint32_t st = smem_u32(stage_base + (size_t)s * L::kStage);
        bulk_g2s(st, a_hi + a_off, L::kA, &full[s]);
        bulk_g2s(st + L::kA, a_lo + a_off, L::kA, &full[s]);
        bulk_g2s(st + 2 * L::kA, b_hi + b_off, L::kB, &full[s]);
        bulk_g2s(st + 2 * L::kA + L::kB, b_lo + b_off, L::kB, &full[s]);
      }
    }
    __syncwarp();
  } else if (warp >= 2) {
    // ---------------------------------------------------------------- MMA warps
    const int ew = warp - 2;
    const int quarter = warp & 3;
    const int half = ew >> 2;
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
    for (int it = 0; it < nkb; ++it) {
      const int s = it % ST;
      mbar_wait(&full[s], (uint32_t)(it / ST) & 1u);
      const uint8_t* st = stage_base + (size_t)s * L::kStage;
#pragma unroll
      for (int k = 0; k < kPkKB / 8; ++k)
        warp_kstep_3xtf32<2, NT>(acc, st, st + L::kA, st + 2 * L::kA, st + 2 * L::kA + L::kB, quarter * 32, half * kCols, 8 * k,
                                 [](int m, int r) { return pk_off(m, r); }, [](int n, int r) { return pk_off(n, r); });
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // every MMA warp is done with the stage buffers: they hold the per-warp transposition patches [32 rows][33]
    asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32) : "memory");
    float* patch = reinterpret_cast<float*>(stage_base) + ew * 32 * 33;
    // r[t] = D[row i0 + 32 quarter + lane][column j0 + half * kCols + c0 + t]
    auto rows_of = [&](int c0, float (&r)[32]) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) patch[frag_row(mt, e) * 33 + frag_col(nt, e)] = acc[mt][c0 / 8 + nt][e];
      __syncwarp();
#pragma unroll
      for (int t = 0; t < 32; ++t) r[t] = patch[lane * 33 + t];
      __syncwarp();
    };
    if constexpr (EPI == 1) {
      const int i = i0 + quarter * 32 + lane;
      const bool row_ok = i < p.MI;
      const int NJ = p.NJ;
      const float* bias = p.bias_j;
      const float* mulrow = p.mul + (long long)((row_ok ? i : 0) / p.mul_div) * p.mul_ld;
      float* e0 = p.e0 ? p.e0 + (long long)i * p.e0_ld : nullptr;
      float* img_hi = p.img_hi; float* img_lo = p.img_lo; float* imgT_hi = p.imgT_hi; float* imgT_lo = p.imgT_lo;
      const long long rg1 = p.img_rg, rgT = p.imgT_rg;
#pragma unroll
      for (int c0 = 0; c0 < kCols; c0 += 32) {
        float r[32];
        rows_of(c0, r);
#pragma unroll
        for (int t = 0; t < 32; t += 4) {
          const int j = j0 + half * kCols + c0 + t;          // NJ % 4 == 0: a group of four is all valid or all invalid
          const bool ok = row_ok && j < NJ;
          float4 h = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok) {
            const float4 b4 = *reinterpret_cast<const float4*>(bias + j);
            float4 v;
            v.x = fmaxf(r[t] + b4.x, 0.f);
            v.y = fmaxf(r[t + 1] + b4.y, 0.f);
            v.z = fmaxf(r[t + 2] + b4.z, 0.f);
            v.w = fmaxf(r[t + 3] + b4.w, 0.f);
            if (e0) *reinterpret_cast<float4*>(e0 + j) = v;
            const float4 m4 = *reinterpret_cast<const float4*>(mulrow + j);
            h = make_float4(v.x * m4.x, v.y * m4.y, v.z * m4.z, v.w * m4.w);
          }
          if (ok) {
            const long long off = pk_index(i, j, rg1);
            float4 hh, ll;
            split_tf32(h, hh, ll);
            *reinterpret_cast<float4*>(img_hi + off) = hh;
            *reinterpret_cast<float4*>(img_lo + off) = ll;
          }
          if (imgT_hi) {                                       // whole warp: 4x4 transpose inside each lane quad
            const float4 ht = quad_transpose(h, lane);         // lane e: h[m0..m0+3] at column j + e
            const int jj = j + (lane & 3), m0 = i & ~3;
            if (m0 < p.MI && jj < NJ) {
              const long long off = pk_index(jj, m0, rgT);
              float4 hh, ll;
              split_tf32(ht, hh, ll);
              *reinterpret_cast<float4*>(imgT_hi + off) = hh;
              *reinterpret_cast<float4*>(imgT_lo + off) = ll;
            }
          }
        }
      }
    } else {
      const int i = i0 + quarter * 32 + lane;
      float* dst = p.C + (long long)split * p.split_stride + (long long)i * p.sc_i;
      const int jb = j0 + half * kCols;
      const bool epi = p.splits == 1;
      const float* bias = epi ? p.bias_j : nullptr;
      const bool relu = epi && p.relu;
      const long long sc_j = p.sc_j;
      const bool v4 = sc_j == 1 && ((reinterpret_cast<uintptr_t>(dst + jb) & 15) == 0) && jb + kCols <= p.NJ;
#pragma unroll
      for (int c0 = 0; c0 < kCols; c0 += 32) {
        float r[32];
        rows_of(c0, r);
        if (i >= p.MI) continue;
#pragma unroll
        for (int t = 0; t < 32; t += 4) {
          float v[4] = {r[t], r[t + 1], r[t + 2], r[t + 3]};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = jb + c0 + t + e;
            if (bias && j < p.NJ) v[e] += bias[j];
            if (relu) v[e] = fmaxf(v[e], 0.f);
          }
          if (v4) {
            *reinterpret_cast<float4*>(dst + jb + c0 + t) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int j = jb + c0 + t + e;
              if (j < p.NJ) dst[(long long)j * sc_j] = v[e];
            }
          }
        }
      }
    }
  }
}

}  // namespace tcp
}  // namespace dz
