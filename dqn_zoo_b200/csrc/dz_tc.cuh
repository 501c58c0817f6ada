// Tensor-core helpers shared by the learner's GEMM kernels (sm_90a): the warp-level m16n8k8 tf32 MMA with the
// shared-memory fragment loads of one k-step, the warpgroup MMA (wgmma) k-step on K-major swizzled tiles, the swizzled
// tile offsets, and the tf32 split
//
//     x = hi + lo,  hi = rn_tf32(x),  lo = rn_tf32(x - hi)      (error-compensated 3xTF32: D += Ah*Bh + Al*Bh + Ah*Bl)
//
// that keeps every contraction within ~2^-21 relative of an fp32 FMA evaluation (the parity bar is 1e-5 on losses and
// gradients).  The kernels themselves: dz_umma.cuh (TMA-fed family: torso + 3136->512 layers at batch 32), dz_umma_net.cu
// (conv1 with the uint8 gather), dz_tcp.cuh (packed-operand GEMM of IQN's 2048-row layers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dz {
namespace tc {

// D += A * B for one 16 x 8 x 8 tile (mma.sync, fragments as in the PTX ISA's m16n8k8 .tf32 layout):
//   a = {A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]},  b = {B[t][g], B[t+4][g]},  d = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}
// with g = lane / 4, t = lane % 4.
__device__ __forceinline__ void mma_16x8x8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// The B fragment loads and MMAs of one k-step of warp_kstep_3xtf32 (below), with the A fragments already in registers
// (ah / al, element q of m-tile mt = A[m0 + 16 mt + g + 8 (q & 1)][k0 + t + 4 (q >> 1)]); a_has_lo: false when A is
// exact (al unused).
template <int MT, int NT, class BOff>
__device__ __forceinline__ void warp_mma_3xtf32(float (&sum)[MT][NT][4], const uint32_t (&ah)[MT][4], const uint32_t (&al)[MT][4],
                                                bool a_has_lo, const uint8_t* b_hi, const uint8_t* b_lo, int n0, int k0, BOff b_off) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    uint32_t bh[2], bl[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint32_t o = b_off(n0 + nt * 8 + g, k0 + t + q * 4);
      bh[q] = *reinterpret_cast<const uint32_t*>(b_hi + o);
      bl[q] = *reinterpret_cast<const uint32_t*>(b_lo + o);
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float p[4] = {0.f, 0.f, 0.f, 0.f};
      if (a_has_lo) mma_16x8x8(p, al[mt], bh);         // small cross terms first
      mma_16x8x8(p, ah[mt], bl);
      mma_16x8x8(p, ah[mt], bh);
#pragma unroll
      for (int e = 0; e < 4; ++e) sum[mt][nt][e] += p[e];
    }
  }
}

// One warp's share of one k-step of 8 reduction elements: rows [m0, m0 + 16 MT) x columns [n0, n0 + 8 NT) of
//     D += Al*Bh + Ah*Bl + Ah*Bh      (Al*Bh skipped when A is exact, i.e. has no lo part: a_lo == nullptr)
// a_off(m, k) / b_off(n, k): byte offset of an element inside one part (hi or lo) of the staged operand, so any
// shared-memory arrangement (K-major or MN-major, swizzled or not) is read as it landed.  The tensor core adds into
// its fp32 accumulator with round-towards-zero, so the three products of a k-step are formed from zero and added
// into `sum` with an ordinary round-to-nearest add.
template <int MT, int NT, class AOff, class BOff>
__device__ __forceinline__ void warp_kstep_3xtf32(float (&sum)[MT][NT][4], const uint8_t* a_hi, const uint8_t* a_lo,
                                                  const uint8_t* b_hi, const uint8_t* b_lo, int m0, int n0, int k0,
                                                  AOff a_off, BOff b_off) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  uint32_t ah[MT][4], al[MT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t o = a_off(m0 + mt * 16 + g + (q & 1) * 8, k0 + t + (q >> 1) * 4);
      ah[mt][q] = *reinterpret_cast<const uint32_t*>(a_hi + o);
      al[mt][q] = a_lo ? *reinterpret_cast<const uint32_t*>(a_lo + o) : 0u;
    }
  }
  warp_mma_3xtf32<MT, NT>(sum, ah, al, a_lo != nullptr, b_hi, b_lo, n0, k0, b_off);
}

// ---- warpgroup MMA (wgmma, sm_90a) on K-major SWIZZLE_128B operands -----------------------------------------------
// Shared-memory matrix descriptor of a K-major SWIZZLE_128B tile (the layout the TMA loads leave): 128-byte rows, groups
// of 8 rows 1024 bytes apart (stride byte offset), 1024-byte aligned tile.  The leading byte offset is unused by this
// layout.  A k-step of 8 tf32 elements further along the rows is the same descriptor with the start address 32 bytes on
// (the swizzle is a function of the absolute address bits, as for the TMA unit that wrote the tile).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Pins the accumulator registers between the asynchronous MMAs and ordinary register accesses (the compiler must not
// move reads of d across a wgmma_wait, nor writes of d across an MMA issue).
template <int NA>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[NA]) {
#pragma unroll
  for (int e = 0; e < NA; ++e) asm volatile("" : "+f"(d[e])::"memory");
}

// D (m64 x N, fp32) = A * B^T (+ D when scale_d != 0), A: 64 x 8, B: N x 8, both tf32 from shared-memory descriptors.
// Per thread: d[4 i + 2 h + e] = D[16 w + g + 8 h][8 i + 2 t + e], w = warp of the warpgroup, g = lane / 4, t = lane % 4.
__device__ __forceinline__ void wgmma_m64k8(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64k8(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

// Issues one k-step of 8 of the error-compensated product of a warpgroup's m64 x N tile as one wgmma group,
//     d = Al*Bh, d += Ah*Bl, d += Ah*Bh        (the order and the zero start of warp_kstep_3xtf32)
// from K-major SWIZZLE_128B hi/lo tiles at shared addresses a_hi / a_lo / b_hi / b_lo; k0: first reduction element.
// The caller retires the group with wgmma_wait and adds d into its fp32 sums with round-to-nearest adds.
template <int NA>
__device__ __forceinline__ void wgmma_kstep_3xtf32(float (&d)[NA], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, int k0) {
  const uint32_t ko = (uint32_t)k0 * 4u;
  const uint64_t ah = wgmma_desc_sw128(a_hi + ko), al = wgmma_desc_sw128(a_lo + ko);
  const uint64_t bh = wgmma_desc_sw128(b_hi + ko), bl = wgmma_desc_sw128(b_lo + ko);
  wgmma_fence_acc(d);
  wgmma_fence();
  wgmma_m64k8(d, al, bh, 0);                        // small cross terms first, from zero
  wgmma_m64k8(d, ah, bl, 1);
  wgmma_m64k8(d, ah, bh, 1);
  wgmma_commit();
  wgmma_fence_acc(d);
}

// D (m64 x 32, fp32) = A * B^T (+ D when scale_d != 0) with A from registers: the warp's 16 rows of the warpgroup's
// 64, a = {A[g][t], A[g + 8][t], A[g][t + 4], A[g + 8][t + 4]} (g = lane / 4, t = lane % 4, the m16n8k8 A layout).
__device__ __forceinline__ void wgmma_m64k8(float (&d)[16], const uint32_t (&a)[4], uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// One k-step of 8 as one wgmma group when A is exact (no lo part) and held in registers:  d = A*Bl, d += A*Bh — the
// products and order of warp_mma_3xtf32 with a_has_lo = false.  B: K-major SWIZZLE_128B hi/lo tiles at shared
// addresses b_hi / b_lo, k0: first reduction element.  The caller keeps `a` unchanged until the group is retired.
__device__ __forceinline__ void wgmma_kstep_exact_a(float (&d)[16], const uint32_t (&a)[4], uint32_t b_hi, uint32_t b_lo, int k0) {
  const uint32_t ko = (uint32_t)k0 * 4u;
  const uint64_t bh = wgmma_desc_sw128(b_hi + ko), bl = wgmma_desc_sw128(b_lo + ko);
  wgmma_fence_acc(d);
  wgmma_fence();
  wgmma_m64k8(d, a, bl, 0);
  wgmma_m64k8(d, a, bh, 1);
  wgmma_commit();
  wgmma_fence_acc(d);
}

// Row / column of D that element e of fragment (mt, nt) of warp_kstep_3xtf32 holds, relative to (m0, n0).
__device__ __forceinline__ int frag_row(int mt, int e) { return mt * 16 + ((threadIdx.x & 31) >> 2) + (e >> 1) * 8; }
__device__ __forceinline__ int frag_col(int nt, int e) { return nt * 8 + 2 * (threadIdx.x & 3) + (e & 1); }

// Byte offsets inside SWIZZLE_128B tiles (1024-byte aligned, 128-byte rows, 16-byte chunk c of row r stored at c ^ (r & 7)):
//   K-major : row = MN index, 32 reduction elements per row
//   MN-major: row = reduction index, 32 MN indices per row, 32-wide MN slabs `lbo` bytes apart
__device__ __forceinline__ uint32_t sw128_kmajor(int mn, int k) {
  return (uint32_t)(mn * 128 + ((((k >> 2) ^ mn) & 7) << 4) + ((k & 3) << 2));
}
__device__ __forceinline__ uint32_t sw128_mnmajor(int mn, int k, uint32_t lbo) {
  return (uint32_t)(mn >> 5) * lbo + (uint32_t)(k * 128 + (((((mn & 31) >> 2) ^ k) & 7) << 4) + ((mn & 3) << 2));
}

// hi = rn_tf32(x), lo = rn_tf32(x - hi): round-to-nearest on both keeps the split error zero-mean
// (a truncating split biases every product towards zero).
__device__ __forceinline__ float rn_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = rn_tf32(x);
  lo = rn_tf32(x - hi);
}
__device__ __forceinline__ void split_tf32(const float4& x, float4& hi, float4& lo) {
  split_tf32(x.x, hi.x, lo.x);
  split_tf32(x.y, hi.y, lo.y);
  split_tf32(x.z, hi.z, lo.z);
  split_tf32(x.w, hi.w, lo.w);
}

// 4x4 transpose across the 4 lanes of an aligned lane quad: on entry lane e holds S[r0+e][b..b+3],
// on exit it holds (S[r0+0..3][b+e]).  Round s: lane R receives from lane (R+s)%4 its component R.
__device__ __forceinline__ float pick(const float4& v, int k) { return k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w)); }
__device__ __forceinline__ float4 quad_transpose(float4 v, int lane) {
  const int e = lane & 3, base = lane & ~3;
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int src = (e + s) & 3;
    float send = pick(v, (e - s) & 3);                 // sender S sends component (S - s) mod 4 == the receiver's index
    float got = __shfl_sync(0xffffffffu, send, base + src);
    r.x = src == 0 ? got : r.x;                        // came from lane S = (e+s)%4 -> reduction element r0+S
    r.y = src == 1 ? got : r.y;
    r.z = src == 2 ? got : r.z;
    r.w = src == 3 ? got : r.w;
  }
  return r;
}

}  // namespace tc
}  // namespace dz
