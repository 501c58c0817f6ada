// Torso (conv1-3) and 3136 -> 512 layer(s) of the batch-32 learner step on the TMA-fed tensor-core kernels.
//   networks.py:181-204 dqn_torso, :82-103 conv, :207-221 dqn_value_head, :137-178 noisy_linear, :224-261 rainbow
// Data flow (all activations are stored once as tf32 hi/lo pairs by the producing epilogue, plus an fp32 copy
// for the layers that are still on the FMA kernels):
//
//   rows (uint8, replay store) --bulk copy--> smem --convert--> conv1 MMA --> act1 {hi,lo,f32} [P*B][h1][w1][32]
//   act1 --TMA im2col boxes--> conv2 MMA --> act2 [P*B][h2][w2][64] --TMA--> conv3 MMA --> act3 = features [P*B][feat]
//   W (fp32, [feat][512]) --TMA, once per blob--> smem --hi/lo split in registers--> MN-major MMA x act3 (every pass
//        applying the blob) --> split-K partials --> finish --> h1
//   dh1 --> W (K-major) MMA --> partials --> finish (ReLU mask) --> dact3 --TMA (zero-filled halo)--> conv3 dgrad --> dact2
//        --> conv2 dgrad (4 stride-parity classes) --> dact1
#include <algorithm>

#include "dz_umma_net.cuh"

namespace dz {

// The plan's launches.  tag: the name dz_test_learner_trace and dz_test_learner_mma_path take; noisy: the name the fc
// launches run under for noisy layers (profiles, timelines), which the MMA-path hook accepts as well.
enum NetLaunch : int { kConv2Fwd, kConv3Fwd, kConv3Dgrad, kConv2Dgrad, kFcFwd, kFcDgrad, kConv3Wgrad, kConv2Wgrad, kNumNetLaunches };
struct NetLaunchName { const char* tag; const char* noisy; };
constexpr NetLaunchName kNetLaunchNames[kNumNetLaunches] = {
    {"conv2_fwd", nullptr},   {"conv3_fwd", nullptr},    {"conv3_dgrad", nullptr}, {"conv2_dgrad", nullptr},
    {"fc1_fwd", "noisy1_fwd"}, {"fc1_dgrad", "noisy1_dgrad"}, {"conv3_wgrad", nullptr}, {"conv2_wgrad", nullptr}};

// Conv layers 1..3 as GEMMs: N output channels x K = (kh, kw, input channel) reduction.  um_pack_conv_kernel states the
// same shapes.  The input-gradient images of conv3 and conv2 are rearrangements of W3 and W2 (as many floats).
constexpr int kConvN[3] = {32, 64, 64}, kConvK[3] = {256, 512, 576};
constexpr int kConvFwdFloats = kConvN[0] * kConvK[0] + kConvN[1] * kConvK[1] + kConvN[2] * kConvK[2];   // per blob

struct UmNet {
  UmNetDesc d;
  int h1, w1, h2, w2, h3, w3, feat, PB;
  UmPlan plan;
  // activations / gradients
  float *act_hi[3], *act_lo[3], *act_f32[3];     // layer 1..3, all passes stacked
  float *dact_hi[3], *dact_lo[3], *dact_f32[3];  // layer 1..3 (pass 0)
  float *h1_buf, *dh1_f32, *dh1_hi, *dh1_lo;
  float *fc_part, *fcd_part;
  int fc_splits, fcd_splits, fc_nprob, fcd_nsrc;
  // conv weight images: [blob][layer] K-major [N][K]; dgrad images (online)
  float *wf_hi[2][3], *wf_lo[2][3], *wd3_hi, *wd3_lo, *wd2_hi, *wd2_lo;
  int map_wf1[2][2];                              // [blob][hi/lo] for the conv1 kernel
  UmLaunch launches[kNumNetLaunches];
  float *wg3_part, *wg2_part, *wg1_part;   // conv3 / conv2 weight-gradient split partials [S][K][64]; conv1: one [256][32] per CTA
  int wg3_splits, wg2_splits, wg1_ctas;
  int map_g1[2];                           // dact1 hi / lo as a flat [B*h1*w1][32] tensor
  float* wg_scratch;                       // bias-gradient chunk sums [3][kWgMaxChunks][64]
  unsigned int* wg_ticket;                 // [4]
  int conv1_stag_bytes, conv1_tiles_per_pass;
  // noise-dependent problem fields (patched when the caller's noise buffer moves)
  struct Patch { int prob; int field; int64_t off; };   // field 0: A.scale_r, 2: A.scale_i, 1: scale_i (epilogue)
  std::vector<Patch> patches;
  const float* noise_cached = nullptr;
  std::string trace_tag;                   // debug: the launch with this tag writes CTA 0's clock stamps to trace_ptr
  long long* trace_ptr = nullptr;
  long long* tr(const char* tag) const { return trace_ptr && trace_tag == tag ? trace_ptr : nullptr; }
  bool fc_per_pass = false;                // tests only: fc forward CTA groups per pass (the umma_gemm_kernel layout)
};

namespace {

using namespace um;

// ------------------------------------------------------------------------------------------------
// Conv weight images: K-major [N][K] tf32 hi/lo for the forward GEMMs (conv1 carries the 1/255 of networks.py:193),
// and the input-gradient arrangements  Wd3[c][(kh,kw,n)] = W3[kh,kw,c,n],  Wd2[py,px][c][(ay,ax,n)] = W2[py+2ay,px+2ax,c,n].
// ------------------------------------------------------------------------------------------------
struct PackArgs {
  const float* blob[2];
  int64_t off_w[3];
  float* wf_hi[2][3]; float* wf_lo[2][3];
  float *wd3_hi, *wd3_lo, *wd2_hi, *wd2_lo;
};

__global__ void __launch_bounds__(256) um_pack_conv_kernel(const __grid_constant__ PackArgs a) {
  dz::pdl_enter();
  constexpr int kN[3] = {32, 64, 64}, kK[3] = {256, 512, 576};
  constexpr int kFwd = 32 * 256 + 64 * 512 + 64 * 576;   // 77824 per blob
  int e = blockIdx.x * 256 + threadIdx.x;
  float v;
  float *hi, *lo;
  if (e < 2 * kFwd) {
    const int b = e / kFwd;
    int r = e - b * kFwd;
    int L = 0;
    if (r >= kN[0] * kK[0]) { r -= kN[0] * kK[0]; L = 1; if (r >= kN[1] * kK[1]) { r -= kN[1] * kK[1]; L = 2; } }
    const int n = r / kK[L], k = r - n * kK[L];
    v = a.blob[b][a.off_w[L] + (int64_t)k * kN[L] + n];
    if (L == 0) v *= 0.0039215688593685627f;   // fl32(1/255): raw bytes are the (exact) MMA operand
    hi = a.wf_hi[b][L] + r; lo = a.wf_lo[b][L] + r;
  } else {
    e -= 2 * kFwd;
    if (e < 64 * 576) {                         // Wd3[c][(kh*3+kw)*64 + n]
      const int c = e / 576, r = e - c * 576, t = r >> 6, n = r & 63;
      v = a.blob[0][a.off_w[2] + ((int64_t)t * 64 + c) * 64 + n];
      hi = a.wd3_hi + e; lo = a.wd3_lo + e;
    } else {
      e -= 64 * 576;
      if (e >= 4 * 32 * 256) return;            // Wd2[(py*2+px)*32 + c][(ay*2+ax)*64 + n]
      const int row = e >> 8, r = e & 255, cls = row >> 5, c = row & 31, py = cls >> 1, px = cls & 1;
      const int t = r >> 6, n = r & 63, ay = t >> 1, ax = t & 1;
      const int kh = py + 2 * ay, kw = px + 2 * ax;
      v = a.blob[0][a.off_w[1] + ((int64_t)(kh * 4 + kw) * 32 + c) * 64 + n];
      hi = a.wd2_hi + e; lo = a.wd2_lo + e;
    }
  }
  float h, l;
  split_tf32(v, h, l);
  *hi = h;
  *lo = l;
}

// ------------------------------------------------------------------------------------------------
// conv1: 8x8 stride 4 over the sampled uint8 observations, read IN PLACE from the replay store (the gather of
// replay.py:718-722 is this kernel's operand load).  Per 128-pixel output tile: one thread bulk-copies the
// contiguous input rows the tile needs (cp.async.bulk, <= 4 segments) into a double-buffered staging area; the
// bytes become exact tf32 values (K = 256 = 8 kernel rows x 32 (kw, c)) that the MMA warps multiply with the resident
// weight image (hi/lo); the bias, ReLU and tf32 hi/lo split of act1 follow.  conv1_wgmma_kernel (the learner's) forms
// the A fragments from the staged bytes in the registers of two MMA warpgroups; conv1_umma_kernel, with eight
// converter warps writing a swizzled A tile for four warps' mma.sync, is kept as the reference it is tested against
// bit for bit (dz_test_conv1_forward).
// ------------------------------------------------------------------------------------------------
struct Conv1Args {
  CUtensorMap wmap[2][2];          // weight image [blob][hi / lo] (grid-constant: descriptor fetch from the constant bank)
  const uint8_t* const* rows[3];
  const float* bias[3];
  int blob[3];
  float *out_hi, *out_lo, *out_f32;
  int npass, B, W, oh, ow, m_pass, tiles_per_pass, ntiles, stag_bytes;
  long long* trace;                // debug: clock stamps of CTA 0
};

constexpr int kC1W = 65536, kC1A = 131072;

// Staging of the uint8 input rows.  For output-pixel tile [m0, m1), every image b the tile touches gets one segment of
// the staging buffer, in image order: the contiguous input rows its output rows of the tile read (8x8 kernel, stride 4),
// starting at input row `row0`.  px: output pixels per image, ow: output width, row_bytes: one input row.
struct Conv1Segment { int row0, bytes; };
__host__ __device__ __forceinline__ Conv1Segment conv1_segment(int b, int m0, int m1, int px, int ow, int row_bytes) {
  const int plo = max(m0, b * px) - b * px, phi = min(m1, (b + 1) * px) - b * px;
  const int oy0 = plo / ow;
  return {4 * oy0, (4 * ((phi - 1) / ow - oy0) + 8) * row_bytes};
}

// Producer: bulk-copies the segments of tile [m0, m1) from the images' row pointers to `dst`, completing on `bar`.
__device__ __forceinline__ void conv1_stage_tile(const uint8_t* const* rows, int m0, int m1, int px, int ow, int row_bytes,
                                                 uint32_t dst, uint64_t* bar) {
  const int b0 = m0 / px, b1 = (m1 - 1) / px;
  uint32_t total = 0;
  for (int b = b0; b <= b1; ++b) total += (uint32_t)conv1_segment(b, m0, m1, px, ow, row_bytes).bytes;
  mbar_expect_tx(bar, total);
  for (int b = b0; b <= b1; ++b) {
    const Conv1Segment seg = conv1_segment(b, m0, m1, px, ow, row_bytes);
    bulk_g2s(dst, rows[b] + (size_t)seg.row0 * row_bytes, (uint32_t)seg.bytes, bar);
    dst += (uint32_t)seg.bytes;
  }
}

// Converter: byte offset inside the staged tile [m0, m1) of the top-left input pixel of output pixel m's window.
__device__ __forceinline__ int conv1_stage_offset(int m, int m0, int m1, int px, int ow, int row_bytes) {
  const int b = m / px, p = m - b * px, oy = p / ow, ox = p - oy * ow;
  int off = 0;
  for (int bb = m0 / px; bb < b; ++bb) off += conv1_segment(bb, m0, m1, px, ow, row_bytes).bytes;
  return off + (4 * oy - conv1_segment(b, m0, m1, px, ow, row_bytes).row0) * row_bytes + 16 * ox;
}

// Converter: one staged 32-byte kernel row (8 pixels x 4 channels) of tile row r, zeros when the row is beyond the batch ...
__device__ __forceinline__ void conv1_load_row(const uint8_t* src, bool valid, uint4 (&u)[2]) {
  if (valid) {
    u[0] = *reinterpret_cast<const uint4*>(src);
    u[1] = *reinterpret_cast<const uint4*>(src + 16);
  } else {
    u[0] = make_uint4(0, 0, 0, 0); u[1] = u[0];
  }
}
// ... expanded to exact floats into row r of kernel row kh's slab of the swizzled K-major A tile [8 kh][128 r][32 (kw, c)].
__device__ __forceinline__ void conv1_expand_row(const uint4 (&u)[2], uint8_t* a_tile, int kh, int r) {
  uint8_t* dstrow = a_tile + kh * 16384 + r * 128;
  const uint32_t w[8] = {u[0].x, u[0].y, u[0].z, u[0].w, u[1].x, u[1].y, u[1].z, u[1].w};
#pragma unroll
  for (int kw = 0; kw < 8; ++kw) {
    // 0x4B000000 | byte = 8388608 + byte exactly; subtracting 2^23 leaves the byte as a float (an exact tf32 number)
    float4 f;
    f.x = __uint_as_float(__byte_perm(w[kw], 0x4B000000u, 0x7440)) - 8388608.0f;
    f.y = __uint_as_float(__byte_perm(w[kw], 0x4B000000u, 0x7441)) - 8388608.0f;
    f.z = __uint_as_float(__byte_perm(w[kw], 0x4B000000u, 0x7442)) - 8388608.0f;
    f.w = __uint_as_float(__byte_perm(w[kw], 0x4B000000u, 0x7443)) - 8388608.0f;
    *reinterpret_cast<float4*>(dstrow + ((kw ^ (r & 7)) << 4)) = f;
  }
}

__global__ void __launch_bounds__(kThreadsU, 1) conv1_umma_kernel(const __grid_constant__ Conv1Args a) {
  if (threadIdx.x < 4) prefetch_tensormap(&a.wmap[threadIdx.x >> 1][threadIdx.x & 1]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem);   // [2] staged input rows landed
  uint64_t* raw_empty = raw_full + 2;                        // [2] converters are done reading them
  uint64_t* w_full = raw_empty + 2;                          // [1] weight image landed (only reloaded when the pass changes)
  uint64_t* a_ready = w_full + 1;                            // [4] kernel-row pair (2j, 2j+1) of the A tile converted
  uint64_t* a_empty = a_ready + 4;                           // [4] ... consumed by the four MMA warps
  uint8_t* w_smem = smem + 1024;
  uint8_t* a_smem = w_smem + kC1W;
  uint8_t* stag = a_smem + kC1A;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(&raw_full[b], 1); mbar_init(&raw_empty[b], kConvWarps); }
    for (int j = 0; j < 4; ++j) { mbar_init(&a_ready[j], kConvWarps); mbar_init(&a_empty[j], 4); }
    mbar_init(w_full, 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  dz::pdl_enter();                        // set-up above overlaps the previous kernel's tail; data accesses start here
  const bool tr = a.trace != nullptr && blockIdx.x == 0;
  if (tr && threadIdx.x == 0) { a.trace[323] = clock64(); a.trace[324] = clock64(); }

  const int px = a.oh * a.ow;             // output pixels per image
  const int row_bytes = a.W * 4;          // one input row of 4-channel pixels
  // consecutive tiles per CTA: the weight image is reloaded only when the pass (online / target parameters) changes
  const int t_begin = (int)(((long long)blockIdx.x * a.ntiles) / gridDim.x);
  const int t_end = (int)(((long long)(blockIdx.x + 1) * a.ntiles) / gridDim.x);

  if (warp == 0) {
    // ---------------------------------------------------------------- producer
    int cur_pass = -1;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int pass = tile / a.tiles_per_pass;
      const int m0 = (tile - pass * a.tiles_per_pass) * 128, m1 = min(m0 + 128, a.m_pass);
      mbar_wait(&raw_empty[buf], (((uint32_t)n >> 1) & 1u) ^ 1u);
      if (elect_one()) {
        conv1_stage_tile(a.rows[pass], m0, m1, px, a.ow, row_bytes, smem_u32(stag + (size_t)buf * a.stag_bytes), &raw_full[buf]);
        if (tr && n < 64) a.trace[n] = clock64();                                                   // [0,64): row copies issued
      }
      __syncwarp();
      if (pass != cur_pass) {
        if (n > 0) mbar_wait(&a_empty[3], ((uint32_t)(n - 1)) & 1u);   // previous tile's MMAs are done with the old image
        if (elect_one()) {
          mbar_expect_tx(w_full, (uint32_t)kC1W);
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            const int part = q >> 3, s = q & 7;
            tma_load_5d(smem_u32(w_smem) + part * 32768 + s * 4096, &a.wmap[a.blob[pass]][part], w_full, 32 * s, 0, 0, 0, 0);
          }
        }
        cur_pass = pass;
      }
      __syncwarp();
    }
  } else if (warp >= 2 && warp < 6) {
    // ---------------------------------------------------------------- MMA + epilogue: D rows [32 q, 32 q + 32) of the tile
    // A (exact tf32 bytes) slab kh = [128 pixels][32 (kw, c)], W slab kh = [32 n][32 (kw, c)] hi | lo, both K-major.
    const int q = warp - 2, mw0 = q * 32;
    auto kmaj = [](int mn, int k) { return sw128_kmajor(mn, k); };
    int cur_pass = -1, wn = 0;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int pass = tile / a.tiles_per_pass;
      const int m0 = (tile - pass * a.tiles_per_pass) * 128, m1 = min(m0 + 128, a.m_pass);
      if (pass != cur_pass) { mbar_wait(w_full, (uint32_t)wn & 1u); ++wn; cur_pass = pass; }
      float sum[2][4][4];
      {   // the bias is the initial value of the sums
        const float* __restrict__ bias = a.bias[pass];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const float2 b2 = *reinterpret_cast<const float2*>(bias + frag_col(nt, 0));
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) { sum[mt][nt][0] = b2.x; sum[mt][nt][1] = b2.y; sum[mt][nt][2] = b2.x; sum[mt][nt][3] = b2.y; }
        }
      }
      for (int slab = 0; slab < 8; ++slab) {
        if ((slab & 1) == 0) mbar_wait(&a_ready[slab >> 1], (uint32_t)n & 1u);
        const uint8_t* as = a_smem + slab * 16384;
        const uint8_t* ws = w_smem + slab * 4096;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          warp_kstep_3xtf32<2, 4>(sum, as, nullptr, ws, ws + 32768, mw0, 0, 8 * k, kmaj, kmaj);
        if (slab & 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_empty[slab >> 1]);
        }
      }
      if (q == 0 && lane == 0 && tile == t_end - 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
      if (tr && warp == 2 && lane == 0 && n < 64) a.trace[192 + n] = clock64();                     // [192,256): tile's MMAs done
      // The warp's 32 rows x 32 channels are ONE contiguous 4 KB block of act1; every store instruction writes eight rows
      // x 32 contiguous bytes (full sectors).
      const long long dst0 = ((long long)pass * a.m_pass + m0 + mw0) * 32;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; e += 2) {
          const int row = frag_row(mt, e);
          if (m0 + mw0 + row >= m1) continue;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const float v0 = fmaxf(sum[mt][nt][e], 0.f), v1 = fmaxf(sum[mt][nt][e + 1], 0.f);
            float h0, l0, h1, l1;
            split_tf32(v0, h0, l0);
            split_tf32(v1, h1, l1);
            const long long o = dst0 + row * 32 + frag_col(nt, e);
            *reinterpret_cast<float2*>(a.out_hi + o) = make_float2(h0, h1);
            *reinterpret_cast<float2*>(a.out_lo + o) = make_float2(l0, l1);
          }
        }
      if (tr && warp == 2 && lane == 0 && n < 64) a.trace[256 + n] = clock64();                     // [256,320): tile stored
    }
    if (t_begin >= t_end && q == 0 && lane == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  } else if (warp >= 6) {
    // ---------------------------------------------------------------- converters: uint8 rows -> exact tf32 A tile
    const int ct = threadIdx.x - 6 * 32;
    const int r = ct & 127, khp = ct >> 7;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int pass = tile / a.tiles_per_pass;
      const int m0 = (tile - pass * a.tiles_per_pass) * 128, m1 = min(m0 + 128, a.m_pass);
      const int m = m0 + r;
      const bool valid = m < m1;
      const int src_off = valid ? conv1_stage_offset(m, m0, m1, px, a.ow, row_bytes) : 0;
      mbar_wait(&raw_full[buf], ((uint32_t)n >> 1) & 1u);
      if (tr && ct == 0 && n < 64) a.trace[64 + n] = clock64();                                     // [64,128): input rows landed
      const uint8_t* src = stag + (size_t)buf * a.stag_bytes + src_off;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int kh = 2 * it + khp;
        uint4 u[2];
        conv1_load_row(src + kh * row_bytes, valid, u);
        mbar_wait(&a_empty[it], ((uint32_t)n & 1u) ^ 1u);     // the previous tile's MMAs have consumed this kernel-row pair
        conv1_expand_row(u, a_smem, kh, r);
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_ready[it]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&raw_empty[buf]);
    }
  }
  if (tr && threadIdx.x == 0) a.trace[322] = clock64();
}

// Warpgroup-MMA conv1.  Producer (row copies, weight image), weight-image layout, epilogue, PDL points and clock-stamp
// slots are those of conv1_umma_kernel; there are no converter warps and no A tile in shared memory.  Warp roles:
// 0 producer | 1 barrier set-up | 2-3 idle | warpgroup 1 (warps 4-7) D rows [0, 64) of the tile, warpgroup 2 (warps
// 8-11) rows [64, 128), all 32 channels.
constexpr int kThreadsC1W = 12 * 32;
// Scratch accumulators a warpgroup rotates through (one MMA group each), as wgmma_gemm_kernel's acc0 / acc1.  Four
// measured no faster than two in the in-graph tile trace.
constexpr int kC1Groups = 2;

__global__ void __launch_bounds__(kThreadsC1W, 1) conv1_wgmma_kernel(const __grid_constant__ Conv1Args a) {
  if (threadIdx.x < 4) prefetch_tensormap(&a.wmap[threadIdx.x >> 1][threadIdx.x & 1]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem);   // [2] staged input rows landed
  uint64_t* raw_empty = raw_full + 2;                        // [2] the 8 MMA warps retired every group of the tile staged there
  uint64_t* w_full = raw_empty + 2;                          // [1] weight image landed (only reloaded when the pass changes)
  uint8_t* w_smem = smem + 1024;
  uint8_t* stag = w_smem + kC1W;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(&raw_full[b], 1); mbar_init(&raw_empty[b], kConsumerWarps); }
    mbar_init(w_full, 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  dz::pdl_enter();                        // set-up above overlaps the previous kernel's tail; data accesses start here
  const bool tr = a.trace != nullptr && blockIdx.x == 0;
  if (tr && threadIdx.x == 0) { a.trace[323] = clock64(); a.trace[324] = clock64(); }

  const int px = a.oh * a.ow;             // output pixels per image
  const int row_bytes = a.W * 4;          // one input row of 4-channel pixels
  const int t_begin = (int)(((long long)blockIdx.x * a.ntiles) / gridDim.x);
  const int t_end = (int)(((long long)(blockIdx.x + 1) * a.ntiles) / gridDim.x);

  if (warp == 0) {
    // ---------------------------------------------------------------- producer
    int cur_pass = -1;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int pass = tile / a.tiles_per_pass;
      const int m0 = (tile - pass * a.tiles_per_pass) * 128, m1 = min(m0 + 128, a.m_pass);
      mbar_wait(&raw_empty[buf], (((uint32_t)n >> 1) & 1u) ^ 1u);
      if (elect_one()) {
        conv1_stage_tile(a.rows[pass], m0, m1, px, a.ow, row_bytes, smem_u32(stag + (size_t)buf * a.stag_bytes), &raw_full[buf]);
        if (tr && n < 64) a.trace[n] = clock64();                                                   // [0,64): row copies issued
      }
      __syncwarp();
      if (pass != cur_pass) {
        // the previous tile's MMAs are done with the old image
        if (n > 0) mbar_wait(&raw_empty[(n - 1) & 1], ((uint32_t)(n - 1) >> 1) & 1u);
        if (elect_one()) {
          mbar_expect_tx(w_full, (uint32_t)kC1W);
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            const int part = q >> 3, s = q & 7;
            tma_load_5d(smem_u32(w_smem) + part * 32768 + s * 4096, &a.wmap[a.blob[pass]][part], w_full, 32 * s, 0, 0, 0, 0);
          }
        }
        cur_pass = pass;
      }
      __syncwarp();
    }
  } else if (warp >= 4) {
    // ---------------------------------------------------------------- MMA warpgroups + epilogue
    // Warpgroup wg: D rows [64 wg, 64 wg + 64) of the tile; this warp's rows r0 and r0 + 8 (plus lane / 4).  A comes
    // from registers: for kernel row kh, thread (g, t) reads the two staged 32-byte kernel rows (8 pixels x 4 channels)
    // of its output pixels and expands byte t of every pixel to an exact float.  k-step s of kernel row kh covers
    // (kw, c) = (2s, 0..3), (2s + 1, 0..3), so a = {X[r0][2s][t], X[r0 + 8][2s][t], X[r0][2s + 1][t], X[r0 + 8][2s + 1][t]}:
    // the wgmma A fragment.  W slab kh = [32 n][32 (kw, c)] at w_smem + 4096 kh, hi | lo 32 KB apart, K-major
    // SWIZZLE_128B, is read through descriptors.  Every k-step is one group into a scratch accumulator; kC1Groups of them
    // rotate, and k-step k is retired (wgmma_wait) and added into the sums once k + kC1Groups - 1 has been issued, so
    // the sums still take the k-steps in order.  The A registers of kernel rows kh and kh + 1 are separate, and every
    // group of kernel row kh - 1 is retired before row kh + 1 is expanded, so no group in flight reads a register
    // being written.  A tile's 32 k-steps are straight-line code and its last group is retired
    // before raw_empty, so no group is in flight across a barrier wait, a branch or a loop edge.  The values the loop
    // branches on are broadcast from lane 0 so that ptxas sees them warp-uniform.
    const int wg = __shfl_sync(0xffffffffu, (warp >> 2) - 1, 0);
    const bool lead = warp == 4 && lane == 0;
    const uint32_t w_base = smem_u32(w_smem);
    const int t = lane & 3, c0 = 2 * t;
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const uint32_t sel = 0x7440u + (uint32_t)t;   // byte t of a word -> low byte of 0x4B0000xx
    float acc[kC1Groups][16];
#pragma unroll
    for (int q = 0; q < kC1Groups; ++q)
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[q][e] = 0.f;
    int cur_pass = -1, wn = 0;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int pass = tile / a.tiles_per_pass;
      const int m0 = (tile - pass * a.tiles_per_pass) * 128, m1 = min(m0 + 128, a.m_pass);
      // an m64 half with no valid pixel issues no MMAs (it still releases the staging buffer)
      const bool active = __shfl_sync(0xffffffffu, (int)(m0 + 64 * wg < m1), 0) != 0;
      // staged offsets of this thread's two pixels; a pixel beyond the batch reads offset 0 and is masked to zeros
      const int ma = m0 + r0, mb = ma + 8;
      const uint32_t mask_a = ma < m1 ? 0xffffffffu : 0u, mask_b = mb < m1 ? 0xffffffffu : 0u;
      const int off_a = ma < m1 ? conv1_stage_offset(ma, m0, m1, px, a.ow, row_bytes) : 0;
      const int off_b = mb < m1 ? conv1_stage_offset(mb, m0, m1, px, a.ow, row_bytes) : 0;
      if (pass != cur_pass) { mbar_wait(w_full, (uint32_t)wn & 1u); ++wn; cur_pass = pass; }
      float sum[16];
      {   // the bias is the initial value of the sums
        const float* __restrict__ bias = a.bias[pass];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 b2 = *reinterpret_cast<const float2*>(bias + 8 * i + c0);
#pragma unroll
          for (int h = 0; h < 2; ++h) { sum[4 * i + 2 * h] = b2.x; sum[4 * i + 2 * h + 1] = b2.y; }
        }
      }
      auto retire = [&](float (&d)[16]) {
        wgmma_fence_acc(d);
#pragma unroll
        for (int e = 0; e < 16; ++e) sum[e] += d[e];
      };
      mbar_wait(&raw_full[buf], ((uint32_t)n >> 1) & 1u);
      if (tr && lead && n < 64) a.trace[64 + n] = clock64();                                       // [64,128): input rows landed
      if (active) {
        const uint8_t* src_a = stag + (size_t)buf * a.stag_bytes + off_a;
        const uint8_t* src_b = stag + (size_t)buf * a.stag_bytes + off_b;
        uint32_t x[2][4][4];   // [kh & 1][k-step][fragment element]
#pragma unroll
        for (int kh = 0; kh < 8; ++kh) {
          const uint4 ua0 = *reinterpret_cast<const uint4*>(src_a + kh * row_bytes);
          const uint4 ua1 = *reinterpret_cast<const uint4*>(src_a + kh * row_bytes + 16);
          const uint4 ub0 = *reinterpret_cast<const uint4*>(src_b + kh * row_bytes);
          const uint4 ub1 = *reinterpret_cast<const uint4*>(src_b + kh * row_bytes + 16);
          const uint32_t wa[8] = {ua0.x, ua0.y, ua0.z, ua0.w, ua1.x, ua1.y, ua1.z, ua1.w};
          const uint32_t wb[8] = {ub0.x, ub0.y, ub0.z, ub0.w, ub1.x, ub1.y, ub1.z, ub1.w};
          // 0x4B000000 | byte = 8388608 + byte exactly; subtracting 2^23 leaves the byte as a float (an exact tf32 number)
          auto expand = [&](uint32_t w, uint32_t mask) {
            return __float_as_uint(__uint_as_float(__byte_perm(w & mask, 0x4B000000u, sel)) - 8388608.0f);
          };
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            x[kh & 1][s][0] = expand(wa[2 * s], mask_a);
            x[kh & 1][s][1] = expand(wb[2 * s], mask_b);
            x[kh & 1][s][2] = expand(wa[2 * s + 1], mask_a);
            x[kh & 1][s][3] = expand(wb[2 * s + 1], mask_b);
          }
          const uint32_t w = w_base + 4096u * (uint32_t)kh;
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            const int ks = 4 * kh + s;
            wgmma_kstep_exact_a(acc[ks % kC1Groups], x[kh & 1][s], w, w + 32768u, 8 * s);
            if (ks >= kC1Groups - 1) {
              wgmma_wait<kC1Groups - 1>();
              retire(acc[(ks + 1) % kC1Groups]);
            }
          }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int ks = 33 - kC1Groups; ks < 32; ++ks) retire(acc[ks % kC1Groups]);
      }
      mbar_arrive_if(&raw_empty[buf], lane == 0);
      if (lead && tile == t_end - 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
      if (tr && lead && n < 64) a.trace[192 + n] = clock64();                                      // [192,256): tile's MMAs done
      // Each store instruction writes eight rows x 32 contiguous bytes of act1 (full sectors).
      const long long dst0 = ((long long)pass * a.m_pass + m0) * 32;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (m0 + row >= m1) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float v0 = fmaxf(sum[4 * i + 2 * h], 0.f), v1 = fmaxf(sum[4 * i + 2 * h + 1], 0.f);
          float h0, l0, h1, l1;
          split_tf32(v0, h0, l0);
          split_tf32(v1, h1, l1);
          const long long o = dst0 + row * 32 + 8 * i + c0;
          *reinterpret_cast<float2*>(a.out_hi + o) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(a.out_lo + o) = make_float2(l0, l1);
        }
      }
      if (tr && lead && n < 64) a.trace[256 + n] = clock64();                                      // [256,320): tile stored
    }
    if (t_begin >= t_end && lead) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }
  if (tr && threadIdx.x == 0) a.trace[322] = clock64();
}

// ------------------------------------------------------------------------------------------------
// conv1 weight gradient: dW1[k][n] = (1/255) * sum_m X[m][k] * dact1[m][n], reduction over the B * h1 * w1 output pixels of
// pass 0.  Same staging as the forward kernel (bulk-copied uint8 rows -> exact tf32 A tile); the MMA warps read the tile
// MN-major (rows = reduction index): A^T is never formed.  G = dact1 hi/lo arrives by TMA.  One partial per CTA.
// ------------------------------------------------------------------------------------------------
struct Conv1WgArgs {
  CUtensorMap gmap[2];             // dact1 hi / lo
  const uint8_t* const* rows;
  float* partial;                // [gridDim.x][256][32]
  int B, W, oh, ow, m_pass, ntiles, stag_bytes;
};

constexpr int kC1G = 32768;      // dact1 tile: hi | lo, [128 rows][32 n] each

__global__ void __launch_bounds__(kThreadsU, 1) conv1_wgrad_umma_kernel(const __grid_constant__ Conv1WgArgs a) {
  if (threadIdx.x < 2) prefetch_tensormap(&a.gmap[threadIdx.x]);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad_1024(smem_raw);
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem);   // [2]
  uint64_t* raw_empty = raw_full + 2;                        // [2]
  uint64_t* g_full = raw_empty + 2;                          // [1] dact1 tile landed
  uint64_t* a_ready = g_full + 1;                            // [4] kernel-row pairs converted
  uint64_t* t_done = a_ready + 4;                            // [1] all MMAs of the tile done (A and G tiles free)
  uint8_t* g_smem = smem + 1024;
  uint8_t* a_smem = g_smem + kC1G;
  uint8_t* stag = a_smem + kC1A;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(&raw_full[b], 1); mbar_init(&raw_empty[b], kConvWarps); }
    for (int j = 0; j < 4; ++j) mbar_init(&a_ready[j], kConvWarps);
    mbar_init(g_full, 1); mbar_init(t_done, 4);
    fence_mbarrier_init();
  }
  __syncthreads();
  dz::pdl_enter();                        // set-up above overlaps the previous kernel's tail; data accesses start here

  const int px = a.oh * a.ow;
  const int row_bytes = a.W * 4;
  const int t_begin = (int)(((long long)blockIdx.x * a.ntiles) / gridDim.x);
  const int t_end = (int)(((long long)(blockIdx.x + 1) * a.ntiles) / gridDim.x);

  if (warp == 0) {
    // ---------------------------------------------------------------- producer
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int m0 = tile * 128, m1 = min(m0 + 128, a.m_pass);
      mbar_wait(&raw_empty[buf], (((uint32_t)n >> 1) & 1u) ^ 1u);
      if (elect_one())
        conv1_stage_tile(a.rows, m0, m1, px, a.ow, row_bytes, smem_u32(stag + (size_t)buf * a.stag_bytes), &raw_full[buf]);
      __syncwarp();
      if (n > 0) mbar_wait(t_done, ((uint32_t)(n - 1)) & 1u);
      if (elect_one()) {
        mbar_expect_tx(g_full, (uint32_t)kC1G);
        tma_load_5d(smem_u32(g_smem), &a.gmap[0], g_full, 0, m0, 0, 0, 0);
        tma_load_5d(smem_u32(g_smem) + 16384, &a.gmap[1], g_full, 0, m0, 0, 0, 0);
      }
      __syncwarp();
    }
  } else if (warp >= 2 && warp < 6) {
    // ---------------------------------------------------------------- MMA warps: rows k = 128 mt + 32 q + [0, 32) of dW1
    // Both tiles are read MN-major (their rows are the reduction index m): A^T from the [8 kh][128 m][32 (kw, c)] tile,
    // G from [128 m][32 n] hi | lo.
    const int q = warp - 2;
    float sum[2][2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) sum[mt][i][nt][e] = 0.f;
    auto a_off = [](int kk, int m) { return sw128_mnmajor(kk, m, 16384u); };
    auto g_off = [](int nn, int m) { return sw128_mnmajor(nn, m, 0u); };
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      mbar_wait(g_full, (uint32_t)n & 1u);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {                      // k 0..127 (kernel rows 0-3) | k 128..255 (kernel rows 4-7)
        mbar_wait(&a_ready[2 * mt], (uint32_t)n & 1u);
        mbar_wait(&a_ready[2 * mt + 1], (uint32_t)n & 1u);
#pragma unroll 4
        for (int k = 0; k < 16; ++k)
          warp_kstep_3xtf32<2, 4>(sum[mt], a_smem, nullptr, g_smem, g_smem + 16384, mt * 128 + q * 32, 0, 8 * k, a_off, g_off);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(t_done);
      if (q == 0 && lane == 0 && tile == t_end - 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    if (t_begin >= t_end && q == 0 && lane == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const float inv255 = 0.0039215688593685627f;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 4; e += 2) {
          float* dst = a.partial + ((long long)blockIdx.x * 256 + mt * 128 + q * 32 + frag_row(i, e)) * 32;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt)
            *reinterpret_cast<float2*>(dst + frag_col(nt, e)) = make_float2(sum[mt][i][nt][e] * inv255, sum[mt][i][nt][e + 1] * inv255);
        }
  } else if (warp >= 6) {
    // ---------------------------------------------------------------- converters
    const int ct = threadIdx.x - 6 * 32;
    const int r = ct & 127, khp = ct >> 7;
    for (int tile = t_begin, n = 0; tile < t_end; ++tile, ++n) {
      const int buf = n & 1;
      const int m0 = tile * 128, m1 = min(m0 + 128, a.m_pass);
      const int m = m0 + r;
      const bool valid = m < m1;
      const int src_off = valid ? conv1_stage_offset(m, m0, m1, px, a.ow, row_bytes) : 0;   // rows beyond the batch add zeros
      mbar_wait(&raw_full[buf], ((uint32_t)n >> 1) & 1u);
      if (n > 0) mbar_wait(t_done, ((uint32_t)(n - 1)) & 1u);     // previous tile's MMAs have consumed the A tile
      const uint8_t* src = stag + (size_t)buf * a.stag_bytes + src_off;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int kh = 2 * it + khp;
        uint4 u[2];
        conv1_load_row(src + kh * row_bytes, valid, u);
        conv1_expand_row(u, a_smem, kh, r);
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_ready[it]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&raw_empty[buf]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Finish kernels of the split FC GEMMs
// ------------------------------------------------------------------------------------------------

// h1[pass][stream][m][n] = relu( sum_s P + b_mu[n] + eps_out[n] * b_sigma[n] )   (networks.py:160-178; P already holds x(Wmu + Wsigma*noise))
struct FcFinishArgs {
  const float* part; int S, B, nstream, noisy, npass;
  const float* bmu[3][2]; const float* bsig[3][2]; const float* eps_out[3][2];
  float* h1;
};

__global__ void __launch_bounds__(256) um_fc_finish_kernel(const __grid_constant__ FcFinishArgs a) {
  dz::pdl_enter();
  const int ps = blockIdx.y, pass = ps / a.nstream, st = ps - pass * a.nstream;
  const int total4 = a.B * 128;
  const long long pstride = (long long)a.B * 512;
  const float* pm = a.part + (long long)ps * a.S * pstride;
  for (int i4 = blockIdx.x * 256 + threadIdx.x; i4 < total4; i4 += gridDim.x * 256) {
    const int i = i4 << 2, n = i & 511;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < a.S; ++s) {
      const float4 x = *reinterpret_cast<const float4*>(pm + s * pstride + i);
      v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
    }
    const float4 b = *reinterpret_cast<const float4*>(a.bmu[pass][st] + n);
    v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    if (a.noisy) {     // the weights' noise went into the GEMM operand; the bias noise is b_sigma * eps_out (networks.py:172-177)
      const float4 bs = *reinterpret_cast<const float4*>(a.bsig[pass][st] + n);
      const float4 eo = *reinterpret_cast<const float4*>(a.eps_out[pass][st] + n);
      v.x = fmaf(bs.x, eo.x, v.x); v.y = fmaf(bs.y, eo.y, v.y); v.z = fmaf(bs.z, eo.z, v.z); v.w = fmaf(bs.w, eo.w, v.w);
    }
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    *reinterpret_cast<float4*>(a.h1 + (long long)ps * pstride + i) = v;
  }
}

// dact3[m][k] = [act3 > 0] * sum over sources and splits of the partials; fp32 + tf32 hi/lo.
__global__ void __launch_bounds__(256) um_fcd_finish_kernel(const float* __restrict__ part, int nparts, long long stride,
                                                            const float* __restrict__ act_hi, float* __restrict__ out,
                                                            float* __restrict__ out_hi, float* __restrict__ out_lo, long long total4) {
  dz::pdl_enter();
  for (long long i4 = blockIdx.x * 256LL + threadIdx.x; i4 < total4; i4 += (long long)gridDim.x * 256) {
    const long long i = i4 << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < nparts; ++s) {
      const float4 x = *reinterpret_cast<const float4*>(part + s * stride + i);
      v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
    }
    const float4 m = *reinterpret_cast<const float4*>(act_hi + i);
    v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f; v.z = m.z > 0.f ? v.z : 0.f; v.w = m.w > 0.f ? v.w : 0.f;
    float4 h, l;
    split_tf32(v, h, l);
    *reinterpret_cast<float4*>(out + i) = v;
    *reinterpret_cast<float4*>(out_hi + i) = h;
    *reinterpret_cast<float4*>(out_lo + i) = l;
  }
}


// Weight-gradient finish: dW[k][n] = sum_s partial[s][k][n] (fixed order), and the bias gradient db[n] = sum_m G[m][n]
// as a deterministic two-level column sum of the (fp32) output gradient: 128-row chunks in parallel, the last block to
// finish adds the chunk sums in chunk order.  One launch covers several layers: blockIdx.y = layer; blocks
// [0, kWgSumBlocks) add the partials, blocks beyond do the bias chunks.
// Partial sums: a block owns 32 consecutive float4 columns; its 8 thread groups stride over the S partials (so the
// up-to-132 loads of one column are 8 independent chains instead of one dependent chain), then group sums are added in
// group order through shared memory — a fixed association, hence bit-deterministic.
constexpr int kWgChunkRows = 128, kWgMaxChunks = 256, kWgGroups = 8;
// norm_part: this layer's slots of the split global gradient norm: [0, sum_blocks) = sum of squares of the dW values each
// sum block wrote, [sum_blocks] = sum of squares of db (dz_learner.cu: split_norm).
struct WgFinish { const float* partial; int S; long long stride; int KN; float* dW; const float* G; int M, N; float* db; float* scratch;
                  unsigned int* ticket; int sum_blocks; float* norm_part; };

__global__ void __launch_bounds__(256) um_wgrad_finish_kernel(const __grid_constant__ WgFinish f) {
  dz::pdl_enter();
  __shared__ float4 red4[256];
  __shared__ bool last;
  if ((int)blockIdx.x >= f.sum_blocks) {
    float* red = reinterpret_cast<float*>(red4);
    const int chunk = blockIdx.x - f.sum_blocks, nchunks = (f.M + kWgChunkRows - 1) / kWgChunkRows;
    if (!f.db || chunk >= nchunks) return;
    const int n = threadIdx.x % f.N, g = threadIdx.x / f.N, G = 256 / f.N;
    const int m1 = min(f.M, (chunk + 1) * kWgChunkRows);
    float acc = 0.f;
    for (int m = chunk * kWgChunkRows + g; m < m1; m += G) acc += f.G[(long long)m * f.N + n];
    red[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < f.N) {
      float t = 0.f;
      for (int q = 0; q < G; ++q) t += red[q * f.N + threadIdx.x];
      f.scratch[chunk * 64 + threadIdx.x] = t;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(f.ticket, 1u) == (unsigned)(nchunks - 1);
    __syncthreads();
    if (last) {
      __threadfence();
      // chunk sums: G thread groups stride over the chunks (independent L2 loads), group sums added in group order
      float t = 0.f;
#pragma unroll 4
      for (int c = g; c < nchunks; c += G) t += __ldcg(f.scratch + c * 64 + n);
      red[threadIdx.x] = t;
      __syncthreads();
      float sq = 0.f;
      if (threadIdx.x < f.N) {
        float tt = 0.f;
        for (int q = 0; q < G; ++q) tt += red[q * f.N + threadIdx.x];
        f.db[threadIdx.x] = tt;
        sq = tt * tt;
      }
      __syncthreads();
      red[threadIdx.x] = sq;
      __syncthreads();
      if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int q = 0; q < f.N; ++q) tot += red[q];
        if (f.norm_part) f.norm_part[f.sum_blocks] = tot;
        *f.ticket = 0;
      }
    }
    return;
  }
  const int total4 = f.KN >> 2;
  const int col = blockIdx.x * 32 + (threadIdx.x & 31), g = threadIdx.x >> 5;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (col < total4) {
    const float* src = f.partial + ((long long)col << 2);
#pragma unroll 4
    for (int s = g; s < f.S; s += kWgGroups) {
      const float4 x = *reinterpret_cast<const float4*>(src + s * f.stride);
      v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
    }
  }
  red4[threadIdx.x] = v;
  __syncthreads();
  if (g == 0) {
    float sq = 0.f;
    if (col < total4) {
#pragma unroll
      for (int q = 1; q < kWgGroups; ++q) {
        const float4 x = red4[q * 32 + threadIdx.x];
        v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
      }
      *reinterpret_cast<float4*>(f.dW + ((long long)col << 2)) = v;
      sq = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
    }
    sq = warp_sum(sq);
    if (threadIdx.x == 0 && f.norm_part) f.norm_part[blockIdx.x] = sq;
  }
}

}  // namespace

int um_split(const float* x, float* hi, float* lo, long long n, void* stream);   // dz_umma.cu

// ------------------------------------------------------------------------------------------------
// Plan
// ------------------------------------------------------------------------------------------------

namespace {
// Bytes of one conv1 staging buffer: the input rows of the worst 128-pixel output tile, rounded up to 128.
int conv1_stag_bytes(int B, int W, int h1, int w1) {
  const int px = h1 * w1, m_pass = B * px;
  int worst = 0;
  for (int m0 = 0; m0 < m_pass; m0 += 128) {
    const int m1 = std::min(m0 + 128, m_pass);
    int tot = 0;
    for (int b = m0 / px; b <= (m1 - 1) / px; ++b) tot += conv1_segment(b, m0, m1, px, w1, W * 4).bytes;
    worst = std::max(worst, tot);
  }
  return (worst + 127) / 128 * 128;
}
// Dynamic shared memory of a conv1 kernel whose resident tiles take `resident` bytes: barriers, those tiles and the
// two staging buffers.
size_t conv1_smem_bytes(int resident, int stag_bytes) { return 2048 + (size_t)resident + 2 * (size_t)stag_bytes; }
}  // namespace

bool um_net_supported(const UmNetDesc& d) {
  if (d.fwd_only ? (d.B < 1 || d.npass != 1) : (d.B < 1 || d.B > 64 || d.npass < 1 || d.npass > 3)) return false;
  if (d.W % 4 || d.H < 36 || d.W < 36) return false;
  const int h1 = conv_out(d.H, 8, 4), w1 = conv_out(d.W, 8, 4);
  if ((h1 & 1) || (w1 & 1)) return false;              // stride-2 parity view of act1
  const int h2 = conv_out(h1, 4, 2), w2 = conv_out(w1, 4, 2);
  const int h3 = conv_out(h2, 3, 1), w3 = conv_out(w2, 3, 1);
  if (h3 < 1 || w3 < 1) return false;
  if (h2 * w2 > 128 || (h1 / 2) * (w1 / 2) > 128 || h3 * w3 > 128) return false;
  if (h1 * w1 < 64) return false;                      // a 128-pixel conv1 tile spans at most 3 images
  // the largest conv1 kernel (conv1_umma_kernel: weight image and A tile resident) fits
  return conv1_smem_bytes(kC1W + kC1A, conv1_stag_bytes(d.B, d.W, h1, w1)) <= 227 * 1024;
}

namespace {

struct Geo { int h1, w1, h2, w2, h3, w3, feat, PB; };
Geo geo_of(const UmNetDesc& d) {
  Geo g;
  g.h1 = conv_out(d.H, 8, 4); g.w1 = conv_out(d.W, 8, 4);
  g.h2 = conv_out(g.h1, 4, 2); g.w2 = conv_out(g.w1, 4, 2);
  g.h3 = conv_out(g.h2, 3, 1); g.w3 = conv_out(g.w2, 3, 1);
  g.feat = g.h3 * g.w3 * 64; g.PB = d.npass * d.B;
  return g;
}

struct Carver {
  char* base; int64_t used = 0;
  float* f(int64_t n) {
    int64_t bytes = (n * 4 + 255) / 256 * 256;
    float* p = base ? reinterpret_cast<float*>(base + used) : nullptr;
    used += bytes;
    return p;
  }
};

int fc_splits_for(int nprob, int nk) { return std::max(1, std::min(std::min(kNumSMs / (nprob * 4), 24), nk)); }

// Forward-only plans: rows of the fc x operand per problem (one NJT 64 tile).
constexpr int kFwdFcRows = 64;

int64_t carve_net(UmNet* n, char* base) {
  const UmNetDesc& d = n->d;
  const Geo g = geo_of(d);
  n->h1 = g.h1; n->w1 = g.w1; n->h2 = g.h2; n->w2 = g.w2; n->h3 = g.h3; n->w3 = g.w3; n->feat = g.feat; n->PB = g.PB;
  Carver c{base};
  const int64_t a1 = (int64_t)g.PB * g.h1 * g.w1 * 32, a2 = (int64_t)g.PB * g.h2 * g.w2 * 64, a3 = (int64_t)g.PB * g.feat;
  const int64_t sz[3] = {a1, a2, a3};
  for (int L = 0; L < 3; ++L) { n->act_hi[L] = c.f(sz[L]); n->act_lo[L] = c.f(sz[L]); n->act_f32[L] = c.f(sz[L]); }
  if (d.fwd_only) {
    for (int L = 0; L < 3; ++L) { n->wf_hi[0][L] = c.f(kConvN[L] * kConvK[L]); n->wf_lo[0][L] = c.f(kConvN[L] * kConvK[L]); }
    n->fc_nprob = n->fcd_nsrc = 0; n->fc_splits = n->fcd_splits = 1;
    if (d.use_fc) {
      n->fc_nprob = d.nstream;
      n->fc_splits = fc_splits_for(d.nstream, g.feat / 32);   // as for one 64-row chunk, whatever B is
      n->h1_buf = c.f((int64_t)d.nstream * d.B * 512);
      n->fc_part = c.f((int64_t)d.nstream * n->fc_splits * d.B * 512);
    }
    return c.used;
  }
  const int64_t dz_[3] = {(int64_t)d.B * g.h1 * g.w1 * 32, (int64_t)d.B * g.h2 * g.w2 * 64, (int64_t)d.B * g.feat};
  for (int L = 0; L < 3; ++L) { n->dact_hi[L] = c.f(dz_[L]); n->dact_lo[L] = c.f(dz_[L]); n->dact_f32[L] = c.f(dz_[L]); }
  for (int b = 0; b < 2; ++b)
    for (int L = 0; L < 3; ++L) { n->wf_hi[b][L] = c.f(kConvN[L] * kConvK[L]); n->wf_lo[b][L] = c.f(kConvN[L] * kConvK[L]); }
  n->wd3_hi = c.f(kConvN[2] * kConvK[2]); n->wd3_lo = c.f(kConvN[2] * kConvK[2]);
  n->wd2_hi = c.f(kConvN[1] * kConvK[1]); n->wd2_lo = c.f(kConvN[1] * kConvK[1]);
  {
    n->wg3_splits = std::max(1, std::min(g.h3, kNumSMs / 5));             // stages = h3 * groups, split over the output rows
    n->wg2_splits = std::max(1, std::min(g.h2, kNumSMs / 8));
    n->wg3_part = c.f((int64_t)n->wg3_splits * 576 * 64);
    n->wg2_part = c.f((int64_t)n->wg2_splits * 512 * 64);
    n->wg1_ctas = std::min(kNumSMs, (d.B * g.h1 * g.w1 + 127) / 128);
    n->wg1_part = c.f((int64_t)n->wg1_ctas * 256 * 32);
    n->wg_scratch = c.f(3 * 256 * 64);
    n->wg_ticket = reinterpret_cast<unsigned int*>(c.f(64));
  }
  n->h1_buf = nullptr; n->dh1_f32 = n->dh1_hi = n->dh1_lo = nullptr; n->fc_part = n->fcd_part = nullptr;
  n->fc_nprob = n->fcd_nsrc = 0; n->fc_splits = n->fcd_splits = 1;
  if (d.use_fc) {
    n->fc_nprob = d.npass * d.nstream;      // noisy layers: mu and sigma are combined in the converter (one GEMM per stream)
    n->fcd_nsrc = d.nstream;
    n->fc_splits = fc_splits_for(n->fc_nprob, g.feat / 32);
    const int ktiles = (g.feat + 127) / 128;
    n->fcd_splits = std::max(1, std::min(kNumSMs / (n->fcd_nsrc * ktiles), 8));
    n->h1_buf = c.f((int64_t)d.npass * d.nstream * d.B * 512);
    n->dh1_f32 = c.f((int64_t)d.nstream * d.B * 512);
    n->dh1_hi = c.f((int64_t)d.nstream * d.B * 512);
    n->dh1_lo = c.f((int64_t)d.nstream * d.B * 512);
    n->fc_part = c.f((int64_t)n->fc_nprob * n->fc_splits * d.B * 512);
    n->fcd_part = c.f((int64_t)n->fcd_nsrc * n->fcd_splits * d.B * g.feat);
  }
  return c.used;
}

// A problem with its operands, k-steps and reduction elements per stage, epilogue and valid extents; the rest zero.
UmProblem make_problem(const UmOperand& A, const UmOperand& Bo, int ksteps, int red_per_stage, uint32_t epi, int MI, int NJ) {
  UmProblem pr;
  memset(&pr, 0, sizeof(pr));
  pr.A = A; pr.B = Bo; pr.ksteps = (uint32_t)ksteps; pr.red_per_stage = (uint32_t)red_per_stage; pr.epi = epi;
  pr.MI = MI; pr.NJ = NJ;
  if (epi == UM_EPI_ROWS) { pr.pw = 1 << 20; pr.rs_outer = 0; pr.rs_inner = 1; }   // tile row r -> dst row row_base + r
  return pr;
}

// Stage of a launch whose operands are K-major hi / lo pairs (A, then B): it may run on the wgmma kernel.
uint32_t kmajor_stage_bytes(const UmOperand& A, const UmOperand& Bo) {
  return std::max(2 * A.part_bytes + 2 * Bo.part_bytes, um_wgmma_min_stage(A.part_bytes));
}

int build_plan(UmNet* n) {
  const UmNetDesc& d = n->d;
  UmPlan& pl = n->plan;
  const int B = d.B, PB = n->PB, h1 = n->h1, w1 = n->w1, h2 = n->h2, w2 = n->w2, h3 = n->h3, w3 = n->w3, feat = n->feat;

  // ---- weight image maps: [blob][layer][part]; box rows = N tile used by the layer
  int m_wf[2][3][2];
  const int nblob = d.fwd_only ? 1 : 2;
  const uint32_t wf_rows[3] = {32, 64, 32};   // conv1: N 32; conv2: full 64; conv3: halves of 32
  for (int b = 0; b < nblob; ++b)
    for (int L = 0; L < 3; ++L) {
      uint64_t dims[2] = {(uint64_t)kConvK[L], (uint64_t)kConvN[L]}, strides[1] = {(uint64_t)kConvK[L] * 4};
      uint32_t box[2] = {32, wf_rows[L]};
      DZ_TRY(pl.add_map_pair(n->wf_hi[b][L], n->wf_lo[b][L], 2, dims, strides, box, m_wf[b][L]));
    }
  for (int b = 0; b < 2; ++b) { n->map_wf1[b][0] = m_wf[b % nblob][0][0]; n->map_wf1[b][1] = m_wf[b % nblob][0][1]; }

  // =========================================================================== conv2 forward
  {
    int m_a[2];
    uint64_t dims[5] = {64, (uint64_t)w1 / 2, 2, (uint64_t)h1 / 2, (uint64_t)PB};
    uint64_t strides[4] = {256, (uint64_t)w1 * 128, (uint64_t)2 * w1 * 128, (uint64_t)h1 * w1 * 128};
    uint32_t box[5] = {32, (uint32_t)w2, 1, (uint32_t)h2, 1};
    DZ_TRY(pl.add_map_pair(n->act_hi[0], n->act_lo[0], 5, dims, strides, box, m_a));
    const int rows = h2 * w2;
    const UmOperand A = um_kmajor(rows, true, false), Bo = um_kmajor(64, true, false);
    const uint32_t a_bytes = A.part_bytes * 2;
    UmLaunch& l = n->launches[kConv2Fwd];
    pl.begin_launch(l, 64, kmajor_stage_bytes(A, Bo));
    for (int p = 0; p < d.npass; ++p) {
      const int blob = d.pass_target[p] ? 1 : 0;
      UmProblem pr = make_problem(A, Bo, 4, 32, UM_EPI_ROWS, rows, 64);
      pr.out_hi = n->act_hi[1]; pr.out_lo = n->act_lo[1]; pr.out_ld = 64;
      pr.bias = (blob ? d.target : d.online) + d.off_conv_b[1]; pr.relu = 1;
      const int prob = pl.add_problem(pr);
      for (int b = 0; b < B; ++b) {
        const int img = p * B + b;
        UmCta& c = pl.begin_cta(prob);
        c.row_base = img * rows; c.ph_valid = 1; c.pw_valid = rows;
        for (int kh = 0; kh < 4; ++kh)
          for (int kw = 0; kw < 4; ++kw) {
            pl.stage();
            pl.op_pair(m_a, 0, A.part_bytes, 32 * (kw & 1), kw >> 1, kh & 1, kh >> 1, img);
            pl.op_pair(m_wf[blob][1], a_bytes, Bo.part_bytes, 32 * (kh * 4 + kw));
          }
        DZ_TRY(pl.end_cta());
      }
    }
    pl.end_launch(l);
  }

  // =========================================================================== conv3 forward (two 32-channel halves)
  {
    // Image pairs per CTA.  A forward-only plan pairs odd B too: its last CTA's second image lies beyond the single
    // pass's B images, where the TMA unit reads zeros, and stores only its first image's rows.
    const int G = ((B % 2 == 0 || d.fwd_only) && 2 * h3 * w3 <= 128) ? 2 : 1;
    int m_a[2];
    uint64_t dims[4] = {64, (uint64_t)w2, (uint64_t)h2, (uint64_t)PB};
    uint64_t strides[3] = {256, (uint64_t)w2 * 256, (uint64_t)h2 * w2 * 256};
    uint32_t box[4] = {32, (uint32_t)w3, (uint32_t)h3, (uint32_t)G};
    DZ_TRY(pl.add_map_pair(n->act_hi[1], n->act_lo[1], 4, dims, strides, box, m_a));
    const int rows = G * h3 * w3;
    const UmOperand A = um_kmajor(rows, true, false), Bo = um_kmajor(32, true, false);
    const uint32_t a_bytes = A.part_bytes * 2;
    UmLaunch& l = n->launches[kConv3Fwd];
    pl.begin_launch(l, 32, kmajor_stage_bytes(A, Bo));
    for (int p = 0; p < d.npass; ++p) {
      const int blob = d.pass_target[p] ? 1 : 0;
      for (int half = 0; half < 2; ++half) {
        UmProblem pr = make_problem(A, Bo, 4, 32, UM_EPI_ROWS, rows, 32);
        pr.out_hi = n->act_hi[2] + 32 * half; pr.out_lo = n->act_lo[2] + 32 * half; pr.out_f32 = n->act_f32[2] + 32 * half;
        pr.out_ld = 64;
        pr.bias = (blob ? d.target : d.online) + d.off_conv_b[2] + 32 * half; pr.relu = 1;
        const int prob = pl.add_problem(pr);
        for (int t = 0; t < (B + G - 1) / G; ++t) {
          const int img = p * B + t * G;
          UmCta& c = pl.begin_cta(prob);
          c.row_base = img * h3 * w3; c.ph_valid = 1; c.pw_valid = std::min(G, B - t * G) * h3 * w3;
          for (int kh = 0; kh < 3; ++kh)
            for (int kw = 0; kw < 3; ++kw)
              for (int ch = 0; ch < 2; ++ch) {
                pl.stage();
                pl.op_pair(m_a, 0, A.part_bytes, 32 * ch, kw, kh, img);
                pl.op_pair(m_wf[blob][2], a_bytes, Bo.part_bytes, 32 * ((kh * 3 + kw) * 2 + ch), 32 * half);
              }
          DZ_TRY(pl.end_cta());
        }
      }
    }
    pl.end_launch(l);
  }

  // =========================================================================== conv3 input gradient
  // dact2[b,y,x,c] = [act2 > 0] * sum_{kh,kw,n} dact3[b, y-kh, x-kw, n] * W3[kh,kw,c,n]; halo zero-filled by the TMA unit
  if (!d.fwd_only) {
    const int nb = 2;                                     // row bands per image
    const int hb = (h2 + nb - 1) / nb;
    int m_a[2], m_w[2];
    for (int part = 0; part < 2; ++part) {
      uint64_t dims[4] = {64, (uint64_t)w3, (uint64_t)h3, (uint64_t)B};
      uint64_t strides[3] = {256, (uint64_t)w3 * 256, (uint64_t)h3 * w3 * 256};
      uint32_t box[4] = {32, (uint32_t)w2, (uint32_t)hb, 1};
      m_a[part] = pl.add_map(part ? n->dact_lo[2] : n->dact_hi[2], 4, dims, strides, box);
      uint64_t wd[2] = {576, 64}, ws[1] = {576 * 4};
      uint32_t wb[2] = {32, 32};
      m_w[part] = pl.add_map(part ? n->wd3_lo : n->wd3_hi, 2, wd, ws, wb);
      if (m_a[part] < 0 || m_w[part] < 0) return DZ_EINVAL;
    }
    const int rows = hb * w2;
    const UmOperand A = um_kmajor(rows, true, false), Bo = um_kmajor(32, true, false);
    const uint32_t a_bytes = A.part_bytes * 2;
    UmLaunch& l = n->launches[kConv3Dgrad];
    pl.begin_launch(l, 32, kmajor_stage_bytes(A, Bo));
    for (int half = 0; half < 2; ++half) {
      UmProblem pr = make_problem(A, Bo, 4, 32, UM_EPI_ROWS, rows, 32);
      pr.out_hi = n->dact_hi[1] + 32 * half; pr.out_lo = n->dact_lo[1] + 32 * half; pr.out_f32 = n->dact_f32[1] + 32 * half;
      pr.out_ld = 64;
      pr.mask = n->act_hi[1] + 32 * half;                 // pass 0 is the first B images
      const int prob = pl.add_problem(pr);
      for (int b = 0; b < B; ++b)
        for (int band = 0; band < nb; ++band) {
          const int y0 = band * hb, y1 = std::min(h2, y0 + hb);
          if (y1 <= y0) continue;
          UmCta& c = pl.begin_cta(prob);
          c.row_base = (b * h2 + y0) * w2; c.ph_valid = 1; c.pw_valid = (y1 - y0) * w2;
          for (int kh = 0; kh < 3; ++kh)
            for (int kw = 0; kw < 3; ++kw)
              for (int nh = 0; nh < 2; ++nh) {
                pl.stage();
                pl.op_pair(m_a, 0, A.part_bytes, 32 * nh, -kw, y0 - kh, b);
                pl.op_pair(m_w, a_bytes, Bo.part_bytes, 32 * ((kh * 3 + kw) * 2 + nh), 32 * half);
              }
          DZ_TRY(pl.end_cta());
        }
    }
    pl.end_launch(l);
  }

  // =========================================================================== conv2 input gradient (4 parity classes)
  // dact1[b, 2i+py, 2j+px, c] = [act1 > 0] * sum_{ay,ax,n} dact2[b, i-ay, j-ax, n] * W2[py+2ay, px+2ax, c, n]
  if (!d.fwd_only) {
    int m_a[2], m_w[2];
    for (int part = 0; part < 2; ++part) {
      uint64_t dims[4] = {64, (uint64_t)w2, (uint64_t)h2, (uint64_t)B};
      uint64_t strides[3] = {256, (uint64_t)w2 * 256, (uint64_t)h2 * w2 * 256};
      uint32_t box[4] = {32, (uint32_t)w1 / 2, (uint32_t)h1 / 2, 1};
      m_a[part] = pl.add_map(part ? n->dact_lo[1] : n->dact_hi[1], 4, dims, strides, box);
      uint64_t wd[2] = {256, 128}, ws[1] = {256 * 4};
      uint32_t wb[2] = {32, 32};
      m_w[part] = pl.add_map(part ? n->wd2_lo : n->wd2_hi, 2, wd, ws, wb);
      if (m_a[part] < 0 || m_w[part] < 0) return DZ_EINVAL;
    }
    const int rows = (h1 / 2) * (w1 / 2);
    const UmOperand A = um_kmajor(rows, true, false), Bo = um_kmajor(32, true, false);
    const uint32_t a_bytes = A.part_bytes * 2;
    UmLaunch& l = n->launches[kConv2Dgrad];
    pl.begin_launch(l, 32, kmajor_stage_bytes(A, Bo));
    UmProblem pr = make_problem(A, Bo, 4, 32, UM_EPI_ROWS, rows, 32);
    pr.out_hi = n->dact_hi[0]; pr.out_lo = n->dact_lo[0]; pr.out_f32 = n->dact_f32[0]; pr.out_ld = 32;
    pr.mask = n->act_hi[0];
    pr.pw = w1 / 2; pr.rs_outer = 2 * w1; pr.rs_inner = 2;
    const int prob = pl.add_problem(pr);
    for (int b = 0; b < B; ++b)
      for (int cls = 0; cls < 4; ++cls) {
        const int py = cls >> 1, pxx = cls & 1;
        UmCta& c = pl.begin_cta(prob);
        c.row_base = b * h1 * w1 + py * w1 + pxx; c.ph_valid = h1 / 2; c.pw_valid = w1 / 2;
        for (int ay = 0; ay < 2; ++ay)
          for (int ax = 0; ax < 2; ++ax)
            for (int nh = 0; nh < 2; ++nh) {
              pl.stage();
              pl.op_pair(m_a, 0, A.part_bytes, 32 * nh, -ax, -ay, b);
              pl.op_pair(m_w, a_bytes, Bo.part_bytes, 32 * ((ay * 2 + ax) * 2 + nh), 32 * cls);
            }
        DZ_TRY(pl.end_cta());
      }
    pl.end_launch(l);
  }

  if (!d.fwd_only) {   // conv1 weight gradient: G operand
    uint64_t dims[2] = {32, (uint64_t)B * h1 * w1}, strides[1] = {128};
    uint32_t box[2] = {32, 128};
    DZ_TRY(pl.add_map_pair(n->dact_hi[0], n->dact_lo[0], 2, dims, strides, box, n->map_g1));
  }
  // =========================================================================== conv3 / conv2 weight gradients
  // dW[k][n] = sum_m A[m][k] G[m][n]: both operands are read through MN-major (transposing) descriptors straight from the
  // NHWC tensors — the same im2col boxes as the forward pass, with the reduction running over (output row, 8 images).
  if (!d.fwd_only) {
    const int groups = (B + 7) / 8;
    // ---- conv3: A = act2 patches (pass 0), G = dact3
    {
      int m_a[2], m_g[2];
      for (int part = 0; part < 2; ++part) {
        uint64_t dims[4] = {64, (uint64_t)w2, (uint64_t)h2, (uint64_t)PB};
        uint64_t strides[3] = {256, (uint64_t)w2 * 256, (uint64_t)h2 * w2 * 256};
        uint32_t box[4] = {32, (uint32_t)w3, 1, 8};
        m_a[part] = pl.add_map(part ? n->act_lo[1] : n->act_hi[1], 4, dims, strides, box);
        uint64_t gd[4] = {64, (uint64_t)w3, (uint64_t)h3, (uint64_t)B};
        uint64_t gs[3] = {256, (uint64_t)w3 * 256, (uint64_t)h3 * w3 * 256};
        m_g[part] = pl.add_map(part ? n->dact_lo[2] : n->dact_hi[2], 4, gd, gs, box);
        if (m_a[part] < 0 || m_g[part] < 0) return DZ_EINVAL;
      }
      const int rows = w3 * 8;                                  // reduction rows per stage (multiple of 8)
      const UmOperand A = um_mnmajor(128, rows, false), Bo = um_mnmajor(64, rows, false);
      const uint32_t a_bytes = A.part_bytes * 2;
      UmLaunch& l = n->launches[kConv3Wgrad];
      pl.begin_launch(l, 64, a_bytes + Bo.part_bytes * 2);
      UmProblem pr = make_problem(A, Bo, rows / 8, rows, UM_EPI_PARTIAL, 576, 64);
      pr.C = n->wg3_part; pr.sc_i = 64; pr.sc_j = 1; pr.split_stride = 576 * 64;
      const int prob = pl.add_problem(pr);
      const int S = n->wg3_splits, per = (h3 + S - 1) / S;
      for (int kt = 0; kt < 5; ++kt)                            // 18 slabs of 32 reduction... k values: 4,4,4,4,2
        for (int sp = 0; sp < S; ++sp) {
          const int oy0 = sp * per, oy1 = std::min(h3, oy0 + per);
          if (oy1 <= oy0) continue;
          const int nslab = std::min(4, 18 - kt * 4);
          UmCta& c = pl.begin_cta(prob);
          c.i0 = kt * 128; c.split = sp;
          for (int oy = oy0; oy < oy1; ++oy)
            for (int gidx = 0; gidx < groups; ++gidx) {
              pl.stage();
              for (int part = 0; part < 2; ++part)
                for (int sl = 0; sl < nslab; ++sl) {
                  const int slab = kt * 4 + sl, tap = slab >> 1, ch = slab & 1, kh = tap / 3, kw = tap % 3;
                  pl.op(m_a[part], part * A.part_bytes + sl * A.lbo, 32 * ch, kw, oy + kh, gidx * 8);
                }
              for (int part = 0; part < 2; ++part)
                for (int nh = 0; nh < 2; ++nh) pl.op(m_g[part], a_bytes + part * Bo.part_bytes + nh * Bo.lbo, 32 * nh, 0, oy, gidx * 8);
            }
          DZ_TRY(pl.end_cta());
        }
      pl.end_launch(l);
    }
    // ---- conv2: A = act1 patches through the stride-2 parity view (pass 0), G = dact2; two 32-column halves
    {
      int m_a[2], m_g[2];
      for (int part = 0; part < 2; ++part) {
        uint64_t dims[5] = {64, (uint64_t)w1 / 2, 2, (uint64_t)h1 / 2, (uint64_t)PB};
        uint64_t strides[4] = {256, (uint64_t)w1 * 128, (uint64_t)2 * w1 * 128, (uint64_t)h1 * w1 * 128};
        uint32_t box[5] = {32, (uint32_t)w2, 1, 1, 8};
        m_a[part] = pl.add_map(part ? n->act_lo[0] : n->act_hi[0], 5, dims, strides, box);
        uint64_t gd[4] = {64, (uint64_t)w2, (uint64_t)h2, (uint64_t)B};
        uint64_t gs[3] = {256, (uint64_t)w2 * 256, (uint64_t)h2 * w2 * 256};
        uint32_t gbox[4] = {32, (uint32_t)w2, 1, 8};
        m_g[part] = pl.add_map(part ? n->dact_lo[1] : n->dact_hi[1], 4, gd, gs, gbox);
        if (m_a[part] < 0 || m_g[part] < 0) return DZ_EINVAL;
      }
      const int rows = w2 * 8;
      const UmOperand A = um_mnmajor(128, rows, false), Bo = um_mnmajor(32, rows, false);
      const uint32_t a_bytes = A.part_bytes * 2;
      UmLaunch& l = n->launches[kConv2Wgrad];
      pl.begin_launch(l, 32, a_bytes + Bo.part_bytes * 2);
      const int S = n->wg2_splits, per = (h2 + S - 1) / S;
      for (int half = 0; half < 2; ++half) {
        UmProblem pr = make_problem(A, Bo, rows / 8, rows, UM_EPI_PARTIAL, 512, 32);
        pr.C = n->wg2_part + 32 * half; pr.sc_i = 64; pr.sc_j = 1; pr.split_stride = 512 * 64;
        const int prob = pl.add_problem(pr);
        for (int kt = 0; kt < 4; ++kt)
          for (int sp = 0; sp < S; ++sp) {
            const int oy0 = sp * per, oy1 = std::min(h2, oy0 + per);
            if (oy1 <= oy0) continue;
            UmCta& c = pl.begin_cta(prob);
            c.i0 = kt * 128; c.split = sp;
            for (int oy = oy0; oy < oy1; ++oy)
              for (int gidx = 0; gidx < groups; ++gidx) {
                pl.stage();
                for (int part = 0; part < 2; ++part)
                  for (int sl = 0; sl < 4; ++sl) {
                    const int tap = kt * 4 + sl, kh = tap >> 2, kw = tap & 3;   // one slab = one (kh, kw) tap x 32 channels
                    pl.op(m_a[part], part * A.part_bytes + sl * A.lbo, 32 * (kw & 1), kw >> 1, kh & 1, oy + (kh >> 1), gidx * 8);
                  }
                pl.op_pair(m_g, a_bytes, Bo.part_bytes, 32 * half, 0, oy, gidx * 8);
              }
            DZ_TRY(pl.end_cta());
          }
      }
      pl.end_launch(l);
    }
  }

  // =========================================================================== fc1 / noisy1 forward and input gradient
  if (d.use_fc) {
    const int njt = d.fwd_only || B > 32 ? 64 : 32;
    const int q = d.noisy ? 2 : 1;
    int m_x[2], m_g[2] = {0, 0};
    for (int part = 0; part < 2; ++part) {
      uint64_t dims[2] = {(uint64_t)feat, (uint64_t)PB}, strides[1] = {(uint64_t)feat * 4};
      uint32_t box[2] = {32, (uint32_t)njt};
      m_x[part] = pl.add_map(part ? n->act_lo[2] : n->act_hi[2], 2, dims, strides, box);
      if (!d.fwd_only) {
        uint64_t gd[2] = {512, (uint64_t)d.nstream * B}, gs[1] = {2048};
        m_g[part] = pl.add_map(part ? n->dh1_lo : n->dh1_hi, 2, gd, gs, box);
      }
      if (m_x[part] < 0 || m_g[part] < 0) return DZ_EINVAL;
    }
    // Forward CTA groups: the passes that apply the same parameter blob share every staged weight tile (online net on
    // s_tm1 and s_t), each group's tiles then span 128 / (passes in the group) weight columns, so a CTA does the same
    // MMA work whether it serves one pass or two.  fc_per_pass (tests only): one group per pass, 128-column tiles.
    // A group member is the x rows [row0, row0 + rows) of one pass: all B of them, or in a forward-only plan one
    // chunk of at most kFwdFcRows, each chunk a group of its own (the same CTAs and reduction order for every row).
    struct FcMember { int pass, row0, rows; };
    std::vector<std::vector<FcMember>> grp;
    std::vector<int> grp_blob;
    if (d.fwd_only) {
      for (int r0 = 0; r0 < B; r0 += kFwdFcRows) { grp.push_back({{0, r0, std::min(kFwdFcRows, B - r0)}}); grp_blob.push_back(0); }
    } else {
      for (int p = 0; p < d.npass; ++p) {
        const int blob = d.pass_target[p] ? 1 : 0;
        int gi = -1;
        if (!n->fc_per_pass)
          for (int k = 0; k < (int)grp.size(); ++k) if (grp_blob[k] == blob) gi = k;
        if (gi < 0) { gi = (int)grp.size(); grp.emplace_back(); grp_blob.push_back(blob); }
        if ((int)grp[gi].size() == kFcMaxProbs) return fail(DZ_EINVAL, "fc forward: more than two passes apply one parameter blob");
        grp[gi].push_back({p, p * B, B});
      }
    }
    const int ngrp = (int)grp.size();
    int fc_rows[2] = {128, 128};   // forward tile columns per blob
    for (int k = 0; k < ngrp; ++k) fc_rows[grp_blob[k]] = 128 / (int)grp[k].size();
    // weight maps: [blob][stream][sigma] x {forward box (32 n, 32 k) x fc_rows / 32, gradient box (32 n, 128 k)}
    int m_wf_fc[2][2][2], m_wd_fc[2][2];
    bool wf3d = true;
    for (int blob = 0; blob < nblob; ++blob)
      for (int s = 0; s < d.nstream; ++s)
        for (int sg = 0; sg < q; ++sg) {
          const float* w = (blob ? d.target : d.online) + (sg ? d.off_fc_sw[s] : d.off_fc_w[s]);
          uint64_t dims[2] = {512, (uint64_t)feat}, strides[1] = {2048};
          // MN-major A operand (rows of W are the reduction): W[k][n] viewed as (n % 32, k, n / 32) so that ONE box of
          // (32, 32, fc_rows / 32) lands as the [32 k][32 n] slabs of a tile, slab-major — one TMA op per tile
          uint64_t dims3[3] = {32, (uint64_t)feat, 16}, strides3[2] = {2048, 128};
          uint32_t box3[3] = {32, 32, (uint32_t)fc_rows[blob] / 32};
          if (wf3d) {
            m_wf_fc[blob][s][sg] = pl.add_map(w, 3, dims3, strides3, box3);
            if (m_wf_fc[blob][s][sg] < 0) wf3d = false;      // driver refused the permuted view: one op per slab instead
          }
          if (!wf3d) {
            if (blob || s || sg) return fail(DZ_EINVAL, "fc weight tensor maps: inconsistent encodings");
            uint32_t box2[2] = {32, 32};
            m_wf_fc[blob][s][sg] = pl.add_map(w, 2, dims, strides, box2);
          }
          if (m_wf_fc[blob][s][sg] < 0) return DZ_EINVAL;
          if (blob == 0 && !d.fwd_only) {
            uint32_t boxd[2] = {32, 128};
            m_wd_fc[s][sg] = pl.add_map(w, 2, dims, strides, boxd);
            if (m_wd_fc[s][sg] < 0) return DZ_EINVAL;
          }
        }
    // ---- forward: D[n, m] = sum_k W[k][n] x[m][k];  noisy: W = Wmu + Wsigma * (eps_in[k] * eps_out[n]), formed in the
    // MMA warps (umma_fc_kernel; with fc_per_pass by the converter warps of umma_gemm_kernel)
    {
      const UmOperand Bo = um_kmajor(njt, true, false);
      const int nk = feat / 32, S = n->fc_splits, per = (nk + S - 1) / S;
      uint32_t stage_bytes = 2 * 16384 + 2 * Bo.part_bytes;
      for (int k = 0; k < ngrp; ++k) {
        const int np = (int)grp[k].size();
        stage_bytes = std::max<uint32_t>(stage_bytes, 2 * 16384 / np + np * 2 * Bo.part_bytes);
      }
      UmLaunch& l = n->launches[kFcFwd];
      pl.begin_launch(l, njt, stage_bytes);
      for (int k = 0; k < ngrp; ++k) {
        const int blob = grp_blob[k], np = (int)grp[k].size(), rows = fc_rows[blob], slabs = rows / 32;
        const UmOperand A = um_mnmajor(rows, 32, true, nullptr);
        const uint32_t a_bytes = 2 * A.part_bytes;
        for (int s = 0; s < d.nstream; ++s) {
          const int prob0 = (int)pl.probs.size();
          for (int gp = 0; gp < np; ++gp) {
            const FcMember& m = grp[k][gp];
            const int p = m.pass, qi = p * d.nstream + s;
            UmProblem pr = make_problem(A, Bo, 4, 32, UM_EPI_PARTIAL, 512, m.rows);
            if (d.noisy) pr.A.convert = 2;
            pr.C = n->fc_part + (int64_t)qi * S * B * 512 + (int64_t)(m.row0 - p * B) * 512;
            pr.sc_i = 1; pr.sc_j = 512; pr.split_stride = (long long)B * 512;
            const int prob = pl.add_problem(pr);
            if (d.noisy) {
              n->patches.push_back({prob, 0, (int64_t)d.noise_apply[p] * d.noise_stride + d.noise_off_in[s]});
              n->patches.push_back({prob, 2, (int64_t)d.noise_apply[p] * d.noise_stride + d.noise_off_out[s]});
            }
          }
          // the column tiles of one k range sit in neighbouring CTAs: together they stream whole 2 KB rows of W
          for (int sp = 0; sp < S; ++sp)
            for (int nt = 0; nt < 512 / rows; ++nt) {
              const int k0 = sp * per, k1 = std::min(nk, k0 + per);
              if (k1 <= k0) continue;
              UmCta& c = pl.begin_cta(prob0);
              c.nprob = (uint32_t)np; c.r0 = 32 * k0; c.i0 = nt * rows; c.split = sp;
              for (int ks = k0; ks < k1; ++ks) {
                pl.stage();
                for (int sg = 0; sg < q; ++sg) {
                  if (wf3d) pl.op(m_wf_fc[blob][s][sg], sg * A.part_bytes, 0, 32 * ks, nt * slabs);
                  else for (int sl = 0; sl < slabs; ++sl) pl.op(m_wf_fc[blob][s][sg], sg * A.part_bytes + sl * 4096, nt * rows + 32 * sl, 32 * ks);
                }
                for (int gp = 0; gp < np; ++gp) pl.op_pair(m_x, a_bytes + gp * 2 * Bo.part_bytes, Bo.part_bytes, 32 * ks, grp[k][gp].row0);
              }
              DZ_TRY(pl.end_cta());
            }
        }
      }
      pl.end_launch(l);
    }
    // ---- input gradient: D[k, m] = sum_n W[k][n] g[m][n];  noisy: W = Wmu + Wsigma * (eps_in[k] * eps_out[n]), formed in the
    // MMA warps (umma_fc_kernel on the K-major tile; with UM_PATH_CONVERTERS by the converter warps of umma_gemm_kernel)
    if (!d.fwd_only) {
      const UmOperand Bo = um_kmajor(njt, true, false);
      const int S = n->fcd_splits, per = (16 + S - 1) / S, ktiles = (feat + 127) / 128;
      UmLaunch& l = n->launches[kFcDgrad];
      pl.begin_launch(l, njt, 2 * 16384 + 2 * Bo.part_bytes);
      for (int s = 0; s < d.nstream; ++s) {
        UmProblem pr = make_problem(um_kmajor(128, true, true, nullptr), Bo, 4, 32, UM_EPI_PARTIAL, feat, B);
        if (d.noisy) pr.A.convert = 2;
        pr.C = n->fcd_part + (int64_t)s * S * B * feat; pr.sc_i = 1; pr.sc_j = feat; pr.split_stride = (long long)B * feat;
        const int prob = pl.add_problem(pr);
        if (d.noisy) {
          n->patches.push_back({prob, 0, (int64_t)d.noise_apply[0] * d.noise_stride + d.noise_off_out[s]});
          n->patches.push_back({prob, 2, (int64_t)d.noise_apply[0] * d.noise_stride + d.noise_off_in[s]});
        }
        for (int kt = 0; kt < ktiles; ++kt)
          for (int sp = 0; sp < S; ++sp) {
            const int n0 = sp * per, n1 = std::min(16, n0 + per);
            if (n1 <= n0) continue;
            UmCta& c = pl.begin_cta(prob);
            c.r0 = 32 * n0; c.i0 = kt * 128; c.split = sp;
            for (int ns = n0; ns < n1; ++ns) {
              pl.stage();
              pl.op(m_wd_fc[s][0], 0, 32 * ns, kt * 128);
              if (d.noisy) pl.op(m_wd_fc[s][1], 16384, 32 * ns, kt * 128);
              pl.op_pair(m_g, 32768, Bo.part_bytes, 32 * ns, s * B);
            }
            DZ_TRY(pl.end_cta());
          }
      }
      pl.end_launch(l);
    }
  }
  return DZ_OK;
}

int apply_noise(UmNet* n, const float* noise, void* stream) {
  if (n->patches.empty() || noise == n->noise_cached) return DZ_OK;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing((cudaStream_t)stream, &cs);
  if (cs != cudaStreamCaptureStatusNone) return fail(DZ_EINVAL, "the noise buffer must not move between graph captures (keep one buffer per learner)");
  for (const auto& p : n->patches) {
    UmProblem& pr = n->plan.probs[p.prob];
    if (p.field == 0) pr.A.scale_r = noise + p.off; else if (p.field == 2) pr.A.scale_i = noise + p.off; else pr.scale_i = noise + p.off;
  }
  DZ_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  DZ_CUDA_OK(cudaMemcpy(n->plan.d_probs, n->plan.probs.data(), n->plan.probs.size() * sizeof(UmProblem), cudaMemcpyHostToDevice));
  n->noise_cached = noise;
  return DZ_OK;
}

}  // namespace

int64_t um_net_workspace_bytes(const UmNetDesc& d) {
  UmNet tmp;
  tmp.d = d;
  return carve_net(&tmp, nullptr);
}

namespace {
int net_create(const UmNetDesc& d, char* base, UmNet** out, bool fc_per_pass) {
  if (!um_net_supported(d)) return fail(DZ_EINVAL, "geometry not supported by the tensor-core path");
  UmNet* n = new UmNet();
  n->d = d;
  n->fc_per_pass = fc_per_pass;
  carve_net(n, base);
  n->conv1_tiles_per_pass = (d.B * n->h1 * n->w1 + 127) / 128;
  n->conv1_stag_bytes = conv1_stag_bytes(d.B, d.W, n->h1, n->w1);
  // gradient buffers start as zeros (hi/lo pairs of layers whose producer has not run yet are never NaN)
  if (!d.fwd_only) cudaMemset(n->wg_ticket, 0, 64 * 4);
  for (int L = 0; L < 3 && !d.fwd_only; ++L) {
    const int64_t cnt[3] = {(int64_t)d.B * n->h1 * n->w1 * 32, (int64_t)d.B * n->h2 * n->w2 * 64, (int64_t)d.B * n->feat};
    cudaMemset(n->dact_hi[L], 0, cnt[L] * 4); cudaMemset(n->dact_lo[L], 0, cnt[L] * 4); cudaMemset(n->dact_f32[L], 0, cnt[L] * 4);
  }
  int rc = build_plan(n);
  for (int i = 0; i < kNumNetLaunches && rc == DZ_OK; ++i)
    if (n->launches[i].nctas > 0) rc = n->plan.localize_maps(n->launches[i]);
  if (rc == DZ_OK) rc = n->plan.upload();
  if (rc == DZ_OK) rc = UmPlan::configure();
  if (rc != DZ_OK) { um_net_destroy(n); return rc; }
  static bool configured = false;
  if (!configured) {
    if (cudaFuncSetAttribute(conv1_umma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(conv1_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(conv1_wgrad_umma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
      um_net_destroy(n);
      return fail(DZ_ECUDA, "conv1 kernels: shared memory attribute");
    }
    configured = true;
  }
  *out = n;
  return DZ_OK;
}
}  // namespace

int um_net_create(const UmNetDesc& d, char* base, UmNet** out) { return net_create(d, base, out, false); }

void um_net_trace(UmNet* n, const char* tag, long long* d_trace) { n->trace_tag = tag ? tag : ""; n->trace_ptr = d_trace; }

int um_net_mma_path(UmNet* n, const char* tag) {
  const std::string t = tag ? tag : "";
  if (t == "conv1_fwd") return UM_PATH_WGMMA;     // conv1_wgmma_kernel (um_forward_torso)
  for (int i = 0; i < kNumNetLaunches; ++i) {
    const NetLaunchName& nm = kNetLaunchNames[i];
    if (t == nm.tag || (nm.noisy && t == nm.noisy)) return n->launches[i].nctas > 0 ? n->plan.path_of(n->launches[i]) : -1;
  }
  return -1;
}

void um_net_destroy(UmNet* n) {
  if (!n) return;
  n->plan.release();
  delete n;
}

// Layers 1 and 2 have no consumer of the exact fp32 activation on this path (the next layer reads the hi/lo pair, the
// ReLU masks read the sign of hi): their "fp32 view" is the tf32 hi image — same activation pattern, values rounded to tf32.
float* um_act_f32(UmNet* n, int layer, int pass) {
  const int64_t per[3] = {(int64_t)n->d.B * n->h1 * n->w1 * 32, (int64_t)n->d.B * n->h2 * n->w2 * 64, (int64_t)n->d.B * n->feat};
  return (layer < 3 ? n->act_hi[layer - 1] : n->act_f32[layer - 1]) + per[layer - 1] * pass;
}
float* um_dact_f32(UmNet* n, int layer) { return n->dact_f32[layer - 1]; }
float* um_act_lo(UmNet* n, int layer) { return layer < 3 ? n->act_lo[layer - 1] : nullptr; }
float* um_dact_hi(UmNet* n, int layer) { return n->dact_hi[layer - 1]; }
float* um_dact_lo(UmNet* n, int layer) { return n->dact_lo[layer - 1]; }
float* um_h1_f32(UmNet* n, int pass, int stream) { return n->h1_buf + ((int64_t)pass * n->d.nstream + stream) * n->d.B * 512; }
float* um_dh1_f32(UmNet* n, int stream) { return n->dh1_f32 + (int64_t)stream * n->d.B * 512; }
float* um_dh1_hi(UmNet* n, int stream) { return n->dh1_hi + (int64_t)stream * n->d.B * 512; }
float* um_dh1_lo(UmNet* n, int stream) { return n->dh1_lo + (int64_t)stream * n->d.B * 512; }

int um_pack_weights(UmNet* n, void* stream) {
  PackArgs a;
  memset(&a, 0, sizeof(a));
  a.blob[0] = n->d.online; a.blob[1] = n->d.target;
  for (int L = 0; L < 3; ++L) a.off_w[L] = n->d.off_conv_w[L];
  for (int b = 0; b < 2; ++b)
    for (int L = 0; L < 3; ++L) { a.wf_hi[b][L] = n->wf_hi[b][L]; a.wf_lo[b][L] = n->wf_lo[b][L]; }
  a.wd3_hi = n->wd3_hi; a.wd3_lo = n->wd3_lo; a.wd2_hi = n->wd2_hi; a.wd2_lo = n->wd2_lo;
  // the kernel's elements run online forward images first: a forward-only plan launches just those
  const int total = n->d.fwd_only ? kConvFwdFloats : 2 * kConvFwdFloats + kConvN[2] * kConvK[2] + kConvN[1] * kConvK[1];
  DZ_LAUNCH_NAMED("conv_pack", um_pack_conv_kernel, (unsigned)ceil_div(total, 256), 256, 0, stream, a);
  return DZ_OK;
}

namespace {
// conv1 forward into act1 hi / lo; reference: conv1_umma_kernel instead of the learner's conv1_wgmma_kernel (tests only).
int launch_conv1(UmNet* n, const uint8_t* const* const* rows, void* stream, bool reference) {
  const UmNetDesc& d = n->d;
  Conv1Args a;
  memset(&a, 0, sizeof(a));
  for (int p = 0; p < d.npass; ++p) {
    const int blob = d.pass_target[p] ? 1 : 0;
    a.rows[p] = rows[p];
    a.bias[p] = (blob ? d.target : d.online) + d.off_conv_b[0];
    a.blob[p] = blob;
  }
  for (int b = 0; b < 2; ++b)
    for (int part = 0; part < 2; ++part) a.wmap[b][part] = n->plan.maps[n->map_wf1[b][part]];
  a.out_hi = n->act_hi[0]; a.out_lo = n->act_lo[0]; a.out_f32 = n->act_f32[0];
  a.npass = d.npass; a.B = d.B; a.W = d.W; a.oh = n->h1; a.ow = n->w1; a.m_pass = d.B * n->h1 * n->w1;
  a.tiles_per_pass = n->conv1_tiles_per_pass; a.ntiles = a.tiles_per_pass * d.npass; a.stag_bytes = n->conv1_stag_bytes;
  a.trace = n->tr("conv1_fwd");
  const size_t smem = conv1_smem_bytes(kC1W + (reference ? kC1A : 0), a.stag_bytes);   // conv1_wgmma_kernel has no A tile
  if (smem > 227 * 1024) return fail(DZ_EINVAL, "conv1 staging does not fit");
  const unsigned grid = (unsigned)std::min(kNumSMs, a.ntiles);
  if (reference) DZ_LAUNCH_NAMED("conv1_fwd", conv1_umma_kernel, grid, kThreadsU, smem, stream, a);
  else DZ_LAUNCH_NAMED("conv1_fwd", conv1_wgmma_kernel, grid, kThreadsC1W, smem, stream, a);
  return DZ_OK;
}

// Launch `id` of the plan under its name; it writes CTA 0's clock stamps when the trace is set on its tag.
int run_launch(UmNet* n, NetLaunch id, void* stream) {
  const NetLaunchName& nm = kNetLaunchNames[id];
  return n->plan.launch(n->d.noisy && nm.noisy ? nm.noisy : nm.tag, n->launches[id], stream, n->tr(nm.tag));
}
}  // namespace

int um_forward_torso(UmNet* n, const uint8_t* const* const* rows, void* stream) {
  DZ_TRY(launch_conv1(n, rows, stream, false));
  DZ_TRY(run_launch(n, kConv2Fwd, stream));
  DZ_TRY(run_launch(n, kConv3Fwd, stream));
  return DZ_OK;
}

int um_forward_fc(UmNet* n, const float* noise, void* stream) {
  const UmNetDesc& d = n->d;
  if (!d.use_fc) return fail(DZ_EINVAL, "fc layers are not on the tensor-core path for this agent");
  if (d.noisy) DZ_TRY(apply_noise(n, noise, stream));
  DZ_TRY(run_launch(n, kFcFwd, stream));
  FcFinishArgs a;
  memset(&a, 0, sizeof(a));
  a.part = n->fc_part; a.S = n->fc_splits; a.B = d.B; a.nstream = d.nstream; a.noisy = d.noisy; a.npass = d.npass; a.h1 = n->h1_buf;
  for (int p = 0; p < d.npass; ++p)
    for (int s = 0; s < d.nstream; ++s) {
      const float* blob = d.pass_target[p] ? d.target : d.online;
      a.bmu[p][s] = blob + d.off_fc_b[s];
      if (d.noisy) {
        a.bsig[p][s] = blob + d.off_fc_sb[s];
        a.eps_out[p][s] = noise + (int64_t)d.noise_apply[p] * d.noise_stride + d.noise_off_out[s];
      }
    }
  dim3 grid((unsigned)std::min<int64_t>(ceil_div((int64_t)d.B * 128, 256), 64), (unsigned)(d.npass * d.nstream));
  DZ_LAUNCH_NAMED("fc_finish", um_fc_finish_kernel, grid, 256, 0, stream, a);
  return DZ_OK;
}

int um_bind_noise(UmNet* n, const float* noise) { return apply_noise(n, noise, nullptr); }

int um_split_dh1(UmNet* n, void* stream) {
  return um_split(n->dh1_f32, n->dh1_hi, n->dh1_lo, (long long)n->d.nstream * n->d.B * 512, stream);
}

int um_backward_fc(UmNet* n, const float* noise, void* stream) {
  const UmNetDesc& d = n->d;
  if (!d.use_fc) return fail(DZ_EINVAL, "fc layers are not on the tensor-core path for this agent");
  if (d.noisy) DZ_TRY(apply_noise(n, noise, stream));
  DZ_TRY(run_launch(n, kFcDgrad, stream));
  const long long total = (long long)d.B * n->feat;
  DZ_LAUNCH_NAMED("fcd_finish", um_fcd_finish_kernel, (unsigned)std::min<long long>(ceil_div(total / 4, 256), kNumSMs * 4), 256, 0, stream,
                  n->fcd_part, n->fcd_nsrc * n->fcd_splits, total, n->act_hi[2], n->dact_f32[2], n->dact_hi[2], n->dact_lo[2], total / 4);
  return DZ_OK;
}

int um_split_dact3(UmNet* n, void* stream) {
  return um_split(n->dact_f32[2], n->dact_hi[2], n->dact_lo[2], (long long)n->d.B * n->feat, stream);
}

int um_wgrad_conv1(UmNet* n, const uint8_t* const* rows0, void* stream) {
  const UmNetDesc& d = n->d;
  Conv1WgArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = rows0; a.gmap[0] = n->plan.maps[n->map_g1[0]]; a.gmap[1] = n->plan.maps[n->map_g1[1]]; a.partial = n->wg1_part;
  a.B = d.B; a.W = d.W; a.oh = n->h1; a.ow = n->w1; a.m_pass = d.B * n->h1 * n->w1;
  a.ntiles = (a.m_pass + 127) / 128; a.stag_bytes = n->conv1_stag_bytes;
  const size_t smem = conv1_smem_bytes(kC1G + kC1A, a.stag_bytes);
  if (smem > 227 * 1024) return fail(DZ_EINVAL, "conv1 wgrad staging does not fit");
  DZ_LAUNCH_NAMED("conv1_wgrad", conv1_wgrad_umma_kernel, (unsigned)n->wg1_ctas, kThreadsU, smem, stream, a);
  return DZ_OK;
}

int um_wgrad_conv3(UmNet* n, void* stream) { return run_launch(n, kConv3Wgrad, stream); }
int um_wgrad_conv2(UmNet* n, void* stream) { return run_launch(n, kConv2Wgrad, stream); }

// dW / db of conv3 and conv2 from the split partials (+ optionally conv1's FMA partials in the same launch).
namespace {
int wg_sum_blocks(int layer) { return (kConvN[layer - 1] * kConvK[layer - 1] / 4 + 31) / 32; }
int wg_slot_base(int layer) { int b = 0; for (int L = 3; L > layer; --L) b += wg_sum_blocks(L) + 1; return b; }
}  // namespace

int um_norm_slots(UmNet*) { return wg_slot_base(1) + wg_sum_blocks(1) + 1; }

// dW / db of one conv layer (1..3) from its split partials; norm_parts (optional): base of the split-norm slot array.
int um_wgrad_finish_layer(UmNet* n, int layer, float* dW, float* db, float* norm_parts, void* stream) {
  float* sc = n->wg_scratch;
  WgFinish f;
  memset(&f, 0, sizeof(f));
  if (layer == 3) f = WgFinish{n->wg3_part, n->wg3_splits, 576 * 64, 576 * 64, dW, n->dact_f32[2], n->d.B * n->h3 * n->w3, 64, db, sc, n->wg_ticket, 0, nullptr};
  else if (layer == 2) f = WgFinish{n->wg2_part, n->wg2_splits, 512 * 64, 512 * 64, dW, n->dact_f32[1], n->d.B * n->h2 * n->w2, 64, db, sc + 256 * 64, n->wg_ticket + 1, 0, nullptr};
  else f = WgFinish{n->wg1_part, n->wg1_ctas, 256 * 32, 256 * 32, dW, n->dact_f32[0], n->d.B * n->h1 * n->w1, 32, db, sc + 2 * 256 * 64, n->wg_ticket + 2, 0, nullptr};
  f.sum_blocks = wg_sum_blocks(layer);
  f.norm_part = norm_parts ? norm_parts + wg_slot_base(layer) : nullptr;
  const int chunks = (f.M + kWgChunkRows - 1) / kWgChunkRows;
  if (chunks > kWgMaxChunks) return fail(DZ_EINVAL, "bias-gradient reduction: too many row chunks");
  const char* tags[3] = {"wgrad_finish1", "wgrad_finish2", "wgrad_finish3"};
  DZ_LAUNCH_NAMED(tags[layer - 1], um_wgrad_finish_kernel, (unsigned)(f.sum_blocks + chunks), 256, 0, stream, f);
  return DZ_OK;
}

int um_backward_conv3(UmNet* n, void* stream) { return run_launch(n, kConv3Dgrad, stream); }
int um_backward_conv2(UmNet* n, void* stream) { return run_launch(n, kConv2Dgrad, stream); }

}  // namespace dz

using namespace dz;

// Test hook: the fc1 / noisy1 forward launch alone, on features x [npass * B][feat] (feat from the H x W observation
// geometry), with the learner's pass layout for npass 1, 2 or 3 (passes 0 and 1 apply the online blob when npass is 3;
// otherwise pass 0 is online and pass 1 target).  Stream s reads the weights at online / target + off_w[s] (mu) and
// + off_sw[s] (sigma, noisy); pass p's noise is apply p: eps_in / eps_out of stream s at noise + p * noise_stride +
// off_in[s] / off_out[s].  per_pass = 0: the learner's plan on umma_fc_kernel; 1: one CTA group per pass with 128-column
// tiles on umma_gemm_kernel and its converter warps.  Writes the split partials [npass][nstream][S][B][512] to d_part
// (room for npass * nstream * 24 * B * 512 floats), S to *splits and the weight-tile bytes the launch stages to
// *weight_bytes.
extern "C" int dz_test_fc_forward(int32_t B, int32_t H, int32_t W, int32_t npass, int32_t nstream, int32_t noisy, const float* online,
                                  const float* target, const int64_t* off_w, const int64_t* off_sw, const float* noise,
                                  int64_t noise_stride, const int64_t* off_in, const int64_t* off_out, const float* x, int32_t per_pass,
                                  float* d_part, int32_t* splits, int64_t* weight_bytes, void* stream) {
  if (nstream < 1 || nstream > 2 || npass < 1 || npass > 3) return fail(DZ_EINVAL, "fc forward test: npass 1..3, nstream 1..2");
  UmNetDesc d;
  memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.npass = npass;
  d.pass_target[0] = 0; d.pass_target[1] = npass == 3 ? 0 : 1; d.pass_target[2] = 1;
  d.online = online; d.target = target;
  d.use_fc = 1; d.nstream = nstream; d.noisy = noisy ? 1 : 0;
  for (int s = 0; s < nstream; ++s) {
    d.off_fc_w[s] = off_w[s];
    if (noisy) { d.off_fc_sw[s] = off_sw[s]; d.noise_off_in[s] = off_in[s]; d.noise_off_out[s] = off_out[s]; }
  }
  for (int p = 0; p < 3; ++p) d.noise_apply[p] = p;
  d.noise_stride = noise_stride;
  if (!um_net_supported(d)) return fail(DZ_EINVAL, "fc forward test: geometry not supported by the tensor-core path");
  char* ws = nullptr;
  DZ_CUDA_OK(cudaMalloc(&ws, (size_t)um_net_workspace_bytes(d)));
  UmNet* n = nullptr;
  int rc = net_create(d, ws, &n, per_pass != 0);
  if (rc == DZ_OK) rc = um_split(x, n->act_hi[2], n->act_lo[2], (long long)n->PB * n->feat, stream);
  if (rc == DZ_OK && noisy) rc = apply_noise(n, noise, stream);
  if (rc == DZ_OK) rc = n->plan.launch("fc1_fwd", n->launches[kFcFwd], stream, nullptr, per_pass ? UM_PATH_CONVERTERS : UM_PATH_AUTO);
  if (rc == DZ_OK) {
    const size_t bytes = (size_t)npass * nstream * n->fc_splits * B * 512 * sizeof(float);
    if (cudaMemcpyAsync(d_part, n->fc_part, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) != cudaSuccess ||
        cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
      rc = fail(DZ_ECUDA, "fc forward test: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (rc == DZ_OK) {
    *splits = n->fc_splits;
    int64_t wb = 0;
    const UmLaunch& l = n->launches[kFcFwd];
    for (int ci = l.cta0; ci < l.cta0 + l.nctas; ++ci) {
      const UmCta& c = n->plan.ctas[ci];
      wb += (int64_t)c.nstages * (noisy ? 2 : 1) * n->plan.probs[c.prob].A.part_bytes;
    }
    *weight_bytes = wb;
  }
  if (n) um_net_destroy(n);
  cudaFree(ws);
  return rc;
}

// Test hook: the fc1 / noisy1 input-gradient launch alone, on the output gradients g [nstream][B][512] (feat from the
// H x W observation geometry).  Stream s reads the online weights at online + off_w[s] (mu) and + off_sw[s] (sigma,
// noisy); its noise is eps_in / eps_out at noise + off_in[s] / off_out[s].  converters = 0: the learner's launch on
// umma_fc_kernel; 1: umma_gemm_kernel and its converter warps.  Writes the split partials [nstream][S][B][feat] to d_part
// (room for nstream * 8 * B * feat floats) and S to *splits.
extern "C" int dz_test_fc_dgrad(int32_t B, int32_t H, int32_t W, int32_t nstream, int32_t noisy, const float* online, const int64_t* off_w,
                                const int64_t* off_sw, const float* noise, const int64_t* off_in, const int64_t* off_out, const float* g,
                                int32_t converters, float* d_part, int32_t* splits, void* stream) {
  if (nstream < 1 || nstream > 2) return fail(DZ_EINVAL, "fc input-gradient test: nstream 1..2");
  UmNetDesc d;
  memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.npass = 1;
  d.online = online; d.target = online;
  d.use_fc = 1; d.nstream = nstream; d.noisy = noisy ? 1 : 0;
  for (int s = 0; s < nstream; ++s) {
    d.off_fc_w[s] = off_w[s];
    if (noisy) { d.off_fc_sw[s] = off_sw[s]; d.noise_off_in[s] = off_in[s]; d.noise_off_out[s] = off_out[s]; }
  }
  if (!um_net_supported(d)) return fail(DZ_EINVAL, "fc input-gradient test: geometry not supported by the tensor-core path");
  char* ws = nullptr;
  DZ_CUDA_OK(cudaMalloc(&ws, (size_t)um_net_workspace_bytes(d)));
  UmNet* n = nullptr;
  int rc = net_create(d, ws, &n, false);
  if (rc == DZ_OK) rc = um_split(g, n->dh1_hi, n->dh1_lo, (long long)nstream * B * 512, stream);
  if (rc == DZ_OK && noisy) rc = apply_noise(n, noise, stream);
  if (rc == DZ_OK) rc = n->plan.launch("fc1_dgrad", n->launches[kFcDgrad], stream, nullptr, converters ? UM_PATH_CONVERTERS : UM_PATH_AUTO);
  if (rc == DZ_OK) {
    const size_t bytes = (size_t)nstream * n->fcd_splits * B * n->feat * sizeof(float);
    if (cudaMemcpyAsync(d_part, n->fcd_part, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) != cudaSuccess ||
        cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
      rc = fail(DZ_ECUDA, "fc input-gradient test: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (rc == DZ_OK) *splits = n->fcd_splits;
  if (n) um_net_destroy(n);
  cudaFree(ws);
  return rc;
}

// Test hook: the conv1 forward launch alone, on the uint8 observations of B x H x W x 4 (rows[p]: host array of the
// npass device row-pointer tables, one observation per pointer), with the pass layout of dz_test_fc_forward (passes 0
// and 1 apply the online blob when npass is 3; otherwise pass 0 is online and pass 1 target).  The conv weights of
// both blobs are at off_conv_w[0..2] (all three layers are packed), conv1's bias at off_conv_b1.  path: 2 the
// learner's conv1_wgmma_kernel, 1 the mma.sync conv1_umma_kernel.  Writes act1 hi / lo [npass * B][h1][w1][32].
extern "C" int dz_test_conv1_forward(int32_t B, int32_t H, int32_t W, int32_t npass, const float* online, const float* target,
                                     const int64_t* off_conv_w, int64_t off_conv_b1, const uint8_t* const* const* rows,
                                     int32_t path, float* d_hi, float* d_lo, void* stream) {
  if (npass < 1 || npass > 3) return fail(DZ_EINVAL, "conv1 forward test: npass 1..3");
  if (path != UM_PATH_MMA_SYNC && path != UM_PATH_WGMMA) return fail(DZ_EINVAL, "conv1 forward test: path 1 (mma.sync) or 2 (wgmma)");
  UmNetDesc d;
  memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.npass = npass;
  d.pass_target[0] = 0; d.pass_target[1] = npass == 3 ? 0 : 1; d.pass_target[2] = 1;
  d.online = online; d.target = target;
  for (int L = 0; L < 3; ++L) d.off_conv_w[L] = off_conv_w[L];
  d.off_conv_b[0] = off_conv_b1;
  if (!um_net_supported(d)) return fail(DZ_EINVAL, "conv1 forward test: geometry not supported by the tensor-core path");
  char* ws = nullptr;
  DZ_CUDA_OK(cudaMalloc(&ws, (size_t)um_net_workspace_bytes(d)));
  UmNet* n = nullptr;
  int rc = net_create(d, ws, &n, false);
  if (rc == DZ_OK) rc = um_pack_weights(n, stream);
  if (rc == DZ_OK) rc = launch_conv1(n, rows, stream, path == UM_PATH_MMA_SYNC);
  if (rc == DZ_OK) {
    const size_t bytes = (size_t)npass * B * n->h1 * n->w1 * 32 * sizeof(float);
    if (cudaMemcpyAsync(d_hi, n->act_hi[0], bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) != cudaSuccess ||
        cudaMemcpyAsync(d_lo, n->act_lo[0], bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream) != cudaSuccess ||
        cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
      rc = fail(DZ_ECUDA, "conv1 forward test: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (n) um_net_destroy(n);
  cudaFree(ws);
  return rc;
}
