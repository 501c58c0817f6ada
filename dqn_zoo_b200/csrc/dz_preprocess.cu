// Atari frame preprocessing on the device (reference: dqn_zoo/processors.py:367-388 rgb2y + resize, :482-501 the
// observation branch of processors.atari()): for every environment stream
//     new = PillowBilinearResize( uint8( luma( max(frame_a, frame_b) ) ) )          (uint8 [out_h][out_w])
// pushed into that stream's frame stack uint8 [out_h][out_w][stack] (a deque: append while it is filling, shift
// left by one channel once it is full; processors.py:492-500).
//
// Byte/integer work, bound by the 2 x 100 KB of raw frame reads per stream: one CTA owns a band of output rows,
// brings exactly the input rows that band needs of both raw frames into shared memory with two cp.async.bulk (TMA)
// copies, takes their byte-wise max (__vmaxu4), converts to luma in float64 with the reference's rounding order (see oracle/processors_oracle.py:rgb2y —
// products rounded separately, summed left to right, truncated), then runs Pillow's two fixed-point passes
// (22-bit coefficients, int32 accumulators, uint8 intermediate image) out of shared memory.
#include "dz_async.cuh"
#include "dz_common.cuh"

namespace dz {
namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;   // Pillow Resample.c PRECISION_BITS for 8-bit images
constexpr int kBandRowsPerCTA = 12;           // output rows per CTA: 84 rows = 7 bands

struct PreprocessArgs {
  const uint8_t* const* frame_a;
  const uint8_t* const* frame_b;
  dz_resample_axis h, v;
  uint8_t* const* stacks;
  const int32_t* counts;
  int stack;
  double wr, wg, wb;
  uint32_t fr, fg, fb;                       // the same weights rounded to 2^-23 (fast-path screen)
  int max_rows;                              // input rows staged per band (shared-memory carve)
  int tab_offset;                            // byte offset of the coefficient tables in shared memory
  int band;                                  // output rows per CTA
};

__device__ __forceinline__ uint8_t clip8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

__global__ void __launch_bounds__(256) atari_preprocess_kernel(const PreprocessArgs a) {
  dz::pdl_enter();
  extern __shared__ __align__(16) uint8_t smem[];
  const int env = blockIdx.y;
  const int kBandRows = a.band;
  const int y0 = blockIdx.x * kBandRows, y1 = min(y0 + kBandRows, a.v.out_size);
  const int in_w = a.h.in_size, out_w = a.h.out_size;
  const int row_bytes = in_w * 3, row_words = row_bytes >> 2;
  // input rows this band touches: windows of consecutive output rows are monotone
  const int r0 = a.v.d_bounds[2 * y0];
  const int r1 = a.v.d_bounds[2 * (y1 - 1)] + a.v.d_bounds[2 * (y1 - 1) + 1];
  const int rows = r1 - r0;
  // shared memory: [raw frame a rows][raw frame b rows][gray][hpass][tables][mbarrier]
  uint32_t* raw_a = reinterpret_cast<uint32_t*>(smem);                       // [max_rows][row_words]
  uint32_t* raw_b = raw_a + (size_t)a.max_rows * row_words;
  uint8_t* gray = smem + (size_t)2 * a.max_rows * row_bytes;                 // [max_rows][in_w]
  uint8_t* hpass = gray + (size_t)a.max_rows * in_w;                         // [max_rows][out_w]
  int32_t* tab = reinterpret_cast<int32_t*>(smem + a.tab_offset);
  int32_t* hb = tab;                                  // [out_w][2]
  int32_t* hk = hb + 2 * out_w;                       // [out_w][ksize_h]
  int32_t* vb = hk + out_w * a.h.ksize;               // [band][2]
  int32_t* vk = vb + 2 * kBandRows;                   // [band][ksize_v]
  uint64_t* bar = reinterpret_cast<uint64_t*>(vk + kBandRows * a.v.ksize + ((kBandRows * a.v.ksize + out_w * a.h.ksize) & 1));

  // The rows a band needs are one contiguous byte range of each raw frame: one thread starts two bulk copies
  // (TMA, completes on the mbarrier) and everybody stages the coefficient tables meanwhile.
  const uint8_t* fa = a.frame_a[env];
  const uint8_t* fb = a.frame_b[env];
  const uint32_t bytes = (uint32_t)rows * (uint32_t)row_bytes;               // multiple of 16 (host-checked)
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbarrier_init();
    mbar_expect_tx(bar, (fa ? bytes : 0u) + (fb ? bytes : 0u));
    if (fa) bulk_g2s(smem_u32(raw_a), fa + (size_t)r0 * row_bytes, bytes, bar);
    if (fb) bulk_g2s(smem_u32(raw_b), fb + (size_t)r0 * row_bytes, bytes, bar);
  }
  for (int i = threadIdx.x; i < 2 * out_w; i += blockDim.x) hb[i] = a.h.d_bounds[i];
  for (int i = threadIdx.x; i < out_w * a.h.ksize; i += blockDim.x) hk[i] = a.h.d_kk[i];
  for (int i = threadIdx.x; i < 2 * (y1 - y0); i += blockDim.x) vb[i] = a.v.d_bounds[2 * y0 + i];
  for (int i = threadIdx.x; i < (y1 - y0) * a.v.ksize; i += blockDim.x) vk[i] = a.v.d_kk[(size_t)y0 * a.v.ksize + i];
  __syncthreads();                                    // barrier initialised + tables visible
  mbar_wait(bar, 0);
  // luma: one thread = 4 consecutive pixels = 12 bytes = 3 aligned words in, 1 word out
  const int n4 = (rows * in_w) >> 2;                  // in_w % 4 == 0 follows from row_bytes % 16 == 0
  uint32_t* gray32 = reinterpret_cast<uint32_t*>(gray);
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    // np.max over the pooled pair (:487); a missing frame is zero padding
    const uint32_t w0 = __vmaxu4(fa ? raw_a[3 * i] : 0u, fb ? raw_b[3 * i] : 0u);
    const uint32_t w1 = __vmaxu4(fa ? raw_a[3 * i + 1] : 0u, fb ? raw_b[3 * i + 1] : 0u);
    const uint32_t w2 = __vmaxu4(fa ? raw_a[3 * i + 2] : 0u, fb ? raw_b[3 * i + 2] : 0u);
    const uint32_t px[4][3] = {{w0 & 255u, (w0 >> 8) & 255u, (w0 >> 16) & 255u},
                               {w0 >> 24, w1 & 255u, (w1 >> 8) & 255u},
                               {(w1 >> 16) & 255u, w1 >> 24, w2 & 255u},
                               {(w2 >> 8) & 255u, (w2 >> 16) & 255u, w2 >> 24}};
    uint32_t out = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // Fast path: 8.23 fixed-point luma in one 32-bit word.  The weights are rounded to 2^-23, so the sum is within
      // 255 * 1.5 * 2^-23 = 4.6e-5 of the exact value, and floor() can only be in doubt when the fractional part is
      // within 2^-13 of an integer.  With the reference's weights the exact luma is a multiple of 0.001 (up to
      // 1e-13), so that is the ~1 colour in 1000 whose luma IS an integer; only those pixels take the reference's
      // float64 sequence (the instruction count is what bounds this kernel).
      const uint32_t v = px[e][0] * a.fr + px[e][1] * a.fg + px[e][2] * a.fb;
      const uint32_t frac = v & ((1u << 23) - 1);
      uint32_t y = v >> 23;
      if (frac < (1u << 10) || frac > (1u << 23) - (1u << 10)) {
        // fl(fl(fl(r*wr) + fl(g*wg)) + fl(b*wb)), truncated: processors.py:367-371 in the golden vector's rounding order
        double t = __dadd_rn(__dadd_rn(__dmul_rn((double)px[e][0], a.wr), __dmul_rn((double)px[e][1], a.wg)),
                             __dmul_rn((double)px[e][2], a.wb));
        y = (uint32_t)(int)t;
      }
      out |= (y & 255u) << (8 * e);
    }
    gray32[i] = out;
  }
  __syncthreads();
  // Resampling passes: one thread owns one output COLUMN xx (window + coefficients in registers, no divisions) and
  // walks down the rows; `lanes` such column-walkers run side by side.
  const int lanes = blockDim.x / out_w;
  const int ksh = a.h.ksize, ksv = a.v.ksize;
  const int count = a.counts[env];
  uint8_t* stack = a.stacks[env];
  if (lanes >= 1 && ksh <= 8) {
    const int xx = threadIdx.x % out_w, lane_row = threadIdx.x / out_w;
    if (lane_row < lanes) {
      const int xmin = hb[2 * xx], cnt = hb[2 * xx + 1];
      int k[8];
#pragma unroll
      for (int x = 0; x < 8; ++x) k[x] = x < cnt ? hk[xx * ksh + x] : 0;
      for (int r = lane_row; r < rows; r += lanes) {                         // horizontal pass
        const uint8_t* src = gray + (size_t)r * in_w + xmin;
        int acc = 1 << (kPrecisionBits - 1);
#pragma unroll
        for (int x = 0; x < 8; ++x) if (x < cnt) acc += (int)src[x] * k[x];
        hpass[r * out_w + xx] = clip8(acc >> kPrecisionBits);
      }
    }
  } else {
    for (int i = threadIdx.x; i < rows * out_w; i += blockDim.x) {
      const int r = i / out_w, xx = i - r * out_w;
      const int xmin = hb[2 * xx], cnt = hb[2 * xx + 1];
      const int32_t* k = hk + xx * ksh;
      const uint8_t* src = gray + (size_t)r * in_w + xmin;
      int acc = 1 << (kPrecisionBits - 1);
      for (int x = 0; x < cnt; ++x) acc += (int)src[x] * k[x];
      hpass[i] = clip8(acc >> kPrecisionBits);
    }
  }
  __syncthreads();
  const bool word_stack = a.stack == 4 && (reinterpret_cast<uintptr_t>(stack) & 3) == 0;
  auto vertical_output = [&](int yl, int xx) {                               // vertical pass + push into the stack
    const int yy = y0 + yl;
    const int ymin = vb[2 * yl], cnt = vb[2 * yl + 1];
    const int32_t* k = vk + yl * ksv;                                        // same yl across a warp: broadcast reads
    const uint8_t* col = hpass + (size_t)(ymin - r0) * out_w + xx;
    int acc = 1 << (kPrecisionBits - 1);
    for (int y = 0; y < cnt; ++y) acc += (int)col[y * out_w] * k[y];
    const uint8_t v = clip8(acc >> kPrecisionBits);
    uint8_t* px = stack + ((size_t)yy * out_w + xx) * a.stack;
    if (count < a.stack) {
      px[count] = v;                                                         // still filling: trailing channels stay zero
    } else if (word_stack) {
      uint32_t* w = reinterpret_cast<uint32_t*>(px);                         // deque(maxlen=4): one word per pixel
      *w = (*w >> 8) | ((uint32_t)v << 24);
    } else {
      for (int c = 0; c + 1 < a.stack; ++c) px[c] = px[c + 1];               // deque(maxlen): drop the oldest frame
      px[a.stack - 1] = v;
    }
  };
  if (lanes >= 1) {
    const int xx = threadIdx.x % out_w, lane_row = threadIdx.x / out_w;
    if (lane_row < lanes)
      for (int yl = lane_row; yl < y1 - y0; yl += lanes) vertical_output(yl, xx);
  } else {
    for (int i = threadIdx.x; i < (y1 - y0) * out_w; i += blockDim.x) vertical_output(i / out_w, i % out_w);
  }
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" int dz_atari_preprocess(const uint8_t* const* d_frame_a, const uint8_t* const* d_frame_b, int32_t n_env,
                                   const dz_resample_axis* horizontal, const dz_resample_axis* vertical,
                                   uint8_t* const* d_stacks, const int32_t* d_counts, int32_t stack, const double* luma3,
                                   int32_t max_band_rows, void* stream) {
  if (n_env <= 0) return DZ_OK;
  if (!d_frame_a || !d_frame_b || !horizontal || !vertical || !d_stacks || !d_counts || !luma3)
    return fail(DZ_EINVAL, "dz_atari_preprocess: null argument");
  if ((horizontal->in_size * 3) % 16) return fail(DZ_EINVAL, "dz_atari_preprocess: row bytes (3 * width) must be a multiple of 16");
  if (stack < 1) return fail(DZ_EINVAL, "dz_atari_preprocess: stack geometry");
  if (max_band_rows < 1 || max_band_rows > vertical->in_size) return fail(DZ_EINVAL, "dz_atari_preprocess: max_band_rows");
  PreprocessArgs a;
  a.frame_a = d_frame_a; a.frame_b = d_frame_b; a.h = *horizontal; a.v = *vertical; a.stacks = d_stacks;
  a.counts = d_counts; a.stack = stack; a.wr = luma3[0]; a.wg = luma3[1]; a.wb = luma3[2];
  a.fr = (uint32_t)llround(luma3[0] * 8388608.0); a.fg = (uint32_t)llround(luma3[1] * 8388608.0);
  a.fb = (uint32_t)llround(luma3[2] * 8388608.0);
  if (luma3[0] < 0 || luma3[1] < 0 || luma3[2] < 0 || luma3[0] + luma3[1] + luma3[2] > 1.0000001)
    return fail(DZ_EINVAL, "dz_atari_preprocess: luma weights must be non-negative and sum to at most 1");
  a.max_rows = max_band_rows;
  size_t smem = (size_t)max_band_rows * (2 * horizontal->in_size * 3 + horizontal->in_size + horizontal->out_size);
  smem = (smem + 15) / 16 * 16;
  a.tab_offset = (int)smem;
  smem += sizeof(int32_t) * ((size_t)horizontal->out_size * (2 + horizontal->ksize) + (size_t)kBandRowsPerCTA * (2 + vertical->ksize) + 1) + 16;
  a.band = kBandRowsPerCTA;
  if (smem > 200 * 1024) return fail(DZ_EINVAL, "dz_atari_preprocess: band does not fit in shared memory");
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    DZ_CUDA_OK(cudaFuncSetAttribute(atari_preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  dim3 grid((unsigned)ceil_div(vertical->out_size, kBandRowsPerCTA), (unsigned)n_env);
  DZ_LAUNCH(atari_preprocess_kernel, grid, 256, smem, stream, a);
  return DZ_OK;
}

extern "C" int32_t dz_atari_preprocess_band_rows(void) { return kBandRowsPerCTA; }
