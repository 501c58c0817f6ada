// Internal (non-ABI) declarations shared between the replay and learner translation units.
#pragma once
#include "dz_common.cuh"

namespace dz {

// Optional per-batch outputs the fused learner path wants straight from the sampler:
// row pointers into the replay store (the gather is fused into the conv1 operand load) and the
// float32/int32 scalars exactly as they enter jit(update).
struct BatchExtras {
  const uint8_t** d_s_tm1_rows;
  const uint8_t** d_s_t_rows;
  int32_t* d_a;
  float* d_r;
  float* d_disc;
  float* d_w;
  int fused;
  // frame-deduplicated replay: the row tables point at [B][2][obs_stride] here, filled by launch_frame_reconstruct
  const uint8_t* recon;
};

int launch_sample(const dz_replay_view* view, int prioritized, const dz_sample_inputs* in, const dz_sample_outputs* out,
                  int batch, const BatchExtras& ex, void* stream);
int launch_update_priorities(const dz_replay_view* view, const int64_t* d_indices, const float* d_priorities, int n,
                             double alpha, int64_t size, void* stream);

// splitmix64 finaliser: the counter hash of the synthetic fills (oracle/replay_oracle.py:_mix64) and the frame hash
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// ---- frame-deduplicated replay layout (dz_frames.cu) ----------------------------------------------------------------
constexpr int kMaxObsChannels = 32;
// One add: resolves the 2*C planes of (src_tm1, src_t) (device pointers, HWC) into row `slot` (see dz_replay_add).
int launch_frame_add(const dz_replay_view* view, int64_t slot, int release_row, const uint8_t* src_tm1,
                     const uint8_t* src_t, void* stream);
// HWC stacks of rows slots[0..batch): s_tm1 of b at dst_tm1 + b * pitch, s_t at dst_t + b * pitch.
int launch_frame_reconstruct(const dz_replay_view* view, const int64_t* d_slots, int batch, uint8_t* dst_tm1,
                             uint8_t* dst_t, int64_t pitch, void* stream);
// Batched add (dz_replay_add_batch): at most kMaxAddBatch adds per call (2 * K leaf writes in one block_tree_set), and
// in the frame-deduplicated layout at most kMaxBatchPlanes = K * 2 * C planes (the resolve kernel's shared memory).
constexpr int kMaxAddBatch = 512;
constexpr int kMaxBatchPlanes = 2048;
// Workspace bytes of the frame pool's part of a batch of up to max_count adds (the planar planes and the match results).
int64_t frame_add_batch_workspace(const dz_replay_view* view, int64_t max_count);
// Plane ids of the rows of `b` (observations at src_tm1 / src_t + k * pitch, device memory); ws: frame_add_batch_workspace bytes.
int launch_frame_add_batch(const dz_replay_view* view, const dz_add_batch* b, const uint8_t* src_tm1,
                           const uint8_t* src_t, int64_t pitch, uint8_t* ws, void* stream);
int launch_frame_pool_reset(const dz_replay_view* view, void* stream);
int launch_frame_fill_stacked(const dz_replay_view* view, int64_t n, uint64_t seed, int64_t episode_len, void* stream);

// Word w of frame f of synthetic episode e (dz_replay_fill_synthetic_stacked); words = H*W/8.
__device__ __forceinline__ uint64_t stacked_frame_word(uint64_t seed, int64_t e, int64_t f, int64_t episode_len,
                                                       int64_t words, int64_t w) {
  return mix64(seed * 0x9E3779B97F4A7C15ull + 0x632BE59BD9B4E019ull +
               (uint64_t)(e * (episode_len + 1) + f) * (uint64_t)words + (uint64_t)w);
}
// Frame held by channel c of the stack after frames 0..step (trailing-zero padded while step + 1 < C); -1 = zeros.
__device__ __forceinline__ int64_t stacked_channel_frame(int64_t step, int c, int C) {
  if (step + 1 < C) return c <= step ? c : -1;
  return step - (C - 1) + c;
}


// ---- packed-operand tensor-core GEMM (dz_tcp.cuh / dz_tcp.cu) ------------------------------------------------------
constexpr int kPkKB = 16;         // reduction elements per k-block / pipeline stage
constexpr int kPkMaxJobs = 8;
constexpr int kPkMaxProblems = 4;

struct PackJob {
  const float* src;
  int ld;
  int red_contig;          // 1: element (row, r) at src[row * ld + r];  0: at src[r * ld + row]
  int rows, red;           // valid extents (everything outside reads as zero)
  int rows_pad, red_pad;   // image extents
  int ones_row;            // row index that reads as 1.0 for every valid r (bias-gradient row), or -1
  float* hi;
  float* lo;
  int tiles_r;             // 64-row tiles per 64-deep slab
  int block0;              // first block of this job in the flattened grid
};
struct PackBatch { PackJob job[kPkMaxJobs]; int n; int blocks; };

struct PkOperand { const float* hi; const float* lo; int rg_total; };   // rg_total = rows_pad / 8
struct PkProblem {
  PkOperand A, B;          // A: 128-row tiles (rows i), B: BNJ-row tiles (rows j)
  int MI, NJ, nkb;         // nkb = red_pad / 16
  float* C;                // partial s at C + s * split_stride; element (i,j) at i * sc_i + j * sc_j
  long long sc_i, sc_j, split_stride;
  int splits;
  const float* bias_j;     // splits == 1 only: + bias_j[j], then optional ReLU
  int relu;
  // EPI 1 (IQN embedding epilogue; dz_tcp.cuh): v = relu(acc + bias_j[j]) -> e0[i * e0_ld + j] (optional);
  // h = v * mul[(i / mul_div) * mul_ld + j] -> hi/lo images with rows i (img_*) and optionally rows j (imgT_*)
  float* e0; int e0_ld;
  const float* mul; int mul_div, mul_ld;
  float *img_hi, *img_lo; int img_rg;
  float *imgT_hi, *imgT_lo; int imgT_rg;
};
struct PkBatch { PkProblem p[kPkMaxProblems]; int n; };


// Packed "tile image" of a GEMM operand (dz_tcp.cuh) with `rows_pad` rows (multiple of the tile height) and `red_pad`
// reduction elements (multiple of 16), rg = rows_pad / 8 row groups: the float index of element (row, r) is
//     (((r / 16) * rg + row / 8) * 4 + (r % 16) / 4) * 32 + (row % 8) * 4 + r % 4
// i.e. per 16-deep k-block all rows are contiguous, in 8-row x 16-byte blocks, so a (TR rows x 16) tile is TR * 64
// contiguous bytes and the m16n8k8 fragment loads from it are bank-conflict free.
__host__ __device__ __forceinline__ long long pk_index(int row, int r, int rg) {
  return ((((long long)(r >> 4) * rg + (row >> 3)) * 4 + ((r & 15) >> 2)) << 5) + (row & 7) * 4 + (r & 3);
}
// Byte offset of element (row, r < kPkKB) inside one k-block of an image, i.e. 4 * pk_index(row, r, 0) in 32-bit
// arithmetic.  Written out rather than through pk_index: the 64-bit form changes the GEMM's MMA loop code.
__device__ __forceinline__ uint32_t pk_off(int row, int r) { return (uint32_t)((((row >> 3) * 4 + (r >> 2)) << 7) + ((row & 7) << 4) + ((r & 3) << 2)); }
inline int64_t pk_image_floats(int rows_pad, int red_pad) { return (int64_t)rows_pad * red_pad; }
int pk_add_job(PackBatch& pb, const float* src, int ld, int red_contig, int rows, int red, int rows_pad, int red_pad,
               int ones_row, float* hi, float* lo);
int launch_pack(const char* tag, const PackBatch& pb, void* stream);
int pk_set_ones_row(float* hi, int rows_pad, int row, int red, void* stream);   // image element (row, r < red) = 1
int launch_pgemm(const char* tag, const PkBatch& kb, void* stream, int epi = 0);
// A tile image an epilogue writes: rg = rows_pad / 8; hi == nullptr: none.
struct PkTarget { float* hi; float* lo; int rg; };
// The EPI 1 problem (IQN embedding, dz_tcp.cuh) of one network apply: rows i < M of the cosine image `cos` against the
// embedding weight image `weT` (rows j < D), nkb k-blocks; v = relu(acc + bias[j]) -> e0 [M][D] (optional), h = v *
// mul[(i / mul_div) * mul_ld + j] -> img (rows i) and imgT (rows j, optional).  The learner's forward and
// dz_test_iqn_embed_packed build their problem with this function.
PkProblem pk_embed_problem(const PkOperand& cos, const PkOperand& weT, int M, int D, int nkb, const float* bias,
                           const float* mul, int mul_div, int mul_ld, float* e0, const PkTarget& img, const PkTarget& imgT);

}  // namespace dz
