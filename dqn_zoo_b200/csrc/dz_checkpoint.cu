// Checkpoint transfers (DESIGN.md §9): the chunk digest, the frame pool's export (live-plane list, plane gather) and
// import (plane scatter, refcount / hash / table rebuild with consistency checks), and the pitched row copies of the
// transition-major layout.
//
// Chunk digest of n bytes: split into 8-byte little-endian words w_0 .. w_{m-1}, m = ceil(n / 8), the last word zero
// padded; digest = mix64(S ^ n) with S = sum_i mix64(w_i ^ ((i + 1) * 0x9E3779B97F4A7C15)) mod 2^64.  The sum is
// taken with wrapping 64-bit adds, which are associative and commutative, so every reduction order (per-thread
// partials, warp shuffles, atomics across CTAs) gives the same S.  For n = frame_stride it is the frame pool's plane
// hash (dz_frames.cu:plane_hash_warp).  Restated in numpy in oracle/checkpoint_oracle.py.
#include "dz_internal.cuh"

namespace dz {

namespace {

constexpr uint64_t kDigestKey = 0x9E3779B97F4A7C15ull;

__host__ __device__ __forceinline__ uint64_t ckpt_mix64(uint64_t x) {
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__host__ __device__ __forceinline__ uint64_t ckpt_word_hash(uint64_t w, int64_t i) {
  return ckpt_mix64(w ^ ((uint64_t)(i + 1) * kDigestKey));
}

// Word i of an n-byte range (the last one zero padded); p is 8-byte aligned.
__host__ __device__ __forceinline__ uint64_t ckpt_word(const uint8_t* p, int64_t n, int64_t i) {
  if (8 * i + 8 <= n) return reinterpret_cast<const uint64_t*>(p)[i];
  uint64_t w = 0;
  for (int64_t b = 8 * i; b < n; ++b) w |= (uint64_t)p[b] << (8 * (b - 8 * i));
  return w;
}

__global__ void __launch_bounds__(256) ckpt_digest_kernel(const uint8_t* __restrict__ p, int64_t n,
                                                          unsigned long long* acc) {
  dz::pdl_enter();
  const int64_t words = (n + 7) >> 3;
  uint64_t s = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < words; i += (int64_t)gridDim.x * blockDim.x)
    s += ckpt_word_hash(ckpt_word(p, n, i), i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(acc, (unsigned long long)s);
}

__global__ void ckpt_digest_final_kernel(unsigned long long* acc, int64_t n) {
  dz::pdl_enter();
  if (threadIdx.x == 0) *acc = ckpt_mix64(*acc ^ (uint64_t)n);
}

static __device__ __forceinline__ uint8_t* pool_plane(const dz_replay_view& v, int64_t id) {
  return v.d_frames + id * v.frame_stride;
}

// Live planes (refcount > 0, plane 0 excluded) in increasing id order, with their hashes: one CTA scans the refcounts
// tile by tile (each thread 8 consecutive ids), so the output order is the id order whatever the timing.
constexpr int kCompactThreads = 1024, kCompactPer = 8;
__global__ void __launch_bounds__(kCompactThreads) pool_compact_kernel(dz_replay_view v, int32_t* out_ids,
                                                                       uint64_t* out_hashes, int64_t* count) {
  dz::pdl_enter();
  __shared__ int32_t s_warp[kCompactThreads / 32];
  __shared__ int64_t s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  const int64_t tile = (int64_t)kCompactThreads * kCompactPer;
  for (int64_t t0 = 0; t0 < v.frame_capacity; t0 += tile) {
    const int64_t first = t0 + (int64_t)threadIdx.x * kCompactPer;
    unsigned live = 0;
#pragma unroll
    for (int k = 0; k < kCompactPer; ++k) {
      const int64_t id = first + k;
      if (id > 0 && id < v.frame_capacity && v.d_refcount[id] > 0) live |= 1u << k;
    }
    const int mine = __popc(live);
    int incl = mine;   // inclusive scan within the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += x;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += x;
      }
      s_warp[lane] = wi - w;   // exclusive prefix of the warps
    }
    __syncthreads();
    int64_t pos = s_base + s_warp[warp] + incl - mine;
    for (int k = 0; k < kCompactPer; ++k)
      if (live >> k & 1u) {
        out_ids[pos] = (int32_t)(first + k);
        out_hashes[pos] = v.d_hashes[first + k];
        ++pos;
      }
    __syncthreads();   // every thread has read s_base and s_warp
    if (threadIdx.x == kCompactThreads - 1) s_base = pos;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = s_base;
}

// Planes ids[0..n) <-> a packed buffer of n * frame_bytes bytes (no stride padding); a warp per plane.  On import the
// padding bytes [frame_bytes, frame_stride) are zeroed, as every add leaves them.
__global__ void __launch_bounds__(256) pool_gather_kernel(dz_replay_view v, const int32_t* __restrict__ ids, int64_t n,
                                                          uint8_t* __restrict__ dst) {
  dz::pdl_enter();
  const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (q >= n) return;
  const uint8_t* src = pool_plane(v, ids[q]);
  uint8_t* out = dst + q * v.frame_bytes;
  const int lane = threadIdx.x & 31;
  if ((v.frame_bytes & 15) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(out);
    for (int64_t i = lane; i < (v.frame_bytes >> 4); i += 32) d4[i] = s4[i];
  } else {
    for (int64_t i = lane; i < v.frame_bytes; i += 32) out[i] = src[i];
  }
}

__global__ void __launch_bounds__(256) pool_scatter_kernel(dz_replay_view v, const int32_t* __restrict__ ids, int64_t n,
                                                           const uint8_t* __restrict__ src, int32_t* bad) {
  dz::pdl_enter();
  const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (q >= n) return;
  const int32_t id = ids[q];
  if (id <= 0 || id >= v.frame_capacity) {
    if ((threadIdx.x & 31) == 0) atomicOr(bad, DZ_CKPT_BAD_PLANE_ID);
    return;
  }
  uint8_t* dst = pool_plane(v, id);
  const uint8_t* in = src + q * v.frame_bytes;
  const int lane = threadIdx.x & 31;
  if ((v.frame_bytes & 15) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(in);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (int64_t i = lane; i < (v.frame_bytes >> 4); i += 32) d4[i] = s4[i];
  } else {
    for (int64_t i = lane; i < v.frame_bytes; i += 32) dst[i] = in[i];
  }
  for (int64_t i = v.frame_bytes + lane; i < v.frame_stride; i += 32) dst[i] = 0;
}

// Refcounts from the plane ids of the live rows (the pool was reset: all 0 but plane 0's permanent reference).
__global__ void __launch_bounds__(256) pool_refcount_kernel(dz_replay_view v, const int64_t* __restrict__ slots,
                                                            int64_t n, int32_t* bad) {
  dz::pdl_enter();
  const int64_t P = 2 * v.obs_channels;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n * P; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t slot = slots[i / P];
    if (slot < 0 || slot >= v.capacity) { atomicOr(bad, DZ_CKPT_BAD_PLANE_ID); continue; }
    const int32_t id = v.d_planes[slot * P + i % P];
    if (id < 0 || id >= v.frame_capacity) { atomicOr(bad, DZ_CKPT_BAD_PLANE_ID); continue; }
    atomicAdd(&v.d_refcount[id], 1);
  }
}

// A warp per listed plane: the list is strictly increasing and names referenced planes only; the recomputed hash
// equals the saved one; the plane goes into the table.  live[0] counts the listed planes (all of them must be live).
__global__ void __launch_bounds__(256) pool_rehash_kernel(dz_replay_view v, const int32_t* __restrict__ ids, int64_t n,
                                                          const uint64_t* __restrict__ saved, int32_t* bad) {
  dz::pdl_enter();
  const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (q >= n) return;
  const int32_t id = ids[q];
  const bool lane0 = (threadIdx.x & 31) == 0;
  if (id <= 0 || id >= v.frame_capacity || (q > 0 && ids[q - 1] >= id)) {
    if (lane0) atomicOr(bad, DZ_CKPT_BAD_PLANE_ID);
    return;
  }
  const uint64_t h = [&] {
    // plane_hash_warp of dz_frames.cu: the digest of the frame_stride bytes of the plane
    const int lane = threadIdx.x & 31;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(pool_plane(v, id));
    uint64_t acc = 0;
    for (int64_t i = lane; i < (v.frame_stride >> 3); i += 32) acc += ckpt_word_hash(w[i], i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    return ckpt_mix64(acc ^ (uint64_t)v.frame_stride);
  }();
  if (!lane0) return;
  if (v.d_refcount[id] <= 0) atomicOr(bad, DZ_CKPT_UNREFERENCED_PLANE);
  if (h != saved[q]) atomicOr(bad, DZ_CKPT_HASH_MISMATCH);
  v.d_hashes[id] = h;
  const int64_t mask = v.table_size - 1;
  int64_t t = (int64_t)(h & (uint64_t)mask);
  while (atomicCAS(&v.d_table[t], -1, id) != -1) t = (t + 1) & mask;
}

// Every referenced plane but plane 0 is listed: the planes with refcount > 0 number exactly n + 1; every free-stack
// entry names an unreferenced plane.
__global__ void __launch_bounds__(256) pool_check_kernel(dz_replay_view v, int64_t n, int64_t top, int32_t* bad) {
  dz::pdl_enter();
  __shared__ unsigned long long s_live;
  if (threadIdx.x == 0) s_live = 0;
  __syncthreads();
  unsigned long long live = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v.frame_capacity; i += (int64_t)gridDim.x * blockDim.x)
    live += v.d_refcount[i] > 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < top; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t id = v.d_free[i];
    if (id <= 0 || id >= v.frame_capacity || v.d_refcount[id] != 0) atomicOr(bad, DZ_CKPT_BAD_FREE_STACK);
  }
  if (live) atomicAdd(&s_live, live);
  __syncthreads();
  if (threadIdx.x == 0 && s_live) atomicAdd(reinterpret_cast<unsigned long long*>(bad + 2), s_live);
}

int grid_for(int64_t work, int block) {
  const int64_t g = ceil_div(work, block);
  return (int)(g < kNumSMs * 16 ? (g > 0 ? g : 1) : kNumSMs * 16);
}

int check_pool(const dz_replay_view* v) {
  if (!v->d_frames || !v->d_planes || !v->d_refcount || !v->d_hashes || !v->d_table || !v->d_free || !v->d_pool_counters)
    return fail(DZ_EINVAL, "not a frame-deduplicated replay view");
  if (v->frame_stride < v->frame_bytes || v->frame_stride % 16 || v->frame_bytes < 1)
    return fail(DZ_EINVAL, "frame_stride must be a multiple of 16 >= frame_bytes");
  if (v->table_size < 2 * v->frame_capacity || (v->table_size & (v->table_size - 1)))
    return fail(DZ_EINVAL, "table_size must be a power of two >= 2 * frame_capacity");
  if (v->obs_channels < 1 || v->obs_channels > kMaxObsChannels) return fail(DZ_EINVAL, "obs_channels must be in [1,32]");
  return DZ_OK;
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_ckpt_digest(const void* d_src, int64_t bytes, uint64_t* d_out, void* stream) {
  if (bytes < 0) return fail(DZ_EINVAL, "bytes must be >= 0");
  if (!d_out || (bytes && !d_src)) return fail(DZ_EINVAL, "null pointer");
  if ((uintptr_t)d_src % 8) return fail(DZ_EINVAL, "the digested range must start 8-byte aligned");
  DZ_CUDA_OK(cudaMemsetAsync(d_out, 0, sizeof(uint64_t), (cudaStream_t)stream));
  if (bytes) {
    const int64_t words = (bytes + 7) >> 3;
    const int grid = (int)std::min<int64_t>(ceil_div(words, 256 * 4), kNumSMs * 8);
    DZ_LAUNCH(ckpt_digest_kernel, grid, 256, 0, stream, static_cast<const uint8_t*>(d_src), bytes,
              reinterpret_cast<unsigned long long*>(d_out));
  }
  DZ_LAUNCH(ckpt_digest_final_kernel, 1, 32, 0, stream, reinterpret_cast<unsigned long long*>(d_out), bytes);
  return DZ_OK;
}

// The same digest computed on the host (the kernel's word hash, compiled for the CPU): digests of host-side files and
// the CPU test-suite's check of the arithmetic.
int dz_ckpt_digest_host(const void* h_src, int64_t bytes, uint64_t* h_out) {
  if (bytes < 0 || !h_out || (bytes && !h_src)) return fail(DZ_EINVAL, "bad argument");
  const uint8_t* p = static_cast<const uint8_t*>(h_src);
  const int64_t words = (bytes + 7) >> 3;
  uint64_t s = 0;
  for (int64_t i = 0; i < words; ++i) {
    uint64_t w = 0;
    memcpy(&w, p + 8 * i, 8 * i + 8 <= bytes ? 8 : (size_t)(bytes - 8 * i));   // little-endian host
    s += ckpt_word_hash(w, i);
  }
  *h_out = ckpt_mix64(s ^ (uint64_t)bytes);
  return DZ_OK;
}

int dz_ckpt_pool_live(const dz_replay_view* view, int32_t* d_ids, uint64_t* d_hashes, int64_t* d_count, void* stream) {
  DZ_TRY(check_pool(view));
  if (!d_ids || !d_hashes || !d_count) return fail(DZ_EINVAL, "null output");
  DZ_LAUNCH(pool_compact_kernel, 1, kCompactThreads, 0, stream, *view, d_ids, d_hashes, d_count);
  return DZ_OK;
}

int dz_ckpt_pool_gather(const dz_replay_view* view, const int32_t* d_ids, int64_t n, uint8_t* d_dst, void* stream) {
  DZ_TRY(check_pool(view));
  if (n < 0) return fail(DZ_EINVAL, "n must be >= 0");
  if (n == 0) return DZ_OK;
  if ((view->frame_bytes & 15) == 0 && (uintptr_t)d_dst % 16) return fail(DZ_EINVAL, "d_dst must be 16-byte aligned");
  DZ_LAUNCH(pool_gather_kernel, (int)ceil_div(n * 32, 256), 256, 0, stream, *view, d_ids, n, d_dst);
  return DZ_OK;
}

int dz_ckpt_pool_scatter(const dz_replay_view* view, const int32_t* d_ids, int64_t n, const uint8_t* d_src,
                         int32_t* d_bad, void* stream) {
  DZ_TRY(check_pool(view));
  if (n < 0 || !d_bad) return fail(DZ_EINVAL, "bad argument");
  if (n == 0) return DZ_OK;
  if ((view->frame_bytes & 15) == 0 && (uintptr_t)d_src % 16) return fail(DZ_EINVAL, "d_src must be 16-byte aligned");
  DZ_LAUNCH(pool_scatter_kernel, (int)ceil_div(n * 32, 256), 256, 0, stream, *view, d_ids, n, d_src, d_bad);
  return DZ_OK;
}

int dz_ckpt_pool_rebuild(const dz_replay_view* view, const int64_t* d_live_slots, int64_t n_live, const int32_t* d_ids,
                         const uint64_t* d_saved_hashes, int64_t n_ids, int64_t top, int32_t* d_bad, void* stream) {
  DZ_TRY(check_pool(view));
  if (n_live < 0 || n_ids < 0 || top < 0 || top > view->frame_capacity || !d_bad)
    return fail(DZ_EINVAL, "bad argument");
  if (n_live)
    DZ_LAUNCH(pool_refcount_kernel, grid_for(n_live * 2 * view->obs_channels, 256), 256, 0, stream, *view, d_live_slots,
              n_live, d_bad);
  if (n_ids)
    DZ_LAUNCH(pool_rehash_kernel, (int)ceil_div(n_ids * 32, 256), 256, 0, stream, *view, d_ids, n_ids, d_saved_hashes,
              d_bad);
  DZ_LAUNCH(pool_check_kernel, grid_for(view->frame_capacity, 256), 256, 0, stream, *view, n_ids, top, d_bad);
  return DZ_OK;
}

int dz_ckpt_rows(const dz_replay_view* view, int64_t first_slot, int64_t n, uint8_t* d_buf, int32_t to_replay,
                 void* stream) {
  if (view->d_planes || !view->d_obs) return fail(DZ_EINVAL, "not a transition-major replay view");
  if (n < 0 || first_slot < 0 || first_slot + n > view->capacity) return fail(DZ_ERANGE, "rows out of range");
  if (n == 0) return DZ_OK;
  uint8_t* rows = view->d_obs + first_slot * 2 * view->obs_stride;
  if (to_replay)
    DZ_CUDA_OK(cudaMemcpy2DAsync(rows, view->obs_stride, d_buf, view->obs_bytes, view->obs_bytes, 2 * n,
                                 cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  else
    DZ_CUDA_OK(cudaMemcpy2DAsync(d_buf, view->obs_bytes, rows, view->obs_stride, view->obs_bytes, 2 * n,
                                 cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return DZ_OK;
}

}  // extern "C"
