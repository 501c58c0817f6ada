// Checkpoint transfers (DESIGN.md §9): the chunk digest, the frame pool's export (live-plane list), the snapshot pass
// that packs either layout's bulk records and digests them per chunk in one read, the pool's
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

// The snapshot pass: records ids[0..n) of the replay's bulk storage packed into dst in file order, and the digest sum S
// of every chunk of that packed stream, in one read of the source.  Record q is `units` pieces of unit_bytes, piece u
// at base + (ids[q] * units + u) * unit_pitch: one plane of the frame pool (units = 1, pitch frame_stride) or the
// s_tm1 | s_t observations of one transition-major row (units = 2, pitch obs_stride).  Chunks hold whole records, so a
// record lies in one chunk; a word may still straddle two records when the record size is not a multiple of 8.
struct SnapSource {
  const uint8_t* base;
  const int32_t* ids;
  int64_t unit_bytes, unit_pitch;
  int units;
};

__device__ __forceinline__ const uint8_t* snap_piece(const SnapSource& s, int64_t q, int u) {
  return s.base + ((int64_t)s.ids[q] * s.units + u) * s.unit_pitch;
}

__device__ __forceinline__ void snap_flush(uint64_t acc, int64_t chunk, unsigned long long* sums) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(&sums[chunk], (unsigned long long)acc);
}

// unit_bytes % 16 == 0 and 16-byte aligned base and dst: a warp per record with 16-byte loads and stores, each warp
// over a contiguous range of records, so it flushes its partial sum once per chunk it touches.
constexpr int kSnapUnroll = 4;
__global__ void __launch_bounds__(256, 4) snapshot_vec_kernel(SnapSource s, int64_t n, uint8_t* __restrict__ dst,
                                                              int64_t recs_per_chunk, unsigned long long* sums) {
  dz::pdl_enter();
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t per = (n + warps - 1) / warps;
  const int64_t q0 = warp * per, q1 = q0 + per < n ? q0 + per : n;
  const int64_t vecs = s.unit_bytes >> 4;                 // 16-byte vectors per piece
  const int64_t rec_words = 2 * vecs * s.units;           // 8-byte words per record
  uint64_t acc = 0;
  int64_t chunk = q0 < q1 ? q0 / recs_per_chunk : 0;
  for (int64_t q = q0; q < q1; ++q) {
    const int64_t k = q / recs_per_chunk;
    if (k != chunk) {
      snap_flush(acc, chunk, sums);
      acc = 0;
      chunk = k;
    }
    uint4* out = reinterpret_cast<uint4*>(dst) + q * vecs * s.units;
    const int64_t w_rec = (q - k * recs_per_chunk) * rec_words;   // the record's first word within its chunk
    for (int u = 0; u < s.units; ++u) {
      const uint4* in = reinterpret_cast<const uint4*>(snap_piece(s, q, u));
      for (int64_t v0 = lane; v0 < vecs; v0 += 32 * kSnapUnroll) {
        uint4 x[kSnapUnroll];
#pragma unroll
        for (int j = 0; j < kSnapUnroll; ++j)
          if (v0 + 32 * j < vecs) x[j] = __ldcs(in + v0 + 32 * j);
#pragma unroll
        for (int j = 0; j < kSnapUnroll; ++j) {
          const int64_t v = v0 + 32 * j;
          if (v < vecs) {
            __stcs(out + u * vecs + v, x[j]);
            const int64_t w = w_rec + 2 * (u * vecs + v);
            acc += ckpt_word_hash((uint64_t)x[j].x | (uint64_t)x[j].y << 32, w) +
                   ckpt_word_hash((uint64_t)x[j].z | (uint64_t)x[j].w << 32, w + 1);
          }
        }
      }
    }
  }
  if (q0 < q1) snap_flush(acc, chunk, sums);
}

// Any geometry: a thread per 8-byte word of a chunk, byte by byte (a word may take bytes of two records and of both
// pieces of a row; the last word of a chunk is zero padded).  Partial sums are flushed when a thread changes chunk.
__global__ void __launch_bounds__(256) snapshot_word_kernel(SnapSource s, int64_t n, uint8_t* __restrict__ dst,
                                                            int64_t chunk_bytes, unsigned long long* sums) {
  dz::pdl_enter();
  const int64_t rec = s.unit_bytes * s.units, total = n * rec;
  const int64_t words_per_chunk = (chunk_bytes + 7) >> 3;
  const int64_t last = (total - 1) / chunk_bytes;
  const int64_t words = last * words_per_chunk + ((total - last * chunk_bytes + 7) >> 3);
  uint64_t acc = 0;
  int64_t chunk = -1;
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < words; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = g / words_per_chunk, i = g - k * words_per_chunk;
    if (k != chunk) {
      if (chunk >= 0 && acc) atomicAdd(&sums[chunk], (unsigned long long)acc);
      acc = 0;
      chunk = k;
    }
    const int64_t c0 = k * chunk_bytes;
    const int64_t end = total - c0 < chunk_bytes ? total - c0 : chunk_bytes;
    uint64_t w = 0;
    for (int64_t b = 8 * i; b < 8 * i + 8 && b < end; ++b) {
      const int64_t p = c0 + b, q = p / rec, r = p - q * rec;
      const int u = (int)(r / s.unit_bytes);
      const uint8_t x = snap_piece(s, q, u)[r - u * s.unit_bytes];
      dst[p] = x;
      w |= (uint64_t)x << (8 * (b - 8 * i));
    }
    acc += ckpt_word_hash(w, i);
  }
  if (chunk >= 0 && acc) atomicAdd(&sums[chunk], (unsigned long long)acc);
}

// digest_k = mix64(S_k ^ bytes of chunk k)
__global__ void __launch_bounds__(256) snapshot_final_kernel(unsigned long long* sums, int64_t nchunks,
                                                             int64_t chunk_bytes, int64_t total) {
  dz::pdl_enter();
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nchunks; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t nk = total - k * chunk_bytes < chunk_bytes ? total - k * chunk_bytes : chunk_bytes;
    sums[k] = ckpt_mix64(sums[k] ^ (uint64_t)nk);
  }
}

// Packed planes -> planes ids[0..n); a warp per plane.  The padding bytes [frame_bytes, frame_stride) are zeroed, as
// every add leaves them.
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

int dz_ckpt_snapshot(const dz_replay_view* view, const int32_t* d_ids, int64_t n, uint8_t* d_dst, int64_t chunk_bytes,
                     uint64_t* d_digests, void* stream) {
  SnapSource s{};
  if (view->d_planes) {
    DZ_TRY(check_pool(view));
    s = SnapSource{view->d_frames, d_ids, view->frame_bytes, view->frame_stride, 1};
  } else {
    if (!view->d_obs || view->obs_bytes < 1 || view->obs_stride < view->obs_bytes)
      return fail(DZ_EINVAL, "neither a frame-deduplicated nor an allocated transition-major replay view");
    s = SnapSource{view->d_obs, d_ids, view->obs_bytes, view->obs_stride, 2};
  }
  const int64_t rec = s.unit_bytes * s.units;
  if (n < 0) return fail(DZ_EINVAL, "n must be >= 0");
  if (chunk_bytes < rec || chunk_bytes % rec) return fail(DZ_EINVAL, "chunk_bytes must be a positive multiple of the record size");
  if (n == 0) return DZ_OK;
  if (!d_ids || !d_dst || !d_digests) return fail(DZ_EINVAL, "null pointer");
  if ((uintptr_t)d_digests % 8) return fail(DZ_EINVAL, "d_digests must be 8-byte aligned");
  const int64_t total = n * rec, nchunks = ceil_div(total, chunk_bytes);
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(d_digests);
  DZ_CUDA_OK(cudaMemsetAsync(d_digests, 0, nchunks * sizeof(uint64_t), (cudaStream_t)stream));
  const bool vec = s.unit_bytes % 16 == 0 && s.unit_pitch % 16 == 0 && (uintptr_t)s.base % 16 == 0 &&
                   (uintptr_t)d_dst % 16 == 0;
  if (vec) {
    const int grid = (int)std::min<int64_t>(ceil_div(n * 32, 256), kNumSMs * 4);
    DZ_LAUNCH(snapshot_vec_kernel, grid, 256, 0, stream, s, n, d_dst, chunk_bytes / rec, sums);
  } else {
    DZ_LAUNCH(snapshot_word_kernel, grid_for(ceil_div(total, 8), 256), 256, 0, stream, s, n, d_dst, chunk_bytes, sums);
  }
  DZ_LAUNCH(snapshot_final_kernel, grid_for(nchunks, 256), 256, 0, stream, sums, nchunks, chunk_bytes, total);
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
