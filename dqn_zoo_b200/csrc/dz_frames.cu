// Frame-deduplicated replay storage (DESIGN.md §3): every distinct H*W plane of the stored frame stacks lives once in
// a device frame pool; each transition keeps 2*C plane ids.  Insert (content-addressed, one CTA per add), reconstruct
// (plane ids -> HWC stacks for the gather and the fused learner), pool reset and the stacked synthetic fill.
//
// Pool rules (pinned by oracle/frame_pool_oracle.py): the planes of an add resolve in order (s_tm1 channels, then s_t
// channels), each to the live plane with identical bytes if there is one, else to a fresh plane popped from a LIFO
// free stack that initially hands out 1, 2, 3, ...; the new row's references are taken before the evicted row's are
// released, and a plane whose refcount drops to 0 is pushed back.  Plane 0 is the all-zero plane and is never freed.
// Lookups go through an open-addressing table (linear probing, backward-shift deletion) keyed by a 64-bit content hash;
// every hash hit is confirmed by a full byte compare.
#include "dz_internal.cuh"

namespace dz {

constexpr uint64_t kWordKey = 0x9E3779B97F4A7C15ull;

static __device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Content hash of one plane (frame_stride bytes, zero padded), computed by one warp; every lane returns it.
static __device__ uint64_t plane_hash_warp(const uint8_t* plane, int64_t frame_stride) {
  const int lane = threadIdx.x & 31;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(plane);
  uint64_t acc = 0;
  for (int64_t i = lane; i < (frame_stride >> 3); i += 32) acc += mix64(w[i] ^ ((uint64_t)(i + 1) * kWordKey));
  return mix64(warp_sum_u64(acc) ^ (uint64_t)frame_stride);
}

static __device__ __forceinline__ const uint8_t* pool_plane(const dz_replay_view& v, int64_t id) {
  return v.d_frames + id * v.frame_stride;   // 64-bit: id * frame_stride exceeds 2^32 at 1M planes of 84x84
}

// Backward-shift deletion of plane `id` from the table (single thread).
static __device__ void table_erase(const dz_replay_view& v, int32_t id) {
  const int64_t mask = v.table_size - 1;
  int64_t i = (int64_t)(v.d_hashes[id] & (uint64_t)mask);
  while (v.d_table[i] != id) i = (i + 1) & mask;
  int64_t j = i;
  for (;;) {
    j = (j + 1) & mask;
    const int32_t x = v.d_table[j];
    if (x < 0) break;
    const int64_t home = (int64_t)(v.d_hashes[x] & (uint64_t)mask);
    // x may move into the hole at i unless its home lies cyclically in (i, j]
    const bool stays = (i <= j) ? (i < home && home <= j) : (i < home || home <= j);
    if (!stays) {
      v.d_table[i] = x;
      i = j;
    }
  }
  v.d_table[i] = -1;
}

// One add.  Phase 1 de-interleaves the two HWC sources into 2*C zero-padded planes in the staging area; phase 2 hashes
// them (a warp per plane); phase 3 resolves them in order (block-wide compares and copies, bookkeeping by thread 0);
// phase 4 writes the row's plane ids and releases the evicted row's references.
__global__ void __launch_bounds__(512) frame_add_kernel(dz_replay_view v, int64_t slot, int release_row,
                                                        const uint8_t* __restrict__ src_tm1,
                                                        const uint8_t* __restrict__ src_t) {
  dz::pdl_enter();
  const int C = (int)v.obs_channels, P = 2 * C;
  const int64_t fb = v.frame_bytes, fs = v.frame_stride;
  uint8_t* stage = v.d_add_staging + 2 * v.obs_stride;   // [P][fs]
  __shared__ uint64_t s_hash[2 * kMaxObsChannels];
  __shared__ int32_t s_id[2 * kMaxObsChannels];
  __shared__ int32_t s_cand;
  __shared__ int s_fresh;
  for (int64_t i = threadIdx.x; i < 2 * fs; i += blockDim.x) {
    const int o = (int)(i / fs);
    const int64_t px = i - o * fs;
    const uint8_t* src = o ? src_t : src_tm1;
    for (int c = 0; c < C; ++c) stage[(o * C + c) * fs + px] = px < fb ? src[px * C + c] : 0;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int p = warp; p < P; p += nwarps) {
    const uint64_t h = plane_hash_warp(stage + p * fs, fs);
    if ((threadIdx.x & 31) == 0) s_hash[p] = h;
  }
  __syncthreads();
  const int64_t mask = v.table_size - 1;
  const int64_t nvec = fs >> 4;
  for (int p = 0; p < P; ++p) {
    const uint64_t h = s_hash[p];
    const uint4* mine = reinterpret_cast<const uint4*>(stage + p * fs);
    int64_t t = (int64_t)(h & (uint64_t)mask);
    int32_t found = -1;
    for (;;) {
      if (threadIdx.x == 0) s_cand = v.d_table[t];
      __syncthreads();
      const int32_t cand = s_cand;
      __syncthreads();   // s_cand is rewritten by the next probe
      if (cand < 0) break;
      if (v.d_hashes[cand] == h) {
        const uint4* theirs = reinterpret_cast<const uint4*>(pool_plane(v, cand));
        int diff = 0;
        for (int64_t i = threadIdx.x; i < nvec; i += blockDim.x) {
          const uint4 a = mine[i], b = theirs[i];
          diff |= (a.x != b.x) | (a.y != b.y) | (a.z != b.z) | (a.w != b.w);
        }
        if (!__syncthreads_or(diff)) { found = cand; break; }
      }
      t = (t + 1) & mask;
    }
    if (threadIdx.x == 0) {
      s_fresh = 0;
      int32_t id = found;
      if (id < 0) {
        const int64_t top = v.d_pool_counters[0];
        if (top == 0) {   // pool exhausted: a data error the host reports at its next sync point
          if (v.d_flags) atomicOr(v.d_flags, DZ_FLAG_FRAME_POOL_FULL);
          id = 0;
        } else {
          id = v.d_free[top - 1];
          v.d_pool_counters[0] = top - 1;
          v.d_hashes[id] = h;
          v.d_table[t] = id;   // t is the empty slot the probe stopped at
          v.d_refcount[id] = 0;
          s_fresh = 1;
        }
      }
      v.d_refcount[id] += 1;
      s_id[p] = id;
    }
    __syncthreads();
    if (s_fresh) {
      uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(pool_plane(v, s_id[p])));
      for (int64_t i = threadIdx.x; i < nvec; i += blockDim.x) dst[i] = mine[i];
    }
    __syncthreads();   // the next plane may match (and compare against) this one
  }
  if (threadIdx.x == 0) {
    int32_t* row = v.d_planes + slot * P;
    int32_t old[2 * kMaxObsChannels];
    for (int p = 0; p < P; ++p) {
      old[p] = row[p];
      row[p] = s_id[p];
    }
    if (release_row) {
      int64_t top = v.d_pool_counters[0];
      for (int p = 0; p < P; ++p) {
        const int32_t id = old[p];
        if (--v.d_refcount[id] == 0) {
          table_erase(v, id);
          v.d_free[top++] = id;
        }
      }
      v.d_pool_counters[0] = top;
    }
  }
}

// ---- batched add (dz_replay_add_batch) -------------------------------------------------------------------------------
// The K adds of a batch have N = K * P planes, plane q = k * P + p.  Phases:
//   1. frame_batch_planes_kernel (a CTA per observation): de-interleave into the planar workspace, hash each plane; gather
//      the plane ids of the rows the batch overwrites.
//   2. frame_batch_match_kernel (a warp per plane): rep[q] = the first plane of the batch with the same bytes, and for
//      each such representative the plane live at batch start with the same bytes.  The only phase that compares bytes.
//   3. frame_batch_resolve_kernel (one CTA, one thread for the rules): replays the pool rules of the K adds on integers in
//      shared memory, then writes rows, refcounts, the free stack and erases the freed planes from the table.
//   4. frame_batch_insert_kernel (a warp per popped plane): bytes, hash and table entry of every plane that ends the
//      batch holding new content.
// Every plane id the batch touches gets a local slot ("loc") in phase 3: [0, N) the batch-start matches, [N, 2N) the ids
// of the overwritten rows, [2N, 3N) the top N entries of the free stack, 3N plane 0.  id_loc[id] (workspace, indexed by
// plane id, written by phases 1-2 and read in phase 3 only) picks one canonical loc per id: any writer may win.

struct FrameBatchWs {
  uint8_t* planar;    // [N][frame_stride]
  uint64_t* hash;     // [N]
  int32_t* rep;       // [N]
  int32_t* match;     // [N] (representatives only; -1 = no live plane with these bytes)
  int32_t* old;       // [N] plane ids of the overwritten rows at batch start
  int32_t* pop_id;    // [N] planes popped by phase 3, in pop order
  int32_t* pop_cls;   // [N] the representative plane whose bytes each popped plane takes
  int32_t* counts;    // [1] pops
  int32_t* id_loc;    // [frame_capacity]
};

static int64_t align256(int64_t x) { return (x + 255) / 256 * 256; }

static FrameBatchWs frame_batch_ws(const dz_replay_view* v, int64_t max_count, uint8_t* base, int64_t* total) {
  const int64_t N = max_count * 2 * v->obs_channels;
  FrameBatchWs w{};
  int64_t off = 0;
  auto take = [&](int64_t bytes) { uint8_t* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  w.planar = take(N * v->frame_stride);
  w.hash = reinterpret_cast<uint64_t*>(take(N * 8));
  w.rep = reinterpret_cast<int32_t*>(take(N * 4));
  w.match = reinterpret_cast<int32_t*>(take(N * 4));
  w.old = reinterpret_cast<int32_t*>(take(N * 4));
  w.pop_id = reinterpret_cast<int32_t*>(take(N * 4));
  w.pop_cls = reinterpret_cast<int32_t*>(take(N * 4));
  w.counts = reinterpret_cast<int32_t*>(take(4));
  w.id_loc = reinterpret_cast<int32_t*>(take(v->frame_capacity * 4));
  if (total) *total = off;
  return w;
}

static __device__ __forceinline__ bool warp_planes_equal(const uint8_t* a, const uint8_t* b, int64_t frame_stride) {
  const uint4* x = reinterpret_cast<const uint4*>(a);
  const uint4* y = reinterpret_cast<const uint4*>(b);
  int diff = 0;
  for (int64_t i = threadIdx.x & 31; i < (frame_stride >> 4); i += 32) {
    const uint4 u = x[i], w = y[i];
    diff |= (u.x != w.x) | (u.y != w.y) | (u.z != w.z) | (u.w != w.w);
  }
  return !__any_sync(0xffffffffu, diff);
}

__global__ void __launch_bounds__(256) frame_batch_planes_kernel(dz_replay_view v, dz_add_batch b,
                                                                 const uint8_t* __restrict__ src_tm1,
                                                                 const uint8_t* __restrict__ src_t, int64_t pitch,
                                                                 FrameBatchWs w) {
  dz::pdl_enter();
  const int C = (int)v.obs_channels, P = 2 * C;
  const int k = blockIdx.x >> 1, o = blockIdx.x & 1;
  const int64_t N = (int64_t)b.count * P, fb = v.frame_bytes, fs = v.frame_stride;
  const uint8_t* src = (o ? src_t : src_tm1) + k * pitch;
  const int64_t q0 = (int64_t)k * P + o * C;
  uint8_t* dst = w.planar + q0 * fs;
  for (int64_t i = threadIdx.x; i < fs; i += blockDim.x)
    for (int c = 0; c < C; ++c) dst[c * fs + i] = i < fb ? src[i * C + c] : 0;
  __syncthreads();
  for (int c = threadIdx.x >> 5; c < C; c += blockDim.x >> 5) {
    const uint64_t h = plane_hash_warp(dst + c * fs, fs);
    if ((threadIdx.x & 31) == 0) w.hash[q0 + c] = h;
  }
  if (o == 0 && threadIdx.x < P) {
    const int64_t slot = (b.first_slot + k) % v.capacity;
    const int32_t id = v.d_planes[slot * P + threadIdx.x];
    w.old[(int64_t)k * P + threadIdx.x] = id;
    if (b.d_release_row[k] && id > 0) w.id_loc[id] = (int32_t)(N + (int64_t)k * P + threadIdx.x);
  }
  if (blockIdx.x == 0) {
    const int64_t top = v.d_pool_counters[0];
    for (int64_t j = threadIdx.x; j < N && j < top; j += blockDim.x) w.id_loc[v.d_free[top - 1 - j]] = (int32_t)(2 * N + j);
  }
}

__global__ void __launch_bounds__(256) frame_batch_match_kernel(dz_replay_view v, int32_t N, FrameBatchWs w) {
  dz::pdl_enter();
  const int q = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  if (q >= N) return;
  const int lane = threadIdx.x & 31;
  const int64_t fs = v.frame_stride;
  const uint64_t h = w.hash[q];
  const uint8_t* mine = w.planar + (int64_t)q * fs;
  int rep = q;
  for (int base = 0; base < q && rep == q; base += 32) {
    const int c = base + lane;
    unsigned m = __ballot_sync(0xffffffffu, c < q && w.hash[c] == h);
    while (m) {
      const int cand = base + __ffs((int)m) - 1;
      if (warp_planes_equal(w.planar + (int64_t)cand * fs, mine, fs)) { rep = cand; break; }
      m &= m - 1;
    }
  }
  if (lane == 0) w.rep[q] = rep;
  if (rep != q) return;
  const int64_t mask = v.table_size - 1;
  int32_t found = -1;
  for (int64_t t = (int64_t)(h & (uint64_t)mask);; t = (t + 1) & mask) {
    const int32_t cand = v.d_table[t];
    if (cand < 0) break;
    if (v.d_hashes[cand] == h && warp_planes_equal(pool_plane(v, cand), mine, fs)) { found = cand; break; }
  }
  if (lane == 0) {
    w.match[q] = found;
    if (found > 0) w.id_loc[found] = q;
  }
}

__global__ void __launch_bounds__(512) frame_batch_resolve_kernel(dz_replay_view v, dz_add_batch b, FrameBatchWs w) {
  dz::pdl_enter();
  const int C = (int)v.obs_channels, P = 2 * C, K = b.count, N = K * P, L = 3 * N + 1;
  extern __shared__ int32_t sm[];
  int32_t* ref = sm;               // [L] refcount of each loc
  int32_t* cls_of = ref + L;       // [L] representative plane whose bytes the loc holds (-1: none in this batch)
  int32_t* loc2id = cls_of + L;    // [L] plane id of the loc (-1: not a canonical loc)
  int32_t* cls_loc = loc2id + L;   // [N] loc holding the bytes of representative q, -1 = none live
  int32_t* rep = cls_loc + N;      // [N]
  int32_t* loc_old = rep + N;      // [N] loc of the plane the overwritten row held (-1: row not released)
  int32_t* new_loc = loc_old + N;  // [N]
  int32_t* pushed = new_loc + N;   // [N] locs pushed onto the free stack by this batch, bottom first
  int32_t* freed = pushed + N;     // [N]
  int32_t* release = freed + N;    // [K]
  __shared__ int s_pops_init, s_pushed;
  const int64_t top0 = v.d_pool_counters[0];
  auto loc_of = [&](int32_t id) { return id == 0 ? 3 * N : w.id_loc[id]; };
  for (int k = threadIdx.x; k < K; k += blockDim.x) release[k] = b.d_release_row[k];
  __syncthreads();
  for (int e = threadIdx.x; e < L; e += blockDim.x) {
    int32_t id = -1;
    if (e == 3 * N) id = 0;
    else if (e >= 2 * N) id = e - 2 * N < top0 ? v.d_free[top0 - 1 - (e - 2 * N)] : -1;
    else if (e >= N) id = release[(e - N) / P] ? w.old[e - N] : -1;
    else if (w.rep[e] == e) id = w.match[e];
    const bool canonical = id == 0 ? e == 3 * N : (id > 0 && (e >= 2 * N || w.id_loc[id] == e));
    loc2id[e] = canonical ? id : -1;
    ref[e] = canonical && e < 2 * N ? v.d_refcount[id] : (e == 3 * N ? v.d_refcount[0] : 0);
    cls_of[e] = -1;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < N; q += blockDim.x) {
    const int r = w.rep[q];
    rep[q] = r;
    loc_old[q] = release[q / P] ? loc_of(w.old[q]) : -1;
    cls_loc[q] = -1;
    if (r == q && w.match[q] >= 0) {
      const int loc = loc_of(w.match[q]);
      cls_loc[q] = loc;
      if (loc != 3 * N) cls_of[loc] = q;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // the pool rules of frame_add_kernel, add after add: resolve, reference, then release the overwritten row
    int pops_init = 0, npush = 0, nfreed = 0, npop = 0;
    bool full = false;
    for (int k = 0; k < K; ++k) {
      for (int q = k * P; q < (k + 1) * P; ++q) {
        const int c = rep[q];
        int loc = cls_loc[c];
        if (loc < 0) {
          if (npush > 0) loc = pushed[--npush];
          else if (pops_init < top0) loc = 2 * N + pops_init++;
          if (loc < 0) {
            full = true;
            loc = 3 * N;
          } else {
            ref[loc] = 0;
            cls_loc[c] = loc;
            cls_of[loc] = c;
            w.pop_id[npop] = loc2id[loc];
            w.pop_cls[npop] = c;
            ++npop;
          }
        }
        ref[loc] += 1;
        new_loc[q] = loc;
      }
      if (release[k]) {
        for (int q = k * P; q < (k + 1) * P; ++q) {
          const int loc = loc_old[q];
          if (--ref[loc] == 0) {
            pushed[npush++] = loc;
            freed[nfreed++] = loc;
            const int c = cls_of[loc];
            if (c >= 0 && cls_loc[c] == loc) cls_loc[c] = -1;
          }
        }
      }
    }
    // every freed plane was live at batch start, so it is in the table under its old hash
    for (int i = 0; i < nfreed; ++i) table_erase(v, loc2id[freed[i]]);
    if (full && v.d_flags) atomicOr(v.d_flags, DZ_FLAG_FRAME_POOL_FULL);
    w.counts[0] = npop;
    s_pops_init = pops_init;
    s_pushed = npush;
  }
  __syncthreads();
  const int pops_init = s_pops_init, npush = s_pushed;
  for (int e = threadIdx.x; e < L; e += blockDim.x)
    if (loc2id[e] >= 0 && (e < 2 * N || e == 3 * N || e - 2 * N < pops_init)) v.d_refcount[loc2id[e]] = ref[e];
  for (int i = threadIdx.x; i < npush; i += blockDim.x) v.d_free[top0 - pops_init + i] = loc2id[pushed[i]];
  if (threadIdx.x == 0) v.d_pool_counters[0] = top0 - pops_init + npush;
  for (int q = threadIdx.x; q < N; q += blockDim.x) {
    const int64_t slot = (b.first_slot + q / P) % v.capacity;
    v.d_planes[slot * P + q % P] = loc2id[new_loc[q]];
  }
}

__global__ void __launch_bounds__(256) frame_batch_insert_kernel(dz_replay_view v, int32_t N, FrameBatchWs w) {
  dz::pdl_enter();
  const int i = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  if (i >= N || i >= w.counts[0]) return;
  const int32_t id = w.pop_id[i];
  const int c = w.pop_cls[i];
  const uint4* src = reinterpret_cast<const uint4*>(w.planar + (int64_t)c * v.frame_stride);
  uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(pool_plane(v, id)));
  for (int64_t j = threadIdx.x & 31; j < (v.frame_stride >> 4); j += 32) dst[j] = src[j];
  if ((threadIdx.x & 31) == 0) {
    const uint64_t h = w.hash[c];
    v.d_hashes[id] = h;
    const int64_t mask = v.table_size - 1;
    int64_t t = (int64_t)(h & (uint64_t)mask);
    while (atomicCAS(&v.d_table[t], -1, id) != -1) t = (t + 1) & mask;
  }
}

// Plane ids -> HWC stacks.  blockIdx.x = 2 * b + which (s_tm1 / s_t of batch entry b), blockIdx.y splits the row.
// C == 4 with 4-byte planes and a 16-byte aligned destination: each thread reads 4 pixels of each plane (one 32-bit
// word per plane) and writes their 16 interleaved bytes as one uint4 (a 4x4 byte transpose with prmt).
__global__ void __launch_bounds__(256) frame_reconstruct_kernel(dz_replay_view v, const int64_t* __restrict__ slots,
                                                                uint8_t* dst_tm1, uint8_t* dst_t, int64_t pitch) {
  dz::pdl_enter();
  const int b = blockIdx.x >> 1, which = blockIdx.x & 1;
  const int C = (int)v.obs_channels;
  __shared__ const uint8_t* s_src[kMaxObsChannels];
  if (threadIdx.x < C) {
    const int32_t id = v.d_planes[slots[b] * 2 * C + which * C + threadIdx.x];
    s_src[threadIdx.x] = pool_plane(v, id);
  }
  __syncthreads();
  uint8_t* dst = (which ? dst_t : dst_tm1) + (int64_t)b * pitch;
  const int64_t stride = (int64_t)gridDim.y * blockDim.x;
  if (C == 4 && (v.frame_bytes & 3) == 0 && ((uintptr_t)dst & 15) == 0) {
    const uint32_t *p0 = reinterpret_cast<const uint32_t*>(s_src[0]), *p1 = reinterpret_cast<const uint32_t*>(s_src[1]),
                   *p2 = reinterpret_cast<const uint32_t*>(s_src[2]), *p3 = reinterpret_cast<const uint32_t*>(s_src[3]);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (int64_t i = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; i < (v.frame_bytes >> 2); i += stride) {
      const uint32_t x0 = __ldg(p0 + i), x1 = __ldg(p1 + i), x2 = __ldg(p2 + i), x3 = __ldg(p3 + i);
      const uint32_t lo01 = __byte_perm(x0, x1, 0x5140), lo23 = __byte_perm(x2, x3, 0x5140);
      const uint32_t hi01 = __byte_perm(x0, x1, 0x7362), hi23 = __byte_perm(x2, x3, 0x7362);
      d4[i] = make_uint4(__byte_perm(lo01, lo23, 0x5410), __byte_perm(lo01, lo23, 0x7632),
                         __byte_perm(hi01, hi23, 0x5410), __byte_perm(hi01, hi23, 0x7632));
    }
  } else {
    for (int64_t i = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; i < v.obs_bytes; i += stride)
      dst[i] = s_src[i % C][i / C];
  }
}

__global__ void frame_pool_init_kernel(dz_replay_view v) {
  dz::pdl_enter();
  const int64_t P = 2 * v.obs_channels;
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v.table_size; i += step) v.d_table[i] = -1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v.frame_capacity; i += step) {
    v.d_refcount[i] = i == 0 ? 1 : 0;
    v.d_free[i] = (int32_t)(v.frame_capacity - 1 - i);   // free[top - 1] = 1 is popped first
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v.capacity * P; i += step) v.d_planes[i] = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v.frame_stride; i += step) v.d_frames[i] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) v.d_pool_counters[0] = v.frame_capacity - 1;
}

// Plane 0 into the table (one warp, after frame_pool_init_kernel zeroed it).
__global__ void __launch_bounds__(32) frame_pool_zero_plane_kernel(dz_replay_view v) {
  dz::pdl_enter();
  const uint64_t h = plane_hash_warp(v.d_frames, v.frame_stride);
  if (threadIdx.x == 0) {
    v.d_hashes[0] = h;
    v.d_table[h & (uint64_t)(v.table_size - 1)] = 0;
  }
}

// Stacked fill, pool side: planes 1..U hold frames in order of first appearance (frame f of episode e is plane
// 1 + e * (episode_len + 1) + f), zero padded to the stride.
__global__ void __launch_bounds__(256) frame_fill_planes_kernel(dz_replay_view v, int64_t U, uint64_t seed,
                                                                int64_t episode_len) {
  dz::pdl_enter();
  const int64_t wps = v.frame_stride >> 3, words = v.frame_bytes >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < U * wps; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = i / wps, w = i - k * wps;
    const int64_t e = k / (episode_len + 1), f = k - e * (episode_len + 1);
    reinterpret_cast<uint64_t*>(const_cast<uint8_t*>(pool_plane(v, k + 1)))[w] =
        w < words ? stacked_frame_word(seed, e, f, episode_len, words, w) : 0ull;
  }
}

// Hash planes 1..U (a warp each) and insert them into the table.
__global__ void __launch_bounds__(256) frame_fill_hash_kernel(dz_replay_view v, int64_t U) {
  dz::pdl_enter();
  const int64_t mask = v.table_size - 1;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t k = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; k < U; k += nw) {
    const int32_t id = (int32_t)(k + 1);
    const uint64_t h = plane_hash_warp(pool_plane(v, id), v.frame_stride);
    if ((threadIdx.x & 31) == 0) {
      v.d_hashes[id] = h;
      int64_t t = (int64_t)(h & (uint64_t)mask);
      while (atomicCAS(&v.d_table[t], -1, id) != -1) t = (t + 1) & mask;
    }
  }
}

// Plane table and refcounts of rows 0..n-1; the free stack top after popping U planes.
__global__ void __launch_bounds__(256) frame_fill_rows_kernel(dz_replay_view v, int64_t n, int64_t U, int64_t episode_len) {
  dz::pdl_enter();
  const int C = (int)v.obs_channels, P = 2 * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n * P; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / P;
    const int p = (int)(i - row * P), o = p / C, c = p % C;
    const int64_t e = row / episode_len, step = row % episode_len + o;
    const int64_t f = stacked_channel_frame(step, c, C);
    const int32_t id = f < 0 ? 0 : (int32_t)(1 + e * (episode_len + 1) + f);
    v.d_planes[i] = id;
    atomicAdd(&v.d_refcount[id], 1);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) v.d_pool_counters[0] = v.frame_capacity - 1 - U;
}

static int grid_for(int64_t work, int block) {
  const int64_t g = ceil_div(work, block);
  return (int)(g < kNumSMs * 32 ? (g > 0 ? g : 1) : kNumSMs * 32);
}

static int check_pool_view(const dz_replay_view* v) {
  if (!v->d_frames || !v->d_planes || !v->d_refcount || !v->d_hashes || !v->d_table || !v->d_free ||
      !v->d_pool_counters || !v->d_add_staging)
    return fail(DZ_EINVAL, "frame pool view lacks a buffer");
  if (v->obs_channels < 1 || v->obs_channels > kMaxObsChannels) return fail(DZ_EINVAL, "obs_channels must be in [1,32]");
  if (v->frame_bytes * v->obs_channels != v->obs_bytes) return fail(DZ_EINVAL, "obs_bytes != frame_bytes * obs_channels");
  if (v->frame_stride < v->frame_bytes || v->frame_stride % 16) return fail(DZ_EINVAL, "frame_stride must be a multiple of 16");
  if (v->table_size < 2 * v->frame_capacity || (v->table_size & (v->table_size - 1)))
    return fail(DZ_EINVAL, "table_size must be a power of two >= 2 * frame_capacity");
  if (v->frame_capacity < 1 || v->frame_capacity > INT32_MAX) return fail(DZ_EINVAL, "frame_capacity out of range");
  return DZ_OK;
}

int launch_frame_add(const dz_replay_view* view, int64_t slot, int release_row, const uint8_t* src_tm1,
                     const uint8_t* src_t, void* stream) {
  DZ_TRY(check_pool_view(view));
  DZ_LAUNCH(frame_add_kernel, 1, 512, 0, stream, *view, slot, release_row, src_tm1, src_t);
  return DZ_OK;
}

int64_t frame_add_batch_workspace(const dz_replay_view* view, int64_t max_count) {
  int64_t total = 0;
  frame_batch_ws(view, max_count, nullptr, &total);
  return total;
}

static size_t resolve_smem_bytes(int64_t N, int64_t K) { return (size_t)(3 * (3 * N + 1) + 6 * N + K) * 4; }

int launch_frame_add_batch(const dz_replay_view* view, const dz_add_batch* b, const uint8_t* src_tm1,
                           const uint8_t* src_t, int64_t pitch, uint8_t* ws, void* stream) {
  DZ_TRY(check_pool_view(view));
  const int64_t K = b->count, N = K * 2 * view->obs_channels;
  if (N > kMaxBatchPlanes) return fail(DZ_EINVAL, "frame-deduplicated batch has more than kMaxBatchPlanes planes");
  static bool smem_set = false;
  if (!smem_set) {
    DZ_CUDA_OK(cudaFuncSetAttribute(frame_batch_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)resolve_smem_bytes(kMaxBatchPlanes, kMaxAddBatch)));
    smem_set = true;
  }
  const FrameBatchWs w = frame_batch_ws(view, K, ws, nullptr);
  const int warp_grid = (int)ceil_div(N * 32, 256);
  DZ_LAUNCH(frame_batch_planes_kernel, (int)(2 * K), 256, 0, stream, *view, *b, src_tm1, src_t, pitch, w);
  DZ_LAUNCH(frame_batch_match_kernel, warp_grid, 256, 0, stream, *view, (int32_t)N, w);
  DZ_LAUNCH(frame_batch_resolve_kernel, 1, 512, resolve_smem_bytes(N, K), stream, *view, *b, w);
  DZ_LAUNCH(frame_batch_insert_kernel, warp_grid, 256, 0, stream, *view, (int32_t)N, w);
  return DZ_OK;
}

int launch_frame_reconstruct(const dz_replay_view* view, const int64_t* d_slots, int batch, uint8_t* dst_tm1,
                             uint8_t* dst_t, int64_t pitch, void* stream) {
  DZ_TRY(check_pool_view(view));
  if (batch <= 0) return DZ_OK;
  const int64_t work = view->obs_channels == 4 ? view->frame_bytes >> 2 : view->obs_bytes;
  const int gy = (int)(ceil_div(work, 256) < 8 ? ceil_div(work, 256) : 8);
  DZ_LAUNCH(frame_reconstruct_kernel, dim3((unsigned)batch * 2u, (unsigned)gy), 256, 0, stream, *view, d_slots, dst_tm1,
            dst_t, pitch);
  return DZ_OK;
}

int launch_frame_pool_reset(const dz_replay_view* view, void* stream) {
  DZ_TRY(check_pool_view(view));
  const int64_t work = view->table_size > view->capacity * 2 * view->obs_channels ? view->table_size
                                                                                    : view->capacity * 2 * view->obs_channels;
  DZ_LAUNCH(frame_pool_init_kernel, grid_for(work, 256), 256, 0, stream, *view);
  DZ_LAUNCH(frame_pool_zero_plane_kernel, 1, 32, 0, stream, *view);
  return DZ_OK;
}

int launch_frame_fill_stacked(const dz_replay_view* view, int64_t n, uint64_t seed, int64_t episode_len, void* stream) {
  DZ_TRY(check_pool_view(view));
  if (view->frame_bytes % 8) return fail(DZ_EINVAL, "stacked fill needs H*W a multiple of 8");
  const int64_t episodes = ceil_div(n, episode_len);
  const int64_t U = n + episodes;   // distinct frames of n transitions of complete stacks
  if (U > view->frame_capacity - 1) return fail(DZ_EINVAL, "frame_capacity too small for the stacked fill");
  DZ_LAUNCH(frame_fill_planes_kernel, grid_for(U * (view->frame_stride >> 3), 256), 256, 0, stream, *view, U, seed,
            episode_len);
  DZ_LAUNCH(frame_fill_hash_kernel, grid_for(U * 32, 256), 256, 0, stream, *view, U);
  DZ_LAUNCH(frame_fill_rows_kernel, grid_for(n * 2 * view->obs_channels, 256), 256, 0, stream, *view, n, U, episode_len);
  return DZ_OK;
}

}  // namespace dz
