/*
 * dqn_zoo_b200 — C ABI of the H100-native replay-sampler + learner-update hot path.
 *
 * The reference (google-deepmind/dqn_zoo) has no FFI layer: its extension point is the
 * duck-typed Python surface `parts.Agent` / `replay.*` (SURVEY.md §8(b)).  This header is
 * the boundary a maintainer would bind from Python (ctypes stub in INTEGRATION.md); each
 * entry point cites the reference code it replaces.  All citations are relative to the
 * reference repository root.
 *
 * Conventions
 *   - every function returns 0 on success, a negative DZ_E* code otherwise;
 *     dz_last_error() returns a thread-local message for the last failure.
 *   - all pointers named d_* are DEVICE pointers (the caller owns the memory — in the
 *     Python host they are torch.Tensor.data_ptr()); h_* are host pointers.
 *   - `stream` is a cudaStream_t passed as void*.  Nothing synchronises the device
 *     unless the comment says so.  Handles are not thread-safe; distinct handles on
 *     distinct streams may run concurrently.
 *   - no torch / C++ types cross this boundary.
 */
#ifndef DQN_ZOO_B200_H_
#define DQN_ZOO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DZ_OK 0
#define DZ_EINVAL (-1)   /* bad argument (ValueError in the Python shim) */
#define DZ_ECUDA (-2)    /* CUDA runtime error */
#define DZ_ERANGE (-3)   /* index / target out of range (IndexError / ValueError) */
#define DZ_ESTATE (-4)   /* device-side sticky error flag was raised by a previous kernel */

const char* dz_last_error(void);
/* "dqn_zoo_b200 <version> sm_90a <build date>"; also proves the library loaded. */
const char* dz_build_info(void);
/* Number of kernels this library has launched in this process (bench.py `gpu_launches`). */
int64_t dz_launch_count(void);
/* Measurement aid (bench.py roofline): between begin and end every kernel launch is bracketed by
 * CUDA events on its own stream; end synchronises the device and writes a JSON object
 * {"<kernel or layer tag>": [launches, total_ms], ...} into `out`.  Never active in a timed run. */
int dz_profile_begin(void);
int dz_profile_end(char* out, int64_t cap);

/* ------------------------------------------------------------------------------------------
 * R1  Sum tree  (replaces replay.py:246-426, class SumTree)
 *
 * d_nodes is float64[2*first_leaf]; node i has children 2i, 2i+1; root = node 1; leaves at
 * [first_leaf, 2*first_leaf).  Internal nodes are always recomputed as fl(left+right)
 * (replay.py:284-290, :394-404), so every function below leaves the tree bit-identical to
 * the reference's after the same call.
 * ---------------------------------------------------------------------------------------- */

/* replay.py:394-404 (_set_values): leaves [n_valid, first_leaf) are zeroed, every internal
 * node resummed bottom-up, node 0 cleared. */
int dz_sumtree_rebuild(double* d_nodes, int64_t first_leaf, int64_t n_valid, void* stream);

/* replay.py:278-290 (set): d_nodes[first_leaf+idx[i]] = values[i] for i in order (duplicates:
 * last write wins), then the root paths are resummed.  Values must be finite and >= 0 and
 * indices in [0,size): violations raise the sticky flag bit DZ_FLAG_BAD_VALUE / _BAD_INDEX
 * in *d_flags (checked by the caller when it next synchronises) and the call is a no-op for
 * that element. */
int dz_sumtree_set(double* d_nodes, int64_t first_leaf, int64_t size, const int64_t* d_idx,
                   const double* d_values, int64_t n, int32_t* d_flags, void* stream);

/* replay.py:299-313,406-426 (query/_query_single): smallest leaf index whose inclusive prefix
 * sum exceeds the target; requires 0 <= target < root else DZ_FLAG_BAD_TARGET. */
int dz_sumtree_query(const double* d_nodes, int64_t first_leaf, const double* d_targets, int64_t n,
                     int64_t* d_out_idx, int32_t* d_flags, void* stream);

/* replay.py:271-276 (get). */
int dz_sumtree_get(const double* d_nodes, int64_t first_leaf, int64_t size, const int64_t* d_idx,
                   int64_t n, double* d_out, int32_t* d_flags, void* stream);

#define DZ_FLAG_BAD_VALUE 1
#define DZ_FLAG_BAD_INDEX 2
#define DZ_FLAG_BAD_TARGET 4
#define DZ_FLAG_ROOT_ZERO 8   /* fused PER step met root == 0 (reference would skip an RNG draw) */
#define DZ_FLAG_NONFINITE_WEIGHT 16
#define DZ_FLAG_FRAME_POOL_FULL 32  /* an add found no free plane (frame_capacity too small); the plane was mapped to 0 */

/* ------------------------------------------------------------------------------------------
 * R5/R6  Replay storage in HBM (replaces the OrderedDict storage of replay.py:120-200 and
 * :654-768; transition-major layout, see DESIGN.md §3)
 * ---------------------------------------------------------------------------------------- */

typedef struct dz_replay_view {
  uint8_t* d_obs;        /* [capacity][2][obs_stride]: s_tm1 then s_t of each transition      */
  int32_t* d_action;     /* [capacity]  a_tm1                                                 */
  double* d_reward;      /* [capacity]  r_t   (float64: n-step returns are built in f64,
                                               replay.py:808-814; rounded to f32 at the learner) */
  double* d_discount;    /* [capacity]  discount_t                                            */
  int64_t capacity;
  int64_t obs_bytes;     /* bytes per observation (84*84*4 = 28224)                           */
  int64_t obs_stride;    /* obs_bytes rounded up to 16                                        */
  /* prioritized replay only (NULL / 0 for uniform) */
  double* d_tree;        /* float64[2*first_leaf]                                             */
  int64_t first_leaf;
  int64_t* d_live;       /* `_active_indices` (replay.py:459): dense list of tree indices     */
  int64_t* d_id_at;      /* `_index_to_id`   (replay.py:455): tree index -> id                */
  /* uniform replay only */
  int64_t* d_ids;        /* `UniformDistribution._ids` (replay.py:49): dense list of ids      */
  int32_t* d_flags;      /* sticky error flags (1 int32)                                      */
  /* frame-deduplicated layout only (d_planes == NULL: transition-major, d_obs holds the rows; DESIGN.md §3).
   * An observation [H][W][C] uint8 is C planes of H*W bytes; each distinct plane is stored once in d_frames and
   * row `slot` keeps 2*C plane ids (s_tm1 channels 0..C-1, then s_t channels 0..C-1).  Plane 0 is the reserved
   * all-zero plane: always live, never freed, its refcount carries one permanent reference. */
  uint8_t* d_frames;     /* [frame_capacity][frame_stride] planar frame pool; offsets are 64-bit */
  int64_t frame_bytes;   /* H*W                                                                */
  int64_t frame_stride;  /* frame_bytes rounded up to 16 (the padding is zero)                 */
  int64_t obs_channels;  /* C (<= 32); also read by dz_replay_fill_synthetic_stacked in either layout */
  int64_t frame_capacity;
  int32_t* d_planes;     /* [capacity][2*C] plane ids                                          */
  int32_t* d_refcount;   /* [frame_capacity] references from live rows (+1 for plane 0)        */
  uint64_t* d_hashes;    /* [frame_capacity] 64-bit content hash of each live plane            */
  int32_t* d_table;      /* [table_size] open-addressing table of live plane ids (-1 = empty)  */
  int64_t table_size;    /* power of two >= 2 * frame_capacity                                  */
  int32_t* d_free;       /* [frame_capacity] LIFO free stack (top = d_pool_counters[0])        */
  int64_t* d_pool_counters; /* [1]: free-stack top; live planes = frame_capacity - top         */
  uint8_t* d_add_staging;   /* [2][obs_stride] host-source copy + [2*C][frame_stride] planar    */
} dz_replay_view;

/* One `add` (replay.py:142-151 / :690-699) after the HOST has done the O(1) integer
 * bookkeeping: copies the two observations from host memory into row `slot`, writes the
 * scalars, applies up to 4 (position,value) patches to the dense id/index lists and, for
 * prioritized replay, sets leaf `tree_index` to `leaf_value` (= priority**alpha, evaluated on
 * the host in float64 as replay.py:507 does) and resums its root path.  `evict_index` >= 0
 * zeroes that leaf first (replay.py:533-534). */
typedef struct dz_add_record {
  int64_t slot;
  int32_t action;
  double reward, discount;
  int32_t n_patches;
  int64_t patch_pos[4];
  int64_t patch_val[4];
  int32_t patch_target[4];   /* 0 = d_live, 1 = d_id_at, 2 = d_ids */
  int64_t tree_index;        /* -1 for uniform replay */
  double leaf_value;
  int64_t evict_index;       /* -1 if nothing evicted */
  int64_t size_after;        /* sum-tree `size` for range checks */
  const float* d_priority;   /* optional: take the priority from this DEVICE float32 (the learner's
                                max_seen_priority, rainbow/agent.py:148-149) instead of leaf_value;
                                leaf = ((double)*d_priority) ** alpha in float64, exact for alpha 0.5 / 1 */
  double alpha;
  int32_t release_row;       /* frame-deduplicated layout: 1 = row `slot` holds a live transition whose plane
                                references are released AFTER the new row's planes are resolved and referenced */
} dz_add_record;

/* s_tm1 / s_t sources may be HOST arrays or DEVICE buffers (cudaMemcpyDefault; NULL = leave the row's bytes).
 * Frame-deduplicated layout (view->d_planes != NULL): both sources are required; host sources are first copied into
 * d_add_staging, device sources are read in place.  One CTA hashes the 2*C planes, resolves each (in order, each
 * seeing the ones before it) to the live plane with identical bytes (hash hit + full byte compare) or to a fresh plane
 * popped from the free stack, then releases the evicted row (refcount 0 -> back on the free stack).  An empty free
 * stack sets DZ_FLAG_FRAME_POOL_FULL and maps the plane to plane 0. */
int dz_replay_add(const dz_replay_view* view, const dz_add_record* rec, const uint8_t* h_s_tm1,
                  const uint8_t* h_s_t, void* stream);

/* K = `count` adds in one call, leaving the replay exactly as K dz_replay_add calls in order k = 0..K-1 would: the
 * same rows, scalars, list patches, sum tree (a pure function of its leaves) and, in the frame-deduplicated layout,
 * the same plane ids, refcounts, free stack (order included), plane bytes and hashes of every live plane, and the same
 * sticky DZ_FLAG_FRAME_POOL_FULL.  The plane table then holds exactly the live planes; its slot layout may differ.
 * Transition k goes to row (first_slot + k) % capacity, so K <= capacity rows are distinct.  The [K] arrays are DEVICE
 * arrays (the Python host fills them with one H2D copy of a pinned block per call). */
typedef struct dz_add_batch {
  int32_t count;
  int64_t first_slot;
  const int32_t* d_action;          /* [K] */
  const double* d_reward;           /* [K] */
  const double* d_discount;         /* [K] */
  const int32_t* d_release_row;     /* [K] as dz_add_record.release_row */
  const int64_t* d_tree_index;      /* [K] prioritized replay; NULL for uniform */
  const int64_t* d_evict_index;     /* [K] -1 = nothing evicted */
  const double* d_leaf_value;       /* [K] priority**alpha in float64 (host), unless d_priority */
  const float* d_priority;          /* optional, shared by the K adds: as dz_add_record.d_priority */
  double alpha;
  int32_t n_patches;                /* list patches of all K adds, applied in order (positions can repeat) */
  const int64_t* d_patch_pos;       /* [n_patches] */
  const int64_t* d_patch_val;       /* [n_patches] */
  const int32_t* d_patch_target;    /* [n_patches] 0 = d_live, 1 = d_id_at, 2 = d_ids */
  const uint8_t* s_tm1;             /* observation k at s_tm1 + k * src_pitch; host or device memory */
  const uint8_t* s_t;
  int64_t src_pitch;
} dz_add_batch;

/* Bytes of the workspace dz_replay_add_batch needs for up to *max_count adds per call.  *max_count is lowered to the
 * most one call takes for this view (the sum-tree update and, in the frame-deduplicated layout, the plane resolution
 * keep their state on chip). */
int dz_replay_add_batch_workspace(const dz_replay_view* view, int32_t* max_count, int64_t* bytes);

/* Host observations are copied H2D once per call, for the whole batch, into the workspace; device observations are
 * read in place.  Argument errors (count above the workspace's or the capacity, first_slot out of range) return
 * DZ_EINVAL / DZ_ERANGE before anything is enqueued.  Frame-deduplicated layout: the planes of the batch are hashed
 * and matched (against the planes live at batch start and against earlier planes of the batch, every hash hit
 * confirmed by a byte compare) in parallel; one thread then replays the pool rules of K sequential adds on integers
 * only; the bytes of the planes that end the batch holding new content are copied in parallel. */
int dz_replay_add_batch(const dz_replay_view* view, const dz_add_batch* batch, void* d_workspace,
                        int64_t workspace_bytes, void* stream);

/* Frame-deduplicated layout: empties the pool (every row's plane ids = 0, free stack hands out 1, 2, 3, ... next,
 * plane 0 zeroed, live and in the table). */
int dz_replay_frame_pool_reset(const dz_replay_view* view, void* stream);
/* Frame-deduplicated layout: live planes (plane 0 included) into *h_frames_in_use.  Synchronises `stream`. */
int dz_replay_frames_in_use(const dz_replay_view* view, int64_t* h_frames_in_use, void* stream);

/* Bulk pre-fill of rows [0, n) of an EMPTY replay with frame stacks, either layout: frame f of episode e is
 * mix64(seed*0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019 + (e*(episode_len+1) + f)*(H*W/8) + w) per 8-byte word w
 * (H*W % 8 == 0).  Transition i is step t = i % episode_len of episode e = i / episode_len; its s_tm1 is the stack
 * after frames 0..t (trailing-zero padded while t + 1 < C: A000, AB00, ...; processors.py:497-504), s_t the stack after
 * frames 0..t+1.  Scalars as dz_replay_fill_synthetic.  Byte-identical to oracle/frame_pool_oracle.py:synthetic_stacked_rows;
 * in the deduplicated layout the plane table, refcounts, hash table and free stack are those n sequential adds leave. */
int dz_replay_fill_synthetic_stacked(const dz_replay_view* view, int64_t n, uint64_t seed, int64_t episode_len,
                                     int32_t num_actions, double discount, void* stream);

/* ------------------------------------------------------------------------------------------
 * Checkpoint transfers (DESIGN.md §9; dz_checkpoint.cu).  A checkpoint streams device arrays
 * through a fixed staging ring in chunks; every chunk is digested on the device before its D2H
 * copy on save and after its H2D copy on load.
 * ---------------------------------------------------------------------------------------- */

/* 64-bit digest of `bytes` bytes at d_src (8-byte aligned): 8-byte little-endian words w_i (the last
 * zero padded), digest = mix64(S ^ bytes), S = sum_i mix64(w_i ^ ((i+1) * 0x9E3779B97F4A7C15)) mod 2^64,
 * mix64 the splitmix64 finaliser.  Wrapping adds make S independent of the reduction order.  Writes
 * the digest to the DEVICE uint64 *d_out. */
int dz_ckpt_digest(const void* d_src, int64_t bytes, uint64_t* d_out, void* stream);
/* The same digest of a HOST range, computed on the CPU. */
int dz_ckpt_digest_host(const void* h_src, int64_t bytes, uint64_t* h_out);

/* Frame-deduplicated layout.  Live planes (refcount > 0, plane 0 excluded) in increasing id order into
 * d_ids[0..*d_count) with their hashes into d_hashes (both sized frame_capacity); *d_count is a DEVICE int64. */
int dz_ckpt_pool_live(const dz_replay_view* view, int32_t* d_ids, uint64_t* d_hashes, int64_t* d_count, void* stream);
/* Either layout: records d_ids[0..n) packed into d_dst in file order, and the digest of each chunk of
 * chunk_bytes (a positive multiple of the record size) of the packed bytes into the DEVICE uint64
 * d_digests[0..ceil(n * record / chunk_bytes)), each equal to dz_ckpt_digest of that chunk, in one read of
 * the replay.  Frame-deduplicated view: record q is plane d_ids[q] (frame_bytes, no stride padding).
 * Transition-major view: record q is row slot d_ids[q], s_tm1 then s_t (2 * obs_bytes).  The ids must name
 * planes / rows of the view; offsets are 64-bit.  16-byte loads and stores when frame_bytes / obs_bytes is a
 * multiple of 16 and d_dst is 16-byte aligned.  n = 0 enqueues nothing. */
int dz_ckpt_snapshot(const dz_replay_view* view, const int32_t* d_ids, int64_t n, uint8_t* d_dst, int64_t chunk_bytes,
                     uint64_t* d_digests, void* stream);
/* Packed planes d_src -> planes d_ids[0..n), stride padding zeroed.  An id outside [1, frame_capacity) sets
 * DZ_CKPT_BAD_PLANE_ID in d_bad[0] and is skipped. */
int dz_ckpt_pool_scatter(const dz_replay_view* view, const int32_t* d_ids, int64_t n, const uint8_t* d_src,
                         int32_t* d_bad, void* stream);
/* After dz_replay_frame_pool_reset, the plane-id table, the planes' bytes and the free stack [0, top): adds one
 * reference per plane id of the live rows d_live_slots[0..n_live); recomputes the hash of each listed plane
 * d_ids[0..n_ids) (strictly increasing), compares it with d_saved_hashes and inserts the plane into the table.
 * d_bad is a zeroed DEVICE int32[4]: d_bad[0] collects DZ_CKPT_* bits, d_bad[2..3] the uint64 count of planes with
 * refcount > 0 (plane 0 included), which the caller checks against n_ids + 1. */
int dz_ckpt_pool_rebuild(const dz_replay_view* view, const int64_t* d_live_slots, int64_t n_live, const int32_t* d_ids,
                         const uint64_t* d_saved_hashes, int64_t n_ids, int64_t top, int32_t* d_bad, void* stream);
#define DZ_CKPT_BAD_PLANE_ID 1        /* a row or the live list names a plane outside the pool, or the list is unsorted */
#define DZ_CKPT_UNREFERENCED_PLANE 2  /* a listed plane has no reference from a live row */
#define DZ_CKPT_HASH_MISMATCH 4       /* a listed plane's bytes do not hash to the saved hash */
#define DZ_CKPT_BAD_FREE_STACK 8      /* a free-stack entry is out of range or names a referenced plane */

/* Transition-major layout: rows [first_slot, first_slot + n) <-> d_buf packed at obs_bytes per observation
 * (s_tm1 then s_t of each row), one pitched device-to-device copy.  to_replay = 0: replay -> d_buf. */
int dz_ckpt_rows(const dz_replay_view* view, int64_t first_slot, int64_t n, uint8_t* d_buf, int32_t to_replay,
                 void* stream);

/* Bulk pre-fill for benchmarks/tests: rows [row0,row0+n) get deterministic pseudo-random
 * contents (splitmix64 counter hash; byte-identical to oracle/replay_oracle.py:synthetic_rows):
 * uint8 observations iid uniform, action uniform, reward in {-1,0,1} w.p. .05/.9/.05, discount_t =
 * `discount` w.p. .99 else 0 (SURVEY §8(d)). */
int dz_replay_fill_synthetic(const dz_replay_view* view, int64_t row0, int64_t n, uint64_t seed,
                             int32_t num_actions, double discount, void* stream);

/* Per-step sampling inputs that live in device memory so that a captured CUDA graph can be
 * replayed: the three host RandomState draws of replay.py:551-567 plus the scalars that
 * change as items are added. */
typedef struct dz_sample_inputs {
  const int64_t* d_rand_pos;   /* [B] randint(size, size=B)            (replay.py:551-554 / :78) */
  const double* d_u_tree;      /* [B] uniform(size=B), scaled by root   (replay.py:559)          */
  const double* d_u_mix;       /* [B] uniform(size=B) < usp             (replay.py:563-567)      */
  const double* d_scalars;     /* [4]: size, beta (IS exponent), usp, normalize(0/1)            */
} dz_sample_inputs;

typedef struct dz_sample_outputs {
  int64_t* d_ids;        /* [B] sampled ids                        (replay.py:578-582)     */
  int64_t* d_indices;    /* [B] tree indices (PER) / list positions (uniform)              */
  int64_t* d_slots;      /* [B] storage rows                                               */
  double* d_probs;       /* [B] sampling probabilities (PER)       (replay.py:569-577)     */
  double* d_weights;     /* [B] importance weights, float64 (PER)  (replay.py:211-243)     */
} dz_sample_outputs;

/* replay.py:547-583 + :706-717 (PER) or :76-82 (uniform): indices, ids, probabilities and
 * importance-sampling weights for one batch.  Warp-cooperative sum-tree descent. */
int dz_replay_sample(const dz_replay_view* view, int32_t prioritized, const dz_sample_inputs* in,
                     const dz_sample_outputs* out, int32_t batch, void* stream);

/* replay.py:718-722 (`get` + np.stack): gather rows d_slots[0..B) into dense batch arrays
 * (uint8 [B][obs_bytes] x2, int64 a, float64 r, float64 discount — the dtypes np.stack
 * yields, SURVEY §8(a) R5). */
int dz_replay_gather(const dz_replay_view* view, const int64_t* d_slots, int32_t batch, uint8_t* d_s_tm1,
                     uint8_t* d_s_t, int64_t* d_a, double* d_r, double* d_disc, void* stream);

/* replay.py:725-730 -> :536-545 -> :203-208 (`update_priorities`, `_power` in FLOAT32 as the
 * priorities arrive as a float32 array, SURVEY §8(a) R3) -> SumTree.set.  d_indices are tree
 * indices (as returned in dz_sample_outputs.d_indices).  alpha == 0.5 uses sqrt.rn.f32. */
int dz_replay_update_priorities(const dz_replay_view* view, const int64_t* d_indices, const float* d_priorities,
                                int32_t n, double alpha, int64_t size, void* stream);

/* ------------------------------------------------------------------------------------------
 * Learner (replaces the jitted `update` closure and `_learn` glue of every agent:
 * dqn/agent.py:85-119,179-189; double_q/agent.py:85-123; prioritized/agent.py:86-129,187-206;
 * c51/agent.py:87-120; qrdqn/agent.py:88-122; rainbow/agent.py:85-123,181-198;
 * iqn/agent.py:178-226; networks: networks.py:58-363)
 * ---------------------------------------------------------------------------------------- */

/* DZ_MUNCHAUSEN: Munchausen DQN (Vieillard, Pietquin & Geist, NeurIPS 2020), outside the reference tree: dqn's
 * network, parameter layout and acting, with the soft, log-policy-augmented target of DESIGN.md §13.
 * DZ_MUNCHAUSEN_IQN: Munchausen-IQN from the same paper: iqn's network, parameter layout, taus and acting, with the
 * soft target over quantile samples of DESIGN.md §14.
 * DZ_FQF: the Fully parameterized Quantile Function (Yang et al., NeurIPS 2019): iqn's network, whose taus a fraction
 * proposal layer computes from the torso features inside the step instead of drawing them (DESIGN.md §15).  Its
 * parameter layout is iqn's followed by "fraction/w" [feat][N] and "fraction/b" [N]; it takes no taus anywhere. */
enum dz_agent_kind { DZ_DQN = 0, DZ_DOUBLE_Q = 1, DZ_PRIORITIZED = 2, DZ_C51 = 3, DZ_QRDQN = 4, DZ_RAINBOW = 5, DZ_IQN = 6,
                     DZ_MUNCHAUSEN = 7, DZ_MUNCHAUSEN_IQN = 8, DZ_FQF = 9 };
enum dz_optimizer_kind { DZ_ADAM = 0, DZ_RMSPROP_CENTERED = 1 };

typedef struct dz_learner_config {
  int32_t kind;              /* dz_agent_kind */
  int32_t num_actions;
  int32_t num_atoms;         /* c51 / rainbow: 51 */
  int32_t num_quantiles;     /* qrdqn: 201 */
  int32_t latent_dim;        /* iqn / munchausen_iqn / fqf: 64 */
  int32_t tau_samples_s_tm1, tau_samples_policy, tau_samples_s_t; /* iqn / munchausen_iqn: N, K, N' (fqf ignores them) */
  int32_t batch;             /* 32 */
  int32_t obs_h, obs_w, obs_c; /* 84,84,4 */
  /* loss hyperparameters, validated for every kind: finite, vmax > 0, grad_error_bound >= 0, huber_param >= 0 */
  float vmax;                /* c51 / rainbow support is linspace(-vmax, vmax, atoms) */
  float grad_error_bound;    /* dqn family: 1/32 (dqn/run_atari.py:79) */
  float huber_param;         /* qrdqn / iqn: 1.0 */
  int32_t optimizer;         /* dz_optimizer_kind */
  float learning_rate, opt_eps, rms_decay, adam_b1, adam_b2;
  float max_global_grad_norm; /* 0 = off (optax.clip_by_global_norm) */
  /* munchausen and munchausen_iqn only (other kinds ignore them, so a zero-filled tail is valid there);
   * dz_learner_create and dz_learner_plan_query return DZ_EINVAL unless all three are finite, tau > 0, alpha >= 0
   * and l0 <= 0 */
  float munchausen_alpha;    /* scale of the log-policy bonus: 0.9 */
  float entropy_temperature; /* tau of the softmax policy of the target network: 0.03 */
  float log_policy_clip;     /* l0, the lower clip of tau * log pi: -1 */
  /* fqf only (other kinds ignore them, so a zero-filled tail is valid there); DZ_EINVAL unless num_fractions is in
   * [2, 128], the learning rate finite and >= 0, eps finite and > 0 and the decay in [0, 1).  The fraction layer is
   * updated by centred RMSProp with these values; the optimizer fields above cover every other tensor, and the clip
   * (when set) and the reported grad norm cover those same tensors. */
  int32_t num_fractions;         /* N: 32 */
  float fraction_learning_rate;  /* 2.5e-9 */
  float fraction_opt_eps;        /* 1e-5 */
  float fraction_rms_decay;      /* 0.95 */
  /* 1: the dueling network (Wang et al., ICML 2016; DESIGN.md §16) in place of the fc1 / head layers, valid for dqn,
   * double_q, prioritized and munchausen (DZ_EINVAL for any other kind; rainbow's network is dueling already).  0, as a
   * zero-filled tail leaves it: the plain network.  The parameter layout after the conv tensors is "adv1/w" [feat][512],
   * "adv1/b" [512], "adv2/w" [512][A], "adv2/b" [A], "val1/w" [feat][512], "val1/b" [512], "val2/w" [512][1],
   * "val2/b" [1], and the head outputs q_a = v + (adv_a - mean_a adv) in every place the plain network's are read. */
  int32_t dueling;
  /* 1: noisy networks (Fortunato et al., ICLR 2018; DESIGN.md §17): every layer after the torso is a factorised-noise
   * layer y = x mu_w + mu_b + ((x * f(eps_in)) sigma_w + sigma_b) * f(eps_out), plain or (with dueling = 1) dueling.
   * Valid for dqn, double_q, prioritized and munchausen (DZ_EINVAL for any other kind; rainbow's network is noisy
   * already).  0, as a zero-filled tail leaves it: no noise.  Each layer L of the network ("fc1", "head"; dueling:
   * "adv1", "adv2", "val1", "val2") holds "L/mu/w", "L/mu/b", "L/sigma/w", "L/sigma/b" in that order after the conv
   * tensors.  The learner then takes noise exactly as rainbow does: noise_floats = 3 applies, dz_learner_noise_stride,
   * per-stream acting noise and the actor's draws. */
  int32_t noisy;
  /* Random-shift image augmentation of the learner step (DrQ, Kostrikov, Yarats & Fergus, ICLR 2021; DESIGN.md §18),
   * valid for every kind and network option.  p in [0, 16] and p < min(obs_h, obs_w) (DZ_EINVAL otherwise); 0, as a
   * zero-filled tail leaves it: off, and the step is what it is without the field.  p > 0: each update reads s_tm1
   * and s_t of example b shifted by (dy0, dx0) and (dy1, dx1) = d_shifts[b][0..3], each in [0, 2p]:
   * out[y][x][c] = in[clamp(y + dy - p, 0, H - 1)][clamp(x + dx - p, 0, W - 1)][c], the observation edge-padded by
   * p and cropped back to H x W.  Every pass over s_tm1 reads the one shifted s_tm1 and every pass over s_t the one
   * shifted s_t; acting never sees a shift. */
  int32_t random_shift_pad;
  /* Prioritized experience replay (Schaul et al., ICLR 2016; DESIGN.md §19) for any kind and network option: 0 or 1
   * (DZ_EINVAL otherwise).  1: every update writes dz_update_outputs.d_priorities and, in dz_learner_learn, updates
   * d_max_seen_priority as max(old, batch max).  0, as a zero-filled tail leaves it: a learner of any kind but
   * prioritized and rainbow writes no priorities, and dz_learner_learn(prioritized = 1) on it returns DZ_EINVAL.
   * DZ_PRIORITIZED and DZ_RAINBOW write them whatever the field says.  The priority of example b, from its UNWEIGHTED
   * loss:
   *   dqn, double_q, prioritized   |td|
   *   munchausen                   |td| against its soft target (not the per-example 0.5 td^2)
   *   c51, rainbow                 clip(|cross entropy|, 0, 100)
   *   qrdqn, iqn, munchausen_iqn,  clip(|quantile Huber loss|, 0, 100), the per-example value (fqf: the quantile
   *   fqf                          loss at the proposed fractions, not the fraction loss)
   * The importance weights d_weights scale each example's loss term and its gradient (fqf: the fraction loss's too)
   * whatever the field says. */
  int32_t prioritized;
  /* Conservative Q-learning, CQL(H) (Kumar, Zhou, Tucker & Levine, NeurIPS 2020; DESIGN.md §20), for every kind and
   * network option: alpha finite and >= 0 (DZ_EINVAL otherwise); 0, as a zero-filled tail leaves it: off, and the step
   * is what it is without the field.  alpha > 0 adds alpha R_b to each example's loss before its importance weight,
   * R_b = logsumexp_a Q_a(s_tm1) - Q_{a_tm1}(s_tm1) >= 0, with Q_a the online network's expected value on s_tm1:
   *   dqn, double_q, prioritized, munchausen   the head output q_a (after the dueling aggregation)
   *   c51, rainbow                             sum_k softmax(logits_a)_k z_k (rainbow: the dueling-aggregated logits)
   *   qrdqn, iqn, munchausen_iqn               the mean of the pass-0 quantiles (iqn: over the N s_tm1 tau samples)
   *   fqf                                      sum_i w_i Z(s_tm1, tau_hat_i, a), the proposal's w_i held constant
   * The gradient of the added term is not clipped by grad_error_bound.  The per-example values, the priorities and
   * fqf's fraction loss are the kind's own, unchanged. */
  float cql_alpha;
} dz_learner_config;

typedef struct dz_learner_plan {
  int64_t param_count;       /* floats in one parameter blob */
  int32_t num_tensors;
  int64_t opt_state_floats;  /* 2*param_count (adam: mu,nu; rmsprop: mu,nu) */
  int64_t workspace_bytes;
  int64_t noise_floats;      /* rainbow and noisy networks: floats of factorised noise for ONE update (3 applies) */
  int64_t tau_floats;        /* iqn / munchausen_iqn: batch*(N+K+N'); fqf: 0 (its taus live in the workspace) */
} dz_learner_plan;

int dz_learner_plan_query(const dz_learner_config* cfg, dz_learner_plan* out);
/* Tensor i of the parameter blob: canonical name ("conv1/w", "adv1/sigma/b", ...), shape
 * (conv w = HWIO, linear w = (in,out); networks_test.py:44,53) and float offset. */
int dz_learner_tensor_info(const dz_learner_config* cfg, int32_t i, char* name64, int64_t* shape4,
                           int32_t* ndim, int64_t* offset);

typedef struct dz_learner_buffers {
  float* d_online;       /* [param_count] */
  float* d_target;       /* [param_count] */
  float* d_grads;        /* [param_count] */
  float* d_opt_state;    /* [opt_state_floats] */
  void* d_workspace;     /* [workspace_bytes] */
  int64_t* d_counters;   /* [4]: 0 = optimizer step count (adam `count`), 1 = rng counter, 2.. reserved */
} dz_learner_buffers;

typedef struct dz_learner dz_learner;
int dz_learner_create(const dz_learner_config* cfg, const dz_learner_buffers* buf, dz_learner** out);
void dz_learner_destroy(dz_learner* l);

/* One batch as device arrays (what `jit(update)` receives after the host->device transfer).
 * Observations are addressed through a pointer table so the fused path can read rows of the
 * replay store in place (gather fused into the conv1 operand load) while the explicit-batch
 * path points into dense arrays. */
typedef struct dz_batch {
  const uint8_t* const* d_s_tm1_rows;  /* [B] device pointers to obs rows */
  const uint8_t* const* d_s_t_rows;    /* [B] */
  const int32_t* d_a_tm1;              /* [B] */
  const float* d_r_t;                  /* [B] float32, as inside jit */
  const float* d_discount_t;           /* [B] */
  const float* d_weights;              /* [B] importance weights (float32) or NULL -> 1 */
  const float* d_taus;                 /* iqn: [B*N | B*K | B*N'] in U[0,1)  (iqn/agent.py:182-190) or NULL; fqf: unused */
  const float* d_noise;                /* rainbow: 3 applies x 8 vectors in the order of networks.py:235-248 (adv1 in/out,
                                          adv2 in/out, val1 in/out, val2 in/out), each padded to a multiple of 4 floats; or NULL.
                                          noisy networks: the same 3 applies (online(s_tm1) | the middle pass | target(s_t)),
                                          each fc1 in/out, head in/out (dueling: rainbow's 8 vectors with one atom) */
  const int32_t* d_shifts;             /* random_shift_pad > 0: [B][4] (dy0, dx0, dy1, dx1), each in [0, 2p]
                                          (dz_learner_generate_shifts); required then (DZ_EINVAL when NULL) and
                                          ignored when the pad is 0 */
} dz_batch;

typedef struct dz_update_outputs {
  float* d_loss;         /* [1] scalar loss (mean of weighted per-example losses) */
  float* d_per_example;  /* [B] per-example losses (c51/rainbow/qr/iqn) or td errors (dqn family) */
  float* d_priorities;   /* [B] new priorities: rainbow clip(|loss|,0,100) (rainbow/agent.py:194),
                                prioritized |td| (prioritized/agent.py:201), any other kind with
                                dz_learner_config.prioritized = 1 by the rule table there; else untouched;
                                may be NULL */
  float* d_grad_norm;    /* [1] global gradient norm before clipping; may be NULL */
  float* d_regularizer;  /* [B] the CQL regulariser R_b (dz_learner_config.cql_alpha), unweighted and without alpha:
                                written when cql_alpha > 0, else untouched; may be NULL */
} dz_update_outputs;

/* jit(update): forward passes, loss, backward, clip, optimizer, parameter update.
 * `apply_update` = 0 stops after the gradients (d_grads holds dLoss/dparams) for parity tests. */
int dz_learner_update(dz_learner* l, const dz_batch* batch, const dz_update_outputs* out, int32_t apply_update,
                      void* stream);

/* The whole `_learn()` (rainbow/agent.py:181-198) in one enqueue: sample -> (rows addressed in
 * place) -> update -> priority write-back.  `d_max_seen_priority` ([1] float32, device) is
 * updated as max(old, batch max) (rainbow/agent.py:196-197) by a learner that writes priorities.
 * `prioritized` = 1 needs such a learner (prioritized, rainbow, or dz_learner_config.prioritized = 1;
 * DZ_EINVAL otherwise, before anything is enqueued) and update_out.d_priorities. */
typedef struct dz_learn_io {
  dz_sample_inputs sample_in;
  dz_sample_outputs sample_out;
  const float* d_taus;
  const float* d_noise;
  dz_update_outputs update_out;
  float* d_max_seen_priority;
  double priority_exponent;  /* alpha */
  const int32_t* d_shifts;   /* as dz_batch.d_shifts */
} dz_learn_io;
int dz_learner_learn(dz_learner* l, const dz_replay_view* replay, int32_t prioritized, const dz_learn_io* io,
                     void* stream);

/* Fills d_taus / d_noise for one update from a counter-based generator (Philox4x32-10 keyed by
 * `seed`, counter d_counters[1] which it advances): taus ~ U[0,1) (iqn/agent.py:45-50); noise =
 * sign(n)*sqrt(|n|), n ~ TruncNormal(-2,2) (networks.py:142-144).  NOT the JAX threefry stream. */
int dz_learner_generate_randomness(dz_learner* l, uint64_t seed, float* d_taus, float* d_noise, void* stream);
/* Same draws, enqueued on the learner's side stream: ordered after the work already on `stream` and before the next
 * dz_learner_learn / dz_learner_update / dz_learner_act_batch on `stream` (they run beside the sampler instead of in
 * front of it).  Any other reader of d_taus / d_noise must synchronise the device first. */
int dz_learner_generate_randomness_async(dz_learner* l, uint64_t seed, float* d_taus, float* d_noise, void* stream);
/* random_shift_pad > 0: the shifts of one update, d_shifts [batch][4] int32, from the same generator at the current
 * counter d_counters[1] on stream id 3, WITHOUT advancing it: example b takes the Philox4x32-10 block at counter
 * (b, 0, ctr low, ctr high ^ (3 << 24)), key = seed, and its words w give (dy0, dx0, dy1, dx1) = floor(w (2p + 1) / 2^32).
 * Enqueue it before the dz_learner_generate_randomness (or _async) of the same step, whose counter step then covers
 * both.  DZ_EINVAL for a learner with the pad at 0 or a NULL buffer. */
int dz_learner_generate_shifts(dz_learner* l, uint64_t seed, int32_t* d_shifts, void* stream);

/* Batched acting for E <= batch independent environment streams (parts.py:342-411 run over many actors;
 * dqn/agent.py:121-131,169-177): online forward on E observations in one enqueue, q-values [E][num_actions] and the
 * epsilon-greedy choice on the device, so a tick costs ONE device-to-host copy of E int32 actions.  E = 1 with
 * d_actions NULL is select_action's network part (rainbow/agent.py:125-133; iqn/agent.py:228-243), the epsilon-greedy
 * draw left to the host.
 *   d_obs      E contiguous uint8 observations (obs_h*obs_w*obs_c bytes each), device memory
 *   d_taus     iqn: [E][tau_samples_policy] (fqf: NULL, its fractions are proposed from the torso features)
 *   d_noise    rainbow and noisy networks: noise_ld = 0, ONE apply shared by the E streams of the tick (they explore in lockstep);
 *              noise_ld = dz_learner_noise_stride, [E][stride] and stream e uses apply e (rainbow/agent.py:125-133 run
 *              by E actors, each drawing its own noise).  When every row carries the same apply the q-values and
 *              actions equal the shared mode's bit for bit.  Other kinds: noise_ld = 0.
 *   d_explore  [2][E] float32 uniforms in [0,1) (device) or NULL for greedy acting:
 *              action = u0[e] < epsilon ? min(floor(u1[e] * num_actions), num_actions - 1) : first argmax of q[e]
 *   d_actions  [E] int32, or NULL for q-values only
 * DZ_EINVAL for E outside [1, batch], a NULL d_obs / d_q_out, missing taus / noise or another noise_ld. */
int dz_learner_act_batch(dz_learner* l, const uint8_t* d_obs, int32_t E, const float* d_taus, const float* d_noise,
                         int64_t noise_ld, const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions,
                         void* stream);

/* Floats of ONE noise apply (rainbow: the 8 factorised-noise vectors; a noisy network: its 4 or 8; each padded to 4
 * floats); DZ_EINVAL for a network without noisy layers. */
int dz_learner_noise_stride(const dz_learner_config* cfg, int64_t* out);
/* E noise applies ([E][stride] floats) for dz_learner_act_batch's per-stream noise from the generator of
 * dz_learner_generate_randomness (same seed and counter: the first min(E, 3) applies equal what it writes); advances
 * d_counters[1] once.  DZ_EINVAL for a learner without noisy layers, E outside [1, batch] or a NULL buffer. */
int dz_learner_generate_stream_noise(dz_learner* l, uint64_t seed, int32_t E, float* d_noise, void* stream);

/* ---- Acting context (SURVEY §8(f) #3: many actor streams per GPU) ----------------------------------------------
 * Batched acting for num_streams in [1, 1024] streams per call (iqn: also num_streams * tau_samples_policy <= 16384;
 * fqf: num_streams * num_fractions <= 16384)
 * over the learner's ONLINE parameters, read in place: an act enqueued on the stream after a learner step sees that
 * step's parameters.  The actor keeps the learner handle (destroy the actor first) and owns only buffers sized for its
 * streams.  On the tensor-core geometries the torso and the 3136 -> 512 layer (noisy layers: with one shared noise
 * apply) run on the learner's sm_90a tensor-core kernels; the heads, and per-stream noisy layers, on the fp32-FMA
 * kernels.  Row e's result does not depend on num_streams. */
typedef struct dz_actor dz_actor;
/* Device workspace bytes of an actor for num_streams streams.  DZ_EINVAL outside the caps. */
int dz_actor_plan_query(const dz_learner_config* cfg, int32_t num_streams, int64_t* workspace_bytes);
int dz_actor_create(dz_learner* l, int32_t num_streams, void* d_workspace, dz_actor** out);
void dz_actor_destroy(dz_actor* a);
/* dz_learner_act_batch's contract for exactly num_streams observations (E below).  Noisy layers: noise_ld = 0, d_noise is
 * one apply shared by the streams; noise_ld = dz_learner_noise_stride, d_noise is [E][stride] and stream e uses apply e.
 * DZ_EINVAL for a NULL buffer, a missing taus / noise or another noise_ld. */
int dz_actor_act(dz_actor* a, const uint8_t* d_obs, const float* d_taus, const float* d_noise, int64_t noise_ld,
                 const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions, void* stream);
/* The learner's generator and counter (d_counters[1], advanced once): iqn taus [E][tau_samples_policy] with the stream
 * of dz_learner_generate_randomness's taus; rainbow and noisy networks one noise apply, or E applies when per_stream is set, with the
 * stream of its noise (so for E <= batch the draws equal those calls' for the same seed and counter).  DZ_EINVAL for
 * other kinds (fqf included: it draws nothing), per_stream on iqn or a NULL buffer. */
int dz_actor_generate_randomness(dz_actor* a, uint64_t seed, int32_t per_stream, float* d_out, void* stream);

/* ---- Frozen acting context (evaluation over a parameter snapshot) -------------------------------------------------
 * The acting context above with its own state: a snapshot of P parameter floats in the learner's layout and a generator
 * counter, both inside its workspace.  The learner handle supplies only the configuration, layout, dims and split
 * counts (the actor keeps a copy of them, not the handle: the learner may be destroyed first).  Acting, randomness and
 * loading read and write only the actor's workspace, the caller's buffers and constant tables, never a learner's device
 * state, so a frozen actor can act on another CUDA stream while a learner trains.  dz_actor_act and
 * dz_actor_generate_randomness take a frozen actor with the same contract; act fails (DZ_EINVAL) before the first
 * load_params.  The live-only calls below fail on a live actor. */
/* Device workspace bytes of a frozen actor; the workspace must be zero-filled before dz_actor_create_frozen, as a live
 * actor's. */
int dz_actor_frozen_plan_query(const dz_learner_config* cfg, int32_t num_streams, int64_t* workspace_bytes);
int dz_actor_create_frozen(dz_learner* l, int32_t num_streams, void* d_workspace, dz_actor** out);
/* snapshot <- d_src (P floats, e.g. a learner's online blob), then the conv weight images are packed once; on stream. */
int dz_actor_load_params(dz_actor* a, const float* d_src, void* stream);
/* d_dst <- the snapshot (P floats), on stream.  DZ_EINVAL before the first load_params. */
int dz_actor_get_params(dz_actor* a, float* d_dst, void* stream);
/* The generator counter (0 at creation; each generate_randomness advances it once), ordered on stream (both calls
 * synchronise with it). */
int dz_actor_get_counter(dz_actor* a, int64_t* out, void* stream);
int dz_actor_set_counter(dz_actor* a, int64_t value, void* stream);

/* target <- online (dqn/agent.py:155-156): device-to-device copy of the blob. */
int dz_learner_sync_target(dz_learner* l, void* stream);

/* Writes the device's uint8 -> float32/255 conversion of 0..255 (the conv1 operand load, networks.py:193)
 * into d_out256 so tests can check it is the correctly rounded quotient. */
int dz_test_u8_to_unit(float* d_out256, void* stream);


/* ---- Atari frame preprocessing (SURVEY §8(f) #3) ---------------------------------------------------------------
 * Replaces the observation branch of processors.atari() — np.max over the pooled frame pair, rgb2y, PIL bilinear
 * resize, frame stack (dqn_zoo/processors.py:367-388, 482-501) — for n_env environment streams per launch.
 * One resampling axis of Pillow's bilinear filter (libImaging/Resample.c): window [first, first + count) and
 * fixed-point (22-bit) coefficients per output index; the tables are host-computed by the caller. */
typedef struct dz_resample_axis {
  const int32_t* d_bounds;   /* [out_size][2] = (first, count) */
  const int32_t* d_kk;       /* [out_size][ksize] */
  int32_t ksize, in_size, out_size;
} dz_resample_axis;
/* d_frame_a/b: [n_env] device pointers to uint8 [in_h][in_w][3] raw frames, 16-byte aligned, 3*in_w % 16 == 0
 * (NULL = zero padding, processors.py:54-66);
 * d_stacks[e]: device pointer to stream e's uint8 [out_h][out_w][stack]; d_counts[e] = frames already in stream e's stack
 * (< stack: the new frame goes to channel count; == stack: channels shift left, new frame last);
 * luma3 = {0.299, 0.587, 1 - (0.299 + 0.587)} (host doubles); max_band_rows = the largest number of input rows any
 * band of dz_atari_preprocess_band_rows() output rows touches (sizes the shared-memory staging). */
int dz_atari_preprocess(const uint8_t* const* d_frame_a, const uint8_t* const* d_frame_b, int32_t n_env,
                        const dz_resample_axis* horizontal, const dz_resample_axis* vertical,
                        uint8_t* const* d_stacks, const int32_t* d_counts, int32_t stack, const double* luma3,
                        int32_t max_band_rows, void* stream);
int32_t dz_atari_preprocess_band_rows(void);

/* ---- JAX-compatible uniform draws (SURVEY §8(f) #2) -----------------------------------------------------------
 * jax.random.uniform(key, (count,), float32) for up to 4 independent keys per launch, bit-identical to jax 0.3.10's
 * threefry2x32 path (iqn/agent.py:45-50 `_sample_tau`).  d_keys: DEVICE uint32 [nblocks][2] (so that a captured CUDA
 * graph can be replayed with fresh keys); counts: HOST int64 [nblocks]; block b is written at
 * d_out + sum(counts[:b]). */
int dz_jax_uniform(const uint32_t* d_keys, const int64_t* counts, int32_t nblocks, float* d_out, void* stream);
/* threefry2x32 (20 rounds) evaluated on the HOST by the same source the kernel compiles; tests only. */
int dz_test_threefry2x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t* out2);

/* ---- Games at Atari geometry on the device (DESIGN.md §10-§12) -------------------------------------------------
 * Catch, Breakout and Pong run E streams each, every stream simulated and rendered as a 210x160x3 uint8 RGB frame in
 * HBM, and share one configuration and one calling convention.  State: int32 [DZ_<GAME>_STATE_FIELDS][E] device array
 * (the fields are listed per game below); a new state is all 0 but over = 1, so that the first tick of every stream is
 * a reset.  Stream e's randomness: key = threefry2x32((0, seed), (stream_offset + e, tag)), tag 0 for Catch, 1 for
 * Breakout, 2 for Pong.
 *
 * dz_<game>_step: one tick of all E streams.  h_control: PINNED int32 [2][E] (row 0 actions, row 1 reset flags:
 * non-zero starts a new episode instead of stepping; so does stepping a stream whose last step was LAST), checked on
 * the host (an action outside [0, A) of a stream that is not reset is DZ_EINVAL) and copied into d_control (device
 * int32 [2][E]).  The kernel updates d_state, writes every stream's frame into d_frames (device uint8 [E][210][160][3],
 * 16-byte aligned) and d_record (device int32 [DZ_<GAME>_RECORD_FIELDS][E]: step_type 0 FIRST / 1 MID / 2 LAST,
 * reward, discount, lives; reward and discount are 0 on FIRST), which is copied to h_record (PINNED, same shape).  All
 * on `stream`; the caller synchronises before reading h_record or reusing h_control.
 * dz_<game>_render: renders every stream's frame from d_state (e.g. after the state was restored); the state is not
 * changed.
 * dz_test_<game>_step: the kernel's tick and picture evaluated on the HOST by the same source: stream id
 * cfg->stream_offset, state int32 [DZ_<GAME>_STATE_FIELDS] updated in place, frame (NULL: not rendered) 210*160*3
 * bytes, record int32 [4]; tests only. */
typedef struct dz_game_config {
  int32_t num_streams;      /* E in [1, DZ_<GAME>_MAX_STREAMS] */
  int32_t num_actions;      /* A in [the game's minimum, 18] */
  int32_t min_noop_steps;   /* 0 <= min <= max <= DZ_<GAME>_MAX_NOOP_STEPS */
  int32_t max_noop_steps;
  uint32_t seed;
  uint32_t stream_offset;   /* stream_offset + E <= 2^32 */
} dz_game_config;

/* Catch (DESIGN.md §10).  State fields paddle_x, ball_x, ball_y, ball_dx, lives, balls_left, counter, noops, over.
 * Actions: A in [3, 18]: 0 stay, 1 left, 2 right, 3.. stay. */
#define DZ_CATCH_HEIGHT 210
#define DZ_CATCH_WIDTH 160
#define DZ_CATCH_STATE_FIELDS 9
#define DZ_CATCH_RECORD_FIELDS 4
#define DZ_CATCH_MAX_STREAMS 4096
#define DZ_CATCH_MAX_NOOP_STEPS 89   /* the first ball lands on the 90th frame after a reset */
typedef dz_game_config dz_catch_config;
int dz_catch_step(const dz_catch_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                  uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream);
int dz_catch_render(const dz_catch_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream);
int dz_test_catch_step(const dz_catch_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                       int32_t* record);

/* The project's own Breakout (not ALE's; DESIGN.md §11).  State fields paddle_x, ball_x, ball_y, ball_dx, ball_dy,
 * in_play, serve_timer, lives, row0..row5 (18-bit brick masks, bit c = brick (r, c) is there), counter, noops, over.
 * Actions: A in [4, 18]: 0 no-op, 1 fire, 2 right, 3 left, 4.. no-op. */
#define DZ_BREAKOUT_HEIGHT 210
#define DZ_BREAKOUT_WIDTH 160
#define DZ_BREAKOUT_BRICK_ROWS 6
#define DZ_BREAKOUT_BRICK_COLS 18
#define DZ_BREAKOUT_STATE_FIELDS 17
#define DZ_BREAKOUT_RECORD_FIELDS 4
#define DZ_BREAKOUT_MAX_STREAMS 4096
#define DZ_BREAKOUT_MAX_NOOP_STEPS 63   /* below the 64-frame serve delay: no ball is served during the no-ops */
typedef dz_game_config dz_breakout_config;
int dz_breakout_step(const dz_breakout_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                     uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream);
int dz_breakout_render(const dz_breakout_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream);
int dz_test_breakout_step(const dz_breakout_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                          int32_t* record);

/* The project's own Pong (not ALE's; DESIGN.md §12), against a scripted opponent.  State fields paddle_y, opponent_y,
 * ball_x, ball_y, ball_dx, ball_dy, in_play, serve_timer, agent_score, opponent_score, counter, noops, over.
 * Actions: A in [6, 18]: 0 no-op, 1 fire, 2 up, 3 down, 4 up + fire, 5 down + fire, 6.. no-op. */
#define DZ_PONG_HEIGHT 210
#define DZ_PONG_WIDTH 160
#define DZ_PONG_STATE_FIELDS 13
#define DZ_PONG_RECORD_FIELDS 4
#define DZ_PONG_MAX_STREAMS 4096
#define DZ_PONG_MAX_NOOP_STEPS 63   /* below the 64-frame serve delay: no ball is served during the no-ops */
typedef dz_game_config dz_pong_config;
int dz_pong_step(const dz_pong_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                 uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream);
int dz_pong_render(const dz_pong_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream);
int dz_test_pong_step(const dz_pong_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                      int32_t* record);

/* Device pointer + element count of an internal learner buffer of the last update (pass 0: "act1", "act2", "act3",
 * "h1", "h1_val", "dh1", "dh1_val", "iqn_e0", "iqn_hi", "iqn_dhi"; the fp32 input gradients of the conv layers' masked
 * outputs "dact1", "dact2", "dact3"; on the tensor-core torso only, where "act1" and "act2" are the tf32 hi images,
 * their lo images "act1_lo", "act2_lo" and the tf32 hi / lo split of each input gradient that the next GEMM reads,
 * "dact1_hi" .. "dact3_hi" and "dact1_lo" .. "dact3_lo" (DZ_EINVAL on the fp32-FMA torso); fqf's proposals: "fqf_tau"
 * [2][B][N+1] and "fqf_tau_hat" [2][B][N], application 0 from online(s_tm1)'s features and 1 from target(s_t)'s, and
 * "fqf_dlogits" [B][N]); tests/tools only. */
int dz_test_learner_buffer(dz_learner* l, const char* name, float** d_ptr, int64_t* count);
/* The per-example arithmetic of the munchausen loss kernel evaluated on the HOST by the same source (fp32, expf / logf):
 * q_tm1 = online(s_tm1), qbar_tm1 = target(s_tm1), qbar_t = target(s_t), each [A] (1 <= A <= 18).  Writes the target
 * out[0], td out[1] and the log-policy bonus alpha * clip(tau * log pi(a_tm1 | s_tm1), l0, 0) out[2].  DZ_EINVAL for
 * A or a_tm1 out of range and for the hyperparameters dz_learner_create rejects; tests only. */
int dz_test_munchausen_example(const float* q_tm1, const float* qbar_tm1, const float* qbar_t, int32_t A, int32_t a_tm1,
                               float r_t, float discount_t, float alpha, float tau, float l0, float* out);
/* The per-example target arithmetic of the munchausen_iqn loss kernel evaluated on the HOST by the same source (fp32,
 * expf / logf): zbar_tm1 = target(s_tm1) at the K policy taus [K][A], zbar_t = target(s_t) at the N' taus [Nt][A]
 * (1 <= A <= 18, 1 <= K, Nt <= 256).  Writes the targets y_j to out[0 .. Nt), the log-policy bonus
 * alpha * clip(tau * log pi(a_tm1 | s_tm1), l0, 0) to out[Nt] and the entropy term sum_a pi(a|s_t) h_t(a) to out[Nt + 1].
 * DZ_EINVAL for sizes or a_tm1 out of range and for the hyperparameters dz_learner_create rejects; tests only. */
int dz_test_munchausen_iqn_example(const float* zbar_tm1, const float* zbar_t, int32_t A, int32_t K, int32_t Nt,
                                   int32_t a_tm1, float r_t, float discount_t, float alpha, float tau, float l0, float* out);
/* The per-example fraction arithmetic of fqf's fraction and loss kernels evaluated on the HOST by the same source
 * (fp32, expf): logits [N] (2 <= N <= 128) -> q = softmax, tau_0..tau_N, tau_hat and the interval weights w; then the
 * fraction gradient from F_tau [N] (F_tau[i] = Z(s_tm1, a_tm1, tau_i), entries 1..N-1 read) and F_hat [N]
 * (Z(s_tm1, a_tm1, tau_hat_i)), chained through the cumulative sum and the softmax and scaled by cot (w_b / B).  Writes
 * q to out[0, N), tau to out[N, 2N+1), tau_hat to out[2N+1, 3N+1), w to out[3N+1, 4N+1) and dlogits to
 * out[4N+1, 5N+1).  DZ_EINVAL for N out of range or a NULL buffer; tests only. */
int dz_test_fqf_example(const float* logits, const float* F_tau, const float* F_hat, int32_t N, float cot, float* out);
/* Host twin of the dueling head's per-row arithmetic (dueling_head_fwd_kernel / dueling_head_bwd_kernel; DESIGN.md
 * §16), the functions those kernels run: from the advantages adv [A], the value v and the q gradient dq [A] it writes
 * q_a = v + (adv_a - m) with m = (sum_a adv_a) / A to out[0, A), dadv_a = dq_a - (sum_a dq_a) / A to out[A, 2A) and
 * dval = sum_a dq_a to out[2A].  Sums run in action order.  DZ_EINVAL for A outside [1, 64] or a NULL buffer; tests only. */
int dz_test_dueling_example(const float* adv, float v, const float* dq, int32_t A, float* out);
/* Host twin of the CQL(H) arithmetic of every loss kernel (DESIGN.md §20), the function their cql variants run: from
 * the expected values q [A] of one example on s_tm1 it writes g_a = cot (softmax(q)_a - [a = a_tm1]) to out[0, A) and
 * R = logsumexp_a q_a - q_{a_tm1} (max-subtracted) to out[A].  Sums run in action order.  DZ_EINVAL for A outside
 * [1, 64], a_tm1 outside [0, A) or a NULL buffer; tests only. */
int dz_test_cql_example(const float* q, int32_t A, int32_t a_tm1, float cot, float* out);
/* The loss section of a learner step (the agent kind's loss kernel, then the scalar loss and the running max priority)
 * on caller-owned device buffers, all enqueued on `stream`; tests only.  cfg is validated as
 * dz_learner_create does, with batch = B and its observation fields replaced by a legal geometry.  d_out[p]: the head
 * outputs of pass p (0 online(s_tm1); dqn: 2 target(s_t) is also the selector; double_q / prioritized: 1 online(s_t)
 * selects; c51: [B][A][K] logits, 2 is target(s_t) and selects; rainbow: advantages [B][A][K] with d_val[p] the value
 * streams [B][K], for online(s_tm1), online(s_t), target(s_t); qrdqn: [B][N][A]; iqn: [B][N_tm1 | N_policy | N_t][A];
 * munchausen / munchausen_iqn: 1 is target(s_tm1)).  d_weights: importance weights [B] or NULL; d_taus: the s_tm1
 * taus [B][N_tm1] (iqn, munchausen_iqn).  Writes d_dout (the gradient wrt pass 0; rainbow: advantages, with d_dval the
 * value stream), d_per_example, d_priorities (required from a configuration that writes priorities: prioritized,
 * rainbow, or cfg->prioritized = 1), d_loss_terms [B], d_loss [1] and, when d_max_seen is given to such a
 * configuration, the running max priority.  fqf's loss needs its fraction buffers: dz_test_loss_fqf. */
int dz_test_loss(const dz_learner_config* cfg, int32_t B, const float* const* d_out, const float* const* d_val,
                 const int32_t* d_a_tm1, const float* d_r_t, const float* d_discount_t, const float* d_weights,
                 const float* d_taus, float* d_dout, float* d_dval, float* d_per_example, float* d_priorities,
                 float* d_loss_terms, float* d_loss, float* d_max_seen, void* stream);
/* fqf's loss section on caller-owned device buffers, as dz_test_loss; tests only.  N = num_fractions: d_out[0]
 * online(s_tm1) at tau_hat [B][N][A], d_out[1] online(s_tm1) at tau_1..tau_N [B][N][A] (the last row, tau_N = 1, is not
 * read), d_out[2] target(s_t) at [tau_hat' | tau_hat] [B][2N][A]; d_tau_hat [B][N], d_w_t the interval weights of
 * s_t's proposal [B][N], d_q_tm1 the fractions of s_tm1's [B][N].  Writes d_dout [B][N][A], d_dlogits [B][N],
 * d_per_example, d_loss_terms [B] and d_loss [1].  It takes no priority buffer, so by dz_test_loss's rule a cfg with
 * prioritized = 1 is DZ_EINVAL here; fqf's priorities are those of a learner step (dz_learner_update). */
int dz_test_loss_fqf(const dz_learner_config* cfg, int32_t B, const float* const* d_out, const int32_t* d_a_tm1,
                     const float* d_r_t, const float* d_discount_t, const float* d_weights, const float* d_tau_hat,
                     const float* d_w_t, const float* d_q_tm1, float* d_dout, float* d_dlogits, float* d_per_example,
                     float* d_loss_terms, float* d_loss, void* stream);
/* The acting tail of every acting entry point on caller-owned device buffers; tests only.  d_out: the head outputs of
 * E observations in the layout of d_out[p] above (iqn: tau_samples_policy samples; rainbow: advantages, d_val the value
 * streams).  Writes the q-values d_q_out [E][A] and, when d_actions is given, the epsilon-greedy actions as
 * dz_learner_act_batch does (d_explore: [2][E] uniforms or NULL).  fqf: dz_test_q_values_fqf. */
int dz_test_q_values(const dz_learner_config* cfg, int32_t E, const float* d_out, const float* d_val, const float* d_explore,
                     float epsilon, float* d_q_out, int32_t* d_actions, void* stream);
/* fqf's acting tail, as dz_test_q_values: d_out [E][N][A] at tau_hat and d_frac_w the interval weights [E][N]. */
int dz_test_q_values_fqf(const dz_learner_config* cfg, int32_t E, const float* d_out, const float* d_frac_w,
                         const float* d_explore, float epsilon, float* d_q_out, int32_t* d_actions, void* stream);
/* fqf's fraction proposal of learner l's layout (num_fractions N, feature width D, the fraction layer of d_params) on
 * caller-owned buffers; tests only.  d_feat: host array of napp (1 or 2) device features [E][D].  d_tau [E][N + 1],
 * d_tau_hat, d_w, d_q [E][N]: host arrays of 2 device pointers, any of them (or the array) NULL; d_pass1 [E][N] and
 * d_pass2 [E][2N] (the learner's pass inputs) may be NULL. */
int dz_test_fraction_forward(dz_learner* l, int32_t E, int32_t napp, const float* const* d_feat, const float* d_params,
                             float* const* d_tau, float* const* d_tau_hat, float* const* d_w, float* const* d_q,
                             float* d_pass1, float* d_pass2, void* stream);
/* The dueling head forward of dueling learner l's layout (plain or noisy) on caller-owned buffers; tests only.  np in
 * 1..3 passes of `rows` rows: d_h1 host array [np][2] of device [rows][512] (advantage, value stream), d_params[i] a
 * parameter blob, d_out[i] q [rows][A].  Noisy: d_noise[i] the pass's noise apply (noise_ld > 0: row r's apply at
 * d_noise[i] + r * noise_ld); NULL and 0 for the plain network. */
int dz_test_dueling_head_fwd(dz_learner* l, int32_t rows, int32_t np, const float* const* d_h1, const float* const* d_params,
                             const float* const* d_noise, int64_t noise_ld, float* const* d_out, void* stream);
/* The dueling head backward of dueling learner l's layout on caller-owned buffers; tests only.  d_dq [rows][A] becomes
 * dadv in place; writes d_dval [rows] and d_dh1[s] [rows][512] (host array of 2) masked by d_h1[s] > 0 and, when d_hi /
 * d_lo (host arrays of 2, or NULL) are given, the tf32 hi/lo pair of each dh1.  Noisy: d_noise is the noise apply. */
int dz_test_dueling_head_bwd(dz_learner* l, int32_t rows, float* d_dq, float* d_dval, const float* const* d_h1,
                             const float* d_params, const float* d_noise, float* const* d_dh1, float* const* d_hi,
                             float* const* d_lo, void* stream);
/* Rainbow's noisy head forward of rainbow learner l's layout on caller-owned buffers; tests only.  np in 1..3 passes of
 * `rows` <= 32 rows: d_h1 host array [np][2] of device [rows][512] (advantage, value stream; 16-byte aligned),
 * d_params[i] a parameter blob (passes with the same blob share its weight tiles), pass i's noise apply at apply i of
 * d_noise, d_out host array [np][2] of device [rows][A * atoms] and [rows][atoms]. */
int dz_test_noisy_head_fwd(dz_learner* l, int32_t rows, int32_t np, const float* const* d_h1, const float* const* d_params,
                           const float* d_noise, float* const* d_out, void* stream);
/* Rainbow's noisy head input gradient on caller-owned buffers; tests only.  d_dout host array of 2 ([rows][A * atoms],
 * [rows][atoms]), the head of d_params through noise apply 0 of d_noise; writes d_dh1[s] [rows][512] masked by
 * d_h1[s] > 0 and, when d_hi / d_lo (host arrays of 2, or NULL) are given, the tf32 hi/lo pair of each dh1. */
int dz_test_noisy_head_bwd(dz_learner* l, int32_t rows, const float* const* d_dout, const float* d_params, const float* d_noise,
                           const float* const* d_h1, float* const* d_dh1, float* const* d_hi, float* const* d_lo, void* stream);
/* IQN's cosine features on caller-owned buffers; tests only: d_out [rows][latent] = cos(fl(fl((j + 1) pi_f) tau_r)) of
 * d_taus [rows]. */
int dz_test_iqn_cos(const float* d_taus, int64_t rows, int32_t latent, float* d_out, void* stream);
/* IQN's value head of IQN-network learner l's layout (A = num_actions <= 18) on caller-owned buffers; tests only.  np in
 * 1..3 applies in one launch: apply i reads d_h1[i] [M[i]][512] (16-byte aligned) and the head of the parameter blob
 * d_params[i], and writes d_out[i] [M[i]][A].  M: host array of np row counts. */
int dz_test_iqn_head_fwd(dz_learner* l, int32_t np, const int32_t* M, const float* const* d_h1, const float* const* d_params,
                         float* const* d_out, void* stream);
/* The value head's input gradient of learner l's layout; tests only: d_dh1 [M][512] = [d_h1 > 0] d_dout W^T with d_dout
 * [M][A] and W the head of d_params (A <= 18). */
int dz_test_iqn_head_dgrad(dz_learner* l, int32_t M, const float* d_dout, const float* d_params, const float* d_h1,
                           float* d_dh1, void* stream);
/* The backward of IQN's Hadamard product E * F; tests only.  d_E, d_dhi [B][N][D], d_F, d_dfeat [B][D]: d_dfeat = [F > 0]
 * sum_n dhi E, dE = [E > 0] dhi F.  packed = 0: dE replaces d_dhi in place (the image arguments are unused).  packed = 1
 * (N = 64, D % 64 = 0): d_dhi is read only and dE is written as the hi/lo tf32 tile image of rows k < D and reduction
 * b * 64 + n into d_img_hi / d_img_lo ([img_rows_pad][B * 64], img_rows_pad a multiple of 128). */
int dz_test_iqn_hadamard_bwd(int32_t packed, int32_t B, int32_t N, int32_t D, float* d_dhi, const float* d_E, const float* d_F,
                             float* d_dfeat, float* d_img_hi, float* d_img_lo, int32_t img_rows_pad, void* stream);
int dz_test_copy(void* d_dst, const void* d_src, int64_t bytes, void* stream);   /* device-to-device, tests only */
/* The learner's random-shift kernel alone, tests only: observations [H][W][C] at d_rows_tm1[b] / d_rows_t[b] shifted by
 * d_shifts[b] (dz_batch.d_shifts; components clamped to [0, 2p]) into d_out [B][2][out_stride] (s_tm1, then s_t), with
 * the out_stride - H*W*C padding bytes of each row zeroed.  DZ_EINVAL unless pad is in [0, 16] and < min(H, W), C % 4 == 0,
 * W * C is a multiple of 16 and at most 32768, out_stride >= H*W*C is a multiple of 16 and d_out is 16-byte aligned;
 * the source rows must be 16-byte aligned. */
int dz_test_random_shift(const uint8_t* const* d_rows_tm1, const uint8_t* const* d_rows_t, const int32_t* d_shifts,
                         int32_t B, int32_t H, int32_t W, int32_t C, int32_t pad, uint8_t* d_out, int64_t out_stride,
                         void* stream);
/* Debug: the tensor-core launch named `tag` writes the clock stamps of its CTA 0 into d_trace (512 int64). */
int dz_test_learner_trace(dz_learner* l, const char* tag, long long* d_trace);
/* Tests: which MMA path the tensor-core launch `tag` (same tags, and "conv1_fwd") takes: *path = 1 warp-level mma.sync,
 * 2 wgmma.  The IQN update's "iqn_embed_fwd", "iqn_fc1_fwd", "iqn_fc1_wgrad", "iqn_fc1_dgrad" and "iqn_embed_wgrad"
 * give 1 when the launch runs on the packed-operand GEMM (csrc/dz_tcp.cuh) and DZ_EINVAL when it runs on the fp32-FMA
 * kernels, independently of the torso's path. */
int dz_test_learner_mma_path(dz_learner* l, const char* tag, int32_t* path);
/* Tests: the same for the actor's forward launches ("conv1_fwd", "conv2_fwd", "conv3_fwd", "fc1_fwd" / "noisy1_fwd");
 * DZ_EINVAL when the actor runs on the fp32-FMA kernels. */
int dz_test_actor_mma_path(dz_actor* a, const char* tag, int32_t* path);
/* Tests: device pointer + element count of the actor's conv3 output "act3" ([E][feat], written by the last act). */
int dz_test_actor_buffer(dz_actor* a, const char* name, float** d_ptr, int64_t* count);
/* Debug: every kernel appends (globaltimer ns, gridDim.x << 32 | gridDim.y << 16 | blockDim.x) to d_buf right after its
 * dependencies completed; d_buf[0] (low 32 bits) counts the entries, entries start at d_buf[2].  d_buf: 2 + 2 * 4000
 * uint64, zeroed by the caller; nullptr switches the stamps off.  Works under CUDA-graph replay (tools/step_timeline.py). */
int dz_debug_timeline(unsigned long long* d_buf);
/* Self-test of the packed-operand tensor-core GEMM (csrc/dz_tcp.cuh; the IQN 3136->512 layer's kernels): packs
 * A (a_rows x red) and B (b_rows x red) from plain fp32 matrices (x_red_contig = 1: element (row, r) at
 * x[row*ld + r]; 0: at x[r*ld + row]) into hi/lo TF32 tile images inside d_work (dz_test_tc_pgemm_work floats),
 * then D[i,j] = sum_r A(i,r) B(j,r).  a_ones_row = a_rows appends a row of ones to A (bias-gradient row), -1: none.
 * splits == 1: + d_bias[j] and ReLU are applied if given; otherwise raw partials at d_C + s*split_stride. */
int64_t dz_test_tc_pgemm_work(int32_t a_rows, int32_t b_rows, int32_t red);
int dz_test_tc_pgemm(const float* d_A, int32_t a_rows, int32_t a_ld, int32_t a_red_contig, const float* d_B,
                     int32_t b_rows, int32_t b_ld, int32_t b_red_contig, int32_t red, int32_t a_ones_row,
                     float* d_work, float* d_C, int64_t sc_i, int64_t sc_j, int32_t splits, int64_t split_stride,
                     const float* d_bias, int32_t relu, void* stream);
/* Self-test of the IQN embedding epilogue of the packed-operand GEMM (the learner's embedding forward): packs d_cos
 * [M][latent] and d_embed_w [latent][D] into d_work (dz_test_tc_pgemm_work(M, D, latent) floats), then with
 * v = relu(cos W + d_bias[j]) writes v to d_e0 [M][D] (or nothing when NULL) and h = v * d_mul[(i / mul_div) * mul_ld + j]
 * as the hi/lo tf32 tile images d_img_hi / d_img_lo (rows i, [ceil(M / 128) 128][ceil(D / 16) 16]) and, when given,
 * d_imgT_hi / d_imgT_lo (rows j, [ceil((D + 1) / 128) 128][ceil(M / 16) 16]).  Only the valid elements of the images
 * are written.  latent <= 128; M, D, mul_ld multiples of 4; mul_ld >= D; d_bias, d_mul, d_e0 16-byte aligned. */
int dz_test_iqn_embed_packed(const float* d_cos, int32_t M, int32_t latent, const float* d_embed_w, int32_t D,
                             const float* d_bias, const float* d_mul, int32_t mul_div, int32_t mul_ld, float* d_work,
                             float* d_e0, float* d_img_hi, float* d_img_lo, float* d_imgT_hi, float* d_imgT_lo,
                             void* stream);
/* Self-test of the TMA-fed tensor-core GEMM family (csrc/dz_umma.cuh; conv / FC layers of the batch-32 step):
 * C[MI][NJ] = sum_r A(i,r) B(j,r), NJ <= 64.  x_mn_major = 0: the operand is stored [rows][R]; 1: [R][rows] (the
 * MMA warps' fragment loads transpose).  convert = 0: operands pre-split into tf32 hi/lo arrays (activation path);
 * 1: raw fp32 tiles split in shared memory by the converter warps (weight path), A optionally scaled by
 * d_scale_r[r].  epi_rows = 1: row epilogue (+ d_bias[j], relu; tf32 hi/lo copies in d_hi / d_lo).  stages: depth of
 * the shared-memory stage ring (0: 4; the launch fails when the ring does not fit).  Synchronizes. */
int dz_test_umma_gemm(const float* d_A, int32_t a_mn_major, const float* d_B, int32_t b_mn_major, int32_t MI, int32_t NJ,
                      int32_t R, int32_t convert, const float* d_scale_r, int32_t stages, int32_t epi_rows,
                      const float* d_bias, int32_t relu, float* d_C, float* d_hi, float* d_lo, void* stream);
/* The same with the MMA kernel chosen by `path`: 0 automatic (as the learner's launches: wgmma when both operands are
 * K-major and pre-split), 1 warp-level mma.sync kernel, 2 wgmma kernel (fails for MN-major or converted operands). */
int dz_test_umma_gemm_path(const float* d_A, int32_t a_mn_major, const float* d_B, int32_t b_mn_major, int32_t MI, int32_t NJ,
                           int32_t R, int32_t convert, const float* d_scale_r, int32_t stages, int32_t epi_rows,
                           const float* d_bias, int32_t relu, float* d_C, float* d_hi, float* d_lo, int32_t path, void* stream);
/* The fc1 / noisy1 forward launch alone (split partials [npass][nstream][S][B][512] of features x [npass * B][feat]
 * against the stream weights at online / target + off_w[s] (mu) and + off_sw[s] (sigma), noise apply p = pass p).
 * per_pass = 0: the learner's plan (passes that apply one blob share each staged weight tile, umma_fc_kernel); 1: one CTA
 * group per pass on umma_gemm_kernel with converter warps.  *weight_bytes: weight-tile bytes the launch stages.
 * d_part holds npass * nstream * 24 * B * 512 floats.  Synchronizes. */
int dz_test_fc_forward(int32_t B, int32_t H, int32_t W, int32_t npass, int32_t nstream, int32_t noisy, const float* online,
                       const float* target, const int64_t* off_w, const int64_t* off_sw, const float* noise, int64_t noise_stride,
                       const int64_t* off_in, const int64_t* off_out, const float* x, int32_t per_pass, float* d_part,
                       int32_t* splits, int64_t* weight_bytes, void* stream);
/* The fc1 / noisy1 input-gradient launch alone (split partials [nstream][S][B][feat] of the output gradients
 * g [nstream][B][512] against the stream weights at online + off_w[s] (mu) and + off_sw[s] (sigma), noise eps_in /
 * eps_out at noise + off_in[s] / off_out[s]).  converters = 0: the learner's umma_fc_kernel; 1: umma_gemm_kernel with
 * converter warps.  d_part holds nstream * 8 * B * feat floats.  Synchronizes. */
int dz_test_fc_dgrad(int32_t B, int32_t H, int32_t W, int32_t nstream, int32_t noisy, const float* online, const int64_t* off_w,
                     const int64_t* off_sw, const float* noise, const int64_t* off_in, const int64_t* off_out, const float* g,
                     int32_t converters, float* d_part, int32_t* splits, void* stream);
/* The conv1 forward launch alone: act1 tf32 hi / lo [npass * B][h1][w1][32] (into d_hi / d_lo) of the uint8
 * observations B x H x W x 4 that rows[p] (host array of npass device tables of B row pointers) point at, pass layout as
 * in dz_test_fc_forward.  off_conv_w: the three conv weight offsets in both blobs; off_conv_b1: conv1's bias.  path: 2 the
 * learner's wgmma kernel, 1 the warp-level mma.sync kernel it is checked against.  Synchronizes. */
int dz_test_conv1_forward(int32_t B, int32_t H, int32_t W, int32_t npass, const float* online, const float* target,
                          const int64_t* off_conv_w, int64_t off_conv_b1, const uint8_t* const* const* rows, int32_t path,
                          float* d_hi, float* d_lo, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DQN_ZOO_B200_H_ */
