// The driver of the device games (dz_catch.cu, dz_breakout.cu, dz_pong.cu; DESIGN.md §10-§12): the tick, the kernel
// that steps or renders E streams, and the bodies of each game's three C entry points.  A game is a trait struct G:
//   State                                a struct of int32 fields ending in counter, noops, over;
//   kName                                "catch", "breakout", "pong": the <game> of the messages and launch names;
//   kTag                                 the second counter word of the stream key (0, 1, 2);
//   kMaxStreams, kMinActions, kMaxNoopSteps, kBackground (packed 0x00BBGGRR);
//   start(State&, k0, k1)                the game's part of a reset, before the no-op frames;
//   frame(State&, action, k0, k1)        one frame of the rules, returning its reward (action 0 is a no-op);
//   over(const State&), lives(const State&);
//   rgb(const State&, x, y)              the colour of pixel (x, y), packed 0x00BBGGRR;
//   span_has_object(const State&, y, xa, xb)   can anything but background touch pixels [xa, xb] of row y?
//                                        Conservative: false means background.
// The kernel and the host twin run the same game_tick, so the twin pins the kernel's rules.
#pragma once
#include "dz_common.cuh"
#include "dz_threefry.cuh"

namespace dz {

// Every game draws a 210x160 RGB frame: rows of 480 bytes, 30 16-byte words.
constexpr int kFrameH = 210, kFrameW = 160;
constexpr int kRowWords = 3 * kFrameW / 16;
constexpr int kFrameBytes = kFrameH * 3 * kFrameW;   // 100,800
constexpr int kGameThreads = 256;
static_assert(3 * kFrameW % 16 == 0, "rows are whole 16-byte words");
static_assert(DZ_CATCH_HEIGHT == kFrameH && DZ_BREAKOUT_HEIGHT == kFrameH && DZ_PONG_HEIGHT == kFrameH &&
                  DZ_CATCH_WIDTH == kFrameW && DZ_BREAKOUT_WIDTH == kFrameW && DZ_PONG_WIDTH == kFrameW,
              "one frame geometry");

struct GameStep { int32_t step_type, reward, discount, lives; };   // a stream's record of one tick
static_assert(sizeof(GameStep) == DZ_CATCH_RECORD_FIELDS * sizeof(int32_t) &&
                  DZ_BREAKOUT_RECORD_FIELDS == DZ_CATCH_RECORD_FIELDS &&
                  DZ_PONG_RECORD_FIELDS == DZ_CATCH_RECORD_FIELDS,
              "one record field per GameStep member");

// floor(u * n / 2^32): a uniform draw in [0, n) from 32 random bits.
__host__ __device__ __forceinline__ int32_t below(uint32_t u, uint32_t n) {
  return (int32_t)(((uint64_t)u * n) >> 32);
}

// State is a struct of int32 fields, stored as one int32 [E] array per field: field i of stream e at st[i * E + e].
template <typename State>
__device__ __forceinline__ State load_state(const int32_t* st, int E, int e) {
  State s;
  int32_t* f = reinterpret_cast<int32_t*>(&s);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(State) / sizeof(int32_t)); ++i) f[i] = st[i * E + e];
  return s;
}

template <typename State>
__device__ __forceinline__ void store_state(const State& s, int32_t* st, int E, int e) {
  const int32_t* f = reinterpret_cast<const int32_t*>(&s);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(State) / sizeof(int32_t)); ++i) st[i * E + e] = f[i];
}

// The 16 bytes of a word whose first byte is channel K of pixel 0 of rgb[0..5] (packed 0x00BBGGRR colours).
template <int K>
__device__ __forceinline__ uint4 pack_word(const uint32_t (&rgb)[6]) {
  uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int b = 0; b < 16; ++b) w[b >> 2] |= ((rgb[(K + b) / 3] >> (8 * ((K + b) % 3))) & 0xFFu) << (8 * (b & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// The checks of a game's configuration; "dz_<game>" prefixes the messages, actions must lie in [min_actions, 18].
inline int check_game_config(const dz_game_config* cfg, const char* game, int max_streams, int min_actions,
                             int max_noop_steps) {
  if (!cfg) return fail(DZ_EINVAL, "dz_%s: null config", game);
  if (cfg->num_streams < 1 || cfg->num_streams > max_streams)
    return fail(DZ_EINVAL, "dz_%s: num_streams must be in [1, %s]", game, std::to_string(max_streams).c_str());
  if (cfg->num_actions < min_actions || cfg->num_actions > 18)
    return fail(DZ_EINVAL, "dz_%s: num_actions must be in [%s, 18]", game, std::to_string(min_actions).c_str());
  if (cfg->min_noop_steps < 0 || cfg->min_noop_steps > cfg->max_noop_steps || cfg->max_noop_steps > max_noop_steps)
    return fail(DZ_EINVAL, "dz_%s: no-op steps must satisfy 0 <= min <= max <= %s", game,
                std::to_string(max_noop_steps).c_str());
  if ((uint64_t)cfg->stream_offset + (uint64_t)cfg->num_streams > (1ull << 32))
    return fail(DZ_EINVAL, "dz_%s: stream_offset + num_streams must be <= 2^32", game);
  return DZ_OK;
}

template <typename G>
int check_config(const dz_game_config* cfg) {
  return check_game_config(cfg, G::kName, G::kMaxStreams, G::kMinActions, G::kMaxNoopSteps);
}

// A tick of one stream: a reset (asked for, or after the episode's LAST step) or one frame with `action`.  Stream
// `stream`'s key is threefry2x32((0, seed), (stream, kTag)); a reset draws its no-op count from (counter, 0).
template <typename G>
__host__ __device__ __forceinline__ GameStep game_tick(typename G::State& s, const dz_game_config& cfg,
                                                       uint32_t stream, int32_t action, bool reset) {
  uint32_t k0, k1;
  threefry2x32(0u, cfg.seed, stream, G::kTag, &k0, &k1);
  if (reset || s.over) {
    uint32_t o0, o1;
    threefry2x32(k0, k1, (uint32_t)s.counter, 0u, &o0, &o1);
    s.counter += 1;
    const int32_t k = cfg.min_noop_steps + below(o0, (uint32_t)(cfg.max_noop_steps - cfg.min_noop_steps + 1));
    G::start(s, k0, k1);
    s.over = 0;
    for (int32_t i = 0; i < k; ++i) G::frame(s, 0, k0, k1);   // kMaxNoopSteps keeps their rewards 0
    s.noops = k;
    return {0, 0, 0, G::lives(s)};
  }
  const int32_t r = G::frame(s, action, k0, k1);
  s.over = G::over(s);
  return {s.over ? 2 : 1, r, s.over ? 0 : 1, G::lives(s)};
}

// A CTA per stream.  Thread 0 ticks the stream (kStep) and writes its record; the CTA then writes the stream's frame
// with aligned 16-byte stores.
template <typename G, bool kStep>
__global__ void __launch_bounds__(kGameThreads) game_kernel(const dz_game_config cfg, int32_t* __restrict__ state,
                                                            const int32_t* __restrict__ control,
                                                            uint8_t* __restrict__ frames,
                                                            int32_t* __restrict__ record) {
  using State = typename G::State;
  dz::pdl_enter();
  __shared__ State s_state;
  const int E = cfg.num_streams, e = blockIdx.x;
  if (threadIdx.x == 0) {
    State s = load_state<State>(state, E, e);
    if (kStep) {
      const GameStep r = game_tick<G>(s, cfg, cfg.stream_offset + (uint32_t)e, control[e], control[E + e] != 0);
      store_state(s, state, E, e);
      record[e] = r.step_type;
      record[E + e] = r.reward;
      record[2 * E + e] = r.discount;
      record[3 * E + e] = r.lives;
    }
    s_state = s;
  }
  __syncthreads();
  const State s = s_state;
  const uint32_t bg[6] = {G::kBackground, G::kBackground, G::kBackground, G::kBackground, G::kBackground,
                          G::kBackground};
  const uint4 bg0 = pack_word<0>(bg), bg1 = pack_word<1>(bg), bg2 = pack_word<2>(bg);
  uint4* out = reinterpret_cast<uint4*>(frames + (int64_t)e * kFrameBytes);
  for (int i = threadIdx.x; i < kFrameH * kRowWords; i += kGameThreads) {
    const int y = i / kRowWords, b0 = 16 * (i - y * kRowWords);
    const int xa = b0 / 3, xb = (b0 + 15) / 3;           // the word covers pixels xa..xb (at most 6)
    // The channel of the word's first byte, k = b0 - 3 xa, is formed in each branch: formed above the test it costs
    // Breakout's step kernel 3 more registers (43).
    uint4 v;
    if (G::span_has_object(s, y, xa, xb)) {
      uint32_t rgb[6];
#pragma unroll
      for (int p = 0; p < 6; ++p) rgb[p] = xa + p <= xb ? G::rgb(s, xa + p, y) : 0u;
      const int k = b0 - 3 * xa;
      v = k == 0 ? pack_word<0>(rgb) : k == 1 ? pack_word<1>(rgb) : pack_word<2>(rgb);
    } else {
      const int k = b0 - 3 * xa;
      v = k == 0 ? bg0 : k == 1 ? bg1 : bg2;
    }
    out[i] = v;
  }
}

// dz_<game>_step: checks, then on `stream` the pinned control in, one launch, the pinned record out.
template <typename G>
int game_step(const dz_game_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
              uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  static const std::string name = std::string(G::kName) + "_kernel<true>";
  DZ_TRY(check_config<G>(cfg));
  if (!d_state || !h_control || !d_control || !d_frames || !d_record || !h_record)
    return fail(DZ_EINVAL, "dz_%s_step: null pointer", G::kName);
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_%s_step: d_frames must be 16-byte aligned", G::kName);
  const int E = cfg->num_streams;
  for (int e = 0; e < E; ++e)
    if (!h_control[E + e] && (h_control[e] < 0 || h_control[e] >= cfg->num_actions))
      return fail(DZ_EINVAL, "dz_%s_step: an action is outside [0, num_actions)", G::kName);
  const cudaStream_t s = (cudaStream_t)stream;
  DZ_CUDA_OK(cudaMemcpyAsync(d_control, h_control, 2 * E * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DZ_LAUNCH_NAMED(name.c_str(), (game_kernel<G, true>), E, kGameThreads, 0, stream, *cfg, d_state, d_control,
                  d_frames, d_record);
  DZ_CUDA_OK(cudaMemcpyAsync(h_record, d_record, E * sizeof(GameStep), cudaMemcpyDeviceToHost, s));
  return DZ_OK;
}

// dz_<game>_render: every stream's frame from d_state, which is not changed.
template <typename G>
int game_render(const dz_game_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  static const std::string name = std::string(G::kName) + "_kernel<false>";
  DZ_TRY(check_config<G>(cfg));
  if (!d_state || !d_frames) return fail(DZ_EINVAL, "dz_%s_render: null pointer", G::kName);
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_%s_render: d_frames must be 16-byte aligned", G::kName);
  DZ_LAUNCH_NAMED(name.c_str(), (game_kernel<G, false>), cfg->num_streams, kGameThreads, 0, stream, *cfg, d_state,
                  (const int32_t*)nullptr, d_frames, (int32_t*)nullptr);
  return DZ_OK;
}

// dz_test_<game>_step: the kernel's tick and picture compiled for the host, on stream cfg->stream_offset.
template <typename G>
int game_host_step(const dz_game_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                   int32_t* record) {
  if (!cfg || !state || !record) return fail(DZ_EINVAL, "dz_test_%s_step: null pointer", G::kName);
  dz_game_config one = *cfg;
  one.num_streams = 1;
  DZ_TRY(check_config<G>(&one));
  if (!reset && (action < 0 || action >= cfg->num_actions))
    return fail(DZ_EINVAL, "dz_test_%s_step: action outside [0, num_actions)", G::kName);
  typename G::State s;
  memcpy(&s, state, sizeof(s));
  const GameStep r = game_tick<G>(s, one, one.stream_offset, action, reset != 0);
  memcpy(state, &s, sizeof(s));
  record[0] = r.step_type; record[1] = r.reward; record[2] = r.discount; record[3] = r.lives;
  if (frame)
    for (int y = 0; y < kFrameH; ++y)
      for (int x = 0; x < kFrameW; ++x) {
        const uint32_t rgb = G::rgb(s, x, y);
        for (int c = 0; c < 3; ++c) frame[(y * kFrameW + x) * 3 + c] = (uint8_t)(rgb >> (8 * c));
      }
  return DZ_OK;
}

}  // namespace dz
