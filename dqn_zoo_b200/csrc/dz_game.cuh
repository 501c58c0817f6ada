// Pieces shared by the device games that draw 210x160 RGB frames with aligned 16-byte stores (dz_breakout.cu,
// dz_pong.cu): the uniform draw, the int32 [fields][E] state load and store, the 16-byte word packer, and the common
// part of the configuration check.
#pragma once
#include <string>

#include "dz_common.cuh"

namespace dz {

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

// The checks every game's configuration (num_streams, num_actions, min/max_noop_steps, seed, stream_offset) shares;
// `game` prefixes the messages, actions must lie in [min_actions, 18].
template <typename Config>
int check_game_config(const Config* cfg, const char* game, int max_streams, int min_actions, int max_noop_steps) {
  if (!cfg) return fail(DZ_EINVAL, "%s: null config", game);
  if (cfg->num_streams < 1 || cfg->num_streams > max_streams)
    return fail(DZ_EINVAL, "%s: num_streams must be in [1, %s]", game, std::to_string(max_streams).c_str());
  if (cfg->num_actions < min_actions || cfg->num_actions > 18)
    return fail(DZ_EINVAL, "%s: num_actions must be in [%s, 18]", game, std::to_string(min_actions).c_str());
  if (cfg->min_noop_steps < 0 || cfg->min_noop_steps > cfg->max_noop_steps || cfg->max_noop_steps > max_noop_steps)
    return fail(DZ_EINVAL, "%s: no-op steps must satisfy 0 <= min <= max <= %s", game,
                std::to_string(max_noop_steps).c_str());
  if ((uint64_t)cfg->stream_offset + (uint64_t)cfg->num_streams > (1ull << 32))
    return fail(DZ_EINVAL, "%s: stream_offset + num_streams must be <= 2^32", game);
  return DZ_OK;
}

}  // namespace dz
