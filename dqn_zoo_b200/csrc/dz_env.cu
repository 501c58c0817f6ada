// Catch at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §10).
//
// One launch per tick: a CTA per stream.  Thread 0 applies the stream's action (or a reset with its random no-op
// frames) to the stream's state, the CTA then writes the stream's whole 210x160x3 RGB frame with aligned 16-byte stores,
// and CTA e's record gets step_type / reward / discount / lives.  The rules live in catch_reset / catch_frame /
// catch_tick and the picture in catch_byte; the kernel and the host twin (dz_test_catch_step) run the same functions,
// and oracle/catch_oracle.py restates them in numpy.
//
// State: int32 [DZ_CATCH_STATE_FIELDS][E] (one array per field, in the order of CatchState).  Randomness is
// counter-based: stream e's key is threefry2x32((0, seed), (stream_offset + e, 0)); a reset draws its no-op count from
// threefry2x32(key, (counter, 0)) and a ball its x and dx from threefry2x32(key, (counter, 1)), each advancing counter.
#include "dz_common.cuh"
#include "dz_threefry.cuh"

namespace dz {

namespace {

constexpr int kH = DZ_CATCH_HEIGHT, kW = DZ_CATCH_WIDTH;
constexpr int kRowBytes = 3 * kW;                         // 480: 30 16-byte words
constexpr int kRowWords = kRowBytes / 16;
constexpr int kFrameBytes = kH * kRowBytes;               // 100,800
constexpr int kPaddleW = 16, kPaddleH = 4, kPaddleY = 188, kPaddleMaxX = kW - kPaddleW, kPaddleStep = 3;
constexpr int kBall = 8, kBallMaxX = kW - kBall, kBallFall = 2, kLandY = kPaddleY - kBall;   // 152, lands at y = 180
constexpr int kLives = 3, kBallsPerEpisode = 20;
constexpr int kLivesY = 4, kLivesH = 6, kLivesX = 8, kLivesPitch = 12, kLivesW = 8;
constexpr int kThreads = 256;
static_assert(kRowBytes % 16 == 0, "rows are whole 16-byte words");
static_assert(kLandY % kBallFall == 0, "the ball reaches its landing row exactly");
static_assert(DZ_CATCH_MAX_NOOP_STEPS < kLandY / kBallFall, "no ball lands during the no-op frames of a reset");

// Channel c of the RGB of the background (24, 26, 167), the paddle (200, 72, 72), the ball (236, 236, 236) and the life
// blocks (92, 186, 92), packed 0x00BBGGRR.
__host__ __device__ __forceinline__ uint8_t catch_colour(int object, int c) {
  const uint32_t rgb = object == 0 ? 0xA71A18u : object == 1 ? 0x4848C8u : object == 2 ? 0xECECECu : 0x5CBA5Cu;
  return (uint8_t)(rgb >> (8 * c));
}

struct CatchState {   // the field order of the state arrays
  int32_t paddle_x, ball_x, ball_y, ball_dx, lives, balls_left, counter, noops, over;
};
static_assert(sizeof(CatchState) == DZ_CATCH_STATE_FIELDS * sizeof(int32_t), "one int32 per field");

struct Step { int32_t step_type, reward, discount, lives; };

// floor(u * n / 2^32): a uniform draw in [0, n) from 32 random bits.
__host__ __device__ __forceinline__ int32_t draw_below(uint32_t u, uint32_t n) {
  return (int32_t)(((uint64_t)u * n) >> 32);
}

__host__ __device__ __forceinline__ void catch_spawn(CatchState& s, uint32_t k0, uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 1u, &o0, &o1);
  s.counter += 1;
  s.ball_x = draw_below(o0, kBallMaxX + 1);
  s.ball_dx = draw_below(o1, 3) - 1;
  s.ball_y = 0;
}

// One frame of the game; returns its reward.
__host__ __device__ __forceinline__ int32_t catch_frame(CatchState& s, int32_t action, uint32_t k0, uint32_t k1) {
  if (action == 1) s.paddle_x = s.paddle_x - kPaddleStep < 0 ? 0 : s.paddle_x - kPaddleStep;
  if (action == 2) s.paddle_x = s.paddle_x + kPaddleStep > kPaddleMaxX ? kPaddleMaxX : s.paddle_x + kPaddleStep;
  if (s.ball_y >= kLandY) {              // the ball landed on the previous frame: a new one
    catch_spawn(s, k0, k1);
    return 0;
  }
  s.ball_y += kBallFall;
  s.ball_x += s.ball_dx;
  if (s.ball_x < 0) { s.ball_x = -s.ball_x; s.ball_dx = -s.ball_dx; }
  if (s.ball_x > kBallMaxX) { s.ball_x = 2 * kBallMaxX - s.ball_x; s.ball_dx = -s.ball_dx; }
  if (s.ball_y != kLandY) return 0;
  s.balls_left -= 1;
  if (s.ball_x < s.paddle_x + kPaddleW && s.ball_x + kBall > s.paddle_x) return 1;
  s.lives -= 1;
  return -1;
}

__host__ __device__ __forceinline__ void catch_reset(CatchState& s, const dz_catch_config& cfg, uint32_t k0, uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 0u, &o0, &o1);
  s.counter += 1;
  const int32_t k = cfg.min_noop_steps + draw_below(o0, (uint32_t)(cfg.max_noop_steps - cfg.min_noop_steps + 1));
  s.paddle_x = kPaddleMaxX / 2;
  s.lives = kLives;
  s.balls_left = kBallsPerEpisode;
  s.over = 0;
  catch_spawn(s, k0, k1);
  for (int32_t i = 0; i < k; ++i) catch_frame(s, 0, k0, k1);   // no landing: their rewards are all 0
  s.noops = k;
}

// A tick of one stream: a reset (asked for, or after the episode's LAST step) or one frame with `action`.
__host__ __device__ __forceinline__ Step catch_tick(CatchState& s, const dz_catch_config& cfg, uint32_t stream,
                                                    int32_t action, bool reset) {
  uint32_t k0, k1;
  threefry2x32(0u, cfg.seed, stream, 0u, &k0, &k1);
  if (reset || s.over) {
    catch_reset(s, cfg, k0, k1);
    return {0, 0, 0, s.lives};
  }
  const int32_t r = catch_frame(s, action, k0, k1);
  s.over = s.lives == 0 || s.balls_left == 0;
  return {s.over ? 2 : 1, r, s.over ? 0 : 1, s.lives};
}

// Which object covers pixel (x, y): 0 background, 1 paddle, 2 ball (drawn last), 3 a life block.
__host__ __device__ __forceinline__ int catch_object(const CatchState& s, int x, int y) {
  if (y >= s.ball_y && y < s.ball_y + kBall && x >= s.ball_x && x < s.ball_x + kBall) return 2;
  if (y >= kPaddleY && y < kPaddleY + kPaddleH && x >= s.paddle_x && x < s.paddle_x + kPaddleW) return 1;
  if (y >= kLivesY && y < kLivesY + kLivesH && x >= kLivesX) {
    const int i = (x - kLivesX) / kLivesPitch;
    if (i < s.lives && x - kLivesX - i * kLivesPitch < kLivesW) return 3;
  }
  return 0;
}

__host__ __device__ __forceinline__ uint8_t catch_byte(const CatchState& s, int x, int y, int c) {
  return catch_colour(catch_object(s, x, y), c);
}

__device__ __forceinline__ CatchState load_state(const int32_t* st, int E, int e) {
  return {st[e], st[E + e], st[2 * E + e], st[3 * E + e], st[4 * E + e], st[5 * E + e], st[6 * E + e], st[7 * E + e],
          st[8 * E + e]};
}

__device__ __forceinline__ void store_state(const CatchState& s, int32_t* st, int E, int e) {
  st[e] = s.paddle_x; st[E + e] = s.ball_x; st[2 * E + e] = s.ball_y; st[3 * E + e] = s.ball_dx;
  st[4 * E + e] = s.lives; st[5 * E + e] = s.balls_left; st[6 * E + e] = s.counter; st[7 * E + e] = s.noops;
  st[8 * E + e] = s.over;
}

// The background's 16-byte word k of every 3 (48 bytes = 16 pixels: the pattern's period).
__device__ __forceinline__ uint4 background_word(int k) {
  uint32_t w[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    w[q] = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) w[q] |= (uint32_t)catch_colour(0, (16 * k + 4 * q + b) % 3) << (8 * b);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Can an object touch the 16 bytes at row y, bytes [b0, b0 + 16) of the row?  Conservative: false means background.
__device__ __forceinline__ bool word_has_object(const CatchState& s, int y, int b0) {
  const int xa = b0 / 3, xb = (b0 + 15) / 3;
  if (y >= s.ball_y && y < s.ball_y + kBall && xb >= s.ball_x && xa < s.ball_x + kBall) return true;
  if (y >= kPaddleY && y < kPaddleY + kPaddleH && xb >= s.paddle_x && xa < s.paddle_x + kPaddleW) return true;
  return y >= kLivesY && y < kLivesY + kLivesH && s.lives > 0 && xb >= kLivesX &&
         xa < kLivesX + (s.lives - 1) * kLivesPitch + kLivesW;
}

template <bool kStep>
__global__ void __launch_bounds__(kThreads) catch_kernel(const dz_catch_config cfg, int32_t* __restrict__ state,
                                                         const int32_t* __restrict__ control,
                                                         uint8_t* __restrict__ frames, int32_t* __restrict__ record) {
  dz::pdl_enter();
  __shared__ CatchState s_state;
  const int E = cfg.num_streams, e = blockIdx.x;
  if (threadIdx.x == 0) {
    CatchState s = load_state(state, E, e);
    if (kStep) {
      const Step r = catch_tick(s, cfg, cfg.stream_offset + (uint32_t)e, control[e], control[E + e] != 0);
      store_state(s, state, E, e);
      record[e] = r.step_type;
      record[E + e] = r.reward;
      record[2 * E + e] = r.discount;
      record[3 * E + e] = r.lives;
    }
    s_state = s;
  }
  __syncthreads();
  const CatchState s = s_state;
  const uint4 bg0 = background_word(0), bg1 = background_word(1), bg2 = background_word(2);
  uint4* out = reinterpret_cast<uint4*>(frames + (int64_t)e * kFrameBytes);
  for (int i = threadIdx.x; i < kH * kRowWords; i += kThreads) {
    const int y = i / kRowWords, cw = i - y * kRowWords, b0 = 16 * cw;
    const int k = cw % 3;
    uint4 v = k == 0 ? bg0 : k == 1 ? bg1 : bg2;
    if (word_has_object(s, y, b0)) {
      uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
      for (int b = 0; b < 16; ++b) w[b >> 2] |= (uint32_t)catch_byte(s, (b0 + b) / 3, y, (b0 + b) % 3) << (8 * (b & 3));
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    out[i] = v;
  }
}

int check_config(const dz_catch_config* cfg) {
  if (!cfg) return fail(DZ_EINVAL, "dz_catch: null config");
  if (cfg->num_streams < 1 || cfg->num_streams > DZ_CATCH_MAX_STREAMS)
    return fail(DZ_EINVAL, "dz_catch: num_streams must be in [1, 4096]");
  if (cfg->num_actions < 3 || cfg->num_actions > 18) return fail(DZ_EINVAL, "dz_catch: num_actions must be in [3, 18]");
  if (cfg->min_noop_steps < 0 || cfg->min_noop_steps > cfg->max_noop_steps ||
      cfg->max_noop_steps > DZ_CATCH_MAX_NOOP_STEPS)
    return fail(DZ_EINVAL, "dz_catch: no-op steps must satisfy 0 <= min <= max <= 89");
  if ((uint64_t)cfg->stream_offset + (uint64_t)cfg->num_streams > (1ull << 32))
    return fail(DZ_EINVAL, "dz_catch: stream_offset + num_streams must be <= 2^32");
  return DZ_OK;
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_catch_step(const dz_catch_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                  uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !h_control || !d_control || !d_frames || !d_record || !h_record)
    return fail(DZ_EINVAL, "dz_catch_step: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_catch_step: d_frames must be 16-byte aligned");
  const int E = cfg->num_streams;
  for (int e = 0; e < E; ++e)
    if (!h_control[E + e] && (h_control[e] < 0 || h_control[e] >= cfg->num_actions))
      return fail(DZ_EINVAL, "dz_catch_step: an action is outside [0, num_actions)");
  const cudaStream_t s = (cudaStream_t)stream;
  DZ_CUDA_OK(cudaMemcpyAsync(d_control, h_control, 2 * E * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DZ_LAUNCH(catch_kernel<true>, E, kThreads, 0, stream, *cfg, d_state, d_control, d_frames, d_record);
  DZ_CUDA_OK(cudaMemcpyAsync(h_record, d_record, DZ_CATCH_RECORD_FIELDS * E * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  return DZ_OK;
}

int dz_catch_render(const dz_catch_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !d_frames) return fail(DZ_EINVAL, "dz_catch_render: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_catch_render: d_frames must be 16-byte aligned");
  DZ_LAUNCH(catch_kernel<false>, cfg->num_streams, kThreads, 0, stream, *cfg, d_state, (const int32_t*)nullptr, d_frames,
            (int32_t*)nullptr);
  return DZ_OK;
}

// The kernel's tick and picture compiled for the host: stream cfg->stream_offset, one state of DZ_CATCH_STATE_FIELDS
// int32 updated in place; frame (may be NULL) gets the 210x160x3 bytes, record the step_type / reward / discount / lives.
int dz_test_catch_step(const dz_catch_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                       int32_t* record) {
  if (!cfg || !state || !record) return fail(DZ_EINVAL, "dz_test_catch_step: null pointer");
  dz_catch_config one = *cfg;
  one.num_streams = 1;
  DZ_TRY(check_config(&one));
  if (!reset && (action < 0 || action >= cfg->num_actions))
    return fail(DZ_EINVAL, "dz_test_catch_step: action outside [0, num_actions)");
  CatchState s;
  memcpy(&s, state, sizeof(s));
  const Step r = catch_tick(s, one, one.stream_offset, action, reset != 0);
  memcpy(state, &s, sizeof(s));
  record[0] = r.step_type; record[1] = r.reward; record[2] = r.discount; record[3] = r.lives;
  if (frame)
    for (int y = 0; y < kH; ++y)
      for (int x = 0; x < kW; ++x)
        for (int c = 0; c < 3; ++c) frame[(y * kW + x) * 3 + c] = catch_byte(s, x, y, c);
  return DZ_OK;
}

}  // extern "C"
