// Breakout at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §11).
//
// The project's own game, not ALE Breakout: a 6 x 18 brick wall worth 7 / 4 / 1 points per row, a paddle, a 4x4 ball
// that is served by FIRE (or a serve timer), 5 lives.  One launch per tick: a CTA per stream.  Thread 0 applies the
// stream's action (or a reset with its random no-op frames) to the stream's state, the CTA then writes the stream's
// whole 210x160x3 RGB frame with aligned 16-byte stores, and CTA e's record gets step_type / reward / discount / lives.
// The rules live in breakout_reset / breakout_frame / breakout_tick and the picture in breakout_rgb; the kernel and the
// host twin (dz_test_breakout_step) run the same functions, and oracle/breakout_oracle.py restates them in numpy.
//
// State: int32 [DZ_BREAKOUT_STATE_FIELDS][E] (one array per field, in the order of BreakoutState); the wall is six
// 18-bit row masks (bit c of row r: brick (r, c) is still there).  Randomness is counter-based: stream e's key is
// threefry2x32((0, seed), (stream_offset + e, 1)) (the 1 tags the game: Catch keys with 0); a reset draws its no-op
// count from threefry2x32(key, (counter, 0)) and a serve its x and dx from threefry2x32(key, (counter, 1)), each
// advancing counter.
#include "dz_game.cuh"
#include "dz_threefry.cuh"

namespace dz {

namespace {

constexpr int kH = DZ_BREAKOUT_HEIGHT, kW = DZ_BREAKOUT_WIDTH;
constexpr int kRowBytes = 3 * kW;                         // 480: 30 16-byte words
constexpr int kRowWords = kRowBytes / 16;
constexpr int kFrameBytes = kH * kRowBytes;               // 100,800
constexpr uint32_t kGameTag = 1;                           // the second counter word of the stream key
// Field: x in [8, 152), y in [25, 196); walls: top y in [17, 25) over the whole width, sides x < 8 and x >= 152 for
// y in [17, 196).
constexpr int kWallTop = 17, kFieldTop = 25, kFieldBottom = 196, kFieldLeft = 8, kFieldRight = 152;
constexpr int kRows = DZ_BREAKOUT_BRICK_ROWS, kCols = DZ_BREAKOUT_BRICK_COLS;
constexpr int kBrickW = 8, kBrickH = 6, kBrickY = 57, kBrickBottom = kBrickY + kRows * kBrickH;   // bricks y in [57, 93)
constexpr uint32_t kFullRow = (1u << kCols) - 1;
constexpr int kPaddleW = 16, kPaddleH = 4, kPaddleY = 189, kPaddleMinX = kFieldLeft,
              kPaddleMaxX = kFieldRight - kPaddleW, kPaddleStep = 4;                                // x in [8, 136]
constexpr int kBall = 4, kBallMinX = kFieldLeft, kBallMaxX = kFieldRight - kBall, kServeY = 100;    // x in [8, 148]
constexpr int kServeDelay = 64, kLives = 5;
constexpr int kLivesY = 4, kLivesH = 6, kLivesX = 8, kLivesPitch = 12, kLivesW = 8;
constexpr int kThreads = 256;
enum { kNoop = 0, kFire = 1, kRight = 2, kLeft = 3 };
static_assert(kRowBytes % 16 == 0, "rows are whole 16-byte words");
static_assert(DZ_BREAKOUT_MAX_NOOP_STEPS < kServeDelay, "no ball is served during the no-op frames of a reset");
static_assert(kFieldLeft + kCols * kBrickW == kFieldRight, "the wall spans the field");
static_assert(kServeY > kBrickBottom && kServeY + kBall < kPaddleY, "a served ball touches no brick and no paddle");

// Packed 0x00BBGGRR colours: background black, walls and life blocks grey, bricks by row, paddle, ball.
constexpr uint32_t kBackground = 0x000000u, kGrey = 0x8E8E8Eu, kPaddleRgb = 0x4848C8u, kBallRgb = 0xECECECu;
__host__ __device__ __forceinline__ uint32_t brick_rgb(int r) {
  return r == 0 ? 0x4848C8u : r == 1 ? 0x3A6CC6u : r == 2 ? 0x307AB4u : r == 3 ? 0x2AA2A2u : r == 4 ? 0x48A048u
                                                                                                     : 0xC84842u;
}
__host__ __device__ __forceinline__ int32_t brick_points(int r) { return r < 2 ? 7 : r < 4 ? 4 : 1; }

struct BreakoutState {   // the field order of the state arrays
  int32_t paddle_x, ball_x, ball_y, ball_dx, ball_dy, in_play, serve_timer, lives;
  int32_t row[kRows];
  int32_t counter, noops, over;
};
static_assert(sizeof(BreakoutState) == DZ_BREAKOUT_STATE_FIELDS * sizeof(int32_t), "one int32 per field");

struct Step { int32_t step_type, reward, discount, lives; };

__host__ __device__ __forceinline__ void breakout_serve(BreakoutState& s, uint32_t k0, uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 1u, &o0, &o1);
  s.counter += 1;
  s.ball_x = kBallMinX + below(o0, kBallMaxX - kBallMinX + 1);
  const int32_t d = below(o1, 4);                          // dx in {-2, -1, +1, +2}
  s.ball_dx = d < 2 ? d - 2 : d - 1;
  s.ball_y = kServeY;
  s.ball_dy = 2;
  s.in_play = 1;
}

// Row r's brick mask by a select chain rather than an indexed load, so the state stays in registers.
__host__ __device__ __forceinline__ uint32_t row_mask(const BreakoutState& s, int r) {
  return (uint32_t)(r == 0 ? s.row[0] : r == 1 ? s.row[1] : r == 2 ? s.row[2] : r == 3 ? s.row[3] : r == 4 ? s.row[4]
                                                                                                   : s.row[5]);
}

// Clears the first live brick the ball overlaps (bottom row first, then left column); returns its points or 0.
__host__ __device__ __forceinline__ int32_t breakout_hit_brick(BreakoutState& s) {
  if (s.ball_y + kBall <= kBrickY || s.ball_y >= kBrickBottom) return 0;
  const int r0 = s.ball_y < kBrickY ? 0 : (s.ball_y - kBrickY) / kBrickH;
  const int r1 = s.ball_y + kBall - 1 >= kBrickBottom ? kRows - 1 : (s.ball_y + kBall - 1 - kBrickY) / kBrickH;
  const int c0 = (s.ball_x - kFieldLeft) / kBrickW, c1 = (s.ball_x + kBall - 1 - kFieldLeft) / kBrickW;
  int hit_r = -1, hit_c = 0;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {      // the last match wins: the bottom row, then its left column
    if (r < r0 || r > r1) continue;
    if ((s.row[r] >> c1) & 1) { hit_r = r; hit_c = c1; }
    if ((s.row[r] >> c0) & 1) { hit_r = r; hit_c = c0; }
  }
  if (hit_r < 0) return 0;
#pragma unroll
  for (int r = 0; r < kRows; ++r)
    if (r == hit_r) s.row[r] &= ~(1 << hit_c);
  s.ball_dy = -s.ball_dy;
  if (hit_r < 2 && (s.ball_dy == 2 || s.ball_dy == -2)) s.ball_dy = s.ball_dy > 0 ? 3 : -3;
  return brick_points(hit_r);
}

// One frame of the game; returns its reward.
__host__ __device__ __forceinline__ int32_t breakout_frame(BreakoutState& s, int32_t action, uint32_t k0, uint32_t k1) {
  if (action == kRight) s.paddle_x = s.paddle_x + kPaddleStep > kPaddleMaxX ? kPaddleMaxX : s.paddle_x + kPaddleStep;
  if (action == kLeft) s.paddle_x = s.paddle_x - kPaddleStep < kPaddleMinX ? kPaddleMinX : s.paddle_x - kPaddleStep;
  if (!s.in_play) {
    s.serve_timer -= 1;
    if (action == kFire || s.serve_timer <= 0) breakout_serve(s, k0, k1);
    return 0;
  }
  s.ball_x += s.ball_dx;
  if (s.ball_x < kBallMinX) { s.ball_x = 2 * kBallMinX - s.ball_x; s.ball_dx = -s.ball_dx; }
  if (s.ball_x > kBallMaxX) { s.ball_x = 2 * kBallMaxX - s.ball_x; s.ball_dx = -s.ball_dx; }
  const int32_t y0 = s.ball_y;
  s.ball_y += s.ball_dy;
  if (s.ball_y < kFieldTop) { s.ball_y = 2 * kFieldTop - s.ball_y; s.ball_dy = -s.ball_dy; }
  const int32_t reward = breakout_hit_brick(s);
  // A falling ball whose bottom crosses the paddle's top row this frame while it overlaps the paddle bounces.
  if (s.ball_dy > 0 && y0 + kBall <= kPaddleY && s.ball_y + kBall > kPaddleY && s.ball_x < s.paddle_x + kPaddleW &&
      s.ball_x + kBall > s.paddle_x) {
    s.ball_y = kPaddleY - kBall;
    s.ball_dy = -s.ball_dy;
    const int32_t zone = 4 * (s.ball_x - s.paddle_x + kBall - 1) / (kPaddleW + kBall - 1);   // offset in [0, 18]
    s.ball_dx = zone < 2 ? zone - 2 : zone - 1;
  }
  if (s.ball_y >= kFieldBottom) {          // out of the field: a life less, no reward
    s.in_play = 0;
    s.lives -= 1;
    s.serve_timer = kServeDelay;
  }
  return reward;
}

__host__ __device__ __forceinline__ void breakout_reset(BreakoutState& s, const dz_breakout_config& cfg, uint32_t k0,
                                                        uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 0u, &o0, &o1);
  s.counter += 1;
  const int32_t k = cfg.min_noop_steps + below(o0, (uint32_t)(cfg.max_noop_steps - cfg.min_noop_steps + 1));
  s.paddle_x = (kPaddleMinX + kPaddleMaxX) / 2;
  s.ball_x = s.ball_y = s.ball_dx = s.ball_dy = 0;
  s.in_play = 0;
  s.serve_timer = kServeDelay;
  s.lives = kLives;
#pragma unroll
  for (int r = 0; r < kRows; ++r) s.row[r] = kFullRow;
  s.over = 0;
  for (int32_t i = 0; i < k; ++i) breakout_frame(s, kNoop, k0, k1);   // no serve: the timer stays above 0
  s.noops = k;
}

// A tick of one stream: a reset (asked for, or after the episode's LAST step) or one frame with `action`.
__host__ __device__ __forceinline__ Step breakout_tick(BreakoutState& s, const dz_breakout_config& cfg, uint32_t stream,
                                                       int32_t action, bool reset) {
  uint32_t k0, k1;
  threefry2x32(0u, cfg.seed, stream, kGameTag, &k0, &k1);
  if (reset || s.over) {
    breakout_reset(s, cfg, k0, k1);
    return {0, 0, 0, s.lives};
  }
  const int32_t r = breakout_frame(s, action, k0, k1);
  int32_t bricks = 0;
#pragma unroll
  for (int i = 0; i < kRows; ++i) bricks |= s.row[i];
  s.over = s.lives == 0 || bricks == 0;
  return {s.over ? 2 : 1, r, s.over ? 0 : 1, s.lives};
}

// The colour of pixel (x, y), objects in drawing order: background, walls, life blocks, bricks, paddle, ball.
__host__ __device__ __forceinline__ uint32_t breakout_rgb(const BreakoutState& s, int x, int y) {
  if (s.in_play && y >= s.ball_y && y < s.ball_y + kBall && x >= s.ball_x && x < s.ball_x + kBall) return kBallRgb;
  if (y >= kPaddleY && y < kPaddleY + kPaddleH && x >= s.paddle_x && x < s.paddle_x + kPaddleW) return kPaddleRgb;
  if (y >= kBrickY && y < kBrickBottom && x >= kFieldLeft && x < kFieldRight) {
    const int r = (y - kBrickY) / kBrickH;
    if ((row_mask(s, r) >> ((x - kFieldLeft) / kBrickW)) & 1) return brick_rgb(r);
  }
  if (y >= kWallTop && y < kFieldTop) return kGrey;
  if (y >= kWallTop && y < kFieldBottom && (x < kFieldLeft || x >= kFieldRight)) return kGrey;
  if (y >= kLivesY && y < kLivesY + kLivesH && x >= kLivesX) {
    const int i = (x - kLivesX) / kLivesPitch;
    if (i < s.lives && x - kLivesX - i * kLivesPitch < kLivesW) return kGrey;
  }
  return kBackground;
}

// Can an object touch pixels [xa, xb] of row y?  Conservative: false means background.  In the wall's rows the test is
// against the row's brick mask, so the cleared part of the wall is written as background.
__device__ __forceinline__ bool span_has_object(const BreakoutState& s, int y, int xa, int xb) {
  if (s.in_play && y >= s.ball_y && y < s.ball_y + kBall && xb >= s.ball_x && xa < s.ball_x + kBall) return true;
  if (y >= kPaddleY && y < kPaddleY + kPaddleH && xb >= s.paddle_x && xa < s.paddle_x + kPaddleW) return true;
  if (y >= kWallTop && y < kFieldTop) return true;
  if (y >= kWallTop && y < kFieldBottom && (xa < kFieldLeft || xb >= kFieldRight)) return true;
  if (y >= kBrickY && y < kBrickBottom) {
    const uint32_t mask = row_mask(s, (y - kBrickY) / kBrickH);
    const int c0 = (xa - kFieldLeft) / kBrickW, c1 = (xb - kFieldLeft) / kBrickW;   // xa, xb in the field here
    return (mask >> c0) & ((2u << (c1 - c0)) - 1u);
  }
  return y >= kLivesY && y < kLivesY + kLivesH && s.lives > 0 && xb >= kLivesX &&
         xa < kLivesX + (s.lives - 1) * kLivesPitch + kLivesW;
}

template <bool kStep>
__global__ void __launch_bounds__(kThreads) breakout_kernel(const dz_breakout_config cfg, int32_t* __restrict__ state,
                                                            const int32_t* __restrict__ control,
                                                            uint8_t* __restrict__ frames,
                                                            int32_t* __restrict__ record) {
  dz::pdl_enter();
  __shared__ BreakoutState s_state;
  const int E = cfg.num_streams, e = blockIdx.x;
  if (threadIdx.x == 0) {
    BreakoutState s = load_state<BreakoutState>(state, E, e);
    if (kStep) {
      const Step r = breakout_tick(s, cfg, cfg.stream_offset + (uint32_t)e, control[e], control[E + e] != 0);
      store_state(s, state, E, e);
      record[e] = r.step_type;
      record[E + e] = r.reward;
      record[2 * E + e] = r.discount;
      record[3 * E + e] = r.lives;
    }
    s_state = s;
  }
  __syncthreads();
  const BreakoutState s = s_state;
  uint4* out = reinterpret_cast<uint4*>(frames + (int64_t)e * kFrameBytes);
  for (int i = threadIdx.x; i < kH * kRowWords; i += kThreads) {
    const int y = i / kRowWords, b0 = 16 * (i - y * kRowWords);
    const int xa = b0 / 3, xb = (b0 + 15) / 3;           // the word covers pixels xa..xb (at most 6)
    uint4 v = make_uint4(0, 0, 0, 0);                      // the background is black
    if (span_has_object(s, y, xa, xb)) {
      uint32_t rgb[6];
#pragma unroll
      for (int p = 0; p < 6; ++p) rgb[p] = xa + p <= xb ? breakout_rgb(s, xa + p, y) : 0u;
      const int k = b0 - 3 * xa;
      v = k == 0 ? pack_word<0>(rgb) : k == 1 ? pack_word<1>(rgb) : pack_word<2>(rgb);
    }
    out[i] = v;
  }
}

int check_config(const dz_breakout_config* cfg) {
  return check_game_config(cfg, "dz_breakout", DZ_BREAKOUT_MAX_STREAMS, 4, DZ_BREAKOUT_MAX_NOOP_STEPS);
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_breakout_step(const dz_breakout_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                     uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !h_control || !d_control || !d_frames || !d_record || !h_record)
    return fail(DZ_EINVAL, "dz_breakout_step: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_breakout_step: d_frames must be 16-byte aligned");
  const int E = cfg->num_streams;
  for (int e = 0; e < E; ++e)
    if (!h_control[E + e] && (h_control[e] < 0 || h_control[e] >= cfg->num_actions))
      return fail(DZ_EINVAL, "dz_breakout_step: an action is outside [0, num_actions)");
  const cudaStream_t s = (cudaStream_t)stream;
  DZ_CUDA_OK(cudaMemcpyAsync(d_control, h_control, 2 * E * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DZ_LAUNCH(breakout_kernel<true>, E, kThreads, 0, stream, *cfg, d_state, d_control, d_frames, d_record);
  DZ_CUDA_OK(cudaMemcpyAsync(h_record, d_record, DZ_BREAKOUT_RECORD_FIELDS * E * sizeof(int32_t),
                             cudaMemcpyDeviceToHost, s));
  return DZ_OK;
}

int dz_breakout_render(const dz_breakout_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !d_frames) return fail(DZ_EINVAL, "dz_breakout_render: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_breakout_render: d_frames must be 16-byte aligned");
  DZ_LAUNCH(breakout_kernel<false>, cfg->num_streams, kThreads, 0, stream, *cfg, d_state, (const int32_t*)nullptr,
            d_frames, (int32_t*)nullptr);
  return DZ_OK;
}

// The kernel's tick and picture compiled for the host: stream cfg->stream_offset, one state of
// DZ_BREAKOUT_STATE_FIELDS int32 updated in place; frame (may be NULL) gets the 210x160x3 bytes, record the
// step_type / reward / discount / lives.
int dz_test_breakout_step(const dz_breakout_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                          int32_t* record) {
  if (!cfg || !state || !record) return fail(DZ_EINVAL, "dz_test_breakout_step: null pointer");
  dz_breakout_config one = *cfg;
  one.num_streams = 1;
  DZ_TRY(check_config(&one));
  if (!reset && (action < 0 || action >= cfg->num_actions))
    return fail(DZ_EINVAL, "dz_test_breakout_step: action outside [0, num_actions)");
  BreakoutState s;
  memcpy(&s, state, sizeof(s));
  const Step r = breakout_tick(s, one, one.stream_offset, action, reset != 0);
  memcpy(state, &s, sizeof(s));
  record[0] = r.step_type; record[1] = r.reward; record[2] = r.discount; record[3] = r.lives;
  if (frame)
    for (int y = 0; y < kH; ++y)
      for (int x = 0; x < kW; ++x) {
        const uint32_t rgb = breakout_rgb(s, x, y);
        for (int c = 0; c < 3; ++c) frame[(y * kW + x) * 3 + c] = (uint8_t)(rgb >> (8 * c));
      }
  return DZ_OK;
}

}  // extern "C"
