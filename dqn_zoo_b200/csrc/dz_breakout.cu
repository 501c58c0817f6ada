// Breakout at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §11).
//
// The project's own game, not ALE Breakout: a 6 x 18 brick wall worth 7 / 4 / 1 points per row, a paddle, a 4x4 ball
// that is served by FIRE (or a serve timer), 5 lives.  The rules live in Breakout::start / frame / over and the
// picture in Breakout::rgb; dz_game.cuh's driver runs them in the kernel and in the host twin (dz_test_breakout_step),
// and oracle/breakout_oracle.py restates them in numpy.
//
// State: int32 [DZ_BREAKOUT_STATE_FIELDS][E] (one array per field, in the order of BreakoutState); the wall is six
// 18-bit row masks (bit c of row r: brick (r, c) is still there).  Randomness is counter-based: stream e's key is
// threefry2x32((0, seed), (stream_offset + e, 1)) (the 1 tags the game: Catch keys with 0); a reset draws its no-op
// count from threefry2x32(key, (counter, 0)) and a serve its x and dx from threefry2x32(key, (counter, 1)), each
// advancing counter.
#include "dz_game.cuh"

namespace dz {

namespace {

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
enum { kNoop = 0, kFire = 1, kRight = 2, kLeft = 3 };
static_assert(DZ_BREAKOUT_MAX_NOOP_STEPS < kServeDelay, "no ball is served during the no-op frames of a reset");
static_assert(kFieldLeft + kCols * kBrickW == kFieldRight, "the wall spans the field");
static_assert(kServeY > kBrickBottom && kServeY + kBall < kPaddleY, "a served ball touches no brick and no paddle");

// Packed 0x00BBGGRR colours: walls and life blocks grey, bricks by row, paddle, ball; the background is black
// (Breakout::kBackground).
constexpr uint32_t kGrey = 0x8E8E8Eu, kPaddleRgb = 0x4848C8u, kBallRgb = 0xECECECu;
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

struct Breakout {
  using State = BreakoutState;
  static constexpr const char* kName = "breakout";
  static constexpr uint32_t kTag = 1;
  static constexpr int kMaxStreams = DZ_BREAKOUT_MAX_STREAMS, kMinActions = 4;
  static constexpr int kMaxNoopSteps = DZ_BREAKOUT_MAX_NOOP_STEPS;
  static constexpr uint32_t kBackground = 0x000000u;

  __host__ __device__ __forceinline__ static void start(State& s, uint32_t, uint32_t) {
    s.paddle_x = (kPaddleMinX + kPaddleMaxX) / 2;
    s.ball_x = s.ball_y = s.ball_dx = s.ball_dy = 0;
    s.in_play = 0;
    s.serve_timer = kServeDelay;
    s.lives = kLives;
#pragma unroll
    for (int r = 0; r < kRows; ++r) s.row[r] = kFullRow;
  }

  // One frame of the game; returns its reward.
  __host__ __device__ __forceinline__ static int32_t frame(State& s, int32_t action, uint32_t k0, uint32_t k1) {
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

  __host__ __device__ __forceinline__ static bool over(const State& s) {
    int32_t bricks = 0;
#pragma unroll
    for (int i = 0; i < kRows; ++i) bricks |= s.row[i];
    return s.lives == 0 || bricks == 0;
  }

  __host__ __device__ __forceinline__ static int32_t lives(const State& s) { return s.lives; }

  // The colour of pixel (x, y), objects in drawing order: background, walls, life blocks, bricks, paddle, ball.
  __host__ __device__ __forceinline__ static uint32_t rgb(const State& s, int x, int y) {
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

  // In the wall's rows the test is against the row's brick mask, so the cleared part of the wall is written as
  // background.
  __device__ __forceinline__ static bool span_has_object(const State& s, int y, int xa, int xb) {
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
};

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_breakout_step(const dz_breakout_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                     uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  return game_step<Breakout>(cfg, d_state, h_control, d_control, d_frames, d_record, h_record, stream);
}

int dz_breakout_render(const dz_breakout_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  return game_render<Breakout>(cfg, d_state, d_frames, stream);
}

int dz_test_breakout_step(const dz_breakout_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                          int32_t* record) {
  return game_host_step<Breakout>(cfg, state, action, reset, frame, record);
}

}  // extern "C"
