// Pong at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §12).
//
// The project's own Pong, not ALE Pong: the agent's paddle on the right against a scripted opponent on the left, a 4x4
// ball that is served by a FIRE action (or a serve timer), +1 or -1 whenever a point ends, 21 points to a game.  The
// rules live in Pong::start / frame / over and the picture in Pong::rgb; dz_game.cuh's driver runs them in the kernel
// and in the host twin (dz_test_pong_step), and oracle/pong_oracle.py restates them in numpy.
//
// State: int32 [DZ_PONG_STATE_FIELDS][E] (one array per field, in the order of PongState).  Randomness is
// counter-based: stream e's key is threefry2x32((0, seed), (stream_offset + e, 2)) (the 2 tags the game: Catch keys
// with 0, Breakout with 1); a reset draws its no-op count from threefry2x32(key, (counter, 0)) and a serve its y, dx and
// dy from threefry2x32(key, (counter, 1)), each advancing counter.
#include "dz_game.cuh"

namespace dz {

namespace {

// Walls y in [24, 34) and [194, 210); the field is y in [34, 194).
constexpr int kWallTop = 24, kFieldTop = 34, kFieldBottom = 194;
constexpr int kPaddleW = 4, kPaddleH = 16, kOppX = 16, kAgentX = 140;
constexpr int kPaddleMin = kFieldTop, kPaddleMax = kFieldBottom - kPaddleH, kPaddleStart = 106, kPaddleStep = 4;
constexpr int kBall = 4, kBallMaxY = kFieldBottom - kBall;                                  // ball y in [34, 190]
constexpr int kServeX = 78, kServeYMin = 50, kServeYMax = 174;
// The opponent's top y moves at most this many px per frame (DESIGN.md §12 gives the tuning).
constexpr int kOppSpeed = 1;
constexpr int kHitDx = 3, kServeDelay = 64, kWin = 21;
// Scores: 12x20 px seven-segment cells with 4 px segments at y in [2, 22); a score's tens cell starts 16 px left of
// its units cell.
constexpr int kDigitY = 2, kDigitW = 12, kDigitH = 20, kSeg = 4, kOppTensX = 20, kAgentTensX = 116, kUnitsDx = 16;
// Glyph of digit d (bit i: segment "abcdefg"[i]): byte d of kGlyphsLo for d < 8, byte d - 8 of kGlyphsHi.
constexpr uint64_t kGlyphsLo = 0x077D6D664F5B063Full;
constexpr uint32_t kGlyphsHi = 0x6F7Fu;
enum { kNoop = 0, kFire = 1, kRight = 2, kLeft = 3, kRightFire = 4, kLeftFire = 5 };
static_assert(DZ_PONG_MAX_NOOP_STEPS < kServeDelay, "no ball is served during the no-op frames of a reset");
static_assert(kServeX > kOppX + kPaddleW && kServeX + kBall < kAgentX, "a served ball touches neither paddle");
static_assert(kServeYMin >= kFieldTop && kServeYMax <= kBallMaxY, "a served ball is in the field");
static_assert((kPaddleStart - kPaddleMin) % kPaddleStep == 0 && (kPaddleMax - kPaddleStart) % kPaddleStep == 0,
              "the agent's paddle reaches both walls");

// Packed 0x00BBGGRR colours; the background (144, 72, 17) is Pong::kBackground.
constexpr uint32_t kWhite = 0xECECECu, kOppRgb = 0x4A82D5u, kAgentRgb = 0x5CBA5Cu;

struct PongState {   // the field order of the state arrays
  int32_t paddle_y, opponent_y, ball_x, ball_y, ball_dx, ball_dy, in_play, serve_timer;
  int32_t agent_score, opponent_score, counter, noops, over;
};
static_assert(sizeof(PongState) == DZ_PONG_STATE_FIELDS * sizeof(int32_t), "one int32 per field");

__host__ __device__ __forceinline__ int32_t clamp_paddle(int32_t y) {
  return y < kPaddleMin ? kPaddleMin : y > kPaddleMax ? kPaddleMax : y;
}

// dy after a paddle hit at offset o = ball_y - paddle_y + 3 in [0, 18]: (-3, -2, -1, +1, +2, +3)[6 o / 19].
__host__ __device__ __forceinline__ int32_t hit_dy(int32_t o) {
  const int32_t zone = 6 * o / (kPaddleH + kBall - 1);
  return zone < 3 ? zone - 3 : zone - 2;
}

__host__ __device__ __forceinline__ void pong_serve(PongState& s, uint32_t k0, uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 1u, &o0, &o1);
  s.counter += 1;
  const int32_t d = below(o1, 8);                          // dx in {-2, +2} x dy in {-2, -1, +1, +2}
  s.ball_x = kServeX;
  s.ball_y = kServeYMin + below(o0, kServeYMax - kServeYMin + 1);
  s.ball_dx = d < 4 ? -2 : 2;
  s.ball_dy = (d & 3) < 2 ? (d & 3) - 2 : (d & 3) - 1;
  s.in_play = 1;
}

// Is pixel (x, y) of the score band lit by `score`, whose tens cell starts at tens_x?
__host__ __device__ __forceinline__ bool score_pixel(int32_t score, int tens_x, int x, int y) {
  int d, cx;
  if (x >= tens_x + kUnitsDx && x < tens_x + kUnitsDx + kDigitW) {
    d = score % 10;
    cx = x - tens_x - kUnitsDx;
  } else if (score >= 10 && x >= tens_x && x < tens_x + kDigitW) {
    d = score / 10;
    cx = x - tens_x;
  } else {
    return false;
  }
  const uint32_t m = d < 8 ? (uint32_t)(kGlyphsLo >> (8 * d)) : kGlyphsHi >> (8 * (d - 8));
  const int cy = y - kDigitY;
  const bool left = cx < kSeg, right = cx >= kDigitW - kSeg;
  const bool upper = cy < kDigitH / 2 + 2, lower = cy >= kDigitH / 2 - 2;
  return ((m & 1) && cy < kSeg) || ((m & 2) && right && upper) || ((m & 4) && right && lower) ||
         ((m & 8) && cy >= kDigitH - kSeg) || ((m & 16) && left && lower) || ((m & 32) && left && upper) ||
         ((m & 64) && upper && lower);
}

struct Pong {
  using State = PongState;
  static constexpr const char* kName = "pong";
  static constexpr uint32_t kTag = 2;
  static constexpr int kMaxStreams = DZ_PONG_MAX_STREAMS, kMinActions = 6, kMaxNoopSteps = DZ_PONG_MAX_NOOP_STEPS;
  static constexpr uint32_t kBackground = 0x114890u;

  __host__ __device__ __forceinline__ static void start(State& s, uint32_t, uint32_t) {
    s.paddle_y = s.opponent_y = kPaddleStart;
    s.ball_x = s.ball_y = s.ball_dx = s.ball_dy = 0;
    s.in_play = 0;
    s.serve_timer = kServeDelay;
    s.agent_score = s.opponent_score = 0;
  }

  // One frame of the game; returns its reward.
  __host__ __device__ __forceinline__ static int32_t frame(State& s, int32_t action, uint32_t k0, uint32_t k1) {
    if (action == kRight || action == kRightFire) s.paddle_y = clamp_paddle(s.paddle_y - kPaddleStep);
    if (action == kLeft || action == kLeftFire) s.paddle_y = clamp_paddle(s.paddle_y + kPaddleStep);
    const int32_t target = s.in_play && s.ball_dx < 0 ? s.ball_y - (kPaddleH - kBall) / 2 : kPaddleStart;
    const int32_t d = target - s.opponent_y;
    s.opponent_y = clamp_paddle(s.opponent_y + (d < -kOppSpeed ? -kOppSpeed : d > kOppSpeed ? kOppSpeed : d));
    if (!s.in_play) {
      s.serve_timer -= 1;
      if (action == kFire || action == kRightFire || action == kLeftFire || s.serve_timer <= 0) pong_serve(s, k0, k1);
      return 0;
    }
    const int32_t x0 = s.ball_x;
    int32_t x = x0 + s.ball_dx, y = s.ball_y + s.ball_dy;
    if (y < kFieldTop) { y = 2 * kFieldTop - y; s.ball_dy = -s.ball_dy; }
    if (y > kBallMaxY) { y = 2 * kBallMaxY - y; s.ball_dy = -s.ball_dy; }
    s.ball_y = y;
    // A paddle returns a ball that crosses its inner column this frame while the two overlap vertically.
    if (s.ball_dx > 0 && x0 + kBall <= kAgentX && x + kBall > kAgentX && y > s.paddle_y - kBall &&
        y < s.paddle_y + kPaddleH) {
      x = kAgentX - kBall;
      s.ball_dx = -kHitDx;
      s.ball_dy = hit_dy(y - s.paddle_y + kBall - 1);
    } else if (s.ball_dx < 0 && x0 >= kOppX + kPaddleW && x < kOppX + kPaddleW && y > s.opponent_y - kBall &&
               y < s.opponent_y + kPaddleH) {
      x = kOppX + kPaddleW;
      s.ball_dx = kHitDx;
      s.ball_dy = hit_dy(y - s.opponent_y + kBall - 1);
    }
    s.ball_x = x;
    if (x > 0 && x < kFrameW - kBall) return 0;
    s.in_play = 0;                                          // a point: the ball left the field past a paddle
    s.serve_timer = kServeDelay;
    if (x <= 0) {
      s.agent_score += 1;
      return 1;
    }
    s.opponent_score += 1;
    return -1;
  }

  __host__ __device__ __forceinline__ static bool over(const State& s) {
    return s.agent_score == kWin || s.opponent_score == kWin;
  }

  __host__ __device__ __forceinline__ static int32_t lives(const State&) { return 0; }

  // The colour of pixel (x, y), objects in drawing order: background, walls, scores, paddles, ball.
  __host__ __device__ __forceinline__ static uint32_t rgb(const State& s, int x, int y) {
    if (s.in_play && y >= s.ball_y && y < s.ball_y + kBall && x >= s.ball_x && x < s.ball_x + kBall) return kWhite;
    if (x >= kAgentX && x < kAgentX + kPaddleW && y >= s.paddle_y && y < s.paddle_y + kPaddleH) return kAgentRgb;
    if (x >= kOppX && x < kOppX + kPaddleW && y >= s.opponent_y && y < s.opponent_y + kPaddleH) return kOppRgb;
    if ((y >= kWallTop && y < kFieldTop) || y >= kFieldBottom) return kWhite;
    if (y >= kDigitY && y < kDigitY + kDigitH) {
      if (score_pixel(s.opponent_score, kOppTensX, x, y)) return kOppRgb;
      if (score_pixel(s.agent_score, kAgentTensX, x, y)) return kAgentRgb;
    }
    return kBackground;
  }

  __device__ __forceinline__ static bool span_has_object(const State& s, int y, int xa, int xb) {
    if (s.in_play && y >= s.ball_y && y < s.ball_y + kBall && xb >= s.ball_x && xa < s.ball_x + kBall) return true;
    if (y >= s.paddle_y && y < s.paddle_y + kPaddleH && xb >= kAgentX && xa < kAgentX + kPaddleW) return true;
    if (y >= s.opponent_y && y < s.opponent_y + kPaddleH && xb >= kOppX && xa < kOppX + kPaddleW) return true;
    if ((y >= kWallTop && y < kFieldTop) || y >= kFieldBottom) return true;
    return y >= kDigitY && y < kDigitY + kDigitH &&
           ((xb >= kOppTensX && xa < kOppTensX + kUnitsDx + kDigitW) ||
            (xb >= kAgentTensX && xa < kAgentTensX + kUnitsDx + kDigitW));
  }
};

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_pong_step(const dz_pong_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                 uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  return game_step<Pong>(cfg, d_state, h_control, d_control, d_frames, d_record, h_record, stream);
}

int dz_pong_render(const dz_pong_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  return game_render<Pong>(cfg, d_state, d_frames, stream);
}

int dz_test_pong_step(const dz_pong_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                      int32_t* record) {
  return game_host_step<Pong>(cfg, state, action, reset, frame, record);
}

}  // extern "C"
