// Catch at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §10).
//
// The rules live in Catch::start / frame / over and the picture in Catch::rgb; dz_game.cuh's driver runs them in the
// kernel and in the host twin (dz_test_catch_step), and oracle/catch_oracle.py restates them in numpy.
//
// State: int32 [DZ_CATCH_STATE_FIELDS][E] (one array per field, in the order of CatchState).  Randomness is
// counter-based: stream e's key is threefry2x32((0, seed), (stream_offset + e, 0)); a reset draws its no-op count from
// threefry2x32(key, (counter, 0)) and a ball its x and dx from threefry2x32(key, (counter, 1)), each advancing counter.
#include "dz_game.cuh"

namespace dz {

namespace {

constexpr int kPaddleW = 16, kPaddleH = 4, kPaddleY = 188, kPaddleMaxX = kFrameW - kPaddleW, kPaddleStep = 3;
constexpr int kBall = 8, kBallMaxX = kFrameW - kBall, kBallFall = 2, kLandY = kPaddleY - kBall;  // 152, lands at 180
constexpr int kLives = 3, kBallsPerEpisode = 20;
constexpr int kLivesY = 4, kLivesH = 6, kLivesX = 8, kLivesPitch = 12, kLivesW = 8;
static_assert(kLandY % kBallFall == 0, "the ball reaches its landing row exactly");
static_assert(DZ_CATCH_MAX_NOOP_STEPS < kLandY / kBallFall, "no ball lands during the no-op frames of a reset");

// Packed 0x00BBGGRR colours: paddle (200, 72, 72), ball (236, 236, 236), life blocks (92, 186, 92); the background
// (24, 26, 167) is Catch::kBackground.
constexpr uint32_t kPaddleRgb = 0x4848C8u, kBallRgb = 0xECECECu, kLivesRgb = 0x5CBA5Cu;

struct CatchState {   // the field order of the state arrays
  int32_t paddle_x, ball_x, ball_y, ball_dx, lives, balls_left, counter, noops, over;
};
static_assert(sizeof(CatchState) == DZ_CATCH_STATE_FIELDS * sizeof(int32_t), "one int32 per field");

__host__ __device__ __forceinline__ void catch_spawn(CatchState& s, uint32_t k0, uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 1u, &o0, &o1);
  s.counter += 1;
  s.ball_x = below(o0, kBallMaxX + 1);
  s.ball_dx = below(o1, 3) - 1;
  s.ball_y = 0;
}

struct Catch {
  using State = CatchState;
  static constexpr const char* kName = "catch";
  static constexpr uint32_t kTag = 0;
  static constexpr int kMaxStreams = DZ_CATCH_MAX_STREAMS, kMinActions = 3, kMaxNoopSteps = DZ_CATCH_MAX_NOOP_STEPS;
  static constexpr uint32_t kBackground = 0xA71A18u;

  __host__ __device__ __forceinline__ static void start(State& s, uint32_t k0, uint32_t k1) {
    s.paddle_x = kPaddleMaxX / 2;
    s.lives = kLives;
    s.balls_left = kBallsPerEpisode;
    catch_spawn(s, k0, k1);
  }

  // One frame of the game; returns its reward.
  __host__ __device__ __forceinline__ static int32_t frame(State& s, int32_t action, uint32_t k0, uint32_t k1) {
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

  __host__ __device__ __forceinline__ static bool over(const State& s) { return s.lives == 0 || s.balls_left == 0; }
  __host__ __device__ __forceinline__ static int32_t lives(const State& s) { return s.lives; }

  // The colour of pixel (x, y): the ball (drawn last), the paddle, a life block or the background.
  __host__ __device__ __forceinline__ static uint32_t rgb(const State& s, int x, int y) {
    if (y >= s.ball_y && y < s.ball_y + kBall && x >= s.ball_x && x < s.ball_x + kBall) return kBallRgb;
    if (y >= kPaddleY && y < kPaddleY + kPaddleH && x >= s.paddle_x && x < s.paddle_x + kPaddleW) return kPaddleRgb;
    if (y >= kLivesY && y < kLivesY + kLivesH && x >= kLivesX) {
      const int i = (x - kLivesX) / kLivesPitch;
      if (i < s.lives && x - kLivesX - i * kLivesPitch < kLivesW) return kLivesRgb;
    }
    return kBackground;
  }

  __device__ __forceinline__ static bool span_has_object(const State& s, int y, int xa, int xb) {
    if (y >= s.ball_y && y < s.ball_y + kBall && xb >= s.ball_x && xa < s.ball_x + kBall) return true;
    if (y >= kPaddleY && y < kPaddleY + kPaddleH && xb >= s.paddle_x && xa < s.paddle_x + kPaddleW) return true;
    return y >= kLivesY && y < kLivesY + kLivesH && s.lives > 0 && xb >= kLivesX &&
           xa < kLivesX + (s.lives - 1) * kLivesPitch + kLivesW;
  }
};

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_catch_step(const dz_catch_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                  uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  return game_step<Catch>(cfg, d_state, h_control, d_control, d_frames, d_record, h_record, stream);
}

int dz_catch_render(const dz_catch_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  return game_render<Catch>(cfg, d_state, d_frames, stream);
}

int dz_test_catch_step(const dz_catch_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                       int32_t* record) {
  return game_host_step<Catch>(cfg, state, action, reset, frame, record);
}

}  // extern "C"
