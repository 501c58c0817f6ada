// Pong at Atari geometry, simulated and rendered on the device for E streams at once (DESIGN.md §12).
//
// The project's own Pong, not ALE Pong: the agent's paddle on the right against a scripted opponent on the left, a 4x4
// ball that is served by a FIRE action (or a serve timer), +1 or -1 whenever a point ends, 21 points to a game.  One
// launch per tick: a CTA per stream.  Thread 0 applies the stream's action (or a reset with its random no-op frames) to
// the stream's state, the CTA then writes the stream's whole 210x160x3 RGB frame with aligned 16-byte stores, and CTA
// e's record gets step_type / reward / discount / lives.  The rules live in pong_reset / pong_frame / pong_tick and the
// picture in pong_rgb; the kernel and the host twin (dz_test_pong_step) run the same functions, and
// oracle/pong_oracle.py restates them in numpy.
//
// State: int32 [DZ_PONG_STATE_FIELDS][E] (one array per field, in the order of PongState).  Randomness is
// counter-based: stream e's key is threefry2x32((0, seed), (stream_offset + e, 2)) (the 2 tags the game: Catch keys
// with 0, Breakout with 1); a reset draws its no-op count from threefry2x32(key, (counter, 0)) and a serve its y, dx and
// dy from threefry2x32(key, (counter, 1)), each advancing counter.
#include "dz_game.cuh"
#include "dz_threefry.cuh"

namespace dz {

namespace {

constexpr int kH = DZ_PONG_HEIGHT, kW = DZ_PONG_WIDTH;
constexpr int kRowBytes = 3 * kW;                         // 480: 30 16-byte words
constexpr int kRowWords = kRowBytes / 16;
constexpr int kFrameBytes = kH * kRowBytes;               // 100,800
constexpr uint32_t kGameTag = 2;                           // the second counter word of the stream key
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
constexpr int kThreads = 256;
enum { kNoop = 0, kFire = 1, kRight = 2, kLeft = 3, kRightFire = 4, kLeftFire = 5 };
static_assert(kRowBytes % 16 == 0, "rows are whole 16-byte words");
static_assert(DZ_PONG_MAX_NOOP_STEPS < kServeDelay, "no ball is served during the no-op frames of a reset");
static_assert(kServeX > kOppX + kPaddleW && kServeX + kBall < kAgentX, "a served ball touches neither paddle");
static_assert(kServeYMin >= kFieldTop && kServeYMax <= kBallMaxY, "a served ball is in the field");
static_assert((kPaddleStart - kPaddleMin) % kPaddleStep == 0 && (kPaddleMax - kPaddleStart) % kPaddleStep == 0,
              "the agent's paddle reaches both walls");

// Packed 0x00BBGGRR colours.
constexpr uint32_t kBackground = 0x114890u, kWhite = 0xECECECu, kOppRgb = 0x4A82D5u, kAgentRgb = 0x5CBA5Cu;

struct PongState {   // the field order of the state arrays
  int32_t paddle_y, opponent_y, ball_x, ball_y, ball_dx, ball_dy, in_play, serve_timer;
  int32_t agent_score, opponent_score, counter, noops, over;
};
static_assert(sizeof(PongState) == DZ_PONG_STATE_FIELDS * sizeof(int32_t), "one int32 per field");

struct Step { int32_t step_type, reward, discount, lives; };

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

// One frame of the game; returns its reward.
__host__ __device__ __forceinline__ int32_t pong_frame(PongState& s, int32_t action, uint32_t k0, uint32_t k1) {
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
  if (x > 0 && x < kW - kBall) return 0;
  s.in_play = 0;                                          // a point: the ball left the field past a paddle
  s.serve_timer = kServeDelay;
  if (x <= 0) {
    s.agent_score += 1;
    return 1;
  }
  s.opponent_score += 1;
  return -1;
}

__host__ __device__ __forceinline__ void pong_reset(PongState& s, const dz_pong_config& cfg, uint32_t k0,
                                                    uint32_t k1) {
  uint32_t o0, o1;
  threefry2x32(k0, k1, (uint32_t)s.counter, 0u, &o0, &o1);
  s.counter += 1;
  const int32_t k = cfg.min_noop_steps + below(o0, (uint32_t)(cfg.max_noop_steps - cfg.min_noop_steps + 1));
  s.paddle_y = s.opponent_y = kPaddleStart;
  s.ball_x = s.ball_y = s.ball_dx = s.ball_dy = 0;
  s.in_play = 0;
  s.serve_timer = kServeDelay;
  s.agent_score = s.opponent_score = 0;
  s.over = 0;
  for (int32_t i = 0; i < k; ++i) pong_frame(s, kNoop, k0, k1);   // no serve: the timer stays above 0
  s.noops = k;
}

// A tick of one stream: a reset (asked for, or after the episode's LAST step) or one frame with `action`.
__host__ __device__ __forceinline__ Step pong_tick(PongState& s, const dz_pong_config& cfg, uint32_t stream,
                                                   int32_t action, bool reset) {
  uint32_t k0, k1;
  threefry2x32(0u, cfg.seed, stream, kGameTag, &k0, &k1);
  if (reset || s.over) {
    pong_reset(s, cfg, k0, k1);
    return {0, 0, 0, 0};
  }
  const int32_t r = pong_frame(s, action, k0, k1);
  s.over = s.agent_score == kWin || s.opponent_score == kWin;
  return {s.over ? 2 : 1, r, s.over ? 0 : 1, 0};
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

// The colour of pixel (x, y), objects in drawing order: background, walls, scores, paddles, ball.
__host__ __device__ __forceinline__ uint32_t pong_rgb(const PongState& s, int x, int y) {
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

// Can an object touch pixels [xa, xb] of row y?  Conservative: false means background.
__device__ __forceinline__ bool span_has_object(const PongState& s, int y, int xa, int xb) {
  if (s.in_play && y >= s.ball_y && y < s.ball_y + kBall && xb >= s.ball_x && xa < s.ball_x + kBall) return true;
  if (y >= s.paddle_y && y < s.paddle_y + kPaddleH && xb >= kAgentX && xa < kAgentX + kPaddleW) return true;
  if (y >= s.opponent_y && y < s.opponent_y + kPaddleH && xb >= kOppX && xa < kOppX + kPaddleW) return true;
  if ((y >= kWallTop && y < kFieldTop) || y >= kFieldBottom) return true;
  return y >= kDigitY && y < kDigitY + kDigitH &&
         ((xb >= kOppTensX && xa < kOppTensX + kUnitsDx + kDigitW) ||
          (xb >= kAgentTensX && xa < kAgentTensX + kUnitsDx + kDigitW));
}

template <bool kStep>
__global__ void __launch_bounds__(kThreads) pong_kernel(const dz_pong_config cfg, int32_t* __restrict__ state,
                                                        const int32_t* __restrict__ control,
                                                        uint8_t* __restrict__ frames, int32_t* __restrict__ record) {
  dz::pdl_enter();
  __shared__ PongState s_state;
  const int E = cfg.num_streams, e = blockIdx.x;
  if (threadIdx.x == 0) {
    PongState s = load_state<PongState>(state, E, e);
    if (kStep) {
      const Step r = pong_tick(s, cfg, cfg.stream_offset + (uint32_t)e, control[e], control[E + e] != 0);
      store_state(s, state, E, e);
      record[e] = r.step_type;
      record[E + e] = r.reward;
      record[2 * E + e] = r.discount;
      record[3 * E + e] = r.lives;
    }
    s_state = s;
  }
  __syncthreads();
  const PongState s = s_state;
  const uint32_t bg[6] = {kBackground, kBackground, kBackground, kBackground, kBackground, kBackground};
  uint4* out = reinterpret_cast<uint4*>(frames + (int64_t)e * kFrameBytes);
  for (int i = threadIdx.x; i < kH * kRowWords; i += kThreads) {
    const int y = i / kRowWords, b0 = 16 * (i - y * kRowWords);
    const int xa = b0 / 3, xb = (b0 + 15) / 3;           // the word covers pixels xa..xb (at most 6)
    const int k = b0 - 3 * xa;                             // the channel of its first byte
    uint4 v;
    if (span_has_object(s, y, xa, xb)) {
      uint32_t rgb[6];
#pragma unroll
      for (int p = 0; p < 6; ++p) rgb[p] = xa + p <= xb ? pong_rgb(s, xa + p, y) : 0u;
      v = k == 0 ? pack_word<0>(rgb) : k == 1 ? pack_word<1>(rgb) : pack_word<2>(rgb);
    } else {
      v = k == 0 ? pack_word<0>(bg) : k == 1 ? pack_word<1>(bg) : pack_word<2>(bg);
    }
    out[i] = v;
  }
}

int check_config(const dz_pong_config* cfg) {
  return check_game_config(cfg, "dz_pong", DZ_PONG_MAX_STREAMS, 6, DZ_PONG_MAX_NOOP_STEPS);
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" {

int dz_pong_step(const dz_pong_config* cfg, int32_t* d_state, const int32_t* h_control, int32_t* d_control,
                 uint8_t* d_frames, int32_t* d_record, int32_t* h_record, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !h_control || !d_control || !d_frames || !d_record || !h_record)
    return fail(DZ_EINVAL, "dz_pong_step: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_pong_step: d_frames must be 16-byte aligned");
  const int E = cfg->num_streams;
  for (int e = 0; e < E; ++e)
    if (!h_control[E + e] && (h_control[e] < 0 || h_control[e] >= cfg->num_actions))
      return fail(DZ_EINVAL, "dz_pong_step: an action is outside [0, num_actions)");
  const cudaStream_t s = (cudaStream_t)stream;
  DZ_CUDA_OK(cudaMemcpyAsync(d_control, h_control, 2 * E * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DZ_LAUNCH(pong_kernel<true>, E, kThreads, 0, stream, *cfg, d_state, d_control, d_frames, d_record);
  DZ_CUDA_OK(cudaMemcpyAsync(h_record, d_record, DZ_PONG_RECORD_FIELDS * E * sizeof(int32_t), cudaMemcpyDeviceToHost,
                             s));
  return DZ_OK;
}

int dz_pong_render(const dz_pong_config* cfg, int32_t* d_state, uint8_t* d_frames, void* stream) {
  DZ_TRY(check_config(cfg));
  if (!d_state || !d_frames) return fail(DZ_EINVAL, "dz_pong_render: null pointer");
  if ((uintptr_t)d_frames % 16) return fail(DZ_EINVAL, "dz_pong_render: d_frames must be 16-byte aligned");
  DZ_LAUNCH(pong_kernel<false>, cfg->num_streams, kThreads, 0, stream, *cfg, d_state, (const int32_t*)nullptr,
            d_frames, (int32_t*)nullptr);
  return DZ_OK;
}

// The kernel's tick and picture compiled for the host: stream cfg->stream_offset, one state of DZ_PONG_STATE_FIELDS
// int32 updated in place; frame (may be NULL) gets the 210x160x3 bytes, record the step_type / reward / discount /
// lives.
int dz_test_pong_step(const dz_pong_config* cfg, int32_t* state, int32_t action, int32_t reset, uint8_t* frame,
                      int32_t* record) {
  if (!cfg || !state || !record) return fail(DZ_EINVAL, "dz_test_pong_step: null pointer");
  dz_pong_config one = *cfg;
  one.num_streams = 1;
  DZ_TRY(check_config(&one));
  if (!reset && (action < 0 || action >= cfg->num_actions))
    return fail(DZ_EINVAL, "dz_test_pong_step: action outside [0, num_actions)");
  PongState s;
  memcpy(&s, state, sizeof(s));
  const Step r = pong_tick(s, one, one.stream_offset, action, reset != 0);
  memcpy(state, &s, sizeof(s));
  record[0] = r.step_type; record[1] = r.reward; record[2] = r.discount; record[3] = r.lives;
  if (frame)
    for (int y = 0; y < kH; ++y)
      for (int x = 0; x < kW; ++x) {
        const uint32_t rgb = pong_rgb(s, x, y);
        for (int c = 0; c < 3; ++c) frame[(y * kW + x) * 3 + c] = (uint8_t)(rgb >> (8 * c));
      }
  return DZ_OK;
}

}  // extern "C"
