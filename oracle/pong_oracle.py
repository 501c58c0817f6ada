"""numpy restatement of the device Pong game (dqn_zoo_b200/csrc/dz_pong.cu, DESIGN.md §12), one stream at a time.
TEST INFRASTRUCTURE ONLY.

This is the project's own Pong, not ALE's: it has no reference implementation, so this module pins the project's
definition of the game, and the kernel and its host-compiled twin are tested against it.  Frames are drawn by plain
array slicing; the randomness is `oracle.jax_prng_oracle.threefry2x32`.

Rules.  Frame 210x160 RGB on (144, 72, 17).  White (236, 236, 236) walls at y in [24, 34) and [194, 210); the field is
y in [34, 194).  Paddles 4x16 px with top y in [34, 178], centred (106) after a reset: the opponent's (213, 130, 74) at
x in [16, 20), the agent's (92, 186, 92) at x in [140, 144).  Ball 4x4 px, (236, 236, 236), drawn last, only while in
play.  Scores: seven-segment numerals (12x20 px cells, 4 px segments) in the paddle's colour, y in [2, 22); the
opponent's units digit at x = 36 (tens at x = 20, from 10 up), the agent's at x = 132 (tens at x = 116).  Actions:
0 NOOP, 1 FIRE, 2 RIGHT (up 4 px), 3 LEFT (down 4 px), 4 RIGHTFIRE, 5 LEFTFIRE, 6.. NOOP.

A frame: (1) the agent's paddle moves (clamped); (2) the opponent's paddle moves at most 1 px toward ball_y - 6 while
the ball is in play and moving left, else toward 106 (clamped); (3) a ball out of play counts its serve timer down and
is served if the action is a FIRE action or the timer reaches 0: x = 78, y = 50 + below(125), (dx, dy) =
((-2, 2)[d // 4], (-2, -1, 1, 2)[d % 4]) for d = below(8) (the frame ends there); (4) a ball in play moves dx, then dy,
reflecting off the walls (y < 34 -> 68 - y, y > 190 -> 380 - y, dy negated); (5) a ball moving right whose right edge
crosses column 140 this frame (x_old + 4 <= 140 < x + 4) while it overlaps the agent's paddle vertically goes to
x = 136, dx = -3; a ball moving left with x_old >= 20 > x that overlaps the opponent's paddle goes to x = 20, dx = +3;
in both cases dy = (-3, -2, -1, 1, 2, 3)[6 * o // 19] for o = ball_y - paddle_y + 3 in [0, 18]; (6) a ball with x <= 0
is the agent's point (+1), one with x >= 156 the opponent's (-1): out of play, serve timer 64.  The episode ends (LAST,
discount 0) on the frame on which a score reaches 21; lives are 0 throughout.  A reset: 0-0, centred paddles, ball out
of play, timer 64, then k no-op frames, k uniform in [min, max] (max <= 63, so nothing is served).  Randomness: key =
threefry2x32((0, seed), (stream, 2)); a reset draws threefry2x32(key, (counter, 0)), a serve
threefry2x32(key, (counter, 1)), each advancing counter; a draw below n of 32 bits u is floor(u * n / 2^32)."""

import numpy as np

from oracle import jax_prng_oracle as jp

HEIGHT, WIDTH = 210, 160
WALL_TOP, FIELD_TOP, FIELD_BOTTOM = 24, 34, 194
OPP_X, AGENT_X, PADDLE_W, PADDLE_H = 16, 140, 4, 16
PADDLE_MIN, PADDLE_MAX, PADDLE_START, PADDLE_STEP = 34, 178, 106, 4
BALL, BALL_MAX_Y = 4, 190
SERVE_X, SERVE_Y_MIN, SERVE_Y_MAX = 78, 50, 174
OPP_SPEED, HIT_DX, SERVE_DELAY, WIN = 1, 3, 64, 21
HIT_DY = (-3, -2, -1, 1, 2, 3)
MAX_NOOP_STEPS = 63
DIGIT_W, DIGIT_H, SEGMENT, DIGIT_Y = 12, 20, 4, 2
OPP_DIGITS_X, AGENT_DIGITS_X = (20, 36), (116, 132)     # (tens, units)
# Seven-segment glyphs of 0..9, bit i = segment 'abcdefg'[i] (a top, b upper right, c lower right, d bottom,
# e lower left, f upper left, g middle).
GLYPHS = (0x3F, 0x06, 0x5B, 0x4F, 0x66, 0x6D, 0x7D, 0x07, 0x7F, 0x6F)
NOOP, FIRE, RIGHT, LEFT, RIGHTFIRE, LEFTFIRE = range(6)
BACKGROUND, WHITE, OPP_RGB, AGENT_RGB = (144, 72, 17), (236, 236, 236), (213, 130, 74), (92, 186, 92)
FIRST, MID, LAST = 0, 1, 2
FIELDS = ('paddle_y', 'opponent_y', 'ball_x', 'ball_y', 'ball_dx', 'ball_dy', 'in_play', 'serve_timer', 'agent_score',
          'opponent_score', 'counter', 'noops', 'over')
GAME_TAG = 2


def check_noops(min_noop_steps, max_noop_steps):
  if not 0 <= min_noop_steps <= max_noop_steps:
    raise ValueError('need 0 <= min_noop_steps <= max_noop_steps, got %d, %d' % (min_noop_steps, max_noop_steps))
  if max_noop_steps > MAX_NOOP_STEPS:
    raise ValueError('max_noop_steps %d > %d: a ball could be served during the no-op frames of a reset'
                     % (max_noop_steps, MAX_NOOP_STEPS))


def _below(u, n):
  return (int(u) * int(n)) >> 32


def _clamp(y):
  return min(max(y, PADDLE_MIN), PADDLE_MAX)


def glyph(d):
  """The 20x12 bool picture of digit d."""
  m = GLYPHS[d]
  g = np.zeros((DIGIT_H, DIGIT_W), bool)
  S, H, W = SEGMENT, DIGIT_H, DIGIT_W
  if m & 1: g[:S] = True                                  # a
  if m & 2: g[:H // 2 + 2, W - S:] = True                 # b
  if m & 4: g[H // 2 - 2:, W - S:] = True                 # c
  if m & 8: g[H - S:] = True                              # d
  if m & 16: g[H // 2 - 2:, :S] = True                    # e
  if m & 32: g[:H // 2 + 2, :S] = True                    # f
  if m & 64: g[H // 2 - 2:H // 2 + 2] = True              # g
  return g


class PongOracle:
  """One stream.  `state` is the dict of the device state fields; `step` / `reset` return
  (frame uint8 [210, 160, 3], step_type, reward, discount, lives) with reward / discount None on FIRST."""

  def __init__(self, seed, stream=0, num_actions=6, min_noop_steps=1, max_noop_steps=30):
    check_noops(min_noop_steps, max_noop_steps)
    if not 6 <= num_actions <= 18:
      raise ValueError('num_actions must be in [6, 18]')
    self.num_actions = num_actions
    self._min, self._max = min_noop_steps, max_noop_steps
    self._key = jp.threefry2x32((0, seed), (stream, GAME_TAG))
    self.state = dict.fromkeys(FIELDS, 0)
    self.state['over'] = 1

  def _serve(self):
    s = self.state
    o0, o1 = jp.threefry2x32(self._key, (s['counter'], 1))
    s['counter'] += 1
    d = _below(o1, 8)
    s.update(ball_x=SERVE_X, ball_y=SERVE_Y_MIN + _below(o0, SERVE_Y_MAX - SERVE_Y_MIN + 1), ball_dx=(-2, 2)[d // 4],
             ball_dy=(-2, -1, 1, 2)[d % 4], in_play=1)

  def _frame(self, action):
    s = self.state
    if action in (RIGHT, RIGHTFIRE):
      s['paddle_y'] = _clamp(s['paddle_y'] - PADDLE_STEP)
    elif action in (LEFT, LEFTFIRE):
      s['paddle_y'] = _clamp(s['paddle_y'] + PADDLE_STEP)
    target = s['ball_y'] - 6 if s['in_play'] and s['ball_dx'] < 0 else PADDLE_START
    s['opponent_y'] = _clamp(s['opponent_y'] + min(max(target - s['opponent_y'], -OPP_SPEED), OPP_SPEED))
    if not s['in_play']:
      s['serve_timer'] -= 1
      if action in (FIRE, RIGHTFIRE, LEFTFIRE) or s['serve_timer'] <= 0:
        self._serve()
      return 0
    x0 = s['ball_x']
    x = x0 + s['ball_dx']
    y = s['ball_y'] + s['ball_dy']
    if y < FIELD_TOP or y > BALL_MAX_Y:
      y = 2 * FIELD_TOP - y if y < FIELD_TOP else 2 * BALL_MAX_Y - y
      s['ball_dy'] = -s['ball_dy']
    s['ball_y'] = y
    for paddle, crossed, new_x, new_dx in (
        (s['paddle_y'], s['ball_dx'] > 0 and x0 + BALL <= AGENT_X < x + BALL, AGENT_X - BALL, -HIT_DX),
        (s['opponent_y'], s['ball_dx'] < 0 and x0 >= OPP_X + PADDLE_W > x, OPP_X + PADDLE_W, HIT_DX)):
      if crossed and paddle - BALL < y < paddle + PADDLE_H:
        x, s['ball_dx'], s['ball_dy'] = new_x, new_dx, HIT_DY[6 * (y - paddle + BALL - 1) // (PADDLE_H + BALL - 1)]
    s['ball_x'] = x
    if x <= 0 or x >= WIDTH - BALL:
      s.update(in_play=0, serve_timer=SERVE_DELAY)
      if x <= 0:
        s['agent_score'] += 1
        return 1
      s['opponent_score'] += 1
      return -1
    return 0

  def reset(self):
    s = self.state
    o0, _ = jp.threefry2x32(self._key, (s['counter'], 0))
    s['counter'] += 1
    k = self._min + _below(o0, self._max - self._min + 1)
    s.update(paddle_y=PADDLE_START, opponent_y=PADDLE_START, ball_x=0, ball_y=0, ball_dx=0, ball_dy=0, in_play=0,
             serve_timer=SERVE_DELAY, agent_score=0, opponent_score=0, over=0)
    for _ in range(k):
      self._frame(NOOP)
    s['noops'] = k
    return self.render(), FIRST, None, None, 0

  def step(self, action):
    out = self.advance(action)
    return (self.render(),) + out

  def advance(self, action):
    """`step` without the frame: (step_type, reward, discount, lives)."""
    if not 0 <= action < self.num_actions:
      raise ValueError('action %d outside [0, %d)' % (action, self.num_actions))
    s = self.state
    if s['over']:
      return self.reset()[1:]
    r = self._frame(action)
    s['over'] = int(s['agent_score'] == WIN or s['opponent_score'] == WIN)
    return LAST if s['over'] else MID, float(r), 0.0 if s['over'] else 1.0, 0

  def render(self):
    s = self.state
    f = np.empty((HEIGHT, WIDTH, 3), np.uint8)
    f[:] = BACKGROUND
    f[WALL_TOP:FIELD_TOP] = WHITE
    f[FIELD_BOTTOM:] = WHITE
    for score, (tens_x, units_x), rgb in ((s['opponent_score'], OPP_DIGITS_X, OPP_RGB),
                                          (s['agent_score'], AGENT_DIGITS_X, AGENT_RGB)):
      digits = [(units_x, score % 10)] + ([(tens_x, score // 10)] if score >= 10 else [])
      for x, d in digits:
        f[DIGIT_Y:DIGIT_Y + DIGIT_H, x:x + DIGIT_W][glyph(d)] = rgb
    f[s['opponent_y']:s['opponent_y'] + PADDLE_H, OPP_X:OPP_X + PADDLE_W] = OPP_RGB
    f[s['paddle_y']:s['paddle_y'] + PADDLE_H, AGENT_X:AGENT_X + PADDLE_W] = AGENT_RGB
    if s['in_play']:
      y, x = s['ball_y'], s['ball_x']
      f[y:y + BALL, x:x + BALL] = WHITE
    return f

  def get_state(self):
    return dict(self.state)

  def set_state(self, state):
    self.state = dict(state)


def random_policy_returns(num_episodes, seed=0, num_actions=6, action_repeat=4):
  """Episode returns of a uniformly random policy that repeats each action `action_repeat` frames, as the agents act."""
  rs = np.random.RandomState(seed)
  env = PongOracle(seed, num_actions=num_actions)
  returns = []
  for _ in range(num_episodes):
    env.reset()
    total, t, action = 0.0, 0, 0
    while True:
      if t % action_repeat == 0:
        action = int(rs.randint(num_actions))
      st, r, _, _ = env.advance(action)
      total += r
      t += 1
      if st == LAST:
        break
    returns.append(total)
  return np.array(returns)
