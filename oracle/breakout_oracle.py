"""numpy restatement of the device Breakout game (dqn_zoo_b200/csrc/dz_breakout.cu, DESIGN.md §11), one stream at a
time.  TEST INFRASTRUCTURE ONLY.

This is the project's own Breakout, not ALE's: it has no reference implementation, so this module pins the project's
definition of the game, and the kernel and its host-compiled twin are tested against it.  Frames are drawn by plain
array slicing; the randomness is `oracle.jax_prng_oracle.threefry2x32`.

Rules.  Frame 210x160 RGB on black.  Grey (142, 142, 142) walls: top y in [17, 25) over the whole width, sides
x in [0, 8) and [152, 160) for y in [17, 196); the field is x in [8, 152), y in [25, 196).  Remaining lives: grey blocks
of 8x6 px at x = 8 + 12 i, y in [4, 10).  Bricks: 6 rows x 18 columns of 8x6 px, brick (r, c) at x in
[8 + 8c, 16 + 8c), y in [57 + 6r, 63 + 6r), coloured by row and worth 7, 7, 4, 4, 1, 1 points (432 in all).  Paddle
16x4 px, (200, 72, 72), y in [189, 193), x in [8, 136], centred (72) after a reset, 4 px per frame.  Ball 4x4 px,
(236, 236, 236), drawn last, only while in play.  Actions: 0 NOOP, 1 FIRE, 2 RIGHT, 3 LEFT, 4.. NOOP.

A frame: (1) the paddle moves; (2) a ball out of play counts its serve timer down and is served if the action is FIRE or
the timer reaches 0: x = 8 + below(141), dx = (-2, -1, 1, 2)[below(4)], y = 100, dy = 2 (the frame ends there);
(3) a ball in play moves dx (x < 8 -> 16 - x, x > 148 -> 296 - x, dx negated), then dy (y < 25 -> 50 - y, dy negated);
(4) of the live bricks it overlaps, the one in the bottom row, then the left column, is cleared: its points are the
reward, dy is negated, and a brick of rows 0-1 raises |dy| from 2 to 3; (5) a falling ball whose bottom row crosses the
paddle's top row this frame (y_old + 4 <= 189 < y + 4) while it overlaps the paddle is put on it (y = 185), dy
negated, dx = (-2, -1, 1, 2)[4 * (x - paddle_x + 3) // 19]; (6) a ball with y >= 196 is lost: out of play, a life
less, serve timer 64, no reward.  An episode has 5 lives; it ends (LAST, discount 0) on the frame that takes the lives
to 0 or clears the last brick.  A reset: full wall, 5 lives, centred paddle, ball out of play, timer 64, then k no-op
frames, k uniform in [min, max] (max <= 63, so nothing is served).  Randomness: key =
threefry2x32((0, seed), (stream, 1)); a reset draws threefry2x32(key, (counter, 0)), a serve
threefry2x32(key, (counter, 1)), each advancing counter; a draw below n of 32 bits u is floor(u * n / 2^32)."""

import numpy as np

from oracle import jax_prng_oracle as jp

HEIGHT, WIDTH = 210, 160
WALL_TOP, FIELD_TOP, FIELD_BOTTOM, FIELD_LEFT, FIELD_RIGHT = 17, 25, 196, 8, 152
ROWS, COLS, BRICK_W, BRICK_H, BRICK_Y = 6, 18, 8, 6, 57
FULL_ROW = (1 << COLS) - 1
POINTS = (7, 7, 4, 4, 1, 1)
PADDLE_W, PADDLE_H, PADDLE_Y, PADDLE_MIN, PADDLE_MAX, PADDLE_STEP = 16, 4, 189, 8, 136, 4
BALL, BALL_MIN, BALL_MAX, SERVE_Y = 4, 8, 148, 100
SERVE_DELAY, LIVES = 64, 5
MAX_NOOP_STEPS = 63
NOOP, FIRE, RIGHT, LEFT = 0, 1, 2, 3
GREY, PADDLE, BALL_RGB = (142, 142, 142), (200, 72, 72), (236, 236, 236)
BRICK_RGB = ((200, 72, 72), (198, 108, 58), (180, 122, 48), (162, 162, 42), (72, 160, 72), (66, 72, 200))
FIRST, MID, LAST = 0, 1, 2
FIELDS = ('paddle_x', 'ball_x', 'ball_y', 'ball_dx', 'ball_dy', 'in_play', 'serve_timer', 'lives',
          'row0', 'row1', 'row2', 'row3', 'row4', 'row5', 'counter', 'noops', 'over')
GAME_TAG = 1


def check_noops(min_noop_steps, max_noop_steps):
  if not 0 <= min_noop_steps <= max_noop_steps:
    raise ValueError('need 0 <= min_noop_steps <= max_noop_steps, got %d, %d' % (min_noop_steps, max_noop_steps))
  if max_noop_steps > MAX_NOOP_STEPS:
    raise ValueError('max_noop_steps %d > %d: a ball could be served during the no-op frames of a reset'
                     % (max_noop_steps, MAX_NOOP_STEPS))


def _below(u, n):
  return (int(u) * int(n)) >> 32


class BreakoutOracle:
  """One stream.  `state` is the dict of the device state fields; `step` / `reset` return
  (frame uint8 [210, 160, 3], step_type, reward, discount, lives) with reward / discount None on FIRST."""

  def __init__(self, seed, stream=0, num_actions=4, min_noop_steps=1, max_noop_steps=30):
    check_noops(min_noop_steps, max_noop_steps)
    if not 4 <= num_actions <= 18:
      raise ValueError('num_actions must be in [4, 18]')
    self.num_actions = num_actions
    self._min, self._max = min_noop_steps, max_noop_steps
    self._key = jp.threefry2x32((0, seed), (stream, GAME_TAG))
    self.state = dict.fromkeys(FIELDS, 0)
    self.state['over'] = 1

  def _serve(self):
    s = self.state
    o0, o1 = jp.threefry2x32(self._key, (s['counter'], 1))
    s['counter'] += 1
    s.update(ball_x=BALL_MIN + _below(o0, BALL_MAX - BALL_MIN + 1), ball_dx=(-2, -1, 1, 2)[_below(o1, 4)],
             ball_y=SERVE_Y, ball_dy=2, in_play=1)

  def _hit_brick(self):
    s = self.state
    x, y = s['ball_x'], s['ball_y']
    for r in range(ROWS - 1, -1, -1):            # the bottom row first, then the left column
      top = BRICK_Y + BRICK_H * r
      if not (y < top + BRICK_H and y + BALL > top):
        continue
      for c in sorted({(x - FIELD_LEFT) // BRICK_W, (x + BALL - 1 - FIELD_LEFT) // BRICK_W}):
        if s['row%d' % r] >> c & 1:
          s['row%d' % r] &= ~(1 << c)
          dy = -s['ball_dy']
          if r < 2 and abs(dy) == 2:
            dy = 3 if dy > 0 else -3
          s['ball_dy'] = dy
          return POINTS[r]
    return 0

  def _frame(self, action):
    s = self.state
    if action == RIGHT:
      s['paddle_x'] = min(s['paddle_x'] + PADDLE_STEP, PADDLE_MAX)
    elif action == LEFT:
      s['paddle_x'] = max(s['paddle_x'] - PADDLE_STEP, PADDLE_MIN)
    if not s['in_play']:
      s['serve_timer'] -= 1
      if action == FIRE or s['serve_timer'] <= 0:
        self._serve()
      return 0
    x = s['ball_x'] + s['ball_dx']
    if x < BALL_MIN or x > BALL_MAX:
      x = 2 * BALL_MIN - x if x < BALL_MIN else 2 * BALL_MAX - x
      s['ball_dx'] = -s['ball_dx']
    s['ball_x'] = x
    y0 = s['ball_y']
    y = y0 + s['ball_dy']
    if y < FIELD_TOP:
      y = 2 * FIELD_TOP - y
      s['ball_dy'] = -s['ball_dy']
    s['ball_y'] = y
    reward = self._hit_brick()
    px = s['paddle_x']
    if (s['ball_dy'] > 0 and y0 + BALL <= PADDLE_Y < s['ball_y'] + BALL
        and px - BALL < s['ball_x'] < px + PADDLE_W):
      s['ball_y'] = PADDLE_Y - BALL
      s['ball_dy'] = -s['ball_dy']
      s['ball_dx'] = (-2, -1, 1, 2)[4 * (s['ball_x'] - px + BALL - 1) // (PADDLE_W + BALL - 1)]
    if s['ball_y'] >= FIELD_BOTTOM:
      s.update(in_play=0, lives=s['lives'] - 1, serve_timer=SERVE_DELAY)
    return reward

  def reset(self):
    s = self.state
    o0, _ = jp.threefry2x32(self._key, (s['counter'], 0))
    s['counter'] += 1
    k = self._min + _below(o0, self._max - self._min + 1)
    s.update(paddle_x=(PADDLE_MIN + PADDLE_MAX) // 2, ball_x=0, ball_y=0, ball_dx=0, ball_dy=0, in_play=0,
             serve_timer=SERVE_DELAY, lives=LIVES, over=0, **{'row%d' % r: FULL_ROW for r in range(ROWS)})
    for _ in range(k):
      self._frame(NOOP)
    s['noops'] = k
    return self.render(), FIRST, None, None, s['lives']

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
    s['over'] = int(s['lives'] == 0 or not any(s['row%d' % i] for i in range(ROWS)))
    return LAST if s['over'] else MID, float(r), 0.0 if s['over'] else 1.0, s['lives']

  def render(self):
    s = self.state
    f = np.zeros((HEIGHT, WIDTH, 3), np.uint8)
    for i in range(s['lives']):
      f[4:10, 8 + 12 * i:16 + 12 * i] = GREY
    f[WALL_TOP:FIELD_BOTTOM, :FIELD_LEFT] = GREY
    f[WALL_TOP:FIELD_BOTTOM, FIELD_RIGHT:] = GREY
    f[WALL_TOP:FIELD_TOP] = GREY
    for r in range(ROWS):
      for c in range(COLS):
        if s['row%d' % r] >> c & 1:
          f[BRICK_Y + BRICK_H * r:BRICK_Y + BRICK_H * (r + 1),
            FIELD_LEFT + BRICK_W * c:FIELD_LEFT + BRICK_W * (c + 1)] = BRICK_RGB[r]
    f[PADDLE_Y:PADDLE_Y + PADDLE_H, s['paddle_x']:s['paddle_x'] + PADDLE_W] = PADDLE
    if s['in_play']:
      y, x = s['ball_y'], s['ball_x']
      f[y:y + BALL, x:x + BALL] = BALL_RGB
    return f

  def get_state(self):
    return dict(self.state)

  def set_state(self, state):
    self.state = dict(state)


def random_policy_returns(num_episodes, seed=0, num_actions=4, action_repeat=4):
  """Episode returns of a uniformly random policy that repeats each action `action_repeat` frames, as the agents act."""
  rs = np.random.RandomState(seed)
  env = BreakoutOracle(seed, num_actions=num_actions)
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
