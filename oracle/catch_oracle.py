"""numpy restatement of the device Catch game (dqn_zoo_b200/csrc/dz_env.cu, DESIGN.md §10), one stream at a time.
TEST INFRASTRUCTURE ONLY.

Catch has no reference implementation: this module pins the project's own definition of the game, and the kernel and
its host-compiled twin are tested against it.  Frames are drawn by plain array slicing; the randomness is
`oracle.jax_prng_oracle.threefry2x32`.

Rules.  Frame 210x160 RGB on a (24, 26, 167) background.  Paddle 16x4 px, (200, 72, 72), top row y = 188, x in
[0, 144], centred (x = 72) at a reset.  Ball 8x8 px, (236, 236, 236), drawn last.  Remaining lives: blocks of 8x6 px,
(92, 186, 92), at x = 8 + 12 i, y in [4, 10).  Actions: 1 moves the paddle 3 px left, 2 moves it 3 px right (clamped),
every other action leaves it.  A frame moves the paddle, then the ball: a ball that landed on the previous frame is
replaced by a new one at y = 0 (no move, no reward); otherwise the ball falls 2 px and moves dx px, reflecting off the
side walls, and lands when y reaches 180 (its bottom on the paddle's top row): +1 if it overlaps the paddle
horizontally, else -1 and one life less.  An episode has 3 lives and 20 balls; it ends (LAST, discount 0) on the frame
that takes lives or balls to 0.  A reset spawns a ball and simulates k no-op frames, k uniform in [min, max] (no ball
can land: max <= 89).  Randomness: key = threefry2x32((0, seed), (stream, 0)); a reset draws
threefry2x32(key, (counter, 0)), a ball threefry2x32(key, (counter, 1)), each advancing counter; a draw below n of 32
bits u is floor(u * n / 2^32)."""

import numpy as np

from oracle import jax_prng_oracle as jp

HEIGHT, WIDTH = 210, 160
PADDLE_W, PADDLE_H, PADDLE_Y, PADDLE_STEP = 16, 4, 188, 3
BALL, FALL, LAND_Y = 8, 2, 180
LIVES, BALLS = 3, 20
MAX_NOOP_STEPS = 89
BACKGROUND, PADDLE, BALL_RGB, LIFE = (24, 26, 167), (200, 72, 72), (236, 236, 236), (92, 186, 92)
FIRST, MID, LAST = 0, 1, 2
FIELDS = ('paddle_x', 'ball_x', 'ball_y', 'ball_dx', 'lives', 'balls_left', 'counter', 'noops', 'over')


def check_noops(min_noop_steps, max_noop_steps):
  if not 0 <= min_noop_steps <= max_noop_steps:
    raise ValueError('need 0 <= min_noop_steps <= max_noop_steps, got %d, %d' % (min_noop_steps, max_noop_steps))
  if max_noop_steps > MAX_NOOP_STEPS:
    raise ValueError('max_noop_steps %d > %d: a ball could land during the no-op frames of a reset'
                     % (max_noop_steps, MAX_NOOP_STEPS))


def _below(u, n):
  return (int(u) * int(n)) >> 32


class CatchOracle:
  """One stream.  `state` is the dict of the device state fields; `step` / `reset` return
  (frame uint8 [210, 160, 3], step_type, reward, discount, lives) with reward / discount None on FIRST."""

  def __init__(self, seed, stream=0, num_actions=6, min_noop_steps=1, max_noop_steps=30):
    check_noops(min_noop_steps, max_noop_steps)
    if not 3 <= num_actions <= 18:
      raise ValueError('num_actions must be in [3, 18]')
    self.num_actions = num_actions
    self._min, self._max = min_noop_steps, max_noop_steps
    self._key = jp.threefry2x32((0, seed), (stream, 0))
    self.state = dict.fromkeys(FIELDS, 0)
    self.state['over'] = 1

  def _spawn(self):
    s = self.state
    o0, o1 = jp.threefry2x32(self._key, (s['counter'], 1))
    s['counter'] += 1
    s['ball_x'] = _below(o0, WIDTH - BALL + 1)
    s['ball_dx'] = _below(o1, 3) - 1
    s['ball_y'] = 0

  def _frame(self, action):
    s = self.state
    if action == 1:
      s['paddle_x'] = max(s['paddle_x'] - PADDLE_STEP, 0)
    elif action == 2:
      s['paddle_x'] = min(s['paddle_x'] + PADDLE_STEP, WIDTH - PADDLE_W)
    if s['ball_y'] >= LAND_Y:
      self._spawn()
      return 0
    s['ball_y'] += FALL
    x = s['ball_x'] + s['ball_dx']
    if x < 0 or x > WIDTH - BALL:
      x = -x if x < 0 else 2 * (WIDTH - BALL) - x
      s['ball_dx'] = -s['ball_dx']
    s['ball_x'] = x
    if s['ball_y'] != LAND_Y:
      return 0
    s['balls_left'] -= 1
    if s['paddle_x'] - BALL < x < s['paddle_x'] + PADDLE_W:
      return 1
    s['lives'] -= 1
    return -1

  def reset(self):
    s = self.state
    o0, _ = jp.threefry2x32(self._key, (s['counter'], 0))
    s['counter'] += 1
    k = self._min + _below(o0, self._max - self._min + 1)
    s.update(paddle_x=(WIDTH - PADDLE_W) // 2, lives=LIVES, balls_left=BALLS, over=0)
    self._spawn()
    for _ in range(k):
      self._frame(0)
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
    s['over'] = int(s['lives'] == 0 or s['balls_left'] == 0)
    return LAST if s['over'] else MID, float(r), 0.0 if s['over'] else 1.0, s['lives']

  def render(self):
    s = self.state
    f = np.empty((HEIGHT, WIDTH, 3), np.uint8)
    f[:] = BACKGROUND
    for i in range(s['lives']):
      f[4:10, 8 + 12 * i:16 + 12 * i] = LIFE
    f[PADDLE_Y:PADDLE_Y + PADDLE_H, s['paddle_x']:s['paddle_x'] + PADDLE_W] = PADDLE
    y, x = s['ball_y'], s['ball_x']
    f[y:y + BALL, x:x + BALL] = BALL_RGB
    return f

  def get_state(self):
    return dict(self.state)

  def set_state(self, state):
    self.state = dict(state)


def random_policy_returns(num_episodes, seed=0, num_actions=6, action_repeat=4):
  """Episode returns of a uniformly random policy that repeats each action `action_repeat` frames, as the agents act."""
  rs = np.random.RandomState(seed)
  env = CatchOracle(seed, num_actions=num_actions)
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
