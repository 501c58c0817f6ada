"""CPU: the Breakout game (DESIGN.md §11) — hand-built scenarios on the numpy oracle (oracle/breakout_oracle.py), the
host-compiled twin of the kernel's tick and picture (dz_test_breakout_step) against the oracle, argument errors, and
the random-policy baseline the GPU learning test is compared with."""

import ctypes as C

import numpy as np
import pytest

from dqn_zoo_b200 import _lib
from oracle import breakout_oracle as bo
from oracle import processors_oracle as po

FIELDS = _lib.BREAKOUT_STATE_FIELDS
NOOP, FIRE, RIGHT, LEFT = bo.NOOP, bo.FIRE, bo.RIGHT, bo.LEFT


def _playing(**fields):
  """A stream just after a reset with a ball in play, then `fields` set by hand."""
  env = bo.BreakoutOracle(seed=5)
  env.reset()
  env.state.update(in_play=1, ball_x=80, ball_y=120, ball_dx=1, ball_dy=2)
  env.state.update(fields)
  return env


def _rows(env):
  return [env.state['row%d' % r] for r in range(bo.ROWS)]


def test_state_fields_match_the_c_abi():
  assert bo.FIELDS == FIELDS
  assert bo.MAX_NOOP_STEPS == _lib.BREAKOUT_MAX_NOOP_STEPS < bo.SERVE_DELAY
  assert sum(bo.POINTS) * bo.COLS == 432


def test_a_reset_waits_for_a_serve():
  env = bo.BreakoutOracle(seed=2)
  frame, st, r, d, lives = env.reset()
  s = env.state
  assert (st, r, d, lives) == (bo.FIRST, None, None, 5)
  assert s['in_play'] == 0 and s['serve_timer'] == bo.SERVE_DELAY - s['noops'] and s['paddle_x'] == 72
  assert _rows(env) == [bo.FULL_ROW] * bo.ROWS
  assert (frame == bo.BALL_RGB).all(axis=2).sum() == 0
  assert (frame[57:63, 8:16] == bo.BRICK_RGB[0]).all() and (frame[87:93, 144:152] == bo.BRICK_RGB[5]).all()
  assert (frame[17:25] == bo.GREY).all() and (frame[25:196, :8] == bo.GREY).all()
  assert (frame[25:196, 152:] == bo.GREY).all() and (frame[196:] == 0).all()
  assert (frame[189:193, 72:88] == bo.PADDLE).all()
  for i in range(5):
    assert (frame[4:10, 8 + 12 * i:16 + 12 * i] == bo.GREY).all()


def test_serve_by_fire():
  env = bo.BreakoutOracle(seed=2)
  env.reset()
  counter = env.state['counter']
  frame, st, r, d, lives = env.step(FIRE)
  s = env.state
  assert (st, r, d, lives) == (bo.MID, 0.0, 1.0, 5)
  assert s['in_play'] == 1 and s['ball_y'] == bo.SERVE_Y and s['ball_dy'] == 2 and s['counter'] == counter + 1
  assert 8 <= s['ball_x'] <= 148 and s['ball_dx'] in (-2, -1, 1, 2)
  assert (frame[100:104, s['ball_x']:s['ball_x'] + 4] == bo.BALL_RGB).all()
  env.step(NOOP)                                   # the ball moves from the next frame on
  assert env.state['ball_y'] == bo.SERVE_Y + 2


def test_serve_by_the_timer():
  env = bo.BreakoutOracle(seed=4)
  env.reset()
  left = env.state['serve_timer']
  for _ in range(left - 1):
    env.step(RIGHT)
    assert env.state['in_play'] == 0
  env.step(LEFT)
  assert env.state['in_play'] == 1 and env.state['ball_y'] == bo.SERVE_Y


def test_serves_cover_positions_and_directions():
  env = bo.BreakoutOracle(seed=8)
  xs, dxs = set(), set()
  for _ in range(200):
    env.reset()
    env.step(FIRE)
    xs.add(env.state['ball_x'])
    dxs.add(env.state['ball_dx'])
  assert dxs == {-2, -1, 1, 2} and min(xs) < 30 and max(xs) > 126


@pytest.mark.parametrize('x,dx,x_after,dx_after', [(9, -2, 9, 2), (8, -1, 9, 1), (147, 2, 147, -2), (148, 1, 147, -1),
                                                   (40, 1, 41, 1), (10, -2, 8, -2)])
def test_side_wall_reflection(x, dx, x_after, dx_after):
  env = _playing(ball_x=x, ball_dx=dx, ball_y=120)
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx'], env.state['ball_y']) == (x_after, dx_after, 122)


@pytest.mark.parametrize('y,dy,y_after,dy_after', [(26, -3, 27, 3), (27, -2, 25, -2), (25, -2, 27, 2)])
def test_top_wall_reflection(y, dy, y_after, dy_after):
  env = _playing(ball_y=y, ball_dy=dy, ball_x=80, ball_dx=1)
  env.state.update({'row%d' % r: 0 for r in range(bo.ROWS)})
  env.state['row0'] = 1                          # a brick far from the ball, so the episode goes on
  assert env.step(NOOP)[1:3] == (bo.MID, 0.0)
  assert (env.state['ball_y'], env.state['ball_dy']) == (y_after, dy_after)


@pytest.mark.parametrize('row,points,dy_after', [(5, 1, 2), (4, 1, 2), (3, 4, 2), (2, 4, 2), (1, 7, 3), (0, 7, 3)])
def test_a_brick_hit_in_each_points_class(row, points, dy_after):
  """A rising ball under brick (row, 4) with the rows below it cleared: the brick goes, its points are the reward, dy
  is negated (and 3 after rows 0-1)."""
  env = _playing(ball_x=40, ball_dx=1, ball_y=bo.BRICK_Y + 6 * row + 7, ball_dy=-2)
  env.state.update({'row%d' % r: 0 for r in range(row + 1, bo.ROWS)})
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d) == (bo.MID, float(points), 1.0)
  assert env.state['row%d' % row] == bo.FULL_ROW & ~(1 << 4) and env.state['ball_dy'] == dy_after
  top = bo.BRICK_Y + 6 * row
  assert (frame[top:top + 5, 40:48] == 0).all()       # the ball now covers only the brick's last row
  assert (frame[top:top + 6, 48:56] == bo.BRICK_RGB[row]).all()


def test_exactly_one_brick_per_frame_bottom_row_then_left_column():
  env = _playing(ball_x=53, ball_dx=1, ball_y=75, ball_dy=-2)   # moves to (54, 73): bricks (2, 5), (2, 6), (3, 5), (3, 6)
  assert env.step(NOOP)[2] == 4.0
  assert env.state['row3'] == bo.FULL_ROW & ~(1 << 5) and env.state['row2'] == bo.FULL_ROW
  assert env.state['ball_dy'] == 2
  env.state.update(ball_x=53, ball_y=75, ball_dy=-2)
  assert env.step(NOOP)[2] == 4.0                  # (3, 5) is gone: (3, 6) next
  assert env.state['row3'] == bo.FULL_ROW & ~(3 << 5) and env.state['row2'] == bo.FULL_ROW
  env.state.update(ball_x=53, ball_y=75, ball_dy=-2)
  assert env.step(NOOP)[2] == 4.0                  # row 3 is open under the ball: (2, 5)
  assert env.state['row2'] == bo.FULL_ROW & ~(1 << 5)


def test_the_speed_up_lasts_until_the_ball_is_lost():
  env = _playing(ball_x=40, ball_dx=1, ball_y=bo.BRICK_Y + 13, ball_dy=-2)
  env.state.update({'row%d' % r: 0 for r in range(2, bo.ROWS)})
  assert env.step(NOOP)[2] == 7.0 and env.state['ball_dy'] == 3
  env.state.update(ball_y=184, paddle_x=40)        # a paddle bounce keeps |dy| = 3
  env.step(NOOP)
  assert env.state['ball_dy'] == -3
  env.state.update(ball_y=195, ball_dy=3)
  env.step(NOOP)
  assert env.state['in_play'] == 0
  env.step(FIRE)
  assert env.state['ball_dy'] == 2


@pytest.mark.parametrize('offset,dx', [(-3, -2), (1, -2), (2, -1), (6, -1), (7, 1), (11, 1), (12, 2), (15, 2)])
def test_paddle_zones(offset, dx):
  env = _playing(paddle_x=60, ball_x=60 + offset - 1, ball_dx=1, ball_y=184, ball_dy=2)
  assert env.step(NOOP)[1:3] == (bo.MID, 0.0)
  assert (env.state['ball_y'], env.state['ball_dy'], env.state['ball_dx']) == (185, -2, dx)


@pytest.mark.parametrize('offset', [-4, 16])
def test_a_ball_beside_the_paddle_falls_through(offset):
  env = _playing(paddle_x=60, ball_x=60 + offset - 1, ball_dx=1, ball_y=184, ball_dy=2)
  env.step(NOOP)
  assert (env.state['ball_y'], env.state['ball_dy']) == (186, 2)


def test_only_a_ball_crossing_the_top_row_bounces():
  env = _playing(paddle_x=60, ball_x=60, ball_dx=1, ball_y=186, ball_dy=2)   # already below the paddle's top row
  env.step(NOOP)
  assert (env.state['ball_y'], env.state['ball_dy']) == (188, 2)


def test_a_miss_costs_a_life_but_not_the_episode():
  env = _playing(ball_x=100, ball_dx=1, ball_y=194, ball_dy=2, paddle_x=8)
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (bo.MID, 0.0, 1.0, 4)
  assert env.state['in_play'] == 0 and env.state['serve_timer'] == bo.SERVE_DELAY
  assert (frame == bo.BALL_RGB).all(axis=2).sum() == 0
  assert (frame[4:10, 8 + 36:16 + 36] == bo.GREY).all() and (frame[4:10, 8 + 48:16 + 48] == 0).all()


def test_last_on_the_last_life_then_a_reset():
  env = _playing(ball_x=100, ball_dx=1, ball_y=194, ball_dy=2, paddle_x=8, lives=1)
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (bo.LAST, 0.0, 0.0, 0)
  assert (frame[4:10] == 0).all()
  frame, st, r, d, lives = env.step(NOOP)          # stepping after LAST starts a new episode
  assert (st, r, d, lives) == (bo.FIRST, None, None, 5)
  assert _rows(env) == [bo.FULL_ROW] * bo.ROWS


def test_last_on_the_last_brick():
  env = _playing(ball_x=40, ball_dx=1, ball_y=bo.BRICK_Y + 37, ball_dy=-2)
  env.state.update({'row%d' % r: 0 for r in range(bo.ROWS)})
  env.state['row5'] = 1 << 4
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (bo.LAST, 1.0, 0.0, 5)
  assert not (frame[57:93, 8:152] == bo.BRICK_RGB[5]).all(axis=2).any()


def test_paddle_moves_and_clamps():
  env = _playing(paddle_x=14)
  env.step(LEFT)
  assert env.state['paddle_x'] == 10
  env.step(LEFT)
  assert env.state['paddle_x'] == 8
  env.state['paddle_x'] = 134
  env.step(RIGHT)
  assert env.state['paddle_x'] == 136
  env.step(RIGHT)
  assert env.state['paddle_x'] == 136


@pytest.mark.parametrize('num_actions', [4, 6, 18])
def test_actions_from_four_up_do_nothing(num_actions):
  env = bo.BreakoutOracle(seed=9, num_actions=num_actions)
  env.reset()
  ref = bo.BreakoutOracle(seed=9, num_actions=num_actions)
  ref.reset()
  rs = np.random.RandomState(0)
  for _ in range(600):
    a = int(rs.randint(num_actions))
    out, want = env.step(a), ref.step(a if a < 4 else 0)
    assert out[1:] == want[1:] and np.array_equal(out[0], want[0])
  with pytest.raises(ValueError):
    env.step(num_actions)


@pytest.mark.parametrize('lo,hi', [(1, 30), (0, 0), (7, 7), (0, 63)])
def test_noop_starts(lo, hi):
  env = bo.BreakoutOracle(seed=3, min_noop_steps=lo, max_noop_steps=hi)
  seen = set()
  for _ in range(60):
    frame, st, r, d, lives = env.reset()
    k = env.state['noops']
    seen.add(k)
    assert lo <= k <= hi and (st, r, d, lives) == (bo.FIRST, None, None, 5)
    assert env.state['in_play'] == 0 and env.state['serve_timer'] == bo.SERVE_DELAY - k >= 1
    assert np.array_equal(frame, env.render())
  assert len(seen) > 1 or hi == lo


@pytest.mark.parametrize('lo,hi', [(0, 64), (1, 200), (5, 4), (-1, 3)])
def test_impossible_noop_ranges_are_rejected(lo, hi):
  with pytest.raises(ValueError):
    bo.BreakoutOracle(seed=0, min_noop_steps=lo, max_noop_steps=hi)
  from dqn_zoo_b200 import environments
  with pytest.raises(ValueError):
    environments.VectorBreakout(4, seed=0, min_noop_steps=lo, max_noop_steps=hi)
  state = np.zeros(len(FIELDS), np.int32)
  with pytest.raises(ValueError):
    _lib.call('dz_test_breakout_step', C.byref(_lib.BreakoutConfig(1, 4, lo, hi, 0, 0)), state.ctypes.data, 0, 1,
              None, np.zeros(4, np.int32).ctypes.data)


def test_the_ball_survives_the_84x84_resize():
  """Every in-play position of the ball on an empty field changes the preprocessed 84x84 frame by at least 100 grey
  levels somewhere (measured: 162), so the agents can see it."""
  env = bo.BreakoutOracle(seed=3)
  env.reset()
  env.state.update({'row%d' % r: 0 for r in range(bo.ROWS)})
  blank = env.render()
  base = po.pooled_gray_resized(blank, blank).astype(int)
  worst = 255
  for y in range(bo.FIELD_TOP, 186, 3):
    for x in range(bo.BALL_MIN, bo.BALL_MAX + 1, 1 if y < 30 else 5):
      env.state.update(in_play=1, ball_x=x, ball_y=y)
      f = env.render()
      worst = min(worst, np.abs(po.pooled_gray_resized(f, f).astype(int) - base).max())
  assert worst >= 100


def _twin(cfg, state, action, reset, render=True):
  frame = np.empty((bo.HEIGHT, bo.WIDTH, 3), np.uint8) if render else None
  rec = np.zeros(4, np.int32)
  _lib.call('dz_test_breakout_step', C.byref(cfg), state.ctypes.data, int(action), int(reset),
            frame.ctypes.data if render else None, rec.ctypes.data)
  return frame, rec


def _new_state():
  state = np.zeros(len(FIELDS), np.int32)
  state[FIELDS.index('over')] = 1
  return state


@pytest.mark.parametrize('seed,num_actions,lo,hi', [(1, 4, 1, 30), (77, 6, 0, 63), (2 ** 32 - 1, 18, 0, 0)])
def test_host_twin_equals_the_oracle(seed, num_actions, lo, hi):
  """Thousands of frames over 12 streams (offsets up to 2^32 - 1), random FIRE-heavy actions and resets: frames
  bit-identical, scalars and every state field exact."""
  rs = np.random.RandomState(seed % 1000)
  p = np.full(num_actions, 0.5 / (num_actions - 1))
  p[FIRE] = 0.5
  for stream in (0, 1, 2, 5, 100, 4095, 65536, 2 ** 31, 2 ** 32 - 12, 2 ** 32 - 5, 2 ** 32 - 2, 2 ** 32 - 1):
    cfg = _lib.BreakoutConfig(1, num_actions, lo, hi, seed, stream)
    state = _new_state()
    ref = bo.BreakoutOracle(seed, stream, num_actions, lo, hi)
    for t in range(400):
      reset = t == 0 or rs.uniform() < 0.005
      a = int(rs.choice(num_actions, p=p))
      render = t % 5 == 0 or reset
      frame, rec = _twin(cfg, state, a, reset, render)
      want = ref.reset() if reset else ref.step(a)
      st, r, d, lives = want[1:]
      assert rec.tolist() == [st, 0 if r is None else int(r), 0 if d is None else int(d), lives]
      assert state.tolist() == [ref.state[k] for k in FIELDS]
      if render:
        assert np.array_equal(frame, want[0])


def _tracker(s, rs):
  """FIRE when the ball is out of play, else follow the ball with a random aim (so that the bounces vary)."""
  if not s['in_play']:
    return FIRE
  aim = s['ball_x'] - s['paddle_x'] - int(rs.randint(-3, 14))
  return RIGHT if aim > 2 else LEFT if aim < -2 else NOOP


def test_host_twin_plays_whole_episodes_like_the_oracle():
  """A paddle that follows the ball: long episodes that clear bricks in every row and end on their own."""
  cfg = _lib.BreakoutConfig(1, 4, 1, 30, 11, 3)
  state = _new_state()
  ref = bo.BreakoutOracle(11, 3)
  rs = np.random.RandomState(0)
  ends, rewards = 0, set()
  cleared = np.zeros(bo.ROWS, bool)
  for t in range(30000):
    a = _tracker(ref.state, rs) if t else 0
    frame, rec = _twin(cfg, state, a, t == 0, render=t % 97 == 0)
    want = ref.reset() if t == 0 else ref.step(a) if t % 97 == 0 else (None,) + ref.advance(a)
    assert rec[0] == want[1] and state.tolist() == [ref.state[k] for k in FIELDS]
    if t % 97 == 0:
      assert np.array_equal(frame, want[0])
    ends += want[1] == bo.LAST
    rewards.add(rec[1])
    cleared |= np.array([ref.state['row%d' % r] != bo.FULL_ROW for r in range(bo.ROWS)])
  assert ends >= 2 and rewards == {0, 1, 4, 7} and cleared.all()


def test_host_twin_rejects_bad_arguments():
  state = _new_state()
  rec = np.zeros(4, np.int32)
  for cfg, action in [(_lib.BreakoutConfig(1, 4, 1, 30, 0, 0), 4), (_lib.BreakoutConfig(1, 4, 1, 30, 0, 0), -1),
                      (_lib.BreakoutConfig(1, 3, 1, 30, 0, 0), 0), (_lib.BreakoutConfig(1, 19, 1, 30, 0, 0), 0),
                      (_lib.BreakoutConfig(1, 4, 1, 64, 0, 0), 0), (_lib.BreakoutConfig(1, 4, 3, 2, 0, 0), 0),
                      (_lib.BreakoutConfig(1, 4, -1, 2, 0, 0), 0)]:
    with pytest.raises(ValueError):
      _lib.call('dz_test_breakout_step', C.byref(cfg), state.ctypes.data, action, 0, None, rec.ctypes.data)
  with pytest.raises(ValueError):
    _lib.call('dz_test_breakout_step', None, state.ctypes.data, 0, 0, None, rec.ctypes.data)
  with pytest.raises(ValueError):
    _lib.call('dz_test_breakout_step', C.byref(_lib.BreakoutConfig(1, 4, 1, 30, 0, 0)), None, 0, 0, None,
              rec.ctypes.data)


def test_breakout_and_catch_streams_do_not_share_draws():
  from oracle import catch_oracle as co
  from oracle import jax_prng_oracle as jp
  assert bo.BreakoutOracle(7, 3)._key != co.CatchOracle(7, 3)._key
  assert tuple(bo.BreakoutOracle(7, 3)._key) == tuple(jp.threefry2x32((0, 7), (3, 1)))


def test_random_policy_baseline():
  """The mean return of a uniformly random policy (actions repeated 4 frames) over 1,000 episodes: the baseline of the
  GPU learning test (DESIGN.md §7).  Measured: 0.823, with 47% of the episodes at 0 and the best at 24."""
  returns = bo.random_policy_returns(1000, seed=0)
  assert returns.min() >= 0 and returns.max() <= 432
  assert 0.75 < returns.mean() < 0.9
