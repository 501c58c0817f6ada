"""CPU: the Catch game (DESIGN.md §10) — hand-built scenarios on the numpy oracle (oracle/catch_oracle.py), the
host-compiled twin of the kernel's tick and picture (dz_test_catch_step) against the oracle, argument errors, and the
random-policy baseline the GPU learning test is compared with."""

import ctypes as C

import numpy as np
import pytest

from dqn_zoo_b200 import _lib
from oracle import catch_oracle as co

FIELDS = _lib.CATCH_STATE_FIELDS


def _playing(**fields):
  env = co.CatchOracle(seed=5)
  env.reset()
  env.state.update(fields)
  return env


def test_state_fields_match_the_c_abi():
  assert co.FIELDS == FIELDS
  assert co.MAX_NOOP_STEPS == _lib.CATCH_MAX_NOOP_STEPS


def test_paddle_under_a_straight_falling_ball_scores():
  env = _playing(ball_x=70, ball_dx=0, ball_y=170, paddle_x=66)
  for _ in range(4):
    assert env.step(0)[1:] == (co.MID, 0.0, 1.0, 3)
  frame, st, r, d, lives = env.step(0)
  assert (st, r, d, lives) == (co.MID, 1.0, 1.0, 3)
  assert env.state['ball_y'] == co.LAND_Y and env.state['balls_left'] == co.BALLS - 1
  assert (frame[co.LAND_Y:co.LAND_Y + 8, 70:78] == co.BALL_RGB).all()
  assert (frame[co.PADDLE_Y:co.PADDLE_Y + 4, 66:82] == co.PADDLE).all()
  env.step(0)                                      # the next frame spawns a new ball at the top
  assert env.state['ball_y'] == 0 and env.state['counter'] == 3


@pytest.mark.parametrize('paddle_x,ball_x,reward', [(0, 100, -1.0), (92, 100, 1.0), (93, 100, 1.0), (84, 100, -1.0),
                                                    (107, 100, 1.0), (108, 100, -1.0)])
def test_overlap_edges(paddle_x, ball_x, reward):
  env = _playing(ball_x=ball_x, ball_dx=0, ball_y=178, paddle_x=paddle_x)
  assert env.step(0)[2] == reward


def test_a_miss_costs_a_life_but_not_the_episode():
  env = _playing(ball_x=100, ball_dx=0, ball_y=178, paddle_x=0)
  frame, st, r, d, lives = env.step(0)
  assert (st, r, d, lives) == (co.MID, -1.0, 1.0, 2)
  assert (frame[4:10, 8:16] == co.LIFE).all() and (frame[4:10, 20:28] == co.LIFE).all()
  assert (frame[4:10, 32:40] == co.BACKGROUND).all()


def test_last_when_lives_reach_zero_then_a_reset():
  env = _playing(ball_x=100, ball_dx=0, ball_y=178, paddle_x=0, lives=1)
  frame, st, r, d, lives = env.step(0)
  assert (st, r, d, lives) == (co.LAST, -1.0, 0.0, 0)
  assert (frame[4:10] == co.BACKGROUND).all()
  frame, st, r, d, lives = env.step(0)             # stepping after LAST starts a new episode
  assert (st, r, d, lives) == (co.FIRST, None, None, 3)


def test_last_when_the_twentieth_ball_lands():
  env = _playing(ball_x=70, ball_dx=0, ball_y=178, paddle_x=66, balls_left=1)
  assert env.step(0)[1:] == (co.LAST, 1.0, 0.0, 3)


@pytest.mark.parametrize('x,dx,x_after,dx_after', [(1, -1, 0, -1), (0, -1, 1, 1), (151, 1, 152, 1), (152, 1, 151, -1),
                                                   (40, 1, 41, 1)])
def test_wall_reflection(x, dx, x_after, dx_after):
  env = _playing(ball_x=x, ball_dx=dx, ball_y=20)
  env.step(0)
  assert (env.state['ball_x'], env.state['ball_dx'], env.state['ball_y']) == (x_after, dx_after, 22)


def test_paddle_moves_and_clamps():
  env = _playing(paddle_x=4, ball_y=20)
  env.step(1)
  assert env.state['paddle_x'] == 1
  env.step(1)
  assert env.state['paddle_x'] == 0
  env.state['paddle_x'] = 142
  env.step(2)
  assert env.state['paddle_x'] == 144
  env.step(2)
  assert env.state['paddle_x'] == 144


@pytest.mark.parametrize('num_actions', [3, 6, 18])
def test_actions_from_three_up_leave_the_paddle(num_actions):
  env = co.CatchOracle(seed=9, num_actions=num_actions)
  env.reset()
  ref = co.CatchOracle(seed=9, num_actions=num_actions)
  ref.reset()
  rs = np.random.RandomState(0)
  for _ in range(300):
    a = int(rs.randint(num_actions))
    out, want = env.step(a), ref.step(a if a < 3 else 0)
    assert out[1:] == want[1:] and np.array_equal(out[0], want[0])
  with pytest.raises(ValueError):
    env.step(num_actions)


@pytest.mark.parametrize('lo,hi', [(1, 30), (0, 0), (7, 7), (0, 89)])
def test_noop_starts(lo, hi):
  env = co.CatchOracle(seed=3, min_noop_steps=lo, max_noop_steps=hi)
  seen = set()
  for _ in range(60):
    frame, st, r, d, lives = env.reset()
    k = env.state['noops']
    seen.add(k)
    assert lo <= k <= hi and (st, r, d, lives) == (co.FIRST, None, None, 3)
    assert env.state['ball_y'] == 2 * k                # the FIRST frame is the last no-op frame
    assert np.array_equal(frame, env.render())
  assert len(seen) > (1 if hi > lo else 0) or hi == lo


@pytest.mark.parametrize('lo,hi', [(0, 90), (1, 200), (5, 4), (-1, 3)])
def test_impossible_noop_ranges_are_rejected(lo, hi):
  with pytest.raises(ValueError):
    co.CatchOracle(seed=0, min_noop_steps=lo, max_noop_steps=hi)
  from dqn_zoo_b200 import environments
  with pytest.raises(ValueError):
    environments.VectorCatch(4, seed=0, min_noop_steps=lo, max_noop_steps=hi)


def _twin(cfg, state, action, reset, render=True):
  frame = np.empty((co.HEIGHT, co.WIDTH, 3), np.uint8) if render else None
  rec = np.zeros(4, np.int32)
  _lib.call('dz_test_catch_step', C.byref(cfg), state.ctypes.data, int(action), int(reset),
            frame.ctypes.data if render else None, rec.ctypes.data)
  return frame, rec


@pytest.mark.parametrize('seed,num_actions,lo,hi', [(1, 6, 1, 30), (77, 3, 0, 89), (2 ** 32 - 1, 18, 0, 0)])
def test_host_twin_equals_the_oracle(seed, num_actions, lo, hi):
  """Several thousand frames over 12 streams (offsets up to 2^32 - 1), random actions and resets: frames bit-identical,
  scalars and every state field exact."""
  rs = np.random.RandomState(seed % 1000)
  for stream in (0, 1, 2, 5, 100, 4095, 65536, 2 ** 31, 2 ** 32 - 12, 2 ** 32 - 5, 2 ** 32 - 2, 2 ** 32 - 1):
    cfg = _lib.CatchConfig(1, num_actions, lo, hi, seed, stream)
    state = np.zeros(len(FIELDS), np.int32)
    state[FIELDS.index('over')] = 1
    ref = co.CatchOracle(seed, stream, num_actions, lo, hi)
    for t in range(250):
      reset = t == 0 or rs.uniform() < 0.01
      a = int(rs.randint(num_actions))
      render = t % 5 == 0 or reset
      frame, rec = _twin(cfg, state, a, reset, render)
      want = ref.reset() if reset else ref.step(a)
      st, r, d, lives = want[1:]
      assert rec.tolist() == [st, 0 if r is None else int(r), 0 if d is None else int(d), lives]
      assert state.tolist() == [ref.state[k] for k in FIELDS]
      if render:
        assert np.array_equal(frame, want[0])


def test_host_twin_plays_whole_episodes_like_the_oracle():
  """A paddle that follows the ball: long episodes, every ball lands, episode ends on the 20th ball."""
  cfg = _lib.CatchConfig(1, 6, 1, 30, 11, 3)
  state = np.zeros(len(FIELDS), np.int32)
  state[FIELDS.index('over')] = 1
  ref = co.CatchOracle(11, 3)
  ends = 0
  for t in range(6000):
    s = ref.state
    a = 2 if s['paddle_x'] + 4 < s['ball_x'] else 1 if s['paddle_x'] > s['ball_x'] + 4 else 0
    frame, rec = _twin(cfg, state, a, t == 0, render=t % 50 == 0)
    want = ref.reset() if t == 0 else ref.step(a)
    assert rec[0] == want[1] and state.tolist() == [ref.state[k] for k in FIELDS]
    if t % 50 == 0:
      assert np.array_equal(frame, want[0])
    ends += want[1] == co.LAST
  assert ends >= 2


def test_host_twin_rejects_bad_arguments():
  state = np.zeros(len(FIELDS), np.int32)
  rec = np.zeros(4, np.int32)
  for cfg, action in [(_lib.CatchConfig(1, 6, 1, 30, 0, 0), 6), (_lib.CatchConfig(1, 6, 1, 30, 0, 0), -1),
                      (_lib.CatchConfig(1, 2, 1, 30, 0, 0), 0), (_lib.CatchConfig(1, 19, 1, 30, 0, 0), 0),
                      (_lib.CatchConfig(1, 6, 1, 90, 0, 0), 0), (_lib.CatchConfig(1, 6, 3, 2, 0, 0), 0)]:
    with pytest.raises(ValueError):
      _lib.call('dz_test_catch_step', C.byref(cfg), state.ctypes.data, action, 0, None, rec.ctypes.data)


def test_random_policy_baseline():
  """The mean return of a uniformly random policy (actions repeated 4 frames) over 1,000 episodes: the baseline of the
  GPU learning test (DESIGN.md §7).  Measured: -2.51."""
  returns = co.random_policy_returns(1000, seed=0)
  assert returns.min() >= -3 and returns.max() <= 20
  assert -2.7 < returns.mean() < -2.3
