"""CPU: the Pong game (DESIGN.md §12) — hand-built scenarios on the numpy oracle (oracle/pong_oracle.py), the
host-compiled twin of the kernel's tick and picture (dz_test_pong_step) against the oracle, the game's invariants
(an edge-aiming policy wins, a ball-centred tracker does not win every point, the random policy's mean return lies
strictly between -21 and 0), argument errors, and the random-policy baseline the GPU learning test is compared with."""

import ctypes as C

import numpy as np
import pytest

from dqn_zoo_b200 import _lib
from oracle import pong_oracle as po
from oracle import processors_oracle as pr

FIELDS = _lib.PONG_STATE_FIELDS
NOOP, FIRE, RIGHT, LEFT, RIGHTFIRE, LEFTFIRE = range(6)


def _playing(**fields):
  """A stream just after a reset with a ball in play, then `fields` set by hand."""
  env = po.PongOracle(seed=5)
  env.reset()
  env.state.update(in_play=1, ball_x=78, ball_y=100, ball_dx=2, ball_dy=1)
  env.state.update(fields)
  return env


def _reflect(y, dy, n):
  for _ in range(n):
    y += dy
    if y < po.FIELD_TOP or y > po.BALL_MAX_Y:
      y = 2 * po.FIELD_TOP - y if y < po.FIELD_TOP else 2 * po.BALL_MAX_Y - y
      dy = -dy
  return y


def edge_aim(s):
  """FIRE out of play; while the ball comes toward the agent, put the paddle where the ball will cross column 140 so
  that one of the paddle's edges returns it steeply (|dy| >= 2), choosing the edge whose return reaches the opponent's
  column farthest from the opponent; otherwise go back to the centre."""
  if not s['in_play']:
    return FIRE
  target = po.PADDLE_START
  if s['ball_dx'] > 0:
    n = (po.AGENT_X - po.BALL - s['ball_x']) // s['ball_dx'] + 1
    y_hit = _reflect(s['ball_y'], s['ball_dy'], n)
    best = -1
    for p in range(y_hit - 15, y_hit + 4):
      o = y_hit - p + po.BALL - 1
      dy = po.HIT_DY[6 * o // (po.PADDLE_H + po.BALL - 1)]
      if abs(dy) < 2 or not po.PADDLE_MIN <= p <= po.PADDLE_MAX or (p - po.PADDLE_START) % po.PADDLE_STEP:
        continue
      miss = abs(_reflect(y_hit, dy, 39) - 6 - s['opponent_y'])
      if miss > best:
        best, target = miss, p
  return RIGHT if s['paddle_y'] > target else LEFT if s['paddle_y'] < target else NOOP


def tracker(s):
  """A ball-centred tracker: FIRE out of play, else move the paddle's centre toward the ball's."""
  if not s['in_play']:
    return FIRE
  aim = s['ball_y'] - 6 - s['paddle_y']
  return LEFT if aim > 2 else RIGHT if aim < -2 else NOOP


def _play(policy, seed, frames, action_repeat):
  """(points won, points lost, games won, games lost) of `policy` over `frames` frames."""
  env = po.PongOracle(seed)
  env.reset()
  won = lost = games_won = games_lost = 0
  a = NOOP
  for t in range(frames):
    if t % action_repeat == 0:
      a = policy(env.state)
    st, r, _, _ = env.advance(a)
    won += r == 1.0
    lost += r == -1.0
    if st == po.LAST:
      games_won += env.state['agent_score'] == po.WIN
      games_lost += env.state['opponent_score'] == po.WIN
  return won, lost, games_won, games_lost


def test_state_fields_match_the_c_abi():
  assert po.FIELDS == FIELDS
  assert po.MAX_NOOP_STEPS == _lib.PONG_MAX_NOOP_STEPS < po.SERVE_DELAY


def test_a_reset_waits_for_a_serve():
  env = po.PongOracle(seed=2)
  frame, st, r, d, lives = env.reset()
  s = env.state
  assert (st, r, d, lives) == (po.FIRST, None, None, 0)
  assert s['in_play'] == 0 and s['serve_timer'] == po.SERVE_DELAY - s['noops']
  assert s['paddle_y'] == s['opponent_y'] == 106 and s['agent_score'] == s['opponent_score'] == 0
  assert (frame == po.WHITE).all(axis=2)[34:194].sum() == 0           # no ball
  assert (frame[24:34] == po.WHITE).all() and (frame[194:] == po.WHITE).all()
  assert (frame[106:122, 140:144] == po.AGENT_RGB).all() and (frame[106:122, 16:20] == po.OPP_RGB).all()
  assert (frame[34:106] == po.BACKGROUND).all() and (frame[22:24] == po.BACKGROUND).all()


@pytest.mark.parametrize('action', [FIRE, RIGHTFIRE, LEFTFIRE])
def test_serve_by_each_fire_action(action):
  env = po.PongOracle(seed=2)
  env.reset()
  counter = env.state['counter']
  frame, st, r, d, lives = env.step(action)
  s = env.state
  assert (st, r, d, lives) == (po.MID, 0.0, 1.0, 0)
  assert s['in_play'] == 1 and s['ball_x'] == po.SERVE_X and s['counter'] == counter + 1
  assert 50 <= s['ball_y'] <= 174 and s['ball_dx'] in (-2, 2) and s['ball_dy'] in (-2, -1, 1, 2)
  assert (frame[s['ball_y']:s['ball_y'] + 4, 78:82] == po.WHITE).all()
  y, dx, dy = s['ball_y'], s['ball_dx'], s['ball_dy']
  env.step(NOOP)                                   # the ball moves from the next frame on
  assert (env.state['ball_x'], env.state['ball_y']) == (78 + dx, y + dy)


def test_serve_by_the_timer():
  env = po.PongOracle(seed=4)
  env.reset()
  left = env.state['serve_timer']
  for _ in range(left - 1):
    env.step(RIGHT)
    assert env.state['in_play'] == 0
  env.step(NOOP)
  assert env.state['in_play'] == 1 and env.state['ball_x'] == po.SERVE_X


def test_serves_cover_positions_and_directions():
  env = po.PongOracle(seed=8)
  ys, dirs = set(), set()
  for _ in range(300):
    env.reset()
    env.step(FIRE)
    ys.add(env.state['ball_y'])
    dirs.add((env.state['ball_dx'], env.state['ball_dy']))
  assert len(dirs) == 8 and min(ys) < 56 and max(ys) > 168 and min(ys) >= 50 and max(ys) <= 174


@pytest.mark.parametrize('y,dy,y_after,dy_after', [(35, -2, 35, 2), (34, -1, 35, 1), (36, -2, 34, -2),
                                                   (189, 2, 189, -2), (190, 1, 189, -1), (188, 2, 190, 2)])
def test_wall_reflection(y, dy, y_after, dy_after):
  env = _playing(ball_y=y, ball_dy=dy, ball_x=78, ball_dx=2)
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_y'], env.state['ball_dy']) == (80, y_after, dy_after)


ZONES = [(0, -3), (3, -3), (4, -2), (6, -2), (7, -1), (9, -1), (10, 1), (12, 1), (13, 2), (15, 2), (16, 3), (18, 3)]


@pytest.mark.parametrize('o,dy', ZONES)
def test_agent_paddle_zones(o, dy):
  env = _playing(paddle_y=100, ball_x=135, ball_dx=2, ball_y=100 + o - 4, ball_dy=1)
  assert env.step(NOOP)[1:] == (po.MID, 0.0, 1.0, 0)
  assert (env.state['ball_x'], env.state['ball_dx'], env.state['ball_dy']) == (136, -3, dy)


@pytest.mark.parametrize('o,dy', ZONES)
def test_opponent_paddle_zones(o, dy):
  """The opponent first moves 1 px toward ball_y - 6, then the ball (dy = +1) crosses its column at offset o."""
  b = 100
  p = b - (o - 5 if o < 10 else o - 3)
  env = _playing(opponent_y=p, ball_x=21, ball_dx=-2, ball_y=b, ball_dy=1)
  env.step(NOOP)
  assert env.state['opponent_y'] == (p - 1 if o < 10 else p + 1)
  assert env.state['ball_y'] - env.state['opponent_y'] + 3 == o
  assert (env.state['ball_x'], env.state['ball_dx'], env.state['ball_dy']) == (20, 3, dy)


@pytest.mark.parametrize('offset', [-1, 19])
def test_a_ball_beside_the_agent_paddle_passes(offset):
  env = _playing(paddle_y=100, ball_x=135, ball_dx=2, ball_y=100 + offset - 4, ball_dy=1)
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx']) == (137, 2)


def test_a_ball_beside_the_opponent_paddle_passes():
  env = _playing(opponent_y=150, ball_x=21, ball_dx=-2, ball_y=60, ball_dy=1)
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx']) == (19, -2)


def test_only_a_crossing_ball_is_returned():
  env = _playing(paddle_y=100, ball_x=137, ball_dx=2, ball_y=104, ball_dy=1)   # already past column 140
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx']) == (139, 2)
  env = _playing(paddle_y=100, ball_x=138, ball_dx=-3, ball_y=104, ball_dy=1)  # moving away
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx']) == (135, -3)
  env = _playing(opponent_y=100, ball_x=19, ball_dx=-2, ball_y=106, ball_dy=0)  # behind the opponent's column
  env.step(NOOP)
  assert (env.state['ball_x'], env.state['ball_dx']) == (17, -2)


def test_a_point_each_way():
  env = _playing(opponent_y=150, ball_x=2, ball_dx=-3, ball_y=60, ball_dy=1)
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (po.MID, 1.0, 1.0, 0)
  s = env.state
  assert (s['agent_score'], s['opponent_score'], s['in_play'], s['serve_timer']) == (1, 0, 0, po.SERVE_DELAY)
  assert (frame == po.WHITE).all(axis=2)[34:194].sum() == 0
  assert (frame[2:22, 132:144][po.glyph(1)] == po.AGENT_RGB).all()
  env = _playing(paddle_y=40, ball_x=154, ball_dx=2, ball_y=150, ball_dy=1)
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (po.MID, -1.0, 1.0, 0)
  assert (env.state['agent_score'], env.state['opponent_score'], env.state['in_play']) == (0, 1, 0)
  assert (frame[2:22, 36:48][po.glyph(1)] == po.OPP_RGB).all()


@pytest.mark.parametrize('agent_wins', [True, False])
def test_last_at_21_then_a_reset(agent_wins):
  if agent_wins:
    env = _playing(opponent_y=150, ball_x=2, ball_dx=-3, ball_y=60, agent_score=20, opponent_score=20)
  else:
    env = _playing(paddle_y=40, ball_x=154, ball_dx=2, ball_y=150, agent_score=20, opponent_score=20)
  frame, st, r, d, lives = env.step(NOOP)
  assert (st, r, d, lives) == (po.LAST, 1.0 if agent_wins else -1.0, 0.0, 0)
  assert env.state['agent_score' if agent_wins else 'opponent_score'] == 21
  frame, st, r, d, lives = env.step(FIRE)          # stepping after LAST starts a new episode
  assert (st, r, d, lives) == (po.FIRST, None, None, 0)
  assert env.state['agent_score'] == env.state['opponent_score'] == 0 and env.state['in_play'] == 0


def test_the_opponent_tracks_at_its_speed_cap_and_returns_to_the_centre():
  env = _playing(opponent_y=106, ball_x=120, ball_dx=-2, ball_y=60, ball_dy=0)
  for t in range(1, 30):
    env.step(NOOP)
    assert env.state['opponent_y'] == 106 - po.OPP_SPEED * t          # toward ball_y - 6 = 54, 1 px per frame
  env = _playing(opponent_y=60, ball_x=120, ball_dx=-2, ball_y=68, ball_dy=0)
  env.step(NOOP)
  env.step(NOOP)
  assert env.state['opponent_y'] == 62 and env.step(NOOP) is not None and env.state['opponent_y'] == 62
  env = _playing(opponent_y=60, ball_x=40, ball_dx=2, ball_y=68, ball_dy=0)   # moving right: back to 106
  for t in range(1, 20):
    env.step(NOOP)
    assert env.state['opponent_y'] == 60 + t
  env = _playing(opponent_y=40, ball_x=120, ball_dx=-2, ball_y=34, ball_dy=0)  # clamped at the top wall
  for _ in range(10):
    env.step(NOOP)
  assert env.state['opponent_y'] == 34


def test_agent_paddle_under_every_action_and_clamping():
  moves = {NOOP: 0, FIRE: 0, RIGHT: -4, LEFT: 4, RIGHTFIRE: -4, LEFTFIRE: 4}
  for a, dy in moves.items():
    env = _playing(paddle_y=100)
    env.step(a)
    assert env.state['paddle_y'] == 100 + dy, a
  env = _playing(paddle_y=38)
  env.step(RIGHT)
  assert env.state['paddle_y'] == 34
  env.step(RIGHTFIRE)
  assert env.state['paddle_y'] == 34
  env.state['paddle_y'] = 174
  env.step(LEFT)
  assert env.state['paddle_y'] == 178
  env.step(LEFTFIRE)
  assert env.state['paddle_y'] == 178


@pytest.mark.parametrize('num_actions', [6, 18])
def test_actions_from_six_up_do_nothing(num_actions):
  env = po.PongOracle(seed=9, num_actions=num_actions)
  env.reset()
  ref = po.PongOracle(seed=9, num_actions=num_actions)
  ref.reset()
  rs = np.random.RandomState(0)
  for _ in range(600):
    a = int(rs.randint(num_actions)) if rs.uniform() < 0.5 else int(rs.randint(6, 19))
    a = a if a < num_actions else NOOP
    out, want = env.step(a), ref.step(a if a < 6 else NOOP)
    assert out[1:] == want[1:] and np.array_equal(out[0], want[0])
  with pytest.raises(ValueError):
    env.step(num_actions)


@pytest.mark.parametrize('lo,hi', [(1, 30), (0, 0), (7, 7), (0, 63)])
def test_noop_starts(lo, hi):
  env = po.PongOracle(seed=3, min_noop_steps=lo, max_noop_steps=hi)
  seen = set()
  for _ in range(60):
    frame, st, r, d, lives = env.reset()
    k = env.state['noops']
    seen.add(k)
    assert lo <= k <= hi and (st, r, d, lives) == (po.FIRST, None, None, 0)
    assert env.state['in_play'] == 0 and env.state['serve_timer'] == po.SERVE_DELAY - k >= 1
    assert np.array_equal(frame, env.render())
  assert len(seen) > 1 or hi == lo


@pytest.mark.parametrize('lo,hi', [(0, 64), (1, 200), (5, 4), (-1, 3)])
def test_impossible_noop_ranges_are_rejected(lo, hi):
  with pytest.raises(ValueError):
    po.PongOracle(seed=0, min_noop_steps=lo, max_noop_steps=hi)
  from dqn_zoo_b200 import environments
  with pytest.raises(ValueError):
    environments.VectorPong(4, seed=0, min_noop_steps=lo, max_noop_steps=hi)
  state = np.zeros(len(FIELDS), np.int32)
  with pytest.raises(ValueError):
    _lib.call('dz_test_pong_step', C.byref(_lib.PongConfig(1, 6, lo, hi, 0, 0)), state.ctypes.data, 0, 1, None,
              np.zeros(4, np.int32).ctypes.data)


def test_numerals_for_every_score():
  """Scores 0 to 21 on both sides: the units digit in its cell, the tens digit only from 10 up, in the paddle's
  colour, and nothing else lit in the band."""
  env = po.PongOracle(seed=1)
  env.reset()
  for score in range(22):
    env.state.update(agent_score=score, opponent_score=21 - score)
    f = env.render()
    band = f[2:22]
    for value, (tens_x, units_x), rgb in ((21 - score, po.OPP_DIGITS_X, po.OPP_RGB),
                                          (score, po.AGENT_DIGITS_X, po.AGENT_RGB)):
      want = np.zeros((20, 28), bool)
      want[:, 16:] = po.glyph(value % 10)
      if value >= 10:
        want[:, :12] = po.glyph(value // 10)
      got = (band[:, tens_x:tens_x + 28] == rgb).all(axis=2)
      assert np.array_equal(got, want), (score, value)
    lit = ~(band == po.BACKGROUND).all(axis=2)
    assert lit.sum() == (po.glyph((21 - score) % 10).sum() + po.glyph(score % 10).sum() +
                         (po.glyph((21 - score) // 10).sum() if 21 - score >= 10 else 0) +
                         (po.glyph(score // 10).sum() if score >= 10 else 0))
  assert [po.glyph(d).sum() for d in range(10)] == [192, 80, 176, 176, 144, 176, 192, 112, 208, 192]


def test_the_ball_survives_the_84x84_resize():
  """Every in-play position of the ball off the paddles changes the preprocessed 84x84 frame by at least 100 grey
  levels somewhere (measured: 102), so the agents can see it."""
  env = po.PongOracle(seed=3)
  env.reset()
  env.state.update(paddle_y=178, opponent_y=34)
  blank = env.render()
  base = pr.pooled_gray_resized(blank, blank).astype(int)
  worst = 255
  for y in range(po.FIELD_TOP, po.BALL_MAX_Y + 1, 1):
    for x in range(1, po.WIDTH - po.BALL, 1 if y < 40 or y > 184 else 5):
      if (po.AGENT_X - po.BALL < x < po.AGENT_X + po.PADDLE_W and y > 178 - po.BALL) or \
         (po.OPP_X - po.BALL < x < po.OPP_X + po.PADDLE_W and y < 34 + po.PADDLE_H):
        continue
      env.state.update(in_play=1, ball_x=x, ball_y=y)
      f = env.render()
      worst = min(worst, np.abs(pr.pooled_gray_resized(f, f).astype(int) - base).max())
  assert worst >= 100


def test_an_edge_aiming_policy_wins_a_game():
  won, lost, games_won, games_lost = _play(edge_aim, seed=2, frames=12000, action_repeat=1)
  assert games_won >= 1 and games_lost == 0 and won > 4 * lost, (won, lost)


def test_a_ball_centred_tracker_does_not_win_every_point():
  """Acting every 4 frames as the agents do, the tracker returns most balls but misses some of the opponent's steep
  returns."""
  won, lost, _, _ = _play(tracker, seed=1, frames=100000, action_repeat=4)
  assert won > 0 and lost > 0, (won, lost)


def _twin(cfg, state, action, reset, render=True):
  frame = np.empty((po.HEIGHT, po.WIDTH, 3), np.uint8) if render else None
  rec = np.zeros(4, np.int32)
  _lib.call('dz_test_pong_step', C.byref(cfg), state.ctypes.data, int(action), int(reset),
            frame.ctypes.data if render else None, rec.ctypes.data)
  return frame, rec


def _new_state():
  state = np.zeros(len(FIELDS), np.int32)
  state[FIELDS.index('over')] = 1
  return state


@pytest.mark.parametrize('seed,num_actions,lo,hi', [(1, 6, 1, 30), (77, 7, 0, 63), (2 ** 32 - 1, 18, 0, 0)])
def test_host_twin_equals_the_oracle(seed, num_actions, lo, hi):
  """Thousands of frames over 12 streams (offsets up to 2^32 - 1), random FIRE-heavy actions and resets, random
  mid-game scores: frames bit-identical, scalars and every state field exact."""
  rs = np.random.RandomState(seed % 1000)
  p = np.full(num_actions, 0.4 / (num_actions - 3))
  p[[FIRE, RIGHTFIRE, LEFTFIRE]] = 0.2
  for stream in (0, 1, 2, 5, 100, 4095, 65536, 2 ** 31, 2 ** 32 - 12, 2 ** 32 - 5, 2 ** 32 - 2, 2 ** 32 - 1):
    cfg = _lib.PongConfig(1, num_actions, lo, hi, seed, stream)
    state = _new_state()
    ref = po.PongOracle(seed, stream, num_actions, lo, hi)
    for t in range(400):
      reset = t == 0 or rs.uniform() < 0.005
      a = int(rs.choice(num_actions, p=p))
      render = t % 5 == 0 or reset
      if t % 100 == 1:                             # random mid-game scores, so games end within the run
        scores = rs.randint(15, 21, size=2)
        ref.state.update(agent_score=int(scores[0]), opponent_score=int(scores[1]))
        state[FIELDS.index('agent_score')], state[FIELDS.index('opponent_score')] = scores
      frame, rec = _twin(cfg, state, a, reset, render)
      want = ref.reset() if reset else ref.step(a)
      st, r, d, lives = want[1:]
      assert rec.tolist() == [st, 0 if r is None else int(r), 0 if d is None else int(d), lives]
      assert state.tolist() == [ref.state[k] for k in FIELDS]
      if render:
        assert np.array_equal(frame, want[0])


def test_host_twin_plays_whole_games_like_the_oracle():
  """Whole games, alternately by the edge-aiming policy and by a random one (actions repeated 4 frames): both sides
  score, and games end both ways."""
  cfg = _lib.PongConfig(1, 6, 1, 30, 11, 3)
  state = _new_state()
  ref = po.PongOracle(11, 3)
  rs = np.random.RandomState(0)
  games, rewards, winners = 0, set(), set()
  a = NOOP
  for t in range(24000):
    if t and (games % 2 == 0 or t % 4 == 0):
      a = edge_aim(ref.state) if games % 2 == 0 else int(rs.randint(6))
    frame, rec = _twin(cfg, state, a, t == 0, render=t % 97 == 0)
    want = ref.reset() if t == 0 else ref.step(a) if t % 97 == 0 else (None,) + ref.advance(a)
    assert rec[0] == want[1] and state.tolist() == [ref.state[k] for k in FIELDS]
    if t % 97 == 0:
      assert np.array_equal(frame, want[0])
    rewards.add(int(rec[1]))
    if want[1] == po.LAST:
      games += 1
      winners.add(ref.state['agent_score'] == po.WIN)
  assert games >= 4 and rewards == {-1, 0, 1} and winners == {True, False}


def test_host_twin_rejects_bad_arguments():
  state = _new_state()
  rec = np.zeros(4, np.int32)
  for cfg, action in [(_lib.PongConfig(1, 6, 1, 30, 0, 0), 6), (_lib.PongConfig(1, 6, 1, 30, 0, 0), -1),
                      (_lib.PongConfig(1, 5, 1, 30, 0, 0), 0), (_lib.PongConfig(1, 19, 1, 30, 0, 0), 0),
                      (_lib.PongConfig(1, 6, 1, 64, 0, 0), 0), (_lib.PongConfig(1, 6, 3, 2, 0, 0), 0),
                      (_lib.PongConfig(1, 6, -1, 2, 0, 0), 0)]:
    with pytest.raises(ValueError):
      _lib.call('dz_test_pong_step', C.byref(cfg), state.ctypes.data, action, 0, None, rec.ctypes.data)
  with pytest.raises(ValueError):
    _lib.call('dz_test_pong_step', None, state.ctypes.data, 0, 0, None, rec.ctypes.data)
  with pytest.raises(ValueError):
    _lib.call('dz_test_pong_step', C.byref(_lib.PongConfig(1, 6, 1, 30, 0, 0)), None, 0, 0, None, rec.ctypes.data)


def test_pong_breakout_and_catch_streams_do_not_share_draws():
  from oracle import breakout_oracle as bo
  from oracle import catch_oracle as co
  from oracle import jax_prng_oracle as jp
  keys = {tuple(po.PongOracle(7, 3)._key), tuple(bo.BreakoutOracle(7, 3)._key), tuple(co.CatchOracle(7, 3)._key)}
  assert len(keys) == 3
  assert tuple(po.PongOracle(7, 3)._key) == tuple(jp.threefry2x32((0, 7), (3, 2)))


RANDOM_EPISODES = 1000


def test_random_policy_baseline():
  """The mean return of a uniformly random policy (actions repeated 4 frames) over RANDOM_EPISODES episodes: the
  baseline of the GPU learning test (DESIGN.md §7), strictly between -21 and 0.  Measured: -7.314, with 8.5% of the
  episodes at 0 or above, the worst at -19 and the best at +8."""
  returns = po.random_policy_returns(RANDOM_EPISODES, seed=0)
  assert returns.min() >= -21 and returns.max() <= 21
  assert -21 < returns.mean() < 0
  assert -7.6 < returns.mean() < -7.0, returns.mean()
