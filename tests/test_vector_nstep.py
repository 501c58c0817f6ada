"""CPU: `replay.VectorNStepAccumulator` (E n-step accumulators as array code) against E per-stream
`oracle.replay_oracle.NStepTransitionAccumulator`s over random interleaved episodes: idle streams, episodes shorter than
n, FIRST straight after LAST, observations overwritten in place between ticks.  Every emitted transition matches in
order, bytes, action and bit-exact float64 return and discount."""

import numpy as np
import pytest
import torch

from oracle import frame_pool_oracle as fpo
from oracle import replay_oracle as ro

OBS = (3, 4, 2)


def _ticks(seed, E, num_ticks):
  """Per tick: (emit, step_type, reward, discount, observations, actions), struct-of-arrays as
  `VectorizedAtariPreprocessor.step_arrays` emits them; the observation array is reused and overwritten in place."""
  rs = np.random.RandomState(seed)
  remaining = np.full(E, -1)     # -1: the next emitted timestep starts an episode
  obs = np.zeros((E,) + OBS, np.uint8)
  out = []
  for _ in range(num_ticks):
    emit = rs.rand(E) < 0.6
    emit[E - 1] = False          # one stream stays idle throughout
    st = np.ones(E, np.int64)
    rw = rs.choice([-1.0, 0.0, 0.5, 1.0, 0.1], size=E)
    dc = rs.choice([0.99, 0.0, 0.9, 1.0 / 3.0], size=E)
    for e in np.nonzero(emit)[0]:
      if remaining[e] < 0:
        st[e] = 0
        remaining[e] = rs.randint(1, 9)    # episodes of 1..8 transitions, some shorter than n
      else:
        remaining[e] -= 1
        if remaining[e] == 0:
          st[e] = 2
          remaining[e] = -1
    rw[st == 0] = np.nan
    dc[st == 0] = np.nan
    obs[emit] = rs.randint(0, 256, size=(int(emit.sum()),) + OBS)
    out.append((emit, st, rw, dc, obs, rs.randint(0, 6, size=E)))
  return out


def _assert_same(got, want):
  if not want:
    assert got is None
    return
  assert got is not None and len(got.r_t) == len(want)
  np.testing.assert_array_equal(got.s_tm1.numpy(), np.stack([w.s_tm1 for w in want]))
  np.testing.assert_array_equal(got.s_t.numpy(), np.stack([w.s_t for w in want]))
  np.testing.assert_array_equal(got.a_tm1, [w.a_tm1 for w in want])
  assert np.asarray(got.r_t, np.float64).tobytes() == np.asarray([w.r_t for w in want], np.float64).tobytes()
  assert np.asarray(got.discount_t, np.float64).tobytes() == np.asarray([w.discount_t for w in want], np.float64).tobytes()


@pytest.mark.parametrize('n', [1, 3, 5])
@pytest.mark.parametrize('seed', [0, 1])
def test_matches_per_stream_accumulators(n, seed):
  from dqn_zoo_b200 import replay as dr
  E = 5
  acc = dr.VectorNStepAccumulator(E, n, device='cpu')
  refs = [ro.NStepTransitionAccumulator(n) for _ in range(E)]
  emitted = 0
  for emit, st, rw, dc, obs, act in _ticks(seed, E, 200):
    want = []
    for e in np.nonzero(emit)[0]:
      ts = fpo._TimeStep(int(st[e]), None if st[e] == 0 else float(rw[e]), None if st[e] == 0 else float(dc[e]),
                         obs[e].copy())
      want.extend(refs[e].step(ts, int(act[e])))
    _assert_same(acc.step(emit, st, rw, dc, obs, act), want)
    emitted += len(want)
  assert emitted > 100


def test_actions_and_observations_as_tensors():
  from dqn_zoo_b200 import replay as dr
  acc = dr.VectorNStepAccumulator(2, 2, device='cpu')
  ref = dr.VectorNStepAccumulator(2, 2, device='cpu')
  for emit, st, rw, dc, obs, act in _ticks(3, 2, 40):
    got = acc.step(emit, st, rw, dc, torch.as_tensor(obs), torch.as_tensor(act, dtype=torch.int32))
    want = ref.step(emit, st, rw, dc, obs, act)
    if want is None:
      assert got is None
      continue
    for g, w in zip(got, want):
      np.testing.assert_array_equal(np.asarray(g), np.asarray(w))


def test_non_first_after_reset_raises():
  from dqn_zoo_b200 import replay as dr
  acc = dr.VectorNStepAccumulator(3, 3, device='cpu')
  obs = np.zeros((3,) + OBS, np.uint8)
  nan = np.full(3, np.nan)
  with pytest.raises(ValueError, match='Expected FIRST timestep'):
    acc.step([False, True, False], [1, 1, 1], nan, nan, obs, [0, 0, 0])
  acc.step([True, True, True], [0, 0, 0], nan, nan, obs, [0, 0, 0])
  assert acc.step([True, True, True], [1, 1, 1], np.ones(3), np.ones(3), obs, [1, 1, 1]) is None
  acc.reset(1)
  with pytest.raises(ValueError, match='Expected FIRST timestep'):
    acc.step([True, True, True], [1, 1, 1], np.ones(3), np.ones(3), obs, [1, 1, 1])
  out = acc.step([True, False, True], [2, 1, 2], np.ones(3), np.ones(3), obs, [1, 1, 1])
  assert len(out.r_t) == 4   # streams 0 and 2: 2-step and 1-step windows each
  acc.reset()
  with pytest.raises(ValueError, match='Expected FIRST timestep'):
    acc.step([True, False, False], [1, 1, 1], np.ones(3), np.ones(3), obs, [1, 1, 1])
