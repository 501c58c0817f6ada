"""CPU: `VectorNStepAccumulator.get_state` / `set_state` — a restored accumulator emits what the original does."""

import numpy as np
import pytest
import torch

from dqn_zoo_b200 import replay as dr


def _tick(rs, E):
  st = rs.choice([1, 1, 1, 2], E)
  return rs.uniform(size=E) < 0.7, st, rs.uniform(-1, 1, E), np.where(st == 2, 0.0, 0.9), rs.randint(0, 6, E)


@pytest.mark.parametrize('n', [1, 3])
def test_round_trip_continues_identically(n):
  E = 5
  rs = np.random.RandomState(n)
  obs = lambda: rs.randint(0, 256, (E, 3, 3, 2)).astype(np.uint8)
  a = dr.VectorNStepAccumulator(E, n, device='cpu')
  a.step(np.ones(E, bool), np.zeros(E), np.full(E, np.nan), np.full(E, np.nan), obs(), rs.randint(0, 6, E))
  for _ in range(4):
    emit, st, r, d, act = _tick(rs, E)
    a.step(emit, np.where(a._has_tm1, st, 0), r, d, obs(), act)
  b = dr.VectorNStepAccumulator(E, n, device='cpu')
  b.set_state(a.get_state())
  for _ in range(12):
    emit, st, r, d, act = _tick(rs, E)
    o = obs()
    x, y = a.step(emit, st, r, d, o, act), b.step(emit, st, r, d, o, act)
    assert (x is None) == (y is None)
    if x is not None:
      for u, v in zip(x, y):
        u = u.numpy() if isinstance(u, torch.Tensor) else u
        v = v.numpy() if isinstance(v, torch.Tensor) else v
        np.testing.assert_array_equal(u, v)


def test_state_of_another_shape_is_refused():
  a = dr.VectorNStepAccumulator(3, 2, device='cpu')
  with pytest.raises(ValueError):
    dr.VectorNStepAccumulator(4, 2, device='cpu').set_state(a.get_state())
