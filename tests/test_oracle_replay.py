"""CPU: the oracle restatement vs (1) golden vectors made from the reference's replay.py,
(2) the reference's known-answer tables."""

import os

import numpy as np
import pytest

from oracle import gen_golden, replay_oracle, scenarios
import replay_contract as rc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.mark.parametrize('name', list(scenarios.ALL))
def test_oracle_reproduces_reference_golden(name):
  rc.check_scenario(replay_oracle, name, 'oracle')


@pytest.mark.parametrize('fn', rc.CONTRACT, ids=lambda f: f.__name__)
def test_oracle_contract(fn):
  fn(replay_oracle)


def test_oracle_matches_reference_on_long_random_per_run():
  """Against the same script run on the original replay.py (tests/golden/replay_long_random_per.npz)."""
  with np.load(os.path.join(GOLDEN, 'replay_long_random_per.npz')) as f:
    want = {k: f[k] for k in f.files}
  got = scenarios.prioritized_replay_script(replay_oracle, **gen_golden.LONG_RANDOM_PER)
  assert sorted(got) == sorted(want)
  for k in want:
    np.testing.assert_array_equal(got[k], want[k], err_msg=k)


def test_synthetic_rows_are_deterministic_and_in_range():
  obs, a, r, d = replay_oracle.synthetic_rows(1, np.arange(100), 64, 6)
  obs2, a2, r2, d2 = replay_oracle.synthetic_rows(1, np.arange(100), 64, 6)
  np.testing.assert_array_equal(obs, obs2)
  assert obs.shape == (100, 2, 64) and obs.dtype == np.uint8
  assert a.min() >= 0 and a.max() < 6
  assert set(np.unique(r)).issubset({-1.0, 0.0, 1.0}) and set(np.unique(d)).issubset({0.0, 0.99})
  obs3, *_ = replay_oracle.synthetic_rows(2, np.arange(100), 64, 6)
  assert (obs3 != obs).mean() > 0.9
