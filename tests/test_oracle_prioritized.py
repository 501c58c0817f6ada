"""CPU: the priority rule of prioritized replay for all ten agent kinds (oracle/prioritized_oracle.py, DESIGN.md §19) on
hand-built oracle outputs, and its agreement with learner_oracle's rule for prioritized and rainbow."""

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo
from oracle import prioritized_oracle as po

TD = torch.tensor([-3.0, 0.0, 2.5, -1e-7, 250.0], dtype=torch.float64)
LOSSES = torch.tensor([150.0, 0.0, 99.99, 100.0, 1e-7], dtype=torch.float64)


def test_the_ten_kinds_are_split_between_the_two_rules():
  assert set(po.KINDS) == {'dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen',
                           'munchausen_iqn', 'fqf'}
  assert not set(po.TD_KINDS) & set(po.LOSS_KINDS)
  with pytest.raises(ValueError):
    po.priorities('ddpg', {'td_errors': TD, 'losses': LOSSES})


@pytest.mark.parametrize('kind', po.TD_KINDS)
def test_td_kinds_take_the_absolute_td_of_either_sign_unclipped(kind):
  # munchausen's per-example value is 0.5 td^2: the priority must come from td, not from the loss
  aux = {'td_errors': TD, 'losses': 0.5 * TD * TD}
  got = po.priorities(kind, aux)
  assert got.dtype == torch.float64
  assert torch.equal(got, torch.tensor([3.0, 0.0, 2.5, 1e-7, 250.0], dtype=torch.float64))


@pytest.mark.parametrize('kind', po.LOSS_KINDS)
def test_loss_kinds_clip_the_absolute_loss_at_100(kind):
  got = po.priorities(kind, {'losses': LOSSES})
  assert torch.equal(got, torch.tensor([100.0, 0.0, 99.99, 100.0, 1e-7], dtype=torch.float64))
  # a negative loss (not produced by these losses, but the rule takes |loss|) and exact zeros
  neg = po.priorities(kind, {'losses': torch.tensor([-7.0, -0.0, -300.0], dtype=torch.float64)})
  assert torch.equal(neg, torch.tensor([7.0, 0.0, 100.0], dtype=torch.float64))
  assert not torch.signbit(neg[1])


def _heads(kind, B, A, K, rs):
  t = lambda *s: torch.tensor(rs.standard_normal(s))
  if kind == 'prioritized':
    return [t(B, A), t(B, A), t(B, A)]
  return [(3 * t(B, A, K), t(B, K)) for _ in range(3)]


@pytest.mark.parametrize('kind', ['prioritized', 'rainbow'])
@pytest.mark.parametrize('weighted', [False, True])
def test_reproduces_the_two_existing_rules_exactly(kind, weighted):
  rs = np.random.RandomState(7)
  B, A, K = 16, 5, 11
  for scale in (1.0, 40.0):   # at the larger scale some rainbow losses pass the clip
    heads = _heads(kind, B, A, K, rs)
    a = torch.tensor(rs.randint(0, A, B))
    r = torch.tensor(scale * rs.choice([-1.0, 0.0, 1.0, 0.37], size=B))
    d = torch.tensor(rs.choice([0.0, 0.99], size=B))
    w = torch.tensor(rs.uniform(0.0, 1.0, B)) if weighted else None
    _, aux = lo.head_loss(kind, heads, a, r, d, w, vmax=5.0, grad=False)
    assert torch.equal(po.priorities(kind, aux), aux['priorities'])
    # learner_oracle.Learner.update hands them on as float32
    assert torch.equal(po.priorities(kind, aux).to(torch.float32), aux['priorities'].to(torch.float32))
