"""CPU: the CQL(H) term of every agent kind (oracle/cql_oracle.py, DESIGN.md §20).

- the oracle's regulariser gradient for every kind's Q definition against central differences in float64;
- hand values (tests/golden/cql_hand_vectors.json): R = log A for equal Q, R -> 0 as Q_{a_tm1} dominates, invariance
  to a constant added to every Q;
- the host twin of the kernels' per-example arithmetic (dz_test_cql_example) within a float32 budget of float64, at
  A = 1, A = 64 and saturated softmaxes;
- cql_alpha's validation in the library and in Learner, and an unchanged layout and plan at alpha > 0.
"""

import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import cql_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
EPS32 = float(np.finfo(np.float32).eps)


def _heads(kind, B, A, rs, N=7, K=11):
  t = lambda *s: torch.tensor(rs.standard_normal(s))
  if kind in ('dqn', 'double_q', 'prioritized', 'munchausen'):
    return t(B, A), None
  if kind == 'c51':
    return 2 * t(B, A, K), None
  if kind == 'rainbow':
    return (2 * t(B, A, K), t(B, K)), None
  w = torch.tensor(rs.dirichlet(np.ones(N), size=B))
  return t(B, N, A), (w if kind == 'fqf' else None)


def _flat(x):
  return list(x) if isinstance(x, tuple) else [x]


@pytest.mark.parametrize('kind', co.KINDS)
def test_the_regularizer_gradient_matches_central_differences(kind):
  rs = np.random.RandomState(3)
  B, A, alpha = 4, 5, 0.7
  head, frac_w = _heads(kind, B, A, rs)
  a = torch.tensor(rs.randint(0, A, B))
  w = torch.tensor([0.0, 0.25, 1.0, 0.6])
  R, g = co.head_grad(kind, head, a, alpha, w, vmax=3.0, frac_w=frac_w)
  assert (R >= 0).all()
  parts = _flat(head)

  def f(ps):
    return float(co.term(co.expected_q(kind, tuple(ps) if kind == 'rainbow' else ps[0], 3.0, frac_w), a, alpha, w)[0])

  h = 1e-6
  for i, (x, gx) in enumerate(zip(parts, _flat(g))):
    num = torch.zeros_like(x)
    flat = x.reshape(-1)
    for j in range(flat.numel()):
      up = [p.clone() for p in parts]
      dn = [p.clone() for p in parts]
      up[i].view(-1)[j] += h
      dn[i].view(-1)[j] -= h
      num.view(-1)[j] = (f(up) - f(dn)) / (2 * h)
    np.testing.assert_allclose(gx.numpy(), num.numpy(), rtol=1e-6, atol=1e-9, err_msg='%s part %d' % (kind, i))
  # an example of weight 0 contributes no gradient; its R is still reported
  for gx in _flat(g):
    assert torch.count_nonzero(gx[0]) == 0
  assert R[0] > 0


def _hand():
  with open(os.path.join(HERE, 'golden', 'cql_hand_vectors.json')) as f:
    return json.load(f)['cases']


@pytest.mark.parametrize('case', _hand(), ids=lambda c: c['name'])
def test_hand_vectors(case):
  q = torch.tensor([case['q']], dtype=torch.float64)
  a = torch.tensor([case['a_tm1']])
  R, g = co.head_grad('dqn', q, a, 1.0)
  np.testing.assert_allclose(float(R[0]), case['R'], rtol=1e-12, atol=1e-15)
  np.testing.assert_allclose(g[0].numpy(), case['grad'], rtol=1e-12, atol=1e-15)


def test_hand_vectors_cover_the_three_properties():
  names = {c['name'] for c in _hand()}
  assert {'equal_q_two', 'equal_q_six', 'one_action', 'taken_action_ahead_by_50', 'shift_-5', 'shift_123'} <= names
  by = {c['name']: c for c in _hand()}
  assert by['shift_-5']['R'] == by['shift_123']['R']
  assert by['taken_action_ahead_by_50']['R'] < 1e-20 < by['taken_action_ahead_by_1']['R']


def _twin(q, a, cot):
  from dqn_zoo_b200 import _lib
  q = np.ascontiguousarray(q, np.float32)
  out = np.zeros(len(q) + 1, np.float32)
  _lib.call('dz_test_cql_example', q.ctypes.data, len(q), int(a), float(cot), out.ctypes.data)
  return out[-1], out[:-1]


def _budget(q, cot):
  """|R - R64| <= 8 eps (|max q| + |q_a| + log A + 1): the max subtraction and the final add each round once at the
  magnitude of the q values, log S at log A; |g - g64| <= |cot| eps (4A + 16 + 2 (max q - min q)): each probability
  carries the rounding of its exponent's argument (up to eps |q_a - max q|), of its exp and of the A-term sum S."""
  q = np.asarray(q, np.float64)
  A = len(q)
  rb = 8 * EPS32 * (abs(q.max()) + np.abs(q).max() + math.log(A) + 1)
  gb = abs(cot) * EPS32 * (4 * A + 16 + 2 * (q.max() - q.min()))
  return rb, gb


CASES = [('A1', [3.5], 0), ('A2-tie', [1.0, 1.0], 1), ('A6', None, 2), ('A18', None, 17), ('A64', None, 63),
         ('A64-offset', 'offset', 5), ('saturated', [0.0, 200.0, -200.0, 30.0], 0),
         ('saturated-taken', [0.0, 200.0, -200.0, 30.0], 1), ('large-equal', [1e4] * 8, 3)]


@pytest.mark.parametrize('name,q,a', CASES, ids=[c[0] for c in CASES])
def test_host_twin_is_within_a_float32_budget_of_float64(name, q, a):
  rs = np.random.RandomState(11)
  if q is None:
    q = rs.standard_normal(int(name[1:])) * 4
  elif q == 'offset':
    q = rs.standard_normal(64) + 500.0
  q = np.asarray(q, np.float32)
  cot = 0.9 / 32
  R, g = _twin(q, a, cot)
  q64 = torch.tensor(q.astype(np.float64))[None]
  R64, g64 = co.head_grad('dqn', q64, torch.tensor([a]), cot)   # one example: the gradient is cot (softmax - onehot)
  g64 = g64[0].numpy()
  rb, gb = _budget(q, cot)
  assert abs(float(R) - float(R64[0])) <= rb, (name, float(R), float(R64[0]), rb)
  assert R >= 0
  assert np.abs(g.astype(np.float64) - g64).max() <= gb, (name, np.abs(g - g64).max(), gb)
  if len(q) == 1:
    assert R == 0 and g[0] == 0


def test_host_twin_refuses_bad_arguments():
  from dqn_zoo_b200 import _lib
  q = np.zeros(65, np.float32)
  out = np.zeros(66, np.float32)
  for A, a in ((0, 0), (65, 0), (4, 4), (4, -1)):
    with pytest.raises(ValueError):
      _lib.call('dz_test_cql_example', q.ctypes.data, A, a, 1.0, out.ctypes.data)


KIND_NETS = [(k, {}) for k in co.KINDS] + [(k, n) for k in ('dqn', 'munchausen')
                                          for n in ({'dueling': 1}, {'noisy': 1}, {'dueling': 1, 'noisy': 1})]


def _cfg(kind, **fields):
  from dqn_zoo_b200 import _lib
  return _lib.LearnerConfig(kind=_lib.AGENT_KINDS[kind], num_actions=6, num_atoms=51, num_quantiles=201, latent_dim=64,
                            tau_samples_s_tm1=8, tau_samples_policy=8, tau_samples_s_t=8, batch=32, obs_h=84, obs_w=84,
                            obs_c=4, learning_rate=1e-4, opt_eps=1e-5, rms_decay=0.95, adam_b1=0.9, adam_b2=0.999,
                            munchausen_alpha=0.9, entropy_temperature=0.03, log_policy_clip=-1.0, **fields)


def _plan(cfg):
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(plan))
  layout = []
  name, shape = C.create_string_buffer(64), (C.c_int64 * 4)()
  ndim, off = C.c_int32(), C.c_int64()
  for i in range(plan.num_tensors):
    _lib.call('dz_learner_tensor_info', C.byref(cfg), i, name, shape, C.byref(ndim), C.byref(off))
    layout.append((name.value, tuple(shape[k] for k in range(ndim.value)), off.value))
  return (plan.param_count, plan.num_tensors, plan.opt_state_floats, plan.workspace_bytes, plan.noise_floats,
          plan.tau_floats), layout


@pytest.mark.parametrize('kind,net', KIND_NETS, ids=['%s%s' % (k, ''.join('-' + o for o in sorted(n))) for k, n in KIND_NETS])
def test_the_library_validates_alpha_and_keeps_the_layout_and_plan(kind, net):
  base = _plan(_cfg(kind, **net))
  for alpha in (0.0, 1e-8, 1.0, 5.0, 1e6):
    assert _plan(_cfg(kind, cql_alpha=alpha, **net)) == base, alpha
  for bad in (-1e-8, -1.0, float('nan'), float('inf'), float('-inf')):
    with pytest.raises(ValueError, match='cql_alpha'):
      _plan(_cfg(kind, cql_alpha=bad, **net))


@pytest.mark.parametrize('bad', [-0.5, float('nan'), float('inf'), '1', True, None])
def test_learner_rejects_a_bad_alpha_before_the_library(bad):
  from dqn_zoo_b200 import learner as dl
  with pytest.raises(ValueError, match='cql_alpha'):
    dl.Learner(dl.NetworkSpec('dqn', 6), cql_alpha=bad)
  assert dl.check_cql_alpha(2) == 2.0 and dl.check_cql_alpha(np.float32(0.5)) == 0.5


def test_update_outputs_default_the_regularizer_to_null():
  from dqn_zoo_b200 import _lib
  out = _lib.UpdateOutputs(1, 2, 3, 4)
  assert out.d_regularizer is None
  assert _lib.LearnIO().update_out.d_regularizer is None
