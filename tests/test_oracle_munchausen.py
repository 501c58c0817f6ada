"""Munchausen DQN's numerics without a GPU: the float64 oracle (oracle/munchausen_oracle.py) against central finite
differences and hand-computed targets, its limits, and the CUDA loss kernel's per-example arithmetic run on the host
(`dz_test_munchausen_example`, the same source as `loss_munchausen_kernel`) against the oracle within an fp32 budget.

The fp32 budget of the host twin (u = 2^-24; every input is an fp32 value, given to the oracle exactly):
  z_a = (qbar_a - v) / tau          relative error <= 2u (subtraction, division)
  e_a = expf(z_a)                   relative error <= 4u (2 ulp on the device) + 2u |z_a|
  S = sum_a e_a (5-level tree)      relative error <= 5u + (4u S + 2u sum_a e_a |z_a|) / S <= u (9 + A)
                                    (z <= 0, so e |z| <= 1/e and S >= 1)
  log S                             absolute error eL <= u (9 + A) + 2u ln A   (1 ulp of log S <= ln A)
  tau log pi = fma(-tau, log S, qbar_a - v)    <= tau eL + u |qbar_a - v| + u |tau log pi|
  bonus = alpha clip(., l0, 0)      <= alpha (that) + u |bonus|   (the clip is 1-Lipschitz)
  boot = fma(tau, log S_t, v_t)     <= tau eL_t + u |boot|
  target = fma(d, boot, r + bonus)  <= |d| (that) + u |r + bonus| + u |target| + (bonus error)
  td = target - q                   + u |td|
"""

import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'munchausen_hand_vectors.json')
U = 2.0 ** -24


def _t(x):
  return torch.tensor(np.asarray(x, dtype=np.float64))


def _golden():
  with open(GOLDEN) as f:
    return json.load(f)['cases']


def test_extra_kind_keeps_the_reference_kinds():
  assert mo.EXTRA_KINDS == ('munchausen',)
  assert 'munchausen' not in lo.AGENT_KINDS and len(lo.AGENT_KINDS) == 7
  spec = lo.NetSpec('munchausen', 6)
  assert mo.param_shapes(spec) == lo.param_shapes(lo.NetSpec('dqn', 6))
  assert mo.head_out(spec) == 6


@pytest.mark.parametrize('case', _golden(), ids=lambda c: c['name'])
def test_oracle_target_matches_the_hand_computed_vectors(case):
  hyper = mo.Hyper(case['alpha'], case['tau'], case['l0'])
  target, bonus = mo.target(_t([case['qbar_tm1']]), _t([case['qbar_t']]), torch.tensor([case['a_tm1']]),
                            _t([case['r_t']]), _t([case['discount_t']]), hyper)
  assert torch.isfinite(target).all()
  assert abs(float(bonus[0]) - case['bonus']) <= 1e-12, case['derivation']
  assert abs(float(target[0]) - case['target']) <= 1e-12 * max(1.0, abs(case['target'])), case['derivation']


def test_golden_covers_the_required_regimes():
  by = {c['name']: c for c in _golden()}
  assert by['clip_active']['bonus'] == -by['clip_active']['alpha'] * 1.0           # clipped at l0 = -1
  assert by['clip_inactive']['l0'] < by['clip_inactive']['bonus'] / by['clip_inactive']['alpha'] < 0
  assert by['terminal_bonus_survives']['discount_t'] == 0 and by['terminal_bonus_survives']['bonus'] < 0
  assert len(by['one_action']['qbar_t']) == 1
  wide = by['wide_q_small_tau_clipped']
  assert wide['tau'] == 0.03 and max(wide['qbar_tm1']) - min(wide['qbar_tm1']) >= 100


def test_alpha_zero_and_small_tau_approach_the_dqn_target():
  rs = np.random.RandomState(0)
  B, A = 64, 6
  qbar_tm1, qbar_t = _t(rs.normal(size=(B, A))), _t(rs.normal(size=(B, A)))
  a = torch.tensor(rs.randint(0, A, B))
  r, d = _t(rs.normal(size=B)), _t(rs.choice([0.0, 0.99], size=B))
  dqn = r + d * qbar_t.max(dim=1).values
  prev = None
  for tau in (1e-1, 1e-2, 1e-3, 1e-5):
    target, bonus = mo.target(qbar_tm1, qbar_t, a, r, d, mo.Hyper(0.0, tau, -1.0))
    assert float(bonus.abs().max()) == 0.0
    gap = target - dqn
    # the soft value exceeds the max by tau log(sum exp((q - v) / tau)), which lies in [0, tau ln A]
    assert float(gap.min()) >= -1e-12 and float((gap - d * tau * math.log(A)).max()) <= 1e-12, tau
    if prev is not None:
      assert float(gap.abs().max()) <= float(prev) + 1e-15
    prev = gap.abs().max()
  assert float(prev) <= 1e-5 * math.log(A)


def _loss(spec, params, target_params, batch, bound, hyper):
  loss, _ = mo.loss_fn(spec, params, target_params, batch, torch.float64, grad_error_bound=bound, hyper=hyper)
  return float(loss)


@pytest.mark.parametrize('hyper', [mo.Hyper(), mo.Hyper(0.5, 1.0, -0.1)], ids=['paper', 'tau1'])
def test_oracle_gradients_match_central_differences(hyper):
  """Every parameter tensor: the autograd gradient of the float64 loss against central differences, along a random
  direction of the whole tensor and at its three largest-gradient elements.  The clip_gradient bound is set out of
  reach so that the loss's derivative is the gradient."""
  spec = lo.NetSpec('munchausen', 4, obs_hw=36)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 1).items()}
  target = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 2).items()}
  rs = np.random.RandomState(4)
  B = 5
  batch = lo.batch_from_numpy(rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8), rs.randint(0, 4, B),
                              rs.choice([-1.0, 0.0, 1.0], B), rs.choice([0.0, 0.99], B),
                              rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8))
  bound = 1e30
  p = {k: v.clone().requires_grad_(True) for k, v in online.items()}
  loss, _ = mo.loss_fn(spec, p, target, batch, torch.float64, grad_error_bound=bound, hyper=hyper)
  loss.backward()
  h = 1e-6
  for name, g in ((k, v.grad) for k, v in p.items()):
    u = torch.tensor(rs.normal(size=g.shape))
    plus = dict(online, **{name: online[name] + h * u})
    minus = dict(online, **{name: online[name] - h * u})
    fd = (_loss(spec, plus, target, batch, bound, hyper) - _loss(spec, minus, target, batch, bound, hyper)) / (2 * h)
    an = float((g * u).sum())
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-8), (name, fd, an)
    for idx in torch.topk(g.abs().reshape(-1), 3).indices.tolist():
      e = torch.zeros(g.numel(), dtype=torch.float64)
      e[idx] = 1.0
      e = e.reshape(g.shape)
      plus = dict(online, **{name: online[name] + h * e})
      minus = dict(online, **{name: online[name] - h * e})
      fd = (_loss(spec, plus, target, batch, bound, hyper) - _loss(spec, minus, target, batch, bound, hyper)) / (2 * h)
      an = float(g.reshape(-1)[idx])
      assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-8), (name, idx, fd, an)


# ---- the CUDA kernel's arithmetic on the host ---------------------------------------------------------------------


def _twin(q_tm1, qbar_tm1, qbar_t, a, r, d, alpha, tau, l0):
  from dqn_zoo_b200 import _lib
  A = len(qbar_tm1)
  arr = [np.ascontiguousarray(x, dtype=np.float32) for x in (q_tm1, qbar_tm1, qbar_t)]
  out = np.zeros(3, np.float32)
  _lib.call('dz_test_munchausen_example', arr[0].ctypes.data, arr[1].ctypes.data, arr[2].ctypes.data, A, int(a),
            float(r), float(d), float(alpha), float(tau), float(l0), out.ctypes.data)
  return out


def _f32(x):
  return float(np.float32(x))


def _budget(q_tm1, qbar_tm1, qbar_t, a, r, d, alpha, tau, l0, target, bonus):
  A = len(qbar_tm1)
  eL = U * (9 + A) + 2 * U * math.log(A)
  v1, v2 = max(qbar_tm1), max(qbar_t)
  s1 = sum(math.exp((q - v1) / tau) for q in qbar_tm1)
  s2 = sum(math.exp((q - v2) / tau) for q in qbar_t)
  tlp = qbar_tm1[a] - v1 - tau * math.log(s1)
  boot = v2 + tau * math.log(s2)
  e_tlp = tau * eL + U * abs(qbar_tm1[a] - v1) + U * abs(tlp)
  e_bonus = alpha * e_tlp + U * abs(bonus)
  e_boot = tau * eL + U * abs(boot)
  e_target = abs(d) * e_boot + e_bonus + U * abs(r + bonus) + U * abs(target)
  e_td = e_target + U * abs(target - q_tm1[a])
  slack = 1e-15 * (abs(r) + abs(boot) + abs(tlp) + abs(q_tm1[a]))   # the oracle's float64 rounding
  return e_target + slack, e_bonus + slack, e_td + slack


def _twin_cases():
  rs = np.random.RandomState(7)
  out = []
  for A in (1, 2, 6, 18):
    for scale in (0.01, 1.0, 30.0):
      for alpha, tau, l0 in ((0.9, 0.03, -1.0), (0.0, 1.0, -0.1), (0.5, 0.3, -0.05), (1.0, 5.0, 0.0)):
        q = [rs.normal(scale=scale, size=A).astype(np.float32) for _ in range(3)]
        out.append((q[0], q[1], q[2], int(rs.randint(A)), _f32(rs.choice([-1.0, 0.0, 0.37, 1.0])),
                    _f32(rs.choice([0.0, 0.99, 0.99 ** 3])), _f32(alpha), _f32(tau), _f32(l0)))
  for c in _golden():
    out.append((np.float32(c['q_tm1']), np.float32(c['qbar_tm1']), np.float32(c['qbar_t']), c['a_tm1'], _f32(c['r_t']),
                _f32(c['discount_t']), _f32(c['alpha']), _f32(c['tau']), _f32(c['l0'])))
  return out


def test_host_twin_within_the_fp32_budget_of_the_oracle():
  worst = 0.0
  clipped = unclipped = 0
  for q_tm1, qbar_tm1, qbar_t, a, r, d, alpha, tau, l0 in _twin_cases():
    got = _twin(q_tm1, qbar_tm1, qbar_t, a, r, d, alpha, tau, l0)
    q64 = [[float(x) for x in v] for v in (q_tm1, qbar_tm1, qbar_t)]
    target, bonus = mo.target(_t([q64[1]]), _t([q64[2]]), torch.tensor([a]), _t([r]), _t([d]), mo.Hyper(alpha, tau, l0))
    target, bonus = float(target[0]), float(bonus[0])
    td = target - q64[0][a]
    b_target, b_bonus, b_td = _budget(q64[0], q64[1], q64[2], a, r, d, alpha, tau, l0, target, bonus)
    for g, w, b in ((got[0], target, b_target), (got[2], bonus, b_bonus), (got[1], td, b_td)):
      assert np.isfinite(g)
      assert abs(float(g) - w) <= b, (g, w, b, len(qbar_tm1), tau)
      worst = max(worst, abs(float(g) - w) / b)
    tlp = float(mo.scaled_log_policy(_t([q64[1]]), tau)[0, a])
    clipped += alpha > 0 and tlp < l0
    unclipped += alpha > 0 and l0 < tlp < 0
  assert clipped and unclipped
  print('worst error / budget %.3f' % worst)


def test_bad_hyperparameters_are_rejected():
  from dqn_zoo_b200 import _lib

  def cfg(kind, alpha, tau, l0):
    c = _lib.LearnerConfig()
    c.kind = _lib.AGENT_KINDS[kind]
    c.num_actions, c.batch, c.obs_h, c.obs_w, c.obs_c = 6, 32, 84, 84, 4
    c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = alpha, tau, l0
    return c

  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', C.byref(cfg('munchausen', 0.9, 0.03, -1.0)), C.byref(plan))
  _lib.call('dz_learner_plan_query', C.byref(cfg('munchausen', 0.0, 1e-6, 0.0)), C.byref(plan))
  bad = [(0.9, 0.0, -1.0), (0.9, -0.03, -1.0), (-0.1, 0.03, -1.0), (0.9, 0.03, 0.5), (math.nan, 0.03, -1.0),
         (0.9, math.inf, -1.0), (0.9, 0.03, -math.inf), (0.9, math.nan, -1.0)]
  for alpha, tau, l0 in bad:
    with pytest.raises(ValueError, match='munchausen'):
      _lib.call('dz_learner_plan_query', C.byref(cfg('munchausen', alpha, tau, l0)), C.byref(plan))
    # dz_learner_create checks the configuration before it reads a buffer
    handle = C.c_void_p()
    with pytest.raises(ValueError, match='munchausen'):
      _lib.call('dz_learner_create', C.byref(cfg('munchausen', alpha, tau, l0)), C.byref(_lib.LearnerBuffers()),
                C.byref(handle))
    q = np.zeros(3, np.float32)
    with pytest.raises(ValueError):
      _lib.call('dz_test_munchausen_example', q.ctypes.data, q.ctypes.data, q.ctypes.data, 3, 0, 0.0, 0.99, alpha, tau,
                l0, np.zeros(3, np.float32).ctypes.data)
  # the other kinds ignore the fields (a zero-filled tail is valid there)
  for kind in lo.AGENT_KINDS:
    c = cfg(kind, -1.0, 0.0, 1.0)
    c.num_atoms, c.num_quantiles, c.latent_dim = 51, 201, 64
    c.tau_samples_s_tm1 = c.tau_samples_policy = c.tau_samples_s_t = 64
    _lib.call('dz_learner_plan_query', C.byref(c), C.byref(plan))
  c = cfg('munchausen', 0.9, 0.03, -1.0)
  c.num_actions = 19
  with pytest.raises(ValueError, match='munchausen'):
    _lib.call('dz_learner_plan_query', C.byref(c), C.byref(plan))


def test_munchausen_parameter_layout_is_dqns():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  layouts = {}
  for kind in ('dqn', 'munchausen'):
    c = _lib.LearnerConfig()
    c.kind = _lib.AGENT_KINDS[kind]
    c.num_actions, c.batch, c.obs_h, c.obs_w, c.obs_c = 6, 32, 84, 84, 4
    c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = 0.9, 0.03, -1.0
    plan = _lib.LearnerPlan()
    _lib.call('dz_learner_plan_query', C.byref(c), C.byref(plan))
    name, shape = C.create_string_buffer(64), (C.c_int64 * 4)()
    ndim, off = C.c_int32(), C.c_int64()
    rows = []
    for i in range(plan.num_tensors):
      _lib.call('dz_learner_tensor_info', C.byref(c), i, name, shape, C.byref(ndim), C.byref(off))
      rows.append((name.value.decode(), tuple(shape[k] for k in range(ndim.value)), off.value))
      assert dl.haiku_name(rows[-1][0], kind) == dl.haiku_name(rows[-1][0], 'dqn')
    layouts[kind] = (plan.param_count, rows)
  assert layouts['dqn'] == layouts['munchausen']
  assert dl.default_optimizer('munchausen') == dl.OptimizerSpec('adam', 0.00005, 0.01 / 32)
