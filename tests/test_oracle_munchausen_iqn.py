"""Munchausen-IQN's numerics without a GPU: the float64 oracle (oracle/munchausen_iqn_oracle.py) against central finite
differences, hand-computed targets and its IQN limit, and the CUDA loss kernel's per-example target arithmetic run on
the host (`dz_test_munchausen_iqn_example`, the same source as `loss_munchausen_iqn_kernel`) against the oracle within
an fp32 budget.

The fp32 budget of the host twin (u = 2^-24; every input is an fp32 value, given to the oracle exactly).  qbar(a) is
a sum of n samples in row order, then a division:
  qbar(a)              absolute error d(a) <= (n + 1) u mean_j |z_j(a)|,   d = max_a d(a)  (d1 at s_tm1, d2 at s_t)
The softmax enters through tau log pi(a) = qbar(a) - tau logsumexp(qbar / tau); logsumexp is 1-Lipschitz in the
max-norm, so the error of qbar moves tau log pi by at most 2 d and pi by a factor within exp(+-2 d / tau).  On top of
that the arithmetic of munchausen's budget (tests/test_oracle_munchausen.py), eL = u (9 + A) + 2u ln A:
  tau log pi(a_tm1)    <= 2 d1 + tau eL + u |qbar_a - v| + u |tau log pi|
  bonus                <= alpha (that) + u |bonus|
  pi(a|s_t)            |dpi_a| <= pi_a (expm1(2 d2 / tau) + (15 + A) u) + u / S   (e_a, S, the division; e |z| <= 1/e)
  h(a) = fma(tau, log S, v - qbar_a)    <= 4 d2 + u |v - qbar_a| + tau eL + u h(a)
  E = sum_a pi h (5-level tree)         <= sum_a (|dpi_a| h_a + pi_a dh_a) + (6 + A) u E
  s_j = sum_a pi zbar_j (fma chain)     <= sum_a |dpi_a| |zbar_j(a)| + (A + 1) u sum_a pi |zbar_j(a)|
  y_j = fma(d, s_j + E, r + bonus)      <= |d| (ds_j + dE + u |s_j + E|) + dbonus + u |r + bonus| + u |y_j|
"""

import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo
from oracle import munchausen_iqn_oracle as mo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'munchausen_iqn_hand_vectors.json')
U = 2.0 ** -24


def _t(x):
  return torch.tensor(np.asarray(x, dtype=np.float64))


def _golden():
  with open(GOLDEN) as f:
    return json.load(f)['cases']


def _target(zbar_tm1, zbar_t, a, r, d, hyper):
  """The oracle's (targets [N'], bonus, entropy) of one example."""
  y, bonus, ent = mo.target(_t([zbar_tm1]), _t([zbar_t]), torch.tensor([a]), _t([r]), _t([d]), hyper)
  return y[0].numpy(), float(bonus[0]), float(ent[0])


def test_extra_kind_keeps_the_reference_kinds():
  assert mo.EXTRA_KINDS == ('munchausen_iqn',)
  assert 'munchausen_iqn' not in lo.AGENT_KINDS and len(lo.AGENT_KINDS) == 7
  spec = lo.NetSpec('munchausen_iqn', 6)
  assert mo.param_shapes(spec) == lo.param_shapes(lo.NetSpec('iqn', 6))
  assert mo.head_out(spec) == 6


@pytest.mark.parametrize('case', _golden(), ids=lambda c: c['name'])
def test_oracle_target_matches_the_hand_computed_vectors(case):
  hyper = mo.Hyper(case['alpha'], case['tau'], case['l0'])
  y, bonus, ent = _target(case['zbar_tm1'], case['zbar_t'], case['a_tm1'], case['r_t'], case['discount_t'], hyper)
  assert np.isfinite(y).all() and math.isfinite(ent) and ent >= 0.0
  assert abs(bonus - case['bonus']) <= 1e-12, case['derivation']
  if case['entropy'] is not None:
    assert abs(ent - case['entropy']) <= 1e-12, case['derivation']
  want = np.asarray(case['targets'])
  assert np.abs(y - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), case['derivation']


def test_golden_covers_the_required_regimes():
  by = {c['name']: c for c in _golden()}
  assert by['clip_active']['bonus'] == -by['clip_active']['alpha'] * 1.0           # clipped at l0 = -1
  assert by['clip_inactive']['l0'] < by['clip_inactive']['bonus'] / by['clip_inactive']['alpha'] < 0
  assert by['terminal_bonus_survives']['discount_t'] == 0 and by['terminal_bonus_survives']['bonus'] < 0
  one = by['one_action']
  assert len(one['zbar_t'][0]) == 1 and one['bonus'] == 0.0
  assert one['targets'] == [one['r_t'] + one['discount_t'] * z[0] for z in one['zbar_t']]
  wide = by['wide_q_small_tau_clipped']
  spread = np.mean(wide['zbar_tm1'], axis=0)
  assert wide['tau'] == 0.03 and spread.max() - spread.min() >= 100


def test_alpha_zero_and_small_tau_approach_the_iqn_loss():
  """With alpha = 0 the bonus vanishes; as tau -> 0 the policy at s_t becomes greedy on the mean of the N' samples and
  h(a*) = tau log S -> 0, so the loss approaches iqn's when iqn's selector taus are tau_t, wherever the argmax margin of
  every example is far above tau ln A."""
  spec = lo.NetSpec('munchausen_iqn', 4, obs_hw=36)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 1).items()}
  target = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 2).items()}
  for k in ('head/w', 'head/b'):
    target[k] = target[k] * 50.0                  # spread the actions' values: margins of order 1e-2 .. 1
  rs = np.random.RandomState(4)
  B, n = 6, 8
  batch = lo.batch_from_numpy(rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8), rs.randint(0, 4, B),
                              rs.choice([-1.0, 0.0, 1.0], B), rs.choice([0.0, 0.99], B),
                              rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8))
  taus = [torch.tensor(rs.uniform(size=(B, n)).astype(np.float32)) for _ in range(3)]
  iqn_spec = lo.NetSpec('iqn', 4, obs_hw=36)
  want, _ = lo.loss_fn(iqn_spec, online, target, batch, torch.float64, taus=(taus[0], taus[2], taus[2]))
  prev = None
  for tau in (1e-1, 1e-2, 1e-3, 1e-5):
    got, aux = mo.loss_fn(spec, online, target, batch, torch.float64, taus, hyper=mo.Hyper(0.0, tau, -1.0))
    assert float(aux['bonus'].abs().max()) == 0.0
    gap = abs(float(got) - float(want))
    if prev is not None:
      assert gap <= prev + 1e-15, tau
    prev = gap
  top2 = aux['qbar_t'].topk(2, dim=1).values
  margin = float((top2[:, 0] - top2[:, 1]).min())
  assert margin >= 1e3 * 1e-5 * math.log(4), margin
  assert prev <= 1e-5 * math.log(4), prev


def _loss(spec, params, target_params, batch, taus, hyper):
  loss, _ = mo.loss_fn(spec, params, target_params, batch, torch.float64, taus, hyper=hyper)
  return float(loss)


@pytest.mark.parametrize('hyper', [mo.Hyper(), mo.Hyper(0.5, 1.0, -0.1)], ids=['paper', 'tau1'])
def test_oracle_gradients_match_central_differences(hyper):
  """Every parameter tensor: the autograd gradient of the float64 loss against central differences, along a random
  direction of the whole tensor and at its three largest-gradient elements."""
  spec = lo.NetSpec('munchausen_iqn', 4, obs_hw=36, latent_dim=16)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 1).items()}
  target = {k: torch.tensor(v, dtype=torch.float64) for k, v in mo.init_params(spec, 2).items()}
  rs = np.random.RandomState(4)
  B = 3
  batch = lo.batch_from_numpy(rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8), rs.randint(0, 4, B),
                              rs.choice([-1.0, 0.0, 1.0], B), rs.choice([0.0, 0.99], B),
                              rs.randint(0, 256, (B, 36, 36, 4)).astype(np.uint8))
  taus = [torch.tensor(rs.uniform(size=(B, k)).astype(np.float32)) for k in (5, 4, 6)]
  p = {k: v.clone().requires_grad_(True) for k, v in online.items()}
  loss, _ = mo.loss_fn(spec, p, target, batch, torch.float64, taus, hyper=hyper)
  loss.backward()
  h = 1e-6
  for name, g in ((k, v.grad) for k, v in p.items()):
    u = torch.tensor(rs.normal(size=g.shape))
    plus = dict(online, **{name: online[name] + h * u})
    minus = dict(online, **{name: online[name] - h * u})
    fd = (_loss(spec, plus, target, batch, taus, hyper) - _loss(spec, minus, target, batch, taus, hyper)) / (2 * h)
    an = float((g * u).sum())
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-8), (name, fd, an)
    for idx in torch.topk(g.abs().reshape(-1), 3).indices.tolist():
      e = torch.zeros(g.numel(), dtype=torch.float64)
      e[idx] = 1.0
      e = e.reshape(g.shape)
      plus = dict(online, **{name: online[name] + h * e})
      minus = dict(online, **{name: online[name] - h * e})
      fd = (_loss(spec, plus, target, batch, taus, hyper) - _loss(spec, minus, target, batch, taus, hyper)) / (2 * h)
      an = float(g.reshape(-1)[idx])
      assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-8), (name, idx, fd, an)


# ---- the CUDA kernel's arithmetic on the host ---------------------------------------------------------------------


def _twin(zbar_tm1, zbar_t, a, r, d, alpha, tau, l0):
  from dqn_zoo_b200 import _lib
  z1 = np.ascontiguousarray(zbar_tm1, dtype=np.float32)
  z2 = np.ascontiguousarray(zbar_t, dtype=np.float32)
  (K, A), Nt = z1.shape, z2.shape[0]
  out = np.zeros(Nt + 2, np.float32)
  _lib.call('dz_test_munchausen_iqn_example', z1.ctypes.data, z2.ctypes.data, A, K, Nt, int(a), float(r), float(d),
            float(alpha), float(tau), float(l0), out.ctypes.data)
  return out[:Nt], float(out[Nt]), float(out[Nt + 1])


def _f32(x):
  return float(np.float32(x))


def _budget(z1, z2, a, r, d, alpha, tau, l0, y, bonus, ent):
  """Per-target, bonus and entropy budgets of the module docstring, from the float64 values."""
  (K, A), Nt = z1.shape, z2.shape[0]
  q1, q2 = z1.mean(axis=0), z2.mean(axis=0)
  d1 = float(((K + 1) * U * np.abs(z1).mean(axis=0)).max())
  d2 = float(((Nt + 1) * U * np.abs(z2).mean(axis=0)).max())
  eL = U * (9 + A) + 2 * U * math.log(A)
  v1, v2 = q1.max(), q2.max()
  s1 = np.exp((q1 - v1) / tau).sum()
  tlp = q1[a] - v1 - tau * math.log(s1)
  e_bonus = alpha * (2 * d1 + tau * eL + U * abs(q1[a] - v1) + U * abs(tlp)) + U * abs(bonus)
  e = np.exp((q2 - v2) / tau)
  s2 = e.sum()
  pi = e / s2
  h = (v2 - q2) + tau * math.log(s2)
  dpi = pi * (math.expm1(2 * d2 / tau) + (15 + A) * U) + U / s2
  dh = 4 * d2 + U * np.abs(v2 - q2) + tau * eL + U * h
  e_ent = float((dpi * h + pi * dh).sum()) + (6 + A) * U * ent
  s = z2 @ pi
  e_s = np.abs(z2) @ dpi + (A + 1) * U * (np.abs(z2) @ pi)
  e_y = abs(d) * (e_s + e_ent + U * np.abs(s + ent)) + e_bonus + U * abs(r + bonus) + U * np.abs(y)
  slack = 1e-14 * (abs(r) + np.abs(z2).max() + np.abs(z1).max() + 1.0)   # the oracle's float64 rounding
  return e_y + slack, e_bonus + slack, e_ent + slack


def _twin_cases():
  rs = np.random.RandomState(7)
  out = []
  for A in (1, 2, 6, 18):
    for K, Nt in ((1, 1), (8, 5), (64, 64)):
      for scale in (0.01, 1.0, 30.0):
        for alpha, tau, l0 in ((0.9, 0.03, -1.0), (0.0, 1.0, -0.1), (0.5, 0.3, -0.05), (1.0, 5.0, 0.0)):
          z1 = rs.normal(scale=scale, size=(K, A)).astype(np.float32)
          z2 = rs.normal(scale=scale, size=(Nt, A)).astype(np.float32)
          out.append((z1, z2, int(rs.randint(A)), _f32(rs.choice([-1.0, 0.0, 0.37, 1.0])),
                      _f32(rs.choice([0.0, 0.99, 0.99 ** 3])), _f32(alpha), _f32(tau), _f32(l0)))
  for c in _golden():
    out.append((np.float32(c['zbar_tm1']), np.float32(c['zbar_t']), c['a_tm1'], _f32(c['r_t']), _f32(c['discount_t']),
                _f32(c['alpha']), _f32(c['tau']), _f32(c['l0'])))
  return out


def test_host_twin_within_the_fp32_budget_of_the_oracle():
  worst = 0.0
  clipped = unclipped = 0
  for z1, z2, a, r, d, alpha, tau, l0 in _twin_cases():
    got_y, got_bonus, got_ent = _twin(z1, z2, a, r, d, alpha, tau, l0)
    z1d, z2d = z1.astype(np.float64), z2.astype(np.float64)
    y, bonus, ent = _target(z1d, z2d, a, r, d, mo.Hyper(alpha, tau, l0))
    b_y, b_bonus, b_ent = _budget(z1d, z2d, a, r, d, alpha, tau, l0, y, bonus, ent)
    assert np.isfinite(got_y).all() and math.isfinite(got_bonus) and got_ent >= 0.0
    err = np.abs(got_y.astype(np.float64) - y)
    assert (err <= b_y).all(), (err.max(), b_y.min(), z1.shape, tau)
    assert abs(got_bonus - bonus) <= b_bonus, (got_bonus, bonus, b_bonus)
    assert abs(got_ent - ent) <= b_ent, (got_ent, ent, b_ent)
    worst = max(worst, float((err / b_y).max()), abs(got_bonus - bonus) / b_bonus, abs(got_ent - ent) / b_ent)
    pi_tm1, h_tm1 = mo.soft_terms(_t(z1d.mean(axis=0)), tau)
    tlp = -float(h_tm1[a])
    clipped += alpha > 0 and tlp < l0
    unclipped += alpha > 0 and l0 < tlp < 0
  assert clipped and unclipped
  print('worst error / budget %.3f' % worst)


def _cfg(kind, alpha=0.9, tau=0.03, l0=-1.0, A=6):
  from dqn_zoo_b200 import _lib
  c = _lib.LearnerConfig()
  c.kind = _lib.AGENT_KINDS[kind]
  c.num_actions, c.batch, c.obs_h, c.obs_w, c.obs_c = A, 32, 84, 84, 4
  c.num_atoms, c.num_quantiles, c.latent_dim = 51, 201, 64
  c.tau_samples_s_tm1 = c.tau_samples_policy = c.tau_samples_s_t = 64
  c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = alpha, tau, l0
  return c


def test_bad_configurations_are_rejected():
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', C.byref(_cfg('munchausen_iqn')), C.byref(plan))
  _lib.call('dz_learner_plan_query', C.byref(_cfg('munchausen_iqn', 0.0, 1e-6, 0.0)), C.byref(plan))
  assert plan.tau_floats == 32 * 3 * 64
  bad = [(0.9, 0.0, -1.0), (0.9, -0.03, -1.0), (-0.1, 0.03, -1.0), (0.9, 0.03, 0.5), (math.nan, 0.03, -1.0),
         (0.9, math.inf, -1.0), (0.9, 0.03, -math.inf), (0.9, math.nan, -1.0)]
  z = np.zeros(6, np.float32)
  for alpha, tau, l0 in bad:
    with pytest.raises(ValueError, match='munchausen'):
      _lib.call('dz_learner_plan_query', C.byref(_cfg('munchausen_iqn', alpha, tau, l0)), C.byref(plan))
    handle = C.c_void_p()   # dz_learner_create checks the configuration before it reads a buffer
    with pytest.raises(ValueError, match='munchausen'):
      _lib.call('dz_learner_create', C.byref(_cfg('munchausen_iqn', alpha, tau, l0)), C.byref(_lib.LearnerBuffers()),
                C.byref(handle))
    with pytest.raises(ValueError):
      _lib.call('dz_test_munchausen_iqn_example', z.ctypes.data, z.ctypes.data, 3, 2, 1, 0, 0.0, 0.99, alpha, tau, l0,
                np.zeros(3, np.float32).ctypes.data)
  with pytest.raises(ValueError, match='munchausen'):
    _lib.call('dz_learner_plan_query', C.byref(_cfg('munchausen_iqn', A=19)), C.byref(plan))
  for field, value in (('latent_dim', 0), ('latent_dim', 24), ('tau_samples_s_tm1', 0), ('tau_samples_policy', 257),
                       ('tau_samples_s_t', -1)):
    c = _cfg('munchausen_iqn')
    setattr(c, field, value)
    with pytest.raises(ValueError):
      _lib.call('dz_learner_plan_query', C.byref(c), C.byref(plan))
  # the other kinds still ignore the fields
  for kind in lo.AGENT_KINDS:
    _lib.call('dz_learner_plan_query', C.byref(_cfg(kind, -1.0, 0.0, 1.0)), C.byref(plan))


def test_munchausen_iqn_parameter_layout_is_iqns():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  layouts = {}
  for kind in ('iqn', 'munchausen_iqn'):
    c = _cfg(kind)
    plan = _lib.LearnerPlan()
    _lib.call('dz_learner_plan_query', C.byref(c), C.byref(plan))
    name, shape = C.create_string_buffer(64), (C.c_int64 * 4)()
    ndim, off = C.c_int32(), C.c_int64()
    rows = []
    for i in range(plan.num_tensors):
      _lib.call('dz_learner_tensor_info', C.byref(c), i, name, shape, C.byref(ndim), C.byref(off))
      rows.append((name.value.decode(), tuple(shape[k] for k in range(ndim.value)), off.value))
      assert dl.haiku_name(rows[-1][0], kind) == dl.haiku_name(rows[-1][0], 'iqn')
    layouts[kind] = (plan.param_count, plan.tau_floats, plan.workspace_bytes > 0, rows)
  assert layouts['iqn'] == layouts['munchausen_iqn']
  assert dl.default_optimizer('munchausen_iqn') == dl.default_optimizer('iqn')
  assert dl.uses_iqn_network('munchausen_iqn') and dl.uses_iqn_network('iqn')
  assert not any(dl.uses_iqn_network(k) for k in ('dqn', 'munchausen', 'rainbow', 'qrdqn'))
