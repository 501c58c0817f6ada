"""CPU: FQF (DESIGN.md §15) -- the float64 oracle (oracle/fqf_oracle.py) against its definition, the hand-derived
vectors in tests/golden/fqf_hand_vectors.json, the library's host twin of the per-example fraction arithmetic, the
configuration checks and the Python surface.

Host-twin budget.  dz_test_fqf_example runs fqf_fractions and fqf_dlogits, the source the fraction and loss kernels
run, in float32 on float32 inputs; the oracle evaluates the same formulas in float64 on the same inputs.  With
u = 2^-24 and every sum serial in index order:
  q_i = expf(l_i - m) / S: the difference l_i - m rounds by up to u |l_i - m| <= u R (R = max_i |l_i - m|), which
      expf turns into a relative error of the same size, expf within 2 ulp, S a sum of N positive terms (relative
      error <= (N + R) u), one division:  |dq_i| <= (N + 4 + 2R) u q_i + 2^-147 (expf and the division of a result in
      the subnormal range, below 2^-126, round to a multiple of 2^-149)
  tau_i = sum_{k<i} q_k: the q errors plus i roundings of a sum <= 1:  |dtau_i| <= T = (2N + 4 + 2R) u
  tau_hat_i: two tau errors halved, one rounding: T + u;  w_i = tau_{i+1} - tau_i: 2T + u
  g_i = (2 F(tau_i) - F(tau_hat_i)) - F(tau_hat_{i-1}): exact inputs, 2 roundings: |dg_i| <= 2 u G_i,
      G_i = 2|F(tau_i)| + |F(tau_hat_i)| + |F(tau_hat_{i-1})|
  dq_k = sum_{i>k} g_i (serial from the end): |ddq_k| <= E_dq = (N + 2) u sum_i G_i
  D = sum_j q_j dq_j (fmaf chain): |dD| <= N u sum_j q_j |dq_j| + sum_j (|dq_j| |dq_j| + q_j E_dq)
  dlogit_k = cot (q_k (dq_k - D)), two roundings: |ddl_k| <= cot (q_k (E_dq + |dD|) + |dq_k| |dq_k - D| + 2 u q_k |dq_k - D|)
The test asserts every element within its budget and prints the worst error / budget.
"""

import ctypes
import json
import math
import os

import numpy as np
import pytest
import torch
from scipy import integrate, stats

from oracle import fqf_oracle as fo
from oracle import learner_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def test_kind_is_an_extra_kind():
  assert 'fqf' not in lo.AGENT_KINDS and len(lo.AGENT_KINDS) == 7 and fo.EXTRA_KINDS == ('fqf',)


# ---- the fraction gradient's definition -----------------------------------------------------------------------------

QUANTILE_FUNCTIONS = {
    'normal_ppf': lambda t: stats.norm.ppf(0.01 + 0.98 * t),
    'exponential_ppf': lambda t: -np.log1p(-0.99 * t),
    'cubic': lambda t: 4.0 * (t - 0.4) ** 3 + t,
}


def w1(F, tau):
  """The 1-Wasserstein error of the staircase at tau_hat: sum_i int_{tau_i}^{tau_{i+1}} |F(w) - F(tau_hat_i)| dw."""
  total = 0.0
  for i in range(len(tau) - 1):
    m = 0.5 * (tau[i] + tau[i + 1])
    fm = F(m)
    total += integrate.quad(lambda x: abs(F(x) - fm), tau[i], tau[i + 1], points=[m], epsabs=1e-13, epsrel=1e-12)[0]
  return total


@pytest.mark.parametrize('name', sorted(QUANTILE_FUNCTIONS))
def test_tau_gradient_is_the_derivative_of_the_w1_error(name):
  F = QUANTILE_FUNCTIONS[name]
  rs = np.random.RandomState(3)
  N = 6
  q = rs.dirichlet(np.ones(N) * 2)
  tau = np.concatenate([[0.0], np.cumsum(q)[:-1], [1.0]])
  hat = 0.5 * (tau[:-1] + tau[1:])
  g = fo.tau_gradient(torch.tensor(F(tau[1:-1]))[None], torch.tensor(F(hat))[None])[0].numpy()
  h = 1e-5
  for i in range(1, N):
    tp, tm = tau.copy(), tau.copy()
    tp[i] += h
    tm[i] -= h
    cd = (w1(F, tp) - w1(F, tm)) / (2 * h)
    assert abs(cd - g[i - 1]) <= 1e-5 * (1 + abs(g[i - 1])), (name, i, cd, g[i - 1])


@pytest.mark.parametrize('name', sorted(QUANTILE_FUNCTIONS))
def test_dlogits_are_the_derivative_of_the_w1_error_through_softmax_and_cumsum(name):
  F = QUANTILE_FUNCTIONS[name]
  rs = np.random.RandomState(4)
  N = 5
  logits = rs.standard_normal(N)

  def objective(lg):
    p = fo.proposal(torch.tensor(lg)[None])
    return w1(F, p['tau'][0].numpy())

  p = fo.proposal(torch.tensor(logits)[None])
  tau, hat = p['tau'][0].numpy(), p['tau_hat'][0].numpy()
  g = fo.tau_gradient(torch.tensor(F(tau[1:-1]))[None], torch.tensor(F(hat))[None])
  dl = fo.dlogits_of(g, p['q'], torch.ones(1, dtype=torch.float64))[0].numpy()
  # the autograd chain of the oracle's surrogate gives the same
  lg = torch.tensor(logits)[None].requires_grad_(True)
  (g.detach() * fo.proposal(lg)['tau'][:, 1:-1]).sum().backward()
  np.testing.assert_allclose(lg.grad[0].numpy(), dl, rtol=1e-12, atol=1e-15)
  h = 1e-5
  for k in range(N):
    lp_, lm_ = logits.copy(), logits.copy()
    lp_[k] += h
    lm_[k] -= h
    cd = (objective(lp_) - objective(lm_)) / (2 * h)
    assert abs(cd - dl[k]) <= 1e-5 * (1 + abs(dl[k])), (name, k, cd, dl[k])


# ---- central differences of the quantile loss ----------------------------------------------------------------------

def _case(B=3, N=6, seed=2):
  spec = lo.NetSpec('fqf', 4, obs_hw=44)
  p = fo.init_params(spec, seed, N)
  p['fraction/w'] = (p['fraction/w'] * 100).astype(np.float32)
  p['fraction/b'] = np.linspace(-1, 1, N).astype(np.float32)
  O = fo.Learner(spec, p, hyper=fo.Hyper(N))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in fo.init_params(spec, seed + 1, N).items()}
  rs = np.random.RandomState(seed)
  batch = lo.batch_from_numpy(rs.randint(0, 256, (B, 44, 44, 4)).astype(np.uint8), rs.randint(0, 4, B),
                              rs.choice([-1.0, 0.5], B), rs.choice([0.0, 0.99], B),
                              rs.randint(0, 256, (B, 44, 44, 4)).astype(np.uint8))
  return spec, O, batch


def test_quantile_loss_central_differences_and_gradient_separation():
  spec, O, batch = _case()
  _, aux = fo.loss_fn(spec, O.online, O.target, batch, torch.float64)
  fixed = (aux['prop_tm1']['tau'].numpy(), aux['prop_tm1']['tau_hat'].numpy(), aux['prop_t']['tau'].numpy(),
           aux['prop_t']['tau_hat'].numpy())
  p = {k: v.clone().requires_grad_(True) for k, v in O.online.items()}
  loss, aux = fo.loss_fn(spec, p, O.target, batch, torch.float64, device_fractions=fixed)
  grads = torch.autograd.grad(loss, list(p.values()), allow_unused=True)
  g = dict(zip(p, grads))
  for name in fo.FRACTION_TENSORS:
    assert g[name] is None or float(g[name].abs().max()) == 0.0, name   # the quantile loss reaches no fraction tensor
  p2 = {k: v.clone().requires_grad_(True) for k, v in O.online.items()}
  _, aux2 = fo.loss_fn(spec, p2, O.target, batch, torch.float64, device_fractions=fixed)
  gf = dict(zip(p2, torch.autograd.grad(aux2['fraction_objective'], list(p2.values()), allow_unused=True)))
  for name in p2:
    if name not in fo.FRACTION_TENSORS:
      assert gf[name] is None or float(gf[name].abs().max()) == 0.0, name   # the fraction loss reaches no torso tensor
  assert float(gf['fraction/w'].abs().max()) > 0
  rs = np.random.RandomState(7)
  h = 1e-6
  for name, value in O.online.items():
    if name in fo.FRACTION_TENSORS:
      continue
    for _ in range(3):
      idx = tuple(rs.randint(0, s) for s in value.shape)
      def at(delta):
        q = {k: v.clone() for k, v in O.online.items()}
        q[name][idx] += delta
        return float(fo.loss_fn(spec, q, O.target, batch, torch.float64, device_fractions=fixed)[0])
      cd = (at(h) - at(-h)) / (2 * h)
      want = float(g[name][idx])
      assert abs(cd - want) <= 1e-6 + 1e-4 * abs(want), (name, idx, cd, want)


# ---- hand vectors ---------------------------------------------------------------------------------------------------

def _hand_cases():
  with open(os.path.join(ROOT, 'tests', 'golden', 'fqf_hand_vectors.json')) as f:
    return json.load(f)['cases']


@pytest.mark.parametrize('case', _hand_cases(), ids=lambda c: c['name'])
def test_hand_vectors(case):
  from dqn_zoo_b200 import _lib
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  p = fo.proposal(t(case['logits'])[None])
  for key in ('q', 'tau', 'tau_hat', 'w'):
    np.testing.assert_allclose(p[key][0].numpy(), case[key], rtol=0, atol=1e-12, err_msg=key)
  g = fo.tau_gradient(t(case['F_tau'][1:])[None], t(case['F_hat'])[None])
  np.testing.assert_allclose(g[0].numpy(), case['tau_grad'], rtol=0, atol=1e-12)
  dl = fo.dlogits_of(g, p['q'], torch.ones(1, dtype=torch.float64))
  np.testing.assert_allclose(dl[0].numpy(), case['dlogits'], rtol=0, atol=1e-12)
  N, A = len(case['logits']), len(case['zsel'][0])
  F_hat = t(case['F_hat'])
  dist0 = F_hat[None, :, None].repeat(1, 1, A)
  ftau = t(case['F_tau'][1:])[None, :, None].repeat(1, 1, A)
  _, aux = fo.head_loss((dist0, ftau, t(case['zsel'])[None], t(case['ztgt'])[None]), [0], [case['r_t']],
                        [case['discount_t']], p['tau_hat'], t(case['w'])[None])
  assert int(aux['a_star'][0]) == case['a_star']
  np.testing.assert_allclose(aux['targets'][0].numpy(), case['targets'], rtol=0, atol=1e-6)
  # the library's float32 twin of the same arithmetic
  out = np.zeros(5 * N + 1, np.float32)
  lg = np.asarray(case['logits'], np.float32)
  ft, fh = np.asarray(case['F_tau'], np.float32), np.asarray(case['F_hat'], np.float32)
  _lib.call('dz_test_fqf_example', lg.ctypes.data, ft.ctypes.data, fh.ctypes.data, N, 1.0, out.ctypes.data)
  for key, lo_, hi_ in (('q', 0, N), ('tau', N, 2 * N + 1), ('tau_hat', 2 * N + 1, 3 * N + 1), ('w', 3 * N + 1, 4 * N + 1),
                        ('dlogits', 4 * N + 1, 5 * N + 1)):
    np.testing.assert_allclose(out[lo_:hi_], case[key], rtol=0, atol=2e-6, err_msg=key)


# ---- the host twin against the oracle within the float32 budget ------------------------------------------------------

@pytest.mark.parametrize('N', [2, 32, 128])
def test_host_twin_within_the_float32_budget(N):
  from dqn_zoo_b200 import _lib
  rs = np.random.RandomState(N)
  worst = 0.0
  for scale in (0.01, 0.1, 1.0, 3.0, 10.0, 30.0):
    for rep in range(4):
      lg = (scale * rs.standard_normal(N)).astype(np.float32)
      ft = np.sort(rs.standard_normal(N)).astype(np.float32)
      fh = np.sort(rs.standard_normal(N)).astype(np.float32)
      cot = np.float32(rs.uniform(0.1, 1.0) / 32)
      out = np.zeros(5 * N + 1, np.float32)
      _lib.call('dz_test_fqf_example', lg.ctypes.data, ft.ctypes.data, fh.ctypes.data, N, float(cot), out.ctypes.data)
      p = fo.proposal(torch.tensor(lg.astype(np.float64))[None])
      q = p['q'][0].numpy()
      g = fo.tau_gradient(torch.tensor(ft[1:].astype(np.float64))[None], torch.tensor(fh.astype(np.float64))[None])
      dl = fo.dlogits_of(g, p['q'], torch.tensor([float(cot)], dtype=torch.float64))[0].numpy()
      G = 2 * np.abs(ft[1:].astype(np.float64)) + np.abs(fh[1:]) + np.abs(fh[:-1])
      gg = np.concatenate([[0.0], g[0].numpy()])
      dq = np.cumsum(gg[::-1])[::-1] - gg
      D = float((q * dq).sum())
      e_dq = (N + 2) * U * G.sum()
      R = float(np.abs(lg.astype(np.float64) - lg.max()).max())
      bq = (N + 4 + 2 * R) * U * q
      T = (2 * N + 4 + 2 * R) * U
      e_D = N * U * float((q * np.abs(dq)).sum()) + float((bq * np.abs(dq) + q * e_dq).sum())
      budgets = {
          'q': (out[:N], q, bq + 2.0 ** -147),
          'tau': (out[N:2 * N + 1], p['tau'][0].numpy(), np.full(N + 1, T)),
          'tau_hat': (out[2 * N + 1:3 * N + 1], p['tau_hat'][0].numpy(), np.full(N, T + U)),
          'w': (out[3 * N + 1:4 * N + 1], p['w'][0].numpy(), np.full(N, 2 * T + U)),
          'dlogits': (out[4 * N + 1:], dl, float(cot) * (q * (e_dq + e_D) + bq * np.abs(dq - D) + 2 * U * q * np.abs(dq - D))
                      + 1e-45),
      }
      for key, (got, want, budget) in budgets.items():
        use = np.abs(got.astype(np.float64) - want) / budget
        assert use.max() <= 1.0, (N, scale, key, float(use.max()))
        worst = max(worst, float(use.max()))
  print('fqf host twin N=%d: worst error / budget %.3f' % (N, worst))


def assert_fraction_invariant(tau, hat, w, N):
  """0 = tau_0 <= tau_1 <= ... <= tau_N = 1, w_i = tau_{i+1} - tau_i >= 0 and tau_i <= tau_hat_i <= tau_{i+1}, exactly in
  float32 (tau [..., N + 1], hat and w [..., N])."""
  tau, hat, w = (np.asarray(x, np.float32) for x in (tau, hat, w))
  assert (tau[..., 0] == 0).all() and (tau[..., N] == 1).all()
  assert (np.diff(tau, axis=-1) >= 0).all() and (tau <= 1).all(), tau.max()
  assert (w >= 0).all() and (w == tau[..., 1:] - tau[..., :-1]).all()
  assert (tau[..., :-1] <= hat).all() and (hat <= tau[..., 1:]).all() and (hat <= 1).all()


@pytest.mark.parametrize('N', [2, 3, 11, 19, 27, 31, 32, 127, 128])
def test_host_twin_fractions_stay_ordered_inside_0_1(N):
  """A saturated last logit leaves the float32 prefix sum of the other N - 1 fractions free to round above 1 (at N = 11
  with logits (0, ..., 0, -30) it gives 1 + 2^-23); the fractions are clamped to 1 so that the invariant holds."""
  from dqn_zoo_b200 import _lib
  rs = np.random.RandomState(100 + N)
  cases = [np.concatenate([np.zeros(N - 1), [-30.0]])]
  for _ in range(60):
    lg = rs.standard_normal(N)
    lg[-1] = -rs.uniform(20, 90)   # the last fraction's share is below float32's rounding of the others' sum
    cases.append(lg)
  for lead in (0, N // 2):         # one fraction takes every other's mass
    lg = np.full(N, -100.0)
    lg[lead] = 0.0
    cases.append(lg)
  cases.append(np.linspace(-80, 80, N))
  z = np.zeros(N, np.float32)
  for lg in cases:
    lg = lg.astype(np.float32)
    out = np.zeros(5 * N + 1, np.float32)
    _lib.call('dz_test_fqf_example', lg.ctypes.data, z.ctypes.data, z.ctypes.data, N, 1.0, out.ctypes.data)
    tau, hat, w = out[N:2 * N + 1], out[2 * N + 1:3 * N + 1], out[3 * N + 1:4 * N + 1]
    assert_fraction_invariant(tau, hat, w, N)
    p = fo.proposal(torch.tensor(lg.astype(np.float64))[None])
    R = float(np.abs(lg.astype(np.float64) - lg.max()).max())
    T = (2 * N + 4 + 2 * R) * U   # the clamp only moves a tau that rounded above 1 back towards the float64 value
    assert np.abs(tau - p['tau'][0].numpy()).max() <= T


# ---- configuration checks and the Python surface ---------------------------------------------------------------------

def _cfg(kind, **fields):
  from dqn_zoo_b200 import _lib
  c = _lib.LearnerConfig(**fields)
  c.kind = _lib.AGENT_KINDS[kind]
  c.num_actions, c.num_atoms, c.num_quantiles, c.latent_dim = 6, 51, 201, 64
  c.tau_samples_s_tm1 = c.tau_samples_policy = c.tau_samples_s_t = 64
  c.batch, c.obs_h, c.obs_w, c.obs_c = 32, 84, 84, 4
  c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = 0.9, 0.03, -1.0
  return c


def test_library_validates_the_fraction_configuration():
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()
  nan, inf = float('nan'), float('inf')
  _lib.call('dz_learner_plan_query', ctypes.byref(_cfg('fqf')), ctypes.byref(plan))
  assert plan.tau_floats == 0
  for ok in (dict(num_fractions=2), dict(num_fractions=128), dict(fraction_learning_rate=0.0),
             dict(fraction_rms_decay=0.0), dict(tau_samples_s_tm1=0)):
    _lib.call('dz_learner_plan_query', ctypes.byref(_cfg('fqf', **ok)), ctypes.byref(plan))
  bad = [('num_fractions', 1), ('num_fractions', 129), ('num_fractions', 0), ('fraction_learning_rate', -1e-9),
         ('fraction_learning_rate', nan), ('fraction_learning_rate', inf), ('fraction_opt_eps', 0.0),
         ('fraction_opt_eps', -1e-5), ('fraction_opt_eps', nan), ('fraction_opt_eps', inf), ('fraction_rms_decay', 1.0),
         ('fraction_rms_decay', -0.1), ('fraction_rms_decay', nan)]
  for field, value in bad:
    with pytest.raises(ValueError, match=field):
      _lib.call('dz_learner_plan_query', ctypes.byref(_cfg('fqf', **{field: value})), ctypes.byref(plan))
  c = _cfg('fqf')
  c.latent_dim = 24
  with pytest.raises(ValueError, match='latent_dim'):
    _lib.call('dz_learner_plan_query', ctypes.byref(c), ctypes.byref(plan))
  # every other kind ignores the tail, whatever it holds
  for kind in _lib.AGENT_KINDS:
    if kind != 'fqf':
      for field, value in bad:
        _lib.call('dz_learner_plan_query', ctypes.byref(_cfg(kind, **{field: value})), ctypes.byref(plan))
  out = np.zeros(5 * 129 + 1, np.float32)
  x = np.zeros(129, np.float32)
  with pytest.raises(ValueError):
    _lib.call('dz_test_fqf_example', x.ctypes.data, x.ctypes.data, x.ctypes.data, 129, 1.0, out.ctypes.data)
  # fqf's loss and acting hooks take only an fqf configuration and its fraction buffers
  heads = (ctypes.c_void_p * 3)(1, 1, 1)
  for kind, w in (('iqn', 1), ('fqf', None)):
    with pytest.raises(ValueError, match='test_loss_fqf'):
      _lib.call('dz_test_loss_fqf', ctypes.byref(_cfg(kind)), 32, heads, 1, 1, 1, None, 1, w, 1, 1, 1, 1, 1, 1, None)
    if w:
      with pytest.raises(ValueError, match='test_q_values_fqf'):
        _lib.call('dz_test_q_values_fqf', ctypes.byref(_cfg(kind)), 4, 1, 1, None, 0.0, 1, None, None)


def test_parameter_layout_and_python_surface():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  for N in (2, 32, 128):
    cfg = _cfg('fqf', num_fractions=N)
    plan = _lib.LearnerPlan()
    _lib.call('dz_learner_plan_query', ctypes.byref(cfg), ctypes.byref(plan))
    want = fo.param_shapes(lo.NetSpec('fqf', 6), N)
    assert plan.num_tensors == len(want)
    name = ctypes.create_string_buffer(64)
    shape = (ctypes.c_int64 * 4)()
    ndim, off = ctypes.c_int32(), ctypes.c_int64()
    for i, (wname, wshape) in enumerate(want.items()):
      _lib.call('dz_learner_tensor_info', ctypes.byref(cfg), i, name, shape, ctypes.byref(ndim), ctypes.byref(off))
      assert name.value.decode() == wname and tuple(shape[k] for k in range(ndim.value)) == tuple(wshape)
    assert list(want)[-2:] == ['fraction/w', 'fraction/b']
  assert dl.uses_iqn_network('fqf') and not dl.draws_taus('fqf')
  assert dl.draws_taus('iqn') and dl.draws_taus('munchausen_iqn') and not dl.draws_taus('dqn')
  assert dl.haiku_name('fraction/w', 'fqf') == ('fraction_proposal/linear', 'w')
  assert dl.default_optimizer('fqf') == dl.OptimizerSpec('adam', 0.00005, 0.01 / 32)
  assert dl.NetworkSpec('fqf', 6).num_fractions == 32
  assert ag.AGENTS['fqf'] is ag.Fqf
