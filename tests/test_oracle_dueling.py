"""CPU: the dueling network (DESIGN.md §16) of dqn, double_q, prioritized and munchausen.

- the float64 oracle (oracle/dueling_oracle.py): autograd against central differences of each kind's loss for every
  tensor, and the aggregation's identities;
- the host twin of the kernels' per-row arithmetic (dz_test_dueling_example) within a float32 budget of float64;
- the C ABI: the parameter layout, and the rejection of dueling=True for every other kind.

Float32 budget of the twin, with u = 2^-24 and sums in action order: the sum of A terms carries at most (A - 1) u of the
sum of magnitudes, the division by A, the subtraction and the addition one u each of their result.  So
  |q_a - q_a*|      <= (A + 3) u (|v| + |adv_a| + mean_a |adv_a|),
  |dadv_a - dadv_a*| <= (A + 2) u (|dq_a| + mean_a |dq_a|),
  |dval - dval*|    <= A u sum_a |dq_a|,
and the test reports the worst error / budget.
"""

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import dueling_oracle as do
from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo

U = 2.0 ** -24
KINDS = do.KINDS
OTHER_KINDS = ('c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen_iqn', 'fqf')


def _case(kind, A=6, hw=36, B=4, seed=0):
  spec = lo.NetSpec(kind, A, obs_hw=hw)
  rs = np.random.RandomState(seed)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in do.init_params(spec, seed).items()}
  target = {k: torch.tensor(v, dtype=torch.float64) for k, v in do.init_params(spec, seed + 1).items()}
  s = rs.randint(0, 256, (2, B, hw, hw, 4)).astype(np.uint8)
  batch = lo.batch_from_numpy(s[0], rs.randint(0, A, B), rs.choice([-1.0, 0.0, 1.0], B), rs.choice([0.0, 0.99], B), s[1])
  w = torch.tensor(rs.uniform(0.1, 1.0, B)) if kind == 'prioritized' else None
  return spec, online, target, batch, w


def _loss(spec, p, target, batch, w):
  # a clip far above every td: rlax.clip_gradient clips the gradient, not the loss, so central differences of the loss
  # match autograd only where it does not fire
  return do.loss_fn(spec, p, target, batch, torch.float64, w, grad_error_bound=1e6)[0]


# ---- the oracle ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', KINDS)
def test_autograd_matches_central_differences_for_every_tensor(kind):
  spec, online, target, batch, w = _case(kind)
  p = {k: v.clone().requires_grad_(True) for k, v in online.items()}
  _loss(spec, p, target, batch, w).backward()
  rs = np.random.RandomState(1)
  h = 1e-6
  for name, value in online.items():
    d = torch.tensor(rs.standard_normal(value.shape))
    d /= d.norm()
    plus = {k: (v + h * d if k == name else v) for k, v in online.items()}
    minus = {k: (v - h * d if k == name else v) for k, v in online.items()}
    fd = float(_loss(spec, plus, target, batch, w) - _loss(spec, minus, target, batch, w)) / (2 * h)
    ad = float((p[name].grad * d).sum())
    scale = max(float(p[name].grad.norm()), 1e-8)
    assert abs(fd - ad) <= 1e-6 * scale, (kind, name, fd, ad)


@pytest.mark.parametrize('A', [1, 6, 18])
def test_aggregation_identities(A):
  spec, online, _, batch, _ = _case('dqn', A=A)
  out = do.apply_net(spec, online, batch['s_tm1'], torch.float64)
  q, adv, v = out['q_values'], out['adv'], out['val']
  torch.testing.assert_close(q - q.mean(1, keepdim=True), adv - adv.mean(1, keepdim=True), rtol=0, atol=1e-12)
  torch.testing.assert_close(q.mean(1), v, rtol=0, atol=1e-12)
  if A == 1:
    assert torch.equal(q[:, 0], v)


@pytest.mark.parametrize('kind', KINDS)
def test_a_constant_advantage_bias_changes_nothing(kind):
  spec, online, target, batch, w = _case(kind)
  shifted = dict(online, **{'adv2/b': online['adv2/b'] + 0.375})
  q0 = do.apply_net(spec, online, batch['s_tm1'], torch.float64)['q_values']
  q1 = do.apply_net(spec, shifted, batch['s_tm1'], torch.float64)['q_values']
  torch.testing.assert_close(q1, q0, rtol=0, atol=1e-12)
  l0 = float(do.loss_fn(spec, online, target, batch, torch.float64, w)[0])
  l1 = float(do.loss_fn(spec, shifted, target, batch, torch.float64, w)[0])
  assert abs(l1 - l0) <= 1e-12 * max(abs(l0), 1.0)


@pytest.mark.parametrize('kind', KINDS)
def test_one_action_is_the_value_stream(kind):
  """At A = 1, q = v exactly and no gradient reaches the advantage stream."""
  spec, online, target, batch, w = _case(kind, A=1)
  p = {k: v.clone().requires_grad_(True) for k, v in online.items()}
  loss = do.loss_fn(spec, p, target, batch, torch.float64, w)[0]
  loss.backward()
  for name in ('adv1/w', 'adv1/b', 'adv2/w', 'adv2/b'):
    assert p[name].grad is None or not p[name].grad.any(), name
  assert p['val2/w'].grad.abs().max() > 0


def test_munchausen_loss_is_the_munchausen_head_on_dueling_q():
  spec, online, target, batch, _ = _case('munchausen')
  q = [do.apply_net(spec, pp, s, torch.float64)['q_values'] for pp, s in
       ((online, batch['s_tm1']), (target, batch['s_tm1']), (target, batch['s_t']))]
  want = mo.head_loss(q, batch['a_tm1'], batch['r_t'], batch['discount_t'], grad=False)[0]
  got = do.loss_fn(spec, online, target, batch, torch.float64)[0]
  assert float(got) == float(want)


# ---- the host twin of the kernels' arithmetic --------------------------------------------------------------------------

def _twin(adv, v, dq):
  from dqn_zoo_b200 import _lib
  A = adv.size
  out = np.zeros(2 * A + 1, np.float32)
  _lib.call('dz_test_dueling_example', adv.ctypes.data, float(v), dq.ctypes.data, A, out.ctypes.data)
  return out[:A], out[A:2 * A], out[2 * A]


@pytest.mark.parametrize('A', [1, 2, 6, 18, 33, 64])
def test_host_twin_within_the_float32_budget(A):
  rs = np.random.RandomState(A)
  worst = 0.0
  for trial in range(200):
    scale = 10.0 ** rs.uniform(-3, 3)
    adv = (scale * rs.standard_normal(A) + (scale * 50 if trial % 4 == 0 else 0.0)).astype(np.float32)
    v = np.float32(scale * rs.standard_normal())
    dq = (scale * rs.standard_normal(A)).astype(np.float32)
    q, dadv, dval = _twin(adv, v, dq)
    a64, v64, g64 = adv.astype(np.float64), float(v), dq.astype(np.float64)
    q_ref = v64 + (a64 - a64.mean())
    dadv_ref = g64 - g64.mean()
    dval_ref = g64.sum()
    worst = max(worst,
                float((np.abs(q - q_ref) / ((A + 3) * U * (abs(v64) + np.abs(a64) + np.abs(a64).mean()))).max()),
                float((np.abs(dadv - dadv_ref) / ((A + 2) * U * (np.abs(g64) + np.abs(g64).mean()) + 1e-300)).max()),
                abs(float(dval) - dval_ref) / (A * U * np.abs(g64).sum() + 1e-300))
    if A == 1:
      assert q[0] == v and dadv[0] == 0.0 and dval == dq[0]
  print('A=%d worst error / budget %.3f' % (A, worst))
  assert worst <= 1.0


def test_host_twin_rejects_bad_arguments():
  from dqn_zoo_b200 import _lib
  x = np.zeros(65, np.float32)
  for A in (0, 65):
    with pytest.raises(ValueError):
      _lib.call('dz_test_dueling_example', x.ctypes.data, 0.0, x.ctypes.data, A, x.ctypes.data)


# ---- the C ABI -------------------------------------------------------------------------------------------------------

def _cfg(kind, dueling, A=6, hw=84):
  from dqn_zoo_b200 import _lib
  cfg = _lib.LearnerConfig(kind=_lib.AGENT_KINDS[kind], num_actions=A, num_atoms=51, num_quantiles=201, latent_dim=64,
                           tau_samples_s_tm1=64, tau_samples_policy=64, tau_samples_s_t=64, batch=32, obs_h=hw, obs_w=hw,
                           obs_c=4, learning_rate=1e-4, opt_eps=1e-5, rms_decay=0.95, adam_b1=0.9, adam_b2=0.999,
                           munchausen_alpha=0.9, entropy_temperature=0.03, log_policy_clip=-1.0)
  cfg.dueling = dueling
  return cfg


def _tensors(cfg):
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(plan))
  name, shape = C.create_string_buffer(64), (C.c_int64 * 4)()
  ndim, off = C.c_int32(), C.c_int64()
  out = []
  for i in range(plan.num_tensors):
    _lib.call('dz_learner_tensor_info', C.byref(cfg), i, name, shape, C.byref(ndim), C.byref(off))
    out.append((name.value.decode(), tuple(shape[k] for k in range(ndim.value)), off.value))
  return plan, out


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('A,hw', [(6, 84), (1, 84), (18, 44), (64, 84)])
def test_layout_names_shapes_and_aligned_offsets(kind, A, hw):
  A = min(A, 18) if kind == 'munchausen' else A   # munchausen's loss takes at most 18 actions
  plan, tensors = _tensors(_cfg(kind, 1, A, hw))
  spec = lo.NetSpec(kind, A, obs_hw=hw)
  want = do.param_shapes(spec)
  assert [(n, s) for n, s, _ in tensors] == list(want.items())
  names = [n for n, _, _ in tensors]
  assert names[6:] == ['adv1/w', 'adv1/b', 'adv2/w', 'adv2/b', 'val1/w', 'val1/b', 'val2/w', 'val2/b']
  end = 0
  for n, s, off in tensors:
    assert off % 4 == 0 and off >= end, n
    end = off + int(np.prod(s))
  assert plan.param_count >= end and plan.noise_floats == 0 and plan.tau_floats == 0
  # the plain network of the same kind is unchanged by the field's existence
  plain = _tensors(_cfg(kind, 0, A, hw))[1]
  assert [n for n, _, _ in plain][6:8] == ['fc1/w', 'fc1/b']


@pytest.mark.parametrize('kind', OTHER_KINDS)
def test_other_kinds_reject_dueling(kind):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  cfg = _cfg(kind, 1)
  with pytest.raises(ValueError, match='dueling'):
    _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(_lib.LearnerPlan()))
  bufs = _lib.LearnerBuffers(0, 0, 0, 0, 0, 0)
  with pytest.raises(ValueError, match='dueling'):
    _lib.call('dz_learner_create', C.byref(cfg), C.byref(bufs), C.byref(C.c_void_p()))
  _tensors(_cfg(kind, 0))   # the same configuration without the field is valid
  with pytest.raises(ValueError, match='dueling'):
    dl.Learner(dl.NetworkSpec(kind, 6, dueling=True))


def test_dueling_field_must_be_zero_or_one():
  from dqn_zoo_b200 import _lib
  with pytest.raises(ValueError, match='dueling'):
    _lib.call('dz_learner_plan_query', C.byref(_cfg('dqn', 2)), C.byref(_lib.LearnerPlan()))


def test_haiku_names_are_stable_and_distinct():
  from dqn_zoo_b200 import learner as dl
  names = list(do.param_shapes(lo.NetSpec('dqn', 6)))
  mods = [dl.haiku_name(n, 'dqn') for n in names]
  assert len(set(mods)) == len(mods)
  assert dl.haiku_name('adv1/w', 'double_q') == ('dueling/advantage/linear', 'w')
  assert dl.haiku_name('val2/b', 'munchausen') == ('dueling/value/linear_1', 'b')
  assert dl.haiku_name('adv1/mu/w', 'rainbow') == ('noisy_linear/mu', 'w')   # rainbow's names are unchanged
