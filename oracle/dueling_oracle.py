"""CPU oracle for the dueling network (TEST INFRASTRUCTURE ONLY): the float64 restatement of dqn, double_q, prioritized
and munchausen on the dueling network of Wang et al., "Dueling Network Architectures for Deep Reinforcement Learning",
ICML 2016 (DESIGN.md §16).

The reference has the dueling aggregation only inside rainbow's noisy, distributional network, so this module is the
specification of the plain one.  After dqn's torso, two streams of the same shape as dqn's fc1 / head:

  adv = relu(feat adv1/w + adv1/b) adv2/w + adv2/b          [B, A]
  v   = relu(feat val1/w + val1/b) val2/w + val2/b          [B, 1]
  q   = v + (adv - mean_a adv)                              (learner_oracle.dueling with one atom)

Every loss, optimizer and priority rule is the kind's own, applied to q: learner_oracle.head_loss for dqn, double_q and
prioritized, munchausen_oracle.head_loss for munchausen.  `learner_oracle.AGENT_KINDS` and its results are unchanged.
"""

from __future__ import annotations

import math

import numpy as np
import torch

from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo

KINDS = ('dqn', 'double_q', 'prioritized', 'munchausen')


def param_shapes(spec):
  """Ordered {name: shape}: the conv tensors, then the advantage stream, then the value stream (the device layout)."""
  d = lo.feature_dim(spec)
  out = {k: v for k, v in lo.param_shapes(spec._replace(kind='dqn')).items() if k.startswith('conv')}
  for stream, n_out in (('adv', spec.num_actions), ('val', 1)):
    out[stream + '1/w'] = (d, 512)
    out[stream + '1/b'] = (512,)
    out[stream + '2/w'] = (512, n_out)
    out[stream + '2/b'] = (n_out,)
  return out


def init_params(spec, seed):
  """The legacy U(+-1/sqrt(fan_in)) init of learner_oracle.init_params for all eight stream tensors, in layout order."""
  rs = np.random.RandomState(seed)
  shapes = param_shapes(spec)
  params = {}
  for name, shape in shapes.items():
    n_in = int(np.prod(shapes[name.rsplit('/', 1)[0] + '/w'][:-1]))
    bound = math.sqrt(1.0 / n_in)
    params[name] = rs.uniform(-bound, bound, size=shape).astype(np.float32)
  return params


def streams(p, feat, tap=None):
  """(adv [B, A], v [B, 1]) of the two streams on torso features feat."""
  h_adv = lo._relu(feat @ p['adv1/w'] + p['adv1/b'], tap, 'adv1')
  h_val = lo._relu(feat @ p['val1/w'] + p['val1/b'], tap, 'val1')
  return h_adv @ p['adv2/w'] + p['adv2/b'], h_val @ p['val2/w'] + p['val2/b']


def aggregate(adv, v):
  """q [B, A] = v + (adv - mean_a adv): learner_oracle.dueling with one atom."""
  return lo.dueling(adv[:, :, None], v)[:, :, 0]


def apply_net(spec, p, obs_u8, dtype, tap=None):
  """One network apply: {'q_values', 'adv', 'val'}.  `tap`: optional learner_oracle.ReluTap (names 'conv1'..'conv3',
  'adv1', 'val1')."""
  adv, v = streams(p, lo.torso(p, obs_u8, dtype, tap), tap)
  return {'q_values': aggregate(adv, v), 'adv': adv, 'val': v[:, 0]}


def default_opt(kind):
  return mo.default_opt() if kind == 'munchausen' else lo.default_opt(kind)


def loss_fn(spec, online, target, batch, dtype, weights=None, grad_error_bound=1.0 / 32, hyper=mo.Hyper(), tap=None):
  """(scalar loss, aux) of the kind's loss on the dueling network's q-values."""
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  q0 = apply_net(spec, online, s_tm1, dtype, tap=tap)['q_values']
  if spec.kind == 'munchausen':
    heads = (q0, apply_net(spec, target, s_tm1, dtype)['q_values'], apply_net(spec, target, s_t, dtype)['q_values'])
    return mo.head_loss(heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], weights,
                        grad_error_bound=grad_error_bound, hyper=hyper, grad=False)
  sel = apply_net(spec, online, s_t, dtype)['q_values'] if spec.kind in ('double_q', 'prioritized') else None
  heads = [q0, sel, apply_net(spec, target, s_t, dtype)['q_values']]
  return lo.head_loss(spec.kind, heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], weights,
                      grad_error_bound=grad_error_bound, grad=False)


class Learner(lo.Learner):
  """learner_oracle.Learner on the dueling network (`update()` is one learner step of the kind)."""

  def __init__(self, spec, params_np, opt=None, dtype=torch.float64, grad_error_bound=1.0 / 32, hyper=mo.Hyper()):
    if spec.kind not in KINDS:
      raise ValueError(spec.kind)
    super().__init__(spec, params_np, opt=opt or default_opt(spec.kind), dtype=dtype, grad_error_bound=grad_error_bound)
    self.hyper = hyper

  def grads(self, batch, weights=None, taus=None, noise=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, weights, self.grad_error_bound, self.hyper, tap=tap)
    loss.backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g

