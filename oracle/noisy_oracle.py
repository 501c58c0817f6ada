"""CPU oracle for noisy networks (TEST INFRASTRUCTURE ONLY): the float64 restatement of dqn, double_q, prioritized and
munchausen on the factorised-noise networks of Fortunato et al., "Noisy Networks for Exploration", ICLR 2018
(DESIGN.md §17).

Every linear layer after dqn's torso is the reference's noisy_linear with a mu bias (learner_oracle._noisy with
with_bias=True):

  y = x mu/w + mu/b + ((x * eps_in) sigma/w + sigma/b) * eps_out

with eps = f(e) = sign(e) sqrt|e| given as an input, one vector per input side and per output side of each layer.

  plain:    q = noisy(relu(noisy(feat, fc1)), head)                                   [B, A]
  dueling:  adv = noisy(relu(noisy(feat, adv1)), adv2), v = noisy(relu(noisy(feat, val1)), val2),
            q = v + (adv - mean_a adv)                                                (dueling_oracle.aggregate)

One learner step takes three noise applies, rainbow's slots: slot 0 online(s_tm1), slot 1 the middle pass
(online(s_t) for double_q and prioritized, target(s_tm1) for munchausen; dqn reads none), slot 2 target(s_t).  Every
loss, optimizer and priority rule is the kind's own (learner_oracle.head_loss, munchausen_oracle.head_loss).
"""

from __future__ import annotations

import math

import numpy as np
import torch

from oracle import dueling_oracle as do
from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo

KINDS = do.KINDS


def layers(spec, dueling):
  """(name, n_in, n_out) of the noisy layers in layout order."""
  d, a = lo.feature_dim(spec), spec.num_actions
  if dueling:
    return [('adv1', d, 512), ('adv2', 512, a), ('val1', d, 512), ('val2', 512, 1)]
  return [('fc1', d, 512), ('head', 512, a)]


def param_shapes(spec, dueling=False):
  """Ordered {name: shape}: the conv tensors, then mu/w, mu/b, sigma/w, sigma/b of each layer (the device layout)."""
  out = {k: v for k, v in lo.param_shapes(spec._replace(kind='dqn')).items() if k.startswith('conv')}
  for name, n_in, n_out in layers(spec, dueling):
    for part in ('mu', 'sigma'):
      out['%s/%s/w' % (name, part)] = (n_in, n_out)
      out['%s/%s/b' % (name, part)] = (n_out,)
  return out


def init_params(spec, seed, dueling=False):
  """mu: the legacy U(+-1/sqrt(fan_in)) for weights and biases; sigma: noisy_sigma0 / sqrt(fan_in) (rainbow's), in
  layout order: the draws of `Learner.init_params`."""
  rs = np.random.RandomState(seed)
  shapes = param_shapes(spec, dueling)
  params = {}
  for name, shape in shapes.items():
    n_in = int(np.prod(shapes[name.rsplit('/', 1)[0] + '/w'][:-1]))
    if '/sigma/' in name:
      params[name] = np.full(shape, spec.noisy_sigma0 / math.sqrt(n_in), dtype=np.float32)
    else:
      bound = math.sqrt(1.0 / n_in)
      params[name] = rs.uniform(-bound, bound, size=shape).astype(np.float32)
  return params


def noise_shapes(spec, dueling=False):
  """(name, length) of the noise vectors of ONE apply, in the device order."""
  return [(v, n) for name, n_in, n_out in layers(spec, dueling) for v, n in ((name + '/in', n_in), (name + '/out', n_out))]


def slot_of_pass(kind):
  """The noise slot each head pass of the learner step reads: (pass 0, middle pass or None, target(s_t))."""
  return (0, None if kind == 'dqn' else 1, 2)


def apply_net(spec, p, obs_u8, dtype, noise, dueling=False, tap=None):
  """One network apply on one noise apply {name: [n]}: {'q_values'} (dueling: also 'adv', 'val').  `tap`: optional
  learner_oracle.ReluTap (names 'conv1'..'conv3' and 'fc1', or 'adv1' and 'val1')."""
  feat = lo.torso(p, obs_u8, dtype, tap)
  n = {name: torch.as_tensor(noise[name]).to(dtype)[None, :] for name, _ in noise_shapes(spec, dueling)}

  def layer(name, x):
    return lo._noisy(p, name, x, n[name + '/in'], n[name + '/out'], True)

  if not dueling:
    return {'q_values': layer('head', lo._relu(layer('fc1', feat), tap, 'fc1'))}
  adv = layer('adv2', lo._relu(layer('adv1', feat), tap, 'adv1'))
  v = layer('val2', lo._relu(layer('val1', feat), tap, 'val1'))
  return {'q_values': do.aggregate(adv, v), 'adv': adv, 'val': v[:, 0]}


def loss_fn(spec, online, target, batch, dtype, noise, dueling=False, weights=None, grad_error_bound=1.0 / 32,
            hyper=mo.Hyper(), tap=None):
  """(scalar loss, aux) of the kind's loss on the noisy network; noise: the step's three applies (slots 0, 1, 2)."""
  s_tm1, s_t = batch['s_tm1'], batch['s_t']

  def q(p, s, slot, tap=None):
    return apply_net(spec, p, s, dtype, noise[slot], dueling, tap)['q_values']

  q0 = q(online, s_tm1, 0, tap)
  if spec.kind == 'munchausen':
    heads = (q0, q(target, s_tm1, 1), q(target, s_t, 2))
    return mo.head_loss(heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], weights,
                        grad_error_bound=grad_error_bound, hyper=hyper, grad=False)
  sel = q(online, s_t, 1) if spec.kind in ('double_q', 'prioritized') else None
  heads = [q0, sel, q(target, s_t, 2)]
  return lo.head_loss(spec.kind, heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], weights,
                      grad_error_bound=grad_error_bound, grad=False)


class Learner(lo.Learner):
  """learner_oracle.Learner on the noisy network (`update()` is one learner step of the kind; `noise` its three
  applies)."""

  def __init__(self, spec, params_np, dueling=False, opt=None, dtype=torch.float64, grad_error_bound=1.0 / 32,
               hyper=mo.Hyper()):
    if spec.kind not in KINDS:
      raise ValueError(spec.kind)
    super().__init__(spec, params_np, opt=opt or do.default_opt(spec.kind), dtype=dtype, grad_error_bound=grad_error_bound)
    self.dueling, self.hyper = dueling, hyper

  def grads(self, batch, weights=None, taus=None, noise=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, noise, self.dueling, weights,
                        self.grad_error_bound, self.hyper, tap=tap)
    loss.backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g
