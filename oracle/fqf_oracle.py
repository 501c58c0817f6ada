"""CPU oracle for FQF (TEST INFRASTRUCTURE ONLY): the float64 restatement of the agent's step.

FQF, the Fully parameterized Quantile Function (Yang et al., "Fully Parameterized Quantile Function for Distributional
Reinforcement Learning", NeurIPS 2019), is not one of the reference's agents, so no reference file pins it; this module
is its specification (DESIGN.md §15).  The quantile network Z(s, a, tau) is iqn's and comes from `learner_oracle`
unchanged, as do `quantile_regression_loss` and the optimizer arithmetic; `AGENT_KINDS` there stays the seven reference
kinds and this kind is listed in `EXTRA_KINDS` here.  With phi / phibar the online / target torso features and
W_f [feat, N], b_f [N] the fraction layer of the online parameters:

  P(phi):    q = softmax(phi W_f + b_f), tau_0 = 0, tau_i = sum_{k<i} q_k, tau_N = 1, tau_hat_i = (tau_i + tau_{i+1}) / 2,
             w_i = tau_{i+1} - tau_i
  s_tm1:     tau, tau_hat = P(stop_grad phi(s_tm1));   s_t: tau', tau_hat' = P(stop_grad phibar(s_t))
  a*         = argmax_a sum_i w'_i Zbar(s_t, a, tau_hat'_i)                     (first maximum)
  y_j        = r_t + discount_t Zbar(s_t, a*, tau_hat_j), j < N                 (stop-gradient)
  loss_b     = quantile_regression_loss(Z(s_tm1, a_tm1, tau_hat_i), i < N, at tau_hat; y; kappa = huber_param)
  dW1/dtau_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}), i = 1..N-1, F(tau) = Z(s_tm1, a_tm1, tau), no gradient into Z
  loss       = mean_b w_b loss_b; the fraction loss takes the same weights: its gradient is
             mean_b w_b sum_i dW1/dtau_i dtau_i/dtheta_f, through the cumsum and the softmax (autograd here)

The per-example values are the quantile losses loss_b.  Optimizers: the configured one (Adam, lr 5e-5, eps 0.01 / 32, no
clip) over every tensor but the fraction layer, whose norm alone is reported; centred RMSProp over the fraction layer.
"""

from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

from oracle import learner_oracle as lo

KIND = 'fqf'
EXTRA_KINDS = (KIND,)
FRACTION_TENSORS = ('fraction/w', 'fraction/b')


class Hyper(NamedTuple):
  num_fractions: int = 32
  fraction_learning_rate: float = 2.5e-9
  fraction_opt_eps: float = 1e-5
  fraction_rms_decay: float = 0.95


def net_spec(kind_spec):
  """The iqn NetSpec with the same geometry: the quantile network of this agent."""
  return kind_spec._replace(kind='iqn')


def param_shapes(spec, num_fractions=32):
  shapes = lo.param_shapes(net_spec(spec))
  shapes['fraction/w'] = (lo.feature_dim(spec), num_fractions)
  shapes['fraction/b'] = (num_fractions,)
  return shapes


def init_params(spec, seed, num_fractions=32):
  """iqn's init for the quantile network (the same RandomState stream, in layout order), then fraction/w
  U(+-0.01/sqrt(fan_in)) and fraction/b zero, as `Learner.init_params`."""
  rs = np.random.RandomState(seed)
  params = {}
  for name, shape in param_shapes(spec, num_fractions).items():
    n_in = int(np.prod(param_shapes(spec, num_fractions)[name.rsplit('/', 1)[0] + '/w'][:-1]))
    bound = math.sqrt(1.0 / n_in)
    if name == 'fraction/w':
      params[name] = rs.uniform(-0.01 * bound, 0.01 * bound, size=shape).astype(np.float32)
    elif name == 'fraction/b':
      params[name] = np.zeros(shape, np.float32)
    else:
      params[name] = rs.uniform(-bound, bound, size=shape).astype(np.float32)
  return params


def default_opt():
  """iqn's Adam over every tensor but the fraction layer: lr 5e-5, eps 0.01 / 32, no global-norm clip."""
  return lo.default_opt('iqn')


def fraction_opt(hyper=Hyper()):
  return lo.OptSpec('rmsprop', hyper.fraction_learning_rate, hyper.fraction_opt_eps, decay=hyper.fraction_rms_decay)


def proposal(logits):
  """P of a batch of logits [B, N]: dict q, tau [B, N+1], tau_hat [B, N], w [B, N] (differentiable in the logits)."""
  q = torch.softmax(logits, dim=-1)
  B = logits.shape[0]
  zero = torch.zeros((B, 1), dtype=logits.dtype)
  tau = torch.cat([zero, torch.cumsum(q, dim=-1)[:, :-1], torch.ones((B, 1), dtype=logits.dtype)], dim=-1)
  return {'logits': logits, 'q': q, 'tau': tau, 'tau_hat': 0.5 * (tau[:, :-1] + tau[:, 1:]), 'w': tau[:, 1:] - tau[:, :-1]}


def fractions(p, feat):
  return proposal(feat @ p['fraction/w'] + p['fraction/b'])


def quantiles(spec, p, obs_u8, dtype, taus, tap=None):
  """Z(s, ., tau) [B, n, A] of iqn's network at taus [B, n]."""
  return lo.apply_net(net_spec(spec), p, obs_u8, dtype, taus=taus, tap=tap)['q_dist']


def tau_gradient(F_tau, F_hat):
  """dW1/dtau_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}) for i = 1..N-1: F_tau [B, N-1] at tau_1..tau_{N-1},
  F_hat [B, N] at tau_hat -> [B, N-1]."""
  return 2.0 * F_tau - F_hat[:, 1:] - F_hat[:, :-1]


def dlogits_of(g, q, cot):
  """The explicit chain of dW1/dtau [B, N-1] (i = 1..N-1) through tau_i = sum_{k<i} q_k and q = softmax(logits):
  dq_k = sum_{i>k} g_i, dlogit_k = q_k (dq_k - sum_j q_j dq_j), scaled by cot [B] (w_b / B)."""
  B, N = q.shape
  gg = torch.cat([torch.zeros((B, 1), dtype=g.dtype), g], dim=-1)                 # index i = 0..N-1 (g_0 unused)
  dq = torch.flip(torch.cumsum(torch.flip(gg, [-1]), -1), [-1]) - gg              # sum_{i > k} g_i
  return cot[:, None] * q * (dq - (q * dq).sum(-1, keepdim=True))


def head_loss(heads, a_tm1, r_t, discount_t, tau_hat, w_t, weights=None, *, huber_param=1.0):
  """The loss from the head outputs: heads = (online(s_tm1) at tau_hat [B, N, A], online(s_tm1) at tau_1..tau_{N-1}
  [B, N-1, A], target(s_t) at tau_hat' [B, N, A], target(s_t) at tau_hat [B, N, A]); tau_hat [B, N]; w_t [B, N] the
  interval weights of s_t's proposal.  Returns (scalar loss, aux): 'losses', 'a_star', 'targets', 'tau_grad'
  (dW1/dtau [B, N-1], detached) and 'cot' (w_b / B)."""
  dist_tm1 = heads[0]
  dtype = dist_tm1.dtype
  a_tm1 = torch.as_tensor(a_tm1).long()
  r = torch.as_tensor(r_t).to(torch.float32).to(dtype)
  disc = torch.as_tensor(discount_t).to(torch.float32).to(dtype)
  rows = torch.arange(a_tm1.shape[0])
  zsel, ztgt = heads[2].detach(), heads[3].detach()
  qsel = (torch.as_tensor(w_t).to(dtype)[:, :, None] * zsel).sum(1)
  a_star = qsel.argmax(dim=1)
  y = (r[:, None] + disc[:, None] * ztgt[rows, :, a_star]).detach()
  losses = lo.quantile_regression_loss(dist_tm1[rows, :, a_tm1], torch.as_tensor(tau_hat).to(dtype).detach(), y,
                                       huber_param)
  w = None if weights is None else torch.as_tensor(weights).to(torch.float32).to(dtype)
  loss = losses.mean() if w is None else (losses * w).mean()
  B = a_tm1.shape[0]
  cot = (torch.ones(B, dtype=dtype) if w is None else w) / B
  g = tau_gradient(heads[1].detach()[rows, :, a_tm1], dist_tm1.detach()[rows, :, a_tm1])
  aux = {'losses': losses.detach(), 'per_example': losses.detach(), 'a_star': a_star, 'targets': y, 'qsel': qsel,
         'tau_grad': g, 'cot': cot, 'dist_tm1': dist_tm1.detach()}
  return loss, aux


def loss_fn(spec, online, target_params, batch, dtype, weights=None, huber_param=1.0, tap=None, device_fractions=None):
  """(scalar loss, aux).  aux['fraction_objective'] is the surrogate sum_b cot_b sum_i dW1/dtau_i tau_i(theta_f), whose
  gradient is the fraction layer's; the loss itself reaches no fraction tensor.  `device_fractions` = (tau, tau_hat) of
  the s_tm1 and s_t proposals as float32 arrays [B, N+1], [B, N] (e.g. read from the device): the quantile network is
  then evaluated at those taus, so both sides feed the same float32 taus to the cosine embedding; the fraction layer's
  own float64 proposals are in aux 'prop_tm1' / 'prop_t' either way."""
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  feat_tm1 = lo.torso(online, s_tm1, dtype).detach()
  feat_t = lo.torso(target_params, s_t, dtype).detach()
  prop0 = fractions(online, feat_tm1)
  prop1 = {k: v.detach() for k, v in fractions(online, feat_t).items()}
  if device_fractions is None:
    tau0, hat0, tau1, hat1 = prop0['tau'].detach(), prop0['tau_hat'].detach(), prop1['tau'], prop1['tau_hat']
  else:
    tau0, hat0, tau1, hat1 = (torch.as_tensor(np.asarray(x, np.float32)).to(dtype) for x in device_fractions)
  heads = (quantiles(spec, online, s_tm1, dtype, hat0, tap=tap),
           quantiles(spec, online, s_tm1, dtype, tau0[:, 1:-1]).detach(),
           quantiles(spec, target_params, s_t, dtype, hat1).detach(),
           quantiles(spec, target_params, s_t, dtype, hat0).detach())
  loss, aux = head_loss(heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], hat0, tau1[:, 1:] - tau1[:, :-1],
                        weights, huber_param=huber_param)
  aux['fraction_objective'] = (aux['cot'][:, None] * aux['tau_grad'] * prop0['tau'][:, 1:-1]).sum()
  aux['prop_tm1'] = {k: v.detach() for k, v in prop0.items()}
  aux['prop_t'] = prop1
  return loss, aux


class Learner(lo.Learner):
  """learner_oracle.Learner with this agent's loss and its two optimizers (`update()` is one learner step)."""

  def __init__(self, spec, params_np, opt=None, dtype=torch.float64, hyper=Hyper(), huber_param=1.0):
    super().__init__(net_spec(spec), params_np, opt=opt or default_opt(), dtype=dtype)
    self.hyper = hyper
    self.huber_param = huber_param
    self.frac_opt = fraction_opt(hyper)

  def grads(self, batch, weights=None, device_fractions=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, weights, self.huber_param, tap=tap,
                        device_fractions=device_fractions)
    (loss + aux['fraction_objective']).backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g

  def update(self, batch, weights=None, device_fractions=None, tap=None):
    loss, aux, g = self.grads(batch, weights, device_fractions, tap=tap)
    main = [k for k in self.online if k not in FRACTION_TENSORS]
    new_p, st, gn = lo.optimizer_step(self.opt, {k: self.online[k] for k in main}, {k: g[k] for k in main}, self.state)
    fst = {'mu': {k: self.state['mu'][k] for k in FRACTION_TENSORS}, 'nu': {k: self.state['nu'][k] for k in FRACTION_TENSORS}}
    new_f, fst, _ = lo.optimizer_step(self.frac_opt, {k: self.online[k] for k in FRACTION_TENSORS},
                                      {k: g[k] for k in FRACTION_TENSORS}, fst)
    for part in ('mu', 'nu'):
      st[part].update(fst[part])
    self.online, self.state = dict(new_p, **new_f), st
    return dict(aux, loss=loss, grads=g, global_norm=gn)
