"""CPU oracle for Munchausen-IQN (TEST INFRASTRUCTURE ONLY): the float64 restatement of the agent's loss.

Munchausen-IQN (Vieillard, Pietquin & Geist, "Munchausen Reinforcement Learning", NeurIPS 2020) is not one of the
reference's agents, so no reference file pins it; this module is its specification (DESIGN.md §14).  The network,
parameter layout, taus and optimizer arithmetic are iqn's and come from `learner_oracle` unchanged, as does
`quantile_regression_loss`; `AGENT_KINDS` there stays the seven reference kinds and this kind is listed in
`EXTRA_KINDS` here.  With Zbar_j the target network's quantile outputs at tau sample j, Z the online one's,
qbar(s, a) the mean of Zbar over that pass's samples and pi(.|s) = softmax(qbar(s, .) / tau):

  h(a)    = v + tau log S - qbar(a) = -tau log pi(a|s),   v = max_a qbar(s, a),  S = sum_a exp((qbar(s, a) - v) / tau)
  bonus   = alpha clip(tau log pi(a_tm1|s_tm1), l0, 0)          (qbar from target(s_tm1) at the K policy taus)
  y_j     = r_t + bonus + discount_t sum_a pi(a|s_t) (Zbar_j(s_t, a) + h_t(a))     j < N'  (qbar at s_t from the same N')
  loss_b  = quantile_regression_loss(Z_i(s_tm1, a_tm1) at tau_tm1_i, i < N; y_j stop-gradient; kappa = huber_param)
  loss    = mean_b w_b loss_b

The per-example values are the losses loss_b.
"""

from __future__ import annotations

from typing import NamedTuple

import torch

from oracle import learner_oracle as lo

KIND = 'munchausen_iqn'
EXTRA_KINDS = (KIND,)


class Hyper(NamedTuple):
  alpha: float = 0.9          # the paper's Atari values
  tau: float = 0.03
  l0: float = -1.0


def net_spec(kind_spec):
  """The iqn NetSpec with the same geometry: the network of this agent."""
  return kind_spec._replace(kind='iqn')


def head_out(spec):
  return lo.head_out(net_spec(spec))


def param_shapes(spec):
  return lo.param_shapes(net_spec(spec))


def init_params(spec, seed):
  return lo.init_params(net_spec(spec), seed)


def apply_net(spec, p, obs_u8, dtype, taus, tap=None):
  return lo.apply_net(net_spec(spec), p, obs_u8, dtype, taus=taus, tap=tap)


def default_opt():
  """iqn's Adam: lr 5e-5, eps 0.01 / 32, no global-norm clip."""
  return lo.default_opt('iqn')


def soft_terms(qbar, tau):
  """(pi, h) over the last axis: the softmax policy pi = softmax(qbar / tau) and h = v + tau log S - qbar >= 0."""
  v = qbar.max(dim=-1, keepdim=True).values
  e = torch.exp((qbar - v) / tau)
  s = e.sum(dim=-1, keepdim=True)
  return e / s, (v - qbar) + tau * torch.log(s)


def target(zbar_tm1, zbar_t, a_tm1, r_t, discount_t, hyper):
  """The targets y [B, N'] of every example, with the bonus [B] and the entropy term sum_a pi h [B]:
  zbar_tm1 [B, K, A] (target(s_tm1) at the policy taus), zbar_t [B, N', A], a_tm1 [B] long, r_t / discount_t [B]."""
  rows = torch.arange(zbar_tm1.shape[0])
  pi_tm1, h_tm1 = soft_terms(zbar_tm1.mean(dim=1), hyper.tau)
  bonus = hyper.alpha * (-h_tm1[rows, a_tm1]).clamp(hyper.l0, 0.0)
  pi_t, h_t = soft_terms(zbar_t.mean(dim=1), hyper.tau)
  ent = (pi_t * h_t).sum(dim=-1)
  boot = (pi_t[:, None, :] * (zbar_t + h_t[:, None, :])).sum(dim=-1)
  return (r_t + bonus)[:, None] + discount_t[:, None] * boot, bonus, ent


def loss_fn(spec, online, target_params, batch, dtype, taus, weights=None, huber_param=1.0, hyper=Hyper(), tap=None):
  """(scalar loss, aux) as learner_oracle.loss_fn; taus = (tau_tm1 [B, N], tau_policy [B, K], tau_t [B, N']).
  aux has 'losses', 'targets', 'bonus', 'entropy', 'dist_tm1', 'qbar_tm1' and 'qbar_t'."""
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  a_tm1 = batch['a_tm1'].long()
  r = batch['r_t'].to(torch.float32).to(dtype)
  disc = batch['discount_t'].to(torch.float32).to(dtype)
  tau_tm1, tau_pol, tau_t = taus
  dist_tm1 = apply_net(spec, online, s_tm1, dtype, tau_tm1, tap=tap)['q_dist']
  zbar_tm1 = apply_net(spec, target_params, s_tm1, dtype, tau_pol)['q_dist'].detach()
  zbar_t = apply_net(spec, target_params, s_t, dtype, tau_t)['q_dist'].detach()
  return head_loss((dist_tm1, zbar_tm1, zbar_t), a_tm1, r, disc, tau_tm1, weights, huber_param=huber_param, hyper=hyper,
                   grad=False)


def head_loss(heads, a_tm1, r_t, discount_t, taus, weights=None, *, huber_param=1.0, hyper=Hyper(), grad=True):
  """learner_oracle.head_loss for this agent: heads = (online(s_tm1) [B, N, A], target(s_tm1) at the policy taus
  [B, K, A], target(s_t) [B, N', A]); taus: the s_tm1 taus [B, N].  aux 'per_example' is the loss."""
  dist_tm1 = heads[0].detach().clone().requires_grad_(True) if grad else heads[0]
  dtype = dist_tm1.dtype
  a_tm1 = torch.as_tensor(a_tm1).long()
  r = torch.as_tensor(r_t).to(torch.float32).to(dtype)
  disc = torch.as_tensor(discount_t).to(torch.float32).to(dtype)
  rows = torch.arange(a_tm1.shape[0])
  zbar_tm1, zbar_t = heads[1].detach(), heads[2].detach()
  y, bonus, ent = target(zbar_tm1, zbar_t, a_tm1, r, disc, hyper)
  losses = lo.quantile_regression_loss(dist_tm1[rows, :, a_tm1], torch.as_tensor(taus).to(dtype), y.detach(), huber_param)
  aux = {'losses': losses.detach(), 'targets': y.detach(), 'bonus': bonus.detach(), 'entropy': ent.detach(),
         'dist_tm1': dist_tm1.detach(), 'qbar_tm1': zbar_tm1.mean(dim=1), 'qbar_t': zbar_t.mean(dim=1)}
  w = None if weights is None else torch.as_tensor(weights).to(torch.float32).to(dtype)
  loss = losses.mean() if w is None else (losses * w).mean()
  aux['per_example'] = aux['losses']
  if grad:
    aux['grad'] = torch.autograd.grad(loss, dist_tm1)[0]
  return loss, aux


class Learner(lo.Learner):
  """learner_oracle.Learner with this agent's loss and hyperparameters (`update()` is one learner step)."""

  def __init__(self, spec, params_np, opt=None, dtype=torch.float64, hyper=Hyper(), huber_param=1.0):
    super().__init__(net_spec(spec), params_np, opt=opt or default_opt(), dtype=dtype)
    self.hyper = hyper
    self.huber_param = huber_param

  def grads(self, batch, weights=None, taus=None, noise=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, taus, weights, self.huber_param, self.hyper,
                        tap=tap)
    loss.backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g
