"""CPU oracle for Munchausen DQN (TEST INFRASTRUCTURE ONLY): the float64 restatement of the agent's loss.

Munchausen DQN (Vieillard, Pietquin & Geist, "Munchausen Reinforcement Learning", NeurIPS 2020) is not one of the
reference's agents, so no reference file pins it; this module is its specification (DESIGN.md §13).  The network,
parameter layout and optimizer arithmetic are dqn's and come from `learner_oracle` unchanged; `AGENT_KINDS` there stays
the seven reference kinds and this kind is listed in `EXTRA_KINDS` here.  With qbar the target network's head, q the
online one's and pi(.|s) = softmax(qbar(s, .) / tau), in the stable form

  tau log pi(a|s) = qbar(s, a) - v - tau log sum_a' exp((qbar(s, a') - v) / tau),   v = max_a' qbar(s, a')
  target = r_t + alpha clip(tau log pi(a_tm1|s_tm1), l0, 0) + discount_t sum_a pi(a|s_t) (qbar(s_t, a) - tau log pi(a|s_t))
  td     = target - q(s_tm1, a_tm1)                      (target is stop-gradient)
  loss   = mean_b 0.5 clip_gradient(td, +-grad_error_bound)^2        (dqn/agent.py's form)

The per-example values are the losses 0.5 td^2.
"""

from __future__ import annotations

from typing import NamedTuple

import torch

from oracle import learner_oracle as lo

KIND = 'munchausen'
EXTRA_KINDS = (KIND,)


class Hyper(NamedTuple):
  alpha: float = 0.9          # the paper's Atari values
  tau: float = 0.03
  l0: float = -1.0


def net_spec(kind_spec):
  """The dqn NetSpec with the same geometry: the network of this agent."""
  return kind_spec._replace(kind='dqn')


def head_out(spec):
  return lo.head_out(net_spec(spec))


def param_shapes(spec):
  return lo.param_shapes(net_spec(spec))


def init_params(spec, seed):
  return lo.init_params(net_spec(spec), seed)


def apply_net(spec, p, obs_u8, dtype, tap=None):
  return lo.apply_net(net_spec(spec), p, obs_u8, dtype, tap=tap)


def default_opt():
  """Adam, lr 5e-5, eps 0.01 / 32, no global-norm clip: the paper's Atari values (no reference file pins them)."""
  return lo.OptSpec('adam', 0.00005, 0.01 / 32)


def scaled_log_policy(q, tau):
  """tau log softmax(q / tau) over the last axis, in the stable form above."""
  v = q.max(dim=-1, keepdim=True).values
  return q - v - tau * torch.log(torch.exp((q - v) / tau).sum(dim=-1, keepdim=True))


def target(qbar_tm1, qbar_t, a_tm1, r_t, discount_t, hyper):
  """The munchausen target of every example: qbar_* [B, A], a_tm1 [B] long, r_t / discount_t [B]."""
  rows = torch.arange(qbar_tm1.shape[0])
  bonus = hyper.alpha * scaled_log_policy(qbar_tm1, hyper.tau)[rows, a_tm1].clamp(hyper.l0, 0.0)
  log_pi_t = scaled_log_policy(qbar_t, hyper.tau)
  pi_t = torch.softmax(qbar_t / hyper.tau, dim=-1)
  boot = (pi_t * (qbar_t - log_pi_t)).sum(dim=-1)
  return r_t + bonus + discount_t * boot, bonus


def loss_fn(spec, online, target_params, batch, dtype, weights=None, grad_error_bound=1.0 / 32, hyper=Hyper(), tap=None):
  """(scalar loss, aux) as learner_oracle.loss_fn: aux has 'losses', 'td_errors', 'q_tm1', 'targets', 'bonus'."""
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  a_tm1 = batch['a_tm1'].long()
  r = batch['r_t'].to(torch.float32).to(dtype)
  disc = batch['discount_t'].to(torch.float32).to(dtype)
  q_tm1 = apply_net(spec, online, s_tm1, dtype, tap=tap)['q_values']
  qbar_tm1 = apply_net(spec, target_params, s_tm1, dtype)['q_values'].detach()
  qbar_t = apply_net(spec, target_params, s_t, dtype)['q_values'].detach()
  return head_loss((q_tm1, qbar_tm1, qbar_t), a_tm1, r, disc, weights, grad_error_bound=grad_error_bound, hyper=hyper,
                   grad=False)


def head_loss(heads, a_tm1, r_t, discount_t, weights=None, *, grad_error_bound=1.0 / 32, hyper=Hyper(), grad=True):
  """learner_oracle.head_loss for this agent: heads = (online(s_tm1), target(s_tm1), target(s_t)), each [B, A].
  aux 'per_example' is the loss 0.5 td^2, as the device writes it."""
  q_tm1 = heads[0].detach().clone().requires_grad_(True) if grad else heads[0]
  dtype = q_tm1.dtype
  a_tm1 = torch.as_tensor(a_tm1).long()
  r = torch.as_tensor(r_t).to(torch.float32).to(dtype)
  disc = torch.as_tensor(discount_t).to(torch.float32).to(dtype)
  rows = torch.arange(a_tm1.shape[0])
  qbar_tm1, qbar_t = heads[1].detach(), heads[2].detach()
  tgt, bonus = target(qbar_tm1, qbar_t, a_tm1, r, disc, hyper)
  td = tgt.detach() - q_tm1[rows, a_tm1]
  td_c = lo._ClipGrad.apply(td, -grad_error_bound, grad_error_bound)
  losses = 0.5 * td_c * td_c
  aux = {'losses': losses.detach(), 'td_errors': td.detach(), 'q_tm1': q_tm1.detach(), 'targets': tgt.detach(),
         'bonus': bonus.detach(), 'qbar_tm1': qbar_tm1, 'qbar_t': qbar_t}
  w = None if weights is None else torch.as_tensor(weights).to(torch.float32).to(dtype)
  loss = losses.mean() if w is None else (losses * w).mean()
  aux['per_example'] = aux['losses']
  if grad:
    aux['grad'] = torch.autograd.grad(loss, q_tm1)[0]
  return loss, aux


class Learner(lo.Learner):
  """learner_oracle.Learner with this agent's loss and hyperparameters (`update()` is one learner step)."""

  def __init__(self, spec, params_np, opt=None, dtype=torch.float64, hyper=Hyper(), grad_error_bound=1.0 / 32):
    super().__init__(spec, params_np, opt=opt or default_opt(), dtype=dtype)
    self.hyper = hyper
    self.grad_error_bound = grad_error_bound

  def grads(self, batch, weights=None, taus=None, noise=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, weights, self.grad_error_bound, self.hyper, tap=tap)
    loss.backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g
