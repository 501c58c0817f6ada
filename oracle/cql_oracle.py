"""CPU oracle for conservative Q-learning (TEST INFRASTRUCTURE ONLY): the float64 restatement of the CQL(H) term that
every agent kind's loss takes when `cql_alpha` > 0 (DESIGN.md §20).

CQL (Kumar, Zhou, Tucker & Levine, "Conservative Q-Learning for Offline Reinforcement Learning", NeurIPS 2020) is not in
the reference, so this module is its specification.  It builds on the kind oracles (learner_oracle, munchausen_oracle,
munchausen_iqn_oracle, fqf_oracle, dueling_oracle, noisy_oracle) without changing them.  For example b, Q_a is the
online network's expected value on s_tm1 from the update's pass-0 head outputs:

  dqn, double_q, prioritized, munchausen (plain, dueling, noisy)   q_a, the head output (after the dueling aggregation)
  c51, rainbow                                                      sum_k softmax(logits_a)_k z_k (rainbow: the
                                                                    dueling-aggregated logits under noise apply 0)
  qrdqn, iqn, munchausen_iqn                                        the mean of the N pass-0 quantiles of action a
  fqf                                                               sum_i w_i Z(s_tm1, tau_hat_i, a), the interval
                                                                    weights w_i of s_tm1's proposal held constant

  R_b  = logsumexp_a Q_a - Q_{a_tm1} >= 0
  loss = mean_b w_b (loss_b + alpha R_b)

loss_b, the per-example values, the priorities and fqf's fraction loss are the kind's own; the added gradient
(alpha w_b / B)(softmax(Q)_a - [a = a_tm1]) wrt Q_a is not clipped by the dqn family's clip_gradient.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import dueling_oracle as do
from oracle import fqf_oracle as fo
from oracle import learner_oracle as lo
from oracle import munchausen_iqn_oracle as mio
from oracle import munchausen_oracle as mo
from oracle import noisy_oracle as no

KINDS = ('dqn', 'double_q', 'prioritized', 'munchausen', 'c51', 'rainbow', 'qrdqn', 'iqn', 'munchausen_iqn', 'fqf')


def regularizer(q, a_tm1):
  """R [B] = logsumexp_a q - q[a_tm1] of expected values q [B, A]."""
  rows = torch.arange(q.shape[0])
  return torch.logsumexp(q, dim=-1) - q[rows, torch.as_tensor(a_tm1).long()]


def expected_q(kind, head0, vmax=10.0, frac_w=None):
  """Q [B, A] of the pass-0 head outputs in the device layout: dqn family [B, A]; c51 logits [B, A, K]; rainbow
  (adv [B, A, K], val [B, K]); qrdqn / iqn / munchausen_iqn / fqf [B, N, A], fqf weighted by frac_w [B, N]."""
  if kind in ('dqn', 'double_q', 'prioritized', 'munchausen'):
    return head0
  if kind in ('c51', 'rainbow'):
    logits = lo.dueling(*head0) if kind == 'rainbow' else head0
    z = torch.tensor(np.linspace(-vmax, vmax, logits.shape[-1]).astype(np.float32)).to(logits.dtype)
    return (F.softmax(logits, dim=-1) * z).sum(-1)
  if kind in ('qrdqn', 'iqn', 'munchausen_iqn'):
    return head0.mean(dim=1)
  if kind == 'fqf':
    return (torch.as_tensor(frac_w).to(head0.dtype)[:, :, None] * head0).sum(1)
  raise ValueError(kind)


def _weights(weights, B, dtype):
  if weights is None:
    return torch.ones(B, dtype=dtype)
  return torch.as_tensor(weights).to(torch.float32).to(dtype)


def term(q, a_tm1, alpha, weights=None):
  """(alpha mean_b w_b R_b, R [B]) of expected values q [B, A]; weights rounded to float32 as the device takes them."""
  R = regularizer(q, a_tm1)
  return alpha * (_weights(weights, q.shape[0], q.dtype) * R).mean(), R


def head_grad(kind, head0, a_tm1, alpha, weights=None, vmax=10.0, frac_w=None):
  """(R [B], the gradient of alpha mean_b w_b R_b wrt the pass-0 head outputs: a tensor, or (d adv, d val) for
  rainbow).  By autograd."""
  parts = list(head0) if kind == 'rainbow' else [head0]
  parts = [x.detach().clone().requires_grad_(True) for x in parts]
  t, R = term(expected_q(kind, tuple(parts) if kind == 'rainbow' else parts[0], vmax, frac_w), a_tm1, alpha, weights)
  g = torch.autograd.grad(t, parts)
  return R.detach(), (tuple(g) if kind == 'rainbow' else g[0])


def pass0_q(O, p, batch, taus=None, noise=None, device_fractions=None, tap=None):
  """Q [B, A] of online(s_tm1) for the kind oracle learner O on parameters p (differentiable in p): the same network
  apply as O's pass 0, with the same taus, noise, fractions and ReluTap."""
  s, dtype, spec = batch['s_tm1'], O.dtype, O.spec
  if isinstance(O, fo.Learner):
    if device_fractions is None:
      prop = fo.fractions(p, lo.torso(p, s, dtype).detach())
      tau0, hat0 = prop['tau'].detach(), prop['tau_hat'].detach()
    else:
      tau0, hat0 = (torch.as_tensor(np.asarray(x, np.float32)).to(dtype) for x in device_fractions[:2])
    return expected_q('fqf', fo.quantiles(spec, p, s, dtype, hat0, tap=tap), frac_w=tau0[:, 1:] - tau0[:, :-1])
  if isinstance(O, mio.Learner):
    return mio.apply_net(spec, p, s, dtype, taus[0], tap=tap)['q_dist'].mean(dim=1)
  if isinstance(O, no.Learner):
    return no.apply_net(spec, p, s, dtype, noise[0], O.dueling, tap)['q_values']
  if isinstance(O, do.Learner):
    return do.apply_net(spec, p, s, dtype, tap=tap)['q_values']
  if isinstance(O, mo.Learner):
    return mo.apply_net(spec, p, s, dtype, tap=tap)['q_values']
  kind = spec.kind
  h = lo.apply_net(spec, p, s, dtype, taus=None if taus is None else taus[0], noise=None if noise is None else noise[0],
                   tap=tap)
  if kind in ('c51', 'rainbow'):
    return expected_q(kind, (h['adv'], h['val']) if kind == 'rainbow' else h['q_logits'], spec.vmax)
  if kind in ('qrdqn', 'iqn'):
    return h['q_dist'].mean(dim=1)
  return h['q_values']


def grads(O, batch, alpha, kind_result, weights=None, taus=None, noise=None, device_fractions=None, tap=None):
  """The CQL update's (loss, aux, grads) from the kind's own `kind_result` = O.grads(...) on the same batch and
  inputs: the loss plus alpha mean_b w_b R_b, aux['regularizer'] = R [B], and the kind's gradients plus the term's.
  The gradient is linear in the loss, so the term's is taken by a second autograd pass over pass 0 alone."""
  loss, aux, g = kind_result
  p = {k: v.clone().requires_grad_(True) for k, v in O.online.items()}
  q = pass0_q(O, p, batch, taus=taus, noise=noise, device_fractions=device_fractions, tap=tap)
  t, R = term(q, batch['a_tm1'], alpha, weights)
  t.backward()
  total = {k: g[k] + (p[k].grad if p[k].grad is not None else torch.zeros_like(p[k])) for k in g}
  return loss + t.detach(), dict(aux, regularizer=R.detach()), total
