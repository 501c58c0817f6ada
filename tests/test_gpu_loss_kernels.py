"""GPU: every agent's loss kernel and the acting tail, example by example, against float64 head-level oracles.

`dz_test_loss` runs the learner's own loss section (launch_loss: the kind's loss kernel, then loss_mean_kernel) on head
outputs given here, and `dz_test_q_values` the acting tail (q_values_kernel, act_select_kernel).  No network runs, so
the inputs can be put exactly on the boundaries where a kernel makes a discrete choice: argmax ties between actions
whose targets differ, target atoms on support points and beyond +-vmax, quantile differences of exactly 0 and +-kappa,
clip_gradient's cotangent at, inside and outside the bound, priorities above rainbow's clamp of 100, and explore
uniforms on epsilon and next to 1.  The references are oracle/learner_oracle.py's `head_loss` (and the Munchausen
oracles' `head_loss`) in float64 on the same fp32 inputs.

Discrete outcomes are compared exactly: the zero gradient of every action but a_tm1, the clipped cotangent (exactly
+-bound where the float64 value is clear of it), a priority clamped to 100, the running max priority and the acting
action.  Continuous outputs get a float32 budget per element, with u = 2^-24 and every input an fp32 value:
  dqn family  td = fma(d, q_t, r) - q_tm1: e_td = 3u (|r| + |d q_t| + |q_tm1|); g = clip(w td / B): |w| e_td / B + 2u |g|;
              the loss term w 0.5 td^2: |w td| e_td + 4u |term|.
  categorical p = softmax(l): relative 2 ulp of expf, the K-term denominator and u |l - max| from the subtraction:
              rel(p_k) = u (|l_k - max| + K + 6) + 2 eL, eL the dueling combine's error (rainbow: (A + 1) u mean_a |adv|
              + 2u (|val| + |adv| + |mean|)); the projection weight of target atom j on support atom i moves by
              (e_zp + 2u (|zp| + |z_i|)) / gap + 2u, e_zp = 2u (|r| + |d z_j|), and proj_i = sum_j w_ij p_j adds
              (K + 1) u; log p_tm1 has absolute error u (|l - max| + |log den| + K + 6) + 2 eL + u |log p|; the loss
              sum_k proj_k log p_k and the gradient cot (p psum - proj) follow term by term.
  quantile    delta_ij = t_j - s_i with e_t = 2u (|r| + |d z|) (munchausen_iqn: the target budget of
              tests/test_oracle_munchausen_iqn.py); a Huber term moves by min(|delta|, kappa) e_delta (kappa = 0: e_delta)
              and its slope by e_delta inside the kink; where |delta| <= e_delta the sign, and with it the weight
              |tau - 1[delta < 0]| and at kappa = 0 the slope, is undetermined in float32, which adds the term's whole
              loss and 2 of slope; sums of n terms add (n + 2) u of their absolute sums.
  munchausen  the target / td budget of tests/test_oracle_munchausen.py (the kernel runs the same arithmetic as the
              host twin checked there), then the dqn family's clip and loss.
  scalar loss loss_mean_kernel's serial fp32 sum over B: sum_b (|w_b| e_b + u |term_b|) / B + (B + 1) u sum_b |term_b| / B.
Every budget carries 1e-12 of its operands for the oracle's own float64 rounding.  `-s` prints error / budget per case.
"""

import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo
from oracle import munchausen_iqn_oracle as miqn
from oracle import munchausen_oracle as mo

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'learner_hand_vectors.json')
Q_KINDS = ('dqn', 'double_q', 'prioritized')
HYPER = mo.Hyper()   # alpha 0.9, tau 0.03, l0 -1 (the same in both Munchausen oracles)


def f32(x):
  return np.asarray(x, dtype=np.float32)


class Case:
  """One call of the loss section: kind, sizes, hyperparameters and fp32 inputs.  heads[p] is pass p's head output
  (rainbow: (adv, val)); heads[1] is None where the kind has no selector pass of its own."""

  def __init__(self, kind, heads, a, r, d, w=None, taus=None, A=None, K=51, N=None, tau_counts=(1, 1, 1), vmax=10.0,
               bound=1.0 / 32, kappa=1.0, max_seen=1.0, name=''):
    self.kind, self.heads, self.name = kind, heads, name
    self.a, self.r, self.d = np.asarray(a, np.int32), f32(r), f32(d)
    self.w = None if w is None else f32(w)
    self.taus = None if taus is None else f32(taus)
    self.B = len(self.a)
    self.A, self.K, self.N, self.tau_counts = A, K, N, tau_counts
    self.vmax, self.bound, self.kappa, self.max_seen = vmax, bound, kappa, max_seen

  def config(self):
    from dqn_zoo_b200 import _lib
    c = _lib.LearnerConfig(vmax=self.vmax, grad_error_bound=self.bound, huber_param=self.kappa)
    c.kind = _lib.AGENT_KINDS[self.kind]
    c.num_actions, c.num_atoms, c.num_quantiles, c.latent_dim = self.A, self.K, self.N or 1, 64
    c.tau_samples_s_tm1, c.tau_samples_policy, c.tau_samples_s_t = self.tau_counts
    c.batch, c.obs_h, c.obs_w, c.obs_c = self.B, 84, 84, 4
    c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = HYPER
    return c


def dev(x):
  return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def run_device(case):
  """The device's outputs of dz_test_loss, every output buffer pre-filled with NaN so that an unwritten element fails."""
  from dqn_zoo_b200 import _lib
  rb = case.kind == 'rainbow'
  passes = [case.heads[p] if case.heads[p] is not None else case.heads[2] for p in range(3)]
  outs = [dev(f32(h[0] if rb else h)) for h in passes]
  vals = [dev(f32(h[1])) for h in passes] if rb else None
  B = case.B
  nan = lambda shape: torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')
  o = dict(dout=nan(outs[0].shape), dval=nan(vals[0].shape) if rb else None, per_example=nan((B,)), priorities=nan((B,)),
           loss_terms=nan((B,)), loss=nan((1,)), max_seen=torch.full((1,), case.max_seen, dtype=torch.float32, device='cuda'))
  keep = dict(a=dev(case.a), r=dev(case.r), d=dev(case.d), w=None if case.w is None else dev(case.w),
              taus=None if case.taus is None else dev(case.taus))
  ptr = lambda t: None if t is None else t.data_ptr()
  _lib.call('dz_test_loss', C.byref(case.config()), B, (C.c_void_p * 3)(*[t.data_ptr() for t in outs]),
            (C.c_void_p * 3)(*[t.data_ptr() for t in vals]) if rb else None, ptr(keep['a']), ptr(keep['r']),
            ptr(keep['d']), ptr(keep['w']), ptr(keep['taus']), ptr(o['dout']), ptr(o['dval']), ptr(o['per_example']),
            ptr(o['priorities']), ptr(o['loss_terms']), ptr(o['loss']), ptr(o['max_seen']) if rb else None,
            torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return {k: None if v is None else v.cpu().numpy().astype(np.float64) for k, v in o.items()}


def t64(x):
  return torch.tensor(np.asarray(x, dtype=np.float64))


def run_oracle(case):
  rb = case.kind == 'rainbow'
  heads = [None if h is None else ((t64(h[0]), t64(h[1])) if rb else t64(h)) for h in case.heads]
  w = None if case.w is None else t64(case.w)
  if case.kind == 'munchausen':
    _, aux = mo.head_loss(heads, case.a, case.r, case.d, w, grad_error_bound=case.bound, hyper=HYPER)
  elif case.kind == 'munchausen_iqn':
    _, aux = miqn.head_loss(heads, case.a, case.r, case.d, t64(case.taus), w, huber_param=case.kappa, hyper=HYPER)
  else:
    _, aux = lo.head_loss(case.kind, heads, case.a, case.r, case.d, w, None if case.taus is None else t64(case.taus),
                          vmax=case.vmax, grad_error_bound=case.bound, huber_param=case.kappa)
  return aux


# ---- budgets ----------------------------------------------------------------------------------------------------------

def _softmax_rel(l, eL):
  """Relative error of each fp32 softmax probability of logits l [..., K] (module docstring)."""
  K = l.shape[-1]
  return U * (np.abs(l - l.max(-1, keepdims=True)) + K + 6) + 2 * eL


def _dueling_err(adv, val):
  """Absolute error bound of rainbow's fp32 logits val + adv - mean_a adv, per example: [B, 1, 1]."""
  A = adv.shape[1]
  m = adv.mean(axis=1, keepdims=True)
  e = (A + 1) * U * np.abs(adv).mean(axis=1, keepdims=True) + 2 * U * (np.abs(val)[:, None, :] + np.abs(adv) + np.abs(m))
  return e.max(axis=(1, 2), keepdims=True)


def budget_q(case, aux):
  B, w = case.B, (np.ones(case.B) if case.w is None else case.w.astype(np.float64))
  td = aux['td_errors'].numpy()
  q_tm1 = aux['q_tm1'].numpy()[np.arange(B), case.a]
  boot = td + q_tm1 - case.r
  e_td = 3 * U * (np.abs(case.r) + np.abs(boot) + np.abs(q_tm1))
  g = w * td / B
  e_g = np.abs(w) * e_td / B + 2 * U * np.abs(g)
  term = w * 0.5 * td * td
  return dict(td=e_td, g=e_g, term=np.abs(w * td) * e_td + 4 * U * np.abs(term), per_example=e_td, priorities=e_td)


def budget_munchausen(case, aux):
  import test_oracle_munchausen as tm
  B, w = case.B, (np.ones(case.B) if case.w is None else case.w.astype(np.float64))
  h = [x.astype(np.float64) for x in case.heads]
  tgt, bonus, td = aux['targets'].numpy(), aux['bonus'].numpy(), aux['td_errors'].numpy()
  e_td = np.array([tm._budget(h[0][b], h[1][b], h[2][b], case.a[b], case.r[b], case.d[b], *HYPER, tgt[b], bonus[b])[2]
                   for b in range(B)])
  g = w * td / B
  loss = 0.5 * td * td
  e_loss = np.abs(td) * e_td + 2 * U * loss
  return dict(g=np.abs(w) * e_td / B + 2 * U * np.abs(g), per_example=e_loss,
              term=np.abs(w) * e_loss + U * np.abs(w * loss))


def budget_categorical(case, aux):
  rb = case.kind == 'rainbow'
  B, A = case.B, case.A
  rows = np.arange(B)
  w = np.ones(B) if case.w is None else case.w.astype(np.float64)
  logits = aux['logits_tm1'].numpy()                     # [B, A, K] float64 (rainbow: after the dueling combine)
  K = logits.shape[-1]
  z = np.linspace(-case.vmax, case.vmax, K).astype(np.float32).astype(np.float64)
  gap = z[1] - z[0]
  a_star = aux['a_star'].numpy()
  if rb:
    eL0 = _dueling_err(case.heads[0][0].astype(np.float64), case.heads[0][1].astype(np.float64))[:, 0, 0]
    eLt = _dueling_err(case.heads[2][0].astype(np.float64), case.heads[2][1].astype(np.float64))[:, 0, 0]
    tl = lo.dueling(t64(case.heads[2][0]), t64(case.heads[2][1])).numpy()[rows, a_star]
  else:
    eL0 = eLt = np.zeros(B)
    tl = case.heads[2].astype(np.float64)[rows, a_star]
  p_t = aux['p_target'].numpy()
  e_pt = p_t * _softmax_rel(tl, eLt[:, None])
  zp = np.clip(case.r[:, None].astype(np.float64) + case.d[:, None] * z[None, :], z[0], z[-1])          # [B, K]
  e_zp = 2 * U * (np.abs(case.r)[:, None] + np.abs(case.d[:, None] * z[None, :]))
  dist = np.abs(zp[:, None, :] - z[None, :, None])                                                     # [B, i, j]
  wij = np.clip(1.0 - dist / gap, 0.0, 1.0)
  near = dist < gap * (1 + 1e-6) + e_zp[:, None, :]
  e_w = near * ((e_zp[:, None, :] + 2 * U * (np.abs(zp)[:, None, :] + np.abs(z)[None, :, None])) / gap + 2 * U)
  proj = aux['target_probs'].numpy()
  e_proj = (p_t[:, None, :] * e_w + wij * (e_pt[:, None, :] + (K + 1) * U * p_t[:, None, :])).sum(-1)   # [B, K]
  l0 = logits[rows, case.a]
  m0 = l0.max(-1, keepdims=True)
  lden = np.log(np.exp(l0 - m0).sum(-1, keepdims=True))
  lp = l0 - m0 - lden
  e_lp = U * (np.abs(l0 - m0) + np.abs(lden) + K + 6) + 2 * eL0[:, None] + U * np.abs(lp)
  loss = aux['losses'].numpy()
  e_loss = (e_proj * np.abs(lp) + proj * e_lp).sum(-1) + (K + 2) * U * np.abs(proj * lp).sum(-1)
  p0 = np.exp(lp)
  e_p0 = p0 * _softmax_rel(l0, eL0[:, None])
  psum = proj.sum(-1, keepdims=True)
  e_psum = e_proj.sum(-1, keepdims=True) + K * U * psum
  cot = (w / B)[:, None]
  dl = cot * (p0 * psum - proj)
  e_dl = cot * (e_p0 * psum + p0 * e_psum + e_proj + 3 * U * (p0 * psum + proj)) + U * np.abs(dl)
  out = dict(per_example=e_loss, priorities=e_loss, term=np.abs(w) * e_loss + U * np.abs(w * loss), dl=e_dl, dl_value=dl)
  return out


def budget_quantile(case, aux, e_tgt=None):
  B = case.B
  rows = np.arange(B)
  w = np.ones(B) if case.w is None else case.w.astype(np.float64)
  src = aux['dist_tm1'].numpy()[rows, :, case.a]                  # [B, N]
  tgt = aux['targets'].numpy()                                     # [B, Nt]
  N, Nt = src.shape[1], tgt.shape[1]
  if case.kind == 'qrdqn':
    tau = np.broadcast_to(((np.arange(N, dtype=np.float32) + np.float32(0.5)) / np.float32(N)).astype(np.float64), (B, N))
  else:
    tau = case.taus.astype(np.float64)
  if e_tgt is None:
    boot = (tgt - case.r[:, None]) / 1.0
    e_tgt = 2 * U * (np.abs(case.r)[:, None] + np.abs(boot))
  k = case.kappa
  delta = tgt[:, None, :] - src[:, :, None]                        # [B, N, Nt]
  ad = np.abs(delta)
  e_d = e_tgt[:, None, :] + U * (np.abs(tgt)[:, None, :] + np.abs(src)[:, :, None])
  amb = ad <= e_d
  wt = np.abs(tau[:, :, None] - (delta < 0))
  if k > 0:
    q = np.minimum(ad, k)
    l = 0.5 * q * q + k * (ad - q)
    dlv = np.clip(delta, -k, k)
    e_l = q * e_d + 3 * U * l + amb * l
    e_dl = (ad < k + e_d) * e_d + amb * (ad + e_d)
  else:
    l, dlv = ad, np.sign(delta)
    e_l = e_d + 3 * U * l + amb * l
    e_dl = amb * 2.0
  acc = (wt * l).sum(-1)
  e_acc = (wt * e_l).sum(-1) + (Nt + 2) * U * acc
  loss = aux['losses'].numpy()
  e_loss = e_acc.sum(-1) / Nt + (N + 10) * U * loss
  cot = w / B
  gacc = (wt * dlv).sum(-1)
  g = -cot[:, None] * gacc / Nt
  e_g = cot[:, None] * ((wt * e_dl).sum(-1) + (Nt + 3) * U * (wt * np.abs(dlv)).sum(-1)) / Nt + 2 * U * np.abs(g)
  return dict(per_example=e_loss, term=np.abs(w) * e_loss + U * np.abs(w * loss), g=e_g, g_value=g)


def budget_munchausen_iqn(case, aux):
  import test_oracle_munchausen_iqn as tmi
  h = [x.astype(np.float64) for x in case.heads]
  y, bonus, ent = aux['targets'].numpy(), aux['bonus'].numpy(), aux['entropy'].numpy()
  e_y = np.stack([tmi._budget(h[1][b], h[2][b], case.a[b], case.r[b], case.d[b], *HYPER, y[b], bonus[b], ent[b])[0]
                  for b in range(case.B)])
  return budget_quantile(case, aux, e_tgt=e_y)


# ---- the comparison ---------------------------------------------------------------------------------------------------

def within(name, got, want, budget, slack_of):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  budget = np.asarray(budget, np.float64) + 1e-12 * np.asarray(slack_of, np.float64) + 1e-30
  assert np.isfinite(got).all(), (name, 'unwritten or non-finite element')
  err = np.abs(got - want)
  ratio = float((err / budget).max()) if err.size else 0.0
  assert ratio <= 1.0, (name, ratio, np.unravel_index(int(np.argmax(err / budget)), err.shape), got.reshape(-1)[:8],
                        want.reshape(-1)[:8])
  return ratio


def check(case):
  """Runs the case on the device and compares every output with the oracle; returns {output: error / budget}."""
  got, aux = run_device(case), run_oracle(case)
  kind, B = case.kind, case.B
  rows = np.arange(B)
  w = np.ones(B) if case.w is None else case.w.astype(np.float64)
  ratios = {}
  dout = got['dout']
  if kind in Q_KINDS or kind == 'munchausen':
    bud = budget_q(case, aux) if kind in Q_KINDS else budget_munchausen(case, aux)
    td = aux['td_errors'].numpy()
    gv = w * td / B
    want_g = np.clip(gv, -case.bound, case.bound)
    # the gradient is -g at a_tm1 and exactly 0 elsewhere
    mask = np.zeros_like(dout, dtype=bool)
    mask[rows, case.a] = True
    assert (dout[~mask] == 0).all(), 'non-zero gradient off a_tm1'
    ratios['dout'] = within('dout', -dout[mask], want_g, bud['g'], np.abs(gv))
    clear = np.abs(gv) > case.bound + bud['g']
    assert (np.abs(dout[mask][clear]) == np.float32(case.bound)).all(), 'a clipped cotangent is not exactly the bound'
    if kind in Q_KINDS:
      ratios['per_example'] = within('td', got['per_example'], td, bud['td'], np.abs(td) + np.abs(case.r))
    else:
      ratios['per_example'] = within('loss', got['per_example'], aux['losses'].numpy(), bud['per_example'], td * td)
    pe_budget = bud['term']
  elif kind in ('c51', 'rainbow'):
    bud = budget_categorical(case, aux)
    loss = aux['losses'].numpy()
    if kind == 'rainbow':
      dval = got['dval']
      ratios['dval'] = within('dval', dval, bud['dl_value'], bud['dl'], np.abs(bud['dl_value']) + 1)
      onehot = (np.arange(case.A)[None, :] == case.a[:, None]).astype(np.float64)
      want_dadv = bud['dl_value'][:, None, :] * (onehot[:, :, None] - 1.0 / case.A)
      e_dadv = bud['dl'][:, None, :] * np.abs(onehot[:, :, None] - 1.0 / case.A) + 2 * U * np.abs(want_dadv)
      ratios['dadv'] = within('dadv', dout, want_dadv, e_dadv, np.abs(want_dadv) + 1)
      g_ref = aux['grad']
      np.testing.assert_allclose(g_ref[1].numpy(), bud['dl_value'], rtol=1e-9, atol=1e-14)   # the budget's own dl
      pri = got['priorities']
      clamped = loss > 100 + bud['priorities']
      assert (pri[clamped] == 100.0).all(), 'a priority above 100 is not clamped to exactly 100'
      ratios['priorities'] = within('priorities', pri[~clamped], np.minimum(np.abs(loss), 100)[~clamped],
                                    bud['priorities'][~clamped], np.abs(loss)[~clamped])
      assert got['max_seen'][0] == max(np.float32(case.max_seen), pri.astype(np.float32).max()), 'running max priority'
    else:
      mask = np.zeros(dout.shape, dtype=bool)
      mask[rows, case.a] = True
      assert (dout[~mask] == 0).all(), 'non-zero gradient off a_tm1'
      ratios['dout'] = within('dout', dout[rows, case.a], bud['dl_value'], bud['dl'], np.abs(bud['dl_value']) + 1)
      np.testing.assert_allclose(aux['grad'].numpy()[rows, case.a], bud['dl_value'], rtol=1e-9, atol=1e-14)
    ratios['per_example'] = within('loss', got['per_example'], loss, bud['per_example'], np.abs(loss) + 1)
    pe_budget = bud['term']
  else:
    bud = budget_quantile(case, aux) if kind != 'munchausen_iqn' else budget_munchausen_iqn(case, aux)
    loss = aux['losses'].numpy()
    mask = np.zeros(dout.shape, dtype=bool)
    mask[rows, :, case.a] = True
    assert (dout[~mask] == 0).all(), 'non-zero gradient off a_tm1'
    np.testing.assert_allclose(aux['grad'].numpy()[rows, :, case.a], bud['g_value'], rtol=1e-9, atol=1e-14)
    ratios['dout'] = within('dout', dout[rows, :, case.a], bud['g_value'], bud['g'], np.abs(bud['g_value']) + 1)
    ratios['per_example'] = within('loss', got['per_example'], loss, bud['per_example'], np.abs(loss) + 1)
    pe_budget = bud['term']
  if kind == 'prioritized':
    ratios['priorities'] = within('priorities', got['priorities'], np.abs(aux['td_errors'].numpy()), bud['priorities'],
                                  np.abs(aux['td_errors'].numpy()))
  terms = w * aux['losses'].numpy()
  ratios['loss_terms'] = within('loss_terms', got['loss_terms'], terms, pe_budget, np.abs(terms) + 1)
  e_mean = (pe_budget.sum() + (B + 1) * U * np.abs(terms).sum()) / B
  ratios['loss'] = within('loss', got['loss'][0], terms.mean(), e_mean, np.abs(terms).mean() + 1)
  print('%-15s %-40s %s' % (kind, case.name, ' '.join('%s %.3f' % kv for kv in sorted(ratios.items()))))
  return ratios, got, aux


# ---- inputs -----------------------------------------------------------------------------------------------------------

def random_case(kind, B, A, rs, K=21, N=16, tau_counts=(8, 5, 7), vmax=10.0, bound=1.0 / 32, kappa=1.0, scale=1.0,
                name='random'):
  r = rs.choice([-1.0, 0.0, 1.0, 0.37], size=B)
  d = rs.choice([0.0, 0.99, 0.99 ** 3, 1.0], size=B)
  a = rs.randint(0, A, B)
  w = rs.uniform(0.1, 1.0, B) if kind in ('prioritized', 'rainbow') else None
  g = lambda *shape: f32(rs.standard_normal(shape) * scale)
  taus = None
  if kind in Q_KINDS or kind == 'munchausen':
    heads = [g(B, A), g(B, A) if kind != 'dqn' else None, g(B, A)]
  elif kind == 'c51':
    heads = [g(B, A, K), None, g(B, A, K)]
  elif kind == 'rainbow':
    heads = [(g(B, A, K), g(B, K)) for _ in range(3)]
  elif kind == 'qrdqn':
    heads = [g(B, N, A), None, g(B, N, A)]
  else:
    n0, n1, n2 = tau_counts
    heads = [g(B, n0, A), g(B, n1, A), g(B, n2, A)]
    taus = f32(rs.uniform(size=(B, n0)))
  return Case(kind, heads, a, r, d, w, taus, A=A, K=K, N=N, tau_counts=tau_counts, vmax=vmax, bound=bound,
              kappa=kappa, name=name)


ALL_KINDS = lo.AGENT_KINDS + mo.EXTRA_KINDS + miqn.EXTRA_KINDS
SHAPES = [(1, 1), (5, 18), (32, 64), (1024, 6)]


@pytest.mark.parametrize('kind', ALL_KINDS)
def test_random_heads_at_every_batch_and_action_count(kind):
  """Generic fp32 heads at B in {1, 5, 32, 1024} and A in {1, 18, 64} (the Munchausen kinds at most 18); B = 1024 puts
  the scalar loss through loss_mean_kernel's 1024-term serial sum."""
  rs = np.random.RandomState(11)
  for B, A in SHAPES:
    if kind.startswith('munchausen'):
      A = min(A, 18)
    big = B == 1024 and kind in ('qrdqn', 'iqn', 'munchausen_iqn')
    check(random_case(kind, B, A, rs, N=4 if big else 16, tau_counts=(3, 2, 4) if big else (8, 5, 7),
                      name='B=%d A=%d' % (B, A)))


# -- argmax ties: the selector ties exactly (in fp32 and float64) between actions whose targets differ; the first wins

def test_double_q_and_prioritized_take_the_first_of_tied_selector_actions():
  for kind in ('double_q', 'prioritized'):
    sel = f32([[1.0, 3.0, 3.0, 0.0], [2.0, 2.0, 2.0, 2.0], [-1.0, -5.0, -1.0, -1.0]])
    tgt = f32([[0.0, 1.0, 5.0, 9.0], [4.0, -4.0, 8.0, 0.5], [-2.0, 7.0, 3.0, 0.25]])
    q_tm1 = f32([[0.1, 0.2, 0.3, 0.4]] * 3)
    case = Case(kind, [q_tm1, sel, tgt], [0, 1, 3], [0.5, 0.0, -1.0], [0.9, 1.0, 0.5],
                [1.0, 0.5, 0.25] if kind == 'prioritized' else None, A=4, bound=1e6, name='tied selector')
    _, got, aux = check(case)
    assert aux['a_star'].tolist() == [1, 0, 0]
    want_td = f32([0.5 + 0.9 * 1.0 - 0.1, 4.0 - 0.2, -1.0 + 0.5 * -2.0 - 0.4])
    np.testing.assert_allclose(got['per_example'], want_td, rtol=1e-6)


def test_categorical_kinds_take_the_first_of_tied_expectations():
  """c51: two target rows with expectation exactly 0 (all mass on the centre atom, half on each of +-z; the other logits
  at -1e4, so exp underflows to exactly 0 in both precisions) and different distributions.  rainbow: identical
  online(s_t) rows (a tied selector) over different target(s_t) rows."""
  K, A = 3, 3
  centre = [-1e4, 0.0, -1e4]
  split = [0.0, -1e4, 0.0]
  c51_t = f32([[split, centre, split], [centre, split, centre]])
  c51_0 = f32(np.random.RandomState(1).standard_normal((2, A, K)))
  _, _, aux = check(Case('c51', [c51_0, None, c51_t], [0, 2], [0.0, 0.5], [1.0, 1.0], A=A, K=K, vmax=1.0,
                         name='tied expectations'))
  assert aux['a_star'].tolist() == [0, 0]
  rs = np.random.RandomState(2)
  adv1 = f32(np.repeat(rs.standard_normal((2, 1, K)), A, axis=1))     # every action's selector logits equal
  val1 = f32(rs.standard_normal((2, K)))
  adv2 = f32(rs.standard_normal((2, A, K)) * 3)
  heads = [(f32(rs.standard_normal((2, A, K))), f32(rs.standard_normal((2, K)))), (adv1, val1), (adv2, f32(rs.standard_normal((2, K))))]
  _, _, aux = check(Case('rainbow', heads, [1, 2], [0.0, 0.3], [0.99, 0.5], w=[1.0, 0.5], A=A, K=K, vmax=1.0,
                         name='tied online(s_t)'))
  assert aux['a_star'].tolist() == [0, 0]


def test_quantile_kinds_take_the_first_of_tied_means():
  """Quantile sets {-1, 1} and {0, 0}: equal means, different targets (qrdqn: the target pass selects; iqn: the
  selector pass, here with the same two sets)."""
  tied = f32([[[-1.0, 0.0, 5.0], [1.0, 0.0, -5.0]]])      # [B=1][N=2][A=3]: means 0, 0, 0
  src = f32([[[0.25, 0.5, 0.75], [0.5, 1.0, 1.5]]])
  for kappa in (0.0, 1.0):
    _, _, aux = check(Case('qrdqn', [src, None, tied], [1], [0.0], [1.0], A=3, N=2, kappa=kappa, name='tied means'))
    assert aux['a_star'].tolist() == [0]
    _, _, aux = check(Case('iqn', [src, tied, tied[:, :, ::-1].copy()], [1], [0.0], [1.0], taus=[[0.2, 0.7]], A=3,
                           tau_counts=(2, 2, 2), kappa=kappa, name='tied means'))
    assert aux['a_star'].tolist() == [0]


def test_munchausen_kinds_with_tied_target_values():
  """qbar ties enter a softmax, not an argmax: a tie is an ordinary input, including a row of A equal values."""
  q = f32([[0.5, 0.5, 0.5, 0.5], [1.0, 2.0, 2.0, -3.0]])
  check(Case('munchausen', [f32([[0.1, 0.2, 0.3, 0.4]] * 2), q, q[:, ::-1].copy()], [1, 2], [0.0, 1.0], [0.99, 0.0], A=4,
             bound=1e6, name='tied qbar'))
  z = np.repeat(q[:, None, :], 3, axis=1)
  check(Case('munchausen_iqn', [f32(np.ones((2, 2, 4))), z, z.copy()], [0, 3], [0.0, 1.0], [0.99, 0.5],
             taus=[[0.25, 0.75]] * 2, A=4, tau_counts=(2, 3, 3), name='tied qbar'))


# -- the categorical projection

@pytest.mark.parametrize('vmax', [1.0, 3.0, 10.0, 100.0])
@pytest.mark.parametrize('K', [2, 3, 51, 128])
def test_projection_on_support_points_beyond_the_edges_and_terminal(vmax, K):
  """r + d z_j exactly on support points (r = 0 with d in {0, 1}, r a multiple of the atom gap with d = 1), targets
  beyond +-vmax that clip onto an edge atom, terminal d = 0, and logits of magnitude 50-80."""
  rs = np.random.RandomState(K)
  gap = float(np.float32(2 * vmax / (K - 1)))
  r = [0.0, 0.0, gap, -2 * gap, 3 * vmax, -5 * vmax, 0.37 * vmax, gap, 0.0]
  d = [1.0, 0.0, 1.0, 1.0, 1.0, 0.5, 0.0, 0.0, 1.0]
  B, A = len(r), 3
  logits = lambda: f32(rs.uniform(50, 80, (B, A, K)) * rs.choice([-1.0, 1.0], (B, A, K)))
  a = rs.randint(0, A, B)
  check(Case('c51', [logits(), None, logits()], a, r, d, A=A, K=K, vmax=vmax, name='vmax=%g K=%d' % (vmax, K)))
  heads = [(logits(), f32(rs.uniform(-60, 60, (B, K)))) for _ in range(3)]
  check(Case('rainbow', heads, a, r, d, w=rs.uniform(0.1, 1, B), A=A, K=K, vmax=vmax, max_seen=5.0,
             name='vmax=%g K=%d' % (vmax, K)))


def test_rainbow_priorities_clamp_at_100_and_update_the_running_max():
  """Losses far above 100 (the taken action's logits put ~-300 of log probability on the projected mass) must give a
  priority of exactly 100, the others their loss, and max_seen the largest of its old value and the priorities."""
  rs = np.random.RandomState(4)
  B, A, K = 6, 2, 51
  adv0 = f32(rs.uniform(-1, 1, (B, A, K)))
  adv0[:3, 0, 25:] = 150.0        # the taken action's mass at the top atoms (logits +-75 after the dueling mean),
  adv0[:3, 0, :25] = -150.0       # far from targets in [-10, 0]
  heads = [(adv0, f32(np.zeros((B, K)))), (f32(rs.standard_normal((B, A, K))), f32(rs.standard_normal((B, K)))),
           (f32(rs.standard_normal((B, A, K))), f32(rs.standard_normal((B, K))))]
  for max_seen in (1.0, 1e3):
    _, got, aux = check(Case('rainbow', heads, [0] * B, [-5.0] * B, [0.5] * B, w=[1.0] * B, A=A, K=K,
                             max_seen=max_seen, name='loss > 100, max_seen=%g' % max_seen))
    assert (aux['losses'].numpy()[:3] > 100).all() and (aux['losses'].numpy()[3:] < 100).all()
    assert (got['priorities'][:3] == 100.0).all()


def test_categorical_at_64_actions_and_128_atoms():
  """The largest configuration validate() accepts: 103,696 bytes of shared memory, over the default 48 KB."""
  rs = np.random.RandomState(5)
  for kind in ('c51', 'rainbow'):
    check(random_case(kind, 32, 64, rs, K=128, scale=3.0, name='A=64 K=128'))


# -- the quantile regression loss

@pytest.mark.parametrize('kappa', [0.0, 0.5, 1.0, 3.0])
def test_quantile_differences_of_exactly_zero_and_kappa(kappa):
  """Targets r + d z with d in {0, 1} and small integers or halves, so that delta = target - source is exact in fp32:
  delta = 0, +-kappa and values on both sides; taus at 0 and at the largest float below 1."""
  k = max(kappa, 1.0)
  src = np.array([0.0, k, -k, 0.5 * k, 2.0 * k, -3.0 * k])                        # N = 6 source quantiles
  tgt = np.array([0.0, 0.0, k, -k, 0.5 * k, 3.0 * k, -2.0 * k])                   # Nt = 7: delta hits 0 and +-k
  A, B = 2, 3
  dist0 = np.zeros((B, 6, A)); dist0[:, :, 1] = src; dist0[:, :, 0] = src[::-1]
  dist_t = np.zeros((B, 7, A)); dist_t[:, :, 0] = tgt; dist_t[:, :, 1] = tgt - 10.0   # action 0 is the greedy one
  below_one = float(np.nextafter(np.float32(1), np.float32(0)))
  taus = np.array([[0.0, below_one, 0.5, 0.25, 0.75, 0.125]] * B)
  for a in (0, 1):
    check(Case('iqn', [f32(dist0), f32(dist_t[:, :1]), f32(dist_t)], [a] * B, [0.0, 0.0, 0.0], [1.0, 1.0, 0.0], taus=taus,
               A=A, tau_counts=(6, 1, 7), kappa=kappa, name='exact deltas a=%d' % a))
  q0 = np.zeros((B, 7, A)); q0[:, :, 1] = np.append(src, 0.0); q0[:, :, 0] = tgt
  check(Case('qrdqn', [f32(q0), None, f32(dist_t)], [1, 0, 1], [0.0, 0.0, k], [1.0, 0.0, 1.0], A=A, N=7, kappa=kappa,
             name='exact deltas'))
  z1 = f32(np.random.RandomState(6).standard_normal((B, 4, A)))
  check(Case('munchausen_iqn', [f32(dist0), z1, f32(dist_t)], [1] * B, [0.0] * B, [1.0, 0.5, 0.0], taus=taus, A=A,
             tau_counts=(6, 4, 7), kappa=kappa, name='exact deltas'))


@pytest.mark.parametrize('kappa', [0.0, 0.5, 1.0, 3.0])
def test_quantile_extreme_sample_counts(kappa):
  """qrdqn with N = 1 and N = 256, iqn with (N, N', N'') = (256, 1, 7) and (1, 256, 256)."""
  rs = np.random.RandomState(7)
  for N in (1, 256):
    check(random_case('qrdqn', 8, 5, rs, N=N, kappa=kappa, name='N=%d' % N))
  for counts in ((256, 1, 7), (1, 256, 256)):
    check(random_case('iqn', 8, 5, rs, tau_counts=counts, kappa=kappa, name='taus=%s' % (counts,)))
    check(random_case('munchausen_iqn', 4, 5, rs, tau_counts=counts, kappa=kappa, name='taus=%s' % (counts,)))


# -- clip_gradient

@pytest.mark.parametrize('bound', [1.0 / 1024, 1.0 / 32, 1.0, 1e6])
def test_clip_gradient_inside_on_and_outside_the_bound(bound):
  """w td / B lands just inside, exactly on and just outside +-bound, and w = 0.  B = 4 and w, td powers of two make
  w td / B exact in fp32; 'just inside / outside' is one part in 2^10 away."""
  B, A = 4, 3
  for kind in ('dqn', 'prioritized', 'munchausen'):
    if kind == 'munchausen':     # the munchausen target is not exact: the clip side is checked where it is clear
      td = np.array([bound * B * 2.0, -bound * B * 0.5, bound * B * 4.0, 1.0])
    else:
      td = np.array([bound * B * (1 - 2.0 ** -10), -bound * B, bound * B * (1 + 2.0 ** -10), -bound * B * 2.0])
    q_tm1 = np.zeros((B, A)); q_t = np.zeros((B, A))
    r = f32(td)
    w = [1.0, 1.0, 1.0, 0.0] if kind == 'prioritized' else None
    heads = [f32(q_tm1), f32(q_t) if kind != 'dqn' else None, f32(q_t)]
    _, got, aux = check(Case(kind, heads, [0, 1, 2, 0], r, [0.0] * B, w, A=A, bound=bound, name='bound=%g' % bound))
    if kind != 'munchausen':
      g = -got['dout'][np.arange(B), [0, 1, 2, 0]]
      want = np.float32([bound * (1 - 2.0 ** -10), -bound, bound, -bound if w is None else 0.0])
      np.testing.assert_array_equal(g.astype(np.float32), want)


# -- the hand-derived fixtures on the device

def test_hand_vectors_through_the_kernels():
  """tests/golden/learner_hand_vectors.json's loss entries through the device kernels: each against its hand-derived
  number as well as against the oracle."""
  with open(GOLDEN) as f:
    hand = json.load(f)
  # the 3-atom projection + cross entropy: vmax = 1, K = 3, target logits log(probs) on the greedy action
  for case in hand['categorical_l2_project']:
    lt = np.log(np.array([case['probs'], [1.0, 1.0, 1.0]]))   # action 1: uniform, expectation 0 < action 0's
    lt[1] -= 1.0
    assert sum(p * z for p, z in zip(case['probs'], case['z_q'])) > 0
    ce = hand['categorical_cross_entropy']
    logits0 = np.array([ce['logits_tm1'], [0.0, 0.0, 0.0]])
    _, got, aux = check(Case('c51', [f32(logits0[None]), None, f32(lt[None])], [0], [case['r_t']], [case['discount_t']],
                             A=2, K=3, vmax=1.0, name='hand projection'))
    np.testing.assert_allclose(aux['target_probs'].numpy()[0], case['expected'], atol=1e-7)
    want = -(np.array(case['expected']) * (np.array(ce['logits_tm1']) - np.log(np.exp(ce['logits_tm1']).sum()))).sum()
    assert abs(got['per_example'][0] - want) <= 1e-6 * abs(want), (got['per_example'][0], want)
    if case['expected'] == ce['target']:
      assert abs(got['per_example'][0] - ce['expected']) <= 1e-6 * ce['expected']
  # quantile Huber at kappa = 1 and kappa = 0: qrdqn with N = 2 has taus (0.25, 0.75), the fixtures' taus
  for case in hand['quantile_regression_loss']:
    assert case['tau'] == [0.25, 0.75]
    src = np.zeros((1, 2, 2)); src[0, :, 0] = case['dist_src']; src[0, :, 1] = -7.0
    tgt = np.zeros((1, 2, 2)); tgt[0, :, 0] = case['target']; tgt[0, :, 1] = -9.0
    _, got, _ = check(Case('qrdqn', [f32(src), None, f32(tgt)], [0], [0.0], [1.0], A=2, N=2, kappa=case['kappa'],
                           name='hand kappa=%g' % case['kappa']))
    assert abs(got['per_example'][0] - case['expected']) <= 4 * U * case['expected'], case['derivation']
  # double Q: the selector picks action 1, the bootstrap 20
  case = hand['double_q_learning']
  heads = [f32([case['q_tm1']]), f32([case['q_t_selector']]), f32([case['q_t_value']])]
  _, got, _ = check(Case('double_q', heads, [case['a_tm1']], [case['r_t']], [case['discount_t']], A=3, bound=1e6,
                         name='hand double_q'))
  assert abs(got['per_example'][0] - case['expected_td']) <= 4 * U * case['expected_td']
  assert abs(got['loss'][0] - case['expected_l2']) <= 8 * U * case['expected_l2']


# ---- acting: q_values_kernel and act_select_kernel --------------------------------------------------------------------

def q_values_device(kind, out, val, A, K=51, nq=1, vmax=10.0, explore=None, eps=0.0):
  from dqn_zoo_b200 import _lib
  E = out.shape[0]
  c = Case(kind, None, np.zeros(E), np.zeros(E), np.zeros(E), A=A, K=K, N=nq, tau_counts=(1, nq, 1), vmax=vmax).config()
  o, v = dev(f32(out)), None if val is None else dev(f32(val))
  ex = None if explore is None else dev(f32(explore))
  q = torch.full((E, A), float('nan'), device='cuda')
  act = torch.full((E,), -1, dtype=torch.int32, device='cuda')
  _lib.call('dz_test_q_values', C.byref(c), E, o.data_ptr(), None if v is None else v.data_ptr(),
            None if ex is None else ex.data_ptr(), float(eps), q.data_ptr(), act.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return q.cpu().numpy().astype(np.float64), act.cpu().numpy()


def greedy_first(q):
  return np.argmax(q, axis=1)      # first maximum, as jnp.argmax


def test_q_values_of_every_network_family():
  rs = np.random.RandomState(8)
  E, A = 7, 5
  for kind in ('dqn', 'c51', 'rainbow', 'qrdqn', 'iqn'):
    for vmax in (1.0, 10.0, 100.0):
      K, nq = 21, 9
      val = None
      if kind == 'dqn':
        out = rs.standard_normal((E, A)); want = f32(out).astype(np.float64); e = np.zeros_like(want)
      elif kind in ('c51', 'rainbow'):
        out = rs.standard_normal((E, A, K)) * 5
        z = np.linspace(-vmax, vmax, K).astype(np.float32).astype(np.float64)
        if kind == 'rainbow':
          val = rs.standard_normal((E, K))
          lg = lo.dueling(t64(f32(out)), t64(f32(val))).numpy()
          eL = _dueling_err(f32(out).astype(np.float64), f32(val).astype(np.float64))
        else:
          lg, eL = f32(out).astype(np.float64), np.zeros((E, 1, 1))
        p = np.exp(lg - lg.max(-1, keepdims=True)); p /= p.sum(-1, keepdims=True)
        want = (p * z).sum(-1)
        e = (p * _softmax_rel(lg, eL) * np.abs(z)).sum(-1) + (K + 4) * U * (p * np.abs(z)).sum(-1)
      else:
        out = rs.standard_normal((E, nq, A))
        want = f32(out).astype(np.float64).mean(1)
        e = (nq + 2) * U * np.abs(f32(out)).mean(1)
      q, act = q_values_device(kind, out, val, A, K=K, nq=nq, vmax=vmax)
      within('q %s' % kind, q, want, e, np.abs(want) + 1)
      np.testing.assert_array_equal(act, greedy_first(q))


def test_act_select_ties_epsilon_boundary_and_uniforms_next_to_one():
  """Greedy ties go to the first maximum; explore[e] == epsilon exactly is greedy (u0 < epsilon explores); an explore
  uniform u1 at the largest float below 1 gives action A - 1, and so does u1 = 1 exactly (outside [0, 1), as a caller's
  own uniforms might be), through the min(., A - 1) clamp."""
  below_one = float(np.nextafter(np.float32(1), np.float32(0)))
  for A in (1, 2, 3, 18, 64):
    q = np.zeros((8, A))
    q[:, A // 2:] = 1.0                                  # a tie over the upper half of the actions
    q[1] = -np.arange(A)                                 # a strict maximum at action 0
    u0 = np.array([0.5, 0.5, 0.25, 0.25, 0.0, 0.25, 0.9, 0.0])
    u1 = np.array([0.0, 0.3, below_one, 1.0, 0.5, 0.0, 0.99, below_one])
    eps = 0.25
    _, act = q_values_device('dqn', q, None, A, explore=np.stack([u0, u1]), eps=eps)
    greedy = greedy_first(f32(q).astype(np.float64))
    explore_a = np.minimum((f32(u1) * np.float32(A)).astype(np.float32).astype(np.int64), A - 1)
    want = np.where(f32(u0) < np.float32(eps), explore_a, greedy)
    np.testing.assert_array_equal(act, want)
    assert act[2] == greedy[2] and act[3] == greedy[3]          # u0 == epsilon: greedy
    assert act[4] == min(A - 1, A // 2) if A > 1 else act[4] == 0
    assert act[7] == A - 1                                       # u1 next to 1 explores the last action
    _, act1 = q_values_device('dqn', q, None, A, explore=np.stack([np.zeros(8), np.ones(8)]), eps=0.5)
    assert (act1 == A - 1).all()                                 # u1 = 1 is clamped to the last action
    _, g = q_values_device('dqn', q, None, A)
    np.testing.assert_array_equal(g, greedy)
